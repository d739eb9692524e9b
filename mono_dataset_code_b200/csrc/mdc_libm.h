// exp and log in double precision, restated so that host and device produce the SAME BITS as the host's glibc.
//
// plotE (main_responseCalib.cpp:72-119) maps every irradiance through log(E + 20) and exp(...) from libm before it truncates the
// result to a colour index; a device version of it is only a drop-in if its exp and log agree with the host's bit for bit.  CUDA's
// exp and log do not.  The pinned implementation is glibc 2.39 (Ubuntu 24.04, libm.so.6) sysdeps/ieee754/dbl-64/e_exp.c and
// e_log.c, the table-driven algorithms of Arm's optimized-routines (exp: 2^(k/128) from a 128-entry table times a degree-5
// polynomial of the reduced argument; log: 128 subintervals of [0x1.6p-1, 0x1.6p0) with 1/c and log(c) from a table and a
// degree-6 polynomial of log1p(r), and a degree-12 polynomial near 1).
//
// The variant matters.  On x86-64 glibc picks, by ifunc, a build of both functions compiled with -mfma -mavx2 when the CPU has
// FMA and AVX2 (x86-64 CPUs of the last decade have both).  In that build e_log.c takes its __FP_FAST_FMA branch (r = fma(z, invc, -1), no chi/clo
// table) and GCC contracted a * b + c into fused multiply-adds at the places marked FMA below; they were read off the
// disassembly of that variant in libm.so.6.  Every other operation is an explicitly rounded IEEE operation (intrinsics on the
// device, -ffp-contract=off on the host).  The tables are glibc's __exp_data.tab and __log_data.tab.
//
// Verified bit for bit against the host's libm (tests/test_libm_restated.py records the glibc version and
// the CPU features that select the variant, and skips where the non-FMA build would run):
// exp on [0, 1] (a dense sweep plus every table-boundary neighbourhood), log on [20, DBL_MAX] (stratified by exponent and
// mantissa), the near-1 and subnormal paths of log, exp's over- and underflow paths, +-0, +-inf and NaN.  NaN results are NaN
// (payloads are not pinned).  On the GPU the same test checks the device build against the host build and libm on the same sweeps.
#pragma once
#include <stdint.h>
#include <string.h>
#if !defined(__CUDA_ARCH__)
#include <math.h>
#endif

#if defined(__CUDA_ARCH__)
#define MDC_LM_ADD(a, b) __dadd_rn((a), (b))
#define MDC_LM_SUB(a, b) __dsub_rn((a), (b))
#define MDC_LM_MUL(a, b) __dmul_rn((a), (b))
#define MDC_LM_FMA(a, b, c) __fma_rn((a), (b), (c))
#define MDC_LM_BITS(x) static_cast<uint64_t>(__double_as_longlong(x))
#define MDC_LM_DBL(u) __longlong_as_double(static_cast<long long>(u))
#define MDC_LM_HD __host__ __device__ __forceinline__
#define MDC_LM_TAB(name) name##_d
#else
#define MDC_LM_ADD(a, b) ((a) + (b))
#define MDC_LM_SUB(a, b) ((a) - (b))
#define MDC_LM_MUL(a, b) ((a) * (b))
#define MDC_LM_FMA(a, b, c) fma((a), (b), (c))
static inline uint64_t mdc_lm_bits(double x) { uint64_t u; memcpy(&u, &x, 8); return u; }
static inline double mdc_lm_dbl(uint64_t u) { double x; memcpy(&x, &u, 8); return x; }
#define MDC_LM_BITS(x) mdc_lm_bits(x)
#define MDC_LM_DBL(u) mdc_lm_dbl(u)
#if defined(__CUDACC__)
#define MDC_LM_HD __host__ __device__ inline
#else
#define MDC_LM_HD static inline
#endif
#define MDC_LM_TAB(name) name##_h
#endif

// __exp_data.tab: for i = 0..127, {bits of the tail of 2^(i/128), bits of 2^(i/128) minus i << 45}
#define MDC_EXP_TAB_INIT { \
    0x0000000000000000ull, 0x3ff0000000000000ull, 0x3c9b3b4f1a88bf6eull, 0x3feff63da9fb3335ull, \
    0xbc7160139cd8dc5dull, 0x3fefec9a3e778061ull, 0xbc905e7a108766d1ull, 0x3fefe315e86e7f85ull, \
    0x3c8cd2523567f613ull, 0x3fefd9b0d3158574ull, 0xbc8bce8023f98efaull, 0x3fefd06b29ddf6deull, \
    0x3c60f74e61e6c861ull, 0x3fefc74518759bc8ull, 0x3c90a3e45b33d399ull, 0x3fefbe3ecac6f383ull, \
    0x3c979aa65d837b6dull, 0x3fefb5586cf9890full, 0x3c8eb51a92fdeffcull, 0x3fefac922b7247f7ull, \
    0x3c3ebe3d702f9cd1ull, 0x3fefa3ec32d3d1a2ull, 0xbc6a033489906e0bull, 0x3fef9b66affed31bull, \
    0xbc9556522a2fbd0eull, 0x3fef9301d0125b51ull, 0xbc5080ef8c4eea55ull, 0x3fef8abdc06c31ccull, \
    0xbc91c923b9d5f416ull, 0x3fef829aaea92de0ull, 0x3c80d3e3e95c55afull, 0x3fef7a98c8a58e51ull, \
    0xbc801b15eaa59348ull, 0x3fef72b83c7d517bull, 0xbc8f1ff055de323dull, 0x3fef6af9388c8deaull, \
    0x3c8b898c3f1353bfull, 0x3fef635beb6fcb75ull, 0xbc96d99c7611eb26ull, 0x3fef5be084045cd4ull, \
    0x3c9aecf73e3a2f60ull, 0x3fef54873168b9aaull, 0xbc8fe782cb86389dull, 0x3fef4d5022fcd91dull, \
    0x3c8a6f4144a6c38dull, 0x3fef463b88628cd6ull, 0x3c807a05b0e4047dull, 0x3fef3f49917ddc96ull, \
    0x3c968efde3a8a894ull, 0x3fef387a6e756238ull, 0x3c875e18f274487dull, 0x3fef31ce4fb2a63full, \
    0x3c80472b981fe7f2ull, 0x3fef2b4565e27cddull, 0xbc96b87b3f71085eull, 0x3fef24dfe1f56381ull, \
    0x3c82f7e16d09ab31ull, 0x3fef1e9df51fdee1ull, 0xbc3d219b1a6fbffaull, 0x3fef187fd0dad990ull, \
    0x3c8b3782720c0ab4ull, 0x3fef1285a6e4030bull, 0x3c6e149289cecb8full, 0x3fef0cafa93e2f56ull, \
    0x3c834d754db0abb6ull, 0x3fef06fe0a31b715ull, 0x3c864201e2ac744cull, 0x3fef0170fc4cd831ull, \
    0x3c8fdd395dd3f84aull, 0x3feefc08b26416ffull, 0xbc86a3803b8e5b04ull, 0x3feef6c55f929ff1ull, \
    0xbc924aedcc4b5068ull, 0x3feef1a7373aa9cbull, 0xbc9907f81b512d8eull, 0x3feeecae6d05d866ull, \
    0xbc71d1e83e9436d2ull, 0x3feee7db34e59ff7ull, 0xbc991919b3ce1b15ull, 0x3feee32dc313a8e5ull, \
    0x3c859f48a72a4c6dull, 0x3feedea64c123422ull, 0xbc9312607a28698aull, 0x3feeda4504ac801cull, \
    0xbc58a78f4817895bull, 0x3feed60a21f72e2aull, 0xbc7c2c9b67499a1bull, 0x3feed1f5d950a897ull, \
    0x3c4363ed60c2ac11ull, 0x3feece086061892dull, 0x3c9666093b0664efull, 0x3feeca41ed1d0057ull, \
    0x3c6ecce1daa10379ull, 0x3feec6a2b5c13cd0ull, 0x3c93ff8e3f0f1230ull, 0x3feec32af0d7d3deull, \
    0x3c7690cebb7aafb0ull, 0x3feebfdad5362a27ull, 0x3c931dbdeb54e077ull, 0x3feebcb299fddd0dull, \
    0xbc8f94340071a38eull, 0x3feeb9b2769d2ca7ull, 0xbc87deccdc93a349ull, 0x3feeb6daa2cf6642ull, \
    0xbc78dec6bd0f385full, 0x3feeb42b569d4f82ull, 0xbc861246ec7b5cf6ull, 0x3feeb1a4ca5d920full, \
    0x3c93350518fdd78eull, 0x3feeaf4736b527daull, 0x3c7b98b72f8a9b05ull, 0x3feead12d497c7fdull, \
    0x3c9063e1e21c5409ull, 0x3feeab07dd485429ull, 0x3c34c7855019c6eaull, 0x3feea9268a5946b7ull, \
    0x3c9432e62b64c035ull, 0x3feea76f15ad2148ull, 0xbc8ce44a6199769full, 0x3feea5e1b976dc09ull, \
    0xbc8c33c53bef4da8ull, 0x3feea47eb03a5585ull, 0xbc845378892be9aeull, 0x3feea34634ccc320ull, \
    0xbc93cedd78565858ull, 0x3feea23882552225ull, 0x3c5710aa807e1964ull, 0x3feea155d44ca973ull, \
    0xbc93b3efbf5e2228ull, 0x3feea09e667f3bcdull, 0xbc6a12ad8734b982ull, 0x3feea012750bdabfull, \
    0xbc6367efb86da9eeull, 0x3fee9fb23c651a2full, 0xbc80dc3d54e08851ull, 0x3fee9f7df9519484ull, \
    0xbc781f647e5a3ecfull, 0x3fee9f75e8ec5f74ull, 0xbc86ee4ac08b7db0ull, 0x3fee9f9a48a58174ull, \
    0xbc8619321e55e68aull, 0x3fee9feb564267c9ull, 0x3c909ccb5e09d4d3ull, 0x3feea0694fde5d3full, \
    0xbc7b32dcb94da51dull, 0x3feea11473eb0187ull, 0x3c94ecfd5467c06bull, 0x3feea1ed0130c132ull, \
    0x3c65ebe1abd66c55ull, 0x3feea2f336cf4e62ull, 0xbc88a1c52fb3cf42ull, 0x3feea427543e1a12ull, \
    0xbc9369b6f13b3734ull, 0x3feea589994cce13ull, 0xbc805e843a19ff1eull, 0x3feea71a4623c7adull, \
    0xbc94d450d872576eull, 0x3feea8d99b4492edull, 0x3c90ad675b0e8a00ull, 0x3feeaac7d98a6699ull, \
    0x3c8db72fc1f0eab4ull, 0x3feeace5422aa0dbull, 0xbc65b6609cc5e7ffull, 0x3feeaf3216b5448cull, \
    0x3c7bf68359f35f44ull, 0x3feeb1ae99157736ull, 0xbc93091fa71e3d83ull, 0x3feeb45b0b91ffc6ull, \
    0xbc5da9b88b6c1e29ull, 0x3feeb737b0cdc5e5ull, 0xbc6c23f97c90b959ull, 0x3feeba44cbc8520full, \
    0xbc92434322f4f9aaull, 0x3feebd829fde4e50ull, 0xbc85ca6cd7668e4bull, 0x3feec0f170ca07baull, \
    0x3c71affc2b91ce27ull, 0x3feec49182a3f090ull, 0x3c6dd235e10a73bbull, 0x3feec86319e32323ull, \
    0xbc87c50422622263ull, 0x3feecc667b5de565ull, 0x3c8b1c86e3e231d5ull, 0x3feed09bec4a2d33ull, \
    0xbc91bbd1d3bcbb15ull, 0x3feed503b23e255dull, 0x3c90cc319cee31d2ull, 0x3feed99e1330b358ull, \
    0x3c8469846e735ab3ull, 0x3feede6b5579fdbfull, 0xbc82dfcd978e9db4ull, 0x3feee36bbfd3f37aull, \
    0x3c8c1a7792cb3387ull, 0x3feee89f995ad3adull, 0xbc907b8f4ad1d9faull, 0x3feeee07298db666ull, \
    0xbc55c3d956dcaebaull, 0x3feef3a2b84f15fbull, 0xbc90a40e3da6f640ull, 0x3feef9728de5593aull, \
    0xbc68d6f438ad9334ull, 0x3feeff76f2fb5e47ull, 0xbc91eee26b588a35ull, 0x3fef05b030a1064aull, \
    0x3c74ffd70a5fddcdull, 0x3fef0c1e904bc1d2ull, 0xbc91bdfbfa9298acull, 0x3fef12c25bd71e09ull, \
    0x3c736eae30af0cb3ull, 0x3fef199bdd85529cull, 0x3c8ee3325c9ffd94ull, 0x3fef20ab5fffd07aull, \
    0x3c84e08fd10959acull, 0x3fef27f12e57d14bull, 0x3c63cdaf384e1a67ull, 0x3fef2f6d9406e7b5ull, \
    0x3c676b2c6c921968ull, 0x3fef3720dcef9069ull, 0xbc808a1883ccb5d2ull, 0x3fef3f0b555dc3faull, \
    0xbc8fad5d3ffffa6full, 0x3fef472d4a07897cull, 0xbc900dae3875a949ull, 0x3fef4f87080d89f2ull, \
    0x3c74a385a63d07a7ull, 0x3fef5818dcfba487ull, 0xbc82919e2040220full, 0x3fef60e316c98398ull, \
    0x3c8e5a50d5c192acull, 0x3fef69e603db3285ull, 0x3c843a59ac016b4bull, 0x3fef7321f301b460ull, \
    0xbc82d52107b43e1full, 0x3fef7c97337b9b5full, 0xbc892ab93b470dc9ull, 0x3fef864614f5a129ull, \
    0x3c74b604603a88d3ull, 0x3fef902ee78b3ff6ull, 0x3c83c5ec519d7271ull, 0x3fef9a51fbc74c83ull, \
    0xbc8ff7128fd391f0ull, 0x3fefa4afa2a490daull, 0xbc8dae98e223747dull, 0x3fefaf482d8e67f1ull, \
    0x3c8ec3bc41aa2008ull, 0x3fefba1bee615a27ull, 0x3c842b94c3a9eb32ull, 0x3fefc52b376bba97ull, \
    0x3c8a64a931d185eeull, 0x3fefd0765b6e4540ull, 0xbc8e37bae43be3edull, 0x3fefdbfdad9cbe14ull, \
    0x3c77893b4d91cd9dull, 0x3fefe7c1819e90d8ull, 0x3c5305c14160cc89ull, 0x3feff3c22b8f71f1ull }
// __log_data.tab: for i = 0..127, {invc, logc} as bit patterns
#define MDC_LOG_TAB_INIT { \
    0x3ff734f0c3e0de9full, 0xbfd7cc7f79e69000ull, 0x3ff713786a2ce91full, 0xbfd76feec20d0000ull, \
    0x3ff6f26008fab5a0ull, 0xbfd713e31351e000ull, 0x3ff6d1a61f138c7dull, 0xbfd6b85b38287800ull, \
    0x3ff6b1490bc5b4d1ull, 0xbfd65d5590807800ull, 0x3ff69147332f0cbaull, 0xbfd602d076180000ull, \
    0x3ff6719f18224223ull, 0xbfd5a8ca86909000ull, 0x3ff6524f99a51ed9ull, 0xbfd54f4356035000ull, \
    0x3ff63356aa8f24c4ull, 0xbfd4f637c36b4000ull, 0x3ff614b36b9ddc14ull, 0xbfd49da7fda85000ull, \
    0x3ff5f66452c65c4cull, 0xbfd445923989a800ull, 0x3ff5d867b5912c4full, 0xbfd3edf439b0b800ull, \
    0x3ff5babccb5b90deull, 0xbfd396ce448f7000ull, 0x3ff59d61f2d91a78ull, 0xbfd3401e17bda000ull, \
    0x3ff5805612465687ull, 0xbfd2e9e2ef468000ull, 0x3ff56397cee76bd3ull, 0xbfd2941b3830e000ull, \
    0x3ff54725e2a77f93ull, 0xbfd23ec58cda8800ull, 0x3ff52aff42064583ull, 0xbfd1e9e129279000ull, \
    0x3ff50f22dbb2bddfull, 0xbfd1956d2b48f800ull, 0x3ff4f38f4734ded7ull, 0xbfd141679ab9f800ull, \
    0x3ff4d843cfde2840ull, 0xbfd0edd094ef9800ull, 0x3ff4bd3ec078a3c8ull, 0xbfd09aa518db1000ull, \
    0x3ff4a27fc3e0258aull, 0xbfd047e65263b800ull, 0x3ff4880524d48434ull, 0xbfcfeb224586f000ull, \
    0x3ff46dce1b192d0bull, 0xbfcf474a7517b000ull, 0x3ff453d9d3391854ull, 0xbfcea4443d103000ull, \
    0x3ff43a2744b4845aull, 0xbfce020d44e9b000ull, 0x3ff420b54115f8fbull, 0xbfcd60a22977f000ull, \
    0x3ff40782da3ef4b1ull, 0xbfccc00104959000ull, 0x3ff3ee8f5d57fe8full, 0xbfcc202956891000ull, \
    0x3ff3d5d9a00b4ce9ull, 0xbfcb81178d811000ull, 0x3ff3bd60c010c12bull, 0xbfcae2c9ccd3d000ull, \
    0x3ff3a5242b75dab8ull, 0xbfca45402e129000ull, 0x3ff38d22cd9fd002ull, 0xbfc9a877681df000ull, \
    0x3ff3755bc5847a1cull, 0xbfc90c6d69483000ull, 0x3ff35dce49ad36e2ull, 0xbfc87120a645c000ull, \
    0x3ff34679984dd440ull, 0xbfc7d68fb4143000ull, 0x3ff32f5cceffcb24ull, 0xbfc73cb83c627000ull, \
    0x3ff3187775a10d49ull, 0xbfc6a39a9b376000ull, 0x3ff301c8373e3990ull, 0xbfc60b3154b7a000ull, \
    0x3ff2eb4ebb95f841ull, 0xbfc5737d76243000ull, 0x3ff2d50a0219a9d1ull, 0xbfc4dc7b8fc23000ull, \
    0x3ff2bef9a8b7fd2aull, 0xbfc4462c51d20000ull, 0x3ff2a91c7a0c1babull, 0xbfc3b08abc830000ull, \
    0x3ff293726014b530ull, 0xbfc31b996b490000ull, 0x3ff27dfa5757a1f5ull, 0xbfc2875490a44000ull, \
    0x3ff268b39b1d3bbfull, 0xbfc1f3b9f879a000ull, 0x3ff2539d838ff5bdull, 0xbfc160c8252ca000ull, \
    0x3ff23eb7aac9083bull, 0xbfc0ce7f57f72000ull, 0x3ff22a012ba940b6ull, 0xbfc03cdc49fea000ull, \
    0x3ff2157996cc4132ull, 0xbfbf57bdbc4b8000ull, 0x3ff201201dd2fc9bull, 0xbfbe370896404000ull, \
    0x3ff1ecf4494d480bull, 0xbfbd17983ef94000ull, 0x3ff1d8f5528f6569ull, 0xbfbbf9674ed8a000ull, \
    0x3ff1c52311577e7cull, 0xbfbadc79202f6000ull, 0x3ff1b17c74cb26e9ull, 0xbfb9c0c3e7288000ull, \
    0x3ff19e010c2c1ab6ull, 0xbfb8a646b372c000ull, 0x3ff18ab07bb670bdull, 0xbfb78d01b3ac0000ull, \
    0x3ff1778a25efbcb6ull, 0xbfb674f145380000ull, 0x3ff1648d354c31daull, 0xbfb55e0e6d878000ull, \
    0x3ff151b990275fddull, 0xbfb4485cdea1e000ull, 0x3ff13f0ea432d24cull, 0xbfb333d94d6aa000ull, \
    0x3ff12c8b7210f9daull, 0xbfb22079f8c56000ull, 0x3ff11a3028ecb531ull, 0xbfb10e4698622000ull, \
    0x3ff107fbda8434afull, 0xbfaffa6c6ad20000ull, 0x3ff0f5ee0f4e6bb3ull, 0xbfadda8d4a774000ull, \
    0x3ff0e4065d2a9fceull, 0xbfabbcece4850000ull, 0x3ff0d244632ca521ull, 0xbfa9a1894012c000ull, \
    0x3ff0c0a77ce2981aull, 0xbfa788583302c000ull, 0x3ff0af2f83c636d1ull, 0xbfa5715e67d68000ull, \
    0x3ff09ddb98a01339ull, 0xbfa35c8a49658000ull, 0x3ff08cabaf52e7dfull, 0xbfa149e364154000ull, \
    0x3ff07b9f2f4e28fbull, 0xbf9e72c082eb8000ull, 0x3ff06ab58c358f19ull, 0xbf9a55f152528000ull, \
    0x3ff059eea5ecf92cull, 0xbf963d62cf818000ull, 0x3ff04949cdd12c90ull, 0xbf9228fb8caa0000ull, \
    0x3ff038c6c6f0ada9ull, 0xbf8c317b20f90000ull, 0x3ff02865137932a9ull, 0xbf8419355daa0000ull, \
    0x3ff0182427ea7348ull, 0xbf781203c2ec0000ull, 0x3ff008040614b195ull, 0xbf60040979240000ull, \
    0x3fefe01ff726fa1aull, 0x3f6feff384900000ull, 0x3fefa11cc261ea74ull, 0x3f87dc41353d0000ull, \
    0x3fef6310b081992eull, 0x3f93cea3c4c28000ull, 0x3fef25f63ceeadcdull, 0x3f9b9fc114890000ull, \
    0x3feee9c8039113e7ull, 0x3fa1b0d8ce110000ull, 0x3feeae8078cbb1abull, 0x3fa58a5bd001c000ull, \
    0x3fee741aa29d0c9bull, 0x3fa95c8340d88000ull, 0x3fee3a91830a99b5ull, 0x3fad276aef578000ull, \
    0x3fee01e009609a56ull, 0x3fb07598e598c000ull, 0x3fedca01e577bb98ull, 0x3fb253f5e30d2000ull, \
    0x3fed92f20b7c9103ull, 0x3fb42edd8b380000ull, 0x3fed5cac66fb5cceull, 0x3fb606598757c000ull, \
    0x3fed272caa5ede9dull, 0x3fb7da76356a0000ull, 0x3fecf26e3e6b2ccdull, 0x3fb9ab434e1c6000ull, \
    0x3fecbe6da2a77902ull, 0x3fbb78c7bb0d6000ull, 0x3fec8b266d37086dull, 0x3fbd431332e72000ull, \
    0x3fec5894bd5d5804ull, 0x3fbf0a3171de6000ull, 0x3fec26b533bb9f8cull, 0x3fc067152b914000ull, \
    0x3febf583eeece73full, 0x3fc147858292b000ull, 0x3febc4fd75db96c1ull, 0x3fc2266ecdca3000ull, \
    0x3feb951e0c864a28ull, 0x3fc303d7a6c55000ull, 0x3feb65e2c5ef3e2cull, 0x3fc3dfc33c331000ull, \
    0x3feb374867c9888bull, 0x3fc4ba366b7a8000ull, 0x3feb094b211d304aull, 0x3fc5933928d1f000ull, \
    0x3feadbe885f2ef7eull, 0x3fc66acd2418f000ull, 0x3feaaf1d31603da2ull, 0x3fc740f8ec669000ull, \
    0x3fea82e63fd358a7ull, 0x3fc815c0f51af000ull, 0x3fea5740ef09738bull, 0x3fc8e92954f68000ull, \
    0x3fea2c2a90ab4b27ull, 0x3fc9bb3602f84000ull, 0x3fea01a01393f2d1ull, 0x3fca8bed1c2c0000ull, \
    0x3fe9d79f24db3c1bull, 0x3fcb5b515c01d000ull, 0x3fe9ae2505c7b190ull, 0x3fcc2967ccbcc000ull, \
    0x3fe9852ef297ce2full, 0x3fccf635d5486000ull, 0x3fe95cbaeea44b75ull, 0x3fcdc1bd3446c000ull, \
    0x3fe934c69de74838ull, 0x3fce8c01b8cfe000ull, 0x3fe90d4f2f6752e6ull, 0x3fcf5509c0179000ull, \
    0x3fe8e6528effd79dull, 0x3fd00e6c121fb800ull, 0x3fe8bfce9fcc007cull, 0x3fd071b80e93d000ull, \
    0x3fe899c0dabec30eull, 0x3fd0d46b9e867000ull, 0x3fe87427aa2317fbull, 0x3fd13687334bd000ull, \
    0x3fe84f00acb39a08ull, 0x3fd1980d67234800ull, 0x3fe82a49e8653e55ull, 0x3fd1f8ffe0cc8000ull, \
    0x3fe8060195f40260ull, 0x3fd2595fd7636800ull, 0x3fe7e22563e0a329ull, 0x3fd2b9300914a800ull, \
    0x3fe7beb377dcb5adull, 0x3fd3187210436000ull, 0x3fe79baa679725c2ull, 0x3fd377266dec1800ull, \
    0x3fe77907f2170657ull, 0x3fd3d54ffbaf3000ull, 0x3fe756cadbd6130cull, 0x3fd432eee32fe000ull }
#if defined(__CUDACC__)
static __device__ const uint64_t mdc_exp_tab_d[256] = MDC_EXP_TAB_INIT;
static __device__ const uint64_t mdc_log_tab_d[256] = MDC_LOG_TAB_INIT;
#endif
static const uint64_t mdc_exp_tab_h[256] = MDC_EXP_TAB_INIT;
static const uint64_t mdc_log_tab_h[256] = MDC_LOG_TAB_INIT;

// exp's special case: |x| > 512 where the scale 2^(k/128) alone would leave the double range
MDC_LM_HD double mdc_exp_special(double tmp, uint64_t sbits, uint64_t ki) {
    if ((ki & 0x80000000ull) == 0) {                      // k > 0: the scale's exponent may have overflowed by <= 460
        const double scale = MDC_LM_DBL(sbits - (1009ull << 52));
        return MDC_LM_MUL(0x1p1009, MDC_LM_FMA(scale, tmp, scale));                                          // FMA
    }
    const double scale = MDC_LM_DBL(sbits + (1022ull << 52));    // k < 0: care in the subnormal range
    const double st = MDC_LM_MUL(scale, tmp);
    double y = MDC_LM_ADD(scale, st);                                                                        // not fused
    if (y < 1.0) {
        double lo = MDC_LM_ADD(MDC_LM_SUB(scale, y), st);
        const double hi = MDC_LM_ADD(1.0, y);
        lo = MDC_LM_ADD(MDC_LM_ADD(MDC_LM_SUB(1.0, hi), y), lo);
        y = MDC_LM_SUB(MDC_LM_ADD(lo, hi), 1.0);
        if (y == 0.0) y = 0.0;
    }
    return MDC_LM_MUL(0x1p-1022, y);
}

MDC_LM_HD double mdc_exp(double x) {
    const uint64_t* T = MDC_LM_TAB(mdc_exp_tab);
    const double InvLn2N = 0x1.71547652b82fep7, Shift = 0x1.8p52, NegLn2hiN = -0x1.62e42fefa0000p-8, NegLn2loN = -0x1.cf79abc9e3b3ap-47;
    const double C2 = 0x1.ffffffffffdbdp-2, C3 = 0x1.555555555543cp-3, C4 = 0x1.55555cf172b91p-5, C5 = 0x1.1111167a4d017p-7;
    uint32_t abstop = static_cast<uint32_t>(MDC_LM_BITS(x) >> 52) & 0x7ff;
    if (abstop - 0x3c9u >= 0x408u - 0x3c9u) {
        if (abstop - 0x3c9u >= 0x80000000u) return MDC_LM_ADD(1.0, x);          // |x| < 2^-54
        if (abstop >= 0x409u) {
            if (MDC_LM_BITS(x) == 0xfff0000000000000ull) return 0.0;
            if (abstop >= 0x7ffu) return MDC_LM_ADD(1.0, x);
            return (MDC_LM_BITS(x) >> 63) ? 0.0 : MDC_LM_DBL(0x7ff0000000000000ull);     // __math_uflow / __math_oflow
        }
        abstop = 0;                                                             // large |x|: special case below
    }
    const double kd0 = MDC_LM_FMA(x, InvLn2N, Shift);                                                        // FMA
    const uint64_t ki = MDC_LM_BITS(kd0);
    const double kd = MDC_LM_SUB(kd0, Shift);
    const double r = MDC_LM_FMA(kd, NegLn2loN, MDC_LM_FMA(kd, NegLn2hiN, x));                                // FMA, FMA
    const uint64_t idx = 2 * (ki % 128), top = ki << 45;
    const double tail = MDC_LM_DBL(T[idx]);
    const uint64_t sbits = T[idx + 1] + top;
    const double r2 = MDC_LM_MUL(r, r);
    const double a = MDC_LM_FMA(MDC_LM_FMA(r, C3, C2), r2, MDC_LM_ADD(tail, r));                             // FMA, FMA
    const double tmp = MDC_LM_FMA(MDC_LM_MUL(r2, r2), MDC_LM_FMA(r, C5, C4), a);                             // FMA, FMA
    if (abstop == 0) return mdc_exp_special(tmp, sbits, ki);
    const double scale = MDC_LM_DBL(sbits);
    return MDC_LM_FMA(scale, tmp, scale);                                                                    // FMA
}

MDC_LM_HD double mdc_log(double x) {
    const uint64_t* T = MDC_LM_TAB(mdc_log_tab);
    const double Ln2hi = 0x1.62e42fefa3800p-1, Ln2lo = 0x1.ef35793c76730p-45;
    const double A0 = -0x1.0000000000001p-1, A1 = 0x1.555555551305bp-2, A2 = -0x1.fffffffeb4590p-3, A3 = 0x1.999b324f10111p-3,
                 A4 = -0x1.55575e506c89fp-3;
    uint64_t ix = MDC_LM_BITS(x);
    const uint32_t top = static_cast<uint32_t>(ix >> 48);
    if (ix - 0x3fee000000000000ull < 0x3090000000000ull) {                      // x in [1 - 2^-4, 1 + 0x1.09p-4)
        const double B0 = -0x1p-1, B1 = 0x1.5555555555577p-2, B2 = -0x1.ffffffffffdcbp-3, B3 = 0x1.999999995dd0cp-3,
                     B4 = -0x1.55555556745a7p-3, B5 = 0x1.24924a344de30p-3, B6 = -0x1.fffffa4423d65p-4, B7 = 0x1.c7184282ad6cap-4,
                     B8 = -0x1.999eb43b068ffp-4, B9 = 0x1.78182f7afd085p-4, B10 = -0x1.5521375d145cdp-4;
        if (ix == 0x3ff0000000000000ull) return 0.0;
        const double r = MDC_LM_SUB(x, 1.0), r2 = MDC_LM_MUL(r, r), r3 = MDC_LM_MUL(r, r2);
        const double a = MDC_LM_FMA(r2, B3, MDC_LM_FMA(r, B2, B1));                                          // FMA, FMA
        const double b = MDC_LM_FMA(r2, B6, MDC_LM_FMA(r, B5, B4));                                          // FMA, FMA
        const double c = MDC_LM_FMA(r3, B10, MDC_LM_FMA(r2, B9, MDC_LM_FMA(r, B8, B7)));                     // FMA x3
        const double p = MDC_LM_FMA(MDC_LM_FMA(c, r3, b), r3, a);                                            // FMA, FMA
        const double rhi = MDC_LM_FMA(-r, 0x1p27, MDC_LM_FMA(r, 0x1p27, r));          // r + w - w, w = r * 2^27: FMA, FMA
        const double rlo = MDC_LM_SUB(r, rhi), rr = MDC_LM_MUL(rhi, rhi);
        const double hi = MDC_LM_FMA(rr, B0, r);                                                             // FMA
        double lo = MDC_LM_FMA(rr, B0, MDC_LM_SUB(r, hi));                                                   // FMA
        lo = MDC_LM_FMA(MDC_LM_MUL(B0, rlo), MDC_LM_ADD(r, rhi), lo);                                        // FMA
        return MDC_LM_ADD(hi, MDC_LM_FMA(p, r3, lo));                                                        // FMA
    }
    if (top - 0x0010u >= 0x7ff0u - 0x0010u) {                                   // x < 2^-1022, inf or NaN
        if (ix * 2 == 0) return MDC_LM_DBL(0xfff0000000000000ull);             // log(+-0) = -inf
        if (ix == 0x7ff0000000000000ull) return x;
        if (x != x) return MDC_LM_ADD(x, x);                                   // NaN
        if (top & 0x8000u) return MDC_LM_DBL(0xfff8000000000000ull);          // x < 0: NaN
        ix = MDC_LM_BITS(MDC_LM_MUL(x, 0x1p52)) - (52ull << 52);                // subnormal: normalise
    }
    const uint64_t tmp = ix - 0x3fe6000000000000ull;
    const int i = static_cast<int>((tmp >> 45) % 128);
    const int k = static_cast<int>(static_cast<int64_t>(tmp) >> 52);
    const double z = MDC_LM_DBL(ix - (tmp & (0xfffull << 52)));
    const double invc = MDC_LM_DBL(T[2 * i]), logc = MDC_LM_DBL(T[2 * i + 1]);
    const double r = MDC_LM_FMA(z, invc, -1.0);                                                              // __FP_FAST_FMA branch
    const double kd = static_cast<double>(k);
    const double w = MDC_LM_FMA(kd, Ln2hi, logc);                                                            // FMA
    const double hi = MDC_LM_ADD(w, r);
    const double lo = MDC_LM_FMA(kd, Ln2lo, MDC_LM_ADD(MDC_LM_SUB(w, hi), r));                               // FMA
    const double r2 = MDC_LM_MUL(r, r);
    const double q = MDC_LM_FMA(MDC_LM_FMA(r, A4, A3), r2, MDC_LM_FMA(r, A2, A1));                           // FMA x3
    const double y = MDC_LM_FMA(MDC_LM_MUL(r, r2), q, MDC_LM_FMA(r2, A0, lo));                               // FMA, FMA
    return MDC_LM_ADD(y, hi);
}
