/*
 * mdc_b200_nccl.h — optional native multi-GPU init for C++ hosts (libmdc_b200_nccl.so, links libnccl).
 *
 * The reference is single-process / single-device; this is the GPU-side equivalent of "construct the
 * DatasetReader's two calibration objects" when frames are sharded over several GPUs (SURVEY.md §8e): rank
 * `root` has parsed the files and built the tables on its host (mdc_fov_create / mdc_photo_create), the four
 * tables travel once over NVLink with ncclBroadcast, and every rank gets a device context that owns its copy.
 * There is no collective after this call.  Python hosts use torch.distributed instead
 * (mono_dataset_code_b200/sharding.py); both paths end in mdc_ctx_create_from_device_tables.
 */
#ifndef MDC_B200_NCCL_H
#define MDC_B200_NCCL_H
#include "mdc_b200.h"
#ifdef __cplusplus
extern "C" {
#endif

/* nccl_comm: an initialised ncclComm_t for this rank (passed as void* to keep nccl.h out of this header).
 * fov / photo: the host models on `root`, ignored (may be NULL) elsewhere.  device: this rank's CUDA device. */
int mdc_ctx_create_broadcast(void* nccl_comm, int rank, int root, int device, const mdc_fov* fov, const mdc_photo* photo,
                             mdc_ctx** out);

/* Communicator set-up for hosts without an NCCL binding of their own: rank 0 calls mdc_nccl_unique_id, ships the 128 bytes to the
 * other ranks by any means (file, socket, the launcher's store), every rank calls mdc_nccl_comm_create. */
int mdc_nccl_unique_id(char id_out[128]);
int mdc_nccl_comm_create(const char id[128], int world, int rank, int device, void** comm_out);
void mdc_nccl_comm_destroy(void* comm);
int mdc_nccl_version(void);

/* responseCalib's optimisation loop (main_responseCalib.cpp:281-362) PIXEL-SHARDED over the ranks of `nccl_comm` (SURVEY.md §8e):
 * d_data_local = this rank's slice of every image, [n][npix_local] u8 (slices of a multiple of 16 pixels keep the fast streaming
 * kernels); d_E_local [npix_local]; d_G [256] is replicated.  The G-step's sums cross the ranks as integers (mdc_rc_gstep_scale /
 * _accumulate_exact / _finish_exact, include/mdc_b200.h): per iteration ncclAllReduce MAX of 4 u64, SUM of 768 int64 and of 256 fp64
 * (+ 256 u64 counts in the first iteration), so d_G and d_E_local hold the same bits for ANY number of ranks, mdc_response_calib's
 * included; the three rmse evaluations all-reduce 2 doubles each; E-step, E-init and rescale are collective-free.  log_host as in
 * mdc_response_calib (global rmse / count).  Same call on every rank.  A rank may hold no pixels (npix_local = 0; d_data_local and
 * d_E_local may then be null): it still takes part in every collective.
 * A rank that fails mid-loop (a CUDA error, a bad argument on that rank only) returns without reaching the remaining collectives, and
 * its peers then wait in an all-reduce that never completes: NCCL has no timeout here, so the host must abort the communicator
 * (ncclCommAbort) or end the processes.  The call does not recover from that. */
int mdc_response_calib_sharded(mdc_ctx* c, void* nccl_comm, int device, const uint8_t* d_data_local, int n, int npix_local,
                               const double* d_t, int nits, double* d_E_local, double* d_G, double* log_host);

#ifdef __cplusplus
}
#endif
#endif
