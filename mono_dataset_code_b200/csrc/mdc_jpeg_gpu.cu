// Baseline-JPEG decoding on the GPU, to the same bytes as the host decoder (mdc_jpeg.cpp):
//   host   the shared marker walk (mdc_jpeg_parse_header) and restart split (mdc_jpeg_split_segments); Huffman / quantisation tables
//          deduplicated over the batch (frames written by one encoder share them)
//   J1     entropy decode: one thread per restart segment, the segments of every frame of the batch at once
//          (mdcj::mdc_jpeg_decode_segment); dequantised coefficients of each luminance block into its own slot
//   J2     inverse DCT: eight threads per 8x8 block (a column each, then a row each), exactly mdcj::idct_block; cropped samples
//          into a u8 batch [n][h][row_pitch]
//   errors per frame in a status word (the first failing segment and its kind), never a trap
// mdc_jpeg_decode_device decodes host buffers.  One device feed (run_device_feed) reads a sequence's frames on the decode-ahead pool
// (mdc_feed.h) and sends them H2D -> J1 -> J2 chunk by chunk: mdc_seq_prepare_device runs K1 on each chunk, mdc_seq_read_gray8_device
// leaves the raw frames in the caller's rows.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <exception>
#include <functional>
#include <map>
#include <memory>
#include <mutex>
#include <string>
#include <vector>

#include "mdc_feed.h"
#include "mdc_internal.h"
#include "mdc_jpeg.h"

#define CU_CHECK(expr)                                                                          \
    do {                                                                                        \
        cudaError_t e__ = (expr);                                                               \
        if (e__ != cudaSuccess) {                                                               \
            mdc_set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(e__), __FILE__, __LINE__); \
            return MDC_ERR_CUDA;                                                                \
        }                                                                                       \
    } while (0)

namespace {

constexpr uint32_t kStatusOk = 0xffffffffu;      // status word of a frame no segment has failed in: (segment << 2) | kind otherwise
constexpr int kJ1Threads = 32;               // one warp per CTA: a batch of long segments spreads over every SM
constexpr int kJ2BlocksPerCta = 32;              // 8 threads per 8x8 block

struct DevFrame {
    mdcj::SegmentFrame sf;       // table pointers into the batch's device table array
    size_t coef_off;             // first coefficient (int32 units) of the frame's padded luminance plane
    int valid;                   // 0: nothing to write (the host rejected the frame, or a restart marker is missing)
    int kind;                    // 0: JPEG; 1: raw pixels at raw_off of the byte buffer, copied by J2
    size_t raw_off;
};
struct DevSeg { size_t begin, end; int frame, index, first_mcu, n_mcus; };

__device__ const uint8_t kZigZagDev[64] = MDC_JPEG_ZIGZAG;

// J1: one thread per restart segment.  The bit state lives in registers; table look-ups go through L1.
__global__ void __launch_bounds__(kJ1Threads) j1_entropy_decode(const uint8_t* __restrict__ bytes, const DevSeg* __restrict__ segs, int n_segs,
                                                                const DevFrame* __restrict__ frames, int32_t* __restrict__ coef,
                                                                uint32_t* __restrict__ status) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n_segs) return;
    const DevSeg s = segs[i];
    const DevFrame& f = frames[s.frame];
    const int rc = mdcj::mdc_jpeg_decode_segment(bytes + s.begin, bytes + s.end, f.sf, s.first_mcu, s.n_mcus, coef + f.coef_off);
    if (rc != mdcj::kSegOk) atomicMin(status + s.frame, (static_cast<uint32_t>(s.index) << 2) | static_cast<uint32_t>(rc));
}

// J2: blockIdx.y = frame, 32 visible 8x8 blocks per CTA, 8 threads per block.  Pass 1 column t of the block, pass 2 row t, both
// through shared memory; exactly mdcj::idct_block (64-bit temporaries).  Raw (non-JPEG) frames are copied row by row instead.
__global__ void __launch_bounds__(8 * kJ2BlocksPerCta) j2_idct(const int32_t* __restrict__ coef, const DevFrame* __restrict__ frames,
                                                               const uint32_t* __restrict__ status, const uint8_t* __restrict__ bytes,
                                                               int w, int h, uint8_t* __restrict__ out, size_t pitch) {
    __shared__ int32_t sc[kJ2BlocksPerCta][64];
    __shared__ mdcj::wide sw[kJ2BlocksPerCta][64];
    const int fi = blockIdx.y;
    const DevFrame& f = frames[fi];
    if (!f.valid || status[fi] != kStatusOk) return;
    uint8_t* dst = out + static_cast<size_t>(fi) * h * pitch;
    if (f.kind == 1) {             // raw pixels: rows of this CTA's slice of the frame
        for (int y = blockIdx.x; y < h; y += gridDim.x)
            for (int x = threadIdx.x; x < w; x += blockDim.x) dst[static_cast<size_t>(y) * pitch + x] = bytes[f.raw_off + static_cast<size_t>(y) * w + x];
        return;
    }
    const int bw = (w + 7) / 8, bh = (h + 7) / 8;
    const int g = threadIdx.x >> 3, t = threadIdx.x & 7;
    const int blk = blockIdx.x * kJ2BlocksPerCta + g;
    const bool live = blk < bw * bh;
    const int by = live ? blk / bw : 0, bx = live ? blk - by * bw : 0;
    if (live) {
        const int32_t* src = coef + f.coef_off + 64 * (static_cast<size_t>(by) * f.sf.blocks_w + bx);
        for (int k = t; k < 64; k += 8) sc[g][kZigZagDev[k]] = src[k];
    }
    __syncthreads();
    if (live) mdcj::idct_column(sc[g], t, sw[g]);
    __syncthreads();
    if (!live) return;
    uint8_t row[8];
    mdcj::idct_row(sw[g], t, row);
    const int y = by * 8 + t;
    if (y >= h) return;
    uint8_t* o = dst + static_cast<size_t>(y) * pitch + bx * 8;
    const int nx = min(8, w - bx * 8);
    for (int x = 0; x < nx; ++x) o[x] = row[x];
}

// ----------------------------------------------------------------------------------------------- host side of a batch
// What a batch needs on the device, built on the host: frame and segment descriptors, the deduplicated tables, and where each
// frame's entropy-coded bytes (or raw pixels) sit in the packed byte buffer.
struct HostBatch {
    std::vector<DevFrame> frames;
    std::vector<DevSeg> segs;
    std::vector<mdcj::HuffTable> tables;
    std::vector<int32_t> qtabs;                      // 64 per distinct quantisation table
    std::map<std::string, int> table_ids, qtab_ids;
    std::vector<int> tab_idx;                        // per frame: dc0 dc1 dc2 ac0 ac1 ac2 (table index), qtab index
    std::vector<std::string> incomplete_msg;         // per frame: the message if a restart marker is missing, else ""
    size_t coef_words = 0, bytes = 0;
    int table_id(const mdcj::HuffTable& t) {
        int total = 0;                               // the table is a function of its code-length counts and its symbols
        for (int l = 1; l <= 16; ++l) total += t.bits[l];
        const std::string key = std::string(reinterpret_cast<const char*>(t.bits + 1), 16) + std::string(reinterpret_cast<const char*>(t.vals), static_cast<size_t>(total));
        auto it = table_ids.find(key);
        if (it != table_ids.end()) return it->second;
        tables.push_back(t);
        return table_ids[key] = static_cast<int>(tables.size()) - 1;
    }
    int qtab_id(const int32_t* q) {
        const std::string key(reinterpret_cast<const char*>(q), 64 * sizeof(int32_t));
        auto it = qtab_ids.find(key);
        if (it != qtab_ids.end()) return it->second;
        qtabs.insert(qtabs.end(), q, q + 64);
        return qtab_ids[key] = static_cast<int>(qtabs.size() / 64) - 1;
    }
    // a frame nothing is decoded for
    void add_skipped() {
        DevFrame f;
        memset(&f, 0, sizeof f);
        frames.push_back(f);
        tab_idx.insert(tab_idx.end(), 7, 0);
        incomplete_msg.emplace_back();
    }
    // a frame of raw pixels (w x h) at byte offset `at`
    void add_raw(size_t at) {
        add_skipped();
        frames.back().valid = 1;
        frames.back().kind = 1;
        frames.back().raw_off = at;
    }
    // a parsed JPEG whose entropy-coded bytes [segs.front().begin, segs.back().end) of the file are packed at byte offset `at`
    void add_jpeg(const mdc_jpeg_header& h, const std::vector<mdc_jpeg_segment>& fs, bool complete, const std::string& name, size_t at) {
        DevFrame f;
        memset(&f, 0, sizeof f);
        f.sf.ncomp = h.ncomp;
        f.sf.mcus_x = h.mcus_x;
        f.sf.blocks_w = h.blocks_w();
        for (int c = 0; c < 3; ++c) { f.sf.h[c] = c < h.ncomp ? h.comp[c].h : 1; f.sf.v[c] = c < h.ncomp ? h.comp[c].v : 1; }
        f.coef_off = coef_words;
        f.valid = complete ? 1 : 0;
        coef_words += static_cast<size_t>(h.blocks_w()) * h.blocks_h() * 64;
        const int fi = static_cast<int>(frames.size());
        for (int c = 0; c < 3; ++c) tab_idx.push_back(table_id(h.dc[h.comp[c < h.ncomp ? c : 0].td]));
        for (int c = 0; c < 3; ++c) tab_idx.push_back(table_id(h.ac[h.comp[c < h.ncomp ? c : 0].ta]));
        tab_idx.push_back(qtab_id(h.qzz));
        const size_t base = fs.empty() ? 0 : fs.front().begin;
        for (size_t k = 0; k < fs.size(); ++k)
            segs.push_back(DevSeg{at + fs[k].begin - base, at + fs[k].end - base, fi, static_cast<int>(k), fs[k].first_mcu, fs[k].n_mcus});
        frames.push_back(f);
        incomplete_msg.push_back(complete ? std::string() : name + ": missing restart marker");
    }
    // metadata layout in one upload: frames | segs | tables | qtabs (each 16-byte aligned)
    size_t off_segs() const { return align(frames.size() * sizeof(DevFrame)); }
    size_t off_tables() const { return off_segs() + align(segs.size() * sizeof(DevSeg)); }
    size_t off_qtabs() const { return off_tables() + align(tables.size() * sizeof(mdcj::HuffTable)); }
    size_t meta_bytes() const { return off_qtabs() + align(qtabs.size() * sizeof(int32_t)); }
    static size_t align(size_t b) { return (b + 15) & ~size_t(15); }
    // writes the metadata for a device copy at d_meta into host memory `m` (meta_bytes())
    void write_meta(uint8_t* m, uint8_t* d_meta) {
        const mdcj::HuffTable* d_tab = reinterpret_cast<const mdcj::HuffTable*>(d_meta + off_tables());
        const int32_t* d_q = reinterpret_cast<const int32_t*>(d_meta + off_qtabs());
        for (size_t i = 0; i < frames.size(); ++i) {
            const int* ti = &tab_idx[7 * i];
            for (int c = 0; c < 3; ++c) { frames[i].sf.dc[c] = d_tab + ti[c]; frames[i].sf.ac[c] = d_tab + ti[3 + c]; }
            frames[i].sf.qzz = d_q + 64 * ti[6];
        }
        if (!frames.empty()) memcpy(m, frames.data(), frames.size() * sizeof(DevFrame));
        if (!segs.empty()) memcpy(m + off_segs(), segs.data(), segs.size() * sizeof(DevSeg));
        if (!tables.empty()) memcpy(m + off_tables(), tables.data(), tables.size() * sizeof(mdcj::HuffTable));
        if (!qtabs.empty()) memcpy(m + off_qtabs(), qtabs.data(), qtabs.size() * sizeof(int32_t));
    }
};

// A decoded frame's message: the kind of the first interval J1 failed in (status word st), else the host's "missing restart
// marker" verdict (`incomplete`, "" if the scan is complete), as the host decoder reports them.  "" for a frame that decoded.
std::string frame_message(uint32_t st, const std::string& name, const std::string& incomplete) {
    if (st == kStatusOk) return incomplete;
    switch (st & 3) {
        case mdcj::kBlockBadDc: return name + ": corrupt JPEG data (DC)";
        case mdcj::kBlockBadAc: return name + ": corrupt JPEG data (AC)";
        default: return name + ": corrupt JPEG data (run past the block)";
    }
}

// Device buffers of one batch in flight, grown as needed.
struct DevSlot {
    uint8_t* bytes = nullptr; size_t bytes_cap = 0;
    uint8_t* meta = nullptr; size_t meta_cap = 0;
    int32_t* coef = nullptr; size_t coef_cap = 0;
    uint32_t* status = nullptr; size_t status_cap = 0;
    uint8_t* u8 = nullptr; size_t u8_cap = 0;
    void release() {
        cudaFree(bytes); cudaFree(meta); cudaFree(coef); cudaFree(status); cudaFree(u8);
        *this = DevSlot();
    }
};
template <class T>
int grow(T** p, size_t* cap, size_t count) {
    if (*cap >= count && *p) return MDC_OK;
    if (*p) cudaFree(*p);
    *p = nullptr; *cap = 0;
    const size_t n = std::max<size_t>(count, 1);
    CU_CHECK(cudaMalloc(reinterpret_cast<void**>(p), n * sizeof(T)));
    *cap = n;
    return MDC_OK;
}

// Enqueues H2D (metadata from `meta_host`, already written for slot.meta, and `nbytes` packed bytes), J1, J2 and the D2H copy of
// the frames' status words.  The device buffers of `slot` must have been grown for this batch (prepare_slot).
int enqueue_batch(const HostBatch& b, DevSlot& slot, const uint8_t* meta_host, const uint8_t* bytes_host, int w, int h, uint8_t* d_out,
                  size_t pitch, uint32_t* status_host, cudaStream_t s) {
    const int n = static_cast<int>(b.frames.size());
    if (n == 0) return MDC_OK;
    CU_CHECK(cudaMemcpyAsync(slot.meta, meta_host, b.meta_bytes(), cudaMemcpyHostToDevice, s));
    if (b.bytes) CU_CHECK(cudaMemcpyAsync(slot.bytes, bytes_host, b.bytes, cudaMemcpyHostToDevice, s));
    CU_CHECK(cudaMemsetAsync(slot.status, 0xff, static_cast<size_t>(n) * sizeof(uint32_t), s));
    if (b.coef_words) CU_CHECK(cudaMemsetAsync(slot.coef, 0, b.coef_words * sizeof(int32_t), s));
    const DevFrame* d_frames = reinterpret_cast<const DevFrame*>(slot.meta);
    const DevSeg* d_segs = reinterpret_cast<const DevSeg*>(slot.meta + b.off_segs());
    const int n_segs = static_cast<int>(b.segs.size());
    if (n_segs) {
        j1_entropy_decode<<<(n_segs + kJ1Threads - 1) / kJ1Threads, kJ1Threads, 0, s>>>(slot.bytes, d_segs, n_segs, d_frames, slot.coef, slot.status);
        CU_CHECK(cudaGetLastError());
    }
    const int vis = ((w + 7) / 8) * ((h + 7) / 8);
    j2_idct<<<dim3((vis + kJ2BlocksPerCta - 1) / kJ2BlocksPerCta, n), 8 * kJ2BlocksPerCta, 0, s>>>(slot.coef, d_frames, slot.status, slot.bytes, w, h,
                                                                                                     d_out, pitch);
    CU_CHECK(cudaGetLastError());
    CU_CHECK(cudaMemcpyAsync(status_host, slot.status, static_cast<size_t>(n) * sizeof(uint32_t), cudaMemcpyDeviceToHost, s));
    return MDC_OK;
}

int prepare_slot(const HostBatch& b, DevSlot& slot) {
    int rc = grow(&slot.meta, &slot.meta_cap, b.meta_bytes());
    if (rc == MDC_OK) rc = grow(&slot.bytes, &slot.bytes_cap, b.bytes);
    if (rc == MDC_OK) rc = grow(&slot.coef, &slot.coef_cap, b.coef_words);
    if (rc == MDC_OK) rc = grow(&slot.status, &slot.status_cap, b.frames.size());
    return rc;
}

}  // namespace

// ------------------------------------------------------------------------------------------------------- decode host buffers
extern "C" int mdc_jpeg_decode_device(mdc_ctx* c, const uint8_t* const* files, const size_t* sizes, int n, int w, int h, uint8_t* d_out,
                                      size_t row_pitch, int* status_host, mdc_stream stream) {
    if (!c || n < 0 || (n > 0 && (!files || !sizes || !d_out)) || w < 1 || h < 1 || row_pitch < static_cast<size_t>(w)) {
        mdc_set_error("mdc_jpeg_decode_device: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    if (n == 0) return MDC_OK;
    CU_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t s = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    HostBatch b;
    std::vector<std::string> msg(static_cast<size_t>(n));
    std::vector<size_t> src_off(static_cast<size_t>(n), 0), src_len(static_cast<size_t>(n), 0);
    const uint8_t* none = nullptr;
    std::vector<const uint8_t*> src(static_cast<size_t>(n), none);
    try {
        static thread_local mdc_jpeg_header hdr;
        std::vector<mdc_jpeg_segment> fs;
        for (int i = 0; i < n; ++i) {
            const std::string name = "frame " + std::to_string(i);
            if (!files[i] || !mdc_jpeg_parse_header(files[i], sizes[i], name, &hdr)) {
                msg[static_cast<size_t>(i)] = files[i] ? mdc_last_error() : name + ": no data";
                b.add_skipped();
                continue;
            }
            if (hdr.width != w || hdr.height != h) {
                msg[static_cast<size_t>(i)] = mdc_dims_message(w, h, hdr.width, hdr.height, name);
                b.add_skipped();
                continue;
            }
            const bool complete = mdc_jpeg_split_segments(files[i], sizes[i], hdr, &fs);
            const size_t begin = fs.empty() ? 0 : fs.front().begin, end = fs.empty() ? 0 : fs.back().end;
            b.add_jpeg(hdr, fs, complete, name, b.bytes);
            src[static_cast<size_t>(i)] = files[i] + begin;
            src_off[static_cast<size_t>(i)] = b.bytes;
            src_len[static_cast<size_t>(i)] = end - begin;
            b.bytes += end - begin;
        }
    } catch (const std::exception& e) {
        mdc_set_error("mdc_jpeg_decode_device: %s", e.what());
        return MDC_ERR_INVALID_ARG;
    }
    DevSlot slot;
    int rc = prepare_slot(b, slot);
    uint8_t* pinned = nullptr;
    uint32_t* st = nullptr;
    const size_t meta = b.meta_bytes();
    if (rc == MDC_OK && mdc_host_alloc(reinterpret_cast<void**>(&pinned), meta + b.bytes + sizeof(uint32_t) * n) != MDC_OK) rc = MDC_ERR_CUDA;
    if (rc == MDC_OK) {
        b.write_meta(pinned, slot.meta);
        for (int i = 0; i < n; ++i)
            if (src_len[static_cast<size_t>(i)]) memcpy(pinned + meta + src_off[static_cast<size_t>(i)], src[static_cast<size_t>(i)], src_len[static_cast<size_t>(i)]);
        st = reinterpret_cast<uint32_t*>(pinned + meta + b.bytes);
        rc = enqueue_batch(b, slot, pinned, pinned + meta, w, h, d_out, row_pitch, st, s);
        const cudaError_t e = cudaStreamSynchronize(s);
        if (rc == MDC_OK && e != cudaSuccess) { mdc_set_error("mdc_jpeg_decode_device: %s", cudaGetErrorString(e)); rc = MDC_ERR_CUDA; }
    }
    int first_bad = -1;
    std::string first_msg;
    if (rc == MDC_OK) {
        for (int i = 0; i < n; ++i) {
            std::string& m = msg[static_cast<size_t>(i)];
            if (m.empty()) m = frame_message(st[i], "frame " + std::to_string(i), b.incomplete_msg[static_cast<size_t>(i)]);
            if (status_host) status_host[i] = m.empty() ? MDC_OK : MDC_ERR_FORMAT;
            if (!m.empty() && first_bad < 0) { first_bad = i; first_msg = m; }
        }
    }
    if (pinned) mdc_host_free(pinned);
    slot.release();
    if (rc != MDC_OK) return rc;
    if (first_bad >= 0) { mdc_set_error("%s", first_msg.c_str()); return MDC_ERR_FORMAT; }
    return MDC_OK;
}

// ------------------------------------------------------------------------------------------------------- sequence feed
namespace {

// what a decode thread leaves for the GPU side, per frame of a chunk
struct FeedFrame {
    std::vector<uint8_t> file;                 // the file's bytes (a JPEG's entropy-coded data is packed from here)
    std::vector<uint8_t> px;                   // PNG / PGM: the decoded 8-bit pixels
    std::unique_ptr<mdc_jpeg_header> hdr;      // JPEG: the parsed header
    std::vector<mdc_jpeg_segment> segs;
    bool jpeg = false, complete = true;
    int status = MDC_OK;                       // MDC_OK: goes to the GPU; MDC_ERR_FORMAT: the host reader fails on it; MDC_ERR_INVALID_ARG: it reads, at another size
    int w = 0, h = 0;                          // the size the host reader reports (0 0 if it fails)
    std::string msg;                           // why the frame is not MDC_OK
};

// the frames a chunk of the device feed holds: more frames decode at once in J1, which keeps more of the GPU busy
int device_feed_chunk(int threads) { return std::min(512, std::max(16, 32 * threads)); }

// Reads frame `id` of `s` into `ff`: the file, then a JPEG's header and restart split (its entropy decoding is the GPU's), or a PNG /
// PGM decoded to 8 bits.  The outcome is the one mdc_seq_read_gray8 would have, with frames of another size than w x h marked.
void read_feed_frame(const mdc_seq* s, int id, int w, int h, FeedFrame& ff, mdc_gray_image& img) {
    const std::string name = mdc_seq_name(s, id);
    ff.jpeg = false;
    ff.status = MDC_ERR_FORMAT;
    ff.w = ff.h = 0;
    ff.msg.clear();
    int fw = 0, fh = 0;
    try {
        if (!mdc_seq_read_file(s, id, &ff.file)) { ff.msg = mdc_last_error(); return; }
        if (ff.file.size() >= 2 && ff.file[0] == 0xff && ff.file[1] == 0xd8) {
            if (!ff.hdr) ff.hdr.reset(new mdc_jpeg_header);
            if (!mdc_jpeg_parse_header(ff.file.data(), ff.file.size(), name, ff.hdr.get())) { ff.msg = mdc_last_error(); return; }
            fw = ff.hdr->width; fh = ff.hdr->height;
            if (fw != w || fh != h) {         // not decoded on the GPU: whether the host decoder accepts it decides its status
                if (!mdc_decode_gray_image(ff.file, name, &img)) { ff.msg = mdc_last_error(); return; }
            } else {
                ff.jpeg = true;
                ff.complete = mdc_jpeg_split_segments(ff.file.data(), ff.file.size(), *ff.hdr, &ff.segs);
            }
        } else {
            if (!mdc_decode_gray_image(ff.file, name, &img)) { ff.msg = mdc_last_error(); return; }
            fw = img.cols; fh = img.rows;
            mdc_gray_to_u8(img, &ff.px);
        }
    } catch (const std::exception& e) {
        ff.jpeg = false;
        ff.msg = name + ": cannot read (" + e.what() + ")";
        return;
    }
    ff.w = fw; ff.h = fh;
    ff.status = MDC_OK;
    if (fw != w || fh != h) {
        ff.jpeg = false;
        ff.status = MDC_ERR_INVALID_ARG;
        ff.msg = mdc_dims_message(w, h, fw, fh, "image " + name);
    }
}

// Chunk [f0, f0 + n) of a device feed after J1 / J2, per frame: the status and size mdc_seq_read_gray8 would give (FeedFrame), its
// message, and where J2 wrote the frames that are MDC_OK ([n][h][pitch]).
struct FeedChunk {
    int f0 = 0, n = 0;
    uint8_t* frames = nullptr;
    std::vector<int> status, sizes;            // sizes: w h per frame
    std::vector<std::string> msg;
};

// The device feed behind mdc_seq_prepare_device and mdc_seq_read_gray8_device: frames ids[0 .. count) of `s`, which the reader
// expects to be w x h, in chunks of device_feed_chunk(threads).  `threads` host threads read the files, parse the JPEG headers,
// split the scans and decode PNG / PGM frames for chunk k+1 while the main thread packs chunk k into the sequence's pinned staging
// and sends it H2D -> J1 -> J2 on `st`.  J2 writes chunk k's frames to d_out + f0 * h * pitch (their slots of the caller's rows) or,
// with d_out NULL, to a scratch buffer of the chunk's slot.  Once a chunk's status words are back, consume(chunk) runs (it may
// enqueue more work on `st` that reads chunk.frames); the feed stops at the first consume that does not return MDC_OK and returns
// that code.  Frames that fail are never written.  Returns after `st` has drained.
int run_device_feed(const mdc_seq* s, const int* ids, int count, int w, int h, int threads, uint8_t* d_out, size_t pitch, cudaStream_t st,
                    const std::function<int(const FeedChunk&)>& consume, const char* who) {
    const int chunk = device_feed_chunk(threads);
    std::lock_guard<std::mutex> feed_lock(mdc_seq_feed_mutex(s));
    mdc_seq_feed_stage* stage = mdc_seq_device_stage(s);

    std::vector<FeedFrame> frames[2];        // the two slots of the pool
    for (int b = 0; b < 2; ++b) frames[b].resize(static_cast<size_t>(std::min(chunk, count)));
    std::vector<mdc_gray_image> img;         // per worker
    mdc_feed_pool pool(count, chunk, threads, [&](int t, int k, int i) {
        read_feed_frame(s, ids[k * chunk + i], w, h, frames[k & 1][static_cast<size_t>(i)], img[static_cast<size_t>(t)]);
        return true;
    });
    img.resize(static_cast<size_t>(pool.workers()));
    if (pool.start(who) != MDC_OK) return MDC_ERR_IO;
    const int n_chunks = pool.chunks();

    HostBatch batch[2];
    FeedChunk done[2];                // the host side of each slot's chunk, kept after its frame slots are handed to chunk k + 2
    DevSlot dev[2];
    cudaEvent_t ev_status[2] = {nullptr, nullptr}, ev_done[2] = {nullptr, nullptr};
    uint32_t* status_pinned[2] = {nullptr, nullptr};
    int rc = MDC_OK;
    for (int b = 0; b < 2 && rc == MDC_OK; ++b)
        if (cudaEventCreateWithFlags(&ev_status[b], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventCreateWithFlags(&ev_done[b], cudaEventDisableTiming) != cudaSuccess ||
            cudaEventRecord(ev_done[b], st) != cudaSuccess) {
            mdc_set_error("%s: cannot create events", who);
            rc = MDC_ERR_CUDA;
        }
    // chunk k: pack into pinned staging, then H2D -> J1 -> J2 (-> status D2H) on the stream
    auto submit = [&](int k) -> int {
        const int b = k & 1, f0 = k * chunk, n = std::min(chunk, count - f0);
        HostBatch& hb = batch[b];
        hb = HostBatch();
        FeedChunk& fc = done[b];
        fc.f0 = f0;
        fc.n = n;
        fc.status.resize(static_cast<size_t>(n));
        fc.sizes.resize(2 * static_cast<size_t>(n));
        fc.msg.resize(static_cast<size_t>(n));
        std::vector<size_t> at(static_cast<size_t>(n));
        for (int i = 0; i < n; ++i) {
            FeedFrame& ff = frames[b][static_cast<size_t>(i)];
            fc.status[static_cast<size_t>(i)] = ff.status;
            fc.sizes[2 * static_cast<size_t>(i)] = ff.w;
            fc.sizes[2 * static_cast<size_t>(i) + 1] = ff.h;
            fc.msg[static_cast<size_t>(i)].swap(ff.msg);
            at[static_cast<size_t>(i)] = hb.bytes;
            if (ff.status != MDC_OK) {
                hb.add_skipped();
            } else if (ff.jpeg) {
                hb.add_jpeg(*ff.hdr, ff.segs, ff.complete, mdc_seq_name(s, ids[f0 + i]), hb.bytes);
                hb.bytes += ff.segs.empty() ? 0 : ff.segs.back().end - ff.segs.front().begin;
            } else {
                hb.add_raw(hb.bytes);
                hb.bytes += ff.px.size();
            }
        }
        const size_t meta = hb.meta_bytes(), need = meta + HostBatch::align(hb.bytes) + sizeof(uint32_t) * static_cast<size_t>(n);
        // the slot's previous chunk (k - 2) has left the staging buffer and the device buffers behind
        CU_CHECK(cudaEventSynchronize(ev_done[b]));
        if (stage->bytes[b] < need) {
            stage->free_slot(b);
            if (mdc_host_alloc(&stage->pinned[b], need + need / 8) != MDC_OK) return MDC_ERR_CUDA;
            stage->bytes[b] = need + need / 8;
        }
        int r = prepare_slot(hb, dev[b]);
        if (r == MDC_OK && !d_out) r = grow(&dev[b].u8, &dev[b].u8_cap, static_cast<size_t>(chunk) * h * pitch);
        if (r != MDC_OK) return r;
        uint8_t* pin = static_cast<uint8_t*>(stage->pinned[b]);
        hb.write_meta(pin, dev[b].meta);
        for (int i = 0; i < n; ++i) {
            const FeedFrame& ff = frames[b][static_cast<size_t>(i)];
            uint8_t* dst = pin + meta + at[static_cast<size_t>(i)];
            if (ff.status != MDC_OK) continue;
            if (ff.jpeg && !ff.segs.empty()) memcpy(dst, ff.file.data() + ff.segs.front().begin, ff.segs.back().end - ff.segs.front().begin);
            else if (!ff.jpeg) memcpy(dst, ff.px.data(), ff.px.size());
        }
        fc.frames = d_out ? d_out + static_cast<size_t>(f0) * h * pitch : dev[b].u8;
        status_pinned[b] = reinterpret_cast<uint32_t*>(pin + meta + HostBatch::align(hb.bytes));
        r = enqueue_batch(hb, dev[b], pin, pin + meta, w, h, fc.frames, pitch, status_pinned[b], st);
        if (r != MDC_OK) return r;
        CU_CHECK(cudaEventRecord(ev_status[b], st));
        return MDC_OK;
    };
    // chunk k after J1 / J2: the GPU's verdict joins the host's, then the consumer
    auto finish = [&](int k) -> int {
        const int b = k & 1;
        FeedChunk& fc = done[b];
        CU_CHECK(cudaEventSynchronize(ev_status[b]));
        for (int i = 0; i < fc.n; ++i) {
            if (fc.status[static_cast<size_t>(i)] != MDC_OK) continue;
            std::string m = frame_message(status_pinned[b][i], mdc_seq_name(s, ids[fc.f0 + i]), batch[b].incomplete_msg[static_cast<size_t>(i)]);
            if (m.empty()) continue;
            fc.status[static_cast<size_t>(i)] = MDC_ERR_FORMAT;
            fc.sizes[2 * static_cast<size_t>(i)] = fc.sizes[2 * static_cast<size_t>(i) + 1] = 0;
            fc.msg[static_cast<size_t>(i)] = m;
        }
        const int r = consume(fc);
        if (r != MDC_OK) return r;
        CU_CHECK(cudaEventRecord(ev_done[b], st));
        return MDC_OK;
    };
    for (int k = 0; k < n_chunks && rc == MDC_OK; ++k) {
        pool.wait(k);
        rc = submit(k);
        pool.release(k);              // frames[k & 1] is packed: chunk k + 2 may be read into it
        if (rc == MDC_OK && k > 0) rc = finish(k - 1);          // overlaps chunk k's J1 / J2 on the GPU
        if (rc == MDC_OK && k == n_chunks - 1) rc = finish(k);
    }
    const cudaError_t drained = cudaStreamSynchronize(st);
    if (rc == MDC_OK && drained != cudaSuccess) { mdc_set_error("%s: %s", who, cudaGetErrorString(drained)); rc = MDC_ERR_CUDA; }
    for (int b = 0; b < 2; ++b) {
        dev[b].release();
        if (ev_status[b]) cudaEventDestroy(ev_status[b]);
        if (ev_done[b]) cudaEventDestroy(ev_done[b]);
    }
    return rc;
}

}  // namespace

extern "C" int mdc_seq_prepare_device(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, float* const* d_out_levels, int levels,
                                      int threads, mdc_stream stream) {
    return mdc_seq_prepare_device_ex(c, s, first, count, flags, MDC_OUT_F32, reinterpret_cast<void* const*>(d_out_levels), levels, threads, stream);
}

extern "C" int mdc_seq_prepare_device_ex(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, int out_type,
                                         void* const* d_out_levels, int levels, int threads, mdc_stream stream) {
    if (mdc_check_out_type(out_type, "mdc_seq_prepare_device") != MDC_OK) return MDC_ERR_INVALID_ARG;
    int in_w = 0, in_h = 0;
    size_t level_px[MDC_MAX_PYR_LEVELS];
    const int checked = mdc_seq_check_prepare(c, s, first, count, flags, d_out_levels, levels, "mdc_seq_prepare_device", &in_w, &in_h, level_px);
    if (checked != MDC_OK || count == 0) return checked;
    if (threads < 1) threads = mdc_seq_default_threads();
    CU_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    // rows padded to 16 bytes keep K1 on its TMA loader; padded rows exist in rectifying mode only (mdc_prepare_batch_pitched)
    const bool rectify = (flags & MDC_RECTIFY) != 0;
    const size_t pitch = rectify ? (static_cast<size_t>(in_w) + 15) / 16 * 16 : static_cast<size_t>(in_w);
    std::vector<int> ids(static_cast<size_t>(count));
    for (int i = 0; i < count; ++i) ids[static_cast<size_t>(i)] = first + i;
    std::string fail_msg;
    // a frame that failed stops the call before its chunk reaches K1; otherwise K1 into the level buffers
    auto prepare = [&](const FeedChunk& fc) -> int {
        for (int i = 0; i < fc.n; ++i)
            if (fc.status[static_cast<size_t>(i)] != MDC_OK) { fail_msg = fc.msg[static_cast<size_t>(i)]; return MDC_ERR_FORMAT; }
        return mdc_prepare_batch_ex(c, fc.frames, pitch, fc.n, flags, out_type, mdc_seq_chunk_levels(d_out_levels, levels, level_px, out_type, fc.f0).data(),
                                    levels, st);
    };
    const int rc = run_device_feed(s, ids.data(), count, in_w, in_h, threads, nullptr, pitch, st, prepare, "mdc_seq_prepare_device");
    if (rc == MDC_ERR_FORMAT) {
        printf("ERROR: %s\n", fail_msg.c_str());
        mdc_set_error("mdc_seq_prepare_device: %s", fail_msg.c_str());
    }
    return rc;
}

extern "C" int mdc_seq_read_gray8_device(mdc_ctx* c, const mdc_seq* s, const int* ids, int n, int w, int h, uint8_t* d_out, size_t row_pitch,
                                         int* status_host, int* sizes_host, int threads, mdc_stream stream) {
    if (n < 0 || (n > 0 && (!c || !s || !ids || !d_out)) || w < 1 || h < 1 || row_pitch < static_cast<size_t>(w)) {
        mdc_set_error("mdc_seq_read_gray8_device: bad argument");
        return MDC_ERR_INVALID_ARG;
    }
    const int n_files = mdc_seq_num_images(s);
    for (int k = 0; k < n; ++k)
        if (ids[k] < 0 || ids[k] >= n_files) {
            mdc_set_error("mdc_seq_read_gray8_device: frame id %d (ids[%d]) outside the sequence's %d", ids[k], k, n_files);
            return MDC_ERR_INVALID_ARG;
        }
    if (n == 0) return MDC_OK;
    if (threads < 1) threads = mdc_seq_default_threads();
    CU_CHECK(cudaSetDevice(mdc_ctx_device_ordinal(c)));
    cudaStream_t st = stream ? static_cast<cudaStream_t>(stream) : static_cast<cudaStream_t>(mdc_ctx_stream_handle(c));
    int first_bad = -1;
    std::string first_msg;
    // every frame's outcome is recorded; J2 has already written the rows of the frames that read
    auto record = [&](const FeedChunk& fc) -> int {
        for (int i = 0; i < fc.n; ++i) {
            const int k = fc.f0 + i;
            if (status_host) status_host[k] = fc.status[static_cast<size_t>(i)];
            if (sizes_host) { sizes_host[2 * k] = fc.sizes[2 * static_cast<size_t>(i)]; sizes_host[2 * k + 1] = fc.sizes[2 * static_cast<size_t>(i) + 1]; }
            if (fc.status[static_cast<size_t>(i)] != MDC_OK && first_bad < 0) { first_bad = k; first_msg = fc.msg[static_cast<size_t>(i)]; }
        }
        return MDC_OK;
    };
    const int rc = run_device_feed(s, ids, n, w, h, threads, d_out, row_pitch, st, record, "mdc_seq_read_gray8_device");
    if (rc != MDC_OK) return rc;
    if (first_bad >= 0) { mdc_set_error("%s", first_msg.c_str()); return MDC_ERR_FORMAT; }
    return MDC_OK;
}
