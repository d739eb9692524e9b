// Internal declarations shared by the host-model, C-ABI and kernel translation units.
#pragma once
#include <stdint.h>
#include <mutex>
#include <string>
#include <vector>

#include "mdc_b200.h"

// Thread-local error message behind mdc_last_error().
void mdc_set_error(const char* fmt, ...);

// Output types of the prepare calls (MDC_OUT_*): element size, and the check every _ex entry point makes first (no device needed):
// MDC_OK, or MDC_ERR_INVALID_ARG with "<where>: unknown output type <t>".
inline size_t mdc_out_elem_size(int out_type) { return out_type == MDC_OUT_F16 ? 2 : out_type == MDC_OUT_U8 ? 1 : 4; }
int mdc_check_out_type(int out_type, const char* where);

// Host-side state of the FOV rectifier (the members of the reference's UndistorterFOV,
// FOVUndistorter.h:85-95, plus bookkeeping).
struct mdc_fov {
    bool valid = false;
    bool dims_known = false;     // lines 1-2 of camera.txt parsed (the reference prints them then)
    bool has_black = false;      // some output pixels have no source (remap = -1)
    int float_math = 0;
    float in_calib[5] = {0, 0, 0, 0, 0};
    float out_calib[5] = {0, 0, 0, 0, 0};
    int in_w = 0, in_h = 0, out_w = 0, out_h = 0;
    float k_rect[9] = {0}, k_org[9] = {0};
    std::vector<float> remap_x, remap_y;
};

// Host-side state of the photometric un-mapper (PhotometricUndistorter.h:47-53).
struct mdc_photo {
    bool valid_gamma = false, valid_vignette = false;
    int w = 0, h = 0;
    float G[256], GInv[256];
    std::vector<float> vmap, vinv;   // allocated (w*h) once gamma parsed, like the reference (:121-122)
};

// Decoded grey image (PNG 8/16-bit grey, or binary PGM).  depth is 8 or 16; 16-bit pixels
// are stored in host byte order.  Returns false (with mdc_set_error) if unreadable/unsupported.
struct mdc_gray_image {
    int rows = 0, cols = 0, depth = 0;
    std::vector<uint8_t> px;
};
bool mdc_read_gray_image(const std::string& path, mdc_gray_image* out);
bool mdc_read_file(const std::string& path, std::vector<uint8_t>* file);                                        // whole file, undecoded
bool mdc_decode_gray_image(const std::vector<uint8_t>& file, const std::string& name, mdc_gray_image* out);      // same, from memory
bool mdc_decode_jpeg_gray(const std::vector<uint8_t>& file, const std::string& name, mdc_gray_image* out);       // baseline JPEG -> luminance (mdc_jpeg.cpp)

// Table builders (strict IEEE float; see mdc_host_models.cpp).
void mdc_fov_build(mdc_fov* f, int mode, const float out_calib_in[5]);
struct mdc_distort_constants { float ocx, ocy, ofx, ofy, d2t, omega, fx, fy, cx, cy; };
void mdc_fov_distort_constants(const mdc_fov* f, mdc_distort_constants* k);
void mdc_fov_distort(const mdc_fov* f, float* xs, float* ys, int n);
void mdc_vc_plane_matrix(const double H[9], int gw, int gh, float facw, float fach, float HK[9]);      // vignetteCalib's H * K_p2idx^-1
bool mdc_photo_set_gamma(mdc_photo* p, const float raw[256]);
void mdc_photo_set_vignette(mdc_photo* p, const void* pixels, int depth);

// Context accessors for translation units that do not see the context's layout (mdc_vignette_calib.cu).
int mdc_ctx_device_ordinal(const mdc_ctx* c);
void* mdc_ctx_stream_handle(mdc_ctx* c);          // the context's own cudaStream_t
void mdc_ctx_add_launches(mdc_ctx* c, int n);
int mdc_ctx_scratch_pool(mdc_ctx* c, void** pool);      // the context's cudaMemPool_t for stream-ordered scratch, kept warm between calls
void mdc_ctx_geometry(const mdc_ctx* c, int* in_w, int* in_h, int* out_w, int* out_h);

// Sequence internals used by the GPU-decoding feed (mdc_jpeg_gpu.cu).
struct mdc_seq_feed_stage {      // a feed's two pinned staging slots, kept between calls
    void* pinned[2] = {nullptr, nullptr};
    size_t bytes[2] = {0, 0};
    void free_slot(int b) { mdc_host_free(pinned[b]); pinned[b] = nullptr; bytes[b] = 0; }
};
bool mdc_seq_read_file(const mdc_seq* s, int id, std::vector<uint8_t>* file);      // frame id's file bytes (folder file or zip entry)
std::mutex& mdc_seq_feed_mutex(const mdc_seq* s);                                   // one feed at a time per sequence object
mdc_seq_feed_stage* mdc_seq_device_stage(const mdc_seq* s);
// 8-bit pixels of a decoded frame, as mdc_seq_read_gray8 returns them: a 16-bit image keeps its high byte (img.px is taken when 8-bit)
void mdc_gray_to_u8(mdc_gray_image& img, std::vector<uint8_t>* px);
// "expected image dimensions <w> x <h>; found <fw> x <fh> (<what>)", BenchmarkDatasetReader.h:194-199
std::string mdc_dims_message(int w, int h, int fw, int fh, const std::string& what);
// The argument checks of mdc_seq_prepare(_ex) and mdc_seq_prepare_device(_ex), "<who>: " messages: first those that need no context
// (sequence and level array, frame range, level count), then the context's input geometry, then a NULL level that has pixels.  On
// MDC_OK, *in_w x *in_h is the input size and level_px[l] the pixels per frame of level l of getImage's result.
int mdc_seq_check_prepare(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, void* const* out_levels, int levels,
                          const char* who, int* in_w, int* in_h, size_t level_px[MDC_MAX_PYR_LEVELS]);
// The level pointers of the chunk that starts at frame f0 of a call's output (a NULL level stays NULL).
std::vector<void*> mdc_seq_chunk_levels(void* const* out_levels, int levels, const size_t* level_px, int out_type, int f0);
// The decode-ahead host feed behind mdc_seq_prepare and mdc_seq_prepare_ex (mdc_sequence.cpp).  Each decoded chunk goes to `prepare`
// (mdc_prepare_batch_host_ex's signature), so that the sequence reader calls nothing of the GPU side but what its caller hands it.
typedef int (*mdc_host_prepare_fn)(mdc_ctx* c, const uint8_t* frames, int n_frames, unsigned flags, int out_type, void* const* out_levels,
                                   int levels);
int mdc_seq_prepare_feed(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, int out_type, void* const* h_out_levels,
                         int levels, int threads, mdc_host_prepare_fn prepare);
int mdc_seq_default_threads();                                                      // threads = 0 of the feeds
