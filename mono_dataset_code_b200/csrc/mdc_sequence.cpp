// Sequence reader: the host side of DatasetReader (BenchmarkDatasetReader.h:83-147, :247-345) without OpenCV / libzip, plus the
// decode-ahead feed of the GPU path (SURVEY.md §8f N1).
//
//   mdc_seq_open      images/ folder (sorted) or, if that is empty, images.zip (central directory, sorted names); times.txt
//   mdc_seq_read_gray8 getImageRaw_internal with CV_LOAD_IMAGE_GRAYSCALE: 8/16-bit grey PNG (16 -> 8 bit by dropping the low byte, as
//                     OpenCV's reader does), binary PGM, baseline JPEG (mdc_jpeg.cpp) - the same bytes as cv::imread returns.
//   mdc_seq_prepare   getImage for a range of frames: the decode-ahead pool (mdc_feed.h) decodes chunk k+1 (two frames per thread,
//                     16..256 frames) into pinned memory while chunk k goes through mdc_prepare_batch_host (H2D, K1, D2H).
//
// The zip reader handles what `zip` / Python's zipfile / the TUM archives produce: stored and deflated entries, no encryption,
// no zip64 (archives < 4 GB, < 65535 entries), CRC-32 verified.
#include <algorithm>
#include <exception>
#include <cstdio>
#include <cstring>
#include <dirent.h>
#include <fstream>
#include <mutex>
#include <string>
#include <sched.h>
#include <thread>
#include <vector>

#include <fcntl.h>
#include <sys/stat.h>
#include <unistd.h>
#include <zlib.h>

#include "mdc_b200.h"
#include "mdc_feed.h"
#include "mdc_internal.h"

namespace {

struct ZipEntry { std::string name; uint16_t method; uint32_t crc, comp_size, size, local_offset; };

uint16_t le16(const uint8_t* p) { return static_cast<uint16_t>(p[0] | (p[1] << 8)); }
uint32_t le32(const uint8_t* p) { return static_cast<uint32_t>(p[0]) | (static_cast<uint32_t>(p[1]) << 8) | (static_cast<uint32_t>(p[2]) << 16) | (static_cast<uint32_t>(p[3]) << 24); }

bool pread_all(int fd, void* dst, size_t n, off_t off) {
    uint8_t* p = static_cast<uint8_t*>(dst);
    while (n) {
        const ssize_t got = pread(fd, p, n, off);
        if (got <= 0) return false;
        p += got; n -= static_cast<size_t>(got); off += got;
    }
    return true;
}

}  // namespace

struct mdc_seq {
    std::string path;                  // with trailing '/'
    bool zipped = false;
    int zip_fd = -1;
    uint64_t zip_bytes = 0;            // size of the archive: no entry can be larger (compressed)
    std::vector<std::string> files;    // full paths (folder) or entry names (zip), sorted
    std::vector<ZipEntry> entries;     // parallel to files when zipped
    std::vector<double> timestamps;
    std::vector<float> exposures;
    // pinned staging of the host feed (mdc_seq_prepare) and of the device feed (mdc_seq_prepare_device, mdc_jpeg_gpu.cu), kept
    // between calls (pinning hundreds of MB costs tens of milliseconds — more than decoding the frames of a short call); one feed at
    // a time per sequence object
    mutable mdc_seq_feed_stage host_stage, device_stage;
    mutable std::mutex feed_mutex;
};

namespace {

// getdir(), BenchmarkDatasetReader.h:44-78: every entry except "." and "..", sorted, prefixed with the directory
int list_dir(std::string dir, std::vector<std::string>* files) {
    DIR* dp = opendir(dir.c_str());
    if (!dp) return -1;
    while (struct dirent* e = readdir(dp)) {
        const std::string name(e->d_name);
        if (name != "." && name != "..") files->push_back(name);
    }
    closedir(dp);
    std::sort(files->begin(), files->end());
    if (dir.empty() || dir[dir.size() - 1] != '/') dir += "/";
    for (size_t i = 0; i < files->size(); ++i) (*files)[i] = dir + (*files)[i];
    return static_cast<int>(files->size());
}

bool read_zip_directory(mdc_seq* s, const std::string& archive) {
    s->zip_fd = open(archive.c_str(), O_RDONLY);
    if (s->zip_fd < 0) { mdc_set_error("cannot open archive %s", archive.c_str()); return false; }
    struct stat st;
    if (fstat(s->zip_fd, &st) != 0 || st.st_size < 22) { mdc_set_error("%s: not a zip archive", archive.c_str()); return false; }
    s->zip_bytes = static_cast<uint64_t>(st.st_size);
    // end-of-central-directory record: last 22 .. 22+65535 bytes
    const size_t tail = static_cast<size_t>(std::min<off_t>(st.st_size, 22 + 65535));
    std::vector<uint8_t> buf(tail);
    if (!pread_all(s->zip_fd, buf.data(), tail, st.st_size - static_cast<off_t>(tail))) { mdc_set_error("%s: read error", archive.c_str()); return false; }
    ssize_t eocd = -1;
    for (ssize_t i = static_cast<ssize_t>(tail) - 22; i >= 0; --i)
        if (le32(&buf[i]) == 0x06054b50u) { eocd = i; break; }
    if (eocd < 0) { mdc_set_error("%s: no zip end-of-central-directory record", archive.c_str()); return false; }
    const uint16_t n_entries = le16(&buf[eocd + 10]);
    const uint32_t cd_size = le32(&buf[eocd + 12]), cd_off = le32(&buf[eocd + 16]);
    if (n_entries == 0xffff || cd_off == 0xffffffffu) { mdc_set_error("%s: zip64 archives are not supported", archive.c_str()); return false; }
    // plausibility before anything is sized from the (untrusted) record: the directory lies inside the archive and holds its entries
    if (static_cast<uint64_t>(cd_off) + cd_size > s->zip_bytes || static_cast<uint64_t>(n_entries) * 46u > cd_size) {
        mdc_set_error("%s: corrupt central directory", archive.c_str());
        return false;
    }
    std::vector<uint8_t> cd(cd_size);
    if (cd_size && !pread_all(s->zip_fd, cd.data(), cd_size, cd_off)) { mdc_set_error("%s: truncated central directory", archive.c_str()); return false; }
    size_t pos = 0;
    std::vector<ZipEntry> all;
    for (int k = 0; k < n_entries; ++k) {
        if (pos + 46 > cd.size() || le32(&cd[pos]) != 0x02014b50u) { mdc_set_error("%s: corrupt central directory", archive.c_str()); return false; }
        ZipEntry e;
        const uint16_t flags = le16(&cd[pos + 8]);
        e.method = le16(&cd[pos + 10]);
        e.crc = le32(&cd[pos + 16]);
        e.comp_size = le32(&cd[pos + 20]);
        e.size = le32(&cd[pos + 24]);
        const uint16_t name_len = le16(&cd[pos + 28]), extra_len = le16(&cd[pos + 30]), comment_len = le16(&cd[pos + 32]);
        e.local_offset = le32(&cd[pos + 42]);
        if (pos + 46 + name_len > cd.size()) { mdc_set_error("%s: corrupt central directory", archive.c_str()); return false; }
        e.name.assign(reinterpret_cast<const char*>(&cd[pos + 46]), name_len);
        pos += 46u + name_len + extra_len + comment_len;
        if (flags & 1) { mdc_set_error("%s: encrypted entry %s", archive.c_str(), e.name.c_str()); return false; }
        if (e.name == "." || e.name == "..") continue;          // :126
        all.push_back(e);
    }
    std::sort(all.begin(), all.end(), [](const ZipEntry& a, const ZipEntry& b) { return a.name < b.name; });      // :131
    s->entries.swap(all);
    for (size_t i = 0; i < s->entries.size(); ++i) s->files.push_back(s->entries[i].name);
    printf("got %d entries and %d files from zipfile!\n", static_cast<int>(n_entries), static_cast<int>(s->files.size()));
    return true;
}

bool read_zip_entry(const mdc_seq* s, const ZipEntry& e, std::vector<uint8_t>* out) {
    uint8_t lh[30];
    if (!pread_all(s->zip_fd, lh, 30, e.local_offset) || le32(lh) != 0x04034b50u) { mdc_set_error("%s: bad local header", e.name.c_str()); return false; }
    const off_t data = static_cast<off_t>(e.local_offset) + 30 + le16(lh + 26) + le16(lh + 28);
    // a corrupt directory must not make us allocate gigabytes: entries cannot be larger than the archive (deflate expands < 1100x)
    if (e.comp_size > s->zip_bytes || static_cast<uint64_t>(data) + e.comp_size > s->zip_bytes || (e.size >> 10) > e.comp_size + 1024u) { mdc_set_error("%s: implausible entry size", e.name.c_str()); return false; }
    out->resize(e.size);
    if (e.method == 0) {
        if (e.comp_size != e.size || (e.size && !pread_all(s->zip_fd, out->data(), e.size, data))) { mdc_set_error("%s: truncated stored entry", e.name.c_str()); return false; }
    } else if (e.method == 8) {
        std::vector<uint8_t> comp(e.comp_size);
        if (e.comp_size && !pread_all(s->zip_fd, comp.data(), e.comp_size, data)) { mdc_set_error("%s: truncated deflated entry", e.name.c_str()); return false; }
        z_stream z;
        memset(&z, 0, sizeof z);
        if (inflateInit2(&z, -MAX_WBITS) != Z_OK) { mdc_set_error("%s: zlib init failed", e.name.c_str()); return false; }
        z.next_in = comp.data(); z.avail_in = e.comp_size;
        z.next_out = out->data(); z.avail_out = e.size;
        const int rc = inflate(&z, Z_FINISH);
        const bool ok = (rc == Z_STREAM_END) && z.total_out == e.size;
        inflateEnd(&z);
        if (!ok) { mdc_set_error("%s: inflate failed (%d)", e.name.c_str(), rc); return false; }
    } else {
        mdc_set_error("%s: unsupported zip compression method %d", e.name.c_str(), static_cast<int>(e.method));
        return false;
    }
    if (static_cast<uint32_t>(crc32(0L, out->data(), e.size)) != e.crc) { mdc_set_error("%s: CRC mismatch", e.name.c_str()); return false; }
    return true;
}

// loadTimestamps(), BenchmarkDatasetReader.h:279-330: "id stamp [exposure]" lines; a count mismatch zeroes everything
void load_times(mdc_seq* s) {
    std::ifstream tr((s->path + "times.txt").c_str());
    std::string line;
    while (std::getline(tr, line)) {
        int id; double stamp; float exposure = 0;
        const int got = sscanf(line.c_str(), "%d %lf %f", &id, &stamp, &exposure);
        if (got == 3) { s->timestamps.push_back(stamp); s->exposures.push_back(exposure); }
        else if (got == 2) { s->timestamps.push_back(stamp); s->exposures.push_back(0); }
    }
    if (s->exposures.size() != s->files.size()) {
        printf("DatasetReader: Mismatch between number of images and number of timestamps / exposure times. Set all to zero.");
        s->timestamps.assign(s->files.size(), 0.0);
        s->exposures.assign(s->files.size(), 0.0f);
    }
}

// 8-bit grey pixels of frame `id` (decoded)
bool read_gray8_unguarded(const mdc_seq* s, int id, std::vector<uint8_t>* px, int* w, int* h) {
    // per-thread scratch (file bytes, decoded image): no multi-megabyte allocation per frame, see mdc_jpeg.cpp
    static thread_local mdc_gray_image img;
    static thread_local std::vector<uint8_t> file;
    if (s->zipped) {
        if (!read_zip_entry(s, s->entries[static_cast<size_t>(id)], &file)) return false;
        if (!mdc_decode_gray_image(file, s->files[static_cast<size_t>(id)], &img)) return false;
    } else if (!mdc_read_gray_image(s->files[static_cast<size_t>(id)], &img)) {
        return false;
    }
    *w = img.cols; *h = img.rows;
    mdc_gray_to_u8(img, px);
    return true;
}
// no exception (bad_alloc / length_error on a hostile file) may cross the C ABI or a std::async worker
bool read_gray8(const mdc_seq* s, int id, std::vector<uint8_t>* px, int* w, int* h) {
    try {
        return read_gray8_unguarded(s, id, px, w, h);
    } catch (const std::exception& e) {
        mdc_set_error("%s: cannot read (%s)", s->files[static_cast<size_t>(id)].c_str(), e.what());
        return false;
    }
}

}  // namespace

bool mdc_seq_read_file(const mdc_seq* s, int id, std::vector<uint8_t>* file) {
    try {
        if (s->zipped) return read_zip_entry(s, s->entries[static_cast<size_t>(id)], file);
        return mdc_read_file(s->files[static_cast<size_t>(id)], file);
    } catch (const std::exception& e) {
        mdc_set_error("%s: cannot read (%s)", s->files[static_cast<size_t>(id)].c_str(), e.what());
        return false;
    }
}
void mdc_gray_to_u8(mdc_gray_image& img, std::vector<uint8_t>* px) {
    if (img.depth == 8) { px->swap(img.px); return; }
    const size_t n = static_cast<size_t>(img.rows) * img.cols;
    px->resize(n);
    const uint16_t* src = reinterpret_cast<const uint16_t*>(img.px.data());
    for (size_t i = 0; i < n; ++i) (*px)[i] = static_cast<uint8_t>(src[i] >> 8);
}
std::string mdc_dims_message(int w, int h, int fw, int fh, const std::string& what) {
    char msg[256];
    snprintf(msg, sizeof msg, "expected image dimensions %d x %d; found %d x %d (%s)", w, h, fw, fh, what.c_str());
    return msg;
}
std::mutex& mdc_seq_feed_mutex(const mdc_seq* s) { return s->feed_mutex; }
mdc_seq_feed_stage* mdc_seq_device_stage(const mdc_seq* s) { return &s->device_stage; }

extern "C" int mdc_seq_open(const char* folder, mdc_seq** out) {
    if (!folder || !out) { mdc_set_error("mdc_seq_open: bad argument"); return MDC_ERR_INVALID_ARG; }
    *out = nullptr;
    mdc_seq* s = nullptr;
    try {
    s = new mdc_seq();
    s->path = folder;
    if (!s->path.empty() && s->path[s->path.size() - 1] != '/') s->path += "/";
    list_dir(s->path + "images/", &s->files);
    if (!s->files.empty()) {
        printf("Load Dataset %s: found %d files in folder /images; assuming that all images are there.\n", s->path.c_str(), static_cast<int>(s->files.size()));
    } else {
        printf("Load Dataset %s: found no in folder /images; assuming that images are zipped.\n", s->path.c_str());
        s->zipped = true;
        if (!read_zip_directory(s, s->path + "images.zip")) {
            printf("ERROR reading archive %s!\n", (s->path + "images.zip").c_str());      // the reference exits here (:117-121)
            if (s->zip_fd >= 0) close(s->zip_fd);
            delete s;
            return MDC_ERR_IO;
        }
    }
    load_times(s);
    printf("Dataset %s: Got %d files!\n", s->path.c_str(), static_cast<int>(s->files.size()));
    } catch (const std::exception& e) {
        mdc_set_error("mdc_seq_open(%s): %s", folder, e.what());
        if (s) { if (s->zip_fd >= 0) close(s->zip_fd); delete s; }
        return MDC_ERR_IO;
    }
    *out = s;
    return MDC_OK;
}

extern "C" void mdc_seq_close(mdc_seq* s) {
    if (!s) return;
    for (int b = 0; b < 2; ++b) { s->host_stage.free_slot(b); s->device_stage.free_slot(b); }
    if (s->zip_fd >= 0) close(s->zip_fd);
    delete s;
}

extern "C" int mdc_seq_num_images(const mdc_seq* s) { return s ? static_cast<int>(s->files.size()) : 0; }
extern "C" int mdc_seq_is_zipped(const mdc_seq* s) { return s && s->zipped; }
extern "C" const char* mdc_seq_name(const mdc_seq* s, int id) {
    return (s && id >= 0 && id < static_cast<int>(s->files.size())) ? s->files[static_cast<size_t>(id)].c_str() : nullptr;
}
// getTimestamp / getExposure, BenchmarkDatasetReader.h:171-186: 0 for an id out of range
extern "C" double mdc_seq_timestamp(const mdc_seq* s, int id) {
    return (s && id >= 0 && id < static_cast<int>(s->timestamps.size())) ? s->timestamps[static_cast<size_t>(id)] : 0.0;
}
extern "C" float mdc_seq_exposure(const mdc_seq* s, int id) {
    return (s && id >= 0 && id < static_cast<int>(s->exposures.size())) ? s->exposures[static_cast<size_t>(id)] : 0.0f;
}

extern "C" int mdc_seq_read_gray8(const mdc_seq* s, int id, uint8_t* out, size_t capacity, int* w, int* h) {
    if (!s || id < 0 || id >= static_cast<int>(s->files.size()) || !w || !h) { mdc_set_error("mdc_seq_read_gray8: bad argument"); return MDC_ERR_INVALID_ARG; }
    std::vector<uint8_t> px;
    if (!read_gray8(s, id, &px, w, h)) return MDC_ERR_FORMAT;
    if (out) {
        if (capacity < px.size()) { mdc_set_error("mdc_seq_read_gray8: buffer of %zu bytes for a %d x %d image", capacity, *w, *h); return MDC_ERR_INVALID_ARG; }
        memcpy(out, px.data(), px.size());
    }
    return MDC_OK;
}

// threads = 0: as many decode threads as the process may keep busy — the CPUs it is allowed to run on, capped by the container's
// CPU-time quota (cgroup v2 cpu.max) where there is one: more busy threads than the quota only get throttled
int mdc_seq_default_threads() {
    int n = static_cast<int>(std::max(1u, std::thread::hardware_concurrency()));
    cpu_set_t set;
    if (sched_getaffinity(0, sizeof set, &set) == 0) n = std::max(1, std::min(n, CPU_COUNT(&set)));
    if (FILE* f = fopen("/sys/fs/cgroup/cpu.max", "r")) {
        long long quota = 0, period = 0;
        if (fscanf(f, "%lld %lld", &quota, &period) == 2 && quota > 0 && period > 0) n = std::max(1, std::min<int>(n, static_cast<int>(quota / period)));
        fclose(f);
    }
    return n;
}

int mdc_seq_check_prepare(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, void* const* out_levels, int levels,
                          const char* who, int* in_w, int* in_h, size_t level_px[MDC_MAX_PYR_LEVELS]) {
    if (!s || !out_levels) { mdc_set_error("%s: bad argument", who); return MDC_ERR_INVALID_ARG; }
    const int n_files = static_cast<int>(s->files.size());
    if (first < 0 || count < 0 || first > n_files || count > n_files - first) {      // first + count can overflow
        mdc_set_error("%s: frames first = %d, count = %d outside the sequence's %d", who, first, count, n_files);
        return MDC_ERR_INVALID_ARG;
    }
    if (levels < 1 || levels > MDC_MAX_PYR_LEVELS) {
        mdc_set_error("%s: %d pyramid levels (1..%d)", who, levels, MDC_MAX_PYR_LEVELS);
        return MDC_ERR_INVALID_ARG;
    }
    if (!c) { mdc_set_error("%s: bad argument", who); return MDC_ERR_INVALID_ARG; }
    int out_w = 0, out_h = 0;
    mdc_ctx_geometry(c, in_w, in_h, &out_w, &out_h);
    if (*in_w < 1 || *in_h < 1) { mdc_set_error("%s: context has no image geometry", who); return MDC_ERR_INVALID_OBJECT; }
    const bool rectify = (flags & MDC_RECTIFY) != 0;
    for (int l = 0; l < levels; ++l) {      // level l of getImage's result: (w >> l) x (h >> l), mdc_prepare_batch
        level_px[l] = static_cast<size_t>((rectify ? out_w : *in_w) >> l) * static_cast<size_t>((rectify ? out_h : *in_h) >> l);
        if (!out_levels[l] && level_px[l] > 0) {      // a level without pixels may be NULL, as for mdc_prepare_batch
            mdc_set_error("%s: output level %d is NULL", who, l);
            return MDC_ERR_INVALID_ARG;
        }
    }
    return MDC_OK;
}

std::vector<void*> mdc_seq_chunk_levels(void* const* out_levels, int levels, const size_t* level_px, int out_type, int f0) {
    std::vector<void*> outs(static_cast<size_t>(levels));
    const size_t esize = mdc_out_elem_size(out_type);
    for (int l = 0; l < levels; ++l)
        outs[static_cast<size_t>(l)] = out_levels[l] ? static_cast<uint8_t*>(out_levels[l]) + static_cast<size_t>(f0) * level_px[l] * esize : nullptr;
    return outs;
}

// getImage(id, ...) for ids [first, first+count): decode ahead on `threads` host threads, prepare on the GPU chunk by chunk.
namespace {
int prepare_host_f32(mdc_ctx* c, const uint8_t* frames, int n_frames, unsigned flags, int, void* const* out_levels, int levels) {
    return mdc_prepare_batch_host(c, frames, n_frames, flags, reinterpret_cast<float* const*>(out_levels), levels);
}
}  // namespace

extern "C" int mdc_seq_prepare(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, float* const* h_out_levels, int levels,
                               int threads) {
    return mdc_seq_prepare_feed(c, s, first, count, flags, MDC_OUT_F32, reinterpret_cast<void* const*>(h_out_levels), levels, threads,
                                prepare_host_f32);
}

// mdc_seq_prepare(_ex): out_type is already checked (mdc_seq_prepare_ex, mdc_capi.cu); `prepare` takes each decoded chunk.
int mdc_seq_prepare_feed(mdc_ctx* c, const mdc_seq* s, int first, int count, unsigned flags, int out_type, void* const* h_out_levels,
                         int levels, int threads, mdc_host_prepare_fn prepare) {
    int in_w = 0, in_h = 0;
    size_t level_px[MDC_MAX_PYR_LEVELS];
    const int checked = mdc_seq_check_prepare(c, s, first, count, flags, h_out_levels, levels, "mdc_seq_prepare", &in_w, &in_h, level_px);
    if (checked != MDC_OK || count == 0) return checked;
    if (threads < 1) threads = mdc_seq_default_threads();
    // a chunk is what the GPU side takes at a time: two frames per decode thread, small enough that the un-overlapped head (first
    // decode) and tail (last H2D / K1 / D2H) of a call stay short
    const int chunk = std::min(256, std::max(16, 2 * threads));
    std::lock_guard<std::mutex> feed_lock(s->feed_mutex);
    const size_t n_in = static_cast<size_t>(in_w) * in_h, need = static_cast<size_t>(chunk) * n_in;
    mdc_seq_feed_stage& stage = s->host_stage;
    if (stage.bytes[0] < need) {      // both slots have one size
        for (int b = 0; b < 2; ++b) stage.free_slot(b);
        for (int b = 0; b < 2; ++b)
            if (mdc_host_alloc(&stage.pinned[b], need) != MDC_OK) { stage.free_slot(0); stage.pinned[1] = nullptr; return MDC_ERR_CUDA; }
        stage.bytes[0] = stage.bytes[1] = need;
    }

    // chunk k is decoded into stage slot k & 1 while chunk k - 1 is prepared.  A frame's error is kept per frame (each frame is read
    // by one worker): an error in chunk k+1 must not stop the call before chunk k, which decoded fine, has been prepared (the
    // reference prepares every frame before the bad one).  A worker takes no further frame of a chunk after an error in it.
    std::vector<std::string> frame_error(static_cast<size_t>(count));
    std::vector<std::vector<uint8_t>> px;      // per worker
    mdc_feed_pool pool(count, chunk, threads, [&](int t, int k, int i) {
        const int f = k * chunk + i;
        std::vector<uint8_t>& p = px[static_cast<size_t>(t)];
        std::string& err = frame_error[static_cast<size_t>(f)];
        int w = 0, h = 0;
        if (!read_gray8(s, first + f, &p, &w, &h)) err = mdc_last_error();
        else if (w != in_w || h != in_h) err = mdc_dims_message(in_w, in_h, w, h, "image " + s->files[static_cast<size_t>(first + f)]);
        else memcpy(static_cast<uint8_t*>(stage.pinned[k & 1]) + static_cast<size_t>(i) * n_in, p.data(), n_in);
        return err.empty();
    });
    px.resize(static_cast<size_t>(pool.workers()));
    if (pool.start("mdc_seq_prepare") != MDC_OK) return MDC_ERR_IO;
    for (int k = 0; k < pool.chunks(); ++k) {
        pool.wait(k);
        const int f0 = k * chunk, n = std::min(chunk, count - f0);
        const auto chunk_end = frame_error.begin() + f0 + n;
        const auto bad = std::find_if(chunk_end - n, chunk_end, [](const std::string& e) { return !e.empty(); });      // its lowest bad frame
        if (bad != chunk_end) {
            printf("ERROR: %s\n", bad->c_str());
            mdc_set_error("mdc_seq_prepare: %s", bad->c_str());
            return MDC_ERR_FORMAT;
        }
        const int rc = prepare(c, static_cast<const uint8_t*>(stage.pinned[k & 1]), n, flags, out_type,
                               mdc_seq_chunk_levels(h_out_levels, levels, level_px, out_type, f0).data(), levels);      // returns after the D2H copy
        if (rc != MDC_OK) return rc;
        pool.release(k);
    }
    return MDC_OK;
}
