// Sequence reader: the host side of DatasetReader (BenchmarkDatasetReader.h:83-147, :247-345) without OpenCV / libzip, plus the
// decode-ahead feed of the GPU path (SURVEY.md §8f N1).
//
//   mdc_seq_open      images/ folder (sorted) or, if that is empty, images.zip (central directory, sorted names); times.txt
//   mdc_seq_read_gray8 getImageRaw_internal with CV_LOAD_IMAGE_GRAYSCALE: 8/16-bit grey PNG (16 -> 8 bit by dropping the low byte, as
//                     OpenCV's reader does), binary PGM, baseline JPEG (mdc_jpeg.cpp) - the same bytes as cv::imread returns.
//   mdc_seq_prepare   getImage for a range of frames: worker threads decode chunk k+1 (two frames per thread, 16..256 frames) into
//                     pinned memory while chunk k goes through mdc_prepare_batch_host (H2D, fused kernel, D2H on three streams).
//
// The zip reader handles what `zip` / Python's zipfile / the TUM archives produce: stored and deflated entries, no encryption,
// no zip64 (archives < 4 GB, < 65535 entries), CRC-32 verified.
#include <algorithm>
#include <atomic>
#include <exception>
#include <cstdio>
#include <cstring>
#include <dirent.h>
#include <fstream>
#include <condition_variable>
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
    // pinned staging buffers of the decode-ahead feed, kept between mdc_seq_prepare calls (pinning hundreds of MB costs tens of
    // milliseconds — more than decoding the frames of a short call); one feed at a time per sequence object
    mutable void* stage[2] = {nullptr, nullptr};
    mutable size_t stage_bytes = 0;
    mutable std::mutex feed_mutex;
    mutable mdc_seq_feed_stage device_stage;      // the same for mdc_seq_prepare_device (mdc_jpeg_gpu.cu)
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

// 8-bit grey pixels of frame `id` (decoded); 16-bit sources keep the high byte
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
    const size_t n = static_cast<size_t>(img.rows) * img.cols;
    *w = img.cols; *h = img.rows;
    if (img.depth == 8) { px->swap(img.px); return true; }
    px->resize(n);
    const uint16_t* src = reinterpret_cast<const uint16_t*>(img.px.data());
    for (size_t i = 0; i < n; ++i) (*px)[i] = static_cast<uint8_t>(src[i] >> 8);
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
    for (int b = 0; b < 2; ++b) if (s->stage[b]) mdc_host_free(s->stage[b]);
    for (int b = 0; b < 2; ++b) if (s->device_stage.pinned[b]) mdc_host_free(s->device_stage.pinned[b]);
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
    // Everything that does not depend on the context is checked first, and all of it before any staging or thread work.  The range
    // test is written so that it cannot overflow (first + count can).
    if (!s || !h_out_levels) { mdc_set_error("mdc_seq_prepare: bad argument"); return MDC_ERR_INVALID_ARG; }
    const int n_files = static_cast<int>(s->files.size());
    if (first < 0 || count < 0 || first > n_files || count > n_files - first) {
        mdc_set_error("mdc_seq_prepare: frames first = %d, count = %d outside the sequence's %d", first, count, n_files);
        return MDC_ERR_INVALID_ARG;
    }
    if (levels < 1 || levels > MDC_MAX_PYR_LEVELS) {
        mdc_set_error("mdc_seq_prepare: %d pyramid levels (1..%d)", levels, MDC_MAX_PYR_LEVELS);
        return MDC_ERR_INVALID_ARG;
    }
    if (!c) { mdc_set_error("mdc_seq_prepare: bad argument"); return MDC_ERR_INVALID_ARG; }
    int in_w = 0, in_h = 0, out_w = 0, out_h = 0;
    mdc_ctx_geometry(c, &in_w, &in_h, &out_w, &out_h);
    if (in_w < 1 || in_h < 1) { mdc_set_error("mdc_seq_prepare: context has no image geometry"); return MDC_ERR_INVALID_OBJECT; }
    const size_t n_in = static_cast<size_t>(in_w) * in_h;
    const bool rectify = (flags & MDC_RECTIFY) != 0;
    std::vector<size_t> level_px(static_cast<size_t>(levels));
    for (int l = 0; l < levels; ++l) {      // level l of getImage's result: (w >> l) x (h >> l), mdc_prepare_batch
        level_px[static_cast<size_t>(l)] = static_cast<size_t>((rectify ? out_w : in_w) >> l) * static_cast<size_t>((rectify ? out_h : in_h) >> l);
        if (!h_out_levels[l] && level_px[static_cast<size_t>(l)] > 0) {      // a level without pixels may be NULL, as for mdc_prepare_batch
            mdc_set_error("mdc_seq_prepare: output level %d is NULL", l);
            return MDC_ERR_INVALID_ARG;
        }
    }
    if (count == 0) return MDC_OK;
    if (threads < 1) threads = mdc_seq_default_threads();
    // a chunk is what the GPU side takes at a time: two frames per decode thread (handed out dynamically, so a slow frame or a
    // descheduled thread does not hold the chunk up), small enough that the un-overlapped head (first decode) and tail (last
    // H2D / K1 / D2H) of a call stay short
    const int chunk = std::min(256, std::max(16, 2 * threads));
    std::lock_guard<std::mutex> feed_lock(s->feed_mutex);
    const size_t need = static_cast<size_t>(chunk) * n_in;
    if (s->stage_bytes < need) {
        for (int b = 0; b < 2; ++b) { if (s->stage[b]) mdc_host_free(s->stage[b]); s->stage[b] = nullptr; }
        s->stage_bytes = 0;
        for (int b = 0; b < 2; ++b)
            if (mdc_host_alloc(&s->stage[b], need) != MDC_OK) {
                if (s->stage[0]) mdc_host_free(s->stage[0]);
                s->stage[0] = s->stage[1] = nullptr;
                return MDC_ERR_CUDA;
            }
        s->stage_bytes = need;
    }
    void* const stage[2] = {s->stage[0], s->stage[1]};

    // Decode pool: `threads` workers live for the whole call.  The workers take the frames of chunk k one by one (an atomic counter per
    // chunk) and decode them into stage[k & 1], then move on to chunk k+1 as soon as the GPU side has released that chunk's buffer
    // (chunk k-1 consumed), so decode of chunk k+1 overlaps H2D / K1 / D2H of chunk k, and nobody creates multi-megabyte buffers per frame.
    const int n_chunks = (count + chunk - 1) / chunk;
    const int workers = std::min(threads, std::min(count, chunk));
    std::mutex mu;
    std::condition_variable cv;
    std::vector<int> decoded(static_cast<size_t>(n_chunks), 0);      // workers finished with chunk k
    std::vector<std::atomic<int>> next_frame(static_cast<size_t>(n_chunks));      // next frame of chunk k nobody has taken yet
    for (auto& a : next_frame) a.store(0, std::memory_order_relaxed);
    int released = 1;                 // chunks whose buffer may be written: 0 .. released (stage[0] and stage[1] are free at the start)
    bool abort = false;
    // first error met in chunk k.  Per chunk, because the workers run one chunk ahead: an error in chunk k+1 must not stop the call
    // before chunk k, which decoded fine, has been prepared (the reference prepares every frame before the bad one).
    std::vector<std::string> chunk_error(static_cast<size_t>(n_chunks));
    auto worker = [&](int) {
        std::vector<uint8_t> px;
        for (int k = 0; k < n_chunks; ++k) {
            {
                std::unique_lock<std::mutex> lk(mu);
                cv.wait(lk, [&] { return abort || k <= released; });
                if (abort) return;
            }
            const int f0 = k * chunk, n = std::min(chunk, count - f0);
            uint8_t* dst = static_cast<uint8_t*>(stage[k & 1]);
            std::string err;
            for (int i; err.empty() && (i = next_frame[static_cast<size_t>(k)].fetch_add(1, std::memory_order_relaxed)) < n;) {
                int w = 0, h = 0;
                if (!read_gray8(s, first + f0 + i, &px, &w, &h)) err = mdc_last_error();
                else if (w != in_w || h != in_h) {      // BenchmarkDatasetReader.h:194-199
                    char msg[256];
                    snprintf(msg, sizeof msg, "expected image dimensions %d x %d; found %d x %d (image %s)", in_w, in_h, w, h, s->files[static_cast<size_t>(first + f0 + i)].c_str());
                    err = msg;
                } else {
                    memcpy(dst + static_cast<size_t>(i) * n_in, px.data(), n_in);
                }
            }
            std::lock_guard<std::mutex> lk(mu);
            if (!err.empty() && chunk_error[static_cast<size_t>(k)].empty()) chunk_error[static_cast<size_t>(k)] = err;
            ++decoded[static_cast<size_t>(k)];
            cv.notify_all();
        }
    };
    std::vector<std::thread> pool;
    try {
        for (int t = 0; t < workers; ++t) pool.emplace_back(worker, t);
    } catch (const std::exception& e) {
        { std::lock_guard<std::mutex> lk(mu); abort = true; }
        cv.notify_all();
        for (auto& th : pool) th.join();
        mdc_set_error("mdc_seq_prepare: cannot start decode threads (%s)", e.what());
        return MDC_ERR_IO;
    }
    int rc = MDC_OK;
    for (int k = 0; k < n_chunks && rc == MDC_OK; ++k) {
        std::string err;
        {
            std::unique_lock<std::mutex> lk(mu);
            cv.wait(lk, [&] { return decoded[static_cast<size_t>(k)] == workers; });
            err = chunk_error[static_cast<size_t>(k)];
        }
        if (!err.empty()) {
            printf("ERROR: %s\n", err.c_str());
            mdc_set_error("mdc_seq_prepare: %s", err.c_str());
            rc = MDC_ERR_FORMAT;
            break;
        }
        const int f0 = k * chunk, n = std::min(chunk, count - f0);
        std::vector<void*> outs(static_cast<size_t>(levels));
        const size_t esize = mdc_out_elem_size(out_type);
        for (int l = 0; l < levels; ++l)
            outs[static_cast<size_t>(l)] = h_out_levels[l] ? static_cast<uint8_t*>(h_out_levels[l]) + static_cast<size_t>(f0) * level_px[static_cast<size_t>(l)] * esize : nullptr;
        rc = prepare(c, static_cast<const uint8_t*>(stage[k & 1]), n, flags, out_type, outs.data(), levels);      // returns after the D2H copy
        std::lock_guard<std::mutex> lk(mu);
        released = k + 2;             // stage[k & 1] is free again: chunk k+2 may be decoded into it
        cv.notify_all();
    }
    {
        std::lock_guard<std::mutex> lk(mu);
        abort = true;                 // error path: wake workers that wait for a buffer that will not be released
    }
    cv.notify_all();
    for (auto& th : pool) th.join();
    return rc;
}
