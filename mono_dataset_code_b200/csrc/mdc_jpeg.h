// The marker walk of a baseline JPEG (mdc_jpeg.cpp), shared by the host decoder and the GPU decoder (mdc_jpeg_gpu.cu): one parser,
// one set of checks and error messages for both.
#pragma once
#include <stddef.h>
#include <stdint.h>
#include <string>
#include <vector>

#include "mdc_jpeg_entropy.cuh"

struct mdc_jpeg_component { int id = 0, h = 1, v = 1, tq = 0, td = 0, ta = 0; };

struct mdc_jpeg_header {
    int width = 0, height = 0;
    int ncomp = 0;                       // 1 or 3; component 0 is the luminance
    mdc_jpeg_component comp[3];          // sampling factors, quantisation / DC / AC table ids
    int32_t qzz[64];                     // luminance quantisation steps in zig-zag (= stream) order
    mdcj::HuffTable dc[4], ac[4];        // as DHT defined them (the ones the scan uses are `defined`)
    int restart_interval = 0;            // MCUs per restart interval, 0 = none
    size_t scan_begin = 0;               // first entropy-coded byte; the scan runs to the first marker after it that is not RSTn
    // scan geometry: an MCU holds yh x yv luminance blocks; the luminance plane is padded to mcus_x * yh x mcus_y * yv blocks
    int mcus_x = 0, mcus_y = 0, yh = 1, yv = 1;
    int blocks_w() const { return mcus_x * yh; }
    int blocks_h() const { return mcus_y * yv; }
};

// Walks the markers up to and including SOS and performs every check the host decoder makes before the entropy-coded data (DQT, DHT
// with the over-subscription check, SOF0/SOF1, DRI, SOS, missing tables, a subsampled luminance).  On failure returns false with
// "<name>: <reason>" in mdc_last_error().
bool mdc_jpeg_parse_header(const uint8_t* d, size_t n, const std::string& name, mdc_jpeg_header* h);

// One restart interval of the scan: its entropy-coded bytes [begin, end) (end = the first marker after begin, or the end of the file)
// and its MCUs [first_mcu, first_mcu + n_mcus).
struct mdc_jpeg_segment { size_t begin, end; int first_mcu, n_mcus; };

// Splits the scan into its restart intervals the way the host decoder walks them: interval k + 1 starts after the first RSTn marker
// at or after the start of interval k.  Returns false if the file ends before a restart marker the scan needs ("missing restart
// marker"); `segs` then holds the intervals in front of the missing marker.
bool mdc_jpeg_split_segments(const uint8_t* d, size_t n, const mdc_jpeg_header& h, std::vector<mdc_jpeg_segment>* segs);
