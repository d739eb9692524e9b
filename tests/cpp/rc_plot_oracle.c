/* plotE and plotG of main_responseCalib.cpp:72-146, restated in plain C and built as the reference is built (-O3, no contraction)
 * against the host's libm: the oracle of the GPU plots (csrc/mdc_rc_plot.cu).  The conversions are C's, so x86-64 makes them as
 * it makes the reference's: float or double to an 8- or 16-bit integer through a 32-bit truncation. */
#include <math.h>
#include <stddef.h>

/* range4 = {min ln(E+20), max ln(E+20), min E, max E}; bgr [npix][3] (cv::Vec3b order), e16 [npix] */
void oport_rc_plot_e_range(const double* E, int npix, double range4[4]) {
    double offset = 20;
    double min = 1e10, max = -1e10, Emin = 1e10, Emax = -1e10;
    for (int i = 0; i < npix; i++) {
        double le = log(E[i] + offset);
        if (le < min) min = le;
        if (le > max) max = le;
        if (E[i] < Emin) Emin = E[i];
        if (E[i] > Emax) Emax = E[i];
    }
    range4[0] = min; range4[1] = max; range4[2] = Emin; range4[3] = Emax;
}

void oport_rc_plot_e_map(const double* E, int npix, const double range4[4], unsigned char* bgr, unsigned short* e16) {
    double offset = 20, min = range4[0], max = range4[1], Emin = range4[2], Emax = range4[3];
    for (int i = 0; i < npix; i++) {
        float val = 3 * (exp((log(E[i] + offset) - min) / (max - min)) - 1) / 1.7183;
        int icP = val;
        float ifP = val - icP;
        icP = icP % 3;
        unsigned char c[3] = {0, 0, 0};
        if (icP == 0) { c[0] = 0; c[1] = 0; c[2] = 255 * ifP; }
        if (icP == 1) { c[0] = 0; c[1] = 255 * ifP; c[2] = 255; }
        if (icP == 2) { c[0] = 255 * ifP; c[1] = 255; c[2] = 255; }
        bgr[3 * i] = c[0]; bgr[3 * i + 1] = c[1]; bgr[3 * i + 2] = c[2];
        e16[i] = 255 * 255 * (E[i] - Emin) / (Emax - Emin);
    }
}

void oport_rc_plot_e(const double* E, int npix, double range4[4], unsigned char* bgr, unsigned short* e16) {
    oport_rc_plot_e_range(E, npix, range4);
    oport_rc_plot_e_map(E, npix, range4, bgr, e16);
}

/* gimg255 [256][256] = GImg * 255, the float image the reference hands to cv::imwrite; minmax = {min G, max G} */
void oport_rc_plot_g(const double* G, float* gimg255, double minmax[2]) {
    double min = 1e10, max = -1e10;
    for (int i = 0; i < 256 * 256; i++) gimg255[i] = 0;
    for (int i = 0; i < 256; i++) {
        if (G[i] < min) min = G[i];
        if (G[i] > max) max = G[i];
    }
    for (int i = 0; i < 256; i++) {
        double val = 256 * (G[i] - min) / (max - min);
        for (int k = 0; k < 256; k++)
            if (val < k) gimg255[k * 256 + i] = k - val;
    }
    for (int i = 0; i < 256 * 256; i++) gimg255[i] = (float)(gimg255[i] * 255.0);
    minmax[0] = min; minmax[1] = max;
}

/* the host's libm itself: out[i] = exp(in[i]) (op 0) or log(in[i]) (op 1) */
void oport_libm(int op, const double* in, double* out, size_t n) {
    for (size_t i = 0; i < n; i++) out[i] = op == 0 ? exp(in[i]) : log(in[i]);
}
