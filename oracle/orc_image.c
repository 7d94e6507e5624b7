/* orc_image.c -- CPU oracle of the image post-processing (DESIGN f-9): AutoExposure, BeamUniformityCorrector and
 * LocalToneMapper of ouster_core/src/image_processing.cpp restated in plain C, in the reference's types and loop
 * order.  Order statistics come from a full sort (nth_element's value is the sorted array's).  Test
 * infrastructure only: built by oracle/image.mk, bound by oracle/image.py. */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define R_LUM 0.299
#define G_LUM 0.587
#define B_LUM 0.114
#define AE_STRIDE 4
#define AE_MIN_NONZERO_POINTS 100
#define BUC_DAMPING 0.92
#define BUC_UPDATE_EVERY 8
#define CLAHE_TILES 8
#define CLAHE_HIST_BINS 1024

/* the layout of ob_image_state / ob_image_params (include/ouster_b200.h) */
typedef struct orc_img_state {
    double lo, hi, lo_state, hi_state;
    int32_t counter, initialized;
    uint32_t dc_rows, reserved;
} orc_img_state;

typedef struct orc_img_params {
    double lo_percentile, hi_percentile;
    int32_t update_every, color_correct;
    double damping, compress_dr_max_lum;
} orc_img_params;

static float orc_fminf_std(float a, float b) { return (b < a) ? b : a; }

/* f16_bits_to_f32_bits_fast_nan_zero (image_processing.cpp:59-65) */
uint32_t orc_f16_bits_fast(uint16_t bits) {
    const uint32_t expanded = (uint32_t)(bits + 0x1C000u) << 13;
    return bits != 0 ? (bits != 0x7e00 ? expanded : 0u) : 0u;
}

void orc_f16_convert(const uint16_t* in, float* out, size_t n) {
    for (size_t i = 0; i < n; ++i) {
        const uint32_t b = orc_f16_bits_fast(in[i]);
        memcpy(&out[i], &b, 4);
    }
}

/* fast_log10 (image_processing.cpp:68-76) */
static float orc_fast_log10(float x) {
    uint32_t bits;
    memcpy(&bits, &x, sizeof(x));
    const float log2_approx = (float)((int32_t)bits - 0x3F800000) * 1.1920929e-7f;
    return log2_approx * 0.30103f;
}

#define T float
#define S _f
#define EPS 1.1920928955078125e-07f
#include "orc_image_t.h"
#undef T
#undef S
#undef EPS

#define T double
#define S _d
#define EPS 2.220446049250313e-16
#include "orc_image_t.h"
#undef T
#undef S
#undef EPS
