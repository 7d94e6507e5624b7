/* orc_frame_ops.c -- CPU oracle of the frame operations (ouster_core/src/frame_ops.cpp:151-286,
 * python/src/ouster/sdk/core/frame_ops.py:83-136).  TEST INFRASTRUCTURE ONLY.
 *
 * Plain loops over one field at a time, in the reference's types: values compared in double, invalid written as
 * a C cast to the field's type (the caller refuses the values where that cast is undefined), NaN handled by the
 * comparisons themselves.  filter_uv "v" is also restated literally (destagger, mask, stagger) so the tests can
 * compare it with the direct staggered-domain form the GPU uses.  Type tags are ChanFieldType's (1..10). */
#include <math.h>
#include <stdint.h>
#include <stdlib.h>
#include <string.h>

#define ORC_TYPES(X)                                                                                          \
    X(1, uint8_t) X(2, uint16_t) X(3, uint32_t) X(4, uint64_t) X(5, int8_t) X(6, int16_t) X(7, int32_t)       \
    X(8, int64_t) X(9, float) X(10, double)

/* ClipOp (frame_ops.cpp:151-163): keep iff lower <= (double)v <= upper, else (T)invalid */
int orc_fo_clip(void* data, int type, size_t n, double lower, double upper, double invalid) {
    switch (type) {
#define X(tag, T)                                                                                             \
    case tag: {                                                                                               \
        T* p = (T*)data;                                                                                      \
        const T inv = (T)invalid;                                                                             \
        for (size_t i = 0; i < n; ++i) {                                                                      \
            const double v = (double)p[i];                                                                    \
            if (!(v >= lower && v <= upper)) p[i] = inv;                                                      \
        }                                                                                                     \
        return 0;                                                                                             \
    }
        ORC_TYPES(X)
#undef X
        default: return -1;
    }
}

/* BuildFilterMaskOp (frame_ops.cpp:165-183): mask[i] = !(lower <= (double)v <= upper); 0 marks invalidation */
int orc_fo_filter_mask(uint8_t* mask, const void* src, int type, size_t n, double lower, double upper) {
    switch (type) {
#define X(tag, T)                                                                                             \
    case tag: {                                                                                               \
        const T* p = (const T*)src;                                                                           \
        for (size_t i = 0; i < n; ++i) {                                                                      \
            const double v = (double)p[i];                                                                    \
            mask[i] = !(v >= lower && v <= upper);                                                            \
        }                                                                                                     \
        return 0;                                                                                             \
    }
        ORC_TYPES(X)
#undef X
        default: return -1;
    }
}

/* ApplyMaskOp (frame_ops.cpp:185-199): where mask == 0, (T)invalid */
int orc_fo_apply_mask(void* data, int type, size_t n, const uint8_t* mask, double invalid) {
    switch (type) {
#define X(tag, T)                                                                                             \
    case tag: {                                                                                               \
        T* p = (T*)data;                                                                                      \
        const T inv = (T)invalid;                                                                             \
        for (size_t i = 0; i < n; ++i)                                                                        \
            if (!mask[i]) p[i] = inv;                                                                         \
        return 0;                                                                                             \
    }
        ORC_TYPES(X)
#undef X
        default: return -1;
    }
}

static size_t true_mod(long long s, size_t w) {
    long long m = s % (long long)w;
    return (size_t)(m < 0 ? m + (long long)w : m);
}

/* filter_uv "v" in the staggered domain: pixel (r, c) is masked iff (c + shift[r]) mod w in [lower, upper) */
void orc_fo_uv_v_mask(uint8_t* mask, const int32_t* shifts, size_t h, size_t w, size_t lower, size_t upper) {
    for (size_t r = 0; r < h; ++r) {
        const size_t s = true_mod(shifts[r], w);
        for (size_t c = 0; c < w; ++c) {
            size_t d = c + s;
            if (d >= w) d -= w;
            mask[r * w + c] = !(d >= lower && d < upper);
        }
    }
}

/* destagger (impl/lidar_frame_impl.h:733-860) of one h x w field of esize-byte pixels: dst(r, (c + s) mod w) =
 * src(r, c) with s = shift (inverse: -shift) taken modulo w */
static void destagger_bytes(uint8_t* dst, const uint8_t* src, const int32_t* shifts, size_t h, size_t w,
                            size_t esize, int inverse) {
    for (size_t r = 0; r < h; ++r) {
        const size_t s = true_mod(inverse ? -(long long)shifts[r] : (long long)shifts[r], w);
        for (size_t c = 0; c < w; ++c) {
            size_t d = c + s;
            if (d >= w) d -= w;
            memcpy(dst + (r * w + d) * esize, src + (r * w + c) * esize, esize);
        }
    }
}

/* filter_uv "v" as the reference writes it (frame_ops.cpp:260-275): destagger, mask destaggered columns
 * [lower, upper), stagger back */
int orc_fo_uv_v_literal(void* data, int type, size_t esize, const int32_t* shifts, size_t h, size_t w, size_t lower,
                        size_t upper, double invalid) {
    const size_t n = h * w;
    uint8_t* tmp = (uint8_t*)malloc(n * esize + 1);
    uint8_t* mask = (uint8_t*)malloc(n + 1);
    if (!tmp || !mask) {
        free(tmp);
        free(mask);
        return -2;
    }
    destagger_bytes(tmp, (const uint8_t*)data, shifts, h, w, esize, 0);
    for (size_t r = 0; r < h; ++r)
        for (size_t c = 0; c < w; ++c) mask[r * w + c] = !(c >= lower && c < upper);
    int rc = orc_fo_apply_mask(tmp, type, n, mask, invalid);
    if (rc == 0) destagger_bytes((uint8_t*)data, tmp, shifts, h, w, esize, 1);
    free(tmp);
    free(mask);
    return rc;
}

/* filter_xyz's mask (frame_ops.py:117-122): pts[..., axis] >= lower & pts[..., axis] <= upper, in the points'
 * type with the bounds rounded to it (NumPy >= 2 comparing an array with a Python float); 1 = invalidate */
void orc_fo_xyz_mask_f64(uint8_t* hit, const double* pts, size_t n, int axis, double lower, double upper) {
    for (size_t i = 0; i < n; ++i) {
        const double v = pts[i * 3 + (size_t)axis];
        hit[i] = v >= lower && v <= upper;
    }
}
void orc_fo_xyz_mask_f32(uint8_t* hit, const float* pts, size_t n, int axis, double lower, double upper) {
    const float lo = (float)lower, hi = (float)upper;
    for (size_t i = 0; i < n; ++i) {
        const float v = pts[i * 3 + (size_t)axis];
        hit[i] = v >= lo && v <= hi;
    }
}
