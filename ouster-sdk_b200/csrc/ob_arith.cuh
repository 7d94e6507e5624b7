// ob_arith.cuh -- the device arithmetic that bit-exact parity with the CPU oracle rests on (DESIGN 2): operations
// rounded one at a time, the summation order of 3-vectors, std::max / std::min, the order-preserving integer image of
// a float or double, x86's cast of a floored double, and the uint64 warp sum.  Every kernel file that needs one of
// them includes this header, so each rounding order is stated once.
#pragma once
#include <cuda/std/limits>

#include <cstdint>

namespace ob {
namespace {

// One rounding per operation.  __f*_rn / __d*_rn are never contracted into an FMA, as nvcc contracts a * b + c by
// default; the reference's x86 build (SSE2, no FMA) and the oracle (-ffp-contract=off) round every step.
__device__ __forceinline__ float mul(float a, float b) { return __fmul_rn(a, b); }
__device__ __forceinline__ double mul(double a, double b) { return __dmul_rn(a, b); }
__device__ __forceinline__ float add(float a, float b) { return __fadd_rn(a, b); }
__device__ __forceinline__ double add(double a, double b) { return __dadd_rn(a, b); }
__device__ __forceinline__ float sub(float a, float b) { return __fsub_rn(a, b); }
__device__ __forceinline__ double sub(double a, double b) { return __dsub_rn(a, b); }
__device__ __forceinline__ float div(float a, float b) { return __fdiv_rn(a, b); }
__device__ __forceinline__ double div(double a, double b) { return __ddiv_rn(a, b); }

// Eigen 3.4's unrolled SSE2 redux of a fixed-size 3-vector: dot product and squaredNorm are (x0 y0 + x1 y1) + x2 y2,
// norm() the square root of that
__device__ __forceinline__ double dot3(const double* a, const double* b) {
    return add(add(mul(a[0], b[0]), mul(a[1], b[1])), mul(a[2], b[2]));
}
__device__ __forceinline__ double sqn3(double a, double b, double c) { return add(add(mul(a, a), mul(b, b)), mul(c, c)); }
__device__ __forceinline__ double norm3(double a, double b, double c) { return sqrt(sqn3(a, b, c)); }
__device__ __forceinline__ double norm3(const double* a) { return norm3(a[0], a[1], a[2]); }

// all three components finite
__device__ __forceinline__ bool finite3(double x, double y, double z) { return isfinite(x) && isfinite(y) && isfinite(z); }
__device__ __forceinline__ bool finite3(const double* v) { return finite3(v[0], v[1], v[2]); }

// std::max(a, b) and std::min(a, b), not fmax / fmin: (a < b) ? b : a and (b < a) ? b : a, so a NaN argument comes
// out where the reference's does
template <typename T>
__device__ __forceinline__ T smax(T a, T b) { return (a < b) ? b : a; }
template <typename T>
__device__ __forceinline__ T smin(T a, T b) { return (b < a) ? b : a; }

// Order-preserving unsigned image of a float or double, and back: unsigned order is "<, then -0.0 before +0.0"
// (NaNs sort outside the numbers).  Order statistics select on it as an unsigned key, because CUB's floating-point
// radix digits fold -0.0 onto +0.0 and std::nth_element / std::sort keep them apart.
__device__ __forceinline__ uint32_t okey(float v) {
    const uint32_t b = __float_as_uint(v);
    return (b & 0x80000000u) ? ~b : (b | 0x80000000u);
}
__device__ __forceinline__ unsigned long long okey(double v) {
    const unsigned long long b = static_cast<unsigned long long>(__double_as_longlong(v));
    return (b >> 63) ? ~b : (b | 0x8000000000000000ull);
}
__device__ __forceinline__ float okey_value(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }
__device__ __forceinline__ double okey_value(unsigned long long k) {
    return __longlong_as_double(static_cast<long long>((k >> 63) ? (k & 0x7fffffffffffffffull) : ~k));
}

// static_cast<I>(std::floor(v)) for I = int32_t or int64_t as x86's cvttsd2si evaluates it: NaN and out-of-range
// values give the integer indefinite, INT32_MIN / INT64_MIN, where the device conversion would saturate
template <typename I>
__device__ __forceinline__ I floor_cast(double v) {
    static_assert(sizeof(I) == 4 || sizeof(I) == 8, "cvttsd2si converts to int32 or int64");
    constexpr double kLimit = sizeof(I) == 4 ? 2147483648.0 : 9223372036854775808.0;  // 2^31, 2^63
    const double f = floor(v);
    if (!(f >= -kLimit && f < kLimit)) return ::cuda::std::numeric_limits<I>::min();
    return static_cast<I>(f);
}

// sum over the 32 lanes of a full warp, every lane gets it
__device__ __forceinline__ unsigned long long warp_sum_u64(unsigned long long v) {
#pragma unroll
    for (int d = 16; d > 0; d >>= 1) v += __shfl_xor_sync(0xffffffffu, v, d);
    return v;
}

}  // namespace
}  // namespace ob
