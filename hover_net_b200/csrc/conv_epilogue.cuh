// Fused convolution epilogue shared by the referee and the wgmma kernels:
// residual add, raw fp32 store, BN(scale/shift)+ReLU -> split fp16 store, or 2x nearest-neighbour
// upsample + skip add -> split store (reference net_utils.py:263-265, net_desc.py:133-139).
#pragma once
#include "conv_params.h"

namespace hvn {

// The range tests are written !(|x| <= 65504) so that NaN, for which every comparison is false, raises the flag too; the
// clamp then stores it as -65504 (fmaxf returns the non-NaN operand), finite like every other flagged value.
__device__ __forceinline__ void split_f32(float x, __half &hi, __half &lo, unsigned int *flag = nullptr) {
    if (flag && !(fabsf(x) <= 65504.f)) *flag = 1u;  // benign race: every writer stores the same value
    x = fminf(fmaxf(x, -65504.f), 65504.f);
    hi = __float2half_rn(x);
    lo = __float2half_rn(x - __half2float(hi));
}

__device__ __forceinline__ float join_f16(__half hi, __half lo) { return __half2float(hi) + __half2float(lo); }

// Single-plane tensors (precision "high": SplitRef::lo == nullptr) store only hi = fp16_rn(x) -- the same hi, with the same
// range check and clamp, as split_f32 -- and read back as hi alone.
__device__ __forceinline__ __half hi_f32(float x, unsigned int *flag = nullptr) {
    if (flag && !(fabsf(x) <= 65504.f)) *flag = 1u;
    return __float2half_rn(fminf(fmaxf(x, -65504.f), 65504.f));
}

// max that returns NaN when either operand is NaN (fmaxf returns the other one): a running maximum built from it carries
// a NaN through to the range test
__device__ __forceinline__ float fmax_nan(float a, float b) {
    float r;
    asm("max.NaN.f32 %0, %1, %2;" : "=f"(r) : "f"(a), "f"(b));
    return r;
}

// Four values at once with the packed conversions (one F2FP per pair): same roundings as split_f32.
// NONNEG: the inputs are already >= 0 (post-ReLU), so only the upper clamp is needed.
template <bool NONNEG = false>
__device__ __forceinline__ void split4_f32(const float t[4], uint2 &hi, uint2 &lo, unsigned int *flag = nullptr) {
    if (flag) {
        const float m = NONNEG ? fmax_nan(fmax_nan(t[0], t[1]), fmax_nan(t[2], t[3]))
                               : fmax_nan(fmax_nan(fabsf(t[0]), fabsf(t[1])), fmax_nan(fabsf(t[2]), fabsf(t[3])));
        if (!(m <= 65504.f)) *flag = 1u;
    }
    float x[4];
#pragma unroll
    for (int i = 0; i < 4; ++i) x[i] = NONNEG ? fminf(t[i], 65504.f) : fminf(fmaxf(t[i], -65504.f), 65504.f);
    const __half2 h01 = __floats2half2_rn(x[0], x[1]), h23 = __floats2half2_rn(x[2], x[3]);
    const float2 f01 = __half22float2(h01), f23 = __half22float2(h23);
    const __half2 l01 = __floats2half2_rn(x[0] - f01.x, x[1] - f01.y), l23 = __floats2half2_rn(x[2] - f23.x, x[3] - f23.y);
    hi = make_uint2(*reinterpret_cast<const uint32_t *>(&h01), *reinterpret_cast<const uint32_t *>(&h23));
    lo = make_uint2(*reinterpret_cast<const uint32_t *>(&l01), *reinterpret_cast<const uint32_t *>(&l23));
}

// hi of split4_f32<true> alone: fp16_rn of four values >= 0, clamped at 65504 (single-plane XF tiles; the caller keeps
// the running maximum for the range guard)
__device__ __forceinline__ uint2 hi4_f32_nonneg(const float t[4]) {
    const __half2 h01 = __floats2half2_rn(fminf(t[0], 65504.f), fminf(t[1], 65504.f));
    const __half2 h23 = __floats2half2_rn(fminf(t[2], 65504.f), fminf(t[3], 65504.f));
    return make_uint2(*reinterpret_cast<const uint32_t *>(&h01), *reinterpret_cast<const uint32_t *>(&h23));
}

// relu(y) split by TRUNCATION, for the XF transform warps whose instruction count paces the tensor core:
//   m  = y with the low 13 mantissa bits cleared  -> exactly an fp16 value for 2^-14 <= |y| < 65536 (one LOP3)
//   hi = cvt.rz.relu.f16x2(m),  lo = cvt.rn.relu.f16x2(y - m)      (y - m is exact, and has the sign of y)
// 4.5 instructions per element with the running maximum, against 7.25 for relu -> clamp -> rn -> unpack -> subtract ->
// rn.  y < 0: both halves relu to 0.  0 <= lo < ulp(hi) instead of |lo| <= ulp/2: hi + lo carries 21 bits instead of 22.
// Below 2^-14 hi is an fp16 subnormal = rz(m) and y - m is not the exact remainder: absolute error < 2^-24 (the rn split
// has 2^-25 there).  y >= 65536: rz saturates hi at 65504 (never Inf); the caller's running maximum raises the range flag.
__device__ __forceinline__ void split4_relu_trunc(const float y[4], uint2 &hi, uint2 &lo) {
    uint32_t h[2], l[2];
#pragma unroll
    for (int i = 0; i < 2; ++i) {
        const float m0 = __uint_as_float(__float_as_uint(y[2 * i]) & 0xFFFFE000u);
        const float m1 = __uint_as_float(__float_as_uint(y[2 * i + 1]) & 0xFFFFE000u);
        const float l0 = y[2 * i] - m0, l1 = y[2 * i + 1] - m1;
        asm("cvt.rz.relu.f16x2.f32 %0, %1, %2;" : "=r"(h[i]) : "f"(m1), "f"(m0));  // d = {upper: a, lower: b}
        asm("cvt.rn.relu.f16x2.f32 %0, %1, %2;" : "=r"(l[i]) : "f"(l1), "f"(l0));
    }
    hi = make_uint2(h[0], h[1]);
    lo = make_uint2(l[0], l[1]);
}

// 4 consecutive output channels c..c+3 of output pixel (n, oy, ox); c % 4 == 0.
__device__ __forceinline__ void conv_epilogue4(const ConvParams &P, int n, int oy, int ox, int c, float v[4]) {
    if (P.w.oscale) {  // undo the per-channel power-of-two weight exponent (exact)
        const float4 ws = *reinterpret_cast<const float4 *>(P.w.oscale + c);
        v[0] *= ws.x; v[1] *= ws.y; v[2] *= ws.z; v[3] *= ws.w;
    }
    if (P.res.p) {
        const float4 r = *reinterpret_cast<const float4 *>(P.res.p + n * P.res.sN + (long long)oy * P.res.sH +
                                                           (long long)ox * P.res.sW + c);
        v[0] += r.x; v[1] += r.y; v[2] += r.z; v[3] += r.w;
    }
    if (P.out_raw.p) {
        float *o = P.out_raw.p + n * P.out_raw.sN + (long long)oy * P.out_raw.sH + (long long)ox * P.out_raw.sW + c;
        *reinterpret_cast<float4 *>(o) = make_float4(v[0], v[1], v[2], v[3]);
    }
    if (P.up2) {
#pragma unroll
        for (int d = 0; d < 4; ++d) {
            int Y = 2 * oy + (d >> 1), X = 2 * ox + (d & 1);
            long long so = n * P.skip.sN + (long long)Y * P.skip.sH + (long long)X * P.skip.sW + c;
            long long oo = n * P.out_split.sN + (long long)Y * P.out_split.sH + (long long)X * P.out_split.sW + c;
            const __half2 *sh = reinterpret_cast<const __half2 *>(P.skip.hi + so);
            const __half2 zero = __float2half2_rn(0.f);
            const __half2 *sl = P.skip.lo ? reinterpret_cast<const __half2 *>(P.skip.lo + so) : nullptr;
            __half2 h01 = sh[0], h23 = sh[1], l01 = sl ? sl[0] : zero, l23 = sl ? sl[1] : zero;
            float t[4] = {v[0] + join_f16(h01.x, l01.x), v[1] + join_f16(h01.y, l01.y),
                          v[2] + join_f16(h23.x, l23.x), v[3] + join_f16(h23.y, l23.y)};
            __half oh[4], ol[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) split_f32(t[i], oh[i], ol[i], P.out_split.flag);
            *reinterpret_cast<uint2 *>(P.out_split.hi + oo) = *reinterpret_cast<uint2 *>(oh);
            if (P.out_split.lo) *reinterpret_cast<uint2 *>(P.out_split.lo + oo) = *reinterpret_cast<uint2 *>(ol);
        }
    } else if (P.out_split.hi) {
        float t[4] = {v[0], v[1], v[2], v[3]};
        if (P.scale) {
            const float4 s = *reinterpret_cast<const float4 *>(P.scale + c);
            const float4 b = *reinterpret_cast<const float4 *>(P.shift + c);
            t[0] = t[0] * s.x + b.x; t[1] = t[1] * s.y + b.y; t[2] = t[2] * s.z + b.z; t[3] = t[3] * s.w + b.w;
        }
        if (P.relu) {
#pragma unroll
            for (int i = 0; i < 4; ++i) t[i] = fmaxf(t[i], 0.f);
        }
        __half oh[4], ol[4];
#pragma unroll
        for (int i = 0; i < 4; ++i) split_f32(t[i], oh[i], ol[i], P.out_split.flag);
        long long oo = n * P.out_split.sN + (long long)oy * P.out_split.sH + (long long)ox * P.out_split.sW + c;
        *reinterpret_cast<uint2 *>(P.out_split.hi + oo) = *reinterpret_cast<uint2 *>(oh);
        if (P.out_split.lo) *reinterpret_cast<uint2 *>(P.out_split.lo + oo) = *reinterpret_cast<uint2 *>(ol);
    }
}

// Epilogue variants of the wgmma kernel (k_conv_tc's MODE): plain, + residual, 2x upsample + skip.
enum { EPI_PLAIN = 0, EPI_RES = 1, EPI_UP2 = 2 };

__device__ __forceinline__ void store_split4(const SplitRef &o, long long off, const float t[4]) {
    uint2 oh, ol;
    split4_f32(t, oh, ol, o.flag);
    *reinterpret_cast<uint2 *>(o.hi + off) = oh;
    if (o.lo) *reinterpret_cast<uint2 *>(o.lo + off) = ol;
}

}  // namespace hvn
