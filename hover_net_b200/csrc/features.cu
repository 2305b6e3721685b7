// Per-instance measurements on the device (include/hvn.h hvn_inst_features*): for every instance-table row the
// HVN_FEAT_LEN columns defined there, from the instance map, the row's contour, the u8 image and the NP channel.
//
// One warp per row does three things.
//   pixel pass   : the bbox in raster order, lanes across a line; exact integer sums A, sum x, sum y, sum x^2,
//                  sum xy, sum y^2 (x, y relative to (cmin, rmin)), per channel sum and sum of squares of the image,
//                  and the fp64 sum of the fp32 NP values.  Integer sums are order-free; the NP sum has a fixed order
//                  (each lane its own pixels in raster order, then a fixed shuffle tree), so calls are repeatable.
//   contour pass : cv2.arcLength (fp32 segment lengths added in fp64 in point order, from the closing segment), the
//                  shoelace area in int64, and the convex hull: the points as (x, y) keys, bitonic-sorted by the warp
//                  in shared memory (global scratch past FEAT_SMEM_POINTS points), deduplicated, then Andrew's
//                  monotone chain on lane 0.  Nothing assumes a simple polygon.  feret_max is the largest squared
//                  distance over hull vertex pairs (int64), rooted once.
//   finishing    : lane 0 evaluates the column formulas in fp64.  This file is built with -fmad=false, so every
//                  product and sum is rounded as written (the Python restatement in tests/features_ref.py computes
//                  the same operations in the same order).
#include <math.h>

#include "../../include/hvn.h"
#include "features.h"

namespace hvn {
namespace {

constexpr int kWarps = 4;  // rows per CTA
constexpr unsigned kFull = 0xffffffffu;

__device__ __forceinline__ int map_of_row(const int *__restrict__ row_offs, int n_maps, long long r) {
    int lo = 0, hi = n_maps - 1;  // last m with row_offs[m] <= r
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (row_offs[mid] <= r) lo = mid;
        else hi = mid - 1;
    }
    return lo;
}

__global__ void k_feat_check(const FeatMap *__restrict__ maps, int n_maps, const int *__restrict__ row_offs,
                             long long n_rows, const long long *__restrict__ table, const int *__restrict__ pts,
                             const int *__restrict__ pt_offs, FeatStatus *__restrict__ st) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    long long err = 0;
    if (i < n_maps) {
        if (row_offs[i] > row_offs[i + 1]) err |= 1;
        if (i == 0 && (row_offs[0] != 0 || row_offs[n_maps] != n_rows)) err |= 1;
    }
    if (i < n_rows) {
        const long long *t = table + i * HVN_ROW_LEN;
        const FeatMap mp = maps[map_of_row(row_offs, n_maps, i)];
        const long long rmin = t[HVN_ROW_RMIN], cmin = t[HVN_ROW_CMIN], rmax = t[HVN_ROW_RMAX], cmax = t[HVN_ROW_CMAX];
        if (!(rmin >= 0 && rmin < rmax && rmax <= mp.H && cmin >= 0 && cmin < cmax && cmax <= mp.W)) err |= 2;
        // a row's points are read only when its range lies inside the call's [pt_offs[0], pt_offs[n_rows]] with
        // pt_offs[0] >= 0: then every read is within the buffer the caller declared, whatever the other rows hold,
        // and any falling offset makes some row fail this test
        const long long lo = pt_offs[0], hi = pt_offs[n_rows], p0 = pt_offs[i], p1 = pt_offs[i + 1];
        if (!(0 <= lo && lo <= p0 && p0 <= p1 && p1 <= hi)) err |= 4;
        if (!(err & 6)) {
            for (long long k = p0; k < p1; ++k) {
                const int x = pts[2 * k], y = pts[2 * k + 1];
                if (x < cmin || x >= cmax || y < rmin || y >= rmax) { err |= 8; break; }
            }
            atomicMax((unsigned long long *)&st->max_pts, (unsigned long long)(p1 - p0));
        }
        if (i == n_rows - 1) st->total_pts = (long long)pt_offs[n_rows] - pt_offs[0];
    }
    if (err) atomicOr((unsigned long long *)&st->err, (unsigned long long)err);
}

template <typename T> __device__ __forceinline__ T warp_sum(T v) {
    for (int d = 16; d > 0; d >>= 1) v += __shfl_down_sync(kFull, v, d);
    return v;  // lane 0 holds the sum
}

// Key of point (x, y) with x, y >= 0: sorts by x, then y.
__device__ __forceinline__ unsigned long long pkey(int x, int y) {
    return ((unsigned long long)(unsigned)x << 32) | (unsigned)y;
}
__device__ __forceinline__ long long kx(unsigned long long k) { return (long long)(k >> 32); }
__device__ __forceinline__ long long ky(unsigned long long k) { return (long long)(k & 0xffffffffull); }
__device__ __forceinline__ long long cross(unsigned long long o, unsigned long long a, unsigned long long b) {
    return (kx(a) - kx(o)) * (ky(b) - ky(o)) - (ky(a) - ky(o)) * (kx(b) - kx(o));
}

// Bitonic sort of keys[0, p2) (p2 a power of two) by one warp; keys may live in shared or global memory.
__device__ void warp_sort(unsigned long long *keys, int p2, int lane) {
    for (int k = 2; k <= p2; k <<= 1) {
        for (int j = k >> 1; j > 0; j >>= 1) {
            for (int i = lane; i < p2; i += 32) {
                const int l = i ^ j;
                if (l > i) {
                    const unsigned long long a = keys[i], b = keys[l];
                    if ((a > b) == ((i & k) == 0)) { keys[i] = b; keys[l] = a; }
                }
            }
            __syncwarp();
        }
    }
}

// Correctly rounded double of the unsigned 128-bit value hi * 2^64 + lo.
__device__ double u128_to_double(unsigned long long hi, unsigned long long lo) {
    if (hi == 0) return __ull2double_rn(lo);
    const int lz = __clzll((long long)hi), sh = 64 - lz;
    const unsigned long long top = lz ? (hi << lz) | (lo >> sh) : hi;
    const unsigned long long rest = lz ? lo << lz : lo;  // the bits shifted out
    return ldexp(__ull2double_rn(top | (rest != 0)), sh);
}

// sqrt(double(A * Q - S^2) / (double(A) * double(A))), the numerator exact in 128 bits and rounded once.
__device__ double pop_std(unsigned long long A, unsigned long long S, unsigned long long Q) {
    const unsigned long long alo = A * Q, ahi = __umul64hi(A, Q);
    const unsigned long long slo = S * S, shi = __umul64hi(S, S);
    const unsigned long long lo = alo - slo, hi = ahi - shi - (alo < slo);
    const double a = (double)A;
    return sqrt(u128_to_double(hi, lo) / (a * a));
}

__global__ void __launch_bounds__(32 * kWarps)
k_feat_rows(const FeatMap *__restrict__ maps, int n_maps, const int *__restrict__ inst_all,
            const unsigned char *__restrict__ img_all, const float *__restrict__ pred_all, int C,
            const long long *__restrict__ table, const int *__restrict__ row_offs, long long n_rows,
            const int *__restrict__ pts, const int *__restrict__ pt_offs, unsigned long long *__restrict__ gkeys,
            int *__restrict__ gstack, double *__restrict__ feats) {
    __shared__ unsigned long long s_keys[kWarps][FEAT_SMEM_POINTS];
    __shared__ int s_stack[kWarps][2 * FEAT_SMEM_POINTS];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const long long r = (long long)blockIdx.x * kWarps + warp;
    if (r >= n_rows) return;
    const long long *t = table + r * HVN_ROW_LEN;
    const int id = (int)t[HVN_ROW_ID];
    const int rmin = (int)t[HVN_ROW_RMIN], cmin = (int)t[HVN_ROW_CMIN];
    const int bh = (int)t[HVN_ROW_RMAX] - rmin, bw = (int)t[HVN_ROW_CMAX] - cmin;
    const FeatMap mp = maps[map_of_row(row_offs, n_maps, r)];

    // ---- pixel pass
    long long A = 0, sx = 0, sy = 0, sxx = 0, sxy = 0, syy = 0, S0 = 0, S1 = 0, S2 = 0, Q0 = 0, Q1 = 0, Q2 = 0;
    double npsum = 0.0;
    for (int y = 0; y < bh; ++y) {
        const long long p_row = mp.px_off + (long long)(rmin + y) * mp.W + cmin;
        for (int x = lane; x < bw; x += 32) {
            const long long p = p_row + x;
            if (inst_all[p] != id) continue;
            ++A;
            sx += x; sy += y;
            sxx += (long long)x * x; sxy += (long long)x * y; syy += (long long)y * y;
            if (img_all) {
                const long long v0 = img_all[3 * p], v1 = img_all[3 * p + 1], v2 = img_all[3 * p + 2];
                S0 += v0; S1 += v1; S2 += v2;
                Q0 += v0 * v0; Q1 += v1 * v1; Q2 += v2 * v2;
            }
            if (pred_all) npsum += (double)pred_all[p * C + (C - 3)];
        }
    }
    A = warp_sum(A); sx = warp_sum(sx); sy = warp_sum(sy);
    sxx = warp_sum(sxx); sxy = warp_sum(sxy); syy = warp_sum(syy);
    S0 = warp_sum(S0); S1 = warp_sum(S1); S2 = warp_sum(S2);
    Q0 = warp_sum(Q0); Q1 = warp_sum(Q1); Q2 = warp_sum(Q2);
    npsum = warp_sum(npsum);

    // ---- contour pass
    const long long p0 = pt_offs[r];
    const int n = (int)(pt_offs[r + 1] - p0);
    const int *P = pts + 2 * p0;
    long long shoe = 0;  // relative to (cmin, rmin): every term is bounded by twice the bbox area
    for (int i = lane; i < n; i += 32) {
        const int j = i ? i - 1 : n - 1;
        shoe += (long long)(P[2 * j] - cmin) * (P[2 * i + 1] - rmin) - (long long)(P[2 * j + 1] - rmin) * (P[2 * i] - cmin);
    }
    shoe = warp_sum(shoe);
    // arcLength: segment i runs from point i - 1 (the last point for i = 0) to point i; lane 0 adds 32 at a time in
    // point order
    double perim = 0.0;
    if (n > 1) {
        for (int b = 0; b < n; b += 32) {
            const int i = b + lane;
            float d = 0.f;
            if (i < n) {
                const int j = i ? i - 1 : n - 1;
                const float dx = (float)P[2 * i] - (float)P[2 * j], dy = (float)P[2 * i + 1] - (float)P[2 * j + 1];
                d = sqrtf(dx * dx + dy * dy);
            }
            for (int k = 0; k < 32 && b + k < n; ++k) {
                const float dk = __shfl_sync(kFull, d, k);
                if (lane == 0) perim += (double)dk;
            }
        }
    }
    // convex hull
    unsigned long long *keys;
    int *stack;
    if (n <= FEAT_SMEM_POINTS) {
        keys = s_keys[warp];
        stack = s_stack[warp];
    } else {
        const long long o = 2 * (p0 - pt_offs[0]);
        keys = gkeys + o;
        stack = gstack + o;
    }
    int p2 = 1;
    while (p2 < n) p2 <<= 1;
    for (int i = lane; i < p2; i += 32) keys[i] = i < n ? pkey(P[2 * i], P[2 * i + 1]) : ~0ull;
    __syncwarp();
    if (n > 1) warp_sort(keys, p2, lane);
    int h = 0;
    long long hull2 = 0;
    if (lane == 0 && n > 0) {
        int m = 1;
        for (int i = 1; i < n; ++i)
            if (keys[i] != keys[m - 1]) keys[m++] = keys[i];
        if (m == 1) {
            stack[0] = 0;
            h = 1;
        } else {
            int k = 0;
            for (int i = 0; i < m; ++i) {
                while (k >= 2 && cross(keys[stack[k - 2]], keys[stack[k - 1]], keys[i]) <= 0) --k;
                stack[k++] = i;
            }
            const int lower = k + 1;
            for (int i = m - 2; i >= 0; --i) {
                while (k >= lower && cross(keys[stack[k - 2]], keys[stack[k - 1]], keys[i]) <= 0) --k;
                stack[k++] = i;
            }
            h = k - 1;  // the last entry repeats the first
            for (int i = 1; i + 1 < h; ++i) hull2 += cross(keys[stack[0]], keys[stack[i]], keys[stack[i + 1]]);
        }
    }
    h = __shfl_sync(kFull, h, 0);
    __syncwarp();
    long long fer2 = 0;
    for (int i = lane; i < h; i += 32) {
        const unsigned long long a = keys[stack[i]];
        for (int j = i + 1; j < h; ++j) {
            const unsigned long long b = keys[stack[j]];
            const long long dx = kx(b) - kx(a), dy = ky(b) - ky(a);
            fer2 = max(fer2, dx * dx + dy * dy);
        }
    }
    for (int d = 16; d > 0; d >>= 1) fer2 = max(fer2, __shfl_down_sync(kFull, fer2, d));

    // ---- finishing
    if (lane != 0) return;
    double *f = feats + r * HVN_FEAT_LEN;
    const double a_px = (double)A;
    const double carea = (double)(shoe < 0 ? -shoe : shoe) * 0.5;
    const double harea = (double)(hull2 < 0 ? -hull2 : hull2) * 0.5;
    f[HVN_FEAT_AREA] = a_px;
    f[HVN_FEAT_CONTOUR_AREA] = carea;
    f[HVN_FEAT_PERIMETER] = perim;
    f[HVN_FEAT_CONVEX_AREA] = harea;
    f[HVN_FEAT_SOLIDITY] = harea != 0.0 ? carea / harea : 0.0;
    f[HVN_FEAT_CIRCULARITY] = perim != 0.0 ? 4.0 * 3.141592653589793 * carea / (perim * perim) : 0.0;
    double major = 0.0, minor = 0.0, ecc = 0.0, orient = 0.0;
    if (A > 0) {
        // cv2.moments' completion (OpenCV completeMomentState): cx = m10 * (1 / m00), mu20 = m20 - m10 * cx, ...
        const double m10 = (double)sx, m01 = (double)sy, inv = 1.0 / a_px;
        const double cx = m10 * inv, cy = m01 * inv;
        const double mu20 = (double)sxx - m10 * cx, mu11 = (double)sxy - m10 * cy, mu02 = (double)syy - m01 * cy;
        const double a = mu20 / a_px, b = mu11 / a_px, c = mu02 / a_px;
        const double hd = (a - c) / 2.0, mid = (a + c) / 2.0;
        const double rr = sqrt(hd * hd + b * b);
        const double l1 = mid + rr, l2 = fmax(mid - rr, 0.0);
        major = 4.0 * sqrt(l1);
        minor = 4.0 * sqrt(l2);
        ecc = l1 != 0.0 ? sqrt(1.0 - l2 / l1) : 0.0;
        orient = 0.5 * atan2(2.0 * b, a - c);
    }
    f[HVN_FEAT_MAJOR_AXIS_LENGTH] = major;
    f[HVN_FEAT_MINOR_AXIS_LENGTH] = minor;
    f[HVN_FEAT_ECCENTRICITY] = ecc;
    f[HVN_FEAT_ORIENTATION] = orient;
    f[HVN_FEAT_FERET_MAX] = sqrt((double)fer2);
    const long long S[3] = {S0, S1, S2}, Q[3] = {Q0, Q1, Q2};
    for (int ch = 0; ch < 3; ++ch) {
        f[HVN_FEAT_MEAN_R + ch] = !img_all ? nan("") : (A > 0 ? (double)S[ch] / a_px : 0.0);
        f[HVN_FEAT_STD_R + ch] = !img_all ? nan("") : (A > 0 ? pop_std(A, S[ch], Q[ch]) : 0.0);
    }
    f[HVN_FEAT_NP_PROB_MEAN] = !pred_all ? nan("") : (A > 0 ? npsum / a_px : 0.0);
}

}  // namespace

int features_check(cudaStream_t stream, const FeatMap *maps, int n_maps, const int *row_offs, long long n_rows,
                   const long long *table, const int *pts, const int *pt_offs, FeatStatus *status) {
    HVN_CUDA(cudaMemsetAsync(status, 0, sizeof(FeatStatus), stream));
    const long long items = n_rows > n_maps ? n_rows : n_maps;
    k_feat_check<<<cdiv(items, 256), 256, 0, stream>>>(maps, n_maps, row_offs, n_rows, table, pts, pt_offs, status);
    HVN_CUDA(cudaGetLastError());
    return 1;
}

int features_rows(cudaStream_t stream, const FeatMap *maps, int n_maps, const int *inst, const unsigned char *img,
                  const float *pred, int C, const long long *table, const int *row_offs, long long n_rows,
                  const int *pts, const int *pt_offs, void *scratch, double *feats, long long total_pts) {
    if (n_rows == 0) return 0;
    unsigned long long *gkeys = (unsigned long long *)scratch;
    int *gstack = scratch ? (int *)(gkeys + 2 * total_pts) : nullptr;
    k_feat_rows<<<cdiv(n_rows, kWarps), 32 * kWarps, 0, stream>>>(maps, n_maps, inst, img, pred, C, table, row_offs,
                                                                  n_rows, pts, pt_offs, gkeys, gstack, feats);
    HVN_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace hvn
