// Instance post-processing on the device (sm_90a): the GPU side of reference
// `process` / `__proc_np_hv` (models/hovernet/post_proc.py:26-90, 94-186).
//
// Bit-exact contract (tests/test_postproc_gpu.py): every integer result (foreground mask, markers,
// inst_map, instance table) equals the CPU oracle; the float64 intermediates (Sobel, energy,
// blurred distance) are produced with the evaluation order pinned against cv2 in SURVEY.md App. A,
// using non-contracted __dmul_rn/__dadd_rn so ptxas cannot fuse them into FMAs.
//
// Stage map (reference line -> kernel):
//   :43      np >= 0.5                         k_threshold_minmax   (+ global min/max of hv_x, hv_y)
//   :45-47   label, remove_small(10), binarise k_ccl_*  k_blob_filter
//   :49-57   normalize x2, Sobel(ksize=21) x2  k_sobel21            (+ global min/max of both Sobels)
//   :59-81   1-normalize, max, energy, marker  k_energy
//   :76      -GaussianBlur(3x3)                k_blur3
//   :82      binary_fill_holes                 k_ccl_* on the complement, k_fill
//   :84      MORPH_OPEN ellipse 5x5            k_erode5 k_dilate5
//   :85-86   label, remove_small(10)           k_ccl_*  k_row_roots k_row_scan k_assign_ids k_marker_labels
//   :88      watershed(dist, marker, mask)     k_watershed          (one exact priority flood per blob)
//   :120-181 per-instance bbox/centroid/type   k_table_accum k_table_rows
#include "common.cuh"
#include "postproc.h"
#include "uf.cuh"

#include <string>
#include <utility>
#include <vector>

namespace hvn {

// ------------------------------------------------------------------------------------------------
// order-preserving integer keys for float / double atomics
__device__ __forceinline__ unsigned int fkey(float f) {
    unsigned int u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __host__ __forceinline__ float fkey_inv(unsigned int k) {
    unsigned int u = (k & 0x80000000u) ? (k & 0x7fffffffu) : ~k;
#ifdef __CUDA_ARCH__
    return __uint_as_float(u);
#else
    float f;
    memcpy(&f, &u, 4);
    return f;
#endif
}
__device__ __forceinline__ unsigned long long dkey(double d) {
    unsigned long long u = (unsigned long long)__double_as_longlong(d);
    return (u >> 63) ? ~u : (u | 0x8000000000000000ull);
}
__device__ __forceinline__ double dkey_inv(unsigned long long k) {
    unsigned long long u = (k >> 63) ? (k & 0x7fffffffffffffffull) : ~k;
    return __longlong_as_double((long long)u);
}

// per-map scalars
struct PPStats {
    unsigned int hmin, hmax, vmin, vmax;            // fkey of raw hv_x / hv_y extrema
    unsigned long long shmin, shmax, svmin, svmax;  // dkey of Sobel extrema
    int nblobs;                                     // foreground components with >= 10 px
    int heap_top;                                   // bump pointer into the per-map heap arena
    int nroots;                                     // marker components before the size filter
    int nrows;                                      // instance-table rows written
    int pad[2];
};

__global__ void k_init_stats(PPStats *st, int n_maps) {
    int m = blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= n_maps) return;
    PPStats s;
    s.hmin = s.vmin = 0xffffffffu;
    s.hmax = s.vmax = 0u;
    s.shmin = s.svmin = ~0ull;
    s.shmax = s.svmax = 0ull;
    s.nblobs = s.heap_top = s.nroots = s.nrows = 0;
    s.pad[0] = s.pad[1] = 0;
    st[m] = s;
}

// cv2.normalize(NORM_MINMAX, 0, 1, CV_32F) scale/shift (SURVEY.md App. A.4)
__device__ __forceinline__ void minmax_scale(double smin, double smax, double &scale, double &shift) {
    double sc = (__dsub_rn(smax, smin) > 2.220446049250313e-16) ? __ddiv_rn(1.0, __dsub_rn(smax, smin)) : 0.0;
    sc = (double)(float)sc;
    scale = sc;
    shift = __dsub_rn(0.0, (double)(float)__dmul_rn(smin, sc));
}

// ------------------------------------------------------------------------------------------------
// :43  blb = np >= 0.5 ; min/max of the two HV channels over the whole map
__global__ void k_threshold_minmax(const float *__restrict__ pred, int C, int off, int N,
                                   unsigned char *__restrict__ fg, PPStats *st) {
    int m = blockIdx.y;
    const float *pm = pred + (size_t)m * N * C + off;
    unsigned char *f = fg + (size_t)m * N;
    float hmin = INFINITY, hmax = -INFINITY, vmin = INFINITY, vmax = -INFINITY;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const float *px = pm + (size_t)p * C;
        float a = px[0], h = px[1], v = px[2];
        f[p] = a >= 0.5f ? 1 : 0;
        hmin = fminf(hmin, h); hmax = fmaxf(hmax, h);
        vmin = fminf(vmin, v); vmax = fmaxf(vmax, v);
    }
    for (int o = 16; o; o >>= 1) {
        hmin = fminf(hmin, __shfl_xor_sync(0xffffffffu, hmin, o));
        hmax = fmaxf(hmax, __shfl_xor_sync(0xffffffffu, hmax, o));
        vmin = fminf(vmin, __shfl_xor_sync(0xffffffffu, vmin, o));
        vmax = fmaxf(vmax, __shfl_xor_sync(0xffffffffu, vmax, o));
    }
    if ((threadIdx.x & 31) == 0 && hmin <= hmax) {
        atomicMin(&st[m].hmin, fkey(hmin)); atomicMax(&st[m].hmax, fkey(hmax));
        atomicMin(&st[m].vmin, fkey(vmin)); atomicMax(&st[m].vmax, fkey(vmax));
    }
}

// ------------------------------------------------------------------------------------------------
// 4-connected component labelling by union-find (uf.cuh); root = smallest linear index of the component,
// i.e. the component's first pixel in raster order (what scipy.ndimage.label numbers by).

// inv = 0: label pixels where src != 0 ; inv = 1: label pixels where src == 0 (for hole filling)
__global__ void k_ccl_init(const unsigned char *__restrict__ src, int inv, int N, int *__restrict__ L) {
    int m = blockIdx.y;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        bool on = (src[(size_t)m * N + p] != 0) != (inv != 0);
        L[(size_t)m * N + p] = on ? p : -1;
    }
}
__global__ void k_ccl_merge(int H, int W, int *__restrict__ Lall) {
    int m = blockIdx.y, N = H * W;
    int *L = Lall + (size_t)m * N;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        if (L[p] < 0) continue;
        int y = p / W, x = p - y * W;
        if (x > 0 && L[p - 1] >= 0) uf_union(L, p, p - 1);
        if (y > 0 && L[p - W] >= 0) uf_union(L, p, p - W);
    }
}
// flatten + component sizes (indexed by root pixel)
__global__ void k_ccl_flatten_count(int N, int *__restrict__ Lall, int *__restrict__ size_all) {
    int m = blockIdx.y;
    int *L = Lall + (size_t)m * N;
    int *sz = size_all + (size_t)m * N;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        if (L[p] < 0) continue;
        int r = uf_find(L, p);
        L[p] = r;  // racy-but-benign: only ever replaces a parent by an ancestor
        atomicAdd(&sz[r], 1);
    }
}

// :46-47 remove components < 10 px and binarise; register surviving blobs for the watershed
__global__ void k_blob_filter(int N, const int *__restrict__ Lall, const int *__restrict__ size_all,
                              unsigned char *__restrict__ fg_all, int *__restrict__ blob_of_root_all,
                              int *__restrict__ blob_root_all, int max_blobs, PPStats *st) {
    int m = blockIdx.y;
    const int *L = Lall + (size_t)m * N;
    const int *sz = size_all + (size_t)m * N;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        int r = L[p];
        bool keep = r >= 0 && sz[r] >= 10;
        fg_all[(size_t)m * N + p] = keep ? 1 : 0;
        if (keep && r == p) {
            int k = atomicAdd(&st[m].nblobs, 1);
            blob_of_root_all[(size_t)m * N + p] = k;
            if (k < max_blobs) blob_root_all[(size_t)m * max_blobs + k] = p;
        }
    }
}
__global__ void k_blob_bbox(int H, int W, const int *__restrict__ Lall, const unsigned char *__restrict__ fg_all,
                            const int *__restrict__ blob_of_root_all, int4 *__restrict__ bbox_all, int max_blobs) {
    int m = blockIdx.y, N = H * W;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        if (!fg_all[(size_t)m * N + p]) continue;
        int k = blob_of_root_all[(size_t)m * N + Lall[(size_t)m * N + p]];
        int y = p / W, x = p - y * W;
        int *bb = (int *)&bbox_all[(size_t)m * max_blobs + k];
        atomicMin(bb + 0, y); atomicMin(bb + 1, x); atomicMax(bb + 2, y); atomicMax(bb + 3, x);
    }
}
__global__ void k_bbox_init(int4 *bbox, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) bbox[i] = make_int4(0x7fffffff, 0x7fffffff, -1, -1);
}

// ------------------------------------------------------------------------------------------------
// :49-57 normalize(hv) -> Sobel(ksize=21), float64, BORDER_REFLECT_101 (SURVEY.md App. A.4-5)
__constant__ double c_deriv[21] = {-1, -18, -152, -798, -2907, -7752, -15504, -23256, -25194, -16796, 0,
                                   16796, 25194, 23256, 15504, 7752, 2907, 798, 152, 18, 1};
__constant__ double c_smooth[21] = {1, 20, 190, 1140, 4845, 15504, 38760, 77520, 125970, 167960, 184756,
                                    167960, 125970, 77520, 38760, 15504, 4845, 1140, 190, 20, 1};

__device__ __forceinline__ int reflect101(int i, int n) {
    if (n == 1) return 0;
    while (i < 0 || i >= n) i = (i < 0) ? -i : 2 * (n - 1) - i;
    return i;
}

constexpr int SB_TW = 32, SB_TH = 16, SB_R = 10;
constexpr int SB_SW = SB_TW + 2 * SB_R, SB_SH = SB_TH + 2 * SB_R;

__global__ void __launch_bounds__(256)
k_sobel21(const float *__restrict__ pred, int C, int off, int H, int W, double *__restrict__ sobh_all,
          double *__restrict__ sobv_all, PPStats *st) {
    __shared__ float s_h[SB_SH][SB_SW + 1];
    __shared__ float s_v[SB_SH][SB_SW + 1];
    __shared__ double r_h[SB_SH][SB_TW];
    __shared__ double r_v[SB_SH][SB_TW];
    int m = blockIdx.z, N = H * W;
    const float *pm = pred + (size_t)m * N * C + off;
    int x0 = blockIdx.x * SB_TW, y0 = blockIdx.y * SB_TH;
    double sc_h, sh_h, sc_v, sh_v;
    minmax_scale((double)fkey_inv(st[m].hmin), (double)fkey_inv(st[m].hmax), sc_h, sh_h);
    minmax_scale((double)fkey_inv(st[m].vmin), (double)fkey_inv(st[m].vmax), sc_v, sh_v);
    // stage the normalised source tile (with reflected halo)
    for (int i = threadIdx.x; i < SB_SH * SB_SW; i += blockDim.x) {
        int ty = i / SB_SW, tx = i - ty * SB_SW;
        int y = reflect101(y0 + ty - SB_R, H), x = reflect101(x0 + tx - SB_R, W);
        const float *px = pm + (size_t)(y * W + x) * C;
        s_h[ty][tx] = (float)__fma_rn((double)px[1], sc_h, sh_h);
        s_v[ty][tx] = (float)__fma_rn((double)px[2], sc_v, sh_v);
    }
    __syncthreads();
    // row pass: acc = sum_{k=0..20} kx[k]*src[x+k-10], left to right, from 0 (no FMA)
    for (int i = threadIdx.x; i < SB_SH * SB_TW; i += blockDim.x) {
        int ty = i / SB_TW, tx = i - ty * SB_TW;
        double ah = 0.0, av = 0.0;
#pragma unroll
        for (int k = 0; k < 21; ++k) {
            ah = __dadd_rn(ah, __dmul_rn(c_deriv[k], (double)s_h[ty][tx + k]));
            av = __dadd_rn(av, __dmul_rn(c_smooth[k], (double)s_v[ty][tx + k]));
        }
        r_h[ty][tx] = ah;
        r_v[ty][tx] = av;
    }
    __syncthreads();
    // column pass: ky[10]*r[y] + sum_{k=1..10} ky[10+k]*(r[y+k] (+|-) r[y-k])
    double lmin_h = INFINITY, lmax_h = -INFINITY, lmin_v = INFINITY, lmax_v = -INFINITY;
    for (int i = threadIdx.x; i < SB_TH * SB_TW; i += blockDim.x) {
        int ty = i / SB_TW, tx = i - ty * SB_TW;
        int y = y0 + ty, x = x0 + tx;
        if (y >= H || x >= W) continue;
        int c = ty + SB_R;
        double ah = __dmul_rn(c_smooth[10], r_h[c][tx]);
        double av = __dmul_rn(c_deriv[10], r_v[c][tx]);
#pragma unroll
        for (int k = 1; k <= 10; ++k) {
            ah = __dadd_rn(ah, __dmul_rn(c_smooth[10 + k], __dadd_rn(r_h[c + k][tx], r_h[c - k][tx])));
            av = __dadd_rn(av, __dmul_rn(c_deriv[10 + k], __dsub_rn(r_v[c + k][tx], r_v[c - k][tx])));
        }
        sobh_all[(size_t)m * N + y * W + x] = ah;
        sobv_all[(size_t)m * N + y * W + x] = av;
        lmin_h = fmin(lmin_h, ah); lmax_h = fmax(lmax_h, ah);
        lmin_v = fmin(lmin_v, av); lmax_v = fmax(lmax_v, av);
    }
    for (int o = 16; o; o >>= 1) {
        lmin_h = fmin(lmin_h, __shfl_xor_sync(0xffffffffu, lmin_h, o));
        lmax_h = fmax(lmax_h, __shfl_xor_sync(0xffffffffu, lmax_h, o));
        lmin_v = fmin(lmin_v, __shfl_xor_sync(0xffffffffu, lmin_v, o));
        lmax_v = fmax(lmax_v, __shfl_xor_sync(0xffffffffu, lmax_v, o));
    }
    if ((threadIdx.x & 31) == 0 && lmin_h <= lmax_h) {
        atomicMin(&st[m].shmin, dkey(lmin_h)); atomicMax(&st[m].shmax, dkey(lmax_h));
        atomicMin(&st[m].svmin, dkey(lmin_v)); atomicMax(&st[m].svmax, dkey(lmax_v));
    }
}

// ------------------------------------------------------------------------------------------------
// :59-81  overall = max(1-norm(sobelh), 1-norm(sobelv)) - (1-blb), clamp; dist_in = (1-overall)*blb;
//         marker0 = clamp(blb - (overall >= 0.4), 0)
__global__ void k_energy(int N, const double *__restrict__ sobh_all, const double *__restrict__ sobv_all,
                         const unsigned char *__restrict__ fg_all, double *__restrict__ din_all,
                         unsigned char *__restrict__ mk0_all, const PPStats *st) {
    int m = blockIdx.y;
    double sc_h, sh_h, sc_v, sh_v;
    minmax_scale(dkey_inv(st[m].shmin), dkey_inv(st[m].shmax), sc_h, sh_h);
    minmax_scale(dkey_inv(st[m].svmin), dkey_inv(st[m].svmax), sc_v, sh_v);
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        size_t i = (size_t)m * N + p;
        float a = __fsub_rn(1.0f, (float)__fma_rn(sobh_all[i], sc_h, sh_h));
        float b = __fsub_rn(1.0f, (float)__fma_rn(sobv_all[i], sc_v, sh_v));
        float o32 = a > b ? a : b;
        int blb = fg_all[i];
        double o = __dsub_rn((double)o32, (double)(1 - blb));
        if (o < 0.0) o = 0.0;
        din_all[i] = __dmul_rn(__dsub_rn(1.0, o), (double)blb);
        int mk = blb - (o >= 0.4 ? 1 : 0);
        mk0_all[i] = mk > 0 ? 1 : 0;
    }
}

// :76  dist = -GaussianBlur(dist_in, (3,3), 0), float64, reflect-101.
// row pass (a*0.25 + b*0.5) + c*0.25 ; column pass b*0.5 + (a + c)*0.25   (pinned vs cv2)
__device__ __forceinline__ double blur_row(const double *row, int x, int W) {
    double a = row[reflect101(x - 1, W)], b = row[x], c = row[reflect101(x + 1, W)];
    return __dadd_rn(__dadd_rn(__dmul_rn(a, 0.25), __dmul_rn(b, 0.5)), __dmul_rn(c, 0.25));
}
__global__ void k_blur3(int H, int W, const double *__restrict__ din_all, double *__restrict__ dist_all) {
    int m = blockIdx.y, N = H * W;
    const double *din = din_all + (size_t)m * N;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        int y = p / W, x = p - y * W;
        double ra = blur_row(din + (size_t)reflect101(y - 1, H) * W, x, W);
        double rb = blur_row(din + (size_t)y * W, x, W);
        double rc = blur_row(din + (size_t)reflect101(y + 1, H) * W, x, W);
        double v = __dadd_rn(__dmul_rn(rb, 0.5), __dmul_rn(__dadd_rn(ra, rc), 0.25));
        dist_all[(size_t)m * N + p] = -v;
    }
}

// ------------------------------------------------------------------------------------------------
// :82 binary_fill_holes == NOT(background 4-connected to the image border)
__global__ void k_border_flag(int H, int W, const int *__restrict__ Lall, unsigned char *__restrict__ flag_all) {
    int m = blockIdx.y, N = H * W;
    int nb = 2 * (H + W);
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < nb; i += gridDim.x * blockDim.x) {
        int p;
        if (i < W) p = i;
        else if (i < 2 * W) p = (H - 1) * W + (i - W);
        else if (i < 2 * W + H) p = (i - 2 * W) * W;
        else p = (i - 2 * W - H) * W + W - 1;
        int r = Lall[(size_t)m * N + p];
        if (r >= 0) flag_all[(size_t)m * N + uf_find(Lall + (size_t)m * N, r)] = 1;
    }
}
__global__ void k_fill(int N, const unsigned char *__restrict__ mk0_all, const int *__restrict__ Lall,
                       const unsigned char *__restrict__ flag_all, unsigned char *__restrict__ out_all) {
    int m = blockIdx.y;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        size_t i = (size_t)m * N + p;
        unsigned char v = 1;
        if (!mk0_all[i]) {
            int r = uf_find(Lall + (size_t)m * N, p);
            v = flag_all[(size_t)m * N + r] ? 0 : 1;
        }
        out_all[i] = v;
    }
}

// :84 MORPH_OPEN with the 5x5 ellipse  00100/11111/11111/11111/00100 ; out-of-image taps ignored
template <bool ERODE>
__global__ void k_morph5(int H, int W, const unsigned char *__restrict__ src_all, unsigned char *__restrict__ dst_all) {
    int m = blockIdx.y, N = H * W;
    const unsigned char *src = src_all + (size_t)m * N;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        int y = p / W, x = p - y * W;
        bool v = ERODE;
#pragma unroll
        for (int j = -2; j <= 2; ++j) {
            int yy = y + j;
            if (yy < 0 || yy >= H) continue;
            int r = (j == -2 || j == 2) ? 0 : 2;
            for (int i = -r; i <= r; ++i) {
                int xx = x + i;
                if (xx < 0 || xx >= W) continue;
                bool s = src[yy * W + xx] != 0;
                if (ERODE) v = v && s; else v = v || s;
            }
        }
        dst_all[(size_t)m * N + p] = v ? 1 : 0;
    }
}

// ------------------------------------------------------------------------------------------------
// :85-86 scipy label numbering: id = 1 + rank of the component's first pixel among all first pixels
__global__ void k_row_roots(int H, int W, const int *__restrict__ Lall, int *__restrict__ rowcnt_all) {
    int m = blockIdx.y, N = H * W;
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int y = warp; y < H; y += nwarps) {
        int c = 0;
        for (int x = lane; x < W; x += 32) c += (Lall[(size_t)m * N + y * W + x] == y * W + x);
        for (int o = 16; o; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
        if (lane == 0) rowcnt_all[(size_t)m * H + y] = c;
    }
}
// exclusive scan over rows, one block per map
__global__ void k_row_scan(int H, int *__restrict__ rowcnt_all, PPStats *st) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    int m = blockIdx.x;
    int *rc = rowcnt_all + (size_t)m * H;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < H; base += blockDim.x) {
        int y = base + threadIdx.x;
        int v = y < H ? rc[y] : 0, incl = v;
        int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        for (int o = 1; o < 32; o <<= 1) {
            int t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        if (lane == 31) s_warp[w] = incl;
        __syncthreads();
        if (w == 0) {
            int nw = blockDim.x >> 5;
            int t = lane < nw ? s_warp[lane] : 0, ti = t;
            for (int o = 1; o < 32; o <<= 1) {
                int u = __shfl_up_sync(0xffffffffu, ti, o);
                if (lane >= o) ti += u;
            }
            s_warp[lane] = ti - t;  // exclusive prefix of warp totals
        }
        __syncthreads();
        int excl = s_carry + s_warp[w] + incl - v;
        if (y < H) rc[y] = excl;
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) s_carry = excl + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) st[m].nroots = s_carry;
}
__global__ void k_assign_ids(int H, int W, const int *__restrict__ Lall, const int *__restrict__ rowoff_all,
                             int *__restrict__ id_all) {
    int m = blockIdx.y, N = H * W;
    int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
    int nwarps = (gridDim.x * blockDim.x) >> 5;
    for (int y = warp; y < H; y += nwarps) {
        int base = rowoff_all[(size_t)m * H + y];
        for (int x0 = 0; x0 < W; x0 += 32) {
            int x = x0 + lane;
            bool root = x < W && Lall[(size_t)m * N + y * W + x] == y * W + x;
            unsigned int b = __ballot_sync(0xffffffffu, root);
            if (root) id_all[(size_t)m * N + y * W + x] = base + __popc(b & ((1u << lane) - 1)) + 1;
            base += __popc(b);
        }
    }
}
// marker labels after remove_small(10); skimage then applies markers * mask; inst starts as markers
__global__ void k_marker_labels(int N, const int *__restrict__ Lall, const int *__restrict__ size_all,
                                const int *__restrict__ id_all, const unsigned char *__restrict__ fg_all,
                                int *__restrict__ inst_all) {
    int m = blockIdx.y;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        size_t i = (size_t)m * N + p;
        int r = Lall[i], v = 0;
        if (r >= 0 && size_all[(size_t)m * N + r] >= 10 && fg_all[i]) v = id_all[(size_t)m * N + r];
        inst_all[i] = v;
    }
}

// A blob that holds exactly one marker label is flooded entirely by that label whatever the order
// (the blob is 4-connected), and a blob without markers stays 0: only blobs with >= 2 distinct labels
// need the ordered flood below.  lab_range[k] = (min,max) marker label inside blob k.
__global__ void k_blob_marker_range(int N, const int *__restrict__ inst_all, const int *__restrict__ L1_all,
                                    const int *__restrict__ blob_of_root_all, int2 *__restrict__ range_all, int max_blobs) {
    int m = blockIdx.y;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        int lab = inst_all[(size_t)m * N + p];
        if (lab <= 0) continue;
        int k = blob_of_root_all[(size_t)m * N + L1_all[(size_t)m * N + p]];
        int *r = (int *)&range_all[(size_t)m * max_blobs + k];
        atomicMin(r, lab);
        atomicMax(r + 1, lab);
    }
}
__global__ void k_blob_fill_single(int N, int *__restrict__ inst_all, const unsigned char *__restrict__ fg_all,
                                   const int *__restrict__ L1_all, const int *__restrict__ blob_of_root_all,
                                   const int2 *__restrict__ range_all, int max_blobs) {
    int m = blockIdx.y;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        if (!fg_all[(size_t)m * N + p]) continue;
        int k = blob_of_root_all[(size_t)m * N + L1_all[(size_t)m * N + p]];
        int2 r = range_all[(size_t)m * max_blobs + k];
        if (r.y > 0 && r.x == r.y) inst_all[(size_t)m * N + p] = r.y;
    }
}
__global__ void k_range_init(int2 *r, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) r[i] = make_int2(0x7fffffff, 0);
}

// ------------------------------------------------------------------------------------------------
// :88 skimage.segmentation.watershed(dist, markers, mask=blb)  (0.17.2; connectivity 1, no
// compactness, no watershed line): a priority flood ordered by (value, age) with the label written
// at push time.  Flooding never leaves a 4-connected component of the mask and entries of different
// components never compare in a way that matters, so each surviving blob is flooded independently
// and exactly by one thread with a private binary heap (same sift rules as heap_general.pxi).
struct __align__(16) HeapItem { double v; int age; int idx; };

// (value, age), then raster index: only age-0 marker pixels can tie on (value, age), and they pop in raster order as in
// the shared-memory floods (DESIGN.md 2)
__device__ __forceinline__ bool h_smaller(const HeapItem &a, const HeapItem &b) {
    if (a.v != b.v) return a.v < b.v;
    if (a.age != b.age) return a.age < b.age;
    return a.idx < b.idx;
}

// 4-ary min-heap on (value, age, idx): the first WS_CAP entries (the hot top levels) live in shared memory,
// the rest in the blob's slice of the global arena.  Keys are a strict total order, so the pop sequence -- all
// that the flood depends on -- is the same as for skimage's binary heap (apart from equal-valued marker pixels,
// which skimage pops in heap-layout order, see DESIGN.md).
constexpr int WS_CAP = 2048;
struct Heap4 {
    HeapItem *s, *g;
    int n;
    __device__ __forceinline__ HeapItem get(int i) const { return i < WS_CAP ? s[i] : g[i - WS_CAP]; }
    __device__ __forceinline__ void set(int i, const HeapItem &e) { if (i < WS_CAP) s[i] = e; else g[i - WS_CAP] = e; }
    __device__ __forceinline__ void push(const HeapItem &e) {
        int i = n++;
        while (i > 0) {
            int p = (i - 1) >> 2;
            HeapItem pe = get(p);
            if (!h_smaller(e, pe)) break;
            set(i, pe);
            i = p;
        }
        set(i, e);
    }
    __device__ __forceinline__ HeapItem pop() {
        HeapItem top = get(0);
        HeapItem last = get(--n);
        int i = 0;
        while (true) {
            int c = 4 * i + 1;
            if (c >= n) break;
            HeapItem best = get(c);
            int bi = c;
            int ce = min(c + 4, n);
            for (int j = c + 1; j < ce; ++j) {
                HeapItem e = get(j);
                if (h_smaller(e, best)) { best = e; bi = j; }
            }
            if (!h_smaller(best, last)) break;
            set(i, best);
            i = bi;
        }
        if (n > 0) set(i, last);
        return top;
    }
};

__global__ void __launch_bounds__(32)
k_watershed(int H, int W, const double *__restrict__ dist_all, const unsigned char *__restrict__ fg_all,
            const int *__restrict__ L1_all, const int *__restrict__ size1_all,
            const int *__restrict__ blob_root_all, const int4 *__restrict__ bbox_all,
            const int2 *__restrict__ range_all, int max_blobs,
            HeapItem *__restrict__ heap_all, int *inst_all, PPStats *st) {
    extern __shared__ __align__(16) unsigned char ws_smem[];
    int m = blockIdx.y, N = H * W;
    int k = blockIdx.x;  // one blob per warp-sized block; lane 0 runs the (inherently sequential) flood
    int nb = st[m].nblobs;
    if (nb > max_blobs) nb = max_blobs;
    if (k >= nb) return;
    { int2 rg = range_all[(size_t)m * max_blobs + k]; if (rg.y == 0 || rg.x == rg.y) return; }
    const int lane = threadIdx.x;
    const double *dist = dist_all + (size_t)m * N;
    const unsigned char *fg = fg_all + (size_t)m * N;
    const int *L1 = L1_all + (size_t)m * N;
    int *inst = inst_all + (size_t)m * N;
    int root = blob_root_all[(size_t)m * max_blobs + k];
    int bsize = size1_all[(size_t)m * N + root];
    int4 bb = bbox_all[(size_t)m * max_blobs + k];
    int goff = 0;
    if (lane == 0) goff = atomicAdd(&st[m].heap_top, bsize);
    goff = __shfl_sync(0xffffffffu, goff, 0);
    Heap4 hp;
    hp.s = reinterpret_cast<HeapItem *>(ws_smem);
    hp.g = heap_all + (size_t)m * N + goff;
    hp.n = 0;
    // marker pixels of this blob, pushed in raster order (age 0); the warp scans the bbox 32 px at a time
    const int bw = bb.w - bb.y + 1, bh = bb.z - bb.x + 1, area = bw * bh;
    for (int base = 0; base < area; base += 32) {
        int i = base + lane;
        bool is = false;
        int p = 0;
        double dv = 0.0;
        if (i < area) {
            int yy = bb.x + i / bw, xx = bb.y + i % bw;
            p = yy * W + xx;
            is = L1[p] == root && inst[p] != 0;
            if (is) dv = dist[p];
        }
        unsigned int msk = __ballot_sync(0xffffffffu, is);
        while (msk) {
            int src = __ffs(msk) - 1;
            msk &= msk - 1;
            int pp = __shfl_sync(0xffffffffu, p, src);
            double dd = __shfl_sync(0xffffffffu, dv, src);
            if (lane == 0) { HeapItem e; e.v = dd; e.age = 0; e.idx = pp; hp.push(e); }
        }
    }
    if (lane == 0) {
        int age = 1;
        while (hp.n > 0) {
            HeapItem e = hp.pop();
            const int y = e.idx / W, x = e.idx - y * W;
            const int lab = inst[e.idx];
            // neighbour order up, left, right, down; label at push time
            int q[4] = {y > 0 ? e.idx - W : -1, x > 0 ? e.idx - 1 : -1, x < W - 1 ? e.idx + 1 : -1,
                        y < H - 1 ? e.idx + W : -1};
            bool take[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) take[j] = q[j] >= 0 && fg[q[j]] && inst[q[j]] == 0;
            double dv[4];
#pragma unroll
            for (int j = 0; j < 4; ++j) dv[j] = take[j] ? dist[q[j]] : 0.0;
#pragma unroll
            for (int j = 0; j < 4; ++j)
                if (take[j]) {
                    age += 1;
                    inst[q[j]] = lab;
                    HeapItem ne; ne.v = dv[j]; ne.age = age; ne.idx = q[j];
                    hp.push(ne);
                }
        }
    }
}

// Patch-sized maps: one CTA per map keeps the per-pixel flood state (-1 outside the mask, 0 unlabelled,
// >0 label) as int16 in shared memory, plus the hot top of one heap per warp; warps pull blobs of the
// map from a shared queue (large blobs first).  Same flood, same order -- only the memory it lives in
// differs from k_watershed, which remains the path for maps too large for shared memory.
constexpr int WT_WARPS = 8;
constexpr int WT_BIG = 2048;      // blobs >= this many px are flooded by warp 0 with the large heap
constexpr int WT_SMALL_CAP = 256; // shared-memory heap entries of warps 1..7 (the rest spills to global)

// Heap entry for maps with < 65536 px, one 64-bit word: [ fkey(float(priority)) | age:16 | idx:16 ].
// float() is monotone, so when the high words differ the u64 order IS the (fp64 value, age) order; when
// they are equal the exact fp64 priorities are fetched and compared, then (age, idx).  Entries of one
// blob therefore pop in exactly the order of skimage's (value, age) heap (equal-valued age-0 marker
// pixels excepted, DESIGN.md 2).  1-based 4-ary heap: children of i are 4i-2..4i+1 (one aligned 32-byte
// group), parent of j is (j+2)>>2; slots past the end hold ~0 so a full group can be read blindly.
typedef unsigned long long u64;
struct HeapQ {
    u64 *s;              // shared part, slots [1, cap]
    u64 *g;              // global spill, slots (cap, ...)
    const double *dist;
    int n, cap;
    __device__ __forceinline__ bool less_exact(u64 a, u64 b) const {
        const double da = dist[(unsigned int)a & 0xffffu], db = dist[(unsigned int)b & 0xffffu];
        if (da != db) return da < db;
        return (unsigned int)a < (unsigned int)b;
    }
    __device__ __forceinline__ bool less(u64 a, u64 b) const {
        if ((a >> 32) != (b >> 32)) return a < b;
        return less_exact(a, b);
    }
    __device__ __forceinline__ u64 get(int i) const { return i <= cap ? s[i] : g[i - cap]; }
    __device__ __forceinline__ void set(int i, u64 e) { if (i <= cap) s[i] = e; else g[i - cap] = e; }
    __device__ __forceinline__ void push(u64 e) {
        int j = ++n;
        while (j > 1) {
            const int p = (j + 2) >> 2;
            const u64 pe = get(p);
            if (!less(e, pe)) break;
            set(j, pe);
            j = p;
        }
        set(j, e);
    }
    __device__ __forceinline__ u64 pop() {
        const u64 top = get(1);
        const u64 last = get(n);
        set(n, ~0ull);
        --n;
        if (n == 0) return top;
        int i = 1;
        while (true) {
            const int c = 4 * i - 2;
            if (c > n) break;
            u64 best;
            int bi;
            if (c + 3 <= cap) {  // whole child group in shared memory (slots past n read as ~0)
                const ulonglong2 q0 = *reinterpret_cast<const ulonglong2 *>(s + c);
                const ulonglong2 q1 = *reinterpret_cast<const ulonglong2 *>(s + c + 2);
                u64 m0 = q0.x < q0.y ? q0.x : q0.y, m1 = q1.x < q1.y ? q1.x : q1.y;
                int i0 = q0.x < q0.y ? c : c + 1, i1 = q1.x < q1.y ? c + 2 : c + 3;
                best = m0 < m1 ? m0 : m1;
                bi = m0 < m1 ? i0 : i1;
                const unsigned int kb = (unsigned int)(best >> 32);
                const int same = ((unsigned int)(q0.x >> 32) == kb) + ((unsigned int)(q0.y >> 32) == kb) +
                                 ((unsigned int)(q1.x >> 32) == kb) + ((unsigned int)(q1.y >> 32) == kb);
                if (same > 1 && kb != 0xffffffffu) {  // fp32 tie among the children: decide exactly
                    best = q0.x; bi = c;
                    if (c + 1 <= n && less(q0.y, best)) { best = q0.y; bi = c + 1; }
                    if (c + 2 <= n && less(q1.x, best)) { best = q1.x; bi = c + 2; }
                    if (c + 3 <= n && less(q1.y, best)) { best = q1.y; bi = c + 3; }
                }
            } else {
                best = get(c); bi = c;
                const int ce = min(c + 3, n);
                for (int j = c + 1; j <= ce; ++j) { const u64 e = get(j); if (less(e, best)) { best = e; bi = j; } }
            }
            if (!less(best, last)) break;
            set(i, best);
            i = bi;
        }
        set(i, last);
        return top;
    }
};

template <bool KK>
__global__ void __launch_bounds__(WT_WARPS * 32)
k_watershed_tile(int H, int W, int big_cap, const double *__restrict__ dist_all,
                 const unsigned char *__restrict__ fg_all, const int *__restrict__ L1_all,
                 const int *__restrict__ size1_all, const int *__restrict__ blob_root_all,
                 const int4 *__restrict__ bbox_all, const int2 *__restrict__ range_all, int max_blobs,
                 HeapItem *__restrict__ heap_all, int *__restrict__ inst_all, PPStats *st) {
    extern __shared__ __align__(16) unsigned char wt_smem[];
    __shared__ int s_next[2];
    // y = idx / W for idx < 2^16 as umulhi(idx, ceil(2^32 / W)) + (idx & wone); for W = 1 the multiplier (2^32) does not
    // fit in 32 bits, so it is 0 there and wone = ~0 passes idx through.
    const unsigned int wmagic = W > 1 ? (unsigned int)((0x100000000ull + (unsigned)W - 1) / (unsigned)W) : 0u;
    const unsigned int wone = W > 1 ? 0u : 0xffffffffu;
    const int m = blockIdx.x, N = H * W;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    // layout: heaps (u64, 16-byte aligned groups) | kk (float per px, optional) | state (int16 per px)
    u64 *heaps = reinterpret_cast<u64 *>(wt_smem);
    const size_t heap_slots = (size_t)(big_cap + 4) + (size_t)(WT_WARPS - 1) * (WT_SMALL_CAP + 4);
    float *kk = reinterpret_cast<float *>(wt_smem + heap_slots * 8);
    short *state = reinterpret_cast<short *>(wt_smem + heap_slots * 8 + (KK ? (((size_t)N * 4 + 15) & ~(size_t)15) : 0));
    const double *dist = dist_all + (size_t)m * N;
    const unsigned char *fg = fg_all + (size_t)m * N;
    const int *L1 = L1_all + (size_t)m * N;
    int *inst = inst_all + (size_t)m * N;
    for (int p = threadIdx.x; p < N; p += blockDim.x) {
        state[p] = fg[p] ? (short)inst[p] : (short)-1;
        if (KK) kk[p] = (float)dist[p] + 0.0f;  // +0.0f: -0.0 and +0.0 are equal priorities, give them one key
    }
    for (size_t i = threadIdx.x; i < heap_slots; i += blockDim.x) heaps[i] = ~0ull;
    if (threadIdx.x < 2) s_next[threadIdx.x] = 0;
    __syncthreads();
    int nb = st[m].nblobs;
    if (nb > max_blobs) nb = max_blobs;
    HeapQ hp;
    hp.dist = dist;
    // warps 0,1: large blobs, one after the other, each with half of the large heap region;
    // warps 2..7: the small ones.  (Slot index c = 4i-2 of every region is 16-byte aligned.)
    const int pass = warp < 2 ? 0 : 1;
    const int half_cap = ((big_cap + 4) / 2 - 4) & ~3;
    hp.s = warp < 2 ? heaps + (size_t)warp * ((big_cap + 4) / 2)
                    : heaps + (big_cap + 4) + (size_t)(warp - 1) * (WT_SMALL_CAP + 4);
    hp.cap = warp < 2 ? half_cap : WT_SMALL_CAP;
    while (true) {
        int k = 0;
        if (lane == 0) k = atomicAdd(&s_next[pass], 1);
        k = __shfl_sync(0xffffffffu, k, 0);
        if (k >= nb) break;
        const int root = blob_root_all[(size_t)m * max_blobs + k];
        const int bsize = size1_all[(size_t)m * N + root];
        if ((bsize >= WT_BIG) != (pass == 0)) continue;
        { const int2 rg = range_all[(size_t)m * max_blobs + k]; if (rg.y == 0 || rg.x == rg.y) continue; }
        const int4 bb = bbox_all[(size_t)m * max_blobs + k];
        int goff = 0;
        if (lane == 0) goff = atomicAdd(&st[m].heap_top, bsize);
        goff = __shfl_sync(0xffffffffu, goff, 0);
        hp.g = reinterpret_cast<u64 *>(heap_all + (size_t)m * N + goff);  // 16 B/px arena >= 8 B/entry
        hp.n = 0;
        const int bw = bb.w - bb.y + 1, bh = bb.z - bb.x + 1, area = bw * bh;
        for (int base = 0; base < area; base += 32) {
            int i = base + lane;
            bool is = false;
            int p = 0;
            unsigned int kv = 0;
            if (i < area) {
                int yy = bb.x + i / bw, xx = bb.y + i % bw;
                p = yy * W + xx;
                is = state[p] > 0 && L1[p] == root;
                if (is) kv = fkey(KK ? kk[p] : (float)dist[p] + 0.0f);
            }
            unsigned int msk = __ballot_sync(0xffffffffu, is);
            while (msk) {
                int src = __ffs(msk) - 1;
                msk &= msk - 1;
                int pp = __shfl_sync(0xffffffffu, p, src);
                unsigned int kq = __shfl_sync(0xffffffffu, kv, src);
                if (lane == 0) hp.push(((u64)kq << 32) | (u64)(unsigned int)pp);  // age 0
            }
        }
        if (lane == 0) {
            unsigned int age = 1;
            const long long t0 = clock64();
            int npop = 0;
            while (hp.n > 0) {
                const u64 e = hp.pop();
                ++npop;
                const int idx = (int)((unsigned int)e & 0xffffu);
                const int y = (int)(__umulhi((unsigned int)idx, wmagic) + ((unsigned int)idx & wone)), x = idx - y * W;
                const short lab = state[idx];
                const int q[4] = {y > 0 ? idx - W : -1, x > 0 ? idx - 1 : -1, x < W - 1 ? idx + 1 : -1, y < H - 1 ? idx + W : -1};
                bool take[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) take[j] = q[j] >= 0 && state[q[j]] == 0;
                unsigned int kq[4];
#pragma unroll
                for (int j = 0; j < 4; ++j) kq[j] = take[j] ? fkey(KK ? kk[q[j]] : (float)__ldg(dist + q[j]) + 0.0f) : 0u;
#pragma unroll
                for (int j = 0; j < 4; ++j)
                    if (take[j]) {
                        age += 1;
                        state[q[j]] = lab;
                        hp.push(((u64)kq[j] << 32) | (u64)((age << 16) | (unsigned int)q[j]));
                    }
            }
            atomicAdd(&st[m].pad[0], npop);                                  // diagnostics: pops / flood cycles per map
            atomicMax(&st[m].pad[1], (int)((clock64() - t0) >> 10));
        }
        __syncwarp();
    }
    __syncthreads();
    for (int p = threadIdx.x; p < N; p += blockDim.x) { short v = state[p]; inst[p] = v > 0 ? (int)v : 0; }
}

// Calendar-queue variant of the per-map flood (used when the fp32 priority table fits in shared memory).
// The heap is replaced by NB buckets over the map's priority range (bucket index monotone in the
// priority), each an exactly-ordered singly linked list threaded through next[px], plus a two-level
// bitmap of non-empty buckets: pop = two find-first-set + unlink the head, push = walk the (short)
// bucket list to the insertion point.  Ordering inside a bucket uses the same exact comparison as the
// heap (fp32 key, then fp64 priority); an entry is placed after all entries with an equal priority,
// i.e. in push (= age) order.  The pop sequence is therefore again the (value, age) order.
constexpr int WC_NB_BIG = 2048, WC_NB_SMALL = 256;
constexpr unsigned short WC_NIL = 0xffffu;

// One record per pixel, one 8-byte shared-memory access: fp32 priority key, link to the next pixel of its bucket list,
// flood state (-1 outside the mask, 0 unlabelled, > 0 label).  Walking a bucket list, testing a neighbour and popping a
// head each used to chase two or three separate arrays (kk / nxt / state); with ~30 dependent shared-memory accesses per
// popped pixel the flood is pure latency, so halving them is what pays.
struct __align__(8) PxRec { float key; unsigned short next; short state; };

__global__ void __launch_bounds__(WT_WARPS * 32)
k_watershed_cal(int H, int W, const double *__restrict__ dist_all, const unsigned char *__restrict__ fg_all,
                const int *__restrict__ L1_all, const int *__restrict__ size1_all, const int *__restrict__ blob_root_all,
                const int4 *__restrict__ bbox_all, const int2 *__restrict__ range_all, int max_blobs,
                int *__restrict__ inst_all, PPStats *st) {
    extern __shared__ __align__(16) unsigned char wc_smem[];
    __shared__ int s_next[2];
    __shared__ unsigned int s_kmin, s_kmax;
    const unsigned int wmagic = W > 1 ? (unsigned int)((0x100000000ull + (unsigned)W - 1) / (unsigned)W) : 0u;  // as in
    const unsigned int wone = W > 1 ? 0u : 0xffffffffu;                                                       // k_watershed_tile
    const int m = blockIdx.x, N = H * W;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const size_t n8 = ((size_t)N * 8 + 15) & ~(size_t)15;
    PxRec *px = reinterpret_cast<PxRec *>(wc_smem);
    unsigned char *qbase = wc_smem + n8;
    // per-warp queue storage: heads u16[NB] | bitmap u32[NB/32]
    const int NB = warp < 2 ? WC_NB_BIG : WC_NB_SMALL;
    const size_t big_bytes = WC_NB_BIG * 2 + WC_NB_BIG / 8, small_bytes = WC_NB_SMALL * 2 + WC_NB_SMALL / 8;
    unsigned char *mine = qbase + (warp < 2 ? warp * big_bytes : 2 * big_bytes + (warp - 2) * small_bytes);
    unsigned short *head = reinterpret_cast<unsigned short *>(mine);
    unsigned int *bitmap = reinterpret_cast<unsigned int *>(mine + NB * 2);
    const double *dist = dist_all + (size_t)m * N;
    const unsigned char *fg = fg_all + (size_t)m * N;
    const int *L1 = L1_all + (size_t)m * N;
    int *inst = inst_all + (size_t)m * N;
    if (threadIdx.x == 0) { s_kmin = 0xffffffffu; s_kmax = 0u; s_next[0] = s_next[1] = 0; }
    __syncthreads();
    unsigned int lmin = 0xffffffffu, lmax = 0u;
    for (int p = threadIdx.x; p < N; p += blockDim.x) {
        const bool f = fg[p] != 0;
        PxRec r;
        r.key = (float)dist[p] + 0.0f;  // +0.0f: -0.0 and +0.0 are equal priorities, give them one key
        r.next = WC_NIL;
        r.state = f ? (short)inst[p] : (short)-1;
        px[p] = r;
        if (f) { const unsigned int ky = fkey(r.key); lmin = min(lmin, ky); lmax = max(lmax, ky); }
    }
    for (int o = 16; o; o >>= 1) {
        lmin = min(lmin, __shfl_xor_sync(0xffffffffu, lmin, o));
        lmax = max(lmax, __shfl_xor_sync(0xffffffffu, lmax, o));
    }
    if (lane == 0) { atomicMin(&s_kmin, lmin); atomicMax(&s_kmax, lmax); }
    for (int i = lane; i < NB; i += 32) head[i] = WC_NIL;
    for (int i = lane; i < NB / 32; i += 32) bitmap[i] = 0u;
    __syncthreads();
    const float kmin = fkey_inv(s_kmin), kmax = fkey_inv(s_kmax);
    const float scale = kmax > kmin ? (float)NB / (kmax - kmin) : 0.f;
    int nb = st[m].nblobs;
    if (nb > max_blobs) nb = max_blobs;
    u64 summary = 0ull;  // bit j <=> bitmap[j] != 0   (NB/32 <= 64 words)

    auto bucket_of = [&](float k) {
        int b = (int)((k - kmin) * scale);
        return b < 0 ? 0 : (b >= NB ? NB - 1 : b);
    };
    // strict exact order "pixel q (key kq) before pixel c (key kc)" (equal => false): fp32 keys, exact fp64 on a tie
    auto precedes = [&](int q, float kq, int c, float kc) {
        if (kq != kc) return kq < kc;
        return dist[q] < dist[c];
    };
    // insert pixel q (key kq, its record's state already written) into its bucket list, after every entry of equal
    // priority (push = age order)
    auto q_push = [&](int q, float kq) {
        const int b = bucket_of(kq);
        unsigned short cur = head[b];
        if (cur == WC_NIL) {
            head[b] = (unsigned short)q; px[q].next = WC_NIL;
            bitmap[b >> 5] |= 1u << (b & 31);
            summary |= 1ull << (b >> 5);
            return;
        }
        PxRec rc = px[cur];
        if (precedes(q, kq, cur, rc.key)) { px[q].next = cur; head[b] = (unsigned short)q; return; }
        unsigned short prev = cur;
        cur = rc.next;
        while (cur != WC_NIL) {
            rc = px[cur];                               // key and link of the next entry in one access
            if (precedes(q, kq, cur, rc.key)) break;
            prev = cur; cur = rc.next;
        }
        px[q].next = cur; px[prev].next = (unsigned short)q;
    };

    // warps 0-1 take the large blobs first (their queues have 2048 buckets), then join the others on the small ones:
    // on nuclei-like maps every blob is small and two of the eight flood lanes used to sit idle
    for (int pass = warp < 2 ? 0 : 1; pass < 2; ++pass)
    while (true) {
        int k = 0;
        if (lane == 0) k = atomicAdd(&s_next[pass], 1);
        k = __shfl_sync(0xffffffffu, k, 0);
        if (k >= nb) break;
        const int root = blob_root_all[(size_t)m * max_blobs + k];
        const int bsize = size1_all[(size_t)m * N + root];
        if ((bsize >= WT_BIG) != (pass == 0)) continue;
        { const int2 rg = range_all[(size_t)m * max_blobs + k]; if (rg.y == 0 || rg.x == rg.y) continue; }
        const int4 bb = bbox_all[(size_t)m * max_blobs + k];
        const int bw = bb.w - bb.y + 1, bh = bb.z - bb.x + 1, area = bw * bh;
        for (int base = 0; base < area; base += 32) {  // marker pixels in raster order
            int i = base + lane;
            bool is = false;
            int p = 0;
            float kp = 0.f;
            if (i < area) {
                int yy = bb.x + i / bw, xx = bb.y + i % bw;
                p = yy * W + xx;
                const PxRec r = px[p];
                is = r.state > 0 && L1[p] == root;
                kp = r.key;
            }
            unsigned int msk = __ballot_sync(0xffffffffu, is);
            while (msk) {
                int src = __ffs(msk) - 1;
                msk &= msk - 1;
                int pp = __shfl_sync(0xffffffffu, p, src);
                float kk = __shfl_sync(0xffffffffu, kp, src);
                if (lane == 0) q_push(pp, kk);
            }
        }
        if (lane == 0) {
            const long long t0 = clock64();
            int npop = 0;
            while (summary) {
                // pop: first non-empty bucket, its head; the head's record gives the next head and the label
                const int j = __ffsll((long long)summary) - 1;
                const unsigned int w = bitmap[j];
                const int bit = __ffs((int)w) - 1, b = j * 32 + bit;
                const int idx = head[b];
                const PxRec e = px[idx];
                head[b] = e.next;
                if (e.next == WC_NIL) {
                    const unsigned int w2 = w & ~(1u << bit);
                    bitmap[j] = w2;
                    if (!w2) summary &= ~(1ull << j);
                }
                ++npop;
                const int y = (int)(__umulhi((unsigned int)idx, wmagic) + ((unsigned int)idx & wone)), x = idx - y * W;
                const short lab = e.state;
                const int q[4] = {y > 0 ? idx - W : -1, x > 0 ? idx - 1 : -1, x < W - 1 ? idx + 1 : -1, y < H - 1 ? idx + W : -1};
                PxRec nr[4];
#pragma unroll
                for (int jn = 0; jn < 4; ++jn) {  // the four neighbour records: independent loads, in flight together
                    nr[jn].state = -1; nr[jn].key = 0.f; nr[jn].next = WC_NIL;
                    if (q[jn] >= 0) nr[jn] = px[q[jn]];
                }
#pragma unroll
                for (int jn = 0; jn < 4; ++jn)  // up, left, right, down; label at push time
                    if (nr[jn].state == 0) { px[q[jn]].state = lab; q_push(q[jn], nr[jn].key); }
            }
            atomicAdd(&st[m].pad[0], npop);
            atomicMax(&st[m].pad[1], (int)((clock64() - t0) >> 10));
        }
        __syncwarp();
    }
    __syncthreads();
    for (int p = threadIdx.x; p < N; p += blockDim.x) { short v = px[p].state; inst[p] = v > 0 ? (int)v : 0; }
}

// ------------------------------------------------------------------------------------------------
// :120-181 per-instance bbox / area / coordinate sums / type histogram, then rows in ascending id
struct InstAcc { int rmin, cmin, rmax, cmax, area, pad; unsigned long long sx, sy; };

__global__ void k_acc_init(InstAcc *acc, size_t n) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i < n) { InstAcc a; a.rmin = a.cmin = 0x7fffffff; a.rmax = a.cmax = -1; a.area = 0; a.pad = 0; a.sx = a.sy = 0; acc[i] = a; }
}
__global__ void k_table_accum(int H, int W, const int *__restrict__ inst_all, const float *__restrict__ pred, int C,
                              int nr_types, InstAcc *__restrict__ acc_all, int *__restrict__ tcnt_all, int max_ids) {
    int m = blockIdx.y, N = H * W;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        int id = inst_all[(size_t)m * N + p];
        if (id <= 0 || id >= max_ids) continue;
        int y = p / W, x = p - y * W;
        InstAcc *a = acc_all + (size_t)m * max_ids + id;
        atomicMin(&a->rmin, y); atomicMin(&a->cmin, x); atomicMax(&a->rmax, y); atomicMax(&a->cmax, x);
        atomicAdd(&a->area, 1);
        atomicAdd(&a->sx, (unsigned long long)x);
        atomicAdd(&a->sy, (unsigned long long)y);
        if (nr_types > 0) {
            int t = (int)pred[((size_t)m * N + p) * C];  // astype(int32) truncation (:111)
            if (t >= 0 && t < nr_types) atomicAdd(&tcnt_all[((size_t)m * max_ids + id) * nr_types + t], 1);
        }
    }
}
// one block per map: ordered compaction of non-empty ids into table rows
__global__ void k_table_rows(const InstAcc *__restrict__ acc_all, const int *__restrict__ tcnt_all, int nr_types,
                             int max_ids, long long *__restrict__ table_all, int max_rows, int *__restrict__ nrows_out,
                             PPStats *st) {
    __shared__ int s_warp[32];
    __shared__ int s_carry;
    int m = blockIdx.x;
    int nid = st[m].nroots + 1;
    if (nid > max_ids) nid = max_ids;
    const InstAcc *acc = acc_all + (size_t)m * max_ids;
    if (threadIdx.x == 0) s_carry = 0;
    __syncthreads();
    for (int base = 0; base < nid; base += blockDim.x) {
        int id = base + threadIdx.x;
        int v = (id > 0 && id < nid && acc[id].area > 0) ? 1 : 0, incl = v;
        int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
        for (int o = 1; o < 32; o <<= 1) { int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
        if (lane == 31) s_warp[w] = incl;
        __syncthreads();
        if (w == 0) {
            int nw = blockDim.x >> 5;
            int t = lane < nw ? s_warp[lane] : 0, ti = t;
            for (int o = 1; o < 32; o <<= 1) { int u = __shfl_up_sync(0xffffffffu, ti, o); if (lane >= o) ti += u; }
            s_warp[lane] = ti - t;
        }
        __syncthreads();
        int row = s_carry + s_warp[w] + incl - v;
        if (v && row < max_rows) {
            InstAcc a = acc[id];
            long long *r = table_all + ((size_t)m * max_rows + row) * 10;
            r[0] = id; r[1] = a.rmin; r[2] = a.cmin; r[3] = a.rmax + 1; r[4] = a.cmax + 1;
            r[5] = a.area; r[6] = (long long)a.sx; r[7] = (long long)a.sy;
            long long type = -1, tc = 0;
            if (nr_types > 0) {
                // sorted by count desc, stable: ties -> smaller type id; if winner is 0 take runner-up
                const int *tcnt = tcnt_all + ((size_t)m * max_ids + id) * nr_types;
                int best = -1, second = -1;
                for (int t = 0; t < nr_types; ++t) {
                    int c = tcnt[t];
                    if (c == 0) continue;
                    if (best < 0 || c > tcnt[best]) { second = best; best = t; }
                    else if (second < 0 || c > tcnt[second]) second = t;
                }
                int pick = best;
                if (best == 0 && second >= 0) pick = second;
                type = pick;
                tc = pick >= 0 ? tcnt[pick] : 0;
            }
            r[8] = type; r[9] = tc;
        }
        __syncthreads();
        if (threadIdx.x == blockDim.x - 1) s_carry = row + v;
        __syncthreads();
    }
    if (threadIdx.x == 0) { st[m].nrows = s_carry; nrows_out[m] = s_carry; }
}

// ------------------------------------------------------------------------------------------------
static int g_flood_impl = 0;  // 0 auto (calendar queue > shared-memory heap > global heap), 1 no calendar queue, 2 global only
void postproc_set_flood_impl(int v) { g_flood_impl = v; }

const char *postproc_flood_name(int k) {
    switch (k) {
    case FLOOD_CAL: return "k_watershed_cal";
    case FLOOD_TILE_KK: return "k_watershed_tile<true>";
    case FLOOD_TILE: return "k_watershed_tile<false>";
    case FLOOD_GLOBAL: return "k_watershed";
    default: return "?";
    }
}

// Shared-memory plan of the per-map flood kernels for an N-px map.  The calendar queue holds one 8-byte record per
// pixel; the heap kernel holds the int16 flood state, optionally the fp32 key table (kk), the small-blob heaps and
// a large-blob heap of `cap` entries (capped at 16384, at least 1024 for the kernel to be worth running).
struct FloodPlan {
    size_t cal_bytes, tile_smem[2];  // tile_smem[kk]
    long long cap[2];
    bool cal_ok, tile_ok[2];
};
static const size_t kFloodBudget = 225 * 1024;

static FloodPlan flood_plan(int N, int max_ids) {
    FloodPlan f;
    const size_t state_bytes = (((size_t)N * 2 + 15) & ~(size_t)15), kk_bytes = (((size_t)N * 4 + 15) & ~(size_t)15);
    f.cal_bytes = (((size_t)N * 8 + 15) & ~(size_t)15) + 2 * (WC_NB_BIG * 2 + WC_NB_BIG / 8) +
                  (WT_WARPS - 2) * (WC_NB_SMALL * 2 + WC_NB_SMALL / 8);
    f.cal_ok = f.cal_bytes <= kFloodBudget && N < 65535 && max_ids < 32000;
    const size_t small_bytes = (size_t)(WT_WARPS - 1) * (WT_SMALL_CAP + 4) * 8;
    for (int kk = 0; kk < 2; ++kk) {
        const size_t fixed = state_bytes + (kk ? kk_bytes : 0) + small_bytes;
        long long cap = fixed + 64 < kFloodBudget ? (long long)((kFloodBudget - fixed) / 8) - 4 : 0;
        cap = std::min<long long>(cap & ~3ll, 16384);
        f.cap[kk] = cap;
        f.tile_smem[kk] = fixed + (size_t)(cap + 4) * 8;
        f.tile_ok[kk] = cap >= 1024 && N < 65536 && max_ids < 32000;
    }
    // the key table is used whenever it leaves room for a 2048-entry large heap
    f.tile_ok[1] = f.tile_ok[1] && state_bytes + kk_bytes + small_bytes + (2048 + 4) * 8 <= kFloodBudget;
    return f;
}

int postproc_flood(cudaStream_t stream, const PostprocBuffers &b, int n, int H, int W, int *inst, int choice) {
    const int N = H * W;
    const FloodPlan f = flood_plan(N, b.max_ids);
    int k = choice;
    if (k == FLOOD_AUTO) {  // patch-sized maps: per-map CTA with the flood state in shared memory; otherwise the generic kernel
        if (f.cal_ok && g_flood_impl == 0) k = FLOOD_CAL;
        else if (f.tile_ok[0] && g_flood_impl <= 1) k = f.tile_ok[1] ? FLOOD_TILE_KK : FLOOD_TILE;
        else k = FLOOD_GLOBAL;
    }
    HVN_CHECK(k >= FLOOD_CAL && k <= FLOOD_GLOBAL, -1, "postproc_flood: unknown flood kernel");
    HVN_CHECK(k != FLOOD_CAL || f.cal_ok, -1, "postproc_flood: the calendar-queue flood does not fit this map");
    HVN_CHECK(k != FLOOD_TILE_KK || f.tile_ok[1], -1, "postproc_flood: the heap flood with key table does not fit this map");
    HVN_CHECK(k != FLOOD_TILE || f.tile_ok[0], -1, "postproc_flood: the shared-memory heap flood does not fit this map");
    static bool attr = false;
    if (!attr) {
        HVN_CUDA(cudaFuncSetAttribute(k_watershed_tile<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFloodBudget + 64));
        HVN_CUDA(cudaFuncSetAttribute(k_watershed_tile<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFloodBudget + 64));
        HVN_CUDA(cudaFuncSetAttribute(k_watershed_cal, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)kFloodBudget + 64));
        attr = true;
    }
    PPStats *st = (PPStats *)b.stats;
    if (k == FLOOD_CAL) {
        k_watershed_cal<<<n, WT_WARPS * 32, f.cal_bytes, stream>>>(H, W, b.dist, b.fg, b.L1, b.size1, b.blob_root, (int4 *)b.bbox,
                                                                 (const int2 *)b.lab_range, b.max_blobs, inst, st);
    } else if (k == FLOOD_TILE_KK) {
        k_watershed_tile<true><<<n, WT_WARPS * 32, f.tile_smem[1], stream>>>(H, W, (int)f.cap[1], b.dist, b.fg, b.L1, b.size1,
            b.blob_root, (int4 *)b.bbox, (const int2 *)b.lab_range, b.max_blobs, (HeapItem *)b.heap, inst, st);
    } else if (k == FLOOD_TILE) {
        k_watershed_tile<false><<<n, WT_WARPS * 32, f.tile_smem[0], stream>>>(H, W, (int)f.cap[0], b.dist, b.fg, b.L1, b.size1,
            b.blob_root, (int4 *)b.bbox, (const int2 *)b.lab_range, b.max_blobs, (HeapItem *)b.heap, inst, st);
    } else {
        k_watershed<<<dim3((unsigned)b.max_blobs, (unsigned)n), 32, WS_CAP * sizeof(HeapItem), stream>>>(
            H, W, b.dist, b.fg, b.L1, b.size1, b.blob_root, (int4 *)b.bbox, (const int2 *)b.lab_range, b.max_blobs,
            (HeapItem *)b.heap, inst, st);
    }
    return k;
}

template <typename A>
static void pp_layout(A &ar, PostprocBuffers &b, int n, int H, int W, int nr_types) {
    size_t N = (size_t)H * W, T = (size_t)n * N;
    b.max_blobs = (int)(N / 10 + 1);
    b.max_ids = postproc_max_ids(H, W);
    b.stats = ar.template take<PPStats>(n);
    b.fg = ar.template take<unsigned char>(T);
    b.L1 = ar.template take<int>(T);
    b.size1 = ar.template take<int>(T);
    b.blob_of_root = ar.template take<int>(T);
    b.blob_root = ar.template take<int>((size_t)n * b.max_blobs);
    b.bbox = ar.template take<int4>((size_t)n * b.max_blobs);
    b.lab_range = ar.template take<int2>((size_t)n * b.max_blobs);
    b.sobh = ar.template take<double>(T);
    b.sobv = ar.template take<double>(T);
    b.din = ar.template take<double>(T);
    b.dist = ar.template take<double>(T);
    b.mk0 = ar.template take<unsigned char>(T);
    b.L2 = ar.template take<int>(T);
    b.flag = ar.template take<unsigned char>(T);
    b.filled = ar.template take<unsigned char>(T);
    b.eroded = ar.template take<unsigned char>(T);
    b.opened = ar.template take<unsigned char>(T);
    b.size3 = ar.template take<int>(T);
    b.id3 = ar.template take<int>(T);
    b.rowcnt = ar.template take<int>((size_t)n * H);
    b.heap = ar.template take<HeapItem>(T);
    b.acc = ar.template take<InstAcc>((size_t)n * b.max_ids);
    b.tcnt = ar.template take<int>((size_t)n * b.max_ids * (nr_types > 0 ? nr_types : 1));
}

int postproc_max_ids(int H, int W) { return (int)((size_t)H * W / 6 + 8); }

size_t postproc_workspace_bytes(int n, int H, int W, int nr_types) {
    ArenaSizer s;
    PostprocBuffers b;
    pp_layout(s, b, n, H, W, nr_types);
    return s.top + 4096;
}

// Runs the whole post-processing path for n maps on `stream`.  Returns the number of kernel launches.
int postproc_run(Arena &arena, cudaStream_t stream, const float *pred, int n, int H, int W, int C, int nr_types,
                 int *inst, long long *table, int max_rows, int *n_rows, std::string *prof) {
    HVN_CHECK(C == 3 || C == 4, -1, "postproc: C must be 3 (np,hv_x,hv_y) or 4 (tp,np,hv_x,hv_y)");
    HVN_CHECK(C == 4 || nr_types == 0, -1, "postproc: nr_types given but the map has no type channel");
    HVN_CHECK(H >= 1 && W >= 1 && n >= 1, -1, "postproc: empty input");
    HVN_CHECK((long long)H * W < (1ll << 30), -1, "postproc: map too large (H*W must be < 2^30)");
    int off = (C == 4) ? 1 : 0;
    int N = H * W;
    size_t T = (size_t)n * N;
    PostprocBuffers b;
    arena.reset();
    arena.reserve(postproc_workspace_bytes(n, H, W, nr_types));
    pp_layout(arena, b, n, H, W, nr_types);
    int launches = 0;
    const int TPB = 256;
    dim3 g1((unsigned)min(cdiv(N, TPB), 1024), (unsigned)n);
    std::vector<std::pair<const char *, cudaEvent_t>> evs;
    auto mark = [&](const char *name) {
        if (!prof) return;
        cudaEvent_t e;
        cudaEventCreate(&e);
        cudaEventRecord(e, stream);
        evs.emplace_back(name, e);
    };
    mark("start");
#define L(...) do { __VA_ARGS__; ++launches; mark(#__VA_ARGS__); } while (0)
    L(k_init_stats<<<cdiv(n, 128), 128, 0, stream>>>((PPStats *)b.stats, n));
    HVN_CUDA(cudaMemsetAsync(b.size1, 0, T * sizeof(int), stream));
    HVN_CUDA(cudaMemsetAsync(b.size3, 0, T * sizeof(int), stream));
    HVN_CUDA(cudaMemsetAsync(b.flag, 0, T, stream));
    HVN_CUDA(cudaMemsetAsync(b.tcnt, 0, (size_t)n * b.max_ids * (nr_types > 0 ? nr_types : 1) * sizeof(int), stream));
    L(k_bbox_init<<<cdiv((size_t)n * b.max_blobs, TPB), TPB, 0, stream>>>((int4 *)b.bbox, (size_t)n * b.max_blobs));
    L(k_range_init<<<cdiv((size_t)n * b.max_blobs, TPB), TPB, 0, stream>>>((int2 *)b.lab_range, (size_t)n * b.max_blobs));
    L(k_acc_init<<<cdiv((size_t)n * b.max_ids, TPB), TPB, 0, stream>>>((InstAcc *)b.acc, (size_t)n * b.max_ids));
    PPStats *st = (PPStats *)b.stats;
    // foreground
    L(k_threshold_minmax<<<g1, TPB, 0, stream>>>(pred, C, off, N, b.fg, st));
    L(k_ccl_init<<<g1, TPB, 0, stream>>>(b.fg, 0, N, b.L1));
    L(k_ccl_merge<<<g1, TPB, 0, stream>>>(H, W, b.L1));
    L(k_ccl_flatten_count<<<g1, TPB, 0, stream>>>(N, b.L1, b.size1));
    L(k_blob_filter<<<g1, TPB, 0, stream>>>(N, b.L1, b.size1, b.fg, b.blob_of_root, b.blob_root, b.max_blobs, st));
    L(k_blob_bbox<<<g1, TPB, 0, stream>>>(H, W, b.L1, b.fg, b.blob_of_root, (int4 *)b.bbox, b.max_blobs));
    // energy landscape
    dim3 gs((unsigned)cdiv(W, SB_TW), (unsigned)cdiv(H, SB_TH), (unsigned)n);
    L(k_sobel21<<<gs, 256, 0, stream>>>(pred, C, off, H, W, b.sobh, b.sobv, st));
    L(k_energy<<<g1, TPB, 0, stream>>>(N, b.sobh, b.sobv, b.fg, b.din, b.mk0, st));
    L(k_blur3<<<g1, TPB, 0, stream>>>(H, W, b.din, b.dist));
    // markers
    L(k_ccl_init<<<g1, TPB, 0, stream>>>(b.mk0, 1, N, b.L2));
    L(k_ccl_merge<<<g1, TPB, 0, stream>>>(H, W, b.L2));
    L(k_border_flag<<<dim3((unsigned)cdiv(2 * (H + W), TPB), (unsigned)n), TPB, 0, stream>>>(H, W, b.L2, b.flag));
    L(k_fill<<<g1, TPB, 0, stream>>>(N, b.mk0, b.L2, b.flag, b.filled));
    L(k_morph5<true><<<g1, TPB, 0, stream>>>(H, W, b.filled, b.eroded));
    L(k_morph5<false><<<g1, TPB, 0, stream>>>(H, W, b.eroded, b.opened));
    L(k_ccl_init<<<g1, TPB, 0, stream>>>(b.opened, 0, N, b.L2));
    L(k_ccl_merge<<<g1, TPB, 0, stream>>>(H, W, b.L2));
    L(k_ccl_flatten_count<<<g1, TPB, 0, stream>>>(N, b.L2, b.size3));
    dim3 gr((unsigned)min(cdiv((long long)H * 32, TPB), 1024), (unsigned)n);
    L(k_row_roots<<<gr, TPB, 0, stream>>>(H, W, b.L2, b.rowcnt));
    L(k_row_scan<<<n, 1024, 0, stream>>>(H, b.rowcnt, st));
    L(k_assign_ids<<<gr, TPB, 0, stream>>>(H, W, b.L2, b.rowcnt, b.id3));
    L(k_marker_labels<<<g1, TPB, 0, stream>>>(N, b.L2, b.size3, b.id3, b.fg, inst));
    // flood
    L(k_blob_marker_range<<<g1, TPB, 0, stream>>>(N, inst, b.L1, b.blob_of_root, (int2 *)b.lab_range, b.max_blobs));
    L(k_blob_fill_single<<<g1, TPB, 0, stream>>>(N, inst, b.fg, b.L1, b.blob_of_root, (int2 *)b.lab_range, b.max_blobs));
    {
        const int fk = postproc_flood(stream, b, n, H, W, inst, FLOOD_AUTO);
        ++launches;
        mark(postproc_flood_name(fk));
    }
    // table
    L(k_table_accum<<<g1, TPB, 0, stream>>>(H, W, inst, pred, C, nr_types, (InstAcc *)b.acc, b.tcnt, b.max_ids));
    L(k_table_rows<<<n, 1024, 0, stream>>>((InstAcc *)b.acc, b.tcnt, nr_types, b.max_ids, table, max_rows, n_rows, st));
#undef L
    HVN_CUDA(cudaGetLastError());
    if (prof) {
        HVN_CUDA(cudaStreamSynchronize(stream));
        prof->clear();
        for (size_t i = 1; i < evs.size(); ++i) {
            float ms = 0.f;
            cudaEventElapsedTime(&ms, evs[i - 1].second, evs[i].second);
            std::string nm(evs[i].first);
            nm = nm.substr(0, nm.find("<<<"));
            char line[160];
            snprintf(line, sizeof(line), "pp %-28s %9.4f ms\n", nm.c_str(), ms);
            *prof += line;
        }
        for (auto &e : evs) cudaEventDestroy(e.second);
        std::vector<PPStats> hs(n);
        HVN_CUDA(cudaMemcpy(hs.data(), st, sizeof(PPStats) * n, cudaMemcpyDeviceToHost));
        long long pops = 0; int pmax = 0, cmax = 0, bl = 0, bmax = 0;
        for (auto &h : hs) { pops += h.pad[0]; pmax = std::max(pmax, h.pad[0]); cmax = std::max(cmax, h.pad[1]); bl += h.nblobs; bmax = std::max(bmax, h.nblobs); }
        char line[256];
        snprintf(line, sizeof(line), "pp stats: maps %d  flood pops total %lld  max/map %d  longest single flood %d kcycles  blobs total %d max/map %d\n",
                 n, pops, pmax, cmax, bl, bmax);
        *prof += line;
    }
    return launches;
}

void postproc_buffers(Arena &arena, int n, int H, int W, int nr_types, PostprocBuffers &b) {
    const size_t top = arena.top;
    arena.reset();
    pp_layout(arena, b, n, H, W, nr_types);
    arena.top = top;
}

// flood-only entry: inst = markers where the size-filtered mask is set, 0 elsewhere (what k_marker_labels leaves)
__global__ void k_mask_markers(int N, const int *__restrict__ markers, const unsigned char *__restrict__ fg_all,
                               int *__restrict__ inst_all) {
    int m = blockIdx.y;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        size_t i = (size_t)m * N + p;
        inst_all[i] = fg_all[i] ? markers[i] : 0;
    }
}

int postproc_flood_only(Arena &arena, cudaStream_t stream, const double *dist, const unsigned char *mask,
                        const int *markers, int n, int H, int W, int *inst, int choice) {
    HVN_CHECK(H >= 1 && W >= 1 && n >= 1, -1, "postproc_flood_only: empty input");
    HVN_CHECK((long long)H * W < (1ll << 30), -1, "postproc_flood_only: map too large (H*W must be < 2^30)");
    const int N = H * W;
    const size_t T = (size_t)n * N;
    PostprocBuffers b;
    arena.reset();
    arena.reserve(postproc_workspace_bytes(n, H, W, 0));
    pp_layout(arena, b, n, H, W, 0);
    const int TPB = 256;
    dim3 g1((unsigned)min(cdiv(N, TPB), 1024), (unsigned)n);
    PPStats *st = (PPStats *)b.stats;
    k_init_stats<<<cdiv(n, 128), 128, 0, stream>>>(st, n);
    HVN_CUDA(cudaMemsetAsync(b.size1, 0, T * sizeof(int), stream));
    k_bbox_init<<<cdiv((size_t)n * b.max_blobs, TPB), TPB, 0, stream>>>((int4 *)b.bbox, (size_t)n * b.max_blobs);
    k_range_init<<<cdiv((size_t)n * b.max_blobs, TPB), TPB, 0, stream>>>((int2 *)b.lab_range, (size_t)n * b.max_blobs);
    HVN_CUDA(cudaMemcpyAsync(b.dist, dist, T * sizeof(double), cudaMemcpyDeviceToDevice, stream));
    k_ccl_init<<<g1, TPB, 0, stream>>>(mask, 0, N, b.L1);
    k_ccl_merge<<<g1, TPB, 0, stream>>>(H, W, b.L1);
    k_ccl_flatten_count<<<g1, TPB, 0, stream>>>(N, b.L1, b.size1);
    k_blob_filter<<<g1, TPB, 0, stream>>>(N, b.L1, b.size1, b.fg, b.blob_of_root, b.blob_root, b.max_blobs, st);
    k_blob_bbox<<<g1, TPB, 0, stream>>>(H, W, b.L1, b.fg, b.blob_of_root, (int4 *)b.bbox, b.max_blobs);
    k_mask_markers<<<g1, TPB, 0, stream>>>(N, markers, b.fg, inst);
    k_blob_marker_range<<<g1, TPB, 0, stream>>>(N, inst, b.L1, b.blob_of_root, (int2 *)b.lab_range, b.max_blobs);
    k_blob_fill_single<<<g1, TPB, 0, stream>>>(N, inst, b.fg, b.L1, b.blob_of_root, (int2 *)b.lab_range, b.max_blobs);
    const int k = postproc_flood(stream, b, n, H, W, inst, choice);
    HVN_CUDA(cudaGetLastError());
    return k;
}

}  // namespace hvn
