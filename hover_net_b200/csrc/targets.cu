// Training targets of the reference on the device: the HV map of models/hovernet/targets.py gen_instance_hv_map
// (after dataloader/augs.py fix_mirror_padding), and the per-batch counts of run_desc.py proc_valid_step_output.
//
// The reference renumbers every later 4-connected piece of an id to a fresh id (fix_mirror_padding), then loops over
// the ids of the cropped map, building a full-map mask per instance: O(instances * pixels), twice.  Here every
// instance is exactly one 4-connected component of equal id, so the kernels work on components and never build the
// renumbered ids:
//   init     parents, accumulators, per-map max id / background / negative-id flags
//   merge    same-id union-find (uf.cuh): root = the component's first pixel in raster order
//   extent   flatten; per component: full-map extent and pixels inside the centre crop; number of components
//   box      per component kept by the size filter (>= 30 px inside the crop, remove_small_objects(crop_ann, 30)):
//            the extent expanded by 2 and sliced with Python slice semantics (a negative start wraps by H, the stop
//            clips at H; a side < 2 skips the instance); count, coordinate sums and extent of its pixels inside the
//            box; whether the crop keeps a background pixel
//   write    per pixel of a kept instance inside its box: offset from the rounded centre of mass (integer sums, one
//            float64 division, int(com + 0.5)), negatives divided by -min and positives by max in IEEE fp32 division
//   flags    per map: no background, no background left in the crop, a box without any of its instance's pixels
//            (the reference fails there converting a NaN centre of mass)
// The per-pixel atomics are aggregated per warp first (__match_any_sync on the root).
#include <algorithm>
#include <climits>

#include "../../include/hvn.h"
#include "cnn_kernels.h"
#include "targets.h"
#include "uf.cuh"

namespace hvn {
namespace {

constexpr int TPB = 256;
constexpr int MIN_IN_CROP = 30;  // remove_small_objects(crop_ann, min_size=30)
constexpr unsigned FULL = 0xffffffffu;

// Python slice [lo - 2 : hi + 2] of an axis of length n (lo inclusive, hi exclusive, hi + 2 > 0): start s0, stop s1.
// False when the slice is shorter than 2 (the reference skips the instance).
__device__ __forceinline__ bool box_side(int lo, int hi, int n, int &s0, int &s1) {
    int a = lo - 2, b = hi + 2;
    if (a < 0) a = max(a + n, 0);
    if (b > n) b = n;
    s0 = a;
    s1 = b;
    return b - a >= 2;
}

struct Box {
    bool ok;
    int r0, r1, c0, c1;
};

__device__ __forceinline__ Box comp_box(const TargetWork &w, size_t r, int H, int W) {
    Box b;
    b.ok = w.ncrop[r] >= MIN_IN_CROP;
    b.ok = b.ok && box_side(w.rmin[r], w.rmax[r] + 1, H, b.r0, b.r1);
    b.ok = b.ok && box_side(w.cmin[r], w.cmax[r] + 1, W, b.c0, b.c1);
    return b;
}

__global__ void __launch_bounds__(TPB) k_tg_init(const int *__restrict__ inst, int N, TargetWork w) {
    const int m = blockIdx.y;
    const size_t base = (size_t)m * N;
    int mx = 0;
    bool zero = false, neg = false;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const size_t i = base + p;
        const int v = inst[i];
        mx = max(mx, v);
        zero |= v == 0;
        neg |= v < 0;
        w.L[i] = v > 0 ? p : -1;
        w.rmin[i] = w.cmin[i] = w.bymin[i] = w.bxmin[i] = INT_MAX;
        w.rmax[i] = w.cmax[i] = w.bymax[i] = w.bxmax[i] = -1;
        w.ncrop[i] = w.nbox[i] = 0;
        w.sy[i] = w.sx[i] = 0;
    }
    mx = __reduce_max_sync(FULL, mx);
    zero = __any_sync(FULL, zero);
    neg = __any_sync(FULL, neg);
    if ((threadIdx.x & 31) == 0) {
        if (mx > 0) atomicMax(&w.maxid[m], mx);
        if (zero) w.has_bg[m] = 1;
        if (neg) atomicOr(w.err, 1);
    }
}

__global__ void __launch_bounds__(TPB) k_tg_merge(const int *__restrict__ inst, int H, int W, TargetWork w) {
    const int m = blockIdx.y, N = H * W;
    const int *I = inst + (size_t)m * N;
    int *L = w.L + (size_t)m * N;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        const int v = I[p];
        if (v <= 0) continue;
        const int y = p / W, x = p - y * W;
        if (x > 0 && I[p - 1] == v) uf_union(L, p, p - 1);
        if (y > 0 && I[p - W] == v) uf_union(L, p, p - W);
    }
}

// Loops below keep every lane of a warp in step (the bound is rounded up to whole strides) so that the warp
// aggregation may use the full mask.
__global__ void __launch_bounds__(TPB) k_tg_extent(int H, int W, int h0, int w0, int ch, int cw, TargetWork w) {
    const int m = blockIdx.y, N = H * W;
    const size_t base = (size_t)m * N;
    const int stride = gridDim.x * blockDim.x;
    int roots = 0;
    for (int q = blockIdx.x * blockDim.x; q < N; q += stride) {
        const int p = q + threadIdx.x;
        int r = -1, y = 0, x = 0;
        if (p < N && w.L[base + p] >= 0) {
            r = uf_find(w.L + base, p);
            w.L[base + p] = r;  // racy-but-benign: only ever replaces a parent by an ancestor
            y = p / W;
            x = p - y * W;
            roots += r == p;
        }
        const bool in_crop = r >= 0 && y >= h0 && y < h0 + ch && x >= w0 && x < w0 + cw;
        const unsigned grp = __match_any_sync(FULL, r);
        const int ymin = __reduce_min_sync(grp, y), ymax = __reduce_max_sync(grp, y);
        const int xmin = __reduce_min_sync(grp, x), xmax = __reduce_max_sync(grp, x);
        const int nc = __popc(grp & __ballot_sync(FULL, in_crop));
        if (r >= 0 && (threadIdx.x & 31) == __ffs(grp) - 1) {
            const size_t R = base + r;
            atomicMin(&w.rmin[R], ymin);
            atomicMax(&w.rmax[R], ymax);
            atomicMin(&w.cmin[R], xmin);
            atomicMax(&w.cmax[R], xmax);
            if (nc) atomicAdd(&w.ncrop[R], nc);
        }
    }
    roots = __reduce_add_sync(FULL, roots);
    if ((threadIdx.x & 31) == 0 && roots) atomicAdd(&w.ncomp[m], roots);
}

__global__ void __launch_bounds__(TPB) k_tg_box(int H, int W, int h0, int w0, int ch, int cw, TargetWork w) {
    const int m = blockIdx.y, N = H * W;
    const size_t base = (size_t)m * N;
    const int stride = gridDim.x * blockDim.x;
    bool bg_crop = false;
    for (int q = blockIdx.x * blockDim.x; q < N; q += stride) {
        const int p = q + threadIdx.x;
        int r = p < N ? w.L[base + p] : -1;
        const int y = p / W, x = p - (p / W) * W;
        const bool in_crop = p < N && y >= h0 && y < h0 + ch && x >= w0 && x < w0 + cw;
        bool in_box = false;
        int dy = 0, dx = 0;
        if (r >= 0) {
            const Box b = comp_box(w, base + r, H, W);
            bg_crop |= in_crop && w.ncrop[base + r] < MIN_IN_CROP;
            in_box = b.ok && y >= b.r0 && y < b.r1 && x >= b.c0 && x < b.c1;
            dy = y - b.r0;
            dx = x - b.c0;
        } else {
            bg_crop |= in_crop;
        }
        if (!in_box) r = -1;
        const unsigned grp = __match_any_sync(FULL, r);
        if (r < 0) continue;  // whole groups leave together: grp holds exactly the lanes with this r
        const int n = __popc(grp);
        const unsigned sy = __reduce_add_sync(grp, (unsigned)dy), sx = __reduce_add_sync(grp, (unsigned)dx);
        const int ymin = __reduce_min_sync(grp, y), ymax = __reduce_max_sync(grp, y);
        const int xmin = __reduce_min_sync(grp, x), xmax = __reduce_max_sync(grp, x);
        if ((threadIdx.x & 31) == __ffs(grp) - 1) {
            const size_t R = base + r;
            atomicAdd(&w.nbox[R], n);
            atomicAdd(&w.sy[R], (unsigned long long)sy);
            atomicAdd(&w.sx[R], (unsigned long long)sx);
            atomicMin(&w.bymin[R], ymin);
            atomicMax(&w.bymax[R], ymax);
            atomicMin(&w.bxmin[R], xmin);
            atomicMax(&w.bxmax[R], xmax);
        }
    }
    if (__any_sync(FULL, bg_crop) && (threadIdx.x & 31) == 0) w.has_bg_crop[m] = 1;
}

// 1..len - com, then negatives / -min and positives / max (IEEE fp32 division; 0 stays 0).
__device__ __forceinline__ float hv_offset(int d, int dmin, int dmax, int com) {
    const int v = d + 1 - com, lo = dmin + 1 - com, hi = dmax + 1 - com;
    const float f = (float)v;
    if (v < 0) return __fdiv_rn(f, (float)-lo);
    if (v > 0) return __fdiv_rn(f, (float)hi);
    return f;
}

__global__ void __launch_bounds__(TPB) k_tg_write(int H, int W, TargetWork w, float2 *__restrict__ hv) {
    const int m = blockIdx.y, N = H * W;
    const size_t base = (size_t)m * N;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < N; p += gridDim.x * blockDim.x) {
        float2 o = make_float2(0.f, 0.f);
        const int r = w.L[base + p];
        if (r >= 0) {
            const size_t R = base + r;
            const Box b = comp_box(w, R, H, W);
            const int cnt = w.nbox[R];
            if (b.ok && cnt == 0 && r == p) w.nan_com[m] = 1;
            const int y = p / W, x = p - y * W;
            if (b.ok && y >= b.r0 && y < b.r1 && x >= b.c0 && x < b.c1) {
                const int comy = (int)((double)w.sy[R] / (double)cnt + 0.5);
                const int comx = (int)((double)w.sx[R] / (double)cnt + 0.5);
                o.x = hv_offset(x - b.c0, w.bxmin[R] - b.c0, w.bxmax[R] - b.c0, comx);
                o.y = hv_offset(y - b.r0, w.bymin[R] - b.r0, w.bymax[R] - b.r0, comy);
            }
        }
        hv[base + p] = o;
    }
}

__global__ void k_tg_flags(int n, TargetWork w, int *__restrict__ flags) {
    for (int m = blockIdx.x * blockDim.x + threadIdx.x; m < n; m += gridDim.x * blockDim.x)
        flags[m] = (w.has_bg[m] ? 0 : HVN_TG_NO_BACKGROUND) | (w.has_bg_crop[m] ? 0 : HVN_TG_NO_BACKGROUND_CROP) |
                   (w.nan_com[m] ? HVN_TG_EMPTY_BOX : 0);
}

template <typename A> void layout(A &a, int n, int H, int W, TargetWork &w) {
    const size_t px = (size_t)n * H * W;
    w.n = n;
    w.H = H;
    w.W = W;
    w.L = a.template take<int>(px);
    w.rmin = a.template take<int>(px);
    w.rmax = a.template take<int>(px);
    w.cmin = a.template take<int>(px);
    w.cmax = a.template take<int>(px);
    w.ncrop = a.template take<int>(px);
    w.nbox = a.template take<int>(px);
    w.sy = a.template take<unsigned long long>(px);
    w.sx = a.template take<unsigned long long>(px);
    w.bymin = a.template take<int>(px);
    w.bymax = a.template take<int>(px);
    w.bxmin = a.template take<int>(px);
    w.bxmax = a.template take<int>(px);
    // the per-map words are one block so that a single memset clears them
    int *per_map = a.template take<int>((size_t)5 * n + 1);
    if (per_map) {
        w.maxid = per_map;
        w.ncomp = per_map + n;
        w.has_bg = per_map + 2 * n;
        w.has_bg_crop = per_map + 3 * n;
        w.nan_com = per_map + 4 * n;
        w.err = per_map + 5 * n;
    }
}

// ---------------------------------------------------------------------------------------------------------------
// Validation counts.  One thread per output pixel, register / shared-memory partials, one set of global atomics per
// block.  Layout of counts: correct, inter, total of (prob_np > 0.5) against (inst > 0), then inter_k, total_k of
// (pred_tp == k) against (type == k) for k in 0..nr_types-1.
__global__ void __launch_bounds__(TPB) k_valid_reduce(const float *__restrict__ pred, const int *__restrict__ inst,
                                                      const int *__restrict__ type, const float2 *__restrict__ hv,
                                                      int H, int W, int h, int w, int h0, int w0, int C, int nr_types,
                                                      unsigned long long *__restrict__ counts, double *__restrict__ sse) {
    __shared__ unsigned s_cnt[3 + 2 * HVN_MAX_TYPES];
    __shared__ double s_sse[TPB / 32];
    for (int i = threadIdx.x; i < 3 + 2 * nr_types; i += blockDim.x) s_cnt[i] = 0;
    __syncthreads();
    const int m = blockIdx.y, npx = h * w;
    const int cnp = C == 4 ? 1 : 0;
    unsigned correct = 0, inter = 0, total = 0;
    double err = 0.0;
    for (int p = blockIdx.x * blockDim.x + threadIdx.x; p < npx; p += gridDim.x * blockDim.x) {
        const int y = p / w, x = p - y * w;
        const size_t o = ((size_t)m * npx + p) * C;
        const size_t t = ((size_t)m * H + y + h0) * W + x + w0;
        const int pn = pred[o + cnp] > 0.5f, tn = inst[t] > 0;
        correct += pn == tn;
        inter += pn & tn;
        total += pn + tn;
        const float2 th = hv[t];
        const float ex = pred[o + C - 2] - th.x, ey = pred[o + C - 1] - th.y;
        err += (double)ex * ex + (double)ey * ey;
        if (nr_types > 0) {
            const int pt = (int)pred[o], tt = type[t];
            if (pt == tt) {
                if (pt >= 0 && pt < nr_types) {
                    atomicAdd(&s_cnt[3 + 2 * pt], 1u);
                    atomicAdd(&s_cnt[4 + 2 * pt], 2u);
                }
            } else {
                if (pt >= 0 && pt < nr_types) atomicAdd(&s_cnt[4 + 2 * pt], 1u);
                if (tt >= 0 && tt < nr_types) atomicAdd(&s_cnt[4 + 2 * tt], 1u);
            }
        }
    }
    correct = __reduce_add_sync(FULL, correct);
    inter = __reduce_add_sync(FULL, inter);
    total = __reduce_add_sync(FULL, total);
    for (int d = 16; d; d >>= 1) err += __shfl_xor_sync(FULL, err, d);
    if ((threadIdx.x & 31) == 0) {
        atomicAdd(&s_cnt[0], correct);
        atomicAdd(&s_cnt[1], inter);
        atomicAdd(&s_cnt[2], total);
        s_sse[threadIdx.x >> 5] = err;
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 3 + 2 * nr_types; i += blockDim.x)
        if (s_cnt[i]) atomicAdd(&counts[i], (unsigned long long)s_cnt[i]);
    if (threadIdx.x == 0) {
        double s = 0.0;
        for (int i = 0; i < TPB / 32; ++i) s += s_sse[i];
        atomicAdd(sse, s);
    }
}

int grid_x(long long px) { return (int)std::min<long long>(std::max<long long>(1, cdiv(px, TPB)), 1024); }

}  // namespace

// Per pixel: 13 words of parents and accumulators (60 B); e.g. 256 maps of 270 x 270 -> 1.1 GB.
size_t targets_workspace_bytes(int n, int H, int W) {
    ArenaSizer s;
    TargetWork w;
    layout(s, n, H, W, w);
    return s.top + 1024;
}

int targets_run(Arena &arena, cudaStream_t stream, const int *inst, int n, int H, int W, int crop_h, int crop_w,
                float *hv, int *flags, TargetWork &w) {
    arena.reset();
    arena.reserve(targets_workspace_bytes(n, H, W));
    layout(arena, n, H, W, w);
    HVN_CUDA(cudaMemsetAsync(w.maxid, 0, ((size_t)5 * n + 1) * sizeof(int), stream));
    const int N = H * W;
    const int h0 = (int)((H - crop_h) * 0.5), w0 = (int)((W - crop_w) * 0.5);  // cropping_center
    const dim3 g(grid_x(N), n);
    k_tg_init<<<g, TPB, 0, stream>>>(inst, N, w);
    k_tg_merge<<<g, TPB, 0, stream>>>(inst, H, W, w);
    k_tg_extent<<<g, TPB, 0, stream>>>(H, W, h0, w0, crop_h, crop_w, w);
    k_tg_box<<<g, TPB, 0, stream>>>(H, W, h0, w0, crop_h, crop_w, w);
    k_tg_write<<<g, TPB, 0, stream>>>(H, W, w, (float2 *)hv);
    k_tg_flags<<<cdiv(n, TPB), TPB, 0, stream>>>(n, w, flags);
    HVN_CUDA(cudaGetLastError());
    return 6;
}

int valid_reduce(cudaStream_t stream, const float *pred, const int *inst, const int *type, const float *hv, int n,
                 int H, int W, int h, int w, int C, int nr_types, long long *counts, double *sse) {
    const int h0 = (int)((H - h) * 0.5), w0 = (int)((W - w) * 0.5);
    k_valid_reduce<<<dim3(grid_x(h * w), n), TPB, 0, stream>>>(pred, inst, type, (const float2 *)hv, H, W, h, w, h0,
                                                                w0, C, nr_types, (unsigned long long *)counts, sse);
    HVN_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace hvn
