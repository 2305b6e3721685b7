// Validation loss on the device: the per-pixel terms of the reference's xentropy_loss, dice_loss, mse_loss and
// msge_loss (models/hovernet/utils.py), summed over a batch (slot layout in loss.h).
//   k_loss_reduce  one block per 32 x 32 tile of one map's crop, 128 threads, 8 pixels each.  The predicted and
//                  target HV of the tile and its 2-pixel halo are staged in shared memory (zero outside the crop:
//                  F.conv2d's padding at the crop border), so the 5 x 5 stencils read no global memory.  The per-pixel
//                  terms are fp32, as the reference computes them; every thread adds them into its own fp64 column
//                  of a shared array, and the block adds the columns in a fixed order into partials[slot][block].
//                  hvn_valid's integer counts come out of the same pass (integer atomics: exact in any order).
//   k_loss_final   one block per slot: a fixed-order sum of that slot's partials.
// No floating-point atomics anywhere, so the sums are bit-identical from call to call.  The pass reads (4 + nt) * 4 B
// of probabilities, 8 B of targets and 4 or 8 B of labels per output pixel: HBM-bound.
#include "../../include/hvn.h"
#include "cnn_kernels.h"
#include "loss.h"

namespace hvn {
namespace {

constexpr int LT = 32;           // tile side
constexpr int LR = 2;            // stencil radius (get_sobel_kernel(5))
constexpr int LH = LT + 2 * LR;  // staged side
constexpr int LTPB = 128;        // threads: 32 columns x 4 rows, 8 rows each
constexpr int FTPB = 256;        // threads of the final pass
constexpr unsigned FULL = 0xffffffffu;

struct LossArgs {
    const float *probs;
    const int *inst, *type;
    const float2 *hv;
    int H, W, h, w, h0, w0, nt, ns, nblk;
    double *part;
    unsigned long long *counts;
    int *err;
};

size_t smem_bytes(int ns) { return (size_t)ns * LTPB * sizeof(double) + 2 * LH * LH * sizeof(float2); }

// -log(clamp(q, eps, 1 - eps)), eps = 10e-8 rounded to fp32 as torch.clamp rounds its bounds
__device__ __forceinline__ float neg_log_clamped(float q) {
    return -logf(fminf(fmaxf(q, (float)10e-8), (float)(1.0 - 10e-8)));
}

__global__ void __launch_bounds__(LTPB) k_loss_reduce(const LossArgs a) {
    extern __shared__ double s_acc[];  // [ns][LTPB]: thread t owns column t
    float2 *s_p = reinterpret_cast<float2 *>(s_acc + (size_t)a.ns * LTPB);  // [LH][LH] predicted HV
    float2 *s_t = s_p + LH * LH;                                             // [LH][LH] target HV
    __shared__ float s_k[25];  // kernel_h of get_sobel_kernel(5); kernel_v is its transpose
    __shared__ unsigned s_cnt[3 + 2 * HVN_MAX_TYPES];
    const int tid = threadIdx.x, lane = tid & 31, wid = tid >> 5;
    const int m = blockIdx.z, ty0 = blockIdx.y * LT, tx0 = blockIdx.x * LT;
    const int C = 4 + a.nt;
    for (int i = tid; i < a.ns * LTPB; i += LTPB) s_acc[i] = 0.0;
    for (int i = tid; i < 3 + 2 * a.nt; i += LTPB) s_cnt[i] = 0;
    if (tid < 25) {
        // torch.meshgrid(h_range, v_range) ('ij'): h varies along rows.  h / (h*h + v*v + 1e-15) in fp32; the
        // 1e-15 only matters at the centre, where h = 0.
        const int i = tid / 5 - LR, j = tid % 5 - LR, d = i * i + j * j;
        s_k[tid] = d ? __fdiv_rn((float)i, (float)d) : 0.f;
    }
    for (int q = tid; q < LH * LH; q += LTPB) {
        const int yy = q / LH, xx = q - yy * LH, y = ty0 + yy - LR, x = tx0 + xx - LR;
        float2 p = make_float2(0.f, 0.f), t = make_float2(0.f, 0.f);
        if (y >= 0 && y < a.h && x >= 0 && x < a.w) {
            const float *pp = a.probs + (((size_t)m * a.h + y) * a.w + x) * C;
            p = make_float2(pp[2], pp[3]);
            t = a.hv[((size_t)m * a.H + y + a.h0) * a.W + x + a.w0];
        }
        s_p[q] = p;
        s_t[q] = t;
    }
    __syncthreads();

    double *acc = s_acc + tid;
    unsigned correct = 0, inter = 0, total = 0;
    bool bad = false;
    const int x = tx0 + lane;
    for (int r = wid; r < LT; r += LTPB / 32) {
        const int y = ty0 + r;
        if (y >= a.h || x >= a.w) continue;
        const float *pp = a.probs + (((size_t)m * a.h + y) * a.w + x) * C;
        const size_t ti = ((size_t)m * a.H + y + a.h0) * a.W + x + a.w0;
        const int fg = a.inst[ti] > 0;
        // NP: cross-entropy and the dice sums
        const float p0 = pp[0], p1 = pp[1], s = p0 + p1;
        acc[LS_NP_CE * LTPB] += (double)neg_log_clamped((fg ? p1 : p0) / s);
        acc[(LS_NP_I + fg) * LTPB] += (double)(fg ? p1 : p0);
        acc[LS_NP_L * LTPB] += (double)p0;
        acc[(LS_NP_L + 1) * LTPB] += (double)p1;
        acc[(LS_NP_R + fg) * LTPB] += 1.0;
        // HV: squared error, and the gradient error inside the nuclei
        const float2 ph = s_p[(r + LR) * LH + lane + LR], th = s_t[(r + LR) * LH + lane + LR];
        const float ex = ph.x - th.x, ey = ph.y - th.y;
        acc[LS_HV_SQ * LTPB] += (double)ex * ex + (double)ey * ey;
        if (fg) {
            float gpx = 0.f, gtx = 0.f, gpy = 0.f, gty = 0.f;
#pragma unroll
            for (int i = 0; i < 5; ++i)
#pragma unroll
                for (int j = 0; j < 5; ++j) {
                    const int q = (r + i) * LH + lane + j;
                    const float kh = s_k[i * 5 + j], kv = s_k[j * 5 + i];
                    gpx = fmaf(kh, s_p[q].x, gpx);
                    gtx = fmaf(kh, s_t[q].x, gtx);
                    gpy = fmaf(kv, s_p[q].y, gpy);
                    gty = fmaf(kv, s_t[q].y, gty);
                }
            const float dh = gpx - gtx, dv = gpy - gty;
            acc[LS_MSGE * LTPB] += (double)dh * dh + (double)dv * dv;
            acc[LS_FOCUS * LTPB] += 1.0;
        }
        // hvn_valid's counts
        const int pn = p1 > 0.5f;
        correct += pn == fg;
        inter += pn & fg;
        total += pn + fg;
        if (a.nt > 0) {
            const float *pt = pp + 4;
            const int tt = a.type[ti];
            int best = 0;
            float bv = pt[0], st = pt[0];
            for (int o = 1; o < a.nt; ++o) {
                st += pt[o];
                if (pt[o] > bv) { bv = pt[o]; best = o; }
            }
            if (tt < 0 || tt >= a.nt) {  // F.one_hot raises: HVN_ERR_INVALID; the counts follow hvn_valid's rule
                bad = true;
                atomicAdd(&s_cnt[4 + 2 * best], 1u);
                continue;
            }
            acc[LS_TP_CE * LTPB] += (double)neg_log_clamped(pt[tt] / st);
            acc[(LS_TP_I + tt) * LTPB] += (double)pt[tt];
            for (int o = 0; o < a.nt; ++o) acc[(LS_TP_I + a.nt + o) * LTPB] += (double)pt[o];
            acc[(LS_TP_I + 2 * a.nt + tt) * LTPB] += 1.0;
            if (best == tt) {
                atomicAdd(&s_cnt[3 + 2 * tt], 1u);
                atomicAdd(&s_cnt[4 + 2 * tt], 2u);
            } else {
                atomicAdd(&s_cnt[4 + 2 * best], 1u);
                atomicAdd(&s_cnt[4 + 2 * tt], 1u);
            }
        }
    }
    correct = __reduce_add_sync(FULL, correct);
    inter = __reduce_add_sync(FULL, inter);
    total = __reduce_add_sync(FULL, total);
    if (lane == 0) {
        atomicAdd(&s_cnt[0], correct);
        atomicAdd(&s_cnt[1], inter);
        atomicAdd(&s_cnt[2], total);
    }
    if (bad) atomicOr(a.err, 1);
    __syncthreads();
    // column sums: warp w adds the slots w, w + 4, ... over the 128 columns in a fixed order
    const int blk = (blockIdx.z * gridDim.y + blockIdx.y) * gridDim.x + blockIdx.x;
    for (int s = wid; s < a.ns; s += LTPB / 32) {
        const double *col = s_acc + (size_t)s * LTPB + lane;
        double v = ((col[0] + col[32]) + (col[64] + col[96]));
        for (int d = 16; d; d >>= 1) v += __shfl_xor_sync(FULL, v, d);
        if (lane == 0) a.part[(size_t)s * a.nblk + blk] = v;
    }
    for (int i = tid; i < 3 + 2 * a.nt; i += LTPB)
        if (s_cnt[i]) atomicAdd(&a.counts[i], (unsigned long long)s_cnt[i]);
}

__global__ void __launch_bounds__(FTPB) k_loss_final(const double *__restrict__ part, int nblk,
                                                     double *__restrict__ sums) {
    __shared__ double s[FTPB];
    const double *p = part + (size_t)blockIdx.x * nblk;
    double v = 0.0;
    for (int b = threadIdx.x; b < nblk; b += FTPB) v += p[b];
    s[threadIdx.x] = v;
    __syncthreads();
    for (int d = FTPB / 2; d; d >>= 1) {
        if (threadIdx.x < d) s[threadIdx.x] += s[threadIdx.x + d];
        __syncthreads();
    }
    if (threadIdx.x == 0) sums[blockIdx.x] = s[0];
}

int nblocks(int n, int h, int w) { return cdiv(w, LT) * cdiv(h, LT) * n; }

}  // namespace

size_t loss_workspace_bytes(int n, int h, int w, int nr_types) {
    ArenaSizer s;
    s.take<double>((size_t)loss_nsums(nr_types) * nblocks(n, h, w));
    s.take<int>(1);
    return s.top + 256;
}

int loss_reduce(Arena &arena, cudaStream_t stream, const float *probs, const int *inst, const int *type,
                const float *hv, int n, int H, int W, int h, int w, int nr_types, double *sums, long long *counts,
                LossWork &lw) {
    HVN_CHECK(nr_types >= 0 && nr_types <= HVN_MAX_TYPES, HVN_ERR_INVALID, "nr_types out of range");
    HVN_CHECK(nr_types == 0 || type, HVN_ERR_INVALID, "a model with nr_types > 0 needs a type map");
    const int ns = loss_nsums(nr_types);
    arena.reset();
    arena.reserve(loss_workspace_bytes(n, h, w, nr_types));
    lw.nblk = nblocks(n, h, w);
    lw.part = arena.take<double>((size_t)ns * lw.nblk);
    lw.err = arena.take<int>(1);
    HVN_CUDA(cudaMemsetAsync(lw.err, 0, sizeof(int), stream));
    LossArgs a;
    a.probs = probs;
    a.inst = inst;
    a.type = type;
    a.hv = reinterpret_cast<const float2 *>(hv);
    a.H = H;
    a.W = W;
    a.h = h;
    a.w = w;
    a.h0 = (int)((H - h) * 0.5);  // cropping_center
    a.w0 = (int)((W - w) * 0.5);
    a.nt = nr_types;
    a.ns = ns;
    a.nblk = lw.nblk;
    a.part = lw.part;
    a.counts = reinterpret_cast<unsigned long long *>(counts);
    a.err = lw.err;
    const size_t smem = smem_bytes(ns);
    HVN_CUDA(cudaFuncSetAttribute(k_loss_reduce, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    k_loss_reduce<<<dim3(cdiv(w, LT), cdiv(h, LT), n), LTPB, smem, stream>>>(a);
    k_loss_final<<<ns, FTPB, 0, stream>>>(lw.part, lw.nblk, sums);
    HVN_CUDA(cudaGetLastError());
    return 2;
}

}  // namespace hvn
