// Test-time augmentation kernels (see tta.h for the view definition and the merge rule).
//   k_tta_views  u8 patches -> their eight dihedral views, view t of input i in slot 8i + t
//   k_tta_merge  the probability head's output on the views -> one k_head-layout map per input
//   k_tta_merge_full  k_head_full's output on the views -> one k_head_full-layout map per input (validation loss)
// Both move a few bytes per pixel against the network's ~1e6 FLOP per pixel: HBM-bound, one thread per pixel.
#include "tta.h"

#include <algorithm>

#include "cnn_kernels.h"
#include "common.cuh"

namespace hvn {

__global__ void __launch_bounds__(256) k_tta_views(const uint8_t *__restrict__ in, int n, int S,
                                                   uint8_t *__restrict__ out) {
    const long long SS = (long long)S * S, total = 8ll * n * SS;
    for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < total; m += (long long)gridDim.x * blockDim.x) {
        const long long slot = m / SS;
        const int p = (int)(m - slot * SS), t = (int)(slot & 7);
        const long long i = slot >> 3;
        int y = p / S, x = p - y * S;
        // V_t = rot90^k(flip^f(x)).  rot90 reads b[y][x] = a[x][S-1-y]: undo the k rotations, then the flip.
        for (int r = 0; r < (t & 3); ++r) { const int ny = x; x = S - 1 - y; y = ny; }
        if (t >> 2) x = S - 1 - x;
        const uint8_t *src = in + ((i * S + y) * S + x) * 3;
        uint8_t *dst = out + m * 3;
        dst[0] = src[0];
        dst[1] = src[1];
        dst[2] = src[2];
    }
}

// FULL = false: probs in k_head_probs' layout [tp p0..?, np, h, v] -> k_head's layout.  FULL = true: probs and out
// both in k_head_full's layout [np p0, np p1, h, v, tp p0..], every channel the mean of the eight views.
template <bool FULL>
__device__ __forceinline__ void tta_merge_body(const float *__restrict__ probs, int n, int h, int nt,
                                               float *__restrict__ out) {
    const long long hh = (long long)h * h, M = (long long)n * hh;
    const int P = FULL ? nt + 4 : nt + 3;
    const int ctp = FULL ? 4 : 0, cnp = FULL ? 1 : nt, chv = FULL ? 2 : nt + 1;  // input channels
    for (long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x; m < M; m += (long long)gridDim.x * blockDim.x) {
        const long long i = m / hh;
        const int p = (int)(m - i * hh), y = p / h, x = p - y * h;
        float tp[HVN_MAX_TYPES], np0 = 0.f, np_ = 0.f, hs = 0.f, vs = 0.f;
#pragma unroll 1
        for (int t = 0; t < 8; ++t) {
            const int k = t & 3;
            // u_t = flip^f(rot90^-k(y_t)): undo the flip, then the k inverse rotations (rot90(., -1) reads
            // b[y][x] = a[h-1-x][y])
            int sy = y, sx = (t >> 2) ? h - 1 - x : x;
            for (int r = 0; r < k; ++r) { const int ny = h - 1 - sx; sx = sy; sy = ny; }
            const float *q = probs + (((i * 8 + t) * h + sy) * h + sx) * P;
            float hv = q[chv], vv = q[chv + 1];
            for (int r = 0; r < k; ++r) { const float nh = -vv; vv = hv; hv = nh; }
            if (t >> 2) hv = -hv;
            if (t == 0) {
                for (int o = 0; o < nt; ++o) tp[o] = q[ctp + o];
                if (FULL) np0 = q[0];
                np_ = q[cnp]; hs = hv; vs = vv;
            } else {
                for (int o = 0; o < nt; ++o) tp[o] += q[ctp + o];
                if (FULL) np0 += q[0];
                np_ += q[cnp]; hs += hv; vs += vv;
            }
        }
        if (FULL) {
            float *o_ = out + m * P;
            o_[0] = np0 * 0.125f;
            o_[1] = np_ * 0.125f;
            o_[2] = hs * 0.125f;
            o_[3] = vs * 0.125f;
            for (int o = 0; o < nt; ++o) o_[4 + o] = tp[o] * 0.125f;
            continue;
        }
        float *o_ = out + m * (nt > 0 ? 4 : 3);
        int c = 0;
        if (nt > 0) {  // argmax of the mean probability, first maximal index, as float (k_head's rule)
            int best = 0;
            float bv = tp[0] * 0.125f;
            for (int o = 1; o < nt; ++o) { const float pv = tp[o] * 0.125f; if (pv > bv) { bv = pv; best = o; } }
            o_[c++] = (float)best;
        }
        o_[c++] = np_ * 0.125f;
        o_[c++] = hs * 0.125f;
        o_[c++] = vs * 0.125f;
    }
}

__global__ void __launch_bounds__(128) k_tta_merge(const float *__restrict__ probs, int n, int h, int nt,
                                                   float *__restrict__ out) {
    tta_merge_body<false>(probs, n, h, nt, out);
}
__global__ void __launch_bounds__(128) k_tta_merge_full(const float *__restrict__ probs, int n, int h, int nt,
                                                        float *__restrict__ out) {
    tta_merge_body<true>(probs, n, h, nt, out);
}

void launch_tta_views(const uint8_t *imgs, int n, int S, uint8_t *views, cudaStream_t s) {
    const long long total = 8ll * n * S * S;
    k_tta_views<<<(int)std::min<long long>(cdiv(total, 256), 132 * 32), 256, 0, s>>>(imgs, n, S, views);
}

void launch_tta_merge(const float *probs, int n, int h, int nr_types, float *out, cudaStream_t s) {
    const long long M = (long long)n * h * h;
    k_tta_merge<<<(int)std::min<long long>(cdiv(M, 128), 132 * 64), 128, 0, s>>>(probs, n, h, nr_types, out);
}

void launch_tta_merge_full(const float *probs, int n, int h, int nr_types, float *out, cudaStream_t s) {
    const long long M = (long long)n * h * h;
    k_tta_merge_full<<<(int)std::min<long long>(cdiv(M, 128), 132 * 64), 128, 0, s>>>(probs, n, h, nr_types, out);
}

}  // namespace hvn
