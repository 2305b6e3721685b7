// Host-side interface of the validation loss reduction (loss.cu): the terms of the reference's training objective
// (models/hovernet/utils.py xentropy_loss, dice_loss, mse_loss, msge_loss) summed over a batch, deterministically.
#pragma once
#include "common.cuh"

namespace hvn {

// Slots of the sums (double), in this order:
//   0 np_ce    sum over pixels of -log q_true, q = p / (p0 + p1) clamped to [1e-7, 1 - 1e-7] (fp32 bounds)
//   1 I0  2 I1 sum of p_c * t_c (NP softmax against the one-hot of inst > 0)
//   3 L0  4 L1 sum of p_c
//   5 R0  6 R1 sum of t_c
//   7 hv_sq    sum of (pred_hv - true_hv)^2 over both channels (fp32 differences; hvn_valid's hv_sse)
//   8 msge_num sum of f * ((G_h(p) - G_h(t))^2 + (G_v(p) - G_v(t))^2), G the 5x5 Sobel of get_sobel_kernel(5) as a
//              cross-correlation with zero padding at the border of the crop, f = inst > 0
//   9 focus    sum of f
// and with nr_types > 0: 10 tp_ce, then I_k (11 + k), L_k (11 + nt + k), R_k (11 + 2 nt + k) for k < nt.
enum LossSlot { LS_NP_CE = 0, LS_NP_I = 1, LS_NP_L = 3, LS_NP_R = 5, LS_HV_SQ = 7, LS_MSGE = 8, LS_FOCUS = 9,
                LS_TP_CE = 10, LS_TP_I = 11 };
inline int loss_nsums(int nr_types) { return 10 + (nr_types > 0 ? 1 + 3 * nr_types : 0); }

struct LossWork {
    int nblk = 0;            // blocks of the per-pixel pass (32 x 32 output pixels of one map each)
    double *part = nullptr;  // [nsums][nblk] per-block partials
    int *err = nullptr;      // [1] a type id outside 0..nr_types-1 inside the crop
};

// Partials and flag: 8 * nsums bytes per 32 x 32 tile of the crop, plus 512.
size_t loss_workspace_bytes(int n, int h, int w, int nr_types);

// probs float32 [n,h,w,4+nr_types] (k_head_full's layout: np p0, np p1, hv x, hv y, tp p0..), inst / type int32
// [n,H,W] (type may be null when nr_types == 0), hv targets float32 [n,H,W,2]; the maps are read on the centre
// h x w crop (cropping_center).  sums double [loss_nsums(nr_types)] is overwritten; counts int64 [3 + 2*nr_types]
// (hvn_valid's counts) is accumulated into.  Per-block partials go to fixed slots and one fixed-order pass adds
// them, so the sums depend on the inputs and shapes only.  After the stream is synchronised, *w.err != 0 means an
// out-of-range type id.  Returns the number of kernels launched.
int loss_reduce(Arena &arena, cudaStream_t stream, const float *probs, const int *inst, const int *type,
                const float *hv, int n, int H, int W, int h, int w, int nr_types, double *sums, long long *counts,
                LossWork &lw);

}  // namespace hvn
