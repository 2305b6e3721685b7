// Host-side interface of the training targets and the validation reduction (targets.cu).
#pragma once
#include "common.cuh"

namespace hvn {

// Device workspace of one targets call, laid out in an Arena by targets_run.  Per-component accumulators are
// indexed by the component's root pixel (its first pixel in raster order), so they are O(pixels), never O(max id).
struct TargetWork {
    int n = 0, H = 0, W = 0;
    int *L = nullptr;                                    // [n*H*W] union-find parents, then roots (-1: background)
    int *rmin = nullptr, *rmax = nullptr, *cmin = nullptr, *cmax = nullptr;  // full-map extent, inclusive
    int *ncrop = nullptr;                                // pixels inside the centre crop
    int *nbox = nullptr;                                 // pixels inside the sliced, expanded box
    unsigned long long *sy = nullptr, *sx = nullptr;     // sums of (y - box row 0), (x - box col 0) over those
    int *bymin = nullptr, *bymax = nullptr, *bxmin = nullptr, *bxmax = nullptr;  // their extent, inclusive
    int *maxid = nullptr, *ncomp = nullptr;              // [n] largest id, number of components
    int *has_bg = nullptr, *has_bg_crop = nullptr, *nan_com = nullptr;  // [n]
    int *err = nullptr;                                  // [1] a negative id was seen
};

size_t targets_workspace_bytes(int n, int H, int W);

// inst int32 [n,H,W] (device) -> hv float32 [n,H,W,2] (x, y) and flags int32 [n] (HVN_TG_* bits), both device.
// After the stream is synchronised, *w.err != 0 means a negative id, and maxid[m] + ncomp[m] > 2^31 - 1 means the
// reference's int32 renumbering would overflow.  Returns the number of kernels launched.
int targets_run(Arena &arena, cudaStream_t stream, const int *inst, int n, int H, int W, int crop_h, int crop_w,
                float *hv, int *flags, TargetWork &w);

// Validation counts of one batch (run_desc.py proc_valid_step_output): pred float32 [n,h,w,C] (C = 3: np, hv_x,
// hv_y; C = 4: tp, np, hv_x, hv_y), inst / type int32 [n,H,W] (type may be null), hv targets [n,H,W,2]; the maps are
// compared on the centre h x w crop.  counts int64 [3 + 2*nr_types] and sse (double) are accumulated into, not
// cleared.  Returns the number of kernels launched.
int valid_reduce(cudaStream_t stream, const float *pred, const int *inst, const int *type, const float *hv, int n,
                 int H, int W, int h, int w, int C, int nr_types, long long *counts, double *sse);

}  // namespace hvn
