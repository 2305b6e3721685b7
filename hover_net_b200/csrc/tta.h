// Test-time augmentation (option "tta"): the eight dihedral views of square patches, and the merge of the heads'
// outputs on those views back into one map per patch.
//
// View t = 0..7 of a patch x (HWC), k = t % 4, f = t / 4:  V_t(x) = rot90(f ? flip(x, 1) : x, k)  (numpy semantics,
// axes (0, 1)).  Its output map y_t is brought back by rot90(y_t, -k), then flip(., 1) if f; the HV vector
// (h = x-offset, v = y-offset) by (h, v) <- (-v, h) k times, then h <- -h if f.  See DESIGN.md §4.5.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace hvn {

// imgs u8 [n,S,S,3] -> views u8 [8n,S,S,3]; view t of input i goes to slot 8i + t
void launch_tta_views(const uint8_t *imgs, int n, int S, uint8_t *views, cudaStream_t s);
// probs f32 [8n,h,h,nr_types+3] (k_head_probs: the TP softmax probabilities if nr_types > 0, then NP, h, v) ->
// out f32 [n,h,h,C] in k_head's layout (C = 4: TP argmax, NP, h, v; C = 3 without TP).  Per output value the eight
// brought-back views are summed in view order in fp32 and scaled by 1/8; TP takes the argmax of the summed
// probabilities (first maximal index).
void launch_tta_merge(const float *probs, int n, int h, int nr_types, float *out, cudaStream_t s);
// probs f32 [8n,h,h,nr_types+4] in k_head_full's layout (np p0, np p1, h, v, tp p0..) -> out f32 [n,h,h,nr_types+4],
// same layout: every channel is the same view-order fp32 sum scaled by 1/8, so np p1, h and v equal
// launch_tta_merge's bit for bit.
void launch_tta_merge_full(const float *probs, int n, int h, int nr_types, float *out, cudaStream_t s);

}  // namespace hvn
