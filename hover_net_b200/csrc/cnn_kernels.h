// Launch interfaces of the CNN kernels (conv_ref.cu, conv_tc.cu).
#pragma once
#include <cuda_runtime.h>
#include "conv_params.h"

#define HVN_MAX_TYPES 16

namespace hvn {

enum HeadKind { HEAD_TP = 0, HEAD_NP = 1, HEAD_HV = 2 };
// what the heads store per pixel: launch_head, launch_head_probs, launch_head_full
enum HeadOut { OUT_PLAIN = 0, OUT_PROBS = 1, OUT_FULL = 2 };

struct HeadParams {
    int nbranch = 0;
    SplitRef feat[3];
    const float *w[3] = {nullptr, nullptr, nullptr};     // [out_ch][64]
    const float *bias[3] = {nullptr, nullptr, nullptr};
    int out_ch[3] = {0, 0, 0};
    int kind[3] = {0, 0, 0};
    int B = 0, h = 0, w_ = 0, C = 0;
    float *out = nullptr;                                 // [B,h,w,C]
};

void launch_conv_ref(const ConvParams &P, cudaStream_t s);
void launch_conv0(const uint8_t *img, int B, int H, int W, int pad, const float *wgt, const float *scale,
                  const float *shift, const SplitRef &out, cudaStream_t s);
// tensor-core stem (conv_tc.cu): same result as launch_conv0 from weights in [1][64][192] split layout
bool conv0_tc_supported(int H, int W, int pad, const SplitRef &out);
void launch_conv0_tc(const uint8_t *img, int B, int H, int W, int pad, const ConvWeights &w, const float *scale,
                     const float *shift, const SplitRef &out, cudaStream_t s);
void launch_bnrelu(const RawRef &in, int B, const float *scale, const float *shift, const SplitRef &out,
                   cudaStream_t s);
void launch_head(const HeadParams &P, cudaStream_t s);
// the heads with the TP branch's out_ch softmax probabilities in place of its argmax: C = out_ch(tp) + 3
void launch_head_probs(const HeadParams &P, cudaStream_t s);
// every softmax probability, in a fixed order whatever the branch order: C = 4 + out_ch(tp) =
// [np p0, np p1, hv x, hv y, tp p0 .. p(nt-1)] (the layout of the validation loss)
void launch_head_full(const HeadParams &P, cudaStream_t s);
void launch_up2_add(const RawRef &in, int B, const SplitRef &skip, const SplitRef &out, cudaStream_t s);

// wgmma path (conv_tc.cu).  tc_plan() decides eligibility and builds the TMA descriptors once per
// (layer, buffer geometry); tc_launch() issues the kernel.
struct TcPlan {
    bool ok = false;
    unsigned char tmap_a_hi[128], tmap_a_lo[128], tmap_w_hi[128], tmap_w_lo[128];
    unsigned char tmap_a2_hi[128], tmap_a2_lo[128];  // second GEMM source (fused shortcut), if any
    // epilogue tensors, 32-channel boxes of one M-tile: residual (load), raw and split outputs (bulk stores)
    unsigned char tmap_res[128], tmap_out_raw[128], tmap_out_hi[128], tmap_out_lo[128];
    int epi_tma = 0;             // 1: the epilogue tensors move by TMA; 0: a flat tile over a cropped view, copied by
                                 // the consumer threads from the same shared-memory staging (no TMA box describes it)
    int bw = 0, bh = 0;          // M-tile = bw x bh output pixels of one image
    int tiles_x = 0, tiles_y = 0;
    int block_n = 0;
    int flat = 0;                // 1x1 stride-1 dense view: M flattened over B*H*W
    int single = 0;              // precision "high": hi planes only, one wgmma per K=16 step (no lo tensor maps)
};
bool tc_plan(const ConvParams &P, TcPlan &plan);
void tc_launch(const ConvParams &P, const TcPlan &plan, cudaStream_t s);
void tc_set_block_n(int n);      // tuning knobs (0 = automatic)
void tc_set_seg_chunks(int n);
void tc_set_prefetch(int n);     // L2 prefetch distance in K-slices for flat (2-D map) operands, 0 = off
void tc_set_xf_trunc(int on);    // XF transform warps: truncating hi/lo split (1, default) or round-to-nearest (0)
// the k_conv_tc instantiation the last tc_launch issued: BLOCK_N | epilogue (EPI_*) << 8 | XF << 12 | ONE << 13
int tc_last_dispatch();

}  // namespace hvn
