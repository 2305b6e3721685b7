// Parameter blocks shared by the CUDA-core referee convolution (conv_ref.cu) and the wgmma
// convolution (conv_tc.cu).  Activations are NHWC.  A "split" tensor stores x as two fp16 planes
// hi = fp16(x), lo = fp16(x - hi): x ~= hi + lo to ~2^-22 relative, which lets the tensor cores
// reproduce fp32-grade products with three fp16 MMAs (hi*hi + hi*lo + lo*hi, fp32 accumulate).
// Precision "high" keeps the hi plane alone (lo == nullptr, read as 0 and never written): one fp16 product per MAC,
// the operand precision of TF32.
#pragma once
#include <cuda_fp16.h>
#include <stdint.h>

namespace hvn {

struct SplitRef {            // view into a split NHWC buffer, already offset to (n=0,y0,x0,c0)
    __half *hi = nullptr, *lo = nullptr;
    long long sN = 0;        // element strides
    int sH = 0, sW = 0;
    int h = 0, w = 0, c = 0; // view extent
    // Range guard: a value outside fp16's finite range (|x| > 65504) cannot be stored as hi + lo.  Every store into a
    // split tensor checks it and raises this device flag (the stored value is clamped so that everything downstream
    // stays finite); the host turns a raised flag into HVN_ERR_RANGE instead of returning a silently clamped result.
    unsigned int *flag = nullptr;
};
struct RawRef {              // view into a raw fp32 NHWC buffer
    float *p = nullptr;
    long long sN = 0;
    int sH = 0, sW = 0;
    int h = 0, w = 0, c = 0;
};

struct ConvWeights {         // [tap][cout][cin_pad] fp16 hi/lo, K-major per tap; cin_pad % 64 == 0
    __half *hi = nullptr, *lo = nullptr;
    // Per-output-channel power-of-two exponent: the stored planes hold w * 2^e[cout] with e chosen so that the largest
    // |w| of the channel lies in [2^13, 2^14) -- both planes then stay in fp16's NORMAL range for every weight down
    // to 2^-17 of the channel's maximum (an unscaled |w| < 2^-3 would leave `lo` subnormal, i.e. fewer than the 22
    // bits the split promises; |w| < 6e-8 would vanish).  oscale[cout] = 2^-e is applied to the fp32 accumulator in
    // the epilogue; scaling by powers of two is exact, so results do not depend on e.
    const float *oscale = nullptr;
    int taps = 0, cout = 0, cin = 0, cin_pad = 0, kh = 0, kw = 0;
};

struct ConvParams {
    SplitRef a;              // input view (bounds of the view are the zero-padding bounds)
    // Optional transformed input (1x1 stride-1 layers): A = split(relu(a_raw * in_scale + in_shift)) is
    // formed on the fly by the kernel's transform warps from the raw fp32 tensor, instead of being read
    // from a pre-transformed split tensor.  `a` must then describe the same view (used by the referee).
    RawRef a_raw;
    const float *in_scale = nullptr, *in_shift = nullptr;
    // Optional second GEMM source accumulated into the same output tile (a residual group's 1x1 shortcut
    // convolution fused into unit 0's conv3): D += A2[pixel * a2_stride] . W[:, cin1 : cin1 + a2.c].
    // `w` then holds both weight matrices concatenated along K (cin = cin1 + a2.c, 1 tap, no padding).
    SplitRef a2;
    int a2_stride = 1, cin1 = 0;
    ConvWeights w;
    int stride = 1, pad_t = 0, pad_l = 0;
    int B = 0, ho = 0, wo = 0;
    // epilogue:  v = acc (+ res) ; out_raw = v ; out_split = split(act(v*scale+shift))
    //            up2: out_split(2y+dy,2x+dx) = split(v + skip(2y+dy,2x+dx))   (no scale/shift)
    RawRef res;              // optional residual (may alias out_raw element-for-element)
    RawRef out_raw;          // optional
    SplitRef out_split;      // optional
    const float *scale = nullptr, *shift = nullptr;  // per-cout; nullptr => identity
    int relu = 0;
    int up2 = 0;
    SplitRef skip;           // used when up2
};

}  // namespace hvn
