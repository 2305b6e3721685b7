// Test-only entry points into the CNN kernels, one operator at a time (tests/test_conv_kernels_gpu.py).
//
// They call the internal launchers of cnn_kernels.h directly on device memory the caller owns, synchronise, and report
// CUDA errors as return codes.  This library is linked from the objects libhvn.so is built from (conv_tc.o, conv_ref.o)
// and is not part of the product or its C ABI.
//
// Views are passed as 8 int64 each: {hi (or fp32 data) pointer, lo pointer (0 = none), sN, sH, sW, h, w, c}, element
// strides, the pointers already offset to the view's origin.  A null first pointer leaves the ConvParams field unset.
#include <cstdio>
#include <cstring>

#include "../../hover_net_b200/csrc/cnn_kernels.h"
#include "../../hover_net_b200/csrc/common.cuh"

using namespace hvn;

namespace {

SplitRef split_view(const long long *v, unsigned int *flag) {
    SplitRef r;
    r.hi = reinterpret_cast<__half *>(v[0]);
    r.lo = reinterpret_cast<__half *>(v[1]);
    r.sN = v[2]; r.sH = (int)v[3]; r.sW = (int)v[4];
    r.h = (int)v[5]; r.w = (int)v[6]; r.c = (int)v[7];
    r.flag = flag;
    return r;
}

RawRef raw_view(const long long *v) {
    RawRef r;
    r.p = reinterpret_cast<float *>(v[0]);
    r.sN = v[2]; r.sH = (int)v[3]; r.sW = (int)v[4];
    r.h = (int)v[5]; r.w = (int)v[6]; r.c = (int)v[7];
    return r;
}

template <typename T> T *ptr(long long p) { return reinterpret_cast<T *>(p); }

int finish() {
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        fprintf(stderr, "conv_probe: %s\n", cudaGetErrorString(e));
        return -2;
    }
    return 0;
}

}  // namespace

// Convolution layout of `d` (int64):
//   [0,8) a   [8,16) a_raw   [16,24) a2   [24,32) res   [32,40) out_raw   [40,48) out_split   [48,56) skip
//   56 w.hi  57 w.lo  58 w.oscale  59 taps  60 cout  61 cin  62 cin_pad  63 kh  64 kw
//   65 in_scale  66 in_shift  67 scale  68 shift  69 range flag (unsigned int *)
//   70 a2_stride  71 cin1  72 stride  73 pad_t  74 pad_l  75 B  76 ho  77 wo  78 relu  79 up2
// path 0: k_conv_tc (return 1 when tc_plan declines the layer), path 1: k_conv_ref (an XF layer first materialises
// split(relu(a_raw * in_scale + in_shift)) into `a` with k_bnrelu, as the engine's referee does).
// info[10]: plan ok, block_n, flat, bw, bh, single, epilogue (EPI_*), XF, ONE as dispatched, BLOCK_N as dispatched.
extern "C" int probe_conv(const long long *d, int path, int *info) {
    unsigned int *flag = ptr<unsigned int>(d[69]);
    ConvParams P;
    P.a = split_view(d + 0, flag);
    if (d[8]) P.a_raw = raw_view(d + 8);
    if (d[16]) P.a2 = split_view(d + 16, flag);
    if (d[24]) P.res = raw_view(d + 24);
    if (d[32]) P.out_raw = raw_view(d + 32);
    if (d[40]) P.out_split = split_view(d + 40, flag);
    if (d[48]) P.skip = split_view(d + 48, flag);
    P.w.hi = ptr<__half>(d[56]); P.w.lo = ptr<__half>(d[57]); P.w.oscale = ptr<const float>(d[58]);
    P.w.taps = (int)d[59]; P.w.cout = (int)d[60]; P.w.cin = (int)d[61]; P.w.cin_pad = (int)d[62];
    P.w.kh = (int)d[63]; P.w.kw = (int)d[64];
    P.in_scale = ptr<const float>(d[65]); P.in_shift = ptr<const float>(d[66]);
    P.scale = ptr<const float>(d[67]); P.shift = ptr<const float>(d[68]);
    P.a2_stride = (int)d[70]; P.cin1 = (int)d[71]; P.stride = (int)d[72]; P.pad_t = (int)d[73]; P.pad_l = (int)d[74];
    P.B = (int)d[75]; P.ho = (int)d[76]; P.wo = (int)d[77]; P.relu = (int)d[78]; P.up2 = (int)d[79];
    memset(info, 0, 10 * sizeof(int));
    try {
        if (path == 0) {
            TcPlan pl;
            if (!tc_plan(P, pl)) return 1;
            info[0] = pl.ok; info[1] = pl.block_n; info[2] = pl.flat; info[3] = pl.bw; info[4] = pl.bh; info[5] = pl.single;
            tc_launch(P, pl, 0);
            const int disp = tc_last_dispatch();
            info[6] = (disp >> 8) & 15; info[7] = (disp >> 12) & 1; info[8] = (disp >> 13) & 1; info[9] = disp & 255;
        } else {
            if (P.in_scale) {
                launch_bnrelu(P.a_raw, P.B, P.in_scale, P.in_shift, P.a, 0);
                P.in_scale = P.in_shift = nullptr;
            }
            launch_conv_ref(P, 0);
        }
    } catch (const Error &e) {
        fprintf(stderr, "conv_probe: %s\n", e.what());
        return e.code;
    }
    return finish();
}

// Stem.  path 0: k_conv0_tc with [64][192] weight planes (w_hi, w_lo, oscale); path 1: k_conv0 with fp32 weights
// [7][7][3][64] (wgt).  Returns 1 when the tensor-core stem does not take the shape.
extern "C" int probe_conv0(long long img, int B, int H, int W, int pad, int path, long long w_hi, long long w_lo,
                           long long oscale, long long wgt, long long scale, long long shift, const long long *out,
                           long long flag) {
    const SplitRef o = split_view(out, ptr<unsigned int>(flag));
    try {
        if (path == 0) {
            if (!conv0_tc_supported(H, W, pad, o)) return 1;
            ConvWeights cw;
            cw.hi = ptr<__half>(w_hi); cw.lo = ptr<__half>(w_lo); cw.oscale = ptr<const float>(oscale);
            cw.taps = 1; cw.kh = cw.kw = 1; cw.cout = 64; cw.cin = 168; cw.cin_pad = 192;
            launch_conv0_tc(ptr<const uint8_t>(img), B, H, W, pad, cw, ptr<const float>(scale), ptr<const float>(shift), o, 0);
        } else {
            launch_conv0(ptr<const uint8_t>(img), B, H, W, pad, ptr<const float>(wgt), ptr<const float>(scale),
                         ptr<const float>(shift), o, 0);
        }
    } catch (const Error &e) {
        fprintf(stderr, "conv_probe: %s\n", e.what());
        return e.code;
    }
    return finish();
}

extern "C" int probe_bnrelu(const long long *in, int B, long long scale, long long shift, const long long *out, long long flag) {
    launch_bnrelu(raw_view(in), B, ptr<const float>(scale), ptr<const float>(shift), split_view(out, ptr<unsigned int>(flag)), 0);
    return finish();
}

extern "C" int probe_up2_add(const long long *in, int B, const long long *skip, const long long *out, long long flag) {
    launch_up2_add(raw_view(in), B, split_view(skip, nullptr), split_view(out, ptr<unsigned int>(flag)), 0);
    return finish();
}

// Heads: feat = 3 split views, w / bias / out_ch / kind per branch; out [B,h,w,C] fp32.
extern "C" int probe_head(int nbranch, const long long *feat, const long long *w, const long long *bias, const int *out_ch,
                          const int *kind, int B, int h, int w_, int C, long long out) {
    HeadParams P;
    P.nbranch = nbranch;
    for (int b = 0; b < nbranch; ++b) {
        P.feat[b] = split_view(feat + 8 * b, nullptr);
        P.w[b] = ptr<const float>(w[b]); P.bias[b] = ptr<const float>(bias[b]);
        P.out_ch[b] = out_ch[b]; P.kind[b] = kind[b];
    }
    P.B = B; P.h = h; P.w_ = w_; P.C = C; P.out = ptr<float>(out);
    launch_head(P, 0);
    return finish();
}

// Process-wide k_conv_tc knobs of this library's copy of conv_tc.o (the engine's defaults: 0, 4, 4, 1).
extern "C" void probe_set_knobs(int block_n, int seg_chunks, int prefetch, int xf_trunc) {
    tc_set_block_n(block_n);
    tc_set_seg_chunks(seg_chunks);
    tc_set_prefetch(prefetch);
    tc_set_xf_trunc(xf_trunc);
}
