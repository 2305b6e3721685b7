// CUDA-core kernels of the CNN path (sm_90a):
//   k_conv_ref   generic NHWC implicit-GEMM convolution in fp32 on split-fp16 operands.  It is the
//                on-device referee for the wgmma kernel (same operands, same epilogue) and the
//                executor for layers the tensor-core kernel does not take.  An absent `lo` plane
//                (precision "high": activations and weights stored as hi only) reads as 0.
//   k_conv0      7x7x3 -> 64 stem on the uint8 image (reference net_desc.py:27-35,103,115)
//   k_bnrelu     BatchNorm(eval)+ReLU raw fp32 -> split (dense-unit preact / blk_bna, net_utils.py:98-99,135-142)
//   k_head       1x1 64->out_ch + bias for every branch, softmax / argmax, concat to [B,h,w,C]
//                (reference net_desc.py:62-68, run_desc.py:185-194)
//   k_head_probs the same with the TP softmax probabilities stored instead of their argmax (test-time augmentation)
//   k_head_full  every softmax probability, [np p0, np p1, hv x, hv y, tp p0..] (validation loss)
#include "common.cuh"
#include "conv_epilogue.cuh"
#include "cnn_kernels.h"

namespace hvn {

// ------------------------------------------------------------------------------------------------
constexpr int RF_BM = 64, RF_BN = 64, RF_BK = 16;

__global__ void __launch_bounds__(256) k_conv_ref(const ConvParams P) {
    __shared__ float As[RF_BK][RF_BM + 4];
    __shared__ float Bs[RF_BK][RF_BN + 4];
    const int tid = threadIdx.x, tx = tid & 15, ty = tid >> 4;
    const int lp = tid >> 2, kq = (tid & 3) * 4;
    const long long M = (long long)P.B * P.ho * P.wo;
    const long long m0 = (long long)blockIdx.x * RF_BM;
    const int n0 = blockIdx.y * RF_BN;
    // loader coordinates
    long long pm = m0 + lp;
    bool pvalid = pm < M;
    int ln = 0, loy = 0, lox = 0;
    if (pvalid) {
        ln = (int)(pm / ((long long)P.ho * P.wo));
        int r = (int)(pm - (long long)ln * P.ho * P.wo);
        loy = r / P.wo;
        lox = r - loy * P.wo;
    }
    const int iy0 = loy * P.stride - P.pad_t, ix0 = lox * P.stride - P.pad_l;
    const bool nvalid = (n0 + lp) < P.w.cout;
    float acc[4][4];
#pragma unroll
    for (int i = 0; i < 4; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    for (int tap = 0; tap < P.w.taps; ++tap) {
        int ky = tap / P.w.kw, kx = tap - ky * P.w.kw;
        int iy = iy0 + ky, ix = ix0 + kx;
        bool inb = pvalid && iy >= 0 && iy < P.a.h && ix >= 0 && ix < P.a.w;
        long long aoff = ln * P.a.sN + (long long)iy * P.a.sH + (long long)ix * P.a.sW;
        long long woff = ((long long)tap * P.w.cout + (n0 + lp)) * P.w.cin_pad;
        const int cend = P.a2.hi ? P.cin1 : P.w.cin;
        for (int c0 = 0; c0 < cend; c0 += RF_BK) {
            float a4[4] = {0.f, 0.f, 0.f, 0.f}, b4[4] = {0.f, 0.f, 0.f, 0.f};
            if (inb) {
                uint2 h = *reinterpret_cast<const uint2 *>(P.a.hi + aoff + c0 + kq);
                uint2 l = P.a.lo ? *reinterpret_cast<const uint2 *>(P.a.lo + aoff + c0 + kq) : make_uint2(0u, 0u);
                const __half *hh = reinterpret_cast<const __half *>(&h);
                const __half *ll = reinterpret_cast<const __half *>(&l);
#pragma unroll
                for (int i = 0; i < 4; ++i) a4[i] = join_f16(hh[i], ll[i]);
            }
            if (nvalid) {
                uint2 h = *reinterpret_cast<const uint2 *>(P.w.hi + woff + c0 + kq);
                uint2 l = P.w.lo ? *reinterpret_cast<const uint2 *>(P.w.lo + woff + c0 + kq) : make_uint2(0u, 0u);
                const __half *hh = reinterpret_cast<const __half *>(&h);
                const __half *ll = reinterpret_cast<const __half *>(&l);
#pragma unroll
                for (int i = 0; i < 4; ++i) b4[i] = join_f16(hh[i], ll[i]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) { As[kq + i][lp] = a4[i]; Bs[kq + i][lp] = b4[i]; }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < RF_BK; ++k) {
                float4 a = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
                float4 b = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
                float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            }
            __syncthreads();
        }
    }
    if (P.a2.hi) {  // second source (fused 1x1 shortcut): pixel (oy*s2, ox*s2), weights at K offset cin1
        const int iy = loy * P.a2_stride, ix = lox * P.a2_stride;
        const bool inb = pvalid && iy < P.a2.h && ix < P.a2.w;
        const long long aoff = ln * P.a2.sN + (long long)iy * P.a2.sH + (long long)ix * P.a2.sW;
        const long long woff = (long long)(n0 + lp) * P.w.cin_pad + P.cin1;
        for (int c0 = 0; c0 < P.a2.c; c0 += RF_BK) {
            float a4[4] = {0.f, 0.f, 0.f, 0.f}, b4[4] = {0.f, 0.f, 0.f, 0.f};
            if (inb) {
                uint2 h = *reinterpret_cast<const uint2 *>(P.a2.hi + aoff + c0 + kq);
                uint2 l = P.a2.lo ? *reinterpret_cast<const uint2 *>(P.a2.lo + aoff + c0 + kq) : make_uint2(0u, 0u);
                const __half *hh = reinterpret_cast<const __half *>(&h);
                const __half *ll = reinterpret_cast<const __half *>(&l);
#pragma unroll
                for (int i = 0; i < 4; ++i) a4[i] = join_f16(hh[i], ll[i]);
            }
            if (nvalid) {
                uint2 h = *reinterpret_cast<const uint2 *>(P.w.hi + woff + c0 + kq);
                uint2 l = P.w.lo ? *reinterpret_cast<const uint2 *>(P.w.lo + woff + c0 + kq) : make_uint2(0u, 0u);
                const __half *hh = reinterpret_cast<const __half *>(&h);
                const __half *ll = reinterpret_cast<const __half *>(&l);
#pragma unroll
                for (int i = 0; i < 4; ++i) b4[i] = join_f16(hh[i], ll[i]);
            }
#pragma unroll
            for (int i = 0; i < 4; ++i) { As[kq + i][lp] = a4[i]; Bs[kq + i][lp] = b4[i]; }
            __syncthreads();
#pragma unroll
            for (int k = 0; k < RF_BK; ++k) {
                float4 a = *reinterpret_cast<const float4 *>(&As[k][ty * 4]);
                float4 b = *reinterpret_cast<const float4 *>(&Bs[k][tx * 4]);
                float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
                for (int i = 0; i < 4; ++i)
#pragma unroll
                    for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
            }
            __syncthreads();
        }
    }
    const int c = n0 + tx * 4;
    if (c >= P.w.cout) return;
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        long long m = m0 + ty * 4 + i;
        if (m >= M) continue;
        int n = (int)(m / ((long long)P.ho * P.wo));
        int r = (int)(m - (long long)n * P.ho * P.wo);
        int oy = r / P.wo, ox = r - oy * P.wo;
        conv_epilogue4(P, n, oy, ox, c, acc[i]);
    }
}

void launch_conv_ref(const ConvParams &P, cudaStream_t s) {
    long long M = (long long)P.B * P.ho * P.wo;
    dim3 grid((unsigned)cdiv(M, RF_BM), (unsigned)cdiv(P.w.cout, RF_BN));
    k_conv_ref<<<grid, 256, 0, s>>>(P);
}

// ------------------------------------------------------------------------------------------------
// stem: x/255 -> 7x7 conv (3->64, fp32) -> BN+ReLU -> split.  pad = 3 in `fast` mode, 0 otherwise.
// One block = 128 consecutive output pixels of one row; a thread owns 4 pixels x 16 output channels
// (64 accumulators), so every input value and every weight float4 read from shared memory feeds 16 FMAs
// (8 shared loads per 64 FMAs; the per-pixel form it replaces issued 16 loads per 64).  The 7 input rows
// of the segment are staged as floats already divided by 255 (the reference's own `imgs / 255.0`), zero
// outside the image.  Accumulation order per output is (ky, kx, channel), as in the reference's direct sum.
// Single-plane output (precision "high"): the staged inputs are rounded to fp16 and the host passes weights already
// rounded to fp16 (under the per-channel exponent), so every product is the one k_conv0_tc forms, exact in fp32.
constexpr int C0_PX = 128, C0_IN = (C0_PX + 6) * 3;
__global__ void __launch_bounds__(128) k_conv0(const uint8_t *__restrict__ img, int B, int H, int W, int pad,
                                               const float *__restrict__ wgt /*[7][7][3][64]*/,
                                               const float *__restrict__ scale, const float *__restrict__ shift,
                                               SplitRef out) {
    extern __shared__ float s_w[];          // 7*7*3*64 weights, then 7 x C0_IN input floats
    float *s_in = s_w + 7 * 7 * 3 * 64;
    const int t = threadIdx.x, ho = out.h, wo = out.w;
    const int x0 = blockIdx.x * C0_PX, oy = blockIdx.y, n = blockIdx.z;
    (void)B; (void)ho;
    for (int i = t; i < 7 * 7 * 3 * 64 / 4; i += 128)
        reinterpret_cast<float4 *>(s_w)[i] = reinterpret_cast<const float4 *>(wgt)[i];
    const uint8_t *im = img + (size_t)n * H * W * 3;
    for (int i = t; i < 7 * C0_IN; i += 128) {
        const int row = i / C0_IN, col = i - row * C0_IN;
        const int pxi = col / 3, ch = col - pxi * 3;
        const int iy = oy + row - pad, ix = x0 + pxi - pad;
        float v = 0.f;
        if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = (float)im[((size_t)iy * W + ix) * 3 + ch] / 255.0f;
        s_in[i] = out.lo ? v : __half2float(__float2half_rn(v));
    }
    __syncthreads();
    const int cg = t & 3, pq = t >> 2;      // 16-channel group, pixel quad
    float acc[4][16];
#pragma unroll
    for (int p = 0; p < 4; ++p)
#pragma unroll
        for (int j = 0; j < 16; ++j) acc[p][j] = 0.f;
    for (int ky = 0; ky < 7; ++ky) {
        const float *in_row = s_in + ky * C0_IN + pq * 12;
#pragma unroll
        for (int kx = 0; kx < 7; ++kx) {
#pragma unroll
            for (int ch = 0; ch < 3; ++ch) {
                float v[4];
#pragma unroll
                for (int p = 0; p < 4; ++p) v[p] = in_row[(p + kx) * 3 + ch];
                const float4 *wr = reinterpret_cast<const float4 *>(s_w + ((ky * 7 + kx) * 3 + ch) * 64 + cg * 16);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float4 w4 = wr[j];
#pragma unroll
                    for (int p = 0; p < 4; ++p) {
                        acc[p][4 * j + 0] = fmaf(v[p], w4.x, acc[p][4 * j + 0]);
                        acc[p][4 * j + 1] = fmaf(v[p], w4.y, acc[p][4 * j + 1]);
                        acc[p][4 * j + 2] = fmaf(v[p], w4.z, acc[p][4 * j + 2]);
                        acc[p][4 * j + 3] = fmaf(v[p], w4.w, acc[p][4 * j + 3]);
                    }
                }
            }
        }
    }
    float sc[16], sh[16];
#pragma unroll
    for (int j = 0; j < 16; ++j) { sc[j] = scale[cg * 16 + j]; sh[j] = shift[cg * 16 + j]; }
#pragma unroll
    for (int p = 0; p < 4; ++p) {
        const int ox = x0 + pq * 4 + p;
        if (ox >= wo) continue;
        const long long oo = n * out.sN + (long long)oy * out.sH + (long long)ox * out.sW + cg * 16;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float tv[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) tv[i] = fmaxf(acc[p][4 * j + i] * sc[4 * j + i] + sh[4 * j + i], 0.f);
            store_split4(out, oo + 4 * j, tv);
        }
    }
}

void launch_conv0(const uint8_t *img, int B, int H, int W, int pad, const float *wgt, const float *scale,
                  const float *shift, const SplitRef &out, cudaStream_t s) {
    static bool attr_set = false;
    const int smem = (7 * 7 * 3 * 64 + 7 * C0_IN) * 4;
    if (!attr_set) {
        cudaFuncSetAttribute(k_conv0, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
        attr_set = true;
    }
    dim3 grid(cdiv(out.w, C0_PX), out.h, B);
    k_conv0<<<grid, 128, smem, s>>>(img, B, H, W, pad, wgt, scale, shift, out);
}

// ------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) k_bnrelu(RawRef in, int B, const float *__restrict__ scale,
                                                const float *__restrict__ shift, SplitRef out) {
    const int c4 = in.c / 4;
    long long total = (long long)B * in.h * in.w * c4;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        int cq = (int)(i % c4);
        long long pix = i / c4;
        int x = (int)(pix % in.w);
        long long t = pix / in.w;
        int y = (int)(t % in.h);
        int n = (int)(t / in.h);
        int c = cq * 4;
        const float4 v = *reinterpret_cast<const float4 *>(in.p + n * in.sN + (long long)y * in.sH +
                                                           (long long)x * in.sW + c);
        const float4 s = *reinterpret_cast<const float4 *>(scale + c);
        const float4 b = *reinterpret_cast<const float4 *>(shift + c);
        float tt[4] = {v.x * s.x + b.x, v.y * s.y + b.y, v.z * s.z + b.z, v.w * s.w + b.w};
        // a NaN input raises the range flag like it does in the XF transform that replaces this pass (the ReLU below
        // would turn it into 0)
        if (out.flag && (tt[0] != tt[0] || tt[1] != tt[1] || tt[2] != tt[2] || tt[3] != tt[3])) *out.flag = 1u;
#pragma unroll
        for (int k = 0; k < 4; ++k) tt[k] = fmaxf(tt[k], 0.f);
        __half oh[4], ol[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) split_f32(tt[k], oh[k], ol[k], out.flag);
        long long oo = n * out.sN + (long long)y * out.sH + (long long)x * out.sW + c;
        *reinterpret_cast<uint2 *>(out.hi + oo) = *reinterpret_cast<uint2 *>(oh);
        if (out.lo) *reinterpret_cast<uint2 *>(out.lo + oo) = *reinterpret_cast<uint2 *>(ol);
    }
}

void launch_bnrelu(const RawRef &in, int B, const float *scale, const float *shift, const SplitRef &out,
                   cudaStream_t s) {
    long long total = (long long)B * in.h * in.w * (in.c / 4);
    int blocks = (int)std::min<long long>(cdiv(total, 256), 132 * 16);
    k_bnrelu<<<blocks, 256, 0, s>>>(in, B, scale, shift, out);
}

// ------------------------------------------------------------------------------------------------
// out(2y+dy, 2x+dx) = split( in(y,x) + skip(2y+dy, 2x+dx) ) : 2x nearest-neighbour upsample + skip add
// (reference net_utils.py:284-294, net_desc.py:133-139) as a streaming pass over the OUTPUT pixels.
__global__ void __launch_bounds__(256) k_up2_add(RawRef in, int B, SplitRef skip, SplitRef out) {
    const int c8 = in.c / 8, oh = 2 * in.h, ow = 2 * in.w;
    const long long total = (long long)B * oh * ow * c8;
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < total;
         i += (long long)gridDim.x * blockDim.x) {
        const int cq = (int)(i % c8);
        long long pix = i / c8;
        const int X = (int)(pix % ow);
        long long t = pix / ow;
        const int Y = (int)(t % oh), n = (int)(t / oh);
        const int c = cq * 8;
        const float *ip = in.p + n * in.sN + (long long)(Y >> 1) * in.sH + (long long)(X >> 1) * in.sW + c;
        const float4 v0 = *reinterpret_cast<const float4 *>(ip), v1 = *reinterpret_cast<const float4 *>(ip + 4);
        const long long so = n * skip.sN + (long long)Y * skip.sH + (long long)X * skip.sW + c;
        const uint4 sh = *reinterpret_cast<const uint4 *>(skip.hi + so);
        const uint4 sl = skip.lo ? *reinterpret_cast<const uint4 *>(skip.lo + so) : make_uint4(0u, 0u, 0u, 0u);
        const __half *hh = reinterpret_cast<const __half *>(&sh), *ll = reinterpret_cast<const __half *>(&sl);
        const float v[8] = {v0.x, v0.y, v0.z, v0.w, v1.x, v1.y, v1.z, v1.w};
        __half oh8[8], ol8[8];
#pragma unroll
        for (int k = 0; k < 8; ++k) split_f32(v[k] + join_f16(hh[k], ll[k]), oh8[k], ol8[k], out.flag);
        const long long oo = n * out.sN + (long long)Y * out.sH + (long long)X * out.sW + c;
        *reinterpret_cast<uint4 *>(out.hi + oo) = *reinterpret_cast<uint4 *>(oh8);
        if (out.lo) *reinterpret_cast<uint4 *>(out.lo + oo) = *reinterpret_cast<uint4 *>(ol8);
    }
}

void launch_up2_add(const RawRef &in, int B, const SplitRef &skip, const SplitRef &out, cudaStream_t s) {
    long long total = (long long)B * 4 * in.h * in.w * (in.c / 8);
    int blocks = (int)std::min<long long>(cdiv(total, 256), 132 * 32);
    k_up2_add<<<blocks, 256, 0, s>>>(in, B, skip, out);
}

// ------------------------------------------------------------------------------------------------
// heads.  feat[b] is the BN+ReLU'd 64-channel map of branch b (order tp?, np, hv).  OUT_PLAIN: [tp argmax?, np p1,
// hv x, hv y].  OUT_PROBS: the TP branch stores its out_ch softmax probabilities instead of their argmax (test-time
// augmentation merges those).  OUT_FULL: [np p0, np p1, hv x, hv y, tp p0..] (the validation loss needs every
// probability).  NP, HV and the TP probabilities come from the same code in all three variants.
template <int OUT> __device__ __forceinline__ void head_body(const HeadParams &P) {
    constexpr bool PROBS = OUT != OUT_PLAIN;
    __shared__ float s_w[3][HVN_MAX_TYPES][64];
    __shared__ float s_b[3][HVN_MAX_TYPES];
    for (int i = threadIdx.x; i < 3 * HVN_MAX_TYPES * 64; i += blockDim.x) {
        int b = i / (HVN_MAX_TYPES * 64), r = i - b * HVN_MAX_TYPES * 64, o = r / 64, k = r - o * 64;
        s_w[b][o][k] = (b < P.nbranch && o < P.out_ch[b]) ? P.w[b][o * 64 + k] : 0.f;
    }
    for (int i = threadIdx.x; i < 3 * HVN_MAX_TYPES; i += blockDim.x) {
        int b = i / HVN_MAX_TYPES, o = i - b * HVN_MAX_TYPES;
        s_b[b][o] = (b < P.nbranch && o < P.out_ch[b]) ? P.bias[b][o] : 0.f;
    }
    __syncthreads();
    long long M = (long long)P.B * P.h * P.w_;
    long long m = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (m >= M) return;
    int n = (int)(m / ((long long)P.h * P.w_));
    int r = (int)(m - (long long)n * P.h * P.w_);
    int y = r / P.w_, x = r - y * P.w_;
    float *out = P.out + m * P.C;
    int oc = 0;
    for (int b = 0; b < P.nbranch; ++b) {
        if (OUT == OUT_FULL) oc = P.kind[b] == HEAD_NP ? 0 : (P.kind[b] == HEAD_HV ? 2 : 4);
        const SplitRef &f = P.feat[b];
        long long fo = n * f.sN + (long long)y * f.sH + (long long)x * f.sW;
        float logit[HVN_MAX_TYPES];
        const int och = P.out_ch[b];
        for (int o = 0; o < och; ++o) logit[o] = 0.f;
        for (int k = 0; k < 64; k += 4) {
            uint2 h = *reinterpret_cast<const uint2 *>(f.hi + fo + k);
            uint2 l = f.lo ? *reinterpret_cast<const uint2 *>(f.lo + fo + k) : make_uint2(0u, 0u);
            const __half *hh = reinterpret_cast<const __half *>(&h);
            const __half *ll = reinterpret_cast<const __half *>(&l);
            float a[4];
#pragma unroll
            for (int i = 0; i < 4; ++i) a[i] = join_f16(hh[i], ll[i]);
            for (int o = 0; o < och; ++o)
#pragma unroll
                for (int i = 0; i < 4; ++i) logit[o] = fmaf(a[i], s_w[b][o][k + i], logit[o]);
        }
        float mx = -INFINITY;
        for (int o = 0; o < och; ++o) { logit[o] += s_b[b][o]; mx = fmaxf(mx, logit[o]); }
        if (P.kind[b] == HEAD_HV) {  // raw regression outputs
            out[oc++] = logit[0];
            out[oc++] = logit[1];
        } else {
            float sum = 0.f, e[HVN_MAX_TYPES];
            for (int o = 0; o < och; ++o) { e[o] = expf(logit[o] - mx); sum += e[o]; }
            if (P.kind[b] == HEAD_NP) {
                if (OUT == OUT_FULL) out[oc++] = e[0] / sum;
                out[oc++] = e[1] / sum;  // softmax(np)[..., 1]
            } else if (PROBS) {          // softmax(tp)
                for (int o = 0; o < och; ++o) out[oc++] = e[o] / sum;
            } else {                     // argmax(softmax(tp)), first maximal index, as float
                int best = 0;
                float bv = e[0] / sum;
                for (int o = 1; o < och; ++o) { float pv = e[o] / sum; if (pv > bv) { bv = pv; best = o; } }
                out[oc++] = (float)best;
            }
        }
    }
}
__global__ void __launch_bounds__(128) k_head(HeadParams P) { head_body<OUT_PLAIN>(P); }
__global__ void __launch_bounds__(128) k_head_probs(HeadParams P) { head_body<OUT_PROBS>(P); }
__global__ void __launch_bounds__(128) k_head_full(HeadParams P) { head_body<OUT_FULL>(P); }

void launch_head(const HeadParams &P, cudaStream_t s) {
    long long M = (long long)P.B * P.h * P.w_;
    k_head<<<cdiv(M, 128), 128, 0, s>>>(P);
}
void launch_head_probs(const HeadParams &P, cudaStream_t s) {
    long long M = (long long)P.B * P.h * P.w_;
    k_head_probs<<<cdiv(M, 128), 128, 0, s>>>(P);
}
void launch_head_full(const HeadParams &P, cudaStream_t s) {
    long long M = (long long)P.B * P.h * P.w_;
    k_head_full<<<cdiv(M, 128), 128, 0, s>>>(P);
}

}  // namespace hvn
