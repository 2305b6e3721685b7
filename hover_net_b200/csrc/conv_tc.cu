// wgmma convolution for sm_90a (Hopper): im2col-free NHWC implicit GEMM.
//
//   D[pixel, cout] = sum_{tap} sum_{cin}  A_tap[pixel, cin] * W_tap[cout, cin]
//
// * A tiles (128 output pixels x 64 input channels, fp16 hi and lo planes) are fetched by TMA
//   straight from the NHWC activation: a 4-D box (64ch, bw, bh, 1 image) whose origin is shifted
//   by the filter tap, so zero padding / valid cropping / stride-2 sampling are tensor-map
//   addressing (out-of-bounds zero fill, elementStrides) -- no im2col buffer exists anywhere.
//   1x1 stride-1 convolutions over a dense buffer use a flat 2-D [pixels, channels] map instead.
// * W tiles (BLOCK_N couts x 64 cin, hi and lo) come from the [tap][cout][cin] K-major weight tensor.
// * Both operands land in 128B-swizzled shared memory and are read from there by wgmma (both K-major).  Per K=16 step
//   three m64nNk16 instructions accumulate a_hi*w_hi + a_hi*w_lo + a_lo*w_hi in fp32 registers: fp32-grade products
//   from fp16 tensor cores.
// * Single-product variant (ONE, precision "high"): activations and weights are stored as hi only, the stages carry no
//   lo tiles, and each K=16 step is one m64nNk16 a_hi*w_hi -- one fp16 product per MAC with fp32 accumulation, the
//   operand precision of TF32.  The freed shared memory holds more stages; the epilogue stores hi only.
// * Persistent CTAs (one per SM), warp-specialised: warp 0 = TMA producer; warpgroups 1 and 2 = consumers, each issuing
//   the wgmma of 64 of the tile's 128 pixel rows over all BLOCK_N columns and running the fused epilogue (BN/ReLU/
//   residual/upsample) from its accumulator fragment.  A shared-memory ring of STAGES operand slots lets the producer
//   run ahead, also across the consumers' epilogue.
// * Epilogue tensors move by TMA (plain and residual epilogues): the producer loads the residual into a staging ring,
//   the consumers finish each 32-channel chunk there and one thread stores it with bulk tensor stores.
// * Accumulation precision: the K loop is cut into segments of G.seg 64-channel slices; each segment accumulates in the
//   wgmma registers from zero and is then added into a separate fp32 sum with round-to-nearest adds, so the number of
//   products chained inside the tensor core stays bounded however large K is.
// * XF variant (1x1 layers fed by a raw fp32 tensor through a pre-activation BatchNorm+ReLU): three
//   extra "transform" warps build the A tiles themselves -- coalesced fp32 loads, y=relu(x*scale+shift),
//   fp16 hi/lo split, 128B-swizzled st.shared, fence.proxy.async -- so the pre-activated copy of the
//   tensor never exists in HBM (no separate BN/ReLU pass, no second output of the producing layer).
// * Flat (2-D map) operands streamed from HBM get a cp.async.bulk.prefetch.tensor L2 cursor a few K-slices ahead.
#include <cuda.h>
#include <cuda_runtime.h>

#include <algorithm>
#include <cstring>
#include <mutex>
#include <type_traits>

#include "common.cuh"
#include "conv_epilogue.cuh"
#include "cnn_kernels.h"

namespace hvn {

// ------------------------------------------------------------------------------------------------
// PTX wrappers
__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint32_t bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(bar), "r"(count) : "memory");
}
__device__ __forceinline__ void mbar_expect_tx(uint32_t bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint32_t bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(bar) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}
__device__ __forceinline__ void tma_2d(uint32_t dst, const void *tmap, uint32_t bar, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
                 ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_3d(uint32_t dst, const void *tmap, uint32_t bar, int c0, int c1, int c2) {
    asm volatile("cp.async.bulk.tensor.3d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5}], [%2];"
                 ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2) : "memory");
}
__device__ __forceinline__ void tma_4d(uint32_t dst, const void *tmap, uint32_t bar, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
                 ::"r"(dst), "l"(tmap), "r"(bar), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
// Bulk tensor stores shared -> global (epilogue).  Elements outside the tensor map's extent are not written.
__device__ __forceinline__ void tma_store_2d(const void *tmap, uint32_t src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(tmap), "r"(src), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const void *tmap, uint32_t src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(tmap), "r"(src), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void bulk_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
// at most N of this thread's bulk groups still reading shared memory / still writing global memory
template <int N> __device__ __forceinline__ void bulk_wait_read() { asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory"); }
template <int N> __device__ __forceinline__ void bulk_wait() { asm volatile("cp.async.bulk.wait_group %0;" ::"n"(N) : "memory"); }
// the 256 consumer threads (warpgroups 1, 2)
__device__ __forceinline__ void consumers_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }

// L2 prefetch of a tensor-map box: no shared memory, no barrier -- used to run several K-slices ahead of the loads on
// operands that come from HBM (the rings below hold 2-4 slices, less than one DRAM round trip under load)
__device__ __forceinline__ void tma_prefetch_2d(const void *tmap, int c0, int c1) {
    asm volatile("cp.async.bulk.prefetch.tensor.2d.L2.global.tile [%0, {%1, %2}];" ::"l"(tmap), "r"(c0), "r"(c1) : "memory");
}

__device__ __forceinline__ void wg_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wg_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N> __device__ __forceinline__ void wg_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
template <int R> __device__ __forceinline__ void wg_fence_regs(float (&d)[R]) {
#pragma unroll
    for (int i = 0; i < R; ++i) asm volatile("" : "+f"(d[i])::"memory");
}

// K-major, 128B-swizzled operand tile (the layout TMA writes with CU_TENSOR_MAP_SWIZZLE_128B): rows of 128 B, 8-row
// groups 1024 B apart (SBO), LBO unused for swizzled K-major layouts.  Tiles start 1024-aligned, so the base offset is 0;
// the K=16 steps inside a 64-channel slice advance the start address by 32 B (the swizzle is applied to address bits).
__device__ __forceinline__ uint64_t wg_desc(uint32_t saddr) {
    uint64_t d = 0;
    d |= (uint64_t)((saddr & 0x3FFFFu) >> 4);
    d |= (uint64_t)1 << 16;
    d |= (uint64_t)(1024 >> 4) << 32;
    d |= (uint64_t)1 << 62;   // SWIZZLE_128B
    return d;
}

// D[64 x N] (+)= A[64 x 16] * B[16 x N], both operands K-major in shared memory, fp32 accumulators in registers.
// Fragment: register 4j + 2h + e holds row (warp & 3) * 16 + lane / 4 + 8h, column 8j + 2 (lane % 4) + e.
// mma: D = A*B + (accum ? D : 0).  mma0: D = A*B with D write-only (scale-d = false), so the accumulator's previous
// contents are dead for the compiler too and its registers are free between a drain and the next segment's first MMA.
template <int N> struct Wgmma;
#define HVN_F8(M, i) M(d[i]), M(d[i + 1]), M(d[i + 2]), M(d[i + 3]), M(d[i + 4]), M(d[i + 5]), M(d[i + 6]), M(d[i + 7])
#define HVN_D16(M) HVN_F8(M, 0), HVN_F8(M, 8)
#define HVN_D32(M) HVN_D16(M), HVN_F8(M, 16), HVN_F8(M, 24)
#define HVN_D64(M) HVN_D32(M), HVN_F8(M, 32), HVN_F8(M, 40), HVN_F8(M, 48), HVN_F8(M, 56)
#define HVN_WGMMA(N, R, DREGS, P, AB, DCONS)                                                                           \
    template <> struct Wgmma<N> {                                                                                      \
        static __device__ __forceinline__ void mma(float (&d)[R], uint64_t a, uint64_t b, uint32_t accum) {            \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, " P ", 0;\n\twgmma.mma_async.sync.aligned.m64n" #N      \
                         "k16.f32.f16.f16 {" DREGS "}, " AB ", p, 1, 1, 0, 0;\n\t}"                                    \
                         : DCONS("+f") : "l"(a), "l"(b), "r"(accum));                                                  \
        }                                                                                                              \
        static __device__ __forceinline__ void mma0(float (&d)[R], uint64_t a, uint64_t b) {                           \
            asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, 0, 0;\n\twgmma.mma_async.sync.aligned.m64n" #N          \
                         "k16.f32.f16.f16 {" DREGS "}, " AB ", p, 1, 1, 0, 0;\n\t}"                                    \
                         : DCONS("=f") : "l"(a), "l"(b));                                                              \
        }                                                                                                              \
    };
HVN_WGMMA(32, 16, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15", "%18", "%16, %17", HVN_D16)
HVN_WGMMA(64, 32, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31", "%34", "%32, %33", HVN_D32)
HVN_WGMMA(128, 64, "%0,%1,%2,%3,%4,%5,%6,%7,%8,%9,%10,%11,%12,%13,%14,%15,%16,%17,%18,%19,%20,%21,%22,%23,%24,%25,%26,%27,%28,%29,%30,%31,%32,%33,%34,%35,%36,%37,%38,%39,%40,%41,%42,%43,%44,%45,%46,%47,%48,%49,%50,%51,%52,%53,%54,%55,%56,%57,%58,%59,%60,%61,%62,%63", "%66", "%64, %65", HVN_D64)
#undef HVN_WGMMA
#undef HVN_D64
#undef HVN_D32
#undef HVN_D16
#undef HVN_F8

// One 64-channel K-slice of the split product: a_hi*w_hi + a_hi*w_lo + a_lo*w_hi (4 K=16 steps, +32 B each).
// ZERO: the slice starts a segment, its first MMA overwrites the accumulator (write-only); zero: the same at run time.
template <int N, bool ZERO = false>
__device__ __forceinline__ void mma_slice(float (&d)[N / 2], uint32_t a_hi, uint32_t a_lo, uint32_t b_hi, uint32_t b_lo,
                                          bool zero = false) {
    const uint64_t dah = wg_desc(a_hi), dal = wg_desc(a_lo), dbh = wg_desc(b_hi), dbl = wg_desc(b_lo);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        const uint64_t ko = (uint64_t)(2 * k);
        if (ZERO && k == 0) Wgmma<N>::mma0(d, dah + ko, dbh + ko);
        else Wgmma<N>::mma(d, dah + ko, dbh + ko, (zero && k == 0) ? 0u : 1u);
        Wgmma<N>::mma(d, dah + ko, dbl + ko, 1u);
        Wgmma<N>::mma(d, dal + ko, dbh + ko, 1u);
    }
}

// One 64-channel K-slice of the single product a_hi*w_hi (precision "high")
template <int N, bool ZERO = false>
__device__ __forceinline__ void mma_slice1(float (&d)[N / 2], uint32_t a_hi, uint32_t b_hi, bool zero = false) {
    const uint64_t dah = wg_desc(a_hi), dbh = wg_desc(b_hi);
#pragma unroll
    for (int k = 0; k < 4; ++k) {
        if (ZERO && k == 0) Wgmma<N>::mma0(d, dah, dbh);
        else Wgmma<N>::mma(d, dah + 2 * k, dbh + 2 * k, (zero && k == 0) ? 0u : 1u);
    }
}

struct TcGeom {
    int flat, bw, bh, tiles_x, tiles_y, tiles_m, tiles_n, kchunks, seg;
    int k1;  // > 0: K-slices [0,k1) come from the first source, [k1,kchunks) from the second (fused shortcut)
    long long m_total;
    int pf;        // flat (2-D map) operands: L2 prefetch distance in K-slices (0 = off)
    int xf_trunc;  // XF transform: truncating hi/lo split (split4_relu_trunc) instead of the round-to-nearest one
    int epi_tma;   // TcPlan::epi_tma
    int eslot, neslots;  // epilogue staging ring: bytes per slot (one 32-channel chunk of every epilogue tensor), slots
};

constexpr int SMEM_LIMIT = 232448;       // opt-in dynamic shared memory per CTA on sm_90 (227 KB)
constexpr int TC_THREADS = 384;          // warpgroup 0: TMA producer (warp 0) + XF transform (warps 1..3); warpgroups 1, 2: wgmma
constexpr int XF_WARPS = 3;
constexpr int CONS_WARPS = 8;
constexpr int A_TILE_BYTES = 128 * 128;  // 128 rows x 64 fp16
constexpr uint32_t RAW_TILE_BYTES = 128 * 64 * 4;

// One operand stage: A then W tiles, hi planes (and, unless ONE, lo planes) -- [a_hi | a_lo | w_hi | w_lo]
template <int BLOCK_N, bool ONE> __host__ __device__ constexpr int tc_stage_bytes() {
    return (ONE ? 1 : 2) * (A_TILE_BYTES + BLOCK_N * 128);
}
// Epilogue staging (EPI_PLAIN, EPI_RES): a ring of slots, each one 32-channel chunk of the tile (128 rows) of every
// epilogue tensor: [raw fp32 16 KB, 128B-swizzled | hi fp16 8 KB | lo fp16 8 KB, 64B-swizzled].  The raw part exists when
// the layer has a residual or a raw output; the residual lands there and the raw output leaves from there.
constexpr int EPI_RAW_BYTES = 128 * 32 * 4, EPI_HALF_BYTES = 128 * 32 * 2;
constexpr int EPI_MAX_SLOTS = 24;
constexpr int BAR_BYTES = 8 * (2 * 16 + 4 + 2 * EPI_MAX_SLOTS);   // up to 16 operand stages
template <int BLOCK_N, bool XF, bool ONE> constexpr int tc_smem(int stages, int ring) {
    return 1024 + stages * tc_stage_bytes<BLOCK_N, ONE>() + (XF ? 2 * (int)RAW_TILE_BYTES : 0) + ring + BAR_BYTES;
}
// EPI_RES (the memory-bound conv3 layers): two operand stages, the rest is staging ring, so that a whole tile's residual
// can be in flight during the tile's MMA.  EPI_PLAIN: a 32 KB ring beside as many stages as fit.  EPI_UP2 stores from
// registers and has no ring.
template <int BLOCK_N, int MODE, bool XF, bool ONE> constexpr int tc_ring() {
    return MODE == EPI_UP2 ? 0 : MODE == EPI_RES ? (SMEM_LIMIT - tc_smem<BLOCK_N, XF, ONE>(2, 0)) / EPI_RAW_BYTES * EPI_RAW_BYTES
                                                 : 2 * EPI_RAW_BYTES;
}
template <int BLOCK_N, int MODE, bool XF, bool ONE> constexpr int tc_stages() {
    if (MODE == EPI_RES) return 2;
    int s = 1;
    while (tc_smem<BLOCK_N, XF, ONE>(s + 1, tc_ring<BLOCK_N, MODE, XF, ONE>()) <= SMEM_LIMIT) ++s;
    return s;
}
static_assert(tc_stages<128, EPI_PLAIN, false, false>() == 3 && tc_stages<128, EPI_PLAIN, true, false>() == 2 &&
                  tc_stages<64, EPI_PLAIN, false, false>() == 4 && tc_stages<64, EPI_PLAIN, true, false>() == 2 &&
                  tc_stages<32, EPI_PLAIN, false, false>() == 4 && tc_stages<128, EPI_UP2, false, false>() == 3,
              "two-plane stage counts");
static_assert(tc_ring<128, EPI_RES, false, false>() == 6 * EPI_RAW_BYTES, "EPI_RES ring: a 64 KB residual tile in flight");
static_assert(tc_stages<32, EPI_PLAIN, false, true>() <= 16 && tc_ring<32, EPI_RES, false, true>() / EPI_RAW_BYTES <= EPI_MAX_SLOTS,
              "barrier area");

// Output element offsets of one accumulator row (pixel) for EPI_UP2; -1 = no such pixel.
struct PixOff {
    long long raw = -1, spl = -1, skip = -1;
};

__device__ __forceinline__ PixOff pix_offsets_up2(const ConvParams &P, bool valid, int n, int oy, int ox) {
    PixOff o;
    if (!valid) return o;
    if (P.out_raw.p) o.raw = n * P.out_raw.sN + (long long)oy * P.out_raw.sH + (long long)ox * P.out_raw.sW;
    o.spl = n * P.out_split.sN + (long long)(2 * oy) * P.out_split.sH + (long long)(2 * ox) * P.out_split.sW;
    o.skip = n * P.skip.sN + (long long)(2 * oy) * P.skip.sH + (long long)(2 * ox) * P.skip.sW;
    return o;
}

template <bool ONE>
__device__ __forceinline__ void store_split2(const SplitRef &o, long long off, float a, float b) {
    if constexpr (ONE) {
        *reinterpret_cast<__half2 *>(o.hi + off) = __halves2half2(hi_f32(a, o.flag), hi_f32(b, o.flag));
        return;
    }
    __half h0, l0, h1, l1;
    split_f32(a, h0, l0, o.flag);
    split_f32(b, h1, l1, o.flag);
    *reinterpret_cast<__half2 *>(o.hi + off) = __halves2half2(h0, h1);
    *reinterpret_cast<__half2 *>(o.lo + off) = __halves2half2(l0, l1);
}

// fp16 pairs parked in fp32 registers (the epilogue's skip batch lives in the dead accumulator)
__device__ __forceinline__ float ld_bits(const __half *p) { return __uint_as_float(*reinterpret_cast<const uint32_t *>(p)); }
__device__ __forceinline__ __half2 bits_h2(float f) {
    const uint32_t u = __float_as_uint(f);
    return *reinterpret_cast<const __half2 *>(&u);
}

// EPI_UP2, channels c, c+1 of one pixel: v already carries the weight exponent's 2^-e.  The skip pairs of the four
// output pixels were read earlier into `pre`: hi (and, unless ONE, lo) as fp16x2 bits, [d * planes + plane].
template <bool ONE>
__device__ __forceinline__ void epi_finish2_up2(const ConvParams &P, const PixOff &o, int c, float v0, float v1, const float *pre) {
    if (o.raw >= 0) *reinterpret_cast<float2 *>(P.out_raw.p + o.raw + c) = make_float2(v0, v1);
#pragma unroll
    for (int d = 0; d < 4; ++d) {
        const long long oo = o.spl + (d >> 1) * P.out_split.sH + (d & 1) * P.out_split.sW + c;
        if constexpr (ONE) {
            const __half2 sh = bits_h2(pre[d]);
            store_split2<true>(P.out_split, oo, v0 + __half2float(sh.x), v1 + __half2float(sh.y));
        } else {
            const __half2 sh = bits_h2(pre[2 * d]), sl = bits_h2(pre[2 * d + 1]);
            store_split2<false>(P.out_split, oo, v0 + join_f16(sh.x, sl.x), v1 + join_f16(sh.y, sl.y));
        }
    }
}

// Byte offsets inside a staging slot of the fragment pair (row, channels 8 jj + 2 q, +1) of a 32-channel chunk
__device__ __forceinline__ int stg_raw_off(int row, int jj, int q) {   // fp32 [128][32], 128B swizzle
    return row * 128 + (((2 * jj + (q >> 1)) ^ (row & 7)) << 4) + (q & 1) * 8;
}
__device__ __forceinline__ int stg_half_off(int row, int jj, int q) {  // fp16 [128][32], 64B swizzle
    return row * 64 + ((jj ^ ((row >> 1) & 3)) << 4) + q * 4;
}

template <int BLOCK_N, int STAGES, int MODE, bool XF, bool ONE>
__global__ void __launch_bounds__(TC_THREADS, 1)
k_conv_tc(const __grid_constant__ CUtensorMap tm_a_hi, const __grid_constant__ CUtensorMap tm_a_lo,
          const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo,
          const __grid_constant__ CUtensorMap tm_a2_hi, const __grid_constant__ CUtensorMap tm_a2_lo,
          const __grid_constant__ CUtensorMap tm_res, const __grid_constant__ CUtensorMap tm_o_raw,
          const __grid_constant__ CUtensorMap tm_o_hi, const __grid_constant__ CUtensorMap tm_o_lo,
          const ConvParams P, const TcGeom G) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    constexpr int STAGE_BYTES = tc_stage_bytes<BLOCK_N, ONE>();
    constexpr int PLANES = ONE ? 1 : 2;
    constexpr int RING = tc_ring<BLOCK_N, MODE, XF, ONE>();
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    const uint32_t raw_base = smem_base + STAGES * STAGE_BYTES;             // XF: 2-slot ring of raw fp32 [128][64] tiles
    const uint32_t ring_base = raw_base + (XF ? 2 * RAW_TILE_BYTES : 0u);  // epilogue staging ring
    const uint32_t bar_base = ring_base + RING;
    // barriers: full[STAGES], empty[STAGES], raw_full[2], raw_empty[2], epi_full[neslots], epi_free[neslots]
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (STAGES + s); };
    auto rfull_bar = [&](int r) { return bar_base + 8u * (2 * STAGES + r); };
    auto rempty_bar = [&](int r) { return bar_base + 8u * (2 * STAGES + 2 + r); };
    auto efull_bar = [&](int e) { return bar_base + 8u * (2 * STAGES + 4 + e); };
    auto efree_bar = [&](int e) { return bar_base + 8u * (2 * STAGES + 4 + EPI_MAX_SLOTS + e); };
    const bool has_raw = MODE == EPI_RES || P.out_raw.p;   // the slot has a raw part

    // warp index broadcast from lane 0: provably warp-uniform, so the role branches below do not count as divergent
    // paths around the wgmma (ptxas would otherwise serialise them)
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    if (threadIdx.x == 0) {
        for (int s = 0; s < STAGES; ++s) { mbar_init(full_bar(s), XF ? 1 + XF_WARPS : 1); mbar_init(empty_bar(s), CONS_WARPS); }
        if (XF) for (int r = 0; r < 2; ++r) { mbar_init(rfull_bar(r), 1); mbar_init(rempty_bar(r), XF_WARPS); }
        if (RING) for (int e = 0; e < G.neslots; ++e) { mbar_init(efull_bar(e), 1); mbar_init(efree_bar(e), 1); }
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    __syncthreads();

    const int total_tiles = G.tiles_m * G.tiles_n;
    const int taps = P.w.taps;
    const int kiters = taps * G.kchunks;
    const uint32_t tx_bytes = (uint32_t)(PLANES * ((G.flat ? 128 : G.bw * G.bh) * 128 + BLOCK_N * 128));

    if (warp == 0) {
        // ===================== TMA producer =====================
        if (lane == 0) {
            int it_global = 0, ec = 0;
            // L2 prefetch cursor, G.pf K-slices ahead of the loads through the same (tile, slice) sequence.  Flat layers
            // only: their A operand is a whole encoder tensor streamed from HBM.
            const bool pf_on = G.flat && G.pf > 0;
            int pf_tile = blockIdx.x, pf_it = 0;
            auto pf_step = [&]() {
                if (pf_tile >= total_tiles) return;
                const int m0p = (pf_tile / G.tiles_n) * 128;
                if constexpr (XF) tma_prefetch_2d(&tm_a_hi, pf_it * 64, m0p);
                else if (G.k1 > 0 && pf_it >= G.k1) {
                    tma_prefetch_2d(&tm_a2_hi, (pf_it - G.k1) * 64, m0p);
                    if constexpr (!ONE) tma_prefetch_2d(&tm_a2_lo, (pf_it - G.k1) * 64, m0p);
                } else {
                    tma_prefetch_2d(&tm_a_hi, pf_it * 64, m0p);
                    if constexpr (!ONE) tma_prefetch_2d(&tm_a_lo, pf_it * 64, m0p);
                }
                if (++pf_it == kiters) { pf_it = 0; pf_tile += gridDim.x; }
            };
            if (pf_on) for (int i = 0; i < G.pf; ++i) pf_step();
            for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
                const int tm = tile / G.tiles_n, tn = tile - tm * G.tiles_n;
                int n_img = 0, y0 = 0, x0 = 0;
                long long m0 = 0;
                if (G.flat) m0 = (long long)tm * 128;
                else {
                    const int per_img = G.tiles_x * G.tiles_y;
                    n_img = tm / per_img;
                    const int r = tm - n_img * per_img;
                    y0 = (r / G.tiles_x) * G.bh;
                    x0 = (r - (r / G.tiles_x) * G.tiles_x) * G.bw;
                }
                for (int it = 0; it < kiters; ++it, ++it_global) {
                    if (pf_on) pf_step();
                    if constexpr (XF) {
                        // raw fp32 A tile of this K-slice -> staging ring (tm_a_hi is the fp32 map).  Issued before the
                        // wait for the operand stage: the raw slot frees up a whole transform earlier than the stage does.
                        const int r = it_global & 1;
                        const uint32_t rph = (uint32_t)(it_global >> 1) & 1u;
                        mbar_wait(rempty_bar(r), rph ^ 1u);
                        mbar_expect_tx(rfull_bar(r), (uint32_t)((G.flat ? 128 : G.bw * G.bh) * 256));
                        if (G.flat) tma_2d(raw_base + r * RAW_TILE_BYTES, &tm_a_hi, rfull_bar(r), it * 64, (int)m0);
                        else tma_4d(raw_base + r * RAW_TILE_BYTES, &tm_a_hi, rfull_bar(r), it * 64, x0, y0, n_img);
                    }
                    const int s = it_global % STAGES;
                    const uint32_t ph = (uint32_t)(it_global / STAGES) & 1u;
                    mbar_wait(empty_bar(s), ph ^ 1u);
                    const uint32_t sa = smem_base + s * STAGE_BYTES;
                    const uint32_t a_hi = sa, a_lo = sa + A_TILE_BYTES, b_hi = sa + PLANES * A_TILE_BYTES,
                                   b_lo = b_hi + BLOCK_N * 128;
                    const int tap = it / G.kchunks, kc = it - tap * G.kchunks;
                    if constexpr (XF) {  // the A planes of the stage are written by the transform warps; weights land beside them
                        mbar_expect_tx(full_bar(s), (uint32_t)(PLANES * BLOCK_N * 128));
                        tma_3d(b_hi, &tm_w_hi, full_bar(s), kc * 64, tn * BLOCK_N, tap);
                        if constexpr (!ONE) tma_3d(b_lo, &tm_w_lo, full_bar(s), kc * 64, tn * BLOCK_N, tap);
                        continue;
                    }
                    mbar_expect_tx(full_bar(s), tx_bytes);
                    if (G.k1 > 0 && kc >= G.k1) {  // second source: fused 1x1 shortcut on the block input
                        const int c2 = (kc - G.k1) * 64;
                        if (G.flat) {
                            tma_2d(a_hi, &tm_a2_hi, full_bar(s), c2, (int)m0);
                            if constexpr (!ONE) tma_2d(a_lo, &tm_a2_lo, full_bar(s), c2, (int)m0);
                        } else {
                            tma_4d(a_hi, &tm_a2_hi, full_bar(s), c2, x0 * P.a2_stride, y0 * P.a2_stride, n_img);
                            if constexpr (!ONE) tma_4d(a_lo, &tm_a2_lo, full_bar(s), c2, x0 * P.a2_stride, y0 * P.a2_stride, n_img);
                        }
                    } else if (G.flat) {
                        tma_2d(a_hi, &tm_a_hi, full_bar(s), kc * 64, (int)m0);
                        if constexpr (!ONE) tma_2d(a_lo, &tm_a_lo, full_bar(s), kc * 64, (int)m0);
                    } else {
                        const int ky = tap / P.w.kw, kx = tap - ky * P.w.kw;
                        const int cx = x0 * P.stride + kx - P.pad_l, cy = y0 * P.stride + ky - P.pad_t;
                        tma_4d(a_hi, &tm_a_hi, full_bar(s), kc * 64, cx, cy, n_img);
                        if constexpr (!ONE) tma_4d(a_lo, &tm_a_lo, full_bar(s), kc * 64, cx, cy, n_img);
                    }
                    tma_3d(b_hi, &tm_w_hi, full_bar(s), kc * 64, tn * BLOCK_N, tap);
                    if constexpr (!ONE) tma_3d(b_lo, &tm_w_lo, full_bar(s), kc * 64, tn * BLOCK_N, tap);
                    if constexpr (MODE == EPI_RES) {
                        // the tile's residual, one 32-channel chunk per staging slot, behind the tile's last K-slice
                        // (a slot may free up only once this tile's first chunks are stored, so every operand of the
                        // tile must be on its way first): in flight while the tile's MMA runs.  res may alias out_raw
                        // element for element: each (tile, chunk) is loaded here before the same CTA stores it from the
                        // same slot, and no two tiles share an address, so a load never sees another tile's store.
                        if (it == kiters - 1 && G.epi_tma) {
                            const uint32_t bytes = (uint32_t)((G.flat ? 128 : G.bw * G.bh) * 128);
                            for (int q = 0; q < BLOCK_N / 32; ++q, ++ec) {
                                const int e = ec % G.neslots;
                                mbar_wait(efree_bar(e), ((uint32_t)(ec / G.neslots) & 1u) ^ 1u);
                                mbar_expect_tx(efull_bar(e), bytes);
                                const uint32_t dst = ring_base + e * G.eslot;
                                const int c = tn * BLOCK_N + 32 * q;
                                if (G.flat) tma_2d(dst, &tm_res, efull_bar(e), c, (int)m0);
                                else tma_4d(dst, &tm_res, efull_bar(e), c, x0, y0, n_img);
                            }
                        }
                    }
                }
            }
        }
    } else if (XF && warp < 4) {
        // ===================== A-operand transform (warps 1..3, XF only) =====================
        // thread -> (row group rg = t>>4, float4 column l16 = t&15), rows rg + 16*i: raw fp32 staging tile
        // (row-major [128][64], filled by TMA) -> y = relu(x*scale+shift) -> fp16 hi/lo -> swizzled A tiles.
        // All row loads of a K-slice are issued before the first value is used.
        const int t = threadIdx.x - 32;
        const int l16 = t & 15, rg = t >> 4;
        const int wl = t & 31;
        constexpr int RG = XF_WARPS * 2;              // row groups: rows rg, rg + RG, ...
        constexpr int XR = (128 + RG - 1) / RG;       // rows per thread (the last one may not exist: 128 % RG)
        uint8_t *smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
        const uint8_t *raw_gen = smem_raw + (raw_base - smem_u32(smem_raw));
        const int vrows = G.flat ? 128 : G.bw * G.bh;  // rows TMA writes; the rest of a partial box keeps stale bits
        int it_global = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            float rmax = 0.f;
            for (int kc = 0; kc < kiters; ++kc, ++it_global) {  // taps == 1: kiters == kchunks
                const int s = it_global % STAGES;
                const uint32_t ph = (uint32_t)(it_global / STAGES) & 1u;
                const int r = it_global & 1;
                const uint32_t rph = (uint32_t)(it_global >> 1) & 1u;
                const int c = kc * 64 + l16 * 4;
                // channels past cin: TMA zero-fills the raw tile there and scale = shift = 0 keeps them 0 (zero weights
                // must not meet Inf/NaN)
                float4 sc = make_float4(0.f, 0.f, 0.f, 0.f), sh = sc;
                if (c < P.w.cin) {
                    sc = *reinterpret_cast<const float4 *>(P.in_scale + c);
                    sh = *reinterpret_cast<const float4 *>(P.in_shift + c);
                }
                mbar_wait(rfull_bar(r), rph);
                const uint8_t *src = raw_gen + r * RAW_TILE_BYTES + rg * 256 + l16 * 16;
                float4 v[XR];
#pragma unroll
                for (int i = 0; i < XR; ++i)  // rows TMA did not write read as 0: finite, and invisible to the range guard
                    v[i] = rg + RG * i < min(vrows, 128) ? *reinterpret_cast<const float4 *>(src + i * RG * 256) : make_float4(0.f, 0.f, 0.f, 0.f);
                // y = x*scale + shift in place: in-order issue puts every instruction below behind the completed LDS of
                // this lane, so the raw slot can go back to the producer now
#pragma unroll
                for (int i = 0; i < XR; ++i)
                    v[i] = make_float4(fmaf(v[i].x, sc.x, sh.x), fmaf(v[i].y, sc.y, sh.y), fmaf(v[i].z, sc.z, sh.z), fmaf(v[i].w, sc.w, sh.w));
                __syncwarp();
                if (wl == 0) mbar_arrive(rempty_bar(r));
                mbar_wait(empty_bar(s), ph ^ 1u);
                uint8_t *a_hi = smem_gen + s * STAGE_BYTES, *a_lo = a_hi + A_TILE_BYTES;
                // range guard: running maximum, tested once per tile (a flag store inside this loop cost the XF layers
                // 40-60 %, measured).  It is taken before the ReLU with a NaN-propagating max (starting from 0, the same
                // maximum for finite values), so a NaN in the raw input raises the flag too.  128B swizzle: 16-byte chunk j of row r lives at chunk (j ^ (r & 7)).
                if constexpr (ONE) {  // hi = fp16_rn(relu(y)): round to nearest -- truncation is only valid with a lo plane
#pragma unroll
                    for (int i = 0; i < XR; ++i) {
                        const int row = rg + RG * i;
                        if (128 % RG != 0 && i == XR - 1 && row >= 128) break;
                        const float y4[4] = {fmaxf(v[i].x, 0.f), fmaxf(v[i].y, 0.f), fmaxf(v[i].z, 0.f), fmaxf(v[i].w, 0.f)};
                        rmax = fmax_nan(fmax_nan(rmax, fmax_nan(v[i].x, v[i].y)), fmax_nan(v[i].z, v[i].w));
                        const int off = row * 128 + ((((l16 >> 1) ^ (row & 7))) << 4) + (l16 & 1) * 8;
                        *reinterpret_cast<uint2 *>(a_hi + off) = hi4_f32_nonneg(y4);
                    }
                } else if (G.xf_trunc) {  // truncating split (conv_epilogue.cuh): 4.5 instead of 7.25 instructions per element
#pragma unroll
                    for (int i = 0; i < XR; ++i) {
                        const int row = rg + RG * i;
                        if (128 % RG != 0 && i == XR - 1 && row >= 128) break;
                        const float y4[4] = {v[i].x, v[i].y, v[i].z, v[i].w};
                        uint2 oh, ol;
                        rmax = fmax_nan(fmax_nan(rmax, fmax_nan(y4[0], y4[1])), fmax_nan(y4[2], y4[3]));
                        split4_relu_trunc(y4, oh, ol);
                        const int off = row * 128 + ((((l16 >> 1) ^ (row & 7))) << 4) + (l16 & 1) * 8;
                        *reinterpret_cast<uint2 *>(a_hi + off) = oh;
                        *reinterpret_cast<uint2 *>(a_lo + off) = ol;
                    }
                } else {
#pragma unroll
                    for (int i = 0; i < XR; ++i) {
                        const int row = rg + RG * i;
                        if (128 % RG != 0 && i == XR - 1 && row >= 128) break;
                        float y4[4] = {fmaxf(v[i].x, 0.f), fmaxf(v[i].y, 0.f), fmaxf(v[i].z, 0.f), fmaxf(v[i].w, 0.f)};
                        uint2 oh, ol;
                        rmax = fmax_nan(fmax_nan(rmax, fmax_nan(v[i].x, v[i].y)), fmax_nan(v[i].z, v[i].w));
                        split4_f32<true>(y4, oh, ol);
                        const int off = row * 128 + ((((l16 >> 1) ^ (row & 7))) << 4) + (l16 & 1) * 8;
                        *reinterpret_cast<uint2 *>(a_hi + off) = oh;
                        *reinterpret_cast<uint2 *>(a_lo + off) = ol;
                    }
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes -> visible to wgmma (async proxy)
                __syncwarp();
                if (wl == 0) mbar_arrive(full_bar(s));
            }
            if (!(rmax <= 65504.f) && P.a.flag) *P.a.flag = 1u;
        }
    } else if (warp >= 4) {
        // ===================== wgmma consumers (warpgroups 1, 2) =====================
        const int wg = (warp >> 2) - 1;                     // rows [64 wg, 64 wg + 64) of the tile
        const int ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);  // fragment rows ra and ra + 8
        constexpr int NR = BLOCK_N / 2;
        float acc[NR], sum[NR];
#pragma unroll
        for (int j = 0; j < NR; ++j) acc[j] = 0.f;
        auto release = [&](int s) {
            __syncwarp();
            if (lane == 0) mbar_arrive(empty_bar(s));
        };
        int it_global = 0, ec = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            const int tm = tile / G.tiles_n, tn = tile - tm * G.tiles_n;
#pragma unroll
            for (int j = 0; j < NR; ++j) sum[j] = 0.f;
            // Segments of G.seg K-slices.  Inside one, a slice's wgmma group is issued before the previous slice's group
            // is waited for, so one group is always in flight; only the segment's end waits for all of them and drains
            // the accumulator into the fp32 sum.  Every exit of the inner loop reaches that wait, and the segment's first
            // MMA does not read the accumulator, so ptxas needs to inject no wait of its own; the register fences keep
            // the accumulator untouched around the asynchronous MMAs.
            int pend;   // stage whose wgmma group may still be reading it
            auto slice = [&](auto zero) {
                const int s = it_global % STAGES;
                mbar_wait(full_bar(s), (uint32_t)(it_global / STAGES) & 1u);
                const uint32_t sa = smem_base + s * STAGE_BYTES + wg * 64 * 128;
                const uint32_t sb = smem_base + s * STAGE_BYTES + PLANES * A_TILE_BYTES;
                wg_fence_regs(acc);
                wg_fence();
                if constexpr (ONE) mma_slice1<BLOCK_N, decltype(zero)::value>(acc, sa, sb);
                else mma_slice<BLOCK_N, decltype(zero)::value>(acc, sa, sa + A_TILE_BYTES, sb, sb + BLOCK_N * 128);
                wg_commit();
                wg_fence_regs(acc);
                wg_wait<1>();                                      // the previous slice's group is done with its stage
                if (pend >= 0) release(pend);
                pend = s;
                ++it_global;
            };
            for (int it0 = 0; it0 < kiters; it0 += G.seg) {
                const int it1 = min(it0 + G.seg, kiters);
                pend = -1;
                slice(std::true_type{});
                for (int it = it0 + 1; it < it1; ++it) slice(std::false_type{});
                wg_wait<0>();                                      // segment complete: drain it into the fp32 sum
                wg_fence_regs(acc);
                release(pend);
#pragma unroll
                for (int j = 0; j < NR; ++j) sum[j] += acc[j];
            }
            // ---- epilogue straight from the fragment: rows ra, ra + 8; two consecutive channels per register pair.
            auto flat_pix = [&](int row, int &n_img, int &oy, int &ox) {
                const long long m = (long long)tm * 128 + row;
                if (m >= G.m_total) return false;
                const long long hw = (long long)P.ho * P.wo;
                n_img = (int)(m / hw);
                const int r = (int)(m - (long long)n_img * hw);
                oy = r / P.wo; ox = r - oy * P.wo;
                return true;
            };
            const int per_img = G.tiles_x * G.tiles_y;
            const int n_box = G.flat ? 0 : tm / per_img, r_box = tm - n_box * per_img;
            const int y_box = G.flat ? 0 : (r_box / G.tiles_x) * G.bh, x_box = G.flat ? 0 : (r_box - (r_box / G.tiles_x) * G.tiles_x) * G.bw;
            bool vrow[2];
            PixOff po[2];
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int row = ra + 8 * h;
                int n_img = n_box, oy = 0, ox = 0;
                if (G.flat) vrow[h] = flat_pix(row, n_img, oy, ox);
                else {
                    const int py = row / G.bw, px = row - py * G.bw;
                    oy = y_box + py; ox = x_box + px;
                    vrow[h] = row < G.bw * G.bh && oy < P.ho && ox < P.wo;
                }
                if constexpr (MODE == EPI_UP2) po[h] = pix_offsets_up2(P, vrow[h], n_img, oy, ox);
            }
            if constexpr (MODE == EPI_UP2) {
                // acc is dead until the next tile's first wgmma (scale-d = 0), so it holds the skip pairs the epilogue
                // reads: batches of JB column groups j, 2 rows x 4 output pixels x planes per j, all of a batch's reads
                // issued before its first store (four round trips per tile).  The compiler cannot hoist them itself,
                // since skip may alias out_split.  JB is the largest batch that stays within 168 registers without
                // spilling at BLOCK_N = 128.
                constexpr int JB = NR / 16;
                static_assert((BLOCK_N / 8) % JB == 0, "epilogue batch must divide the column groups");
#pragma unroll
                for (int j0 = 0; j0 < BLOCK_N / 8; j0 += JB) {
                    float2 ws[JB];
#pragma unroll
                    for (int jj = 0; jj < JB; ++jj) {
                        const int c = tn * BLOCK_N + 8 * (j0 + jj) + 2 * (lane & 3);
                        ws[jj] = __ldg(reinterpret_cast<const float2 *>(P.w.oscale + c));
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            if (po[h].skip >= 0)
#pragma unroll
                                for (int d = 0; d < 4; ++d) {
                                    const long long so = po[h].skip + (d >> 1) * P.skip.sH + (d & 1) * P.skip.sW + c;
                                    float *pre = &acc[((jj * 2 + h) * 4 + d) * PLANES];
                                    pre[0] = ld_bits(P.skip.hi + so);
                                    if constexpr (!ONE) pre[1] = ld_bits(P.skip.lo + so);
                                }
                    }
#pragma unroll
                    for (int jj = 0; jj < JB; ++jj) {
                        const int j = j0 + jj;
                        const int c = tn * BLOCK_N + 8 * j + 2 * (lane & 3);
#pragma unroll
                        for (int h = 0; h < 2; ++h)
                            if (po[h].spl >= 0)
                                epi_finish2_up2<ONE>(P, po[h], c, sum[4 * j + 2 * h] * ws[jj].x, sum[4 * j + 2 * h + 1] * ws[jj].y,
                                                     &acc[(jj * 2 + h) * 4 * PLANES]);
                    }
                }
            } else {
                // Chunks of 32 channels through the staging ring: the fragment goes into the slot (added to the residual
                // TMA put there), then one thread hands the slot to TMA as bulk tensor stores, which clip rows past
                // m_total and pixels past ho / wo.  Per element: sum * oscale (+ res) -> raw ; BN, ReLU -> split.
                const bool bn = P.scale && P.out_split.hi;
                const int q4 = lane & 3, ct = threadIdx.x - 128;
#pragma unroll
                for (int q = 0; q < BLOCK_N / 32; ++q, ++ec) {
                    const int e = ec % G.neslots;
                    const uint32_t eph = (uint32_t)(ec / G.neslots) & 1u;
                    const uint32_t s_raw = ring_base + e * G.eslot, s_hi = s_raw + (has_raw ? EPI_RAW_BYTES : 0),
                                   s_lo = s_hi + EPI_HALF_BYTES;
                    uint8_t *g_raw = smem_raw + (s_raw - smem_u32(smem_raw)), *g_hi = smem_raw + (s_hi - smem_u32(smem_raw)),
                            *g_lo = g_hi + EPI_HALF_BYTES;
                    const int cq = tn * BLOCK_N + 32 * q;
                    if (G.epi_tma) {
                        if (MODE == EPI_RES) mbar_wait(efull_bar(e), eph);   // the chunk's residual has landed
                        else mbar_wait(efree_bar(e), eph ^ 1u);             // the slot's previous store has read it
                    } else if (MODE == EPI_RES) {                           // cropped view: copy the residual in
#pragma unroll
                        for (int i = 0; i < 4; ++i) {
                            const int p = ct + 256 * i, row = p >> 3, k = p & 7;
                            int n_img, oy, ox;
                            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
                            if (flat_pix(row, n_img, oy, ox))
                                v = *reinterpret_cast<const float4 *>(P.res.p + n_img * P.res.sN + (long long)oy * P.res.sH +
                                                                      (long long)ox * P.res.sW + cq + 4 * k);
                            *reinterpret_cast<float4 *>(g_raw + row * 128 + ((k ^ (row & 7)) << 4)) = v;
                        }
                        consumers_sync();
                    }
#pragma unroll
                    for (int jj = 0; jj < 4; ++jj) {
                        const int j = 4 * q + jj;
                        const int c = cq + 8 * jj + 2 * q4;
                        const float2 ws = __ldg(reinterpret_cast<const float2 *>(P.w.oscale + c));
                        float2 sc = make_float2(1.f, 1.f), sh = make_float2(0.f, 0.f);
                        if (bn) { sc = __ldg(reinterpret_cast<const float2 *>(P.scale + c)); sh = __ldg(reinterpret_cast<const float2 *>(P.shift + c)); }
#pragma unroll
                        for (int h = 0; h < 2; ++h) {
                            const int row = ra + 8 * h;
                            float v0 = sum[4 * j + 2 * h] * ws.x, v1 = sum[4 * j + 2 * h + 1] * ws.y;
                            const int ro = stg_raw_off(row, jj, q4);
                            if constexpr (MODE == EPI_RES) {
                                const float2 r = *reinterpret_cast<const float2 *>(g_raw + ro);
                                v0 += r.x; v1 += r.y;
                            }
                            if (P.out_raw.p) *reinterpret_cast<float2 *>(g_raw + ro) = make_float2(v0, v1);
                            if (P.out_split.hi) {
                                float t0 = v0, t1 = v1;
                                if (P.scale) { t0 = t0 * sc.x + sh.x; t1 = t1 * sc.y + sh.y; }
                                if (P.relu) { t0 = fmaxf(t0, 0.f); t1 = fmaxf(t1, 0.f); }
                                unsigned int *flag = vrow[h] ? P.out_split.flag : nullptr;   // rows that are stored
                                const int so = stg_half_off(row, jj, q4);
                                if constexpr (ONE) {
                                    *reinterpret_cast<__half2 *>(g_hi + so) = __halves2half2(hi_f32(t0, flag), hi_f32(t1, flag));
                                } else {
                                    __half h0, l0, h1, l1;
                                    split_f32(t0, h0, l0, flag);
                                    split_f32(t1, h1, l1, flag);
                                    *reinterpret_cast<__half2 *>(g_hi + so) = __halves2half2(h0, h1);
                                    *reinterpret_cast<__half2 *>(g_lo + so) = __halves2half2(l0, l1);
                                }
                            }
                        }
                    }
                    if (G.epi_tma) {
                        asm volatile("fence.proxy.async.shared::cta;" ::: "memory");  // generic writes -> visible to TMA
                        consumers_sync();
                        if (threadIdx.x == 128) {
                            if (G.flat) {
                                if (P.out_raw.p) tma_store_2d(&tm_o_raw, s_raw, cq, tm * 128);
                                if (P.out_split.hi) {
                                    tma_store_2d(&tm_o_hi, s_hi, cq, tm * 128);
                                    if constexpr (!ONE) tma_store_2d(&tm_o_lo, s_lo, cq, tm * 128);
                                }
                            } else {
                                if (P.out_raw.p) tma_store_4d(&tm_o_raw, s_raw, cq, x_box, y_box, n_box);
                                if (P.out_split.hi) {
                                    tma_store_4d(&tm_o_hi, s_hi, cq, x_box, y_box, n_box);
                                    if constexpr (!ONE) tma_store_4d(&tm_o_lo, s_lo, cq, x_box, y_box, n_box);
                                }
                            }
                            bulk_commit();
                            // a slot goes back (to the producer's residual load, or to the next chunk written into it)
                            // once its store has read it: the previous chunk's, so that this store stays in flight
                            if (G.neslots > 1) {
                                bulk_wait_read<1>();
                                if (ec > 0) mbar_arrive(efree_bar((ec - 1) % G.neslots));
                            } else {
                                bulk_wait_read<0>();
                                mbar_arrive(efree_bar(e));
                            }
                        }
                    } else {  // cropped view: copy the chunk out, 16 bytes per thread and step
                        consumers_sync();
                        if (P.out_raw.p)
#pragma unroll
                            for (int i = 0; i < 4; ++i) {
                                const int p = ct + 256 * i, row = p >> 3, k = p & 7;
                                int n_img, oy, ox;
                                if (flat_pix(row, n_img, oy, ox))
                                    *reinterpret_cast<float4 *>(P.out_raw.p + n_img * P.out_raw.sN + (long long)oy * P.out_raw.sH +
                                                                (long long)ox * P.out_raw.sW + cq + 4 * k) =
                                        *reinterpret_cast<const float4 *>(g_raw + row * 128 + ((k ^ (row & 7)) << 4));
                            }
                        if (P.out_split.hi)
#pragma unroll
                            for (int i = 0; i < 2; ++i) {
                                const int p = ct + 256 * i, row = p >> 2, k = p & 3;
                                int n_img, oy, ox;
                                if (flat_pix(row, n_img, oy, ox)) {
                                    const long long o = n_img * P.out_split.sN + (long long)oy * P.out_split.sH +
                                                        (long long)ox * P.out_split.sW + cq + 8 * k;
                                    const int so = row * 64 + ((k ^ ((row >> 1) & 3)) << 4);
                                    *reinterpret_cast<uint4 *>(P.out_split.hi + o) = *reinterpret_cast<const uint4 *>(g_hi + so);
                                    if constexpr (!ONE) *reinterpret_cast<uint4 *>(P.out_split.lo + o) = *reinterpret_cast<const uint4 *>(g_lo + so);
                                }
                            }
                        consumers_sync();
                    }
                }
            }
        }
        if (threadIdx.x == 128) bulk_wait<0>();   // every bulk store complete before the CTA exits
    }
}

// ------------------------------------------------------------------------------------------------
// Stem on the tensor core: conv0 7x7x3 -> 64 on the uint8 image (reference net_desc.py:27-35,103,115), BN+ReLU,
// split store.  GEMM view: M = output pixels, N = 64, K = 7 rows x 24 (21 bytes of one image row = 7 taps x 3 channels,
// padded to 24) = 168, padded to 192 = three 64-wide K-slices; the 8th "row" and the 3 pad bytes carry zero weights.
// No operand of this GEMM exists in memory.  Per tile the eight producer warps fetch the 8 input rows it touches, push
// every byte ONCE through a 256-entry table holding (float)v / 255.0f (the reference's own `imgs / 255.0`, an IEEE
// division) already split into fp16 hi | lo, and keep the converted strip in shared memory; an A row's 16-byte chunk is
// then 8 consecutive words of that strip (hi halves to one plane, lo halves to the other), written 128B-swizzled where
// wgmma reads it.  Weights (64 x 192 x {hi, lo} = 48 KB) stay resident in shared memory.
// A tile = 128 consecutive output pixels of one image in raster order (at most two output rows, wo >= 128).
// ONE (precision "high"): the table's hi half and w_hi only, one wgmma per K=16 step, hi-only store; the lo slots of the
// shared-memory layout stay unused.
// Warps: 0 = weight TMA, 4..11 = wgmma consumers (two warpgroups of 64 rows), 12..19 = A-operand producers.
constexpr int C0T_PROD_WARPS = 8, C0T_STAGES = 3, C0T_K = 192, C0T_ROWS = 8, C0T_STRIDE = 832;
constexpr int C0T_PSTRIDE = 833;  // words per row of the converted strip: odd, so the 7 filter rows fall into different banks
constexpr int C0T_PROD0 = 4 + CONS_WARPS;   // first producer warp
constexpr int C0T_THREADS = (C0T_PROD0 + C0T_PROD_WARPS) * 32;
constexpr int C0T_SMEM = 1024 + C0T_STAGES * 2 * A_TILE_BYTES + 3 * 2 * 64 * 128 + 2 * C0T_ROWS * C0T_PSTRIDE * 4 + 256 * 4 + 256;

template <bool ONE>
__global__ void __launch_bounds__(C0T_THREADS, 1)
k_conv0_tc(const __grid_constant__ CUtensorMap tm_w_hi, const __grid_constant__ CUtensorMap tm_w_lo,
           const uint8_t *__restrict__ img, int B, int H, int W, int pad, const float *__restrict__ oscale,
           const float *__restrict__ scale, const float *__restrict__ shift, const SplitRef out) {
    extern __shared__ __align__(1024) uint8_t smem_raw[];
    const uint32_t smem_base = (smem_u32(smem_raw) + 1023u) & ~1023u;
    uint8_t *smem_gen = smem_raw + (smem_base - smem_u32(smem_raw));
    constexpr uint32_t STAGE = 2 * A_TILE_BYTES;                 // a_hi | a_lo of one 64-wide K-slice
    constexpr uint32_t W_OFF = C0T_STAGES * STAGE;               // 3 x [w_hi 8 KB | w_lo 8 KB]
    constexpr uint32_t STRIP_OFF = W_OFF + 3 * 2 * 64 * 128;     // 2 x [8 rows][833 words] converted strip (hi | lo << 16)
    constexpr uint32_t LUT_OFF = STRIP_OFF + 2 * C0T_ROWS * C0T_PSTRIDE * 4;  // [256] (hi | lo << 16) of v / 255
    constexpr uint32_t BAR_OFF = LUT_OFF + 256 * 4;
    const uint32_t bar_base = smem_base + BAR_OFF;
    auto full_bar = [&](int s) { return bar_base + 8u * s; };
    auto empty_bar = [&](int s) { return bar_base + 8u * (C0T_STAGES + s); };
    const uint32_t wfull_bar = bar_base + 8u * (2 * C0T_STAGES);
    // warp index broadcast from lane 0: provably warp-uniform, so the role branches below do not count as divergent
    // paths around the wgmma (ptxas would otherwise serialise them)
    const int warp = __shfl_sync(0xffffffffu, (int)(threadIdx.x >> 5), 0), lane = threadIdx.x & 31;
    const int ho = out.h, wo = out.w, hw = ho * wo;
    const int tiles_img = (hw + 127) >> 7, total_tiles = B * tiles_img;

    if (threadIdx.x == 0) {
        for (int s = 0; s < C0T_STAGES; ++s) { mbar_init(full_bar(s), C0T_PROD_WARPS); mbar_init(empty_bar(s), CONS_WARPS); }
        mbar_init(wfull_bar, 1);
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    {   // (float)v / 255.0f as fp16 hi | lo
        uint32_t *lut = reinterpret_cast<uint32_t *>(smem_gen + LUT_OFF);
        for (int i = threadIdx.x; i < 256; i += blockDim.x) {
            const float f = (float)i / 255.0f;
            const __half h = __float2half_rn(f), l = __float2half_rn(f - __half2float(h));
            lut[i] = (uint32_t)__half_as_ushort(h) | (ONE ? 0u : (uint32_t)__half_as_ushort(l) << 16);
        }
    }
    __syncthreads();

    if (warp == 0) {
        if (lane == 0) {  // resident weights: three K-slices, hi and lo
            mbar_expect_tx(wfull_bar, (ONE ? 1 : 2) * 3 * 64 * 128);
            for (int s = 0; s < 3; ++s) {
                tma_3d(smem_base + W_OFF + s * 16384, &tm_w_hi, wfull_bar, s * 64, 0, 0);
                if constexpr (!ONE) tma_3d(smem_base + W_OFF + s * 16384 + 8192, &tm_w_lo, wfull_bar, s * 64, 0, 0);
            }
        }
    } else if (warp < 4) {
        // idle warps of the producer warpgroup
    } else if (warp < C0T_PROD0) {
        // ===================== wgmma + epilogue: BN+ReLU -> split store =====================
        const int wg = (warp >> 2) - 1;
        const int ra = wg * 64 + (warp & 3) * 16 + (lane >> 2);
        float acc[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) acc[j] = 0.f;
        mbar_wait(wfull_bar, 0);
        int it = 0;
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
            for (int ks = 0; ks < 3; ++ks, ++it) {
                const int s = it % C0T_STAGES;
                mbar_wait(full_bar(s), (uint32_t)(it / C0T_STAGES) & 1u);
                const uint32_t sa = smem_base + s * STAGE + wg * 64 * 128, sb = smem_base + W_OFF + ks * 16384;
                wg_fence();
                if constexpr (ONE) mma_slice1<64>(acc, sa, sb, ks == 0);
                else mma_slice<64>(acc, sa, sa + A_TILE_BYTES, sb, sb + 8192, ks == 0);
                wg_commit();
                wg_wait<0>();
                wg_fence_regs(acc);
                __syncwarp();
                if (lane == 0) mbar_arrive(empty_bar(s));
            }
            const int n = tile / tiles_img;
#pragma unroll
            for (int h = 0; h < 2; ++h) {
                const int p = (tile - n * tiles_img) * 128 + ra + 8 * h;
                if (p >= hw) continue;
                const int oy = p / wo, ox = p - oy * wo;
                const long long oo = n * out.sN + (long long)oy * out.sH + (long long)ox * out.sW;
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const int c = 8 * j + 2 * (lane & 3);
                    // 2^-e folds into the BN scale exactly
                    const float2 w2 = __ldg(reinterpret_cast<const float2 *>(oscale + c));
                    const float2 s2 = __ldg(reinterpret_cast<const float2 *>(scale + c));
                    const float2 b2 = __ldg(reinterpret_cast<const float2 *>(shift + c));
                    const float t0 = fmaxf(acc[4 * j + 2 * h] * (w2.x * s2.x) + b2.x, 0.f);
                    const float t1 = fmaxf(acc[4 * j + 2 * h + 1] * (w2.y * s2.y) + b2.y, 0.f);
                    store_split2<ONE>(out, oo + c, t0, t1);
                }
            }
        }
    } else {
        // ===================== A-operand producers (warps 12..19) =====================
        const int t = threadIdx.x - C0T_PROD0 * 32;                 // 0..255
        const int j = t & 7;                                        // 16-byte chunk of the A row = group inside the K-slice
        const uint32_t *lut = reinterpret_cast<const uint32_t *>(smem_gen + LUT_OFF);
        const int row_bytes = W * 3;
        // input rows y0 - pad .. y0 - pad + 7 of image n, columns from -pad: zero outside the image.  26 bytes per
        // thread: all loads are issued first (load_strip, early in a tile) and stored late (store_strip), so their
        // global latency hides behind the A tiles built in between.
        constexpr int SB = C0T_ROWS * C0T_STRIDE / (C0T_PROD_WARPS * 32);
        static_assert(SB * C0T_PROD_WARPS * 32 == C0T_ROWS * C0T_STRIDE, "strip bytes must divide evenly");
        uint8_t sreg[SB];
        auto load_strip = [&](int tile) {
            const int n = tile / tiles_img, p0 = (tile - n * tiles_img) * 128;
            const int y0 = p0 / wo;
            const uint8_t *im = img + (size_t)n * H * W * 3;
#pragma unroll
            for (int k = 0; k < SB; ++k) {
                const int i = t + k * C0T_PROD_WARPS * 32;
                const int r = i / C0T_STRIDE, cbyte = i - r * C0T_STRIDE;
                const int iy = y0 - pad + r, ib = cbyte - pad * 3;
                sreg[k] = (iy >= 0 && iy < H && ib >= 0 && ib < row_bytes) ? __ldg(im + (size_t)iy * row_bytes + ib) : (uint8_t)0;
            }
        };
        auto store_strip = [&](int buf) {  // convert once per input byte
            uint32_t *strip = reinterpret_cast<uint32_t *>(smem_gen + STRIP_OFF) + buf * C0T_ROWS * C0T_PSTRIDE;
#pragma unroll
            for (int k = 0; k < SB; ++k) {
                const int i = t + k * C0T_PROD_WARPS * 32;
                const int r = i / C0T_STRIDE, cbyte = i - r * C0T_STRIDE;
                strip[r * C0T_PSTRIDE + cbyte] = lut[sreg[k]];
            }
        };
        int it = 0, tcnt = 0;
        if ((int)blockIdx.x < total_tiles) { load_strip(blockIdx.x); store_strip(0); }
        asm volatile("bar.sync 2, %0;" ::"n"(C0T_PROD_WARPS * 32) : "memory");
        for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x, ++tcnt) {
            const int n = tile / tiles_img, p0 = (tile - n * tiles_img) * 128;
            const int y0 = p0 / wo;
            const uint32_t *strip = reinterpret_cast<const uint32_t *>(smem_gen + STRIP_OFF) + (tcnt & 1) * C0T_ROWS * C0T_PSTRIDE;
            const bool more = tile + (int)gridDim.x < total_tiles;
            if (more) load_strip(tile + gridDim.x);   // next tile's rows: in flight while this tile is built
            for (int ks = 0; ks < 3; ++ks, ++it) {
                const int s = it % C0T_STAGES;
                mbar_wait(empty_bar(s), ((uint32_t)(it / C0T_STAGES) & 1u) ^ 1u);
                uint8_t *a_hi = smem_gen + s * STAGE, *a_lo = a_hi + A_TILE_BYTES;
                const int G = ks * 8 + j, ky = G / 3, g = G - ky * 3;   // K = ky * 24 + g * 8 + i
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int r = (t >> 3) + 32 * q;                      // A row = pixel inside the tile
                    uint4 vh = make_uint4(0u, 0u, 0u, 0u), vl = vh;
                    if (ky < 7) {
                        int p = p0 + r;
                        p = p < hw ? p : hw - 1;                          // rows past the image repeat its last pixel (never stored)
                        const int y = p / wo, x = p - y * wo;
                        const uint32_t *src = strip + (y - y0 + ky) * C0T_PSTRIDE + x * 3 + g * 8;
                        uint32_t e[8];
#pragma unroll
                        for (int i = 0; i < 8; ++i) e[i] = src[i];
                        vh = make_uint4(__byte_perm(e[0], e[1], 0x5410), __byte_perm(e[2], e[3], 0x5410),
                                        __byte_perm(e[4], e[5], 0x5410), __byte_perm(e[6], e[7], 0x5410));
                        if constexpr (!ONE)
                            vl = make_uint4(__byte_perm(e[0], e[1], 0x7632), __byte_perm(e[2], e[3], 0x7632),
                                            __byte_perm(e[4], e[5], 0x7632), __byte_perm(e[6], e[7], 0x7632));
                    }
                    const int off = r * 128 + ((j ^ (r & 7)) << 4);       // 128B swizzle: chunk j of row r at (j ^ (r & 7))
                    *reinterpret_cast<uint4 *>(a_hi + off) = vh;
                    if constexpr (!ONE) *reinterpret_cast<uint4 *>(a_lo + off) = vl;
                }
                asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
                __syncwarp();
                if (lane == 0) mbar_arrive(full_bar(s));
            }
            if (more) store_strip((tcnt + 1) & 1);   // the other buffer: last read one tile ago, before the barrier below
            asm volatile("bar.sync 2, %0;" ::"n"(C0T_PROD_WARPS * 32) : "memory");  // next strip complete; this one free again
        }
    }
}

// ------------------------------------------------------------------------------------------------
// host side
typedef CUresult (*EncodeTiledFn)(CUtensorMap *, CUtensorMapDataType, cuuint32_t, void *, const cuuint64_t *,
                                  const cuuint64_t *, const cuuint32_t *, const cuuint32_t *, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn encode_fn() {
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void *p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    });
    return fn;
}

static bool encode(unsigned char *dst, const void *base, int rank, const cuuint64_t *dims, const cuuint64_t *strides_bytes,
                   const cuuint32_t *box, const cuuint32_t *estr, CUtensorMapDataType dt = CU_TENSOR_MAP_DATA_TYPE_FLOAT16,
                   CUtensorMapSwizzle sw = CU_TENSOR_MAP_SWIZZLE_128B) {
    EncodeTiledFn fn = encode_fn();
    if (!fn) return false;
    alignas(64) CUtensorMap tm;
    CUresult r = fn(&tm, dt, (cuuint32_t)rank, const_cast<void *>(base), dims, strides_bytes, box, estr,
                    CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return false;
    memcpy(dst, &tm, sizeof(tm));
    return true;
}
constexpr CUtensorMapDataType TM_F32 = CU_TENSOR_MAP_DATA_TYPE_FLOAT32;

// One epilogue tensor (element size es, strides in elements) as 32-channel boxes of an M-tile: flat tiles a 2-D
// [pixels, channels] map over the view's rows, box tiles a 4-D (C, bw, bh, 1) box.  fp32 boxes (128 B per pixel) are
// 128B-swizzled, fp16 boxes (64 B per pixel) 64B-swizzled, the layouts stg_raw_off / stg_half_off write.
static bool encode_epi(unsigned char *dst, const void *base, long long sN, int sH, int sW, int es, const ConvParams &P,
                       const TcPlan &plan) {
    const CUtensorMapDataType dt = es == 4 ? TM_F32 : CU_TENSOR_MAP_DATA_TYPE_FLOAT16;
    const CUtensorMapSwizzle sw = es == 4 ? CU_TENSOR_MAP_SWIZZLE_128B : CU_TENSOR_MAP_SWIZZLE_64B;
    cuuint32_t ones[4] = {1, 1, 1, 1};
    if (plan.flat) {
        cuuint64_t dims[2] = {(cuuint64_t)P.w.cout, (cuuint64_t)((long long)P.B * P.ho * P.wo)};
        cuuint64_t str[1] = {(cuuint64_t)sW * es};
        cuuint32_t box[2] = {32, 128};
        return encode(dst, base, 2, dims, str, box, ones, dt, sw);
    }
    cuuint64_t dims[4] = {(cuuint64_t)P.w.cout, (cuuint64_t)P.wo, (cuuint64_t)P.ho, (cuuint64_t)P.B};
    cuuint64_t str[3] = {(cuuint64_t)sW * es, (cuuint64_t)sH * es, (cuuint64_t)sN * es};
    cuuint32_t box[4] = {32, (cuuint32_t)plan.bw, (cuuint32_t)plan.bh, 1};
    return encode(dst, base, 4, dims, str, box, ones, dt, sw);
}

static int g_force_block_n = 0;
static int g_seg_chunks = 4;  // 64-channel slices per accumulation segment (4 -> 48 chained wgmma)
static int g_pf = 4;          // L2 prefetch distance (K-slices) for flat operands; 0 = off
static int g_xf_trunc = 1;
static int g_last_dispatch = 0;
int tc_last_dispatch() { return g_last_dispatch; }
void tc_set_prefetch(int n) { g_pf = n < 0 ? 0 : n; }
void tc_set_xf_trunc(int on) { g_xf_trunc = on; }
void tc_set_block_n(int n) { g_force_block_n = n; }
void tc_set_seg_chunks(int n) { g_seg_chunks = n < 1 ? 1 : n; }

static int num_sms() {
    static int sms = 0;
    if (!sms) {
        int dev = 0;
        cudaGetDevice(&dev);
        cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
    }
    return sms;
}

bool tc_plan(const ConvParams &P, TcPlan &plan) {
    plan.ok = false;
    const ConvWeights &w = P.w;
    // precision "high": weights without a lo plane; every split operand of the layer then has one plane too
    const bool one = w.lo == nullptr;
    plan.single = one ? 1 : 0;
    if (!P.in_scale && (P.a.lo == nullptr) != one) return false;
    if (P.a2.hi && (P.a2.lo == nullptr) != one) return false;
    if (P.out_split.hi && (P.out_split.lo == nullptr) != one) return false;
    if (P.up2 && (P.skip.lo == nullptr) != one) return false;
    if (w.cin_pad % 64 != 0 || w.cout % 32 != 0) return false;
    if (P.stride != 1 && P.stride != 2) return false;
    if (P.pad_t != P.pad_l) return false;
    const bool two = P.a2.hi != nullptr;
    if (two) {
        if (w.taps != 1 || P.stride != 1 || P.pad_t != 0 || P.in_scale || (P.cin1 % 64) || (P.a2.c % 64)) return false;
        if ((reinterpret_cast<uintptr_t>(P.a2.hi) & 15) || (reinterpret_cast<uintptr_t>(P.a2.lo) & 15)) return false;
        if ((P.a2.sW % 8) || (P.a2.sH % 8) || (P.a2.sN % 8)) return false;
    }
    const bool xf = P.in_scale != nullptr;
    if (xf) {
        if (w.taps != 1 || P.stride != 1 || P.pad_t != 0 || P.res.p) return false;
        if ((reinterpret_cast<uintptr_t>(P.a_raw.p) & 15) || (P.a_raw.sW % 4) || (P.a_raw.sH % 4) || (P.a_raw.sN % 4)) return false;
        if ((long long)P.B * P.a_raw.sN >= (1ll << 31)) return false;
    } else {
        if ((reinterpret_cast<uintptr_t>(P.a.hi) & 15) || (reinterpret_cast<uintptr_t>(P.a.lo) & 15)) return false;
        if ((P.a.sW % 8) || (P.a.sH % 8) || (P.a.sN % 8)) return false;
    }
    int bn = w.cout >= 128 ? 128 : (w.cout >= 64 ? 64 : 32);
    if (g_force_block_n && w.cout % g_force_block_n == 0) bn = g_force_block_n;
    if (w.cout % bn) return false;
    plan.block_n = bn;
    const bool dense_rows = xf ? ((long long)P.a_raw.sW * P.a_raw.w == P.a_raw.sH && (long long)P.a_raw.sH * P.a_raw.h == P.a_raw.sN)
                               : ((long long)P.a.sW * P.a.w == P.a.sH && (long long)P.a.sH * P.a.h == P.a.sN);
    const int ah = xf ? P.a_raw.h : P.a.h, aw = xf ? P.a_raw.w : P.a.w;
    plan.flat = (w.taps == 1 && P.stride == 1 && P.pad_t == 0 && dense_rows && P.ho == ah && P.wo == aw) ? 1 : 0;
    if (two) {  // both sources must share the tile -> pixel mapping
        const bool dense2 = (long long)P.a2.sW * P.a2.w == P.a2.sH && (long long)P.a2.sH * P.a2.h == P.a2.sN;
        if (!(P.a2_stride == 1 && dense2 && P.a2.h == P.ho && P.a2.w == P.wo)) plan.flat = 0;
    }
    if (xf && bn != 128 && bn != 64) return false;
    cuuint32_t ones[4] = {1, 1, 1, 1};
    if (plan.flat) {
        cuuint64_t dims[2] = {(cuuint64_t)P.a.c, (cuuint64_t)((long long)P.B * P.a.h * P.a.w)};
        cuuint64_t str[1] = {(cuuint64_t)P.a.sW * 2};
        cuuint32_t box[2] = {64, 128};
        if (!xf) {
            if (!encode(plan.tmap_a_hi, P.a.hi, 2, dims, str, box, ones)) return false;
            if (!one && !encode(plan.tmap_a_lo, P.a.lo, 2, dims, str, box, ones)) return false;
        } else {
            cuuint64_t rdims[2] = {(cuuint64_t)P.a_raw.c, (cuuint64_t)((long long)P.B * P.a_raw.h * P.a_raw.w)};
            cuuint64_t rstr[1] = {(cuuint64_t)P.a_raw.sW * 4};
            if (!encode(plan.tmap_a_hi, P.a_raw.p, 2, rdims, rstr, box, ones, TM_F32, CU_TENSOR_MAP_SWIZZLE_NONE)) return false;
        }
        plan.bw = 128; plan.bh = 1; plan.tiles_x = plan.tiles_y = 0;
        if (two) {
            cuuint64_t d2[2] = {(cuuint64_t)P.a2.c, (cuuint64_t)((long long)P.B * P.a2.h * P.a2.w)};
            cuuint64_t s2[1] = {(cuuint64_t)P.a2.sW * 2};
            if (!encode(plan.tmap_a2_hi, P.a2.hi, 2, d2, s2, box, ones)) return false;
            if (!one && !encode(plan.tmap_a2_lo, P.a2.lo, 2, d2, s2, box, ones)) return false;
        }
    } else {
        // choose the (bw x bh <= 128) pixel rectangle that wastes the fewest accumulator rows
        int best_bw = 0, best_bh = 0;
        double best = -1;
        const int maxb = 256 / P.stride;
        for (int bw = 1; bw <= std::min(128, maxb); ++bw) {
            int bh = std::min(128 / bw, maxb);
            if (bh < 1) continue;
            for (; bh >= 1; --bh) {
                double cover = (double)P.ho * P.wo / ((double)cdiv(P.wo, bw) * cdiv(P.ho, bh) * 128.0);
                if (cover > best + 1e-9) { best = cover; best_bw = bw; best_bh = bh; }
            }
        }
        plan.bw = best_bw; plan.bh = best_bh;
        plan.tiles_x = cdiv(P.wo, plan.bw); plan.tiles_y = cdiv(P.ho, plan.bh);
        cuuint64_t dims[4] = {(cuuint64_t)P.a.c, (cuuint64_t)P.a.w, (cuuint64_t)P.a.h, (cuuint64_t)P.B};
        cuuint64_t str[3] = {(cuuint64_t)P.a.sW * 2, (cuuint64_t)P.a.sH * 2, (cuuint64_t)P.a.sN * 2};
        cuuint32_t box[4] = {64, (cuuint32_t)(plan.bw * P.stride), (cuuint32_t)(plan.bh * P.stride), 1};
        cuuint32_t estr[4] = {1, (cuuint32_t)P.stride, (cuuint32_t)P.stride, 1};
        if (!xf) {
            if (!encode(plan.tmap_a_hi, P.a.hi, 4, dims, str, box, estr)) return false;
            if (!one && !encode(plan.tmap_a_lo, P.a.lo, 4, dims, str, box, estr)) return false;
        } else {
            cuuint64_t rdims[4] = {(cuuint64_t)P.a_raw.c, (cuuint64_t)P.a_raw.w, (cuuint64_t)P.a_raw.h, (cuuint64_t)P.B};
            cuuint64_t rstr[3] = {(cuuint64_t)P.a_raw.sW * 4, (cuuint64_t)P.a_raw.sH * 4, (cuuint64_t)P.a_raw.sN * 4};
            if (!encode(plan.tmap_a_hi, P.a_raw.p, 4, rdims, rstr, box, estr, TM_F32, CU_TENSOR_MAP_SWIZZLE_NONE)) return false;
        }
        if (two) {
            const int s2 = P.a2_stride;
            if (plan.bw * s2 > 256 || plan.bh * s2 > 256) return false;
            cuuint64_t d2[4] = {(cuuint64_t)P.a2.c, (cuuint64_t)P.a2.w, (cuuint64_t)P.a2.h, (cuuint64_t)P.B};
            cuuint64_t st2[3] = {(cuuint64_t)P.a2.sW * 2, (cuuint64_t)P.a2.sH * 2, (cuuint64_t)P.a2.sN * 2};
            cuuint32_t box2[4] = {64, (cuuint32_t)(plan.bw * s2), (cuuint32_t)(plan.bh * s2), 1};
            cuuint32_t es2[4] = {1, (cuuint32_t)s2, (cuuint32_t)s2, 1};
            if (!encode(plan.tmap_a2_hi, P.a2.hi, 4, d2, st2, box2, es2)) return false;
            if (!one && !encode(plan.tmap_a2_lo, P.a2.lo, 4, d2, st2, box2, es2)) return false;
        }
    }
    {
        cuuint64_t dims[3] = {(cuuint64_t)w.cin_pad, (cuuint64_t)w.cout, (cuuint64_t)w.taps};
        cuuint64_t str[2] = {(cuuint64_t)w.cin_pad * 2, (cuuint64_t)w.cin_pad * w.cout * 2};
        cuuint32_t box[3] = {64, (cuuint32_t)bn, 1};
        if (!encode(plan.tmap_w_hi, w.hi, 3, dims, str, box, ones)) return false;
        if (!one && !encode(plan.tmap_w_lo, w.lo, 3, dims, str, box, ones)) return false;
    }
    if (!P.up2) {
        // epilogue tensors: 16-byte aligned bases and strides (TMA, and the staged copy of a cropped flat view)
        auto al16 = [](const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; };
        if (P.res.p && (!al16(P.res.p) || P.res.sW % 4 || P.res.sH % 4 || P.res.sN % 4)) return false;
        if (P.out_raw.p && (!al16(P.out_raw.p) || P.out_raw.sW % 4 || P.out_raw.sH % 4 || P.out_raw.sN % 4)) return false;
        if (P.out_split.hi && (!al16(P.out_split.hi) || (!one && !al16(P.out_split.lo)) || P.out_split.sW % 8 ||
                               P.out_split.sH % 8 || P.out_split.sN % 8)) return false;
        // a flat tile is 128 consecutive pixels: one TMA box only where the view's rows are dense
        auto rows_dense = [&](long long sN, int sH, int sW) { return (long long)sW * P.wo == sH && (long long)sH * P.ho == sN; };
        plan.epi_tma = 1;
        if (plan.flat && ((P.res.p && !rows_dense(P.res.sN, P.res.sH, P.res.sW)) ||
                          (P.out_raw.p && !rows_dense(P.out_raw.sN, P.out_raw.sH, P.out_raw.sW)) ||
                          (P.out_split.hi && !rows_dense(P.out_split.sN, P.out_split.sH, P.out_split.sW))))
            plan.epi_tma = 0;
        if (plan.epi_tma) {
            if (P.res.p && !encode_epi(plan.tmap_res, P.res.p, P.res.sN, P.res.sH, P.res.sW, 4, P, plan)) return false;
            if (P.out_raw.p && !encode_epi(plan.tmap_out_raw, P.out_raw.p, P.out_raw.sN, P.out_raw.sH, P.out_raw.sW, 4, P, plan))
                return false;
            if (P.out_split.hi) {
                const SplitRef &o = P.out_split;
                if (!encode_epi(plan.tmap_out_hi, o.hi, o.sN, o.sH, o.sW, 2, P, plan)) return false;
                if (!one && !encode_epi(plan.tmap_out_lo, o.lo, o.sN, o.sH, o.sW, 2, P, plan)) return false;
            }
        }
    }
    plan.ok = true;
    return true;
}

template <int BLOCK_N, int MODE, bool XF, bool ONE>
static void launch_tm(const ConvParams &P, const TcPlan &plan, TcGeom G, cudaStream_t s) {
    constexpr int STAGES = tc_stages<BLOCK_N, MODE, XF, ONE>();
    constexpr int RING = tc_ring<BLOCK_N, MODE, XF, ONE>();
    constexpr int smem = tc_smem<BLOCK_N, XF, ONE>(STAGES, RING);
    static_assert(smem <= SMEM_LIMIT, "shared memory budget exceeded");
    static bool attr = false;
    if (!attr) {
        HVN_CUDA(cudaFuncSetAttribute(k_conv_tc<BLOCK_N, STAGES, MODE, XF, ONE>, cudaFuncAttributeMaxDynamicSharedMemorySize, smem));
        attr = true;
    }
    G.eslot = (MODE == EPI_RES || P.out_raw.p ? EPI_RAW_BYTES : 0) + (P.out_split.hi ? (ONE ? 1 : 2) * EPI_HALF_BYTES : 0);
    G.neslots = RING && G.eslot ? std::min(RING / G.eslot, EPI_MAX_SLOTS) : 1;
    if (RING && G.eslot) HVN_CHECK(G.neslots >= 1, -1, "conv_tc: epilogue staging ring too small");
    const int grid = std::min(G.tiles_m * G.tiles_n, num_sms());
    CUtensorMap t[10];
    const unsigned char *src[10] = {plan.tmap_a_hi, plan.tmap_a_lo, plan.tmap_w_hi, plan.tmap_w_lo, plan.tmap_a2_hi,
                                    plan.tmap_a2_lo, plan.tmap_res, plan.tmap_out_raw, plan.tmap_out_hi, plan.tmap_out_lo};
    for (int i = 0; i < 10; ++i) memcpy(&t[i], src[i], 128);
    k_conv_tc<BLOCK_N, STAGES, MODE, XF, ONE><<<grid, TC_THREADS, smem, s>>>(t[0], t[1], t[2], t[3], t[4], t[5], t[6], t[7], t[8],
                                                                            t[9], P, G);
    g_last_dispatch = BLOCK_N | MODE << 8 | (XF ? 1 : 0) << 12 | (ONE ? 1 : 0) << 13;
}

template <int BLOCK_N, bool ONE>
static void launch_t(const ConvParams &P, const TcPlan &plan, const TcGeom &G, cudaStream_t s) {
    if (P.in_scale) {  // transformed input: only the shapes the plan produces (1x1, plain or upsample epilogue)
        if constexpr (BLOCK_N == 128 || BLOCK_N == 64) {
            if (P.up2) launch_tm<BLOCK_N, EPI_UP2, true, ONE>(P, plan, G, s);
            else launch_tm<BLOCK_N, EPI_PLAIN, true, ONE>(P, plan, G, s);
            return;
        }
        throw Error(-1, "conv_tc: transformed input with unsupported tile shape");
    }
    if (P.up2) launch_tm<BLOCK_N, EPI_UP2, false, ONE>(P, plan, G, s);
    else if (P.res.p) launch_tm<BLOCK_N, EPI_RES, false, ONE>(P, plan, G, s);
    else launch_tm<BLOCK_N, EPI_PLAIN, false, ONE>(P, plan, G, s);
}

// Stem launcher.  `w` = conv0 weights as [1 tap][64 cout][192 k] split fp16 (k = ky * 24 + kx * 3 + ch, zeros elsewhere).
bool conv0_tc_supported(int H, int W, int pad, const SplitRef &out) {
    return out.w >= 128 && out.c == 64 && (W + 2 * pad) * 3 + 3 <= C0T_STRIDE && out.h == H + 2 * pad - 6 && out.w == W + 2 * pad - 6 &&
           !(reinterpret_cast<uintptr_t>(out.hi) & 15) && !(reinterpret_cast<uintptr_t>(out.lo) & 15) && out.sW % 8 == 0 &&
           out.sH % 8 == 0 && out.sN % 8 == 0;
}

template <bool ONE> static void set_conv0_smem() {
    static bool attr = false;
    if (!attr) {
        HVN_CUDA(cudaFuncSetAttribute(k_conv0_tc<ONE>, cudaFuncAttributeMaxDynamicSharedMemorySize, C0T_SMEM));
        attr = true;
    }
}

void launch_conv0_tc(const uint8_t *img, int B, int H, int W, int pad, const ConvWeights &w, const float *scale,
                     const float *shift, const SplitRef &out, cudaStream_t s) {
    HVN_CHECK(w.taps == 1 && w.cout == 64 && w.cin_pad == C0T_K, -1, "conv0_tc: unexpected weight layout");
    const bool one = w.lo == nullptr;
    HVN_CHECK((out.lo == nullptr) == one, -1, "conv0_tc: weights and output differ in their number of fp16 planes");
    static_assert(C0T_SMEM <= SMEM_LIMIT, "conv0_tc: shared memory budget exceeded");
    alignas(64) CUtensorMap w_hi, w_lo;
    cuuint32_t ones[3] = {1, 1, 1};
    cuuint64_t dims[3] = {(cuuint64_t)w.cin_pad, (cuuint64_t)w.cout, 1};
    cuuint64_t str[2] = {(cuuint64_t)w.cin_pad * 2, (cuuint64_t)w.cin_pad * w.cout * 2};
    cuuint32_t box[3] = {64, 64, 1};
    memset(&w_lo, 0, sizeof(w_lo));
    HVN_CHECK(encode((unsigned char *)&w_hi, w.hi, 3, dims, str, box, ones) && (one || encode((unsigned char *)&w_lo, w.lo, 3, dims, str, box, ones)),
              -2, "conv0_tc: tensor map encode failed");
    const int tiles = B * cdiv((long long)out.h * out.w, 128);
    const int grid = std::min(tiles, num_sms());
    if (one) {
        set_conv0_smem<true>();
        k_conv0_tc<true><<<grid, C0T_THREADS, C0T_SMEM, s>>>(w_hi, w_lo, img, B, H, W, pad, w.oscale, scale, shift, out);
    } else {
        set_conv0_smem<false>();
        k_conv0_tc<false><<<grid, C0T_THREADS, C0T_SMEM, s>>>(w_hi, w_lo, img, B, H, W, pad, w.oscale, scale, shift, out);
    }
}

void tc_launch(const ConvParams &P, const TcPlan &plan, cudaStream_t s) {
    TcGeom G;
    G.flat = plan.flat; G.bw = plan.bw; G.bh = plan.bh; G.tiles_x = plan.tiles_x; G.tiles_y = plan.tiles_y;
    G.kchunks = P.w.cin_pad / 64;
    G.seg = g_seg_chunks;
    G.k1 = P.a2.hi ? P.cin1 / 64 : 0;
    G.m_total = (long long)P.B * P.ho * P.wo;
    G.tiles_m = plan.flat ? cdiv(G.m_total, 128) : P.B * plan.tiles_x * plan.tiles_y;
    G.tiles_n = P.w.cout / plan.block_n;
    G.xf_trunc = g_xf_trunc;
    G.pf = g_pf;
    G.epi_tma = plan.epi_tma;
    if (plan.single) {
        switch (plan.block_n) {
        case 128: launch_t<128, true>(P, plan, G, s); break;
        case 64: launch_t<64, true>(P, plan, G, s); break;
        default: launch_t<32, true>(P, plan, G, s); break;
        }
    } else {
        switch (plan.block_n) {
        case 128: launch_t<128, false>(P, plan, G, s); break;
        case 64: launch_t<64, false>(P, plan, G, s); break;
        default: launch_t<32, false>(P, plan, G, s); break;
        }
    }
}

}  // namespace hvn
