// Contingency table of two instance maps: for every map, every distinct (true id, pred id) pair that occurs at a
// pixel where either id is non-zero, with its pixel count.  It is the only per-pixel quantity the reference's
// instance metrics need (metrics/stats_utils.py: get_fast_aji, get_fast_aji_plus, get_fast_pq, the dice scores,
// remap_label): intersections are the entries, areas the row and column sums.  The reference instead builds a
// full-map mask per instance and per overlapping pair, O(instances * pixels).
//
// One streaming pass reads both maps once (8 B per pixel).  Instance maps are spatially coherent, so the pass
// aggregates before it touches global memory: each CTA owns an 8 x 128 pixel tile, every warp reads one row of
// it 32 pixels at a time, lanes holding the same key are merged with __match_any_sync, and the group leader adds
// the group's count to a shared-memory open-addressed table (2048 slots, at most 1024 keys, so the load is <= 1/2).
// The tile's distinct pairs go to a per-tile list in global memory.  The sum of the list lengths of a map bounds
// its number of distinct pairs, so the per-map global hash table uses next_pow2(2 * bound) slots (load <= 1/2):
// only that prefix is cleared and scanned, and the work after the pass scales with pairs, not pixels.  Then the
// lists are merged into the hash table, the pairs are counted, offs is an exclusive scan of the counts, and the
// occupied slots are compacted into the output in no particular order (the host sorts O(pairs) rows).
//
// Integers only: counts are exact and independent of the order of the atomics.  Keys pack (t << 32) | p with
// t, p >= 0, so the all-ones word is free to mark an empty slot.
#include <algorithm>

#include "stats.h"

namespace hvn {
namespace {

constexpr int TH = 8, TW = 128, TPX = TH * TW;   // tile: one row per warp, 4 x 32 pixels per row
constexpr int SLOTS = 2 * TPX;                   // shared table of a tile
constexpr int THREADS = TH * 32;
constexpr unsigned long long EMPTY = ~0ull;

__device__ __forceinline__ unsigned long long mix(unsigned long long k) {  // splitmix64 finaliser
    k ^= k >> 30;
    k *= 0xbf58476d1ce4e5b9ull;
    k ^= k >> 27;
    k *= 0x94d049bb133111ebull;
    k ^= k >> 31;
    return k;
}

// Open addressing with linear probing; the caller guarantees a free slot (load <= 1/2).  Returns true when this
// call claimed the slot for a new key.
__device__ __forceinline__ bool table_add(unsigned long long *keys, unsigned *cnt, unsigned long long mask,
                                          unsigned long long key, unsigned c) {
    unsigned long long s = mix(key) & mask;
    for (;;) {
        const unsigned long long prev = atomicCAS(&keys[s], EMPTY, key);
        if (prev == EMPTY || prev == key) {
            atomicAdd(&cnt[s], c);
            return prev == EMPTY;
        }
        s = (s + 1) & mask;
    }
}

__global__ void __launch_bounds__(THREADS) k_pairs_tile(const int *__restrict__ tru, const int *__restrict__ pred,
                                                        int H, int W, int tiles_x, int tiles,
                                                        unsigned long long *__restrict__ lkey,
                                                        unsigned *__restrict__ lcnt, int *__restrict__ tile_n,
                                                        int *__restrict__ err) {
    __shared__ unsigned long long skey[SLOTS];
    __shared__ unsigned scnt[SLOTS];
    __shared__ int s_n;
    const int tile = blockIdx.x, m = blockIdx.y;
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    for (int i = threadIdx.x; i < SLOTS; i += THREADS) {
        skey[i] = EMPTY;
        scnt[i] = 0;
    }
    if (threadIdx.x == 0) s_n = 0;
    const int ty = tile / tiles_x, tx = tile - ty * tiles_x;
    const int y = ty * TH + warp;
    const int *tr = tru + ((size_t)m * H + y) * W;
    const int *pr = pred ? pred + ((size_t)m * H + y) * W : nullptr;
    int tv[TW / 32], pv[TW / 32];
#pragma unroll
    for (int j = 0; j < TW / 32; ++j) {  // all loads first: 8 in flight per thread
        const int x = tx * TW + j * 32 + lane;
        const bool in = y < H && x < W;
        tv[j] = in ? __ldg(tr + x) : 0;
        pv[j] = (in && pr) ? __ldg(pr + x) : 0;
    }
    __syncthreads();
    bool neg = false;
#pragma unroll
    for (int j = 0; j < TW / 32; ++j) {
        const int t = tv[j], p = pv[j];
        neg |= (t | p) < 0;
        const unsigned long long key =
            (t | p) > 0 ? ((unsigned long long)(unsigned)t << 32) | (unsigned)p : EMPTY;  // skips (0,0), negatives
        const unsigned grp = __match_any_sync(0xffffffffu, key);
        if (key != EMPTY && lane == __ffs(grp) - 1) table_add(skey, scnt, SLOTS - 1, key, __popc(grp));
    }
    if (__any_sync(0xffffffffu, neg) && lane == 0) atomicOr(err, 1);
    __syncthreads();
    const size_t lbase = ((size_t)m * tiles + tile) * TPX;
    for (int i = threadIdx.x; i < SLOTS; i += THREADS) {
        const unsigned long long k = skey[i];
        if (k != EMPTY) {
            const int o = atomicAdd(&s_n, 1);
            lkey[lbase + o] = k;
            lcnt[lbase + o] = scnt[i];
        }
    }
    __syncthreads();
    if (threadIdx.x == 0) tile_n[(size_t)m * tiles + tile] = s_n;
}

// One block per map: bound = sum of the tile list lengths -> slots in use = next_pow2(2 * bound).
__global__ void __launch_bounds__(1024) k_pairs_bound(const int *__restrict__ tile_n, int tiles,
                                                      long long *__restrict__ hcap, int *__restrict__ npairs,
                                                      int *__restrict__ cursor) {
    __shared__ long long part[32];
    const int m = blockIdx.x;
    long long s = 0;
    for (int i = threadIdx.x; i < tiles; i += blockDim.x) s += tile_n[(size_t)m * tiles + i];
    for (int d = 16; d; d >>= 1) s += __shfl_xor_sync(0xffffffffu, s, d);
    if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = s;
    __syncthreads();
    if (threadIdx.x == 0) {
        long long b = 0;
        for (int i = 0; i < (int)(blockDim.x >> 5); ++i) b += part[i];
        long long cap = 0;
        if (b > 0) {
            cap = 1;
            while (cap < 2 * b) cap <<= 1;
        }
        hcap[m] = cap;
        npairs[m] = 0;
        cursor[m] = 0;
    }
}

__global__ void k_pairs_clear(unsigned long long *__restrict__ hkey, unsigned *__restrict__ hcnt, long long stride,
                              const long long *__restrict__ hcap) {
    const int m = blockIdx.y;
    const long long cap = hcap[m];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < cap; i += (long long)gridDim.x * blockDim.x) {
        hkey[m * stride + i] = EMPTY;
        hcnt[m * stride + i] = 0;
    }
}

// One block per tile list: merge into the map's hash table and count the new keys.
__global__ void __launch_bounds__(128) k_pairs_merge(const unsigned long long *__restrict__ lkey,
                                                     const unsigned *__restrict__ lcnt, const int *__restrict__ tile_n,
                                                     int tiles, unsigned long long *__restrict__ hkey,
                                                     unsigned *__restrict__ hcnt, long long stride,
                                                     const long long *__restrict__ hcap, int *__restrict__ npairs) {
    const int tile = blockIdx.x, m = blockIdx.y;
    const size_t t = (size_t)m * tiles + tile;
    const int n = tile_n[t];
    if (n == 0) return;
    const unsigned long long mask = (unsigned long long)hcap[m] - 1;
    int fresh = 0;
    for (int i = threadIdx.x; i < n; i += blockDim.x)
        fresh += table_add(hkey + m * stride, hcnt + m * stride, mask, lkey[t * TPX + i], lcnt[t * TPX + i]);
    for (int d = 16; d; d >>= 1) fresh += __shfl_xor_sync(0xffffffffu, fresh, d);
    if ((threadIdx.x & 31) == 0 && fresh) atomicAdd(&npairs[m], fresh);
}

// offs = exclusive scan of the per-map pair counts (n is small: maps of one call).
__global__ void k_pairs_offs(const int *__restrict__ npairs, int n, long long *__restrict__ offs) {
    long long s = 0;
    for (int m = 0; m < n; ++m) {
        offs[m] = s;
        s += npairs[m];
    }
    offs[n] = s;
}

__global__ void k_pairs_emit(const unsigned long long *__restrict__ hkey, const unsigned *__restrict__ hcnt,
                             long long stride, const long long *__restrict__ hcap, const long long *__restrict__ offs,
                             int n, const int *__restrict__ err, int *__restrict__ cursor, long long *__restrict__ out,
                             long long cap) {
    if (*err || offs[n] > cap) return;
    const int m = blockIdx.y;
    const long long hc = hcap[m], base = offs[m];
    for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < hc; i += (long long)gridDim.x * blockDim.x) {
        const unsigned long long k = hkey[m * stride + i];
        if (k == EMPTY) continue;
        const long long r = base + atomicAdd(&cursor[m], 1);
        out[3 * r] = (long long)(k >> 32);
        out[3 * r + 1] = (long long)(k & 0xffffffffull);
        out[3 * r + 2] = (long long)hcnt[m * stride + i];
    }
}

long long next_pow2(long long v) {
    long long p = 1;
    while (p < v) p <<= 1;
    return p;
}

template <typename A> void layout(A &a, int n, int H, int W, PairWork &w) {
    w.n = n;
    w.H = H;
    w.W = W;
    w.tiles = cdiv(H, TH) * cdiv(W, TW);
    w.stride = next_pow2(2ll * H * W);
    const size_t lists = (size_t)n * w.tiles * TPX, slots = (size_t)n * w.stride;
    w.lkey = a.template take<unsigned long long>(lists);
    w.lcnt = a.template take<unsigned>(lists);
    w.tile_n = a.template take<int>((size_t)n * w.tiles);
    w.hkey = a.template take<unsigned long long>(slots);
    w.hcnt = a.template take<unsigned>(slots);
    w.hcap = a.template take<long long>(n);
    w.npairs = a.template take<int>(n);
    w.cursor = a.template take<int>(n);
    w.err = a.template take<int>(1);
}

// Blocks per map for the loops over hash slots: enough for a full table, few when the maps are small.
int slot_blocks(long long stride) { return (int)std::min<long long>(128, std::max<long long>(1, stride / (256 * 32))); }

}  // namespace

// Per pixel: 12 B of tile lists (tiles padded to 8 x 128) + 12 B per hash slot, next_pow2(2 * H * W) slots per map
// (24..48 B); e.g. 14 maps of 1000 x 1000 -> 0.52 GB, one 4096 x 4096 map -> 0.6 GB.
size_t inst_pairs_workspace_bytes(int n, int H, int W) {
    ArenaSizer s;
    PairWork w;
    layout(s, n, H, W, w);
    return s.top + 1024;
}

int inst_pairs_count(Arena &arena, cudaStream_t stream, const int *tru, const int *pred, int n, int H, int W,
                     long long *offs, PairWork &w) {
    arena.reset();
    arena.reserve(inst_pairs_workspace_bytes(n, H, W));
    layout(arena, n, H, W, w);
    w.offs = offs;
    HVN_CUDA(cudaMemsetAsync(w.err, 0, sizeof(int), stream));
    const int tiles_x = cdiv(W, TW);
    k_pairs_tile<<<dim3(w.tiles, n), THREADS, 0, stream>>>(tru, pred, H, W, tiles_x, w.tiles, w.lkey, w.lcnt, w.tile_n,
                                                           w.err);
    k_pairs_bound<<<n, 1024, 0, stream>>>(w.tile_n, w.tiles, w.hcap, w.npairs, w.cursor);
    k_pairs_clear<<<dim3(slot_blocks(w.stride), n), 256, 0, stream>>>(w.hkey, w.hcnt, w.stride, w.hcap);
    k_pairs_merge<<<dim3(w.tiles, n), 128, 0, stream>>>(w.lkey, w.lcnt, w.tile_n, w.tiles, w.hkey, w.hcnt, w.stride,
                                                        w.hcap, w.npairs);
    k_pairs_offs<<<1, 1, 0, stream>>>(w.npairs, n, offs);
    HVN_CUDA(cudaGetLastError());
    return 5;
}

int inst_pairs_emit(cudaStream_t stream, const PairWork &w, long long *pairs, long long cap) {
    k_pairs_emit<<<dim3(slot_blocks(w.stride), w.n), 256, 0, stream>>>(w.hkey, w.hcnt, w.stride, w.hcap, w.offs, w.n,
                                                                       w.err, w.cursor, pairs, cap);
    HVN_CUDA(cudaGetLastError());
    return 1;
}

}  // namespace hvn
