// Host-side interface of the instance-statistics pair table (stats.cu).
#pragma once
#include "common.cuh"

namespace hvn {

// Device workspace of one inst_pairs call, laid out in an Arena by inst_pairs_count and read again by
// inst_pairs_emit (the arena must not be reset in between).
struct PairWork {
    int n = 0, H = 0, W = 0, tiles = 0;
    long long stride = 0;                    // hash slots reserved per map: next_pow2(2*H*W)
    unsigned long long *lkey = nullptr;      // per-tile pair lists [n*tiles*1024]
    unsigned *lcnt = nullptr;
    int *tile_n = nullptr;                   // [n*tiles]
    unsigned long long *hkey = nullptr;      // per-map hash tables [n*stride]
    unsigned *hcnt = nullptr;
    long long *hcap = nullptr;               // [n] slots in use per map
    int *npairs = nullptr, *cursor = nullptr, *err = nullptr;
    long long *offs = nullptr;
};

size_t inst_pairs_workspace_bytes(int n, int H, int W);

// true/pred int32 [n,H,W] (device; pred may be null = all zero) -> offs [n+1] int64 (device) and the per-map hash
// tables in `w`.  *w.err becomes non-zero on a negative id.  Returns the number of kernels launched.
int inst_pairs_count(Arena &arena, cudaStream_t stream, const int *tru, const int *pred, int n, int H, int W,
                     long long *offs, PairWork &w);
// Writes the rows (t, p, count) int64 of every map at [offs[m], offs[m+1]) of `pairs` when offs[n] <= cap and no
// negative id was seen; writes nothing otherwise.  Returns the number of kernels launched.
int inst_pairs_emit(cudaStream_t stream, const PairWork &w, long long *pairs, long long cap);

}  // namespace hvn
