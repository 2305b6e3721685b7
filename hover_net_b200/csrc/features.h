// Host-side interface of the per-instance measurements (features.cu): shape, intensity and NP statistics of every
// instance-table row, HVN_FEAT_LEN float64 per row (include/hvn.h HVN_FEAT_*).
#pragma once
#include "common.cuh"

namespace hvn {

// Rows whose contour has at most this many points sort and hull them in shared memory; longer rows use a global
// scratch of FEAT_SCRATCH_BYTES_PER_POINT per contour point of the call (taken only when such a row exists).
constexpr int FEAT_SMEM_POINTS = 512;
constexpr size_t FEAT_SCRATCH_BYTES_PER_POINT = 24;

// Map m of a packed group: H x W pixels starting at pixel px_off.
struct FeatMap {
    long long px_off;
    int H, W;
};

// What the check pass found: err != 0 on an inconsistent argument (bit 1 row offsets, 2 a table row's bbox outside
// its map or empty, 4 point offsets, 8 a point outside its row's bbox); the longest row's point count; and the points
// of the call (pt_offs[n_rows] - pt_offs[0]).
struct FeatStatus {
    long long err, max_pts, total_pts;
};

// Validates the packed layout on the device and writes *status (device).  Returns the number of kernels launched.
int features_check(cudaStream_t stream, const FeatMap *maps, int n_maps, const int *row_offs, long long n_rows,
                   const long long *table, const int *pts, const int *pt_offs, FeatStatus *status);

// One warp per row: the pixel pass over the bbox, the contour pass and the finishing arithmetic, into feats
// [n_rows,HVN_FEAT_LEN].  img (u8 [H,W,3] per map) and pred (f32 [H,W,C] per map, NP at channel C - 3) may be null:
// their columns are NaN then.  scratch: FEAT_SCRATCH_BYTES_PER_POINT * total_pts bytes (total_pts the status' count)
// when some row has more than FEAT_SMEM_POINTS points, else unused.  Only input that passed features_check may be
// given.  Returns the number of kernels launched.
int features_rows(cudaStream_t stream, const FeatMap *maps, int n_maps, const int *inst, const unsigned char *img,
                  const float *pred, int C, const long long *table, const int *row_offs, long long n_rows,
                  const int *pts, const int *pt_offs, void *scratch, double *feats, long long total_pts);

}  // namespace hvn
