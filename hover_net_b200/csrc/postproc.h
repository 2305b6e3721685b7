// Host-side interface of the device post-processing path (postproc.cu).
#pragma once
#include <string>

#include "common.cuh"

namespace hvn {

struct PostprocBuffers {
    int max_blobs = 0, max_ids = 0;
    void *stats = nullptr;
    unsigned char *fg = nullptr, *mk0 = nullptr, *flag = nullptr, *filled = nullptr, *eroded = nullptr, *opened = nullptr;
    int *L1 = nullptr, *size1 = nullptr, *blob_of_root = nullptr, *blob_root = nullptr;
    void *bbox = nullptr, *lab_range = nullptr;
    double *sobh = nullptr, *sobv = nullptr, *din = nullptr, *dist = nullptr;
    int *L2 = nullptr, *size3 = nullptr, *id3 = nullptr, *rowcnt = nullptr;
    void *heap = nullptr, *acc = nullptr;
    int *tcnt = nullptr;
};

void postproc_set_flood_impl(int v);  // test hook: 0 auto, 1 no calendar queue, 2 global-memory heap only
size_t postproc_workspace_bytes(int n, int H, int W, int nr_types);
// Instance ids a map can hold (ids 1 .. postproc_max_ids - 1): an upper bound on the table rows of one H x W map.
int postproc_max_ids(int H, int W);

// Watershed flood kernels.  FLOOD_AUTO picks by map size (calendar queue, shared-memory heap with or without the fp32
// key table, global-memory heap; "flood_impl" narrows the choice); the others force one kernel.
enum FloodKernel { FLOOD_AUTO = 0, FLOOD_CAL = 1, FLOOD_TILE_KK = 2, FLOOD_TILE = 3, FLOOD_GLOBAL = 4 };
const char *postproc_flood_name(int k);
// Launches the flood over the laid-out buffers `b` (markers already in inst, single-label blobs filled).  Returns the
// FloodKernel launched; a forced kernel that does not fit the map throws Error(-1) without launching.
int postproc_flood(cudaStream_t stream, const PostprocBuffers &b, int n, int H, int W, int *inst, int choice);

// Test hooks.  postproc_buffers: the stage buffers of the last postproc_run on `arena` for the same (n, H, W, nr_types)
// (the layout is deterministic; nothing is launched).  postproc_flood_only: the watershed stage alone on caller-owned
// device maps dist f64 / mask u8 / markers i32 [n,H,W] -> inst i32: the mask's components, the < 10 px filter, boxes,
// marker ranges, single-label fill and the flood kernel `choice`, the same kernels postproc_run launches.  Marker
// labels must lie in [0, postproc_max_ids(H, W)).  Returns the FloodKernel launched.
void postproc_buffers(Arena &arena, int n, int H, int W, int nr_types, PostprocBuffers &b);
int postproc_flood_only(Arena &arena, cudaStream_t stream, const double *dist, const unsigned char *mask,
                        const int *markers, int n, int H, int W, int *inst, int choice);

// pred [n,H,W,C] f32 (device) -> inst [n,H,W] i32, table [n,max_rows,10] i64, n_rows [n] i32 (device).
// Returns the number of kernels launched on `stream`.
int postproc_run(Arena &arena, cudaStream_t stream, const float *pred, int n, int H, int W, int C, int nr_types,
                 int *inst, long long *table, int max_rows, int *n_rows, std::string *prof = nullptr);

// Contours of every table row (contour.cu): offs [n*max_rows + 1] i32 exclusive prefix of the per-row point
// counts, pts [cap][2] i32 (x, y) in map coordinates.  All pointers are device pointers.  Returns the number
// of kernels launched.
int contours_run(cudaStream_t stream, const int *inst, const long long *table, const int *n_rows, int n_maps, int H,
                 int W, int max_rows, int *pts, long long cap, int *offs);
// The three phases of contours_run, for the packed layout of a tile group: per-row point counts cnt [n*max_rows]
// (0 past n_rows); exclusive scan of offs [0, total) in place, offs[total] = sum; and the write pass of one size class
// at its packed positions (row r of class map m is packed row row_offs[img_of[m].img] + r, its points
// pts[pt_offs[row] : pt_offs[row+1]]; nothing is written when row_offs[n_out] > rows_cap or past cap).
struct TileImage;
int contours_count(cudaStream_t stream, const int *inst, const long long *table, const int *n_rows, int n_maps, int H,
                   int W, int max_rows, int *cnt);
int contours_scan(cudaStream_t stream, int *offs, int total);
int contours_write_packed(cudaStream_t stream, const int *inst, const long long *table, const int *n_rows, int n_maps,
                          int H, int W, int max_rows, const TileImage *img_of, const int *row_offs, int n_out,
                          long long rows_cap, const int *pt_offs, int *pts, long long cap);

}  // namespace hvn
