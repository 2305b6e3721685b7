// Host-side interface of the whole-image tile path (tile.cu).
#pragma once
#include <vector>

#include "common.cuh"

namespace hvn {

struct Model;

// One image of a tile group, as the gather / scatter kernels see it (a small device table, one entry per slot).
struct TileImage {
    long long in_off;    // byte offset of the image in the packed input (input order)
    long long pred_off;  // float offset of its [H,W,C] map in the prediction buffer (slot order)
    long long cell0;     // global index of its first patch: prefix sum of the cell counts of the earlier slots
    long long row0;      // first row of its padded instance table in the group's table workspace
    int H, W, rows, cols;
    int img;             // its index in input order
    int max_rows;        // rows of its padded table: min(rows_cap, id bound of H x W), the same for its size class
};

// patch grid of reference infer/tile.py:60-69 for an H x W image and a patch_out step
void tile_grid(int H, int W, int patch_out, int *rows, int *cols);
size_t tile_workspace_bytes(int patch_in, int patch_out, int C, int batch);
// Lays out a group of n images, shapes [n][2] (H, W): slots[s] for slot s, slot_of[i] = slot of input image i.  Slots
// are ordered by size class (classes in order of first appearance, input order within a class) so that each class's
// maps are contiguous in the prediction buffer.  Returns the number of size classes.
int tile_plan(const int *shapes, int n, int step, int C, std::vector<TileImage> &slots, std::vector<int> &slot_of);
// Runs global patches [cell_lo, cell_hi) of the group img [n_img] (device table in slot order) through the network in
// batches of `batch` and writes each patch's map into its image's region of pred (device).  Pixels of other patches
// are left untouched.  Returns its own kernel launches.
int tile_predict(Model &model, Arena &ws, cudaStream_t s, const uint8_t *imgs, const TileImage *img, int n_img,
                 long long cell_lo, long long cell_hi, int patch_in, int batch, int chunk, float *pred);

// Instance tables [n,max_rows,10] -> packed [<= cap rows,10], offs [n+1] (offs[n] = total rows; rows past cap are not
// written).  Device pointers.  Returns its kernel launches.
// Tile-group form (geo not null): output map m is slot slot[m], whose padded table starts at row geo[s].row0 of `table`
// and holds geo[s].max_rows rows (n_rows and cnt are indexed by slot / by table row alike); offs count every row of
// n_rows, so offs[n] is the true total; cnt (may be null) is packed to packed_cnt like the rows.
int pack_tables(cudaStream_t s, const long long *table, const int *n_rows, int n, int max_rows, long long *packed,
                long long cap, int *offs, const int *slot = nullptr, const TileImage *geo = nullptr,
                const int *cnt = nullptr, int *packed_cnt = nullptr);

}  // namespace hvn
