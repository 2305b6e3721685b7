// Whole-image tile path on the device (SURVEY.md row f1; reference infer/tile.py:46-143 and its multi-file loop
// :236-369): reflect-pad + patch grid (`_prepare_patching`), the batch loop over patches, and the stitch + crop of
// `_post_process_patches` -- as index arithmetic, over a group of images of any sizes.  The padded images never
// exist: a patch pixel reads its source image through numpy's "reflect" index map (no edge repeat, period
// 2*(L-1)), and every patch output pixel is written straight to its place in that image's [H,W,C] prediction map
// (pixels past H/W are the crop).  Geometry per image: step = patch_out; rows = ceil((H - step)/step) + 1
// (tile.py:60-69); pad top/left = (patch_in - patch_out)/2; patch (r, c) covers padded rows [r*step, r*step +
// patch_in).  The patches of the group form one list (image after image, row-major within an image); a batch
// is any contiguous range of it, so it may start in one image and end in another, as in the reference.
#include <algorithm>

#include "cnn.h"
#include "tile.h"

namespace hvn {
namespace {

__device__ __forceinline__ int reflect_index(int i, int L) {
    if (L == 1) return 0;
    const int p = 2 * (L - 1);
    int t = i % p;
    if (t < 0) t += p;
    return t < L ? t : p - t;
}

// The image that holds global patch `cell`: the last entry with cell0 <= cell (cell0 ascending, img[0].cell0 = 0).
__device__ __forceinline__ int find_image(const TileImage *__restrict__ img, int n_img, long long cell) {
    int lo = 0, hi = n_img - 1;
    while (lo < hi) {
        const int mid = (lo + hi + 1) >> 1;
        if (img[mid].cell0 <= cell) lo = mid; else hi = mid - 1;
    }
    return lo;
}

// patches [n, win, win, 3] u8 for global patches first .. first+n-1; blockIdx.y = patch in the batch
__global__ void k_tile_gather(const uint8_t *__restrict__ src, const TileImage *__restrict__ img, int n_img, int win,
                              int step, int pad, long long first, uint8_t *__restrict__ patches) {
    __shared__ TileImage s_img;
    const int p = blockIdx.y;
    if (threadIdx.x == 0) s_img = img[find_image(img, n_img, first + p)];
    __syncthreads();
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= win * win) return;
    const int py = r / win, px = r - py * win;
    const int cell = (int)(first + p - s_img.cell0);
    const int gr = cell / s_img.cols, gc = cell - gr * s_img.cols;
    const int sy = reflect_index(gr * step + py - pad, s_img.H), sx = reflect_index(gc * step + px - pad, s_img.W);
    const uint8_t *s = src + s_img.in_off + ((size_t)sy * s_img.W + sx) * 3;
    uint8_t *d = patches + ((size_t)p * win * win + r) * 3;
    d[0] = s[0]; d[1] = s[1]; d[2] = s[2];
}

// outputs [n, step, step, C] f32 -> each patch's image map [H, W, C] at pred + pred_off, at (row*step, col*step),
// cropped to H x W
__global__ void k_tile_scatter(const float *__restrict__ outs, const TileImage *__restrict__ img, int n_img, int step,
                               int C, long long first, float *__restrict__ pred) {
    __shared__ TileImage s_img;
    const int p = blockIdx.y;
    if (threadIdx.x == 0) s_img = img[find_image(img, n_img, first + p)];
    __syncthreads();
    const int r = blockIdx.x * blockDim.x + threadIdx.x;
    if (r >= step * step) return;
    const int py = r / step, px = r - py * step;
    const int cell = (int)(first + p - s_img.cell0);
    const int gr = cell / s_img.cols, gc = cell - gr * s_img.cols;
    const int y = gr * step + py, x = gc * step + px;
    if (y >= s_img.H || x >= s_img.W) return;
    const float *s = outs + ((size_t)p * step * step + r) * C;
    float *d = pred + s_img.pred_off + ((size_t)y * s_img.W + x) * C;
    for (int c = 0; c < C; ++c) d[c] = s[c];
}

// Instance tables [n, max_rows, 10] (padded) -> packed rows [sum n_rows, 10] + offs [n + 1].  One block per map: its
// offset is the sum of the earlier maps' row counts (n is a batch size: a strided sum), min(n_rows, max_rows) each.
// Tile-group form (geo not null): output map m is slot s = slot[m], whose padded table starts at row geo[s].row0 and
// holds geo[s].max_rows rows; offsets count all n_rows (a caller sizing its buffer from offs[n] needs the true total);
// the per-row contour point counts cnt (same layout as the table rows) move to packed_cnt with the rows.  `packed` may
// equal `table` (and packed_cnt cnt) when n == 1: the rows are then already in place.
__global__ void k_pack_tables(const long long *table, const int *__restrict__ n_rows, int n, int max_rows,
                              long long *packed, long long cap, int *__restrict__ offs, const int *__restrict__ slot,
                              const TileImage *__restrict__ geo, const int *cnt, int *packed_cnt) {
    __shared__ int s_part[32];
    __shared__ int s_off;
    const int m = blockIdx.x;
    int part = 0;
    for (int i = threadIdx.x; i < m; i += blockDim.x) {
        const int k = n_rows[geo ? slot[i] : i];
        part += geo ? k : min(k, max_rows);
    }
    for (int o = 16; o; o >>= 1) part += __shfl_xor_sync(0xffffffffu, part, o);
    if ((threadIdx.x & 31) == 0) s_part[threadIdx.x >> 5] = part;
    __syncthreads();
    const int sm = geo ? slot[m] : m;
    const int k = n_rows[sm];
    const int stride = geo ? geo[sm].max_rows : max_rows;
    const size_t row0 = geo ? (size_t)geo[sm].row0 : (size_t)sm * max_rows;
    if (threadIdx.x == 0) {
        int t = 0;
        for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += s_part[w];
        s_off = t;
        offs[m] = t;
        if (m == n - 1) offs[n] = t + (geo ? k : min(k, max_rows));
    }
    __syncthreads();
    const int off = s_off, nr = min(k, stride);
    if (packed != table) {
        const long long *src = table + row0 * 10;
        for (int i = threadIdx.x; i < nr * 10; i += blockDim.x) {
            const long long row = off + i / 10;
            if (row < cap) packed[(size_t)off * 10 + i] = src[i];
        }
    }
    if (cnt && packed_cnt != cnt)
        for (int i = threadIdx.x; i < nr; i += blockDim.x)
            if (off + i < cap) packed_cnt[off + i] = cnt[row0 + i];
}

}  // namespace

int pack_tables(cudaStream_t s, const long long *table, const int *n_rows, int n, int max_rows, long long *packed,
                long long cap, int *offs, const int *slot, const TileImage *geo, const int *cnt, int *packed_cnt) {
    k_pack_tables<<<n, 256, 0, s>>>(table, n_rows, n, max_rows, packed, cap, offs, slot, geo, cnt, packed_cnt);
    HVN_CUDA(cudaGetLastError());
    return 1;
}

void tile_grid(int H, int W, int patch_out, int *rows, int *cols) {
    auto steps = [&](int L) { return (L <= patch_out ? 0 : (L - patch_out + patch_out - 1) / patch_out) + 1; };
    *rows = steps(H);
    *cols = steps(W);
}

size_t tile_workspace_bytes(int patch_in, int patch_out, int C, int batch) {
    return ((size_t)batch * patch_in * patch_in * 3 + 255) / 256 * 256 + ((size_t)batch * patch_out * patch_out * C * 4 + 255) / 256 * 256;
}

int tile_plan(const int *shapes, int n, int step, int C, std::vector<TileImage> &slots, std::vector<int> &slot_of) {
    HVN_CHECK(n >= 1, -1, "a tile group needs at least one image");
    std::vector<long long> in_off(n);
    long long off = 0;
    for (int i = 0; i < n; ++i) {
        const int H = shapes[2 * i], W = shapes[2 * i + 1];
        HVN_CHECK(H >= 1 && W >= 1 && (long long)H * W < (1ll << 30), -1,
                  "image " + std::to_string(i) + ": bad shape " + std::to_string(H) + "x" + std::to_string(W));
        in_off[i] = off;
        off += (long long)H * W * 3;
    }
    // slot order: size classes in order of first appearance, input order within a class
    slots.clear();
    slot_of.assign(n, -1);
    int classes = 0;
    long long cell0 = 0, pred_off = 0;
    for (int i = 0; i < n; ++i) {
        if (slot_of[i] >= 0) continue;
        ++classes;
        for (int j = i; j < n; ++j) {
            if (shapes[2 * j] != shapes[2 * i] || shapes[2 * j + 1] != shapes[2 * i + 1]) continue;
            TileImage t;
            t.in_off = in_off[j];
            t.pred_off = pred_off;
            t.cell0 = cell0;
            t.H = shapes[2 * j];
            t.W = shapes[2 * j + 1];
            tile_grid(t.H, t.W, step, &t.rows, &t.cols);
            t.img = j;
            t.row0 = 0;      // the padded-table layout is the caller's (it depends on rows_cap)
            t.max_rows = 0;
            slot_of[j] = (int)slots.size();
            slots.push_back(t);
            cell0 += (long long)t.rows * t.cols;
            pred_off += (long long)t.H * t.W * C;
        }
    }
    HVN_CHECK(cell0 < (1ll << 31), -1, "too many patches in one tile group");
    return classes;
}

int tile_predict(Model &model, Arena &ws, cudaStream_t s, const uint8_t *imgs, const TileImage *img, int n_img,
                 long long cell_lo, long long cell_hi, int patch_in, int batch, int chunk, float *pred) {
    int oh, ow, oc;
    model.out_shape(patch_in, patch_in, oh, ow, oc);
    HVN_CHECK(oh == ow && oh >= 1, -1, "unsupported patch size for this model mode");
    const int step = oh, pad = (patch_in - step) / 2;
    if (batch < 1) batch = 64;
    batch = std::min(batch, 65535);  // gridDim.y of the gather / scatter; the forward does not depend on the split
    uint8_t *patches = ws.take<uint8_t>((size_t)batch * patch_in * patch_in * 3);
    float *outs = ws.take<float>((size_t)batch * step * step * oc);
    int launches = 0;
    for (long long first = cell_lo; first < cell_hi; first += batch) {
        const int n = (int)std::min<long long>(batch, cell_hi - first);
        k_tile_gather<<<dim3(cdiv(patch_in * patch_in, 256), n), 256, 0, s>>>(imgs, img, n_img, patch_in, step, pad, first,
                                                                               patches);
        model.forward(patches, n, patch_in, patch_in, outs, chunk, s);
        k_tile_scatter<<<dim3(cdiv(step * step, 256), n), 256, 0, s>>>(outs, img, n_img, step, oc, first, pred);
        launches += 2;
    }
    HVN_CUDA(cudaGetLastError());
    return launches;
}

}  // namespace hvn
