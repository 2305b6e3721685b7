// Instance contours on the device (SURVEY.md row f3): for every instance-table row the outer border of the
// instance, point for point what the reference obtains from
//     cv2.findContours(inst_map[rmin:rmax, cmin:cmax] == id, RETR_TREE, CHAIN_APPROX_SIMPLE)[0][0] + (cmin, rmin)
// (reference models/hovernet/post_proc.py:133-147).  OpenCV's border following (Suzuki-Abe; contours.cpp
// icvFetchContour) is sequential per contour but instances are independent: one thread traces one
// instance straight on inst_map (pixels outside the bbox or of another id read as background, which is what
// the crop-and-compare does), first to count the CHAIN_APPROX_SIMPLE points, then -- after an exclusive
// scan of the counts -- to write them.  Direction codes 0..7 = E,NE,N,NW,W,SW,S,SE; the trace starts at the
// first pixel in raster order, takes as "previous" pixel the first neighbour clockwise from NW, searches
// counter-clockwise from the previous pixel at every step and keeps a point only where the step direction
// changes.  A flood region is 4-connected, hence a single 8-connected component whose outer border is the
// first contour cv2 returns.
#include "postproc.h"
#include "tile.h"

namespace hvn {
namespace {

__device__ __forceinline__ int cdx(int s) { return s == 0 || s == 1 || s == 7 ? 1 : (s >= 3 && s <= 5 ? -1 : 0); }
__device__ __forceinline__ int cdy(int s) { return s >= 1 && s <= 3 ? -1 : (s >= 5 && s <= 7 ? 1 : 0); }

struct Box { int rmin, cmin, rmax, cmax; };

__device__ __forceinline__ bool fg(const int *__restrict__ inst, int W, int id, const Box &b, int y, int x) {
    return y >= b.rmin && y < b.rmax && x >= b.cmin && x < b.cmax && inst[(size_t)y * W + x] == id;
}

// Traces the outer border; writes points (x, y) when WRITE.  Returns the number of points, 0 on
// inconsistent input (no pixel of `id` in the first bbox row, or a walk that does not close).
template <bool WRITE>
__device__ int trace(const int *__restrict__ inst, int W, int id, const Box &b, int *__restrict__ out) {
    int x0 = b.cmin;
    while (x0 < b.cmax && inst[(size_t)b.rmin * W + x0] != id) ++x0;
    if (x0 >= b.cmax) return 0;
    const int y0 = b.rmin;
    int s = 4;
    do {
        s = (s - 1) & 7;
        if (fg(inst, W, id, b, y0 + cdy(s), x0 + cdx(s))) break;
    } while (s != 4);
    if (s == 4) {  // isolated pixel
        if (WRITE) { out[0] = x0; out[1] = y0; }
        return 1;
    }
    const int y1 = y0 + cdy(s), x1 = x0 + cdx(s);
    int y3 = y0, x3 = x0, prev_s = s ^ 4, n = 0;
    const long long max_steps = 4ll * (b.rmax - b.rmin) * (b.cmax - b.cmin) + 8;
    for (long long step = 0; step < max_steps; ++step) {
        int y4, x4;
        for (;;) {
            ++s;
            y4 = y3 + cdy(s & 7); x4 = x3 + cdx(s & 7);
            if (fg(inst, W, id, b, y4, x4)) break;
        }
        s &= 7;
        if (s != prev_s) {
            if (WRITE) { out[2 * n] = x3; out[2 * n + 1] = y3; }
            ++n;
            prev_s = s;
        }
        if (y4 == y0 && x4 == x0 && y3 == y1 && x3 == x1) return n;
        y3 = y4; x3 = x4;
        s = (s + 4) & 7;
    }
    return 0;
}

template <bool WRITE>
__global__ void k_contour_trace(const int *__restrict__ inst_all, const long long *__restrict__ table,
                                const int *__restrict__ n_rows, int n_maps, int H, int W, int max_rows,
                                int *__restrict__ offs, int *__restrict__ pts, long long cap) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_maps * max_rows) return;
    const int m = idx / max_rows, r = idx - m * max_rows;
    const int rows = min(n_rows[m], max_rows);
    if (r >= rows) {
        if (!WRITE) offs[idx] = 0;
        return;
    }
    const long long *row = table + (size_t)idx * 10;
    Box b = {(int)row[1], (int)row[2], (int)row[3], (int)row[4]};
    const int *inst = inst_all + (size_t)m * H * W;
    if (!WRITE) {
        offs[idx] = trace<false>(inst, W, (int)row[0], b, nullptr);
    } else {
        const long long o = offs[idx], n = offs[idx + 1] - o;
        if (n > 0 && o + n <= cap) trace<true>(inst, W, (int)row[0], b, pts + 2 * o);
    }
}

// Write pass of a size class of a tile group into the packed layout: padded map m of the class is output image
// img_of[m] (a TileImage slot table, read at .img); its row r is packed row row_offs[img] + r, whose points are
// pts[pt_offs[row] : pt_offs[row + 1]].  Nothing is written when the packed table did not fit (row_offs[n_out] >
// rows_cap) or a row's points do not fit in cap.
__global__ void k_contour_write_packed(const int *__restrict__ inst_all, const long long *__restrict__ table,
                                       const int *__restrict__ n_rows, int n_maps, int H, int W, int max_rows,
                                       const TileImage *__restrict__ img_of, const int *__restrict__ row_offs, int n_out,
                                       long long rows_cap, const int *__restrict__ pt_offs, int *__restrict__ pts,
                                       long long cap) {
    const int idx = blockIdx.x * blockDim.x + threadIdx.x;
    if (idx >= n_maps * max_rows || row_offs[n_out] > rows_cap) return;
    const int m = idx / max_rows, r = idx - m * max_rows;
    if (r >= min(n_rows[m], max_rows)) return;
    const long long row = (long long)row_offs[img_of[m].img] + r;
    const long long o = pt_offs[row], n = pt_offs[row + 1] - o;
    if (n <= 0 || o + n > cap) return;
    const long long *t = table + (size_t)idx * 10;
    Box b = {(int)t[1], (int)t[2], (int)t[3], (int)t[4]};
    trace<true>(inst_all + (size_t)m * H * W, W, (int)t[0], b, pts + 2 * o);
}

// counts[0..total) -> exclusive prefix in place, offs[total] = sum.  One block.
__global__ void __launch_bounds__(1024) k_contour_scan(int *__restrict__ offs, int total) {
    __shared__ int part[1024];
    const int t = threadIdx.x;
    const int chunk = (total + 1023) / 1024;
    const int lo = min(t * chunk, total), hi = min(lo + chunk, total);
    int s = 0;
    for (int i = lo; i < hi; ++i) s += offs[i];
    part[t] = s;
    __syncthreads();
    for (int d = 1; d < 1024; d <<= 1) {
        int v = t >= d ? part[t - d] : 0;
        __syncthreads();
        part[t] += v;
        __syncthreads();
    }
    int run = part[t] - s;
    for (int i = lo; i < hi; ++i) {
        const int c = offs[i];
        offs[i] = run;
        run += c;
    }
    if (t == 1023) offs[total] = part[1023];
}

}  // namespace

int contours_count(cudaStream_t stream, const int *inst, const long long *table, const int *n_rows, int n_maps, int H,
                   int W, int max_rows, int *cnt) {
    k_contour_trace<false><<<cdiv((long long)n_maps * max_rows, 128), 128, 0, stream>>>(inst, table, n_rows, n_maps, H, W,
                                                                                      max_rows, cnt, nullptr, 0);
    HVN_CUDA(cudaGetLastError());
    return 1;
}

int contours_scan(cudaStream_t stream, int *offs, int total) {
    k_contour_scan<<<1, 1024, 0, stream>>>(offs, total);
    HVN_CUDA(cudaGetLastError());
    return 1;
}

int contours_write_packed(cudaStream_t stream, const int *inst, const long long *table, const int *n_rows, int n_maps,
                          int H, int W, int max_rows, const TileImage *img_of, const int *row_offs, int n_out,
                          long long rows_cap, const int *pt_offs, int *pts, long long cap) {
    k_contour_write_packed<<<cdiv((long long)n_maps * max_rows, 128), 128, 0, stream>>>(
        inst, table, n_rows, n_maps, H, W, max_rows, img_of, row_offs, n_out, rows_cap, pt_offs, pts, cap);
    HVN_CUDA(cudaGetLastError());
    return 1;
}

int contours_run(cudaStream_t stream, const int *inst, const long long *table, const int *n_rows, int n_maps, int H,
                 int W, int max_rows, int *pts, long long cap, int *offs) {
    const int total = n_maps * max_rows;
    const int threads = 128, blocks = cdiv(total, threads);
    contours_count(stream, inst, table, n_rows, n_maps, H, W, max_rows, offs);
    contours_scan(stream, offs, total);
    k_contour_trace<true><<<blocks, threads, 0, stream>>>(inst, table, n_rows, n_maps, H, W, max_rows, offs, pts, cap);
    HVN_CUDA(cudaGetLastError());
    return 3;
}

}  // namespace hvn
