// Test-only entry points into the post-processing kernels, one stage at a time (tests/test_postproc_stages_gpu.py).
//
// pp_probe_run runs the whole post-processing path (postproc_run, the product's own code in postproc.o) on a
// probe-owned arena, so that pp_probe_buffers can then hand out the stage buffers it left there.  pp_probe_flood runs
// the watershed stage alone through the same kernels (postproc_flood_only) with a forced or automatic flood kernel.
// All buffers are device pointers the caller owns; every entry synchronises and reports errors as return codes.  This
// library (libhvn_pp_probe.so, built by build_pp_probe.py) is linked from postproc.o, the object libhvn.so is built
// from, and is not part of the product or its C ABI.
#include <cstdio>

#include "../../hover_net_b200/csrc/common.cuh"
#include "../../hover_net_b200/csrc/postproc.h"

using namespace hvn;

namespace {

Arena g_arena;

int finish(int rc_ok) {
    cudaError_t e = cudaDeviceSynchronize();
    if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) {
        fprintf(stderr, "pp_probe: %s\n", cudaGetErrorString(e));
        return -2;
    }
    return rc_ok;
}

template <typename F> int guarded(F f) {
    try {
        return f();
    } catch (const Error &e) {
        fprintf(stderr, "pp_probe: %s\n", e.what());
        cudaDeviceSynchronize();
        return e.code;
    }
}

}  // namespace

// pred [n,H,W,C] f32 -> inst [n,H,W] i32, table [n,max_rows,10] i64, nrows [n] i32.  *launches: kernels launched.
extern "C" int pp_probe_run(long long pred, int n, int H, int W, int C, int nr_types, long long inst, long long table,
                            int max_rows, long long nrows, int *launches) {
    return guarded([&] {
        *launches = postproc_run(g_arena, 0, reinterpret_cast<const float *>(pred), n, H, W, C, nr_types,
                                 reinterpret_cast<int *>(inst), reinterpret_cast<long long *>(table), max_rows,
                                 reinterpret_cast<int *>(nrows));
        return finish(0);
    });
}

// Stage buffers of the last pp_probe_run with the same (n, H, W, nr_types), as device addresses:
//   0 fg (u8, after the < 10 px filter)  1 sobh  2 sobv  3 din  4 dist (f64)  5 mk0  6 filled  7 opened (u8)
//   8 L2 (i32, root pixel of each opened-marker component, -1 off)  9 size3 (i32, component size by root)
//   10 id3 (i32, scipy label id by root)  11 L1 (i32, root of each foreground component)  12 size1
extern "C" int pp_probe_buffers(int n, int H, int W, int nr_types, long long *out) {
    return guarded([&] {
        PostprocBuffers b;
        postproc_buffers(g_arena, n, H, W, nr_types, b);
        const void *p[13] = {b.fg, b.sobh, b.sobv, b.din, b.dist, b.mk0, b.filled, b.opened, b.L2, b.size3, b.id3,
                             b.L1, b.size1};
        for (int i = 0; i < 13; ++i) out[i] = (long long)(size_t)p[i];
        return 0;
    });
}

// dist f64, mask u8, markers i32 [n,H,W] -> inst i32.  choice: FloodKernel (0 auto, 1 calendar queue, 2 heap with key
// table, 3 heap without, 4 global heap).  *kernel: the FloodKernel that ran.  -1: the forced kernel does not fit the map.
extern "C" int pp_probe_flood(long long dist, long long mask, long long markers, int n, int H, int W, long long inst,
                              int choice, int *kernel) {
    return guarded([&] {
        *kernel = postproc_flood_only(g_arena, 0, reinterpret_cast<const double *>(dist),
                                      reinterpret_cast<const unsigned char *>(mask), reinterpret_cast<const int *>(markers),
                                      n, H, W, reinterpret_cast<int *>(inst), choice);
        return finish(0);
    });
}

// bytes from device address src into host memory dst
extern "C" int pp_probe_d2h(void *dst, long long src, long long bytes) {
    cudaError_t e = cudaMemcpy(dst, reinterpret_cast<const void *>(src), (size_t)bytes, cudaMemcpyDeviceToHost);
    return e == cudaSuccess ? 0 : -2;
}

extern "C" int pp_probe_max_ids(int H, int W) { return postproc_max_ids(H, W); }

extern "C" void pp_probe_release() { g_arena.release(); }
