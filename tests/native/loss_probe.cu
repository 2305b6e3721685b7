// Test-only entry point into the validation loss reduction (tests/test_loss_gpu.py): loss_reduce, the product's own
// code in loss.o, on caller-owned device buffers, so that the kernels can be checked alone on recorded cases.  This
// library (libhvn_loss_probe.so, built by build_loss_probe.py) is not part of the product or its C ABI.
#include <cstdio>

#include "../../hover_net_b200/csrc/common.cuh"
#include "../../hover_net_b200/csrc/loss.h"

using namespace hvn;

namespace {
Arena g_arena;
}

// probs f32 [n,h,w,4+nt], inst / type i32 [n,H,W] (type may be 0 when nt == 0), hv f32 [n,H,W,2], all device
// addresses -> sums f64 [loss_nsums(nt)] and counts i64 [3 + 2 nt] (both device; counts accumulated into).
// *bad: the out-of-range type flag.  Synchronises; returns 0, or an HVN_ERR_* code.
extern "C" int loss_probe_reduce(long long probs, long long inst, long long type, long long hv, int n, int H, int W,
                                 int h, int w, int nt, long long sums, long long counts, int *bad) {
    try {
        LossWork lw;
        loss_reduce(g_arena, 0, reinterpret_cast<const float *>(probs), reinterpret_cast<const int *>(inst),
                    reinterpret_cast<const int *>(type), reinterpret_cast<const float *>(hv), n, H, W, h, w, nt,
                    reinterpret_cast<double *>(sums), reinterpret_cast<long long *>(counts), lw);
        cudaError_t e = cudaDeviceSynchronize();
        if (e == cudaSuccess) e = cudaMemcpy(bad, lw.err, sizeof(int), cudaMemcpyDeviceToHost);
        if (e != cudaSuccess) {
            fprintf(stderr, "loss_probe: %s\n", cudaGetErrorString(e));
            return -2;
        }
        return 0;
    } catch (const Error &e) {
        fprintf(stderr, "loss_probe: %s\n", e.what());
        cudaDeviceSynchronize();
        return e.code;
    }
}

extern "C" int loss_probe_nsums(int nt) { return loss_nsums(nt); }

extern "C" void loss_probe_release() { g_arena.release(); }
