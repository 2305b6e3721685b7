// Probe: how many bytes per clock can the SMs pull out of L2 with bulk async copies (the path every operand tile of
// k_conv_tc takes), and does a cluster multicast raise the per-SM rate?
//   mode 0  unicast, every CTA streams its own tiles from a 64 MB (L2-resident) buffer
//   mode 1  unicast, the two CTAs of a cluster fetch the SAME tile (32 KB each)
//   mode 2  multicast, each CTA of a cluster fetches half a tile (16 KB) and multicasts it to both: 32 KB land per CTA
//   mode 3  unicast from a 4 GB buffer (HBM)
//   nvcc -gencode arch=compute_90a,code=sm_90a -O2 -o tools/tma_bw_probe tools/tma_bw_probe.cu
#include <cuda_runtime.h>
#include <cstdint>
#include <cstdio>

constexpr int TILE = 32768, SLOTS = 4;

__device__ __forceinline__ uint32_t smem_u32(const void *p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_wait(uint32_t bar, uint32_t parity) {
    uint32_t ok;
    do {
        asm volatile("{\n\t.reg .pred p;\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}"
                     : "=r"(ok) : "r"(bar), "r"(parity) : "memory");
    } while (!ok);
}

__global__ void __cluster_dims__(2, 1, 1) __launch_bounds__(128, 1)
probe(const uint8_t *buf, size_t buf_bytes, int mode, int iters, long long *cycles) {
    extern __shared__ __align__(1024) uint8_t raw[];
    __shared__ __align__(8) uint64_t full[SLOTS];
    const uint32_t base = (smem_u32(raw) + 1023u) & ~1023u;
    uint32_t rank;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(rank));
    const size_t ntiles = buf_bytes / TILE;
    if (threadIdx.x == 0) {
        for (int s = 0; s < SLOTS; ++s) asm volatile("mbarrier.init.shared::cta.b64 [%0], 1;" ::"r"(smem_u32(&full[s])) : "memory");
        asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    }
    asm volatile("barrier.cluster.arrive.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
    long long t0 = 0;
    if (threadIdx.x == 0) t0 = clock64();
    for (int lap = 0; lap < iters / SLOTS; ++lap) {
        if (threadIdx.x == 0) {
            for (int s = 0; s < SLOTS; ++s) {
                const int i = lap * SLOTS + s;
                const uint32_t bar = smem_u32(&full[s]), dst = base + s * TILE;
                asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(bar), "r"(TILE) : "memory");
                if (mode == 2) {
                    const size_t tile = ((size_t)i * (gridDim.x / 2) + blockIdx.x / 2) % ntiles;
                    const uint8_t *src = buf + tile * TILE + rank * (TILE / 2);
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes.multicast::cluster [%0], [%1], %2, [%3], %4;"
                                 ::"r"(dst + rank * (TILE / 2)), "l"(src), "r"(TILE / 2), "r"(bar), "h"((uint16_t)3) : "memory");
                } else {
                    const size_t tile = (mode == 1 ? ((size_t)i * (gridDim.x / 2) + blockIdx.x / 2) : ((size_t)i * gridDim.x + blockIdx.x)) % ntiles;
                    asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
                                 ::"r"(dst), "l"(buf + tile * TILE), "r"(TILE), "r"(bar) : "memory");
                }
            }
            for (int s = 0; s < SLOTS; ++s) mbar_wait(smem_u32(&full[s]), (uint32_t)lap & 1u);
        }
        if (mode == 2) asm volatile("barrier.cluster.arrive.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
        else __syncthreads();
    }
    if (threadIdx.x == 0) cycles[blockIdx.x] = clock64() - t0;
    asm volatile("barrier.cluster.arrive.aligned;\n\tbarrier.cluster.wait.aligned;" ::: "memory");
}

int main() {
    uint8_t *buf;
    const size_t big = 4ull << 30, small = 64ull << 20;
    if (cudaMalloc(&buf, big) != cudaSuccess) { printf("alloc failed\n"); return 1; }
    cudaMemset(buf, 1, big);
    long long *d;
    cudaMalloc(&d, 8 * 148);
    const int smem = SLOTS * TILE + 1024;
    cudaFuncSetAttribute(probe, cudaFuncAttributeMaxDynamicSharedMemorySize, smem);
    const int iters = 4096;
    const char *names[4] = {"unicast, own tiles, L2-resident (64 MB)", "unicast, cluster pair fetches the same tile", "multicast, half a tile per CTA to both",
                            "unicast, own tiles, HBM (4 GB)"};
    printf("bulk-copy rate into shared memory, 148 CTAs (74 clusters of 2), %d x 32 KB per CTA, 4 in flight\n", iters);
    for (int mode = 0; mode < 4; ++mode) {
        for (int rep = 0; rep < 2; ++rep) {
            cudaEvent_t a, b;
            cudaEventCreate(&a); cudaEventCreate(&b);
            cudaEventRecord(a);
            probe<<<148, 128, smem>>>(buf, mode == 3 ? big : small, mode, iters, d);
            cudaEventRecord(b);
            cudaError_t e = cudaDeviceSynchronize();
            if (e != cudaSuccess) { printf("mode %d: CUDA error %s\n", mode, cudaGetErrorString(e)); return 1; }
            float ms;
            cudaEventElapsedTime(&ms, a, b);
            long long c[148], mx = 0;
            cudaMemcpy(c, d, sizeof(c), cudaMemcpyDeviceToHost);
            for (int i = 0; i < 148; ++i) mx = c[i] > mx ? c[i] : mx;
            if (rep == 1)
                printf("mode %d  %-46s %7.3f ms  %6.1f B/clk per SM landed  %7.2f TB/s landed chip-wide\n", mode, names[mode], ms,
                       (double)iters * TILE / (double)mx, 148.0 * iters * TILE / (ms * 1e-3) / 1e12);
        }
    }
    return 0;
}
