// Shared helpers for libhvn (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <stdexcept>

namespace hvn {

struct Error : public std::runtime_error {
    int code;
    Error(int c, const std::string &m) : std::runtime_error(m), code(c) {}
};

#define HVN_CUDA(expr)                                                                         \
    do {                                                                                       \
        cudaError_t e__ = (expr);                                                              \
        if (e__ != cudaSuccess)                                                                \
            throw ::hvn::Error(-2, std::string(#expr) + ": " + cudaGetErrorString(e__) + " @" + \
                                       __FILE__ + ":" + std::to_string(__LINE__));             \
    } while (0)

#define HVN_CHECK(cond, code, msg)                         \
    do {                                                   \
        if (!(cond)) throw ::hvn::Error((code), (msg));    \
    } while (0)

static inline int cdiv(long long a, long long b) { return (int)((a + b - 1) / b); }

// Grow-only device arena: one cudaMalloc per high-water mark, bump allocation per call.
struct Arena {
    char *base = nullptr;
    size_t cap = 0, top = 0;
    void reset() { top = 0; }
    void reserve(size_t bytes) {
        if (bytes <= cap) return;
        if (base) HVN_CUDA(cudaFree(base));
        base = nullptr;
        cap = 0;
        HVN_CUDA(cudaMalloc((void **)&base, bytes));
        cap = bytes;
    }
    template <typename T> T *take(size_t n) {
        size_t bytes = (n * sizeof(T) + 255) & ~(size_t)255;
        if (top + bytes > cap) throw Error(-2, "arena overflow (internal sizing bug)");
        T *p = (T *)(base + top);
        top += bytes;
        return p;
    }
    void release() {
        if (base) cudaFree(base);
        base = nullptr;
        cap = top = 0;
    }
};

// Counts bytes like Arena::take without allocating (sizing pass).
struct ArenaSizer {
    size_t top = 0;
    template <typename T> T *take(size_t n) {
        top += (n * sizeof(T) + 255) & ~(size_t)255;
        return nullptr;
    }
};

}  // namespace hvn
