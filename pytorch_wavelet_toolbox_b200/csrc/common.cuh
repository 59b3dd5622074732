// common.cuh -- shared device helpers for the H100 (sm_90a) wavelet filter bank.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#include "../../include/wtb200.h"
#include "knobs.cuh"

#include <mutex>
#include <unordered_map>

namespace wtb {

// Opt a kernel in to `bytes` of dynamic shared memory.  cudaFuncSetAttribute is a driver call whose cost is far from
// negligible when the value CHANGES from launch to launch (milliseconds of host time per call), so the limit is only ever raised, once per (device, kernel), and kernels whose
// need varies with the problem ask for their maximum up front.
template <typename K>
static cudaError_t ensure_dyn_smem(K kern, size_t bytes) {
    static std::mutex mu;
    static std::unordered_map<uint64_t, size_t> cur;
    int dev = 0;
    cudaGetDevice(&dev);
    const uint64_t key = (uint64_t)(uintptr_t)kern * 64u + (uint64_t)(dev & 63);
    std::lock_guard<std::mutex> g(mu);
    size_t& v = cur[key];
    if (bytes <= v) return cudaSuccess;
    const cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bytes);
    if (e == cudaSuccess) v = bytes;
    return e;
}
constexpr size_t WTB_MAX_DYN_SMEM = 227 * 1024;

// SM count of the current device (132 on an H100 SXM): the grid-size heuristics fill the machine with it.
static inline int sm_count() {
    int dev = 0, n = 0;
    cudaGetDevice(&dev);
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n < 1) n = 132;
    return n;
}


// Filter taps travel as kernel parameters (no __constant__ symbols), so concurrent
// streams may run different wavelets.
template <typename T>
struct Taps {
    T lo[WT_MAX_FILT_LEN];
    T hi[WT_MAX_FILT_LEN];
};

// Boundary extension ext(x)[j] for j outside [0, n).  Returns the source index, or -1
// when the sample is an implicit zero.  Restates the five ptwt modes
// (reference src/ptwt/_util.py:36-44, :163-195; torch F.pad semantics for the rest).
__device__ __forceinline__ int64_t ext_index(int64_t j, int64_t n, int mode) {
    if (j >= 0 && j < n) return j;
    switch (mode) {
        case WT_MODE_ZERO:
            return -1;
        case WT_MODE_CONSTANT:
            return j < 0 ? 0 : n - 1;
        case WT_MODE_REFLECT: {
            if (n == 1) return 0;
            const int64_t p = 2 * n - 2;
            j %= p;
            if (j < 0) j += p;
            return j < n ? j : p - j;
        }
        case WT_MODE_PERIODIC: {
            j %= n;
            if (j < 0) j += n;
            return j;
        }
        default: {  // WT_MODE_SYMMETRIC
            const int64_t p = 2 * n;
            j %= p;
            if (j < 0) j += p;
            return j < n ? j : p - 1 - j;
        }
    }
}

// 32-bit flavour for tile kernels (extents < 2^31).
__device__ __forceinline__ int ext_index32(int j, int n, int mode) {
    if (j >= 0 && j < n) return j;
    switch (mode) {
        case WT_MODE_ZERO:
            return -1;
        case WT_MODE_CONSTANT:
            return j < 0 ? 0 : n - 1;
        case WT_MODE_REFLECT: {
            if (n == 1) return 0;
            const int p = 2 * n - 2;
            j %= p;
            if (j < 0) j += p;
            return j < n ? j : p - j;
        }
        case WT_MODE_PERIODIC: {
            j %= n;
            if (j < 0) j += n;
            return j;
        }
        default: {
            const int p = 2 * n;
            j %= p;
            if (j < 0) j += p;
            return j < n ? j : p - 1 - j;
        }
    }
}

}  // namespace wtb
