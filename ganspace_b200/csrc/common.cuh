// Shared helpers for the ganspace_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include <stdio.h>
#include "../../include/ganspace_b200.h"

namespace gsb {

void set_error(const char *fmt, ...);

#define GSB_CHECK_ARG(cond, ...)                                  \
    do {                                                          \
        if (!(cond)) {                                            \
            gsb::set_error(__VA_ARGS__);                          \
            return GSB_ERR_ARG;                                   \
        }                                                         \
    } while (0)

#define GSB_CHECK_CUDA(expr)                                                              \
    do {                                                                                  \
        cudaError_t _e = (expr);                                                          \
        if (_e != cudaSuccess) {                                                          \
            gsb::set_error("%s failed: %s (%s:%d)", #expr, cudaGetErrorString(_e),        \
                           __FILE__, __LINE__);                                           \
            return GSB_ERR_CUDA;                                                          \
        }                                                                                 \
    } while (0)

#define GSB_CHECK_LAUNCH() GSB_CHECK_CUDA(cudaGetLastError())

static inline size_t align_up(size_t x, size_t a) { return (x + a - 1) / a * a; }

__device__ __forceinline__ double warp_sum(double v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_sum(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}

// Sum over a CTA; every thread gets the result.  `red` = shared scratch of >= 33 doubles.
__device__ __forceinline__ double block_sum(double v, double *red) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, nw = (blockDim.x + 31) >> 5;
    v = warp_sum(v);
    __syncthreads();  // protect `red` from the previous use
    if (lane == 0) red[warp] = v;
    __syncthreads();
    double t = (lane < nw) ? red[lane] : 0.0;
    t = warp_sum(t);
    return t;
}

// Warp-wide argmax of |x| (svd_flip's sign rule): each lane holds a candidate (best = |x|, idx, val = x); every lane gets
// the winner.  Ties go to the lower index, as np.argmax's first occurrence.
template <class T, class I>
__device__ __forceinline__ void warp_argmax_abs(T &best, I &idx, T &val) {
    for (int o = 16; o > 0; o >>= 1) {
        const T ob = __shfl_xor_sync(0xffffffffu, best, o), ov = __shfl_xor_sync(0xffffffffu, val, o);
        const I oi = __shfl_xor_sync(0xffffffffu, idx, o);
        if (ob > best || (ob == best && oi < idx)) { best = ob; idx = oi; val = ov; }
    }
}

int num_sms();

// Raises `kernel`'s dynamic shared-memory limit to `bytes` unless an earlier call already set at least that much (the
// largest size set so far is remembered per kernel, process-wide).
int raise_dyn_smem(const void *kernel, size_t bytes);
template <class F>
int raise_dyn_smem(F *kernel, size_t bytes) { return raise_dyn_smem(reinterpret_cast<const void *>(kernel), bytes); }

}  // namespace gsb
