// Pack kernels shared by the tap-GEMM generators (declared in tap_conv.cuh).
#include "tap_conv.cuh"

namespace gsb {

__global__ void scale_copy_kernel(const float *__restrict__ src, int64_t count, float scale, const float *__restrict__ dev_scale,
                                  float *__restrict__ dst) {
    const float s = dev_scale ? scale * dev_scale[0] : scale;
    for (int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; i < count; i += (int64_t)gridDim.x * blockDim.x)
        dst[i] = src[i] * s;
}

__global__ void const_nhwc_kernel(const float *__restrict__ src, int C, float *__restrict__ dst) {
    for (int i = blockIdx.x * blockDim.x + threadIdx.x; i < 16 * C; i += gridDim.x * blockDim.x) dst[(i % 16) * C + i / 16] = src[i];
}

}  // namespace gsb
