// Pieces shared by the three tap-GEMM generators: StyleGAN2 (synthesis.cu), ProGAN (progan.cu) and StyleGAN v1 (stylegan.cu).
// Each of them runs a conv as one tc_gemm_plain contraction per tap into the tap planes Y[b, p, tap, co] at the input
// resolution, followed by a gather.  The gather's epilogue (demodulation, PixelNorm, instance statistics, ...) stays in the
// generator's own file.
#pragma once
#include "tc_common.cuh"

namespace gsb {

// fp32 elements of the largest per-chunk buffer of a ProGAN / StyleGAN layer: 2048 x 9 x 512 = 38 MB of the 50 MB L2, so that a
// chunk's tap planes stay in L2 between the GEMM and its gather
constexpr int64_t TAP_CHUNK_ELEMS = (int64_t)2048 * 9 * 512;

// 3x3 conv (padding 1) of channels [4q, 4q + 4) at output pixel (y, x) of sample b on an R x R map, from tap planes Y with `ld`
// floats per row: the sum, over ky then kx, of Y[b, (yy, xx), ky * 3 + kx, 4q ..] for yy = y + ky - 1, xx = x + kx - 1 inside
// [0, R).  UP: the conv reads the nearest-x2 up-sampled input, so Y is at resolution R/2 and the source pixel is (yy>>1, xx>>1).
template <bool UP>
__device__ __forceinline__ float4 tap_sum3x3(const float *__restrict__ Y, int ld, int64_t b, int y, int x, int R, int c, int q) {
    const int H = UP ? (R >> 1) : R;
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int yy = y + ky - 1;
        if (yy < 0 || yy >= R) continue;
        const int ys = UP ? (yy >> 1) : yy;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int xx = x + kx - 1;
            if (xx < 0 || xx >= R) continue;
            const int xs = UP ? (xx >> 1) : xx;
            const float4 v = *reinterpret_cast<const float4 *>(Y + ((b * H + ys) * H + xs) * (int64_t)ld + (ky * 3 + kx) * c + 4 * q);
            acc.x += v.x; acc.y += v.y; acc.z += v.z; acc.w += v.w;
        }
    }
    return acc;
}

// Sum of v over the c/4 threads that hold one pixel's channels (consecutive threads, cq = c/4 a power of two that divides the
// block size; every thread of the block calls this).  Shuffles inside a warp, then for c >= 256 the 2 .. 8 warps of the pixel
// are added in warp order from shared memory: the same order for every pixel, batch size and launch.
__device__ __forceinline__ float pixel_sum(float v, int cq) {
    const int span = cq < 32 ? cq : 32;
    for (int off = span >> 1; off > 0; off >>= 1) v += __shfl_xor_sync(0xffffffffu, v, off);
    if (cq > 32) {
        __shared__ float red[8];
        const int wib = threadIdx.x >> 5, wpp = cq >> 5;            // warp in block, warps per pixel
        __syncthreads();                                            // the previous call's readers are done
        if ((threadIdx.x & 31) == 0) red[wib] = v;
        __syncthreads();
        const int w0 = wib / wpp * wpp;
        v = 0.f;
        for (int k = 0; k < wpp; ++k) v += red[w0 + k];
    }
    return v;
}

// ---- pack kernels (tap_conv.cu) -----------------------------------------------------------------------------------------
// dst[i] = src[i] * s for i < count, with s = scale, or scale * dev_scale[0] when dev_scale is given (a scalar on the device)
__global__ void scale_copy_kernel(const float *__restrict__ src, int64_t count, float scale, const float *__restrict__ dev_scale,
                                  float *__restrict__ dst);
// a learned constant [C, 4, 4] (NCHW of one sample) -> [16, C] (NHWC)
__global__ void const_nhwc_kernel(const float *__restrict__ src, int C, float *__restrict__ dst);

}  // namespace gsb
