// Component strips (notebooks/notebook_utils.py create_strip / create_strip_centered, latent mode).
//
// gsb_strip_latents builds the per-layer latents of every frame of a strip set in two launches:
//   strip_dots_kernel   one warp per (component, latent) pair: nrm = sqrt(sum(zc^2) + 1e-8) and, when centring,
//                       dotp = sum((z - mean) * (zc / nrm)); each lane sums a fixed stride of d in fp32, then a fixed xor
//                       butterfly -- deterministic, independent of the launch shape;
//   strip_apply_kernel  out[l][f][:] = z - dotp * (zc / nrm) + (zc * sigma) * stdev for l in [layer_start, layer_end), z
//                       elsewhere; every operation rounded on its own (no contraction), in the reference's order, so a frame
//                       whose dotp matches is bit-identical to the reference's torch expression.
// gsb_strip_offsets writes the activation edits of frames [f0, f0 + n) of a strip set (mode 'activation' / 'both'): the dots
// come from strip_dots_kernel over the layer's unedited values a_i and the activation components x_c, then
//   strip_offset_kernel  out[f - f0][:] = (xc * sigma) * stdev - (xc / nrm) * dotp, the centring term only when centring;
//                        rounded one operation at a time in the reference's order, so without centring the offsets are the
//                        reference's delta * act_stdev bit for bit.
// gsb_strip_pack_frames clamps the generator's [n, 3, H, W] images (any strides) to [0, 1] as np.clip does and writes NHWC
// fp32 frames, or uint8 frames with np.uint8(frame * 255) semantics.
#include "common.cuh"
#include <math.h>

namespace gsb {

// dots[2 * p] = nrm of component c, dots[2 * p + 1] = dotp of pair p = c * n_lat + i (0 without centring)
__global__ void strip_dots_kernel(const float *__restrict__ lat, int n_lat, const float *__restrict__ comp, int n_comp,
                                  const float *__restrict__ mean, int D, int center, float *__restrict__ dots) {
    const int p = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (p >= n_comp * n_lat) return;
    const int c = p / n_lat, i = p % n_lat;
    const float *zc = comp + (int64_t)c * D;
    float s = 0.f;
    for (int d = lane; d < D; d += 32) s = __fadd_rn(s, __fmul_rn(zc[d], zc[d]));
    const float nrm = __fsqrt_rn(__fadd_rn(warp_sum(s), 1e-8f));
    float dot = 0.f;
    if (center) {
        const float *z = lat + (int64_t)i * D;
        for (int d = lane; d < D; d += 32)
            dot = __fadd_rn(dot, __fmul_rn(__fsub_rn(z[d], mean[d]), __fdiv_rn(zc[d], nrm)));
        dot = warp_sum(dot);
    }
    if (lane == 0) {
        dots[2 * p] = nrm;
        dots[2 * p + 1] = dot;
    }
}

// grid (F, ceil(D / 128), L); frame f = (c * n_lat + i) * n_frames + k
__global__ void strip_apply_kernel(const float *__restrict__ lat, int n_lat, const float *__restrict__ comp,
                                   const float *__restrict__ stdev, const float *__restrict__ sigmas, int n_frames,
                                   const float *__restrict__ dots, int D, int64_t F, int layer_start, int layer_end, int center,
                                   float *__restrict__ out) {
    const int64_t f = blockIdx.x;
    const int d = blockIdx.y * blockDim.x + threadIdx.x;
    const int l = blockIdx.z;
    if (d >= D) return;
    const int64_t p = f / n_frames;
    const int k = (int)(f % n_frames);
    const int c = (int)(p / n_lat), i = (int)(p % n_lat);
    float v = lat[(int64_t)i * D + d];
    if (l >= layer_start && l < layer_end) {
        const float zc = comp[(int64_t)c * D + d];
        if (center) v = __fsub_rn(v, __fmul_rn(dots[2 * p + 1], __fdiv_rn(zc, dots[2 * p])));
        v = __fadd_rn(v, __fmul_rn(__fmul_rn(zc, sigmas[k]), stdev[c]));
    }
    out[((int64_t)l * F + f) * D + d] = v;
}

// grid (n, ceil(W / 128)); frame f = f0 + blockIdx.x = (c * n_lat + i) * n_frames + k
__global__ void strip_offset_kernel(const float *__restrict__ comp, int n_lat, const float *__restrict__ stdev,
                                    const float *__restrict__ sigmas, int n_frames, const float *__restrict__ dots, int W, int64_t f0,
                                    int center, float *__restrict__ out) {
    const int64_t f = f0 + blockIdx.x;
    const int d = blockIdx.y * blockDim.x + threadIdx.x;
    if (d >= W) return;
    const int64_t p = f / n_frames;
    const int k = (int)(f % n_frames);
    const int c = (int)(p / n_lat);
    const float xc = comp[(int64_t)c * W + d];
    float v = __fmul_rn(__fmul_rn(xc, sigmas[k]), stdev[c]);
    if (center) v = __fsub_rn(v, __fmul_rn(__fdiv_rn(xc, dots[2 * p]), dots[2 * p + 1]));
    out[(int64_t)blockIdx.x * W + d] = v;
}

// one thread per output byte-group: frame n, pixel (y, x), channel ch; src strides in elements
template <bool U8>
__global__ void strip_pack_kernel(const float *__restrict__ src, int64_t sn, int64_t sc, int64_t sh, int64_t sw, int64_t total,
                                  int H, int W, void *__restrict__ dst) {
    const int64_t t = (int64_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (t >= total) return;
    const int ch = (int)(t % 3);
    const int64_t px = t / 3;
    const int x = (int)(px % W);
    const int64_t r = px / W;
    const int y = (int)(r % H);
    const int64_t n = r / H;
    float v = src[n * sn + ch * sc + y * sh + x * sw];
    // np.clip(v, 0, 1) = min(max(v, 0), 1) with NaN kept: max(a, b) = isnan(a) ? a : (a > b ? a : b), min likewise with <
    if (!isnan(v)) {
        v = v > 0.f ? v : 0.f;
        v = v < 1.f ? v : 1.f;
    }
    if (U8)
        static_cast<unsigned char *>(dst)[t] = (unsigned char)__fmul_rn(v, 255.f);
    else
        static_cast<float *>(dst)[t] = v;
}

}  // namespace gsb

extern "C" size_t gsb_strip_workspace_bytes(int n_lat, int n_comp) { return (size_t)2 * n_lat * n_comp * sizeof(float); }

extern "C" int gsb_strip_latents(const float *d_latents, int n_lat, const float *d_comps, int n_comp, const float *d_stdev,
                                 const float *d_mean, const float *d_sigmas, int n_frames, int layer_start, int layer_end, int L,
                                 int D, int center, float *d_out, void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_latents && d_comps && d_stdev && d_sigmas && d_out && d_workspace, "strip_latents: null pointer");
    GSB_CHECK_ARG(!center || d_mean, "strip_latents: centring needs lat_mean");
    GSB_CHECK_ARG(n_lat >= 1 && n_comp >= 1 && n_frames >= 1 && L >= 1 && L <= 65535 && D >= 1 && D <= 65535 * 128,
                  "strip_latents: bad shape (n_lat=%d, n_comp=%d, n_frames=%d, L=%d, D=%d)", n_lat, n_comp, n_frames, L, D);
    GSB_CHECK_ARG(0 <= layer_start && layer_start <= layer_end && layer_end <= L,
                  "strip_latents: layer range [%d, %d) outside [0, %d]", layer_start, layer_end, L);
    const int64_t F = (int64_t)n_comp * n_lat * n_frames;
    GSB_CHECK_ARG(F <= 2147483647LL, "strip_latents: %lld frames", (long long)F);
    GSB_CHECK_ARG(workspace_bytes >= gsb_strip_workspace_bytes(n_lat, n_comp), "strip_latents: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    float *dots = static_cast<float *>(d_workspace);
    const int pairs = n_comp * n_lat;
    strip_dots_kernel<<<(pairs + 7) / 8, 256, 0, st>>>(d_latents, n_lat, d_comps, n_comp, d_mean, D, center, dots);
    GSB_CHECK_LAUNCH();
    dim3 grid((unsigned)F, (unsigned)((D + 127) / 128), (unsigned)L);
    strip_apply_kernel<<<grid, 128, 0, st>>>(d_latents, n_lat, d_comps, d_stdev, d_sigmas, n_frames, dots, D, F, layer_start,
                                             layer_end, center, d_out);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_strip_offsets(const float *d_acts, int n_lat, const float *d_comps, int n_comp, const float *d_stdev,
                                 const float *d_mean, const float *d_sigmas, int n_frames, int W, int center, int64_t f0, int64_t n,
                                 float *d_out, void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_comps && d_stdev && d_sigmas && d_out && d_workspace, "strip_offsets: null pointer");
    GSB_CHECK_ARG(!center || (d_acts && d_mean), "strip_offsets: centring needs the layer's values and act_mean");
    GSB_CHECK_ARG(n_lat >= 1 && n_comp >= 1 && n_frames >= 1 && W >= 1 && W <= 65535 * 128,
                  "strip_offsets: bad shape (n_lat=%d, n_comp=%d, n_frames=%d, W=%d)", n_lat, n_comp, n_frames, W);
    const int64_t F = (int64_t)n_comp * n_lat * n_frames;
    GSB_CHECK_ARG(0 <= f0 && 1 <= n && n <= 2147483647LL && f0 + n <= F,
                  "strip_offsets: frames [%lld, %lld) outside [0, %lld)", (long long)f0, (long long)(f0 + n), (long long)F);
    GSB_CHECK_ARG(workspace_bytes >= gsb_strip_workspace_bytes(n_lat, n_comp), "strip_offsets: workspace too small");
    cudaStream_t st = (cudaStream_t)stream;
    float *dots = static_cast<float *>(d_workspace);
    const int pairs = n_comp * n_lat;
    strip_dots_kernel<<<(pairs + 7) / 8, 256, 0, st>>>(d_acts, n_lat, d_comps, n_comp, d_mean, W, center, dots);
    GSB_CHECK_LAUNCH();
    dim3 grid((unsigned)n, (unsigned)((W + 127) / 128));
    strip_offset_kernel<<<grid, 128, 0, st>>>(d_comps, n_lat, d_stdev, d_sigmas, n_frames, dots, W, f0, center, d_out);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_strip_pack_frames(const float *d_src, int64_t sn, int64_t sc, int64_t sh, int64_t sw, int64_t n, int H, int W,
                                     int as_uint8, void *d_dst, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_src && d_dst, "strip_pack_frames: null pointer");
    GSB_CHECK_ARG(n >= 0 && H >= 1 && W >= 1, "strip_pack_frames: bad shape (n=%lld, H=%d, W=%d)", (long long)n, H, W);
    const int64_t total = n * H * W * 3;
    if (total == 0) return GSB_OK;
    const unsigned blocks = (unsigned)((total + 255) / 256);
    if (as_uint8)
        strip_pack_kernel<true><<<blocks, 256, 0, (cudaStream_t)stream>>>(d_src, sn, sc, sh, sw, total, H, W, d_dst);
    else
        strip_pack_kernel<false><<<blocks, 256, 0, (cudaStream_t)stream>>>(d_src, sn, sc, sh, sw, total, H, W, d_dst);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}
