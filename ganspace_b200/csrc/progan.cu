// ProGAN generator: layer1 .. layerK and the RGB output block.
//
// Replaces netdissect/proggan.py:93-171 (ProgressiveGenerator.forward: NormConvBlock, NormUpscaleConvBlock, OutputConvBlock) as
// driven by models/wrappers.py:500-522 (ProGAN.forward, partial_forward).
//
// Every block is  x^ = PixelNorm(x)  ->  (nearest x2)  ->  conv without bias  ->  * gain/sqrt(cin) + b  ->  leaky-ReLU 0.2.
// The weights are shared by all samples, so each conv is one dense contraction over ci per tap (the formulation of
// synthesis.cu, same wgmma GEMM with fp16 hi/lo operands) followed by a gather:
//     Y[b,p,tap,co]   = sum_ci (scale W)[co,ci,tap] x^[b,p,ci]                                K = ci, N = taps * co
//     layer1   :  the 1x1 latent under a 4x4 kernel with padding 3 meets tap (3-y, 3-x) at output pixel (y, x): the weights are
//                 packed with the taps reversed and Y[b, 0, (y,x), co] IS the 4x4 output
//     stride 1 :  out[b,y,x,co] = sum_tap Y[b,(y+ky-1, x+kx-1),tap,co]
//     upsample :  nearest x2 only replicates pixels and PixelNorm is per pixel, so up(x^)[u,v] = x^[u>>1, v>>1] and
//                 out[b,y,x,co] = sum_tap Y[b,((y+ky-1)>>1, (x+kx-1)>>1),tap,co]   for 0 <= y+ky-1, x+kx-1 < 2H:
//                 the GEMM runs at the INPUT resolution (a quarter of the rows the reference convolves)
//     f = leaky_relu_0.2(out + b[co]);  the next block's operand is its PixelNorm  f / sqrt(mean_c f^2 + 1e-8)
// The output block (PixelNorm, 1x1 conv to RGB, * 1/sqrt(c) + b) is fused behind the last block's epilogue.
//
// Layout: NHWC activations; between blocks they travel PixelNorm-ed (|x^| <= sqrt(c)) as fp16 hi/lo pairs.  The hooked block's
// activation is written as fp32 NHWC rows with a caller-given row stride.  Samples are processed in chunks whose tap planes
// fit the L2.  The per-pixel reductions over channels use warp shuffles and a fixed-order shared-memory step: a sample's
// result does not depend on the batch it is part of.
#include "tap_conv.cuh"
#include <math.h>

namespace gsb {

constexpr int PG_MAX_BLOCKS = 24;

static int pg_taps(const gsb_progan_block &c) { return c.ksize * c.ksize; }
static int pg_res_out(const gsb_progan_block &c) { return c.ksize == 4 ? 4 : (c.upsample ? 2 * c.res_in : c.res_in); }
// samples per chunk: the tap planes of one GEMM launch fit TAP_CHUNK_ELEMS
static int64_t pg_chunk_samples(const gsb_progan_block &c) {
    const int64_t per_sample = (int64_t)c.res_in * c.res_in * pg_taps(c) * c.cout;
    const int64_t spc = TAP_CHUNK_ELEMS / per_sample;
    return spc < 1 ? 1 : spc;
}

// ---- packed layout ----------------------------------------------------------------------------------------
struct PgBlockView {
    __half *w_hi, *w_lo;      // [taps*cout, cin]   row = tap*cout + co
    float *scal;              // [4]: inv_wscale, wscale, absmax
    float *bias;              // [cout]
};
struct PgView {
    unsigned *overflow;
    float *out_w;             // [3, c_last] * 1/sqrt(c_last)
    float *out_b;             // [3]
    PgBlockView L[PG_MAX_BLOCKS];
    size_t bytes;
};
static PgView pg_view(void *base, const gsb_progan_block *blocks, int n_blocks) {
    PgView v;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    v.overflow = (unsigned *)take(256);
    v.out_w = (float *)take((size_t)3 * blocks[n_blocks - 1].cout * 4);
    v.out_b = (float *)take(16);
    for (int l = 0; l < n_blocks; ++l) {
        const gsb_progan_block &c = blocks[l];
        const size_t wcount = (size_t)pg_taps(c) * c.cout * c.cin;
        v.L[l].w_hi = (__half *)take(wcount * 2);
        v.L[l].w_lo = (__half *)take(wcount * 2);
        v.L[l].scal = (float *)take(16);
        v.L[l].bias = (float *)take((size_t)c.cout * 4);
    }
    v.bytes = off;
    return v;
}

static int pg_check(const gsb_progan_block *blocks, int n_blocks) {
    GSB_CHECK_ARG(blocks && n_blocks >= 1 && n_blocks <= PG_MAX_BLOCKS, "progan: need 1..%d blocks", PG_MAX_BLOCKS);
    for (int l = 0; l < n_blocks; ++l) {
        const gsb_progan_block &c = blocks[l];
        GSB_CHECK_ARG(c.cin % 32 == 0 && c.cin >= 32 && c.cout >= 32 && c.cout <= 1024 && (c.cout & (c.cout - 1)) == 0,
                      "progan: block %d needs cin%%32==0 and cout a power of two in [32, 1024] (cin=%d cout=%d)", l, c.cin, c.cout);
        if (l == 0) GSB_CHECK_ARG(c.ksize == 4 && c.res_in == 1 && !c.upsample, "progan: block 0 is the 4x4 conv on the 1x1 latent");
        else GSB_CHECK_ARG(c.ksize == 3 && c.cin == blocks[l - 1].cout && c.res_in == pg_res_out(blocks[l - 1]) && c.res_in <= 1024,
                           "progan: block %d does not chain", l);
    }
    return GSB_OK;
}

// ---- forward kernels ------------------------------------------------------------------------------------
// PixelNorm of the latent (one warp per row) -> fp16 hi/lo operand of layer1
__global__ void __launch_bounds__(256)
pg_latent_norm_kernel(const float *__restrict__ z, int64_t n, int c, __half *__restrict__ hi, __half *__restrict__ lo, unsigned *overflow) {
    const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= n) return;
    const float *zr = z + row * c;
    float ss = 0.f;
    for (int k = 4 * lane; k < c; k += 128) {
        const float4 v = *reinterpret_cast<const float4 *>(zr + k);
        ss += (v.x * v.x + v.y * v.y) + (v.z * v.z + v.w * v.w);
    }
    ss = warp_sum(ss);
    const float den = sqrtf(ss / (float)c + 1e-8f);
    bool ovf = false;
    for (int k = 4 * lane; k < c; k += 128) {
        const float4 v = *reinterpret_cast<const float4 *>(zr + k);
        const float f[4] = {v.x / den, v.y / den, v.z / den, v.w / den};
        tc::store_split4(f, hi, lo, row * c + k, ovf);
    }
    if (ovf) atomicOr(overflow, 1u);
}

struct PgEpi {
    const float *bias;           // [c]
    __half *out_hi, *out_lo;     // [nb, hw, c] (chunk-local) PixelNorm-ed operand of the next block, or nullptr
    float *out_f32;              // hooked block: row b at out_f32 + b*ld, or nullptr
    int64_t ld;
    const float *rgb_w, *rgb_b;  // output block: [3, c] (scaled) and [3], or nullptr
    float *rgb_out;              // [nb, hw, 3] (chunk-local)
    unsigned *overflow;
};
// conv result (4 channels of one pixel) -> bias, leaky-ReLU -> the fp32 activation and / or the next block's PixelNorm-ed operand
// and / or the RGB pixel.  Threads past the end of the launch (`valid` false) take part in the reductions with zeros.
__device__ __forceinline__ void pg_epilogue(const PgEpi &e, float4 acc, bool valid, int64_t b, int pix, int hw, int c, int q) {
    float f[4] = {0.f, 0.f, 0.f, 0.f};
    if (valid) {
        const float4 bs = *reinterpret_cast<const float4 *>(e.bias + 4 * q);
        f[0] = acc.x + bs.x; f[1] = acc.y + bs.y; f[2] = acc.z + bs.z; f[3] = acc.w + bs.w;
#pragma unroll
        for (int k = 0; k < 4; ++k) f[k] = (f[k] >= 0.f) ? f[k] : 0.2f * f[k];
        if (e.out_f32) *reinterpret_cast<float4 *>(e.out_f32 + b * e.ld + (int64_t)pix * c + 4 * q) = make_float4(f[0], f[1], f[2], f[3]);
    }
    if (!e.out_hi && !e.rgb_w) return;
    const int cq = c >> 2;
    const float ss = pixel_sum((f[0] * f[0] + f[1] * f[1]) + (f[2] * f[2] + f[3] * f[3]), cq);
    const float den = sqrtf(ss / (float)c + 1e-8f);
    const float g[4] = {f[0] / den, f[1] / den, f[2] / den, f[3] / den};
    if (e.out_hi && valid) {
        bool ovf = false;
        tc::store_split4(g, e.out_hi, e.out_lo, (b * hw + pix) * (int64_t)c + 4 * q, ovf);
        if (ovf) atomicOr(e.overflow, 1u);
    }
    if (e.rgb_w) {
#pragma unroll
        for (int o = 0; o < 3; ++o) {
            const float4 wv = *reinterpret_cast<const float4 *>(e.rgb_w + (int64_t)o * c + 4 * q);
            const float r = pixel_sum((g[0] * wv.x + g[1] * wv.y) + (g[2] * wv.z + g[3] * wv.w), cq);
            if (valid && q == 0) e.rgb_out[(b * hw + pix) * 3 + o] = r + e.rgb_b[o];
        }
    }
}

// MODE 0: layer1 (Y is the 4x4 output); 1: stride-1 3x3 gather; 2: 3x3 on the nearest-x2 up-sampled input, Y at the input
// resolution R/2.  Y [nb * H * H, taps * c];  one thread per 4 channels of an output pixel
template <int MODE>
__global__ void __launch_bounds__(256)
pg_gather_kernel(const float *__restrict__ Y, int64_t nb, int R, int c, PgEpi e) {
    const int cq = c >> 2;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const bool valid = idx < nb * R * R * cq;
    const int q = (int)(idx % cq);
    const int64_t pixg = idx / cq;
    const int x = (int)(pixg % R), y = (int)((pixg / R) % R);
    const int64_t b = pixg / ((int64_t)R * R);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
    if (valid) {
        if (MODE == 0) acc = *reinterpret_cast<const float4 *>(Y + pixg * c + 4 * q);
        else acc = tap_sum3x3<MODE == 2>(Y, 9 * c, b, y, x, R, c, q);
    }
    pg_epilogue(e, acc, valid, b, y * R + x, R * R, c, q);
}

// ---- workspace --------------------------------------------------------------------------------------------
struct PgWs {
    __half *z[2];           // PixelNorm-ed latent, hi/lo
    __half *act[2][2];      // [ping-pong][hi/lo]
    float *Y;
    unsigned *queue;        // tile queue of the tap GEMM launches
    size_t bytes;
};
static PgWs pg_ws(void *base, const gsb_progan_block *blocks, int n_run, int64_t n) {
    PgWs w;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    size_t act_elems = 64, y_elems = 0;
    for (int l = 0; l < n_run; ++l) {
        const gsb_progan_block &c = blocks[l];
        const size_t ro = (size_t)pg_res_out(c);
        if (l + 1 < n_run) { const size_t e = (size_t)n * ro * ro * c.cout; act_elems = act_elems > e ? act_elems : e; }
        const int64_t spc = pg_chunk_samples(c) < n ? pg_chunk_samples(c) : n;
        const size_t ye = (size_t)spc * c.res_in * c.res_in * pg_taps(c) * c.cout;
        y_elems = y_elems > ye ? y_elems : ye;
    }
    for (int h = 0; h < 2; ++h) w.z[h] = (__half *)take((size_t)n * blocks[0].cin * 2);
    for (int a = 0; a < 2; ++a)
        for (int h = 0; h < 2; ++h) w.act[a][h] = (__half *)take(act_elems * 2);
    w.Y = (float *)take(y_elems * 4);
    w.queue = (unsigned *)take(sizeof(unsigned));
    w.bytes = off;
    return w;
}

}  // namespace gsb

extern "C" size_t gsb_progan_packed_bytes(const gsb_progan_block *blocks, int n_blocks) {
    if (gsb::pg_check(blocks, n_blocks)) return 0;
    return gsb::pg_view(nullptr, blocks, n_blocks).bytes;
}

extern "C" int gsb_progan_pack(const gsb_progan_block *blocks, int n_blocks, const float *d_out_weight, const float *d_out_bias,
                               void *d_packed, size_t packed_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (int r = pg_check(blocks, n_blocks)) return r;
    GSB_CHECK_ARG(d_out_weight && d_out_bias && d_packed, "progan_pack: null pointer");
    PgView v = pg_view(d_packed, blocks, n_blocks);
    if (packed_bytes < v.bytes) { set_error("progan_pack: buffer too small (%zu < %zu)", packed_bytes, v.bytes); return GSB_ERR_WORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CHECK_CUDA(cudaMemsetAsync(d_packed, 0, v.bytes, st));
    for (int l = 0; l < n_blocks; ++l) {
        const gsb_progan_block &c = blocks[l];
        GSB_CHECK_ARG(c.conv_weight && c.bias, "progan_pack: block %d has a null parameter pointer", l);
        // WScaleLayer.scale = gain / sqrt(fan_in), gain = sqrt2 / kernel_size, fan_in = in_channels (proggan.py:113,129-130)
        const float scale = (float)(sqrt(2.0) / c.ksize / sqrt((double)c.cin));
        const int taps = pg_taps(c);
        // layer1's taps are stored reversed (see the top of this file)
        if (int r = tc_split_weight(c.conv_weight, c.cout, c.cin, taps, scale, c.ksize == 4, taps * c.cout, v.L[l].w_hi, v.L[l].w_lo,
                                    v.L[l].scal, nullptr, st)) return r;
        scale_copy_kernel<<<4, 256, 0, st>>>(c.bias, c.cout, 1.0f, nullptr, v.L[l].bias);
        GSB_CHECK_LAUNCH();
    }
    const int cl = blocks[n_blocks - 1].cout;
    scale_copy_kernel<<<4, 256, 0, st>>>(d_out_weight, (int64_t)3 * cl, (float)(1.0 / sqrt((double)cl)), nullptr, v.out_w);   // gain 1 (proggan.py:163)
    GSB_CHECK_LAUNCH();
    scale_copy_kernel<<<1, 32, 0, st>>>(d_out_bias, 3, 1.0f, nullptr, v.out_b);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" size_t gsb_progan_workspace_bytes(const gsb_progan_block *blocks, int n_run, int64_t n) {
    if (!blocks || n_run < 1 || n_run > gsb::PG_MAX_BLOCKS || n < 1) return 0;
    return gsb::pg_ws(nullptr, blocks, n_run, n).bytes;
}

extern "C" int gsb_progan_forward(const void *d_packed, const gsb_progan_block *blocks, int n_blocks, int n_run, const float *d_z,
                                  int64_t n, float *d_act_out, int64_t ld_act, float *d_rgb_out, void *d_workspace,
                                  size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (int r = pg_check(blocks, n_blocks)) return r;
    GSB_CHECK_ARG(d_packed && d_z && d_workspace && (d_act_out || d_rgb_out), "progan: null pointer");
    GSB_CHECK_ARG(n_run >= 1 && n_run <= n_blocks && n >= 0, "progan: n_run / n out of range");
    GSB_CHECK_ARG(!d_rgb_out || n_run == n_blocks, "progan: the image needs every block (n_run == n_blocks)");
    if (n == 0) return GSB_OK;
    const gsb_progan_block &last = blocks[n_run - 1];
    const int ro_last = pg_res_out(last);
    GSB_CHECK_ARG(!d_act_out || (ld_act >= (int64_t)ro_last * ro_last * last.cout && ld_act % 4 == 0), "progan: bad ld_act");
    PgView v = pg_view(const_cast<void *>(d_packed), blocks, n_blocks);
    PgWs w = pg_ws(d_workspace, blocks, n_run, n);
    if (workspace_bytes < w.bytes) { set_error("progan: workspace too small (%zu < %zu)", workspace_bytes, w.bytes); return GSB_ERR_WORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;

    pg_latent_norm_kernel<<<(unsigned)((n + 7) / 8), 256, 0, st>>>(d_z, n, blocks[0].cin, w.z[0], w.z[1], v.overflow);
    GSB_CHECK_LAUNCH();
    for (int l = 0; l < n_run; ++l) {
        const gsb_progan_block &c = blocks[l];
        const int dst = l & 1;                                         // block l reads act[dst ^ 1] (block 0: the latent), writes act[dst]
        const __half *a_hi = l ? w.act[dst ^ 1][0] : w.z[0], *a_lo = l ? w.act[dst ^ 1][1] : w.z[1];
        const bool is_last = (l == n_run - 1);
        const int H = c.res_in, ro = pg_res_out(c), hw_in = H * H, hw_out = ro * ro, taps = pg_taps(c);
        const int64_t spc = pg_chunk_samples(c);
        for (int64_t b0 = 0; b0 < n; b0 += spc) {
            const int64_t nb = (b0 + spc <= n) ? spc : (n - b0);
            if (int r = tc_gemm_plain(a_hi + b0 * hw_in * c.cin, a_lo + b0 * hw_in * c.cin, nb * hw_in, c.cin, v.L[l].w_hi, v.L[l].w_lo,
                                      taps * c.cout, v.L[l].scal, w.Y, v.overflow, w.queue, 0, st)) return r;
            PgEpi e;
            e.bias = v.L[l].bias;
            e.out_hi = is_last ? nullptr : w.act[dst][0] + b0 * hw_out * c.cout;
            e.out_lo = is_last ? nullptr : w.act[dst][1] + b0 * hw_out * c.cout;
            e.out_f32 = (is_last && d_act_out) ? d_act_out + b0 * ld_act : nullptr;
            e.ld = ld_act;
            e.rgb_w = (is_last && d_rgb_out) ? v.out_w : nullptr;
            e.rgb_b = v.out_b;
            e.rgb_out = (is_last && d_rgb_out) ? d_rgb_out + b0 * hw_out * 3 : nullptr;
            e.overflow = v.overflow;
            const int64_t total = nb * hw_out * (c.cout / 4);
            const unsigned grid = (unsigned)((total + 255) / 256);
            if (l == 0) pg_gather_kernel<0><<<grid, 256, 0, st>>>(w.Y, nb, ro, c.cout, e);
            else if (c.upsample) pg_gather_kernel<2><<<grid, 256, 0, st>>>(w.Y, nb, ro, c.cout, e);
            else pg_gather_kernel<1><<<grid, 256, 0, st>>>(w.Y, nb, ro, c.cout, e);
            GSB_CHECK_LAUNCH();
        }
    }
    return GSB_OK;
}

extern "C" int gsb_progan_status(const void *d_packed, const gsb_progan_block *blocks, int n_blocks, unsigned *h_flags) {
    using namespace gsb;
    if (int r = pg_check(blocks, n_blocks)) return r;
    GSB_CHECK_ARG(d_packed && h_flags, "progan_status: null pointer");
    PgView v = pg_view(const_cast<void *>(d_packed), blocks, n_blocks);
    GSB_CHECK_CUDA(cudaMemcpy(h_flags, v.overflow, sizeof(unsigned), cudaMemcpyDeviceToHost));
    return GSB_OK;
}
