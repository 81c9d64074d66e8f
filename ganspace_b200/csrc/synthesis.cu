// StyleGAN2 synthesis blocks up to a hooked StyledConv (BASELINE config 5 family: layer = conv1 | convs.k).
//
// Replaces models/stylegan2/stylegan2-pytorch/model.py:181-277 (ModulatedConv2d), :280-291 (NoiseInjection),
// :294-304 (ConstantInput), :307-341 (StyledConv), op/fused_act.py:86-92 (FusedLeakyReLU), model.py:75-91 +
// op/upfirdn2d.py:144-198 (Blur after the stride-2 transposed conv), as driven by models/wrappers.py:224-255.
//
// The reference builds per-sample weights  w[b] = scale * W * s[b,ci] * demod[b,co]  ([B,co,ci,3,3] = 9.4 MB per
// sample and layer) and runs a grouped conv.  Here the SHARED weights are used:
//     xs[b,p,ci]      = x[b,p,ci] * s[b,ci]                               (modulation moved to the input)
//     Y[b,p,tap,co]   = sum_ci (scale W)[co,ci,tap] xs[b,p,ci]            one dense contraction, K = ci, N = 9 co
//                                                                        -> wgmma GEMM (mapping_tc.cu, fp16 hi/lo split)
//     stride 1 :  out[b,y,x,co] = sum_tap Y[b,(y+ky-1,x+kx-1),tap,co]
//     upsample :  T[b,u,v,co]   = sum_{tap: u-ky, v-kx even} Y[b,((u-ky)/2,(v-kx)/2),tap,co]      (2H+1 grid)
//                 out[b,y,x,co] = sum_{i,j<4} k[i]k[j]/16 * T[b,y+i-1,x+j-1,co],  k = [1,3,3,1]     (Blur, pad (1,1))
//     out = out * demod[b,co] + noise_w * noise[y,x] + bias[co];  out = sqrt2 * leaky_relu_0.2(out)
//     demod[b,co] = rsqrt( sum_ci s[b,ci]^2 * sum_tap (scale W)[co,ci,tap]^2 + 1e-8 )
// which is algebraically the reference's computation (oracle: styled_conv_taps == styled_conv_forward).
//
// Layout: activations are NHWC ([b, y, x, c]) so that the GEMM operand is K-major and the gathers are coalesced
// over channels; between layers they travel as fp16 hi/lo pairs already multiplied by the NEXT layer's style.
// The hooked layer's activation is written as fp32 NHWC rows of length res*res*co with a caller-given row stride
// (directly into the large-d IPCA batch buffer).  Samples are processed in chunks whose tap planes (Y) fit the L2.
#include "tap_conv.cuh"
#include <math.h>

namespace gsb {

constexpr int SY_MAX_LAYERS = 24;
constexpr int SY_MAX_RGB = SY_MAX_LAYERS / 2 + 1;
constexpr int SY_CHUNK_ROWS = 2048;       // GEMM rows per launch: 2048 x 9*512 fp32 tap planes = 38 MB (fits the 50 MB L2)

// ---- packed layout ----------------------------------------------------------------------------------------
struct SynthLayerView {
    __half *w_hi, *w_lo;      // [9*cout, cin]   row = tap*cout + co
    float *scal;              // [4]: inv_wscale, wscale, absmax
    float *wsq;               // [cout, cin]  sum_tap (scale W)^2
    float *modw;              // [cin, style_dim]  modulation.weight * (1/sqrt(style_dim))
    float *modb;              // [cin]
    float *actb;              // [cout]
    float *noise;             // [res_out^2]  noise_weight * noise
};
struct SynthRgbView {         // the ToRGB that follows layer 2j (cin = that layer's cout)
    float *modw;              // [cin, style_dim]  modulation.weight * (1/sqrt(style_dim))
    float *modb;              // [cin]
    float *convw;             // [3, cin]  conv.weight (unscaled)
    float *bias;              // [3]
};
struct SynthView {
    float *const_nhwc;        // [16, c0]
    float *zeros;             // [max channels]
    unsigned *overflow;
    SynthLayerView L[SY_MAX_LAYERS];
    SynthRgbView R[SY_MAX_RGB];
    size_t bytes;
};
static int res_out_of(const gsb_styled_conv &l) { return l.upsample ? 2 * l.res_in : l.res_in; }
static int rgbs_of(int n_layers) { return (n_layers + 1) / 2; }    // ToRGB j follows layer 2j

static SynthView synth_view(void *base, const gsb_styled_conv *layers, int n_layers, int style_dim) {
    SynthView v;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    int cmax = 0;
    for (int l = 0; l < n_layers; ++l) { cmax = cmax > layers[l].cin ? cmax : layers[l].cin; cmax = cmax > layers[l].cout ? cmax : layers[l].cout; }
    v.const_nhwc = (float *)take((size_t)16 * (n_layers ? layers[0].cin : 0) * 4);
    v.zeros = (float *)take((size_t)cmax * 4);
    v.overflow = (unsigned *)take(256);
    for (int l = 0; l < n_layers; ++l) {
        const gsb_styled_conv &c = layers[l];
        const int ro = res_out_of(c);
        v.L[l].w_hi = (__half *)take((size_t)9 * c.cout * c.cin * 2);
        v.L[l].w_lo = (__half *)take((size_t)9 * c.cout * c.cin * 2);
        v.L[l].scal = (float *)take(16);
        v.L[l].wsq = (float *)take((size_t)c.cout * c.cin * 4);
        v.L[l].modw = (float *)take((size_t)c.cin * style_dim * 4);
        v.L[l].modb = (float *)take((size_t)c.cin * 4);
        v.L[l].actb = (float *)take((size_t)c.cout * 4);
        v.L[l].noise = (float *)take((size_t)ro * ro * 4);
    }
    for (int j = 0; j < rgbs_of(n_layers); ++j) {
        const size_t cin = layers[2 * j].cout;
        v.R[j].modw = (float *)take(cin * style_dim * 4);
        v.R[j].modb = (float *)take(cin * 4);
        v.R[j].convw = (float *)take(3 * cin * 4);
        v.R[j].bias = (float *)take(3 * 4);
    }
    v.bytes = off;
    return v;
}

static int check_layers(const gsb_styled_conv *layers, int n_layers, int style_dim) {
    GSB_CHECK_ARG(layers && n_layers >= 1 && n_layers <= SY_MAX_LAYERS, "synthesis: need 1..%d layers", SY_MAX_LAYERS);
    GSB_CHECK_ARG(style_dim > 0 && style_dim % 16 == 0, "synthesis: style_dim %% 16");
    for (int l = 0; l < n_layers; ++l) {
        const gsb_styled_conv &c = layers[l];
        GSB_CHECK_ARG(c.cin % 32 == 0 && c.cout % 32 == 0 && c.cin >= 32 && c.cout >= 32,
                      "synthesis: layer %d needs cin%%32==0, cout%%32==0 (cin=%d cout=%d)", l, c.cin, c.cout);
        GSB_CHECK_ARG(c.res_in >= 4 && c.res_in <= 1024, "synthesis: layer %d bad res_in", l);
        if (l == 0) GSB_CHECK_ARG(c.res_in == 4 && !c.upsample, "synthesis: layer 0 is conv1 on the 4x4 constant");
        else GSB_CHECK_ARG(c.cin == layers[l - 1].cout && c.res_in == res_out_of(layers[l - 1]), "synthesis: layer %d does not chain", l);
    }
    return GSB_OK;
}

// ---- forward kernels ------------------------------------------------------------------------------------
__global__ void sy_square_kernel(const float *__restrict__ x, int64_t count, float *__restrict__ y) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < count) { const float v = x[i]; y[i] = v * v; }
}
__global__ void sy_rsqrt_eps_kernel(float *__restrict__ x, int64_t count) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i < count) x[i] = 1.0f / sqrtf(x[i] + 1e-8f);
}

// ConstantInput (model.py:300-304) times the first layer's style: out[b,p,c] = const[p,c] * s[b,c]  -> hi/lo
__global__ void sy_const_modulate_kernel(const float *__restrict__ cst, const float *__restrict__ s, int64_t n, int hw, int c,
                                         __half *__restrict__ hi, __half *__restrict__ lo, unsigned *overflow) {
    const int cq = c >> 2;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= n * hw * cq) return;
    const int q = (int)(idx % cq);
    const int64_t pix = idx / cq;
    const int p = (int)(pix % hw);
    const int64_t b = pix / hw;
    const float4 cv = *reinterpret_cast<const float4 *>(cst + (int64_t)p * c + 4 * q);
    const float4 sv = *reinterpret_cast<const float4 *>(s + b * c + 4 * q);
    const float f[4] = {cv.x * sv.x, cv.y * sv.y, cv.z * sv.z, cv.w * sv.w};
    bool ovf = false;
    tc::store_split4(f, hi, lo, pix * c + 4 * q, ovf);
    if (ovf) atomicOr(overflow, 1u);
}

// y[n, N] = x[n, K] W[N, K]^T + bias: one thread per output, for the style / demodulation products of blocks whose channel
// count is below the GEMM kernels' 128-wide tiles (64- and 32-channel blocks at 512^2 / 1024^2)
__global__ void sy_small_linear_kernel(const float *__restrict__ x, const float *__restrict__ w, const float *__restrict__ bias,
                                       float *__restrict__ y, int64_t n, int N, int K) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= n * N) return;
    const int j = (int)(idx % N);
    const int64_t r = idx / N;
    const float *xr = x + r * K, *wr = w + (int64_t)j * K;
    float a0 = 0.f, a1 = 0.f, a2 = 0.f, a3 = 0.f;
    int k = 0;
    for (; k + 3 < K; k += 4) {
        const float4 xv = *reinterpret_cast<const float4 *>(xr + k), wv = *reinterpret_cast<const float4 *>(wr + k);
        a0 = fmaf(xv.x, wv.x, a0); a1 = fmaf(xv.y, wv.y, a1); a2 = fmaf(xv.z, wv.z, a2); a3 = fmaf(xv.w, wv.w, a3);
    }
    for (; k < K; ++k) a0 = fmaf(xr[k], wr[k], a0);
    y[idx] = (a0 + a1) + (a2 + a3) + bias[j];
}
static int sy_linear(const float *x, const float *w, const float *bias, float *y, int64_t n, int N, int K, gsb_stream_t stream) {
    if (N % 128 == 0 && K % 16 == 0) return gsb_linear_forward(x, w, bias, y, n, N, K, 0, nullptr, 0, stream);
    const int64_t total = n * N;
    sy_small_linear_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(x, w, bias, y, n, N, K);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

struct EpiParams {
    const float *demod;     // [nb, c]  (chunk-local rows)
    const float *noise;     // [H*W] pre-multiplied by NoiseInjection.weight
    const float *bias;      // [c]
    const float *s_next;    // [nb, c] next layer's style, or nullptr on the hooked layer
    __half *out_hi, *out_lo;   // [nb, H*W, c] (chunk-local)
    float *out_f32;         // hooked layer: row b at out_f32 + b*ld
    int64_t ld;
    unsigned *overflow;
    // ToRGB of this resolution (model.py:344-363), fused: rgb[b,pix,o] += sum_c (scale W)[o,c] s_rgb[b,c] f[b,pix,c]
    const float *rgb_w;     // [3, c] ToRGB.conv.weight (unscaled), or nullptr
    const float *rgb_s;     // [nb, c] ToRGB style (chunk-local rows)
    float *rgb_out;         // [nb, H*W, 3] (chunk-local), pre-initialised with bias + up-sampled skip
    float rgb_scale;        // 1 / sqrt(c)
};
// conv result (4 channels) -> demod, noise, bias, leaky-ReLU * sqrt2 -> next layer's operand or the fp32 activation
__device__ __forceinline__ void sy_epilogue(const EpiParams &e, float4 acc, int64_t b, int pix, int hw, int c, int q) {
    const float4 dm = *reinterpret_cast<const float4 *>(e.demod + b * c + 4 * q);
    const float4 bs = *reinterpret_cast<const float4 *>(e.bias + 4 * q);
    const float nz = e.noise[pix];
    float f[4] = {fmaf(acc.x, dm.x, nz) + bs.x, fmaf(acc.y, dm.y, nz) + bs.y, fmaf(acc.z, dm.z, nz) + bs.z,
                  fmaf(acc.w, dm.w, nz) + bs.w};
    const float sqrt2 = 1.41421356237309515f;
#pragma unroll
    for (int k = 0; k < 4; ++k) f[k] = sqrt2 * ((f[k] >= 0.f) ? f[k] : 0.2f * f[k]);
    if (e.rgb_w) {
        // the channel quads of one pixel sit in consecutive lanes (c/4 of them, a power of two; >= 32: whole warps)
        const float4 sr = *reinterpret_cast<const float4 *>(e.rgb_s + b * c + 4 * q);
        const float g[4] = {f[0] * sr.x, f[1] * sr.y, f[2] * sr.z, f[3] * sr.w};
        float r[3];
#pragma unroll
        for (int o = 0; o < 3; ++o) {
            const float4 wv = *reinterpret_cast<const float4 *>(e.rgb_w + (int64_t)o * c + 4 * q);
            r[o] = e.rgb_scale * (g[0] * wv.x + g[1] * wv.y + g[2] * wv.z + g[3] * wv.w);
        }
        const int cq = c >> 2, span = cq < 32 ? cq : 32;
        for (int off = span >> 1; off > 0; off >>= 1) {
#pragma unroll
            for (int o = 0; o < 3; ++o) r[o] += __shfl_xor_sync(0xffffffffu, r[o], off);
        }
        float *dst = e.rgb_out + (b * hw + pix) * 3;
        if (cq <= 32) {
            // one lane per pixel holds the sum: a plain read-modify-write, deterministic
            if ((q & (span - 1)) == 0) { dst[0] += r[0]; dst[1] += r[1]; dst[2] += r[2]; }
        } else {
            // 256 / 512 channels: the pixel's quads span 2 / 4 warps of this block (blocks hold whole pixels: 256 % cq == 0 and
            // the launch has no partial blocks); combine them through shared memory in a fixed order
            __shared__ float rgb_red[8][3];
            const int wib = threadIdx.x >> 5, wpp = cq >> 5;                    // warp in block, warps per pixel
            if ((threadIdx.x & 31) == 0) { rgb_red[wib][0] = r[0]; rgb_red[wib][1] = r[1]; rgb_red[wib][2] = r[2]; }
            __syncthreads();
            if ((threadIdx.x & 31) == 0 && (wib % wpp) == 0) {
                float t0 = 0.f, t1 = 0.f, t2 = 0.f;
                for (int k = 0; k < wpp; ++k) { t0 += rgb_red[wib + k][0]; t1 += rgb_red[wib + k][1]; t2 += rgb_red[wib + k][2]; }
                dst[0] += t0; dst[1] += t1; dst[2] += t2;
            }
            __syncthreads();
        }
    }
    if (e.s_next) {
        const float4 sn = *reinterpret_cast<const float4 *>(e.s_next + b * c + 4 * q);
        f[0] *= sn.x; f[1] *= sn.y; f[2] *= sn.z; f[3] *= sn.w;
        bool ovf = false;
        tc::store_split4(f, e.out_hi, e.out_lo, (b * hw + pix) * (int64_t)c + 4 * q, ovf);
        if (ovf) atomicOr(e.overflow, 1u);
    } else if (e.out_f32) {
        *reinterpret_cast<float4 *>(e.out_f32 + b * e.ld + (int64_t)pix * c + 4 * q) = make_float4(f[0], f[1], f[2], f[3]);
    }
}

// rgb[b, y, x, o] = bias[o] (+ Upsample(prev)[b, y, x, o]):  upfirdn2d(prev, [1,3,3,1] outer * 4 / 64, up = 2, pad = (2, 1))
// (model.py:33-51, op/upfirdn2d.py:157-198): zero-insertion puts prev[i] at 2i; out[y] = sum_i k[i] up[y + i - 2].
__global__ void sy_rgb_init_kernel(const float *__restrict__ bias, const float *__restrict__ prev, int64_t n, int R, float *__restrict__ rgb) {
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= n * R * R) return;
    const int x = (int)(idx % R), y = (int)((idx / R) % R);
    const int64_t b = idx / ((int64_t)R * R);
    float acc[3] = {bias[0], bias[1], bias[2]};
    if (prev) {
        const int Rp = R >> 1;
        const float k1[4] = {1.f, 3.f, 3.f, 1.f};
#pragma unroll
        for (int i = 0; i < 4; ++i) {
            const int u = y + i - 2;
            if (u < 0 || (u & 1) || (u >> 1) >= Rp) continue;
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const int v = x + j - 2;
                if (v < 0 || (v & 1) || (v >> 1) >= Rp) continue;
                const float kw = k1[i] * k1[j] * 0.0625f;
                const float *pp = prev + ((b * Rp + (u >> 1)) * Rp + (v >> 1)) * 3;
                acc[0] = fmaf(kw, pp[0], acc[0]); acc[1] = fmaf(kw, pp[1], acc[1]); acc[2] = fmaf(kw, pp[2], acc[2]);
            }
        }
    }
    float *o = rgb + idx * 3;
    o[0] = acc[0]; o[1] = acc[1]; o[2] = acc[2];
}

// stride-1 3x3: gather the nine tap planes.  Y [nb*R*R, 9*c]
__global__ void __launch_bounds__(256)
sy_conv_gather_kernel(const float *__restrict__ Y, int64_t nb, int R, int c, EpiParams e) {
    const int cq = c >> 2;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= nb * R * R * cq) return;
    const int q = (int)(idx % cq);
    const int64_t pixg = idx / cq;
    const int x = (int)(pixg % R), y = (int)((pixg / R) % R);
    const int64_t b = pixg / ((int64_t)R * R);
    sy_epilogue(e, tap_sum3x3<false>(Y, 9 * c, b, y, x, R, c, q), b, y * R + x, R * R, c, q);
}

// stride-2 transposed conv: T[b,u,v,:] on the (2H+1) x (2W+1) grid = sum of the tap planes that land on (u,v)
__global__ void __launch_bounds__(256)
sy_upconv_scatter_kernel(const float *__restrict__ Y, int64_t nb, int H, int W, int c, float *__restrict__ T) {
    const int cq = c >> 2, TH = 2 * H + 1, TW = 2 * W + 1;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= nb * TH * TW * cq) return;
    const int q = (int)(idx % cq);
    const int64_t pixg = idx / cq;
    const int v = (int)(pixg % TW), u = (int)((pixg / TW) % TH);
    const int64_t b = pixg / ((int64_t)TW * TH);
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int t = u - ky;
        if (t < 0 || (t & 1) || (t >> 1) >= H) continue;
        const int yy = t >> 1;
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int s = v - kx;
            if (s < 0 || (s & 1) || (s >> 1) >= W) continue;
            const int xx = s >> 1;
            const float4 w = *reinterpret_cast<const float4 *>(Y + ((b * H + yy) * W + xx) * (int64_t)(9 * c) + (ky * 3 + kx) * c + 4 * q);
            acc.x += w.x; acc.y += w.y; acc.z += w.z; acc.w += w.w;
        }
    }
    *reinterpret_cast<float4 *>(T + pixg * c + 4 * q) = acc;
}

// Blur([1,3,3,1] outer / 64 * 4, pad (1,1)) of T -> 2H x 2W, then the shared epilogue
__global__ void __launch_bounds__(256)
sy_blur_epilogue_kernel(const float *__restrict__ T, int64_t nb, int H2, int W2, int c, EpiParams e) {
    const int cq = c >> 2, TH = H2 + 1, TW = W2 + 1;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= nb * H2 * W2 * cq) return;
    const int q = (int)(idx % cq);
    const int64_t pixg = idx / cq;
    const int x = (int)(pixg % W2), y = (int)((pixg / W2) % H2);
    const int64_t b = pixg / ((int64_t)W2 * H2);
    const float k1[4] = {1.f, 3.f, 3.f, 1.f};
    float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
    for (int i = 0; i < 4; ++i) {
        const int u = y + i - 1;
        if (u < 0 || u >= TH) continue;
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const int v = x + j - 1;
            if (v < 0 || v >= TW) continue;
            const float kw = k1[i] * k1[j] * 0.0625f;
            const float4 t = *reinterpret_cast<const float4 *>(T + ((b * TH + u) * TW + v) * (int64_t)c + 4 * q);
            acc.x = fmaf(kw, t.x, acc.x); acc.y = fmaf(kw, t.y, acc.y); acc.z = fmaf(kw, t.z, acc.z); acc.w = fmaf(kw, t.w, acc.w);
        }
    }
    sy_epilogue(e, acc, b, y * W2 + x, H2 * W2, c, q);
}

// ---- workspace --------------------------------------------------------------------------------------------
struct SynthWs {
    float *S[SY_MAX_LAYERS], *D[SY_MAX_LAYERS];
    float *s2;
    __half *act[2][2];     // [ping-pong][hi/lo]
    float *Y, *T;
    unsigned *queue;        // tile queue of the tap GEMM launches
    float *rgb[2];          // with ToRGBs: skip images (ping-pong)
    float *rgb_s[SY_MAX_RGB];   // with the style stage: ToRGB styles
    size_t bytes;
};
static int chunk_samples(const gsb_styled_conv &c) {
    int spc = SY_CHUNK_ROWS / (c.res_in * c.res_in);
    return spc < 1 ? 1 : spc;
}
// own_styles: the workspace also holds the styles S[l] and rgb_s[j] (j < n_rgb) that the style stage writes; without it the caller
// passes them (gsb_synthesis_forward_styled)
static SynthWs synth_ws(void *base, const gsb_styled_conv *layers, int n_run, int n_rgb, int64_t n, bool own_styles) {
    SynthWs w;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    size_t cmax = 0, act_elems = 0, y_elems = 0, t_elems = 0;
    for (int l = 0; l < n_run; ++l) {
        const gsb_styled_conv &c = layers[l];
        w.S[l] = own_styles ? (float *)take((size_t)n * c.cin * 4) : nullptr;
        w.D[l] = (float *)take((size_t)n * c.cout * 4);
        cmax = cmax > (size_t)c.cin ? cmax : (size_t)c.cin;
        const size_t in_elems = (size_t)n * c.res_in * c.res_in * c.cin;
        act_elems = act_elems > in_elems ? act_elems : in_elems;
        const size_t spc = (size_t)chunk_samples(c);
        const size_t ye = spc * c.res_in * c.res_in * 9 * c.cout;
        y_elems = y_elems > ye ? y_elems : ye;
        if (c.upsample) {
            const size_t te = spc * (2 * c.res_in + 1) * (2 * c.res_in + 1) * c.cout;
            t_elems = t_elems > te ? t_elems : te;
        }
    }
    w.s2 = (float *)take((size_t)n * cmax * 4);
    for (int a = 0; a < 2; ++a)
        for (int h = 0; h < 2; ++h) w.act[a][h] = (__half *)take(act_elems * 2);
    w.Y = (float *)take(y_elems * 4);
    w.T = (float *)take((t_elems ? t_elems : 64) * 4);
    w.queue = (unsigned *)take(sizeof(unsigned));
    w.rgb[0] = w.rgb[1] = nullptr;
    for (int j = 0; j < SY_MAX_RGB; ++j) w.rgb_s[j] = nullptr;
    if (n_rgb > 0) {
        const int ro = res_out_of(layers[n_run - 1]);
        for (int a = 0; a < 2; ++a) w.rgb[a] = (float *)take((size_t)n * ro * ro * 3 * 4);
        for (int j = 0; own_styles && j < n_rgb; ++j) w.rgb_s[j] = (float *)take((size_t)n * layers[2 * j].cout * 4);
    }
    w.bytes = off;
    return w;
}

// ToRGB j follows layer 2j of layers[0..n_following): its cin is that layer's cout, a power of two (the epilogue's lane reduction)
static int check_rgbs(const gsb_styled_conv *layers, int n_following, const gsb_to_rgb *rgbs) {
    GSB_CHECK_ARG(rgbs, "synthesis: null ToRGB list");
    for (int j = 0; j < rgbs_of(n_following); ++j) {
        const gsb_to_rgb &t = rgbs[j];
        const int c = layers[2 * j].cout;
        GSB_CHECK_ARG(t.conv_weight && t.bias && t.mod_weight && t.mod_bias && t.cin == c && (c & (c - 1)) == 0,
                      "synthesis: ToRGB %d does not match layer %d (cin=%d, cout=%d)", j, 2 * j, t.cin, c);
    }
    return GSB_OK;
}
static bool aligned16(const void *p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

}  // namespace gsb

extern "C" size_t gsb_synthesis_packed_bytes(const gsb_styled_conv *layers, int n_layers, int style_dim) {
    if (gsb::check_layers(layers, n_layers, style_dim)) return 0;
    return gsb::synth_view(nullptr, layers, n_layers, style_dim).bytes;
}

extern "C" int gsb_synthesis_pack(const gsb_styled_conv *layers, int n_layers, int style_dim, const gsb_to_rgb *rgbs,
                                  const float *d_const_input, void *d_packed, size_t packed_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (int r = check_layers(layers, n_layers, style_dim)) return r;
    if (int r = check_rgbs(layers, n_layers, rgbs)) return r;
    GSB_CHECK_ARG(d_const_input && d_packed, "synthesis_pack: null pointer");
    SynthView v = synth_view(d_packed, layers, n_layers, style_dim);
    if (packed_bytes < v.bytes) { set_error("synthesis_pack: buffer too small (%zu < %zu)", packed_bytes, v.bytes); return GSB_ERR_WORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CHECK_CUDA(cudaMemsetAsync(d_packed, 0, v.bytes, st));
    const int c0 = layers[0].cin;
    const_nhwc_kernel<<<8, 256, 0, st>>>(d_const_input, c0, v.const_nhwc);
    GSB_CHECK_LAUNCH();
    const float mscale = (float)(1.0 / sqrt((double)style_dim));                  // EqualLinear.scale, lr_mul = 1 (model.py:143)
    for (int l = 0; l < n_layers; ++l) {
        const gsb_styled_conv &c = layers[l];
        GSB_CHECK_ARG(c.conv_weight && c.mod_weight && c.mod_bias && c.act_bias && c.noise && c.noise_weight,
                      "synthesis_pack: layer %d has a null parameter pointer", l);
        const float scale = (float)(1.0 / sqrt((double)c.cin * 9.0));           // ModulatedConv2d.scale (model.py:219-220)
        if (int r = tc_split_weight(c.conv_weight, c.cout, c.cin, 9, scale, false, 9 * c.cout, v.L[l].w_hi, v.L[l].w_lo, v.L[l].scal,
                                    v.L[l].wsq, st)) return r;
        scale_copy_kernel<<<128, 256, 0, st>>>(c.mod_weight, (int64_t)c.cin * style_dim, mscale, nullptr, v.L[l].modw);
        GSB_CHECK_LAUNCH();
        scale_copy_kernel<<<4, 256, 0, st>>>(c.mod_bias, c.cin, 1.0f, nullptr, v.L[l].modb);
        GSB_CHECK_LAUNCH();
        scale_copy_kernel<<<4, 256, 0, st>>>(c.act_bias, c.cout, 1.0f, nullptr, v.L[l].actb);
        GSB_CHECK_LAUNCH();
        const int ro = res_out_of(c);
        scale_copy_kernel<<<64, 256, 0, st>>>(c.noise, (int64_t)ro * ro, 1.0f, c.noise_weight, v.L[l].noise);
        GSB_CHECK_LAUNCH();
    }
    for (int j = 0; j < rgbs_of(n_layers); ++j) {
        const gsb_to_rgb &t = rgbs[j];
        scale_copy_kernel<<<64, 256, 0, st>>>(t.mod_weight, (int64_t)t.cin * style_dim, mscale, nullptr, v.R[j].modw);
        GSB_CHECK_LAUNCH();
        scale_copy_kernel<<<4, 256, 0, st>>>(t.mod_bias, t.cin, 1.0f, nullptr, v.R[j].modb);
        GSB_CHECK_LAUNCH();
        scale_copy_kernel<<<4, 256, 0, st>>>(t.conv_weight, 3 * t.cin, 1.0f, nullptr, v.R[j].convw);
        GSB_CHECK_LAUNCH();
        scale_copy_kernel<<<1, 32, 0, st>>>(t.bias, 3, 1.0f, nullptr, v.R[j].bias);
        GSB_CHECK_LAUNCH();
    }
    return GSB_OK;
}

extern "C" size_t gsb_synthesis_workspace_bytes(const gsb_styled_conv *layers, int n_run, int n_rgb, int64_t n) {
    if (!layers || n_run < 1 || n_run > gsb::SY_MAX_LAYERS || n < 1) return 0;
    return gsb::synth_ws(nullptr, layers, n_run, n_rgb, n, true).bytes;
}

namespace gsb {

// run stage: layers[0 .. n_run) on the styles S[l] [n, cin_l]; optional fp32 activation of the last layer (d_out), optional ToRGB
// chain: ToRGB j < n_rgb follows layer 2j with style rgb_s[j] [n, cin_j].  The demodulation factors are derived from S here
// (model.py:239).
static int synthesis_run(const SynthView &v, const gsb_styled_conv *layers, int n_run, int n_rgb, const float *const *S,
                         const float *const *rgb_s, int64_t n, float *d_out, int64_t ld_out, float *d_rgb_out, const SynthWs &w,
                         gsb_stream_t stream) {
    cudaStream_t st = (cudaStream_t)stream;
    for (int l = 0; l < n_run; ++l) {
        const gsb_styled_conv &c = layers[l];
        const int64_t cnt = n * c.cin;
        sy_square_kernel<<<(unsigned)((cnt + 255) / 256), 256, 0, st>>>(S[l], cnt, w.s2);
        GSB_CHECK_LAUNCH();
        if (int r = sy_linear(w.s2, v.L[l].wsq, v.zeros, w.D[l], n, c.cout, c.cin, stream)) return r;
        const int64_t cnt2 = n * c.cout;
        sy_rsqrt_eps_kernel<<<(unsigned)((cnt2 + 255) / 256), 256, 0, st>>>(w.D[l], cnt2);
        GSB_CHECK_LAUNCH();
    }
    {   // ConstantInput * style of conv1
        const int64_t total = n * 16 * (layers[0].cin / 4);
        sy_const_modulate_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(v.const_nhwc, S[0], n, 16, layers[0].cin, w.act[0][0],
                                                                                w.act[0][1], v.overflow);
        GSB_CHECK_LAUNCH();
    }
    const float *rgb_prev = nullptr;
    for (int l = 0; l < n_run; ++l) {
        const gsb_styled_conv &c = layers[l];
        const int src = l & 1, dst = src ^ 1;
        const bool hooked = (l == n_run - 1);
        const int H = c.res_in, ro = res_out_of(c), hw_in = H * H, hw_out = ro * ro;
        const int spc = chunk_samples(c);
        // ToRGB after conv1 and after the second conv of every resolution (model.py:546-561)
        const int j = l / 2;
        const bool with_rgb = (l % 2 == 0) && j < n_rgb;
        float *rgb_cur = nullptr;
        if (with_rgb) {
            rgb_cur = (j == n_rgb - 1) ? d_rgb_out : w.rgb[j & 1];
            const int64_t tot = n * hw_out;
            sy_rgb_init_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(v.R[j].bias, rgb_prev, n, ro, rgb_cur);
            GSB_CHECK_LAUNCH();
        }
        for (int64_t b0 = 0; b0 < n; b0 += spc) {
            const int64_t nb = (b0 + spc <= n) ? spc : (n - b0);
            const int64_t rows = nb * hw_in;
            if (int r = tc_gemm_plain(w.act[src][0] + b0 * hw_in * c.cin, w.act[src][1] + b0 * hw_in * c.cin, rows, c.cin, v.L[l].w_hi,
                                      v.L[l].w_lo, 9 * c.cout, v.L[l].scal, w.Y, v.overflow, w.queue, 0, st)) return r;
            EpiParams e;
            e.demod = w.D[l] + b0 * c.cout;
            e.noise = v.L[l].noise;
            e.bias = v.L[l].actb;
            e.s_next = hooked ? nullptr : S[l + 1] + b0 * c.cout;
            e.out_hi = hooked ? nullptr : w.act[dst][0] + b0 * hw_out * c.cout;
            e.out_lo = hooked ? nullptr : w.act[dst][1] + b0 * hw_out * c.cout;
            e.out_f32 = (hooked && d_out) ? d_out + b0 * ld_out : nullptr;
            e.ld = ld_out;
            e.overflow = v.overflow;
            e.rgb_w = with_rgb ? v.R[j].convw : nullptr;
            e.rgb_s = with_rgb ? rgb_s[j] + b0 * c.cout : nullptr;
            e.rgb_out = with_rgb ? rgb_cur + b0 * hw_out * 3 : nullptr;
            e.rgb_scale = (float)(1.0 / sqrt((double)c.cout));
            const int cq = c.cout / 4;
            if (c.upsample) {
                const int64_t t_total = nb * (2 * H + 1) * (2 * H + 1) * cq;
                sy_upconv_scatter_kernel<<<(unsigned)((t_total + 255) / 256), 256, 0, st>>>(w.Y, nb, H, H, c.cout, w.T);
                GSB_CHECK_LAUNCH();
                const int64_t o_total = nb * hw_out * cq;
                sy_blur_epilogue_kernel<<<(unsigned)((o_total + 255) / 256), 256, 0, st>>>(w.T, nb, ro, ro, c.cout, e);
                GSB_CHECK_LAUNCH();
            } else {
                const int64_t o_total = nb * hw_out * cq;
                sy_conv_gather_kernel<<<(unsigned)((o_total + 255) / 256), 256, 0, st>>>(w.Y, nb, H, c.cout, e);
                GSB_CHECK_LAUNCH();
            }
        }
        if (with_rgb) rgb_prev = rgb_cur;
    }
    return GSB_OK;
}

// argument checks shared by the two chain entries; *w receives the workspace layout
static int check_run(const void *d_packed, const gsb_styled_conv *layers, int n_layers, int n_run, int n_rgb, int style_dim, int64_t n,
                     float *d_out, int64_t ld_out, float *d_rgb_out, void *d_workspace, size_t workspace_bytes, bool own_styles,
                     SynthWs *w) {
    if (int r = check_layers(layers, n_layers, style_dim)) return r;
    GSB_CHECK_ARG(d_packed && d_workspace && (d_out || d_rgb_out), "synthesis: null pointer");
    GSB_CHECK_ARG(n_run >= 1 && n_run <= n_layers, "synthesis: n_run out of range");
    GSB_CHECK_ARG(n_rgb >= 0 && n_rgb <= rgbs_of(n_run), "synthesis: ToRGB %d has no layer %d to follow", n_rgb - 1, 2 * (n_rgb - 1));
    GSB_CHECK_ARG(n_rgb == 0 || d_rgb_out, "synthesis: ToRGBs without an image output");
    GSB_CHECK_ARG(n >= 0, "synthesis: bad n");
    if (n == 0) return GSB_OK;
    const gsb_styled_conv &last = layers[n_run - 1];
    const int ro_last = res_out_of(last);
    GSB_CHECK_ARG(!d_out || (ld_out >= (int64_t)ro_last * ro_last * last.cout && ld_out % 4 == 0), "synthesis: bad n / ld_out");
    *w = synth_ws(d_workspace, layers, n_run, n_rgb, n, own_styles);
    if (workspace_bytes < w->bytes) { set_error("synthesis: workspace too small (%zu < %zu)", workspace_bytes, w->bytes); return GSB_ERR_WORKSPACE; }
    return GSB_OK;
}

// style stage (model.py:226,234): s = w modw^T + modb with the modulation weight scaled at pack time.  Layer l reads latent entry
// min(l, w_layers - 1), ToRGB j entry min(2j + 1, w_layers - 1); a NULL S[l] / rgb_s[j] (or array) skips that style.
static int style_stage(const SynthView &v, const gsb_styled_conv *layers, int n_conv, int n_rgb, int style_dim, const float *d_w,
                       int w_layers, int64_t n, float *const *S, float *const *rgb_s, gsb_stream_t stream) {
    auto latent = [&](int idx) { return d_w + (size_t)(idx < w_layers ? idx : w_layers - 1) * n * style_dim; };
    for (int l = 0; S && l < n_conv; ++l)
        if (S[l])
            if (int r = sy_linear(latent(l), v.L[l].modw, v.L[l].modb, S[l], n, layers[l].cin, style_dim, stream)) return r;
    for (int j = 0; rgb_s && j < n_rgb; ++j)
        if (rgb_s[j])
            if (int r = sy_linear(latent(2 * j + 1), v.R[j].modw, v.R[j].modb, rgb_s[j], n, layers[2 * j].cout, style_dim, stream))
                return r;
    return GSB_OK;
}

}  // namespace gsb

// Generator.forward (model.py:493-571) up to layer n_run-1 and ToRGB n_rgb-1: the style stage into the workspace, then the run stage
extern "C" int gsb_synthesis_forward(const void *d_packed, const gsb_styled_conv *layers, int n_layers, int n_run, int n_rgb,
                                     int style_dim, const float *d_w, int w_layers, int64_t n, float *d_act_out, int64_t ld_act,
                                     float *d_rgb_out, void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_w && w_layers >= 1, "synthesis: no latents");
    SynthWs w;
    if (int r = check_run(d_packed, layers, n_layers, n_run, n_rgb, style_dim, n, d_act_out, ld_act, d_rgb_out, d_workspace,
                          workspace_bytes, true, &w)) return r;
    if (n == 0) return GSB_OK;
    const SynthView v = synth_view(const_cast<void *>(d_packed), layers, n_layers, style_dim);
    if (int r = style_stage(v, layers, n_run, n_rgb, style_dim, d_w, w_layers, n, w.S, w.rgb_s, stream)) return r;
    return synthesis_run(v, layers, n_run, n_rgb, w.S, w.rgb_s, n, d_act_out, ld_act, d_rgb_out, w, stream);
}

extern "C" int gsb_synthesis_styles(const void *d_packed, const gsb_styled_conv *layers, int n_layers, int style_dim, const float *d_w,
                                    int w_layers, int64_t n, float *const *d_S, float *const *d_rgb_s, gsb_stream_t stream) {
    using namespace gsb;
    if (int r = check_layers(layers, n_layers, style_dim)) return r;
    GSB_CHECK_ARG(d_packed && d_w && w_layers >= 1 && n >= 0, "synthesis_styles: null pointer or bad n");
    if (n == 0) return GSB_OK;
    const SynthView v = synth_view(const_cast<void *>(d_packed), layers, n_layers, style_dim);
    return style_stage(v, layers, n_layers, rgbs_of(n_layers), style_dim, d_w, w_layers, n, d_S, d_rgb_s, stream);
}

extern "C" size_t gsb_synthesis_forward_styled_workspace_bytes(const gsb_styled_conv *layers, int n_run, int n_rgb, int64_t n) {
    if (!layers || n_run < 1 || n_run > gsb::SY_MAX_LAYERS || n < 1) return 0;
    return gsb::synth_ws(nullptr, layers, n_run, n_rgb, n, false).bytes;
}

extern "C" int gsb_synthesis_forward_styled(const void *d_packed, const gsb_styled_conv *layers, int n_layers, int n_run, int n_rgb,
                                            int style_dim, const float *const *d_S, const float *const *d_rgb_s, int64_t n,
                                            float *d_act_out, int64_t ld_act, float *d_rgb_out, void *d_workspace,
                                            size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    SynthWs w;
    if (int r = check_run(d_packed, layers, n_layers, n_run, n_rgb, style_dim, n, d_act_out, ld_act, d_rgb_out, d_workspace,
                          workspace_bytes, false, &w)) return r;
    GSB_CHECK_ARG(d_S && (n_rgb == 0 || d_rgb_s), "synthesis_forward_styled: null style list");
    for (int l = 0; l < n_run; ++l)
        GSB_CHECK_ARG(d_S[l] && aligned16(d_S[l]), "synthesis_forward_styled: style of layer %d is null or not 16-byte aligned", l);
    for (int j = 0; j < n_rgb; ++j)
        GSB_CHECK_ARG(d_rgb_s[j] && aligned16(d_rgb_s[j]), "synthesis_forward_styled: style of ToRGB %d is null or not 16-byte aligned", j);
    if (n == 0) return GSB_OK;
    const SynthView v = synth_view(const_cast<void *>(d_packed), layers, n_layers, style_dim);
    return synthesis_run(v, layers, n_run, n_rgb, d_S, d_rgb_s, n, d_act_out, ld_act, d_rgb_out, w, stream);
}

extern "C" int gsb_synthesis_status(const void *d_packed, const gsb_styled_conv *layers, int n_layers, int style_dim, unsigned *h_flags) {
    using namespace gsb;
    if (int r = check_layers(layers, n_layers, style_dim)) return r;
    GSB_CHECK_ARG(d_packed && h_flags, "synthesis_status: null pointer");
    SynthView v = synth_view(const_cast<void *>(d_packed), layers, n_layers, style_dim);
    GSB_CHECK_CUDA(cudaMemcpy(h_flags, v.overflow, sizeof(unsigned), cudaMemcpyDeviceToHost));
    return GSB_OK;
}
