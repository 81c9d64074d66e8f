// StyleGAN (v1) synthesis network: g_synthesis.blocks.4x4 .. RxR and torgb.
//
// Replaces models/stylegan/model.py:270-376 (InputBlock, GSynthesisBlock, LayerEpilogue, G_synthesis.forward) as driven by
// models/wrappers.py:330-417 (StyleGAN.forward, partial_forward).
//
// Layers run in execution order, two per block.  Layer l is
//     x  ->  conv (l > 0)  ->  + bias  ->  + noise_weight[c] noise[y,x]  ->  leaky-ReLU 0.2  ->  InstanceNorm  ->  StyleMod(w_l)
// with  layer 0 : x = const (the InputBlock's learned [C, 4, 4] tensor, shared by all samples)
//       conv    : 3x3, padding 1, weight * sqrt2 / sqrt(9 cin)
//       up-conv : nearest x2, 3x3 conv, then the [1,2,1] x [1,2,1] / 16 depthwise blur with zero padding of the conv OUTPUT.
//                 From 128 px on the reference takes the conv_transpose2d branch (model.py:82-91) instead: that equals nearest x2
//                 followed by a 3x3 correlation with the kernel flipped in both spatial axes, so those layers pack the flipped
//                 kernel and share the rest of the path.
// InstanceNorm is per sample and channel over H*W (biased variance, eps 1e-5); StyleMod is  x (s0 + 1) + s1  with
// [s0 | s1] = w_l (A / sqrt(dlatent))^T + b.  Together:  y = (x - mean) * (rstd (s0 + 1)) + s1,  one affine per (sample, channel).
//
// Per layer and chunk of samples:
//     tap GEMM      Y[b,p,tap,co] = sum_ci (scale W)[co,ci,tap] x[b,p,ci]    (tc_gemm_plain, fp16 hi/lo, wgmma), at the INPUT
//                                 resolution: nearest x2 only replicates pixels (the formulation of progan.cu)
//     up gather     U = the up-conv output (up-conv layers only; the blur reads it)
//     epilogue      gather / blur, bias, noise, leaky-ReLU -> pre-norm activation A (fp32 NHWC) and per-(sample, tile, channel)
//                   fp64 sums and sums of squares
//     finish        one warp per (sample, channel): the tiles' sums in a fixed order -> mean and the affine
//     apply         the affine -> the next layer's operand as fp16 hi/lo, and / or the hooked activation as fp32 NHWC rows with a
//                   caller-given row stride, and / or (last layer) the 1x1 torgb conv
// The StyleMod vectors of every layer come from one style GEMM launch before the first layer (the style stage); the rest is the
// run stage, which gsb_stylegan_forward_styled runs on caller-given styles.  No float atomics; every reduction runs in
// a fixed order inside one sample, so a sample's result does not depend on the batch it is part of.
//
// Channel counts: cin and cout are powers of two in [16, 512].  The 16-channel layers of the 1024-px generators run on the same
// path: the GEMM needs only K % 8 == 0, and its N = 9 cout is padded with zero weight rows to a multiple of 32.
#include "tap_conv.cuh"
#include <math.h>

namespace gsb {

constexpr int SG_MAX_LAYERS = 18;
constexpr int SG_TILE_PASSES = 8;                                 // pixel passes of one epilogue block (the statistics tile)

static int sg_np(const gsb_stylegan_layer &c) { return (9 * c.cout + 31) / 32 * 32; }           // GEMM N (padded)
static int sg_res_in(const gsb_stylegan_layer &c) { return c.upsample ? c.res_out / 2 : c.res_out; }
// up-conv layers from 128 px on run the reference's conv_transpose2d branch: the flipped kernel
static bool sg_flipped(const gsb_stylegan_layer &c) { return c.upsample && c.res_out >= 128; }
static int sg_tile_px(const gsb_stylegan_layer &c) {
    const int hw = c.res_out * c.res_out, ppp = 1024 / c.cout;    // pixels per pass of a 256-thread block
    return hw < ppp * SG_TILE_PASSES ? hw : ppp * SG_TILE_PASSES;
}
static int64_t sg_chunk_samples(const gsb_stylegan_layer &c) {
    const int64_t hw_in = (int64_t)sg_res_in(c) * sg_res_in(c), hw = (int64_t)c.res_out * c.res_out;
    int64_t per = hw * c.cout;
    if (c.conv_weight && hw_in * sg_np(c) > per) per = hw_in * sg_np(c);
    const int64_t spc = TAP_CHUNK_ELEMS / per;
    return spc < 1 ? 1 : spc;
}

// ---- packed layout ----------------------------------------------------------------------------------------
struct SgLayerView {
    __half *w_hi, *w_lo;      // [np, cin]  row = tap*cout + co (rows >= 9 cout are zero)
    float *scal;              // [4]: inv_wscale, wscale, absmax
    float *bias, *noise_w;    // [cout]
    float *noise;             // [res_out^2]
    int style_off;            // column of s0 in the style matrix (s1 follows at + cout)
};
struct SgView {
    unsigned *overflow;
    float *cst;               // [16, c0] NHWC
    float *style_wt;          // [dlatent, s_total]  A^T / sqrt(dlatent), all layers side by side
    float *style_b;           // [s_total]
    int s_total;
    float *rgb_w;             // [3, c_last] / sqrt(c_last)
    float *rgb_b;             // [3]
    SgLayerView L[SG_MAX_LAYERS];
    size_t bytes;
};
static SgView sg_view(void *base, const gsb_stylegan_layer *layers, int n_layers, int dlatent) {
    SgView v;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    v.s_total = 0;
    for (int l = 0; l < n_layers; ++l) v.s_total += 2 * layers[l].cout;
    v.overflow = (unsigned *)take(256);
    v.cst = (float *)take((size_t)16 * layers[0].cout * 4);
    v.style_wt = (float *)take((size_t)dlatent * v.s_total * 4);
    v.style_b = (float *)take((size_t)v.s_total * 4);
    v.rgb_w = (float *)take((size_t)3 * layers[n_layers - 1].cout * 4);
    v.rgb_b = (float *)take(16);
    int soff = 0;
    for (int l = 0; l < n_layers; ++l) {
        const gsb_stylegan_layer &c = layers[l];
        const size_t wcount = c.conv_weight ? (size_t)sg_np(c) * c.cin : 0;
        v.L[l].w_hi = (__half *)take(wcount * 2);
        v.L[l].w_lo = (__half *)take(wcount * 2);
        v.L[l].scal = (float *)take(16);
        v.L[l].bias = (float *)take((size_t)c.cout * 4);
        v.L[l].noise_w = (float *)take((size_t)c.cout * 4);
        v.L[l].noise = (float *)take((size_t)c.res_out * c.res_out * 4);
        v.L[l].style_off = soff;
        soff += 2 * c.cout;
    }
    v.bytes = off;
    return v;
}

static bool sg_pow2(int x, int lo, int hi) { return x >= lo && x <= hi && (x & (x - 1)) == 0; }

static int sg_check(const gsb_stylegan_layer *layers, int n_layers, int dlatent) {
    GSB_CHECK_ARG(layers && n_layers >= 1 && n_layers <= SG_MAX_LAYERS, "stylegan: need 1..%d layers", SG_MAX_LAYERS);
    GSB_CHECK_ARG(dlatent >= 1 && dlatent <= 4096, "stylegan: bad dlatent %d", dlatent);
    for (int l = 0; l < n_layers; ++l) {
        const gsb_stylegan_layer &c = layers[l];
        GSB_CHECK_ARG(sg_pow2(c.cout, 16, 512) && (l == 0 || sg_pow2(c.cin, 16, 512)),
                      "stylegan: layer %d needs cin, cout powers of two in [16, 512] (cin=%d cout=%d)", l, c.cin, c.cout);
        if (l == 0) GSB_CHECK_ARG(!c.conv_weight && !c.upsample && c.res_out == 4, "stylegan: layer 0 is the 4x4 constant input");
        else GSB_CHECK_ARG(c.conv_weight && c.cin == layers[l - 1].cout && sg_res_in(c) == layers[l - 1].res_out && c.res_out <= 1024,
                           "stylegan: layer %d does not chain", l);
    }
    return GSB_OK;
}

// ---- pack kernels ---------------------------------------------------------------------------------------
// A [rows, K] (StyleMod lin.weight) -> dst[k * ld + r] = A[r, k] * scale
__global__ void sg_transpose_scale_kernel(const float *__restrict__ A, int rows, int K, float scale, float *__restrict__ dst, int64_t ld) {
    for (int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x; idx < (int64_t)rows * K; idx += (int64_t)gridDim.x * blockDim.x) {
        const int r = (int)(idx / K), k = (int)(idx % K);
        dst[(int64_t)k * ld + r] = A[idx] * scale;
    }
}

// ---- style GEMM -------------------------------------------------------------------------------------------
// The StyleMod rows of a set of layers:  S_l[b, j] = w_{lat(l)}[b] . style_wt[:, col0(l) + j] + style_b[col0(l) + j],  every
// element computed as  acc = 0; acc = fmaf(w[k], wt[k][j], acc) for k = 0 .. dlatent-1 in order; acc + bias  -- so a row does not
// depend on the tile, the batch or the launch it is computed in.
// Register-tiled FP32 GEMM: a CTA computes 32 TM rows x SGS_BN = 32 columns, 256 threads of TM rows x 4 columns; operands are
// staged through shared memory in BK-deep slices by a cp.async double buffer.  Small batches (TM <= 2) take deeper slices and
// four CTAs per SM: with little arithmetic per slice, the loads in flight -- the slices' latency -- set the kernel's time.  Every 2 cout is a multiple of
// 32, so a column tile lies inside one layer and reads one latent per sample.  The grid is linear, column tiles fastest: the
// CTAs that share a slice of latent rows run side by side (the rows come from L2 once per column tile, from HBM once).
constexpr int SGS_BN = 32, SGS_THREADS = 256, SGS_PAD = 4;

struct SgStyleJob {
    const float *w;                       // [w_layers, n, dlatent]
    const float *wt, *bias;               // packed: [dlatent, s_total], [s_total]
    int64_t n;
    int dlatent, s_total, n_sel;
    int col0[SG_MAX_LAYERS];              // selected layer s: its first column in the packed style matrix
    int tile0[SG_MAX_LAYERS + 1];         // its first column tile (prefix sums; tile0[n_sel] = all column tiles)
    int lat[SG_MAX_LAYERS];               // the latent it reads
    float *out[SG_MAX_LAYERS];            // its rows: out[s] + b * ld[s] + j
    int64_t ld[SG_MAX_LAYERS];
};

__device__ __forceinline__ void sgs_cp16(float *dst, const float *src, bool valid) {
    const unsigned sa = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16, %2;" ::"r"(sa), "l"(src), "r"(valid ? 16 : 0) : "memory");
}

template <int TM, int BK>
__global__ void __launch_bounds__(SGS_THREADS, TM <= 2 ? 4 : 2)
sg_style_gemm_kernel(const __grid_constant__ SgStyleJob J) {
    constexpr int BM = 32 * TM;
    __shared__ __align__(16) float As[2][BM][BK + SGS_PAD];
    __shared__ __align__(16) float Bs[2][BK][SGS_BN];
    const int n_ct = J.tile0[J.n_sel];
    const int ct = (int)(blockIdx.x % (unsigned)n_ct);
    const int64_t r0 = (int64_t)(blockIdx.x / (unsigned)n_ct) * BM;
    int s = 0;
    while (ct >= J.tile0[s + 1]) ++s;
    const int jl = (ct - J.tile0[s]) * SGS_BN;                      // first column of the tile inside its layer
    const int jg = J.col0[s] + jl;                                  // ... in the packed style matrix
    const float *wl = J.w + (int64_t)J.lat[s] * J.n * J.dlatent;
    const int tid = threadIdx.x, tc = tid & 7, tr = tid >> 3;
    const int nk = (J.dlatent + BK - 1) / BK;

    auto load = [&](int kt, int buf) {
        const int k0 = kt * BK;
        for (int c = tid; c < BM * BK / 4; c += SGS_THREADS) {      // A: BM rows x BK/4 quads (rows past n are zero-filled)
            const int row = c / (BK / 4), kq = (c % (BK / 4)) * 4;
            const int64_t b = r0 + row < J.n ? r0 + row : J.n - 1;
            const bool ok = k0 + kq < J.dlatent && r0 + row < J.n;
            sgs_cp16(&As[buf][row][kq], wl + b * J.dlatent + (ok ? k0 + kq : 0), ok);
        }
        for (int c = tid; c < BK * SGS_BN / 4; c += SGS_THREADS) {  // B: BK rows x 8 quads
            const int k = c >> 3, jq = (c & 7) * 4;
            const bool ok = k0 + k < J.dlatent;
            sgs_cp16(&Bs[buf][k][jq], J.wt + (int64_t)(ok ? k0 + k : 0) * J.s_total + jg + jq, ok);
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };

    float acc[TM][4];
#pragma unroll
    for (int i = 0; i < TM; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    load(0, 0);
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) {
            load(kt + 1, buf ^ 1);
            asm volatile("cp.async.wait_group 1;" ::: "memory");
        } else {
            asm volatile("cp.async.wait_group 0;" ::: "memory");
        }
        __syncthreads();
        const int kmax = J.dlatent - kt * BK;                       // only the last slice of a dlatent % BK != 0 is partial
        if (kmax >= BK) {
#pragma unroll
            for (int kq = 0; kq < BK; kq += 4) {
                float4 bq[4];
#pragma unroll
                for (int q = 0; q < 4; ++q) bq[q] = *reinterpret_cast<const float4 *>(&Bs[buf][kq + q][tc * 4]);
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    const float4 a = *reinterpret_cast<const float4 *>(&As[buf][tr + 32 * i][kq]);
                    const float av[4] = {a.x, a.y, a.z, a.w};
#pragma unroll
                    for (int q = 0; q < 4; ++q) {
                        acc[i][0] = fmaf(av[q], bq[q].x, acc[i][0]);
                        acc[i][1] = fmaf(av[q], bq[q].y, acc[i][1]);
                        acc[i][2] = fmaf(av[q], bq[q].z, acc[i][2]);
                        acc[i][3] = fmaf(av[q], bq[q].w, acc[i][3]);
                    }
                }
            }
        } else {
            for (int k = 0; k < kmax; ++k) {
                const float4 bq = *reinterpret_cast<const float4 *>(&Bs[buf][k][tc * 4]);
#pragma unroll
                for (int i = 0; i < TM; ++i) {
                    const float a = As[buf][tr + 32 * i][k];
                    acc[i][0] = fmaf(a, bq.x, acc[i][0]);
                    acc[i][1] = fmaf(a, bq.y, acc[i][1]);
                    acc[i][2] = fmaf(a, bq.z, acc[i][2]);
                    acc[i][3] = fmaf(a, bq.w, acc[i][3]);
                }
            }
        }
        __syncthreads();                                            // the slice is read before the next load overwrites it
    }
    const float4 bv = *reinterpret_cast<const float4 *>(J.bias + jg + tc * 4);
#pragma unroll
    for (int i = 0; i < TM; ++i) {
        const int64_t b = r0 + tr + 32 * i;
        if (b >= J.n) continue;
        float *o = J.out[s] + b * J.ld[s] + jl + tc * 4;
        o[0] = acc[i][0] + bv.x;
        o[1] = acc[i][1] + bv.y;
        o[2] = acc[i][2] + bv.z;
        o[3] = acc[i][3] + bv.w;
    }
}

// One launch of the style GEMM over the layers of `J` (n_sel, col0, lat, out, ld filled in by the caller); rows are tiled by the
// smallest TM whose 32 TM rows hold n, at most 8.
static int sg_style_launch(SgStyleJob &J, const SgView &v, const gsb_stylegan_layer *layers, const int *sel, cudaStream_t st) {
    int t = 0;
    for (int s = 0; s < J.n_sel; ++s) {
        J.tile0[s] = t;
        t += 2 * layers[sel[s]].cout / SGS_BN;
    }
    J.tile0[J.n_sel] = t;
    J.wt = v.style_wt;
    J.bias = v.style_b;
    J.s_total = v.s_total;
    if (J.n == 0 || t == 0) return GSB_OK;
    const int TM = J.n <= 32 ? 1 : J.n <= 64 ? 2 : J.n <= 128 ? 4 : 8;
    const int64_t blocks = (J.n + 32 * TM - 1) / (32 * TM) * t;
    GSB_CHECK_ARG(blocks <= 0x7fffffff, "stylegan: %lld style tiles exceed one launch", (long long)blocks);
    switch (TM) {
        case 1: sg_style_gemm_kernel<1, 64><<<(unsigned)blocks, SGS_THREADS, 0, st>>>(J); break;
        case 2: sg_style_gemm_kernel<2, 32><<<(unsigned)blocks, SGS_THREADS, 0, st>>>(J); break;
        case 4: sg_style_gemm_kernel<4, 16><<<(unsigned)blocks, SGS_THREADS, 0, st>>>(J); break;
        default: sg_style_gemm_kernel<8, 16><<<(unsigned)blocks, SGS_THREADS, 0, st>>>(J); break;
    }
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// ---- forward kernels ------------------------------------------------------------------------------------

// the 3x3 conv outputs of an up-conv layer (before the blur), from Y at the input resolution R/2 with row length np.  One thread
// per 4 channels of an output pixel.
__global__ void __launch_bounds__(256)
sg_up_gather_kernel(const float *__restrict__ Y, int64_t nb, int R, int c, int np, float *__restrict__ U) {
    const int cq = c >> 2;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= nb * R * R * cq) return;
    const int q = (int)(idx % cq);
    const int64_t pixg = idx / cq;
    const int x = (int)(pixg % R), y = (int)((pixg / R) % R);
    const int64_t b = pixg / ((int64_t)R * R);
    *reinterpret_cast<float4 *>(U + pixg * c + 4 * q) = tap_sum3x3<true>(Y, np, b, y, x, R, c, q);
}

// MODE 0: the constant input (src = const [16, c]); 1: stride-1 3x3 gather (src = Y [nb*R*R, np]); 2: the blur of the up-conv
// output (src = U [nb, R, R, c], zero padding).  Then + bias + noise_w noise[p], leaky-ReLU -> A, and the tile's fp64 sums.
// Grid (tiles, nb), 256 threads: thread = (pixel lane pl, channel quad q); a block covers `tile` consecutive pixels of one sample.
template <int MODE>
__global__ void __launch_bounds__(256)
sg_epilogue_kernel(const float *__restrict__ src, int R, int c, int np, int tile, const float *__restrict__ bias,
                   const float *__restrict__ noise_w, const float *__restrict__ noise, float *__restrict__ A, double *__restrict__ part) {
    __shared__ double red[2][256][4];
    const int cq = c >> 2, ppp = 256 / cq;
    const int q = threadIdx.x % cq, pl = threadIdx.x / cq;
    const int64_t b = blockIdx.y;
    const int hw = R * R;
    const float4 bs = *reinterpret_cast<const float4 *>(bias + 4 * q);
    const float4 nw = *reinterpret_cast<const float4 *>(noise_w + 4 * q);
    double s[4] = {0.0, 0.0, 0.0, 0.0}, ss[4] = {0.0, 0.0, 0.0, 0.0};
    for (int p = blockIdx.x * tile + pl; p < (blockIdx.x + 1) * tile; p += ppp) {
        const int y = p / R, x = p % R;
        float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
        if (MODE == 0) {
            acc = *reinterpret_cast<const float4 *>(src + (int64_t)p * c + 4 * q);
        } else if (MODE == 1) {
            acc = tap_sum3x3<false>(src, np, b, y, x, R, c, q);
        } else {
#pragma unroll
            for (int ky = 0; ky < 3; ++ky) {
                const int yy = y + ky - 1;
                if (yy < 0 || yy >= R) continue;
#pragma unroll
                for (int kx = 0; kx < 3; ++kx) {
                    const int xx = x + kx - 1;
                    if (xx < 0 || xx >= R) continue;
                    const float wgt = (float)((ky == 1 ? 2 : 1) * (kx == 1 ? 2 : 1)) * 0.0625f;
                    const float4 v = *reinterpret_cast<const float4 *>(src + ((b * R + yy) * R + xx) * (int64_t)c + 4 * q);
                    acc.x = fmaf(wgt, v.x, acc.x); acc.y = fmaf(wgt, v.y, acc.y); acc.z = fmaf(wgt, v.z, acc.z); acc.w = fmaf(wgt, v.w, acc.w);
                }
            }
        }
        const float nz = noise[p];
        float f[4] = {acc.x + bs.x, acc.y + bs.y, acc.z + bs.z, acc.w + bs.w};
        const float g[4] = {nw.x, nw.y, nw.z, nw.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            f[k] = fmaf(g[k], nz, f[k]);
            f[k] = (f[k] >= 0.f) ? f[k] : 0.2f * f[k];
            s[k] += (double)f[k];
            ss[k] += (double)f[k] * (double)f[k];
        }
        *reinterpret_cast<float4 *>(A + (b * hw + p) * (int64_t)c + 4 * q) = make_float4(f[0], f[1], f[2], f[3]);
    }
#pragma unroll
    for (int k = 0; k < 4; ++k) { red[0][threadIdx.x][k] = s[k]; red[1][threadIdx.x][k] = ss[k]; }
    __syncthreads();
    if (pl == 0) {
        for (int j = 1; j < ppp; ++j)
#pragma unroll
            for (int k = 0; k < 4; ++k) { s[k] += red[0][j * cq + q][k]; ss[k] += red[1][j * cq + q][k]; }
        double *o = part + ((b * gridDim.x + blockIdx.x) * (int64_t)c + 4 * q) * 2;
#pragma unroll
        for (int k = 0; k < 4; ++k) { o[2 * k] = s[k]; o[2 * k + 1] = ss[k]; }
    }
}

// one warp per (sample, channel): tiles summed lane-strided in order, then a fixed shuffle tree.  aff[b, c] = {mean, rstd (s0+1), s1}
__global__ void __launch_bounds__(256)
sg_finish_kernel(const double *__restrict__ part, int64_t nb, int c, int tiles, int hw, const float *__restrict__ S, int64_t s_ld,
                 int s_off, float4 *__restrict__ aff) {
    const int64_t wid = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (wid >= nb * c) return;
    const int64_t b = wid / c;
    const int ch = (int)(wid % c);
    double s = 0.0, ss = 0.0;
    for (int t = lane; t < tiles; t += 32) {
        const double *o = part + ((b * tiles + t) * (int64_t)c + ch) * 2;
        s += o[0];
        ss += o[1];
    }
    s = warp_sum(s);
    ss = warp_sum(ss);
    if (lane == 0) {
        const double mean = s / hw;
        double var = ss / hw - mean * mean;
        var = var > 0.0 ? var : 0.0;
        const float rstd = (float)(1.0 / sqrt(var + 1e-5));
        const float s0 = S[b * s_ld + s_off + ch], s1 = S[b * s_ld + s_off + c + ch];
        aff[wid] = make_float4((float)mean, rstd * (s0 + 1.f), s1, 0.f);
    }
}

struct SgApply {
    const float *A;              // [nb, hw, c] pre-norm activation (chunk-local)
    const float4 *aff;           // [nb, c]
    __half *out_hi, *out_lo;     // [nb, hw, c] (chunk-local) operand of the next layer, or nullptr
    float *out_f32;              // hooked layer: row b at out_f32 + b*ld, or nullptr
    int64_t ld;
    const float *rgb_w, *rgb_b;  // torgb: [3, c] (scaled) and [3], or nullptr
    float *rgb_out;              // [nb, hw, 3] (chunk-local)
    unsigned *overflow;
};
// y = (x - mean) a + s1 for 4 channels of one pixel -> the enabled outputs.  Threads past the end take part in the RGB sums.
__global__ void __launch_bounds__(256)
sg_apply_kernel(SgApply e, int64_t nb, int hw, int c) {
    const int cq = c >> 2;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    const bool valid = idx < nb * hw * cq;
    const int q = (int)(idx % cq);
    const int64_t pixg = idx / cq;
    const int64_t b = pixg / hw;
    const int pix = (int)(pixg % hw);
    float y[4] = {0.f, 0.f, 0.f, 0.f};
    if (valid) {
        const float4 x = *reinterpret_cast<const float4 *>(e.A + pixg * c + 4 * q);
        const float xv[4] = {x.x, x.y, x.z, x.w};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float4 a = e.aff[b * c + 4 * q + k];
            y[k] = fmaf(xv[k] - a.x, a.y, a.z);
        }
        if (e.out_f32) *reinterpret_cast<float4 *>(e.out_f32 + b * e.ld + (int64_t)pix * c + 4 * q) = make_float4(y[0], y[1], y[2], y[3]);
        if (e.out_hi) {
            bool ovf = false;
            tc::store_split4(y, e.out_hi, e.out_lo, pixg * c + 4 * q, ovf);
            if (ovf) atomicOr(e.overflow, 1u);
        }
    }
    if (e.rgb_w) {
#pragma unroll
        for (int o = 0; o < 3; ++o) {
            const float4 wv = *reinterpret_cast<const float4 *>(e.rgb_w + (int64_t)o * c + 4 * q);
            const float r = pixel_sum((y[0] * wv.x + y[1] * wv.y) + (y[2] * wv.z + y[3] * wv.w), cq);
            if (valid && q == 0) e.rgb_out[pixg * 3 + o] = r + e.rgb_b[o];
        }
    }
}

// ---- workspace --------------------------------------------------------------------------------------------
struct SgWs {
    float *S;               // [n, s_run]  (gsb_stylegan_forward only: the styled run reads the caller's)
    __half *act[2][2];      // [ping-pong][hi/lo]
    float *Y, *U, *A;
    double *part;
    float4 *aff;
    unsigned *queue;        // tile queue of the tap GEMM launches
    size_t bytes;
};
static SgWs sg_ws(void *base, const gsb_stylegan_layer *layers, int n_run, int64_t n, bool own_styles) {
    SgWs w;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    size_t s_run = 0, act_elems = 64, y_elems = 64, a_elems = 64, part_elems = 64, aff_elems = 64;
    for (int l = 0; l < n_run; ++l) {
        const gsb_stylegan_layer &c = layers[l];
        s_run += 2 * c.cout;
        const size_t hw = (size_t)c.res_out * c.res_out, hw_in = (size_t)sg_res_in(c) * sg_res_in(c);
        if (l + 1 < n_run) act_elems = act_elems > n * hw * c.cout ? act_elems : n * hw * c.cout;
        const size_t spc = (size_t)(sg_chunk_samples(c) < n ? sg_chunk_samples(c) : n);
        if (c.conv_weight) y_elems = y_elems > spc * hw_in * sg_np(c) ? y_elems : spc * hw_in * sg_np(c);
        a_elems = a_elems > spc * hw * c.cout ? a_elems : spc * hw * c.cout;
        const size_t pe = spc * (hw / sg_tile_px(c)) * c.cout * 2;
        part_elems = part_elems > pe ? part_elems : pe;
        aff_elems = aff_elems > spc * c.cout ? aff_elems : spc * c.cout;
    }
    w.S = own_styles ? (float *)take((size_t)n * s_run * 4) : nullptr;
    for (int a = 0; a < 2; ++a)
        for (int h = 0; h < 2; ++h) w.act[a][h] = (__half *)take(act_elems * 2);
    w.Y = (float *)take(y_elems * 4);
    w.U = (float *)take(a_elems * 4);
    w.A = (float *)take(a_elems * 4);
    w.part = (double *)take(part_elems * 8);
    w.aff = (float4 *)take(aff_elems * 16);
    w.queue = (unsigned *)take(sizeof(unsigned));
    w.bytes = off;
    return w;
}

static int sg_s_run(const gsb_stylegan_layer *layers, int n_run) {
    int s_run = 0;
    for (int l = 0; l < n_run; ++l) s_run += 2 * layers[l].cout;
    return s_run;
}

// The arguments gsb_stylegan_forward and gsb_stylegan_forward_styled share.
static int sg_run_check(const gsb_stylegan_layer *layers, int n_layers, int n_run, int dlatent, int64_t n, const float *d_act_out,
                        int64_t ld_act, const float *d_rgb_out) {
    if (int r = sg_check(layers, n_layers, dlatent)) return r;
    GSB_CHECK_ARG(n_run >= 1 && n_run <= n_layers && n >= 0, "stylegan: n_run / n out of range");
    GSB_CHECK_ARG(!d_rgb_out || n_run == n_layers, "stylegan: the image needs every layer (n_run == n_layers)");
    if (n == 0) return GSB_OK;
    GSB_CHECK_ARG(n <= 65535, "stylegan: at most 65535 samples per call (n = %lld)", (long long)n);
    const gsb_stylegan_layer &last = layers[n_run - 1];
    GSB_CHECK_ARG(!d_act_out || (ld_act >= (int64_t)last.res_out * last.res_out * last.cout && ld_act % 4 == 0), "stylegan: bad ld_act");
    return GSB_OK;
}

// The style GEMM's operand rules: 16-byte cp.async slices of the latent rows.
static int sg_latents_check(const float *d_w, int dlatent) {
    GSB_CHECK_ARG(dlatent % 4 == 0 && ((uintptr_t)d_w & 15) == 0,
                  "stylegan: the style GEMM needs dlatent %% 4 == 0 and 16-byte aligned latents (dlatent = %d)", dlatent);
    return GSB_OK;
}

// The run stage: layers 0 .. n_run-1 on the styles S [n, s_run] (the chain's column order).
static int sg_run(const SgView &v, const SgWs &w, const gsb_stylegan_layer *layers, int n_run, const float *S, int64_t n, float *d_act_out,
                  int64_t ld_act, float *d_rgb_out, cudaStream_t st) {
    const int s_run = sg_s_run(layers, n_run);
    for (int l = 0; l < n_run; ++l) {
        const gsb_stylegan_layer &c = layers[l];
        const int dst = l & 1;                                         // layer l reads act[dst ^ 1], writes act[dst]
        const __half *a_hi = w.act[dst ^ 1][0], *a_lo = w.act[dst ^ 1][1];
        const bool is_last = (l == n_run - 1);
        const int R = c.res_out, H = sg_res_in(c), hw = R * R, hw_in = H * H, np = sg_np(c), tile = sg_tile_px(c), tiles = hw / tile;
        const int64_t spc = sg_chunk_samples(c);
        for (int64_t b0 = 0; b0 < n; b0 += spc) {
            const int64_t nb = (b0 + spc <= n) ? spc : (n - b0);
            const dim3 egrid((unsigned)tiles, (unsigned)nb);
            if (!c.conv_weight) {
                sg_epilogue_kernel<0><<<egrid, 256, 0, st>>>(v.cst, R, c.cout, 0, tile, v.L[l].bias, v.L[l].noise_w, v.L[l].noise, w.A, w.part);
            } else {
                if (int r = tc_gemm_plain(a_hi + b0 * hw_in * c.cin, a_lo + b0 * hw_in * c.cin, nb * hw_in, c.cin, v.L[l].w_hi, v.L[l].w_lo,
                                          np, v.L[l].scal, w.Y, v.overflow, w.queue, 0, st)) return r;
                if (c.upsample) {
                    const int64_t total = nb * hw * (c.cout / 4);
                    sg_up_gather_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(w.Y, nb, R, c.cout, np, w.U);
                    GSB_CHECK_LAUNCH();
                    sg_epilogue_kernel<2><<<egrid, 256, 0, st>>>(w.U, R, c.cout, np, tile, v.L[l].bias, v.L[l].noise_w, v.L[l].noise, w.A, w.part);
                } else {
                    sg_epilogue_kernel<1><<<egrid, 256, 0, st>>>(w.Y, R, c.cout, np, tile, v.L[l].bias, v.L[l].noise_w, v.L[l].noise, w.A, w.part);
                }
            }
            GSB_CHECK_LAUNCH();
            sg_finish_kernel<<<(unsigned)((nb * c.cout + 7) / 8), 256, 0, st>>>(w.part, nb, c.cout, tiles, hw, S + b0 * s_run, s_run,
                                                                               v.L[l].style_off, w.aff);
            GSB_CHECK_LAUNCH();
            SgApply e;
            e.A = w.A;
            e.aff = w.aff;
            e.out_hi = is_last ? nullptr : w.act[dst][0] + b0 * hw * c.cout;
            e.out_lo = is_last ? nullptr : w.act[dst][1] + b0 * hw * c.cout;
            e.out_f32 = (is_last && d_act_out) ? d_act_out + b0 * ld_act : nullptr;
            e.ld = ld_act;
            e.rgb_w = (is_last && d_rgb_out) ? v.rgb_w : nullptr;
            e.rgb_b = v.rgb_b;
            e.rgb_out = (is_last && d_rgb_out) ? d_rgb_out + b0 * hw * 3 : nullptr;
            e.overflow = v.overflow;
            const int64_t total = nb * hw * (c.cout / 4);
            sg_apply_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(e, nb, hw, c.cout);
            GSB_CHECK_LAUNCH();
        }
    }
    return GSB_OK;
}

}  // namespace gsb

extern "C" size_t gsb_stylegan_packed_bytes(const gsb_stylegan_layer *layers, int n_layers, int dlatent) {
    if (gsb::sg_check(layers, n_layers, dlatent)) return 0;
    return gsb::sg_view(nullptr, layers, n_layers, dlatent).bytes;
}

extern "C" int gsb_stylegan_pack(const gsb_stylegan_layer *layers, int n_layers, int dlatent, const float *d_const,
                                 const float *d_rgb_weight, const float *d_rgb_bias, void *d_packed, size_t packed_bytes,
                                 gsb_stream_t stream) {
    using namespace gsb;
    if (int r = sg_check(layers, n_layers, dlatent)) return r;
    GSB_CHECK_ARG(d_const && d_rgb_weight && d_rgb_bias && d_packed, "stylegan_pack: null pointer");
    SgView v = sg_view(d_packed, layers, n_layers, dlatent);
    if (packed_bytes < v.bytes) { set_error("stylegan_pack: buffer too small (%zu < %zu)", packed_bytes, v.bytes); return GSB_ERR_WORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CHECK_CUDA(cudaMemsetAsync(d_packed, 0, v.bytes, st));
    const_nhwc_kernel<<<8, 256, 0, st>>>(d_const, layers[0].cout, v.cst);
    GSB_CHECK_LAUNCH();
    for (int l = 0; l < n_layers; ++l) {
        const gsb_stylegan_layer &c = layers[l];
        GSB_CHECK_ARG(c.bias && c.noise && c.noise_weight && c.style_weight && c.style_bias,
                      "stylegan_pack: layer %d has a null parameter pointer", l);
        if (c.conv_weight) {
            // MyConv2d with use_wscale, gain sqrt2, lrmul 1: w_mul = sqrt2 / sqrt(cin * 9) (model.py:51-62)
            const float scale = (float)(sqrt(2.0) / sqrt(9.0 * c.cin));
            // the flipped kernel (both spatial axes) of a 3x3 conv is its taps in reverse order
            if (int r = tc_split_weight(c.conv_weight, c.cout, c.cin, 9, scale, sg_flipped(c), sg_np(c), v.L[l].w_hi, v.L[l].w_lo,
                                        v.L[l].scal, nullptr, st)) return r;
        }
        scale_copy_kernel<<<4, 256, 0, st>>>(c.bias, c.cout, 1.0f, nullptr, v.L[l].bias);
        GSB_CHECK_LAUNCH();
        scale_copy_kernel<<<4, 256, 0, st>>>(c.noise_weight, c.cout, 1.0f, nullptr, v.L[l].noise_w);
        GSB_CHECK_LAUNCH();
        scale_copy_kernel<<<64, 256, 0, st>>>(c.noise, (int64_t)c.res_out * c.res_out, 1.0f, nullptr, v.L[l].noise);
        GSB_CHECK_LAUNCH();
        // StyleMod lin: MyLinear(dlatent, 2 cout, gain 1, use_wscale): w_mul = 1 / sqrt(dlatent), b_mul = 1 (model.py:121-131)
        sg_transpose_scale_kernel<<<256, 256, 0, st>>>(c.style_weight, 2 * c.cout, dlatent, (float)(1.0 / sqrt((double)dlatent)),
                                                       v.style_wt + v.L[l].style_off, v.s_total);
        GSB_CHECK_LAUNCH();
        scale_copy_kernel<<<4, 256, 0, st>>>(c.style_bias, 2 * c.cout, 1.0f, nullptr, v.style_b + v.L[l].style_off);
        GSB_CHECK_LAUNCH();
    }
    const int cl = layers[n_layers - 1].cout;
    // torgb: MyConv2d(c, 3, 1, gain 1, use_wscale): w_mul = 1 / sqrt(c)
    scale_copy_kernel<<<4, 256, 0, st>>>(d_rgb_weight, (int64_t)3 * cl, (float)(1.0 / sqrt((double)cl)), nullptr, v.rgb_w);
    GSB_CHECK_LAUNCH();
    scale_copy_kernel<<<1, 32, 0, st>>>(d_rgb_bias, 3, 1.0f, nullptr, v.rgb_b);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" size_t gsb_stylegan_workspace_bytes(const gsb_stylegan_layer *layers, int n_run, int64_t n) {
    if (!layers || n_run < 1 || n_run > gsb::SG_MAX_LAYERS || n < 1) return 0;
    return gsb::sg_ws(nullptr, layers, n_run, n, true).bytes;
}

extern "C" size_t gsb_stylegan_forward_styled_workspace_bytes(const gsb_stylegan_layer *layers, int n_run, int64_t n) {
    if (!layers || n_run < 1 || n_run > gsb::SG_MAX_LAYERS || n < 1) return 0;
    return gsb::sg_ws(nullptr, layers, n_run, n, false).bytes;
}

extern "C" int gsb_stylegan_forward(const void *d_packed, const gsb_stylegan_layer *layers, int n_layers, int n_run, int dlatent,
                                    const float *d_w, int w_layers, int64_t n, float *d_act_out, int64_t ld_act, float *d_rgb_out,
                                    void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (int r = sg_run_check(layers, n_layers, n_run, dlatent, n, d_act_out, ld_act, d_rgb_out)) return r;
    GSB_CHECK_ARG(d_packed && d_w && d_workspace && (d_act_out || d_rgb_out), "stylegan: null pointer");
    GSB_CHECK_ARG(w_layers == 1 || w_layers >= n_run, "stylegan: w_layers must be 1 or cover every layer run (%d < %d)", w_layers, n_run);
    if (n == 0) return GSB_OK;
    if (int r = sg_latents_check(d_w, dlatent)) return r;
    SgView v = sg_view(const_cast<void *>(d_packed), layers, n_layers, dlatent);
    SgWs w = sg_ws(d_workspace, layers, n_run, n, true);
    if (workspace_bytes < w.bytes) { set_error("stylegan: workspace too small (%zu < %zu)", workspace_bytes, w.bytes); return GSB_ERR_WORKSPACE; }
    cudaStream_t st = (cudaStream_t)stream;

    // the style stage: every layer run, in the chain's column order, into S [n, s_run]
    SgStyleJob J;
    J.w = d_w;
    J.n = n;
    J.dlatent = dlatent;
    J.n_sel = n_run;
    int sel[SG_MAX_LAYERS];
    const int s_run = sg_s_run(layers, n_run);
    for (int l = 0; l < n_run; ++l) {
        sel[l] = l;
        J.col0[l] = v.L[l].style_off;
        J.lat[l] = w_layers == 1 ? 0 : l;
        J.out[l] = w.S + v.L[l].style_off;
        J.ld[l] = s_run;
    }
    if (int r = sg_style_launch(J, v, layers, sel, st)) return r;
    return sg_run(v, w, layers, n_run, w.S, n, d_act_out, ld_act, d_rgb_out, st);
}

extern "C" int gsb_stylegan_forward_styled(const void *d_packed, const gsb_stylegan_layer *layers, int n_layers, int n_run, int dlatent,
                                           const float *d_S, int64_t n, float *d_act_out, int64_t ld_act, float *d_rgb_out,
                                           void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    if (int r = sg_run_check(layers, n_layers, n_run, dlatent, n, d_act_out, ld_act, d_rgb_out)) return r;
    GSB_CHECK_ARG(d_packed && d_S && d_workspace && (d_act_out || d_rgb_out), "stylegan_forward_styled: null pointer");
    if (n == 0) return GSB_OK;
    SgView v = sg_view(const_cast<void *>(d_packed), layers, n_layers, dlatent);
    SgWs w = sg_ws(d_workspace, layers, n_run, n, false);
    if (workspace_bytes < w.bytes) {
        set_error("stylegan_forward_styled: workspace too small (%zu < %zu)", workspace_bytes, w.bytes);
        return GSB_ERR_WORKSPACE;
    }
    return sg_run(v, w, layers, n_run, d_S, n, d_act_out, ld_act, d_rgb_out, (cudaStream_t)stream);
}

extern "C" int gsb_stylegan_styles(const void *d_packed, const gsb_stylegan_layer *layers, int n_layers, int dlatent, const float *d_w,
                                   int w_layers, int64_t n, const int *layer_idx, int n_idx, float *const *d_S, gsb_stream_t stream) {
    using namespace gsb;
    if (int r = sg_check(layers, n_layers, dlatent)) return r;
    GSB_CHECK_ARG(d_packed && (d_w || n == 0) && n >= 0 && w_layers >= 1, "stylegan_styles: null pointer or bad n / w_layers");
    GSB_CHECK_ARG(n_idx >= 1 && n_idx <= n_layers && layer_idx && d_S, "stylegan_styles: need 1..%d layers (n_idx = %d)", n_layers, n_idx);
    SgStyleJob J;
    J.w = d_w;
    J.n = n;
    J.dlatent = dlatent;
    J.n_sel = n_idx;
    SgView v = sg_view(const_cast<void *>(d_packed), layers, n_layers, dlatent);
    for (int s = 0; s < n_idx; ++s) {
        const int l = layer_idx[s];
        GSB_CHECK_ARG(l >= 0 && l < n_layers, "stylegan_styles: layer index %d out of [0, %d)", l, n_layers);
        GSB_CHECK_ARG(d_S[s] || n == 0, "stylegan_styles: null output for layer %d", l);
        GSB_CHECK_ARG(w_layers == 1 || l < w_layers, "stylegan_styles: layer %d needs latent %d (w_layers = %d)", l, l, w_layers);
        J.col0[s] = v.L[l].style_off;
        J.lat[s] = w_layers == 1 ? 0 : l;
        J.out[s] = d_S[s];
        J.ld[s] = 2 * layers[l].cout;
    }
    if (n == 0) return GSB_OK;
    if (int r = sg_latents_check(d_w, dlatent)) return r;
    return sg_style_launch(J, v, layers, layer_idx, (cudaStream_t)stream);
}

extern "C" int gsb_stylegan_status(const void *d_packed, const gsb_stylegan_layer *layers, int n_layers, int dlatent, unsigned *h_flags) {
    using namespace gsb;
    if (int r = sg_check(layers, n_layers, dlatent)) return r;
    GSB_CHECK_ARG(d_packed && h_flags, "stylegan_status: null pointer");
    SgView v = sg_view(const_cast<void *>(d_packed), layers, n_layers, dlatent);
    GSB_CHECK_CUDA(cudaMemcpy(h_flags, v.overflow, sizeof(unsigned), cudaMemcpyDeviceToHost));
    return GSB_OK;
}
