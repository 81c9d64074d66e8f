// BigGAN-deep generator: GenBlock, SelfAttn and the RGB tail (pytorch_pretrained_biggan/model.py:57-253 as driven by
// models/wrappers.py:599-648), the kernels behind ganspace_b200/models/biggan.py.
//
// Every convolution (and both attention products) is one implicit GEMM on fp32 NHWC activations:
//     out[b, y, x, co] = alpha * (sum_{tap, ci} op(X)[b, src(y, x, tap), ci] W[tap * cin + ci, co] + bias[co]) + res[b, y', x', co]
//     op(X)   = ReLU((X - m[ci]) * a[b, ci] + o[b, ci])      the conditional BatchNorm + ReLU before the conv, applied while the
//               operand tile is loaded (the block input stays raw for the skip path and the hooks); zero padding is applied
//               AFTER it, as the reference pads the normalised tensor
//     src     = (y + ky - p, x + kx - p), read at ((y + ky - p) >> 1, (x + kx - p) >> 1) of the half-resolution input when the
//               conv follows a nearest x2 up-sampling: BN and ReLU are per pixel, so they commute with the up-sampling and the
//               up-sampled operand is never materialised
//     res     = the GenBlock skip path (the first cout channels of the block input, nearest x2 when the block up-samples) or the
//               SelfAttn input; alpha = SelfAttn's gamma
// The weights are shared by all samples except in the two attention products, where the "weights" are the sample's own
// pooled phi / g maps (w_sample_stride).
//
// Arithmetic is plain fp32 FMA in a fixed order over k for every output element: BigGAN's activations have no bound (no
// PixelNorm; ReLU and residual sums grow), so there is no fp16 operand split to overflow, and a sample's result does not
// depend on the batch it is part of or on its position in it (no split-K, no atomics).
#include "common.cuh"
#include <math.h>

namespace gsb {

constexpr int BB_BM = 128, BB_BN = 64, BB_BK = 16, BB_THREADS = 256;

// ---- implicit-GEMM convolution ------------------------------------------------------------------------------------------
template <bool PROLOGUE>
__global__ void __launch_bounds__(BB_THREADS)
bb_conv_kernel(const gsb_biggan_conv c, int64_t n) {
    __shared__ __align__(16) float As[2][BB_BK][BB_BM + 4];
    __shared__ __align__(16) float Bs[2][BB_BK][BB_BN];
    const int tid = threadIdx.x;
    const int R = c.upsample ? 2 * c.res_in : c.res_in;            // output resolution
    const int64_t hw = (int64_t)R * R, M = n * hw;
    const int K = c.ksize * c.ksize * c.cin, pad = c.ksize >> 1;
    const int64_t m0 = (int64_t)blockIdx.x * BB_BM;
    const int n0 = blockIdx.y * BB_BN;

    // this thread's operand row (fixed over k) and the 8 consecutive k of each tile it loads
    const int arow = tid >> 1, akh = (tid & 1) * 8;
    const int64_t am = m0 + arow;
    const bool arow_ok = am < M;
    const int64_t ab = arow_ok ? am / hw : 0;
    const int apix = arow_ok ? (int)(am % hw) : 0;
    const int ay = apix / R, ax = apix % R;
    const float *xb = c.x + ab * ((int64_t)c.res_in * c.res_in) * c.ldx;
    // per-sample weights: every row of a tile belongs to one sample (hw is a multiple of the tile height, checked on the host)
    const float *wt = c.weight + (c.w_sample_stride ? (m0 / hw) * c.w_sample_stride : 0);
    const int bk = tid >> 4, bn4 = (tid & 15) * 4;

    float4 ra[2], rb;
    auto load = [&](int k0) {
        const int tap = k0 / c.cin, ci = k0 % c.cin + akh;
        const int yy = ay + tap / c.ksize - pad, xx = ax + tap % c.ksize - pad;
        ra[0] = ra[1] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (arow_ok && yy >= 0 && yy < R && xx >= 0 && xx < R) {
            const int ys = c.upsample ? (yy >> 1) : yy, xs = c.upsample ? (xx >> 1) : xx;
            const float *p = xb + ((int64_t)ys * c.res_in + xs) * c.ldx + ci;
            ra[0] = *reinterpret_cast<const float4 *>(p);
            ra[1] = *reinterpret_cast<const float4 *>(p + 4);
            if (PROLOGUE) {
                float *v = reinterpret_cast<float *>(ra);
#pragma unroll
                for (int j = 0; j < 8; ++j) {
                    const float t = (v[j] - c.bn_mean[ci + j]) * c.bn_scale[ab * c.cin + ci + j] + c.bn_offset[ab * c.cin + ci + j];
                    v[j] = t > 0.f ? t : 0.f;
                }
            }
        }
        rb = make_float4(0.f, 0.f, 0.f, 0.f);
        if (n0 + bn4 < c.cout) rb = *reinterpret_cast<const float4 *>(wt + (int64_t)(k0 + bk) * c.cout + n0 + bn4);
    };
    auto store = [&](int s) {
        const float *v = reinterpret_cast<const float *>(ra);
#pragma unroll
        for (int j = 0; j < 8; ++j) As[s][akh + j][arow] = v[j];
        *reinterpret_cast<float4 *>(&Bs[s][bk][bn4]) = rb;
    };

    const int ty = tid >> 4, tx = tid & 15;                  // rows ty*8 .. +8, columns tx*4 .. +4
    float acc[8][4];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 4; ++j) acc[i][j] = 0.f;

    const int nk = K / BB_BK;
    load(0);
    store(0);
    __syncthreads();
    for (int kt = 0; kt < nk; ++kt) {
        const int s = kt & 1;
        if (kt + 1 < nk) load((kt + 1) * BB_BK);
#pragma unroll
        for (int k = 0; k < BB_BK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&As[s][k][ty * 8]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&As[s][k][ty * 8 + 4]);
            const float4 b = *reinterpret_cast<const float4 *>(&Bs[s][k][tx * 4]);
            const float av[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 4; ++j) acc[i][j] = fmaf(av[i], bv[j], acc[i][j]);
        }
        if (kt + 1 < nk) store(s ^ 1);
        __syncthreads();
    }

    const int co = n0 + tx * 4;
    if (co >= c.cout) return;
    const float4 bias = c.bias ? *reinterpret_cast<const float4 *>(c.bias + co) : make_float4(0.f, 0.f, 0.f, 0.f);
    const int Rr = c.res_upsample ? (R >> 1) : R;
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int64_t m = m0 + ty * 8 + i;
        if (m >= M) break;
        const int64_t b = m / hw;
        const int pix = (int)(m % hw);
        float4 v = make_float4(c.alpha * (acc[i][0] + bias.x), c.alpha * (acc[i][1] + bias.y), c.alpha * (acc[i][2] + bias.z),
                               c.alpha * (acc[i][3] + bias.w));
        if (c.res) {
            const int y = pix / R, x = pix % R;
            const int yr = c.res_upsample ? (y >> 1) : y, xr = c.res_upsample ? (x >> 1) : x;
            const float4 r = *reinterpret_cast<const float4 *>(c.res + ((b * Rr + yr) * Rr + xr) * c.ldres + co);
            v.x += r.x; v.y += r.y; v.z += r.z; v.w += r.w;
        }
        *reinterpret_cast<float4 *>(c.out + m * c.ldo + co) = v;
    }
}

// ---- conditional BatchNorm rows and tables --------------------------------------------------------------------------------
// The rows s = cond_b . Ws[ch] and o = cond_b . Wo[ch] of one (sample, channel), reduced across the calling warp: lane-strided
// fmaf over k, then warp_sum.  Every kernel that forms these rows calls this, so the fused tables and the tables built from
// materialised rows hold the same bits.
__device__ __forceinline__ float2 bb_cond_rows(const float *__restrict__ cond_b, const float *__restrict__ ws_ch,
                                               const float *__restrict__ wo_ch, int cdim, int lane) {
    float s = 0.f, o = 0.f;
    for (int k = lane; k < cdim; k += 32) {
        const float z = cond_b[k];
        s = fmaf(z, ws_ch[k], s);
        o = fmaf(z, wo_ch[k], o);
    }
    return make_float2(warp_sum(s), warp_sum(o));
}

// scale[b, ch] = (1 + cond_b . Ws[ch]) / sqrt(var[ch] + eps),  offset[b, ch] = cond_b . Wo[ch]   (one warp per (b, ch))
__global__ void __launch_bounds__(256)
bb_bn_table_kernel(const float *__restrict__ cond, int64_t n, int cdim, const float *__restrict__ ws, const float *__restrict__ wo,
                   const float *__restrict__ var, float eps, int C, float *__restrict__ scale, float *__restrict__ offset) {
    const int64_t w = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (w >= n * C) return;
    const int64_t b = w / C;
    const int ch = (int)(w % C);
    const float2 r = bb_cond_rows(cond + b * cdim, ws + (int64_t)ch * cdim, wo + (int64_t)ch * cdim, cdim, lane);
    if (lane == 0) {
        scale[w] = (1.f + r.x) / sqrtf(var[ch] + eps);
        offset[w] = r.y;
    }
}

// The rows of up to GSB_BIGGAN_BN_ROWS_MAX BatchNorms of one block in one launch: one warp per (b, channel of the concatenated
// [C_0 | C_1 | ...]), s and o written to the BatchNorm's own [n, C_j] outputs.
struct bb_bn_rows_args {
    gsb_biggan_bn_rows_desc d[GSB_BIGGAN_BN_ROWS_MAX];
    int64_t start[GSB_BIGGAN_BN_ROWS_MAX + 1];     // prefix sums of the widths
    int count;
};

__global__ void __launch_bounds__(256)
bb_bn_rows_kernel(const float *__restrict__ cond, int64_t n, int cdim, const bb_bn_rows_args a) {
    const int64_t w = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    const int64_t total = a.start[a.count];
    if (w >= n * total) return;
    const int64_t b = w / total;
    const int64_t g = w % total;
    int j = 0;
    while (g >= a.start[j + 1]) ++j;
    const gsb_biggan_bn_rows_desc &d = a.d[j];
    const int ch = (int)(g - a.start[j]);
    const float2 r = bb_cond_rows(cond + b * cdim, d.w_scale + (int64_t)ch * cdim, d.w_offset + (int64_t)ch * cdim, cdim, lane);
    if (lane == 0) {
        d.scale_rows[b * d.c + ch] = r.x;
        d.offset_rows[b * d.c + ch] = r.y;
    }
}

// tables from given rows: scale[b, ch] = (1 + s[b, ch]) / sqrt(var[ch] + eps), offset[b, ch] = o[b, ch]; row b of s at s + b ld_s
// (ld_s = 0: one row for every sample), likewise o.  One thread per element.
__global__ void __launch_bounds__(256)
bb_bn_table_rows_kernel(const float *__restrict__ s, int64_t ld_s, const float *__restrict__ o, int64_t ld_o, int64_t n,
                        const float *__restrict__ var, float eps, int C, float *__restrict__ scale, float *__restrict__ offset) {
    const int64_t i = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (i >= n * C) return;
    const int64_t b = i / C;
    const int ch = (int)(i % C);
    scale[i] = (1.f + s[b * ld_s + ch]) / sqrtf(var[ch] + eps);
    offset[i] = o[b * ld_o + ch];
}

// ---- SelfAttn: 2x2 max-pool of phi (written K-major for the score product) and g -------------------------------------------
// tpg [n, R, R, C/8 (theta) | C/8 (phi) | C/2 (g)] -> phi_t [n, C/8, (R/2)^2], g [n, (R/2)^2, C/2]
__global__ void __launch_bounds__(256)
bb_attn_pool_kernel(const float *__restrict__ tpg, int64_t n, int R, int C, float *__restrict__ phi_t, float *__restrict__ g) {
    const int c8 = C / 8, c2 = C / 2, ct = c8 + c8 + c2, ch = c8 + c2, Rp = R / 2, hwp = Rp * Rp;
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= n * hwp * ch) return;
    const int k = (int)(idx % ch);
    const int64_t q = idx / ch;
    const int p = (int)(q % hwp);
    const int64_t b = q / hwp;
    const int y = 2 * (p / Rp), x = 2 * (p % Rp);
    const float *s = tpg + ((b * R + y) * R + x) * (int64_t)ct + c8 + k;
    const float v = fmaxf(fmaxf(s[0], s[ct]), fmaxf(s[(int64_t)R * ct], s[(int64_t)R * ct + ct]));
    if (k < c8) phi_t[(b * c8 + k) * hwp + p] = v;
    else g[(b * hwp + p) * c2 + (k - c8)] = v;
}

// ---- SelfAttn: softmax over the keys, in place, one warp per query row (fixed reduction order) ----------------------------
__global__ void __launch_bounds__(256)
bb_softmax_rows_kernel(float *__restrict__ s, int64_t rows, int cols) {
    const int64_t row = blockIdx.x * (int64_t)(blockDim.x >> 5) + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (row >= rows) return;
    float *r = s + row * cols;
    float mx = -INFINITY;
    for (int k = lane; k < cols; k += 32) mx = fmaxf(mx, r[k]);
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
    for (int k = lane; k < cols; k += 32) sum += expf(r[k] - mx);
    sum = warp_sum(sum);
    for (int k = lane; k < cols; k += 32) r[k] = expf(r[k] - mx) / sum;
}

// ---- tail: BN (per-channel affine) -> ReLU -> 3x3 conv to the 3 kept channels -> tanh -> 0.5 (x + 1) ----------------------
// one thread per output pixel; weight [3, C, 3, 3] (the first three output channels of conv_to_rgb), image NHWC [n, R, R, 3]
constexpr int BB_RGB_MAX_C = 256;
__global__ void __launch_bounds__(128)
bb_rgb_kernel(const float *__restrict__ x, int64_t n, int R, int C, const float *__restrict__ mean, const float *__restrict__ scale,
              const float *__restrict__ offset, const float *__restrict__ weight, const float *__restrict__ bias, float *__restrict__ img) {
    __shared__ float wsm[9][BB_RGB_MAX_C][3];
    __shared__ float aff[3][BB_RGB_MAX_C];
    for (int i = threadIdx.x; i < 3 * C * 9; i += blockDim.x) {
        const int o = i / (C * 9), ci = (i / 9) % C, t = i % 9;
        wsm[t][ci][o] = weight[i];
    }
    for (int i = threadIdx.x; i < C; i += blockDim.x) { aff[0][i] = mean[i]; aff[1][i] = scale[i]; aff[2][i] = offset[i]; }
    __syncthreads();
    const int64_t idx = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (idx >= n * R * R) return;
    const int pix = (int)(idx % ((int64_t)R * R));
    const int64_t b = idx / ((int64_t)R * R);
    const int y = pix / R, xq = pix % R;
    float acc[3] = {0.f, 0.f, 0.f};
    for (int t = 0; t < 9; ++t) {
        const int yy = y + t / 3 - 1, xx = xq + t % 3 - 1;
        if (yy < 0 || yy >= R || xx < 0 || xx >= R) continue;
        const float *p = x + ((b * R + yy) * R + xx) * (int64_t)C;
        for (int ci = 0; ci < C; ci += 4) {
            const float4 v4 = *reinterpret_cast<const float4 *>(p + ci);
            const float v[4] = {v4.x, v4.y, v4.z, v4.w};
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                float a = (v[j] - aff[0][ci + j]) * aff[1][ci + j] + aff[2][ci + j];
                a = a > 0.f ? a : 0.f;
#pragma unroll
                for (int o = 0; o < 3; ++o) acc[o] = fmaf(a, wsm[t][ci + j][o], acc[o]);
            }
        }
    }
#pragma unroll
    for (int o = 0; o < 3; ++o) img[idx * 3 + o] = 0.5f * (tanhf(acc[o] + bias[o]) + 1.f);
}

}  // namespace gsb

extern "C" int gsb_biggan_conv_forward(const gsb_biggan_conv *c, int64_t n, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(c && c->x && c->weight && c->out && n >= 0, "biggan_conv: null pointer");
    GSB_CHECK_ARG((c->ksize == 1 || c->ksize == 3) && c->cin % BB_BK == 0 && c->cin > 0 && c->cout % 4 == 0 && c->cout > 0 &&
                      c->res_in > 0 && c->ldx % 4 == 0 && c->ldx >= c->cin && c->ldo % 4 == 0 && c->ldo >= c->cout,
                  "biggan_conv: need ksize 1|3, cin%%16 == 0, cout%%4 == 0, ld%%4 == 0 (ksize=%d cin=%d cout=%d)", c->ksize, c->cin,
                  c->cout);
    GSB_CHECK_ARG(!c->res || (c->ldres % 4 == 0 && c->ldres >= c->cout), "biggan_conv: bad ldres");
    GSB_CHECK_ARG(!c->bn_mean || (c->bn_scale && c->bn_offset), "biggan_conv: incomplete BN prologue");
    const int R = c->upsample ? 2 * c->res_in : c->res_in;
    GSB_CHECK_ARG(!c->w_sample_stride || ((int64_t)R * R) % BB_BM == 0,
                  "biggan_conv: per-sample weights need a multiple of %d output pixels per sample", BB_BM);
    GSB_CHECK_ARG(!c->res_upsample || R % 2 == 0, "biggan_conv: res_upsample needs an even resolution");
    if (n == 0) return GSB_OK;
    const int64_t M = n * R * R;
    const dim3 grid((unsigned)((M + BB_BM - 1) / BB_BM), (unsigned)((c->cout + BB_BN - 1) / BB_BN));
    GSB_CHECK_ARG(grid.y <= 65535, "biggan_conv: cout too large");
    cudaStream_t st = (cudaStream_t)stream;
    if (c->bn_mean) bb_conv_kernel<true><<<grid, BB_THREADS, 0, st>>>(*c, n);
    else bb_conv_kernel<false><<<grid, BB_THREADS, 0, st>>>(*c, n);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_biggan_bn_table(const float *d_cond, int64_t n, int cdim, const float *d_w_scale, const float *d_w_offset,
                                   const float *d_var, float eps, int c, float *d_scale, float *d_offset, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_cond && d_w_scale && d_w_offset && d_var && d_scale && d_offset && n >= 0 && cdim > 0 && c > 0,
                  "biggan_bn_table: bad argument");
    if (n == 0) return GSB_OK;
    const int64_t warps = n * c;
    bb_bn_table_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, (cudaStream_t)stream>>>(d_cond, n, cdim, d_w_scale, d_w_offset, d_var,
                                                                                     eps, c, d_scale, d_offset);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_biggan_bn_rows(const float *d_cond, int64_t n, int cdim, const gsb_biggan_bn_rows_desc *descs, int count,
                                  gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_cond && descs && n >= 0 && cdim > 0 && count >= 1 && count <= GSB_BIGGAN_BN_ROWS_MAX,
                  "biggan_bn_rows: bad argument (count=%d, at most %d)", count, GSB_BIGGAN_BN_ROWS_MAX);
    bb_bn_rows_args a;
    a.count = count;
    a.start[0] = 0;
    for (int j = 0; j < count; ++j) {
        const gsb_biggan_bn_rows_desc &d = descs[j];
        GSB_CHECK_ARG(d.w_scale && d.w_offset && d.scale_rows && d.offset_rows && d.c > 0, "biggan_bn_rows: bad descriptor %d", j);
        a.d[j] = d;
        a.start[j + 1] = a.start[j] + d.c;
    }
    if (n == 0) return GSB_OK;
    const int64_t warps = n * a.start[count];
    bb_bn_rows_kernel<<<(unsigned)((warps + 7) / 8), 256, 0, (cudaStream_t)stream>>>(d_cond, n, cdim, a);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_biggan_bn_table_rows(const float *d_scale_rows, int64_t ld_scale_rows, const float *d_offset_rows,
                                        int64_t ld_offset_rows, int64_t n, const float *d_var, float eps, int c, float *d_scale,
                                        float *d_offset, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_scale_rows && d_offset_rows && d_var && d_scale && d_offset && n >= 0 && c > 0 &&
                      (ld_scale_rows == 0 || ld_scale_rows >= c) && (ld_offset_rows == 0 || ld_offset_rows >= c),
                  "biggan_bn_table_rows: bad argument (c=%d, ld=%lld, %lld)", c, (long long)ld_scale_rows, (long long)ld_offset_rows);
    if (n == 0) return GSB_OK;
    const int64_t total = n * c;
    bb_bn_table_rows_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(
        d_scale_rows, ld_scale_rows, d_offset_rows, ld_offset_rows, n, d_var, eps, c, d_scale, d_offset);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_biggan_attn_pool(const float *d_tpg, int64_t n, int res, int c, float *d_phi_t, float *d_g, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_tpg && d_phi_t && d_g && n >= 0 && res % 2 == 0 && c % 8 == 0, "biggan_attn_pool: bad argument");
    if (n == 0) return GSB_OK;
    const int64_t total = n * (int64_t)(res / 2) * (res / 2) * (c / 8 + c / 2);
    bb_attn_pool_kernel<<<(unsigned)((total + 255) / 256), 256, 0, (cudaStream_t)stream>>>(d_tpg, n, res, c, d_phi_t, d_g);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_biggan_softmax_rows(float *d_s, int64_t rows, int cols, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_s && rows >= 0 && cols > 0, "biggan_softmax_rows: bad argument");
    if (rows == 0) return GSB_OK;
    bb_softmax_rows_kernel<<<(unsigned)((rows + 7) / 8), 256, 0, (cudaStream_t)stream>>>(d_s, rows, cols);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_biggan_rgb(const float *d_x, int64_t n, int res, int c, const float *d_mean, const float *d_scale,
                              const float *d_offset, const float *d_weight, const float *d_bias, float *d_img, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_x && d_mean && d_scale && d_offset && d_weight && d_bias && d_img && n >= 0 && res > 0,
                  "biggan_rgb: null pointer");
    GSB_CHECK_ARG(c % 4 == 0 && c > 0 && c <= BB_RGB_MAX_C, "biggan_rgb: need c%%4 == 0 and c <= %d (c=%d)", BB_RGB_MAX_C, c);
    if (n == 0) return GSB_OK;
    const int64_t total = n * (int64_t)res * res;
    bb_rgb_kernel<<<(unsigned)((total + 127) / 128), 128, 0, (cudaStream_t)stream>>>(d_x, n, res, c, d_mean, d_scale, d_offset, d_weight,
                                                                                    d_bias, d_img);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}
