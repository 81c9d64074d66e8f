// Incremental-PCA chain, large-d engine (d up to ~10^6 features: conv feature maps, BASELINE config 5).
//
// Replaces estimators.py:55-81 (IPCAEstimator.fit_partial / get_components) -> scikit-learn
// IncrementalPCA.partial_fit (_incremental_pca.py:254-380) when the d x d Gram of the small-d engine (ipca.cu) is out
// of reach (d = 524,288 -> 2 TB).  sklearn stacks
//        M = [ S * Vt            (c rows:  singular_values_ * components_)
//              X - mean_b        (n_b rows: the centred batch)
//              sqrt(n_seen n_b / n_tot) (mean - mean_b) ]          (1 row)
// and takes the top-c right singular vectors of M.  Here M (fp32, [c + n_b + 1, d]) stays in HBM -- the producer
// (synthesis.cu) writes the batch rows in place -- and the SVD goes through the SMALL side:
//        T = M M^T  (n_s x n_s, n_s = c + n_b + 1 ~ 2100; fp32 products summed in fp32 over 8192-long chunks of d,
//                    chunks accumulated in fp64)
//        T = U diag(lambda) U^T  (top c; fp64 direct solver: L2-resident Householder tridiagonalisation, bisection,
//                    inverse iteration (eig.cu))
//        S_new = sqrt(lambda),   (S * Vt)_new = U^T M      (one skinny GEMM over M; rows 0..c-1 of M for the next step)
// followed by sklearn's svd_flip sign rule on the rows and the Chan mean / variance merge per feature
// (extmath._incremental_mean_and_var).  Nothing of size d x d or n_b x d ever leaves the device.
#include "eig.cuh"
#include "tc_common.cuh"
#include <math.h>

namespace gsb {

constexpr int BD_HDR = 4;
constexpr int BD_KCHUNK = 8192;

static inline int bigd_rows(int c, int nb_max) { return (c + nb_max + 1 + 31) / 32 * 32; }

struct BigState { double *hdr, *mean, *unnorm, *S; };
static BigState big_state(void *p, int64_t d, int c) {
    BigState s;
    s.hdr = reinterpret_cast<double *>(p);
    s.mean = s.hdr + BD_HDR;
    s.unnorm = s.mean + d;
    s.S = s.unnorm + d;
    return s;
}

struct BigWs {
    Workspace ew;          // ew.A doubles as T; ew.evecs (U) and ew.lam carry the solve over to the commit
    double *mean_b;
    float *Dnew, *rowmax;
    void *tc;              // operands of the tensor-core Gram (flags & GSB_BIGD_GRAM_TC)
    size_t bytes;
};
static BigWs big_ws(void *base, int64_t d, int c, int nb_max, int flags) {
    BigWs w;
    const int np = bigd_rows(c, nb_max);
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    const size_t eb = carve(nullptr, np, c).bytes;
    w.ew = carve(take(eb), np, c);
    w.mean_b = (double *)take((size_t)d * 8);
    w.Dnew = (float *)take((size_t)c * d * 4);
    w.rowmax = (float *)take((size_t)2 * c * 4);
    w.tc = ((flags & GSB_BIGD_GRAM_TC) && gram_tc_supported(d)) ? take(gram_tc_workspace_bytes(np, d)) : nullptr;
    w.bytes = off;
    return w;
}

// ---------------------------------------------------------------------------------------------
// per-feature pass: batch mean, centring in place, batch sum of squares, mean-correction row, Chan merge
// (_incremental_pca.py:327-347, extmath.py:1118-1265).  One thread per feature; warps read 128 contiguous bytes per row.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256)
bigd_center_kernel(float *__restrict__ M, int64_t d, int c, int nb, int n_pad, double n_seen, double *__restrict__ mean,
                   double *__restrict__ unnorm, double *__restrict__ mean_b) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= d) return;
    float *col = M + (size_t)c * d + j;
    double s0 = 0.0, s1 = 0.0, s2 = 0.0, s3 = 0.0;
    int r = 0;
    for (; r + 4 <= nb; r += 4) {
        s0 += (double)col[(size_t)r * d];
        s1 += (double)col[(size_t)(r + 1) * d];
        s2 += (double)col[(size_t)(r + 2) * d];
        s3 += (double)col[(size_t)(r + 3) * d];
    }
    for (; r < nb; ++r) s0 += (double)col[(size_t)r * d];
    const double n_b = (double)nb;
    const double mb = ((s0 + s1) + (s2 + s3)) / n_b;
    double q0 = 0.0, q1 = 0.0;
    r = 0;
    for (; r + 2 <= nb; r += 2) {
        const double d0 = (double)col[(size_t)r * d] - mb, d1 = (double)col[(size_t)(r + 1) * d] - mb;
        q0 += d0 * d0; q1 += d1 * d1;
        col[(size_t)r * d] = (float)d0;                    // X -= col_batch_mean (float32 array -= float64 vector)
        col[(size_t)(r + 1) * d] = (float)d1;
    }
    for (; r < nb; ++r) {
        const double d0 = (double)col[(size_t)r * d] - mb;
        q0 += d0 * d0;
        col[(size_t)r * d] = (float)d0;
    }
    const double ss = q0 + q1;
    float corr = 0.f;
    if (n_seen > 0) {
        const double n_tot = n_seen + n_b, mo = mean[j];
        corr = (float)(sqrt((n_seen / n_tot) * n_b) * (mo - mb));                 // mean_correction (:340-343)
        mean[j] = (mo * n_seen + mb * n_b) / n_tot;
        const double ratio = n_seen / n_b;
        const double tq = (mo * n_seen) / ratio - mb * n_b;
        unnorm[j] = unnorm[j] + ss + ratio / n_tot * tq * tq;
    } else {
        mean[j] = mb;
        unnorm[j] = ss;
    }
    M[(size_t)(c + nb) * d + j] = corr;
    for (int rr = c + nb + 1; rr < n_pad; ++rr) M[(size_t)rr * d + j] = 0.f;
    mean_b[j] = mb;
}

// ---------------------------------------------------------------------------------------------
// T += M[:, k-chunk] M[:, k-chunk]^T   (upper tile pairs; mirrored on the fly).  128 x 128 x 16 tiles, 8 x 8 per thread.
// ---------------------------------------------------------------------------------------------
constexpr int GB = 128, GK = 16;
__global__ void __launch_bounds__(256, 2)
bigd_gram_kernel(const float *__restrict__ M, int n_rows, int64_t d, int kchunk, double *__restrict__ T, int ldt) {
    __shared__ __align__(16) float As[2][GK][GB + 4];
    __shared__ __align__(16) float Bs[2][GK][GB + 4];
    const int tid = threadIdx.x;
    const int nt = (n_rows + GB - 1) / GB;
    int ti = 0, rem = blockIdx.x;
    while (rem >= nt - ti) { rem -= nt - ti; ++ti; }
    const int tj = ti + rem;
    const int m0 = ti * GB, n0 = tj * GB;
    const int64_t kbeg = (int64_t)blockIdx.y * kchunk;
    const int64_t kend = (kbeg + kchunk < d) ? kbeg + kchunk : d;
    const int tx = tid & 15, ty = tid >> 4;
    const int lr = tid >> 2, lk = (tid & 3) * 4;
    float acc[8][8];
#pragma unroll
    for (int i = 0; i < 8; ++i)
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[i][j] = 0.f;
    float4 ra[2], rb[2];
    auto gload = [&](int64_t k0) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = lr + 64 * h;
            ra[h] = (m0 + r < n_rows) ? *reinterpret_cast<const float4 *>(M + (size_t)(m0 + r) * d + k0 + lk) : make_float4(0.f, 0.f, 0.f, 0.f);
            rb[h] = (n0 + r < n_rows) ? *reinterpret_cast<const float4 *>(M + (size_t)(n0 + r) * d + k0 + lk) : make_float4(0.f, 0.f, 0.f, 0.f);
        }
    };
    auto sstore = [&](int buf) {
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int r = lr + 64 * h;
            As[buf][lk + 0][r] = ra[h].x; As[buf][lk + 1][r] = ra[h].y; As[buf][lk + 2][r] = ra[h].z; As[buf][lk + 3][r] = ra[h].w;
            Bs[buf][lk + 0][r] = rb[h].x; Bs[buf][lk + 1][r] = rb[h].y; Bs[buf][lk + 2][r] = rb[h].z; Bs[buf][lk + 3][r] = rb[h].w;
        }
    };
    gload(kbeg);
    sstore(0);
    __syncthreads();
    const int nk = (int)((kend - kbeg) / GK);
    for (int kt = 0; kt < nk; ++kt) {
        const int buf = kt & 1;
        if (kt + 1 < nk) gload(kbeg + (int64_t)(kt + 1) * GK);
#pragma unroll
        for (int k = 0; k < GK; ++k) {
            const float4 a0 = *reinterpret_cast<const float4 *>(&As[buf][k][ty * 4]);
            const float4 a1 = *reinterpret_cast<const float4 *>(&As[buf][k][64 + ty * 4]);
            const float4 b0 = *reinterpret_cast<const float4 *>(&Bs[buf][k][tx * 4]);
            const float4 b1 = *reinterpret_cast<const float4 *>(&Bs[buf][k][64 + tx * 4]);
            const float a[8] = {a0.x, a0.y, a0.z, a0.w, a1.x, a1.y, a1.z, a1.w};
            const float b[8] = {b0.x, b0.y, b0.z, b0.w, b1.x, b1.y, b1.z, b1.w};
#pragma unroll
            for (int i = 0; i < 8; ++i)
#pragma unroll
                for (int j = 0; j < 8; ++j) acc[i][j] = fmaf(a[i], b[j], acc[i][j]);
        }
        if (kt + 1 < nk) {
            sstore(buf ^ 1);
            __syncthreads();
        }
    }
#pragma unroll
    for (int i = 0; i < 8; ++i) {
        const int gm = m0 + ((i < 4) ? (ty * 4 + i) : (64 + ty * 4 + i - 4));
        if (gm >= n_rows) continue;
#pragma unroll
        for (int j = 0; j < 8; ++j) {
            const int gn = n0 + ((j < 4) ? (tx * 4 + j) : (64 + tx * 4 + j - 4));
            if (gn >= n_rows) continue;
            const double v = (double)acc[i][j];
            atomicAdd(&T[(size_t)gm * ldt + gn], v);
            if (ti != tj) atomicAdd(&T[(size_t)gn * ldt + gm], v);
        }
    }
}

// ---------------------------------------------------------------------------------------------
// Dnew[t, j] = sum_r U[t, r] M[r, j]     (c <= 128 rows out; one CTA per 128 features, 32-row slabs of M)
// ---------------------------------------------------------------------------------------------
constexpr int PJ_COLS = 128, PJ_SLAB = 32, PJ_CMAX = 128;
__global__ void __launch_bounds__(256)
bigd_project_kernel(const double *__restrict__ U, int ldu, const float *__restrict__ M, int n_rows, int64_t d, int c,
                    float *__restrict__ Dnew) {
    __shared__ __align__(16) float Ms[PJ_SLAB][PJ_COLS];
    __shared__ float Us[PJ_SLAB][PJ_CMAX + 1];
    const int tid = threadIdx.x, tx = tid & 31, ty = tid >> 5;         // tx: 4 features; ty: components ty, ty+8, ...
    const int64_t j0 = (int64_t)blockIdx.x * PJ_COLS;
    float acc[16][4];
#pragma unroll
    for (int i = 0; i < 16; ++i)
#pragma unroll
        for (int q = 0; q < 4; ++q) acc[i][q] = 0.f;
    for (int r0 = 0; r0 < n_rows; r0 += PJ_SLAB) {
        for (int idx = tid; idx < PJ_SLAB * (PJ_COLS / 4); idx += 256) {
            const int rr = idx / (PJ_COLS / 4), q4 = idx % (PJ_COLS / 4);
            const int r = r0 + rr;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r < n_rows && j0 + 4 * q4 < d) v = *reinterpret_cast<const float4 *>(M + (size_t)r * d + j0 + 4 * q4);
            *reinterpret_cast<float4 *>(&Ms[rr][4 * q4]) = v;
        }
        for (int idx = tid; idx < PJ_SLAB * PJ_CMAX; idx += 256) {
            const int t = idx / PJ_SLAB, rr = idx % PJ_SLAB;               // consecutive threads read consecutive r of U[t, :]
            const int r = r0 + rr;
            Us[rr][t] = (t < c && r < n_rows) ? (float)U[(size_t)t * ldu + r] : 0.f;
        }
        __syncthreads();
#pragma unroll 4
        for (int rr = 0; rr < PJ_SLAB; ++rr) {
            const float4 m = *reinterpret_cast<const float4 *>(&Ms[rr][4 * tx]);
#pragma unroll
            for (int i = 0; i < 16; ++i) {
                const float u = Us[rr][ty + 8 * i];
                acc[i][0] = fmaf(u, m.x, acc[i][0]); acc[i][1] = fmaf(u, m.y, acc[i][1]);
                acc[i][2] = fmaf(u, m.z, acc[i][2]); acc[i][3] = fmaf(u, m.w, acc[i][3]);
            }
        }
        __syncthreads();
    }
    const int64_t j = j0 + 4 * tx;
    if (j >= d) return;
#pragma unroll
    for (int i = 0; i < 16; ++i) {
        const int t = ty + 8 * i;
        if (t < c) *reinterpret_cast<float4 *>(Dnew + (size_t)t * d + j) = make_float4(acc[i][0], acc[i][1], acc[i][2], acc[i][3]);
    }
}

// svd_flip (u_based_decision=False): the entry of largest magnitude of every row becomes positive (first index on
// ties).  Phase 1: rowmax[t] = (max |.|, its signed value) over this device's features.  One CTA per row.
__global__ void __launch_bounds__(1024)
bigd_rowmax_kernel(const float *__restrict__ Dnew, int64_t d, float *__restrict__ rowmax) {
    __shared__ float s_best[32];
    __shared__ float s_val[32];
    __shared__ long long s_idx[32];
    const int t = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const float *row = Dnew + (size_t)t * d;
    float best = -1.f, bval = 0.f;
    long long bi = 0;
    for (int64_t i = tid; i < d; i += 1024) {
        const float v = row[i], av = fabsf(v);
        if (av > best) { best = av; bval = v; bi = i; }
    }
    warp_argmax_abs(best, bi, bval);
    if (lane == 0) { s_best[warp] = best; s_val[warp] = bval; s_idx[warp] = bi; }
    __syncthreads();
    if (warp == 0) {
        best = s_best[lane]; bval = s_val[lane]; bi = s_idx[lane];
        warp_argmax_abs(best, bi, bval);
        if (lane == 0) { rowmax[2 * t] = best; rowmax[2 * t + 1] = bval; }
    }
}
// Phase 2: rows [0, c) of M <- sign * Dnew, S = sqrt(lambda).  `signs` == nullptr: the sign of this device's own
// row maximum (single GPU); otherwise the signs agreed across the feature shards.
__global__ void __launch_bounds__(1024)
bigd_commit_kernel(const float *__restrict__ Dnew, int64_t d, const double *__restrict__ lam, const float *__restrict__ rowmax,
                   const float *__restrict__ signs, float *__restrict__ M, double *__restrict__ S, double *__restrict__ hdr,
                   double n_tot) {
    const int t = blockIdx.x, tid = threadIdx.x;
    const float sgn = signs ? ((signs[t] < 0.f) ? -1.f : 1.f) : ((rowmax[2 * t + 1] < 0.f) ? -1.f : 1.f);
    const float *row = Dnew + (size_t)t * d;
    float *dst = M + (size_t)t * d;
    for (int64_t i = tid; i < d; i += 1024) dst[i] = sgn * row[i];
    if (tid == 0) {
        S[t] = sqrt(fmax(lam[t], 0.0));
        if (t == 0) { hdr[0] = n_tot; hdr[1] += 1.0; }
    }
}

__global__ void bigd_export_comp_kernel(const float *__restrict__ M, const double *__restrict__ S, int64_t d, int c,
                                        float *__restrict__ comp) {
    const int t = blockIdx.y;
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= d) return;
    const double s = S[t];
    comp[(size_t)t * d + j] = (s > 0.0) ? (float)((double)M[(size_t)t * d + j] / s) : 0.f;
}
__global__ void bigd_export_vec_kernel(const double *__restrict__ mean, const double *__restrict__ unnorm, int64_t d, double n_seen,
                                       double *__restrict__ o_mean, double *__restrict__ o_var) {
    const int64_t j = blockIdx.x * (int64_t)blockDim.x + threadIdx.x;
    if (j >= d) return;
    if (o_mean) o_mean[j] = mean[j];
    if (o_var) o_var[j] = unnorm[j] / n_seen;
}
__global__ void __launch_bounds__(1024)
bigd_export_small_kernel(const double *__restrict__ unnorm, const double *__restrict__ S, int64_t d, int c, double n_seen,
                         double *o_sv, double *o_ev, double *o_evr) {
    __shared__ double red[64];
    double part = 0.0;
    for (int64_t i = threadIdx.x; i < d; i += blockDim.x) part += unnorm[i];
    const double tot = block_sum(part, red);
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        const double s = S[i];
        if (o_sv) o_sv[i] = s;
        if (o_ev) o_ev[i] = s * s / (n_seen - 1.0);
        if (o_evr) o_evr[i] = s * s / tot;
    }
}

// NHWC -> NCHW of whole rows: dst[r][ch * hw + p] = src[r][p * c + ch].  Each row is an [hw, c] matrix transposed through a
// 32 x 33 shared-memory tile (the extra column keeps the column reads free of bank conflicts): one CTA per (channel tile,
// pixel tile, row), 32-lane reads along the channels of a pixel and 32-lane writes along the pixels of a channel, both
// coalesced.  A pure copy: the output holds the input's bits.
constexpr int TP_TILE = 32, TP_ROWS = 8;
template <typename T>
__global__ void __launch_bounds__(TP_TILE * TP_ROWS)
nhwc_to_nchw_kernel(const T *__restrict__ src, int64_t ld_src, T *__restrict__ dst, int64_t ld_dst, int hw, int c) {
    __shared__ T tile[TP_TILE][TP_TILE + 1];
    const int64_t r = blockIdx.z;
    const int ch0 = blockIdx.x * TP_TILE, p0 = blockIdx.y * TP_TILE;
    const T *s = src + r * ld_src;
    T *o = dst + r * ld_dst;
    for (int i = threadIdx.y; i < TP_TILE; i += TP_ROWS) {
        const int p = p0 + i, ch = ch0 + threadIdx.x;
        if (p < hw && ch < c) tile[i][threadIdx.x] = s[(int64_t)p * c + ch];
    }
    __syncthreads();
    for (int i = threadIdx.y; i < TP_TILE; i += TP_ROWS) {
        const int ch = ch0 + i, p = p0 + threadIdx.x;
        if (p < hw && ch < c) o[(int64_t)ch * hw + p] = tile[threadIdx.x][i];
    }
}

static int bigd_check(int64_t d, int c, int nb_max) {
    GSB_CHECK_ARG(d >= 1024 && d % 16 == 0 && d < (1ll << 31), "bigd: need d >= 1024, d %% 16 == 0 (d=%lld)", (long long)d);
    GSB_CHECK_ARG(c >= 1 && c <= PJ_CMAX, "bigd: need 1 <= c <= %d (c=%d)", PJ_CMAX, c);
    GSB_CHECK_ARG(nb_max >= 1 && bigd_rows(c, nb_max) <= 4096, "bigd: c + nb_max + 1 must be <= 4096 (nb_max=%d)", nb_max);
    return GSB_OK;
}

}  // namespace gsb

extern "C" int gsb_bigd_rows(int c, int nb_max) { return gsb::bigd_rows(c, nb_max); }

extern "C" size_t gsb_bigd_state_bytes(int64_t d, int c) { return (size_t)(gsb::BD_HDR + 2 * (size_t)d + c) * sizeof(double); }

extern "C" size_t gsb_bigd_workspace_bytes(int64_t d, int c, int nb_max, int flags) {
    if (gsb::bigd_check(d, c, nb_max)) return 0;
    return gsb::big_ws(nullptr, d, c, nb_max, flags).bytes;
}

extern "C" int gsb_bigd_reset(void *d_state, float *d_M, int64_t d, int c, int nb_max, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && d_M, "bigd_reset: null pointer");
    if (int r = gsb::bigd_check(d, c, nb_max)) return r;
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CHECK_CUDA(cudaMemsetAsync(d_state, 0, gsb_bigd_state_bytes(d, c), st));
    GSB_CHECK_CUDA(cudaMemsetAsync(d_M, 0, (size_t)gsb::bigd_rows(c, nb_max) * d * sizeof(float), st));
    return GSB_OK;
}

namespace gsb {
struct StepCtx { BigWs w; BigState s; int np, n_rows; cudaStream_t st; };
static int step_ctx(StepCtx &x, void *d_state, float *d_M, int64_t d, int c, int nb_max, int64_t n_seen, int nb, int flags,
                    void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && d_M && d_workspace, "bigd step: null pointer");
    if (int r = bigd_check(d, c, nb_max)) return r;
    GSB_CHECK_ARG(nb >= 1 && nb <= nb_max && n_seen >= 0, "bigd step: bad batch size %d (nb_max=%d)", nb, nb_max);
    GSB_CHECK_ARG(n_seen > 0 || c <= nb, "bigd step: n_components=%d > first batch size %d", c, nb);
    x.w = big_ws(d_workspace, d, c, nb_max, flags);
    if (workspace_bytes < x.w.bytes) { set_error("bigd step: workspace too small (%zu < %zu)", workspace_bytes, x.w.bytes); return GSB_ERR_WORKSPACE; }
    x.s = big_state(d_state, d, c);
    x.np = bigd_rows(c, nb_max);
    x.n_rows = c + nb + 1;
    x.st = (cudaStream_t)stream;
    return GSB_OK;
}
}  // namespace gsb

extern "C" void *gsb_bigd_gram_matrix(void *d_workspace, int64_t d, int c, int nb_max) {
    if (!d_workspace || gsb::bigd_check(d, c, nb_max)) return nullptr;
    return gsb::big_ws(d_workspace, d, c, nb_max, 0).ew.A;         // T is the first block of the workspace for any flags
}

// phase 1: centre the batch rows, update mean / variance, T = M M^T over THIS device's features
extern "C" int gsb_bigd_step_gram(void *d_state, float *d_M, int64_t d, int c, int nb_max, int64_t n_seen, int nb, int flags,
                                  double *d_batch_mean, void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    StepCtx x;
    if (int r = step_ctx(x, d_state, d_M, d, c, nb_max, n_seen, nb, flags, d_workspace, workspace_bytes, stream)) return r;
    bigd_center_kernel<<<(unsigned)((d + 255) / 256), 256, 0, x.st>>>(d_M, d, c, nb, x.np, (double)n_seen, x.s.mean, x.s.unnorm, x.w.mean_b);
    GSB_CHECK_LAUNCH();
    if (d_batch_mean) GSB_CHECK_CUDA(cudaMemcpyAsync(d_batch_mean, x.w.mean_b, (size_t)d * sizeof(double), cudaMemcpyDeviceToDevice, x.st));
    double *T = x.w.ew.A;
    GSB_CHECK_CUDA(cudaMemsetAsync(T, 0, (size_t)x.np * x.np * sizeof(double), x.st));
    if (x.w.tc) return gram_tc(d_M, x.n_rows, x.np, d, x.w.tc, T, x.st);      // tensor cores, promoted accumulator (gram_tc.cu)
    const int nt = (x.n_rows + GB - 1) / GB;
    dim3 grid((unsigned)(nt * (nt + 1) / 2), (unsigned)((d + BD_KCHUNK - 1) / BD_KCHUNK));
    bigd_gram_kernel<<<grid, 256, 0, x.st>>>(d_M, x.n_rows, d, BD_KCHUNK, T, x.np);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// phase 2: top-c eigenpairs of T (summed over the feature shards by the caller), Dnew = U^T M, per-row maxima
extern "C" int gsb_bigd_step_solve(void *d_state, float *d_M, int64_t d, int c, int nb_max, int64_t n_seen, int nb, int flags,
                                   float *d_rowmax, void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    StepCtx x;
    if (int r = step_ctx(x, d_state, d_M, d, c, nb_max, n_seen, nb, flags, d_workspace, workspace_bytes, stream)) return r;
    if (int r = eig_top(x.w.ew, x.np, c, x.w.ew.lam, x.w.ew.evecs, x.st)) return r;      // ew.A holds T (and is destroyed)
    bigd_project_kernel<<<(unsigned)((d + PJ_COLS - 1) / PJ_COLS), 256, 0, x.st>>>(x.w.ew.evecs, x.np, d_M, x.n_rows, d, c, x.w.Dnew);
    GSB_CHECK_LAUNCH();
    bigd_rowmax_kernel<<<c, 1024, 0, x.st>>>(x.w.Dnew, d, x.w.rowmax);
    GSB_CHECK_LAUNCH();
    if (d_rowmax) GSB_CHECK_CUDA(cudaMemcpyAsync(d_rowmax, x.w.rowmax, (size_t)2 * c * sizeof(float), cudaMemcpyDeviceToDevice, x.st));
    return GSB_OK;
}

// phase 3: commit  S*Vt <- sign * Dnew  (d_signs [c], or NULL = this device's own row maxima), S, sample count
extern "C" int gsb_bigd_step_commit(void *d_state, float *d_M, int64_t d, int c, int nb_max, int64_t n_seen, int nb, int flags,
                                    const float *d_signs, void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    using namespace gsb;
    StepCtx x;
    if (int r = step_ctx(x, d_state, d_M, d, c, nb_max, n_seen, nb, flags, d_workspace, workspace_bytes, stream)) return r;
    bigd_commit_kernel<<<c, 1024, 0, x.st>>>(x.w.Dnew, d, x.w.ew.lam, x.w.rowmax, d_signs, d_M, x.s.S, x.s.hdr, (double)(n_seen + nb));
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_bigd_chain_step(void *d_state, float *d_M, int64_t d, int c, int nb_max, int64_t n_seen, int nb, int flags,
                                   double *d_batch_mean, void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    if (int r = gsb_bigd_step_gram(d_state, d_M, d, c, nb_max, n_seen, nb, flags, d_batch_mean, d_workspace, workspace_bytes, stream)) return r;
    if (int r = gsb_bigd_step_solve(d_state, d_M, d, c, nb_max, n_seen, nb, flags, nullptr, d_workspace, workspace_bytes, stream)) return r;
    return gsb_bigd_step_commit(d_state, d_M, d, c, nb_max, n_seen, nb, flags, nullptr, d_workspace, workspace_bytes, stream);
}

extern "C" int gsb_bigd_export(const void *d_state, const float *d_M, int64_t d, int c, int64_t n_seen, float *d_components,
                               double *d_singular_values, double *d_mean, double *d_var, double *d_explained_variance,
                               double *d_explained_variance_ratio, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_state && d_M, "bigd_export: null pointer");
    GSB_CHECK_ARG(n_seen > 1 && c >= 1 && d >= 1, "bigd_export: nothing fitted yet");
    cudaStream_t st = (cudaStream_t)stream;
    BigState s = big_state(const_cast<void *>(d_state), d, c);
    if (d_components) {
        dim3 grid((unsigned)((d + 255) / 256), c);
        bigd_export_comp_kernel<<<grid, 256, 0, st>>>(d_M, s.S, d, c, d_components);
        GSB_CHECK_LAUNCH();
    }
    if (d_mean || d_var) {
        bigd_export_vec_kernel<<<(unsigned)((d + 255) / 256), 256, 0, st>>>(s.mean, s.unnorm, d, (double)n_seen, d_mean, d_var);
        GSB_CHECK_LAUNCH();
    }
    bigd_export_small_kernel<<<1, 1024, 0, st>>>(s.unnorm, s.S, d, c, (double)n_seen, d_singular_values, d_explained_variance,
                                                  d_explained_variance_ratio);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_nhwc_to_nchw_rows(const void *d_src, int64_t ld_src, void *d_dst, int64_t ld_dst, int64_t rows, int hw, int c,
                                     int elem_bytes, gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_src && d_dst && d_src != d_dst, "nhwc_to_nchw_rows: null or aliased pointer");
    GSB_CHECK_ARG(elem_bytes == 4 || elem_bytes == 8, "nhwc_to_nchw_rows: elements of 4 (fp32) or 8 (fp64) bytes (got %d)", elem_bytes);
    GSB_CHECK_ARG(rows >= 0 && rows <= 65535 && hw >= 1 && c >= 1, "nhwc_to_nchw_rows: bad shape (rows=%lld, hw=%d, c=%d)",
                  (long long)rows, hw, c);
    GSB_CHECK_ARG(ld_src >= (int64_t)hw * c && ld_dst >= (int64_t)hw * c, "nhwc_to_nchw_rows: row pitch below hw * c");
    if (rows == 0) return GSB_OK;
    dim3 grid((unsigned)((c + TP_TILE - 1) / TP_TILE), (unsigned)((hw + TP_TILE - 1) / TP_TILE), (unsigned)rows);
    GSB_CHECK_ARG(grid.y <= 65535, "nhwc_to_nchw_rows: hw = %d has too many pixel tiles", hw);
    if (elem_bytes == 4)
        nhwc_to_nchw_kernel<float><<<grid, dim3(TP_TILE, TP_ROWS), 0, (cudaStream_t)stream>>>(
            static_cast<const float *>(d_src), ld_src, static_cast<float *>(d_dst), ld_dst, hw, c);
    else
        nhwc_to_nchw_kernel<double><<<grid, dim3(TP_TILE, TP_ROWS), 0, (cudaStream_t)stream>>>(
            static_cast<const double *>(d_src), ld_src, static_cast<double *>(d_dst), ld_dst, hw, c);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}
