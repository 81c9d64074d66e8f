// Per-group sufficient statistics of the small-d incremental PCA on the Hopper tensor cores (wgmma + TMA).
//
//   mean_g[d]   = (1/nb) sum_r x[g nb + r, :]                          fp64 accumulation of the fp32 samples
//   gram_g[d,d] = sum_r (x[r,:] - mean_g)^T (x[r,:] - mean_g)          fp32-grade products, promoted accumulation
// for G consecutive groups of nb rows in ONE call.  These replace what sklearn's IncrementalPCA.partial_fit reads off a
// batch (estimators.py:68-76 -> _incremental_pca.py:332-357), exactly like stats.cu (the fp32 FMA form, kept for feature
// counts that are not a multiple of 128); the chain (subspace.cu / ipca.cu) consumes them in the reference's group order.
//
// Three kernels per call:
//   colsum_groups_kernel     column sums per (group, 256-row slice) (fp64), coalesced reads; mean_groups_kernel adds the
//                            slices in a fixed order (no atomics: the means are bitwise reproducible) -> mean, mean32
//   center_split_t_kernel    xt[g][c][r] = fp16 hi/lo split of (x[g nb + r][c] - mean32[c]) * 2^e_g (e_g: per-group power of two
//                            that puts 2 max|x| into [8192, 32768), so hi keeps 11 bits and nothing overflows), i.e. the centred samples
//                            TRANSPOSED so that the sample index is the contiguous (K) dimension of both MMA operands
//   gram_tc_kernel           (gram_tc.cu, Store epilogue) the centred Gram of every group: persistent wgmma kernel over
//                            (group, upper 128 x 128 tile pair) work items, 3 MMAs per product, promoted accumulation;
//                            samples beyond nb are zero-filled by the TMA unit (no padding is ever read); each tile is
//                            scaled by 2^-2e and stored (with its mirror image) as fp64.
// Algorithmic work: 2 d^2 FLOP per sample (x3 MMAs); HBM traffic: x read twice (4 B), xt written and read (4 + 4 B per element,
// the re-reads of the 10 tile pairs come out of L2).
#include "tc_common.cuh"
#include <stdlib.h>
#include <string.h>

namespace gsb {

namespace stc {

// ---- column sums per group ----------------------------------------------------------------------------------------
constexpr int SUM_ROWS = 256;               // rows per column-sum slice

// one (column block, row slice, group) block of column sums; part: [G][ny][d]
__device__ __forceinline__ void colsum_groups_body(const float *__restrict__ x, int64_t nb, int d, int64_t ld, int rows_per_cta,
                                                   double *__restrict__ part, float *__restrict__ absmax, int bx, int by, int ny,
                                                   int g) {
    const int col = bx * blockDim.x + threadIdx.x;
    const int64_t r0 = (int64_t)by * rows_per_cta;
    const int64_t r1 = r0 + rows_per_cta < nb ? r0 + rows_per_cta : nb;
    const float *xg = x + (size_t)g * nb * ld;
    double a0 = 0.0, a1 = 0.0;              // fp64 sum of the fp32 samples, as sklearn's _safe_accumulator_op does
    float mx = 0.f;
    if (col < d) {
        int64_t r = r0;
        for (; r + 1 < r1; r += 2) {
            const float v0 = xg[r * ld + col], v1 = xg[(r + 1) * ld + col];
            a0 += (double)v0; a1 += (double)v1;
            mx = fmaxf(mx, fmaxf(fabsf(v0), fabsf(v1)));
        }
        if (r < r1) { const float v0 = xg[r * ld + col]; a0 += (double)v0; mx = fmaxf(mx, fabsf(v0)); }
        part[((size_t)g * ny + by) * d + col] = a0 + a1;
    }
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if ((threadIdx.x & 31) == 0) atomicMax(reinterpret_cast<int *>(absmax + g), __float_as_int(mx));   // mx >= 0: int order == float order
}

__global__ void colsum_groups_kernel(const float *__restrict__ x, int64_t nb, int d, int64_t ld, int rows_per_cta,
                                     double *__restrict__ part /* [G][ny][d] */, float *__restrict__ absmax /* [G], zeroed */) {
    colsum_groups_body(x, nb, d, ld, rows_per_cta, part, absmax, blockIdx.x, blockIdx.y, gridDim.y, blockIdx.z);
}

// mean per (group, feature); scale exponent per group: |x - mean| <= 2 max|x|, and 2 max|x| 2^e lands in [8192, 32768)
__device__ __forceinline__ void mean_groups_body(const double *__restrict__ part, int ny, int n_groups, int d, double nd,
                                                 double *__restrict__ mean, float *__restrict__ mean32, const float *__restrict__ absmax,
                                                 int *__restrict__ exps, int i) {
    if (i < n_groups * d) {
        const int g = i / d, c = i % d;
        double t = 0.0;
        for (int y = 0; y < ny; ++y) t += part[((size_t)g * ny + y) * d + c];
        const double m = t / nd;
        mean[i] = m;
        mean32[i] = (float)m;
    }
    if (i < n_groups) {
        const float a = absmax[i];
        int e = 0;
        if (a > 0.f && a < 1.0e38f) { int ex; frexpf(2.f * a, &ex); e = 14 - ex; }
        exps[i] = e;
    }
}

__global__ void mean_groups_kernel(const double *__restrict__ part, int ny, int n_groups, int d, double nd, double *__restrict__ mean,
                                   float *__restrict__ mean32, const float *__restrict__ absmax, int *__restrict__ exps) {
    mean_groups_body(part, ny, n_groups, d, nd, mean, mean32, absmax, exps, blockIdx.x * blockDim.x + threadIdx.x);
}

// ---- centre, scale, split, transpose ---------------------------------------------------------------------------------
// tile: 64 samples x 64 features; 256 threads.  xt_hi / xt_lo: [G][d][nbp] fp16 (nbp = nb rounded up to 64).
__device__ __forceinline__ void center_split_t_body(const float *__restrict__ x, int64_t nb, int d, int64_t ld, int64_t nbp,
                                                    const float *__restrict__ mean32, const int *__restrict__ exps,
                                                    __half *__restrict__ xt_hi, __half *__restrict__ xt_lo, int bx, int by, int g) {
    __shared__ float tile[64][65];
    const int64_t r0 = (int64_t)bx * 64;
    const int c0 = by * 64;
    const int tid = threadIdx.x;
    const float *xg = x + (size_t)g * nb * ld;
    const float *mg = mean32 + (size_t)g * d;
    {
        const int c4 = (tid & 15) * 4, rr = tid >> 4;
        const float4 m = *reinterpret_cast<const float4 *>(mg + c0 + c4);
        const float sc = ldexpf(1.f, exps[g]);                  // power of two: exact
#pragma unroll
        for (int p = 0; p < 4; ++p) {
            const int r = rr + 16 * p;
            float4 v = make_float4(0.f, 0.f, 0.f, 0.f);
            if (r0 + r < nb) {
                v = *reinterpret_cast<const float4 *>(xg + (r0 + r) * ld + c0 + c4);
                v.x = (v.x - m.x) * sc; v.y = (v.y - m.y) * sc; v.z = (v.z - m.z) * sc; v.w = (v.w - m.w) * sc;
            }
            tile[r][c4] = v.x; tile[r][c4 + 1] = v.y; tile[r][c4 + 2] = v.z; tile[r][c4 + 3] = v.w;
        }
    }
    __syncthreads();
    {
        const int warp = tid >> 5, lane = tid & 31;
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const int c = warp * 8 + q;
            uint32_t hi, lo;
            tc::split2(tile[2 * lane][c], tile[2 * lane + 1][c], hi, lo);
            const size_t o = ((size_t)g * d + c0 + c) * nbp + r0 + 2 * lane;
            *reinterpret_cast<uint32_t *>(xt_hi + o) = hi;
            *reinterpret_cast<uint32_t *>(xt_lo + o) = lo;
        }
    }
}

__global__ void __launch_bounds__(256)
center_split_t_kernel(const float *__restrict__ x, int64_t nb, int d, int64_t ld, int64_t nbp, const float *__restrict__ mean32,
                      const int *__restrict__ exps, __half *__restrict__ xt_hi, __half *__restrict__ xt_lo) {
    center_split_t_body(x, nb, d, ld, nbp, mean32, exps, xt_hi, xt_lo, blockIdx.x, blockIdx.y, blockIdx.z);
}

struct WsView {
    double *sum;
    float *mean32;
    __half *xt_hi, *xt_lo;
    float *absmax;
    int *exps;
    size_t bytes;
};
static WsView carve(void *base, int n_groups, int64_t nb, int d) {
    WsView w;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 1024); return q; };
    const int64_t nbp = (nb + 63) / 64 * 64;
    const int64_t ny = (nb + SUM_ROWS - 1) / SUM_ROWS;
    w.sum = (double *)take((size_t)n_groups * ny * d * sizeof(double));       // column sums per (group, row slice)
    w.absmax = (float *)take((size_t)n_groups * sizeof(float));
    w.exps = (int *)take((size_t)n_groups * sizeof(int));
    w.mean32 = (float *)take((size_t)n_groups * d * sizeof(float));
    w.xt_hi = (__half *)take((size_t)n_groups * d * nbp * 2);
    w.xt_lo = (__half *)take((size_t)n_groups * d * nbp * 2);
    w.bytes = off;
    return w;
}

// ---- grouped: the three preparation kernels for several inputs per launch -------------------------------------------
// Each kernel's blocks are the concatenation of what the plain launches of the descriptors would run, in descriptor order;
// a block finds its descriptor by its first block index and runs the plain kernel's body on the decoded coordinates.
struct PrepDesc {
    const float *x;
    int64_t nb, ld, nbp;
    int d, n_groups, ny;
    double *mean, *sum;
    float *mean32, *absmax;
    int *exps;
    __half *xt_hi, *xt_lo;
    int blk_colsum, blk_mean, blk_center;       // first block of the descriptor in each launch
};
struct PrepParams {
    PrepDesc desc[GRAM_GROUPED_MAX];
    int n_desc;
};

template <int PrepDesc::*FIRST>
__device__ __forceinline__ const PrepDesc &find_desc(const PrepParams &p, int b) {
    int i = 0;
    while (i + 1 < p.n_desc && b >= p.desc[i + 1].*FIRST) ++i;
    return p.desc[i];
}

__global__ void colsum_grouped_kernel(const __grid_constant__ PrepParams p) {
    const PrepDesc &q = find_desc<&PrepDesc::blk_colsum>(p, blockIdx.x);
    const int local = blockIdx.x - q.blk_colsum, gx = (q.d + 127) / 128;
    colsum_groups_body(q.x, q.nb, q.d, q.ld, SUM_ROWS, q.sum, q.absmax, local % gx, (local / gx) % q.ny, q.ny, local / (gx * q.ny));
}

__global__ void mean_grouped_kernel(const __grid_constant__ PrepParams p) {
    const PrepDesc &q = find_desc<&PrepDesc::blk_mean>(p, blockIdx.x);
    const int local = blockIdx.x - q.blk_mean;
    mean_groups_body(q.sum, q.ny, q.n_groups, q.d, (double)q.nb, q.mean, q.mean32, q.absmax, q.exps, local * blockDim.x + threadIdx.x);
}

__global__ void __launch_bounds__(256) center_split_t_grouped_kernel(const __grid_constant__ PrepParams p) {
    const PrepDesc &q = find_desc<&PrepDesc::blk_center>(p, blockIdx.x);
    const int local = blockIdx.x - q.blk_center, gx = (int)(q.nbp / 64), gy = q.d / 64;
    center_split_t_body(q.x, q.nb, q.d, q.ld, q.nbp, q.mean32, q.exps, q.xt_hi, q.xt_lo, local % gx, (local / gx) % gy,
                        local / (gx * gy));
}

// Workspace of one set of grouped launches: the scale maxima of every group first (one memset zeroes them all), then each
// descriptor's column-sum slices, fp32 means and split operands (carve's layout)
static size_t carve_grouped(void *base, const gsb_stats_desc *descs, int n, PrepDesc *out) {
    char *p = reinterpret_cast<char *>(base);
    int total_groups = 0;
    for (int i = 0; i < n; ++i) total_groups += descs[i].n_groups;
    size_t off = align_up((size_t)total_groups * sizeof(float), 1024);
    int g0 = 0;
    for (int i = 0; i < n; ++i) {
        const gsb_stats_desc &s = descs[i];
        WsView w = carve(p ? p + off : nullptr, s.n_groups, s.rows_per_group, s.d);
        if (out) {
            PrepDesc &q = out[i];
            q.x = s.x; q.nb = s.rows_per_group; q.ld = s.ld; q.nbp = (s.rows_per_group + 63) / 64 * 64;
            q.d = s.d; q.n_groups = s.n_groups; q.ny = (int)((s.rows_per_group + SUM_ROWS - 1) / SUM_ROWS);
            q.mean = s.mean_out; q.sum = w.sum; q.mean32 = w.mean32; q.exps = w.exps;
            q.absmax = reinterpret_cast<float *>(p) + g0;
            q.xt_hi = w.xt_hi; q.xt_lo = w.xt_lo;
        }
        g0 += s.n_groups;
        off += w.bytes;
    }
    return off;
}

}  // namespace stc

bool stats_tc_supported(int64_t nb, int d) {
    static int mode = -1;
    if (mode == -1) {
        const char *env = getenv("GANSPACE_B200_STATS");
        mode = (env && strcmp(env, "simt") == 0) ? 0 : 1;
    }
    return mode == 1 && d % 128 == 0 && d >= 128 && d <= 1024 && nb >= 1;
}

size_t stats_tc_workspace_bytes(int n_groups, int64_t nb, int d) { return stc::carve(nullptr, n_groups, nb, d).bytes; }

// mean[G][d], gram[G][d][d] of G consecutive groups of nb rows of x (row stride ld)
int stats_tc(const float *x, int n_groups, int64_t nb, int d, int64_t ld, double *mean, double *gram, void *ws, cudaStream_t st) {
    using namespace stc;
    WsView w = carve(ws, n_groups, nb, d);
    const int64_t nbp = (nb + 63) / 64 * 64;
    GSB_CHECK_CUDA(cudaMemsetAsync(w.absmax, 0, (size_t)n_groups * sizeof(float), st));
    {
        const int ny = (int)((nb + SUM_ROWS - 1) / SUM_ROWS);
        dim3 grid((d + 127) / 128, (unsigned)ny, (unsigned)n_groups);
        colsum_groups_kernel<<<grid, 128, 0, st>>>(x, nb, d, ld, SUM_ROWS, w.sum, w.absmax);
        GSB_CHECK_LAUNCH();
        mean_groups_kernel<<<(n_groups * d + 255) / 256, 256, 0, st>>>(w.sum, ny, n_groups, d, (double)nb, mean, w.mean32, w.absmax, w.exps);
        GSB_CHECK_LAUNCH();
    }
    {
        dim3 grid((unsigned)(nbp / 64), (unsigned)(d / 64), (unsigned)n_groups);
        center_split_t_kernel<<<grid, 256, 0, st>>>(x, nb, d, ld, nbp, w.mean32, w.exps, w.xt_hi, w.xt_lo);
        GSB_CHECK_LAUNCH();
    }
    return gram_tc_launch(GramEpilogue::Store, w.xt_hi, w.xt_lo, nb, nbp, n_groups, d, d, w.exps, gram, st);
}

bool stats_tc_grouped_width(int d) { return d % 128 == 0 && d >= 128 && d <= 1024; }

size_t stats_tc_grouped_workspace_bytes(const gsb_stats_desc *descs, int n_desc) {
    size_t bytes = 0;
    for (int i0 = 0; i0 < n_desc; i0 += GRAM_GROUPED_MAX) {
        const int n = n_desc - i0 < GRAM_GROUPED_MAX ? n_desc - i0 : GRAM_GROUPED_MAX;
        const size_t b = stc::carve_grouped(nullptr, descs + i0, n, nullptr);
        bytes = b > bytes ? b : bytes;
    }
    return bytes;
}

// descriptors already checked: one set of four launches (+ one memset) per GRAM_GROUPED_MAX descriptors, sharing ws
int stats_tc_grouped(const gsb_stats_desc *descs, int n_desc, void *ws, cudaStream_t st) {
    using namespace stc;
    for (int i0 = 0; i0 < n_desc; i0 += GRAM_GROUPED_MAX) {
        const int n = n_desc - i0 < GRAM_GROUPED_MAX ? n_desc - i0 : GRAM_GROUPED_MAX;
        PrepParams p;
        memset(&p, 0, sizeof(p));
        p.n_desc = n;
        carve_grouped(ws, descs + i0, n, p.desc);
        int total_groups = 0, b_col = 0, b_mean = 0, b_ctr = 0;
        GramGroupedOperand ops[GRAM_GROUPED_MAX];
        for (int i = 0; i < n; ++i) {
            PrepDesc &q = p.desc[i];
            q.blk_colsum = b_col; q.blk_mean = b_mean; q.blk_center = b_ctr;
            b_col += ((q.d + 127) / 128) * q.ny * q.n_groups;
            b_mean += (q.n_groups * q.d + 255) / 256;
            b_ctr += (int)(q.nbp / 64) * (q.d / 64) * q.n_groups;
            total_groups += q.n_groups;
            ops[i] = GramGroupedOperand{q.xt_hi, q.xt_lo, q.nb, q.nbp, q.d, q.n_groups, q.exps, descs[i0 + i].gram_out};
        }
        GSB_CHECK_CUDA(cudaMemsetAsync(ws, 0, (size_t)total_groups * sizeof(float), st));
        colsum_grouped_kernel<<<b_col, 128, 0, st>>>(p);
        GSB_CHECK_LAUNCH();
        mean_grouped_kernel<<<b_mean, 256, 0, st>>>(p);
        GSB_CHECK_LAUNCH();
        center_split_t_grouped_kernel<<<b_ctr, 256, 0, st>>>(p);
        GSB_CHECK_LAUNCH();
        if (int r = gram_tc_grouped_launch(ops, n, st)) return r;
    }
    return GSB_OK;
}

}  // namespace gsb
