// Per-batch sufficient statistics for the Gram-form incremental PCA (fp32 FMA path).
//
//   mean[d]   = (1/n) sum_r x[r,:]                       fp64 accumulation of the fp32 samples
//   gram[d,d] = sum_r (x[r,:]-mean)^T (x[r,:]-mean)      fp32 products, fp32 partial sums over <=512 rows,
//                                                        fp64 accumulation across row chunks
// These replace what sklearn's IncrementalPCA.partial_fit reads off the batch
// (estimators.py:68-76 -> _incremental_pca.py:332-357: col_mean/col_var merge, X -= col_batch_mean,
// and the X rows of the stacked matrix whose SVD it takes): the right singular vectors/values of the
// stack [S*V; Xc; m] are the eigenpairs of V^T S^2 V + Xc^T Xc + m m^T (SURVEY.md section 0.3).
//
// Kernels: column sums (coalesced, fp64 atomics), then a 64x64-tile SYRK over the upper triangle of
// tile pairs, split over row chunks; each CTA adds its fp32 tile into the fp64 Gram with atomics and
// mirrors off-diagonal tiles so the chain reads a full symmetric matrix.
#include "tc_common.cuh"

namespace gsb {

__global__ void colsum_kernel(const float *__restrict__ x, int64_t n, int d, int64_t ld, int rows_per_cta,
                              double *__restrict__ sum) {
    int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= d) return;
    int64_t r0 = (int64_t)blockIdx.y * rows_per_cta;
    int64_t r1 = r0 + rows_per_cta < n ? r0 + rows_per_cta : n;
    double acc = 0.0;   // fp64 sum of the fp32 samples, as sklearn's _safe_accumulator_op does
    for (int64_t r = r0; r < r1; ++r) acc += (double)x[r * ld + col];
    atomicAdd(&sum[col], acc);
}

__global__ void mean_finalize_kernel(const double *__restrict__ sum, int d, double nd,
                                     double *__restrict__ mean, float *__restrict__ mean32) {
    int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i < d) {
        double m = sum[i] / nd;
        mean[i] = m;
        mean32[i] = (float)m;
    }
}

constexpr int GT = 64;       // tile edge
constexpr int GK = 16;       // rows per smem stage
constexpr int GRAM_THREADS = 256;

__global__ void __launch_bounds__(GRAM_THREADS, 2)
gram_centered_kernel(const float *__restrict__ x, int64_t n, int d, int64_t ld, int rows_per_cta,
                     const float *__restrict__ mean32, double *__restrict__ gram) {
    // blockIdx.x enumerates tile pairs (ti <= tj) of the upper triangle
    const int nt = (d + GT - 1) / GT;
    int p = blockIdx.x, ti = 0;
    while (p >= nt - ti) { p -= nt - ti; ++ti; }
    const int tj = ti + p;
    const int64_t r0 = (int64_t)blockIdx.y * rows_per_cta;
    const int64_t r1 = r0 + rows_per_cta < n ? r0 + rows_per_cta : n;

    __shared__ __align__(16) float Xi[2][GK][GT];
    __shared__ __align__(16) float Xj[2][GK][GT];
    const int tid = threadIdx.x;
    const int tx = tid & 15, ty = tid >> 4;   // 16x16 threads, 4x4 outputs each
    const int lrow = tid >> 4;                // loader: 16 rows x 16 float4
    const int lcol = (tid & 15) * 4;
    const bool ci_ok = ti * GT + lcol < d, cj_ok = tj * GT + lcol < d;   // d % 4 == 0
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    const float4 mi = ci_ok ? *reinterpret_cast<const float4 *>(mean32 + ti * GT + lcol) : zero4;
    const float4 mj = cj_ok ? *reinterpret_cast<const float4 *>(mean32 + tj * GT + lcol) : zero4;

    float acc[4][4];
#pragma unroll
    for (int a = 0; a < 4; ++a)
#pragma unroll
        for (int b = 0; b < 4; ++b) acc[a][b] = 0.f;

    float4 vi, vj;
    auto gload = [&](int64_t rbase) {
        int64_t r = rbase + lrow;
        if (r < r1) {
            vi = ci_ok ? *reinterpret_cast<const float4 *>(x + r * ld + ti * GT + lcol) : zero4;
            vj = cj_ok ? *reinterpret_cast<const float4 *>(x + r * ld + tj * GT + lcol) : zero4;
            vi.x -= mi.x; vi.y -= mi.y; vi.z -= mi.z; vi.w -= mi.w;
            vj.x -= mj.x; vj.y -= mj.y; vj.z -= mj.z; vj.w -= mj.w;
        } else {
            vi = make_float4(0.f, 0.f, 0.f, 0.f);
            vj = vi;
        }
    };
    gload(r0);
    *reinterpret_cast<float4 *>(&Xi[0][lrow][lcol]) = vi;
    *reinterpret_cast<float4 *>(&Xj[0][lrow][lcol]) = vj;
    __syncthreads();
    int buf = 0;
    for (int64_t rb = r0; rb < r1; rb += GK) {
        bool more = rb + GK < r1;
        if (more) gload(rb + GK);
#pragma unroll
        for (int k = 0; k < GK; ++k) {
            float4 a = *reinterpret_cast<const float4 *>(&Xi[buf][k][ty * 4]);
            float4 b = *reinterpret_cast<const float4 *>(&Xj[buf][k][tx * 4]);
            float av[4] = {a.x, a.y, a.z, a.w}, bv[4] = {b.x, b.y, b.z, b.w};
#pragma unroll
            for (int q = 0; q < 4; ++q)
#pragma unroll
                for (int s = 0; s < 4; ++s) acc[q][s] = fmaf(av[q], bv[s], acc[q][s]);
        }
        if (more) {
            *reinterpret_cast<float4 *>(&Xi[buf ^ 1][lrow][lcol]) = vi;
            *reinterpret_cast<float4 *>(&Xj[buf ^ 1][lrow][lcol]) = vj;
            __syncthreads();
            buf ^= 1;
        }
    }
#pragma unroll
    for (int q = 0; q < 4; ++q)
#pragma unroll
        for (int s = 0; s < 4; ++s) {
            int gi = ti * GT + ty * 4 + q, gj = tj * GT + tx * 4 + s;
            if (gi >= d || gj >= d) continue;
            double v = (double)acc[q][s];
            atomicAdd(&gram[(int64_t)gi * d + gj], v);
            if (ti != tj) atomicAdd(&gram[(int64_t)gj * d + gi], v);
        }
}

}  // namespace gsb

extern "C" size_t gsb_batch_stats_workspace_bytes(int64_t n, int d) {
    if (gsb::stats_tc_supported(n, d)) return gsb::stats_tc_workspace_bytes(1, n, d);
    return gsb::align_up((size_t)d * sizeof(double), 256) + gsb::align_up((size_t)d * sizeof(float), 256);
}

extern "C" size_t gsb_batch_stats_multi_workspace_bytes(int n_groups, int64_t rows_per_group, int d) {
    if (gsb::stats_tc_supported(rows_per_group, d)) return gsb::stats_tc_workspace_bytes(n_groups, rows_per_group, d);
    return gsb_batch_stats_workspace_bytes(rows_per_group, d);
}

// Statistics of n_groups consecutive groups of rows_per_group rows: d_mean [G][d], d_gram [G][d][d].  One set of launches for
// all groups on the tensor-core path (d % 128 == 0); a loop over the fp32 FMA kernels otherwise.
extern "C" int gsb_batch_stats_multi(const float *d_x, int n_groups, int64_t rows_per_group, int d, int64_t ld, double *d_mean,
                                     double *d_gram, void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_x && d_mean && d_gram && d_workspace, "batch_stats_multi: null pointer");
    GSB_CHECK_ARG(n_groups > 0 && n_groups <= 65535 && rows_per_group > 0 && d > 0 && d % 4 == 0 && ld >= d && ld % 4 == 0,
                  "batch_stats_multi: need 0<groups<=65535, rows>0, d%%4==0, ld>=d, ld%%4==0 (groups=%d rows=%lld d=%d ld=%lld)",
                  n_groups, (long long)rows_per_group, d, (long long)ld);
    if (workspace_bytes < gsb_batch_stats_multi_workspace_bytes(n_groups, rows_per_group, d)) {
        gsb::set_error("batch_stats_multi: workspace too small");
        return GSB_ERR_WORKSPACE;
    }
    if (gsb::stats_tc_supported(rows_per_group, d))
        return gsb::stats_tc(d_x, n_groups, rows_per_group, d, ld, d_mean, d_gram, d_workspace, (cudaStream_t)stream);
    for (int g = 0; g < n_groups; ++g) {
        int r = gsb_batch_stats(d_x + (size_t)g * rows_per_group * ld, rows_per_group, d, ld, d_mean + (size_t)g * d,
                                d_gram + (size_t)g * d * d, d_workspace, workspace_bytes, stream);
        if (r) return r;
    }
    return GSB_OK;
}

static int check_grouped(const gsb_stats_desc *descs, int n_desc) {
    GSB_CHECK_ARG(descs && n_desc > 0, "batch_stats_grouped: need a non-empty descriptor array (n_desc=%d)", n_desc);
    for (int i = 0; i < n_desc; ++i) {
        const gsb_stats_desc &s = descs[i];
        GSB_CHECK_ARG(s.x && s.mean_out && s.gram_out, "batch_stats_grouped: null pointer in descriptor %d", i);
        GSB_CHECK_ARG(gsb::stats_tc_grouped_width(s.d),
                      "batch_stats_grouped: descriptor %d has d=%d; the grouped statistics take d %% 128 == 0, 128 <= d <= 1024 "
                      "(other widths: gsb_batch_stats_multi)", i, s.d);
        GSB_CHECK_ARG(s.n_groups > 0 && s.n_groups <= 65535 && s.rows_per_group > 0 && s.ld >= s.d && s.ld % 4 == 0,
                      "batch_stats_grouped: descriptor %d needs 0<groups<=65535, rows>0, ld>=d, ld%%4==0 (groups=%d rows=%lld "
                      "ld=%lld)", i, s.n_groups, (long long)s.rows_per_group, (long long)s.ld);
    }
    return GSB_OK;
}

extern "C" size_t gsb_batch_stats_grouped_workspace_bytes(const gsb_stats_desc *descs, int n_desc) {
    if (check_grouped(descs, n_desc)) return 0;
    return gsb::stats_tc_grouped_workspace_bytes(descs, n_desc);
}

// Statistics of several inputs in one set of launches per 32 descriptors; every descriptor is checked before anything runs.
extern "C" int gsb_batch_stats_grouped(const gsb_stats_desc *descs, int n_desc, void *d_workspace, size_t workspace_bytes,
                                       gsb_stream_t stream) {
    if (int r = check_grouped(descs, n_desc)) return r;
    GSB_CHECK_ARG(d_workspace, "batch_stats_grouped: null workspace");
    if (workspace_bytes < gsb::stats_tc_grouped_workspace_bytes(descs, n_desc)) {
        gsb::set_error("batch_stats_grouped: workspace too small");
        return GSB_ERR_WORKSPACE;
    }
    return gsb::stats_tc_grouped(descs, n_desc, d_workspace, (cudaStream_t)stream);
}

extern "C" int gsb_batch_stats(const float *d_x, int64_t n, int d, int64_t ld, double *d_mean,
                               double *d_gram, void *d_workspace, size_t workspace_bytes,
                               gsb_stream_t stream) {
    GSB_CHECK_ARG(d_x && d_mean && d_gram && d_workspace, "batch_stats: null pointer");
    GSB_CHECK_ARG(n > 0 && d > 0 && d % 4 == 0 && ld >= d && ld % 4 == 0,
                  "batch_stats: need n>0, d%%4==0, ld>=d, ld%%4==0 (n=%lld d=%d ld=%lld)", (long long)n, d,
                  (long long)ld);
    if (workspace_bytes < gsb_batch_stats_workspace_bytes(n, d)) {
        gsb::set_error("batch_stats: workspace too small");
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    if (gsb::stats_tc_supported(n, d)) return gsb::stats_tc(d_x, 1, n, d, ld, d_mean, d_gram, d_workspace, st);
    double *sum = reinterpret_cast<double *>(d_workspace);
    float *mean32 = reinterpret_cast<float *>(reinterpret_cast<char *>(d_workspace) +
                                              gsb::align_up((size_t)d * sizeof(double), 256));
    GSB_CHECK_CUDA(cudaMemsetAsync(sum, 0, (size_t)d * sizeof(double), st));
    GSB_CHECK_CUDA(cudaMemsetAsync(d_gram, 0, (size_t)d * d * sizeof(double), st));
    {
        int rows = 128;
        dim3 grid((d + 127) / 128, (unsigned)((n + rows - 1) / rows));
        gsb::colsum_kernel<<<grid, 128, 0, st>>>(d_x, n, d, ld, rows, sum);
        GSB_CHECK_LAUNCH();
        gsb::mean_finalize_kernel<<<(d + 255) / 256, 256, 0, st>>>(sum, d, (double)n, d_mean, mean32);
        GSB_CHECK_LAUNCH();
    }
    {
        int nt = (d + gsb::GT - 1) / gsb::GT;
        int pairs = nt * (nt + 1) / 2;
        // fp32 partial sums over at most 512 rows; enough chunks to fill the machine
        int rows = 512;
        while (rows > 128 && (int64_t)pairs * ((n + rows - 1) / rows) < 2 * gsb::num_sms()) rows /= 2;
        dim3 grid(pairs, (unsigned)((n + rows - 1) / rows));
        gsb::gram_centered_kernel<<<grid, gsb::GRAM_THREADS, 0, st>>>(d_x, n, d, ld, rows, mean32, d_gram);
        GSB_CHECK_LAUNCH();
    }
    return GSB_OK;
}
