// Projection statistics and the latent-regression accumulators (fp32 products, fp64 moments).
//
//   gsb_project_std      decomposition.py:313-316 (random_stdevs) and :326-329 (lat_stdev)
//   gsb_linreg_*         decomposition.py:77-139  (linreg_lstsq): instead of materialising
//                        A[n_samp,c] and Z[n_samp,L] on the host and calling gelsd, every batch adds
//                        A^T A, A^T Z and sum(Z) into fp64 accumulators; the c x c solve is a Cholesky.
#include "common.cuh"

namespace gsb {

constexpr int PJ_ROWS = 64, PJ_COMPS = 32, PJ_K = 32;

// p[r,k] = sum_i (x[r,i] - sub[i]) * dirs[k,i]   (optionally / stdev[k])
// SUBMODE 0: no subtraction; 1: fp64 sub (x rounded to fp32 after an fp64 subtract, as numpy's
// float32_array -= float64_array does, decomposition.py:291); 2: fp32 sub (decomposition.py:120).
template <int SUBMODE>
__device__ __forceinline__ void project_tile(const float *__restrict__ x, int64_t n, int d, int64_t ld,
                                             const float *__restrict__ dirs, int c,
                                             const double *__restrict__ sub64,
                                             const float *__restrict__ sub32, int64_t r0, int k0,
                                             float (&acc)[8], float (*Xs)[PJ_K + 1], float (*Cs)[PJ_K + 1],
                                             int i_begin = 0, int i_end = -1) {
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
#pragma unroll
    for (int r = 0; r < 8; ++r) acc[r] = 0.f;
    if (i_end < 0 || i_end > d) i_end = d;
    for (int i0 = i_begin; i0 < i_end; i0 += PJ_K) {
        for (int rr = ty; rr < PJ_ROWS; rr += 8) {
            int64_t r = r0 + rr;
            int i = i0 + tx;
            float v = 0.f;
            if (r < n && i < i_end) {
                v = x[r * ld + i];
                if (SUBMODE == 1) v = (float)((double)v - sub64[i]);
                if (SUBMODE == 2) v = v - sub32[i];
            }
            Xs[rr][tx] = v;
        }
        for (int kk = ty; kk < PJ_COMPS; kk += 8) {
            int k = k0 + kk, i = i0 + tx;
            Cs[kk][tx] = (k < c && i < i_end) ? dirs[(int64_t)k * d + i] : 0.f;
        }
        __syncthreads();
#pragma unroll 8
        for (int kk = 0; kk < PJ_K; ++kk) {
            float cv = Cs[tx][kk];
#pragma unroll
            for (int r = 0; r < 8; ++r) acc[r] = fmaf(Xs[ty + 8 * r][kk], cv, acc[r]);
        }
        __syncthreads();
    }
}

__global__ void __launch_bounds__(256)
project_moments_kernel(const float *__restrict__ x, int64_t n, int d, int64_t ld,
                       const float *__restrict__ dirs, int c, const double *__restrict__ sub,
                       double *__restrict__ mom /* [2][c] */) {
    __shared__ float Xs[PJ_ROWS][PJ_K + 1], Cs[PJ_COMPS][PJ_K + 1];
    __shared__ double s1[8][32], s2[8][32];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int k0 = blockIdx.y * PJ_COMPS;
    const int64_t r0 = (int64_t)blockIdx.x * PJ_ROWS;
    float acc[8];
    if (sub) project_tile<1>(x, n, d, ld, dirs, c, sub, nullptr, r0, k0, acc, Xs, Cs);
    else project_tile<0>(x, n, d, ld, dirs, c, nullptr, nullptr, r0, k0, acc, Xs, Cs);
    double a1 = 0.0, a2 = 0.0;
#pragma unroll
    for (int r = 0; r < 8; ++r)
        if (r0 + ty + 8 * r < n) { double p = (double)acc[r]; a1 += p; a2 += p * p; }
    s1[ty][tx] = a1; s2[ty][tx] = a2;
    __syncthreads();
    if (ty == 0 && k0 + tx < c) {
        for (int q = 1; q < 8; ++q) { a1 += s1[q][tx]; a2 += s2[q][tx]; }
        atomicAdd(&mom[k0 + tx], a1);
        atomicAdd(&mom[c + k0 + tx], a2);
    }
}

__global__ void moments_to_std_kernel(const double *__restrict__ mom, int c, double n, float *__restrict__ out) {
    int k = blockIdx.x * blockDim.x + threadIdx.x;
    if (k < c) {
        double m = mom[k] / n, v = mom[c + k] / n - m * m;   // population std (numpy ddof=0)
        out[k] = (float)sqrt(fmax(v, 0.0));
    }
}

// A[r,k] = ((act[r,:] - mean) . comp[k,:]) / stdev[k]      decomposition.py:119-123
// gridDim.z > 1 (conv feature maps, d ~ 10^5..10^6): the feature axis is split into gridDim.z slabs of a multiple of PJ_K
// features; CTA z stores its partial coordinates, undivided, in part[z][row][k] -- every (z, row < n, k < c) slot, an
// empty slab's zeros included -- and linreg_split_sum_kernel adds them in z order.  No atomics: the result does not depend
// on the order the CTAs run in.
__global__ void __launch_bounds__(256)
linreg_coords_kernel(const float *__restrict__ act, int64_t n, int d, const float *__restrict__ comp, int c,
                     const float *__restrict__ mean, const float *__restrict__ stdev, float *__restrict__ A,
                     float *__restrict__ part) {
    __shared__ float Xs[PJ_ROWS][PJ_K + 1], Cs[PJ_COMPS][PJ_K + 1];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int k0 = blockIdx.y * PJ_COMPS;
    const int64_t r0 = (int64_t)blockIdx.x * PJ_ROWS;
    float acc[8];
    const int slab = (int)(((int64_t)d + gridDim.z - 1) / gridDim.z + PJ_K - 1) / PJ_K * PJ_K;
    const int i_begin = blockIdx.z * slab;
    project_tile<2>(act, n, d, d, comp, c, nullptr, mean, r0, k0, acc, Xs, Cs, i_begin, i_begin + slab);
    const int k = k0 + tx;
    if (k >= c) return;
    const float sd = stdev[k];
    float *slot = part + (size_t)blockIdx.z * n * c;
#pragma unroll
    for (int r = 0; r < 8; ++r) {
        int64_t row = r0 + ty + 8 * r;
        if (row >= n) continue;
        if (gridDim.z == 1) A[row * c + k] = acc[r] / sd;
        else slot[row * c + k] = acc[r];
    }
}

// A[row,k] = (sum_{z < splits} part[z][row][k]) / stdev[k], the sum in z order; one division, after the sum.  A separate
// kernel rather than a pass folded into linreg_normal_eq_kernel's loader: that loader reads each A element once per
// 32-column output tile, so folding would re-read all the partials (c + L) / 32 times.
__global__ void __launch_bounds__(256)
linreg_split_sum_kernel(const float *__restrict__ part, int splits, int64_t n, int c, const float *__restrict__ stdev,
                        float *__restrict__ A) {
    const int64_t nc = n * c;
    for (int64_t e = (int64_t)blockIdx.x * blockDim.x + threadIdx.x; e < nc; e += (int64_t)gridDim.x * blockDim.x) {
        float s = 0.f;
        for (int z = 0; z < splits; ++z) s += part[z * nc + e];
        A[e] = s / stdev[e % c];
    }
}

// acc[c, c+L] += A^T [A | Z]  and  sumZ += column sums of Z, over rows [r0, r1)
constexpr int NE_T = 32, NE_ROWS = 256;
__global__ void __launch_bounds__(256)
linreg_normal_eq_kernel(const float *__restrict__ A, const float *__restrict__ Z, int64_t n, int c, int L,
                        double *__restrict__ AtA, double *__restrict__ AtZ, double *__restrict__ sumZ) {
    __shared__ float As[NE_T][NE_T + 1], Bs[NE_T][NE_T + 1];
    const int tx = threadIdx.x & 31, ty = threadIdx.x >> 5;
    const int i0 = blockIdx.y * NE_T;              // rows of the output: components
    const int j0 = blockIdx.x * NE_T;              // cols of the output: [A | Z] columns
    const int64_t r0 = (int64_t)blockIdx.z * NE_ROWS;
    const int64_t r1 = r0 + NE_ROWS < n ? r0 + NE_ROWS : n;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    float zs = 0.f;
    for (int64_t rb = r0; rb < r1; rb += NE_T) {
        for (int rr = ty; rr < NE_T; rr += 8) {
            int64_t r = rb + rr;
            int i = i0 + tx, j = j0 + tx;
            As[rr][tx] = (r < r1 && i < c) ? A[r * c + i] : 0.f;
            float b = 0.f;
            if (r < r1) {
                if (j < c) b = A[r * c + j];
                else if (j < c + L) b = Z[r * L + (j - c)];
            }
            Bs[rr][tx] = b;
        }
        __syncthreads();
#pragma unroll 8
        for (int rr = 0; rr < NE_T; ++rr) {
            float b = Bs[rr][tx];
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[q] = fmaf(As[rr][ty + 8 * q], b, acc[q]);
            if (ty == 0) zs += b;
        }
        __syncthreads();
    }
    const int j = j0 + tx;
    if (j < c + L) {
#pragma unroll
        for (int q = 0; q < 4; ++q) {
            int i = i0 + ty + 8 * q;
            if (i >= c) continue;
            if (j < c) atomicAdd(&AtA[(size_t)i * c + j], (double)acc[q]);
            else atomicAdd(&AtZ[(size_t)i * L + (j - c)], (double)acc[q]);
        }
        if (ty == 0 && blockIdx.y == 0 && j >= c) atomicAdd(&sumZ[j - c], (double)zs);
    }
}

// single-CTA Cholesky solve  M = AtA^-1 AtZ  (c <= 512), fp64, on a copy of AtA (`fac`).  A pivot that is not clearly
// positive (<= 1e-6 of the largest diagonal entry: the columns of A are numerically dependent, or hold NaN) sets info = k + 1
// and zeroes M; the caller then takes the minimum-norm route (linreg_pinv_kernel), which is what the reference's
// scipy.linalg.lstsq(..., lapack_driver='gelsd') returns for a rank-deficient A (decomposition.py:133).
__global__ void __launch_bounds__(1024)
linreg_solve_kernel(const double *__restrict__ AtA_in, double *__restrict__ AtA, const double *__restrict__ AtZ,
                    const double *__restrict__ sumZ, int c, int L, double n_total, double *__restrict__ M,
                    double *__restrict__ zmean, int *__restrict__ info) {
    const int tid = threadIdx.x, nt = blockDim.x;
    __shared__ double red[64];
    double dmax = 0.0;
    for (int i = tid; i < c * c; i += nt) {
        const double v = AtA_in[i];
        AtA[i] = v;
        if (i / c == i % c) dmax = fmax(dmax, v);
    }
    for (int o = 16; o > 0; o >>= 1) dmax = fmax(dmax, __shfl_xor_sync(0xffffffffu, dmax, o));
    if ((tid & 31) == 0) red[tid >> 5] = dmax;
    __syncthreads();
    dmax = 0.0;
    for (int q = 0; q < (nt >> 5); ++q) dmax = fmax(dmax, red[q]);
    const double floor_ = 1e-6 * dmax;
    for (int col = tid; col < L; col += nt) zmean[col] = sumZ[col] / n_total;
    // right-looking Cholesky, lower factor stored in AtA
    for (int k = 0; k < c; ++k) {
        __syncthreads();
        double dkk = AtA[(size_t)k * c + k];
        if (!(dkk > floor_)) {
            if (tid == 0) *info = k + 1;
            for (int i = tid; i < c * L; i += nt) M[i] = 0.0;
            return;
        }
        double lkk = sqrt(dkk);
        __syncthreads();
        for (int i = k + tid; i < c; i += nt) AtA[(size_t)i * c + k] = (i == k) ? lkk : AtA[(size_t)i * c + k] / lkk;
        __syncthreads();
        for (int idx = tid; idx < (c - k - 1) * (c - k - 1); idx += nt) {
            int i = k + 1 + idx / (c - k - 1), j = k + 1 + idx % (c - k - 1);
            if (j <= i) AtA[(size_t)i * c + j] -= AtA[(size_t)i * c + k] * AtA[(size_t)j * c + k];
        }
    }
    __syncthreads();
    // each thread solves columns of the right-hand side:  L y = b ; L^T x = y
    for (int col = tid; col < L; col += nt) {
        for (int i = 0; i < c; ++i) {
            double s = AtZ[(size_t)i * L + col];
            for (int k = 0; k < i; ++k) s -= AtA[(size_t)i * c + k] * M[(size_t)k * L + col];
            M[(size_t)i * L + col] = s / AtA[(size_t)i * c + i];
        }
        for (int i = c - 1; i >= 0; --i) {
            double s = M[(size_t)i * L + col];
            for (int k = i + 1; k < c; ++k) s -= AtA[(size_t)k * c + i] * M[(size_t)k * L + col];
            M[(size_t)i * L + col] = s / AtA[(size_t)i * c + i];
        }
    }
    if (tid == 0) *info = 0;
}

// Minimum-norm least squares from the eigen-decomposition AtA = sum_i lam_i v_i v_i^T:  M = sum_{lam_i > rcond lam_max}
// v_i (v_i^T AtZ) / lam_i.   evecs[c][c]: rows are eigenvectors (descending eigenvalues).  grid.x = L columns in chunks of 128.
__global__ void __launch_bounds__(128)
linreg_pinv_kernel(const double *__restrict__ lam, const double *__restrict__ evecs, const double *__restrict__ AtZ, int c, int L,
                   double rcond, double *__restrict__ M) {
    const int col = blockIdx.x * blockDim.x + threadIdx.x;
    if (col >= L) return;
    const double cut = rcond * fmax(lam[0], 0.0);
    for (int i = 0; i < c; ++i) M[(size_t)i * L + col] = 0.0;
    for (int t = 0; t < c; ++t) {
        const double l = lam[t];
        if (!(l > cut)) continue;
        const double *v = evecs + (size_t)t * c;
        double proj = 0.0;
        for (int k = 0; k < c; ++k) proj = fma(v[k], AtZ[(size_t)k * L + col], proj);
        proj /= l;
        for (int i = 0; i < c; ++i) M[(size_t)i * L + col] = fma(v[i], proj, M[(size_t)i * L + col]);
    }
}

struct LinregView { double *AtA, *AtZ, *sumZ, *fac; int *info; size_t bytes; };
static LinregView linreg_view(void *p, int c, int L) {
    LinregView v;
    char *b = reinterpret_cast<char *>(p);
    size_t off = 0;
    v.AtA = (double *)(b + off); off += align_up((size_t)c * c * 8, 256);
    v.AtZ = (double *)(b + off); off += align_up((size_t)c * L * 8, 256);
    v.sumZ = (double *)(b + off); off += align_up((size_t)L * 8, 256);
    v.info = (int *)(b + off); off += 256;
    v.fac = (double *)(b + off); off += align_up((size_t)c * c * 8, 256);
    v.bytes = off;
    return v;
}

}  // namespace gsb

extern "C" size_t gsb_project_std_workspace_bytes(int c) { return gsb::align_up((size_t)2 * c * sizeof(double), 256); }

extern "C" int gsb_project_std(const float *d_x, int64_t n, int d, int64_t ld, const float *d_dirs, int c,
                               const double *d_sub, float *d_out_std, void *d_workspace,
                               size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_x && d_dirs && d_out_std && d_workspace, "project_std: null pointer");
    GSB_CHECK_ARG(n > 0 && d > 0 && c > 0 && ld >= d, "project_std: bad sizes");
    if (workspace_bytes < gsb_project_std_workspace_bytes(c)) {
        gsb::set_error("project_std: workspace too small");
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    double *mom = reinterpret_cast<double *>(d_workspace);
    GSB_CHECK_CUDA(cudaMemsetAsync(mom, 0, (size_t)2 * c * sizeof(double), st));
    dim3 grid((unsigned)((n + gsb::PJ_ROWS - 1) / gsb::PJ_ROWS), (c + gsb::PJ_COMPS - 1) / gsb::PJ_COMPS);
    gsb::project_moments_kernel<<<grid, 256, 0, st>>>(d_x, n, d, ld, d_dirs, c, d_sub, mom);
    GSB_CHECK_LAUNCH();
    gsb::moments_to_std_kernel<<<(c + 127) / 128, 128, 0, st>>>(mom, c, (double)n, d_out_std);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" size_t gsb_linreg_state_bytes(int c, int latent_dim) { return gsb::linreg_view(nullptr, c, latent_dim).bytes; }

extern "C" int gsb_linreg_reset(void *d_state, int c, int latent_dim, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && c > 0 && latent_dim > 0, "linreg_reset: bad arguments");
    GSB_CHECK_CUDA(cudaMemsetAsync(d_state, 0, gsb_linreg_state_bytes(c, latent_dim), (cudaStream_t)stream));
    return GSB_OK;
}

// Few row tiles and a long feature axis: split d over 2..64 CTAs.  The doubling stops once tiles * splits reaches
// 8 * SMs, so splits * n * c stays under 2 * 8 * SMs * PJ_ROWS * PJ_COMPS floats for any n.
extern "C" int gsb_linreg_feature_splits(int64_t n, int c, int d) {
    if (n <= 0 || c <= 0 || d <= 0) return 1;
    const int64_t tiles = ((n + gsb::PJ_ROWS - 1) / gsb::PJ_ROWS) * ((c + gsb::PJ_COMPS - 1) / gsb::PJ_COMPS);
    int splits = 1;
    while (splits < 64 && tiles * splits < 8 * gsb::num_sms() && d / (2 * splits) >= 4096) splits *= 2;
    return splits;
}

extern "C" size_t gsb_linreg_workspace_bytes(int64_t n, int c, int d) {
    const int splits = gsb_linreg_feature_splits(n, c, d);
    const size_t a = gsb::align_up((size_t)n * c * sizeof(float), 256);
    return splits > 1 ? a + gsb::align_up((size_t)splits * n * c * sizeof(float), 256) : a;
}

extern "C" int gsb_linreg_accumulate(void *d_state, int c, int latent_dim, const float *d_act, int64_t n, int d,
                                     const float *d_comp, const float *d_mean, const float *d_stdev,
                                     const float *d_z, void *d_workspace, size_t workspace_bytes,
                                     gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && d_act && d_comp && d_mean && d_stdev && d_z && d_workspace, "linreg_accumulate: null pointer");
    GSB_CHECK_ARG(n > 0 && c > 0 && c <= 512 && d > 0 && latent_dim > 0, "linreg_accumulate: bad sizes");
    if (workspace_bytes < gsb_linreg_workspace_bytes(n, c, d)) {
        gsb::set_error("linreg_accumulate: workspace too small");
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    gsb::LinregView v = gsb::linreg_view(d_state, c, latent_dim);
    float *A = reinterpret_cast<float *>(d_workspace);
    float *part = reinterpret_cast<float *>(reinterpret_cast<char *>(d_workspace) +
                                            gsb::align_up((size_t)n * c * sizeof(float), 256));
    const int splits = gsb_linreg_feature_splits(n, c, d);
    dim3 g1((unsigned)((n + gsb::PJ_ROWS - 1) / gsb::PJ_ROWS), (c + gsb::PJ_COMPS - 1) / gsb::PJ_COMPS, splits);
    gsb::linreg_coords_kernel<<<g1, 256, 0, st>>>(d_act, n, d, d_comp, c, d_mean, d_stdev, A, part);
    GSB_CHECK_LAUNCH();
    if (splits > 1) {
        const int64_t nc = n * c;
        const int64_t want = (nc + 255) / 256, cap = 8 * gsb::num_sms();
        gsb::linreg_split_sum_kernel<<<(unsigned)(want < cap ? want : cap), 256, 0, st>>>(part, splits, n, c, d_stdev, A);
        GSB_CHECK_LAUNCH();
    }
    dim3 g2((c + latent_dim + gsb::NE_T - 1) / gsb::NE_T, (c + gsb::NE_T - 1) / gsb::NE_T,
            (unsigned)((n + gsb::NE_ROWS - 1) / gsb::NE_ROWS));
    gsb::linreg_normal_eq_kernel<<<g2, 256, 0, st>>>(A, d_z, n, c, latent_dim, v.AtA, v.AtZ, v.sumZ);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_linreg_solve(void *d_state, int c, int latent_dim, int64_t n_total, double *d_M_t,
                                double *d_z_mean, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && d_M_t && d_z_mean && c > 0 && c <= 512 && n_total > 0, "linreg_solve: bad arguments");
    gsb::LinregView v = gsb::linreg_view(d_state, c, latent_dim);
    gsb::linreg_solve_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(v.AtA, v.fac, v.AtZ, v.sumZ, c, latent_dim,
                                                                  (double)n_total, d_M_t, d_z_mean, v.info);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// 0 = the Cholesky solve succeeded; k > 0 = pivot k was not positive (rank-deficient / non-finite normal equations): M was
// zeroed, call gsb_linreg_solve_pinv.  Synchronises the stream.
extern "C" int gsb_linreg_solve_status(const void *d_state, int c, int latent_dim, int *h_info, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && h_info && c > 0 && latent_dim > 0, "linreg_solve_status: bad arguments");
    gsb::LinregView v = gsb::linreg_view(const_cast<void *>(d_state), c, latent_dim);
    GSB_CHECK_CUDA(cudaMemcpyAsync(h_info, v.info, sizeof(int), cudaMemcpyDeviceToHost, (cudaStream_t)stream));
    GSB_CHECK_CUDA(cudaStreamSynchronize((cudaStream_t)stream));
    return GSB_OK;
}

extern "C" const double *gsb_linreg_normal_matrix(const void *d_state, int c, int latent_dim) {
    return gsb::linreg_view(const_cast<void *>(d_state), c, latent_dim).AtA;
}

// Minimum-norm solution from the eigenpairs of the normal matrix (gsb_sym_eig_top of gsb_linreg_normal_matrix, all c of them):
// eigenvalues <= rcond * largest are dropped, as gelsd drops small singular values.
extern "C" int gsb_linreg_solve_pinv(const void *d_state, int c, int latent_dim, const double *d_evals, const double *d_evecs,
                                     double rcond, double *d_M_t, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && d_evals && d_evecs && d_M_t && c > 0 && c <= 512 && rcond >= 0.0, "linreg_solve_pinv: bad arguments");
    gsb::LinregView v = gsb::linreg_view(const_cast<void *>(d_state), c, latent_dim);
    gsb::linreg_pinv_kernel<<<(latent_dim + 127) / 128, 128, 0, (cudaStream_t)stream>>>(d_evals, d_evecs, v.AtZ, c, latent_dim, rcond,
                                                                                     d_M_t);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}
