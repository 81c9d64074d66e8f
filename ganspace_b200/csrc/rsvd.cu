// Facebook PCA (fbpca.pca, raw=True, m >= n) from pooled batch statistics, fp64 (DESIGN.md section 5g).
//
// The reference's FacebookPCAEstimator (estimators.py:124-160) stacks all N + NB samples and calls fbpca.pca on them.  For
// m >= n its randomized branch depends on the samples X only through the Gram G = X^T X:
//     Q = orth(X G^2 Omega)     (fbpca: LU-normalised power iterations and a final QR),   Va, s = svd(Q^T X)
// With Y an orthonormal basis of range(G^2 Omega), P = G Y, L = chol(Y^T P) and F = P L^-T  (d x l):  Q^T X = F^T, so Va and s
// are the top-c left singular vectors / singular values of F, i.e. from the eigenpairs (W, s^2) of the l x l matrix F^T F:
// Va^T = F W diag(1/s).  The exact branch (l >= m/1.25 or l >= n/1.25) is the top-c eigenpairs of G itself.
//
// State: pooled (n, mean[d], centred scatter S[d,d]), folded from per-group statistics with Chan's update in the caller's order.
// The driver's samples are centred by their mean, so its G is S; fit() on raw rows uses G = S + n mean mean^T.
//
// Products are fp64 on the tensor cores (mma.sync m8n8k4, as subspace.cu); the range basis is orthonormalised by CholQR2
// between the products.  Everything is deterministic: no atomics on values, fixed reduction orders.
#include "eig.cuh"
#include <math.h>

namespace gsb {

namespace {

constexpr int FB_HDR = 32;     // doubles: [0] = n; status word (int) at [2]

struct FbState {
    double *hdr, *mean, *S;
    int *status;
    size_t bytes;
};

FbState fb_state(void *base, int d) {
    FbState s;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    s.hdr = (double *)take(FB_HDR * sizeof(double));
    s.mean = (double *)take((size_t)d * sizeof(double));
    s.S = (double *)take((size_t)d * d * sizeof(double));
    s.status = reinterpret_cast<int *>(s.hdr + 2);
    s.bytes = off;
    return s;
}

int lpad(int l) { return (l + 31) / 32 * 32; }

struct FbWs {
    double *G, *Y, *P, *Sm, *comp, *T;
    Workspace eig;         // eig.lam / eig.evecs: the eigenpairs of F^T F
    size_t bytes;
};

FbWs fb_carve(void *base, int d, int c, int l) {
    FbWs w;
    const int lp = lpad(l), de = d > lp ? d : lp;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    w.G = (double *)take((size_t)d * d * 8);
    w.Y = (double *)take((size_t)d * lp * 8);
    w.P = (double *)take((size_t)d * lp * 8);
    w.Sm = (double *)take((size_t)lp * lp * 8);
    w.comp = (double *)take((size_t)c * d * 8);
    w.T = (double *)take((size_t)d * c * 8);
    const size_t eig_off = off;
    off += carve(nullptr, de, c).bytes;
    w.eig = carve(base ? p + eig_off : nullptr, de, c);
    w.bytes = off;
    return w;
}

int check_fb_dims(int d) {
    GSB_CHECK_ARG(d >= 32 && d <= 1024 && d % 32 == 0, "fbpca: needs 32 <= d <= 1024, d%%32==0 (d=%d)", d);
    return GSB_OK;
}

}  // namespace

// ---------------------------------------------------------------------------------------------
// Pooling: Chan's update of (n, mean, S) by n_groups groups of nb rows, in order.  Group g has mean mg[g] and centred Gram
// Cg[g]; a NULL mg / Cg is a group of zero rows (mean 0, Gram 0).
//   S += Cg + (n nb / (n + nb)) (mg - mean)(mg - mean)^T,   mean += (mg - mean) nb / (n + nb),   n += nb
// ---------------------------------------------------------------------------------------------
__global__ void fb_pool_scatter_kernel(double *__restrict__ S, const double *__restrict__ mean, const double *__restrict__ hdr,
                                       const double *__restrict__ mg, const double *__restrict__ Cg, int n_groups, double nb,
                                       int d) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
    if (j >= d) return;
    double n = hdr[0], mi = mean[i], mj = mean[j], s = S[(size_t)i * d + j];
    for (int g = 0; g < n_groups; ++g) {
        const double gi = mg ? mg[(size_t)g * d + i] : 0.0, gj = mg ? mg[(size_t)g * d + j] : 0.0;
        const double nn = n + nb, di = gi - mi, dj = gj - mj;
        s += (Cg ? Cg[((size_t)g * d + i) * d + j] : 0.0) + (n * nb / nn) * di * dj;
        mi += di * (nb / nn);
        mj += dj * (nb / nn);
        n = nn;
    }
    S[(size_t)i * d + j] = s;
}

// one CTA of d threads (d <= 1024): every thread reads n before thread 0 advances it
__global__ void fb_pool_mean_kernel(double *__restrict__ mean, double *__restrict__ hdr, const double *__restrict__ mg,
                                    int n_groups, double nb, int d) {
    const int i = threadIdx.x;
    double n = hdr[0];
    __syncthreads();
    if (i < d) {
        double m = mean[i];
        for (int g = 0; g < n_groups; ++g) {
            const double nn = n + nb;
            m += ((mg ? mg[(size_t)g * d + i] : 0.0) - m) * (nb / nn);
            n = nn;
        }
        mean[i] = m;
    } else {
        n += nb * n_groups;
    }
    if (i == 0) hdr[0] = n;
}

// ---------------------------------------------------------------------------------------------
// fp64 GEMM on the tensor cores: C[M,N] = op(A)[M,K] op(B)[K,N]
//   A: TA = false -> A[m * lda + k],  TA = true -> A[k * lda + m];   B: TB = false -> B[k * ldb + n],  TB = true -> B[n * ldb + k]
// A warp computes an 8 x 32 tile (one A fragment against four B fragments per k-step of 4); a CTA of 4 warps a 32 x 32 tile.
// Operands are read through L1/L2 (these matrices are at most 8 MB); out-of-range fragments load zeros.
// ---------------------------------------------------------------------------------------------
constexpr int FG_NT = 4;

__device__ __forceinline__ void fb_dmma(double &c0, double &c1, double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}

template <bool TA, bool TB>
__global__ void __launch_bounds__(128) fb_gemm_kernel(int M, int N, int K, const double *__restrict__ A, int lda,
                                                      const double *__restrict__ B, int ldb, double *__restrict__ C, int ldc) {
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, g = lane >> 2, t = lane & 3;
    const int am = blockIdx.y * 32 + warp * 8 + g, n0 = blockIdx.x * 32;
    double acc[FG_NT][2];
#pragma unroll
    for (int b = 0; b < FG_NT; ++b) { acc[b][0] = 0.0; acc[b][1] = 0.0; }
    for (int k0 = 0; k0 < K; k0 += 4) {
        const int k = k0 + t;
        double a = 0.0;
        if (am < M && k < K) a = TA ? A[(size_t)k * lda + am] : A[(size_t)am * lda + k];
#pragma unroll
        for (int b = 0; b < FG_NT; ++b) {
            const int n = n0 + 8 * b + g;
            double bv = 0.0;
            if (n < N && k < K) bv = TB ? B[(size_t)n * ldb + k] : B[(size_t)k * ldb + n];
            fb_dmma(acc[b][0], acc[b][1], a, bv);
        }
    }
    const int row = blockIdx.y * 32 + warp * 8 + g;
    if (row >= M) return;
#pragma unroll
    for (int b = 0; b < FG_NT; ++b) {
        const int col = n0 + 8 * b + 2 * t;
        if (col < N) C[(size_t)row * ldc + col] = acc[b][0];
        if (col + 1 < N) C[(size_t)row * ldc + col + 1] = acc[b][1];
    }
}

template <bool TA, bool TB>
int fb_gemm(int M, int N, int K, const double *A, int lda, const double *B, int ldb, double *C, int ldc, cudaStream_t st) {
    dim3 grid((N + 31) / 32, (M + 31) / 32);
    fb_gemm_kernel<TA, TB><<<grid, 128, 0, st>>>(M, N, K, A, lda, B, ldb, C, ldc);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// ---------------------------------------------------------------------------------------------
// Omega' = Q^T Omega  [r, l]:  Q [d, r] fp64, Omega [d, l] fp32 (fbpca's test matrix as drawn), a reduction over a long d
// (32768 at BigGAN's gen_z).  fb_gemm_kernel's warp tile, with the k-steps of d dealt round-robin to FP_SPLIT groups of
// four warps; the groups' partial 32 x 32 tiles are then summed in shared memory in group order (deterministic).
// ---------------------------------------------------------------------------------------------
constexpr int FP_SPLIT = 4;

__global__ void __launch_bounds__(128 * FP_SPLIT) fb_project_kernel(int r, int l, int d, const double *__restrict__ Q,
                                                                    const float *__restrict__ Om, double *__restrict__ out) {
    __shared__ double part[FP_SPLIT - 1][32][33];
    const int lane = threadIdx.x & 31, warp = (threadIdx.x >> 5) & 3, grp = threadIdx.x >> 7, g = lane >> 2, t = lane & 3;
    const int row = blockIdx.y * 32 + warp * 8 + g, n0 = blockIdx.x * 32;
    double acc[FG_NT][2];
#pragma unroll
    for (int b = 0; b < FG_NT; ++b) { acc[b][0] = 0.0; acc[b][1] = 0.0; }
#pragma unroll 4
    for (int k0 = 4 * grp; k0 < d; k0 += 4 * FP_SPLIT) {
        const int k = k0 + t;
        double a = 0.0;
        if (row < r && k < d) a = Q[(size_t)k * r + row];
#pragma unroll
        for (int b = 0; b < FG_NT; ++b) {
            const int n = n0 + 8 * b + g;
            double bv = 0.0;
            if (n < l && k < d) bv = (double)Om[(size_t)k * l + n];
            fb_dmma(acc[b][0], acc[b][1], a, bv);
        }
    }
    const int lr = warp * 8 + g;                 // accumulator (lr, 8 b + 2 t + {0, 1}) of the CTA's tile
    if (grp > 0) {
#pragma unroll
        for (int b = 0; b < FG_NT; ++b) {
            part[grp - 1][lr][8 * b + 2 * t] = acc[b][0];
            part[grp - 1][lr][8 * b + 2 * t + 1] = acc[b][1];
        }
    }
    __syncthreads();
    if (grp > 0 || row >= r) return;
#pragma unroll
    for (int b = 0; b < FG_NT; ++b) {
        double s0 = acc[b][0], s1 = acc[b][1];
        for (int q = 0; q < FP_SPLIT - 1; ++q) {
            s0 += part[q][lr][8 * b + 2 * t];
            s1 += part[q][lr][8 * b + 2 * t + 1];
        }
        const int col = n0 + 8 * b + 2 * t;
        if (col < l) out[(size_t)row * l + col] = s0;
        if (col + 1 < l) out[(size_t)row * l + col + 1] = s1;
    }
}

// ---------------------------------------------------------------------------------------------
// In-place lower Cholesky of A[n,n] (row stride lda; the upper triangle is ignored), one CTA, Crout order: column j is
//   L_jj = sqrt(A_jj - sum_k<j L_jk^2),   L_ij = (A_ij - sum_k<j L_ik L_jk) / L_jj   (i > j, one warp per row, coalesced)
// A pivot <= 1e-12 max_i A_ii (the matrix is not numerically positive definite: the data's rank is below l) sets bit0 of
// *status and stops before its square root.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(1024) fb_chol_kernel(double *__restrict__ A, int n, int lda, int *__restrict__ status) {
    __shared__ double red[33];
    __shared__ int fail;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    double mx = 0.0;
    for (int i = tid; i < n; i += blockDim.x) mx = fmax(mx, A[(size_t)i * lda + i]);
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmax(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    if (lane == 0) red[warp] = mx;
    if (tid == 0) fail = 0;
    __syncthreads();
    mx = 0.0;
    for (int w = 0; w < nw; ++w) mx = fmax(mx, red[w]);
    const double tol = 1e-12 * mx;
    for (int j = 0; j < n; ++j) {
        const double *Lj = A + (size_t)j * lda;
        if (warp == 0) {
            double s = 0.0;
            for (int k = lane; k < j; k += 32) s += Lj[k] * Lj[k];
            s = warp_sum(s);
            if (lane == 0) {
                const double piv = Lj[j] - s;
                if (piv > tol) A[(size_t)j * lda + j] = sqrt(piv);
                else fail = 1;
            }
        }
        __syncthreads();
        if (fail) break;
        const double ljj = Lj[j];
        for (int i = j + 1 + warp; i < n; i += nw) {
            double *Li = A + (size_t)i * lda;
            double s = 0.0;
            for (int k = lane; k < j; k += 32) s += Li[k] * Lj[k];
            s = warp_sum(s);
            if (lane == 0) Li[j] = (Li[j] - s) / ljj;
        }
        __syncthreads();
    }
    if (tid == 0 && fail) atomicOr(status, 1);
}

// Y[rows, l] <- Y L^-T  (forward substitution, one warp per row staged in shared memory; L from fb_chol_kernel).  Skipped
// once *status is set, so a failed factorisation leaves finite values behind for the remaining kernels.
constexpr int FT_WARPS = 4;
__global__ void __launch_bounds__(FT_WARPS * 32) fb_trsm_rows_kernel(double *__restrict__ Y, int rows, int l, int ldy,
                                                                     const double *__restrict__ L, int ldl,
                                                                     const int *__restrict__ status) {
    extern __shared__ double ys[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, r = blockIdx.x * FT_WARPS + warp;
    if (r >= rows || *status) return;
    double *y = ys + (size_t)warp * l, *yg = Y + (size_t)r * ldy;
    for (int k = lane; k < l; k += 32) y[k] = yg[k];
    __syncwarp();
    for (int j = 0; j < l; ++j) {
        const double *Lj = L + (size_t)j * ldl;
        double s = 0.0;
        for (int k = lane; k < j; k += 32) s += Lj[k] * y[k];
        s = warp_sum(s);
        if (lane == 0) y[j] = (y[j] - s) / Lj[j];
        __syncwarp();
    }
    for (int k = lane; k < l; k += 32) yg[k] = y[k];
}

static int fb_trsm_rows(double *Y, int rows, int l, int ldy, const double *L, int ldl, const int *status, cudaStream_t st) {
    fb_trsm_rows_kernel<<<(rows + FT_WARPS - 1) / FT_WARPS, FT_WARPS * 32, (size_t)FT_WARPS * l * sizeof(double), st>>>(
        Y, rows, l, ldy, L, ldl, status);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// G = S + (raw ? n mean mean^T : 0)
__global__ void fb_form_g_kernel(double *__restrict__ G, const double *__restrict__ S, const double *__restrict__ mean,
                                 const double *__restrict__ hdr, int d, int raw) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
    if (j >= d) return;
    const size_t o = (size_t)i * d + j;
    G[o] = raw ? S[o] + hdr[0] * mean[i] * mean[j] : S[o];
}

// W[k, :] /= s_k  (s_k^2 = evals[k]; the eigenvector rows of F^T F become the columns of diag(1/s) W^T)
__global__ void fb_scale_rows_kernel(double *__restrict__ W, int c, int n, const double *__restrict__ evals) {
    const int k = blockIdx.x;
    const double e = evals[k], inv = e > 0.0 ? 1.0 / sqrt(e) : 0.0;
    for (int j = threadIdx.x; j < n; j += blockDim.x) W[(size_t)k * n + j] *= inv;
}

// stdev_k = sqrt(v_k^T S v_k / n) (= std(X v_k), X centred), total_var = tr S / n; rows re-sorted by descending stdev
// (np.argsort(stdev)[::-1]: equal values keep descending index order), var_ratio = stdev^2 / total_var.  T = S V^T [d, c].
__global__ void __launch_bounds__(512) fb_finish_kernel(const double *__restrict__ S, const double *__restrict__ hdr,
                                                          const double *__restrict__ V, const double *__restrict__ T, int d, int c,
                                                          double *__restrict__ out, double *__restrict__ stdev,
                                                          double *__restrict__ var_ratio) {
    __shared__ double red[33];
    __shared__ double q[1024];
    __shared__ int perm[1024];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = blockDim.x >> 5;
    double tr = 0.0;
    for (int i = tid; i < d; i += blockDim.x) tr += S[(size_t)i * d + i];
    tr = block_sum(tr, red);
    for (int k = warp; k < c; k += nw) {
        double s = 0.0;
        for (int i = lane; i < d; i += 32) s += V[(size_t)k * d + i] * T[(size_t)i * c + k];
        s = warp_sum(s);
        if (lane == 0) q[k] = s;
    }
    __syncthreads();
    for (int k = tid; k < c; k += blockDim.x) {
        int rank = 0;
        for (int j = 0; j < c; ++j) rank += (q[j] > q[k]) || (q[j] == q[k] && j > k);
        perm[rank] = k;
    }
    __syncthreads();
    const double n = hdr[0];
    for (int r = tid; r < c; r += blockDim.x) {
        const double qk = fmax(q[perm[r]], 0.0);
        stdev[r] = sqrt(qk / n);
        var_ratio[r] = qk / tr;
    }
    for (size_t idx = tid; idx < (size_t)c * d; idx += blockDim.x) {
        const int r = (int)(idx / d), i = (int)(idx % d);
        out[idx] = V[(size_t)perm[r] * d + i];
    }
}

}  // namespace gsb

extern "C" size_t gsb_fbpca_state_bytes(int d) {
    return gsb::fb_state(nullptr, d).bytes;
}

extern "C" int gsb_fbpca_reset(void *d_state, int d, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state, "fbpca_reset: null state");
    if (int r = gsb::check_fb_dims(d)) return r;
    GSB_CHECK_CUDA(cudaMemsetAsync(d_state, 0, gsb_fbpca_state_bytes(d), (cudaStream_t)stream));
    return GSB_OK;
}

static int fb_pool(void *d_state, int d, int n_groups, int64_t rows_per_group, const double *d_means, const double *d_grams,
                   cudaStream_t st) {
    gsb::FbState s = gsb::fb_state(d_state, d);
    dim3 grid((d + 127) / 128, d);
    gsb::fb_pool_scatter_kernel<<<grid, 128, 0, st>>>(s.S, s.mean, s.hdr, d_means, d_grams, n_groups, (double)rows_per_group, d);
    GSB_CHECK_LAUNCH();
    gsb::fb_pool_mean_kernel<<<1, (d + 31) / 32 * 32, 0, st>>>(s.mean, s.hdr, d_means, n_groups, (double)rows_per_group, d);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_fbpca_accumulate(void *d_state, int d, int n_groups, int64_t rows_per_group, const double *d_means,
                                    const double *d_grams, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && d_means && d_grams, "fbpca_accumulate: null pointer");
    if (int r = gsb::check_fb_dims(d)) return r;
    GSB_CHECK_ARG(n_groups >= 1 && rows_per_group >= 1, "fbpca_accumulate: bad counts");
    return fb_pool(d_state, d, n_groups, rows_per_group, d_means, d_grams, (cudaStream_t)stream);
}

extern "C" int gsb_fbpca_add_zero_rows(void *d_state, int d, int64_t n_zero, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state, "fbpca_add_zero_rows: null state");
    if (int r = gsb::check_fb_dims(d)) return r;
    GSB_CHECK_ARG(n_zero >= 0, "fbpca_add_zero_rows: bad count");
    if (n_zero == 0) return GSB_OK;
    return fb_pool(d_state, d, 1, n_zero, nullptr, nullptr, (cudaStream_t)stream);
}

extern "C" size_t gsb_fbpca_workspace_bytes(int d, int c, int l) {
    return gsb::fb_carve(nullptr, d, c, l).bytes;
}

extern "C" int gsb_fbpca_solve(void *d_state, int d, int c, int l, int flags, const double *d_omega, double *d_components,
                               double *d_stdev, double *d_var_ratio, double *d_mean, void *d_workspace, size_t workspace_bytes,
                               gsb_stream_t stream) {
    using namespace gsb;
    GSB_CHECK_ARG(d_state && d_components && d_stdev && d_var_ratio && d_workspace, "fbpca_solve: null pointer");
    if (int r = check_fb_dims(d)) return r;
    GSB_CHECK_ARG(c >= 1 && c <= d && l >= c && (d_omega == nullptr || l < d), "fbpca_solve: need 1 <= c <= l (< d) (c=%d l=%d d=%d)",
                  c, l, d);
    GSB_CHECK_ARG((flags & ~GSB_FBPCA_RAW) == 0, "fbpca_solve: unknown flags %d", flags);
    FbWs w = fb_carve(d_workspace, d, c, l);
    if (workspace_bytes < w.bytes) {
        set_error("fbpca_solve: workspace too small (%zu < %zu)", workspace_bytes, w.bytes);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    FbState s = fb_state(d_state, d);
    const int lp = lpad(l);
    dim3 gd((d + 127) / 128, d);
    if (d_omega == nullptr) {
        // exact branch: the top-c right singular vectors of X are the top-c eigenvectors of G
        fb_form_g_kernel<<<gd, 128, 0, st>>>(w.eig.A, s.S, s.mean, s.hdr, d, flags & GSB_FBPCA_RAW);
        GSB_CHECK_LAUNCH();
        if (int r = eig_top(w.eig, d, c, w.eig.lam, w.comp, st)) return r;
    } else {
        GSB_CHECK_CUDA(cudaMemsetAsync(w.Y, 0, (size_t)d * lp * 8, st));
        GSB_CHECK_CUDA(cudaMemsetAsync(w.P, 0, (size_t)d * lp * 8, st));
        GSB_CHECK_CUDA(cudaMemsetAsync(w.Sm, 0, (size_t)lp * lp * 8, st));
        fb_form_g_kernel<<<gd, 128, 0, st>>>(w.G, s.S, s.mean, s.hdr, d, flags & GSB_FBPCA_RAW);
        GSB_CHECK_LAUNCH();
        // Y = orth(G^2 Omega): two products, each followed by CholQR2 (Y <- Y chol(Y^T Y)^-T, twice)
        const double *src = d_omega;
        for (int it = 0; it < 2; ++it) {
            if (int r = fb_gemm<false, false>(d, l, d, w.G, d, src, it == 0 ? l : lp, w.Y, lp, st)) return r;
            for (int rep = 0; rep < 2; ++rep) {
                if (int r = fb_gemm<true, false>(l, l, d, w.Y, lp, w.Y, lp, w.Sm, lp, st)) return r;
                fb_chol_kernel<<<1, 1024, 0, st>>>(w.Sm, l, lp, s.status);
                GSB_CHECK_LAUNCH();
                if (int r = fb_trsm_rows(w.Y, d, l, lp, w.Sm, lp, s.status, st)) return r;
            }
            if (it == 0) {
                GSB_CHECK_CUDA(cudaMemcpyAsync(w.P, w.Y, (size_t)d * lp * 8, cudaMemcpyDeviceToDevice, st));
                src = w.P;
            }
        }
        // P = G Y,  L = chol(Y^T P),  F = P L^-T  (in place in P)
        if (int r = fb_gemm<false, false>(d, l, d, w.G, d, w.Y, lp, w.P, lp, st)) return r;
        if (int r = fb_gemm<true, false>(l, l, d, w.Y, lp, w.P, lp, w.Sm, lp, st)) return r;
        fb_chol_kernel<<<1, 1024, 0, st>>>(w.Sm, l, lp, s.status);
        GSB_CHECK_LAUNCH();
        if (int r = fb_trsm_rows(w.P, d, l, lp, w.Sm, lp, s.status, st)) return r;
        // F^T F (lp x lp, zero-padded so that the eigensolver sees a multiple of 32) -> top-c (s^2, W)
        if (int r = fb_gemm<true, false>(lp, lp, d, w.P, lp, w.P, lp, w.eig.A, lp, st)) return r;
        if (int r = eig_top(w.eig, lp, c, w.eig.lam, w.eig.evecs, st)) return r;
        // Va = diag(1/s) W^T F^T  [c, d]
        fb_scale_rows_kernel<<<c, 128, 0, st>>>(w.eig.evecs, c, lp, w.eig.lam);
        GSB_CHECK_LAUNCH();
        if (int r = fb_gemm<false, true>(c, d, lp, w.eig.evecs, lp, w.P, lp, w.comp, d, st)) return r;
    }
    // stdevs from the centred scatter, sort, sign rule (largest-|.| entry of each row positive)
    if (int r = fb_gemm<false, true>(d, c, d, s.S, d, w.comp, d, w.T, c, st)) return r;
    fb_finish_kernel<<<1, 512, 0, st>>>(s.S, s.hdr, w.comp, w.T, d, c, d_components, d_stdev, d_var_ratio);
    GSB_CHECK_LAUNCH();
    if (int r = sign_rows(d_components, c, d, st)) return r;
    if (d_mean) GSB_CHECK_CUDA(cudaMemcpyAsync(d_mean, s.mean, (size_t)d * 8, cudaMemcpyDeviceToDevice, st));
    return GSB_OK;
}

extern "C" int gsb_fbpca_project_omega(const double *d_Q, int d, int r, const float *d_omega, int l, double *d_omega_r,
                                       gsb_stream_t stream) {
    GSB_CHECK_ARG(d_Q && d_omega && d_omega_r, "fbpca_project_omega: null pointer");
    GSB_CHECK_ARG(d >= 1 && r >= 1 && r <= 1024 && l >= 1 && l <= 1024,
                  "fbpca_project_omega: needs d >= 1, 1 <= r <= 1024, 1 <= l <= 1024 (d=%d r=%d l=%d)", d, r, l);
    dim3 grid((l + 31) / 32, (r + 31) / 32);
    gsb::fb_project_kernel<<<grid, 128 * gsb::FP_SPLIT, 0, (cudaStream_t)stream>>>(r, l, d, d_Q, d_omega, d_omega_r);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_fbpca_status(void *d_state, int d, unsigned *h_flags, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && h_flags, "fbpca_status: null pointer");
    if (int r = gsb::check_fb_dims(d)) return r;
    gsb::FbState s = gsb::fb_state(d_state, d);
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CHECK_CUDA(cudaMemcpyAsync(h_flags, s.status, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    GSB_CHECK_CUDA(cudaMemsetAsync(s.status, 0, sizeof(int), st));
    GSB_CHECK_CUDA(cudaStreamSynchronize(st));
    return GSB_OK;
}
