// Incremental-PCA chain, small-d engine (d <= 1024): all state and arithmetic fp64, on device.
//
// Replaces estimators.py:55-81 (IPCAEstimator.fit_partial / get_components), i.e. scikit-learn's
// IncrementalPCA.partial_fit (_incremental_pca.py:254-380) in its Gram form (SURVEY.md section 0.3):
//     G = V^T S^2 V + Xc^T Xc + m m^T,   m = sqrt(n_seen*n_b/n_tot) (mean - mean_b)
//     top-c eigenpairs of G  ->  components_ (svd_flip sign rule), singular_values_ = sqrt(lambda)
//     mean/var merge of extmath._incremental_mean_and_var (Chan et al.), batch variance = diag(Xc^T Xc)
//
// The symmetric eigensolver is the classical direct route, written for one GPU:
//   1. tridiag_kernel   Householder tridiagonalisation spread over P = n/8 CTAs (column-cyclic, each CTA's
//                       columns resident in its shared memory), ONE grid barrier per reflector: the fused
//                       pass applies the pending rank-2 update, accumulates A v for the next reflector and
//                       extracts the next pivot row; every CTA rebuilds v / w redundantly from the two
//                       exchanged n-vectors, so nothing else crosses SMs.
//   2. bisect_kernel    top-c eigenvalues of T by 32-way multisection (one warp per eigenvalue, Sturm counts).
//   3. invit_kernel     eigenvectors of T by inverse iteration on the pivoted LU of T - lambda I.
//   4. backtransform_kernel  applies the reflectors (one warp per eigenvector) and the sign rule.
#include "ipca_internal.cuh"
#include <math.h>

namespace gsb {

// state header doubles: [0] n_seen, [1] steps, [2] form (0: (V, S) valid; 1: subspace form, (Q, H) authoritative),
// [3] current Q buffer, [4] iterations of the last subspace step, [5] its relative residual, [6] max residual, [7] total iterations
constexpr int ST_HDR = 24;   // [8..23]: clocks per phase of the subspace steps (CTA 0), a profiling aid

struct StateView {
    double *hdr, *mean, *unnorm, *S, *V;
    double *H, *Qbuf;        // subspace form: H[c,c], Q[2][d][c+4] (ping-pong)
    void *eig_ws;            // workspace of the export-time eigen-decomposition of H
    size_t bytes;
};
static inline size_t export_eig_n(int c) { return (size_t)(c + 31) / 32 * 32; }
inline StateView state_view(void *p, int d, int c) {
    StateView s;
    s.hdr = reinterpret_cast<double *>(p);
    s.mean = s.hdr + ST_HDR;
    s.unnorm = s.mean + d;
    s.S = s.unnorm + d;
    s.V = s.S + c;
    size_t off = align_up((size_t)(ST_HDR + 2 * (size_t)d + c + (size_t)c * d) * sizeof(double), 256);
    s.H = s.Qbuf = nullptr; s.eig_ws = nullptr;
    if (subspace_applicable(d, c)) {
        char *b = reinterpret_cast<char *>(p);
        s.H = reinterpret_cast<double *>(b + off); off += align_up((size_t)c * c * 8, 256);
        s.Qbuf = reinterpret_cast<double *>(b + off); off += align_up((size_t)2 * d * (c + 4) * 8, 256);
        s.eig_ws = b + off; off += carve(nullptr, (int)export_eig_n(c), c).bytes;
    }
    s.bytes = off;
    return s;
}

Workspace carve(void *base, int d, int c) {
    Workspace w;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    w.A = (double *)take((size_t)d * d * 8);
    w.dg = (double *)take((size_t)d * 8);
    w.e = (double *)take((size_t)d * 8);
    w.beta = (double *)take((size_t)d * 8);
    w.Vh = (double *)take((size_t)d * d * 8);
    w.lam = (double *)take((size_t)c * 8);
    w.Z = (double *)take((size_t)c * d * 8);
    w.evecs = (double *)take((size_t)c * d * 8);
    w.lu = (double *)take((size_t)5 * d * c * 8);
    w.swp = (unsigned char *)take((size_t)d * c);
    w.xch = (double *)take((size_t)4 * d * 8);
    w.qx = (double *)take((size_t)2 * 16 * 512 * 8);
    w.counter = (unsigned *)take(256);
    w.bytes = off;
    return w;
}

// ---------------------------------------------------------------------------------------------
// G = gram_b + m m^T + sum_t S_t^2 v_t v_t^T      (first step: G = gram_b)
// ---------------------------------------------------------------------------------------------
constexpr int BG_T = 32;
__global__ void build_g_kernel(const double *__restrict__ gram_b, const double *__restrict__ mean_b,
                               const double *__restrict__ mean, const double *__restrict__ S,
                               const double *__restrict__ V, int d, int c, double n_seen, double n_b,
                               double *__restrict__ G) {
    __shared__ double Vi[BG_T][33], Vj[BG_T][33], s2[BG_T];
    const int tx = threadIdx.x, ty = threadIdx.y;   // 32 x 8
    const int j = blockIdx.x * 32 + tx;
    const int i0 = blockIdx.y * 32;
    double acc[4] = {0, 0, 0, 0};
    if (n_seen > 0) {
        for (int t0 = 0; t0 < c; t0 += BG_T) {
            for (int tt = ty; tt < BG_T; tt += 8) {
                int t = t0 + tt;
                bool ok = t < c;
                Vi[tt][tx] = (ok && i0 + tx < d) ? V[(size_t)t * d + i0 + tx] : 0.0;
                Vj[tt][tx] = (ok && j < d) ? V[(size_t)t * d + j] : 0.0;
                if (tx == 0) { double s = ok ? S[t] : 0.0; s2[tt] = s * s; }
            }
            __syncthreads();
#pragma unroll 8
            for (int tt = 0; tt < BG_T; ++tt) {
                double vj = Vj[tt][tx] * s2[tt];
#pragma unroll
                for (int r = 0; r < 4; ++r) acc[r] += Vi[tt][ty + 8 * r] * vj;
            }
            __syncthreads();
        }
    }
    if (j >= d) return;
    const double f = (n_seen > 0) ? sqrt((n_seen / (n_seen + n_b)) * n_b) : 0.0;
    const double mj = (n_seen > 0) ? f * (mean[j] - mean_b[j]) : 0.0;
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        int i = i0 + ty + 8 * r;
        if (i >= d) continue;
        double mi = (n_seen > 0) ? f * (mean[i] - mean_b[i]) : 0.0;
        G[(size_t)i * d + j] = gram_b[(size_t)i * d + j] + mi * mj + acc[r];
    }
}

// ---------------------------------------------------------------------------------------------
// grid barrier (all CTAs of the launch are co-resident: grid <= #SMs, 1 CTA each fits trivially)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned *p) {
    unsigned v;
    asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
    return v;
}
__device__ __forceinline__ void grid_barrier(unsigned *counter, unsigned target) {
    __syncthreads();
    if (threadIdx.x == 0) {
        __threadfence();
        atomicAdd(counter, 1u);
        while (ld_acquire_u32(counter) < target) { }
        __threadfence();
    }
    __syncthreads();
}

// ---------------------------------------------------------------------------------------------
// Householder tridiagonalisation  A = Q T Q^T,  Q = H_0 H_1 ... H_{n-3},  H_k = I - beta_k v_k v_k^T
// ---------------------------------------------------------------------------------------------
constexpr int TRI_THREADS_GRID = 256;      // global-barrier variant: P = n/8 CTAs
constexpr int TRI_THREADS_CLUSTER = 512;   // cluster variant: one 16-CTA cluster, hardware barrier
constexpr int TRI_CLUSTER = 16;

__device__ __forceinline__ void cluster_barrier() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// CLUSTER = false: any number of co-resident CTAs, software barrier on a global counter.
// CLUSTER = true : the grid is ONE thread-block cluster (16 CTAs, non-portable size); the per-reflector
//                  exchange is ordered by barrier.cluster (release/acquire), ~5x cheaper than the atomic
//                  counter, and the column blocks (n/16 columns = 128 KB for n = 512) stay in shared memory.
template <bool CLUSTER>
__global__ void __launch_bounds__(CLUSTER ? TRI_THREADS_CLUSTER : TRI_THREADS_GRID, 1)
tridiag_kernel(const double *__restrict__ A, int n, double *__restrict__ dg, double *__restrict__ e,
               double *__restrict__ beta, double *__restrict__ Vh, double *__restrict__ xch,
               unsigned *__restrict__ counter) {
    extern __shared__ double smd[];
    const int TRI_THREADS = blockDim.x;
    const int P = gridDim.x, me = blockIdx.x, tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = TRI_THREADS / 32;
    const int ncl = n / P;
    double *Aloc = smd;               // [ncl][n]   owned columns j = me + P*l
    double *a = Aloc + (size_t)ncl * n;   // current pivot column (rows > k valid)
    double *v = a + n;
    double *w = v + n;
    double *pv = w + n;               // pending rank-2 update (v_{k-1}, w_{k-1})
    double *pw = pv + n;
    double *red = pw + n;             // [64]

    for (int l = 0; l < ncl; ++l) {
        const double *src = A + (size_t)(me + P * l) * n;   // row j == column j (symmetric)
        for (int i = tid; i < n; i += TRI_THREADS) Aloc[(size_t)l * n + i] = src[i];
    }
    for (int i = tid; i < n; i += TRI_THREADS) {
        a[i] = A[i];
        pv[i] = 0.0;
        pw[i] = 0.0;
        w[i] = 0.0;
    }
    if (me == 0 && tid == 0) dg[0] = A[0];
    __syncthreads();

    unsigned target = 0;
    for (int k = 0; k <= n - 3; ++k) {
        const int par = k & 1;
        double *Pbuf = xch + (size_t)par * 2 * n, *Rbuf = Pbuf + n;
        // ---- 1. reflector from a[k+1 .. n-1] (redundant in every CTA) ---------------------------
        const double x0 = a[k + 1];
        double part = 0.0;
        for (int i = k + 2 + tid; i < n; i += TRI_THREADS) part += a[i] * a[i];
        const double sigma = block_sum(part, red);
        double alpha, bk, v0;
        if (sigma == 0.0) {
            alpha = x0; bk = 0.0; v0 = 0.0;
        } else {
            const double nrm = sqrt(x0 * x0 + sigma);
            alpha = (x0 > 0.0) ? -nrm : nrm;
            v0 = x0 - alpha;
            bk = 1.0 / (nrm * (nrm + fabs(x0)));     // 2 / (v^T v)
        }
        for (int i = tid; i < n; i += TRI_THREADS)
            v[i] = (i <= k || bk == 0.0) ? 0.0 : ((i == k + 1) ? v0 : a[i]);
        __syncthreads();
        if (me == 0) {
            if (tid == 0) { e[k] = alpha; beta[k] = bk; }
            for (int i = tid; i < n; i += TRI_THREADS) Vh[(size_t)k * n + i] = v[i];
        }
        // ---- 2. fused local pass: pending update, p = A v, next pivot row ------------------------
        for (int l = warp; l < ncl; l += nwarps) {
            const int j = me + P * l;
            if (j <= k) continue;
            double *col = Aloc + (size_t)l * n;
            const double pvj = pv[j], pwj = pw[j];
            double acc = 0.0, rj = 0.0;
            for (int i = k + 1 + lane; i < n; i += 32) {
                double x = col[i] - pv[i] * pwj - pw[i] * pvj;
                col[i] = x;
                acc += x * v[i];
                if (i == k + 1) rj = x;
            }
            acc = warp_sum(acc);
            if (lane == 0) {
                __stcg(&Pbuf[j], bk * acc);
                __stcg(&Rbuf[j], rj);
            }
        }
        // ---- 3. exchange ---------------------------------------------------------------------
        if (CLUSTER) {
            __syncthreads();
            cluster_barrier();
        } else {
            target += (unsigned)P;
            grid_barrier(counter, target);
        }
        // ---- 4. w, next pivot column (redundant in every CTA) -------------------------------------
        part = 0.0;
        for (int i = k + 1 + tid; i < n; i += TRI_THREADS) {
            double pi = __ldcg(&Pbuf[i]);
            w[i] = pi;
            a[i] = __ldcg(&Rbuf[i]);
            part += pi * v[i];
        }
        const double ptv = block_sum(part, red);
        const double K2 = 0.5 * bk * ptv;
        for (int i = k + 1 + tid; i < n; i += TRI_THREADS) w[i] -= K2 * v[i];
        __syncthreads();
        const double vk1 = v[k + 1], wk1 = w[k + 1];
        for (int i = k + 1 + tid; i < n; i += TRI_THREADS) a[i] -= vk1 * w[i] + wk1 * v[i];
        __syncthreads();
        if (me == 0 && tid == 0) dg[k + 1] = a[k + 1];
        double *t = pv; pv = v; v = t;
        t = pw; pw = w; w = t;
    }
    // last 2x2 block: e[n-2] = A[n-1,n-2] (held in a[n-1]); dg[n-1] needs the pending update
    if (me == 0 && tid == 0) { e[n - 2] = a[n - 1]; e[n - 1] = 0.0; beta[n - 2] = 0.0; beta[n - 1] = 0.0; }
    if (me == (n - 1) % P && tid == 0) {
        int l = (n - 1) / P;
        dg[n - 1] = Aloc[(size_t)l * n + (n - 1)] - 2.0 * pv[n - 1] * pw[n - 1];
    }
}

// ---------------------------------------------------------------------------------------------
// L2-resident variant for 1024 < n <= 4096 (the small side of the large-d engine, n = c + NB + 1 ~ 2100): the
// matrix (n^2 fp64 = 36 MB at n = 2112) does not fit the shared memory of the machine but sits in the 50 MB L2.
// Same algorithm and exchange as tridiag_kernel<false> (one software grid barrier per reflector); the owned
// columns j = me + P l are updated IN PLACE in global memory (row j of the symmetric input == column j), one warp
// per column, four independent 256-byte segments in flight per lane.  P ~ n/16 co-resident CTAs of 16 warps.
// ---------------------------------------------------------------------------------------------
constexpr int TRL_THREADS = 512;
__global__ void __launch_bounds__(TRL_THREADS, 1)
tridiag_l2_kernel(double *__restrict__ A, int n, double *__restrict__ dg, double *__restrict__ e,
                  double *__restrict__ beta, double *__restrict__ Vh, double *__restrict__ xch,
                  unsigned *__restrict__ counter) {
    extern __shared__ double smd[];
    const int P = gridDim.x, me = blockIdx.x, tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = TRL_THREADS / 32;
    const int ncl = (n + P - 1) / P;
    double *a = smd;                  // current pivot column (rows > k valid)
    double *v = a + n;
    double *w = v + n;
    double *pv = w + n;               // pending rank-2 update (v_{k-1}, w_{k-1})
    double *pw = pv + n;
    double *red = pw + n;             // [64]

    for (int i = tid; i < n; i += TRL_THREADS) {
        a[i] = A[i];                  // column 0 (never modified: only columns j > k are touched)
        pv[i] = 0.0;
        pw[i] = 0.0;
        w[i] = 0.0;
    }
    if (me == 0 && tid == 0) dg[0] = A[0];
    __syncthreads();

    unsigned target = 0;
    for (int k = 0; k <= n - 3; ++k) {
        const int par = k & 1;
        double *Pbuf = xch + (size_t)par * 2 * n, *Rbuf = Pbuf + n;
        // ---- 1. reflector from a[k+1 .. n-1] (redundant in every CTA) ---------------------------
        const double x0 = a[k + 1];
        double part = 0.0;
        for (int i = k + 2 + tid; i < n; i += TRL_THREADS) part += a[i] * a[i];
        const double sigma = block_sum(part, red);
        double alpha, bk, v0;
        if (sigma == 0.0) {
            alpha = x0; bk = 0.0; v0 = 0.0;
        } else {
            const double nrm = sqrt(x0 * x0 + sigma);
            alpha = (x0 > 0.0) ? -nrm : nrm;
            v0 = x0 - alpha;
            bk = 1.0 / (nrm * (nrm + fabs(x0)));     // 2 / (v^T v)
        }
        for (int i = tid; i < n; i += TRL_THREADS)
            v[i] = (i <= k || bk == 0.0) ? 0.0 : ((i == k + 1) ? v0 : a[i]);
        __syncthreads();
        if (me == 0) {
            if (tid == 0) { e[k] = alpha; beta[k] = bk; }
            for (int i = tid; i < n; i += TRL_THREADS) Vh[(size_t)k * n + i] = v[i];
        }
        // ---- 2. fused pass over the owned columns: pending update, p = A v, next pivot row ---------
        for (int l = warp; l < ncl; l += nwarps) {
            const int j = me + P * l;
            if (j >= n || j <= k) continue;
            double *col = A + (size_t)j * n;
            const double pvj = pv[j], pwj = pw[j];
            double acc = 0.0, rj = 0.0;
            int i = k + 1 + lane;
            for (; i + 96 < n; i += 128) {
                const double c0 = col[i], c1 = col[i + 32], c2 = col[i + 64], c3 = col[i + 96];
                const double x0_ = c0 - pv[i] * pwj - pw[i] * pvj;
                const double x1_ = c1 - pv[i + 32] * pwj - pw[i + 32] * pvj;
                const double x2_ = c2 - pv[i + 64] * pwj - pw[i + 64] * pvj;
                const double x3_ = c3 - pv[i + 96] * pwj - pw[i + 96] * pvj;
                col[i] = x0_; col[i + 32] = x1_; col[i + 64] = x2_; col[i + 96] = x3_;
                acc += x0_ * v[i] + x1_ * v[i + 32] + x2_ * v[i + 64] + x3_ * v[i + 96];
                if (i == k + 1) rj = x0_;
            }
            for (; i < n; i += 32) {
                const double x = col[i] - pv[i] * pwj - pw[i] * pvj;
                col[i] = x;
                acc += x * v[i];
                if (i == k + 1) rj = x;
            }
            acc = warp_sum(acc);
            if (lane == 0) {                    // lane 0 owns row k+1 (i starts at k+1+lane)
                __stcg(&Pbuf[j], bk * acc);
                __stcg(&Rbuf[j], rj);
            }
        }
        // ---- 3. exchange ---------------------------------------------------------------------
        target += (unsigned)P;
        grid_barrier(counter, target);
        // ---- 4. w, next pivot column (redundant in every CTA) -------------------------------------
        part = 0.0;
        for (int i = k + 1 + tid; i < n; i += TRL_THREADS) {
            double pi = __ldcg(&Pbuf[i]);
            w[i] = pi;
            a[i] = __ldcg(&Rbuf[i]);
            part += pi * v[i];
        }
        const double ptv = block_sum(part, red);
        const double K2 = 0.5 * bk * ptv;
        for (int i = k + 1 + tid; i < n; i += TRL_THREADS) w[i] -= K2 * v[i];
        __syncthreads();
        const double vk1 = v[k + 1], wk1 = w[k + 1];
        for (int i = k + 1 + tid; i < n; i += TRL_THREADS) a[i] -= vk1 * w[i] + wk1 * v[i];
        __syncthreads();
        if (me == 0 && tid == 0) dg[k + 1] = a[k + 1];
        double *t = pv; pv = v; v = t;
        t = pw; pw = w; w = t;
    }
    if (me == 0 && tid == 0) { e[n - 2] = a[n - 1]; e[n - 1] = 0.0; beta[n - 2] = 0.0; beta[n - 1] = 0.0; }
    if (me == (n - 1) % P && tid == 0)
        dg[n - 1] = A[(size_t)(n - 1) * n + (n - 1)] - 2.0 * pv[n - 1] * pw[n - 1];
}

// ---------------------------------------------------------------------------------------------
// Register-resident variant of the cluster tridiagonalisation (n <= 512, n % 16 == 0).
// The shared-memory variants above spend their time on shared-memory bandwidth (every matrix element
// is read and written once per reflector, plus three vector operands).  Here the CTA's column block
// lives in REGISTERS: thread (warp w, lane l) owns row i = nw l + w (nw = 16 or 8 warps) of the CTA's <= 32 columns
// j = me + 16 c.  Per reflector a thread applies the pending rank-2 update to its 32 elements with the
// column operands broadcast from shared memory, the per-column sums are formed by a 31-shuffle
// transpose-reduce inside each warp and a 16-way add across warps, and all row-indexed vector work
// (v_i, w_i, next pivot column) is O(1) per thread.
// ---------------------------------------------------------------------------------------------
constexpr int TRR_NC = 32;   // columns per CTA (registers)
// qx: [2][16][512] doubles of per-CTA partial products (row-permuted so that a warp reads 256 contiguous bytes)
__global__ void __launch_bounds__(TRI_THREADS_CLUSTER, 1)
tridiag_reg_kernel(const double *__restrict__ A, int n, double *__restrict__ dg, double *__restrict__ e,
                   double *__restrict__ beta, double *__restrict__ Vh, double *__restrict__ xch,
                   double *__restrict__ qx) {
    __shared__ double vsh[512];                 // v_k by row / column index
    __shared__ double2 pvw[512];                // pending (v_{k-1}, w_{k-1}) by row / column index
    __shared__ double red[64];
    const int me = blockIdx.x, tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int nc = n / TRI_CLUSTER;             // active columns of this CTA
    const int nw = blockDim.x >> 5;             // 16 warps (n <= 512) or 8 warps (n <= 256): one row per thread
    const int i = nw * lane + warp;             // own row
    const bool row_ok = i < n;

    double Areg[TRR_NC];
#pragma unroll
    for (int c = 0; c < TRR_NC; ++c) {
        const int j = me + TRI_CLUSTER * c;
        Areg[c] = (row_ok && c < nc) ? A[(size_t)j * n + i] : 0.0;      // A[i][j] == A[j][i]
    }
    double a_i = row_ok ? A[i] : 0.0;            // pivot column 0 (row 0 of A), own row
    double pv_i = 0.0, pw_i = 0.0;
    for (int q = tid; q < 512; q += blockDim.x) pvw[q] = make_double2(0.0, 0.0);
    if (me == 0 && tid == 0) dg[0] = A[0];
    __syncthreads();

    for (int k = 0; k <= n - 3; ++k) {
        const int par = k & 1;
        double *Rbuf = xch + (size_t)par * n;
        double *Qbuf = qx + (size_t)par * TRI_CLUSTER * 512;
        // ---- 1. reflector (redundant in every CTA; one row per thread) ---------------------------
        if (i == k + 1) red[32] = a_i;
        const double sigma = block_sum((row_ok && i > k + 1) ? a_i * a_i : 0.0, red);
        const double x0 = red[32];
        double alpha, bk, v0;
        if (sigma == 0.0) {
            alpha = x0; bk = 0.0; v0 = 0.0;
        } else {
            const double nrm = sqrt(x0 * x0 + sigma);
            alpha = (x0 > 0.0) ? -nrm : nrm;
            v0 = x0 - alpha;
            bk = 1.0 / (nrm * (nrm + fabs(x0)));
        }
        const double v_i = (!row_ok || i <= k || bk == 0.0) ? 0.0 : ((i == k + 1) ? v0 : a_i);
        if (row_ok) vsh[i] = v_i;                                // every index < n has exactly one owner
        __syncthreads();
        if (me == 0) {
            if (tid == 0) { e[k] = alpha; beta[k] = bk; }
            for (int q = tid; q < n; q += blockDim.x) Vh[(size_t)k * n + q] = vsh[q];
        }
        // ---- 2. pending rank-2 update + this CTA's share of (A v)_i, row-wise (A is symmetric) ----------
        // columns j = me + 16 c with j > k are live:  c0 <= c < nc
        const int c0 = (k >= me) ? ((k - me) / TRI_CLUSTER + 1) : 0;
        const bool pivot_row = (i == k + 1);
        double q = 0.0;
#pragma unroll
        for (int c = 0; c < TRR_NC; ++c) {
            if ((unsigned)(c - c0) < (unsigned)(nc - c0)) {
                const int j = me + TRI_CLUSTER * c;
                const double2 pj = pvw[j];                       // broadcast: (pv_j, pw_j)
                const double x = Areg[c] - pv_i * pj.y - pw_i * pj.x;
                Areg[c] = x;
                q += x * vsh[j];
                if (pivot_row) __stcg(&Rbuf[j], x);              // pivot row of A^(k)
            }
        }
        __stcg(&Qbuf[me * 512 + tid], q);                        // row i's partial, permuted index = tid
        // ---- 3. exchange -------------------------------------------------------------------------
        cluster_barrier();
        // ---- 4. p, w, next pivot column (one row per thread) ------------------------------------------
        const bool act = row_ok && i > k;
        double p_i = 0.0;
        if (act) {
            double t0 = 0.0, t1 = 0.0;
#pragma unroll
            for (int r = 0; r < TRI_CLUSTER; r += 2) {
                t0 += __ldcg(&Qbuf[r * 512 + tid]);
                t1 += __ldcg(&Qbuf[(r + 1) * 512 + tid]);
            }
            p_i = bk * (t0 + t1);
        }
        const double r_i = act ? __ldcg(&Rbuf[i]) : 0.0;
        const double ptv = block_sum(p_i * v_i, red);
        const double w_i = p_i - 0.5 * bk * ptv * v_i;
        if (i == k + 1) { red[33] = v_i; red[34] = w_i; }
        if (row_ok) pvw[i] = make_double2(v_i, w_i);
        __syncthreads();
        const double vk1 = red[33], wk1 = red[34];
        a_i = act ? (r_i - vk1 * w_i - wk1 * v_i) : 0.0;
        pv_i = v_i; pw_i = w_i;
        if (me == 0 && i == k + 1) dg[k + 1] = a_i;
    }
    // last 2x2 block
    if (me == 0 && i == n - 1) { e[n - 2] = a_i; e[n - 1] = 0.0; beta[n - 2] = 0.0; beta[n - 1] = 0.0; }
    if (me == (n - 1) % TRI_CLUSTER && i == n - 1) {
        const int cl = (n - 1) / TRI_CLUSTER;
        double last = 0.0;
#pragma unroll
        for (int c = 0; c < TRR_NC; ++c) if (c == cl) last = Areg[c];
        dg[n - 1] = last - 2.0 * pv_i * pw_i;
    }
}

// ---------------------------------------------------------------------------------------------
// top-c eigenvalues of the tridiagonal T: 128-way multisection on Sturm counts, one CTA per eigenvalue.
// The count uses the division-free three-term recurrence  p_i = (d_i - x) p_{i-1} - e_{i-1}^2 p_{i-2}
// (q_i = p_i / p_{i-1} are the LDL^T pivots whose negative signs are counted); T is pre-scaled by a power
// of two so that |d - x| <= 2, e^2 <= 1, and (p_i, p_{i-1}) is renormalised by an exact power of two every
// 8 steps.  The dependent chain is one DFMA per row instead of a division.
// ---------------------------------------------------------------------------------------------
constexpr int BIS_THREADS = 128;
__global__ void __launch_bounds__(BIS_THREADS)
bisect_kernel(const double *__restrict__ dg, const double *__restrict__ e, int n, int c,
              double *__restrict__ lam) {
    extern __shared__ double smd[];
    double *sd = smd, *se2 = smd + n, *red = se2 + n;   // red[64]
    __shared__ double s_x[BIS_THREADS];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    double gl = 1e300, gu = -1e300;
    for (int i = tid; i < n; i += BIS_THREADS) {
        double di = dg[i];
        double el = (i > 0) ? fabs(e[i - 1]) : 0.0, er = (i < n - 1) ? fabs(e[i]) : 0.0;
        gl = fmin(gl, di - el - er);
        gu = fmax(gu, di + el + er);
    }
    for (int o = 16; o > 0; o >>= 1) {
        gl = fmin(gl, __shfl_xor_sync(0xffffffffu, gl, o));
        gu = fmax(gu, __shfl_xor_sync(0xffffffffu, gu, o));
    }
    if (lane == 0) { red[warp] = gl; red[8 + warp] = gu; }
    __syncthreads();
    gl = red[0]; gu = red[8];
    for (int q = 1; q < BIS_THREADS / 32; ++q) { gl = fmin(gl, red[q]); gu = fmax(gu, red[8 + q]); }
    const double eps = 2.220446049250313e-16;
    double tnorm = fmax(fabs(gl), fabs(gu));
    if (!(tnorm > 0.0)) tnorm = 1.0;
    int ex;
    frexp(tnorm, &ex);
    const double sc = ldexp(1.0, -ex);               // power of two: scaled spectrum within [-1, 1]
    for (int i = tid; i < n; i += BIS_THREADS) {
        sd[i] = dg[i] * sc;
        double es = (i < n - 1) ? e[i] * sc : 0.0;
        se2[i] = es * es;
    }
    __syncthreads();
    const int t = blockIdx.x;                         // t-th largest
    const int m = n - 1 - t;                          // ascending index
    const double margin = 4.0 * eps * n;
    double lo = gl * sc - margin, hi = gu * sc + margin;
    for (int it = 0; it < 12; ++it) {
        const double width = hi - lo;
        const double x = lo + width * ((double)(tid + 1) / (double)(BIS_THREADS + 1));
        // number of eigenvalues < x  =  number of sign changes p_{i-1} -> p_i  (sign bits of the high
        // words; an exact zero is taken as positive and shows up as a change one row later)
        int cnt = 0;
        double pm = 1.0, pc = sd[0] - x;              // p_{-1}, p_0
        cnt += (unsigned)__double2hiint(pc) >> 31;
        for (int i0 = 1; i0 < n; i0 += 8) {
            const int i1 = (i0 + 8 < n) ? i0 + 8 : n;
#pragma unroll 8
            for (int i = i0; i < i1; ++i) {
                const double pn = (sd[i] - x) * pc - se2[i - 1] * pm;
                cnt += (unsigned)(__double2hiint(pn) ^ __double2hiint(pc)) >> 31;
                pm = pc; pc = pn;
            }
            // renormalise by an exact power of two (keeps signs and the ratio)
            const double mag = fmax(fabs(pc), fabs(pm));
            const int eb = ((__double2hiint(mag) >> 20) & 0x7ff) - 1023;
            if (eb > 200 || eb < -200) {
                const double f = (mag > 0.0) ? __hiloint2double((1023 - eb) << 20, 0) : 1.0;
                pc *= f; pm *= f;
                if (mag == 0.0) { pc = 1e-300; pm = 0.0; }
            }
        }
        s_x[tid] = x;
        __syncthreads();
        // first probe with count >= m+1 bounds the eigenvalue from above
        unsigned mask = __ballot_sync(0xffffffffu, cnt >= m + 1);
        if (lane == 0) reinterpret_cast<unsigned *>(red)[warp] = mask;
        __syncthreads();
        int f = BIS_THREADS;
        for (int q = BIS_THREADS / 32 - 1; q >= 0; --q) {
            unsigned mq = reinterpret_cast<unsigned *>(red)[q];
            if (mq) f = q * 32 + __ffs(mq) - 1;
        }
        const double nhi = (f < BIS_THREADS) ? s_x[f] : hi;
        const double nlo = (f > 0) ? s_x[f - 1] : lo;
        __syncthreads();
        hi = nhi; lo = nlo;
        if (hi - lo <= 2.0 * eps * fmax(fabs(lo), fabs(hi)) + 1e-300 || hi - lo >= width) break;
    }
    if (tid == 0) lam[t] = 0.5 * (lo + hi) / sc;
}

// ---------------------------------------------------------------------------------------------
// eigenvectors of T: inverse iteration on the partially pivoted LU of T - lambda I
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ double hash_unit(unsigned i, unsigned t) {
    unsigned h = i * 2654435761u ^ (t + 1u) * 40503u;
    h ^= h >> 15; h *= 2246822519u; h ^= h >> 13; h *= 3266489917u; h ^= h >> 16;
    return ((double)(h & 0xffffffu) / 8388608.0) - 1.0;   // [-1, 1)
}

// One warp per eigenvector; the pivoted LU (stored as reciprocal pivots so that the solves are FMA chains)
// and the iterate live in shared memory.  Lane 0 walks the three sequential recurrences, all lanes share
// the O(n) parallel parts.
constexpr int IV_WARPS = 4;
__global__ void __launch_bounds__(IV_WARPS * 32)
invit_kernel(const double *__restrict__ dg, const double *__restrict__ e, const double *__restrict__ lam, int n,
             int c, double *__restrict__ Z) {
    extern __shared__ double smd[];
    const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5;
    const int t = blockIdx.x * (blockDim.x >> 5) + warp;      // 4 warps per CTA, 1 when n > 1024 (shared memory)
    if (t >= c) return;
    double *u0i = smd + (size_t)warp * (5 * (size_t)n + (size_t)(n + 7) / 8);   // 1/pivot
    double *u1 = u0i + n, *u2 = u1 + n, *ml = u2 + n, *xb = ml + n;
    unsigned char *swp = reinterpret_cast<unsigned char *>(xb + n);
    const double lambda = lam[t];
    double tn = 0.0;
    for (int i = lane; i < n; i += 32)
        tn = fmax(tn, fabs(dg[i]) + ((i < n - 1) ? fabs(e[i]) : 0.0) + ((i > 0) ? fabs(e[i - 1]) : 0.0));
    for (int o = 16; o > 0; o >>= 1) tn = fmax(tn, __shfl_xor_sync(0xffffffffu, tn, o));
    const double tiny = fmax(2.220446049250313e-16 * tn, 1e-300);
    // stage T - lambda I:  u1 <- diagonal, u2 <- off-diagonal (overwritten by the factorisation)
    for (int i = lane; i < n; i += 32) {
        u1[i] = dg[i] - lambda;
        u2[i] = (i < n - 1) ? e[i] : 0.0;
        xb[i] = hash_unit((unsigned)i, (unsigned)t);
    }
    __syncwarp();
    if (lane == 0) {
        double p = u1[0], q = u2[0];
        for (int i = 0; i < n - 1; ++i) {
            const double sub = u2[i];
            const double dn = u1[i + 1];
            const double sn = u2[i + 1];            // 0 for the last row
            if (fabs(p) >= fabs(sub)) {
                if (fabs(p) < tiny) p = (p < 0.0) ? -tiny : tiny;
                const double pinv = 1.0 / p;
                const double mult = sub * pinv;
                u0i[i] = pinv; u1[i] = q; u2[i] = 0.0; ml[i] = mult; swp[i] = 0;
                p = dn - mult * q;
                q = sn;
            } else {
                const double sinv = 1.0 / sub;
                const double mult = p * sinv;
                u0i[i] = sinv; u1[i] = dn; u2[i] = sn; ml[i] = mult; swp[i] = 1;
                p = q - mult * dn;
                q = -mult * sn;
            }
        }
        if (fabs(p) < tiny) p = (p < 0.0) ? -tiny : tiny;
        u0i[n - 1] = 1.0 / p; u1[n - 1] = 0.0; u2[n - 1] = 0.0;
    }
    __syncwarp();
    // fold the reciprocal pivots into the upper factor: x_i = c0_i - c1_i x_{i+1} - c2_i x_{i+2}, so the
    // dependent chain of the back substitution is one DFMA per row
    for (int i = lane; i < n; i += 32) { u1[i] *= u0i[i]; u2[i] *= u0i[i]; }
    __syncwarp();
    for (int iter = 0; iter < 2; ++iter) {
        if (lane == 0) {
            double bi = xb[0], bn = xb[1];
            for (int i = 0; i < n - 1; ++i) {             // forward: replay the row operations
                const double bnn = (i + 2 < n) ? xb[i + 2] : 0.0;   // prefetch off the dependent chain
                double lo_ = bi, hi_ = bn;
                if (swp[i]) { lo_ = bn; hi_ = bi; }
                xb[i] = lo_;
                bi = hi_ - ml[i] * lo_;
                bn = bnn;
            }
            xb[n - 1] = bi;
        }
        __syncwarp();
        for (int i = lane; i < n; i += 32) xb[i] *= u0i[i];   // c0
        __syncwarp();
        if (lane == 0) {
            double x1 = 0.0, x2 = 0.0;
            for (int i = n - 1; i >= 0; --i) {            // backward: U x = b
                const double t0 = xb[i] - u2[i] * x2;     // x2 is one step old: off the chain
                const double x = t0 - u1[i] * x1;
                xb[i] = x;
                x2 = x1; x1 = x;
            }
        }
        __syncwarp();
        double amax = 0.0;
        for (int i = lane; i < n; i += 32) amax = fmax(amax, fabs(xb[i]));
        for (int o = 16; o > 0; o >>= 1) amax = fmax(amax, __shfl_xor_sync(0xffffffffu, amax, o));
        double inv = 1.0 / amax, ss = 0.0;
        for (int i = lane; i < n; i += 32) { double x = xb[i] * inv; ss += x * x; }
        ss = warp_sum(ss);
        inv = inv / sqrt(ss);
        for (int i = lane; i < n; i += 32) xb[i] *= inv;
        __syncwarp();
    }
    for (int i = lane; i < n; i += 32) Z[(size_t)t * n + i] = xb[i];
}

// ---------------------------------------------------------------------------------------------
// Re-orthogonalise eigenvectors of (numerically) repeated eigenvalues.  Inverse iteration gives
// orthogonality ~ eps*||T||/gap, so only clusters with gaps below 1e-7*||T|| need it (LAPACK dstein
// uses 1e-3; with distinct eigenvalues -- every GAN activation spectrum seen here -- this kernel
// finds no cluster and returns after one pass over lam).  Classical Gram-Schmidt applied twice.
// ---------------------------------------------------------------------------------------------
constexpr int CO_THREADS = 1024;
__global__ void __launch_bounds__(CO_THREADS)
cluster_orth_kernel(const double *__restrict__ lam, const double *__restrict__ dg, const double *__restrict__ e,
                    int n, int c, double *__restrict__ Z) {
    extern __shared__ double smd[];
    double *zt = smd;            // [n]
    double *dots = zt + n;       // [c]
    double *red = dots + c;      // [64]
    int *start = reinterpret_cast<int *>(red + 64);   // [c]
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, nw = CO_THREADS / 32;
    double tn = 0.0;
    for (int i = tid; i < n; i += CO_THREADS)
        tn = fmax(tn, fabs(dg[i]) + ((i < n - 1) ? fabs(e[i]) : 0.0) + ((i > 0) ? fabs(e[i - 1]) : 0.0));
    for (int o = 16; o > 0; o >>= 1) tn = fmax(tn, __shfl_xor_sync(0xffffffffu, tn, o));
    if (lane == 0) red[warp] = tn;
    __syncthreads();
    if (tid == 0) {
        double t = 0.0;
        for (int q = 0; q < nw; ++q) t = fmax(t, red[q]);
        const double tol = 1e-7 * t;
        int any = 0;
        start[0] = 0;
        for (int k = 1; k < c; ++k) {
            start[k] = (fabs(lam[k - 1] - lam[k]) <= tol) ? start[k - 1] : k;
            any |= (start[k] != k);
        }
        red[32] = (double)any;
    }
    __syncthreads();
    if (red[32] == 0.0) return;
    for (int t = 0; t < c; ++t) {
        const int s0 = start[t];
        if (s0 == t) continue;
        for (int pass = 0; pass < 2; ++pass) {
            for (int i = tid; i < n; i += CO_THREADS) zt[i] = Z[(size_t)t * n + i];
            __syncthreads();
            for (int s = s0 + warp; s < t; s += nw) {
                double d = 0.0;
                for (int i = lane; i < n; i += 32) d += Z[(size_t)s * n + i] * zt[i];
                d = warp_sum(d);
                if (lane == 0) dots[s] = d;
            }
            __syncthreads();
            double nrm = 0.0;
            for (int i = tid; i < n; i += CO_THREADS) {
                double x = zt[i];
                for (int s = s0; s < t; ++s) x -= dots[s] * Z[(size_t)s * n + i];
                zt[i] = x;
                nrm += x * x;
            }
            nrm = block_sum(nrm, red);
            const double inv = (nrm > 0.0) ? 1.0 / sqrt(nrm) : 0.0;
            for (int i = tid; i < n; i += CO_THREADS) Z[(size_t)t * n + i] = zt[i] * inv;
            __syncthreads();
        }
    }
}

// ---------------------------------------------------------------------------------------------
// eigenvectors of A:  x = H_0 H_1 ... H_{n-3} z ; then the svd_flip sign rule (largest |.| entry > 0)
// ---------------------------------------------------------------------------------------------
// One CTA = 8 warps = 8 eigenvectors, each held in its warp's registers (NR = n/32 doubles per lane); the
// reflectors stream from L2 through a cp.async ring shared by the 8 warps (BT_DEPTH pairs in flight), two
// reflectors per barrier, so the ~510 dependent steps are paced by the per-step dot/axpy.
constexpr int BT_WARPS = 8;
constexpr int BT_DEPTH = 4;      // ring slots, each holding a PAIR of reflectors
template <int NR>
__global__ void __launch_bounds__(BT_WARPS * 32)
backtransform_kernel(const double *__restrict__ Z, const double *__restrict__ Vh,
                     const double *__restrict__ beta, int n, int c, double *__restrict__ out) {
    extern __shared__ double smd[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int t = blockIdx.x * BT_WARPS + warp;
    const bool active = t < c;
    double *ring = smd;                                    // [BT_DEPTH][2][n]
    double z[NR];
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        const int i = lane + 32 * r;
        z[r] = (active && i < n) ? Z[(size_t)t * n + i] : 0.0;
    }
    const int nchunk = n;                                  // 16-byte chunks per reflector pair (2 * n/2)
    const int npairs = (n - 2 + 1) / 2;                    // reflectors k = n-3 .. 0, processed (k, k-1)
    auto prefetch = [&](int pidx) {                        // pair pidx holds reflectors k = n-3-2*pidx and k-1
        if (pidx < npairs) {
            const int k = n - 3 - 2 * pidx;
            double *dst = ring + (size_t)(pidx % BT_DEPTH) * 2 * n;
            for (int ch = tid; ch < nchunk; ch += BT_WARPS * 32) {
                const int which = ch / (n / 2), off = ch % (n / 2);
                const int kk = k - which;
                if (kk >= 0) {
                    unsigned sa = (unsigned)__cvta_generic_to_shared(dst + (size_t)which * n + 2 * off);
                    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(Vh + (size_t)kk * n + 2 * off)
                                 : "memory");
                }
            }
        }
        asm volatile("cp.async.commit_group;" ::: "memory");
    };
    for (int j = 0; j < BT_DEPTH - 1; ++j) prefetch(j);
    for (int pidx = 0; pidx < npairs; ++pidx) {
        prefetch(pidx + BT_DEPTH - 1);
        asm volatile("cp.async.wait_group %0;" ::"n"(BT_DEPTH - 1) : "memory");
        __syncthreads();
        const double *base = ring + (size_t)(pidx % BT_DEPTH) * 2 * n;
#pragma unroll
        for (int which = 0; which < 2; ++which) {
            const int k = n - 3 - 2 * pidx - which;
            if (k < 0) break;
            const double bk = beta[k];
            if (bk == 0.0) continue;
            const double *vk = base + (size_t)which * n;
            double vr[NR], s = 0.0;
#pragma unroll
            for (int r = 0; r < NR; ++r) {
                const int i = lane + 32 * r;
                vr[r] = (i > k && i < n) ? vk[i] : 0.0;
                s += vr[r] * z[r];
            }
            s = warp_sum(s) * bk;
#pragma unroll
            for (int r = 0; r < NR; ++r) z[r] -= s * vr[r];
        }
        __syncthreads();                                   // the slot is refilled by the next prefetch
    }
    if (!active) return;
    // argmax |z| (first index on ties, as np.argmax)
    double best = -1.0;
    int bi = 0;
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        const int i = lane + 32 * r;
        const double az = fabs(z[r]);
        if (i < n && az > best) { best = az; bi = i; }
    }
    double bval = 0.0;
#pragma unroll
    for (int r = 0; r < NR; ++r) if (lane + 32 * r == bi) bval = z[r];
    for (int o = 16; o > 0; o >>= 1) {
        double ob = __shfl_xor_sync(0xffffffffu, best, o);
        int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        double ov = __shfl_xor_sync(0xffffffffu, bval, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; bval = ov; }
    }
    const double sgn = (bval < 0.0) ? -1.0 : 1.0;
#pragma unroll
    for (int r = 0; r < NR; ++r) {
        const int i = lane + 32 * r;
        if (i < n) out[(size_t)t * n + i] = sgn * z[r];
    }
}

// n > 1024: the eigenvector does not fit a warp's registers.  One CTA per eigenvector, z in shared memory, the
// reflectors stream from L2; one block reduction per reflector (used once per large-d run, in the cold first step).
__global__ void __launch_bounds__(256)
backtransform_big_kernel(const double *__restrict__ Z, const double *__restrict__ Vh, const double *__restrict__ beta,
                         int n, int c, double *__restrict__ out) {
    extern __shared__ double smd[];
    double *z = smd, *red = smd + n;                       // red[64]
    const int tid = threadIdx.x, t = blockIdx.x;
    for (int i = tid; i < n; i += 256) z[i] = Z[(size_t)t * n + i];
    __syncthreads();
    for (int k = n - 3; k >= 0; --k) {
        const double bk = beta[k];
        if (bk == 0.0) continue;
        const double *vk = Vh + (size_t)k * n;
        double vr[16];                                     // n <= 4096
        double s = 0.0;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int i = k + 1 + tid + 256 * r;
            vr[r] = (i < n) ? vk[i] : 0.0;
            s += (i < n) ? vr[r] * z[i] : 0.0;
        }
        s = block_sum(s, red) * bk;
#pragma unroll
        for (int r = 0; r < 16; ++r) {
            const int i = k + 1 + tid + 256 * r;
            if (i < n) z[i] -= s * vr[r];
        }
        __syncthreads();
    }
    if (tid == 0) {                                        // svd_flip sign rule: first largest |z| positive
        double best = -1.0, bval = 0.0;
        for (int i = 0; i < n; ++i) { const double az = fabs(z[i]); if (az > best) { best = az; bval = z[i]; } }
        red[40] = (bval < 0.0) ? -1.0 : 1.0;
    }
    __syncthreads();
    const double sgn = red[40];
    for (int i = tid; i < n; i += 256) out[(size_t)t * n + i] = sgn * z[i];
}

template <int NR>
static int launch_backtransform(const double *Z, const double *Vh, const double *beta, int d, int c, double *evecs,
                                cudaStream_t st) {
    const size_t smem = (size_t)BT_DEPTH * 2 * d * sizeof(double);
    static size_t smem_set = 0;
    if (smem > smem_set) {
        GSB_CHECK_CUDA(cudaFuncSetAttribute(backtransform_kernel<NR>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        smem_set = smem;
    }
    backtransform_kernel<NR><<<(c + BT_WARPS - 1) / BT_WARPS, BT_WARPS * 32, smem, st>>>(Z, Vh, beta, d, c, evecs);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// ---------------------------------------------------------------------------------------------
// state update after the eigensolve
// ---------------------------------------------------------------------------------------------
__global__ void finalize_kernel(double *hdr, double *mean, double *unnorm, double *S, double *V,
                                const double *__restrict__ mean_b, const double *__restrict__ gram_b,
                                const double *__restrict__ lam, const double *__restrict__ evecs, int d,
                                int c, double n_seen, double n_b) {
    const size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    const double n_tot = n_seen + n_b;
    if (idx < (size_t)c * d) V[idx] = evecs[idx];
    if (idx < (size_t)c) S[idx] = sqrt(fmax(lam[idx], 0.0));
    if (idx < (size_t)d) {
        const double mb = mean_b[idx], vb = gram_b[idx * (size_t)d + idx];
        if (n_seen > 0) {
            const double mo = mean[idx];
            // extmath._incremental_mean_and_var: updated_mean = (last_sum + new_sum) / updated_count
            mean[idx] = (mo * n_seen + mb * n_b) / n_tot;
            // last_unnorm + new_unnorm + last_over_new/updated * (last_sum/last_over_new - new_sum)^2
            const double r = n_seen / n_b;
            const double tq = (mo * n_seen) / r - mb * n_b;
            unnorm[idx] = unnorm[idx] + vb + r / n_tot * tq * tq;
        } else {
            mean[idx] = mb;
            unnorm[idx] = vb;
        }
    }
    if (idx == 0) { hdr[0] = n_tot; hdr[1] += 1.0; }
}

__global__ void export_kernel(const double *hdr, const double *mean, const double *unnorm, const double *S,
                              const double *V, int d, int c, double n_seen, double *o_comp, double *o_sv,
                              double *o_mean, double *o_var, double *o_ev, double *o_evr) {
    __shared__ double red[64];
    double part = 0.0;
    for (int i = threadIdx.x; i < d; i += blockDim.x) part += unnorm[i];
    const double tot = block_sum(part, red);
    for (size_t i = threadIdx.x; i < (size_t)c * d; i += blockDim.x)
        if (o_comp) o_comp[i] = V[i];
    for (int i = threadIdx.x; i < d; i += blockDim.x) {
        if (o_mean) o_mean[i] = mean[i];
        if (o_var) o_var[i] = unnorm[i] / n_seen;
    }
    for (int i = threadIdx.x; i < c; i += blockDim.x) {
        const double s = S[i];
        if (o_sv) o_sv[i] = s;
        if (o_ev) o_ev[i] = s * s / (n_seen - 1.0);
        if (o_evr) o_evr[i] = s * s / tot;
    }
}

// ---------------------------------------------------------------------------------------------
static int eig_top_big(const Workspace &w, int d, int c, double *evals, double *evecs, cudaStream_t st);
static size_t g_iv_smem_set = 0, g_bis_smem_set = 0;     // largest dynamic-smem opt-in made so far (shared by both paths)

__device__ int g_eig_status = 0;
int *eig_status_device_ptr() {
    static int *p = nullptr;
    if (!p && cudaGetSymbolAddress((void **)&p, g_eig_status) != cudaSuccess) p = nullptr;
    return p;
}

int eig_top(const Workspace &w, int d, int c, double *evals, double *evecs, cudaStream_t st) {
    if (d > 1024) return eig_top_big(w, d, c, evals, evecs, st);
    // Preferred: one 16-CTA cluster (hardware barrier) when the column blocks fit in shared memory.
    static int cluster_ok = -1;     // -1 unknown, 0 unavailable, 1 usable
    const size_t cl_smem = ((size_t)(d / TRI_CLUSTER) * d + 5 * (size_t)d + 64) * sizeof(double);
    bool use_cluster = (d % TRI_CLUSTER == 0) && cl_smem <= 227 * 1024;
    if (use_cluster && cluster_ok == -1) {
        cluster_ok = 1;
        if (cudaFuncSetAttribute(tridiag_kernel<true>, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess ||
            cudaFuncSetAttribute(tridiag_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, 227 * 1024) != cudaSuccess) {
            cluster_ok = 0;
            (void)cudaGetLastError();
        }
        if (cluster_ok) {
            cudaLaunchConfig_t q{};
            q.gridDim = dim3(TRI_CLUSTER); q.blockDim = dim3(TRI_THREADS_CLUSTER); q.dynamicSmemBytes = cl_smem;
            cudaLaunchAttribute at[1];
            at[0].id = cudaLaunchAttributeClusterDimension;
            at[0].val.clusterDim.x = TRI_CLUSTER; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
            q.attrs = at; q.numAttrs = 1;
            int nclusters = 0;
            if (cudaOccupancyMaxActiveClusters(&nclusters, tridiag_kernel<true>, &q) != cudaSuccess || nclusters < 1) {
                cluster_ok = 0;
                (void)cudaGetLastError();
            }
        }
    }
    if (use_cluster && cluster_ok == 1) {
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(TRI_CLUSTER); cfg.blockDim = dim3(TRI_THREADS_CLUSTER);
        cfg.dynamicSmemBytes = cl_smem; cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = TRI_CLUSTER; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        static int reg_variant = -1;
        if (reg_variant == -1) {
            reg_variant = 1;
            if (cudaFuncSetAttribute(tridiag_reg_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1) != cudaSuccess) {
                reg_variant = 0;
                (void)cudaGetLastError();
            }
        }
        if (reg_variant && d <= 512) {
            cfg.dynamicSmemBytes = 0;
            if (d <= 256) cfg.blockDim = dim3(256);          // one row per thread: 8 warps suffice, cheaper barriers
            GSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, tridiag_reg_kernel, (const double *)w.A, d, w.dg, w.e, w.beta, w.Vh,
                                              w.xch, w.qx));
        } else {
            GSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, tridiag_kernel<true>, (const double *)w.A, d, w.dg, w.e, w.beta,
                                              w.Vh, w.xch, w.counter));
        }
    } else {
        // P CTAs, 8 columns each (n % 8 == 0); all must be co-resident for the software grid barrier
        int P = d / 8;
        while (P > 128) P /= 2;
        GSB_CHECK_ARG(d % P == 0, "sym_eig: d=%d not divisible by P=%d", d, P);
        const int ncl = d / P;
        const size_t tri_smem = ((size_t)ncl * d + 5 * (size_t)d + 64) * sizeof(double);
        GSB_CHECK_ARG(tri_smem <= 200 * 1024, "sym_eig: d=%d too large for the small-d engine", d);
        static size_t tri_smem_set = 0;
        if (tri_smem > tri_smem_set) {
            GSB_CHECK_CUDA(cudaFuncSetAttribute(tridiag_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                                (int)tri_smem));
            tri_smem_set = tri_smem;
        }
        GSB_CHECK_CUDA(cudaMemsetAsync(w.counter, 0, 256, st));
        tridiag_kernel<false><<<P, TRI_THREADS_GRID, tri_smem, st>>>(w.A, d, w.dg, w.e, w.beta, w.Vh, w.xch, w.counter);
        GSB_CHECK_LAUNCH();
    }
    const size_t bis_smem = (2 * (size_t)d + 64) * sizeof(double);
    bisect_kernel<<<c, BIS_THREADS, bis_smem, st>>>(w.dg, w.e, d, c, evals);
    GSB_CHECK_LAUNCH();
    const size_t iv_smem = (size_t)IV_WARPS * (5 * (size_t)d + (size_t)(d + 7) / 8) * sizeof(double);
    if (iv_smem > g_iv_smem_set) {
        GSB_CHECK_CUDA(cudaFuncSetAttribute(invit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)iv_smem));
        g_iv_smem_set = iv_smem;
    }
    invit_kernel<<<(c + IV_WARPS - 1) / IV_WARPS, IV_WARPS * 32, iv_smem, st>>>(w.dg, w.e, evals, d, c, w.Z);
    GSB_CHECK_LAUNCH();
    const size_t co_smem = ((size_t)d + c + 64) * sizeof(double) + (size_t)c * sizeof(int);
    cluster_orth_kernel<<<1, CO_THREADS, co_smem, st>>>(evals, w.dg, w.e, d, c, w.Z);
    GSB_CHECK_LAUNCH();
    if (d <= 128) { if (int r = launch_backtransform<4>(w.Z, w.Vh, w.beta, d, c, evecs, st)) return r; }
    else if (d <= 256) { if (int r = launch_backtransform<8>(w.Z, w.Vh, w.beta, d, c, evecs, st)) return r; }
    else if (d <= 512) { if (int r = launch_backtransform<16>(w.Z, w.Vh, w.beta, d, c, evecs, st)) return r; }
    else { if (int r = launch_backtransform<32>(w.Z, w.Vh, w.beta, d, c, evecs, st)) return r; }
    return GSB_OK;
}

// 1024 < d <= 4096: L2-resident tridiagonalisation, then the same bisection / inverse iteration (one warp per CTA:
// the LU of T - lambda I takes 5 d doubles of shared memory) and the shared-memory back-transform.
static int eig_top_big(const Workspace &w, int d, int c, double *evals, double *evecs, cudaStream_t st) {
    GSB_CHECK_ARG(d % 32 == 0 && d <= 4096, "sym_eig: large variant needs d %% 32 == 0, d <= 4096 (d=%d)", d);
    int P = (d + 15) / 16;                                  // one column per warp
    const int maxp = num_sms() - 8;
    if (P > maxp) P = maxp;
    const size_t tri_smem = (5 * (size_t)d + 64) * sizeof(double);
    const size_t bis_smem = (2 * (size_t)d + 64) * sizeof(double);
    const size_t iv_smem = (5 * (size_t)d + (size_t)(d + 7) / 8) * sizeof(double);
    const size_t bt_smem = ((size_t)d + 64) * sizeof(double);
    static size_t tri_set = 0, bt_set = 0;
    if (tri_smem > tri_set) {
        GSB_CHECK_CUDA(cudaFuncSetAttribute(tridiag_l2_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)tri_smem));
        tri_set = tri_smem;
    }
    if (bis_smem > g_bis_smem_set && bis_smem > 48 * 1024) {
        GSB_CHECK_CUDA(cudaFuncSetAttribute(bisect_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bis_smem));
        g_bis_smem_set = bis_smem;
    }
    if (iv_smem > g_iv_smem_set) {
        GSB_CHECK_CUDA(cudaFuncSetAttribute(invit_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)iv_smem));
        g_iv_smem_set = iv_smem;
    }
    if (bt_smem > bt_set) {
        GSB_CHECK_CUDA(cudaFuncSetAttribute(backtransform_big_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)bt_smem));
        bt_set = bt_smem;
    }
    GSB_CHECK_CUDA(cudaMemsetAsync(w.counter, 0, 256, st));
    tridiag_l2_kernel<<<P, TRL_THREADS, tri_smem, st>>>(w.A, d, w.dg, w.e, w.beta, w.Vh, w.xch, w.counter);
    GSB_CHECK_LAUNCH();
    bisect_kernel<<<c, BIS_THREADS, bis_smem, st>>>(w.dg, w.e, d, c, evals);
    GSB_CHECK_LAUNCH();
    invit_kernel<<<c, 32, iv_smem, st>>>(w.dg, w.e, evals, d, c, w.Z);
    GSB_CHECK_LAUNCH();
    const size_t co_smem = ((size_t)d + c + 64) * sizeof(double) + (size_t)c * sizeof(int);
    cluster_orth_kernel<<<1, CO_THREADS, co_smem, st>>>(evals, w.dg, w.e, d, c, w.Z);
    GSB_CHECK_LAUNCH();
    backtransform_big_kernel<<<c, 256, bt_smem, st>>>(w.Z, w.Vh, w.beta, d, c, evecs);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// svd_flip sign rule on the rows of V[c,d] (largest |.| entry positive; first index on ties)
__global__ void sign_rows_kernel(double *__restrict__ V, int c, int d) {
    const int lane = threadIdx.x & 31, t = blockIdx.x * (blockDim.x >> 5) + (threadIdx.x >> 5);
    if (t >= c) return;
    double *row = V + (size_t)t * d;
    double best = -1.0, bval = 0.0;
    int bi = 0;
    for (int i = lane; i < d; i += 32) {
        const double az = fabs(row[i]);
        if (az > best) { best = az; bi = i; bval = row[i]; }
    }
    for (int o = 16; o > 0; o >>= 1) {
        const double ob = __shfl_xor_sync(0xffffffffu, best, o), ov = __shfl_xor_sync(0xffffffffu, bval, o);
        const int oi = __shfl_xor_sync(0xffffffffu, bi, o);
        if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; bval = ov; }
    }
    if (bval < 0.0)
        for (int i = lane; i < d; i += 32) row[i] = -row[i];
}

int sign_rows(double *V, int c, int d, cudaStream_t st) {
    sign_rows_kernel<<<(c + 7) / 8, 256, 0, st>>>(V, c, d);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

static int g_chain_force_direct = 0;     // host-side switch, read when a step is enqueued (not thread-safe across handles, as the ABI states)
bool chain_forced_direct() { return g_chain_force_direct != 0; }

static int check_dims(int d, int c) {
    GSB_CHECK_ARG(d >= 32 && d <= 1024 && d % 32 == 0, "ipca: small-d engine needs 32 <= d <= 1024, d%%32==0 (d=%d)", d);
    GSB_CHECK_ARG(c >= 1 && c <= d, "ipca: need 1 <= c <= d (c=%d d=%d)", c, d);
    return GSB_OK;
}

}  // namespace gsb

extern "C" size_t gsb_ipca_state_bytes(int d, int c) {
    return gsb::state_view(nullptr, d, c).bytes;
}

extern "C" size_t gsb_ipca_workspace_bytes(int d, int c) {
    size_t b = gsb::carve(nullptr, d, c).bytes;
    if (gsb::subspace_applicable(d, c)) b += gsb::carve_subspace(nullptr, d, c).bytes;
    return b;
}

extern "C" int gsb_ipca_reset(void *d_state, int d, int c, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state, "ipca_reset: null state");
    if (int r = gsb::check_dims(d, c)) return r;
    GSB_CHECK_CUDA(cudaMemsetAsync(d_state, 0, gsb_ipca_state_bytes(d, c), (cudaStream_t)stream));
    return GSB_OK;
}

extern "C" int gsb_ipca_chain_step(void *d_state, int d, int c, int64_t n_seen, int64_t n_batch,
                                   const double *d_mean_b, const double *d_gram_b, void *d_workspace,
                                   size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state && d_mean_b && d_gram_b && d_workspace, "ipca_chain_step: null pointer");
    if (int r = gsb::check_dims(d, c)) return r;
    GSB_CHECK_ARG(n_seen >= 0 && n_batch > 0, "ipca_chain_step: bad counts");
    // sklearn: "n_components must be <= the batch number of samples for the first partial_fit call"
    GSB_CHECK_ARG(n_seen > 0 || c <= n_batch, "ipca_chain_step: n_components=%d > first batch size %lld", c,
                  (long long)n_batch);
    gsb::Workspace w = gsb::carve(d_workspace, d, c);
    if (workspace_bytes < w.bytes) {
        gsb::set_error("ipca_chain_step: workspace too small (%zu < %zu)", workspace_bytes, w.bytes);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    gsb::StateView s = gsb::state_view(d_state, d, c);
    const bool subspace = gsb::subspace_applicable(d, c);
    if (subspace && n_seen > 0) {
        // steps 2..K: orthogonal iteration on (Q, H), one cluster launch (subspace.cu)
        const size_t off = w.bytes;
        gsb::SubspaceWs sw = gsb::carve_subspace(reinterpret_cast<char *>(d_workspace) + off, d, c);
        if (workspace_bytes < off + sw.bytes) {
            gsb::set_error("ipca_chain_step: workspace too small (%zu < %zu)", workspace_bytes, off + sw.bytes);
            return GSB_ERR_WORKSPACE;
        }
        return gsb::subspace_step(s.hdr, s.mean, s.unnorm, s.H, s.Qbuf, d_mean_b, d_gram_b, sw, d, c, (double)n_seen,
                                  (double)n_batch, st);
    }
    dim3 grid((d + 31) / 32, (d + 31) / 32), block(32, 8);
    gsb::build_g_kernel<<<grid, block, 0, st>>>(d_gram_b, d_mean_b, s.mean, s.S, s.V, d, c, (double)n_seen,
                                                (double)n_batch, w.A);
    GSB_CHECK_LAUNCH();
    if (int r = gsb::eig_top(w, d, c, w.lam, w.evecs, st)) return r;
    size_t tot = (size_t)c * d;
    gsb::finalize_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(
        s.hdr, s.mean, s.unnorm, s.S, s.V, d_mean_b, d_gram_b, w.lam, w.evecs, d, c, (double)n_seen,
        (double)n_batch);
    GSB_CHECK_LAUNCH();
    // the first step seeds the subspace form: Q = V^T, H = diag(S^2)
    if (subspace) return gsb::to_subspace_form(s.hdr, s.S, s.V, s.H, s.Qbuf, d, c, st);
    return GSB_OK;
}

// 0 = the environment's choice (default: orthogonal iteration where it applies), 1 = direct solve for every step.
//   replaces: nothing in the reference (sklearn always solves exactly, _incremental_pca.py:352-368); this is the exact route the
//   host falls back to when gsb_eig_status reports an iteration cap.
extern "C" int gsb_ipca_set_chain_mode(int mode) {
    GSB_CHECK_ARG(mode == 0 || mode == 1, "ipca_set_chain_mode: mode must be 0 or 1");
    gsb::g_chain_force_direct = mode;
    return GSB_OK;
}

extern "C" int gsb_ipca_export(const void *d_state, int d, int c, int64_t n_seen, double *d_components,
                               double *d_singular_values, double *d_mean, double *d_var,
                               double *d_explained_variance, double *d_explained_variance_ratio,
                               gsb_stream_t stream) {
    GSB_CHECK_ARG(d_state, "ipca_export: null state");
    if (int r = gsb::check_dims(d, c)) return r;
    GSB_CHECK_ARG(n_seen > 1, "ipca_export: nothing fitted yet");
    gsb::StateView s = gsb::state_view(const_cast<void *>(d_state), d, c);
    if (gsb::subspace_applicable(d, c)) {
        // the chain ran on (Q, H): one eigen-decomposition of H gives sklearn's (components_, singular_values_)
        if (int r = gsb::materialise_components(s.hdr, s.S, s.V, s.H, s.Qbuf, s.eig_ws, d, c, (cudaStream_t)stream)) return r;
    }
    gsb::export_kernel<<<1, 1024, 0, (cudaStream_t)stream>>>(s.hdr, s.mean, s.unnorm, s.S, s.V, d, c,
                                                            (double)n_seen, d_components, d_singular_values,
                                                            d_mean, d_var, d_explained_variance,
                                                            d_explained_variance_ratio);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

extern "C" int gsb_eig_status(unsigned *h_flags, gsb_stream_t stream) {
    GSB_CHECK_ARG(h_flags, "eig_status: null pointer");
    int *dp = gsb::eig_status_device_ptr();
    GSB_CHECK_ARG(dp, "eig_status: no device status word");
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CHECK_CUDA(cudaMemcpyAsync(h_flags, dp, sizeof(unsigned), cudaMemcpyDeviceToHost, st));
    GSB_CHECK_CUDA(cudaMemsetAsync(dp, 0, sizeof(int), st));
    GSB_CHECK_CUDA(cudaStreamSynchronize(st));
    return GSB_OK;
}

extern "C" int gsb_sym_eig_top(double *d_a, int d, int c, double *d_evals, double *d_evecs,
                               void *d_workspace, size_t workspace_bytes, gsb_stream_t stream) {
    GSB_CHECK_ARG(d_a && d_evals && d_evecs && d_workspace, "sym_eig_top: null pointer");
    GSB_CHECK_ARG(d >= 32 && d <= 4096 && d % 32 == 0 && c >= 1 && c <= d, "sym_eig_top: need 32 <= d <= 4096, d%%32==0, 1 <= c <= d");
    gsb::Workspace w = gsb::carve(d_workspace, d, c);
    if (workspace_bytes < w.bytes) {
        gsb::set_error("sym_eig_top: workspace too small (%zu < %zu)", workspace_bytes, w.bytes);
        return GSB_ERR_WORKSPACE;
    }
    cudaStream_t st = (cudaStream_t)stream;
    GSB_CHECK_CUDA(cudaMemcpyAsync(w.A, d_a, (size_t)d * d * sizeof(double), cudaMemcpyDeviceToDevice, st));
    return gsb::eig_top(w, d, c, d_evals, d_evecs, st);
}
