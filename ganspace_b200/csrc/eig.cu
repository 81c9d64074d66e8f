// fp64 symmetric eigensolver: top-c eigenpairs of a d x d matrix (32 <= d <= 4096), the classical direct route on one GPU.
//   1. tridiag_kernel   Householder tridiagonalisation, column-cyclic over the CTAs, ONE barrier per reflector: the fused pass
//                       applies the pending rank-2 update, accumulates A v for the next reflector and extracts the next pivot
//                       row; every CTA rebuilds v / w redundantly from the two exchanged n-vectors, so nothing else crosses SMs.
//                       The owned columns live in registers (tridiag_reg_kernel, d <= 512), in shared memory (a 16-CTA cluster,
//                       d <= 640; d/8 grid-barrier CTAs, d <= 1024) or in place in L2 (d <= 4096).
//   2. bisect_kernel    top-c eigenvalues of T by multisection on Sturm counts.
//   3. invit_kernel     eigenvectors of T by inverse iteration on the pivoted LU of T - lambda I.
//   4. backtransform_kernel  applies the reflectors and the svd_flip sign rule.
#include "eig.cuh"
#include <math.h>

namespace gsb {

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
    w.xch = (double *)take((size_t)4 * d * 8);
    w.qx = (double *)take((size_t)2 * 16 * 512 * 8);
    w.counter = (unsigned *)take(256);
    w.bytes = off;
    return w;
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

__device__ __forceinline__ void cluster_barrier() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}

// ---------------------------------------------------------------------------------------------
// Householder tridiagonalisation  A = Q T Q^T,  Q = H_0 H_1 ... H_{n-3},  H_k = I - beta_k v_k v_k^T
// ---------------------------------------------------------------------------------------------
constexpr int TRI_CLUSTER = 16;

// reflector H = I - bk v v^T that maps x = (x0, x[1..]) (sigma = sum x[1..]^2) onto alpha e_0; v = (v0, x[1..])
struct Reflector { double alpha, bk, v0; };
__device__ __forceinline__ Reflector householder(double x0, double sigma) {
    if (sigma == 0.0) return {x0, 0.0, 0.0};
    const double nrm = sqrt(x0 * x0 + sigma);
    const double alpha = (x0 > 0.0) ? -nrm : nrm;
    return {alpha, 1.0 / (nrm * (nrm + fabs(x0))), x0 - alpha};     // bk = 2 / (v^T v)
}

// Where a CTA's owned columns j = me + P l live:
//   Cluster: the grid is ONE 16-CTA thread-block cluster (non-portable size), columns in shared memory; the per-reflector
//            exchange is ordered by barrier.cluster (release/acquire), ~5x cheaper than the atomic counter.  n <= 640.
//   Grid:    P = n/8 co-resident CTAs, columns in shared memory, a software barrier on a global counter.  n <= 1024.
//   L2:      P ~ n/16 co-resident CTAs of 16 warps, columns updated IN PLACE in global memory (row j of the symmetric input ==
//            column j): n^2 fp64 (36 MB at n = 2112) does not fit the machine's shared memory but sits in the 50 MB L2.
//            One warp per column, four independent 256-byte segments in flight per lane.  n <= 4096.
enum class Cols { Cluster, Grid, L2 };
template <Cols S> constexpr int tri_threads() { return S == Cols::Grid ? 256 : 512; }

template <Cols S>
__global__ void __launch_bounds__(tri_threads<S>(), 1)
tridiag_kernel(double *__restrict__ A, int n, double *__restrict__ dg, double *__restrict__ e,
               double *__restrict__ beta, double *__restrict__ Vh, double *__restrict__ xch,
               unsigned *__restrict__ counter) {
    constexpr bool SMEM = S != Cols::L2;
    // the shared-memory variants stride by blockDim.x: with a constant stride the compiler unrolls their loops and needs
    // 8-25 more registers
    const int NT = SMEM ? (int)blockDim.x : tri_threads<S>();
    extern __shared__ double smd[];
    const int P = gridDim.x, me = blockIdx.x, tid = threadIdx.x;
    const int lane = tid & 31, warp = tid >> 5, nwarps = NT / 32;
    const int ncl = SMEM ? n / P : (n + P - 1) / P;     // SMEM: n % P == 0
    double *Aloc = smd;                                  // SMEM: [ncl][n] owned columns
    double *a = smd + (SMEM ? (size_t)ncl * n : 0);      // current pivot column (rows > k valid)
    double *v = a + n;
    double *w = v + n;
    double *pv = w + n;               // pending rank-2 update (v_{k-1}, w_{k-1})
    double *pw = pv + n;
    double *red = pw + n;             // [64]
    auto owned = [&](int l, int j) { return SMEM ? Aloc + (size_t)l * n : A + (size_t)j * n; };

    if (SMEM) {
        for (int l = 0; l < ncl; ++l) {
            const double *src = A + (size_t)(me + P * l) * n;   // row j == column j (symmetric)
            for (int i = tid; i < n; i += NT) Aloc[(size_t)l * n + i] = src[i];
        }
    }
    for (int i = tid; i < n; i += NT) {
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
        for (int i = k + 2 + tid; i < n; i += NT) part += a[i] * a[i];
        const Reflector h = householder(x0, block_sum(part, red));
        const double bk = h.bk;
        for (int i = tid; i < n; i += NT)
            v[i] = (i <= k || bk == 0.0) ? 0.0 : ((i == k + 1) ? h.v0 : a[i]);
        __syncthreads();
        if (me == 0) {
            if (tid == 0) { e[k] = h.alpha; beta[k] = bk; }
            for (int i = tid; i < n; i += NT) Vh[(size_t)k * n + i] = v[i];
        }
        // ---- 2. fused pass over the owned columns: pending update, p = A v, next pivot row ---------
        for (int l = warp; l < ncl; l += nwarps) {
            const int j = me + P * l;
            if ((!SMEM && j >= n) || j <= k) continue;
            double *col = owned(l, j);
            const double pvj = pv[j], pwj = pw[j];
            double acc = 0.0, rj = 0.0;
            int i = k + 1 + lane;
            if constexpr (!SMEM) {
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
        if constexpr (S == Cols::Cluster) {
            __syncthreads();
            cluster_barrier();
        } else {
            target += (unsigned)P;
            grid_barrier(counter, target);
        }
        // ---- 4. w, next pivot column (redundant in every CTA) -------------------------------------
        part = 0.0;
        for (int i = k + 1 + tid; i < n; i += NT) {
            double pi = __ldcg(&Pbuf[i]);
            w[i] = pi;
            a[i] = __ldcg(&Rbuf[i]);
            part += pi * v[i];
        }
        const double ptv = block_sum(part, red);
        const double K2 = 0.5 * bk * ptv;
        for (int i = k + 1 + tid; i < n; i += NT) w[i] -= K2 * v[i];
        __syncthreads();
        const double vk1 = v[k + 1], wk1 = w[k + 1];
        for (int i = k + 1 + tid; i < n; i += NT) a[i] -= vk1 * w[i] + wk1 * v[i];
        __syncthreads();
        if (me == 0 && tid == 0) dg[k + 1] = a[k + 1];
        double *t = pv; pv = v; v = t;
        t = pw; pw = w; w = t;
    }
    // last 2x2 block: e[n-2] = A[n-1,n-2] (held in a[n-1]); dg[n-1] needs the pending update
    if (me == 0 && tid == 0) { e[n - 2] = a[n - 1]; e[n - 1] = 0.0; beta[n - 2] = 0.0; beta[n - 1] = 0.0; }
    if (me == (n - 1) % P && tid == 0)
        dg[n - 1] = owned((n - 1) / P, n - 1)[n - 1] - 2.0 * pv[n - 1] * pw[n - 1];
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
__global__ void __launch_bounds__(512, 1)
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
        const Reflector h = householder(red[32], sigma);
        const double bk = h.bk;
        const double v_i = (!row_ok || i <= k || bk == 0.0) ? 0.0 : ((i == k + 1) ? h.v0 : a_i);
        if (row_ok) vsh[i] = v_i;                                // every index < n has exactly one owner
        __syncthreads();
        if (me == 0) {
            if (tid == 0) { e[k] = h.alpha; beta[k] = bk; }
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
constexpr int IV_WARPS = 4;      // per CTA for n <= 1024; 1 above (shared memory)
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
    warp_argmax_abs(best, bi, bval);
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
    warp_argmax_abs(best, bi, bval);
    if (bval < 0.0)
        for (int i = lane; i < d; i += 32) row[i] = -row[i];
}

int sign_rows(double *V, int c, int d, cudaStream_t st) {
    sign_rows_kernel<<<(c + 7) / 8, 256, 0, st>>>(V, c, d);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// ---------------------------------------------------------------------------------------------
// launch plan: each stage's variant is picked by d
// ---------------------------------------------------------------------------------------------
int eig_top(const Workspace &w, int d, int c, double *evals, double *evecs, cudaStream_t st) {
    GSB_CHECK_ARG(d >= 32 && d <= 4096 && d % 32 == 0, "sym_eig: need 32 <= d <= 4096, d %% 32 == 0 (d=%d)", d);
    // 1. tridiagonalisation
    if (d <= 640) {
        // one 16-CTA cluster (hardware barrier) while its column blocks fit 227 KiB of shared memory: columns in registers up
        // to d = 512 (8 warps suffice up to 256), else in shared memory
        cudaLaunchConfig_t cfg{};
        cfg.gridDim = dim3(TRI_CLUSTER); cfg.blockDim = dim3(d <= 256 ? 256 : 512); cfg.stream = st;
        cudaLaunchAttribute at[1];
        at[0].id = cudaLaunchAttributeClusterDimension;
        at[0].val.clusterDim.x = TRI_CLUSTER; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
        cfg.attrs = at; cfg.numAttrs = 1;
        if (d <= 512) {
            GSB_CHECK_CUDA(cudaFuncSetAttribute(tridiag_reg_kernel, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
            GSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, tridiag_reg_kernel, (const double *)w.A, d, w.dg, w.e, w.beta, w.Vh,
                                              w.xch, w.qx));
        } else {
            auto kern = tridiag_kernel<Cols::Cluster>;
            cfg.dynamicSmemBytes = ((size_t)(d / TRI_CLUSTER) * d + 5 * (size_t)d + 64) * sizeof(double);
            GSB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
            if (int r = raise_dyn_smem(kern, cfg.dynamicSmemBytes)) return r;
            GSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, w.A, d, w.dg, w.e, w.beta, w.Vh, w.xch, w.counter));
        }
    } else {
        GSB_CHECK_CUDA(cudaMemsetAsync(w.counter, 0, 256, st));
        if (d <= 1024) {
            // P = d/8 CTAs of 8 columns each; all co-resident for the software grid barrier
            const size_t smem = (8 * (size_t)d + 5 * (size_t)d + 64) * sizeof(double);
            if (int r = raise_dyn_smem(tridiag_kernel<Cols::Grid>, smem)) return r;
            tridiag_kernel<Cols::Grid><<<d / 8, tri_threads<Cols::Grid>(), smem, st>>>(w.A, d, w.dg, w.e, w.beta, w.Vh, w.xch,
                                                                                      w.counter);
        } else {
            // columns in L2, one per warp
            int P = (d + 15) / 16;
            if (P > num_sms() - 8) P = num_sms() - 8;
            const size_t smem = (5 * (size_t)d + 64) * sizeof(double);
            if (int r = raise_dyn_smem(tridiag_kernel<Cols::L2>, smem)) return r;
            tridiag_kernel<Cols::L2><<<P, tri_threads<Cols::L2>(), smem, st>>>(w.A, d, w.dg, w.e, w.beta, w.Vh, w.xch, w.counter);
        }
        GSB_CHECK_LAUNCH();
    }
    // 2. eigenvalues
    const size_t bis_smem = (2 * (size_t)d + 64) * sizeof(double);
    if (int r = raise_dyn_smem(bisect_kernel, bis_smem)) return r;
    bisect_kernel<<<c, BIS_THREADS, bis_smem, st>>>(w.dg, w.e, d, c, evals);
    GSB_CHECK_LAUNCH();
    // 3. eigenvectors of T; above d = 1024 one warp's LU takes most of a CTA's shared memory
    const int iv_warps = d <= 1024 ? IV_WARPS : 1;
    const size_t iv_smem = (size_t)iv_warps * (5 * (size_t)d + (size_t)(d + 7) / 8) * sizeof(double);
    if (int r = raise_dyn_smem(invit_kernel, iv_smem)) return r;
    invit_kernel<<<(c + iv_warps - 1) / iv_warps, iv_warps * 32, iv_smem, st>>>(w.dg, w.e, evals, d, c, w.Z);
    GSB_CHECK_LAUNCH();
    const size_t co_smem = ((size_t)d + c + 64) * sizeof(double) + (size_t)c * sizeof(int);
    cluster_orth_kernel<<<1, CO_THREADS, co_smem, st>>>(evals, w.dg, w.e, d, c, w.Z);
    GSB_CHECK_LAUNCH();
    // 4. eigenvectors of A
    if (d > 1024) {
        const size_t smem = ((size_t)d + 64) * sizeof(double);
        if (int r = raise_dyn_smem(backtransform_big_kernel, smem)) return r;
        backtransform_big_kernel<<<c, 256, smem, st>>>(w.Z, w.Vh, w.beta, d, c, evecs);
    } else {
        auto kern = d <= 128 ? backtransform_kernel<4> : d <= 256 ? backtransform_kernel<8>
                  : d <= 512 ? backtransform_kernel<16> : backtransform_kernel<32>;
        const size_t smem = (size_t)BT_DEPTH * 2 * d * sizeof(double);
        if (int r = raise_dyn_smem(kern, smem)) return r;
        kern<<<(c + BT_WARPS - 1) / BT_WARPS, BT_WARPS * 32, smem, st>>>(w.Z, w.Vh, w.beta, d, c, evecs);
    }
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

}  // namespace gsb

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
