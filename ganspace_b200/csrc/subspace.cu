// Incremental-PCA chain step WITHOUT a per-step eigen-decomposition (round 2; DESIGN.md section 5b).
//
// sklearn's partial_fit (estimators.py:68-76 -> _incremental_pca.py:254-380) keeps (components_, singular_values_) and
// re-enters them in the next batch only through   V^T S^2 V  =  P G P   (P = projector on the top-c eigenspace of G).
// With ANY orthonormal basis Q[d,c] of that eigenspace and H = Q^T G Q  this is  Q H Q^T  exactly, so the chain state
// can be (Q, H) and a step only has to find the top-c INVARIANT SUBSPACE of
//        G = Q H Q^T + C_b + m m^T ,        m = sqrt(n_seen n_b / n_tot) (mean - mean_b)
// which is well separated from the rest of the spectrum from the second batch on (the kept part has seen k batches, the
// discarded tail only one: lambda_{c+1}/lambda_c ~ 1/k), although the eigen-gaps INSIDE it are tiny (0.3 %).  Orthogonal
// (subspace) iteration  Q <- orth(G Q)  converges like (lambda_{c+1}/lambda_c)^it -- 2-3 iterations per step for most of a
// run (tools/study_subspace_chain.py: 242 iterations over the 100 steps of config 2 at tol 1e-5, exported components
// equal to the exact chain to cos 0.999999999) -- and every operation is a GEMM or a c x c Cholesky.  The single
// eigen-decomposition of the final H happens at export (materialise_*).  The first step (one batch: no gap) uses the
// direct solver of ipca.cu.
//
// One launch = one chain step = one 16-CTA thread-block cluster; CTA q owns rows [q d/16, (q+1) d/16) of every d-row
// operand.  All products run on the fp64 tensor-core path (mma.sync m8n8k4: measured 64 FMA/clk/SM, the same peak as
// DFMA, but with 6 shared-memory operand loads per 5 MMAs instead of 2 per FMA).  Per iteration:
//     Y_q = G_q Q                (operands streamed from L2 through a 3-stage cp.async ring)
//     H~ = sum_q Q_q^T Y_q ,  W = sum_q Y_q^T Y_q        (two-stage reduction through L2, two cluster barriers)
//     residual ||Y - Q H~||_F / min diag H~ <= tol  ->  H = sym(H~), done
//     W = L L^T, Q_q <- Y_q L^-T  (Cholesky in shared memory, the triangular solve rides along as extra rows)
#include "ipca_internal.cuh"
#include <math.h>
#include <stdlib.h>
#include <string.h>

namespace gsb {

constexpr int SC_CL = 16;          // CTAs per cluster
constexpr int SC_WARPS = 8;
constexpr int SC_THREADS = SC_WARPS * 32;
constexpr int SC_KT = 32;          // rows of Q per pipeline stage (K extent of a stage)
constexpr int SC_LDA = SC_KT + 4;  // padded row length of a G tile (bank-conflict-free fragment loads)
constexpr int SC_STAGES = 3;
constexpr int SC_NB = 5;           // column tiles (8 wide) sharing one A fragment
constexpr int SC_MAXG = 2;         // tile groups per warp in the pipelined product

struct SubspaceParams {
    double *hdr, *mean, *unnorm, *H, *Qbuf;      // chain state (device)
    const double *mean_b, *gram_b;               // statistics of this batch
    double *Gt, *Part, *Red, *Slots;             // workspace: G tiles, per-CTA partial (H~, W), reduced (H~, W), scalars
    double *Prof;                                // [16] clocks per phase, accumulated by CTA 0 (profiling aid)
    int d, c;
    double n_seen, n_b, tol;
    double dbl;                                  // residual > dbl * tol: two multiplications by G per orthonormalisation
    int maxit;
    int *status;
};

__device__ __forceinline__ void dmma884(double &c0, double &c1, double a, double b) {
    asm("mma.sync.aligned.m8n8k4.row.col.f64.f64.f64.f64 {%0,%1}, {%2}, {%3}, {%0,%1};" : "+d"(c0), "+d"(c1) : "d"(a), "d"(b));
}
__device__ __forceinline__ void sc_cluster_sync() {
    asm volatile("barrier.cluster.arrive.release.aligned;" ::: "memory");
    asm volatile("barrier.cluster.wait.acquire.aligned;" ::: "memory");
}
__device__ __forceinline__ void cp_async16(double *dst, const double *src) {
    const unsigned sa = (unsigned)__cvta_generic_to_shared(dst);
    asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(sa), "l"(src) : "memory");
}
__device__ __forceinline__ void cta_copy_async(double *dst, const double *src, int ndoubles) {
    for (int ch = threadIdx.x; ch < ndoubles / 2; ch += SC_THREADS) cp_async16(dst + 2 * ch, src + 2 * ch);
}

// One A fragment against up to SC_NB B fragments, `ksteps` k-steps of 4.
//   A[m][k]:  AT = false -> As[m * lda + k]     AT = true -> As[k * lda + m]
//   B[k][n]:  BT = false -> Bs[k * ldb + n]     BT = true -> Bs[n * ldb + k]
template <bool AT, bool BT>
__device__ __forceinline__ void mma_group(const double *__restrict__ As, int lda, const double *__restrict__ Bs, int ldb,
                                          int ksteps, int m0, int n0, int nb, double (&acc)[SC_NB][2]) {
    const int lane = threadIdx.x & 31, g = lane >> 2, t = lane & 3;
    const double *ap = AT ? (As + (size_t)t * lda + m0 + g) : (As + (size_t)(m0 + g) * lda + t);
    const double *bp = BT ? (Bs + (size_t)(n0 + g) * ldb + t) : (Bs + (size_t)t * ldb + n0 + g);
    const int astep = AT ? 4 * lda : 4, bstep = BT ? 4 : 4 * ldb, bnext = BT ? 8 * ldb : 8;
#pragma unroll 2
    for (int ks = 0; ks < ksteps; ++ks) {
        const double a = ap[(size_t)ks * astep];
#pragma unroll
        for (int b = 0; b < SC_NB; ++b) {
            if (b < nb) {
                const double bv = bp[(size_t)ks * bstep + (size_t)b * bnext];
                dmma884(acc[b][0], acc[b][1], a, bv);
            }
        }
    }
}

// 1/sqrt(x) for a positive normal x: hardware approximation (2^-22) + two Newton steps; ~80 clocks on the dependent chain of the
// Cholesky instead of ~200 for the library routine with its special-case handling
__device__ __forceinline__ double fast_rsqrt(double x) {
    double y;
    asm("rsqrt.approx.ftz.f64 %0, %1;" : "=d"(y) : "d"(x));
    const double h = 0.5 * x;
    double t = fma(-h * y, y, 0.5);
    y = fma(y, t, y);
    t = fma(-h * y, y, 0.5);
    y = fma(y, t, y);
    return y;
}

__device__ __forceinline__ void zero_acc(double (&acc)[SC_NB][2]) {
#pragma unroll
    for (int b = 0; b < SC_NB; ++b) { acc[b][0] = 0.0; acc[b][1] = 0.0; }
}

// tile groups of an (mt x nt) grid of 8x8 tiles: group g -> row tile g % mt, column tiles [nbsel * (g / mt), +nbsel)
struct Grouping { int mt, nt, nbsel, ngroups; };
__device__ __forceinline__ Grouping make_grouping(int mt, int nt) {
    Grouping q;
    q.mt = mt; q.nt = nt;
    int nb = (mt * nt + SC_WARPS - 1) / SC_WARPS;
    nb = nb < 1 ? 1 : (nb > SC_NB ? SC_NB : nb);
    q.nbsel = nb;
    q.ngroups = mt * ((nt + nb - 1) / nb);
    return q;
}


// Cholesky of W[c,c] with the RPC rows of Y riding along (Y <- Y L^-T), all in REGISTERS: the (c + RPC) x c array is
// spread over a 16 x 16 thread grid, thread (ry, cx) holds rows ry + 16 a (a < RA) and columns cx + 16 b (b < CB).  Only the Y
// rows are written back (L is not needed).  Panels of 8 columns: a per-column barrier + rsqrt + broadcast costs 0.59 us per
// column (47 us for c = 80) although the arithmetic is 0.07 us.  Per panel: (1) the owners publish the panel's 8 columns; (2) warp 0
// factors the 8 x 8 diagonal block with shuffles (lane l owns row l), then one thread per remaining row solves X = P L^-T (the Y
// rows of the panel are final here and go straight to Ys); (3) every thread applies the rank-8 update to its registers.
// Two barriers per panel instead of eight.
template <int RA, int CB>
__device__ __forceinline__ void chol_solve_blocked(const double *__restrict__ Ws, double *__restrict__ Ys, int c, int cp, int RPC,
                                                   double *__restrict__ buf /* [2 * 16 * RA * 9 + 80] */) {
    const int tid = threadIdx.x, ry = tid >> 4, cx = tid & 15, lane = tid & 31;
    const int nrows = c + RPC, CL = 16 * RA;
    double *P = buf, *XS = buf + (size_t)CL * 9, *Lb = XS + (size_t)CL * 9;        // Lb: [8][9] factor, [72..79] inverse diagonal
    double A[RA][CB];
#pragma unroll
    for (int a = 0; a < RA; ++a) {
        const int r = ry + 16 * a;
#pragma unroll
        for (int b = 0; b < CB; ++b) {
            const int q = cx + 16 * b;
            double v = 0.0;
            if (r < nrows && q < c) v = (r < c) ? Ws[(size_t)r * cp + q] : Ys[(size_t)(r - c) * cp + q];
            A[a][b] = v;
        }
    }
    // pivots below 1e-26 x the first (= largest-scale) diagonal entry are clamped: numerically dependent columns
    const double floor_ = fmax(fabs(Ws[0]) * 1e-26, 1e-300);
    __syncthreads();
    for (int p = 0; p < c / 8; ++p) {
        const int j0 = 8 * p, pb = p >> 1, pc = (p & 1) * 8;
        // (1) panel columns -> P[row][k]
        if (cx >= pc && cx < pc + 8) {
#pragma unroll
            for (int b = 0; b < CB; ++b)
                if (b == pb) {
#pragma unroll
                    for (int a = 0; a < RA; ++a) P[(size_t)(ry + 16 * a) * 9 + (cx - pc)] = A[a][b];
                }
        }
        __syncthreads();
        // (2a) 8 x 8 Cholesky of the diagonal block in warp 0: lane l (< 8) owns row l
        if (tid < 32) {
            const int l = lane & 7;
            double row[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) row[k] = P[(size_t)(j0 + l) * 9 + k];
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                double piv = __shfl_sync(0xffffffffu, row[j], j);
                if (!(piv > floor_)) piv = floor_;
                const double inv = fast_rsqrt(piv);
                const double lij = row[j] * inv;                       // L[l][j] for l >= j
#pragma unroll
                for (int k = j + 1; k < 8; ++k) {
                    const double lkj = __shfl_sync(0xffffffffu, lij, k);
                    row[k] = fma(-lij, lkj, row[k]);
                }
                row[j] = lij;
                if (lane == j) Lb[72 + j] = inv;                       // 1 / L[j][j]
            }
            if (lane < 8) {
#pragma unroll
                for (int k = 0; k < 8; ++k) Lb[l * 9 + k] = (k <= l) ? row[k] : 0.0;
            }
        }
        __syncthreads();
        // (2b) X[r][:] = P[r][:] L^-T for the rows below the panel; one thread per row
        for (int r = j0 + 8 + tid; r < nrows; r += SC_THREADS) {
            double x[8];
#pragma unroll
            for (int k = 0; k < 8; ++k) {
                double sacc = P[(size_t)r * 9 + k];
#pragma unroll
                for (int m = 0; m < k; ++m) sacc = fma(-x[m], Lb[k * 9 + m], sacc);
                x[k] = sacc * Lb[72 + k];
            }
#pragma unroll
            for (int k = 0; k < 8; ++k) XS[(size_t)r * 9 + k] = x[k];
            if (r >= c) {
#pragma unroll
                for (int k = 0; k < 8; ++k) Ys[(size_t)(r - c) * cp + j0 + k] = x[k];
            }
        }
        __syncthreads();
        // (3) rank-8 update of the trailing columns (q >= j0 + 8) for the rows below the panel
        double xr[RA][8];
#pragma unroll
        for (int a = 0; a < RA; ++a) {
            const int r = ry + 16 * a;
            const bool ok = (r >= j0 + 8) && (r < nrows);
#pragma unroll
            for (int k = 0; k < 8; ++k) xr[a][k] = ok ? XS[(size_t)r * 9 + k] : 0.0;
        }
#pragma unroll
        for (int b = 0; b < CB; ++b) {
            const int q = cx + 16 * b;
            if (q >= j0 + 8 && q < c) {
                double xq[8];
#pragma unroll
                for (int k = 0; k < 8; ++k) xq[k] = XS[(size_t)q * 9 + k];
#pragma unroll
                for (int a = 0; a < RA; ++a) {
                    double v = A[a][b];
#pragma unroll
                    for (int k = 0; k < 8; ++k) v = fma(-xr[a][k], xq[k], v);
                    A[a][b] = v;
                }
            }
        }
    }
    __syncthreads();
}

// One chain step by the whole cluster.  All data written by one CTA and read by another travels through L2 (.cg loads /
// cp.async.cg) or after a cluster barrier.
template <int RA, int CB>
__global__ void __launch_bounds__(SC_THREADS, 1)
subspace_step_kernel(const SubspaceParams p) {
    extern __shared__ __align__(16) double sc_smem[];
    const int d = p.d, c = p.c, cp = c + 4, RPC = d / SC_CL, RT = RPC / 8, CT = c / 8, nkt = d / SC_KT;
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5, fg = lane >> 2, ft = lane & 3;
    uint32_t me_u;
    asm volatile("mov.u32 %0, %%cluster_ctarank;" : "=r"(me_u));
    const int me = (int)me_u;

    double *As = sc_smem;                                   // [STAGES][RPC][SC_LDA]
    double *Bs = As + (size_t)SC_STAGES * RPC * SC_LDA;     // [STAGES][SC_KT][cp]
    double *Ys = Bs + (size_t)SC_STAGES * SC_KT * cp;       // [RPC][cp]   Y_q / T_q / new Q_q
    double *Qq = Ys + (size_t)RPC * cp;                     // [RPC][cp]   own rows of the current Q
    double *Ws = Qq + (size_t)RPC * cp;                     // [c][cp]     H, then W -> L
    double *mv = Ws + (size_t)c * cp;                       // [d]         mean-correction vector m
    double *red = mv + d;                                   // [64]
    double *cholbuf = red + 64;                             // [2 * 16 * RA * 9 + 80]  Cholesky panels
    long long tprev = clock64();
    double prof[10] = {0, 0, 0, 0, 0, 0, 0, 0, 0, 0};
#define PROF(k) do { const long long tn_ = clock64(); prof[k] += (double)(tn_ - tprev); tprev = tn_; } while (0)

    const double n_seen = p.n_seen, n_b = p.n_b, n_tot = n_seen + n_b;
    int cur = (int)__ldcg(p.hdr + 3);
    double *Qc = p.Qbuf + (size_t)cur * d * cp, *Qn = p.Qbuf + (size_t)(cur ^ 1) * d * cp;
    const size_t tileA = (size_t)RPC * SC_LDA, tileB = (size_t)SC_KT * cp;
    double *Gmine = p.Gt + (size_t)me * nkt * tileA;

    // ------------------------------------------------------------------ phase 0: m, own rows of Q, H
    {
        const double f = sqrt((n_seen / n_tot) * n_b);
        for (int i = tid; i < d; i += SC_THREADS) mv[i] = f * (__ldcg(p.mean + i) - __ldcg(p.mean_b + i));
        const double *src = Qc + (size_t)me * RPC * cp;
        for (int i = tid; i < RPC * cp; i += SC_THREADS) Qq[i] = __ldcg(src + i);
        for (int i = tid; i < c * c; i += SC_THREADS) Ws[(i / c) * cp + i % c] = __ldcg(p.H + i);
    }
    __syncthreads();
    // ------------------------------------------------------------------ phase 1a: T_q = Q_q H  -> Ys
    {
        const Grouping gr = make_grouping(RT, CT);
        for (int g = warp; g < gr.ngroups; g += SC_WARPS) {
            const int rt = g % gr.mt, ct0 = (g / gr.mt) * gr.nbsel;
            const int nb = (gr.nt - ct0 < gr.nbsel) ? gr.nt - ct0 : gr.nbsel;
            double acc[SC_NB][2];
            zero_acc(acc);
            mma_group<false, false>(Qq, cp, Ws, cp, c / 4, rt * 8, ct0 * 8, nb, acc);
#pragma unroll
            for (int b = 0; b < SC_NB; ++b)
                if (b < nb) {
                    double *o = Ys + (size_t)(rt * 8 + fg) * cp + (ct0 + b) * 8 + 2 * ft;
                    o[0] = acc[b][0]; o[1] = acc[b][1];
                }
        }
    }
    __syncthreads();
    PROF(0);
    // ------------------------------------------------------------------ phase 1b: G_q = T_q Q^T + C_q + m_q m^T  -> tiles in L2
    {
        const Grouping gr = make_grouping(RT, SC_KT / 8);
        // the C_b block of this CTA's rows and the stage's 32 columns rides along in the (otherwise unused) A stage
        auto copy_c = [&](int stage, int kt_) {
            double *dstc = As + (size_t)stage * tileA;
            for (int ch = tid; ch < RPC * (SC_KT / 2); ch += SC_THREADS) {
                const int r = ch / (SC_KT / 2), o2 = ch % (SC_KT / 2);
                cp_async16(dstc + (size_t)r * SC_LDA + 2 * o2, p.gram_b + (size_t)(me * RPC + r) * d + kt_ * SC_KT + 2 * o2);
            }
        };
        for (int s = 0; s < SC_STAGES - 1; ++s) {
            if (s < nkt) { cta_copy_async(Bs + (size_t)s * tileB, Qc + (size_t)s * tileB, (int)tileB); copy_c(s, s); }
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        for (int kt = 0; kt < nkt; ++kt) {
            asm volatile("cp.async.wait_group %0;" ::"n"(SC_STAGES - 2) : "memory");
            __syncthreads();
            {
                const int nx = kt + SC_STAGES - 1;
                if (nx < nkt) {
                    cta_copy_async(Bs + (size_t)(nx % SC_STAGES) * tileB, Qc + (size_t)nx * tileB, (int)tileB);
                    copy_c(nx % SC_STAGES, nx);
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
            }
            const double *Bt = Bs + (size_t)(kt % SC_STAGES) * tileB, *Cst = As + (size_t)(kt % SC_STAGES) * tileA;
            for (int g = warp; g < gr.ngroups; g += SC_WARPS) {
                const int rt = g % gr.mt, ct0 = (g / gr.mt) * gr.nbsel;
                const int nb = (gr.nt - ct0 < gr.nbsel) ? gr.nt - ct0 : gr.nbsel;
                double acc[SC_NB][2];
                zero_acc(acc);
                mma_group<false, true>(Ys, cp, Bt, cp, c / 4, rt * 8, ct0 * 8, nb, acc);
                const int lrow = rt * 8 + fg, grow = me * RPC + lrow;
                const double mr = mv[grow];
#pragma unroll
                for (int b = 0; b < SC_NB; ++b)
                    if (b < nb) {
                        const int lcol = (ct0 + b) * 8 + 2 * ft, gcol = kt * SC_KT + lcol;
                        const double2 cb = *reinterpret_cast<const double2 *>(Cst + (size_t)lrow * SC_LDA + lcol);
                        double2 o;
                        o.x = acc[b][0] + cb.x + mr * mv[gcol];
                        o.y = acc[b][1] + cb.y + mr * mv[gcol + 1];
                        *reinterpret_cast<double2 *>(Gmine + (size_t)kt * tileA + (size_t)lrow * SC_LDA + lcol) = o;
                    }
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
    }
    __syncthreads();
    PROF(1);

    // ------------------------------------------------------------------ phase 2: orthogonal iteration
    const Grouping gy = make_grouping(RT, CT);              // RPC x c outputs
    const Grouping gh = make_grouping(CT, CT);              // c x c outputs
    const int E = 2 * c * c, slice = (E + SC_CL - 1) / SC_CL;
    double rel = 0.0;
    int it = 0;
    bool conv = false;
    // Y_q (or Z_q) = G_q B  -> Ys   (K = d streamed in stages of SC_KT; B = the current Q, or the published Y of a double step)
    auto gemm_into_ys = [&](const double *Bsrc) {
        {
        double acc[SC_MAXG][SC_NB][2];
#pragma unroll
        for (int q = 0; q < SC_MAXG; ++q) zero_acc(acc[q]);
        for (int s = 0; s < SC_STAGES - 1; ++s) {
            if (s < nkt) {
                cta_copy_async(As + (size_t)s * tileA, Gmine + (size_t)s * tileA, (int)tileA);
                cta_copy_async(Bs + (size_t)s * tileB, Bsrc + (size_t)s * tileB, (int)tileB);
            }
            asm volatile("cp.async.commit_group;" ::: "memory");
        }
        for (int kt = 0; kt < nkt; ++kt) {
            asm volatile("cp.async.wait_group %0;" ::"n"(SC_STAGES - 2) : "memory");
            __syncthreads();
            {
                const int nx = kt + SC_STAGES - 1;
                if (nx < nkt) {
                    cta_copy_async(As + (size_t)(nx % SC_STAGES) * tileA, Gmine + (size_t)nx * tileA, (int)tileA);
                    cta_copy_async(Bs + (size_t)(nx % SC_STAGES) * tileB, Bsrc + (size_t)nx * tileB, (int)tileB);
                }
                asm volatile("cp.async.commit_group;" ::: "memory");
            }
            const double *At = As + (size_t)(kt % SC_STAGES) * tileA, *Bt = Bs + (size_t)(kt % SC_STAGES) * tileB;
#pragma unroll
            for (int q = 0; q < SC_MAXG; ++q) {
                const int g = warp + q * SC_WARPS;
                if (g < gy.ngroups) {
                    const int rt = g % gy.mt, ct0 = (g / gy.mt) * gy.nbsel;
                    const int nb = (gy.nt - ct0 < gy.nbsel) ? gy.nt - ct0 : gy.nbsel;
                    mma_group<false, false>(At, SC_LDA, Bt, cp, SC_KT / 4, rt * 8, ct0 * 8, nb, acc[q]);
                }
            }
        }
        asm volatile("cp.async.wait_group 0;" ::: "memory");
#pragma unroll
        for (int q = 0; q < SC_MAXG; ++q) {
            const int g = warp + q * SC_WARPS;
            if (g < gy.ngroups) {
                const int rt = g % gy.mt, ct0 = (g / gy.mt) * gy.nbsel;
                const int nb = (gy.nt - ct0 < gy.nbsel) ? gy.nt - ct0 : gy.nbsel;
#pragma unroll
                for (int b = 0; b < SC_NB; ++b)
                    if (b < nb) {
                        double *o = Ys + (size_t)(rt * 8 + fg) * cp + (ct0 + b) * 8 + 2 * ft;
                        o[0] = acc[q][b][0]; o[1] = acc[q][b][1];
                    }
            }
        }
    }
    };
    // partial H~ = Q_q^T Ys and W = Ys^T Ys -> L2, reduced over the cluster into p.Red (two cluster barriers)
    auto partial_reduce = [&]() {
    // ---- partial H~ = Q_q^T Y_q and W = Y_q^T Y_q  -> L2
    {
        double *Ph = p.Part + (size_t)me * E, *Pw = Ph + (size_t)c * c;
        for (int g = warp; g < gh.ngroups; g += SC_WARPS) {
            const int mt = g % gh.mt, ct0 = (g / gh.mt) * gh.nbsel;
            const int nb = (gh.nt - ct0 < gh.nbsel) ? gh.nt - ct0 : gh.nbsel;
            double ah[SC_NB][2], aw[SC_NB][2];
            zero_acc(ah); zero_acc(aw);
            mma_group<true, false>(Qq, cp, Ys, cp, RPC / 4, mt * 8, ct0 * 8, nb, ah);
            mma_group<true, false>(Ys, cp, Ys, cp, RPC / 4, mt * 8, ct0 * 8, nb, aw);
#pragma unroll
            for (int b = 0; b < SC_NB; ++b)
                if (b < nb) {
                    const size_t o = (size_t)(mt * 8 + fg) * c + (ct0 + b) * 8 + 2 * ft;
                    *reinterpret_cast<double2 *>(Ph + o) = make_double2(ah[b][0], ah[b][1]);
                    *reinterpret_cast<double2 *>(Pw + o) = make_double2(aw[b][0], aw[b][1]);
                }
        }
    }
    __syncthreads();
    sc_cluster_sync();                                   // (1) all partials are in L2
    for (int q0 = 0; q0 < slice; q0 += 4 * SC_THREADS) {                  // 64 loads in flight per thread
        double v[4][SC_CL];
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int el = me * slice + q0 + u * SC_THREADS + tid;
            const bool ok = (q0 + u * SC_THREADS + tid < slice) && el < E;
#pragma unroll
            for (int r = 0; r < SC_CL; ++r) v[u][r] = ok ? __ldcg(p.Part + (size_t)r * E + el) : 0.0;
        }
#pragma unroll
        for (int u = 0; u < 4; ++u) {
            const int el = me * slice + q0 + u * SC_THREADS + tid;
            if ((q0 + u * SC_THREADS + tid < slice) && el < E) {
                double s = 0.0;
#pragma unroll
                for (int r = 0; r < SC_CL; ++r) s += v[u][r];                       // fixed order: deterministic
                p.Red[el] = s;
            }
        }
    }
    __syncthreads();
    sc_cluster_sync();                                   // (2) reduced H~ and W are in L2
    };
    for (;;) {
        gemm_into_ys(Qc);
        __syncthreads();
        PROF(2);
        partial_reduce();
        for (int i = tid; i < c * c; i += SC_THREADS) Ws[(i / c) * cp + i % c] = __ldcg(p.Red + i);
        __syncthreads();
        PROF(4);
        // ---- residual  R_q = Y_q - Q_q H~
        double rs = 0.0;
        for (int g = warp; g < gy.ngroups; g += SC_WARPS) {
            const int rt = g % gy.mt, ct0 = (g / gy.mt) * gy.nbsel;
            const int nb = (gy.nt - ct0 < gy.nbsel) ? gy.nt - ct0 : gy.nbsel;
            double acc[SC_NB][2];
            zero_acc(acc);
            mma_group<false, false>(Qq, cp, Ws, cp, c / 4, rt * 8, ct0 * 8, nb, acc);
#pragma unroll
            for (int b = 0; b < SC_NB; ++b)
                if (b < nb) {
                    const double *y = Ys + (size_t)(rt * 8 + fg) * cp + (ct0 + b) * 8 + 2 * ft;
                    const double r0 = y[0] - acc[b][0], r1 = y[1] - acc[b][1];
                    rs = fma(r0, r0, rs);
                    rs = fma(r1, r1, rs);
                }
        }
        rs = block_sum(rs, red);
        if (tid == 0) p.Slots[me] = rs;
        __syncthreads();
        sc_cluster_sync();                                   // (3) every CTA's residual share is in L2
        {
            double sl[SC_CL];
#pragma unroll
            for (int r = 0; r < SC_CL; ++r) sl[r] = __ldcg(p.Slots + r);
            double hmin = 1e300;
            for (int i = lane; i < c; i += 32) hmin = fmin(hmin, Ws[(size_t)i * cp + i]);
            for (int o = 16; o > 0; o >>= 1) hmin = fmin(hmin, __shfl_xor_sync(0xffffffffu, hmin, o));
            double tot = 0.0;
#pragma unroll
            for (int r = 0; r < SC_CL; ++r) tot += sl[r];
            rel = (hmin > 0.0) ? sqrt(tot) / hmin : 1e300;
            conv = rel <= p.tol;
        }
        PROF(5);
        if (conv || it >= p.maxit) break;
        ++it;
        if (rel > p.dbl * p.tol && it < p.maxit) {
            // Far from converged: multiply by G once more before orthonormalising, Z = G Y (two iterations of convergence for
            // one Cholesky; cond(Z) <= (lambda_1 / lambda_c)^2, harmless in fp64).  Y becomes the B operand: publish it.
            double *dst = Qn + (size_t)me * RPC * cp;
            for (int i = tid; i < RPC * cp; i += SC_THREADS) dst[i] = ((i % cp) < c) ? Ys[i] : 0.0;
            __syncthreads();
            sc_cluster_sync();                               // Y is complete in L2
            gemm_into_ys(Qn);
            __syncthreads();
            partial_reduce();                                // only W = Z^T Z is used
            ++it;
            PROF(2);
        }
        // ---- W = L L^T in shared memory; the rows of Y_q (Z_q) ride along:  Q_q <- Y_q L^-T
        for (int i = tid; i < c * c; i += SC_THREADS) Ws[(i / c) * cp + i % c] = __ldcg(p.Red + (size_t)c * c + i);
        __syncthreads();
        chol_solve_blocked<RA, CB>(Ws, Ys, c, cp, RPC, cholbuf);
        PROF(6);
        // ---- publish the new rows of Q
        {
            double *dst = Qn + (size_t)me * RPC * cp;
            for (int i = tid; i < RPC * cp; i += SC_THREADS) {
                const double v = ((i % cp) < c) ? Ys[i] : 0.0;
                Qq[i] = v;
                dst[i] = v;
            }
        }
        __syncthreads();
        sc_cluster_sync();                                   // (4) the new Q is complete in L2
        { double *t_ = Qc; Qc = Qn; Qn = t_; }
        cur ^= 1;
        PROF(7);
    }
    // ------------------------------------------------------------------ commit: H = sym(H~), running mean / variance, header
    if (me == 0) {
        for (int i = tid; i < c * c; i += SC_THREADS) {
            const int a = i / c, b = i % c;
            p.H[i] = 0.5 * (Ws[(size_t)a * cp + b] + Ws[(size_t)b * cp + a]);
        }
    }
    for (int l = tid; l < RPC; l += SC_THREADS) {
        const int i = me * RPC + l;
        const double mb = __ldcg(p.mean_b + i), vb = __ldcg(p.gram_b + (size_t)i * d + i), mo = __ldcg(p.mean + i);
        // extmath._incremental_mean_and_var (same arithmetic as finalize_kernel in ipca.cu)
        const double r = n_seen / n_b;
        const double tq = (mo * n_seen) / r - mb * n_b;
        p.unnorm[i] = __ldcg(p.unnorm + i) + vb + r / n_tot * tq * tq;
        p.mean[i] = (mo * n_seen + mb * n_b) / n_tot;
    }
    __syncthreads();
    if (me == 0 && tid == 0) {
        p.hdr[0] = n_tot;
        p.hdr[1] += 1.0;
        p.hdr[2] = 1.0;                   // subspace form: (Q, H) are authoritative, (V, S) are stale
        p.hdr[3] = (double)cur;
        p.hdr[4] = (double)it;
        p.hdr[5] = rel;
        p.hdr[6] = fmax(p.hdr[6], rel);
        p.hdr[7] += (double)it;
        if (!conv) atomicOr(p.status, 2);
        PROF(8);
        for (int q = 0; q < 9; ++q) p.Prof[q] += prof[q];
        p.Prof[9] += (double)it;
        p.Prof[10] += 1.0;
    }
    __syncthreads();
    sc_cluster_sync();
}
#undef PROF

// (V, S) of the direct first step -> (Q, H):  Q[i][t] = V[t][i], H = diag(S^2)
__global__ void to_subspace_kernel(double *hdr, const double *__restrict__ S, const double *__restrict__ V, double *__restrict__ H,
                                   double *__restrict__ Qbuf, int d, int c) {
    const int cp = c + 4;
    const size_t idx = blockIdx.x * (size_t)blockDim.x + threadIdx.x;
    if (idx < (size_t)d * cp) {
        const int i = (int)(idx / cp), t = (int)(idx % cp);
        Qbuf[idx] = (t < c) ? V[(size_t)t * d + i] : 0.0;
    }
    if (idx < (size_t)c * c) {
        const int a = (int)(idx / c), b = (int)(idx % c);
        H[idx] = (a == b) ? S[a] * S[a] : 0.0;
    }
    if (idx == 0) { hdr[2] = 1.0; hdr[3] = 0.0; hdr[4] = 0.0; hdr[5] = 0.0; hdr[6] = 0.0; hdr[7] = 0.0; }
}

// H[c,c] embedded in an n x n matrix (n = c rounded up to 32) whose padding diagonal lies below the spectrum of H
__global__ void embed_h_kernel(const double *__restrict__ hdr, const double *__restrict__ H, int c, int n, double *__restrict__ A) {
    if (hdr[2] == 0.0) {              // eigen form: (V, S) are valid already; hand the solver a harmless diagonal matrix
        for (int i = threadIdx.x; i < n * n; i += blockDim.x) A[i] = (i / n == i % n) ? -(double)(i / n + 1) : 0.0;
        return;
    }
    __shared__ double red[64];
    double m = 0.0;
    for (int i = threadIdx.x; i < c * c; i += blockDim.x) m = fmax(m, fabs(H[i]));
    for (int o = 16; o > 0; o >>= 1) m = fmax(m, __shfl_xor_sync(0xffffffffu, m, o));
    if ((threadIdx.x & 31) == 0) red[threadIdx.x >> 5] = m;
    __syncthreads();
    m = 0.0;
    for (int q = 0; q < (int)(blockDim.x >> 5); ++q) m = fmax(m, red[q]);
    const double padv = -(m * c + 1.0);
    for (int i = threadIdx.x; i < n * n; i += blockDim.x) {
        const int a = i / n, b = i % n;
        A[i] = (a < c && b < c) ? H[(size_t)a * c + b] : ((a == b) ? padv : 0.0);
    }
}

// V[t][i] = sum_s Z[t][s] Q[i][s]  (Z rows = eigenvectors of H), S[t] = sqrt(lam_t).  Grid (d / 128, c / 8): a thread owns one
// feature i and eight components t (this kernel sits on the tail of every run: two 256-thread blocks took 0.93 ms)
constexpr int ROT_T = 8;
__global__ void __launch_bounds__(128)
rotate_kernel(const double *__restrict__ hdr, const double *__restrict__ Z, int n, const double *__restrict__ lam,
              const double *__restrict__ Qbuf, int d, int c, double *__restrict__ V, double *__restrict__ S) {
    if (hdr[2] == 0.0) return;
    __shared__ double zs[ROT_T][132];                        // this block's ROT_T rows of Z (c <= 128)
    const int cp = c + 4, t0 = blockIdx.y * ROT_T;
    const double *Q = Qbuf + (size_t)((int)hdr[3]) * d * cp;
    for (int k = threadIdx.x; k < ROT_T * c; k += blockDim.x) {
        const int t = k / c, sidx = k % c;
        zs[t][sidx] = (t0 + t < c) ? Z[(size_t)(t0 + t) * n + sidx] : 0.0;
    }
    __syncthreads();
    if (blockIdx.x == 0 && threadIdx.x < ROT_T && t0 + threadIdx.x < c) S[t0 + threadIdx.x] = sqrt(fmax(lam[t0 + threadIdx.x], 0.0));
    const int i = blockIdx.x * blockDim.x + threadIdx.x;     // feature index
    if (i >= d) return;
    const double *qrow = Q + (size_t)i * cp;
    double acc0[ROT_T], acc1[ROT_T];
#pragma unroll
    for (int t = 0; t < ROT_T; ++t) acc0[t] = acc1[t] = 0.0;
    // same summation order per output as before: even / odd partial sums, then their sum
    int sidx = 0;
    for (; sidx + 1 < c; sidx += 2) {
        const double q0 = qrow[sidx], q1 = qrow[sidx + 1];
#pragma unroll
        for (int t = 0; t < ROT_T; ++t) { acc0[t] = fma(zs[t][sidx], q0, acc0[t]); acc1[t] = fma(zs[t][sidx + 1], q1, acc1[t]); }
    }
    if (sidx < c) {
        const double q0 = qrow[sidx];
#pragma unroll
        for (int t = 0; t < ROT_T; ++t) acc0[t] = fma(zs[t][sidx], q0, acc0[t]);
    }
#pragma unroll
    for (int t = 0; t < ROT_T; ++t)
        if (t0 + t < c) V[(size_t)(t0 + t) * d + i] = acc0[t] + acc1[t];
}

// ------------------------------------------------------------------------------------------------------------------
bool subspace_applicable(int d, int c) {
    if (chain_forced_direct()) return false;
    static int mode = -1;
    if (mode == -1) {
        const char *env = getenv("GANSPACE_B200_CHAIN");
        mode = (env && strcmp(env, "direct") == 0) ? 0 : 1;
    }
    return mode == 1 && d % 128 == 0 && d >= 128 && d <= 512 && c % 8 == 0 && c >= 8 && c <= 128 && 2 * c <= d + d / 4 &&
           subspace_smem_bytes(d, c) <= 227 * 1024;
}

size_t subspace_smem_bytes(int d, int c) {
    const int cp = c + 4, RPC = d / SC_CL;
    return ((size_t)SC_STAGES * RPC * SC_LDA + (size_t)SC_STAGES * SC_KT * cp + 2 * (size_t)RPC * cp + (size_t)c * cp + d + 64 +
            2 * 16 * 10 * 9 + 80) * sizeof(double);
}

SubspaceWs carve_subspace(void *base, int d, int c) {
    SubspaceWs w;
    char *p = reinterpret_cast<char *>(base);
    size_t off = 0;
    auto take = [&](size_t bytes) { char *q = p + off; off += align_up(bytes, 256); return q; };
    const int RPC = d / SC_CL, nkt = d / SC_KT;
    w.Gt = (double *)take((size_t)SC_CL * nkt * RPC * SC_LDA * 8);
    w.Part = (double *)take((size_t)SC_CL * 2 * c * c * 8);
    w.Red = (double *)take((size_t)2 * c * c * 8);
    w.Slots = (double *)take(SC_CL * 8);
    w.bytes = off;
    return w;
}

// residual / tolerance ratio above which an iteration multiplies by G twice before orthonormalising (GANSPACE_B200_SUBSPACE_DBL;
// 0 = never).  One multiplication gains a factor lambda_{c+1}/lambda_c ~ 1/k at step k, so "more than 10x away" means at least
// two more iterations early in a run and costs at most one spare GEMM late in it.
static double double_step_factor() {
    static double f = -1.0;
    if (f < 0.0) {
        const char *e = getenv("GANSPACE_B200_SUBSPACE_DBL");
        f = e ? atof(e) : 10.0;                                // measured with the blocked Cholesky: 314 -> 213 us per step, same digits
        if (!(f > 0.0)) f = 1e300;
    }
    return f;
}

int subspace_step(double *hdr, double *mean, double *unnorm, double *H, double *Qbuf, const double *mean_b, const double *gram_b,
                  const SubspaceWs &w, int d, int c, double n_seen, double n_b, cudaStream_t st) {
    static double tol = -1.0;
    static int maxit = 0;
    if (tol < 0.0) {
        const char *e1 = getenv("GANSPACE_B200_SUBSPACE_TOL"), *e2 = getenv("GANSPACE_B200_SUBSPACE_MAXIT");
        // residual tolerance ||G Q - Q H||_F / min diag H: 1e-4 reproduces the exact chain to cos 0.99999997 over 40 steps of
        // config 2 (tools/study_subspace_chain.py; 1e-3: 0.999998, 1e-2: 0.99992) with ~25 % fewer iterations than 1e-5
        tol = e1 ? atof(e1) : 1e-4;
        if (!(tol > 0.0)) tol = 1e-4;
        maxit = e2 ? atoi(e2) : 60;
        if (maxit < 1) maxit = 60;
    }
    const size_t smem = subspace_smem_bytes(d, c);
    const bool small = (c <= 80 && c + d / SC_CL <= 112);   // register tile of the Cholesky: 7 x 5 or 10 x 8 per thread
    auto kern = small ? subspace_step_kernel<7, 5> : subspace_step_kernel<10, 8>;
    static bool cluster_set[2] = {false, false};
    if (!cluster_set[small]) {
        GSB_CHECK_CUDA(cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1));
        cluster_set[small] = true;
    }
    if (int r = raise_dyn_smem(kern, smem)) return r;
    SubspaceParams p;
    p.hdr = hdr; p.mean = mean; p.unnorm = unnorm; p.H = H; p.Qbuf = Qbuf;
    p.mean_b = mean_b; p.gram_b = gram_b;
    p.Gt = w.Gt; p.Part = w.Part; p.Red = w.Red; p.Slots = w.Slots; p.Prof = hdr + 8;
    p.d = d; p.c = c; p.n_seen = n_seen; p.n_b = n_b; p.tol = tol; p.maxit = maxit; p.dbl = double_step_factor();
    p.status = eig_status_device_ptr();
    GSB_CHECK_ARG(p.status, "subspace_step: no device status word");
    cudaLaunchConfig_t cfg{};
    cfg.gridDim = dim3(SC_CL); cfg.blockDim = dim3(SC_THREADS); cfg.dynamicSmemBytes = smem; cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeClusterDimension;
    at[0].val.clusterDim.x = SC_CL; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    GSB_CHECK_CUDA(cudaLaunchKernelEx(&cfg, kern, p));
    return GSB_OK;
}

int to_subspace_form(double *hdr, const double *S, const double *V, double *H, double *Qbuf, int d, int c, cudaStream_t st) {
    const size_t tot = (size_t)d * (c + 4);
    to_subspace_kernel<<<(unsigned)((tot + 255) / 256), 256, 0, st>>>(hdr, S, V, H, Qbuf, d, c);
    GSB_CHECK_LAUNCH();
    return GSB_OK;
}

// (Q, H) -> (V, S): eigen-decomposition of H with the direct solver, V = Z Q^T, svd_flip sign rule.  No-ops on the device
// when the state is still in eigen form (hdr[2] == 0).
int materialise_components(double *hdr, double *S, double *V, const double *H, const double *Qbuf, void *eig_ws, int d, int c,
                           cudaStream_t st) {
    const int n = (c + 31) / 32 * 32;
    Workspace w = carve(eig_ws, n, c);
    embed_h_kernel<<<1, 256, 0, st>>>(hdr, H, c, n, w.A);
    GSB_CHECK_LAUNCH();
    if (int r = eig_top(w, n, c, w.lam, w.evecs, st)) return r;
    GSB_CHECK_ARG(c <= 128, "materialise_components: c <= 128");
    rotate_kernel<<<dim3((unsigned)((d + 127) / 128), (unsigned)((c + ROT_T - 1) / ROT_T)), 128, 0, st>>>(hdr, w.evecs, n, w.lam, Qbuf, d,
                                                                                                    c, V, S);
    GSB_CHECK_LAUNCH();
    return sign_rows(V, c, d, st);
}

}  // namespace gsb
