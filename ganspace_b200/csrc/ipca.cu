// Incremental-PCA chain, small-d engine (d <= 1024): all state and arithmetic fp64, on device.
//
// Replaces estimators.py:55-81 (IPCAEstimator.fit_partial / get_components), i.e. scikit-learn's
// IncrementalPCA.partial_fit (_incremental_pca.py:254-380) in its Gram form (SURVEY.md section 0.3):
//     G = V^T S^2 V + Xc^T Xc + m m^T,   m = sqrt(n_seen*n_b/n_tot) (mean - mean_b)
//     top-c eigenpairs of G  ->  components_ (svd_flip sign rule), singular_values_ = sqrt(lambda)
//     mean/var merge of extmath._incremental_mean_and_var (Chan et al.), batch variance = diag(Xc^T Xc)
//
// The eigenpairs come from the fp64 direct solver (eig.cu).
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

__device__ int g_eig_status = 0;
int *eig_status_device_ptr() {
    static int *p = nullptr;
    if (!p && cudaGetSymbolAddress((void **)&p, g_eig_status) != cudaSuccess) p = nullptr;
    return p;
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
