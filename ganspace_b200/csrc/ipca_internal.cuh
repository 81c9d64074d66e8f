// Internal interfaces of the small-d chain, shared by ipca.cu and subspace.cu.
#pragma once
#include "eig.cuh"

namespace gsb {

// sticky device-side status word of the chain kernels (bit1: a subspace step hit its iteration cap)
int *eig_status_device_ptr();

// subspace.cu: chain step as orthogonal iteration on (Q, H) (no per-step eigen-decomposition)
struct SubspaceWs {
    double *Gt, *Part, *Red, *Slots;
    size_t bytes;
};
bool subspace_applicable(int d, int c);
// gsb_ipca_set_chain_mode(1): every chain step is the direct solve until it is set back to 0 (the host's fallback after a run
// whose iteration hit its cap, i.e. data without a spectral gap after component c)
bool chain_forced_direct();
size_t subspace_smem_bytes(int d, int c);
SubspaceWs carve_subspace(void *base, int d, int c);
int subspace_step(double *hdr, double *mean, double *unnorm, double *H, double *Qbuf, const double *mean_b, const double *gram_b,
                  const SubspaceWs &w, int d, int c, double n_seen, double n_b, cudaStream_t st);
int to_subspace_form(double *hdr, const double *S, const double *V, double *H, double *Qbuf, int d, int c, cudaStream_t st);
int materialise_components(double *hdr, double *S, double *V, const double *H, const double *Qbuf, void *eig_ws, int d, int c,
                           cudaStream_t st);

}  // namespace gsb
