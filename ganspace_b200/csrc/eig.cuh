// Interface of the fp64 symmetric eigensolver (eig.cu), used by the small-d chain (ipca.cu, subspace.cu), the large-d engine
// (bigd.cu) and fbpca (rsvd.cu).
#pragma once
#include "common.cuh"

namespace gsb {

struct Workspace {
    double *A, *dg, *e, *beta, *Vh, *lam, *Z, *evecs, *xch, *qx;
    unsigned *counter;
    size_t bytes;
};
Workspace carve(void *base, int d, int c);
// top-c eigenpairs (descending) of the symmetric matrix held in w.A (destroyed), 32 <= d <= 4096, d % 32 == 0; evecs rows are
// sign-normalised
int eig_top(const Workspace &w, int d, int c, double *evals, double *evecs, cudaStream_t st);

// svd_flip sign rule on the rows of V[c,d]
int sign_rows(double *V, int c, int d, cudaStream_t st);

}  // namespace gsb
