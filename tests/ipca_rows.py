"""Rows with a known spectrum for the IPCA parity tests (test_large_d_engine_gpu.py, test_small_d_chain_gpu.py)."""
import numpy as np


class Data:
    """Batches X = Z diag(sigma) B^T + noise + shift with a known spectrum ("gapped": sigma_k^2 = 0.97^k; "power":
    sigma_k^2 = 1/(k+1)), generated on the host from fixed RandomState seeds so that the device and the oracle see the same
    fp32 rows; batch i depends on (seed, i).

    B is an orthonormal d x r basis (r = c + 16, at most d, or ``rank``) and Z is centred with orthogonal columns of norm
    sqrt(nb), so every batch's centred scatter is exactly diag(sigma^2) nb in B.  The noise floor sits 10x below the smallest
    signal eigenvalue of a batch (``noise=False``: no noise, the rows lie in an affine r-dimensional subspace).  The mean
    alternates by +-delta u between batches (u orthogonal to B when r < d, delta^2 = 1.5 sigma_0^2): only the
    mean-correction row carries that direction into the state, and from the second batch on it is the top component."""

    def __init__(self, d, c, nb, spectrum, seed, spikes=(), rank=None, noise=True):
        rng = np.random.RandomState(seed)
        self.d, self.seed, self.r = d, seed, min(c + 16, d) if rank is None else rank
        k = np.arange(self.r, dtype=np.float64)
        self.sig2 = 0.97 ** k if spectrum == "gapped" else 1.0 / (k + 1.0)
        G = rng.standard_normal((d, self.r)) / np.sqrt(d)
        for i, col in enumerate(spikes):
            G[d - 1 - 97 * i, col] = 0.25                 # global maximum: last feature quarter
            G[11 + 97 * i, col] = -0.15                   # shard 0's maximum, opposite sign
        self.B = np.linalg.qr(G)[0]
        u = rng.standard_normal(d)
        if self.r < d:
            u -= self.B @ (self.B.T @ u)
        self.u = u / np.linalg.norm(u)
        self.shift = 2.0 * rng.standard_normal(d)
        # a batch's noise eigenvalues (Marchenko-Pastur edge nu^2 (sqrt d + sqrt nb)^2) 10x below nb sigma_{r-1}^2
        self.nu = np.sqrt(0.1 * self.sig2[-1] * nb / (np.sqrt(d) + np.sqrt(nb)) ** 2) if noise else 0.0
        self.delta = np.sqrt(1.5 * self.sig2[0])

    def batch(self, i, nb):
        """Batch i of nb >= r rows (fp32)."""
        rng = np.random.RandomState([self.seed, i])
        Z = rng.standard_normal((nb, self.r))
        Z -= Z.mean(axis=0)
        Z = np.linalg.qr(Z)[0] * np.sqrt(nb)              # centred, Z^T Z = nb I
        X = (Z * np.sqrt(self.sig2)) @ self.B.T
        if self.nu:
            X += self.nu * rng.standard_normal((nb, self.d))
        X += self.shift + (1.0 if i % 2 == 0 else -1.0) * self.delta * self.u
        return X.astype(np.float32)
