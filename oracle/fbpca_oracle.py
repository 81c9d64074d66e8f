"""ORACLE -- test infrastructure only: the Facebook PCA estimator (--est fbpca) restated in NumPy.

Two restatements, both pinned by tests/test_fbpca.py:
  * ``pca``: the published fbpca algorithm (fbpca.pca, Facebook's randomized PCA package) for the case the reference uses --
    dense real A, raw=True -- with both of its branches for m >= n: exact SVD when l >= m/1.25 or l >= n/1.25, otherwise a
    uniform(-1, 1) test matrix drawn from NumPy's global state, LU-normalised power iterations, a final QR and the SVD of
    Q^T A.  fbpca is a third-party package (absent here and not part of the reference); ``oracle/gen_golden_fbpca.py``
    installs this module as ``sys.modules['fbpca']`` when it runs the unmodified reference.
  * ``gram_solve``: the same fit from G = A^T A alone, in fp64 -- the form csrc/rsvd.cu computes on the device:
    Y = orth(G^n_iter Omega) (CholQR2 between the products), P = G Y, L = chol(Y^T P), F = P L^-T; Q^T A = F^T, so
    (Va, s) are the top-k left singular vectors / singular values of F, from the eigenpairs of F^T F.

``compute_path_fbpca`` restates decomposition.compute (:150-341) for estimator='fbpca' on top of ganspace_oracle's sampling,
mapping and regression restatements.  The product package never imports this module.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

from oracle import ganspace_oracle as orc

INT32_MAX = 2147483647


# --------------------------------------------------------------------------------------------
# fbpca.pca (raw=True, dense real input)
# --------------------------------------------------------------------------------------------
def pca(A, k=6, raw=False, n_iter=2, l=None):
    """fbpca.pca restated for dense real A with raw=True (the reference's only call, estimators.py:136)."""
    if l is None:
        l = k + 2
    m, n = A.shape
    assert k > 0 and k <= min(m, n) and n_iter >= 0 and l >= k
    if not raw:
        raise NotImplementedError("only raw=True is restated (the reference passes raw=True)")
    if l >= m / 1.25 or l >= n / 1.25:
        U, s, Va = scipy.linalg.svd(A, full_matrices=False)
        return U[:, :k], s[:k], Va[:k, :]
    if m < n:
        raise NotImplementedError("only m >= n is restated (the reference's sample matrices are tall)")
    Q = np.random.uniform(low=-1.0, high=1.0, size=(n, l)).astype(A.dtype)
    Q = A.dot(Q)
    if n_iter == 0:
        Q, _ = scipy.linalg.qr(Q, mode="economic")
    else:
        Q, _ = scipy.linalg.lu(Q, permute_l=True)
    for it in range(n_iter):
        Q = Q.T.dot(A).T
        Q, _ = scipy.linalg.lu(Q, permute_l=True)
        Q = A.dot(Q)
        if it + 1 < n_iter:
            Q, _ = scipy.linalg.lu(Q, permute_l=True)
        else:
            Q, _ = scipy.linalg.qr(Q, mode="economic")
    QA = Q.T.dot(A)
    R, s, Va = scipy.linalg.svd(QA, full_matrices=False)
    U = Q.dot(R)
    return U[:, :k], s[:k], Va[:k, :]


# --------------------------------------------------------------------------------------------
# the Gram form (what the device computes)
# --------------------------------------------------------------------------------------------
def _cholqr2(Y):
    for _ in range(2):
        L = np.linalg.cholesky(Y.T @ Y)
        Y = scipy.linalg.solve_triangular(L, Y.T, lower=True).T
    return Y


def gram_solve(G, omega, k, n_iter=2):
    """(Va [k, n], s [k]) of fbpca.pca(A, k, n_iter, raw=True, l) from G = A^T A (fp64); omega [n, l] = fbpca's test matrix,
    None = the exact branch (top-k eigenpairs of G)."""
    G = np.asarray(G, np.float64)
    if omega is None:
        lam, V = np.linalg.eigh(G)
        lam, V = lam[::-1][:k], V[:, ::-1][:, :k]
        return V.T.copy(), np.sqrt(np.maximum(lam, 0.0))
    Y = np.asarray(omega, np.float64)
    for _ in range(n_iter):
        Y = _cholqr2(G @ Y)
    P = G @ Y
    L = np.linalg.cholesky(Y.T @ P)
    F = scipy.linalg.solve_triangular(L, P.T, lower=True).T
    lam, W = np.linalg.eigh(F.T @ F)
    lam, W = lam[::-1][:k], W[:, ::-1][:, :k]
    s = np.sqrt(lam)
    return (F @ W / s).T.copy(), s


def randomized(k, m, n):
    """fbpca's branch for an [m, n] input with l = 2k: True = randomized range finder, False = exact SVD."""
    l = 2 * k
    return not (l >= m / 1.25 or l >= n / 1.25)


def sign_normalise(out):
    """Apply the sign rule of the device (largest-|.| entry of each act_comp row positive) to act_comp and, with the same
    signs, to lat_comp (fbpca's signs are LAPACK's choice; the regression is linear in them)."""
    c = out["act_comp"].shape[0]
    a = np.asarray(out["act_comp"]).reshape(c, -1)
    _, signs = orc.svd_flip_v(a.astype(np.float64))
    res = dict(out)
    res["act_comp"] = (a * signs[:, None].astype(a.dtype)).reshape(out["act_comp"].shape).astype(out["act_comp"].dtype)
    lat = np.asarray(out["lat_comp"])
    res["lat_comp"] = (lat.reshape(c, -1) * signs[:, None].astype(lat.dtype)).reshape(lat.shape).astype(lat.dtype)
    return res


# --------------------------------------------------------------------------------------------
# decomposition.compute (:150-341) with estimator='fbpca'
# --------------------------------------------------------------------------------------------
def fit_estimator(X, c, form, omega_draw=True):
    """FacebookPCAEstimator.fit (estimators.py:135-156) on the centred [m, d] samples X (float32); the test matrix comes from
    the global NumPy state at the moment of the call, as in fbpca.  Returns (components, stdev, var_ratio)."""
    m, d = X.shape
    if form == "literal":
        _, _, Va = pca(X, k=c, n_iter=2, raw=True, l=2 * c)
    else:
        omega = np.random.uniform(low=-1.0, high=1.0, size=(d, 2 * c)).astype(np.float32) if randomized(c, m, d) else None
        X64 = X.astype(np.float64)
        Va, _ = gram_solve(X64.T @ X64, omega, c)
    total_var = X.var(axis=0).sum()
    stdev = np.dot(Va, X.T).std(axis=1)
    idx = np.argsort(stdev)[::-1]
    return Va[idx].copy(), stdev[idx], stdev[idx] ** 2 / total_var


def compute_path_fbpca(sample, activate, latent_dims: int, feat_dims: int, n: int, B: int, c: int, samples_are_latents: bool,
                       seed=None, use_w: bool = False, form: str = "gram", regress: bool = True):
    """decomposition.compute for estimator='fbpca' (non-batched: decomposition.py:222-224, 245-267, 276-287).
        sample(seed, B) -> one model.sample_latent(B) call;  activate(latents) -> hooked activations [B, feat_dims]
    ``form``: 'literal' = fbpca restatement on the stacked matrix, 'gram' = the fp64 Gram form."""
    d = feat_dims
    c = min(c, d)
    N, NB, n_lat, K = orc.plan(n, B, c)
    np.random.seed(seed or orc.SEED_SAMPLING)
    seeds = [int(np.random.randint(INT32_MAX)) for _ in range(n_lat // B)]     # one sample_latent(B) per call (:232-236)
    latents = np.concatenate([sample(s, B) for s in seeds], axis=0)
    samples = np.zeros((N + NB, d), np.float32)                                  # :224 (rows past K NB stay zero)
    for gi in range(0, N, NB):
        rows = latents[gi:gi + NB]
        samples[gi:gi + NB] = rows if samples_are_latents else activate(rows)
    X_global_mean = samples.mean(axis=0, keepdims=True, dtype=np.float32)       # :278
    X = samples - X_global_mean
    X_comp, X_stdev, X_var_ratio = fit_estimator(X, c, form)                    # global state: Omega right after phase A
    X_comp = X_comp.astype(np.float64) if form == "gram" else X_comp

    if samples_are_latents:
        Z_comp, Z_mean = X_comp, X_global_mean
    elif not regress:
        Z_comp, Z_mean = np.ones((c, latent_dims)), np.zeros((1, latent_dims))
    else:
        Z_comp, Z_mean = orc.linreg(sample, activate, latent_dims, X_comp, X_global_mean, X_stdev, n, B)
    Z_comp = Z_comp / np.linalg.norm(Z_comp, axis=-1, keepdims=True)
    if samples_are_latents:
        X_comp = Z_comp

    random_dirs = orc.get_random_dirs(c, d)
    n_rand = min(5000, X.shape[0])
    X_stdev_random = np.dot(random_dirs, X[:n_rand].T).std(axis=1)              # first rows of the whole matrix

    lat_stdev = np.ones_like(X_stdev)
    if use_w:
        lat_seed = int(np.random.randint(INT32_MAX))                              # :327, after fbpca's draw
        coords = np.dot(Z_comp.reshape(-1, latent_dims), sample(lat_seed, 5000).T)
        lat_stdev = coords.std(axis=1)
    return {
        "act_comp": X_comp.reshape(-1, 1, d).astype(np.float32),
        "act_mean": X_global_mean.reshape(1, d).astype(np.float32),
        "act_stdev": X_stdev.astype(np.float32),
        "lat_comp": Z_comp.reshape(-1, 1, latent_dims).astype(np.float32),
        "lat_mean": np.asarray(Z_mean).reshape(1, latent_dims).astype(np.float32),
        "lat_stdev": lat_stdev.astype(np.float32),
        "var_ratio": X_var_ratio.astype(np.float32),
        "random_stdevs": X_stdev_random.astype(np.float32),
    }


def compute_stylegan2_style_fbpca(weights, biases, n: int, B: int, c: int, use_w: bool, seed=None, form: str = "gram"):
    """model=StyleGAN2, layer='style', --est fbpca (W space: the samples are the latents; Z space: mapping(z), regression)."""
    mapping = lambda z: orc.mapping_forward(z, weights, biases)
    normals = lambda s, B_: orc.standard_normal_f32(s, 512 * B_).reshape(B_, 512)
    if use_w:
        sample = lambda s, B_: mapping(normals(s, B_))
        return compute_path_fbpca(sample, None, 512, 512, n, B, c, True, seed=seed, use_w=True, form=form)
    return compute_path_fbpca(normals, mapping, 512, 512, n, B, c, False, seed=seed, form=form)
