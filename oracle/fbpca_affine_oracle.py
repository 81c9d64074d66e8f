"""ORACLE -- test infrastructure only: --est fbpca on a layer that is affine in the latent (BigGAN-512 generator.gen_z).

  * ``pca``: fbpca.pca (raw=True, dense real input) with BOTH of its randomized branches.  oracle/fbpca_oracle.py restates
    the tall one (m >= n); a gen_z run with N + NB < 32768 samples takes the wide one (m < n), which draws its test matrix
    over the rows, uniform(-1, 1) of shape (l, m).  ``oracle/gen_golden_fbpca_affine.py`` installs this module as
    ``sys.modules['fbpca']`` when it runs the unmodified reference.
  * ``compute_genz_literal``: decomposition.compute with estimator='fbpca' on the materialised [N + NB, 32768] activations,
    fbpca's literal algorithm in fp64 -- independent of the low-rank shortcut the device takes (DESIGN.md section 5g).
  * ``linear_form`` / ``lifted_solve``: that shortcut restated in NumPy (fp64), for the CPU tests.
"""
from __future__ import annotations

import numpy as np
import scipy.linalg

from oracle import fbpca_oracle as fbo
from oracle import ganspace_oracle as orc


def pca(A, k=6, raw=False, n_iter=2, l=None):
    """fbpca.pca restated for dense real A with raw=True, both shapes."""
    if l is None:
        l = k + 2
    m, n = A.shape
    if m >= n or l >= m / 1.25 or l >= n / 1.25:
        return fbo.pca(A, k=k, raw=raw, n_iter=n_iter, l=l)
    assert k > 0 and k <= min(m, n) and n_iter >= 0 and l >= k and raw
    R = np.random.uniform(low=-1.0, high=1.0, size=(l, m)).astype(A.dtype)
    Q = R.dot(A).T
    if n_iter == 0:
        Q, _ = scipy.linalg.qr(Q, mode="economic")
    else:
        Q, _ = scipy.linalg.lu(Q, permute_l=True)
    for it in range(n_iter):
        Q = A.dot(Q)
        Q, _ = scipy.linalg.lu(Q, permute_l=True)
        Q = Q.T.dot(A).T
        if it + 1 < n_iter:
            Q, _ = scipy.linalg.lu(Q, permute_l=True)
        else:
            Q, _ = scipy.linalg.qr(Q, mode="economic")
    U, s, Ra = scipy.linalg.svd(A.dot(Q), full_matrices=False)
    Va = Ra.dot(Q.T)
    return U[:, :k], s[:k], Va[:k, :]


def fit_literal(X, c):
    """FacebookPCAEstimator.fit (estimators.py:135-156) on the centred samples X, fbpca in X's dtype.
    Returns (components, stdev, var_ratio)."""
    _, _, Va = pca(X, k=c, n_iter=2, raw=True, l=2 * c)
    stdev = np.dot(Va, X.T).std(axis=1)
    idx = np.argsort(stdev)[::-1]
    return Va[idx].copy(), stdev[idx], stdev[idx] ** 2 / X.var(axis=0).sum()


# --------------------------------------------------------------------------------------------
# the shortcut: act = y Q^T + offset  ->  act = yt Qt^T with yt = [y + Q^T offset, |offset_perp|]
# --------------------------------------------------------------------------------------------
def linear_form(Q, offset):
    """(Qt [d, r+1], t [r+1]): Q with the unit offset component outside range(Q) appended, and the coordinate shift."""
    a = Q.T @ offset
    perp = offset - Q @ a
    b = np.linalg.norm(perp)
    return np.concatenate([Q, (perp / b)[:, None]], axis=1), np.concatenate([a, [b]])


def lifted_solve(Y, n_zero, Qt, t, omega, c):
    """fbpca on [y_i Q^T + offset; n_zero zero rows] (centred), from the coordinates alone: the pooled (mean, scatter) of
    yt = [y + a, b] and the zero rows, Omega' = Qt^T Omega (None: exact branch), the Gram-form solve, lifted through Qt.
    Returns (components [c, d], stdev, var_ratio, mean [d])."""
    Yt = np.concatenate([np.asarray(Y, np.float64) + t[None, :-1], np.full((len(Y), 1), t[-1])], axis=1)
    Yt = np.concatenate([Yt, np.zeros((n_zero, Yt.shape[1]))])
    mean = Yt.mean(0)
    S = (Yt - mean).T @ (Yt - mean)
    Va, _ = fbo.gram_solve(S, None if omega is None else Qt.T @ np.asarray(omega, np.float64), c)
    q = np.einsum("kd,de,ke->k", Va, S, Va)
    idx = np.argsort(q)[::-1]
    m = len(Yt)
    return Va[idx] @ Qt.T, np.sqrt(q[idx] / m), q[idx] / np.trace(S), mean @ Qt.T


# --------------------------------------------------------------------------------------------
# compact fixtures: gen_z's activation-space arrays lie in span(W_z, offset), 129 columns of the layer's own weights
# --------------------------------------------------------------------------------------------
SPAN_KEYS = ("act_comp", "act_mean")


def genz_span(params, class_idx: int = 248):
    """M [32768, 129] fp64 = [W_z, offset]: every activation row, every centred row and every component of gen_z's
    decomposition is a combination of these columns (offset = bias + W_embed @ embedding)."""
    w = params["w_eff"].astype(np.float64)
    offset = params["bias"].astype(np.float64) + w[:, 128:] @ params["emb"][:, class_idx].astype(np.float64)
    return np.concatenate([w[:, :128], offset[:, None]], axis=1)


def encode_span(arrays, params):
    """act_comp / act_mean as least-squares coefficients over genz_span (``<key>_coef``, fp64) and the relative residual of
    each row (``<key>_resid``); the other arrays unchanged.  129 numbers per row instead of 32768."""
    M = genz_span(params)
    out = {k: v for k, v in arrays.items() if k not in SPAN_KEYS}
    for k in SPAN_KEYS:
        rows = np.asarray(arrays[k], np.float64).reshape(-1, M.shape[0])
        coef = np.linalg.lstsq(M, rows.T, rcond=None)[0].T
        out[f"{k}_coef"] = coef
        out[f"{k}_resid"] = np.linalg.norm(rows - coef @ M.T, axis=1) / np.linalg.norm(rows, axis=1)
        out[f"{k}_shape"] = np.array(np.shape(arrays[k]))
    return out


def decode_span(fixture, params):
    """The 8-array dict of an encode_span fixture; act_comp / act_mean rebuilt from their coefficients (float32)."""
    M = genz_span(params)
    out = {k: fixture[k] for k in ("dump_name", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio",
                                   "random_stdevs")}
    for k in SPAN_KEYS:
        out[k] = (fixture[f"{k}_coef"] @ M.T).reshape(tuple(fixture[f"{k}_shape"])).astype(np.float32)
    return out


# --------------------------------------------------------------------------------------------
# decomposition.compute (:150-341), estimator='fbpca', layer generator.gen_z, on the materialised activations
# --------------------------------------------------------------------------------------------
def compute_genz_literal(params, n: int, B: int, c: int, class_idx: int = 248, dtype=np.float64):
    """The reference's compute path with fbpca's literal algorithm run in ``dtype`` on the stacked activations."""
    sample = lambda s, B_: orc.truncated_noise_sample(s, B_)
    activate = lambda z: orc.genz_forward(z, params, class_idx)
    d = params["w_eff"].shape[0]
    N, NB, n_lat, K = orc.plan(n, B, c)
    np.random.seed(orc.SEED_SAMPLING)
    seeds = [int(np.random.randint(fbo.INT32_MAX)) for _ in range(n_lat // B)]
    latents = np.concatenate([sample(s, B) for s in seeds], axis=0)
    samples = np.zeros((N + NB, d), np.float32)
    for gi in range(0, N, NB):
        samples[gi:gi + NB] = activate(latents[gi:gi + NB])
    X_global_mean = samples.mean(axis=0, keepdims=True, dtype=np.float32)
    samples -= X_global_mean
    X = samples.astype(dtype)
    del samples
    X_comp, X_stdev, X_var_ratio = fit_literal(X, c)
    Z_comp, Z_mean = orc.linreg(sample, activate, 128, X_comp, X_global_mean, X_stdev, n, B)
    Z_comp = Z_comp / np.linalg.norm(Z_comp, axis=-1, keepdims=True)
    random_dirs = orc.get_random_dirs(c, d)
    X_stdev_random = np.dot(random_dirs, X[:min(5000, X.shape[0])].T).std(axis=1)
    return {
        "act_comp": X_comp.reshape(-1, 1, d).astype(np.float32),
        "act_mean": X_global_mean.reshape(1, d).astype(np.float32),
        "act_stdev": X_stdev.astype(np.float32),
        "lat_comp": Z_comp.reshape(-1, 1, 128).astype(np.float32),
        "lat_mean": np.asarray(Z_mean).reshape(1, 128).astype(np.float32),
        "lat_stdev": np.ones_like(X_stdev).astype(np.float32),
        "var_ratio": X_var_ratio.astype(np.float32),
        "random_stdevs": X_stdev_random.astype(np.float32),
    }
