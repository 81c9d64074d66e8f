"""ORACLE -- test infrastructure only.

CPU restatement (numpy + the plain-C RNG in ``mt19937_legacy.c``) of the reference's
activation-sampling + incremental-PCA hot path.  Only ``tests/``, ``__graft_entry__.smoke()`` and
``bench.py``'s cpu_baseline / ``--impl reference`` legs may import this module; the product package
``ganspace_b200`` never does (tests/test_no_oracle_in_product.py enforces it).

Every function cites the reference file:line it follows (paths relative to /root/reference).

Parity pinning (SURVEY.md section 8c): the reference holds no golden vectors for this path that can be
regenerated offline, so the oracle is pinned against *outputs of the reference itself run in the
build container*: ``oracle/gen_golden.py`` imports the unmodified reference (``decomposition.py``,
``models/wrappers.py``, the vendored StyleGAN2 generator) plus scikit-learn 1.9.0 /
NumPy 2.3.5 / SciPy 1.18.1, and writes the fixtures under ``tests/golden/``;
``tests/test_oracle_golden.py`` checks this restatement against them.

Third-party arithmetic restated here (absent from /root/reference, un-pinned by environment.yml:14-15):
  * NumPy legacy RandomState (MT19937, polar normals, masked randint)      -> mt19937_legacy.c
  * scikit-learn IncrementalPCA.partial_fit / _incremental_mean_and_var / svd_flip
      sklearn/decomposition/_incremental_pca.py:254-380, sklearn/utils/extmath.py:1118-1265,924-982
  * scipy.linalg.lstsq(gelsd) (decomposition.py:133), scipy.stats.truncnorm.rvs (biggan utils.py:32)
"""
from __future__ import annotations

import ctypes
import os
import subprocess
from pathlib import Path

import numpy as np

_HERE = Path(__file__).resolve().parent
_LIB = None


def build_c(force: bool = False) -> Path:
    """Compile the C restatement (gcc) into oracle/_build/."""
    out = _HERE / "_build" / "libmt19937_legacy.so"
    src = _HERE / "mt19937_legacy.c"
    if force or not out.exists() or out.stat().st_mtime < src.stat().st_mtime:
        out.parent.mkdir(exist_ok=True)
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-ffp-contract=off",
                               "-o", str(out), str(src), "-lm"])
    return out


def _lib():
    global _LIB
    if _LIB is None:
        _LIB = ctypes.CDLL(str(build_c()))
    return _LIB


# --------------------------------------------------------------------------------------------
# RNG  (models/wrappers.py:167-175; decomposition.py:226-227)
# --------------------------------------------------------------------------------------------
INT32_MAX = 2147483647


def seed_sequence(seed0: int, count: int) -> np.ndarray:
    """np.random.seed(seed0); [np.random.randint(np.iinfo(np.int32).max) for _ in range(count)]
    -- the per-call seeds StyleGAN2.sample_latent draws from the global state (wrappers.py:168-169)."""
    out = np.empty(count, np.uint32)
    _lib().gso_randint_sequence(ctypes.c_uint32(seed0), ctypes.c_uint32(INT32_MAX),
                                ctypes.c_int64(count), out.ctypes.data_as(ctypes.c_void_p))
    return out


def standard_normal_f32(seed: int, n: int) -> np.ndarray:
    """RandomState(seed).standard_normal(n) cast to float32 (wrappers.py:171-174)."""
    out = np.empty(n, np.float32)
    _lib().gso_standard_normal_f32(ctypes.c_uint32(seed), ctypes.c_int64(n),
                                   out.ctypes.data_as(ctypes.c_void_p))
    return out


def standard_normal_f64(seed: int, n: int) -> np.ndarray:
    out = np.empty(n, np.float64)
    _lib().gso_standard_normal_f64(ctypes.c_uint32(seed), ctypes.c_int64(n),
                                   out.ctypes.data_as(ctypes.c_void_p))
    return out


def random_sample_f64(seed: int, n: int) -> np.ndarray:
    out = np.empty(n, np.float64)
    _lib().gso_random_sample_f64(ctypes.c_uint32(seed), ctypes.c_int64(n),
                                 out.ctypes.data_as(ctypes.c_void_p))
    return out


def raw_u32(seed: int, n: int) -> np.ndarray:
    out = np.empty(n, np.uint32)
    _lib().gso_raw_u32(ctypes.c_uint32(seed), ctypes.c_int64(n), out.ctypes.data_as(ctypes.c_void_p))
    return out


# --------------------------------------------------------------------------------------------
# StyleGAN2 mapping network  (stylegan2-pytorch/model.py:14-19,132-161,400-409; op/fused_act.py:86-92)
# --------------------------------------------------------------------------------------------
LR_MLP = 0.01
SQRT2_F32 = np.float32(2 ** 0.5)


def mapping_random_init(seed: int = 1234, n_mlp: int = 8, dim: int = 512):
    """The random-init mapping weights the BASELINE configs name: ``torch.manual_seed(seed)`` followed
    by ``Generator(size, 512, 8)`` -- the mapping EqualLinear weights are the first RNG consumers
    (model.py:400-409, weight = randn(out,in)/lr_mul :138, bias = 0 :141)."""
    import torch
    g = torch.Generator().manual_seed(seed)
    ws = [torch.randn(dim, dim, generator=g).div_(LR_MLP).numpy() for _ in range(n_mlp)]
    bs = [np.zeros(dim, np.float32) for _ in range(n_mlp)]
    return ws, bs


def pixel_norm(x: np.ndarray) -> np.ndarray:
    """model.py:14-19  input * rsqrt(mean(input**2, dim=1) + 1e-8), float32."""
    x = x.astype(np.float32, copy=False)
    ms = np.mean(x * x, axis=1, keepdims=True, dtype=np.float32) + np.float32(1e-8)
    return (x * (np.float32(1.0) / np.sqrt(ms))).astype(np.float32)


def mapping_forward_np(z: np.ndarray, weights, biases, lr_mul: float = LR_MLP) -> np.ndarray:
    """Generator.style in plain numpy: PixelNorm then 8x EqualLinear(activation='fused_lrelu')
    (model.py:151-161: F.linear(x, W*scale) ; fused_leaky_relu(out, bias*lr_mul) = sqrt2*lrelu_0.2(out+b))."""
    x = pixel_norm(z)
    for w, b in zip(weights, biases):
        scale = np.float32((1.0 / np.sqrt(w.shape[1])) * lr_mul)
        ws = (w.astype(np.float32) * scale).astype(np.float32)
        y = x @ ws.T + (b.astype(np.float32) * np.float32(lr_mul))
        y = np.where(y >= 0, y, y * np.float32(0.2)).astype(np.float32)
        x = (SQRT2_F32 * y).astype(np.float32)
    return x


def mapping_forward(z: np.ndarray, weights, biases, lr_mul: float = LR_MLP) -> np.ndarray:
    """Same network through the CPU kernels the reference itself calls (torch F.linear / leaky_relu on
    the host), so that the CPU baseline timed from this oracle spends its time where the reference does.
    model.py:14-19 (PixelNorm), :151-161 (EqualLinear.forward), op/fused_act.py:86-92 (CPU fallback)."""
    import math
    import torch
    import torch.nn.functional as F
    with torch.no_grad():
        x = torch.from_numpy(np.ascontiguousarray(z, dtype=np.float32))
        x = x * torch.rsqrt(torch.mean(x ** 2, dim=1, keepdim=True) + 1e-8)
        for w, b in zip(weights, biases):
            wt, bt = torch.from_numpy(w), torch.from_numpy(b)
            scale = (1 / math.sqrt(wt.shape[1])) * lr_mul
            out = F.linear(x, wt * scale)
            x = (2 ** 0.5) * F.leaky_relu(out + (bt * lr_mul).view(1, -1), negative_slope=0.2)
        return x.numpy()


# --------------------------------------------------------------------------------------------
# Incremental PCA  (estimators.py:55-81 -> sklearn IncrementalPCA.partial_fit)
# --------------------------------------------------------------------------------------------
class IPCAState:
    def __init__(self, n_components: int):
        self.n_components = n_components
        self.n_samples_seen = 0
        self.mean = 0.0
        self.var = 0.0
        self.components = None
        self.singular_values = None
        self.explained_variance = None
        self.explained_variance_ratio = None


def incremental_mean_and_var(X, last_mean, last_var, last_n):
    """sklearn/utils/extmath.py:1118-1265 (no NaNs, no sample weights), float64 accumulators."""
    X64 = X.astype(np.float64)
    n_new = X.shape[0]
    last_sum = last_mean * last_n
    new_sum = X64.sum(axis=0)
    n_tot = last_n + n_new
    mean = (last_sum + new_sum) / n_tot
    T = new_sum / n_new
    temp = X64 - T
    corr = temp.sum(axis=0)
    new_unnorm = (temp ** 2).sum(axis=0) - corr ** 2 / n_new
    if last_n == 0:
        unnorm = new_unnorm
    else:
        last_unnorm = last_var * last_n
        r = last_n / n_new
        unnorm = last_unnorm + new_unnorm + r / n_tot * (last_sum / r - new_sum) ** 2
    return mean, unnorm / n_tot, n_tot


def svd_flip_v(Vt):
    """sklearn svd_flip(u_based_decision=False): the largest-|.| entry of each row becomes positive."""
    idx = np.argmax(np.abs(Vt), axis=1)
    signs = np.sign(Vt[np.arange(Vt.shape[0]), idx])
    return Vt * signs[:, None], signs


def ipca_partial_fit(st: IPCAState, X: np.ndarray) -> IPCAState:
    """sklearn/decomposition/_incremental_pca.py:254-380 restated (SVD form, dtype behaviour kept:
    first batch float32 SVD, stacked matrix float64 afterwards)."""
    import scipy.linalg
    X = np.array(X, copy=True)
    n_samples = X.shape[0]
    col_mean, col_var, n_total = incremental_mean_and_var(X, st.mean, st.var, st.n_samples_seen)
    if st.n_samples_seen == 0:
        X -= col_mean
    else:
        col_batch_mean = np.mean(X, axis=0)
        X -= col_batch_mean
        mean_correction = np.sqrt((st.n_samples_seen / n_total) * n_samples) * (st.mean - col_batch_mean)
        X = np.vstack((st.singular_values.reshape((-1, 1)) * st.components, X, mean_correction))
    U, S, Vt = scipy.linalg.svd(X, full_matrices=False, check_finite=False)
    Vt, _ = svd_flip_v(Vt)
    c = st.n_components
    st.explained_variance = (S ** 2 / (n_total - 1))[:c]
    st.explained_variance_ratio = (S ** 2 / np.sum(col_var * n_total))[:c]
    st.n_samples_seen = n_total
    st.components = Vt[:c]
    st.singular_values = S[:c]
    st.mean = col_mean
    st.var = col_var
    return st


def ipca_partial_fit_small_side(st: IPCAState, X: np.ndarray) -> IPCAState:
    """The same partial_fit (_incremental_pca.py:254-380) for d >> rows: the thin SVD of the stacked matrix M [rows, d] through
    its small-side Gram  M M^T = U S^2 U^T,  Vt = S^-1 U^T M  (fp64) instead of LAPACK gesdd on M -- the same factorisation up to
    rounding, at rows^2 d instead of rows d min(rows, d) ... with a 30x smaller constant for rows = 2081, d = 32768."""
    X = np.array(X, copy=True)
    n_samples = X.shape[0]
    col_mean, col_var, n_total = incremental_mean_and_var(X, st.mean, st.var, st.n_samples_seen)
    if st.n_samples_seen == 0:
        M = X.astype(np.float64) - col_mean
    else:
        col_batch_mean = np.mean(X.astype(np.float64), axis=0)
        mean_correction = np.sqrt((st.n_samples_seen / n_total) * n_samples) * (st.mean - col_batch_mean)
        M = np.vstack((st.singular_values.reshape((-1, 1)) * st.components, X.astype(np.float64) - col_batch_mean, mean_correction))
    c = st.n_components
    lam, U = np.linalg.eigh(M @ M.T)
    lam, U = lam[::-1][:c], U[:, ::-1][:, :c]
    S = np.sqrt(np.maximum(lam, 0.0))
    Vt = (U.T @ M) / S[:, None]
    Vt, _ = svd_flip_v(Vt)
    st.explained_variance = S ** 2 / (n_total - 1)
    st.explained_variance_ratio = S ** 2 / np.sum(col_var * n_total)
    st.n_samples_seen = n_total
    st.components = Vt
    st.singular_values = S
    st.mean = col_mean
    st.var = col_var
    return st


def batch_stats(X: np.ndarray):
    """Per-batch sufficient statistics of the Gram-form chain: (n, mean[d], centred Gram[d,d]) in fp64."""
    X64 = X.astype(np.float64)
    m = X64.mean(axis=0)
    Xc = X64 - m
    return X.shape[0], m, Xc.T @ Xc


def ipca_gram_step(st: IPCAState, n_b: int, mean_b: np.ndarray, gram_b: np.ndarray) -> IPCAState:
    """Gram-form restatement of one partial_fit (SURVEY.md section 0.3 / Appendix B):
        G = V^T S^2 V + Xc^T Xc + m m^T,  m = sqrt(n_seen*n_b/n_tot) (mean - mean_b)
    eigh(G) -> top-c (lambda, v); S = sqrt(lambda); sign rule of svd_flip.  The running mean/var merge is
    Chan et al. exactly as _incremental_mean_and_var does it, using diag(Xc^T Xc) as the batch's
    unnormalised variance."""
    c = st.n_components
    n_tot = st.n_samples_seen + n_b
    new_unnorm = np.diag(gram_b).copy()
    if st.n_samples_seen == 0:
        G = gram_b.copy()
        mean = mean_b.copy()
        unnorm = new_unnorm
    else:
        V, S = st.components.astype(np.float64), st.singular_values.astype(np.float64)
        m = np.sqrt((st.n_samples_seen / n_tot) * n_b) * (st.mean - mean_b)
        G = (V.T * (S ** 2)) @ V + gram_b + np.outer(m, m)
        mean = (st.mean * st.n_samples_seen + mean_b * n_b) / n_tot
        unnorm = st.var * st.n_samples_seen + new_unnorm + \
            (st.n_samples_seen * n_b / n_tot) * (st.mean - mean_b) ** 2
    lam, Q = np.linalg.eigh(G)
    lam = lam[::-1][:c]
    Vt = Q[:, ::-1][:, :c].T
    Vt, _ = svd_flip_v(Vt)
    S = np.sqrt(np.maximum(lam, 0.0))
    st.components = Vt
    st.singular_values = S
    st.explained_variance = S ** 2 / (n_tot - 1)
    st.explained_variance_ratio = S ** 2 / np.sum(unnorm)
    st.mean = mean
    st.var = unnorm / n_tot
    st.n_samples_seen = n_tot
    return st


# --------------------------------------------------------------------------------------------
# decomposition.compute  (decomposition.py:150-358) for StyleGAN2 layer='style'
# --------------------------------------------------------------------------------------------
SEED_SAMPLING, SEED_RANDOM_DIRS, SEED_LINREG = 1, 2, 3   # decomposition.py:34-37


def plan(n: int, B: int, c: int):
    """decomposition.py:201,220,232:  N, NB, n_lat, number of partial_fit groups."""
    N = n // B * B
    NB = max(B, max(2000, 3 * c))
    n_lat = ((N + NB - 1) // B + 1) * B
    K = (N + NB - 1) // NB
    return N, NB, n_lat, K


def get_random_dirs(components: int, dimensions: int) -> np.ndarray:
    """decomposition.py:42-46."""
    gen = np.random.RandomState(seed=SEED_RANDOM_DIRS)
    dirs = gen.normal(size=(components, dimensions))
    dirs /= np.sqrt(np.sum(dirs ** 2, axis=1, keepdims=True))
    return dirs.astype(np.float32)


class _GlobalSeeds:
    """The module-level NumPy state the reference threads through sample_latent calls."""

    def __init__(self, seed0):
        self.seed0, self.i, self._cache = seed0, 0, np.empty(0, np.uint32)

    def next(self):
        if self.i >= len(self._cache):
            self._cache = seed_sequence(self.seed0, max(64, 2 * (self.i + 1)))
        s = int(self._cache[self.i])
        self.i += 1
        return s


def compute_path(sample, activate, latent_dims: int, feat_dims: int, n: int, B: int, c: int,
                 samples_are_latents: bool, seed=None, ipca: str = "svd", use_w: bool = False, return_aux=False,
                 regress: bool = True):
    """Restated decomposition.compute (:150-341) for estimator='ipca'.
        sample(seed, B)   -> one model.sample_latent(B) call (latents [B, latent_dims], float32)
        activate(latents) -> the hooked layer's activations flattened to [B, feat_dims]
    ``ipca``: 'svd' = sklearn-form partial_fit restatement, 'gram' = Gram-chain restatement (d x d), 'small' = small-side
    restatement (rows x rows; for d >> rows)."""
    d = feat_dims
    c = min(c, d)                                                    # :191
    N, NB, n_lat, K = plan(n, B, c)
    seeds = _GlobalSeeds(seed or SEED_SAMPLING)                      # :226-227

    # Phase A (:232-236): one sample_latent(B) per micro-batch
    latents = np.zeros((n_lat, latent_dims), np.float32)
    for i in range(n_lat // B):
        latents[i * B:(i + 1) * B] = sample(seeds.next(), B)

    # Phase B (:239-265)
    st = IPCAState(c)
    X = None
    for gi in range(0, N, NB):
        rows = latents[gi:gi + NB]
        X = (rows if samples_are_latents else activate(rows)).astype(np.float32).copy()
        if ipca == "svd":
            ipca_partial_fit(st, X)
        elif ipca == "small":
            ipca_partial_fit_small_side(st, X)
        else:
            ipca_gram_step(st, *batch_stats(X))

    X_global_mean = st.mean.reshape(1, d)                            # :289
    X = (X.astype(np.float64) - X_global_mean).astype(np.float32)    # :291 (float32 array -= float64)
    X_comp = np.array(st.components, dtype=np.float64, copy=True)
    X_stdev = np.sqrt(st.explained_variance)
    X_var_ratio = st.explained_variance_ratio

    if samples_are_latents:                                          # :297-299
        Z_comp, Z_mean = X_comp, X_global_mean
    elif not regress:                                                # (test shortcut: PCA half only, lat_* left as placeholders)
        Z_comp, Z_mean = np.ones((c, latent_dims)), np.zeros((1, latent_dims))
    else:                                                            # :301-305 -> linreg_lstsq :77-139
        Z_comp, Z_mean = linreg(sample, activate, latent_dims, X_comp, X_global_mean, X_stdev, n, B)
    Z_comp = Z_comp / np.linalg.norm(Z_comp, axis=-1, keepdims=True)  # :308
    if samples_are_latents:
        X_comp = Z_comp                                              # same ndarray in the reference

    random_dirs = get_random_dirs(c, d)                              # :312
    n_rand = min(5000, X.shape[0])
    X_stdev_random = np.dot(random_dirs, X[:n_rand].T).std(axis=1)   # :313-316

    lat_stdev = np.ones_like(X_stdev)                                # :325
    if use_w:                                                        # :326-329
        samples = sample(seeds.next(), 5000)
        coords = np.dot(Z_comp.reshape(-1, latent_dims), samples.T)
        lat_stdev = coords.std(axis=1)

    out = {                                                          # :331-341
        "act_comp": X_comp.reshape(-1, 1, d).astype(np.float32),
        "act_mean": X_global_mean.reshape(1, d).astype(np.float32),
        "act_stdev": X_stdev.astype(np.float32),
        "lat_comp": Z_comp.reshape(-1, 1, latent_dims).astype(np.float32),
        "lat_mean": np.asarray(Z_mean).reshape(1, latent_dims).astype(np.float32),
        "lat_stdev": lat_stdev.astype(np.float32),
        "var_ratio": X_var_ratio.astype(np.float32),
        "random_stdevs": X_stdev_random.astype(np.float32),
    }
    if return_aux:
        return out, dict(state=st, N=N, NB=NB, n_lat=n_lat, K=K)
    return out


def linreg(sample, activate, latent_dims, comp, mean, stdev, n: int, B: int):
    """decomposition.py:77-139: regress the latent on the scaled PC coordinates of the activations."""
    import scipy.linalg
    seeds = _GlobalSeeds(SEED_LINREG)                                # :80-81
    seeds.next()   # :88 get_latent_dims() -> get_latent_shape() -> sample_latent(1) eats one global draw
    comp32 = comp.astype(np.float32)
    mean32 = np.asarray(mean).astype(np.float32).reshape(1, -1)
    stdev32 = stdev.astype(np.float32)
    n_samp = max(10_000, n) // B * B                                 # :87
    A = np.zeros((n_samp, comp.shape[0]), np.float32)
    Z = np.zeros((n_samp, latent_dims), np.float32)
    for i in range(n_samp // B):                                     # :115-126
        z = sample(seeds.next(), B)
        act = activate(z) - mean32
        coords = act @ comp32.T
        A[i * B:(i + 1) * B] = coords / stdev32
        Z[i * B:(i + 1) * B] = z
    M_t = scipy.linalg.lstsq(A, Z, lapack_driver="gelsd")[0]        # :133
    return M_t[:comp.shape[0], :].astype(np.float64), np.mean(Z, axis=0, keepdims=True)


def compute_stylegan2_style(weights, biases, n: int, B: int, c: int, use_w: bool, seed=None,
                            ipca: str = "svd", return_aux: bool = False):
    """model=StyleGAN2, layer='style' (wrappers.py:167-179,194-222): W space (--use_w: sample_latent applies the
    mapping, samples are the latents) or Z space (activations = mapping(z), regression back to z)."""
    mapping = lambda z: mapping_forward(z, weights, biases)
    normals = lambda s, B_: standard_normal_f32(s, 512 * B_).reshape(B_, 512)
    if use_w:
        sample = lambda s, B_: mapping(normals(s, B_))
        return compute_path(sample, None, 512, 512, n, B, c, True, seed=seed, ipca=ipca, use_w=True,
                            return_aux=return_aux)
    return compute_path(normals, mapping, 512, 512, n, B, c, False, seed=seed, ipca=ipca, return_aux=return_aux)


# --------------------------------------------------------------------------------------------
# BigGAN generator.gen_z  (wrappers.py:562-569,611-648; biggan utils.py:21-33, model.py:51-52,211-212,291)
# --------------------------------------------------------------------------------------------
def truncated_noise_sample(seed: int, batch_size: int, dim_z: int = 128, truncation: float = 1.0) -> np.ndarray:
    """biggan utils.py:21-33: truncnorm.rvs(-2, 2, size, random_state=RandomState(seed)).astype(f32)*truncation.
    SciPy's truncnorm draws RandomState.uniform and applies the inverse CDF ndtri(Phi(a) + u (Phi(b)-Phi(a)))."""
    from scipy.special import ndtr, ndtri
    u = random_sample_f64(seed, batch_size * dim_z)
    pa, pb = ndtr(-2.0), ndtr(2.0)
    vals = ndtri(pa + u * (pb - pa)).astype(np.float32).reshape(batch_size, dim_z)
    return (np.float32(truncation) * vals).astype(np.float32)


def biggan_genz_random_init(seed: int = 4321, z_dim: int = 128, out_features: int = 4 * 4 * 16 * 128, eps: float = 1e-4):
    """Random-init tensors of the reference's BigGAN that gen_z depends on: torch.manual_seed(seed) followed
    by BigGAN(config) creates embeddings (nn.Linear(1000,128,bias=False)) and then
    generator.gen_z = spectral_norm(nn.Linear(256, 32768)) before anything else (biggan model.py:288-293,204-212)."""
    import torch
    from torch import nn
    torch.manual_seed(seed)
    emb = nn.Linear(1000, z_dim, bias=False)
    lin = nn.utils.spectral_norm(nn.Linear(2 * z_dim, out_features), eps=eps)
    w = lin.weight_orig.detach()
    sigma = torch.dot(lin.weight_u, torch.mv(w, lin.weight_v))      # eval mode: no power iteration
    return {"w_eff": (w / sigma).numpy(), "bias": lin.bias.detach().numpy(), "emb": emb.weight.detach().numpy(),
            "weight_orig": w.numpy(), "u": lin.weight_u.numpy(), "v": lin.weight_v.numpy()}


def genz_forward(z: np.ndarray, params, class_idx: int = 248) -> np.ndarray:
    """cond = cat(z, embeddings(one_hot)); act = gen_z(cond)  (wrappers.py:627-636), through torch's CPU F.linear."""
    import torch
    import torch.nn.functional as F
    with torch.no_grad():
        zt = torch.from_numpy(np.ascontiguousarray(z, dtype=np.float32))
        embed = torch.from_numpy(params["emb"][:, class_idx]).unsqueeze(0).expand(zt.shape[0], -1)
        cond = torch.cat((zt, embed), dim=1)
        return F.linear(cond, torch.from_numpy(params["w_eff"]), torch.from_numpy(params["bias"])).numpy()


def compute_biggan_genz(params, n: int, B: int, c: int, class_idx: int = 248, seed=None, ipca: str = "svd"):
    """model=BigGAN-512, layer='generator.gen_z' (BASELINE.json config 4)."""
    sample = lambda s, B_: truncated_noise_sample(s, B_)
    activate = lambda z: genz_forward(z, params, class_idx)
    return compute_path(sample, activate, 128, params["w_eff"].shape[0], n, B, c, False, seed=seed, ipca=ipca)


# --------------------------------------------------------------------------------------------
# comparison metric of BASELINE.json (sign-normalised cosine, explained-variance ratios)
# --------------------------------------------------------------------------------------------
def compare_npz(ours: dict, ref: dict) -> dict:
    a = np.asarray(ours["act_comp"], np.float64).reshape(ours["act_comp"].shape[0], -1)
    b = np.asarray(ref["act_comp"], np.float64).reshape(ref["act_comp"].shape[0], -1)
    cos = np.sum(a * b, axis=1) / (np.linalg.norm(a, axis=1) * np.linalg.norm(b, axis=1))
    la = np.asarray(ours["lat_comp"], np.float64).reshape(a.shape[0], -1)
    lb = np.asarray(ref["lat_comp"], np.float64).reshape(a.shape[0], -1)
    lcos = np.sum(la * lb, axis=1) / (np.linalg.norm(la, axis=1) * np.linalg.norm(lb, axis=1))

    def rel(k):
        x, y = np.asarray(ours[k], np.float64).ravel(), np.asarray(ref[k], np.float64).ravel()   # [1,C,H,W] vs [1,d] layouts
        return float(np.max(np.abs(x - y)) / max(np.max(np.abs(y)), 1e-30))

    return {
        "min_abs_cos": float(np.min(np.abs(cos))),
        "min_signed_cos": float(np.min(cos)),
        "min_lat_signed_cos": float(np.min(lcos)),
        "max_abs_dvar_ratio": float(np.max(np.abs(np.asarray(ours["var_ratio"], np.float64) -
                                                  np.asarray(ref["var_ratio"], np.float64)))),
        "act_mean_rel": rel("act_mean"), "act_stdev_rel": rel("act_stdev"),
        "lat_mean_rel": rel("lat_mean"), "lat_stdev_rel": rel("lat_stdev"),
        "random_stdevs_rel": rel("random_stdevs"),
    }


# --------------------------------------------------------------------------------------------
# StyleGAN2 synthesis up to a hooked StyledConv  (wrappers.py:194-259; stylegan2-pytorch/model.py:181-341)
# --------------------------------------------------------------------------------------------
STYLEGAN2_CHANNELS = {4: 512, 8: 512, 16: 512, 32: 512, 64: 512, 128: 256, 256: 128, 512: 64, 1024: 32}


def synthesis_layer_names(upto: str):
    """Hookable StyledConv layers in execution order up to ``upto`` ('conv1', 'convs.0', ...) (wrappers.py:224-255)."""
    names = ["conv1"]
    if upto != "conv1":
        k = int(upto.split(".")[1])
        names += [f"convs.{i}" for i in range(k + 1)]
    return names


def synthesis_random_init(seed: int = 1234, size: int = 1024, upto: str = "convs.4"):
    """Random-init synthesis tensors of ``Generator(size, 512, 8)`` under ``torch.manual_seed(seed)``, replaying the
    reference's parameter creation order (model.py:384-469): style (8 x randn(512,512)), input (randn(1,512,4,4) :298),
    conv1 [ModulatedConv2d weight randn(1,co,ci,3,3) :222-224, modulation EqualLinear randn(ci,512) bias 1 :226],
    to_rgb1 [weight randn(1,3,512,1,1), modulation], the ``noises`` buffers (:434-437), then per resolution
    convs[2j] (upsample), convs[2j+1], to_rgbs[j].  NoiseInjection.weight = 0 (:284), FusedLeakyReLU.bias = 0."""
    import math
    import torch
    g = torch.Generator().manual_seed(seed)
    rn = lambda *s: torch.randn(*s, generator=g)
    for _ in range(8):
        rn(512, 512)                                                  # mapping network (mapping_random_init)
    log_size = int(math.log(size, 2))
    ch = STYLEGAN2_CHANNELS
    const = rn(1, ch[4], 4, 4).numpy()[0]

    def styled(ci, co, upsample, res_out):
        w = rn(1, co, ci, 3, 3).numpy()[0]
        mw = rn(ci, 512).numpy()
        return dict(weight=w, mod_weight=mw, mod_bias=np.ones(ci, np.float32), noise_weight=np.float32(0.0),
                    act_bias=np.zeros(co, np.float32), upsample=upsample, res_out=res_out)

    def to_rgb(ci):
        # ToRGB (:344-363): ModulatedConv2d(ci, 3, 1, demodulate=False) weight randn(1,3,ci,1,1), modulation randn(ci,512) bias 1, bias 0
        w = rn(1, 3, ci, 1, 1).numpy()[0, :, :, 0, 0]
        mw = rn(ci, 512).numpy()
        rgbs.append(dict(weight=w, mod_weight=mw, mod_bias=np.ones(ci, np.float32), bias=np.zeros(3, np.float32)))

    rgbs = []
    layers = {"conv1": styled(ch[4], ch[4], False, 4)}
    to_rgb(ch[4])
    for layer_idx in range((log_size - 2) * 2 + 1):
        res = (layer_idx + 5) // 2
        rn(1, 1, 2 ** res, 2 ** res)
    wanted = synthesis_layer_names(upto)
    in_ch = ch[4]
    for i in range(3, log_size + 1):
        out_ch = ch[2 ** i]
        layers[f"convs.{2 * (i - 3)}"] = styled(in_ch, out_ch, True, 2 ** i)
        layers[f"convs.{2 * (i - 3) + 1}"] = styled(out_ch, out_ch, False, 2 ** i)
        to_rgb(out_ch)
        in_ch = out_ch
        if wanted[-1] in layers:
            break
    return dict(const=const, layers={k: layers[k] for k in wanted}, to_rgbs=rgbs)     # to_rgbs[0] = to_rgb1, [j + 1] = to_rgbs.j


def fixed_noise(seed: int = 0, size: int = 1024):
    """wrappers.py:261-267 set_noise_seed: torch.manual_seed(seed); randn(1,1,4,4); two maps per resolution 8..size."""
    import math
    import torch
    g = torch.Generator().manual_seed(seed)
    noise = [torch.randn(1, 1, 4, 4, generator=g).numpy()[0, 0]]
    for i in range(3, int(math.log(size, 2)) + 1):
        for _ in range(2):
            noise.append(torch.randn(1, 1, 2 ** i, 2 ** i, generator=g).numpy()[0, 0])
    return noise


BLUR_K2D = (np.outer([1, 3, 3, 1], [1, 3, 3, 1]).astype(np.float32) / np.float32(64.0)) * np.float32(4.0)   # model.py:47-57,81-84


def styled_conv_forward(x, w, L, noise):
    """One StyledConv exactly as the reference computes it on the CPU: per-sample modulated + demodulated weights,
    grouped conv / stride-2 transposed conv + upfirdn2d blur (model.py:232-277), NoiseInjection (:287-291),
    FusedLeakyReLU CPU fallback (fused_act.py:86-90).  x [B,ci,H,W], w [B,512] float32 -> [B,co,H',W']."""
    import math
    import torch
    import torch.nn.functional as F
    x = torch.from_numpy(np.ascontiguousarray(x, np.float32))
    w = torch.from_numpy(np.ascontiguousarray(w, np.float32))
    weight = torch.from_numpy(L["weight"])[None]                         # [1,co,ci,3,3]
    co, ci = weight.shape[1], weight.shape[2]
    B, _, H, W = x.shape
    mscale = 1 / math.sqrt(512)                                           # EqualLinear.scale, lr_mul = 1 (:143)
    style = F.linear(w, torch.from_numpy(L["mod_weight"]) * mscale, bias=torch.from_numpy(L["mod_bias"]) * 1.0)
    style = style.view(B, 1, ci, 1, 1)
    weight = (1 / math.sqrt(ci * 9)) * weight * style                    # :236
    demod = torch.rsqrt(weight.pow(2).sum([2, 3, 4]) + 1e-8)             # :239
    weight = weight * demod.view(B, co, 1, 1, 1)
    weight = weight.view(B * co, ci, 3, 3)
    if L["upsample"]:
        inp = x.reshape(1, B * ci, H, W)
        wt = weight.view(B, co, ci, 3, 3).transpose(1, 2).reshape(B * ci, co, 3, 3)
        out = F.conv_transpose2d(inp, wt, padding=0, stride=2, groups=B)   # :255
        out = out.view(B, co, 2 * H + 1, 2 * W + 1)
        # Blur(pad=(1,1), kernel*4) -> upfirdn2d_native: pad, true convolution (flipped kernel) (upfirdn2d.py:157-198)
        out = F.pad(out, [1, 1, 1, 1]).reshape(B * co, 1, 2 * H + 3, 2 * W + 3)
        kflip = torch.flip(torch.from_numpy(BLUR_K2D), [0, 1]).view(1, 1, 4, 4)
        out = F.conv2d(out, kflip).view(B, co, 2 * H, 2 * W)
    else:
        inp = x.reshape(1, B * ci, H, W)
        out = F.conv2d(inp, weight, padding=1, groups=B).view(B, co, H, W)   # :272
    out = out + torch.tensor(float(L["noise_weight"])) * torch.from_numpy(np.asarray(noise, np.float32))[None, None]
    out = (2 ** 0.5) * F.leaky_relu(out + torch.from_numpy(L["act_bias"]).view(1, -1, 1, 1), negative_slope=0.2)
    return out.numpy()


def styled_conv_shared(x, w, L, noise, dtype=np.float32):
    """styled_conv_forward with the per-sample weights factored out (identical algebra, used for bulk oracle runs: the
    reference form builds a [B,co,ci,3,3] weight tensor per call): scale the input channels by the style, convolve with
    the SHARED scale*W through the same torch CPU conv kernels, multiply by demod afterwards (the blur is linear and
    per-channel, so the demodulation commutes with it).  ``dtype``: the arithmetic's type (float64 for the per-layer parity
    references of tests/test_render_gpu.py)."""
    import math
    import torch
    import torch.nn.functional as F
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype))
    x, w = T(x), T(w)
    W = T(L["weight"]) * (1 / math.sqrt(L["weight"].shape[1] * 9))                               # [co,ci,3,3]
    B, ci, H, _ = x.shape
    style = F.linear(w, T(L["mod_weight"]) * (1 / math.sqrt(512)), bias=T(L["mod_bias"]))
    demod = torch.rsqrt((style * style) @ (W * W).sum([2, 3]).T + 1e-8)                       # [B,co]
    xs = x * style.view(B, ci, 1, 1)
    if L["upsample"]:
        out = F.conv_transpose2d(xs, W.transpose(0, 1), padding=0, stride=2)                   # [B,co,2H+1,2H+1]
        co = out.shape[1]
        out = F.pad(out, [1, 1, 1, 1]).reshape(B * co, 1, 2 * H + 3, 2 * H + 3)
        kflip = torch.flip(T(BLUR_K2D), [0, 1]).view(1, 1, 4, 4)
        out = F.conv2d(out, kflip).view(B, co, 2 * H, 2 * H)
    else:
        out = F.conv2d(xs, W, padding=1)
    out = out * demod.view(B, -1, 1, 1)
    out = out + torch.tensor(float(L["noise_weight"]), dtype=out.dtype) * T(noise)[None, None]
    out = (2 ** 0.5) * F.leaky_relu(out + T(L["act_bias"]).view(1, -1, 1, 1), negative_slope=0.2)
    return out.numpy()


def styled_conv_taps(x_nhwc, w, L, noise):
    """The same StyledConv in the form the CUDA path uses (numpy, float64 accumulation): scale the INPUT channels by
    the style, one dense contraction per 3x3 tap with the shared weights (Y[b,p,tap,co] = sum_ci W[co,ci,tap] xs[b,p,ci]),
    gather the nine tap planes (stride-1) or scatter them on the 2x grid and blur (upsample), multiply by
    demod[b,co] = rsqrt(sum_ci s^2 sum_k (scale W)^2 + 1e-8), add noise and bias, leaky-ReLU * sqrt2.
    x_nhwc [B,H,W,ci] -> [B,H',W',co].  Algebraically identical to styled_conv_forward."""
    x = np.asarray(x_nhwc, np.float64)
    B, H, W, ci = x.shape
    Wt = L["weight"].astype(np.float64) / np.sqrt(ci * 9.0)              # [co,ci,3,3]
    co = Wt.shape[0]
    s = np.asarray(w, np.float64) @ (L["mod_weight"].astype(np.float64) / np.sqrt(512.0)).T + L["mod_bias"]
    demod = 1.0 / np.sqrt((s * s) @ (Wt ** 2).sum(axis=(2, 3)).T + 1e-8)     # [B,co]
    xs = x * s[:, None, None, :]
    Y = np.einsum("bhwi,oikl->bhwklo", xs, Wt)                           # [B,H,W,ky,kx,co]
    if L["upsample"]:
        T = np.zeros((B, 2 * H + 1, 2 * W + 1, co))
        for ky in range(3):
            for kx in range(3):
                T[:, ky:ky + 2 * H:2, kx:kx + 2 * W:2, :] += Y[:, :, :, ky, kx, :]   # out_t[2y+ky, 2x+kx]
        Tp = np.pad(T, [(0, 0), (1, 1), (1, 1), (0, 0)])
        out = np.zeros((B, 2 * H, 2 * W, co))
        kb = BLUR_K2D.astype(np.float64)
        for i in range(4):
            for j in range(4):
                out += kb[i, j] * Tp[:, i:i + 2 * H, j:j + 2 * W, :]
    else:
        Yp = np.pad(Y, [(0, 0), (1, 1), (1, 1), (0, 0), (0, 0), (0, 0)])
        out = np.zeros((B, H, W, co))
        for ky in range(3):
            for kx in range(3):
                out += Yp[:, ky:ky + H, kx:kx + W, ky, kx, :]           # in[y+ky-1, x+kx-1]
    out = out * demod[:, None, None, :]
    out = out + float(L["noise_weight"]) * np.asarray(noise, np.float64)[None, :, :, None] + L["act_bias"].astype(np.float64)
    out = np.sqrt(2.0) * np.where(out >= 0, out, 0.2 * out)
    return out


def to_rgb_forward(x, w, R, skip=None, dtype=np.float32):
    """ToRGB (model.py:344-363): 1x1 modulated conv WITHOUT demodulation (ModulatedConv2d(ci, 3, 1, demodulate=False), scale
    1/sqrt(ci), :219-220,236), + bias, + Upsample(skip) (:33-51: upfirdn2d(skip, [1,3,3,1] outer / 16, up=2, pad=(2,1)),
    native form op/upfirdn2d.py:157-198: zero insertion, pad, true convolution).  x [B,ci,H,W], w [B,512] -> [B,3,H,W], in
    ``dtype`` arithmetic."""
    import math
    import torch
    import torch.nn.functional as F
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype))
    x, w = T(x), T(w)
    B, ci, H, W = x.shape
    style = F.linear(w, T(R["mod_weight"]) * (1 / math.sqrt(512)), bias=T(R["mod_bias"]))
    weight = (1 / math.sqrt(ci)) * T(R["weight"]).view(1, 3, ci, 1, 1) * style.view(B, 1, ci, 1, 1)
    out = F.conv2d(x.reshape(1, B * ci, H, W), weight.view(B * 3, ci, 1, 1), padding=0, groups=B).view(B, 3, H, W)
    out = out + T(R["bias"]).view(1, 3, 1, 1)
    if skip is not None:
        sk = T(skip)
        h = sk.shape[2]
        up = torch.zeros(B, 3, 2 * h, 2 * h, dtype=sk.dtype)
        up[:, :, ::2, ::2] = sk
        up = F.pad(up, [2, 1, 2, 1]).reshape(B * 3, 1, 2 * h + 3, 2 * h + 3)
        kflip = torch.flip(T(BLUR_K2D), [0, 1]).view(1, 1, 4, 4)
        out = out + F.conv2d(up, kflip).view(B, 3, 2 * h, 2 * h)
    return out.numpy()


def render_forward(w_layers, params, noises, form: str = "shared", keep=()):
    """Generator.forward (model.py:493-571) from per-layer W latents ``w_layers`` [B, n_latent, 512] (one global latent: the same
    row repeated, wrappers.py:202-205): conv1(latent 0) -> to_rgb1(latent 1); per resolution convs[2j](latent 2j+1),
    convs[2j+1](latent 2j+2), to_rgbs[j](latent 2j+3, skip).  ``params`` = synthesis_random_init(upto = the last StyledConv);
    returns (image = the last skip, before the wrapper's 0.5 (x + 1), and {name: activation} for the names in ``keep``)."""
    fn = {"reference": styled_conv_forward, "shared": styled_conv_shared}[form]
    names = list(params["layers"].keys())
    B = w_layers.shape[0]
    kept = {}
    x = np.repeat(params["const"][None], B, axis=0)
    x = fn(x, w_layers[:, 0], params["layers"]["conv1"], noises[0])
    if "conv1" in keep:
        kept["conv1"] = x
    skip = to_rgb_forward(x, w_layers[:, 1], params["to_rgbs"][0])
    if "to_rgb1" in keep:
        kept["to_rgb1"] = skip
    i = 1
    for j in range((len(names) - 1) // 2):
        for q in range(2):
            name = f"convs.{2 * j + q}"
            x = fn(x, w_layers[:, i + q], params["layers"][name], noises[i + q])
            if name in keep:
                kept[name] = x
        skip = to_rgb_forward(x, w_layers[:, i + 2], params["to_rgbs"][j + 1], skip)
        if f"to_rgbs.{j}" in keep:
            kept[f"to_rgbs.{j}"] = skip
        i += 2
    return skip, kept


def synthesis_forward(w, params, noises, upto: str, form: str = "reference"):
    """wrappers.py:224-255 for one global latent: input -> conv1(noise[0]) -> convs.0(noise[1]) -> convs.1(noise[2]) ...
    (every layer's style is the same w: latent[:, i] of the repeated [B,n_latent,512] tensor :202-205).
    Returns the hooked layer's activation [B,co,H,W] float32."""
    B = w.shape[0]
    x = np.repeat(params["const"][None], B, axis=0)                      # ConstantInput (:300-304)
    if form == "taps":
        x = x.transpose(0, 2, 3, 1)
    for idx, name in enumerate(synthesis_layer_names(upto)):
        L = params["layers"][name]
        fn = {"reference": styled_conv_forward, "shared": styled_conv_shared, "taps": styled_conv_taps}[form]
        x = fn(x, w, L, noises[idx])
    return x.transpose(0, 3, 1, 2) if form == "taps" else x


def compute_stylegan2_layer(weights, biases, params, layer: str, n: int, B: int, c: int, size: int = 1024, seed=None,
                            return_aux: bool = False, regress: bool = True, form: str = "shared"):
    """model=StyleGAN2, layer=conv1|convs.k, Z space (decomposition.py:150-341): activations = synthesis(mapping(z))
    flattened NCHW; IncrementalPCA in its sklearn (stacked-SVD) form; regression back to z."""
    noises = fixed_noise(0, size)
    normals = lambda s, B_: standard_normal_f32(s, 512 * B_).reshape(B_, 512)

    def activate(z):
        out = []
        for i in range(0, z.shape[0], 256):
            out.append(synthesis_forward(mapping_forward(z[i:i + 256], weights, biases), params, noises, layer, form=form))
        a = np.concatenate(out, axis=0)
        return a.reshape(a.shape[0], -1)

    L = params["layers"][layer]
    d = L["weight"].shape[0] * L["res_out"] ** 2
    return compute_path(normals, activate, 512, d, n, B, c, False, seed=seed, ipca="svd", return_aux=return_aux,
                        regress=regress)
