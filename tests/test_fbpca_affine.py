"""--est fbpca on a layer that is affine in the latent, host side: the fp64 literal-fbpca oracle against the fixtures the
unmodified reference wrote on BigGAN-512 generator.gen_z (oracle/gen_golden_fbpca_affine.py), the low-rank formulation the
device solves (DESIGN.md section 5g) against fbpca's literal algorithm on the full-width matrix, and the driver on the CPU
stand-ins of the device layer, single process and on two gloo ranks."""
import os
import socket
import sys
from pathlib import Path

import numpy as np
import pytest
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

ROOT = Path(__file__).resolve().parents[1]


@pytest.fixture(scope="module")
def fao():
    from oracle import fbpca_affine_oracle
    return fbpca_affine_oracle


def test_oracle_matches_reference_golden_exact_branch(golden, oracle, fao):
    """c = 80, N = 4000: the reference took fbpca's wide branch with l = 160 >= rank 129; the fp64 literal restatement
    (same branch, same draws) reproduces it."""
    params = oracle.biggan_genz_random_init(4321)
    g = fao.decode_span(golden("fbpca_e_biggan512_husky_genz_n4000_b1000_c80.npz"), params)
    ref = fao.compute_genz_literal(params, 4_000, 1_000, 80)
    cmp = oracle.compare_npz(ref, g)
    assert cmp["min_abs_cos"] >= 0.9999 and cmp["max_abs_dvar_ratio"] <= 1e-6, cmp
    for k in ("act_mean_rel", "act_stdev_rel", "random_stdevs_rel", "lat_mean_rel"):
        assert cmp[k] < 1e-4, (k, cmp)


def test_shortcut_matches_reference_golden_randomized_branch(golden, oracle, fao):
    """c = 16, N = 32000 (fbpca's tall branch, l = 32 < rank): the fp64 coordinate-space solve with the reference's test
    matrix (the draw after the sampling seeds) reproduces the reference's components, stdevs and ratios."""
    p = oracle.biggan_genz_random_init(4321)
    g = fao.decode_span(golden("fbpca_d_biggan512_husky_genz_n32000_b1000_c16.npz"), p)
    n, B, c = 32_000, 1_000, 16
    N, NB, n_lat, K = oracle.plan(n, B, c)
    np.random.seed(1)
    seeds = [int(np.random.randint(2147483647)) for _ in range(n_lat // B)]
    omega = np.random.uniform(-1.0, 1.0, (32768, 2 * c)).astype(np.float32)
    z = np.concatenate([oracle.truncated_noise_sample(s, B) for s in seeds])[:K * NB].astype(np.float64)
    w = p["w_eff"].astype(np.float64)
    o = p["bias"].astype(np.float64) + w[:, 128:] @ p["emb"][:, 248].astype(np.float64)
    Q, R = np.linalg.qr(w[:, :128])
    Qt, t = fao.linear_form(Q, o)
    comp, stdev, ratio, mean = fao.lifted_solve(z @ R.T, N + NB - K * NB, Qt, t, omega, c)
    gc = g["act_comp"].reshape(c, -1).astype(np.float64)
    assert np.abs(np.sum(comp * gc, axis=1)).min() >= 0.999
    assert np.max(np.abs(ratio - g["var_ratio"])) <= 1e-4
    assert np.allclose(stdev, g["act_stdev"], rtol=1e-3)
    assert np.max(np.abs(mean - g["act_mean"].ravel())) < 1e-4 * np.max(np.abs(g["act_mean"]))


@pytest.mark.parametrize("name", ["fbpca_d_biggan512_husky_genz_n32000_b1000_c16.npz",
                                  "fbpca_e_biggan512_husky_genz_n4000_b1000_c80.npz"])
def test_compact_fixtures_rebuild_the_reference_arrays(golden, oracle, fao, name):
    """act_comp / act_mean are stored as coefficients over gen_z's [W_z, offset]; the reference's rows lie in that span up to
    float32 rounding, and the rebuilt rows are unit-norm and mutually orthogonal like fbpca's."""
    g = golden(name)
    assert g["act_comp_resid"].max() < 1e-5 and g["act_mean_resid"].max() < 1e-5
    out = fao.decode_span(g, oracle.biggan_genz_random_init(4321))
    assert set(out) == {"dump_name", "act_comp", "act_mean", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio",
                        "random_stdevs"}
    c = out["act_stdev"].shape[0]
    assert out["act_comp"].shape == (c, 1, 32768) and out["act_mean"].shape == (1, 32768)
    A = out["act_comp"].reshape(c, -1).astype(np.float64)
    assert np.max(np.abs(A @ A.T - np.eye(c))) < 1e-4


@pytest.mark.parametrize("c", [5, 6, 7, 8, 10])
def test_lifted_solve_equals_literal_fbpca(fao, c):
    """Rows y Q^T + offset (rank r = 11 in D = 96) followed by zero rows: the centred matrix has rank r + 1 = 12.  l = 2c = 10
    is below it (randomized), 12 is equal and 14, 16, 20 above it (exact)."""
    rng = np.random.RandomState(c)
    D, r, m_data, n_zero = 96, 11, 300, 100
    Q = np.linalg.qr(rng.standard_normal((D, r)))[0]
    offset = 3.0 * rng.standard_normal(D)
    Y = rng.standard_normal((m_data, r)) * (0.8 ** np.arange(r))[None, :] * 4.0
    A = np.concatenate([Y @ Q.T + offset, np.zeros((n_zero, D))])
    X = A - A.mean(0)
    assert np.linalg.matrix_rank(X) == r + 1
    np.random.seed(7)
    Va, stdev, ratio = fao.fit_literal(X, c)
    np.random.seed(7)
    omega = np.random.uniform(-1.0, 1.0, (D, 2 * c))
    Qt, t = fao.linear_form(Q, offset)
    comp, st, ra, mean = fao.lifted_solve(Y, n_zero, Qt, t, omega if 2 * c < r + 1 else None, c)
    assert np.abs(np.sum(comp * Va, axis=1)).min() >= 1 - 1e-9
    assert np.allclose(st, stdev, rtol=1e-9) and np.allclose(ra, ratio, rtol=1e-9)
    assert np.allclose(mean, A.mean(0), atol=1e-12)


def test_lifted_solve_without_the_offset_direction_differs(fao):
    """Pooling the plain r-coordinates (a zero row read as y = 0, i.e. act = offset) is not fbpca on the stacked matrix."""
    rng = np.random.RandomState(3)
    D, r, m_data, n_zero, c = 96, 11, 300, 100, 8
    Q = np.linalg.qr(rng.standard_normal((D, r)))[0]
    offset = 3.0 * rng.standard_normal(D)
    Y = rng.standard_normal((m_data, r)) * 2.0
    A = np.concatenate([Y @ Q.T + offset, np.zeros((n_zero, D))])
    _, stdev, ratio = fao.fit_literal(A - A.mean(0), c)
    Yz = np.concatenate([Y, np.zeros((n_zero, r))])
    S = (Yz - Yz.mean(0)).T @ (Yz - Yz.mean(0))
    lam = np.linalg.eigvalsh(S)[::-1][:c]
    assert not np.allclose(np.sqrt(lam / len(Yz)), stdev, rtol=1e-3)


# ---- the driver on CPU stand-ins of the device layer ---------------------------------------------------------------------
N, B, LAT, D = 4000, 500, 24, 512


class FakeFBPCAPool:
    """Interface of _native.FBPCAPool: Chan-pooled (n, mean, scatter) and the Gram-form solve of oracle/fbpca_oracle.py."""

    def __init__(self, d, device):
        self.d, self.n = int(d), 0
        self.mean, self.S = np.zeros(self.d), np.zeros((self.d, self.d))

    def _fold(self, nb, mg, Cg):
        nn = self.n + nb
        dm = mg - self.mean
        self.S = self.S + Cg + (self.n * nb / nn) * np.outer(dm, dm)
        self.mean = self.mean + dm * (nb / nn)
        self.n = nn

    def accumulate(self, rows_per_group, means, grams):
        means = means.reshape(-1, self.d).numpy()
        grams = grams.reshape(-1, self.d, self.d).numpy()
        for g in range(means.shape[0]):
            self._fold(int(rows_per_group), means[g], grams[g])

    def add_zero_rows(self, n_zero):
        if n_zero > 0:
            self._fold(int(n_zero), np.zeros(self.d), np.zeros((self.d, self.d)))

    def solve(self, c, l, omega=None, raw=False):
        from oracle import fbpca_oracle as fbo
        assert not raw and (omega is None or omega.shape == (self.d, l))
        Va, _ = fbo.gram_solve(self.S, None if omega is None else omega.numpy(), c)
        q = np.einsum("kd,de,ke->k", Va, self.S, Va)
        idx = np.argsort(q)[::-1]
        Va = fbo.orc.svd_flip_v(Va[idx])[0]
        t = lambda a: torch.from_numpy(np.ascontiguousarray(a, np.float64))
        return {"components": t(Va), "stdev": t(np.sqrt(q[idx] / self.n)), "var_ratio": t(q[idx] / np.trace(self.S)),
                "mean": t(self.mean)}


def _fake_linear(x, w, bias=None, lrelu=False, bounded=False):
    y = x.float() @ w.float().T
    return y + bias.float() if bias is not None else y


def _run_driver(c):
    sys.path.insert(0, str(ROOT / "tests"))
    sys.path.insert(0, str(ROOT))
    import fakes
    from ganspace_b200 import _native, decomposition, estimators
    from ganspace_b200.config import Config
    from ganspace_b200.models.biggan import AffineLayer
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    fakes.install(_native, estimators)
    _native.FBPCAPool = FakeFBPCAPool
    _native.linear = _fake_linear
    _native.fbpca_project_omega = lambda Q, om: Q.T @ om.double()

    class FakeAffineModel(fakes.FakeFeatureModel):
        """Layer 'feat' = z W^T + o: affine in the latent, exposed through affine_layer like BigGAN's gen_z."""

        def __init__(self):
            super().__init__(C=1, H=1, W=D, latent=LAT, seed=13)
            g = torch.Generator().manual_seed(14)
            self.Wm = torch.randn(D, LAT, generator=g, dtype=torch.float64) * (0.85 ** torch.arange(LAT))[None, :]
            self.o = 2.0 * torch.randn(D, generator=g, dtype=torch.float64)

        def act_nchw_flat(self, z):
            return (z.reshape(-1, LAT).double() @ self.Wm.T + self.o).float()

        def feature_layout(self, layer_name):
            return None

        def affine_layer(self, layer_name):
            Q, R = torch.linalg.qr(self.Wm)
            return AffineLayer(Q, R, self.o.clone())

    model = FakeAffineModel()
    inst = InstrumentedModel(model)
    inst.retain_layer("feat")
    cfg = Config(model="Fake", layer="feat", output_class="none", components=c, n=N, batch_size=B, use_w=False,
                 estimator="fbpca")
    return decomposition.compute_arrays(cfg, inst), model


def _expected(oracle, model, c):
    from oracle import fbpca_oracle as fbo
    sample = lambda seed, b: np.random.RandomState(seed).standard_normal(LAT * b).reshape(b, LAT).astype(np.float32)
    activate = lambda z: model.act_nchw_flat(torch.from_numpy(np.ascontiguousarray(z, np.float32))).numpy()
    return fbo.sign_normalise(fbo.compute_path_fbpca(sample, activate, LAT, D, N, B, c, False, form="literal"))


_PATCHED = ("BigIPCA", "IPCAChain", "batch_stats", "batch_stats_multi", "LinregAccumulator", "project_std", "require_cuda",
            "FBPCAPool", "linear", "fbpca_project_omega")


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_path, c):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    out, _ = _run_driver(c)
    if rank == 0:
        np.savez(out_path, **out)
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.parametrize("c", [6, 16])
def test_driver_one_and_two_ranks(oracle, monkeypatch, tmp_path, c):
    """c = 6: l = 12 < rank 25 (randomized, Omega projected); c = 16: l = 32 >= 25 (exact).  Against the reference's path
    restated with fbpca's literal algorithm on the stacked [6000, 512] matrix; two gloo ranks give the same arrays."""
    from ganspace_b200 import _native
    for name in _PATCHED:
        monkeypatch.setattr(_native, name, getattr(_native, name))
    out, model = _run_driver(c)
    cmp = oracle.compare_npz(out, _expected(oracle, model, c))
    assert cmp["min_signed_cos"] > 1 - 1e-4 and cmp["min_lat_signed_cos"] > 1 - 1e-4 and cmp["max_abs_dvar_ratio"] < 1e-5, cmp
    for k in ("act_mean_rel", "act_stdev_rel", "random_stdevs_rel", "lat_mean_rel"):
        assert cmp[k] < 1e-4, (k, cmp)
    out_path = str(tmp_path / "two.npz")
    mp.spawn(_worker, args=(2, _free_port(), out_path, c), nprocs=2, join=True)
    with np.load(out_path) as data:
        for k in data.files:
            if k == "lat_comp":                            # the regression's all-reduce sums in another order
                a, b = out[k].reshape(c, -1).astype(np.float64), data[k].reshape(c, -1).astype(np.float64)
                assert np.sum(a * b, axis=1).min() >= 1 - 1e-6
            else:
                assert np.array_equal(out[k], data[k]), k
