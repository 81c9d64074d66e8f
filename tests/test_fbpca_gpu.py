"""--est fbpca on the device (csrc/rsvd.cu through estimators.FacebookPCAEstimator and decomposition.compute): parity with the
fixtures the unmodified reference wrote (oracle/gen_golden_fbpca.py), the device solve against the oracle's fp64 Gram form,
the rank check, determinism, Ctrl-C and the 2-GPU run."""
import os
import socket
import sys
import tempfile
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
ROOT = Path(__file__).resolve().parents[1]

COS_TOL = 0.999
RATIO_TOL = 1e-3
AUX_TOL = 1e-4        # as tests/test_e2e_gpu.py

FIXTURES = [
    ("fbpca_a_stylegan2_ffhq_style_w_n10000_b1000_c32.npz", dict(n=10_000, b=1_000, c=32, use_w=True)),
    ("fbpca_b_stylegan2_ffhq_style_z_n5000_b500_c16.npz", dict(n=5_000, b=500, c=16, use_w=False)),
    ("fbpca_c_stylegan2_ffhq_style_w_n4000_b1000_c210.npz", dict(n=4_000, b=1_000, c=210, use_w=True)),
]


@pytest.fixture(scope="module")
def fbo():
    from oracle import fbpca_oracle
    return fbpca_oracle


def _run(n, b, c, use_w, tmp=None, layer="style"):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model, StyleGAN2
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=model, use_w=use_w)
    cfg = Config(model="StyleGAN2", layer=layer, output_class="ffhq", components=c, n=n, batch_size=b, use_w=use_w,
                 estimator="fbpca")
    with tempfile.TemporaryDirectory() as t:
        tmp = tmp or t
        path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        with np.load(path, allow_pickle=False) as data:
            out = {k: data[k] for k in data.files}
    inst.close()
    return out, path.name


def _check(cmp):
    assert cmp["min_signed_cos"] >= COS_TOL and cmp["min_lat_signed_cos"] >= COS_TOL, cmp
    assert cmp["max_abs_dvar_ratio"] <= RATIO_TOL, cmp
    assert cmp["act_mean_rel"] < AUX_TOL and cmp["act_stdev_rel"] < AUX_TOL, cmp
    assert cmp["lat_stdev_rel"] < AUX_TOL and cmp["random_stdevs_rel"] < AUX_TOL, cmp


@pytest.mark.parametrize("name,kw", FIXTURES)
def test_get_or_compute_vs_reference_golden(golden, oracle, fbo, name, kw):
    g = golden(name)
    out, fname = _run(kw["n"], kw["b"], kw["c"], kw["use_w"])
    assert fname == str(g["dump_name"])
    for k in g:
        if k != "dump_name":
            assert out[k].shape == g[k].shape and out[k].dtype == np.float32, k
    # the device applies the sign rule already; the reference's signs are LAPACK's
    assert np.array_equal(fbo.sign_normalise(out)["act_comp"], out["act_comp"])
    cmp = oracle.compare_npz(out, fbo.sign_normalise(g))
    _check(cmp)
    if not kw["use_w"]:
        assert cmp["lat_mean_rel"] < AUX_TOL, cmp
        assert np.array_equal(out["lat_stdev"], np.ones(kw["c"], np.float32))


def test_two_runs_are_bit_identical():
    a, _ = _run(10_000, 1_000, 32, True)
    b, _ = _run(10_000, 1_000, 32, True)
    for k in a:
        assert np.array_equal(a[k], b[k]), k


def _spectrum(kind, d):
    if kind == "power":
        return (1.0 + np.arange(d)) ** -1.0
    if kind == "clustered":
        return np.concatenate([np.linspace(10, 9, 8), np.linspace(5, 4.5, 8), 0.5 * 0.95 ** np.arange(d - 16)])
    return 0.97 ** np.arange(d)


@pytest.mark.parametrize("kind,d,c,m", [("power", 512, 32, 40_000), ("clustered", 256, 24, 20_000), ("exact", 128, 60, 8_000)])
def test_device_solve_vs_oracle_gram_form(fbo, kind, d, c, m):
    """Pooled statistics of 4 groups (fp64, uploaded), then the solve, against the oracle's Gram form on the whole matrix."""
    from ganspace_b200 import _native
    rng = np.random.RandomState(17)
    basis, _ = np.linalg.qr(rng.standard_normal((d, d)))
    X = (rng.standard_normal((m, d)) * _spectrum(kind, d)[None, :]) @ basis.T + rng.standard_normal(d)
    groups = np.split(X, 4)
    means = np.stack([g.mean(0) for g in groups])
    grams = np.stack([(g - g.mean(0)).T @ (g - g.mean(0)) for g in groups])
    dev = torch.device("cuda:0")
    pool = _native.FBPCAPool(d, dev)
    pool.accumulate(m // 4, torch.from_numpy(means[:1]).to(dev), torch.from_numpy(grams[:1]).to(dev))
    pool.accumulate(m // 4, torch.from_numpy(means[1:]).to(dev), torch.from_numpy(grams[1:]).to(dev))
    pool.add_zero_rows(1000)
    Xz = np.concatenate([X, np.zeros((1000, d))])
    mean = Xz.mean(0)
    S = (Xz - mean).T @ (Xz - mean)
    randomized = fbo.randomized(c, m + 1000, d)
    assert randomized == (kind != "exact")
    omega = rng.uniform(-1.0, 1.0, (d, 2 * c)) if randomized else None
    out = pool.solve(c, 2 * c, omega=torch.from_numpy(omega) if randomized else None)
    Va, _ = fbo.gram_solve(S, omega, c)
    q = np.einsum("kd,de,ke->k", Va, S, Va)
    order = np.argsort(q)[::-1]
    Va, q = fbo.orc.svd_flip_v(Va[order])[0], q[order]
    comp = out["components"].cpu().numpy()
    cos = np.sum(comp * Va, axis=1)
    assert cos.min() >= 1 - 1e-9, cos.min()
    assert np.allclose(out["stdev"].cpu().numpy(), np.sqrt(q / (m + 1000)), rtol=1e-9)
    assert np.allclose(out["var_ratio"].cpu().numpy(), q / np.trace(S), rtol=1e-9)
    assert np.allclose(out["mean"].cpu().numpy(), mean, rtol=1e-12, atol=1e-12)


def test_fit_on_raw_rows_vs_fbpca_restatement(fbo):
    """FacebookPCAEstimator.fit (raw=True: uncentred X^T X) on a host ndarray against the restated fbpca.pca, same Omega."""
    from ganspace_b200.estimators import FacebookPCAEstimator
    rng = np.random.RandomState(3)
    d, m, c = 256, 6_000, 16
    X = ((rng.standard_normal((m, d)) * (0.95 ** np.arange(d))[None, :]) + 0.5).astype(np.float32)
    est = FacebookPCAEstimator(c)
    np.random.seed(9)
    est.fit(X)
    comp, stdev, ratio = est.get_components()
    np.random.seed(9)
    _, _, Va = fbo.pca(X.astype(np.float64), k=c, n_iter=2, raw=True, l=2 * c)
    Va = Va.copy()
    st = np.dot(Va, X.T.astype(np.float64)).std(axis=1)
    order = np.argsort(st)[::-1]
    Va = fbo.orc.svd_flip_v(Va[order])[0]
    assert np.sum(comp * Va, axis=1).min() >= 1 - 1e-6
    assert np.allclose(stdev, st[order], rtol=1e-5)
    assert np.allclose(ratio, st[order] ** 2 / X.astype(np.float64).var(0).sum(), rtol=1e-5)
    assert np.allclose(est.transformer.mean_, X.astype(np.float64).mean(0, keepdims=True), atol=1e-6)


def test_rank_deficient_samples_raise():
    from ganspace_b200 import _native
    from ganspace_b200.estimators import FacebookPCAEstimator
    rng = np.random.RandomState(4)
    X = (rng.standard_normal((5_000, 10)) @ rng.standard_normal((10, 128))).astype(np.float32)    # rank 10 < l = 16
    with pytest.raises(_native.FBPCARankError, match="numerical rank below l = 16"):
        FacebookPCAEstimator(8).fit(X)
    # the pool's status word is cleared: a well-posed solve afterwards succeeds
    est = FacebookPCAEstimator(4)
    est.fit(X)
    assert np.all(np.isfinite(est.get_components()[0]))


def test_keyboard_interrupt_exits_without_a_file(monkeypatch):
    """Ctrl-C while collecting: the reference exits with status 1 and writes nothing (decomposition.py:268-270)."""
    from ganspace_b200 import estimators
    calls = {"n": 0}
    orig = estimators.FacebookPCAEstimator.fit_partial_stats

    def interrupting(self, *a):
        calls["n"] += 1
        if calls["n"] == 2:
            raise KeyboardInterrupt
        return orig(self, *a)

    monkeypatch.setattr(estimators.FacebookPCAEstimator, "fit_partial_stats", interrupting)
    with tempfile.TemporaryDirectory() as tmp:
        with pytest.raises(SystemExit) as ex:
            _run(10_000, 1_000, 32, True, tmp=tmp)
        assert ex.value.code == 1
        assert not list(Path(tmp).rglob("*.npz"))


def test_conv_feature_maps_are_not_available():
    with pytest.raises(NotImplementedError, match="conv feature maps"):
        _run(4_000, 500, 8, False, layer="convs.1")


def _free_port():
    with socket.socket() as s:
        s.bind(("127.0.0.1", 0))
        return s.getsockname()[1]


def _worker(rank, world, port, out_path):
    sys.path.insert(0, str(ROOT))
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port))
    import torch.distributed as dist
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world)
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import StyleGAN2, get_instrumented_model
    dev = torch.device("cuda", rank)
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    inst = get_instrumented_model("StyleGAN2", "ffhq", "style", dev, model=model, use_w=False)
    cfg = Config(model="StyleGAN2", layer="style", output_class="ffhq", components=16, n=5_000, batch_size=500,
                 use_w=False, estimator="fbpca")
    with tempfile.TemporaryDirectory() as tmp:
        path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        if rank == 0:
            with np.load(path) as data:
                np.savez(out_path, **{k: data[k] for k in data.files})
    dist.barrier()
    dist.destroy_process_group()


@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_two_gpus_equal_one_gpu(tmp_path):
    import torch.multiprocessing as mp
    out_path = str(tmp_path / "two_gpu.npz")
    mp.spawn(_worker, args=(2, _free_port(), out_path), nprocs=2, join=True)
    with np.load(out_path) as data:
        two = {k: data[k] for k in data.files}
    one, _ = _run(5_000, 500, 16, False)
    for k in ("act_comp", "act_mean", "act_stdev", "var_ratio", "random_stdevs"):
        assert np.array_equal(one[k], two[k]), k
    a, b = one["lat_comp"].reshape(16, -1).astype(np.float64), two["lat_comp"].reshape(16, -1).astype(np.float64)
    assert np.sum(a * b, axis=1).min() >= 1 - 1e-6          # the regression's all-reduce sums in another order
