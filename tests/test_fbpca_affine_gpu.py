"""--est fbpca on BigGAN-512 generator.gen_z (BASELINE config 4's layer) on the device: parity with the fixtures the unmodified
reference wrote (oracle/gen_golden_fbpca_affine.py), with fbpca's literal algorithm in fp64 on the materialised activations,
the test-matrix projection, and a config-4-sized run against an fp64 restatement."""
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

COS_TOL = 0.999
RATIO_TOL = 1e-3
AUX_TOL = 1e-4

FIXTURES = [
    ("fbpca_d_biggan512_husky_genz_n32000_b1000_c16.npz", dict(n=32_000, c=16)),     # l = 32 < rank: randomized branch
    ("fbpca_e_biggan512_husky_genz_n4000_b1000_c80.npz", dict(n=4_000, c=80)),       # l = 160 >= rank: exact branch
]


@pytest.fixture(scope="module")
def model():
    from ganspace_b200.models.biggan import BigGAN
    return BigGAN(torch.device("cuda:0"), 512, "husky", random_init=4321)


@pytest.fixture(scope="module")
def fao():
    from oracle import fbpca_affine_oracle
    return fbpca_affine_oracle


def _run(model, n, b, c):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model
    inst = get_instrumented_model("BigGAN-512", "husky", "generator.gen_z", torch.device("cuda:0"), model=model)
    cfg = Config(model="BigGAN-512", layer="generator.gen_z", output_class="husky", components=c, n=n, batch_size=b,
                 estimator="fbpca")
    with tempfile.TemporaryDirectory() as tmp:
        path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        with np.load(path) as data:
            out = {k: data[k] for k in data.files}
    inst.close()
    return out, path.name


@pytest.mark.parametrize("name,kw", FIXTURES)
def test_get_or_compute_vs_reference_golden(model, golden, oracle, fao, name, kw):
    from oracle import fbpca_oracle as fbo
    g = fao.decode_span(golden(name), oracle.biggan_genz_random_init(4321))      # act_comp / act_mean rebuilt from the span
    out, fname = _run(model, kw["n"], 1_000, kw["c"])
    assert fname == str(g["dump_name"])
    for k in g:
        if k != "dump_name":
            assert out[k].shape == g[k].shape and out[k].dtype == np.float32, k
    assert np.array_equal(fbo.sign_normalise(out)["act_comp"], out["act_comp"])
    cmp = oracle.compare_npz(out, fbo.sign_normalise(g))
    assert cmp["min_signed_cos"] >= COS_TOL and cmp["min_lat_signed_cos"] >= COS_TOL, cmp
    assert cmp["max_abs_dvar_ratio"] <= RATIO_TOL, cmp
    for k in ("act_mean_rel", "act_stdev_rel", "random_stdevs_rel", "lat_mean_rel"):
        assert cmp[k] < AUX_TOL, (k, cmp)
    assert np.array_equal(out["lat_stdev"], np.ones(kw["c"], np.float32))


@pytest.mark.parametrize("c", [16, 80])
def test_get_or_compute_vs_fp64_literal_fbpca(model, oracle, fao, c):
    """N = 4000 against fbpca's literal algorithm in fp64 on the stacked [6000, 32768] activations.  c = 80 is the exact
    branch; c = 16 (l = 32 < rank with fewer samples than features: fbpca's wide branch) is refused."""
    from oracle import fbpca_oracle as fbo
    if c == 16:
        with pytest.raises(NotImplementedError, match="needs N \\+ NB >= 32768"):
            _run(model, 4_000, 1_000, 16)
        return
    ref = fao.compute_genz_literal(oracle.biggan_genz_random_init(4321), 4_000, 1_000, c)
    out, _ = _run(model, 4_000, 1_000, c)
    cmp = oracle.compare_npz(out, fbo.sign_normalise(ref))
    assert cmp["min_signed_cos"] >= 1 - 1e-5 and cmp["min_lat_signed_cos"] >= 1 - 1e-4, cmp
    assert cmp["max_abs_dvar_ratio"] <= 1e-6, cmp
    for k in ("act_stdev_rel", "random_stdevs_rel", "lat_mean_rel"):
        assert cmp[k] < 1e-5, (k, cmp)
    assert cmp["act_mean_rel"] < 5e-5, cmp          # the reference's mean is a float32 sum over 6000 rows


@pytest.mark.parametrize("d,r,l", [(32768, 256, 32), (32768, 256, 128), (1000, 40, 7)])
def test_project_omega_equals_qt_omega(d, r, l):
    from ganspace_b200 import _native
    rng = np.random.RandomState(d + r + l)
    Q = np.linalg.qr(rng.standard_normal((d, r)))[0]
    om = rng.uniform(-1, 1, (d, l)).astype(np.float32)
    dev = torch.device("cuda:0")
    got = _native.fbpca_project_omega(torch.from_numpy(Q).to(dev), torch.from_numpy(om).to(dev)).cpu().numpy()
    want = Q.T @ om.astype(np.float64)
    assert got.shape == (r, l) and np.max(np.abs(got - want)) <= 1e-12 * np.max(np.abs(want))


def test_config4_shape_n1e6_c80(model):
    """N = 10^6, B = 10^4, c = 80: finite, orthonormal components equal to the exact top-80 PCA of the stacked matrix, restated
    in fp64 in an orthonormal basis of span(W_z, offset) taken independently of the layer's own factorisation."""
    from ganspace_b200 import plan
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import compute_arrays, _draw_seeds
    from ganspace_b200.models import get_instrumented_model
    n, b, c = 1_000_000, 10_000, 80
    inst = get_instrumented_model("BigGAN-512", "husky", "generator.gen_z", torch.device("cuda:0"), model=model)
    cfg = Config(model="BigGAN-512", layer="generator.gen_z", output_class="husky", components=c, n=n, batch_size=b,
                 estimator="fbpca")
    out = compute_arrays(cfg, inst)
    inst.close()
    A = out["act_comp"].reshape(c, -1).astype(np.float64)
    assert np.all(np.isfinite(A)) and np.all(np.isfinite(out["lat_comp"]))
    assert np.max(np.abs(A @ A.T - np.eye(c))) < 1e-5

    pl = plan.make_plan(n, b, c)
    np.random.seed(1)
    seeds = _draw_seeds(pl.n_calls)
    z = model.sample_latents_multi(b, seeds)[:pl.K * pl.NB].double()
    gz = model.model.generator.gen_z
    w = gz.effective_weight().double()
    o = gz.bias.detach().double() + w[:, 128:] @ model._embed().double()
    basis, _ = torch.linalg.qr(torch.cat([w[:, :128], o[:, None]], dim=1))
    u = z @ (basis.T @ w[:, :128]).T + basis.T @ o                  # coordinates of the activation rows
    m = pl.N + pl.NB
    mean = u.sum(0) / m                                                # zero rows: pl.N + pl.NB - K NB of them
    S = (u - mean).T @ (u - mean) + (m - u.shape[0]) * torch.outer(mean, mean)
    lam, V = torch.linalg.eigh(S)
    V = (basis @ V[:, -c:].flip(1)).T.cpu().numpy()
    lam = lam[-c:].flip(0).cpu().numpy()
    cos = np.abs(np.sum(A * V, axis=1))
    assert cos.min() >= 1 - 1e-5, cos.min()
    assert np.allclose(out["var_ratio"], lam / float(torch.trace(S)), rtol=1e-5)
    assert np.allclose(out["act_stdev"], np.sqrt(lam / m), rtol=1e-5)
