"""--est fbpca on the host side: the oracle's Gram-form solve against its restatement of fbpca.pca, the oracle's
compute path against the fixtures the unmodified reference wrote (oracle/gen_golden_fbpca.py), fbpca's test-matrix draw
from the global NumPy state, and the estimator's surface and cache name."""
import numpy as np
import pytest

FIXTURES = [
    ("fbpca_a_stylegan2_ffhq_style_w_n10000_b1000_c32.npz", dict(n=10_000, B=1_000, c=32, use_w=True)),
    ("fbpca_b_stylegan2_ffhq_style_z_n5000_b500_c16.npz", dict(n=5_000, B=500, c=16, use_w=False)),
    ("fbpca_c_stylegan2_ffhq_style_w_n4000_b1000_c210.npz", dict(n=4_000, B=1_000, c=210, use_w=True)),
]


@pytest.fixture(scope="module")
def fbo():
    from oracle import fbpca_oracle
    return fbpca_oracle


def _synthetic(rng, m, d, decay):
    basis, _ = np.linalg.qr(rng.standard_normal((d, d)))
    return (rng.standard_normal((m, d)) * decay[None, :]) @ basis.T


@pytest.mark.parametrize("m,d,k,kind", [(3000, 64, 8, "power"), (4000, 96, 12, "clustered"), (500, 64, 30, "exact")])
def test_gram_solve_equals_fbpca_restatement(fbo, m, d, k, kind):
    rng = np.random.RandomState(5)
    if kind == "clustered":
        decay = np.concatenate([np.linspace(10, 9, 6), np.linspace(5, 4.5, 6), 0.5 * 0.95 ** np.arange(d - 12)])
    else:
        decay = 0.9 ** np.arange(d)
    X = _synthetic(rng, m, d, decay)                      # fp64 input: Omega is the same array in both forms
    np.random.seed(123)
    _, s_lit, Va_lit = fbo.pca(X, k=k, n_iter=2, raw=True, l=2 * k)
    np.random.seed(123)
    omega = np.random.uniform(-1.0, 1.0, (d, 2 * k)) if fbo.randomized(k, m, d) else None
    assert (omega is None) == (kind == "exact")
    Va, s = fbo.gram_solve(X.T @ X, omega, k)
    cos = np.abs(np.sum(Va * Va_lit, axis=1))
    assert cos.min() >= 1 - 1e-10, cos.min()
    assert np.max(np.abs(s - s_lit) / s_lit) <= 1e-10


def _cmp(oracle, ours, ref, fbo):
    return oracle.compare_npz(fbo.sign_normalise(ours), fbo.sign_normalise(ref))


@pytest.mark.parametrize("form", ["literal", "gram"])
@pytest.mark.parametrize("name,kw", FIXTURES)
def test_compute_restatement_vs_reference(oracle, golden, mapping_weights, fbo, name, kw, form):
    g = golden(name)
    ws, bs = mapping_weights
    out = fbo.compute_stylegan2_style_fbpca(ws, bs, kw["n"], kw["B"], kw["c"], kw["use_w"], form=form)
    cmp = _cmp(oracle, out, g, fbo)
    assert cmp["min_signed_cos"] > 1 - 1e-6 and cmp["min_lat_signed_cos"] > 1 - 1e-6, cmp
    assert cmp["max_abs_dvar_ratio"] < 1e-6, cmp
    for k in ("act_mean_rel", "act_stdev_rel", "lat_mean_rel", "lat_stdev_rel", "random_stdevs_rel"):
        assert cmp[k] < 1e-5, (k, cmp)
    for k in out:
        assert out[k].shape == g[k].shape and out[k].dtype == g[k].dtype, k


@pytest.mark.parametrize("use_w,randomized", [(True, True), (False, True), (True, False)])
def test_host_omega_is_the_reference_draw(monkeypatch, use_w, randomized):
    """The driver's draws -- phase A seeds, fbpca's Omega, then (W space) the lat_stdev seed -- equal the reference's sequence:
    the seeds of every sample_latent(B) call, then fbpca's uniform(-1, 1) draw inside fit, then sample_latent(5000)."""
    from ganspace_b200 import decomposition, plan
    from ganspace_b200.estimators import FacebookPCAEstimator
    n, B, c, d = (10_000, 1_000, 32, 512) if randomized else (4_000, 1_000, 210, 512)
    pl = plan.make_plan(n, B, c)
    est = FacebookPCAEstimator(c)
    np.random.seed(1)
    seeds = decomposition._draw_seeds(pl.n_calls)
    omega = est.draw_omega(pl.N + pl.NB, d)
    after = decomposition._draw_seeds(1)[0] if use_w else None
    # the reference: sample_latent draws one randint per call (models/wrappers.py:168-169), fbpca draws Omega in fit
    np.random.seed(1)
    ref_seeds = [np.random.randint(np.iinfo(np.int32).max) for _ in range(pl.n_calls)]
    ref_omega = np.random.uniform(low=-1.0, high=1.0, size=(d, 2 * c)).astype(np.float32) if randomized else None
    ref_after = np.random.randint(np.iinfo(np.int32).max) if use_w else None
    assert seeds == ref_seeds
    if randomized:
        assert omega.dtype == np.float32 and omega.shape == (d, 2 * c) and np.array_equal(omega, ref_omega)
    else:
        assert omega is None
    assert after == ref_after


def test_estimator_surface_and_cache_name():
    from ganspace_b200.estimators import FacebookPCAEstimator, get_estimator
    est = get_estimator("fbpca", 80, 1.0)
    assert isinstance(est, FacebookPCAEstimator)
    assert not est.batch_support and est.n_iter == 2 and est.l == 160
    assert est.get_param_str() == "fbpca_c80_it2_l160"
    assert est.randomized(1_010_000, 512)
    assert not FacebookPCAEstimator(205).randomized(10 ** 6, 512) and FacebookPCAEstimator(204).randomized(10 ** 6, 512)
    for name in ("pca", "ica", "spca"):
        with pytest.raises(RuntimeError):
            get_estimator(name, 3, 1.0)


def test_cache_name(monkeypatch, tmp_path):
    """get_or_compute's cache file (decomposition.py:384-394) carries fbpca's parameter string."""
    from types import SimpleNamespace
    from ganspace_b200 import decomposition
    from ganspace_b200.config import Config
    calls = []
    monkeypatch.setattr(decomposition, "compute", lambda cfg, path, model: calls.append(path))
    cfg = Config(model="StyleGAN2", layer="style", output_class="ffhq", estimator="fbpca", components=32, n=10_000,
                 use_w=True, seed=3)
    path = decomposition.get_or_compute(cfg, submit_config=SimpleNamespace(run_dir=str(tmp_path), run_dir_root=str(tmp_path)))
    assert path.name == "stylegan2-ffhq_style_fbpca_c32_it2_l64_n10000_w_seed3.npz" and calls == [path]


def test_fixture_names_match_the_reference_cache_names(golden):
    for name, kw in FIXTURES:
        g = golden(name)
        want = "stylegan2-ffhq_style_fbpca_c{c}_it2_l{l}_n{n}{w}.npz".format(c=kw["c"], l=2 * kw["c"], n=kw["n"],
                                                                            w="_w" if kw["use_w"] else "")
        assert str(g["dump_name"]) == want
