"""Parity of the StyleGAN2 synthesis chain (csrc/synthesis.cu via the C ABI) and of the large-d IPCA engine
(csrc/bigd.cu) against the committed reference fixtures and the oracle (SURVEY.md section 8 row a5, config-5 family)."""
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

COS_TOL = 0.999        # BASELINE.json north_star tolerances
RATIO_TOL = 1e-3
ACT_TOL = 2e-4         # activations: max |diff| / max |ref| (fp16 hi/lo tensor-core products, ~1e-5 per layer)


def _perturb(model, names):
    """Same deterministic non-zero noise weights / biases as oracle/gen_golden.py perturb_synthesis."""
    mods = dict(model.named_modules())
    for i, name in enumerate(names):
        with torch.no_grad():
            mods[name].noise.weight.fill_(0.1 * (i + 1))
            b = mods[name].activate.bias
            b.copy_((0.1 * torch.sin(torch.arange(b.shape[0], dtype=torch.float32) + i)).to(b.device))


@pytest.fixture(scope="module")
def perturbed_model():
    from ganspace_b200.models import StyleGAN2
    m = StyleGAN2(torch.device("cuda:0"), "ffhq", random_init=1234)
    _perturb(m.model, ["conv1"] + [f"convs.{i}" for i in range(5)])
    return m


def test_partial_forward_known_answers(golden, perturbed_model):
    """Reference partial_forward (wrappers.py:224-255) outputs for 4 seeded latents, layers conv1 .. convs.4."""
    from ganspace_b200.models import get_instrumented_model
    g = golden("synthesis_known_answers.npz")
    m = perturbed_model
    dev = m.device
    m.use_z()
    z = m.sample_latent(4, seed=21)
    assert np.array_equal(z.cpu().numpy(), g["z"])
    for layer, keep in (("conv1", 4), ("convs.0", 4), ("convs.1", 4), ("convs.2", 2), ("convs.3", 1), ("convs.4", 1)):
        inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=m, use_w=False)
        m.partial_forward(z[:keep], layer)
        act = inst.retained_features()[layer]
        key = layer.replace(".", "_")
        a = act.cpu().numpy()
        if f"act_{key}" in g:
            ref = g[f"act_{key}"]
            assert a.shape == ref.shape, (layer, a.shape, ref.shape)
        else:
            ref = g[f"act_{key}_sub"]
            a_sub = a[:, ::4, ::2, ::2]
            assert a_sub.shape == ref.shape
            sums = np.array([a.astype(np.float64).sum(), (a.astype(np.float64) ** 2).sum()])
            assert np.allclose(sums, g[f"sum_{key}"], rtol=1e-4), (layer, sums, g[f"sum_{key}"])
            a = a_sub
        err = np.abs(a - ref).max() / np.abs(ref).max()
        assert err < ACT_TOL, (layer, err)
        inst.close()
    m.check_numerics()


def test_synthesis_chunking_and_native_layout(oracle, perturbed_model):
    """A batch that spans several sample chunks with a ragged tail (33 samples at 16x16: chunks of 8), written through
    activations_into into a row-strided buffer, against the oracle's reference-form StyledConv chain."""
    m = perturbed_model
    m.use_w()
    rng = np.random.RandomState(5)
    w = rng.standard_normal((33, 512)).astype(np.float32)
    params = oracle.synthesis_random_init(1234, 1024, "convs.3")
    for i, name in enumerate(oracle.synthesis_layer_names("convs.3")):
        params["layers"][name]["noise_weight"] = np.float32(0.1 * (i + 1))
        params["layers"][name]["act_bias"] = (0.1 * np.sin(np.arange(512, dtype=np.float32) + i)).astype(np.float32)
    ref = oracle.synthesis_forward(w, params, oracle.fixed_noise(0, 1024), "convs.3")      # [33,512,16,16]
    d = 512 * 16 * 16
    buf = torch.zeros((40, d + 64), dtype=torch.float32, device=m.device)
    out = buf[3:36, :d]
    assert m.feature_layout("convs.3") == ("nhwc", (16, 16, 512))
    m.activations_into(torch.from_numpy(w).to(m.device), "convs.3", out)
    got = out.view(33, 16, 16, 512).permute(0, 3, 1, 2).cpu().numpy()
    err = np.abs(got - ref).max() / np.abs(ref).max()
    assert err < ACT_TOL, err
    assert float(buf[:3].abs().max()) == 0.0 and float(buf[36:].abs().max()) == 0.0 and float(buf[:, d:].abs().max()) == 0.0
    m.use_z()


@pytest.mark.parametrize("n,c", [(1088, 16), (2112, 80)])
def test_sym_eig_large(n, c):
    """L2-resident tridiagonalisation + bisection + inverse iteration for 1024 < n <= 4096 (small side of the large-d engine)."""
    from ganspace_b200 import _native
    torch.manual_seed(n)
    dev = torch.device("cuda:0")
    q, _ = torch.linalg.qr(torch.randn(n, n, dtype=torch.float64, device=dev))
    lam = torch.cat([torch.logspace(3, 0, 200, dtype=torch.float64, device=dev),
                     1e-3 * torch.rand(n - 200, dtype=torch.float64, device=dev)])
    a = (q * lam) @ q.T
    a = 0.5 * (a + a.T)
    evals, evecs = _native.sym_eig_top(a, c)
    ref = torch.linalg.eigvalsh(a).flip(0)[:c]
    assert torch.allclose(evals, ref, rtol=1e-10, atol=1e-10 * float(ref[0]))
    resid = (a @ evecs.T - evecs.T * evals).norm(dim=0) / float(ref[0])
    assert float(resid.max()) < 1e-10, float(resid.max())
    gram = evecs @ evecs.T
    assert float((gram - torch.eye(c, dtype=torch.float64, device=dev)).abs().max()) < 1e-9


def _synthetic_batches(d, nb, k, seed):
    rng = np.random.RandomState(seed)
    basis = rng.standard_normal((d, 64)).astype(np.float32) * (0.85 ** np.arange(64, dtype=np.float32))[None, :]
    shift = 2.0 * rng.standard_normal(d).astype(np.float32)
    return [((rng.standard_normal((nb, 64)).astype(np.float32) @ basis.T) + 0.05 * rng.standard_normal((nb, d)).astype(np.float32)
             + shift).astype(np.float32) for _ in range(k)]


def test_gram_tc_matches_fp64(monkeypatch):
    """Small-side Gram on the tensor cores with the promoted accumulator vs the fp32-FMA kernel vs fp64, three chunks of d with a
    ragged tail, rows of very different magnitude (per-row power-of-two scaling)."""
    from ganspace_b200 import _native
    dev = torch.device("cuda:0")
    d, nb, c = 20480, 300, 12
    g = torch.Generator(device="cpu").manual_seed(3)
    base = torch.randn(nb + c, d, generator=g)
    base[:c] *= 1000.0                       # "S * Vt" rows
    base[c + 5] *= 1e-3
    base[c + 6] *= 50.0
    base[c:] += 0.7                          # non-zero batch mean
    res = {}
    for gram in ("simt", "tc"):
        eng = _native.BigIPCA(d, c, nb, dev, gram=gram)
        eng.M[:c].copy_(base[:c])
        eng.batch_rows(nb).copy_(base[c:])
        eng.n_seen = 900                      # a previous state: the correction row is live
        T = eng.gram_only(nb).clone()
        M64 = eng.M[:c + nb + 1].double()     # centred in place by phase 1
        ref = M64 @ M64.T
        n = c + nb + 1
        scale = torch.sqrt(torch.outer(torch.diag(ref), torch.diag(ref)))
        res[gram] = float(((T[:n, :n] - ref).abs() / scale).max())
        assert float(((T[:n, :n] - T[:n, :n].T).abs() / scale).max()) < 1e-12
        assert float(T[n:].abs().max()) == 0.0 and float(T[:, n:].abs().max()) == 0.0
    print("gram error vs fp64 (relative to sqrt(T_ii T_jj)):", res)
    assert res["simt"] < 5e-6, res          # measured 2.4e-6 (8192-long fp32 FMA chains)
    assert res["tc"] < 5e-6, res            # measured 1.6e-6 (48 truncating MMA steps per promotion)


@pytest.mark.parametrize("gram", ["simt", "tc"])
@pytest.mark.parametrize("d,nb,c,k", [(4096, 300, 12, 4), (2048, 1100, 16, 3)])
def test_large_d_chain_vs_sklearn_form(oracle, monkeypatch, d, nb, c, k, gram):
    """IPCAEstimator with d > 1024 (small-side engine) against the oracle's restatement of IncrementalPCA.partial_fit.
    (2048, 1100, 16): small side 1117 -> 1120 > 1024 exercises the L2 eigensolver on every step."""
    from ganspace_b200.estimators import get_estimator
    monkeypatch.setenv("GANSPACE_B200_BIGD_GRAM", gram)
    Xs = _synthetic_batches(d, nb, k, seed=d + nb)
    est = get_estimator("ipca", c, 1.0)
    st = oracle.IPCAState(c)
    for i, X in enumerate(Xs):
        if i % 2 == 0:
            assert est.fit_partial(torch.from_numpy(X).cuda())
        else:
            assert est.fit_partial(X.copy())
        oracle.ipca_partial_fit(st, X.copy())
        comp, stdev, ratio = est.get_components()
        cos = np.sum(np.asarray(comp, np.float64) * st.components, axis=1)
        assert cos.min() > 1 - 1e-5, (i, cos.min())
        assert np.allclose(stdev, np.sqrt(st.explained_variance), rtol=2e-5), i
        assert np.abs(ratio - st.explained_variance_ratio).max() < 1e-5, i
        assert np.allclose(est.transformer.mean_, st.mean, rtol=1e-6, atol=1e-6)
        assert np.allclose(est.transformer.var_, st.var, rtol=1e-5)
    assert est.transformer.is_large_d and int(est.transformer.n_samples_seen_) == nb * k
    # a later, larger batch grows the device buffer and keeps the state
    Xl = _synthetic_batches(d, nb + 40, 1, seed=7)[0]
    assert est.fit_partial(Xl.copy())
    oracle.ipca_partial_fit(st, Xl.copy())
    comp, stdev, _ = est.get_components()
    assert np.sum(np.asarray(comp, np.float64) * st.components, axis=1).min() > 1 - 1e-5


def _run_layer(layer, n, b, c, perturb=None):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model, StyleGAN2
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    if perturb:
        _perturb(model.model, perturb)
    inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=model, use_w=False)
    cfg = Config(model="StyleGAN2", layer=layer, output_class="ffhq", components=c, n=n, batch_size=b, use_w=False,
                 estimator="ipca")
    with tempfile.TemporaryDirectory() as tmp:
        path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        with np.load(path, allow_pickle=False) as data:
            out = {k: data[k] for k in data.files}
    inst.close()
    return out, path.name


@pytest.mark.parametrize("fixture,layer,n,b,c", [
    ("c5s_stylegan2_ffhq_convs1_z_n4000_b500_c8.npz", "convs.1", 4000, 500, 8),
    ("c5s_stylegan2_ffhq_convs2_z_n4000_b250_c6.npz", "convs.2", 4000, 250, 6),
])
def test_conv_layer_pca_vs_reference_golden(golden, oracle, fixture, layer, n, b, c):
    """get_or_compute on a StyledConv feature map (d = 32768 / 131072), Z space with the regression pass, against the
    unmodified reference's .npz (config-5 family at a size the reference finishes on the build container's CPU)."""
    from conftest import GOLDEN
    if not (GOLDEN / fixture).exists():
        pytest.skip(f"fixture {fixture} not generated")
    g = golden(fixture)
    out, name = _run_layer(layer, n, b, c)
    assert name == str(g["dump_name"])
    for k in ("act_comp", "act_mean", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio", "random_stdevs"):
        assert out[k].shape == g[k].shape and out[k].dtype == g[k].dtype, k
    cmp = oracle.compare_npz(out, g)
    assert cmp["min_signed_cos"] >= COS_TOL, cmp
    assert cmp["max_abs_dvar_ratio"] <= RATIO_TOL, cmp
    assert cmp["min_lat_signed_cos"] >= COS_TOL, cmp
    assert cmp["act_mean_rel"] < 1e-3 and cmp["act_stdev_rel"] < 1e-3 and cmp["random_stdevs_rel"] < 1e-3, cmp


def test_conv_layer_pca_nonzero_noise_vs_reference_golden(golden, oracle):
    """End to end with NON-ZERO NoiseInjection weights and activation biases (both are 0 at random init, which leaves the noise
    path of the fused epilogue untested at the PCA level): layer=convs.1, Z space + regression, against the reference's .npz
    (oracle/gen_golden_r2.py G10; fixed noise maps from set_noise_seed(0) on the CPU generator, as the reference's CPU run)."""
    g = golden("c5n_stylegan2_ffhq_convs1_z_noise_n4000_b500_c8.npz")
    out, name = _run_layer("convs.1", 4000, 500, 8, perturb=[str(x) for x in g["perturbed"]])
    assert name == str(g["dump_name"])
    if int(g.get("lat_placeholder", 0)):
        for k in ("lat_comp", "lat_mean", "lat_stdev"):
            g[k] = out[k]
    cmp = oracle.compare_npz(out, g)
    assert cmp["min_signed_cos"] >= COS_TOL and cmp["max_abs_dvar_ratio"] <= RATIO_TOL, cmp
    assert cmp["act_mean_rel"] < 1e-3 and cmp["act_stdev_rel"] < 1e-3 and cmp["random_stdevs_rel"] < 1e-3, cmp
    # the perturbation matters: the zero-noise fixture of the same layer has a different mean
    g0 = golden("c5s_stylegan2_ffhq_convs1_z_n4000_b500_c8.npz")
    assert np.abs(g["act_mean"] - g0["act_mean"]).max() > 1e-2


def test_config5_layer_convs4_vs_reference_golden(golden, oracle):
    """BASELINE config 5's layer itself: convs.4 (d = 524288), Z space, N = 4000, through the large-d engine with the
    tensor-core Gram, against the unmodified reference's PCA stage (oracle/gen_golden_r2.py G9; act_comp stored as float16).
    The reference's regression stage does not fit the 62 GB fixture container at this d, so the fixture's lat_* arrays are
    placeholders and only the act_* / variance arrays are compared (the regression itself: the convs.1 / convs.2 fixtures)."""
    from conftest import GOLDEN
    fixture = "c5_stylegan2_ffhq_convs4_z_n4000_b500_c4.npz"
    if not (GOLDEN / fixture).exists():
        pytest.skip(f"fixture {fixture} not generated")
    g = dict(golden(fixture))
    g["act_comp"] = g.pop("act_comp_f16").astype(np.float32)
    out, name = _run_layer("convs.4", 4000, 500, 4)
    assert name == str(g["dump_name"]) and out["act_comp"].shape == (4, 1, 512, 32, 32)
    if int(g.get("lat_placeholder", 0)):
        for k in ("lat_comp", "lat_mean", "lat_stdev"):
            g[k] = out[k]
    cmp = oracle.compare_npz(out, g)
    assert cmp["min_signed_cos"] >= COS_TOL and cmp["max_abs_dvar_ratio"] <= RATIO_TOL, cmp
    assert cmp["act_mean_rel"] < 1e-3 and cmp["act_stdev_rel"] < 1e-3 and cmp["random_stdevs_rel"] < 1e-3, cmp
