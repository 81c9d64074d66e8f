"""StyleGAN2 feature maps at 64 x 64 and 128 x 128 (convs.6 / convs.7: d = 2,097,152; convs.8 / convs.9: d = 4,194,304) through the
large-d IPCA engine: the engine against fp64 at full width, the synthesis kernels writing rows whose element offsets pass 2^31,
the device NHWC -> NCHW export permutation, get_or_compute end to end against an fp64 restatement on the same activations, and
the guards (StyleGAN2's bound, the device-memory check)."""
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch
from ipca_rows import Data

pytestmark = pytest.mark.gpu

COS_TOL = 0.999        # signed cosine per component
RATIO_TOL = 1e-3       # |explained-variance ratio - fp64|
D64, D128 = 64 * 64 * 512, 128 * 128 * 256


def _signed_cos(a, b):
    a = np.asarray(a, np.float64)
    b = np.asarray(b, np.float64)
    return np.sum(a * b, axis=1) / (np.linalg.norm(a, axis=1) * np.linalg.norm(b, axis=1))


# ---- 1. the engine at full width against fp64 --------------------------------------------------------------------------
@pytest.mark.parametrize("d", [D64, D128])
def test_engine_parity_full_width(oracle, d):
    """Three 64-row batches at c = 8 through BigIPCA (tensor-core Gram, operands split into 524,288-column slabs) against
    ``oracle.ipca_partial_fit_small_side`` after every step."""
    from ganspace_b200 import _native
    c, nb = 8, 64
    dev = torch.device("cuda:0")
    data = Data(d, c, nb, "gapped", seed=77 + d % 1000)
    eng = _native.BigIPCA(d, c, nb, dev)
    st = oracle.IPCAState(c)
    for i in range(3):
        X = data.batch(i, nb)
        eng.batch_rows(nb).copy_(torch.from_numpy(X).to(dev))
        eng.step(nb)
        oracle.ipca_partial_fit_small_side(st, X)
        got = {k: v.cpu().numpy().astype(np.float64) for k, v in eng.export().items()}
        cos = np.sum(got["components"] * st.components, axis=1)
        ratio = np.abs(got["explained_variance_ratio"] - st.explained_variance_ratio)
        assert cos.min() >= COS_TOL, (d, i, int(np.argmin(cos)), cos.min())
        assert ratio.max() <= RATIO_TOL, (d, i, ratio.max())
        assert np.allclose(got["mean"], st.mean, rtol=1e-6, atol=1e-6), (d, i, "mean")
        assert np.allclose(got["var"], st.var, rtol=1e-5), (d, i, "var")
    del eng
    torch.cuda.empty_cache()


# ---- 2. synthesis straight into the engine's rows ----------------------------------------------------------------------
@pytest.fixture(scope="module")
def sg2():
    from ganspace_b200.models import get_instrumented_model, StyleGAN2
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    inst = get_instrumented_model("StyleGAN2", "ffhq", "convs.6", dev, model=model)
    yield inst
    inst.close()


@pytest.mark.parametrize("layer,d", [("convs.6", D64), ("convs.8", D128)])
def test_activations_into_past_2_31(sg2, layer, d):
    """``activations_into`` into rows of a buffer whose first written element lies past 2^31 equals ``partial_forward``'s hooked
    activation (permuted to NHWC) bit for bit; the rows around the written ones are untouched."""
    model = sg2.model
    n = 6
    row0 = (1 << 31) // d + 3
    buf = torch.full((row0 + n + 1, d), -7.0, dtype=torch.float32, device=model.device)
    assert row0 * d > (1 << 31)
    z = model.sample_latent(n, seed=4321)
    model.activations_into(z, layer, buf[row0:row0 + n])
    sg2.retain_layer(layer)
    with torch.no_grad():
        model.partial_forward(z, layer)
    ref = sg2.retained_features()[layer]                       # [n, C, H, W]
    ref_nhwc = ref.permute(0, 2, 3, 1).reshape(n, -1)
    assert torch.equal(buf[row0:row0 + n], ref_nhwc)
    assert bool((buf[row0 - 1] == -7.0).all()) and bool((buf[row0 + n] == -7.0).all())
    del buf
    torch.cuda.empty_cache()


def test_activations_into_slices_large_batches(sg2, monkeypatch):
    """Batches whose synthesis workspace passes the budget run in slices of rows, with the bits of one call."""
    model = sg2.model
    z = model.sample_latent(40, seed=99)
    whole = model.activations_into(z, "convs.6", torch.empty((40, D64), device=model.device))
    monkeypatch.setattr(type(model), "SYNTH_WORKSPACE_BUDGET", 200 << 20)
    n_run = model.synthesis_layer_names().index("convs.6") + 1
    assert model._synthesis(n_run).rows_within(n_run, 40, 200 << 20) < 40
    sliced = model.activations_into(z, "convs.6", torch.empty((40, D64), device=model.device))
    assert torch.equal(whole, sliced)


# ---- 3. the export permutation ----------------------------------------------------------------------------------------
@pytest.mark.parametrize("rows,h,c,dtype", [(3, 7, 3, np.float32), (2, 5, 512, np.float32), (5, 33, 40, np.float32),
                                            (1, 1, 1, np.float32), (4, 17, 3, np.float64), (2, 64, 512, np.float64)])
def test_nhwc_to_nchw_rows_ragged(rows, h, c, dtype):
    from ganspace_b200 import _native
    rng = np.random.RandomState(rows * 1000 + h * 10 + c)
    x = rng.standard_normal((rows, h * h * c)).astype(dtype)
    want = np.ascontiguousarray(x.reshape(rows, h, h, c).transpose(0, 3, 1, 2)).reshape(rows, -1)
    got = _native.nhwc_to_nchw_rows(torch.from_numpy(x).cuda(), h * h, c).cpu().numpy()
    assert got.dtype == dtype and np.array_equal(got.view(np.uint8), want.view(np.uint8))
    # row-strided source and destination
    src = torch.zeros((rows, h * h * c + 8), dtype=torch.float64 if dtype == np.float64 else torch.float32, device="cuda")
    src[:, :h * h * c] = torch.from_numpy(x).cuda()
    dst = torch.zeros_like(src)
    _native.nhwc_to_nchw_rows(src[:, :h * h * c], h * h, c, out=dst[:, :h * h * c])
    assert np.array_equal(dst[:, :h * h * c].cpu().numpy(), want) and bool((dst[:, h * h * c:] == 0).all())


def test_nhwc_to_nchw_rows_full_components():
    """One full [80, 128*128*256] array (the components of convs.8 at c = 80)."""
    from ganspace_b200 import _native
    rows, h, c = 80, 128, 256
    x = torch.randn((rows, h * h * c), generator=torch.Generator().manual_seed(5)).numpy()
    got = _native.nhwc_to_nchw_rows(torch.from_numpy(x).cuda(), h * h, c).cpu().numpy()
    want = np.ascontiguousarray(x.reshape(rows, h, h, c).transpose(0, 3, 1, 2)).reshape(rows, -1)
    assert np.array_equal(got, want)


def test_nhwc_to_nchw_rows_refusals():
    from ganspace_b200 import _native
    x = torch.zeros((2, 48), device="cuda")
    with pytest.raises(_native.NativeError):
        _native._check(_native.load().gsb_nhwc_to_nchw_rows(_native._ptr(x), 48, _native._ptr(x), 48, 2, 16, 3, 4,
                                                            _native._stream()), "gsb_nhwc_to_nchw_rows")
    with pytest.raises(_native.NativeError):
        y = torch.zeros_like(x)
        _native._check(_native.load().gsb_nhwc_to_nchw_rows(_native._ptr(x), 48, _native._ptr(y), 48, 2, 16, 3, 2,
                                                            _native._stream()), "gsb_nhwc_to_nchw_rows")


# ---- 4. end to end ---------------------------------------------------------------------------------------------------
def _fp64_ipca(groups, c, d, dev, chunk=1 << 16):
    """sklearn IncrementalPCA.partial_fit over ``groups`` ([nb, d] fp32 device tensors, produced lazily) restated in fp64
    through the small side of the stacked matrix, column chunk by column chunk (the stacked matrix never exists in fp64 at
    once).  Returns (components [c, d] with svd_flip signs, explained_variance_ratio [c])."""
    f64 = dict(dtype=torch.float64, device=dev)
    n_seen, mean, var, comps, S = 0, torch.zeros(d, **f64), torch.zeros(d, **f64), None, None
    for X in groups:
        nb = X.shape[0]
        bmean = torch.zeros(d, **f64)
        bunnorm = torch.zeros(d, **f64)
        for j in range(0, d, chunk):
            Xc = X[:, j:j + chunk].double()
            bmean[j:j + chunk] = Xc.mean(0)
            bunnorm[j:j + chunk] = ((Xc - bmean[j:j + chunk]) ** 2).sum(0)
        n_tot = n_seen + nb
        if n_seen == 0:
            new_mean, new_var = bmean, bunnorm / n_tot
            corr = None
        else:
            r = n_seen / nb
            unnorm = var * n_seen + bunnorm + r / n_tot * (mean * n_seen / r - bmean * nb) ** 2
            corr = np.sqrt((n_seen / n_tot) * nb) * (mean - bmean)
            new_mean, new_var = (mean * n_seen + bmean * nb) / n_tot, unnorm / n_tot

        def block(j):
            Xc = X[:, j:j + chunk].double() - bmean[j:j + chunk]
            if n_seen == 0:
                return Xc
            return torch.cat([S[:, None] * comps[:, j:j + chunk], Xc, corr[None, j:j + chunk]])
        rows = nb if n_seen == 0 else c + nb + 1
        G = torch.zeros((rows, rows), **f64)
        for j in range(0, d, chunk):
            Mb = block(j)
            G += Mb @ Mb.T
        lam, U = torch.linalg.eigh(G)
        lam, U = lam.flip(0)[:c], U.flip(1)[:, :c]
        S_new = lam.clamp_min(0).sqrt()
        V = torch.empty((c, d), **f64)
        for j in range(0, d, chunk):
            V[:, j:j + chunk] = (U.T @ block(j)) / S_new[:, None]
        idx = V.abs().argmax(1)
        V *= torch.sign(V[torch.arange(c, device=dev), idx])[:, None]
        comps, S, mean, var, n_seen = V, S_new, new_mean, new_var, n_tot
    ratio = S ** 2 / (var.sum() * n_seen)
    return comps, ratio


@pytest.mark.parametrize("layer,shape", [("convs.6", (512, 64, 64)), ("convs.8", (256, 128, 128))])
def test_get_or_compute_end_to_end(layer, shape):
    """get_or_compute on a 64 x 64 and a 128 x 128 layer (Z space, N = 6000, B = 2000, c = 8): the reference's eight arrays in its
    shapes; act_comp and var_ratio against the fp64 restatement fed with ``partial_forward``'s activations of the latents the
    fit consumed; a second run writes byte-identical arrays."""
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model, StyleGAN2
    dev = torch.device("cuda:0")
    c, n, b = 8, 6000, 2000
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=model)
    seen = []
    into = model.activations_into

    def recording(x, layer_name, out):
        seen.append(x.detach().clone())
        return into(x, layer_name, out)
    model.activations_into = recording
    cfg = Config(model="StyleGAN2", layer=layer, output_class="ffhq", components=c, n=n, batch_size=b, use_w=False,
                 estimator="ipca")
    files = []
    with tempfile.TemporaryDirectory() as tmp:
        for rep in range(2):
            run_dir = f"{tmp}/{rep}"
            path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=run_dir, run_dir_root=run_dir),
                                  force_recompute=True)
            with np.load(path, allow_pickle=False) as data:
                files.append({k: data[k] for k in data.files})
            if rep == 0:
                fit_latents = torch.cat(seen)[:n]
    out = files[0]
    model.activations_into = into
    for k in out:         # every member byte for byte (the .npz container itself stamps the time of writing)
        assert out[k].tobytes() == files[1][k].tobytes(), f"two runs wrote different {k}"
    assert sorted(out) == sorted(["act_comp", "act_mean", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio",
                                  "random_stdevs"])
    want = {"act_comp": (c, 1, *shape), "act_mean": (1, *shape), "act_stdev": (c,), "lat_comp": (c, 1, 512), "lat_mean": (1, 512),
            "lat_stdev": (c,), "var_ratio": (c,), "random_stdevs": (c,)}
    for k, s in want.items():
        assert out[k].shape == s and out[k].dtype == np.float32, (k, out[k].shape, s)
    assert fit_latents.shape[0] == n
    torch.cuda.empty_cache()

    d = int(np.prod(shape))

    def groups():
        X = torch.empty((b, d), dtype=torch.float32, device=dev)       # one buffer: each group is consumed before the next
        for g0 in range(0, n, b):
            for r in range(0, b, 250):
                with torch.no_grad():
                    model.partial_forward(fit_latents[g0 + r:g0 + r + 250], layer)
                X[r:r + 250] = inst.retained_features()[layer].reshape(250, -1)
            yield X
    comps, ratio = _fp64_ipca(groups(), c, d, dev)
    cos = _signed_cos(out["act_comp"].reshape(c, -1), comps.cpu().numpy())
    assert cos.min() >= COS_TOL, (layer, cos)
    assert np.abs(out["var_ratio"] - ratio.cpu().numpy()).max() <= RATIO_TOL, (layer, out["var_ratio"], ratio)
    inst.close()
    torch.cuda.empty_cache()


# ---- 5. guards -------------------------------------------------------------------------------------------------------
def test_convs10_exceeds_bound():
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model, StyleGAN2
    dev = torch.device("cuda:0")
    model = StyleGAN2(dev, "ffhq", random_init=1234)
    with pytest.raises(NotImplementedError, match="exceeds"):
        model.feature_layout("convs.10")
    inst = get_instrumented_model("StyleGAN2", "ffhq", "convs.10", dev, model=model)
    with tempfile.TemporaryDirectory() as tmp:
        with pytest.raises(NotImplementedError, match="exceeds"):
            get_or_compute(Config(model="StyleGAN2", layer="convs.10", output_class="ffhq", components=8, n=4000,
                                  batch_size=2000), inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp),
                           force_recompute=True)
    inst.close()


def test_engine_that_cannot_fit_raises_before_allocating():
    """c = 128 and 3967-row batches at d = 4,194,304: a 68.7 GB stacked matrix plus its workspace, more than an 80 GB card
    holds next to a 20 GB reserve -- refused before anything is allocated or launched."""
    from ganspace_b200 import _native
    dev = torch.device("cuda:0")
    torch.cuda.synchronize()
    before = torch.cuda.memory_allocated(dev)
    need = _native.BigIPCA.device_bytes(D128, 128, 3967)
    assert need > 68e9
    with pytest.raises(_native.DeviceMemoryError, match=f"{need + (20 << 30):,} bytes"):
        _native.BigIPCA(D128, 128, 3967, dev, reserve=20 << 30)
    assert torch.cuda.memory_allocated(dev) == before
