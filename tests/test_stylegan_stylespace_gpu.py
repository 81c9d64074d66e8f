"""StyleGAN (v1) style space on the device: the rows of every StyleMod layer ('g_synthesis.blocks.RxR.epi{1,2}.style_mod.lin')
against the unmodified reference (oracle/gen_golden_stylegan_stylespace.py) and fp64, the styled run against the chain's own,
partial_forward to a style layer without a synthesis launch, forward with style hooks bit-identical to forward without them,
style edits against the reference and fp64, the notebook strip flow, get_or_compute on style layers, and the hook guards."""
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ganspace_oracle as go
from oracle import stylegan_oracle as so
from oracle import stylegan_stylespace_oracle as sso

pytestmark = pytest.mark.gpu

MAP_TOL = 2e-5         # the mapping network's bar (test_kernels_gpu.py): one fp32 product of K = 512 per layer
ROW_TOL = 1e-5         # one fp32 dot product of K = 512 against fp64, relative to max(1, max |ref|)
COS_TOL, RATIO_TOL, REL_TOL = 0.999, 1e-3, 1e-3
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def ka(golden):
    return golden("stylegan_stylespace_known_answers.npz")


@pytest.fixture(scope="module")
def models():
    from ganspace_b200.models import StyleGAN, stylegan
    out = {}
    for cls in ("ffhq", "bedrooms"):
        m = StyleGAN(DEV, cls, random_init=1234)
        stylegan.synthesis_fill(m.model, 7)
        m.use_z()
        out[cls] = m
    return out


def _key(name):
    return name[len("g_synthesis.blocks."):].replace(".", "_")


def _names(m):
    return [t[0] for t in m.model.style_layers()]


def _inst(m, layers, use_w=False):
    from ganspace_b200.models import get_instrumented_model
    return get_instrumented_model("StyleGAN", m.outclass, layers, DEV, model=m, use_w=use_w)


def _close(got, ref, tol, what):
    got, ref = got.cpu().numpy() if torch.is_tensor(got) else got, ref
    assert got.shape == ref.shape, (what, got.shape, ref.shape)
    err = np.abs(got.astype(np.float64) - ref).max()
    assert err < tol * max(1.0, np.abs(ref).max()), (what, err)


@pytest.mark.parametrize("cls", ["ffhq", "bedrooms"])
def test_style_rows_vs_reference(ka, models, cls):
    """Every style layer, retained from forward and from partial_forward, for Z, W and 18 distinct W latents."""
    m = models[cls]
    names = _names(m)
    inst = _inst(m, names)
    assert all(tuple(inst.feature_shape[n]) == (1, t[3]) for n, t in zip(names, m.model.style_layers()))
    z4 = torch.tensor(ka[f"{cls}_z4"], device=DEV)
    w18 = [torch.tensor(w, device=DEV) for w in so.w18_latents()]
    runs = [("z4", "forward", lambda: m.forward(z4)), ("z4", "partial", lambda: m.partial_forward(z4, names[-1]))]
    for tag, how, run in runs:
        run()
        for name, rows in inst.retained_features().items():
            _close(rows, ka[f"{cls}_{tag}_{_key(name)}"], MAP_TOL, (how, tag, name))
    m.use_w()
    try:
        w4 = m.model.g_mapping(z4)
        for how, run in (("forward", lambda: m.forward(w4)), ("partial", lambda: m.partial_forward(w4, names[-1]))):
            run()
            for name, rows in inst.retained_features().items():
                _close(rows, ka[f"{cls}_z4_{_key(name)}"], MAP_TOL, ("W", how, name))
        for how, run in (("forward", lambda: m.forward(w18)), ("partial", lambda: m.partial_forward(w18, names[-1]))):
            run()
            for name, rows in inst.retained_features().items():
                _close(rows, ka[f"{cls}_w18_{_key(name)}"], MAP_TOL, ("w18", how, name))
    finally:
        m.use_z()
        inst.close()


@pytest.mark.parametrize("n", [1, 127, 129, 1000, 70_000])
def test_styles_vs_fp64(models, n):
    """gsb_stylegan_styles on every element of every style layer, one latent per layer and sample; 70,000 rows is above the
    65,535 rows one launch of the former one-thread-per-element kernel could take."""
    m = models["ffhq"]
    packed = m.model.g_synthesis.packed()
    table = m.model.style_layers()
    w = torch.randn((18, n, 512), generator=torch.Generator(device=DEV).manual_seed(n), dtype=torch.float32, device=DEV)
    S = packed.styles(w, range(18))
    epis = m.model.g_synthesis.layer_modules()
    for name, l, lat, width in table:
        lin = epis[l][1].style_mod.lin
        ref = w[lat].double() @ (lin.weight.detach().double() / np.sqrt(512)).T + lin.bias.detach().double()
        assert S[l].shape == (n, width), name
        err = float((S[l].double() - ref).abs().max())
        assert err < ROW_TOL * max(1.0, float(ref.abs().max())), (name, n, err)
    # a subset, one latent for every layer: the same rows as the full set on that latent
    sub = packed.styles(w[:1], [17, 3])
    full = packed.styles(w[:1], range(18))
    assert sorted(sub) == [3, 17] and torch.equal(sub[3], full[3]) and torch.equal(sub[17], full[17])


def test_styles_arguments(models):
    from ganspace_b200 import _native
    m = models["bedrooms"]
    packed = m.model.g_synthesis.packed()
    w = torch.randn((1, 0, 512), device=DEV)
    assert packed.styles(w, [0, 13])[13].shape == (0, 128)
    lib = _native.load()
    import ctypes as C
    w = torch.randn((1, 4, 512), device=DEV)
    out = torch.empty((4, 1024), device=DEV)
    for idx, ptr in (([14], out.data_ptr()), ([-1], out.data_ptr()), ([0], None)):
        rc = lib.gsb_stylegan_styles(_native._ptr(packed.packed), packed.desc, packed.n_layers, 512, _native._ptr(w), 1, 4,
                                     (C.c_int * 1)(*idx), 1, (C.c_void_p * 1)(ptr), _native._stream())
        assert rc != 0, idx


@pytest.mark.parametrize("cls,n,Lw,n_run", [("ffhq", 5, 18, 18), ("ffhq", 130, 1, 8), ("bedrooms", 9, 1, 14), ("bedrooms", 300, 18, 6)])
def test_styled_run_is_the_chain_run(models, cls, n, Lw, n_run):
    """gsb_stylegan_forward_styled on gsb_stylegan_styles' rows equals gsb_stylegan_forward: the image and the block output."""
    m = models[cls]
    packed = m.model.g_synthesis.packed()
    w = torch.randn((Lw, n, 512), generator=torch.Generator().manual_seed(n), dtype=torch.float32).to(DEV)
    S = packed.styles(w, range(n_run))
    full = n_run == packed.n_layers
    act, img = packed.forward(w[:n_run] if Lw > 1 else w, n_run, want_act=True, want_rgb=full)
    act2, img2 = packed.forward_styled(S, n_run, want_act=True, want_rgb=full)
    assert torch.equal(act, act2)
    assert (img is None and img2 is None) or torch.equal(img, img2)
    m.check_numerics()


def test_forward_with_style_hooks_is_bit_identical(models):
    m = models["ffhq"]
    z = m.sample_latent(3, seed=11)
    plain = m.forward(z)
    inst = _inst(m, ["g_synthesis.blocks.32x32"])
    m.forward(z)
    act = inst.retained_features()["g_synthesis.blocks.32x32"].clone()
    inst.retain_layers(_names(m))
    assert torch.equal(m.forward(z), plain)
    assert torch.equal(inst.retained_features()["g_synthesis.blocks.32x32"], act)
    inst.edit_layer("g_synthesis.blocks.8x8.epi1.style_mod.lin", offset=torch.zeros(1, 1024, device=DEV))
    inst.edit_layer("g_synthesis.blocks.1024x1024.epi2.style_mod.lin", offset=torch.zeros(3, 32, device=DEV))
    assert torch.equal(m.forward(z), plain)
    assert torch.equal(inst.retained_features()["g_synthesis.blocks.32x32"], act)
    inst.close()
    lin = dict(m.model.named_modules())["g_synthesis.blocks.8x8.epi1.style_mod.lin"]
    h = lin.register_forward_hook(lambda mod, i, o: torch.zeros(2, 1024, device=DEV))
    with pytest.raises(ValueError, match="must keep the style's shape"):
        m.forward(z)
    h.remove()


def test_partial_forward_to_style_layer_runs_no_synthesis(models):
    from ganspace_b200 import _native
    m = models["ffhq"]
    packed = m.model.g_synthesis.packed()
    for layer, l in (("g_synthesis.blocks.4x4.epi1.style_mod.lin", 0), ("g_synthesis.blocks.32x32.epi2.style_mod.lin", 7),
                     ("g_synthesis.blocks.1024x1024.epi2.style_mod.lin", 17)):
        inst = _inst(m, layer)
        z = m.sample_latent(200, seed=9)
        _native.instrument.reset()
        m.partial_forward(z, layer)
        assert "stylegan" not in _native.instrument.rows and _native.instrument.rows.get("styles") == 200, layer
        got = inst.retained_features()[layer]
        assert torch.equal(got, packed.styles(m.model.g_mapping.packed().forward(z), [l])[l]), layer
        inst.close()


@pytest.mark.parametrize("which", ["offset", "ablate"])
def test_edited_images_vs_reference(ka, models, which):
    m = models["ffhq"]
    inst = _inst(m, "g_synthesis.blocks.8x8.epi1.style_mod.lin")
    if which == "offset":
        inst.edit_layer("g_synthesis.blocks.16x16.epi2.style_mod.lin", offset=torch.tensor(ka["edit_offset"], device=DEV))
    else:
        inst.edit_layer("g_synthesis.blocks.4x4.epi1.style_mod.lin", ablation=0.5,
                        replacement=torch.tensor(ka["edit_replacement"], device=DEV))
    img = m.forward(torch.tensor(ka["ffhq_z4"][:2], device=DEV)).cpu().numpy()
    inst.close()
    ref = ka[f"img_{which}_sub"]
    scale = np.abs(ref - 0.5).max()
    assert np.abs(img[:, :, ::16, ::16] - ref).max() < 1e-3 * scale, np.abs(img[:, :, ::16, ::16] - ref).max() / scale
    assert abs((img.astype(np.float64) ** 2).sum() - ka[f"img_{which}_sum"][1]) < 2e-3 * ka[f"img_{which}_sum"][1]
    assert np.abs(ka["img4_sub"] - ref).max() > 1e-2 * scale


def test_edited_image_vs_fp64(models):
    """forward with a style edit on blocks.8x8.epi1 against the fp64 oracle rendering the device's own edited styles."""
    m = models["ffhq"]
    names = _names(m)
    inst = _inst(m, names)
    z = m.sample_latent(1, seed=12)
    delta = torch.tensor(np.random.RandomState(3).standard_normal((1, 1024)).astype(np.float32), device=DEV)
    inst.edit_layer("g_synthesis.blocks.8x8.epi1.style_mod.lin", offset=delta)
    img = m.forward(z).double()
    S = {k: v.double() for k, v in inst.retained_features().items()}          # retained before the edit
    inst.close()
    S["g_synthesis.blocks.8x8.epi1.style_mod.lin"] = S["g_synthesis.blocks.8x8.epi1.style_mod.lin"] + delta.double()
    noise = {int(n.split(".")[2].split("x")[0]): mod.noise.reshape(mod.noise.shape[-2:])
             for n, mod in m.model.named_modules() if n.endswith("top_epi.noise")}
    ref = sso.render_styled(S, m.model.state_dict(), noise, 1024, device=DEV)
    scale = float((ref - 0.5).abs().max())
    err = float((img - ref).abs().max())
    assert err < 1e-3 * scale, err / scale
    assert float((ref - m.forward(z).double()).abs().max()) > 1e-2 * scale            # the edit shows


def test_style_edit_reaches_downstream_block(models):
    """A style edit upstream of a retained block changes that block, and partial_forward to it equals forward's hand-off."""
    m = models["bedrooms"]
    z = m.sample_latent(4, seed=13)
    inst = _inst(m, ["g_synthesis.blocks.64x64"])
    m.forward(z)
    plain = inst.retained_features()["g_synthesis.blocks.64x64"].clone()
    inst.edit_layer("g_synthesis.blocks.16x16.epi1.style_mod.lin", offset=torch.full((1, 1024), 0.3, device=DEV))
    m.forward(z)
    edited = inst.retained_features()["g_synthesis.blocks.64x64"].clone()
    assert (edited - plain).abs().max() > 1e-2 * plain.abs().max()
    m.partial_forward(z, "g_synthesis.blocks.64x64")
    assert torch.equal(inst.retained_features()["g_synthesis.blocks.64x64"], edited)
    # an 18-latent list: latent l reaches layer l and the edit still applies
    w18 = [m.model.g_mapping(m.sample_latent(4, seed=30 + l)) for l in range(18)]
    m.use_w()
    try:
        m.forward(w18)
        a = inst.retained_features()["g_synthesis.blocks.64x64"].clone()
        m.partial_forward(w18, "g_synthesis.blocks.64x64")
        assert torch.equal(inst.retained_features()["g_synthesis.blocks.64x64"], a)
    finally:
        m.use_z()
    inst.close()


def test_each_style_hook_fires_once(models):
    m = models["ffhq"]
    calls = {}
    mods = dict(m.model.named_modules())
    names = ["g_synthesis.blocks.4x4.epi1.style_mod.lin", "g_synthesis.blocks.8x8.epi2.style_mod.lin",
             "g_synthesis.blocks.16x16.epi1.style_mod.lin", "g_synthesis.blocks.256x256.epi2.style_mod.lin"]
    inst = _inst(m, ["g_synthesis.blocks.16x16", "g_synthesis.blocks.4x4"])
    handles = [mods[n].register_forward_hook(lambda mod, i, o, n=n: calls.__setitem__(n, calls.get(n, 0) + 1)) for n in names]
    z = m.sample_latent(2, seed=14)
    m.forward(z)
    assert calls == {n: 1 for n in names}
    calls.clear()
    m.partial_forward(z, "g_synthesis.blocks.16x16")
    assert calls == {n: 1 for n in names[:3]}
    calls.clear()
    m.partial_forward(z, "g_synthesis.blocks.8x8.epi2.style_mod.lin")          # stops after block 8x8
    assert calls == {n: 1 for n in names[:2]}
    inst.close()
    for h in handles:
        h.remove()


def test_notebook_activation_strip_on_style_layer(models):
    """notebook_utils._create_strip_batch_sigma, mode 'activation', center=True, restated: retain, centre along a component,
    per-frame offsets [B, 2C], sample_np.  Equals the styled chain on explicitly edited styles."""
    m = models["bedrooms"]
    layer = "g_synthesis.blocks.16x16.epi2.style_mod.lin"
    inst = _inst(m, layer)
    z_single = m.sample_latent(1, seed=15)
    comp = torch.tensor(np.random.RandomState(4).standard_normal((1, 1024)).astype(np.float32), device=DEV)
    act_mean = torch.tensor(np.random.RandomState(5).standard_normal((1, 1024)).astype(np.float32), device=DEV)
    act_stdev, B = 2.0, 5
    normalize = lambda v: v / torch.sqrt(torch.sum(v ** 2, dim=-1, keepdim=True) + 1e-8)
    inst.retain_layer(layer)
    inst.model.sample_np(z_single)
    value = inst.retained_features()[layer].clone()
    zero = normalize(comp) * torch.sum((value - act_mean) * normalize(comp), dim=-1, keepdim=True)
    sigmas = torch.linspace(-2, 2, B, device=DEV)
    delta = comp.repeat_interleave(B, axis=0) * sigmas.reshape(-1, 1)
    inst.edit_layer(layer, offset=delta * act_stdev - zero)
    frames = inst.model.sample_np(z_single.repeat_interleave(B, axis=0))
    inst.close()
    packed = m.model.g_synthesis.packed()
    S = packed.styles(m.model.g_mapping(z_single.repeat_interleave(B, axis=0)), range(14))
    S[5] = S[5] + (delta * act_stdev - zero)
    _, img = packed.forward_styled(S, 14, want_act=False, want_rgb=True)
    ref = np.clip((0.5 * (img.permute(0, 3, 1, 2) + 1)).permute(0, 2, 3, 1).cpu().numpy(), 0.0, 1.0)
    assert np.array_equal(frames, ref)
    assert np.abs(frames[0] - frames[-1]).max() > 1e-2


def _run(models, layer, n, b, c, use_w, est="ipca"):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    m = models["ffhq"]
    inst = _inst(m, layer, use_w=use_w)
    cfg = Config(model="StyleGAN", layer=layer, output_class="ffhq", components=c, n=n, batch_size=b, use_w=use_w, estimator=est)
    try:
        with tempfile.TemporaryDirectory() as tmp:
            path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
            with np.load(path, allow_pickle=False) as data:
                out = {k: data[k] for k in data.files}
    finally:
        inst.close()
        m.use_z()
    return out, path.name


def _check(cmp):
    assert cmp["min_signed_cos"] >= COS_TOL and cmp["max_abs_dvar_ratio"] <= RATIO_TOL, cmp
    assert cmp["min_lat_signed_cos"] >= COS_TOL, cmp
    assert cmp["act_mean_rel"] < REL_TOL and cmp["act_stdev_rel"] < REL_TOL and cmp["random_stdevs_rel"] < REL_TOL, cmp


@pytest.mark.parametrize("fixture,layer,use_w", [
    ("sv_stylegan_ffhq_8x8epi1lin_z_n4000_b500_c16.npz", "g_synthesis.blocks.8x8.epi1.style_mod.lin", False),
    ("sv_stylegan_ffhq_32x32epi2lin_w_n4000_b500_c16.npz", "g_synthesis.blocks.32x32.epi2.style_mod.lin", True),
])
def test_get_or_compute_vs_reference_golden(golden, oracle, models, fixture, layer, use_w):
    g = golden(fixture)
    out, name = _run(models, layer, 4000, 500, 16, use_w)
    assert name == str(g["dump_name"])
    for k in ("act_comp", "act_mean", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio", "random_stdevs"):
        assert out[k].shape == g[k].shape and out[k].dtype == g[k].dtype, k
    _check(oracle.compare_npz(out, g))


def test_get_or_compute_fbpca_vs_oracle(oracle, models):
    """--est fbpca on blocks.16x16.epi1.style_mod.lin (W space, regression) against the oracle's fbpca restatement (fp64 Gram)."""
    from oracle import fbpca_oracle as fbo
    m = models["ffhq"]
    sd = {k: v.cpu() for k, v in m.model.state_dict().items()}
    epi = "g_synthesis.blocks.16x16.epi1"
    sample = lambda s, B_: so.mapping(go.standard_normal_f32(s, 512 * B_).reshape(B_, 512), sd).astype(np.float32)
    activate = lambda w: sso.style_rows(w, sd, epi).astype(np.float32)
    ref = fbo.compute_path_fbpca(sample, activate, 512, 1024, 4000, 500, 16, False, use_w=True)
    out, _ = _run(models, f"{epi}.style_mod.lin", 4000, 500, 16, True, est="fbpca")
    _check(oracle.compare_npz(out, fbo.sign_normalise(ref)))


def test_hook_guards(models):
    from ganspace_b200.models import get_instrumented_model
    m = models["bedrooms"]
    z = m.sample_latent(2, seed=16)
    inst = get_instrumented_model("StyleGAN", "bedrooms", "g_synthesis.blocks.8x8.epi1.style_mod.lin", DEV, model=m)
    assert tuple(inst.feature_shape["g_synthesis.blocks.8x8.epi1.style_mod.lin"]) == (1, 1024)
    inst.close()
    for bad in ("g_synthesis.blocks.8x8.epi1.style_mod", "g_synthesis.blocks.8x8.epi1", "g_synthesis.blocks.8x8.epi2.top_epi.noise",
                "g_synthesis.blocks.8x8.conv1", "g_synthesis.torgb", "g_mapping.dense3"):
        with pytest.raises(NotImplementedError, match="hookable layers") as e:
            get_instrumented_model("StyleGAN", "bedrooms", bad, DEV, model=m)
        assert "style_mod.lin" in str(e.value)
        assert not any(len(mod._forward_hooks) for _, mod in m.model.named_modules()), bad
    # a block's activation edit stays refused; a style edit is taken
    inst = _inst(m, "g_synthesis.blocks.8x8")
    inst.edit_layer("g_synthesis.blocks.8x8", offset=torch.ones(1, 512, 8, 8, device=DEV))
    with pytest.raises(NotImplementedError, match="cannot be propagated"):
        m.forward(z)
    inst.close()
    m.forward(z)
