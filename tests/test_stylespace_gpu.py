"""StyleGAN2 style space on the device: the rows of every modulation layer ('*.conv.modulation') against the unmodified
reference (oracle/gen_golden_stylespace.py) and fp64, partial_forward to a style layer without a synthesis launch, forward with
style hooks bit-identical to forward without them, style edits against the reference and fp64, the notebook strip flow,
get_or_compute on style layers, and the refused sub-module hooks."""
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from oracle import ganspace_oracle as go
from oracle import stylespace_oracle as so

pytestmark = pytest.mark.gpu

MAP_TOL = 2e-5         # the mapping network's bar (test_kernels_gpu.py): one fp32 product of K = 512 per layer
COS_TOL, RATIO_TOL, REL_TOL = 0.999, 1e-3, 1e-3
SUB = 16               # the fixture's images keep every 16th pixel each way (oracle/gen_golden_stylespace.py)
DEV = torch.device("cuda:0")


def _perturb(model):
    """oracle/stylespace_oracle.perturb on the module tree (gen_golden_r2.py G11's values)."""
    convs, rgbs = model.chain_layers()
    with torch.no_grad():
        for i, (_, m) in enumerate(convs):
            m.noise.weight.fill_(0.1 * (i + 1))
            m.activate.bias.copy_((0.1 * torch.sin(torch.arange(m.activate.bias.shape[0], dtype=torch.float32) + i)).to(DEV))
        for j, (_, m) in enumerate(rgbs):
            m.bias.copy_((0.05 * torch.tensor([1.0, -2.0, 3.0]).view(1, 3, 1, 1) * (j + 1)).to(DEV))


@pytest.fixture(scope="module")
def ka(golden):
    return golden("stylespace_known_answers.npz")


@pytest.fixture(scope="module")
def model():
    from ganspace_b200.models import StyleGAN2
    m = StyleGAN2(DEV, "ffhq", random_init=1234)
    _perturb(m.model)
    m.use_z()
    return m


@pytest.fixture(scope="module")
def params():
    return so.perturb(go.synthesis_random_init(1234, 1024, upto="convs.15"))


def _inst(model, layers):
    from ganspace_b200.models import get_instrumented_model
    return get_instrumented_model("StyleGAN2", "ffhq", layers, DEV, model=model, use_w=False)


def _names(model):
    return [t[0] for t in model.model.style_layers()]


def test_style_rows_vs_reference(ka, model):
    """Every S layer, retained from forward, for four latents and for a list of 18 per-layer latents."""
    names = _names(model)
    inst = _inst(model, names)
    model.forward(torch.tensor(ka["z4"], device=DEV))
    got4 = {k: v.cpu().numpy() for k, v in inst.retained_features().items()}
    model.forward([torch.tensor(z, device=DEV) for z in ka["z18"]])
    got18 = {k: v.cpu().numpy() for k, v in inst.retained_features().items()}
    inst.close()
    for name in names:
        key = name.replace(".", "_")
        for got, ref in ((got4[name], ka["s4_" + key]), (got18[name], ka["s18_" + key])):
            assert got.shape == ref.shape, name
            assert np.abs(got - ref).max() < MAP_TOL * max(1.0, np.abs(ref).max()), name


@pytest.mark.parametrize("n", [100, 130])
@pytest.mark.parametrize("w_layers", [1, 18])
def test_style_rows_vs_fp64(model, params, n, w_layers):
    """gsb_synthesis_styles on every element of every S layer, below and above the 128-row switch of gsb_linear_forward."""
    w = torch.tensor(np.random.RandomState(n + w_layers).standard_normal((w_layers, n, 512)).astype(np.float32), device=DEV)
    syn = model._synthesis(17)
    table = model.model.style_layers()
    S = syn.styles(w, range(len(table)))
    convs, rgbs = model.model.chain_layers()
    conv_idx = {f"{n}.conv.modulation": i for i, (n, _) in enumerate(convs)}
    rgb_idx = {f"{n}.conv.modulation": j for j, (n, _) in enumerate(rgbs)}
    wn = w.double().cpu().numpy()
    for name, k, entry, width in table:
        got = S[k].cpu().numpy()
        P = list(params["layers"].values())[conv_idx[name]] if name in conv_idx else params["to_rgbs"][rgb_idx[name]]
        ref = so.modulation_forward(wn[min(entry, w_layers - 1)], P["mod_weight"], P["mod_bias"])
        assert got.shape == (n, width), name
        assert np.abs(got - ref).max() < MAP_TOL * max(1.0, np.abs(ref).max()), (name, np.abs(got - ref).max())


def test_partial_forward_to_style_layer_runs_no_synthesis(model):
    from ganspace_b200 import _native
    syn = model._synthesis(17)
    keys = {t[0]: k for k, t in enumerate(model.model.style_layers())}
    for layer in ("convs.4.conv.modulation", "to_rgbs.2.conv.modulation", "convs.12.conv.modulation", "conv1.conv.modulation"):
        inst = _inst(model, layer)
        z = model.sample_latent(200, seed=9)
        _native.instrument.reset()
        model.partial_forward(z, layer)
        assert "synthesis" not in _native.instrument.rows, layer
        got = inst.retained_features()[layer]
        w = model.model.style(z)
        k = keys[layer]
        assert torch.equal(got, syn.styles(w[None], [k])[k]), layer
        inst.close()


def test_forward_with_style_hooks_is_bit_identical(model):
    z = model.sample_latent(3, seed=11)
    plain = model.forward(z)
    inst = _inst(model, ["convs.8"])
    model.forward(z)
    act = inst.retained_features()["convs.8"].clone()
    inst.retain_layers(_names(model))
    assert torch.equal(model.forward(z), plain)
    assert torch.equal(inst.retained_features()["convs.8"], act)
    inst.edit_layer("convs.5.conv.modulation", offset=torch.zeros(1, 512, device=DEV))
    inst.edit_layer("to_rgbs.2.conv.modulation", offset=torch.zeros(3, 512, device=DEV))
    assert torch.equal(model.forward(z), plain)
    assert torch.equal(inst.retained_features()["convs.8"], act)
    inst.close()


def test_styled_run_is_the_chain_run(model):
    """gsb_synthesis_forward_styled on gsb_synthesis_styles' rows equals gsb_synthesis_forward, with and without ToRGBs."""
    syn = model._synthesis(17)
    # the whole chain at a small batch; to convs.7 (64 x 64) at a batch past the 128-row switch of the style GEMMs
    for n, Lw, n_run in ((5, 18, 17), (130, 1, 9)):
        n_rgb = (n_run - 1) // 2 + 1
        w = torch.tensor(np.random.RandomState(n).standard_normal((Lw, n, 512)).astype(np.float32), device=DEV)
        S = syn.styles(w, [syn.slot_of["conv", l] for l in range(n_run)] + [syn.slot_of["rgb", j] for j in range(n_rgb)])
        act, img = syn.forward(w, n_run, n_rgb=n_rgb)
        act2, img2 = syn.forward_styled(S, n_run, n_rgb=n_rgb)
        assert torch.equal(act, act2) and torch.equal(img, img2)
        if Lw == 1:
            a5 = syn.forward(w[0], 6)[0]
            assert torch.equal(a5, syn.forward_styled(S, 6)[0])
    model.check_numerics()


@pytest.mark.parametrize("which", ["offset", "ablate"])
def test_edited_images_vs_reference(ka, model, which):
    inst = _inst(model, "convs.5.conv.modulation")
    if which == "offset":
        inst.edit_layer("convs.5.conv.modulation", offset=torch.tensor(ka["edit_offset"], device=DEV))
    else:
        inst.edit_layer("to_rgbs.2.conv.modulation", ablation=0.5, replacement=torch.tensor(ka["edit_replacement"], device=DEV))
    img = model.forward(torch.tensor(ka["z4"][:2], device=DEV)).cpu().numpy()
    inst.close()
    ref = ka[f"img_{which}_sub"]
    scale = np.abs(ref - 0.5).max()
    assert np.abs(img[:, :, ::SUB, ::SUB] - ref).max() < 1e-3 * scale, np.abs(img[:, :, ::SUB, ::SUB] - ref).max() / scale
    assert abs((img.astype(np.float64) ** 2).sum() - ka[f"img_{which}_sum"][1]) < 2e-3 * ka[f"img_{which}_sum"][1]
    # the edit shows: the unedited image is far from this one
    assert np.abs(ka["img4_sub"][:2] - ref).max() > 1e-2 * scale


def test_edited_image_vs_fp64(model, params):
    """One sample: forward with an S edit on convs.2 against the fp64 oracle rendering the device's own edited styles."""
    names = _names(model)
    inst = _inst(model, names)
    z = model.sample_latent(1, seed=12)
    delta = torch.tensor(np.random.RandomState(3).standard_normal((1, 512)).astype(np.float32), device=DEV)
    inst.edit_layer("convs.2.conv.modulation", offset=delta)
    img = model.forward(z).double().cpu().numpy()
    S = {k: v.double().cpu().numpy() for k, v in inst.retained_features().items()}      # retained before the edit
    inst.close()
    S["convs.2.conv.modulation"] = S["convs.2.conv.modulation"] + delta.double().cpu().numpy()
    ref, _ = so.render(S, params, go.fixed_noise(0, 1024))
    ref = 0.5 * (ref + 1)
    scale = np.abs(ref - 0.5).max()
    assert np.abs(img - ref).max() < 1e-3 * scale, np.abs(img - ref).max() / scale


def test_style_edit_reaches_downstream_activation(model):
    """An S edit upstream of a retained StyledConv changes that activation, and partial_forward to it equals forward."""
    z = model.sample_latent(4, seed=13)
    inst = _inst(model, ["convs.8"])
    model.forward(z)
    plain = inst.retained_features()["convs.8"].clone()
    inst.edit_layer("convs.5.conv.modulation", offset=torch.full((1, 512), 0.3, device=DEV))
    model.forward(z)
    edited = inst.retained_features()["convs.8"].clone()
    assert (edited - plain).abs().max() > 1e-2 * plain.abs().max()
    model.partial_forward(z, "convs.8")
    assert torch.equal(inst.retained_features()["convs.8"], edited)
    inst.close()


def test_each_style_hook_fires_once(model):
    calls = {}
    mods = dict(model.model.named_modules())
    names = ["conv1.conv.modulation", "to_rgb1.conv.modulation", "convs.3.conv.modulation", "to_rgbs.4.conv.modulation",
             "convs.15.conv.modulation"]
    inst = _inst(model, ["convs.6"])
    handles = [mods[n].register_forward_hook(lambda m, i, o, n=n: calls.__setitem__(n, calls.get(n, 0) + 1)) for n in names]
    z = model.sample_latent(2, seed=14)
    model.forward(z)
    assert calls == {n: 1 for n in names}
    calls.clear()
    model.partial_forward(z, "convs.6")        # runs conv1 .. convs.6 and to_rgb1 .. to_rgbs.2
    assert calls == {n: 1 for n in names[:3]}
    inst.close()
    for h in handles:
        h.remove()


def test_notebook_activation_strip_on_style_layer(model):
    """notebook_utils._create_strip_batch_sigma, mode 'activation', center=True, restated: retain, centre along a component,
    per-frame offsets [B, cin], sample_np.  Equals forward on explicitly edited styles."""
    layer = "convs.3.conv.modulation"
    inst = _inst(model, layer)
    z_single = model.sample_latent(1, seed=15)
    comp = torch.tensor(np.random.RandomState(4).standard_normal((1, 512)).astype(np.float32), device=DEV)
    act_mean = torch.tensor(np.random.RandomState(5).standard_normal((1, 512)).astype(np.float32), device=DEV)
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
    # explicitly: the styles of the batch, edited, through the styled chain
    syn = model._synthesis(17)
    keys = {t[0]: k for k, t in enumerate(model.model.style_layers())}
    w = model.model.style(z_single.repeat_interleave(B, axis=0))[None]
    S = syn.styles(w, keys.values())
    S[keys[layer]] = S[keys[layer]] + (delta * act_stdev - zero)
    _, img = syn.forward_styled(S, 17, want_act=False, n_rgb=9)
    ref = np.clip((0.5 * (img + 1)).cpu().numpy(), 0.0, 1.0)
    assert np.array_equal(frames, ref)
    assert np.abs(frames[0] - frames[-1]).max() > 1e-2


def _run(layer, n, b, c, use_w, est="ipca"):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model, StyleGAN2
    model = StyleGAN2(DEV, "ffhq", random_init=1234)
    _perturb(model.model)
    inst = get_instrumented_model("StyleGAN2", "ffhq", layer, DEV, model=model, use_w=use_w)
    cfg = Config(model="StyleGAN2", layer=layer, output_class="ffhq", components=c, n=n, batch_size=b, use_w=use_w, estimator=est)
    with tempfile.TemporaryDirectory() as tmp:
        path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        with np.load(path, allow_pickle=False) as data:
            out = {k: data[k] for k in data.files}
    inst.close()
    return out, path.name


def _check(cmp):
    assert cmp["min_signed_cos"] >= COS_TOL and cmp["max_abs_dvar_ratio"] <= RATIO_TOL, cmp
    assert cmp["min_lat_signed_cos"] >= COS_TOL, cmp
    assert cmp["act_mean_rel"] < REL_TOL and cmp["act_stdev_rel"] < REL_TOL and cmp["random_stdevs_rel"] < REL_TOL, cmp


@pytest.mark.parametrize("fixture,layer,use_w", [
    ("c6_stylegan2_ffhq_convs1mod_z_n4000_b500_c16.npz", "convs.1.conv.modulation", False),
    ("c6_stylegan2_ffhq_torgb1mod_w_n4000_b500_c16.npz", "to_rgb1.conv.modulation", True),
])
def test_get_or_compute_vs_reference_golden(golden, oracle, fixture, layer, use_w):
    g = golden(fixture)
    out, name = _run(layer, 4000, 500, 16, use_w)
    assert name == str(g["dump_name"])
    for k in ("act_comp", "act_mean", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio", "random_stdevs"):
        assert out[k].shape == g[k].shape and out[k].dtype == g[k].dtype, k
    _check(oracle.compare_npz(out, g))


def test_get_or_compute_fbpca_vs_oracle(oracle, mapping_weights, params):
    """--est fbpca on convs.3.conv.modulation (W space, regression) against the oracle's fbpca restatement (fp64 Gram form)."""
    from oracle import fbpca_oracle as fbo
    ws, bs = mapping_weights
    P = params["layers"]["convs.3"]
    sample = lambda s, B_: go.mapping_forward(go.standard_normal_f32(s, 512 * B_).reshape(B_, 512), ws, bs)
    activate = lambda w: so.modulation_forward(w, P["mod_weight"], P["mod_bias"]).astype(np.float32)
    ref = fbo.compute_path_fbpca(sample, activate, 512, 512, 4000, 500, 16, False, use_w=True)
    out, _ = _run("convs.3.conv.modulation", 4000, 500, 16, True, est="fbpca")
    _check(oracle.compare_npz(out, fbo.sign_normalise(ref)))


def test_sub_module_hooks_are_refused(model):
    from ganspace_b200.models import get_instrumented_model
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    z = model.sample_latent(1, seed=16)
    guarded = model.model.unhookable_layers()
    assert len(guarded) == 76
    for name in guarded:
        with pytest.raises(NotImplementedError, match="hookable synthesis layers"):
            get_instrumented_model("StyleGAN2", "ffhq", name, DEV, model=model, use_w=False)
        inst = InstrumentedModel(model)
        inst.retain_layer(name)
        with pytest.raises(NotImplementedError, match=name.replace(".", r"\.")):
            model.partial_forward(z, "convs.8")
        with pytest.raises(NotImplementedError, match=name.replace(".", r"\.")):
            model.forward(z)
        inst.close()
    # activation edits on StyledConv / ToRGB layers stay refused
    for layer, shape in (("convs.3", (1, 512, 16, 16)), ("to_rgbs.1", (1, 3, 16, 16))):
        inst = _inst(model, layer)
        inst.edit_layer(layer, offset=torch.ones(shape, device=DEV))
        with pytest.raises(NotImplementedError):
            model.forward(z)
        inst.close()
    # nothing is left hooked: a plain forward works
    model.forward(z)
