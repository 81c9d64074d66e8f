"""Activation-mode component strips on the GPU (ganspace_b200.strips with mode 'activation' / 'both', csrc/strips.cu
gsb_strip_offsets): the offsets kernel against fp64, the frames against the reference's loop over ``inst.edit_layer`` and the
package's own sample_np (tests/act_strip_reference.py), the keyword options, the refusals and the state a call leaves, on
StyleGAN2, StyleGAN and BigGAN-deep with random-init weights."""
import numpy as np
import pytest
import torch

from ganspace_b200 import _native
from ganspace_b200.netdissect.nethook import InstrumentedModel
from ganspace_b200.strips import create_strip, create_strip_centered
from act_strip_reference import reference_act_strip, strip_offsets_fp64

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
OFFSET_TOL = 1e-6       # max |diff| / max |fp64| of the offsets (a few fp32 roundings)
# centred frames: the centring's dot product (of the activation in mode 'activation', of the latent in 'both') is summed in
# another order than torch.sum's, a last-bit change of the edit (test_centred_offsets_match_torch); what the generator makes of
# it, max |diff| on the [0, 1] scale, measured on an H100 80GB HBM3 (random init 1234) over the cases below: StyleGAN2 1.0e-5,
# StyleGAN 3.6e-5, BigGAN-512 9.8e-2 (generator.gen_z in mode 'activation': its dot product runs over 32768 values, and the
# random-init chain amplifies a last-bit change of its output the most; 8.2e-3 on generator.layers.3.bn_2.scale).  The bounds
# are those with a margin.
CENTRED_TOL = {"StyleGAN2": 5e-5, "StyleGAN": 2e-4, "BigGAN": 0.15}


# ---- the offsets kernel --------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("n_lat,n_comp,W", [(1, 1, 512), (3, 4, 1024), (6, 3, 32768), (2, 14, 4608)])
@pytest.mark.parametrize("center", [False, True], ids=["plain", "centred"])
def test_strip_offsets_fp64(n_lat, n_comp, W, center):
    g = torch.Generator().manual_seed(n_lat * 100 + n_comp * 10 + W + center)
    acts = torch.randn(n_lat, W, generator=g) * 0.7 + 0.2
    comps = torch.randn(n_comp, W, generator=g) / np.sqrt(W)
    stdev = torch.rand(n_comp, generator=g) * 3 + 0.5
    mean = torch.randn(W, generator=g) * 0.1
    n_frames = 5
    sigmas = torch.from_numpy(np.linspace(-3.0, 3.0, n_frames).astype(np.float32))
    d = [t.to(DEV).contiguous() for t in (acts, comps, stdev, mean, sigmas)]
    F = n_comp * n_lat * n_frames
    for f0, n in ((0, F), (F // 3, F - F // 3), (F - 1, 1)):
        got = _native.strip_offsets(d[0], d[1], d[2], d[3] if center else None, d[4], n_lat, f0, n, center)
        ref = strip_offsets_fp64(acts.numpy(), comps.numpy(), stdev.numpy(), mean.numpy(), sigmas.numpy(), n_lat, f0, n, center)
        out = got.cpu().numpy()
        assert out.shape == ref.shape == (n, W)
        err = np.abs(out - ref).max() / np.abs(ref).max()
        assert err <= OFFSET_TOL, (f0, n, err)
        assert torch.equal(got, _native.strip_offsets(d[0], d[1], d[2], d[3] if center else None, d[4], n_lat, f0, n, center))
        if not center:
            # the reference's torch expression delta * act_stdev - 0, bit for bit
            f = torch.arange(f0, f0 + n, device=DEV)
            c, k = f // n_frames // n_lat, f % n_frames
            assert torch.equal(got, d[1][c] * d[4][k][:, None] * d[2][c][:, None] - 0)


def test_strip_offsets_refuses_bad_ranges():
    x = torch.zeros(1, 8, device=DEV)
    one = torch.ones(1, device=DEV)
    with pytest.raises(_native.NativeError, match="frames"):
        _native.strip_offsets(None, x, one, None, one, 1, 0, 2, False)
    with pytest.raises(_native.NativeError, match="frames"):
        _native.strip_offsets(None, x, one, None, one, 1, -1, 1, False)


# ---- models --------------------------------------------------------------------------------------------------------------
_MODELS = {}


def _model(name):
    from ganspace_b200.models import ProGAN, StyleGAN, StyleGAN2, stylegan
    from ganspace_b200.models.biggan import BigGAN
    if name not in _MODELS:
        if name == "StyleGAN2":
            m = StyleGAN2(DEV, "ffhq", random_init=1234)
        elif name == "StyleGAN":
            m = StyleGAN(DEV, "bedrooms", random_init=1234)
            stylegan.synthesis_fill(m.model, 7)
        elif name == "BigGAN":
            m = BigGAN(DEV, 512, "husky", random_init=1234)
        else:
            m = ProGAN(DEV, "bedroom", random_init=1234)
        m.eval()
        _MODELS[name] = m
    return _MODELS[name]


@pytest.fixture(scope="module", autouse=True)
def _release_models():
    yield
    _MODELS.clear()
    torch.cuda.empty_cache()


def _inst(name, space):
    model = _model(name)
    if hasattr(model, "use_w"):
        model.use_w() if space == "W" else model.use_z()
    return InstrumentedModel(model)


def _values(inst, layer, x):
    """The layer's unedited values of latents x, [n, W]."""
    inst.close()
    inst.retain_layer(layer)
    with torch.no_grad():
        inst.model.partial_forward(x, layer)
    v = inst.retained_layer(layer).clone()
    inst.close()
    return v.reshape(v.shape[0], -1)


def _edit_inputs(inst, layer, n_comp):
    """Six latents, latent and activation components with stdevs and means, from 64 samples."""
    model = inst.model
    lats = [model.sample_latent(1, seed=100 + i).reshape(1, -1) for i in range(6)]
    D = lats[0].shape[1]
    many = model.sample_latent(64, seed=5).reshape(64, D)
    acts = _values(inst, layer, many)
    W = acts.shape[1]
    g = torch.Generator().manual_seed(11)
    z_comp = (torch.randn(n_comp, D, generator=g) / np.sqrt(D)).to(DEV)
    x_comp = (torch.randn(n_comp, W, generator=g) / np.sqrt(W)).to(DEV)
    scale = torch.linspace(1.5, 0.5, n_comp, device=DEV)
    return dict(lats=lats, z_comp=z_comp, x_comp=x_comp, lat_stdev=many.std(0).mean() * scale,
                act_stdev=acts.std(0).mean() * scale, lat_mean=many.mean(0, keepdim=True), act_mean=acts.mean(0, keepdim=True))


def _max_diff(a, b):
    return max(float(np.abs(np.asarray(x, np.float64) - np.asarray(y, np.float64)).max()) for fa, fb in zip(a, b)
               for x, y in zip(fa, fb))


def _batch_spread(model, lats):
    """The most a frame changes with the batch it is rendered in (one batch, groups of 5, one by one); 0: batch-invariant."""
    w = torch.cat(lats, 0)
    full = model.sample_np(w).reshape(len(w), -1)
    parts = np.concatenate([model.sample_np(w[i:i + 5]).reshape(-1, full.shape[1]) for i in range(0, len(w), 5)])
    ones = np.stack([model.sample_np(w[i:i + 1]).reshape(-1) for i in range(len(w))])
    return float(max(np.abs(full - parts).max(), np.abs(full - ones).max()))


LAYERS = [
    ("StyleGAN2", "style", "Z"),
    ("StyleGAN2", "convs.3.conv.modulation", "W"),
    ("StyleGAN2", "to_rgbs.1.conv.modulation", "Z"),
    ("StyleGAN", "g_mapping", "Z"),
    ("StyleGAN", "g_synthesis.blocks.16x16.epi1.style_mod.lin", "W"),
    ("BigGAN", "generator.gen_z", "Z"),
    ("BigGAN", "generator.layers.3.bn_2.scale", "Z"),
]


@pytest.mark.parametrize("name,layer,space", LAYERS, ids=[f"{n}-{l}-{s}" for n, l, s in LAYERS])
@pytest.mark.parametrize("n_lat,num_frames", [(1, 7), (6, 3)], ids=["batch-over-sigma", "batch-over-latents"])
@pytest.mark.parametrize("mode", ["activation", "both"])
def test_frames_match_reference_loop(name, layer, space, n_lat, num_frames, mode):
    inst = _inst(name, space)
    model = inst.model
    assert model.edit_reaches_image(layer)
    e = _edit_inputs(inst, layer, 1)
    lats = e["lats"][:n_lat]
    L = model.get_max_latents()
    ls, le = (2, 9) if L > 2 else (0, -1)
    spread = _batch_spread(model, lats + [v + 0.01 for v in lats])
    args = (lats, e["x_comp"], e["z_comp"], e["act_stdev"][0], e["lat_stdev"][0])
    ref = reference_act_strip(inst, mode, layer, *args, None, None, 2.5, ls, le, num_frames, False)
    got = create_strip(inst, mode, layer, *args, 2.5, ls, le, num_frames)
    assert len(got) == n_lat and all(len(s) == num_frames for s in got)
    assert all(f.dtype == np.float32 and f.shape == ref[0][0].shape and f.ndim == 3 for s in got for f in s)
    d = _max_diff(got, ref)
    print(f"{name} {layer} {space} {mode} {n_lat}x{num_frames}: batch spread {spread:.3g}, create_strip max |diff| {d:.3g}")
    assert spread == 0.0, f"the {name} chain gives a latent other bits in another batch (max |diff| {spread:.3g})"
    assert d == 0.0, f"{name} {layer}: frames differ by {d} from the reference loop's"
    ref = reference_act_strip(inst, mode, layer, *args, e["act_mean"], e["lat_mean"], 2.5, ls, le, num_frames, True)
    got = create_strip_centered(inst, mode, layer, *args, e["act_mean"], e["lat_mean"], 2.5, ls, le, num_frames)
    d = _max_diff(got, ref)
    print(f"{name} {layer} {space} {mode} {n_lat}x{num_frames}: create_strip_centered max |diff| {d:.3g}")
    assert d <= CENTRED_TOL[name], f"{name} {layer}: centred frames differ by {d}"
    inst.close()


@pytest.mark.parametrize("name,layer,space", [LAYERS[0], LAYERS[5]], ids=["StyleGAN2-style-Z", "BigGAN-gen_z"])
def test_centred_offsets_match_torch(name, layer, space):
    """The centred offsets of the kernel and of the reference's torch expression, on the layer's real values, are both within a
    few fp32 roundings of fp64: what differs in the centred frames is the generator's response to the last bits."""
    inst = _inst(name, space)
    e = _edit_inputs(inst, layer, 1)
    acts = _values(inst, layer, torch.cat(e["lats"][:3])).contiguous()
    x, sd, mean = e["x_comp"], e["act_stdev"][:1].contiguous(), e["act_mean"].reshape(-1).contiguous()
    sig = torch.tensor([-2.0, 0.5, 3.0], device=DEV)
    got = _native.strip_offsets(acts, x, sd, mean, sig, 3, 0, 9, True)
    unit = x / torch.sqrt(torch.sum(x ** 2, dim=-1, keepdim=True) + 1e-8)
    dotp = torch.sum((acts - mean) * unit, dim=-1, keepdim=True)
    ref = ((x * sig[:, None] * sd)[None] - (unit * dotp)[:, None]).reshape(9, -1)
    fp64 = strip_offsets_fp64(acts.cpu().numpy(), x.cpu().numpy(), sd.cpu().numpy(), mean.cpu().numpy(), sig.cpu().numpy(), 3, 0, 9,
                              True)
    scale = np.abs(fp64).max()
    err_got = np.abs(got.cpu().numpy() - fp64).max() / scale
    err_ref = np.abs(ref.cpu().numpy() - fp64).max() / scale
    print(f"{name} {layer}: centred offsets against fp64, kernel {err_got:.3g}, torch {err_ref:.3g}")
    assert err_got <= OFFSET_TOL and err_ref <= OFFSET_TOL, (err_got, err_ref)
    inst.close()


def _same(a, b, what):
    d = _max_diff(a, b)
    assert d == 0.0, f"{what}: frames differ by {d}"


@pytest.mark.parametrize("name,layer,space", [LAYERS[1], LAYERS[5]], ids=["StyleGAN2-modulation-W", "BigGAN-gen_z"])
@pytest.mark.parametrize("mode", ["activation", "both"])
def test_components_batch_sizes_uint8(name, layer, space, mode):
    inst = _inst(name, space)
    e = _edit_inputs(inst, layer, 3)
    lats = e["lats"][:2]
    call = lambda x, z, a_sd, l_sd, **kw: create_strip_centered(inst, mode, layer, lats, x, z, a_sd, l_sd, e["act_mean"],
                                                               e["lat_mean"], 2.0, 0, -1, 4, **kw)
    multi = call(e["x_comp"], e["z_comp"], e["act_stdev"], e["lat_stdev"], per_component=True)
    assert len(multi) == 3 and all(len(m) == 2 and len(m[0]) == 4 for m in multi)
    for c in range(3):
        single = call(e["x_comp"][c:c + 1], e["z_comp"][c:c + 1], e["act_stdev"][c], e["lat_stdev"][c])
        _same(multi[c], single, f"{name} component {c}")
    for bs in (1, 7, None):
        forced = call(e["x_comp"], e["z_comp"], e["act_stdev"], e["lat_stdev"], per_component=True, batch_size=bs)
        _same(sum(multi, []), sum(forced, []), f"{name} batch size {bs}")
    f32 = call(e["x_comp"][:1], e["z_comp"][:1], e["act_stdev"][0], e["lat_stdev"][0], batch_size=3)
    u8 = call(e["x_comp"][:1], e["z_comp"][:1], e["act_stdev"][0], e["lat_stdev"][0], batch_size=3, as_uint8=True)
    for sa, sb in zip(f32, u8):
        for a, b in zip(sa, sb):
            assert b.dtype == np.uint8 and np.array_equal(b, np.uint8(a * 255))
    inst.close()


# ---- which layers are taken, and the state a call leaves ------------------------------------------------------------------
def test_edit_reaches_image():
    s2 = _model("StyleGAN2")
    s2.use_z()
    assert all(s2.edit_reaches_image(t[0]) for t in s2.model.style_layers()) and s2.edit_reaches_image("style")
    assert not any(s2.edit_reaches_image(n) for n in ("convs.4", "conv1", "to_rgbs.0", "to_rgb1", "input"))
    s2.use_w()
    assert all(s2.edit_reaches_image(t[0]) for t in s2.model.style_layers()) and not s2.edit_reaches_image("style")
    s1 = _model("StyleGAN")
    s1.use_z()
    assert all(s1.edit_reaches_image(t[0]) for t in s1.model.style_layers()) and s1.edit_reaches_image("g_mapping")
    assert not any(s1.edit_reaches_image(n) for n in s1.model.block_names())
    s1.use_w()
    assert all(s1.edit_reaches_image(t[0]) for t in s1.model.style_layers()) and not s1.edit_reaches_image("g_mapping")
    bg = _model("BigGAN")
    assert bg.edit_reaches_image("generator.gen_z") and all(bg.edit_reaches_image(n) for n, _ in bg.model.style_layers())
    assert not any(bg.edit_reaches_image(f"generator.layers.{k}") for k in range(len(bg.model.generator.layers)))
    pg = _model("ProGAN")
    assert not any(pg.edit_reaches_image(n) for n in pg.model.block_names())


@pytest.mark.parametrize("name,layer,space", [("StyleGAN2", "convs.4", "Z"), ("StyleGAN2", "style", "W"), ("ProGAN", "layer3", "Z"),
                                              ("BigGAN", "generator.layers.2", "Z")])
@pytest.mark.parametrize("mode", ["activation", "both"])
def test_refusals_leave_inst_untouched(name, layer, space, mode):
    inst = _inst(name, space)
    model = inst.model
    z = model.sample_latent(1, seed=3).reshape(1, -1)
    inst.retain_layer(layer)
    with pytest.raises(NotImplementedError, match="cannot be propagated"):
        create_strip(inst, mode, layer, [z], torch.zeros(1, 8, device=DEV), torch.zeros_like(z), 1.0, 1.0, 2.0, 0, -1, 3)
    assert layer in inst.retained_features() and inst._handles, "inst was closed before the refusal"
    inst.close()


@pytest.mark.parametrize("name,layer,space", [LAYERS[0], LAYERS[4], LAYERS[6]], ids=["StyleGAN2-style-Z", "StyleGAN-lin-W",
                                                                                    "BigGAN-bn"])
def test_call_leaves_no_hook_and_no_edit(name, layer, space):
    inst = _inst(name, space)
    model = inst.model
    e = _edit_inputs(inst, layer, 1)
    z = torch.cat(e["lats"][:2])
    with torch.no_grad():
        before = model.forward(z).cpu()
    create_strip_centered(inst, "activation", layer, e["lats"][:2], e["x_comp"], None, e["act_stdev"][0], None, e["act_mean"], None,
                          2.0, 0, -1, 3)
    assert not inst._handles and not inst._offset and not inst._retained
    assert all(not m._forward_hooks for _, m in model.named_modules())
    with torch.no_grad():
        after = model.forward(z).cpu()
    assert torch.equal(before, after)
