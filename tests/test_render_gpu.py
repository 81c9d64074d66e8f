"""Full synthesis to RGB (SURVEY.md section 8 rows a5 / f2): every StyledConv of the 1024^2 generator (512 ... 32 channels), the
ToRGB / skip chain, StyleGAN2.forward with one latent, per-layer latents and style mixing -- against known answers written by
the unmodified reference (oracle/gen_golden_r2.py G11), plus the reference's own test invariants (tests/partial_forward_test.py:
partial == full at the hooked layer; tests/layerwise_z_test.py: forward(z) == forward(n_latents * [z])).
convs.10 .. convs.15 are checked against the reference's full forward: its partial_forward never reaches them (substring match on
the layer name, wrappers.py:241-246 -- INTEGRATION.md section 3).  Every StyledConv and every ToRGB is also checked on its own
against fp64, on every element, fed the chain's own input."""
import numpy as np
import pytest
import torch

from layer_parity import assert_spans_chunks, check, nhwc_to_nchw, parity_batch, stylegan2_chunk_samples
from oracle import ganspace_oracle as oracle_go

pytestmark = pytest.mark.gpu

ACT_TOL = 5e-4         # max |diff| / max |ref| after up to 17 fused layers (fp16 hi/lo tensor-core products, ~1e-5 per layer)
LAYER_TOL = 9e-6       # one StyledConv fed the chain's own input, against fp64, per sample: ~3x the worst measured
RGB_TOL = 2e-6         # one ToRGB (fp32 1x1 conv + skip) fed the chain's own inputs, against fp64, per sample: ~3x the worst measured


def _perturb(model, conv_names, rgb_names):
    mods = dict(model.named_modules())
    for i, name in enumerate(conv_names):
        with torch.no_grad():
            mods[name].noise.weight.fill_(0.1 * (i + 1))
            b = mods[name].activate.bias
            b.copy_((0.1 * torch.sin(torch.arange(b.shape[0], dtype=torch.float32) + i)).to(b.device))
    for i, name in enumerate(rgb_names):
        with torch.no_grad():
            mods[name].bias.copy_((0.05 * torch.tensor([1.0, -2.0, 3.0]).view(1, 3, 1, 1) * (i + 1)).to(mods[name].bias.device))


@pytest.fixture(scope="module")
def deep(golden):
    from conftest import GOLDEN
    if not (GOLDEN / "synthesis_deep_known_answers.npz").exists():
        pytest.skip("fixture synthesis_deep_known_answers.npz not generated")
    return golden("synthesis_deep_known_answers.npz")


@pytest.fixture(scope="module")
def model(deep):
    from ganspace_b200.models import StyleGAN2
    m = StyleGAN2(torch.device("cuda:0"), "ffhq", random_init=1234)
    _perturb(m.model, [str(x) for x in deep["conv_names"]], [str(x) for x in deep["rgb_names"]])
    return m


def _sub(act):
    step = max(1, act.shape[-1] // 32)
    return act[:, ::max(1, act.shape[1] // 16), ::step, ::step]


CONV_NAMES = ["conv1"] + [f"convs.{i}" for i in range(16)]
RGB_NAMES = ["to_rgb1"] + [f"to_rgbs.{j}" for j in range(8)]


@pytest.fixture(scope="module")
def perturbed():
    """The 1024^2 generator with non-zero noise weights and activation biases in every StyledConv and non-zero ToRGB biases."""
    from ganspace_b200.models import StyleGAN2
    m = StyleGAN2(torch.device("cuda:0"), "ffhq", random_init=1234)
    _perturb(m.model, CONV_NAMES, RGB_NAMES)
    return m


def _np(t):
    return t.detach().float().cpu().numpy()


def _per_layer_latents(seed, n):
    return np.random.RandomState(seed).standard_normal((18, n, 512)).astype(np.float32)


@pytest.mark.parametrize("name", CONV_NAMES)
def test_each_styled_conv_vs_fp64(perturbed, name):
    """StyledConv ``name`` (layer l of the chain, latent l) fed the chain's own output of layer l-1 (the constant input for
    conv1) against the oracle's shared-weight form in fp64, on every element of a batch that spans two sample chunks of the
    layer, one latent per sample and layer (gsb_synthesis_forward).  Measured on an H100 80GB HBM3 (700 W): worst
    2.8e-6 (conv1), 1.7e-6 to 2.6e-6 for the 512-channel layers, under 1.4e-6 from convs.9 on."""
    m = perturbed
    l = CONV_NAMES.index(name)
    mod = ([m.model.conv1] + list(m.model.convs))[l]
    syn = m._synthesis(len(CONV_NAMES))
    res_in = 4 if l == 0 else syn.shapes[l - 1][0]
    spc = stylegan2_chunk_samples(res_in)
    n = parity_batch(spc)
    assert_spans_chunks(n, spc)
    w = _per_layer_latents(300 + l, n)
    wd = torch.from_numpy(w).to(m.device)
    if l == 0:
        x = np.repeat(_np(m.model.input.input).astype(np.float64), n, axis=0)
    else:
        x = nhwc_to_nchw(syn.forward(wd, l)[0], n, *syn.shapes[l - 1])
    got = nhwc_to_nchw(syn.forward(wd, l + 1)[0], n, *syn.shapes[l])
    r = syn.shapes[l][0]
    L = dict(weight=_np(mod.conv.weight[0]), mod_weight=_np(mod.conv.modulation.weight), mod_bias=_np(mod.conv.modulation.bias),
             noise_weight=float(mod.noise.weight), act_bias=_np(mod.activate.bias), upsample=mod.conv.upsample)
    ref = oracle_go.styled_conv_shared(x, w[l], L, _np(m.noise[l]).reshape(r, r), dtype=np.float64)
    check(got, ref, LAYER_TOL, name, chunk_of=spc)
    m.check_numerics()


@pytest.mark.parametrize("name", RGB_NAMES)
def test_each_to_rgb_vs_fp64(perturbed, name):
    """ToRGB ``name`` (j; it follows layer 0 for j = 0, else layer 2j, and reads latent 2j + 1) fed the chain's own StyledConv
    output and the chain's own previous skip image, against to_rgb_forward in fp64 (modulated 1x1 conv without demodulation,
    bias, [1,3,3,1] up-sampled skip), on every element of a batch that spans two chunks of the layer it is fused into.
    Measured on an H100 80GB HBM3 (700 W): worst 6.3e-7 (to_rgb1), 2.2e-7 to 4.7e-7 for the others."""
    m = perturbed
    j = RGB_NAMES.index(name)
    lj = 2 * j
    mods = [m.model.to_rgb1] + list(m.model.to_rgbs)
    rgbs = [t.describe() for t in mods]
    syn = m._synthesis(len(CONV_NAMES))
    spc = stylegan2_chunk_samples(4 if lj == 0 else syn.shapes[lj - 1][0])
    n = parity_batch(spc)
    assert_spans_chunks(n, spc)
    w = _per_layer_latents(400 + j, n)
    wd = torch.from_numpy(w).to(m.device)
    act, img = syn.forward(wd, lj + 1, n_rgb=j + 1)
    x = nhwc_to_nchw(act, n, *syn.shapes[lj])
    got = img.permute(0, 3, 1, 2).double().cpu().numpy()
    skip = None
    if j > 0:
        skip = syn.forward(wd, lj - 1, want_act=False, n_rgb=j)[1].permute(0, 3, 1, 2).double().cpu().numpy()
    R = {k: _np(v) for k, v in rgbs[j].items()}
    R["weight"] = R.pop("conv_weight")
    ref = oracle_go.to_rgb_forward(x, w[lj + 1], R, skip, dtype=np.float64)
    check(got, ref, RGB_TOL, name, chunk_of=spc)
    m.check_numerics()


def test_deep_layers_and_to_rgb_known_answers(deep, model):
    from ganspace_b200.models import get_instrumented_model
    dev = torch.device("cuda:0")
    model.use_z()
    z = torch.tensor(deep["z"]).to(dev)
    layers = [f"convs.{i}" for i in range(5, 16)] + [str(x) for x in deep["rgb_names"]]
    for layer in layers:
        inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=model, use_w=False)
        model.partial_forward(z[:1], layer)
        act = inst.retained_features()[layer].float().cpu().numpy()
        key = layer.replace(".", "_")
        assert tuple(act.shape) == tuple(deep[f"shape_{key}"]), layer
        ref = deep[f"act_{key}_sub"]
        scale = np.abs(ref).max()
        assert np.abs(_sub(act) - ref).max() < ACT_TOL * scale, (layer, np.abs(_sub(act) - ref).max() / scale)
        s1, s2 = act.astype(np.float64).sum(), (act.astype(np.float64) ** 2).sum()
        assert abs(s2 - deep[f"sum_{key}"][1]) < 2e-3 * deep[f"sum_{key}"][1], layer
        assert abs(s1 - deep[f"sum_{key}"][0]) < 2e-3 * np.sqrt(deep[f"sum_{key}"][1] * act.size), layer
        inst.close()
    model.check_numerics()


def test_forward_images_vs_reference(deep, model):
    dev = torch.device("cuda:0")
    model.use_z()
    z = torch.tensor(deep["z"]).to(dev)
    img = model.forward(z).float().cpu().numpy()
    assert img.shape == (2, 3, 1024, 1024)
    ref = deep["img_sub"]
    scale = np.abs(ref - 0.5).max()
    assert np.abs(img[:, :, ::4, ::4] - ref).max() < 1e-3 * scale, np.abs(img[:, :, ::4, ::4] - ref).max() / scale
    assert abs((img.astype(np.float64) ** 2).sum() - deep["img_sum"][1]) < 2e-3 * deep["img_sum"][1]
    # one latent per layer (tests/layerwise_z_test.py:59-69) and style mixing with a per-layer list
    n_lat = model.get_max_latents()
    same = model.forward([z[:1]] * n_lat).float().cpu().numpy()
    assert np.abs(same - img[:1]).max() < 1e-5 * max(1.0, np.abs(img).max())
    mixed = model.forward([z[:1]] * 8 + [z[1:2]] * (n_lat - 8)).float().cpu().numpy()
    refm = deep["mixed_sub"]
    assert np.abs(mixed[:, :, ::4, ::4] - refm).max() < 1e-3 * np.abs(refm - 0.5).max()
    model.check_numerics()


def test_partial_forward_equals_forward_at_hooked_layer(model):
    """The reference's tests/partial_forward_test.py:112-121 invariant on random-init weights, plus latent lists in partial_forward
    (tests/layerwise_z_test.py:51-56) and the batch-size probe without a layer (decomposition.get_max_batch_size)."""
    from ganspace_b200.decomposition import get_max_batch_size
    from ganspace_b200.models import get_instrumented_model
    dev = torch.device("cuda:0")
    model.use_z()
    for layer in ("convs.0", "convs.7", "to_rgbs.2"):
        inst = get_instrumented_model("StyleGAN2", "ffhq", layer, dev, model=model, use_w=False)
        z = model.sample_latent(3, seed=5)
        model.partial_forward(z, layer)
        a = inst.retained_features()[layer].clone()
        model.forward(z)
        b = inst.retained_features()[layer].clone()
        assert torch.equal(a, b), layer
        model.partial_forward(model.get_max_latents() * [z], layer)
        c = inst.retained_features()[layer]
        assert torch.allclose(a, c, rtol=0, atol=1e-6 * float(a.abs().max())), layer
        # negative control (partial_forward_test.py:93-98): different latents differ
        model.partial_forward(model.sample_latent(3, seed=6), layer)
        assert not torch.equal(a, inst.retained_features()[layer])
        inst.close()
    inst = get_instrumented_model("StyleGAN2", "ffhq", "convs.0", dev, model=model, use_w=False)
    assert get_max_batch_size(inst, dev, None) >= 2
    # an activation edit cannot be re-fed into the fused chain: loud, not silent
    inst.edit_layer("convs.0", offset=torch.ones(1, 512, 8, 8, device=dev))
    with pytest.raises(NotImplementedError):
        model.forward(model.sample_latent(1, seed=1))
    inst.remove_edits()
    inst.close()


def test_to_rgb_edit_in_place_repacks():
    """The ToRGBs are packed with the chain: an in-place edit of a ToRGB's bias and modulation weight after a forward call shows in
    the next image exactly as in a wrapper built with the edited weights."""
    from ganspace_b200.models import StyleGAN2
    dev = torch.device("cuda:0")

    def edit(m):
        with torch.no_grad():
            m.model.to_rgbs[2].bias.add_(0.25)
            m.model.to_rgbs[2].conv.modulation.weight.mul_(1.5)
    m = StyleGAN2(dev, "cat", random_init=3)
    z = m.sample_latent(3, seed=2)
    before = m.forward(z)
    edit(m)
    after = m.forward(z)
    fresh = StyleGAN2(dev, "cat", random_init=3)
    edit(fresh)
    assert torch.equal(after, fresh.forward(z))
    assert (after - before).abs().max() > 1e-2
    m.check_numerics()
