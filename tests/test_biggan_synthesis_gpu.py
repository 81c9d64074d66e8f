"""BigGAN-deep synthesis on the GPU (csrc/biggan.cu through models.biggan.BigGAN): every generator.layers.k and the images against
known answers the unmodified reference wrote (oracle/gen_golden_biggan_synth.py), every layer and the RGB tail of the 512 and the
128 generator on their own against an fp64 restatement on every element, one GenBlock and the SelfAttn at scaled random inputs, batch independence,
hooks, edits and the get_or_compute guard."""
import numpy as np
import pytest
import torch
import torch.nn.functional as F

from layer_parity import assert_spans_chunks, biggan_chunk_samples, biggan_tile, check, parity_batch

pytestmark = pytest.mark.gpu

ACT_TOL = 5e-4         # max |diff| / max |ref|: the bar of test_progan_gpu.py
UNIT_TOL = 2e-5        # one module against its fp64 restatement
LAYER_TOL = 4.5e-6     # one layer fed the chain's own input, against fp64, per sample: ~3x the worst measured (test_each_layer_vs_fp64)


@pytest.fixture(scope="module")
def ka(golden):
    return golden("biggan_synthesis_known_answers.npz")


@pytest.fixture(scope="module")
def model():
    from ganspace_b200.models.biggan import BigGAN
    return BigGAN(torch.device("cuda:0"), 512, "husky", random_init=4321)


def _sub(act):
    c, r = act.shape[1], act.shape[2]
    return act[:, ::max(1, c // 8), ::max(1, r // 16), ::max(1, r // 16)]


def _err(a, b):
    return float(np.abs(np.asarray(a, np.float64) - b).max() / np.abs(b).max())


def test_every_layer_vs_reference(ka, model):
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    dev = torch.device("cuda:0")
    names = [f"generator.layers.{k}" for k in range(15)]
    inst = InstrumentedModel(model)
    inst.retain_layers(names)
    try:
        model.partial_forward(torch.tensor(ka["z"]).to(dev), names[-1])
        feats = inst.retained_features()
        for k, name in enumerate(names):
            act = feats[name]
            assert tuple(act.shape) == tuple(ka[f"act{k}_shape"]), name
            a = act.double()
            err = _err(_sub(act).cpu().numpy(), ka[f"act{k}_sub"])
            assert err < ACT_TOL, (name, err)
            np.testing.assert_allclose(a.pow(2).sum(dim=(1, 2, 3)).cpu().numpy(), ka[f"act{k}_sq"], rtol=1e-3, err_msg=name)
            scale = float(np.sqrt(ka[f"act{k}_sq"].max()))          # sums: against the tensor's l2 norm
            assert np.abs(a.sum(dim=(1, 2, 3)).cpu().numpy() - ka[f"act{k}_sum"]).max() < 1e-3 * scale * np.sqrt(a[0].numel()), name
    finally:
        inst.close()


def test_images_vs_reference(ka, model):
    dev = torch.device("cuda:0")
    img = model.forward(torch.tensor(ka["z"]).to(dev))
    assert tuple(img.shape) == (2, 3, 512, 512)
    assert _err(img[:, :, ::8, ::8].cpu().numpy(), ka["img_t100_sub"]) < ACT_TOL
    np.testing.assert_allclose(img.double().sum(dim=(1, 2, 3)).cpu().numpy(), ka["img_t100_sum"], rtol=1e-4)
    z_list = [torch.tensor(z).to(dev) for z in ka["z_list"]]
    img = model.forward(z_list)
    assert _err(img[:, :, ::8, ::8].cpu().numpy(), ka["img_list_sub"]) < ACT_TOL
    model.truncation = 0.37
    try:
        img = model.forward(torch.tensor(ka["z37"]).to(dev))
        assert _err(img[:, :, ::8, ::8].cpu().numpy(), ka["img_t037_sub"]) < ACT_TOL
        np.testing.assert_allclose(img.double().sum(dim=(1, 2, 3)).cpu().numpy(), ka["img_t037_sum"], rtol=1e-4)
    finally:
        model.truncation = 1.0


def test_biggan128_images_vs_reference(ka):
    from ganspace_b200.models.biggan import BigGAN
    m = BigGAN(torch.device("cuda:0"), 128, "husky", random_init=4321)
    img = m.forward(torch.tensor(ka["z"]).cuda())
    assert tuple(img.shape) == (2, 3, 128, 128)
    assert _err(img[:, :, ::2, ::2].cpu().numpy(), ka["img128_sub"]) < ACT_TOL
    np.testing.assert_allclose(img.double().sum(dim=(1, 2, 3)).cpu().numpy(), ka["img128_sum"], rtol=1e-4)


def test_biggan256_shapes():
    from ganspace_b200.models.biggan import BigGAN
    m = BigGAN(torch.device("cuda:0"), 256, "husky", random_init=1)
    img = m.forward(m.sample_latent(1, seed=3))
    assert tuple(img.shape) == (1, 3, 256, 256) and bool(torch.isfinite(img).all())


# ---- single modules against an fp64 restatement of model.py ------------------------------------------------------------------
def _bn64(bn, x, cond, t):
    mean, var = (v.double().cpu() for v in bn.stats(t))
    w = 1 + cond @ bn.scale.effective_weight().double().cpu().t()
    b = cond @ bn.offset.effective_weight().double().cpu().t()
    return (x - mean[None, :, None, None]) / torch.sqrt(var + bn.eps)[None, :, None, None] * w[:, :, None, None] + b[:, :, None, None]


def _conv64(m, x):
    w = m.effective_weight().double().cpu()
    return F.conv2d(x, w, None if m.bias is None else m.bias.detach().double().cpu(), padding=w.shape[-1] // 2)


def _block64(blk, x, cond, t):
    h = _conv64(blk.conv_0, F.relu(_bn64(blk.bn_0, x, cond, t)))
    h = F.relu(_bn64(blk.bn_1, h, cond, t))
    if blk.up_sample:
        h = F.interpolate(h, scale_factor=2, mode="nearest")
    h = _conv64(blk.conv_1, h)
    h = _conv64(blk.conv_2, F.relu(_bn64(blk.bn_2, h, cond, t)))
    h = _conv64(blk.conv_3, F.relu(_bn64(blk.bn_3, h, cond, t)))
    x0 = x[:, :x.shape[1] // 2] if blk.drop_channels else x
    if blk.up_sample:
        x0 = F.interpolate(x0, scale_factor=2, mode="nearest")
    return h + x0


def _attn64(sa, x):
    n, ch, h, w = x.shape
    theta = _conv64(sa.snconv1x1_theta, x).view(n, ch // 8, h * w)
    phi = F.max_pool2d(_conv64(sa.snconv1x1_phi, x), 2).view(n, ch // 8, h * w // 4)
    attn = torch.softmax(torch.bmm(theta.permute(0, 2, 1), phi), dim=-1)
    g = F.max_pool2d(_conv64(sa.snconv1x1_g, x), 2).view(n, ch // 2, h * w // 4)
    o = _conv64(sa.snconv1x1_o_conv, torch.bmm(g, attn.permute(0, 2, 1)).view(n, ch // 2, h, w))
    return x + sa.gamma.detach().double().cpu() * o


def test_genblock_up_and_drop_vs_fp64(model):
    """The up-sampling, channel-dropping GenBlock on random inputs three times the unit scale and arbitrary condition vectors:
    a regime the chain's own activations and the model's condition vectors (test_each_layer_vs_fp64) do not reach."""
    blk = model.model.generator.layers[3]                  # (up, 2048 -> 1024) at 8x8 -> 16x16
    assert blk.up_sample and blk.drop_channels
    gen = torch.Generator().manual_seed(5)
    x = torch.randn(3, 2048, 8, 8, generator=gen, dtype=torch.float64) * 3
    cond = torch.randn(3, 256, generator=gen, dtype=torch.float64) * 0.5
    chain = model._chain()
    out = chain.block(3, x.float().permute(0, 2, 3, 1).contiguous().cuda(), cond.float().cuda()).permute(0, 3, 1, 2)
    ref = _block64(blk, x.float().double(), cond.float().double(), model.truncation)
    assert _err(out.cpu().numpy(), ref.numpy()) < UNIT_TOL


def _rgb64(g, x, t):
    mean, var = (v.double().cpu() for v in g.bn.stats(t))
    h = (x - mean[None, :, None, None]) / torch.sqrt(var + g.bn.eps)[None, :, None, None]
    h = h * g.bn.weight.detach().double().cpu()[None, :, None, None] + g.bn.bias.detach().double().cpu()[None, :, None, None]
    w = g.conv_to_rgb.effective_weight().double().cpu()[:3]            # the image keeps the first three output channels
    return 0.5 * (torch.tanh(F.conv2d(F.relu(h), w, g.conv_to_rgb.bias.detach().double().cpu()[:3], padding=1)) + 1)


@pytest.fixture(scope="module")
def model128():
    from ganspace_b200.models.biggan import BigGAN
    return BigGAN(torch.device("cuda:0"), 128, "husky", random_init=4321)


def _layer_cases():
    from ganspace_b200.models.biggan import _LAYERS
    cases = []
    for res in (512, 128):
        n_mod = len(_LAYERS[res]) + 1                      # the GenBlocks and the SelfAttn
        cases += [pytest.param(res, k, id=f"{res}-layers.{k}") for k in range(n_mod)] + [pytest.param(res, "rgb", id=f"{res}-rgb")]
    return cases


@pytest.mark.parametrize("res,layer", _layer_cases())
def test_each_layer_vs_fp64(model, model128, res, layer):
    """generator.layers.k (GenBlock or SelfAttn) fed the chain's own output of layers.k-1 (of gen_z for k = 0), taken from the
    retain hooks, with the condition vector the chain gives that block, against the fp64 restatement, on every element; the RGB
    tail fed the last layer's output.  One latent per sample and per GenBlock, so a condition index that slips fails.  The batch
    spans two 128-row tiles of the layer's input resolution and, at 4x4 and 8x8, ends in a ragged tile.  Measured on an H100
    80GB HBM3 (700 W), both generators: worst 1.4e-6 (layers.3, the 8 -> 16 up-block with 2048 input channels), under 1e-6 for
    every other GenBlock and the SelfAttn (3.7e-7 at 64x64), under 1e-6 for the RGB tail."""
    from ganspace_b200.models.biggan import GenBlock
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    m = model if res == 512 else model128
    g = m.model.generator
    mods = list(g.layers)
    k = len(mods) - 1 if layer == "rgb" else layer
    r_in = 4
    for mod in mods[:k]:
        r_in *= 2 if isinstance(mod, GenBlock) and mod.up_sample else 1
    r_last = r_in * (2 if isinstance(mods[k], GenBlock) and mods[k].up_sample else 1)
    spc = biggan_chunk_samples(r_last if layer == "rgb" else r_in)
    n = parity_batch(spc)
    assert_spans_chunks(n, spc)
    zs = [m.sample_latent(n, seed=500 + 31 * k + i) for i in range(m.model.n_latents)]
    conds = [c.double().cpu() for c in m._conds(zs)]
    prev = "generator.gen_z" if k == 0 else f"generator.layers.{k - 1}"
    names = [prev, f"generator.layers.{k}"]
    inst = InstrumentedModel(m)
    inst.retain_layers(names)
    try:
        if layer == "rgb":
            got = m.forward(zs)
            x = inst.retained_layer(names[1]).double().cpu()
            ref = _rgb64(g, x, m.truncation)
            tile = lambda s: biggan_tile(s, r_last)
        else:
            m.partial_forward(zs, names[1])
            x = inst.retained_layer(prev)
            x = (x.view(n, 4, 4, -1).permute(0, 3, 1, 2) if k == 0 else x).double().cpu()
            got = inst.retained_layer(names[1])
            if isinstance(mods[k], GenBlock):
                ci = 1 + sum(isinstance(mod, GenBlock) for mod in mods[:k])
                ref = _block64(mods[k], x, conds[ci], m.truncation)
            else:
                ref = _attn64(mods[k], x)
            tile = lambda s: biggan_tile(s, r_in)
        check(got.double().cpu().numpy(), ref.numpy(), LAYER_TOL, f"BigGAN-{res} {names[1] if layer != 'rgb' else 'rgb'}", chunk_of=tile)
    finally:
        inst.close()


def test_selfattn_vs_fp64(model):
    sa = model.model.generator.layers[8]
    gen = torch.Generator().manual_seed(6)
    # scaled so that the scores are O(10): at unit inputs they reach ~1e4, where fp32 rounding of the scores alone moves the
    # softmax by ~1e-3 (a property of fp32 scores, the reference's included, not of the kernels)
    x = torch.randn(2, 512, 64, 64, generator=gen, dtype=torch.float64) * 0.05
    out = model._chain().attn(8, x.float().permute(0, 2, 3, 1).contiguous().cuda()).permute(0, 3, 1, 2)
    ref = _attn64(sa, x.float().double())
    err = _err(out.cpu().numpy(), ref.numpy())
    delta = _err((out.cpu().double() - x.float().double()).numpy(), (ref - x.float().double()).numpy())
    assert err < UNIT_TOL and delta < 1e-4, (err, delta)


# ---- batch independence, hooks, edits ----------------------------------------------------------------------------------------
def test_sample_alone_equals_sample_in_batch(model):
    z = model.sample_latent(7, seed=21)
    full = model.forward(z)
    alone = model.forward(z[4:5].clone())
    assert torch.equal(full[4:5], alone)


def test_instrumented_layers_hooks_and_edits(model):
    from ganspace_b200.models import get_instrumented_model
    dev = torch.device("cuda:0")
    inst = get_instrumented_model("BigGAN-512", "husky", "generator.layers.3", dev, model=model)
    try:
        assert tuple(inst.feature_shape["generator.layers.3"]) == (1, 1024, 16, 16)
        z = model.sample_latent(2, seed=5)
        model.partial_forward(z, "generator.layers.3")
        a = inst.retained_layer("generator.layers.3").clone()
        model.partial_forward(z, "generator.layers.5")           # the hooked layer fires on the way, with the same values
        assert torch.equal(inst.retained_layer("generator.layers.3"), a)
        inst.edit_layer("generator.layers.3", offset=1.0)
        model.partial_forward(z, "generator.layers.3")           # an edit on the last layer run has nothing downstream
        with pytest.raises(NotImplementedError):
            model.partial_forward(z, "generator.layers.4")
        with pytest.raises(NotImplementedError):
            model.forward(z)
    finally:
        inst.close()
    # quirk: a name outside generator.layers runs 14 of the 15 modules and never the tail
    inst = get_instrumented_model("BigGAN-512", "husky", ["generator.layers.13", "generator.layers.14"], dev, model=model)
    try:
        inst.retained_features()
        z = model.sample_latent(1, seed=9)
        inst._retained["generator.layers.14"] = None
        model.partial_forward(z, "generator.conv_to_rgb")
        assert inst.retained_layer("generator.layers.13") is not None and inst.retained_layer("generator.layers.14") is None
    finally:
        inst.close()


def test_get_or_compute_guard(model):
    from types import SimpleNamespace
    import tempfile
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model
    inst = get_instrumented_model("BigGAN-512", "husky", "generator.layers.1", torch.device("cuda:0"), model=model)
    cfg = Config(model="BigGAN-512", layer="generator.layers.1", output_class="husky", components=4, n=100, batch_size=50)
    try:
        with tempfile.TemporaryDirectory() as tmp, pytest.raises(NotImplementedError, match="generator.gen_z"):
            get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
    finally:
        inst.close()


def test_outputs_finite(ka, model):
    img = model.forward(torch.tensor(ka["z"]).cuda())
    assert bool(torch.isfinite(img).all()) and float(img.min()) >= 0.0 and float(img.max()) <= 1.0
