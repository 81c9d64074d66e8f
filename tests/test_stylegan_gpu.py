"""StyleGAN (v1) on the GPU (csrc/stylegan.cu and the mapping kernels through models.wrappers.StyleGAN): every block and the image
for ffhq and bedrooms against known answers written by the unmodified reference, in Z mode and for 18 distinct W; one block of
each kind against the fp64 oracle fed its own input; every layer and torgb on its own against fp64 on every element, fed the
chain's own input; the sampler against NumPy; partial == full at a hooked block; independence of the
batch size; the three get_or_compute runs against the reference's own .npz (oracle/gen_golden_stylegan.py); and the guards."""
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from layer_parity import assert_spans_chunks, check, nhwc_to_nchw, parity_batch, stylegan_chunk_samples
from oracle import stylegan_oracle as so

pytestmark = pytest.mark.gpu

ACT_TOL = 5e-4         # max |diff| / max |ref| after up to 18 fused layers (the bar of test_render_gpu.py / test_progan_gpu.py)
LAYER_TOL = 1e-4       # one layer fed the oracle's own input, against fp64
PARITY_TOL = 1.3e-5    # one layer fed the chain's own input, against fp64, per sample: ~3x the worst measured (test_each_layer_vs_fp64)
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def ka(golden):
    return golden("stylegan_known_answers.npz")


@pytest.fixture(scope="module")
def models():
    from ganspace_b200.models import StyleGAN, stylegan
    out = {}
    for cls in ("ffhq", "bedrooms"):
        m = StyleGAN(DEV, cls, random_init=1234)
        stylegan.synthesis_fill(m.model, 7)
        out[cls] = m
    return out


def _sub(act):
    step = max(1, act.shape[-1] // 16)
    return act[:, ::max(1, act.shape[1] // 8), ::step, ::step]


@pytest.mark.parametrize("cls", ["ffhq", "bedrooms"])
def test_every_block_and_image_vs_reference(ka, models, cls):
    from ganspace_b200.models import get_instrumented_model
    m = models[cls]
    names = m.model.block_names()
    z = torch.tensor(ka[f"{cls}_z"]).to(DEV)
    w = m.model.g_mapping(z).cpu().numpy()
    ref_w = ka[f"{cls}_w"]
    assert np.abs(w - ref_w).max() <= 2e-5 * max(1.0, np.abs(ref_w).max())
    inst = get_instrumented_model("StyleGAN", cls, names, DEV, model=m)
    assert inst.input_shape == (1, 512)
    w18 = [torch.tensor(x).to(DEV) for x in so.w18_latents()]
    for tag, run in (("z", lambda: m.forward(z)), ("w18", lambda: (m.use_w(), m.forward(w18))[1])):
        img = run().float().cpu().numpy()
        m.use_z()
        for name, act in inst.retained_features().items():
            b = name.rsplit(".", 1)[1]
            act = act.float().cpu().numpy()
            assert tuple(act.shape) == tuple(ka[f"{cls}_{b}_shape"]), name
            ref = ka[f"{cls}_{tag}_{b}_sub"]
            err = np.abs(_sub(act) - ref).max() / np.abs(ref).max()
            assert err < ACT_TOL, (tag, name, err)
            s2 = (act.astype(np.float64).reshape(4, -1) ** 2).sum(1)
            assert np.abs(s2 - ka[f"{cls}_{tag}_{b}_sums"][:, 1]).max() < 2e-3 * ka[f"{cls}_{tag}_{b}_sums"][:, 1].max(), (tag, name)
        R = m.resolution
        assert img.shape == (4, 3, R, R)
        ref = ka[f"{cls}_{tag}_image_sub"]
        step = max(1, R // 32)
        err = np.abs(img[:, :, ::step, ::step] - ref).max() / np.abs(ref - 0.5).max()
        assert err < ACT_TOL, (tag, err)
    inst.close()
    with pytest.raises(AssertionError, match="1 or 18"):
        m.forward([z, z])
    m.check_numerics()


def test_one_layer_of_each_kind_vs_fp64_oracle(models):
    """The 4x4 input block, an up-conv below 128 px (8x8), one from 128 px (128x128, flipped kernel) and a 16-channel layer
    (1024x1024): the chain run to the block before, its output fed to the fp64 oracle, and the chain's block output compared."""
    m = models["ffhq"]
    sd = m.model.state_dict()
    noise = so.fixed_noise(1024)
    w = m.model.g_mapping.packed().forward(m.sample_latent(1, seed=4))
    packed = m.model.g_synthesis.packed()
    lays = so.layers(sd, 1024)
    wn = w.double().cpu().numpy()
    for blk in ("4x4", "8x8", "128x128", "1024x1024"):
        bi = so.block_names(1024).index(blk)
        x = None
        if bi:
            act = packed.forward(w, 2 * bi)[0]
            r, c = packed.shapes[2 * bi - 1]
            x = act.view(1, r, r, c).permute(0, 3, 1, 2).double().cpu().numpy()
        for l in (2 * bi, 2 * bi + 1):
            _, conv, epi, up, r = lays[l]
            x = so.layer_taps(x, wn, sd, conv, epi, up, noise[r])
        got = packed.forward(w, 2 * bi + 2)[0]
        r, c = packed.shapes[2 * bi + 1]
        got = got.view(1, r, r, c).permute(0, 3, 1, 2).double().cpu().numpy()
        err = np.abs(got - x).max() / np.abs(x).max()
        assert err < LAYER_TOL, (blk, err)
    m.check_numerics()


def _layer_cases():
    cases = []
    for cls, res in (("ffhq", 1024), ("bedrooms", 256)):
        for l, (b, conv, _, _, _) in enumerate(so.layers({}, res)):
            cases.append(pytest.param(cls, l, id=f"{cls}-{l:02d}-{b}.{'const' if conv is None else conv.rsplit('.', 1)[1]}"))
        cases.append(pytest.param(cls, "torgb", id=f"{cls}-torgb"))
    return cases


@pytest.mark.parametrize("cls,layer", _layer_cases())
def test_each_layer_vs_fp64(models, cls, layer):
    """Layer ``layer`` of the synthesis chain (the input block's constant layer, a 3x3 conv, an up-conv below 128 px and one
    from 128 px, which packs the flipped kernel) fed the chain's own output of the layer before, against the reference form in
    fp64 (oracle layer_reference), on every element of a batch that spans two chunks of that layer; torgb fed the last layer's
    output.  Every sample and every layer has its own latent ([L, n, 512]), so a latent or style index that slips by a layer
    or by a sample fails.  Measured on an H100 80GB HBM3 (700 W), both classes: worst 4.3e-6 (the 4x4 conv and the 8x8 up-conv),
    1e-6 to 3.5e-6 up to 64x64, under 1e-6 from 128x128 on (flipped kernel included), 1.4e-7 for torgb."""
    m = models[cls]
    sd = m.model.state_dict()
    packed = m.model.g_synthesis.packed()
    lays = so.layers(sd, m.resolution)
    rgb = layer == "torgb"
    l = len(lays) - 1 if rgb else layer
    _, conv, epi, up, r = lays[l]
    spc = stylegan_chunk_samples(r, packed.shapes[l][1], up, conv is not None)
    n = parity_batch(spc)
    assert_spans_chunks(n, spc)
    w = np.random.RandomState(200 + l).standard_normal((len(lays), n, 512)).astype(np.float32)
    wd = torch.from_numpy(w).to(DEV)
    if rgb:
        act, img = packed.forward(wd, len(lays), want_rgb=True)
        got = img.permute(0, 3, 1, 2).double().cpu().numpy()
        ref = so.torgb(nhwc_to_nchw(act, n, *packed.shapes[l]), sd)
    else:
        x = None if l == 0 else nhwc_to_nchw(packed.forward(wd, l)[0], n, *packed.shapes[l - 1])
        got = nhwc_to_nchw(packed.forward(wd, l + 1)[0], n, *packed.shapes[l])
        noise = m.model.g_synthesis.layer_modules()[l][1].top_epi.noise.noise.reshape(r, r)
        ref = so.layer_reference(x, w[l], sd, conv, epi, up, noise)
    check(got, ref, PARITY_TOL, f"{cls} {layer}", chunk_of=spc)
    m.check_numerics()


def test_sample_latent_and_small_api(models):
    m = models["bedrooms"]
    z = m.sample_latent(7, seed=11)
    want = np.random.RandomState(11).standard_normal(7 * 512).reshape(7, 512).astype(np.float32)
    assert z.shape == (7, 512) and np.array_equal(z.cpu().numpy(), want)
    np.random.seed(5)
    seed = np.random.randint(np.iinfo(np.int32).max)
    np.random.seed(5)
    assert torch.equal(m.sample_latent(2), m.sample_latent(2, seed=seed))
    rs = np.random.RandomState(5)
    rs.randint(np.iinfo(np.int32).max)
    np.random.seed(5)
    assert m.get_latent_shape() == (1, 512) and np.random.randint(1 << 30) == rs.randint(1 << 30)
    assert m.get_max_latents() == 18 and m.latent_space_name() == "Z" and m.has_latent_residual
    m.use_w()
    try:
        assert m.latent_space_name() == "W"
        z2 = torch.tensor(np.random.RandomState(2).standard_normal(3 * 512).reshape(3, 512).astype(np.float32)).to(DEV)
        assert torch.equal(m.sample_latent(3, seed=2), m.z_to_latent(z2))
        lat, ensure = m.sample_latents_multi(4, [2, 3], lazy=True)
        ensure(8)
        assert torch.equal(lat[:3], m.sample_latent(3, seed=2)) and torch.equal(lat[4:8], m.sample_latent(4, seed=3))
    finally:
        m.use_z()
    with pytest.raises(RuntimeError, match="cannot change output class"):
        m.set_output_class("cats")
    m.set_noise_seed(1)
    maps = [mod.noise for n, mod in m.model.named_modules() if n.endswith("top_epi.noise")]
    torch.manual_seed(1)
    assert torch.equal(maps[-1].cpu(), torch.randn(1, 1, 256, 256)) and torch.equal(maps[-1], maps[-2])
    m.set_noise_seed(0)


def test_partial_equals_full_hooks_and_guards(models):
    from ganspace_b200.models import get_instrumented_model
    m = models["bedrooms"]
    z = m.sample_latent(3, seed=5)
    for layer in ("g_synthesis.blocks.4x4", "g_synthesis.blocks.64x64", "g_synthesis.blocks.256x256"):
        inst = get_instrumented_model("StyleGAN", "bedrooms", layer, DEV, model=m)
        m.partial_forward(z, layer)
        a = inst.retained_features()[layer].clone()
        m.forward(z)
        assert torch.equal(a, inst.retained_features()[layer]), layer
        inst.close()
    # the reference's substring stop rule: 'blocks.16x16.conv1' stops after block 16x16, so a hook on 32x32 does not fire
    calls = []
    h = m.model.g_synthesis.blocks["32x32"].register_forward_hook(lambda *a: calls.append(1))
    m.partial_forward(z, "blocks.16x16.conv1")
    assert not calls
    m.partial_forward(z, "g_synthesis.blocks.32x32")
    assert len(calls) == 1
    h.remove()
    with pytest.raises(RuntimeError, match="not encountered"):
        m.partial_forward(z, "g_synthesis.blocks.99")
    # g_mapping: Z mode fires in partial_forward; W mode in sample_latent (the reference's quirk)
    inst = get_instrumented_model("StyleGAN", "bedrooms", "g_mapping", DEV, model=m)
    m.partial_forward(z, "g_mapping")
    assert torch.equal(inst.retained_features()["g_mapping"], m.model.g_mapping.packed().forward(z))
    m.use_w()
    w = m.sample_latent(2, seed=8)
    assert torch.equal(inst.retained_features()["g_mapping"], w)
    m.use_z()
    inst.close()
    for bad in ("g_mapping.dense3", "g_synthesis.blocks.8x8.epi1", "g_synthesis.blocks.8x8.conv1", "g_synthesis", "g_synthesis.torgb"):
        with pytest.raises(NotImplementedError, match="hookable layers"):
            get_instrumented_model("StyleGAN", "bedrooms", bad, DEV, model=m)
        for _, mod in m.model.named_modules():
            mod._forward_hooks.clear()
    inst = get_instrumented_model("StyleGAN", "bedrooms", "g_synthesis.blocks.8x8", DEV, model=m)
    inst.edit_layer("g_synthesis.blocks.8x8", offset=torch.ones(1, 512, 8, 8, device=DEV))
    with pytest.raises(NotImplementedError, match="cannot be propagated"):
        m.forward(z)
    inst.remove_edits()
    inst.close()
    with pytest.raises(RuntimeError, match="Unknown layer"):
        get_instrumented_model("StyleGAN", "bedrooms", "g_synthesis.blocks.99x99", DEV, model=m)
    with pytest.raises(RuntimeError, match="outside the GPU hot path"):
        from ganspace_b200.models import get_model
        get_model("DCGAN", "x", DEV)
    with pytest.raises(NotImplementedError, match="exceeds"):
        m.feature_layout("g_synthesis.blocks.64x64")
    m.check_numerics()


def test_tf_checkpoint_without_conversion_raises(tmp_path, monkeypatch):
    from ganspace_b200.models import StyleGAN
    (tmp_path / "stylegan").mkdir()
    (tmp_path / "stylegan" / "stylegan_vases_1024.pkl").write_bytes(b"x")
    monkeypatch.setenv("GANCONTROL_CHECKPOINT_DIR", str(tmp_path))
    monkeypatch.delenv("GANSPACE_B200_RANDOM_INIT", raising=False)
    with pytest.raises(RuntimeError, match="TensorFlow"):
        StyleGAN(DEV, "vases")


def test_rows_do_not_depend_on_batch_size(models):
    m = models["bedrooms"]
    layer = "g_synthesis.blocks.32x32"
    z = m.sample_latent(500, seed=9)
    d = 32 * 32 * 512
    full = torch.empty((500, d), device=DEV)
    m.activations_into(z, layer, full)
    for n in (1, 3, 127, 128):
        part = torch.empty((n, d), device=DEV)
        m.activations_into(z[:n], layer, part)
        assert torch.equal(part, full[:n]), n
    strided = torch.zeros((4, d + 64), device=DEV)
    m.activations_into(z[:4], layer, strided[:, :d])
    assert torch.equal(strided[:, :d], full[:4]) and float(strided[:, d:].abs().max()) == 0.0
    img1 = m.forward(z[:1])
    assert torch.equal(img1, m.forward(z[:5])[:1])
    m.check_numerics()


@pytest.mark.parametrize("layer,use_w,c", [("g_mapping", False, 16), ("g_mapping", True, 16), ("g_synthesis.blocks.8x8", False, 8)])
def test_get_or_compute_vs_reference(golden, oracle, models, layer, use_w, c):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model
    short = layer.rsplit(".", 1)[-1]
    g = golden(f"sg_stylegan_ffhq_{short}_{'w' if use_w else 'z'}_n4000_b500_c{c}.npz")
    if "act_comp_f16" in g:
        g["act_comp"] = g.pop("act_comp_f16").astype(np.float32)
    m = models["ffhq"]
    inst = get_instrumented_model("StyleGAN", "ffhq", layer, DEV, model=m, use_w=use_w)
    cfg = Config(model="StyleGAN", layer=layer, output_class="ffhq", components=c, n=4000, batch_size=500, estimator="ipca", use_w=use_w)
    with tempfile.TemporaryDirectory() as tmp:
        path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        with np.load(path, allow_pickle=False) as data:
            out = {k: data[k] for k in data.files}
    assert path.name == str(g["dump_name"])
    for k in ("act_comp", "act_mean", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio", "random_stdevs"):
        assert out[k].shape == g[k].shape, k
    cmp = oracle.compare_npz(out, g)
    assert cmp["min_signed_cos"] >= 0.999 and cmp["max_abs_dvar_ratio"] <= 1e-3 and cmp["min_lat_signed_cos"] >= 0.999, cmp
    assert cmp["act_mean_rel"] < 1e-3 and cmp["act_stdev_rel"] < 1e-3 and cmp["random_stdevs_rel"] < 1e-3, cmp
    m.use_z()
    if layer != "g_mapping":
        # a latent-space edit along the first direction renders and changes the image
        z = m.sample_latent(2, seed=3)
        base = m.forward(z)
        moved = m.forward(z + 2 * torch.from_numpy(out["lat_comp"][0]).to(DEV).reshape(1, 512))
        assert moved.shape == (2, 3, 1024, 1024) and bool(torch.isfinite(moved).all())
        assert float((moved - base).abs().max()) > 1e-3
    m.check_numerics()
    inst.close()
