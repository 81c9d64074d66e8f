"""ProGAN on the GPU (csrc/progan.cu through models.wrappers.ProGAN): every block and the image against known answers written by
the unmodified reference, every block on its own against fp64 on every element, the latent sampler against NumPy, partial ==
full at a hooked layer, independence of the batch size, and get_or_compute at layer4 against the reference's own .npz
(oracle/gen_golden_progan.py)."""
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from layer_parity import assert_spans_chunks, check, nhwc_to_nchw, parity_batch, progan_chunk_samples
from oracle import progan_oracle as po

pytestmark = pytest.mark.gpu

ACT_TOL = 5e-4         # max |diff| / max |ref| after up to 15 fused blocks (the bar of test_render_gpu.py)
LAYER_TOL = 8e-6       # one block fed the chain's own input, against fp64, per sample: ~3x the worst measured (test_each_block_vs_fp64)


@pytest.fixture(scope="module")
def ka(golden):
    return golden("progan_known_answers.npz")


@pytest.fixture(scope="module")
def model():
    from ganspace_b200.models import ProGAN
    return ProGAN(torch.device("cuda:0"), "bedroom", random_init=1234)


def _sub(act):
    step = max(1, act.shape[-1] // 16)
    return act[:, ::max(1, act.shape[1] // 8), ::step, ::step]


def test_every_block_and_image_vs_reference(ka, model):
    from ganspace_b200.models import get_instrumented_model
    dev = torch.device("cuda:0")
    names = [str(x) for x in ka["names"]]
    assert [n for n, _ in model.named_modules() if n and "." not in n] == names
    z = torch.tensor(ka["z"]).to(dev)
    inst = get_instrumented_model("ProGAN", "bedroom", names, dev, model=model)
    assert inst.input_shape == (1, 512, 1, 1) and tuple(inst.feature_shape["layer10"]) == (1, 128, 64, 64)
    img = model.forward(z).float().cpu().numpy()
    for name, act in inst.retained_features().items():
        act = act.float().cpu().numpy()
        assert tuple(act.shape) == tuple(ka[f"shape_{name}"]), name
        ref = ka[f"act_{name}_sub"]
        scale = np.abs(ref).max()
        assert np.abs(_sub(act) - ref).max() < ACT_TOL * scale, (name, np.abs(_sub(act) - ref).max() / scale)
        s2 = (act.astype(np.float64) ** 2).sum()
        assert abs(s2 - ka[f"sum_{name}"][1]) < 2e-3 * ka[f"sum_{name}"][1], name
    inst.close()
    assert img.shape == (4, 3, 256, 256)
    ref = ka["img_sub"]
    assert np.abs(img[:, :, ::8, ::8] - ref).max() < ACT_TOL * np.abs(ref - 0.5).max()
    assert abs((img.astype(np.float64) ** 2).sum() - ka["img_sum"][1]) < 2e-3 * ka["img_sum"][1]
    assert np.array_equal(model.forward([z]).cpu().numpy(), img)                 # a one-element list is the same latent
    with pytest.raises(AssertionError, match="single global latent"):
        model.forward([z, z])
    model.check_numerics()


@pytest.mark.parametrize("name", [spec[0] for spec in po.block_specs()])
def test_each_block_vs_fp64(model, name):
    """Block ``name`` fed the chain's own output of the block before (the latent for layer1) against the reference form in
    fp64, on every element of a batch that spans two GEMM chunks of that block (the output block: of layer14, behind whose
    epilogue it is fused), one latent per sample.  Measured on an H100 80GB HBM3 (700 W): worst 2.4e-6 (layer2, fp16 hi/lo
    tensor-core products over 4608 terms), 1e-6 to 2e-6 at 4x4 .. 32x32, under 1e-6 from 64x64 on, 1.6e-7 for the output
    block."""
    params = po.progan_random_init(1234)                    # the model's weights (tests/test_progan.py pins the init order)
    names = list(params)
    i = names.index(name)
    out_block = name.startswith("output")
    packed = model.model.packed()
    conv = i - 1 if out_block else i                         # the conv block whose chunks the batch must cross
    res_in = 1 if conv == 0 else packed.shapes[conv - 1][0]
    spc = progan_chunk_samples(res_in, params[names[conv]]["ksize"], packed.shapes[conv][1])
    n = parity_batch(spc)
    assert_spans_chunks(n, spc)
    z = torch.from_numpy(np.random.RandomState(100 + i).standard_normal((n, 512)).astype(np.float32)).to(model.device)
    if out_block:
        act, rgb = packed.forward(z, i, want_rgb=True)
        x = nhwc_to_nchw(act, n, *packed.shapes[i - 1])
        got = rgb.permute(0, 3, 1, 2).double().cpu().numpy()
    else:
        x = z.double().cpu().numpy().reshape(n, 512, 1, 1) if i == 0 else nhwc_to_nchw(packed.forward(z, i)[0], n, *packed.shapes[i - 1])
        got = nhwc_to_nchw(packed.forward(z, i + 1)[0], n, *packed.shapes[i])
    ref = po.progan_block_forward(x, params[name], output=out_block, dtype=np.float64)
    check(got, ref, LAYER_TOL, name, chunk_of=spc)
    model.check_numerics()


def test_sample_latent_bit_exact_vs_numpy(model):
    z = model.sample_latent(7, seed=11)
    want = np.random.RandomState(11).standard_normal(7 * 512).reshape(7, 512).astype(np.float32)
    assert z.shape == (7, 512, 1, 1) and np.array_equal(z.cpu().numpy().reshape(7, 512), want)
    np.random.seed(5)
    seed = np.random.randint(np.iinfo(np.int32).max)
    np.random.seed(5)
    assert torch.equal(model.sample_latent(2), model.sample_latent(2, seed=seed))          # global-seed semantics
    rs = np.random.RandomState(5)                                                 # get_latent_shape consumes one global draw, as the reference's
    rs.randint(np.iinfo(np.int32).max)
    np.random.seed(5)
    assert model.get_latent_shape() == (1, 512, 1, 1) and np.random.randint(1 << 30) == rs.randint(1 << 30)
    assert model.get_max_latents() == 1 and model.latent_space_name() == "Z"
    with pytest.raises(RuntimeError, match="cannot change output class"):
        model.set_output_class("kitchen")


def test_partial_equals_full_and_rejects_unknown_layers(model):
    from ganspace_b200.models import get_instrumented_model
    dev = torch.device("cuda:0")
    z = model.sample_latent(3, seed=5)
    for layer in ("layer1", "layer5", "layer8", "output_256x256"):
        inst = get_instrumented_model("ProGAN", "bedroom", layer, dev, model=model)
        model.partial_forward(z, layer)
        a = inst.retained_features()[layer].clone()
        model.forward(z)
        assert torch.equal(a, inst.retained_features()[layer]), layer
        model.partial_forward(model.sample_latent(3, seed=6), layer)
        assert not torch.equal(a, inst.retained_features()[layer])
        inst.close()
    with pytest.raises(RuntimeError, match="not encountered"):
        model.partial_forward(z, "layer1.conv")                                  # exact block names only, as the reference
    inst = get_instrumented_model("ProGAN", "bedroom", "layer3", dev, model=model)
    inst.edit_layer("layer3", offset=torch.ones(1, 512, 8, 8, device=dev))
    with pytest.raises(NotImplementedError):                                     # an edit cannot be re-fed into the fused chain: loud
        model.forward(z)
    inst.remove_edits()
    inst.close()
    with pytest.raises(RuntimeError, match="Unknown layer"):
        get_instrumented_model("ProGAN", "bedroom", "layer99", dev, model=model)


def test_rows_do_not_depend_on_batch_size(model):
    """Chunk boundaries (layer4 runs 32 samples per GEMM launch, layer1 1152) and ragged last tiles: a sample's activation is
    bit-identical whatever batch it is part of."""
    z = model.sample_latent(500, seed=9)
    d = 8 * 8 * 512
    full = torch.empty((500, d), device=z.device)
    model.activations_into(z, "layer4", full)
    for n in (1, 3, 127, 128):
        part = torch.empty((n, d), device=z.device)
        model.activations_into(z[:n], "layer4", part)
        assert torch.equal(part, full[:n]), n
    strided = torch.zeros((4, d + 64), device=z.device)                          # row-strided destination (the engine's batch rows)
    model.activations_into(z[:4], "layer4", strided[:, :d])
    assert torch.equal(strided[:, :d], full[:4]) and float(strided[:, d:].abs().max()) == 0.0
    model.check_numerics()


def test_get_or_compute_layer4_vs_reference(golden, oracle, model):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model
    g = golden("pg_progan_bedroom_layer4_n4000_b500_c8.npz")
    g["act_comp"] = g.pop("act_comp_f16").astype(np.float32)               # stored as float16 to keep the fixture small
    dev = torch.device("cuda:0")
    inst = get_instrumented_model("ProGAN", "bedroom", "layer4", dev, model=model)
    cfg = Config(model="ProGAN", layer="layer4", output_class="bedroom", components=8, n=4000, batch_size=500, estimator="ipca")
    with tempfile.TemporaryDirectory() as tmp:
        path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
        with np.load(path, allow_pickle=False) as data:
            out = {k: data[k] for k in data.files}
    assert path.name == str(g["dump_name"])
    for k in ("act_comp", "act_mean", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio", "random_stdevs"):
        assert out[k].shape == g[k].shape and out[k].dtype == np.float32, k
    assert out["lat_comp"].shape == (8, 1, 512, 1, 1) and out["act_comp"].shape == (8, 1, 512, 8, 8)
    cmp = oracle.compare_npz(out, g)
    assert cmp["min_signed_cos"] >= 0.999 and cmp["max_abs_dvar_ratio"] <= 1e-3 and cmp["min_lat_signed_cos"] >= 0.999, cmp
    assert cmp["act_mean_rel"] < 1e-3 and cmp["act_stdev_rel"] < 1e-3 and cmp["random_stdevs_rel"] < 1e-3, cmp
    assert np.array_equal(out["lat_stdev"], np.ones(8, np.float32))
    # a latent-space edit along the first direction renders and changes the image
    z = model.sample_latent(2, seed=3)
    base = model.forward(z)
    moved = model.forward(z + 2 * torch.from_numpy(out["lat_comp"][0]).to(dev))
    assert moved.shape == (2, 3, 256, 256) and bool(torch.isfinite(moved).all())
    assert float((moved - base).abs().max()) > 1e-3
    model.check_numerics()
    inst.close()
    with pytest.raises(RuntimeError, match="Cannot change latent space"):
        get_or_compute(Config(model="ProGAN", output_class="bedroom", layer="layer4", n=100, use_w=True))
    with pytest.raises(NotImplementedError, match="exceeds"):
        model.feature_layout("layer12")
