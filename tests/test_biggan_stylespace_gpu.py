"""BigGAN-deep conditional-BatchNorm row layers (generator.layers.k.bn_j.scale / .offset) on the GPU: retained rows against the rows
the unmodified reference retained (oracle/gen_golden_biggan_stylespace.py) and against fp64, no conv launch for a rows-only partial
run, bit-identity of a retain-only hooked forward, edits against the reference's edited images and an fp64 chain, get_or_compute
against the reference's fixtures and the fp64 oracle, and the guards."""
import os
import tempfile
from types import SimpleNamespace

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import biggan_stylespace_oracle as bso

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
ACT_TOL = 5e-4         # images: max |diff| / max |ref|, the bar of test_biggan_synthesis_gpu.py
ROW_TOL = 2e-5         # rows against the reference's fp32 rows and against fp64, relative to the layer's max |row|
COS_TOL = 0.999
RATIO_TOL = 1e-3
AUX_TOL = 1e-3


@pytest.fixture(scope="module")
def ka(golden):
    return golden("biggan_stylespace_known_answers.npz")


@pytest.fixture(scope="module")
def models():
    from ganspace_b200.models.biggan import BigGAN
    return {512: BigGAN(DEV, 512, "husky", random_init=4321), 128: BigGAN(DEV, 128, "husky", random_init=4321)}


@pytest.fixture(scope="module")
def nets():
    return {512: bso.net(512), 128: bso.net(128)}


def _inst(m, layers):
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    inst = InstrumentedModel(m)
    inst.retain_layers(layers)
    return inst


def _err(a, b):
    a, b = np.asarray(a, np.float64), np.asarray(b, np.float64)
    return float(np.abs(a - b).max() / np.abs(b).max())


def _cond_index(m):
    from ganspace_b200.models.biggan import GenBlock
    layers = list(m.model.generator.layers)
    return {k: 1 + sum(isinstance(l, GenBlock) for l in layers[:k]) for k in range(len(layers))}


# ---- 1. rows ---------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("res", [512, 128])
def test_rows_vs_reference_and_fp64(ka, models, nets, res):
    m, net = models[res], nets[res]
    names = [n for n, _ in m.model.style_layers()]
    ci = _cond_index(m)
    z = torch.tensor(ka["z"]).to(DEV)
    z_big = m.sample_latent(37, seed=5)                       # 37 x C warps: many CTAs per layer
    z_list = [torch.tensor(t).to(DEV) for t in ka["z_list"]]
    inst = _inst(m, names)
    try:
        runs = [("forward z", lambda: m.forward(z), lambda k: ka["z"], "z"),
                ("partial z", lambda: m.partial_forward(z, names[-1]), lambda k: ka["z"], "z"),
                ("partial big", lambda: m.partial_forward(z_big, names[-1]), lambda k: z_big.cpu().numpy(), None)]
        if res == 512:
            runs += [("forward list", lambda: m.forward(z_list), lambda k: ka["z_list"][ci[k]], "list"),
                     ("partial list", lambda: m.partial_forward(z_list, names[-1]), lambda k: ka["z_list"][ci[k]], "list")]
        known = {tag: bso.known_rows(ka, res, tag) for tag in (("z", "list") if res == 512 else ("z",))}
        for what, run, z_of, tag in runs:
            run()
            feats = inst.retained_features()
            for name in names:
                got = feats[name].cpu().numpy()
                k = int(name.split(".")[2])
                r64 = bso.rows64(net, name, z_of(k))
                assert got.shape == r64.shape, (what, name)
                assert _err(got, r64) < ROW_TOL, (what, name, _err(got, r64))
                if tag is not None:
                    errs = bso.known_rows_err(got, known[tag][name])
                    assert max(errs) < ROW_TOL, (what, name, errs)
    finally:
        inst.close()


# ---- 2. rows only: no conv ---------------------------------------------------------------------------------------------------
def test_partial_forward_to_row_layer_launches_no_conv(models):
    from ganspace_b200 import _native
    m = models[512]
    layers = ["generator.layers.9.bn_1.scale", "generator.layers.9.bn_3.offset", "generator.layers.2.bn_0.offset"]
    inst = _inst(m, layers)
    z = m.sample_latent(4, seed=2)
    old = _native.instrument.timing
    try:
        _native.instrument.timing = True
        _native.instrument.reset()
        m.partial_forward(z, layers[0])
        secs = _native.instrument.section_ms()
        assert not any(k.startswith("biggan layers.") or k == "biggan rgb" for k in secs), secs
        assert secs["biggan rows"][1] == 2, secs                     # one row launch per block with a hooked row layer
        assert all(tuple(inst.retained_layer(n).shape) == (4, m.model.get_submodule(n).weight_orig.shape[0]) for n in layers)
    finally:
        _native.instrument.timing = old
        inst.close()


# ---- 3. bit-identity ---------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("res", [512, 128])
@pytest.mark.parametrize("truncation", [1.0, 0.37])
def test_retain_hooks_are_bit_identical(models, res, truncation):
    m = models[res]
    m.truncation = truncation
    try:
        z = m.sample_latent(3, seed=7, truncation=truncation)
        plain = m.forward(z).clone()
        for k in (0, 3, 9):
            inst = _inst(m, [f"generator.layers.{k}.bn_{j}.{kind}" for j in range(4) for kind in ("scale", "offset")])
            try:
                hooked = m.forward(z)
            finally:
                inst.close()
            assert torch.equal(hooked, plain), (res, truncation, k)
    finally:
        m.truncation = 1.0


# ---- 4. edits ----------------------------------------------------------------------------------------------------------------
def _d(t):
    """A parameter in fp64 on the device (the synthesis weights of the module tree stay on the host)."""
    return t.detach().double().to(DEV)


def _bn64(bn, x, t, s, o):
    mean, var = (_d(v) for v in bn.stats(t))
    return (x - mean[None, :, None, None]) / torch.sqrt(var + bn.eps)[None, :, None, None] * (1 + s)[:, :, None, None] \
        + o[:, :, None, None]


def _conv64(m, x):
    w = _d(m.effective_weight())
    return F.conv2d(x, w, None if m.bias is None else _d(m.bias), padding=w.shape[-1] // 2)


def _chain64(m, z, t, edit=None):
    """The generator in fp64 on the device, with every row layer's rows cond W_eff^T and ``edit(name, rows) -> rows`` applied."""
    from ganspace_b200.models.biggan import GenBlock
    g = m.model.generator
    e = _d(m.model.embeddings.weight)[:, 248]
    cond = torch.cat((z.double(), e[None].expand(z.shape[0], -1)), dim=1)
    h = F.linear(cond, _d(g.gen_z.effective_weight()), _d(g.gen_z.bias))
    x = h.view(-1, 4, 4, h.shape[1] // 16).permute(0, 3, 1, 2)
    for k, blk in enumerate(g.layers):
        if isinstance(blk, GenBlock):
            def bn(j, x):
                rows = []
                for kind in ("scale", "offset"):
                    r = cond @ _d(getattr(getattr(blk, f"bn_{j}"), kind).effective_weight()).T
                    rows.append(edit(f"generator.layers.{k}.bn_{j}.{kind}", r) if edit else r)
                return F.relu(_bn64(getattr(blk, f"bn_{j}"), x, t, *rows))
            hh = _conv64(blk.conv_0, bn(0, x))
            hh = bn(1, hh)
            if blk.up_sample:
                hh = F.interpolate(hh, scale_factor=2, mode="nearest")
            hh = _conv64(blk.conv_2, bn(2, _conv64(blk.conv_1, hh)))
            hh = _conv64(blk.conv_3, bn(3, hh))
            x0 = x[:, :x.shape[1] // 2] if blk.drop_channels else x
            if blk.up_sample:
                x0 = F.interpolate(x0, scale_factor=2, mode="nearest")
            x = hh + x0
        else:
            n, ch, hgt, wid = x.shape
            theta = _conv64(blk.snconv1x1_theta, x).view(n, ch // 8, hgt * wid)
            phi = F.max_pool2d(_conv64(blk.snconv1x1_phi, x), 2).view(n, ch // 8, hgt * wid // 4)
            attn = torch.softmax(torch.bmm(theta.permute(0, 2, 1), phi), dim=-1)
            gg = F.max_pool2d(_conv64(blk.snconv1x1_g, x), 2).view(n, ch // 2, hgt * wid // 4)
            x = x + _d(blk.gamma) * _conv64(blk.snconv1x1_o_conv, torch.bmm(gg, attn.permute(0, 2, 1)).view(n, ch // 2, hgt, wid))
    mean, var = (_d(v) for v in g.bn.stats(t))
    hh = (x - mean[None, :, None, None]) / torch.sqrt(var + g.bn.eps)[None, :, None, None]
    hh = hh * _d(g.bn.weight)[None, :, None, None] + _d(g.bn.bias)[None, :, None, None]
    w = _d(g.conv_to_rgb.effective_weight())[:3]
    return 0.5 * (torch.tanh(F.conv2d(F.relu(hh), w, _d(g.conv_to_rgb.bias)[:3], padding=1)) + 1)


EDITS = [("scale", "generator.layers.11.bn_2.scale"), ("offset", "generator.layers.13.bn_1.offset"),
         ("ablate", "generator.layers.10.bn_0.offset")]


@pytest.mark.parametrize("tag,layer", EDITS)
def test_edit_vs_reference_and_fp64(ka, models, tag, layer):
    m = models[512]
    z = torch.tensor(ka["z"]).to(DEV)
    prev = f"generator.layers.{int(layer.split('.')[2]) - 1}"
    kw = {k[len(f"edit_{tag}_"):]: ka[k] for k in ka if k.startswith(f"edit_{tag}_")}
    inst = _inst(m, [prev])
    try:
        img_plain = m.forward(z).clone()
        prev_plain = inst.retained_layer(prev).clone()
    finally:
        inst.close()
    inst = _inst(m, [layer, prev])
    try:
        inst.edit_layer(layer, **{k: (torch.tensor(v).to(DEV) if np.ndim(v) else float(v)) for k, v in kw.items()})
        img = m.forward(z)
        prev_edit = inst.retained_layer(prev)
    finally:
        inst.close()
    assert _err(img[:, :, ::16, ::16].cpu().numpy(), ka[f"img_{tag}_sub"]) < ACT_TOL, tag
    np.testing.assert_allclose(img.double().sum(dim=(1, 2, 3)).cpu().numpy(), ka[f"img_{tag}_sum"], rtol=1e-4)
    assert torch.equal(prev_edit, prev_plain)                  # block k-1 is upstream of the edit
    np.testing.assert_allclose(prev_edit.double().pow(2).sum(dim=(1, 2, 3)).cpu().numpy(), ka[f"prev_{tag}_sq"], rtol=1e-3)

    def edit(name, r):
        if name != layer:
            return r
        if "offset" in kw:
            return r + torch.tensor(kw["offset"]).double().to(DEV)
        a = float(kw["ablation"])
        return r * (1 - a) + a * torch.tensor(kw["replacement"]).double().to(DEV)[None]
    with torch.no_grad():
        ref64 = _chain64(m, z, m.truncation, edit)
        plain64 = _chain64(m, z, m.truncation)
    assert _err(img.cpu().numpy(), ref64.cpu().numpy()) < ACT_TOL, tag
    delta64 = ref64 - plain64
    assert float(delta64.abs().max()) > 1e-3                            # the edit is visible in the image
    assert _err((img - img_plain).cpu().numpy(), delta64.cpu().numpy()) < 0.02, tag       # and it is the fp64 chain's change


def test_edit_shape_is_checked(models):
    m = models[128]
    layer = "generator.layers.2.bn_1.scale"
    inst = _inst(m, [layer])
    try:
        inst.edit_layer(layer, offset=torch.ones(2, 1, 512, device=DEV))        # broadcasts to [2, 2, 512]
        with pytest.raises(ValueError, match="must keep the rows' shape"):
            m.forward(m.sample_latent(2, seed=1))
    finally:
        inst.close()


# ---- 5, 6. get_or_compute ----------------------------------------------------------------------------------------------------
def _run(m, layer, n, b, c, est="ipca"):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model
    inst = get_instrumented_model("BigGAN-512", "husky", layer, DEV, model=m)
    cfg = Config(model="BigGAN-512", layer=layer, output_class="husky", components=c, n=n, batch_size=b, estimator=est)
    try:
        with tempfile.TemporaryDirectory() as tmp:
            path = get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
            with np.load(path) as data:
                out = {k: data[k] for k in data.files}
    finally:
        inst.close()
    return out, path.name


def _check(cmp, aux=("act_mean_rel", "act_stdev_rel", "random_stdevs_rel")):
    assert cmp["min_signed_cos"] >= COS_TOL and cmp["min_lat_signed_cos"] >= COS_TOL, cmp
    assert cmp["max_abs_dvar_ratio"] <= RATIO_TOL, cmp
    for k in aux:
        assert cmp[k] < AUX_TOL, (k, cmp)


@pytest.mark.parametrize("fixture,layer,est", [
    ("bs_biggan512_husky_l0bn1scale_z_n4000_b1000_c16.npz", "generator.layers.0.bn_1.scale", "ipca"),
    ("bs_biggan512_husky_l1bn0offset_z_n4000_b1000_c16_fbpca.npz", "generator.layers.1.bn_0.offset", "fbpca"),
])
def test_get_or_compute_vs_reference_golden(golden, oracle, models, fixture, layer, est):
    from oracle import fbpca_oracle as fbo
    g = golden(fixture)
    m = models[512]
    assert m.affine_layer(layer) is not None and m.affine_layer(layer).rank == 128
    out, name = _run(m, layer, 4000, 1000, 16, est)
    assert name == str(g["dump_name"])
    for k in ("act_comp", "act_mean", "act_stdev", "lat_comp", "lat_mean", "lat_stdev", "var_ratio", "random_stdevs"):
        assert out[k].shape == g[k].shape and out[k].dtype == g[k].dtype, k
    _check(oracle.compare_npz(out, fbo.sign_normalise(g) if est == "fbpca" else g))


def test_narrow_layer_vs_oracle(oracle, models, nets):
    """C = 32 <= 128: the rows are materialised (gsb_biggan_bn_rows) and go to the small-d engine; against the oracle's IPCA on
    the fp64 rows."""
    m, layer = models[512], "generator.layers.13.bn_2.offset"
    assert m.model.get_submodule(layer).weight_orig.shape[0] == 32 and m.affine_layer(layer) is None
    out, _ = _run(m, layer, 4000, 1000, 8)
    ref = bso.compute_rows(nets[512], layer, 4000, 1000, 8)
    _check(oracle.compare_npz(out, ref))


def test_materialised_rows_cross_check(oracle, models):
    """GANSPACE_B200_BIGGAN_AFFINE=0 on a C = 512 layer: materialised rows through the small-d engine against the affine path."""
    m, layer = models[512], "generator.layers.4.bn_3.scale"
    assert m.model.get_submodule(layer).weight_orig.shape[0] == 256
    affine, _ = _run(m, layer, 4000, 1000, 16)
    old = os.environ.get("GANSPACE_B200_BIGGAN_AFFINE")
    os.environ["GANSPACE_B200_BIGGAN_AFFINE"] = "0"
    try:
        assert m.affine_layer(layer) is None
        rows, _ = _run(m, layer, 4000, 1000, 16)
    finally:
        if old is None:
            del os.environ["GANSPACE_B200_BIGGAN_AFFINE"]
        else:
            os.environ["GANSPACE_B200_BIGGAN_AFFINE"] = old
    _check(oracle.compare_npz(rows, affine))


# ---- 7. guards and ABI -------------------------------------------------------------------------------------------------------
def test_guards(models):
    from ganspace_b200.config import Config
    from ganspace_b200.decomposition import get_or_compute
    from ganspace_b200.models import get_instrumented_model
    m = models[512]
    layer = "generator.layers.0.bn_1.scale"
    inst = get_instrumented_model("BigGAN-512", "husky", layer, DEV, model=m)
    assert tuple(inst.feature_shape[layer]) == (1, 512)
    cfg = Config(model="BigGAN-512", layer=layer, output_class="husky", components=129, n=1000, batch_size=500)
    try:
        with tempfile.TemporaryDirectory() as tmp, pytest.raises(NotImplementedError, match="exceeds the rank"):
            get_or_compute(cfg, inst, submit_config=SimpleNamespace(run_dir=tmp, run_dir_root=tmp), force_recompute=True)
    finally:
        inst.close()
    for bad in ("generator.layers.0.bn_1", "generator.layers.3.conv_2", "generator.layers.8.snconv1x1_g"):
        with pytest.raises(NotImplementedError, match="materialises the outputs"):
            get_instrumented_model("BigGAN-512", "husky", bad, DEV, model=m)
        assert not any(len(mod._forward_hooks) for _, mod in m.model.named_modules()), bad
        inst = _inst(m, [bad])
        try:
            with pytest.raises(NotImplementedError, match="materialises the outputs"):
                m.forward(m.sample_latent(1, seed=1))
        finally:
            inst.close()
    for bad in ("generator.layers.3", "generator.layers.0.bn_1", "generator.bn"):
        with pytest.raises(NotImplementedError, match="generator.gen_z"):
            m.affine_layer(bad)


def test_abi_symbols():
    from ganspace_b200 import _native
    lib = _native.load()
    for sym in ("gsb_biggan_bn_rows", "gsb_biggan_bn_table_rows", "gsb_biggan_bn_table"):
        assert hasattr(lib, sym), sym
