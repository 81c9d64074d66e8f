"""BigGAN-deep conditional-BatchNorm row layers on the host: the row-layer table of ganspace_b200.models.biggan at 128, 256 and 512,
the fp64 oracle's rows against the rows the unmodified reference retained (oracle/gen_golden_biggan_stylespace.py), and the list of
sub-modules whose hooks the chain still refuses (the device runs are tests/test_biggan_stylespace_gpu.py)."""
import numpy as np
import pytest

from oracle import biggan_stylespace_oracle as bso

ROW_TOL = 2e-5         # fp64 oracle against the reference's fp32 rows, relative to the layer's max |row|: fp32 sigma and K = 256 products


@pytest.fixture(scope="module")
def ka(golden):
    return golden("biggan_stylespace_known_answers.npz")


@pytest.fixture(scope="module")
def nets():
    return {512: bso.net(512), 128: bso.net(128)}


@pytest.mark.parametrize("res,count,lo,hi", [(512, 112, 32, 2048), (256, 96, 64, 2048), (128, 80, 64, 2048)])
def test_row_layer_table(res, count, lo, hi):
    from ganspace_b200.models import biggan
    net = biggan._BigGANNet(res)
    table = net.style_layers()
    widths = [c for _, c in table]
    assert len(table) == count and min(widths) == lo and max(widths) == hi
    mods = dict(net.named_modules())
    blocks = [k for k, layer in enumerate(net.generator.layers) if isinstance(layer, biggan.GenBlock)]
    assert 8 not in blocks                       # generator.layers.8 is the SelfAttn
    expect = [f"generator.layers.{k}.bn_{j}.{kind}" for k in blocks for j in range(4) for kind in ("scale", "offset")]
    assert [n for n, _ in table] == expect       # execution order: block by block, bn_0 .. bn_3, scale before offset
    for name, c in table:
        m = mods[name]
        assert isinstance(m, biggan.SNLinear) and tuple(m.weight_orig.shape) == (c, 256) and m.bias is None, name
        assert mods[name.rsplit(".", 1)[0]].num_features == c


@pytest.mark.parametrize("res", [512, 128])
def test_oracle_rows_vs_reference(ka, nets, res):
    """The fixture holds a strided sub-sample of each layer's rows and the per-sample sums and sums of squares of the whole rows."""
    net = nets[res]
    table = net.style_layers()
    assert [str(n) for n in ka[f"r{res}_names"]] == [n for n, _ in table]
    assert [int(c) for c in ka[f"r{res}_widths"]] == [c for _, c in table]
    cases = [("z", lambda k: ka["z"])]
    if res == 512:
        from ganspace_b200.models import biggan
        ci = {k: 1 + sum(isinstance(m, biggan.GenBlock) for m in list(net.generator.layers)[:k]) for k in range(len(net.generator.layers))}
        cases.append(("list", lambda k: ka["z_list"][ci[k]]))
    for tag, z_of in cases:
        known = bso.known_rows(ka, res, tag)
        for name, c in table:
            got = bso.rows64(net, name, z_of(int(name.split(".")[2])))
            assert got.shape == (2, c), name
            errs = bso.known_rows_err(got, known[name])
            assert max(errs) < ROW_TOL, (tag, name, errs)


def test_guard_list():
    """Every module inside a block other than the row layers, generator.bn and conv_to_rgb: hooks on them still raise."""
    from ganspace_b200.models import biggan
    net = biggan._BigGANNet(512)
    rows = {n for n, _ in net.style_layers()}
    guarded = net.unhookable_layers()
    assert not rows & set(guarded)
    for name in ("generator.layers.0.bn_0", "generator.layers.0.conv_0", "generator.layers.3.bn_2", "generator.layers.13.conv_3",
                 "generator.layers.8.snconv1x1_theta", "generator.layers.8.snconv1x1_o_conv", "generator.bn",
                 "generator.conv_to_rgb"):
        assert name in guarded, name
    for name in ("generator.gen_z", "generator.layers.0", "generator.layers.8", "embeddings"):
        assert name not in guarded, name
    inner = [n for n, _ in net.named_modules() if n.startswith("generator.layers.") and n.count(".") >= 3]
    assert sorted(set(inner) - rows) == sorted(n for n in guarded if n.count(".") >= 3)
    assert net.unhookable_layers(2, tail=False) == [n for n in guarded if n.startswith(("generator.layers.0.", "generator.layers.1."))]
