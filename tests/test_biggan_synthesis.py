"""BigGAN-deep module tree on the CPU: names, state-dict keys and shapes of the reference's (a pytorch_model.bin loads by key), and the
random init plus the shared post-init fill against the checksums the reference wrote (oracle/gen_golden_biggan_synth.py)."""
import numpy as np
import pytest
import torch


@pytest.fixture(scope="module")
def ka(golden):
    return golden("biggan_synthesis_known_answers.npz")


def _net(resolution, seed=4321):
    from ganspace_b200.models import biggan
    torch.manual_seed(seed)
    net = biggan._BigGANNet(resolution)
    biggan.synthesis_fill(net, seed)
    return net


def _check_init(sd, keys, sums, sq):
    assert list(sd) == [str(k) for k in keys]
    fill = ("running_means", "running_vars", "gamma", "generator.bn.weight", "generator.bn.bias")
    for k, s, q in zip(keys, sums, sq):
        t = sd[str(k)].double()
        if any(f in str(k) for f in fill):
            # the fill propagates second moments with fp64 matrix products: last-bit differences between BLAS builds
            np.testing.assert_allclose([t.sum().item(), t.pow(2).sum().item()], [s, q], rtol=1e-6, err_msg=str(k))
        else:                                       # torch's own init under manual_seed: bit-identical
            assert t.sum().item() == s and t.pow(2).sum().item() == q, str(k)


def test_512_tree_keys_shapes_and_init(ka):
    net = _net(512)
    sd = net.state_dict()
    assert [str(tuple(v.shape)) for v in sd.values()] == [str(s) for s in ka["sd512_shapes"]]
    _check_init(sd, ka["sd512_keys"], ka["sd512_sum"], ka["sd512_sq"])
    layers = net.generator.layers
    assert len(layers) == 15 and type(layers[8]).__name__ == "SelfAttn"
    assert [type(m).__name__ for i, m in enumerate(layers) if i != 8] == ["GenBlock"] * 14
    names = {n for n, _ in net.named_modules()}
    assert {"generator.gen_z", "generator.layers.14", "generator.layers.8.snconv1x1_o_conv", "generator.layers.3.bn_2.scale",
            "generator.bn", "generator.conv_to_rgb"} <= names


def test_128_init_matches_reference(ka):
    net = _net(128)
    assert len(net.generator.layers) == 11 and type(net.generator.layers[8]).__name__ == "SelfAttn"
    _check_init(net.state_dict(), ka["sd128_keys"], ka["sd128_sum"], ka["sd128_sq"])


def test_256_shapes():
    net = _net(256, seed=1)
    layers = net.generator.layers
    assert len(layers) == 13 and type(layers[8]).__name__ == "SelfAttn"
    ups = sum(bool(m.up_sample) for m in layers if type(m).__name__ == "GenBlock")
    assert 4 * 2 ** ups == 256
    assert net.generator.conv_to_rgb.weight_orig.shape == (128, 128, 3, 3)
    assert net.generator.layers[-1].conv_3.weight_orig.shape == (128, 64, 1, 1)


def test_gen_z_init_is_a_prefix(golden):
    """gen_z's weights do not change with the synthesis modules added behind it (config 4's known answers)."""
    from ganspace_b200.models import biggan
    torch.manual_seed(4321)
    net = biggan._BigGANNet(512)
    g = golden("biggan_known_answers.npz")
    gz = net.generator.gen_z
    assert np.array_equal(gz.weight_orig[:4, :6].detach().numpy(), g["weight_orig_head"])
    assert np.array_equal(gz.bias[:8].detach().numpy(), g["bias_head"])
    assert np.array_equal(gz.weight_u[:8].numpy(), g["u_head"]) and np.array_equal(gz.weight_v[:8].numpy(), g["v_head"])
    assert np.array_equal(net.embeddings.weight[:4, :6].detach().numpy(), g["emb_head"])


def test_fixture_loads(ka):
    assert ka["z"].shape == (2, 128) and ka["z_list"].shape == (15, 2, 128)
    for k in range(15):
        assert np.isfinite(ka[f"act{k}_sub"]).all()
    assert ka["img_t100_sub"].shape == (2, 3, 64, 64) and ka["img128_sub"].shape == (2, 3, 64, 64)
