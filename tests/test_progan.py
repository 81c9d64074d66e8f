"""ProGAN on the host: the oracle's two forms of a block against each other and against the known answers written by the
unmodified reference (oracle/gen_golden_progan.py), and the module tree / random init / checkpoint loading of
ganspace_b200.models.progan (parameters only -- the arithmetic is the GPU chain, tests/test_progan_gpu.py)."""
import numpy as np
import pytest
import torch

from oracle import progan_oracle as po


@pytest.fixture(scope="module")
def ka(golden):
    return golden("progan_known_answers.npz")


@pytest.fixture(scope="module")
def params():
    return po.progan_random_init(1234)


def _sub(act):
    step = max(1, act.shape[-1] // 16)
    return act[:, ::max(1, act.shape[1] // 8), ::step, ::step]


def test_oracle_matches_reference_known_answers(ka, params):
    names = [str(x) for x in ka["names"]]
    upto = "layer8"                                        # 32 x 32: the deeper blocks are the same two code paths at CPU-minutes cost
    acts = po.progan_forward(ka["z"].reshape(4, -1), params, upto=upto, keep=names)
    for name in names[:names.index(upto) + 1]:
        act, ref = acts[name], ka[f"act_{name}_sub"]
        assert tuple(act.shape) == tuple(ka[f"shape_{name}"]), name
        assert np.abs(_sub(act) - ref).max() < 1e-5 * np.abs(ref).max(), name
        assert abs((act.astype(np.float64) ** 2).sum() - ka[f"sum_{name}"][1]) < 1e-5 * ka[f"sum_{name}"][1], name


def test_tap_form_equals_reference_form(params):
    """The low-resolution tap GEMM + gather of csrc/progan.cu is the reference's block, for all four block kinds."""
    rng = np.random.RandomState(3)
    small = po.progan_random_init(5, sizes=[64, 32, 32])
    x = rng.standard_normal((2, 64, 1, 1)).astype(np.float32)
    for name, L in small.items():
        out = name.startswith("output")
        a, b = po.progan_block_forward(x, L, output=out), po.progan_block_taps(x, L, output=out)
        assert a.shape == b.shape, name
        assert np.abs(a - b).max() <= 5e-6 * np.abs(a).max(), (name, np.abs(a - b).max() / np.abs(a).max())
        x = a
    assert x.shape == (2, 3, 8, 8)


def test_random_init_reproduces_reference_tensors(ka):
    from ganspace_b200.models import progan
    m = progan.random_init(1234)
    sd = m.state_dict()
    assert list(sd) == [str(k) for k in ka["state_dict_keys"]]
    for name in ("layer1", "layer7", "output_256x256"):
        assert np.array_equal(sd[f"{name}.conv.weight"].reshape(-1)[:64].numpy(), ka[f"init_{name}_w"]), name
        assert np.array_equal(sd[f"{name}.wscale.b"].reshape(-1)[:3].numpy(), ka[f"init_{name}_b"]), name
    p = po.progan_random_init(1234)
    for name in ("layer2", "layer13"):
        assert np.array_equal(sd[f"{name}.conv.weight"].numpy(), p[name]["weight"]) and np.array_equal(sd[f"{name}.wscale.b"].numpy(), p[name]["b"])
    assert m.block_names() == [str(x) for x in ka["names"]]
    assert [(blk.upsample, blk.conv.kernel_size[0]) for blk in m][:4] == [(False, 4), (False, 3), (True, 3), (False, 3)]
    assert abs(m.layer3.wscale.scale - np.sqrt(2) / 3 / np.sqrt(512)) < 1e-12 and abs(m.output_256x256.wscale.scale - 1 / np.sqrt(32)) < 1e-12


def test_both_checkpoint_key_formats_load():
    from ganspace_b200.models import progan
    torch.manual_seed(0)
    src = progan.ProgressiveGenerator(sizes=[64, 32, 32])
    sd = src.state_dict()
    a = progan.from_state_dict({"state_dict": dict(sd)})
    old = {}
    for k, v in sd.items():
        block, rest = k.split(".", 1)
        old[("output." if block.startswith("output") else f"features.{int(block[5:]) - 1}.") + rest] = v
    b = progan.from_state_dict(old)
    for m in (a, b):
        assert m.block_names() == ["layer1", "layer2", "layer3", "layer4", "output_8x8"]
        assert all(torch.equal(m.state_dict()[k], sd[k]) for k in sd)
    with pytest.raises(NotImplementedError):
        a.layer1(torch.zeros(1, 64, 1, 1))
