"""StyleGAN (v1) on the host: the oracle's two forms of a layer against each other (including an up-conv layer from 128 px, the
reference's conv_transpose2d branch) and against the known answers written by the unmodified reference
(oracle/gen_golden_stylegan.py), and the module tree / random init / fill of ganspace_b200.models.stylegan (parameters only -- the
arithmetic is the GPU chain, tests/test_stylegan_gpu.py)."""
import numpy as np
import pytest
import torch

from oracle import stylegan_oracle as so


@pytest.fixture(scope="module")
def ka(golden):
    return golden("stylegan_known_answers.npz")


def _sub(act):
    step = max(1, act.shape[-1] // 16)
    return act[:, ::max(1, act.shape[1] // 8), ::step, ::step]


def _sd(res):
    from ganspace_b200.models import stylegan
    return stylegan.random_init(1234, res, fill=7).state_dict()


def test_module_tree_and_init_match_reference(ka):
    from ganspace_b200.models import stylegan
    for cls, res in (("ffhq", 1024), ("bedrooms", 256)):
        m = stylegan.random_init(1234, res, fill=7)
        sd = m.state_dict()
        assert list(sd) == [str(k) for k in ka[f"{cls}_state_dict_keys"]], cls
        assert len(list(m.named_modules())) == int(ka[f"{cls}_n_modules"]), cls
        for k in [k for k in ka if k.startswith(f"{cls}_init_")]:
            assert np.array_equal(sd[k[len(cls) + 6:]].reshape(-1)[:64].numpy(), ka[k]), k
    assert int(ka["ffhq_n_modules"]) == 166
    assert m.block_names()[-1] == "g_synthesis.blocks.256x256" and m.g_synthesis.blocks["256x256"].conv1.weight.shape[0] == 64
    torch.manual_seed(1234)
    plain = stylegan.StyleGAN_G(256)
    assert float(plain.g_synthesis.blocks["4x4"].epi1.top_epi.noise.weight.detach().abs().max()) == 0.0      # the reference's degenerate init
    with pytest.raises(NotImplementedError):
        m.g_synthesis.blocks["8x8"](torch.zeros(1, 512, 4, 4))
    with pytest.raises(NotImplementedError):
        m.g_synthesis.blocks["8x8"].conv0_up(torch.zeros(1, 512, 4, 4))


def test_mapping_oracle_matches_reference(ka):
    sd = _sd(256)
    w = so.mapping(ka["bedrooms_z"], sd)
    ref = ka["bedrooms_w"]
    assert np.abs(w - ref).max() <= 1e-5 * np.abs(ref).max()


def test_oracle_matches_reference_known_answers(ka):
    """bedrooms, blocks 4x4 .. 32x32 in both forms and both latent modes (the deeper blocks are the same code paths at CPU-minutes
    cost, except the >= 128 px up-conv, which test_tap_form_equals_reference_form covers)."""
    sd = _sd(256)
    noise = so.fixed_noise(256)
    w = so.mapping(ka["bedrooms_z"], sd)
    for tag, lat in (("z", w), ("w18", np.stack(so.w18_latents()).astype(np.float64))):
        for form in ("reference", "taps"):
            out = so.synthesis(lat, sd, noise, 256, upto="32x32", form=form)
            for b, act in out.items():
                ref = ka[f"bedrooms_{tag}_{b}_sub"]
                assert act.shape[1:] == tuple(ka[f"bedrooms_{b}_shape"][1:]), b
                err = np.abs(_sub(act) - ref).max() / np.abs(ref).max()
                assert err < 1e-4, (tag, form, b, err)


def test_tap_form_equals_reference_form():
    """The low-resolution tap GEMM + gather + blur + one affine of csrc/stylegan.cu is the reference's layer: the constant input,
    a stride-1 conv, an up-conv below 128 px and one at 128 px (the conv_transpose2d branch, flipped kernel), at 16 channels."""
    rng = np.random.RandomState(3)
    sd, C = {}, 16
    for name, ci in (("c", C), ("u", C)):
        sd[f"{name}.weight"] = rng.standard_normal((C, ci, 3, 3))
        sd[f"{name}.bias"] = rng.standard_normal(C)
    for e in ("e0", "e1", "e2", "e3"):
        sd[f"{e}.top_epi.noise.weight"] = rng.standard_normal(C)
        sd[f"{e}.style_mod.lin.weight"] = rng.standard_normal((2 * C, 512))
        sd[f"{e}.style_mod.lin.bias"] = rng.standard_normal(2 * C) * 0.5
    sd["blk.const"], sd["blk.bias"] = rng.standard_normal((1, C, 4, 4)), rng.standard_normal(C)
    sd.update({k.replace("e0.", "blk.e0."): v for k, v in sd.items() if k.startswith("e0.")})     # the constant input's epilogue
    w = rng.standard_normal((2, 512))
    cases = [(None, "blk.e0", False, 4), ("c", "e1", False, 4), ("u", "e2", True, 8), ("u", "e3", True, 128)]
    for conv, epi, up, r in cases:
        x = rng.standard_normal((2, C, r // 2 if up else r, r // 2 if up else r))
        noise = rng.standard_normal((r, r))
        a = so.layer_reference(x, w, sd, conv, epi, up, noise)
        b = so.layer_taps(x, w, sd, conv, epi, up, noise)
        assert a.shape == b.shape == (2, C, r, r), (conv, r)
        err = np.abs(a - b).max() / np.abs(a).max()
        assert err <= 1e-6, (conv, epi, r, err)
    # without the flip the 128 px up-conv is a different function: the check above would catch a port that treats both alike
    x = rng.standard_normal((2, C, 64, 64))
    s = dict(sd)
    s["u.weight"] = sd["u.weight"][:, :, ::-1, ::-1]
    a = so.layer_reference(x, w, sd, "u", "e3", True, np.zeros((128, 128)))
    b = so.layer_taps(x, w, s, "u", "e3", True, np.zeros((128, 128)))
    assert np.abs(a - b).max() > 1e-2 * np.abs(a).max()


def test_unknown_class_and_model_fail_as_the_reference():
    from ganspace_b200.models import get_model
    with pytest.raises(AssertionError, match="Invalid StyleGAN class"):
        get_model("StyleGAN", "nope", torch.device("cpu"))
    with pytest.raises(RuntimeError, match="DCGAN"):
        get_model("DCGAN", "x", torch.device("cpu"))
