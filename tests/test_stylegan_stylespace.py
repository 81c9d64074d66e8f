"""StyleGAN (v1) style space on the host: the oracle's style rows and styled render against the unmodified reference
(oracle/gen_golden_stylegan_stylespace.py), the style-layer table of ganspace_b200.models.stylegan for the 256-, 512- and
1024-px classes, and which hooks the StyleGAN wrapper accepts (the device runs are tests/test_stylegan_stylespace_gpu.py)."""
import numpy as np
import pytest
import torch

from oracle import stylegan_oracle as so
from oracle import stylegan_stylespace_oracle as sso

ROW_TOL = 2e-5         # fp64 oracle against the reference's fp32 rows (K = 512 products after an fp32 mapping network)
IMG_TOL = 1e-3         # fp64 render against the reference's fp32 image, relative to max |img - 0.5|


@pytest.fixture(scope="module")
def ka(golden):
    return golden("stylegan_stylespace_known_answers.npz")


def _key(name):
    return name[len("g_synthesis.blocks."):].replace(".", "_")


def _sd(res):
    from ganspace_b200.models import stylegan
    return stylegan.random_init(1234, res, fill=7).state_dict()


@pytest.mark.parametrize("cls,res", [("ffhq", 1024), ("bedrooms", 256)])
def test_oracle_style_rows_vs_reference(ka, cls, res):
    sd = _sd(res)
    names = sso.style_layer_names(res)
    assert len(names) == {1024: 18, 256: 14}[res]
    w4 = so.mapping(ka[f"{cls}_z4"], sd)
    w18 = so.w18_latents()
    for l, name in enumerate(names):
        epi = name[:-len(".style_mod.lin")]
        for got, ref in ((sso.style_rows(w4, sd, epi), ka[f"{cls}_z4_{_key(name)}"]),
                         (sso.style_rows(w18[l], sd, epi), ka[f"{cls}_w18_{_key(name)}"])):
            assert got.shape == ref.shape == (4, sd[f"{name}.weight"].shape[0]), name
            assert np.abs(got - ref).max() < ROW_TOL * max(1.0, np.abs(ref).max()), (name, np.abs(got - ref).max())


def test_oracle_styled_render_vs_reference_edits(ka):
    """The two edited ffhq images: the oracle's rows, edited as nethook edits them, through the styled fp64 render."""
    sd = _sd(1024)
    names = sso.style_layer_names(1024)
    w2 = so.mapping(ka["ffhq_z4"][:2], sd)
    S = {n: sso.style_rows(w2, sd, n[:-len(".style_mod.lin")]) for n in names}
    off, abl = dict(S), dict(S)
    off["g_synthesis.blocks.16x16.epi2.style_mod.lin"] = S["g_synthesis.blocks.16x16.epi2.style_mod.lin"] + ka["edit_offset"]
    a = "g_synthesis.blocks.4x4.epi1.style_mod.lin"
    abl[a] = 0.5 * S[a] + 0.5 * ka["edit_replacement"][None]
    both = {n: np.concatenate([off[n], abl[n]]) for n in names}
    img = sso.render_styled(both, sd, so.fixed_noise(1024), 1024).numpy()
    for which, got in (("offset", img[:2]), ("ablate", img[2:])):
        ref = ka[f"img_{which}_sub"]
        scale = np.abs(ref - 0.5).max()
        assert np.abs(got[:, :, ::16, ::16] - ref).max() < IMG_TOL * scale, which
        assert abs((got ** 2).sum() - ka[f"img_{which}_sum"][1]) < 1e-4 * ka[f"img_{which}_sum"][1], which
        assert np.abs(ref - ka["img4_sub"]).max() > 1e-2 * scale, which          # the edit shows


@pytest.mark.parametrize("res,widths", [
    (256, [1024] * 8 + [512] * 2 + [256] * 2 + [128] * 2),
    (512, [1024] * 8 + [512] * 2 + [256] * 2 + [128] * 2 + [64] * 2),
    (1024, [1024] * 8 + [512] * 2 + [256] * 2 + [128] * 2 + [64] * 2 + [32] * 2),
])
def test_style_layer_table(res, widths):
    from ganspace_b200.models import stylegan
    net = stylegan.StyleGAN_G(res)
    table = net.style_layers()
    assert [t[0] for t in table] == sso.style_layer_names(res)
    assert [t[1] for t in table] == list(range(len(widths))) and [t[2] for t in table] == list(range(len(widths)))
    assert [t[3] for t in table] == widths
    assert all(w <= 1024 and w % 32 == 0 for w in widths)
    mods = dict(net.named_modules())
    epis = net.g_synthesis.layer_modules()
    for name, l, _, width in table:
        assert mods[name] is epis[l][1].style_mod.lin and mods[name].weight.shape == (width, 512)
    rows = torch.randn(3, widths[0])
    assert mods[table[0][0]](_result=rows) is rows
    with pytest.raises(NotImplementedError):
        mods[table[0][0]](rows[:, :512])


def _wrapper(res):
    """A StyleGAN wrapper around a host module tree, for the hook rules alone (no device, no kernels)."""
    from ganspace_b200.models import stylegan
    from ganspace_b200.models.wrappers import StyleGAN
    m = StyleGAN.__new__(StyleGAN)
    torch.nn.Module.__init__(m)
    m.model = stylegan.StyleGAN_G(res)
    return m


def test_hook_guard_list():
    m = _wrapper(256)
    hookable = m._hookable()
    assert hookable == ["g_mapping"] + m.model.block_names() + sso.style_layer_names(256)
    mods = dict(m.model.named_modules())
    for name in sso.style_layer_names(256)[::3] + ["g_mapping", "g_synthesis.blocks.8x8"]:
        h = mods[name].register_forward_hook(lambda *a: None)
        m._reject_sub_module_hooks()
        h.remove()
    refused = ["g_synthesis.blocks.8x8.epi1.style_mod", "g_synthesis.blocks.8x8.epi1", "g_synthesis.blocks.8x8.epi2.top_epi.noise",
               "g_synthesis.blocks.8x8.epi1.top_epi", "g_synthesis.blocks.8x8.conv1", "g_synthesis.blocks.8x8.conv0_up",
               "g_synthesis.blocks.4x4.conv", "g_synthesis.torgb", "g_mapping.dense3", "g_synthesis"]
    for name in refused:
        h = mods[name].register_forward_hook(lambda *a: None)
        with pytest.raises(NotImplementedError, match="hookable layers") as e:
            m._reject_sub_module_hooks()
        assert "g_synthesis.blocks.256x256.epi2.style_mod.lin" in str(e.value) and f"'{name}'" in str(e.value)
        h.remove()
    m._reject_sub_module_hooks()
