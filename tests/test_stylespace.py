"""StyleGAN2 style space on the host: the oracle's modulation outputs and S-edited images against the unmodified reference
(oracle/gen_golden_stylespace.py S1), the name -> (chain layer, latent entry, width) table of every S layer of the eight
classes, and the list of synthesis sub-modules whose hooks are refused."""
import numpy as np
import pytest

from oracle import ganspace_oracle as go
from oracle import stylespace_oracle as so

SUB = 16               # the fixture's images keep every 16th pixel each way (oracle/gen_golden_stylespace.py)
CLASSES = {"ffhq": 1024, "car": 512, "cat": 256, "church": 256, "horse": 256, "bedrooms": 256, "kitchen": 256, "places": 256}


@pytest.fixture(scope="module")
def ka(golden):
    return golden("stylespace_known_answers.npz")


@pytest.fixture(scope="module")
def params():
    return so.perturb(go.synthesis_random_init(1234, 1024, upto="convs.15"))


def test_oracle_styles_vs_reference(ka, params, mapping_weights):
    """Every S layer's rows for four latents (one global latent) and for a list of 18 per-layer latents."""
    ws, bs = mapping_weights
    names = [str(n) for n in ka["s_names"]]
    assert sorted(names) == sorted(n for n, _, _ in so.style_layers(params)) and len(names) == 26
    w4 = go.mapping_forward(ka["z4"], ws, bs).astype(np.float64)
    S4 = so.styles(np.repeat(w4[:, None], 18, axis=1), params)
    w18 = np.stack([go.mapping_forward(z, ws, bs) for z in ka["z18"]], axis=1).astype(np.float64)      # [2, 18, 512]
    S18 = so.styles(w18, params)
    for name in names:
        key = name.replace(".", "_")
        for got, ref in ((S4[name], ka["s4_" + key]), (S18[name], ka["s18_" + key])):
            assert got.shape == ref.shape, name
            assert np.abs(got - ref).max() < 2e-5 * np.abs(ref).max(), (name, np.abs(got - ref).max() / np.abs(ref).max())
    # the 18 latents differ per layer, so the entries matter: convs.4 reads entry 5, to_rgbs.2 entry 7
    assert np.abs(S18["convs.4.conv.modulation"] - so.modulation_forward(w18[:, 4], params["layers"]["convs.4"]["mod_weight"],
                                                                        params["layers"]["convs.4"]["mod_bias"])).max() > 1e-2


def edited_styles(ka, params, mapping_weights, which, samples=slice(0, 1)):
    """The styles of S1's edit images (latents z4[:2]) with the edit ``which`` applied as nethook applies it."""
    ws, bs = mapping_weights
    w = go.mapping_forward(ka["z4"][:2], ws, bs).astype(np.float64)[samples]
    S = so.styles(np.repeat(w[:, None], 18, axis=1), params)
    if which == "offset":
        S["convs.5.conv.modulation"] = S["convs.5.conv.modulation"] + ka["edit_offset"][samples]
    else:
        s = S["to_rgbs.2.conv.modulation"]
        S["to_rgbs.2.conv.modulation"] = s * (1 - 0.5) + ka["edit_replacement"][None] * 0.5
    return S


@pytest.mark.parametrize("which", ["offset", "ablate"])
def test_oracle_edited_images_vs_reference(ka, params, mapping_weights, which):
    """The first sample of each S1 edit image, rendered in fp64 from the edited styles."""
    img, _ = so.render(edited_styles(ka, params, mapping_weights, which), params, go.fixed_noise(0, 1024))
    img = 0.5 * (img + 1)
    ref = ka[f"img_{which}_sub"][:1]
    scale = np.abs(ref - 0.5).max()
    assert np.abs(img[:, :, ::SUB, ::SUB] - ref).max() < 1e-4 * scale, np.abs(img[:, :, ::SUB, ::SUB] - ref).max() / scale
    # the edit is visible: the unedited image differs
    assert np.abs(ka[f"img_{which}_sub"][:1] - ka["img4_sub"][:1]).max() > 1e-2 * scale


@pytest.mark.parametrize("cls", sorted(CLASSES))
def test_style_layer_table(cls):
    """name -> (key, latent entry, width) for every modulation layer of the class's generator; the key is the position in the
    table, in execution order."""
    from ganspace_b200.models import stylegan2
    g = stylegan2.Generator(CLASSES[cls], 512, 8)
    table = g.style_layers()
    mods = dict(g.named_modules())
    assert {t[0] for t in table} == {n for n in mods if n.endswith(".conv.modulation")}
    n_conv = len(g.convs) + 1
    assert len(table) == n_conv + len(g.to_rgbs) + 1 == {1024: 26, 512: 23, 256: 20}[CLASSES[cls]]
    for pos, (name, key, entry, width) in enumerate(table):
        assert mods[name].weight.shape == (width, 512), name
        assert key == pos, name
        if name == "conv1.conv.modulation":
            assert (key, entry, width) == (0, 0, 512)
        elif name == "to_rgb1.conv.modulation":
            assert (key, entry, width) == (1, 1, 512)
        elif name.startswith("convs."):
            k = int(name.split(".")[1])            # chain layer l = k + 1, after the ToRGBs of layers 0, 2, .., < l
            assert (key, entry, width) == (k + 1 + (k + 2) // 2, k + 1, g.convs[k].conv.in_channel), name
        else:
            j = int(name.split(".")[1])            # ToRGB j + 1, after chain layer 2j + 2
            assert (key, entry, width) == (3 * (j + 1) + 1, 2 * j + 3, g.convs[2 * j + 1].conv.out_channel), name
        assert entry < g.n_latent
    # execution order: conv1, to_rgb1, then per resolution convs.2j, convs.2j+1, to_rgbs.j
    assert [t[0].split(".conv")[0] for t in table[:5]] == ["conv1", "to_rgb1", "convs.0", "convs.1", "to_rgbs.0"]


def test_guard_list():
    from ganspace_b200.models import stylegan2
    g = stylegan2.Generator(256, 512, 8)
    guarded = g.unhookable_layers()
    for name in ("conv1.conv", "conv1.noise", "conv1.activate", "convs.0.conv", "convs.0.conv.blur", "convs.0.noise",
                 "convs.0.activate", "convs.11.conv", "to_rgb1.conv", "to_rgbs.0.conv", "to_rgbs.0.upsample", "to_rgbs.5.upsample"):
        assert name in guarded, name
    hookable = {"conv1", "to_rgb1", "style", "input"} | {f"convs.{k}" for k in range(len(g.convs))} | \
        {f"to_rgbs.{j}" for j in range(len(g.to_rgbs))} | {t[0] for t in g.style_layers()}
    assert not hookable & set(guarded)
    chain = ("conv1.", "to_rgb1.", "convs.", "to_rgbs.")
    expected = {n for n, _ in g.named_modules() if n.startswith(chain) and n.count(".") >= (1 if n.startswith(chain[:2]) else 2)}
    assert set(guarded) == expected - {t[0] for t in g.style_layers()}
    assert "conv1.conv.blur" not in guarded and "to_rgb1.upsample" not in guarded      # neither exists
