"""Component strips on the GPU (ganspace_b200.strips, csrc/strips.cu): the latent kernel against fp64, and the frames of
create_strip / create_strip_centered against the reference's five-frames-per-call loop over the package's own sample_np
(tests/strip_reference.py), for StyleGAN2, StyleGAN, BigGAN-deep and ProGAN with random-init weights."""
import numpy as np
import pytest
import torch

from ganspace_b200 import _native
from ganspace_b200.strips import create_strip, create_strip_centered
from strip_reference import reference_strip, strip_latents_fp64

pytestmark = pytest.mark.gpu

DEV = torch.device("cuda:0")
LATENT_TOL = 1e-6       # max |diff| / max |fp64| of the per-layer latents (a few fp32 roundings, ~2e-7 measured)
# centred frames: the centring's dot product is summed in another order than torch.sum's, a last-bit change of the edited
# latent; what the generator makes of it, max |diff| on the [0, 1] scale, measured on an H100 (random init 1234):
# StyleGAN2 3.2e-6, StyleGAN 1.5e-5, ProGAN 7.2e-7, BigGAN-512 1.4e-2 (its random-init chain amplifies a last-bit change)
CENTRED_TOL = {"StyleGAN2": 2e-5, "StyleGAN": 1e-4, "ProGAN": 5e-6, "BigGAN": 5e-2}


# ---- the latent kernel ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("L,D", [(18, 512), (16, 128), (1, 512)], ids=["StyleGAN2-StyleGAN", "BigGAN-512", "ProGAN"])
@pytest.mark.parametrize("center", [False, True], ids=["plain", "centred"])
@pytest.mark.parametrize("inside", [True, False], ids=["some-layers", "all-layers"])
def test_strip_latents_fp64(L, D, center, inside):
    g = torch.Generator().manual_seed(L * 1000 + D + 7 * center)
    n_lat, n_comp = 3, 4
    lat = torch.randn(n_lat, D, generator=g) * 0.8 + 0.3
    comps = torch.randn(n_comp, D, generator=g) / np.sqrt(D)
    stdev = torch.rand(n_comp, generator=g) * 3 + 0.5
    mean = torch.randn(D, generator=g) * 0.1
    sigmas = torch.from_numpy(np.linspace(-2.5, 2.5, 7).astype(np.float32))
    start, end = ((2, 9) if L > 1 else (0, 1)) if inside else (0, L)
    dev = [t.to(DEV).contiguous() for t in (lat, comps, stdev, mean, sigmas)]
    got = _native.strip_latents(*dev[:3], dev[3] if center else None, dev[4], start, end, L, center)
    torch.cuda.synchronize()
    ref = strip_latents_fp64(lat.numpy(), comps.numpy(), stdev.numpy(), mean.numpy(), sigmas.numpy(), start, end, L, center)
    out = got.cpu().numpy()
    assert out.shape == ref.shape == (L, n_comp * n_lat * 7, D)
    err = np.abs(out - ref).max() / np.abs(ref).max()
    assert err <= LATENT_TOL, err
    # layers outside [start, end) are the latents' own bits
    for l in list(range(start)) + list(range(end, L)):
        assert np.array_equal(out[l], np.repeat(lat.numpy(), 7, axis=0)[None].repeat(n_comp, 0).reshape(-1, D))
    again = _native.strip_latents(*dev[:3], dev[3] if center else None, dev[4], start, end, L, center)
    assert torch.equal(got, again)                       # deterministic
    if not center:
        # the reference's torch expression z + z_comp * sigma * lat_stdev, bit for bit
        z = dev[0].repeat_interleave(7, 0).repeat(n_comp, 1)
        zc = dev[1].repeat_interleave(n_lat * 7, 0)
        sd = dev[2].repeat_interleave(n_lat * 7, 0)[:, None]
        s = dev[4].repeat(n_comp * n_lat)[:, None]
        assert torch.equal(got[start], z - 0 + zc * s * sd)


def test_strip_latents_refuses_bad_ranges():
    x = torch.zeros(1, 8, device=DEV)
    one = torch.ones(1, device=DEV)
    with pytest.raises(_native.NativeError, match="layer range"):
        _native.strip_latents(x, x, one, None, one, 3, 2, 4, False)
    with pytest.raises(_native.NativeError, match="layer range"):
        _native.strip_latents(x, x, one, None, one, 0, 5, 4, False)


# ---- frames --------------------------------------------------------------------------------------------------------------
def _model(name):
    from ganspace_b200.models import get_instrumented_model
    from ganspace_b200.models import ProGAN, StyleGAN, StyleGAN2, stylegan
    from ganspace_b200.models.biggan import BigGAN
    if name == "StyleGAN2":
        m = StyleGAN2(DEV, "ffhq", random_init=1234)
        return get_instrumented_model("StyleGAN2", "ffhq", "style", DEV, model=m, use_w=True)
    if name == "StyleGAN":
        m = StyleGAN(DEV, "bedrooms", random_init=1234)
        stylegan.synthesis_fill(m.model, 7)
        return get_instrumented_model("StyleGAN", "bedrooms", "g_mapping", DEV, model=m, use_w=True)
    if name == "BigGAN":
        m = BigGAN(DEV, 512, "husky", random_init=1234)
        return get_instrumented_model("BigGAN-512", "husky", "generator.gen_z", DEV, model=m)
    m = ProGAN(DEV, "bedroom", random_init=1234)
    return get_instrumented_model("ProGAN", "bedroom", "layer3", DEV, model=m)


MODELS = ["StyleGAN2", "StyleGAN", "BigGAN", "ProGAN"]


@pytest.fixture(scope="module", params=MODELS)
def setup(request):
    inst = _model(request.param)
    model = inst.model
    lats = [model.sample_latent(1, seed=100 + i).reshape(1, -1) for i in range(6)]
    D = lats[0].shape[1]
    many = model.sample_latent(64, seed=5).reshape(64, D)
    mean = many.mean(0, keepdim=True)
    g = torch.Generator().manual_seed(11)
    comps = (torch.randn(3, D, generator=g) / np.sqrt(D)).to(DEV)
    stdev = torch.tensor([0.9, 1.7, 2.3], device=DEV) * many.std(0).mean()
    yield request.param, inst, lats, mean, comps, stdev
    inst.close()
    del model, inst
    torch.cuda.empty_cache()


def _batch_spread(model, lats):
    """The most a frame of the generator changes with the batch it is rendered in: the same per-layer latents rendered as one
    batch, in groups of 5 (as the reference's loop) and one by one; max |diff|.  0 means the chain is batch-invariant."""
    w = torch.cat(lats, 0)
    L = model.get_max_latents()
    full = model.sample_np([w] * L).reshape(len(w), -1)
    parts = np.concatenate([model.sample_np([w[i:i + 5]] * L).reshape(-1, full.shape[1]) for i in range(0, len(w), 5)])
    ones = np.stack([model.sample_np([w[i:i + 1]] * L).reshape(-1) for i in range(len(w))])
    return float(max(np.abs(full - parts).max(), np.abs(full - ones).max()))


def _max_diff(a, b):
    return max(float(np.abs(np.asarray(x, np.float64) - np.asarray(y, np.float64)).max()) for fa, fb in zip(a, b)
               for x, y in zip(fa, fb))


@pytest.mark.parametrize("n_lat,num_frames", [(1, 7), (6, 3)], ids=["batch-over-sigma", "batch-over-latents"])
def test_frames_match_reference_loop(setup, n_lat, num_frames):
    name, inst, lats, mean, comps, stdev = setup
    model = inst.model
    lats = lats[:n_lat]
    L = model.get_max_latents()
    ls, le = (2, 9) if L > 1 else (0, -1)
    spread = _batch_spread(model, lats + [l + 0.01 for l in lats])
    print(f"{name}: the chain's own batch spread {spread:.3g}")
    ref = reference_strip(model, lats, comps[:1], stdev[0], None, 3.0, ls, le, num_frames, False)
    got = create_strip(inst, "latent", None, lats, None, comps[:1], None, stdev[0], 3.0, ls, le, num_frames)
    assert len(got) == n_lat and all(len(s) == num_frames for s in got)
    assert all(f.dtype == np.float32 and f.shape == ref[0][0].shape and f.ndim == 3 for s in got for f in s)
    d = _max_diff(got, ref)
    print(f"{name} {n_lat}x{num_frames}: create_strip max |diff| {d:.3g}")
    assert spread == 0.0, f"the {name} chain gives a latent other bits in another batch (max |diff| {spread:.3g})"
    assert d == 0.0, f"{name}: frames differ by {d} from the reference loop's"
    ref = reference_strip(model, lats, comps[:1], stdev[0], mean, 3.0, ls, le, num_frames, True)
    got = create_strip_centered(inst, "latent", None, lats, None, comps[:1], None, stdev[0], None, mean, 3.0, ls, le, num_frames)
    d = _max_diff(got, ref)
    print(f"{name} {n_lat}x{num_frames}: create_strip_centered max |diff| {d:.3g}")
    assert d <= CENTRED_TOL[name], f"{name}: centred frames differ by {d}"


def _assert_same(a, b, what):
    """Equal frames, bit for bit (every chain is batch-invariant)."""
    d = _max_diff(a, b)
    assert d == 0.0, f"{what}: frames differ by {d}"


def test_components_and_batch_sizes(setup):
    name, inst, lats, mean, comps, stdev = setup
    lats = lats[:2]
    multi = create_strip_centered(inst, "latent", None, lats, None, comps, None, stdev, None, mean, 2.0, 0, -1, 4,
                                  per_component=True)
    assert len(multi) == 3 and all(len(m) == 2 and len(m[0]) == 4 for m in multi)
    for c in range(3):
        single = create_strip_centered(inst, "latent", None, lats, None, comps[c:c + 1], None, stdev[c], None, mean, 2.0, 0, -1, 4)
        _assert_same(multi[c], single, f"{name} component {c}")
    for bs in (1, 7):
        forced = create_strip_centered(inst, "latent", None, lats, None, comps, None, stdev, None, mean, 2.0, 0, -1, 4,
                                       per_component=True, batch_size=bs)
        again = create_strip_centered(inst, "latent", None, lats, None, comps, None, stdev, None, mean, 2.0, 0, -1, 4,
                                      per_component=True, batch_size=bs)
        _assert_same(sum(multi, []), sum(forced, []), f"{name} batch size {bs}")
        _assert_same(forced[0], again[0], f"{name} batch size {bs}, run twice")


def test_uint8_frames(setup):
    name, inst, lats, mean, comps, stdev = setup
    f32 = create_strip(inst, "latent", None, lats[:2], None, comps[:1], None, stdev[0], 4.0, 0, -1, 3, batch_size=4)
    u8 = create_strip(inst, "latent", None, lats[:2], None, comps[:1], None, stdev[0], 4.0, 0, -1, 3, as_uint8=True, batch_size=4)
    for sa, sb in zip(f32, u8):
        for a, b in zip(sa, sb):
            assert b.dtype == np.uint8 and np.array_equal(b, np.uint8(a * 255))
