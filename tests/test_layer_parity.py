"""The per-layer comparator of tests/layer_parity.py catches the defects a generator chain's kernels are prone to (CPU only).

Each case restates one layer with the oracle's fp64 forms at a small shape that keeps the structure (a few channels, an 8 -> 16
px up-conv, a 64 -> 128 px up-conv), injects one defect into the kernels' form (oracle/stylegan_oracle.layer_taps) or into the
output, and requires the comparator to report at least 10x the per-layer bar of the GPU tests -- and to point at the cause
(sample, chunk, border ring).  The defect-free kernels' form stays far under the bar."""
import numpy as np
import pytest

from layer_parity import (assert_spans_chunks, compare, parity_batch, progan_chunk_samples, stylegan2_chunk_samples,
                          stylegan_chunk_samples, biggan_chunk_samples)
from oracle import ganspace_oracle as go
from oracle import stylegan_oracle as so

BAR = 1.3e-5           # the loosest per-layer bar of the GPU family tests (StyleGAN v1's PARITY_TOL)
SPC = 4                # samples per chunk of the small cases
BLK = "g_synthesis.blocks.16x16"


def _sg_layer(rng, ci, co, conv, epi):
    """A StyleGAN (v1) layer's parameters in the reference's key format, every term non-zero."""
    return {f"{conv}.weight": rng.standard_normal((co, ci, 3, 3)), f"{conv}.bias": 0.5 * rng.standard_normal(co),
            f"{epi}.top_epi.noise.weight": 0.5 * rng.standard_normal(co),
            f"{epi}.style_mod.lin.weight": rng.standard_normal((2 * co, 512)), f"{epi}.style_mod.lin.bias": 0.5 * rng.standard_normal(2 * co)}


def _upconv_case(res_out=16, n=2, seed=0):
    rng = np.random.RandomState(seed)
    blk = f"g_synthesis.blocks.{res_out}x{res_out}"
    conv, epi = f"{blk}.conv0_up", f"{blk}.epi1"
    sd = _sg_layer(rng, 4, 4, conv, epi)
    x = rng.standard_normal((n, 4, res_out // 2, res_out // 2))
    w = rng.standard_normal((3, n, 512))                   # three layers' latents: l - 1, l, l + 1
    noise = rng.standard_normal((res_out, res_out))
    ref = so.layer_reference(x, w[1], sd, conv, epi, True, noise)
    return sd, conv, epi, x, w, noise, ref


def _bad_gather(Y, R, up):
    """oracle _gather with the up-sampled source row / column off by one: (y + ky) >> 1 instead of (y + ky - 1) >> 1."""
    B, co = Y.shape[0], Y.shape[-1]
    out = np.zeros((B, R, R, co))
    idx = np.arange(R)
    for ky in range(3):
        yy = idx + ky - 1
        my = (yy >= 0) & (yy < R)
        ys = np.minimum((yy[my] + 1) >> 1, R // 2 - 1) if up else yy[my]
        for kx in range(3):
            xx = idx + kx - 1
            mx = (xx >= 0) & (xx < R)
            xs = np.minimum((xx[mx] + 1) >> 1, R // 2 - 1) if up else xx[mx]
            out[np.ix_(np.arange(B), idx[my], idx[mx])] += Y[:, ys][:, :, xs][:, :, :, ky, kx, :]
    return out


def _assert_caught(r, factor=10):
    assert r.err > factor * BAR, str(r)


def test_defect_free_kernel_form_is_far_under_the_bar():
    for res in (16, 128):
        sd, conv, epi, x, w, noise, ref = _upconv_case(res)
        r = compare(so.layer_taps(x, w[1], sd, conv, epi, True, noise), ref, f"up-conv to {res}")
        assert r.err < 1e-3 * BAR, str(r)


def test_neighbours_latent_in_second_chunk():
    n = parity_batch(SPC)
    sd, conv, epi, x, w, noise, ref = _upconv_case(n=n)
    bad = w[1].copy()
    bad[SPC] = bad[SPC - 1]                               # the first sample of chunk 1 reads the last latent of chunk 0
    r = compare(so.layer_taps(x, bad, sd, conv, epi, True, noise), ref, "chunk-local latent", chunk_of=SPC)
    _assert_caught(r)
    assert r.worst[0] == SPC and r.chunk == 1 and (r.per_sample[:SPC] < 1e-10).all(), str(r)


def test_unflipped_kernel_of_the_128px_up_conv():
    sd, conv, epi, x, w, noise, ref = _upconv_case(128)
    bad = dict(sd)
    bad[f"{conv}.weight"] = sd[f"{conv}.weight"][:, :, ::-1, ::-1]      # layer_taps flips it back: the unflipped kernel
    _assert_caught(compare(so.layer_taps(x, w[1], bad, conv, epi, True, noise), ref, "unflipped 128 px"))


def test_up_sample_gather_off_by_one(monkeypatch):
    sd, conv, epi, x, w, noise, ref = _upconv_case(16)
    monkeypatch.setattr(so, "_gather", _bad_gather)
    _assert_caught(compare(so.layer_taps(x, w[1], sd, conv, epi, True, noise), ref, "gather (y + ky) >> 1"))


def test_transposed_noise_map():
    sd, conv, epi, x, w, noise, ref = _upconv_case(16)
    _assert_caught(compare(so.layer_taps(x, w[1], sd, conv, epi, True, noise.T), ref, "transposed noise"))


@pytest.mark.parametrize("axis", [2, 3])
def test_wrong_last_output_row_or_column(axis):
    sd, conv, epi, x, w, noise, ref = _upconv_case(16)
    got = so.layer_taps(x, w[1], sd, conv, epi, True, noise)
    src = [slice(None)] * 4
    dst = [slice(None)] * 4
    src[axis], dst[axis] = -2, -1
    got[tuple(dst)] = got[tuple(src)]                     # e.g. a clamped source index on the far border
    r = compare(got, ref, "last row / column")
    _assert_caught(r)
    assert r.on_border and r.worst[axis] == ref.shape[axis] - 1, str(r)


@pytest.mark.parametrize("slip", [-1, 1])
def test_per_layer_latent_index_slip_stylegan(slip):
    sd, conv, epi, x, w, noise, ref = _upconv_case(16)
    _assert_caught(compare(so.layer_taps(x, w[1 + slip], sd, conv, epi, True, noise), ref, f"latent l{slip:+d}"))


def _s2_layer(rng, ci, co, upsample):
    return dict(weight=rng.standard_normal((co, ci, 3, 3)).astype(np.float32), mod_weight=rng.standard_normal((ci, 512)).astype(np.float32),
                mod_bias=np.ones(ci, np.float32), noise_weight=np.float32(0.3), act_bias=(0.1 * rng.standard_normal(co)).astype(np.float32),
                upsample=upsample)


@pytest.mark.parametrize("slip", [-1, 1])
def test_per_layer_latent_index_slip_stylegan2(slip):
    rng = np.random.RandomState(3)
    L = _s2_layer(rng, 4, 4, True)
    x = rng.standard_normal((2, 4, 8, 8))
    w = rng.standard_normal((3, 2, 512))
    noise = rng.standard_normal((16, 16))
    ref = go.styled_conv_shared(x, w[1], L, noise, dtype=np.float64)
    assert compare(go.styled_conv_taps(x.transpose(0, 2, 3, 1), w[1], L, noise).transpose(0, 3, 1, 2), ref).err < 1e-3 * BAR
    _assert_caught(compare(go.styled_conv_shared(x, w[1 + slip], L, noise, dtype=np.float64), ref, f"latent l{slip:+d}"))


def test_to_rgb_skip_without_up_sampling():
    rng = np.random.RandomState(4)
    R = dict(weight=rng.standard_normal((3, 4)).astype(np.float32), mod_weight=rng.standard_normal((4, 512)).astype(np.float32),
             mod_bias=np.ones(4, np.float32), bias=np.array([0.05, -0.1, 0.15], np.float32))
    x = rng.standard_normal((2, 4, 16, 16))
    w = rng.standard_normal((2, 512))
    skip = rng.standard_normal((2, 3, 8, 8))
    ref = go.to_rgb_forward(x, w, R, skip, dtype=np.float64)
    nearest = skip.repeat(2, axis=2).repeat(2, axis=3)
    _assert_caught(compare(go.to_rgb_forward(x, w, R, None, dtype=np.float64) + nearest, ref, "skip not blurred"))


def test_oracle_dtype_default_is_unchanged():
    """The fp32 default of the oracle forms the reference comparisons use is what it was; fp64 agrees with it to fp32 rounding."""
    rng = np.random.RandomState(5)
    L = _s2_layer(rng, 4, 4, False)
    x = rng.standard_normal((2, 4, 8, 8)).astype(np.float32)
    w = rng.standard_normal((2, 512)).astype(np.float32)
    noise = rng.standard_normal((8, 8)).astype(np.float32)
    a, b = go.styled_conv_shared(x, w, L, noise), go.styled_conv_shared(x, w, L, noise, dtype=np.float64)
    assert a.dtype == np.float32 and b.dtype == np.float64 and compare(a, b).err < 1e-5


def test_chunk_rules_and_batches():
    assert progan_chunk_samples(1, 4, 512) == 1152 and progan_chunk_samples(8, 3, 512) == 32     # layer1, layer4
    assert progan_chunk_samples(256, 3, 32) == 1
    assert stylegan_chunk_samples(4, 512, False, False) == 1152 and stylegan_chunk_samples(4, 512, False, True) == 128
    assert stylegan_chunk_samples(1024, 16, True, True) == 1
    assert stylegan2_chunk_samples(4) == 128 and stylegan2_chunk_samples(16) == 8 and stylegan2_chunk_samples(64) == 1
    assert biggan_chunk_samples(4) == 8 and biggan_chunk_samples(8) == 2 and biggan_chunk_samples(16) == 1
    for spc in (1, 2, 8, 128, 1152):
        n = parity_batch(spc)
        assert_spans_chunks(n, spc)
    with pytest.raises(AssertionError):
        assert_spans_chunks(8, 8)
    with pytest.raises(AssertionError):
        assert_spans_chunks(16, 8)
