"""Host rules of ganspace_b200.strips against the reference's (notebook_utils.py:31-172, utils.py:26-41): frame padding,
the batching branch and its sigma ladder, the edited layer range, and the refusal of activation edits."""
import numpy as np
import pytest
import torch

from ganspace_b200 import strips


def _pad_reference(strip, horiz, vert, value):
    # utils.py:26-41, restated
    dtype = strip[0].dtype
    if value is None:
        value = 1.0 if dtype in [np.float32, np.float64] else np.iinfo(dtype).max
    out = [strip[0]]
    for f in strip[1:]:
        if horiz > 0:
            out.append(value * np.ones((f.shape[0], f.shape[1] // horiz, 3), dtype=dtype))
        elif vert > 0:
            out.append(value * np.ones((f.shape[0] // vert, f.shape[1], 3), dtype=dtype))
        out.append(f)
    return out


@pytest.mark.parametrize("dtype", [np.float32, np.float64, np.uint8])
@pytest.mark.parametrize("horiz,vert,value", [(64, 0, None), (4, 0, None), (0, 2, None), (0, 0, None), (8, 0, 0.5), (3, 5, 7)])
def test_pad_frames_matches_reference(dtype, horiz, vert, value):
    rng = np.random.default_rng(3)
    strip = [(rng.random((16, 24, 3)) * 200).astype(dtype) for _ in range(4)]
    got = strips.pad_frames(strip, horiz, vert, value)
    want = _pad_reference(strip, horiz, vert, value)
    assert len(got) == len(want)
    for g, w in zip(got, want):
        assert g.dtype == w.dtype and g.shape == w.shape and np.array_equal(g, w)
    assert strips.pad_frames(strip[:1]) == [strip[0]]


@pytest.mark.parametrize("n_lat,num_frames", [(1, 1), (1, 5), (1, 7), (5, 5), (6, 5), (5, 10), (10, 5), (3, 2), (12, 9),
                                              (2, 33), (40, 7)])
@pytest.mark.parametrize("sigma", [2.0, 3.7, 13.0])
def test_sigma_ladder_and_branch(n_lat, num_frames, sigma):
    over_lat = strips.batches_over_latents(n_lat, num_frames)
    assert over_lat == (n_lat > num_frames)                  # _create_strip_impl's test: len(latents) > num_frames
    if over_lat:                                              # _create_strip_batch_lat
        want = np.linspace(-sigma, sigma, num_frames, dtype=np.float32)
    else:                                                     # _create_strip_batch_sigma: float64, padded, then .float()
        B = min(num_frames, 5)
        padded = ((num_frames - 1) // B + 1) * B
        ladder = np.concatenate([np.linspace(-sigma, sigma, num_frames), np.zeros(padded - num_frames)])
        want = torch.from_numpy(ladder).float().numpy()[:num_frames]
    got = strips.sigma_ladder(sigma, num_frames, n_lat)
    assert got.dtype == np.float32 and np.array_equal(got, want)


@pytest.mark.parametrize("max_lat", [1, 14, 16, 18])
@pytest.mark.parametrize("start,end", [(0, -1), (0, 18), (0, 19), (0, 100), (3, 8), (-4, 6), (10, 5), (20, -1), (5, 0),
                                       (0, 1), (7, 7), (2, -30)])
def test_layer_range_matches_reference(max_lat, start, end):
    # _create_strip_impl
    want_end = max_lat if (end < 0 or end > max_lat) else end
    want_start = np.clip(start, 0, want_end)
    got = strips.layer_range(max_lat, start, end)
    assert got == (want_start, want_end)
    assert 0 <= got[0] <= got[1] <= max_lat


class _NoModel:
    """An instrumented model stand-in: the mode is refused before the model is touched."""
    model = None

    def close(self):
        raise AssertionError("closed before the mode was checked")


@pytest.mark.parametrize("mode", ["activation", "both"])
def test_activation_modes_raise(mode):
    z = [torch.zeros(1, 512)]
    with pytest.raises(NotImplementedError, match="cannot be propagated"):
        strips.create_strip(_NoModel(), mode, "style", z, None, torch.zeros(1, 512), 1.0, 1.0, 2.0, 0, -1, 5)
    with pytest.raises(NotImplementedError, match="cannot be propagated"):
        strips.create_strip_centered(_NoModel(), mode, "style", z, None, torch.zeros(1, 512), 1.0, 1.0, None, torch.zeros(1, 512),
                                     2.0, 0, -1, 5)


def test_unknown_mode_raises():
    with pytest.raises(ValueError, match="unknown create_strip mode"):
        strips.create_strip(_NoModel(), "latnet", "style", [torch.zeros(1, 512)], None, torch.zeros(1, 512), 1.0, 1.0, 2.0, 0, -1)
