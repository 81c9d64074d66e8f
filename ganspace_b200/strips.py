"""Component strips on the GPU: ``create_strip``, ``create_strip_centered`` and ``pad_frames``.

The reference's notebooks/notebook_utils.py:22-172 and utils.py:26-41, with the same signatures and results, for
``mode='latent'`` on StyleGAN2, StyleGAN (v1), BigGAN-deep and ProGAN.  Where the reference renders five frames per
``sample_np`` call and builds the edited per-layer latent list in PyTorch for each call, here

* one ``gsb_strip_latents`` launch pair builds the edited latents of every frame (all latents, components and sigmas) as
  one [L, F, D] device buffer (csrc/strips.cu);
* the frames go through the model's own ``forward`` in launch groups of many frames, sized from free device memory;
* one ``gsb_strip_pack_frames`` launch per group clamps the images and writes NHWC frames, and one device -> host copy per
  group brings them back (through a pinned buffer, overlapped with the next group's rendering).

Each latent and component is taken as a flat D-vector: the centring dot product and the component's norm run over all
of its D entries (the reference's ``dim=-1``, which is the same for the [1, D] latents of StyleGAN2, StyleGAN and BigGAN).

Like the reference, a call first runs ``inst.close()``: the instrumented model's retained layers and edits are dropped.
Activation edits (``mode='activation'`` / ``'both'``) would have to be re-fed into the fused chains, which is not built:
they raise ``NotImplementedError``.
"""
from __future__ import annotations

import numpy as np
import torch

from . import _native

_PROBE_FRAMES = 4               # frames of the first launch group, whose peak allocation sizes the later groups
_MAX_GROUP_BYTES = 256 << 20    # host staging per launch group (two pinned buffers of this size at most)


def pad_frames(strip, pad_fract_horiz=64, pad_fract_vert=0, pad_value=None):
    """utils.py:26-41: the frames of ``strip`` with a bar of ``pad_value`` (1.0 for float frames, the dtype's maximum for
    integer frames) between consecutive frames, W // pad_fract_horiz wide (or, with pad_fract_horiz = 0, H // pad_fract_vert
    tall); returns the list of frames and bars."""
    dtype = strip[0].dtype
    if pad_value is None:
        pad_value = 1.0 if dtype in (np.float32, np.float64) else np.iinfo(dtype).max
    out = [strip[0]]
    for frame in strip[1:]:
        H, W = frame.shape[0], frame.shape[1]
        if pad_fract_horiz > 0:
            out.append(pad_value * np.ones((H, W // pad_fract_horiz, 3), dtype=dtype))
        elif pad_fract_vert > 0:
            out.append(pad_value * np.ones((H // pad_fract_vert, W, 3), dtype=dtype))
        out.append(frame)
    return out


def layer_range(max_lat, layer_start, layer_end):
    """The edited layers [start, end) of ``_create_strip_impl``: an end below 0 or past ``max_lat`` means ``max_lat``; the
    start is clipped to [0, end]."""
    end = max_lat if (layer_end < 0 or layer_end > max_lat) else layer_end
    return int(np.clip(layer_start, 0, end)), int(end)


def batches_over_latents(n_lat, num_frames):
    """The reference's branch: ``_create_strip_batch_lat`` when there are more latents than frames, else
    ``_create_strip_batch_sigma``."""
    return n_lat > num_frames


def sigma_ladder(sigma, num_frames, n_lat):
    """The fp32 sigmas of a strip as the reference's branch builds them: ``np.linspace`` in float64 cast to float32
    (batch over sigma), or ``np.linspace(..., dtype=np.float32)`` (batch over latents)."""
    if batches_over_latents(n_lat, num_frames):
        return np.linspace(-sigma, sigma, num_frames, dtype=np.float32)
    return np.linspace(-sigma, sigma, num_frames).astype(np.float32)


def create_strip(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, sigma, layer_start, layer_end, num_frames=5,
                 *, per_component=False, as_uint8=False, batch_size=None):
    """notebook_utils.py:22-24: ``frames[i_lat] = [frame_0, ..., frame_{num_frames-1}]``, latent ``i_lat`` moved along
    ``z_comp`` by ``sigma_k * lat_stdev`` (sigma_k from -sigma to sigma) in layers [layer_start, layer_end); float32 [H, W, 3]
    frames in [0, 1].  See ``create_strip_centered`` for the keyword-only arguments."""
    return _strips(inst, mode, latents, z_comp, lat_stdev, None, sigma, layer_start, layer_end, num_frames, False, per_component,
                   as_uint8, batch_size)


def create_strip_centered(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, act_mean, lat_mean, sigma, layer_start,
                          layer_end, num_frames=5, *, per_component=False, as_uint8=False, batch_size=None):
    """notebook_utils.py:26-29: as ``create_strip``, with each latent first moved onto ``lat_mean`` along the component.

    Keyword-only extensions:

    * ``per_component``: ``z_comp`` holds n_comp components [n_comp, ...] and ``lat_stdev`` their n_comp stdevs (or one for
      all); returns ``frames[i_comp][i_lat]``, all of them rendered in the same launch groups;
    * ``as_uint8``: uint8 frames, ``np.uint8(frame * 255)`` of the float frames;
    * ``batch_size``: frames per launch group; None sizes the groups from free device memory.  The frames do not depend on it.

    ``x_comp``, ``act_stdev`` and ``act_mean`` are the activation edit's, which the latent mode does not read."""
    return _strips(inst, mode, latents, z_comp, lat_stdev, lat_mean, sigma, layer_start, layer_end, num_frames, True, per_component,
                   as_uint8, batch_size)


def _flat_rows(x, rows, dev, what):
    t = (x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))).to(device=dev, dtype=torch.float32)
    if t.numel() % rows:
        raise ValueError(f"{what}: {t.numel()} values do not split into {rows} rows")
    return t.reshape(rows, -1).contiguous()


def _strips(inst, mode, latents, z_comp, lat_stdev, lat_mean, sigma, layer_start, layer_end, num_frames, center, per_component,
            as_uint8, batch_size):
    if mode in ("activation", "both"):
        raise NotImplementedError(f"create_strip mode '{mode}': an activation edit cannot be propagated through the fused "
                                  "chains; only mode='latent' is built")
    if mode != "latent":
        raise ValueError(f"unknown create_strip mode '{mode}'")
    if num_frames < 1:
        raise ValueError(f"num_frames = {num_frames}")
    model = inst.model
    inst.close()                                   # as the reference: no retained layer, no edit
    dev = model.device
    L = model.get_max_latents()
    start, end = layer_range(L, layer_start, layer_end)
    latents = latents if isinstance(latents, list) else list(latents)
    n_lat = len(latents)
    z = torch.cat([_flat_rows(v, 1, dev, "latent") for v in latents])
    D = z.shape[1]
    n_comp = (z_comp.shape[0] if per_component else 1)
    comps = _flat_rows(z_comp, n_comp, dev, "z_comp")
    stdev = _flat_rows(lat_stdev, 1, dev, "lat_stdev").reshape(-1)
    if stdev.numel() == 1:
        stdev = stdev.expand(n_comp).contiguous()
    if comps.shape[1] != D or stdev.numel() != n_comp:
        raise ValueError(f"z_comp rows of {comps.shape[1]} values and {stdev.numel()} lat_stdev values for {n_comp} components "
                         f"of latents of {D} values")
    mean = _flat_rows(lat_mean, 1, dev, "lat_mean").reshape(-1) if center else None
    if center and mean.numel() != D:
        raise ValueError(f"lat_mean has {mean.numel()} values, the latents {D}")
    sigmas = torch.from_numpy(sigma_ladder(sigma, num_frames, n_lat)).to(dev)
    with torch.no_grad(), torch.cuda.device(dev):
        w = _native.strip_latents(z, comps, stdev, mean, sigmas, start, end, L, center)
        frames = _render(model, w, torch.uint8 if as_uint8 else torch.float32, batch_size)
    out = [[[frames[(c * n_lat + i) * num_frames + k] for k in range(num_frames)] for i in range(n_lat)] for c in range(n_comp)]
    return out if per_component else out[0]


_pinned = {}        # (slot, dtype) -> grow-only pinned host staging buffer


def _staging(slot, numel, dtype):
    buf = _pinned.get((slot, dtype))
    if buf is None or buf.numel() < numel:
        buf = _pinned[(slot, dtype)] = torch.empty(numel, dtype=dtype, pin_memory=True)
    return buf[:numel]


def _render(model, w, dtype, batch_size):
    """The frames of the per-layer latents ``w`` [L, F, D] through ``model.forward``, packed as one host array [F, H, W, 3]."""
    F = w.shape[1]
    stream = torch.cuda.current_stream()
    frames = None
    pending = None                                  # (event, pinned buffer, first frame, frame count) of the previous group

    def drain():
        ev, buf, f0, n = pending
        ev.synchronize()
        frames[f0:f0 + n] = buf.numpy().reshape(n, *frames.shape[1:])

    f0, group, k = 0, batch_size, 0
    while f0 < F:
        n = min(F - f0, group or _PROBE_FRAMES)
        if group is None:                           # the first group measures the bytes a frame takes
            base = torch.cuda.memory_allocated()
            torch.cuda.reset_peak_memory_stats()
        img = model.forward(list(w[:, f0:f0 + n].unbind(0)))
        if frames is None:
            frames = np.empty((F, img.shape[2], img.shape[3], 3), dtype=np.uint8 if dtype == torch.uint8 else np.float32)
        dev_frames = _native.pack_frames(img, torch.empty((n, img.shape[2], img.shape[3], 3), dtype=dtype, device=img.device))
        del img
        if group is None:
            group = _group_size((torch.cuda.max_memory_allocated() - base) / n, dev_frames[0].numel() * dev_frames.element_size())
        buf = _staging(k % 2, dev_frames.numel(), dtype)
        buf.copy_(dev_frames.reshape(-1), non_blocking=True)
        ev = torch.cuda.Event()
        ev.record(stream)
        if pending is not None:
            drain()
        pending = (ev, buf, f0, n)
        f0, k = f0 + n, k + 1
    drain()
    return frames


def _group_size(frame_bytes, host_frame_bytes):
    """Frames per launch group: half of the device memory that is free (or cached by PyTorch) over the peak bytes one frame of
    the first group took, at most _MAX_GROUP_BYTES of frames on the host, at least one."""
    free, _ = torch.cuda.mem_get_info()
    free += torch.cuda.memory_reserved() - torch.cuda.memory_allocated()
    n = min(int(0.5 * free / max(frame_bytes, 1.0)), _MAX_GROUP_BYTES // host_frame_bytes)
    return max(1, n)
