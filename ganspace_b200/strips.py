"""Component strips on the GPU: ``create_strip``, ``create_strip_centered`` and ``pad_frames``.

The reference's notebooks/notebook_utils.py:22-172 and utils.py:26-41, with the same signatures and results, on StyleGAN2,
StyleGAN (v1), BigGAN-deep and ProGAN.  Where the reference renders five frames per ``sample_np`` call and builds the edited
per-layer latent list (and the activation offset) in PyTorch for each call, here

* one ``gsb_strip_latents`` launch pair builds the edited latents of every frame (all latents, components and sigmas) as
  one [L, F, D] device buffer (csrc/strips.cu);
* the frames go through the model's own ``forward`` in launch groups of many frames, sized from free device memory;
* with an activation edit (``mode='activation'`` / ``'both'``), one ``gsb_strip_offsets`` launch pair per group writes the
  group's [n, W] offsets, which ``inst.edit_layer`` hands to the layer's hook for that group's ``forward``;
* one ``gsb_strip_pack_frames`` launch per group clamps the images and writes NHWC frames, and one device -> host copy per
  group brings them back (through a pinned buffer, overlapped with the next group's rendering).

Each latent, component and activation is taken as a flat vector: the centring dot product and the component's norm run over
all of its entries (the reference's ``dim=-1``, which is the same for the [1, D] latents and [n, W] rows taken here).

Activation edits are taken on the layers whose edit reaches the image (``model.edit_reaches_image``): style-space rows, the
mapping network's output in Z space and BigGAN's gen_z.  On any other layer (a conv map, which the fused chains cannot take
back) they raise ``NotImplementedError`` before ``inst`` is touched.  Like the reference, a call first runs ``inst.close()``;
unlike it, a call also ends with ``inst.close()``, so no retained layer or edit is left behind.
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
    ``z_comp`` by ``sigma_k * lat_stdev`` (sigma_k from -sigma to sigma) in layers [layer_start, layer_end) (mode 'latent'),
    and/or ``layer``'s value moved by ``x_comp * sigma_k * act_stdev`` (mode 'activation'); 'both' does both; float32 [H, W, 3]
    frames in [0, 1].  See ``create_strip_centered`` for the keyword-only arguments."""
    return _strips(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, None, None, sigma, layer_start, layer_end,
                   num_frames, False, per_component, as_uint8, batch_size)


def create_strip_centered(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, act_mean, lat_mean, sigma, layer_start,
                          layer_end, num_frames=5, *, per_component=False, as_uint8=False, batch_size=None):
    """notebook_utils.py:26-29: as ``create_strip``, with each sample first moved onto the mean along the component: in mode
    'activation' the layer's value onto ``act_mean`` along ``x_comp``, else the latent onto ``lat_mean`` along ``z_comp`` (in
    'both' the activation is not centred, as in the reference).

    Keyword-only extensions:

    * ``per_component``: ``z_comp`` / ``x_comp`` hold n_comp components [n_comp, ...] (the same count in 'both') and
      ``lat_stdev`` / ``act_stdev`` their n_comp stdevs (or one for all); returns ``frames[i_comp][i_lat]``, all of them rendered
      in the same launch groups;
    * ``as_uint8``: uint8 frames, ``np.uint8(frame * 255)`` of the float frames;
    * ``batch_size``: frames per launch group; None sizes the groups from free device memory.  The frames do not depend on it.

    The latent mode does not read ``x_comp``, ``act_stdev`` and ``act_mean``; the activation mode does not read ``z_comp``,
    ``lat_stdev`` and ``lat_mean``."""
    return _strips(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, act_mean, lat_mean, sigma, layer_start,
                   layer_end, num_frames, True, per_component, as_uint8, batch_size)


def _flat_rows(x, rows, dev, what):
    t = (x if torch.is_tensor(x) else torch.as_tensor(np.asarray(x))).to(device=dev, dtype=torch.float32)
    if t.numel() % rows:
        raise ValueError(f"{what}: {t.numel()} values do not split into {rows} rows")
    return t.reshape(rows, -1).contiguous()


def _component_rows(comp, stdev, per_component, dev, what):
    """The [n_comp, width] components and their [n_comp] stdevs (one stdev may serve all)."""
    n_comp = comp.shape[0] if per_component else 1
    comps = _flat_rows(comp, n_comp, dev, what)
    sd = _flat_rows(stdev, 1, dev, f"{what} stdev").reshape(-1)
    if sd.numel() == 1:
        sd = sd.expand(n_comp).contiguous()
    if sd.numel() != n_comp:
        raise ValueError(f"{sd.numel()} stdevs for {n_comp} components of {what}")
    return comps, sd


def _strips(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, act_mean, lat_mean, sigma, layer_start, layer_end,
            num_frames, center, per_component, as_uint8, batch_size):
    if mode not in ("latent", "activation", "both"):
        raise ValueError(f"unknown create_strip mode '{mode}'")
    model = inst.model
    if mode != "latent" and not getattr(model, "edit_reaches_image", lambda _: False)(layer):
        raise NotImplementedError(f"create_strip mode '{mode}': an activation edit on '{layer}' cannot be propagated through the "
                                  "fused chains; activation edits are built on style-space rows, on the mapping network's output "
                                  "in Z space and on BigGAN's generator.gen_z")
    if num_frames < 1:
        raise ValueError(f"num_frames = {num_frames}")
    inst.close()                                   # as the reference: no retained layer, no edit
    try:
        return _strips_closed(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, act_mean, lat_mean, sigma,
                              layer_start, layer_end, num_frames, center, per_component, as_uint8, batch_size)
    finally:
        inst.close()                               # unlike the reference: the last group's edit is not left in place


def _strips_closed(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, act_mean, lat_mean, sigma, layer_start,
                   layer_end, num_frames, center, per_component, as_uint8, batch_size):
    model = inst.model
    dev = model.device
    latents = latents if isinstance(latents, list) else list(latents)
    n_lat = len(latents)
    z = torch.cat([_flat_rows(v, 1, dev, "latent") for v in latents])
    D = z.shape[1]
    sigmas = torch.from_numpy(sigma_ladder(sigma, num_frames, n_lat)).to(dev)
    lat_center = center and mode != "activation"       # in 'both' the reference centres the latent, not the activation
    if mode == "activation":
        # the latents go in unedited: a zero component on an empty layer range, and one latent per frame ([1, F, D])
        n_comp = x_comp.shape[0] if per_component else 1
        comps, stdev = torch.zeros((n_comp, D), device=dev), torch.zeros(n_comp, device=dev)
        L, start, end = 1, 0, 0
    else:
        comps, stdev = _component_rows(z_comp, lat_stdev, per_component, dev, "z_comp")
        n_comp = comps.shape[0]
        if comps.shape[1] != D:
            raise ValueError(f"z_comp rows of {comps.shape[1]} values for latents of {D} values")
        L = model.get_max_latents()
        start, end = layer_range(L, layer_start, layer_end)
    mean = _flat_rows(lat_mean, 1, dev, "lat_mean").reshape(-1) if lat_center else None
    if lat_center and mean.numel() != D:
        raise ValueError(f"lat_mean has {mean.numel()} values, the latents {D}")
    edit = None
    if mode != "latent":
        edit = _activation_edit(inst, layer, z, x_comp, act_stdev, act_mean, sigmas, n_comp, center and mode == "activation",
                                per_component)
    with torch.no_grad(), torch.cuda.device(dev):
        w = _native.strip_latents(z, comps, stdev, mean, sigmas, start, end, L, lat_center)
        frames = _render(model, w[0] if mode == "activation" else w, torch.uint8 if as_uint8 else torch.float32, batch_size, edit)
    out = [[[frames[(c * n_lat + i) * num_frames + k] for k in range(num_frames)] for i in range(n_lat)] for c in range(n_comp)]
    return out if per_component else out[0]


def _activation_edit(inst, layer, z, x_comp, act_stdev, act_mean, sigmas, n_comp, center, per_component):
    """The per-group step of an activation edit: ``edit(f0, n)`` sets the offsets of frames [f0, f0 + n) on ``layer``.  The
    layer's unedited values of the n_lat latents come from one ``partial_forward``; they give its width and, when centring, the
    dot products."""
    model = inst.model
    dev = z.device
    n_lat = z.shape[0]
    with torch.no_grad():
        inst.retain_layer(layer)
        model.partial_forward(z, layer)
        acts = _flat_rows(inst.retained_layer(layer).clone(), n_lat, dev, f"'{layer}' values")
        inst.close()
    W = acts.shape[1]
    comps, stdev = _component_rows(x_comp, act_stdev, per_component, dev, "x_comp")
    if comps.shape[0] != n_comp:
        raise ValueError(f"{comps.shape[0]} x_comp components and {n_comp} z_comp components")
    if comps.shape[1] != W:
        raise ValueError(f"x_comp rows of {comps.shape[1]} values for '{layer}' of {W} values")
    mean = _flat_rows(act_mean, 1, dev, "act_mean").reshape(-1) if center else None
    if center and mean.numel() != W:
        raise ValueError(f"act_mean has {mean.numel()} values, '{layer}' {W}")
    acts = acts if center else None

    def edit(f0, n):
        inst.edit_layer(layer, offset=_native.strip_offsets(acts, comps, stdev, mean, sigmas, n_lat, f0, n, center))
    return edit


_pinned = {}        # (slot, dtype) -> grow-only pinned host staging buffer


def _staging(slot, numel, dtype):
    buf = _pinned.get((slot, dtype))
    if buf is None or buf.numel() < numel:
        buf = _pinned[(slot, dtype)] = torch.empty(numel, dtype=dtype, pin_memory=True)
    return buf[:numel]


def _render(model, w, dtype, batch_size, edit=None):
    """The frames of the per-layer latents ``w`` [L, F, D] (or of the single latents [F, D]) through ``model.forward``, packed as
    one host array [F, H, W, 3].  ``edit(f0, n)``, when given, runs before the forward of frames [f0, f0 + n)."""
    F = w.shape[-2]
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
        if edit is not None:
            edit(f0, n)
        img = model.forward(w[f0:f0 + n] if w.dim() == 2 else list(w[:, f0:f0 + n].unbind(0)))
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
