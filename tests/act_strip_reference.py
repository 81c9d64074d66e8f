"""A plain restatement of the reference's strip loops in every mode (notebook_utils.py:31-172) over ``inst.edit_layer`` and the
package's own ``model.sample_np``: five frames (or five latents) per call, the activation offset and the edited per-layer latent
list built with torch ops per call; and an fp64 restatement of gsb_strip_offsets.  What the activation modes of
``ganspace_b200.strips`` are compared with (tests/test_activation_strips_gpu.py) and timed against (tools/bench_strips.py)."""
import numpy as np
import torch

from ganspace_b200.strips import batches_over_latents, layer_range
from strip_reference import _images, _unit


def reference_act_strip(inst, mode, layer, latents, x_comp, z_comp, act_stdev, lat_stdev, act_mean, lat_mean, sigma, layer_start,
                        layer_end, num_frames, center):
    """frames[i_lat] of notebook_utils.py:31-172 in any mode, restated over ``inst.edit_layer`` and the package's ``sample_np``:
    five frames (or five latents) per call, the offsets and latents built with torch ops per call.  One difference: the layer is
    retained for the centring with the previous call's edit removed, since the retained value is the unedited one either way and
    an edit with five rows cannot be applied to the one-latent run the reference makes there.  Leaves ``inst`` closed."""
    model = inst.model
    L = model.get_max_latents()
    start, end = layer_range(L, layer_start, layer_end)
    n_lat = len(latents)
    frames = [[] for _ in range(n_lat)]

    def unedited(z):
        inst.remove_edits(layer)
        inst.retain_layer(layer)
        model.sample_np(z)
        return inst.retained_features()[layer].clone()

    inst.close()
    with torch.no_grad():
        if not batches_over_latents(n_lat, num_frames):
            B = min(num_frames, 5)
            n_pad = -(-num_frames // B) * B
            ladder = np.concatenate([np.linspace(-sigma, sigma, num_frames), np.zeros(n_pad - num_frames)])
            ladder = torch.from_numpy(ladder).float().to(model.device)
            for g in range(n_pad // B):
                sig = ladder[g * B:(g + 1) * B]
                for i, z1 in enumerate(latents):
                    off_act, off_lat = 0, 0
                    if center and mode == "activation":
                        value = unedited(z1)
                        off_act = _unit(x_comp) * torch.sum((value - act_mean) * _unit(x_comp), dim=-1, keepdim=True)
                    elif center:
                        off_lat = torch.sum((z1 - lat_mean) * _unit(z_comp), dim=-1, keepdim=True) * _unit(z_comp)
                    z = z1.repeat_interleave(B, axis=0)
                    if mode in ("latent", "both"):
                        z = [z] * L
                        delta = z_comp * sig.reshape([-1] + [1] * (z_comp.ndim - 1)) * lat_stdev
                        for l in range(start, end):
                            z[l] = z[l] - off_lat + delta
                    if mode in ("activation", "both"):
                        comp_batch = x_comp.repeat_interleave(B, axis=0)
                        delta = comp_batch * sig.reshape([-1] + [1] * (comp_batch.ndim - 1))
                        inst.edit_layer(layer, offset=delta * act_stdev - off_act)
                    for j, img in enumerate(_images(model, z)):
                        if g * B + j < num_frames:
                            frames[i].append(img)
        else:
            B = min(n_lat, 5)
            ladder = np.linspace(-sigma, sigma, num_frames, dtype=np.float32)
            for g in range(-(-n_lat // B)):
                zg = torch.cat(latents[g * B:(g + 1) * B], 0)
                inst.close()
                off_act, off_lat = 0, 0
                if center and mode == "activation":
                    value = unedited(zg)
                    off_act = _unit(x_comp) * torch.sum((value - act_mean) * _unit(x_comp), dim=-1, keepdim=True)
                elif center:
                    off_lat = torch.sum((zg - lat_mean) * _unit(z_comp), dim=-1, keepdim=True) * _unit(z_comp)
                for s in ladder:
                    z = [zg] * L
                    if mode in ("latent", "both"):
                        delta = z_comp * s * lat_stdev
                        for l in range(start, end):
                            z[l] = z[l] - off_lat + delta
                    if mode in ("activation", "both"):
                        inst.edit_layer(layer, offset=x_comp * s * act_stdev - off_act)
                    for j, img in enumerate(_images(model, z)):
                        frames[g * B + j].append(img)
    inst.close()
    return frames


def strip_offsets_fp64(acts, comps, stdev, mean, sigmas, n_lat, f0, n, center):
    """fp64 NumPy [n, W] offsets of gsb_strip_offsets for frames [f0, f0 + n) (frame (c * n_lat + i) * n_frames + k)."""
    x = np.asarray(comps, np.float64)
    n_frames = len(sigmas)
    unit = x / np.sqrt((x ** 2).sum(1, keepdims=True) + 1e-8)
    out = np.empty((n, x.shape[1]))
    for f in range(f0, f0 + n):
        c, i, k = f // n_frames // n_lat, f // n_frames % n_lat, f % n_frames
        out[f - f0] = x[c] * float(sigmas[k]) * float(stdev[c])
        if center:
            out[f - f0] -= unit[c] * ((np.asarray(acts[i], np.float64) - np.asarray(mean, np.float64)) * unit[c]).sum()
    return out
