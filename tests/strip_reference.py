"""A plain restatement of the reference's latent-mode strip loops (notebook_utils.py:31-172) over the package's own
``model.sample_np``: five frames (or five latents) per call, the edited per-layer latent list built with torch ops per call.
What ``ganspace_b200.strips`` is compared with (tests/test_strips_gpu.py) and timed against (tools/bench_strips.py)."""
import numpy as np
import torch

from ganspace_b200.strips import batches_over_latents, layer_range


def _unit(v):
    return v / torch.sqrt(torch.sum(v ** 2, dim=-1, keepdim=True) + 1e-8)


def _images(model, zs):
    img = model.sample_np(zs)
    return img[None] if img.ndim == 3 else img


def reference_strip(model, latents, z_comp, lat_stdev, lat_mean, sigma, layer_start, layer_end, num_frames, center):
    """frames[i_lat] = [num_frames float32 frames], as the reference renders them (latents [1, D] device tensors)."""
    L = model.get_max_latents()
    start, end = layer_range(L, layer_start, layer_end)
    n_lat = len(latents)
    frames = [[] for _ in range(n_lat)]
    with torch.no_grad():
        if not batches_over_latents(n_lat, num_frames):
            B = min(num_frames, 5)
            n_pad = -(-num_frames // B) * B
            ladder = np.concatenate([np.linspace(-sigma, sigma, num_frames), np.zeros(n_pad - num_frames)])
            ladder = torch.from_numpy(ladder).float().to(model.device)
            for g in range(n_pad // B):
                sig = ladder[g * B:(g + 1) * B]
                for i, z1 in enumerate(latents):
                    off = 0
                    if center:
                        off = torch.sum((z1 - lat_mean) * _unit(z_comp), dim=-1, keepdim=True) * _unit(z_comp)
                    zb = z1.repeat_interleave(B, axis=0)
                    delta = z_comp * sig.reshape([-1] + [1] * (z_comp.ndim - 1)) * lat_stdev
                    zs = [zb] * L
                    for l in range(start, end):
                        zs[l] = zs[l] - off + delta
                    for j, img in enumerate(_images(model, zs)):
                        if g * B + j < num_frames:
                            frames[i].append(img)
        else:
            B = min(n_lat, 5)
            ladder = np.linspace(-sigma, sigma, num_frames, dtype=np.float32)
            for g in range(-(-n_lat // B)):
                zg = torch.cat(latents[g * B:(g + 1) * B], 0)
                off = 0
                if center:
                    off = torch.sum((zg - lat_mean) * _unit(z_comp), dim=-1, keepdim=True) * _unit(z_comp)
                for s in ladder:
                    zs = [zg] * L
                    delta = z_comp * s * lat_stdev
                    for l in range(start, end):
                        zs[l] = zs[l] - off + delta
                    for j, img in enumerate(_images(model, zs)):
                        frames[g * B + j].append(img)
    return frames


def strip_latents_fp64(latents, comps, stdev, mean, sigmas, start, end, L, center):
    """fp64 NumPy [L, F, D] per-layer latents of gsb_strip_latents (frame (c * n_lat + i) * n_frames + k)."""
    z, zc = np.asarray(latents, np.float64), np.asarray(comps, np.float64)
    n_lat, D = z.shape
    n_comp, n_frames = zc.shape[0], len(sigmas)
    unit = zc / np.sqrt((zc ** 2).sum(1, keepdims=True) + 1e-8)
    out = np.empty((L, n_comp * n_lat * n_frames, D))
    for c in range(n_comp):
        for i in range(n_lat):
            dot = ((z[i] - np.asarray(mean, np.float64)) * unit[c]).sum() if center else 0.0
            for k, s in enumerate(np.asarray(sigmas, np.float64)):
                f = (c * n_lat + i) * n_frames + k
                out[:, f] = z[i]
                out[start:end, f] = z[i] - dot * unit[c] + zc[c] * s * float(stdev[c])
    return out
