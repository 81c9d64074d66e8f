"""ORACLE / TEST INFRASTRUCTURE -- StyleGAN (v1) generator (models/stylegan/model.py:26-376), restated from its equations twice:

  * ``layer_reference``  the reference's own form, fp64 torch on the host: nearest x2 + F.conv2d below 128 px, the pad-and-sum
                         4x4 kernel under F.conv_transpose2d from 128 px, the blur as a depthwise conv, InstanceNorm, StyleMod
  * ``layer_taps``       the form the kernels of csrc/stylegan.cu compute, fp64 NumPy: one contraction over ci per tap at the INPUT
                         resolution and a gather (the kernel flipped in both axes from 128 px), the blur with explicit zero padding,
                         InstanceNorm and StyleMod as one affine per (sample, channel)
tests/test_stylegan.py pins the two to each other.  Parameters are a state dict in the reference's key format (NumPy or torch
values); ``mapping`` restates g_mapping.  Nothing under ganspace_b200/ imports this module.
"""
import numpy as np

DLATENT = 512


def _np(t):
    return t.detach().cpu().numpy() if hasattr(t, "detach") else np.asarray(t)


def block_names(resolution):
    return [f"{2 ** r}x{2 ** r}" for r in range(2, int(np.log2(resolution)) + 1)]


def layers(sd, resolution):
    """[(block, conv_prefix or None, epi_prefix, upsample, res_out)] in execution order, two per block."""
    out = []
    for i, b in enumerate(block_names(resolution)):
        r, p = int(b.split("x")[0]), f"g_synthesis.blocks.{b}"
        if i == 0:
            out += [(b, None, f"{p}.epi1", False, r), (b, f"{p}.conv", f"{p}.epi2", False, r)]
        else:
            out += [(b, f"{p}.conv0_up", f"{p}.epi1", True, r), (b, f"{p}.conv1", f"{p}.epi2", False, r)]
    return out


def mapping(z, sd):
    """g_mapping in fp64: PixelNorm, then 8 x lrelu_0.2(x (W sqrt2 0.01 / sqrt512)^T + 0.01 b)."""
    x = np.asarray(z, np.float64).reshape(len(z), -1)
    x = x / np.sqrt(np.mean(x * x, axis=1, keepdims=True) + 1e-8)
    for i in range(8):
        W, b = _np(sd[f"g_mapping.dense{i}.weight"]).astype(np.float64), _np(sd[f"g_mapping.dense{i}.bias"]).astype(np.float64)
        x = x @ (W * (np.sqrt(2) * 0.01 / np.sqrt(DLATENT))).T + 0.01 * b
        x = np.where(x >= 0, x, 0.2 * x)
    return x


def style(w, sd, epi):
    """StyleMod vectors (s0, s1), each [n, C], for dlatents w [n, 512]."""
    A, b = _np(sd[f"{epi}.style_mod.lin.weight"]).astype(np.float64), _np(sd[f"{epi}.style_mod.lin.bias"]).astype(np.float64)
    s = np.asarray(w, np.float64) @ (A / np.sqrt(DLATENT)).T + b
    C = A.shape[0] // 2
    return s[:, :C], s[:, C:]


def layer_reference(x, w, sd, conv, epi, up, noise):
    """One layer in the reference's form (fp64 torch on the host).  x [n, ci, H, H] (ignored for the constant input), w [n, 512]."""
    import torch
    T = lambda a: torch.from_numpy(np.ascontiguousarray(_np(a), dtype=np.float64))
    keys = [k for k in sd if k.startswith((epi.rsplit(".", 1)[0] + ".", f"{conv}.", f"{epi}."))]
    return layer_torch(None if x is None else T(x), T(w), {k: T(sd[k]) for k in keys}, conv, epi, up, T(noise)).numpy()


def layer_torch(t, w, sd, conv, epi, up, noise):
    """``layer_reference`` on torch tensors of any dtype and device (tools/bench_stylegan.py's plain-PyTorch baseline)."""
    import torch
    import torch.nn.functional as F
    if conv is None:
        blk = epi.rsplit(".", 1)[0]
        t = sd[f"{blk}.const"].expand(len(w), -1, -1, -1) + sd[f"{blk}.bias"].view(1, -1, 1, 1)
    else:
        W = sd[f"{conv}.weight"]
        W = W * float(np.sqrt(2) / np.sqrt(W.shape[1] * 9))
        if up and t.shape[2] * 2 >= 128:                   # model.py:82-91
            k = F.pad(W.permute(1, 0, 2, 3), (1, 1, 1, 1))
            k = k[:, :, 1:, 1:] + k[:, :, :-1, 1:] + k[:, :, 1:, :-1] + k[:, :, :-1, :-1]
            t = F.conv_transpose2d(t, k, stride=2, padding=(k.size(-1) - 1) // 2)
        else:
            if up:
                t = t.repeat_interleave(2, dim=2).repeat_interleave(2, dim=3)
            t = F.conv2d(t, W, None, padding=1)
        if up:
            k = torch.tensor([1.0, 2.0, 1.0], dtype=t.dtype, device=t.device)
            k = (k[:, None] * k[None, :] / 16)[None, None].expand(t.shape[1], -1, -1, -1)
            t = F.conv2d(t, k, padding=1, groups=t.shape[1])
        t = t + sd[f"{conv}.bias"].view(1, -1, 1, 1)
    t = t + sd[f"{epi}.top_epi.noise.weight"].view(1, -1, 1, 1) * noise.view(1, 1, *t.shape[2:])
    t = F.leaky_relu(t, 0.2)
    t = F.instance_norm(t, eps=1e-5)
    A = sd[f"{epi}.style_mod.lin.weight"]
    s = w @ (A / float(np.sqrt(DLATENT))).T + sd[f"{epi}.style_mod.lin.bias"]
    C = A.shape[0] // 2
    return t * (s[:, :C, None, None] + 1) + s[:, C:, None, None]


def _gather(Y, R, up):
    """sum_tap Y[b, src(y + ky - 1), src(x + kx - 1), ky, kx, :] over in-range taps; src = >>1 on the up-sampled grid."""
    B, co = Y.shape[0], Y.shape[-1]
    out = np.zeros((B, R, R, co))
    idx = np.arange(R)
    for ky in range(3):
        yy = idx + ky - 1
        my = (yy >= 0) & (yy < R)
        ys = (yy[my] >> 1) if up else yy[my]
        for kx in range(3):
            xx = idx + kx - 1
            mx = (xx >= 0) & (xx < R)
            xs = (xx[mx] >> 1) if up else xx[mx]
            out[np.ix_(np.arange(B), idx[my], idx[mx])] += Y[:, ys][:, :, xs][:, :, :, ky, kx, :]
    return out


def layer_taps(x, w, sd, conv, epi, up, noise):
    """One layer in the kernels' form (fp64 NumPy, NHWC inside, NCHW in and out)."""
    n = len(w)
    if conv is None:
        blk = epi.rsplit(".", 1)[0]
        f = np.broadcast_to(_np(sd[f"{blk}.const"]).astype(np.float64).transpose(0, 2, 3, 1), (n, 4, 4, _np(sd[f"{blk}.bias"]).shape[0]))
        f = f + _np(sd[f"{blk}.bias"]).astype(np.float64)
    else:
        xh = np.asarray(x, np.float64).transpose(0, 2, 3, 1)
        W = _np(sd[f"{conv}.weight"]).astype(np.float64)
        W = W * (np.sqrt(2) / np.sqrt(W.shape[1] * 9))
        R = 2 * xh.shape[1] if up else xh.shape[1]
        if up and R >= 128:                                # the conv_transpose2d branch: the flipped kernel
            W = W[:, :, ::-1, ::-1]
        f = _gather(np.tensordot(xh, W, axes=([3], [1])).transpose(0, 1, 2, 4, 5, 3), R, up)      # [B, H, H, 3, 3, co]
        if up:                                             # [1,2,1]^2 / 16 blur, zero padding of the conv output
            p = np.pad(f, ((0, 0), (1, 1), (1, 1), (0, 0)))
            k = np.array([1.0, 2.0, 1.0]) / 4
            f = sum(k[dy] * k[dx] * p[:, dy:dy + R, dx:dx + R] for dy in range(3) for dx in range(3))
        f = f + _np(sd[f"{conv}.bias"]).astype(np.float64)
    f = f + _np(sd[f"{epi}.top_epi.noise.weight"]).astype(np.float64) * np.asarray(_np(noise), np.float64).reshape(1, *f.shape[1:3], 1)
    f = np.where(f >= 0, f, 0.2 * f)
    mean = f.mean(axis=(1, 2), keepdims=True)
    var = (f * f).mean(axis=(1, 2), keepdims=True) - mean * mean
    s0, s1 = style(w, sd, epi)
    a = (s0 + 1)[:, None, None, :] / np.sqrt(var + 1e-5)
    return ((f - mean) * a + s1[:, None, None, :]).transpose(0, 3, 1, 2)


def torgb(x, sd):
    W = _np(sd["g_synthesis.torgb.weight"]).astype(np.float64)[:, :, 0, 0]
    out = np.einsum("bchw,oc->bohw", np.asarray(x, np.float64), W / np.sqrt(W.shape[1]))
    return out + _np(sd["g_synthesis.torgb.bias"]).astype(np.float64).reshape(1, 3, 1, 1)


def synthesis(w_layers, sd, noise, resolution, upto=None, form="reference"):
    """{block name: output} for blocks 4x4 .. ``upto`` (default: all, plus 'image' = 0.5 (torgb + 1)).  ``w_layers``: [n, 512]
    (one dlatent for every layer) or [18, n, 512]; ``noise``: {res: [res, res] map}."""
    fn = layer_reference if form == "reference" else layer_taps
    w_layers = np.asarray(w_layers, np.float64)
    per_layer = w_layers.ndim == 3
    out, x = {}, None
    for l, (b, conv, epi, up, r) in enumerate(layers(sd, resolution)):
        x = fn(x, w_layers[l] if per_layer else w_layers, sd, conv, epi, up, noise[r])
        if l % 2 == 1:
            out[b] = x
            if b == upto:
                return out
    out["image"] = 0.5 * (torgb(x, sd) + 1)
    return out


def w18_latents():
    """The 18 distinct W latents (4 samples each) of the known answers' per-layer forward: any W is a valid synthesis input."""
    return [np.random.RandomState(100 + i).standard_normal((4, 512)).astype(np.float32) for i in range(18)]


def fixed_noise(resolution, seed=0):
    """set_noise_seed(seed): torch.randn(1, 1, R, R) right after manual_seed(seed), per resolution."""
    import torch
    maps = {}
    for b in block_names(resolution):
        r = int(b.split("x")[0])
        torch.manual_seed(seed)
        maps[r] = torch.randn(1, 1, r, r).numpy()[0, 0]
    return maps
