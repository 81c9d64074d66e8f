"""ORACLE -- StyleGAN2 style space: the modulation layers and a render that takes its styles from the caller.

The style of a StyledConv or ToRGB is s = w (A / sqrt(512))^T + b (EqualLinear, model.py:132-166, 226, 234).  An S-space edit
replaces s; the layer then modulates (and, for a StyledConv, demodulates) with the edited s.  These restate
ganspace_oracle.styled_conv_shared / to_rgb_forward / render_forward with the style as an input, in any dtype; the originals
are left as they are.
"""
import math

import numpy as np

from oracle.ganspace_oracle import BLUR_K2D


def modulation_forward(w, mod_weight, mod_bias, dtype=np.float64):
    """The modulation EqualLinear: w [B, 512] -> s [B, cin]."""
    w = np.asarray(w, dtype)
    return w @ (np.asarray(mod_weight, dtype) * (1 / math.sqrt(512))).T + np.asarray(mod_bias, dtype)


def style_layers(params):
    """(name, params entry, latent entry) of every modulation layer of ``params`` (synthesis_random_init), in execution order."""
    out = []
    for l, name in enumerate(params["layers"]):
        out.append((f"{name}.conv.modulation", params["layers"][name], l))
        if l % 2 == 0 and l // 2 < len(params["to_rgbs"]):
            j = l // 2
            out.append((f"{'to_rgb1' if j == 0 else f'to_rgbs.{j - 1}'}.conv.modulation", params["to_rgbs"][j], 2 * j + 1))
    return out


def styles(w_layers, params, dtype=np.float64):
    """{S layer name: s [B, cin]} for per-layer latents w_layers [B, n_latent, 512]."""
    return {name: modulation_forward(w_layers[:, e], P["mod_weight"], P["mod_bias"], dtype) for name, P, e in style_layers(params)}


def styled_conv(x, s, L, noise, dtype=np.float64):
    """StyledConv (model.py:232-277, 287-291, fused_act.py:86-90) with the style s [B, ci] given; the shared-weight form of
    ganspace_oracle.styled_conv_shared."""
    import torch
    import torch.nn.functional as F
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype))
    x, style = T(x), T(s)
    W = T(L["weight"]) * (1 / math.sqrt(L["weight"].shape[1] * 9))
    B, ci, H, _ = x.shape
    demod = torch.rsqrt((style * style) @ (W * W).sum([2, 3]).T + 1e-8)
    xs = x * style.view(B, ci, 1, 1)
    if L["upsample"]:
        out = F.conv_transpose2d(xs, W.transpose(0, 1), padding=0, stride=2)
        co = out.shape[1]
        out = F.pad(out, [1, 1, 1, 1]).reshape(B * co, 1, 2 * H + 3, 2 * H + 3)
        out = F.conv2d(out, torch.flip(T(BLUR_K2D), [0, 1]).view(1, 1, 4, 4)).view(B, co, 2 * H, 2 * H)
    else:
        out = F.conv2d(xs, W, padding=1)
    out = out * demod.view(B, -1, 1, 1)
    out = out + torch.tensor(float(L["noise_weight"]), dtype=out.dtype) * T(noise)[None, None]
    return ((2 ** 0.5) * F.leaky_relu(out + T(L["act_bias"]).view(1, -1, 1, 1), negative_slope=0.2)).numpy()


def to_rgb(x, s, R, skip=None, dtype=np.float64):
    """ToRGB (model.py:344-363) with the style s [B, ci] given: 1x1 modulated conv without demodulation, bias, up-sampled skip."""
    import torch
    import torch.nn.functional as F
    T = lambda a: torch.from_numpy(np.ascontiguousarray(a, dtype))
    x, style = T(x), T(s)
    B, ci, H, _ = x.shape
    out = torch.einsum("oc,bchw->bohw", T(R["weight"]) * (1 / math.sqrt(ci)), x * style.view(B, ci, 1, 1))
    out = out + T(R["bias"]).view(1, 3, 1, 1)
    if skip is not None:
        sk = T(skip)
        h = sk.shape[2]
        up = torch.zeros(B, 3, 2 * h, 2 * h, dtype=sk.dtype)
        up[:, :, ::2, ::2] = sk
        up = F.pad(up, [2, 1, 2, 1]).reshape(B * 3, 1, 2 * h + 3, 2 * h + 3)
        out = out + F.conv2d(up, torch.flip(T(BLUR_K2D), [0, 1]).view(1, 1, 4, 4)).view(B, 3, 2 * h, 2 * h)
    return out.numpy()


def render(S, params, noises, dtype=np.float64, keep=()):
    """Generator.forward (model.py:493-571) on the styles S {S layer name: [B, cin]} (from ``styles``, possibly edited) instead of
    latents.  Returns (the last skip image, before the wrapper's 0.5 (x + 1), {name: activation} for the StyledConv names in
    ``keep``)."""
    names = list(params["layers"].keys())
    first = next(iter(S.values()))
    x = np.repeat(np.asarray(params["const"], dtype)[None], first.shape[0], axis=0)
    skip, kept = None, {}
    for l, name in enumerate(names):
        x = styled_conv(x, S[f"{name}.conv.modulation"], params["layers"][name], noises[l], dtype)
        if name in keep:
            kept[name] = x
        if l % 2 == 0 and l // 2 < len(params["to_rgbs"]):
            j = l // 2
            rname = "to_rgb1" if j == 0 else f"to_rgbs.{j - 1}"
            skip = to_rgb(x, S[f"{rname}.conv.modulation"], params["to_rgbs"][j], skip, dtype)
    return skip, kept


def perturb(params):
    """gen_golden_r2.py G11's perturbation on oracle parameters: noise weight 0.1 (i + 1) and activation bias 0.1 sin(c + i) on
    StyledConv i, bias 0.05 [1, -2, 3] (j + 1) on ToRGB j."""
    for i, L in enumerate(params["layers"].values()):
        L["noise_weight"] = np.float32(0.1 * (i + 1))
        L["act_bias"] = (0.1 * np.sin(np.arange(L["act_bias"].shape[0], dtype=np.float32) + i)).astype(np.float32)
    for j, R in enumerate(params["to_rgbs"]):
        R["bias"] = (0.05 * np.array([1.0, -2.0, 3.0]) * (j + 1)).astype(np.float32)
    return params
