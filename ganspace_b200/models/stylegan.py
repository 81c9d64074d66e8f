"""StyleGAN (v1) generator: the module tree of models/stylegan/model.py:212-376 (``StyleGAN_G`` with ``g_mapping`` and
``g_synthesis``) with the same names, parameter shapes and creation order, so that its ``.pt`` state dicts load by key,
``named_modules()`` hooks attach, and ``torch.manual_seed(s); StyleGAN_G(res)`` gives the reference's initial weights bit for bit.

The arithmetic is not here.  ``g_mapping`` runs the packed mapping kernels (csrc/mapping*.cu): v1's layer
``lrelu(x (W w_mul)^T + b 0.01)`` with ``w_mul = sqrt2 0.01 / sqrt512`` equals ``sqrt2 lrelu(x (W 0.01 / sqrt512)^T + (b / sqrt2) 0.01)``
(leaky-ReLU is positively homogeneous), which is the StyleGAN2 layer the kernels compute, with the bias divided by sqrt2 on the host.
The synthesis network runs in ``_native.PackedStyleGAN`` (csrc/stylegan.cu); a block's ``forward(_result=act)`` and a StyleMod
``lin``'s ``forward(_result=rows)`` only hand the chain's result to the forward hooks.  Every other module has no stand-alone forward and raises.
"""
from __future__ import annotations

import math
from collections import OrderedDict

import torch
import torch.nn as nn

from .. import _native

DLATENT = 512


class _NotBuilt(nn.Module):
    def forward(self, *a, **k):
        raise NotImplementedError(
            f"{self.__class__.__name__} has no stand-alone forward: StyleGAN runs g_mapping and the synthesis blocks as fused "
            "kernels (StyleGAN.forward / partial_forward to 'g_mapping' or 'g_synthesis.blocks.RxR'); there is no PyTorch fallback")


class MyLinear(_NotBuilt):
    """model.py:26-48, parameters only (equalized learning rate: ``weight * w_mul``, ``bias * b_mul``).  A StyleMod's ``lin`` is a
    style layer: StyleGAN.forward / partial_forward compute its rows [n, 2C] on the device and ``forward(_result=rows)`` hands them
    to the forward hooks, returning what the hooks return (an edit replaces the style)."""

    def __init__(self, input_size, output_size, gain=2 ** 0.5, use_wscale=True, lrmul=1.0):
        super().__init__()
        he_std = gain * input_size ** (-0.5)
        init_std = 1.0 / lrmul
        self.w_mul = he_std * lrmul
        self.weight = nn.Parameter(torch.randn(output_size, input_size) * init_std)
        self.bias = nn.Parameter(torch.zeros(output_size))
        self.b_mul = lrmul

    def forward(self, *a, _result=None, **k):
        if _result is None:
            return super().forward(*a, **k)
        return _result


class Upscale2d(_NotBuilt):
    pass


class BlurLayer(_NotBuilt):
    """model.py:144-166: the [1,2,1] x [1,2,1] / 16 kernel, a buffer of the state dict."""

    def __init__(self):
        super().__init__()
        k = torch.tensor([1, 2, 1], dtype=torch.float32)
        k = k[:, None] * k[None, :]
        self.register_buffer("kernel", (k / k.sum())[None, None])


class MyConv2d(_NotBuilt):
    """model.py:50-105, parameters only."""

    def __init__(self, input_channels, output_channels, kernel_size, gain=2 ** 0.5, intermediate=None, upscale=False):
        super().__init__()
        self.upscale = Upscale2d() if upscale else None
        self.w_mul = gain * (input_channels * kernel_size ** 2) ** (-0.5)
        self.kernel_size = kernel_size
        self.weight = nn.Parameter(torch.randn(output_channels, input_channels, kernel_size, kernel_size))
        self.bias = nn.Parameter(torch.zeros(output_channels))
        self.intermediate = intermediate


class NoiseLayer(_NotBuilt):
    """model.py:107-119.  ``noise`` [1, 1, H, W] (set by ``StyleGAN.set_noise_seed`` or by hand) is the map every sample gets."""

    def __init__(self, channels):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(channels))
        self.noise = None


class PixelNormLayer(_NotBuilt):
    pass


class InstanceNorm(_NotBuilt):
    """nn.InstanceNorm2d(channels): no parameters, eps 1e-5."""


class StyleMod(_NotBuilt):
    def __init__(self, latent_size, channels):
        super().__init__()
        self.lin = MyLinear(latent_size, channels * 2, gain=1.0)


class LayerEpilogue(_NotBuilt):
    """model.py:228-253: top_epi (noise, activation, instance_norm) and style_mod."""

    def __init__(self, channels, activation):
        super().__init__()
        self.top_epi = nn.Sequential(OrderedDict([("noise", NoiseLayer(channels)), ("activation", activation),
                                                  ("instance_norm", InstanceNorm())]))
        self.style_mod = StyleMod(DLATENT, channels)


class _Block(nn.Module):
    def forward(self, *a, _result=None, **k):
        if _result is None:
            raise NotImplementedError("StyleGAN synthesis blocks run as part of the fused chain (StyleGAN.forward / "
                                      "partial_forward); a stand-alone per-block call is not built and there is no PyTorch fallback")
        return _result


class InputBlock(_Block):
    def __init__(self, nf, activation):
        super().__init__()
        self.const = nn.Parameter(torch.ones(1, nf, 4, 4))
        self.bias = nn.Parameter(torch.ones(nf))
        self.epi1 = LayerEpilogue(nf, activation)
        self.conv = MyConv2d(nf, nf, 3)
        self.epi2 = LayerEpilogue(nf, activation)


class GSynthesisBlock(_Block):
    def __init__(self, in_channels, out_channels, activation):
        super().__init__()
        blur = BlurLayer()
        self.conv0_up = MyConv2d(in_channels, out_channels, 3, intermediate=blur, upscale=True)
        self.epi1 = LayerEpilogue(out_channels, activation)
        self.conv1 = MyConv2d(out_channels, out_channels, 3)
        self.epi2 = LayerEpilogue(out_channels, activation)


def nf(stage):
    """Channel count of stage ``log2(R) - 1`` (fmap_base 8192, fmap_decay 1, fmap_max 512)."""
    return min(int(8192 / (2.0 ** stage)), 512)


class G_mapping(nn.Sequential):
    """PixelNorm + 8 x (MyLinear(512, 512, lrmul 0.01), LeakyReLU 0.2).  As in the reference one LeakyReLU instance is registered
    under all eight ``denseK_act`` names (so ``named_modules()`` lists only ``dense0_act``).  forward = one packed-kernel call."""

    def __init__(self):
        act = nn.LeakyReLU(negative_slope=0.2)
        layers = [("pixel_norm", PixelNormLayer())]
        for i in range(8):
            layers += [(f"dense{i}", MyLinear(DLATENT, DLATENT, gain=math.sqrt(2), lrmul=0.01)), (f"dense{i}_act", act)]
        super().__init__(OrderedDict(layers))
        self.pack_cache = _native.Repacked()

    def packed(self) -> "_native.PackedMapping":
        lins = [getattr(self, f"dense{i}") for i in range(8)]
        return self.pack_cache.get([t for l in lins for t in (l.weight, l.bias)], lambda: _native.PackedMapping(
            torch.stack([l.weight.detach() for l in lins]), torch.stack([l.bias.detach() for l in lins]) / math.sqrt(2), 0.01))

    def forward(self, z):
        return self.packed().forward(z, pixelnorm=True)


class G_synthesis(nn.Module):
    """model.py:277-364 for the reference's defaults.  ``torgb`` is registered before ``blocks``, as there."""

    def __init__(self, resolution=1024):
        super().__init__()
        log2 = int(math.log2(resolution))
        assert resolution == 2 ** log2 and resolution >= 4
        act = nn.LeakyReLU(negative_slope=0.2)
        blocks, last = [], None
        for res in range(2, log2 + 1):
            channels = nf(res - 1)
            name = f"{2 ** res}x{2 ** res}"
            blocks.append((name, InputBlock(channels, act) if res == 2 else GSynthesisBlock(last, channels, act)))
            last = channels
        self.torgb = MyConv2d(last, 3, 1, gain=1)
        self.blocks = nn.ModuleDict(OrderedDict(blocks))
        self.resolution = resolution
        self.pack_cache = _native.Repacked()

    def forward(self, *a, **k):
        raise NotImplementedError("g_synthesis runs as the fused chain: call StyleGAN.forward / partial_forward")

    def layer_modules(self):
        """(conv, epilogue, upsample, res_out) of every layer in execution order; conv is None for the constant input."""
        out = []
        for i, (name, blk) in enumerate(self.blocks.items()):
            r = int(name.split("x")[0])
            if i == 0:
                out += [(None, blk.epi1, False, r), (blk.conv, blk.epi2, False, r)]
            else:
                out += [(blk.conv0_up, blk.epi1, True, r), (blk.conv1, blk.epi2, False, r)]
        return out

    def packed(self) -> "_native.PackedStyleGAN":
        """The chain packed for the kernels; re-packed when a parameter or a noise map changes."""
        layers = self.layer_modules()
        noise = [epi.top_epi.noise.noise for _, epi, _, _ in layers]
        if any(n is None for n in noise):
            raise RuntimeError("StyleGAN: a NoiseLayer has no noise map (StyleGAN.set_noise_seed sets them)")

        def build():
            inp = self.blocks["4x4"]
            descs = []
            for (conv, epi, up, r), nz in zip(layers, noise):
                descs.append(dict(conv_weight=None if conv is None else conv.weight, bias=inp.bias if conv is None else conv.bias,
                                  noise=nz, noise_weight=epi.top_epi.noise.weight, style_weight=epi.style_mod.lin.weight,
                                  style_bias=epi.style_mod.lin.bias, upsample=up, res_out=r))
            return _native.PackedStyleGAN(descs, inp.const, self.torgb.weight, self.torgb.bias, DLATENT)
        return self.pack_cache.get(list(self.parameters()) + noise, build)


class StyleGAN_G(nn.Sequential):
    def __init__(self, resolution):
        self.resolution = resolution
        super().__init__(OrderedDict([("g_mapping", G_mapping()), ("g_synthesis", G_synthesis(resolution=resolution))]))

    def forward(self, *a, **k):
        raise NotImplementedError("call StyleGAN.forward / partial_forward (models/wrappers.py): they drive the fused kernels")

    def block_names(self):
        return [f"g_synthesis.blocks.{n}" for n in self.g_synthesis.blocks]

    def style_layers(self):
        """(name, chain layer, latent index, width 2C) of every style layer ``g_synthesis.blocks.RxR.epi{1,2}.style_mod.lin``, in
        execution order: chain layer l is the l-th epilogue and reads latent l of an 18-latent input.  The chain layer is also the
        layer's position in this table, the key of its rows (``PackedStyleGAN.styles``)."""
        out = []
        for l, (_, epi, _, _) in enumerate(self.g_synthesis.layer_modules()):
            blk = self.block_names()[l // 2]
            out.append((f"{blk}.epi{l % 2 + 1}.style_mod.lin", l, l, epi.style_mod.lin.weight.shape[0]))
        return out

    def hookable_layers(self):
        return ["g_mapping"] + self.block_names() + [t[0] for t in self.style_layers()]

    def unhookable_layers(self):
        """Sub-modules that run inside the fused kernels and have no output of their own to hook: every one but
        ``hookable_layers()``."""
        hookable = set(self.hookable_layers())
        return [n for n, _ in self.named_modules() if n and n not in hookable]


def synthesis_fill(net, seed):
    """Seeded values for what the reference's init leaves degenerate (zero biases and noise weights, an all-ones constant whose
    first InstanceNorm is exactly 0): under ``torch.manual_seed(seed)``, in module order, every InputBlock ``const`` and ``bias``,
    NoiseLayer ``weight``, MyConv2d ``bias`` of the synthesis network (torgb's included) and StyleMod ``lin.bias`` is drawn from
    N(0, 1) * 0.5.  oracle/gen_golden_stylegan.py applies the same fill to the reference's generator."""
    g = net.g_synthesis if hasattr(net, "g_synthesis") else net._modules["g_synthesis"]
    torch.manual_seed(int(seed))
    with torch.no_grad():
        for name, p in g.named_parameters():
            if name.endswith(("const", ".bias", "noise.weight")) or name == "bias":
                p.copy_(torch.randn(p.shape) * 0.5)
    return net


def random_init(seed, resolution=1024, fill=None):
    """``torch.manual_seed(seed); StyleGAN_G(resolution)``: the reference's initial weights; with ``fill``, then
    ``synthesis_fill(net, fill)``."""
    torch.manual_seed(int(seed))
    net = StyleGAN_G(resolution)
    if fill is not None:
        synthesis_fill(net, fill)
    return net
