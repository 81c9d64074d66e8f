"""StyleGAN2 generator: parameter layout + the CUDA-backed mapping network.

Mirror of the module tree of /root/reference/models/stylegan2/stylegan2-pytorch/model.py:384-469
(``Generator``): same sub-module names (so ``named_modules()`` / layer validation / rosinality
``g_ema`` checkpoints line up) and the same parameter creation order (so ``torch.manual_seed(s)``
followed by ``Generator(size, 512, 8)`` gives the reference's random init bit-for-bit -- the
BASELINE.json configs use random-init weights).

Only the hot path computes: ``Generator.style`` (PixelNorm + 8 x EqualLinear, model.py:400-409) runs
the hand-written mapping kernels through the C ABI, and the StyledConv chain conv1, convs.0 .. convs.k runs
as ONE C-ABI call (csrc/synthesis.cu) driven by ``models.wrappers.StyleGAN2.partial_forward``; the modules
below hold the parameters in the reference's layout and give the hooks their names.  ToRGB / full image
synthesis are not on the path and raise.
"""
from __future__ import annotations

import math
import random

import torch
from torch import nn

from .. import _native

LR_MLP = 0.01


class PixelNorm(nn.Module):
    """model.py:14-19.  Runs the CUDA PixelNorm kernel (only reached when a ``style.k`` child is hooked)."""

    def forward(self, x):
        return _native.mapping_pixelnorm(x)


class EqualLinear(nn.Module):
    """model.py:132-166 parameter holder; forward = one fused linear+bias+lrelu kernel."""

    def __init__(self, in_dim, out_dim, bias=True, bias_init=0.0, lr_mul=1.0, activation=None):
        super().__init__()
        self.weight = nn.Parameter(torch.randn(out_dim, in_dim).div_(lr_mul))
        self.bias = nn.Parameter(torch.zeros(out_dim).fill_(bias_init)) if bias else None
        self.activation = activation
        self.scale = (1 / math.sqrt(in_dim)) * lr_mul
        self.lr_mul = lr_mul
        self.pack_cache = _native.Repacked()

    def forward(self, x=None, _result=None):
        if _result is not None:
            # a ModulatedConv2d.modulation layer: its style rows come from the fused chain's style stage
            # (models.wrappers.StyleGAN2); this call only hands them to the forward hooks, which may return edited rows
            return _result
        if self.activation != "fused_lrelu" or self.weight.shape[0] != self.weight.shape[1]:
            raise NotImplementedError("EqualLinear outside the mapping network is not built yet (SURVEY 8 a5)")
        packed = self.pack_cache.get([self.weight, self.bias], lambda: _native.PackedMapping(
            self.weight.detach()[None], self.bias.detach()[None], self.lr_mul))
        return packed.forward(x, pixelnorm=False)

    def __repr__(self):
        return f"{self.__class__.__name__}({self.weight.shape[1]}, {self.weight.shape[0]})"


class MappingNetwork(nn.Sequential):
    """``Generator.style``: children '0' (PixelNorm) and '1'..'8' (EqualLinear), as in the reference.

    forward() runs the whole chain in one C-ABI call unless a child module carries a forward hook
    (someone retained ``style.k``), in which case the children run one by one so the hooks fire."""

    def __init__(self, style_dim, n_mlp, lr_mlp):
        layers = [PixelNorm()]
        for _ in range(n_mlp):
            layers.append(EqualLinear(style_dim, style_dim, lr_mul=lr_mlp, activation="fused_lrelu"))
        super().__init__(*layers)
        self.style_dim, self.n_mlp, self.lr_mlp = style_dim, n_mlp, lr_mlp
        self.pack_cache = _native.Repacked()

    def packed(self) -> "_native.PackedMapping":
        lins = list(self)[1:]
        return self.pack_cache.get([t for l in lins for t in (l.weight, l.bias)], lambda: _native.PackedMapping(
            torch.stack([l.weight.detach() for l in lins]), torch.stack([l.bias.detach() for l in lins]), self.lr_mlp))

    def forward(self, z):
        if any(len(m._forward_hooks) or len(m._forward_pre_hooks) for m in self):
            return super().forward(z)
        return self.packed().forward(z, pixelnorm=True)


def _make_kernel(k):
    k = torch.tensor(k, dtype=torch.float32)
    if k.ndim == 1:
        k = k[None, :] * k[:, None]
    return k / k.sum()


class _NotBuilt(nn.Module):
    def forward(self, *a, **k):
        raise NotImplementedError(
            f"{self.__class__.__name__} has no stand-alone forward: the StyledConv chain runs as one fused C-ABI call "
            "(StyleGAN2.partial_forward(x, 'conv1' | 'convs.k')); ToRGB / image synthesis are not on the GPU hot path. "
            "There is no PyTorch/CPU fallback.")


class Blur(_NotBuilt):
    def __init__(self, kernel, pad, upsample_factor=1):
        super().__init__()
        kernel = _make_kernel(kernel)
        if upsample_factor > 1:
            kernel = kernel * (upsample_factor ** 2)
        self.register_buffer("kernel", kernel)
        self.pad = pad


class Upsample(_NotBuilt):
    def __init__(self, kernel, factor=2):
        super().__init__()
        self.factor = factor
        self.register_buffer("kernel", _make_kernel(kernel) * (factor ** 2))
        p = self.kernel.shape[0] - factor
        self.pad = ((p + 1) // 2 + factor - 1, p // 2)


class ModulatedConv2d(_NotBuilt):
    def __init__(self, in_channel, out_channel, kernel_size, style_dim, demodulate=True, upsample=False,
                 blur_kernel=(1, 3, 3, 1)):
        super().__init__()
        self.eps = 1e-8
        self.kernel_size, self.in_channel, self.out_channel = kernel_size, in_channel, out_channel
        self.upsample, self.downsample = upsample, False
        if upsample:
            factor = 2
            p = (len(blur_kernel) - factor) - (kernel_size - 1)
            self.blur = Blur(blur_kernel, pad=((p + 1) // 2 + factor - 1, p // 2 + 1), upsample_factor=factor)
        self.scale = 1 / math.sqrt(in_channel * kernel_size ** 2)
        self.padding = kernel_size // 2
        self.weight = nn.Parameter(torch.randn(1, out_channel, in_channel, kernel_size, kernel_size))
        self.modulation = EqualLinear(style_dim, in_channel, bias_init=1)
        self.demodulate = demodulate


class NoiseInjection(_NotBuilt):
    def __init__(self):
        super().__init__()
        self.weight = nn.Parameter(torch.zeros(1))


class ConstantInput(nn.Module):
    def __init__(self, channel, size=4):
        super().__init__()
        self.input = nn.Parameter(torch.randn(1, channel, size, size))

    def forward(self, input):
        return self.input.repeat(input.shape[0], 1, 1, 1)      # model.py:300-304


class FusedLeakyReLU(_NotBuilt):
    def __init__(self, channel, negative_slope=0.2, scale=2 ** 0.5):
        super().__init__()
        self.bias = nn.Parameter(torch.zeros(channel))
        self.negative_slope, self.scale = negative_slope, scale


class StyledConv(nn.Module):
    """model.py:307-341.  The arithmetic of the whole conv1 .. convs.k chain is one fused C-ABI call
    (``_native.PackedSynthesis``); ``forward(_result=act)`` only hands that result to the forward hooks."""

    def __init__(self, in_channel, out_channel, kernel_size, style_dim, upsample=False, blur_kernel=(1, 3, 3, 1),
                 demodulate=True):
        super().__init__()
        self.conv = ModulatedConv2d(in_channel, out_channel, kernel_size, style_dim, upsample=upsample,
                                    blur_kernel=blur_kernel, demodulate=demodulate)
        self.noise = NoiseInjection()
        self.activate = FusedLeakyReLU(out_channel)

    def forward(self, input=None, style=None, noise=None, _result=None):
        if _result is None:
            raise NotImplementedError(
                "StyledConv runs as part of the fused synthesis chain (StyleGAN2.partial_forward(x, 'convs.k')); a "
                "stand-alone per-layer call is not built and there is no PyTorch fallback")
        return _result

    def describe(self, noise_map, res_in):
        """Layer descriptor for _native.PackedSynthesis (device tensors in PyTorch layout)."""
        c = self.conv
        return dict(conv_weight=c.weight[0], mod_weight=c.modulation.weight, mod_bias=c.modulation.bias,
                    act_bias=self.activate.bias, noise=noise_map.reshape(-1), noise_weight=self.noise.weight,
                    upsample=c.upsample, res_in=res_in)


class ToRGB(nn.Module):
    """model.py:344-363.  The arithmetic (1x1 modulated conv without demodulation, bias, up-sampled skip) is fused into the
    epilogue of the StyledConv it follows (gsb_synthesis_forward); ``forward(_result=skip)`` hands the result to the hooks."""

    def __init__(self, in_channel, style_dim, upsample=True, blur_kernel=(1, 3, 3, 1)):
        super().__init__()
        if upsample:
            self.upsample = Upsample(blur_kernel)
        self.conv = ModulatedConv2d(in_channel, 3, 1, style_dim, demodulate=False)
        self.bias = nn.Parameter(torch.zeros(1, 3, 1, 1))

    def forward(self, input=None, style=None, skip=None, _result=None):
        if _result is None:
            raise NotImplementedError("ToRGB runs inside the fused synthesis chain (Generator.forward / partial_forward)")
        return _result

    def describe(self):
        """ToRGB descriptor for _native.PackedSynthesis, which copies the parameters at pack time."""
        c = self.conv
        return dict(conv_weight=c.weight[0, :, :, 0, 0], mod_weight=c.modulation.weight, mod_bias=c.modulation.bias,
                    bias=self.bias.reshape(3))


class NamedTensor(nn.Module):
    def forward(self, x):
        return x


class StridedStyle(nn.ModuleList):
    """model.py:374-382: gives each per-layer style a hookable name."""

    def __init__(self, n_latents):
        super().__init__([NamedTensor() for _ in range(n_latents)])
        self.n_latents = n_latents

    def forward(self, x):
        return torch.stack([self[i](x[:, i, :]) for i in range(self.n_latents)], dim=1)


class Generator(nn.Module):
    def __init__(self, size, style_dim, n_mlp, channel_multiplier=2, blur_kernel=(1, 3, 3, 1), lr_mlp=LR_MLP):
        super().__init__()
        self.size, self.style_dim = size, style_dim
        self.style = MappingNetwork(style_dim, n_mlp, lr_mlp)
        self.channels = {4: 512, 8: 512, 16: 512, 32: 512, 64: 256 * channel_multiplier,
                         128: 128 * channel_multiplier, 256: 64 * channel_multiplier,
                         512: 32 * channel_multiplier, 1024: 16 * channel_multiplier}
        self.input = ConstantInput(self.channels[4])
        self.conv1 = StyledConv(self.channels[4], self.channels[4], 3, style_dim, blur_kernel=blur_kernel)
        self.to_rgb1 = ToRGB(self.channels[4], style_dim, upsample=False)
        self.log_size = int(math.log(size, 2))
        self.num_layers = (self.log_size - 2) * 2 + 1
        self.convs, self.upsamples, self.to_rgbs = nn.ModuleList(), nn.ModuleList(), nn.ModuleList()
        self.noises = nn.Module()
        in_channel = self.channels[4]
        for layer_idx in range(self.num_layers):
            res = (layer_idx + 5) // 2
            self.noises.register_buffer(f"noise_{layer_idx}", torch.randn(1, 1, 2 ** res, 2 ** res))
        for i in range(3, self.log_size + 1):
            out_channel = self.channels[2 ** i]
            self.convs.append(StyledConv(in_channel, out_channel, 3, style_dim, upsample=True, blur_kernel=blur_kernel))
            self.convs.append(StyledConv(out_channel, out_channel, 3, style_dim, blur_kernel=blur_kernel))
            self.to_rgbs.append(ToRGB(out_channel, style_dim))
            in_channel = out_channel
        self.n_latent = self.log_size * 2 - 2
        self.strided_style = StridedStyle(self.n_latent)

    def get_latent(self, z):
        return self.style(z)

    def chain_layers(self):
        """(name, module) of the StyledConv layers conv1, convs.0, ... and of the ToRGB layers to_rgb1, to_rgbs.0, ..."""
        return ([("conv1", self.conv1)] + [(f"convs.{k}", m) for k, m in enumerate(self.convs)],
                [("to_rgb1", self.to_rgb1)] + [(f"to_rgbs.{j}", m) for j, m in enumerate(self.to_rgbs)])

    def style_layers(self):
        """The style space: (name, key, latent entry, width) of every modulation layer, in execution order (conv1, to_rgb1, convs.0,
        convs.1, to_rgbs.0, ...; ToRGB j follows StyledConv 2j).  The key is the layer's position in this table, which keys its rows
        (``PackedSynthesis.styles``); the latent entry is the [N, n_latent, 512] latent's column the layer reads
        (model.py:546-561); width = the layer's input channels."""
        convs, rgbs = self.chain_layers()
        out = []
        for l, (name, m) in enumerate(convs):
            out.append((f"{name}.conv.modulation", len(out), l, m.conv.in_channel))
            if l % 2 == 0:
                j = l // 2
                out.append((f"{rgbs[j][0]}.conv.modulation", len(out), 2 * j + 1, rgbs[j][1].conv.in_channel))
        return out

    def unhookable_layers(self):
        """Sub-modules of the StyledConv and ToRGB layers that run inside the fused chain and have no output of their own to
        hook: every one except the '.conv.modulation' style layers."""
        convs, rgbs = self.chain_layers()
        return [f"{name}.{c}" for name, m in convs + rgbs for c, _ in m.named_modules() if c and c != "conv.modulation"]

    def latent(self, styles, inject_index=None, truncation=1, truncation_latent=None, input_is_w=False):
        """The [N, n_latent, style_dim] per-layer latent of a forward call (model.py:511-552)."""
        if not input_is_w:
            styles = [self.style(s) for s in styles]
        if truncation < 1:
            styles = [truncation_latent + truncation * (s - truncation_latent) for s in styles]
        return self.latents_per_layer(styles, inject_index)

    def latents_per_layer(self, styles, inject_index=None):
        """model.py:527-552: the [N, n_latent, style_dim] latent of a forward call from one, two or n_latent styles."""
        if len(styles) == 1:
            if styles[0].ndim < 3:
                return styles[0].unsqueeze(1).repeat(1, self.n_latent, 1)
            return styles[0]
        if len(styles) == 2:
            if inject_index is None:
                inject_index = random.randint(1, self.n_latent - 1)
            latent = styles[0].unsqueeze(1).repeat(1, inject_index, 1)
            latent2 = styles[1].unsqueeze(1).repeat(1, self.n_latent - inject_index, 1)
            return self.strided_style(torch.cat([latent, latent2], 1))
        assert len(styles) == self.n_latent, f"Expected {self.n_latent} latents, got {len(styles)}"
        return self.strided_style(torch.stack(styles, dim=1))

    def forward(self, styles, return_latents=False, inject_index=None, truncation=1, truncation_latent=None, input_is_w=False,
                noise=None, randomize_noise=True, _synthesis=None):
        """model.py:493-571 on the fused chain (``_synthesis``: the wrapper's PackedSynthesis over all StyledConv layers, which
        holds the fixed noise maps -- the reference wrapper always passes them, wrappers.py:188-192)."""
        if _synthesis is None:
            raise NotImplementedError("Generator.forward needs the wrapper's packed synthesis chain (StyleGAN2.forward); "
                                      "randomised noise is not built")
        latent = self.latent(styles, inject_index, truncation, truncation_latent, input_is_w)     # [N, n_latent, S]
        w_layers = latent.permute(1, 0, 2).contiguous()
        _, img = _synthesis.forward(w_layers, len(self.convs) + 1, want_act=False, n_rgb=len(self.to_rgbs) + 1)
        image = img.permute(0, 3, 1, 2)                                            # NCHW view of the NHWC skip image
        return (image, latent) if return_latents else (image, None)
