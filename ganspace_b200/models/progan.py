"""ProGAN generator: the module tree of netdissect/proggan.py:34-171 (names ``layer1 .. layerK``, ``output_RxR``; parameters
``<block>.conv.weight`` and ``<block>.wscale.b``) so that its checkpoints load and ``named_modules()`` hooks attach.

The arithmetic is not here: the whole chain runs in ``_native.PackedProGAN`` (csrc/progan.cu).  A block's
``forward(_result=act)`` only hands the chain's result to the forward hooks, the convention of ``stylegan2.StyledConv``.
The parameter-free children of the reference's blocks (``norm``, ``up``, ``relu``) have nothing to hook that the block itself
does not give and are not mirrored.
"""
from __future__ import annotations

import itertools
import math
from collections import OrderedDict

import torch
import torch.nn as nn

from .. import _native

RESOLUTION_SIZES = {
    8: [512, 512, 512], 16: [512, 512, 512, 512], 32: [512, 512, 512, 512, 256], 64: [512, 512, 512, 512, 256, 128],
    128: [512, 512, 512, 512, 256, 128, 64], 256: [512, 512, 512, 512, 256, 128, 64, 32],
    1024: [512, 512, 512, 512, 512, 256, 128, 64, 32, 16],
}


class WScale(nn.Module):
    """proggan.py:110-121: ``x * gain / sqrt(fan_in) + b``; ``b`` is drawn from N(0, 1) at construction, as there."""

    def __init__(self, size, fan_in, gain):
        super().__init__()
        self.scale = gain / math.sqrt(fan_in)
        self.b = nn.Parameter(torch.randn(size))


class Block(nn.Module):
    """NormConvBlock / NormUpscaleConvBlock / OutputConvBlock (proggan.py:123-171), parameters only."""

    def __init__(self, in_channels, out_channels, kernel_size, padding, upsample=False, gain=None):
        super().__init__()
        self.upsample = upsample
        self.conv = nn.Conv2d(in_channels, out_channels, kernel_size, 1, padding, bias=False)
        self.wscale = WScale(out_channels, in_channels, math.sqrt(2) / kernel_size if gain is None else gain)

    def forward(self, x=None, _result=None):
        if _result is None:
            raise NotImplementedError("ProGAN blocks run as part of the fused chain (ProGAN.forward / partial_forward); a "
                                      "stand-alone per-block call is not built and there is no PyTorch fallback")
        return _result

    def describe(self):
        return dict(conv_weight=self.conv.weight, bias=self.wscale.b, upsample=self.upsample)


class ProgressiveGenerator(nn.Sequential):
    """proggan.py:34-96.  ``sizes`` = [z dim, 4x4 depth, 8x8 depth, ...]; modules are created in the reference's order, so one
    ``torch.manual_seed`` before construction gives the reference's initial parameters."""

    def __init__(self, resolution=None, sizes=None):
        assert (resolution is None) != (sizes is None)
        sizes = RESOLUTION_SIZES[resolution] if sizes is None else list(sizes)
        seq = [Block(sizes[0], sizes[1], 4, 3), Block(sizes[1], sizes[1], 3, 1)]
        for si, so in zip(sizes[1:-1], sizes[2:]):
            seq += [Block(si, so, 3, 1, upsample=True), Block(so, so, 3, 1)]
        dim = 4 * 2 ** (len(seq) // 2 - 1)
        named = [(f"layer{i + 1}", m) for i, m in enumerate(seq)]
        named.append((f"output_{dim}x{dim}", Block(sizes[-1], 3, 1, 0, gain=1)))
        super().__init__(OrderedDict(named))
        self.resolution = dim
        self.pack_cache = _native.Repacked()

    def block_names(self):
        return list(self._modules)

    def packed(self) -> "_native.PackedProGAN":
        """The chain packed for the kernels; re-packed when a parameter changes."""
        mods = list(self._modules.values())
        return self.pack_cache.get([p for m in mods for p in (m.conv.weight, m.wscale.b)], lambda: _native.PackedProGAN(
            [m.describe() for m in mods[:-1]], mods[-1].conv.weight, mods[-1].wscale.b))

    def forward(self, x):
        raise NotImplementedError("call ProGAN.forward / partial_forward (models/wrappers.py): they drive the fused chain")


def sizes_from_state_dict(params):
    """Channel depths from the conv shapes (proggan.py:197-214)."""
    sizes = []
    for i in itertools.count():
        weight = params.get(f"layer{i + 1}.conv.weight")
        if weight is None:
            break
        if i == 0:
            sizes.append(weight.shape[1])
        if i % 2 == 0:
            sizes.append(weight.shape[0])
    return sizes


def state_dict_from_old_names(params):
    """``features.<i>`` / ``output`` keys of the older checkpoints -> ``layer<i+1>`` / ``output_RxR`` (proggan.py:271-298)."""
    result, i = {}, 0
    while f"features.{i}.conv.weight" in params:
        result[f"layer{i + 1}.conv.weight"] = params[f"features.{i}.conv.weight"]
        result[f"layer{i + 1}.wscale.b"] = params[f"features.{i}.wscale.b"]
        i += 1
    res = 4 * 2 ** ((i - 1) // 2)
    result[f"output_{res}x{res}.conv.weight"] = params["output.conv.weight"]
    result[f"output_{res}x{res}.wscale.b"] = params["output.wscale.b"]
    return result


def from_state_dict(state_dict):
    """proggan.py:15-28 after ``torch.load``: accepts a bare state dict or one under 'state_dict', in either key format."""
    if "state_dict" in state_dict:
        state_dict = state_dict["state_dict"]
    if "features.0.conv.weight" in state_dict:
        state_dict = state_dict_from_old_names(state_dict)
    model = ProgressiveGenerator(sizes=sizes_from_state_dict(state_dict))
    model.load_state_dict(state_dict)
    return model


def random_init(seed, resolution=256):
    """Random weights in the parametrisation WScaleLayer assumes: under ``torch.manual_seed(seed)`` the generator is built in the
    reference's creation order (Conv2d default init, then ``wscale.b ~ N(0, 1)``, block by block), then every ``conv.weight`` is
    drawn from N(0, 1) in module order.  (PyTorch's default Conv2d init, std ~ 1/sqrt(3 fan_in), under the additional
    gain / sqrt(cin) of WScaleLayer would leave every activation dominated by its bias.)"""
    torch.manual_seed(int(seed))
    model = ProgressiveGenerator(resolution=resolution)
    with torch.no_grad():
        for m in model._modules.values():
            m.conv.weight.copy_(torch.randn(m.conv.weight.shape))
    return model
