"""BigGAN wrapper of the hot path: latent sampler + ``generator.gen_z`` (BASELINE.json config 4).

Mirror of /root/reference/models/wrappers.py:525-648 (``BigGAN(BaseModel)``) restricted to what
``decomposition.compute`` reaches for ``layer='generator.gen_z'`` (``partial_forward`` stops after gen_z
with n_layers = 0, wrappers.py:611-648):

    z      = truncated_noise_sample(seed)                  biggan utils.py:21-33   -> gsb_legacy_truncnorm_f32
    embed  = embeddings(one_hot(class))                    biggan model.py:291     (constant per class)
    act    = gen_z(cat(z, embed))                          biggan model.py:211-212,232
           = spectral_norm(Linear(256, 4*4*16*ch)): weight_orig / sigma, sigma = u^T W v with the stored u, v
             (eval mode: no power iteration)               -> folded once into W_eff, gsb_linear_forward

Low-rank activation path.  gen_z is affine in z:  act = z A^T + const,  A = W_eff[:, :128]  (d = 32768, r = 128).
With the thin QR  A = Q R  every centred activation is  (z - zbar) R^T Q^T, so sklearn's IncrementalPCA on the
32768-dim activations equals IncrementalPCA on y = z R^T (128-dim) followed by  components = components_y Q^T
(the SVD of the stacked matrix is equivariant under the isometry Q).  ``affine_layer()`` exposes that
factorisation; the decomposition driver then never materialises the [N, 32768] activations (131 GB at N=1e6)
and reuses the small-d engine.  ``partial_forward`` still produces the full activation for API users.

Synthesis (``forward``, ``partial_forward`` to ``generator.layers.k``): the reference's module tree (GenBlock, SelfAttn,
BigGANBatchNorm, generator.bn, conv_to_rgb; same names, shapes and creation order) holds the parameters, and ``_Chain`` runs
them on the kernels of csrc/biggan.cu (DESIGN.md section 5i).  The conditional-BatchNorm row layers generator.layers.k.bn_j.scale /
.offset are affine in z as well (``affine_layer``, ``style_layers``); decomposing any other generator layer raises.
"""
from __future__ import annotations

import math
import os
import re

import numpy as np
import torch
from torch import nn

from .. import _native
from .wrappers import _checkpoint, _DeviceGenerator, _global_seed

# ImageNet class ids for the names GANSpace's configs use (the reference resolves names through
# nltk/WordNet, biggan utils.py:174-216, which is not available offline)
_CLASS_IDS = {"husky": 248, "siberian_husky": 250, "golden_retriever": 207, "lion": 291, "tiger": 292,
              "mushroom": 947, "barn": 425, "church": 497, "castle": 483, "volcano": 980, "lakeside": 975}

# (up-sample, in, out) per GenBlock, in units of channel_width.  128: the reference's BigGANConfig defaults; 512: its
# biggan-deep-512 configuration; 256: the same pattern with six up-samplings (the published config is not available offline)
_LAYERS = {
    128: [(False, 16, 16), (True, 16, 16), (False, 16, 16), (True, 16, 8), (False, 8, 8), (True, 8, 4), (False, 4, 4),
          (True, 4, 2), (False, 2, 2), (True, 2, 1)],
    256: [(False, 16, 16), (True, 16, 16), (False, 16, 16), (True, 16, 8), (False, 8, 8), (True, 8, 8), (False, 8, 8),
          (True, 8, 4), (False, 4, 4), (True, 4, 2), (False, 2, 2), (True, 2, 1)],
    512: [(False, 16, 16), (True, 16, 16), (False, 16, 16), (True, 16, 8), (False, 8, 8), (True, 8, 8), (False, 8, 8),
          (True, 8, 4), (False, 4, 4), (True, 4, 2), (False, 2, 2), (True, 2, 1), (False, 1, 1), (True, 1, 1)],
}
_CHANNEL_WIDTH = 128


_ROW_LAYER = re.compile(r"^generator\.layers\.([0-9]+)\.bn_([0-3])\.(scale|offset)$")


def _row_layer(name):
    """(k, j, 'scale' | 'offset') of a row-layer name generator.layers.k.bn_j.scale / .offset, else None."""
    m = _ROW_LAYER.match(name)
    return None if m is None else (int(m[1]), int(m[2]), m[3])


class _Config:
    def __init__(self, resolution):
        self.output_dim = resolution
        self.z_dim = 128
        self.class_embed_dim = 128
        self.channel_width = _CHANNEL_WIDTH
        self.num_classes = 1000
        self.layers = list(_LAYERS[resolution])
        self.attention_layer_position = 8
        self.eps = 1e-4
        self.n_stats = 51


class _SNParams(nn.Module):
    """The tensors of a ``torch.nn.utils.spectral_norm`` module (``bias``, ``weight_orig``, ``weight_u``, ``weight_v``), copied from
    one built with torch so that its random init (layer init, then the normal draws of u and v) is the reference's.  In eval mode
    the effective weight is W_orig / sigma with sigma = u^T W_orig.view(out, -1) v: no power iteration."""

    def __init__(self, sn):
        super().__init__()
        if sn.bias is not None:
            self.bias = nn.Parameter(sn.bias.detach().clone())
        else:
            self.register_parameter("bias", None)
        self.weight_orig = nn.Parameter(sn.weight_orig.detach().clone())
        self.register_buffer("weight_u", sn.weight_u.detach().clone())
        self.register_buffer("weight_v", sn.weight_v.detach().clone())
        self.weight_cache = _native.Repacked()

    def effective_weight(self) -> torch.Tensor:
        def build():
            w = self.weight_orig.detach()
            sigma = torch.dot(self.weight_u, torch.mv(w.reshape(w.shape[0], -1), self.weight_v))      # torch spectral_norm, eval mode
            return (w / sigma).contiguous()
        return self.weight_cache.get([self.weight_orig, self.weight_u, self.weight_v], build)


class SNLinear(_SNParams):
    """``spectral_norm(nn.Linear)`` in eval mode: y = x (W_orig / sigma)^T + b."""

    def forward(self, x=None, _result=None):
        # the conditional-BatchNorm linears (generator.layers.k.bn_j.scale / .offset) run in the BigGAN chain, which hands their
        # rows to the hooks with forward(_result=rows), the convention of _FusedModule
        if _result is not None:
            return _result
        # latents are truncated normals in [-2, 2] * truncation and the class embedding is a fixed vector: inside fp16's range,
        # so batches of >= 128 rows run on the tensor cores (fp32-grade hi/lo split)
        return _native.linear(x, self.effective_weight(), self.bias.detach(), bounded=bool(x.abs().max() < 6e4) if x.shape[0] >= 128 else False)


class SNConv2d(_SNParams):
    """``spectral_norm(nn.Conv2d)`` in eval mode, parameters only: the convolution runs in csrc/biggan.cu."""

    def __init__(self, in_channels, out_channels, kernel_size, padding=0, bias=True, eps=1e-12):
        super().__init__(nn.utils.spectral_norm(nn.Conv2d(in_channels, out_channels, kernel_size, padding=padding, bias=bias), eps=eps))

    def gemm_weight(self) -> torch.Tensor:
        """W_eff as the GEMM operand of gsb_biggan_conv_forward: [ksize^2 cin, cout], row (ky ksize + kx) cin + ci."""
        w = self.effective_weight()
        return w.permute(2, 3, 1, 0).reshape(-1, w.shape[0]).contiguous()


def _sn_linear(cin, cout, eps, bias=True):
    return SNLinear(nn.utils.spectral_norm(nn.Linear(cin, cout, bias=bias), eps=eps))


class _FusedModule(nn.Module):
    """A module whose arithmetic runs in the BigGAN chain (BigGAN.forward / partial_forward): ``forward(_result=act)`` only hands
    the chain's result to the forward hooks, the convention of stylegan2.StyledConv and progan.Block."""

    def forward(self, *args, _result=None, **kwargs):
        if _result is None:
            raise NotImplementedError(f"{type(self).__name__} runs as part of the BigGAN chain (BigGAN.forward / partial_forward); "
                                      "a stand-alone call is not built and there is no PyTorch fallback")
        return _result


class BigGANBatchNorm(_FusedModule):
    """model.py:99-149: BatchNorm with the statistics interpolated from 51 per-truncation tables; conditional: weight
    1 + scale(cond) and bias offset(cond), bias-free spectral-norm linears of the condition vector."""

    def __init__(self, num_features, condition_vector_dim=None, n_stats=51, eps=1e-4, conditional=True):
        super().__init__()
        self.num_features = num_features
        self.eps = eps
        self.conditional = conditional
        self.register_buffer("running_means", torch.zeros(n_stats, num_features))
        self.register_buffer("running_vars", torch.ones(n_stats, num_features))
        self.step_size = 1.0 / (n_stats - 1)
        if conditional:
            self.scale = _sn_linear(condition_vector_dim, num_features, eps, bias=False)
            self.offset = _sn_linear(condition_vector_dim, num_features, eps, bias=False)
        else:
            self.weight = nn.Parameter(torch.empty(num_features))         # uninitialised in the reference (torch.Tensor(n))
            self.bias = nn.Parameter(torch.empty(num_features))

    def stats(self, truncation):
        """(mean, var) at ``truncation``, interpolated exactly as the reference orders it (model.py:128-135)."""
        coef, start = math.modf(truncation / self.step_size)
        start = int(start)
        rm, rv = self.running_means.detach(), self.running_vars.detach()
        if coef != 0.0:
            return rm[start] * coef + rm[start + 1] * (1 - coef), rv[start] * coef + rv[start + 1] * (1 - coef)
        return rm[start], rv[start]


class GenBlock(_FusedModule):
    """model.py:152-202: bn_0 -> ReLU -> conv_0 (1x1) -> bn_1 -> ReLU -> [nearest x2] -> conv_1 (3x3) -> bn_2 -> ReLU -> conv_2 (3x3)
    -> bn_3 -> ReLU -> conv_3 (1x1), plus the skip path (first in/2 channels when in != out, nearest x2 when up-sampling)."""

    def __init__(self, in_size, out_size, condition_vector_dim, reduction_factor=4, up_sample=False, n_stats=51, eps=1e-12):
        super().__init__()
        self.up_sample = up_sample
        self.drop_channels = in_size != out_size
        mid = in_size // reduction_factor
        self.bn_0 = BigGANBatchNorm(in_size, condition_vector_dim, n_stats=n_stats, eps=eps)
        self.conv_0 = SNConv2d(in_size, mid, 1, eps=eps)
        self.bn_1 = BigGANBatchNorm(mid, condition_vector_dim, n_stats=n_stats, eps=eps)
        self.conv_1 = SNConv2d(mid, mid, 3, padding=1, eps=eps)
        self.bn_2 = BigGANBatchNorm(mid, condition_vector_dim, n_stats=n_stats, eps=eps)
        self.conv_2 = SNConv2d(mid, mid, 3, padding=1, eps=eps)
        self.bn_3 = BigGANBatchNorm(mid, condition_vector_dim, n_stats=n_stats, eps=eps)
        self.conv_3 = SNConv2d(mid, out_size, 1, eps=eps)


class SelfAttn(_FusedModule):
    """model.py:57-96: theta, phi, g 1x1 convs (C/8, C/8, C/2, no bias), 2x2 max-pool of phi and g, softmax over the keys,
    o_conv (C/2 -> C), out = x + gamma o."""

    def __init__(self, in_channels, eps=1e-12):
        super().__init__()
        self.in_channels = in_channels
        self.snconv1x1_theta = SNConv2d(in_channels, in_channels // 8, 1, bias=False, eps=eps)
        self.snconv1x1_phi = SNConv2d(in_channels, in_channels // 8, 1, bias=False, eps=eps)
        self.snconv1x1_g = SNConv2d(in_channels, in_channels // 2, 1, bias=False, eps=eps)
        self.snconv1x1_o_conv = SNConv2d(in_channels // 2, in_channels, 1, bias=False, eps=eps)
        self.gamma = nn.Parameter(torch.zeros(1))


class _Generator(nn.Module):
    """model.py:204-229, modules created in the reference's order."""

    def __init__(self, gen_z, config):
        super().__init__()
        self.config = config
        ch = config.channel_width
        cdim = 2 * config.z_dim
        self.gen_z = gen_z
        layers = []
        for i, (up, cin, cout) in enumerate(config.layers):
            if i == config.attention_layer_position:
                layers.append(SelfAttn(ch * cin, eps=config.eps))
            layers.append(GenBlock(ch * cin, ch * cout, cdim, up_sample=up, n_stats=config.n_stats, eps=config.eps))
        self.layers = nn.ModuleList(layers)
        self.bn = BigGANBatchNorm(ch, n_stats=config.n_stats, eps=config.eps, conditional=False)
        self.conv_to_rgb = SNConv2d(ch, ch, 3, padding=1, eps=config.eps)


class _BigGANNet(nn.Module):
    """Module tree, parameter and buffer names of pytorch_pretrained_biggan.BigGAN (a pytorch_model.bin loads by key)."""

    def __init__(self, resolution):
        super().__init__()
        self.config = _Config(resolution)
        # creation order == the reference's (embeddings, then Generator: gen_z, layers, bn, conv_to_rgb), so that
        # torch.manual_seed(s) reproduces the reference's random init bit-for-bit (gen_z's is a prefix of it)
        self.embeddings = nn.Linear(self.config.num_classes, self.config.z_dim, bias=False)
        self.generator = _Generator(_sn_linear(2 * self.config.z_dim, 4 * 4 * 16 * self.config.channel_width, self.config.eps),
                                    self.config)
        self.n_latents = len(self.config.layers) + 1

    def style_layers(self):
        """(name, width) of every conditional-BatchNorm row layer ``generator.layers.k.bn_j.scale`` / ``.offset``, in execution order
        (per GenBlock k: bn_0 .. bn_3, scale before offset, as BigGANBatchNorm.forward calls them)."""
        return [(f"generator.layers.{k}.bn_{j}.{kind}", getattr(layer, f"bn_{j}").num_features)
                for k, layer in enumerate(self.generator.layers) if isinstance(layer, GenBlock)
                for j in range(4) for kind in ("scale", "offset")]

    def unhookable_layers(self, n_modules=None, tail=True):
        """The sub-modules the chain gives no output of their own, in generator.layers[:n_modules] (all by default) and, with
        ``tail``, generator.bn and generator.conv_to_rgb: every module inside a block except the row layers."""
        rows = {name for name, _ in self.style_layers()}
        out = [name for i, layer in enumerate(list(self.generator.layers)[:n_modules])
               for name, m in layer.named_modules(prefix=f"generator.layers.{i}") if m is not layer and name not in rows]
        return out + (["generator.bn", "generator.conv_to_rgb"] if tail else [])


@torch.no_grad()
def synthesis_fill(net, seed=0):
    """Seeded values for what a random init leaves degenerate or undefined: the BatchNorm statistics tables (zeros and ones),
    ``SelfAttn.gamma`` (zero) and ``generator.bn.weight`` / ``bias`` (uninitialised).  Works on this module tree and on the
    reference's (same attribute names), so that both get the same weights.

    Spectral normalisation with random u, v does not bound a random conv (sigma = u^T W v is not its norm), so a BatchNorm with
    unit statistics would let the activations grow by orders of magnitude per conv.  The tables are therefore scaled to the
    second moment each BatchNorm's input would have if every conv input were independent and zero-mean (propagated per channel
    through the effective weights, in fp64), then perturbed per truncation row: every BatchNorm re-normalises and the 51 rows
    differ, so the interpolation is visible.  The tail BatchNorm's weight is scaled so that ``conv_to_rgb`` stays out of tanh's
    saturation."""
    gen = torch.Generator().manual_seed(int(seed))
    randn = lambda *s: torch.randn(*s, generator=gen, dtype=torch.float64)
    rand = lambda *s: torch.rand(*s, generator=gen, dtype=torch.float64)
    g = net.generator
    cfg = net.config

    def w_eff(m):
        w = m.weight_orig.detach().double().cpu()
        return w / torch.dot(m.weight_u.double().cpu(), torch.mv(w.reshape(w.shape[0], -1), m.weight_v.double().cpu()))

    def conv_m2(m, m2):
        out = w_eff(m).pow(2).flatten(2).sum(2) @ m2
        return out if m.bias is None else out + m.bias.detach().double().cpu().pow(2)

    cond_m2 = torch.cat([torch.ones(cfg.z_dim, dtype=torch.float64),
                         net.embeddings.weight.detach().double().cpu().pow(2).mean(1)])

    def fill_bn(bn, m2):
        c = m2.numel()
        sd = m2.clamp_min(1e-12).sqrt()
        bn.running_means.copy_(0.3 * sd * randn(cfg.n_stats, c))
        bn.running_vars.copy_(m2.clamp_min(1e-12) * (0.5 + rand(cfg.n_stats, c)))
        if bn.conditional:                     # E[((1 + s) x^ + o)^2] with x^ of unit second moment, then ReLU halves it
            return 0.5 * (1 + w_eff(bn.scale).pow(2) @ cond_m2 + w_eff(bn.offset).pow(2) @ cond_m2)
        return None

    wz = w_eff(g.gen_z)
    m2 = (wz.pow(2) @ cond_m2 + g.gen_z.bias.detach().double().cpu().pow(2)).view(16, -1).mean(0)      # NHWC [4, 4, 16 ch]
    for layer in g.layers:
        if hasattr(layer, "snconv1x1_theta"):
            # o_conv's output is not normalised: gamma brings it to the scale of its input, so that neither term drowns the other
            o2 = conv_m2(layer.snconv1x1_o_conv, conv_m2(layer.snconv1x1_g, m2))
            gamma = (0.5 + 0.5 * rand(1)) * torch.sqrt(m2.mean() / o2.mean())
            layer.gamma.copy_(gamma)
            m2 = m2 + gamma.pow(2) * o2
            continue
        h = m2
        for bn, conv in ((layer.bn_0, layer.conv_0), (layer.bn_1, layer.conv_1), (layer.bn_2, layer.conv_2), (layer.bn_3, layer.conv_3)):
            h = conv_m2(conv, fill_bn(bn, h))
        m2 = h + m2[:h.numel()]
    fill_bn(g.bn, m2)
    kappa = 1.0 / torch.sqrt(0.5 * w_eff(g.conv_to_rgb)[:3].pow(2).flatten(1).sum(1).mean())
    c = m2.numel()
    g.bn.weight.copy_(kappa * (0.5 + rand(c)))
    g.bn.bias.copy_(0.2 * kappa * randn(c))


class AffineLayer:
    """act = y Q^T + offset,  y = z R^T  (see module docstring).  All device tensors."""

    def __init__(self, Q64, R64, offset64, shift64=None, rank=None):
        self.Q = Q64                                   # [d, r] fp64, orthonormal columns
        self.Q32 = Q64.float().contiguous()
        self.R32 = R64.float().contiguous()           # [r, r]
        self.offset = offset64                         # [d] fp64: b + W_eff[:, r:] @ embed
        self.shift32 = None if shift64 is None else shift64.float().contiguous()
        self.rank = Q64.shape[1] if rank is None else rank
        self.dim = Q64.shape[0]

    def coords(self, z: torch.Tensor) -> torch.Tensor:
        """y = z R^T (+ shift) through the fp32 GEMM kernel."""
        return _native.linear(z, self.R32, self.shift32)

    def linear_form(self):
        """The same map with no offset: act = yt Qt^T, Qt = [Q, q_o, 0] and yt = z Rt^T + t = [y + Q^T offset, |o_perp|, 0],
        where o_perp = offset - Q Q^T offset and q_o = o_perp / |o_perp|.  A zero activation row is then a zero coordinate
        row, which fbpca's zero-padded sample matrix needs (DESIGN.md section 5g).  The width is padded to a multiple of 128
        (the GEMM kernel's output tile); ``rank`` is r + 1, or r when the offset lies in range(Q)."""
        d, r = self.Q.shape
        w = (r + 1 + 127) // 128 * 128
        a = self.Q.T @ self.offset
        perp = self.offset - self.Q @ a
        b = torch.linalg.vector_norm(perp)
        inside = bool(b <= 1e-12 * torch.linalg.vector_norm(self.offset))
        Qt = torch.zeros((d, w), dtype=torch.float64, device=self.Q.device)
        Qt[:, :r] = self.Q
        Rt = torch.zeros((w, self.R32.shape[1]), dtype=torch.float64, device=self.Q.device)
        Rt[:r] = self.R32.double()
        t = torch.zeros(w, dtype=torch.float64, device=self.Q.device)
        t[:r] = a
        if not inside:
            Qt[:, r] = perp / b
            t[r] = b
        return AffineLayer(Qt, Rt, torch.zeros_like(self.offset), shift64=t, rank=r + (0 if inside else 1))

    def lift_rows(self, rows64: torch.Tensor) -> torch.Tensor:
        """rows [k, r] in y-space -> [k, d] in activation space (directions: no offset); in-tree GEMM kernel, fp32 (the
        results are stored as float32)."""
        return _native.linear(rows64.float().contiguous(), self.Q32).double()


class _Chain:
    """The synthesis weights folded at one truncation and uploaded for csrc/biggan.cu, and the launch sequence of each module.
    Per GenBlock BatchNorm: the interpolated mean and variance and the effective scale / offset weights, whose products with the
    samples' condition vectors become per-(sample, channel) affine tables at run time; per conv: W_eff as a [k^2 cin, cout]
    GEMM operand; SelfAttn: theta | phi | g as one GEMM operand; tail: the BatchNorm as a per-channel affine and the first three
    output channels of conv_to_rgb (the only ones the image keeps)."""

    def __init__(self, net, truncation, device):
        f = lambda t: t.detach().to(device=device, dtype=torch.float32).contiguous()
        g = net.generator
        self.device = device
        self.steps = []
        for layer in g.layers:
            if isinstance(layer, SelfAttn):
                w = torch.cat([m.gemm_weight() for m in (layer.snconv1x1_theta, layer.snconv1x1_phi, layer.snconv1x1_g)], dim=1)
                self.steps.append(dict(w_tpg=f(w), w_o=f(layer.snconv1x1_o_conv.gemm_weight()), gamma=float(layer.gamma.detach())))
                continue
            bns = []
            for bn in (layer.bn_0, layer.bn_1, layer.bn_2, layer.bn_3):
                mean, var = bn.stats(truncation)
                bns.append(dict(mean=f(mean), var=f(var), ws=f(bn.scale.effective_weight()), wo=f(bn.offset.effective_weight()),
                                eps=bn.eps))
            convs = [dict(w=f(c.gemm_weight()), b=f(c.bias)) for c in (layer.conv_0, layer.conv_1, layer.conv_2, layer.conv_3)]
            cin, mid, cout = layer.conv_0.weight_orig.shape[1], layer.conv_0.weight_orig.shape[0], layer.conv_3.weight_orig.shape[0]
            assert cout == cin or 2 * cout == cin
            self.steps.append(dict(cin=cin, mid=mid, cout=cout, up=bool(layer.up_sample), bns=bns, convs=convs))
        mean, var = g.bn.stats(truncation)
        self.tail = dict(mean=f(mean), scale=f(g.bn.weight.detach() / torch.sqrt(var + g.bn.eps)), offset=f(g.bn.bias),
                         w=f(g.conv_to_rgb.effective_weight()[:3]), b=f(g.conv_to_rgb.bias[:3]))

    def _empty(self, *shape):
        return torch.empty(shape, dtype=torch.float32, device=self.device)

    def rows(self, i, cond, js):
        """The rows (cond W_scale^T, cond W_offset^T) [n, C_j] of BatchNorms ``js`` of GenBlock i, in one launch: what the hooks of
        generator.layers.i.bn_j.scale / .offset receive."""
        bns = self.steps[i]["bns"]
        with _native.instrument.section("biggan rows"):
            return _native.biggan_bn_rows(cond, [(bns[j]["ws"], bns[j]["wo"]) for j in js])

    def table(self, i, j, n, scale_rows, offset_rows):
        """The (scale, offset) tables [n, C] of BatchNorm j of GenBlock i from given rows ([n, C], row-strided, or [1, C])."""
        bn = self.steps[i]["bns"][j]
        c = bn["mean"].numel()
        scale, offset = self._empty(n, c), self._empty(n, c)
        with _native.instrument.section("biggan rows"):
            _native.biggan_bn_table_rows(scale_rows, offset_rows, bn["var"], bn["eps"], scale, offset)
        return scale, offset

    def block(self, i, x, cond, tables=None):
        """GenBlock i on NHWC x [n, R, R, cin] with condition vectors cond [n, 256] -> [n, R', R', cout].  ``tables``: {j: (scale,
        offset)} caller-built tables [n, C_j] for BatchNorm j (``table``); the others are folded from cond here."""
        p = self.steps[i]
        n, R = x.shape[0], x.shape[1]
        R2 = 2 * R if p["up"] else R
        mid, cin, cout = p["mid"], p["cin"], p["cout"]
        tables = tables or {}
        with _native.instrument.section(f"biggan layers.{i}"):
            tabs = []
            for j, bn in enumerate(p["bns"]):
                if j in tables:
                    tabs.append((bn["mean"], *tables[j]))
                    continue
                c = bn["mean"].numel()
                scale, offset = self._empty(n, c), self._empty(n, c)
                _native.biggan_bn_table(cond, bn["ws"], bn["wo"], bn["var"], bn["eps"], scale, offset)
                tabs.append((bn["mean"], scale, offset))
            (w0, w1, w2, w3) = p["convs"]
            t0 = self._empty(n, R, R, mid)
            _native.biggan_conv(x, n, cin, R, 1, w0["w"], mid, t0, bn=tabs[0], bias=w0["b"])
            t1 = self._empty(n, R2, R2, mid)
            _native.biggan_conv(t0, n, mid, R, 3, w1["w"], mid, t1, upsample=p["up"], bn=tabs[1], bias=w1["b"])
            t2 = self._empty(n, R2, R2, mid)
            _native.biggan_conv(t1, n, mid, R2, 3, w2["w"], mid, t2, bn=tabs[2], bias=w2["b"])
            out = self._empty(n, R2, R2, cout)
            _native.biggan_conv(t2, n, mid, R2, 1, w3["w"], cout, out, bn=tabs[3], bias=w3["b"], res=x, ldres=cin,
                                res_upsample=p["up"])
        _native.instrument.add_rows("biggan", n if i == 0 else 0)
        return out

    def attn(self, i, x):
        """SelfAttn i on NHWC x [n, R, R, C]: theta | phi | g in one GEMM, 2x2 max-pool, scores against the pooled keys, softmax
        over the keys, the weighted sum of the pooled g, then o_conv with x + gamma o in its epilogue."""
        p = self.steps[i]
        n, R, C = x.shape[0], x.shape[1], x.shape[3]
        c8, c2, hwp = C // 8, C // 2, R * R // 4
        ct = 2 * c8 + c2
        with _native.instrument.section(f"biggan layers.{i}"):
            tpg = self._empty(n, R, R, ct)
            _native.biggan_conv(x, n, C, R, 1, p["w_tpg"], ct, tpg)
            phi_t, gp = self._empty(n, c8, hwp), self._empty(n, hwp, c2)
            _native.biggan_attn_pool(tpg, n, R, C, phi_t, gp)
            s = self._empty(n, R * R, hwp)
            _native.biggan_conv(tpg, n, c8, R, 1, phi_t, hwp, s, ldx=ct, w_sample_stride=c8 * hwp)
            _native.biggan_softmax_rows(s, n * R * R, hwp)
            o = self._empty(n, R * R, c2)
            _native.biggan_conv(s, n, hwp, R, 1, gp, c2, o, w_sample_stride=hwp * c2)
            out = self._empty(n, R, R, C)
            _native.biggan_conv(o, n, c2, R, 1, p["w_o"], C, out, alpha=p["gamma"], res=x)
        return out

    def rgb(self, x):
        """Tail on NHWC x [n, R, R, ch]: image 0.5 (tanh(conv_to_rgb(ReLU(bn(x)))[:3]) + 1), NHWC [n, R, R, 3]."""
        n, R, C = x.shape[0], x.shape[1], x.shape[3]
        t = self.tail
        img = self._empty(n, R, R, 3)
        with _native.instrument.section("biggan rgb"):
            _native.biggan_rgb(x, n, R, C, t["mean"], t["scale"], t["offset"], t["w"], t["b"], img)
        return img


class BigGAN(_DeviceGenerator):
    _latent_shape = (1, 128)

    def __init__(self, device, resolution, class_name, truncation=1.0, random_init=None):
        super().__init__(f"BigGAN-{resolution}", class_name)
        self.device = _native.require_cuda(device)
        self.truncation = truncation
        self._random_init = random_init
        self.resolution = int(resolution)
        self.load_model(f"biggan-deep-{resolution}")
        self.set_output_class(class_name or "husky")
        self.name = f"BigGAN-{resolution}-{self.outclass}-t{self.truncation}"
        self.has_latent_residual = True
        self._affine = {}

    def load_model(self, name):
        if self.resolution not in _LAYERS:
            raise RuntimeError("Unknown BigGAN model name", name)
        source = self._weight_source(_checkpoint(f"{name}/pytorch_model.bin"), overrides=("GANSPACE_B200_RANDOM_INIT_BIGGAN",))
        if isinstance(source, int):
            torch.manual_seed(source)
            net = _BigGANNet(self.resolution)
            synthesis_fill(net, source)
        else:
            net = _BigGANNet(self.resolution)
            net.load_state_dict(torch.load(source, map_location="cpu"), strict=False)      # as BigGAN.from_pretrained
        # only the embedding and gen_z go to the device here: the synthesis weights are folded and uploaded on the first
        # synthesis call (_chain), so that gen_z-only runs (decomposition of generator.gen_z) never touch them
        net.embeddings.to(self.device)
        net.generator.gen_z.to(self.device)
        self.model = net
        self._chain_cache = _native.Repacked()

    # ---- latents ----------------------------------------------------------------------------------
    def sample_latent(self, n_samples=1, truncation=None, seed=None):
        if seed is None:
            seed = _global_seed()
        t = truncation or self.truncation
        return _native.legacy_truncnorm([seed], 128 * n_samples, -2.0, 2.0, float(t), self.device).view(n_samples, 128)

    def sample_latents_multi(self, n_samples, seeds, out=None):
        z = _native.legacy_truncnorm(list(seeds), 128 * n_samples, -2.0, 2.0, float(self.truncation), self.device)
        return z.view(len(seeds) * n_samples, 128)

    def get_max_latents(self):
        return len(self.model.config.layers) + 1

    def get_conditional_state(self, z):
        return self.v_class

    def set_conditional_state(self, z, c):
        self.v_class = c

    def is_valid_class(self, class_id):
        if isinstance(class_id, int):
            return class_id < 1000
        if isinstance(class_id, str):
            return class_id.replace(" ", "_").lower() in _CLASS_IDS
        raise RuntimeError(f"Unknown class identifier {class_id}")

    def set_output_class(self, class_id):
        if isinstance(class_id, int):
            idx = class_id
            self.outclass = f"class{class_id}"
        elif isinstance(class_id, str):
            key = class_id.replace(" ", "_").lower()
            if key not in _CLASS_IDS:
                raise RuntimeError(f"Unknown class identifier {class_id} (WordNet lookup is not available offline; "
                                   f"known names: {sorted(_CLASS_IDS)}; or pass the ImageNet class index)")
            idx = _CLASS_IDS[key]
            self.outclass = class_id.replace(" ", "_")
        else:
            raise RuntimeError(f"Unknown class identifier {class_id}")
        one_hot = torch.zeros(1, 1000, dtype=torch.float32)
        one_hot[0, idx] = 1.0
        self.v_class = one_hot.to(self.device)
        self._class_idx = idx
        self._affine = {}
        if hasattr(self, "model"):
            self.affine_layer("generator.gen_z")       # thin QR of the folded weight: model/class set-up, not part of a run

    def _embed(self) -> torch.Tensor:
        """embeddings(one_hot) = column `idx` of the embedding matrix  -> [128] fp32."""
        return self.model.embeddings.weight.detach()[:, self._class_idx].contiguous()

    # ---- synthesis: GenBlock / SelfAttn chain and the RGB tail (csrc/biggan.cu) --------------------------------------------
    def _conds(self, x):
        """cond[k] = cat(z[k], embed) for the n_latents latents (one z is used for all of them), model.py:295-309."""
        n_lat = self.model.n_latents
        zs = x if isinstance(x, list) else n_lat * [x]
        assert len(zs) == n_lat, f"Expected {n_lat} latents, got {len(zs)}"
        e = self._embed().unsqueeze(0)
        return [torch.cat((z.reshape(z.shape[0], -1).float(), e.expand(z.shape[0], -1)), dim=1).contiguous() for z in zs]

    def _chain(self):
        """The synthesis weights folded and uploaded at the current truncation (again when a parameter or buffer changes)."""
        g = self.model.generator
        tensors = [t for m in (g.layers, g.bn, g.conv_to_rgb) for t in list(m.parameters()) + list(m.buffers())]
        return self._chain_cache.get(tensors, lambda: _Chain(self.model, float(self.truncation), self.device), float(self.truncation))

    def _synthesize(self, x, n_modules, want_image):
        """gen_z, then generator.layers[:n_modules] (and the tail when ``want_image``), firing the hooks of every layer on the
        way.  A hook's result on gen_z is what the chain continues from; an edit on a later layer would have to be re-fed into the
        chain, which is not built -- it raises instead of being silently ignored (except on the last layer of a partial run).
        The row layers generator.layers.k.bn_j.scale / .offset are the exception: a hooked block's rows are computed from its own
        condition vectors and handed to the hooks, and its BatchNorm tables are built from what they return, so an edit there
        reaches block k and everything after it.  A partial run (no image) with no generator.layers.k hooked computes only the
        hooked rows and launches no conv."""
        g = self.model.generator
        layers = list(g.layers)[:n_modules]
        mods = self._modules_by_name()
        for name in self.model.unhookable_layers(n_modules, tail=want_image):
            if len(mods[name]._forward_hooks):
                raise NotImplementedError(f"a hook on '{name}': the BigGAN chain materialises the outputs of gen_z and of "
                                          "generator.layers.k only")
        hooked_rows = {}                                # block index -> [(j, kind, name)] of its hooked row layers
        for name, _ in self.model.style_layers():
            k, j, kind = _row_layer(name)
            if k < len(layers) and len(mods[name]._forward_hooks):
                hooked_rows.setdefault(k, []).append((j, kind, name))
        conds = self._conds(x)
        chain = self._chain()
        if hooked_rows and not want_image and not any(len(m._forward_hooks) for m in layers):
            if len(g.gen_z._forward_hooks):
                g.gen_z(conds[0])
            for k in sorted(hooked_rows):
                self._block_tables(chain, k, self._block_cond(conds, k), hooked_rows[k], build=False)
            return None
        h = g.gen_z(conds[0])
        act = h.contiguous().view(h.shape[0], 4, 4, -1)                 # gen_z's output is NHWC [4, 4, 16 ch] already
        ci = 1
        for i, mod in enumerate(layers):
            if isinstance(mod, GenBlock):
                tables = self._block_tables(chain, i, conds[ci], hooked_rows[i]) if i in hooked_rows else None
                act = chain.block(i, act, conds[ci], tables)
                ci += 1
            else:
                act = chain.attn(i, act)
            if len(mod._forward_hooks):
                self._hand_off(mod, act, act.shape[1], act.shape[3], want_image or i < len(layers) - 1, f"generator.layers.{i}")
        return chain.rgb(act).permute(0, 3, 1, 2) if want_image else None

    def edit_reaches_image(self, layer_name):
        """gen_z's output is what the chain continues from, and a row layer's rows are what its block's BatchNorm tables are built
        from; an edit on generator.layers.k would have to be re-fed into the chain."""
        return layer_name == "generator.gen_z" or layer_name in dict(self.model.style_layers())

    def _modules_by_name(self):
        mods = getattr(self, "_by_name", None)
        if mods is None:
            mods = self._by_name = dict(self.model.named_modules())
        return mods

    def _block_cond(self, conds, k):
        """The condition vectors of the GenBlock at generator.layers[k] (one per GenBlock, after gen_z's)."""
        return conds[1 + sum(isinstance(m, GenBlock) for m in list(self.model.generator.layers)[:k])]

    def _block_tables(self, chain, k, cond, hooked, build=True):
        """The rows of the BatchNorms of GenBlock k that have a hooked row layer (one launch), handed to the hooks; returns {j:
        (scale, offset)} tables built from what the hooks return (``build``; a rows-only run builds none)."""
        mods = self._modules_by_name()
        js = sorted({j for j, _, _ in hooked})
        rows = dict(zip(js, chain.rows(k, cond, js)))
        tables = {}
        for j in js:
            s, o = rows[j]
            for jj, kind, name in hooked:
                if jj == j and kind == "scale":
                    s = self._hand_rows(mods[name], s, name)
                elif jj == j:
                    o = self._hand_rows(mods[name], o, name)
            if build:
                tables[j] = chain.table(k, j, cond.shape[0], s, o)
        return tables

    @staticmethod
    def _hand_rows(module, rows, name):
        """Hands a row layer's rows [n, C] to its hooks and returns what the tables are built from: the rows, or the hooks' edit
        (a [1, C] edit applies to every sample, as nethook broadcasts it)."""
        out = module(_result=rows)
        if out is rows:
            return rows
        if not (out.dim() == 2 and out.shape[1] == rows.shape[1] and out.shape[0] in (1, rows.shape[0])):
            raise ValueError(f"an edit on '{name}' must keep the rows' shape {tuple(rows.shape)} (or [1, {rows.shape[1]}]), got "
                             f"{tuple(out.shape)}")
        out = out.to(device=rows.device, dtype=torch.float32)
        return out if out.stride(1) == 1 else out.contiguous()

    def forward(self, x):
        """wrappers.py:599-607: images 0.5 (G(z) + 1) in [0, 1], [n, 3, R, R] (an NCHW view of NHWC storage), from one latent or
        a list of n_latents (one per layer)."""
        return self._synthesize(x, len(self.model.generator.layers), True)

    def partial_forward(self, x, layer_name):
        """wrappers.py:611-648, including its quirks: 'generator.layers.k' runs layers[:k+1] of the ModuleList (SelfAttn is one of
        them); any other name but embeddings / gen_z runs layers[:len(config.layers)], one module short of the ModuleList, and
        never the tail.  Returns None; results reach the caller through hooks."""
        if layer_name in ("embeddings", "generator.gen_z"):
            z = x[0] if isinstance(x, list) else x
            cond = torch.cat((z, self._embed().unsqueeze(0).expand(z.shape[0], -1)), dim=1).contiguous()
            self.model.generator.gen_z(cond)             # hook retains [B, 4*4*16*ch]
            return None
        if "generator.layers" in layer_name:
            m = re.match(r"^generator\.layers\.[0-9]+", layer_name)
            if m is None:
                raise RuntimeError(f"Unknown layer '{layer_name}'")
            n_layers = int(m[0].split(".")[-1]) + 1
        else:
            n_layers = len(self.model.config.layers)
        self._synthesize(x, n_layers, False)
        return None

    # ---- low-rank structure of gen_z and of the row layers ------------------------------------------------
    def affine_layer(self, layer_name):
        """The exact factorisation act = (z R^T) Q^T + offset of a layer that is affine in z, or None when the decomposition
        driver is to materialise the layer's activations.  gen_z: A = W_eff[:, :128], offset = b + W_eff[:, 128:] embed.  A row
        layer generator.layers.k.bn_j.scale / .offset of width C: rows = z A^T + W_eff[:, 128:] embed (no bias), rank min(C, 128);
        C <= 128 gives no saving, so its rows are materialised (gsb_biggan_bn_rows) and go to the small-d engine.
        GANSPACE_B200_BIGGAN_AFFINE=0: no low-rank shortcut -- gen_z's activations are materialised and go through the general
        large-d engine (csrc/bigd.cu), and so are the rows of every row layer with C <= 1024 (the small-d engine), a cross-check
        of the shortcut."""
        widths = dict(self.model.style_layers())
        if layer_name.startswith("generator.") and layer_name != "generator.gen_z" and layer_name not in widths:
            raise NotImplementedError(f"BigGAN: decomposing '{layer_name}' is not built; of the generator's layers only "
                                      "generator.gen_z and the conditional-BatchNorm row layers generator.layers.k.bn_j.scale / "
                                      ".offset can be decomposed")
        if layer_name != "generator.gen_z" and layer_name not in widths:
            return None
        no_shortcut = os.environ.get("GANSPACE_B200_BIGGAN_AFFINE", "1") == "0"
        if layer_name == "generator.gen_z" and no_shortcut:
            return None
        r = self.model.config.z_dim
        if layer_name in widths and (widths[layer_name] <= r or (no_shortcut and widths[layer_name] <= 1024)):
            return None
        if layer_name not in self._affine:
            g = self._modules_by_name()[layer_name]
            w = g.effective_weight().to(self.device).double()                # [d, 256] (the row layers' weights stay on the host)
            Q, R = torch.linalg.qr(w[:, :r].contiguous(), mode="reduced")   # one-time setup (like weight packing)
            offset = w[:, r:] @ self._embed().double()
            if g.bias is not None:
                offset = g.bias.detach().double() + offset
            self._affine[layer_name] = AffineLayer(Q.contiguous(), R.contiguous(), offset.contiguous())
        return self._affine[layer_name]
