"""Model wrappers of the hot path: ``BaseModel``, ``StyleGAN2``, ``get_model``, ``get_instrumented_model``.

Mirror of /root/reference/models/wrappers.py (BaseModel :27-94, StyleGAN2 :97-267, factories :651-735):
same class and method names, argument meaning and error behaviour, so ``decomposition.get_or_compute``,
``visualize.py`` and the notebooks call them unchanged.  Differences, all on the device side:

* ``sample_latent`` draws the NumPy-legacy normal stream ON THE GPU (bit-exact MT19937 + polar method,
  csrc/rng.cu) -- the seed is still taken from NumPy's global state on the host exactly as the reference
  does (wrappers.py:168-169), so seeds and latents are identical.
* ``Generator.style`` runs the hand-written mapping kernels (csrc/mapping*.cu).
* ``partial_forward(x, 'style')`` stops right after the mapping network; the reference first builds the
  ``[B, n_latent, 512]`` repeat+stack that the early exit then throws away (wrappers.py:202-222).
* checkpoints: no network here.  A rosinality ``g_ema`` checkpoint under $GANCONTROL_CHECKPOINT_DIR is
  loaded when present; otherwise ``random_init=<seed>`` (or env GANSPACE_B200_RANDOM_INIT) reproduces the
  reference's default initialisation under ``torch.manual_seed(seed)`` (the BASELINE.json configs).
"""
from __future__ import annotations

import os
from abc import ABC as AbstractBaseClass, abstractmethod
from functools import singledispatch
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import torch

from .. import _native
from ..config import Config
from ..netdissect.nethook import InstrumentedModel
from . import stylegan2

INT32_MAX = int(np.iinfo(np.int32).max)


def _global_seed() -> int:
    """``np.random.randint(np.iinfo(np.int32).max)`` on NumPy's global legacy state (wrappers.py:169)."""
    return int(np.random.randint(INT32_MAX))


class BaseModel(AbstractBaseClass, torch.nn.Module):
    def __init__(self, model_name, class_name):
        super().__init__()
        self.model_name = model_name
        self.outclass = class_name

    @abstractmethod
    def partial_forward(self, x, layer_name):
        """Run the network only up to ``layer_name`` (hooks fire as a side effect); returns None."""

    @abstractmethod
    def sample_latent(self, n_samples=1, seed=None, truncation=None):
        """Batch of latents on ``self.device``."""

    def get_max_latents(self):
        return 1

    def latent_space_name(self):
        return "Z"

    def get_latent_shape(self):
        return tuple(self.sample_latent(1).shape)

    def get_latent_dims(self):
        return np.prod(self.get_latent_shape())

    def set_output_class(self, new_class):
        self.outclass = new_class

    def forward(self, x):
        out = self.model.forward(x)
        return 0.5 * (out + 1)

    def sample_np(self, z=None, n_samples=1, seed=None):
        if z is None:
            z = self.sample_latent(n_samples, seed=seed)
        elif isinstance(z, list):
            z = [torch.tensor(l).to(self.device) if not torch.is_tensor(l) else l for l in z]
        elif not torch.is_tensor(z):
            z = torch.tensor(z).to(self.device)
        img = self.forward(z)
        img_np = img.permute(0, 2, 3, 1).cpu().detach().numpy()
        return np.clip(img_np, 0.0, 1.0).squeeze()

    def get_conditional_state(self, z):
        return None

    def set_conditional_state(self, z, c):
        return z

    def named_modules(self, *args, **kwargs):
        return self.model.named_modules(*args, **kwargs)


def _checkpoint(relpath) -> Path:
    return Path(os.environ.get("GANCONTROL_CHECKPOINT_DIR", Path(__file__).parent / "checkpoints")) / relpath


class _DeviceGenerator(BaseModel):
    """What the wrappers of the generators that run on the device (StyleGAN2, StyleGAN, ProGAN, BigGAN) share: where the weights
    come from, the latent shape, the fixed output class, handing a fused chain's activations to the hooks, and the largest
    feature map that is decomposed."""

    _latent_shape = (1, 512)
    MAX_DECOMPOSITION_DIMS = None               # None: no bound

    def _weight_source(self, checkpoint: Path, overrides=()):
        """The seed of random-init weights, an int: ``random_init=``, else env GANSPACE_B200_RANDOM_INIT (whose value the first
        set variable of ``overrides`` replaces).  Without a seed, ``checkpoint`` if it is a file; else raises.  The answer is
        kept as ``weight_source`` (a saved decomposition state names the weights it was fitted with)."""
        seed = self._random_init
        if seed is None and os.environ.get("GANSPACE_B200_RANDOM_INIT"):
            seed = next(os.environ[e] for e in (*overrides, "GANSPACE_B200_RANDOM_INIT") if os.environ.get(e))
        if seed is not None:
            self.weight_source = int(seed)
            return int(seed)
        if checkpoint.is_file():
            self.weight_source = checkpoint
            return checkpoint
        raise RuntimeError(f"{self.model_name} checkpoint {checkpoint} not found and no network access to download it; pass "
                           "random_init=<seed> (or set GANSPACE_B200_RANDOM_INIT) for random-init weights")

    def get_latent_shape(self):
        """The reference samples one latent for its shape (wrappers.py:60-61).  The draw from the global NumPy stream that this
        sample_latent(1) consumes is kept (later seeds depend on it); the kernels behind it are not launched."""
        _global_seed()
        return self._latent_shape

    def set_output_class(self, new_class):
        if self.outclass != new_class:
            raise RuntimeError(f"{self.model_name}: cannot change output class without reloading")

    def edit_reaches_image(self, layer_name):
        """Whether an ``edit_layer`` offset on ``layer_name`` reaches the image ``forward`` returns.  A chain output (a conv map,
        a ToRGB image, a block) is handed to the hooks as a view that the fused chain cannot take back: not by default."""
        return False

    def _hand_off(self, module, act, res, channels, downstream, name):
        """Hands the fused chain's NHWC activation ``act`` of layer ``name`` to the forward hooks of ``module`` as an NCHW view,
        and returns the view.  A hook that returns another tensor edits the layer.  The chain cannot take an edit back, so when
        the run goes on past this layer (``downstream``) the edit raises instead of being silently ignored."""
        view = act.view(-1, res, res, channels).permute(0, 3, 1, 2)
        if module(_result=view) is not view and downstream:
            raise NotImplementedError(f"an edit on layer '{name}' cannot be propagated through the fused {self.model_name} chain")
        return view

    def _nhwc_layout(self, layer_name, res, channels):
        """``feature_layout`` of a conv layer: ('nhwc', (H, W, C)), the device order of ``activations_into``; the reference's
        flattening is NCHW -- a fixed permutation, applied once to the exported components."""
        d = res * res * channels
        if self.MAX_DECOMPOSITION_DIMS is not None and d > self.MAX_DECOMPOSITION_DIMS:
            raise NotImplementedError(
                f"{self.model_name} {layer_name}: d = {d} exceeds {self.MAX_DECOMPOSITION_DIMS}, the largest feature map the large-d "
                "IPCA engine is run at: its stacked matrix holds (components + batch + 1) rows of d floats in HBM")
        return ("nhwc", (res, res, channels))


class _StyledGenerator(_DeviceGenerator):
    """A device generator with a mapping network and a style space (StyleGAN2, StyleGAN): latents are in Z, or in W after
    ``use_w``; ``forward`` and ``partial_forward`` share one skeleton.  Each model describes its fused chain as data:

    * ``_chain_outputs()``: (name, n_run, n_rgb) of every hookable chain output in execution order, with the chain run that ends
      at it: ``n_run`` layers and ``n_rgb`` ToRGBs.  The output is the run's last activation when ``n_rgb`` is 0, else its image;
    * ``_style_layers()``: (name, n_run, n_rgb) of every style layer, in the order of ``model.style_layers()`` (execution order),
      with the chain run that reaches it; style rows are keyed by their position in this table;
    * ``_image_run()``: the (n_run, n_rgb) of the image ``forward`` returns;
    * ``_stop(layer_name)``: the index of the chain output at which ``partial_forward`` stops (the reference's stop rule);
    * ``_chain(n_run)``: the packed chain (``forward``, ``styles``, ``forward_styled``, ``shapes``) covering ``n_run`` layers;
    * ``_w_layers(ws, truncate)``: the [Lw, n, 512] per-layer latents of a call ([1, n, 512] for one latent);
    * ``_stops_before_chain(layer_name, ws)``: whether ``partial_forward`` ends before the fused chain (in the mapping network);
    * ``model.unhookable_layers()`` and ``_unhookable_message(name)``: the sub-modules the chain gives no output of their own."""

    def latent_space_name(self):
        return "W" if self.w_primary else "Z"

    def use_w(self):
        self.w_primary = True

    def use_z(self):
        self.w_primary = False

    def _draw_z(self, n_samples, seed):
        return _native.legacy_normal([seed], 512 * n_samples, self.device).view(n_samples, 512)

    def sample_latent(self, n_samples=1, seed=None, truncation=None):
        z = self._draw_z(n_samples, _global_seed() if seed is None else seed)
        # a module call: the mapping network's hooks fire here in W mode, as in the reference
        return self._mapping()(z) if self.w_primary else z

    @staticmethod
    def _hand_style(module, rows, name):
        """Hands a style layer's rows [n, width] to its hooks and returns what the chain uses: the rows, or the hooks' edit (a
        [1, width] edit applies to every sample, as nethook broadcasts it)."""
        out = module(_result=rows)
        if out is rows:
            return rows
        if out.dim() == 2 and out.shape[0] == 1:
            out = out.expand(rows.shape[0], -1)
        if tuple(out.shape) != tuple(rows.shape):
            raise ValueError(f"an edit on '{name}' must keep the style's shape {tuple(rows.shape)} (or [1, {rows.shape[1]}]), got "
                             f"{tuple(out.shape)}")
        return out.to(device=rows.device, dtype=torch.float32).contiguous()

    def edit_reaches_image(self, layer_name):
        """Style layers: their rows are handed to the hooks before the chain consumes them, in Z and in W.  The mapping network's
        output: in Z only, where ``forward`` calls it as a module and continues from its result; in W ``forward`` never runs it."""
        if layer_name in {t[0] for t in self._style_layers()}:
            return True
        return layer_name == self._MAPPING_LAYER and not self.w_primary

    def _module(self, name):
        mods = getattr(self, "_by_name", None)
        if mods is None:
            mods = self._by_name = dict(self.model.named_modules())
        return mods[name]

    def _reject_sub_module_hooks(self, layer_name=None):
        """Refuses hooks on, and ``partial_forward`` to, the sub-modules that run inside the fused chain."""
        guarded = getattr(self, "_guarded", None)
        if guarded is None:
            guarded = self._guarded = {n: self._module(n) for n in self.model.unhookable_layers()}
        for name, m in guarded.items():
            if len(m._forward_hooks) or len(m._forward_pre_hooks):
                raise NotImplementedError(self._unhookable_message(name))
        if layer_name in guarded:
            raise NotImplementedError(self._unhookable_message(layer_name))

    def forward(self, x):
        """wrappers.py: images in [0, 1] (before clamping) from one latent or a list of per-layer latents.  Hooked chain outputs
        receive their activations (retain_layer works); an edit of one would have to be re-fed into the fused chain, which is not
        built -- it raises instead of being silently ignored.  Hooked style layers receive their style rows once per call, and what
        their hooks return is what every chain run of the call uses."""
        return 0.5 * (self._synthesize(x, None).permute(0, 3, 1, 2) + 1)

    def partial_forward(self, x, layer_name):
        """Runs the network up to the chain output the reference's stop rule names for ``layer_name``; the side effect is that the
        hooks on the way fire.  An edit is accepted on that last output alone.  With only style layers hooked, only their rows
        are computed (no synthesis launch)."""
        self._synthesize(x, layer_name)

    def _hooked(self, name):
        return len(self._module(name)._forward_hooks) > 0

    def _synthesize(self, x, layer_name):
        """The skeleton of ``forward`` (``layer_name`` None; returns the NHWC image) and ``partial_forward``."""
        self._reject_sub_module_hooks(layer_name)
        ws = x if isinstance(x, list) else [x]
        if not self.w_primary:
            ws = [self._mapping()(s) for s in ws]          # module calls: the mapping network's hooks fire
        if layer_name is not None and self._stops_before_chain(layer_name, ws):
            return None
        w_layers = self._w_layers(ws, layer_name is None)
        outs = self._chain_outputs()
        outs = outs if layer_name is None else outs[:self._stop(layer_name) + 1]
        image = self._image_run() if layer_name is None else None
        n_run, n_rgb = image or (max(o[1] for o in outs), max(o[2] for o in outs))
        hooked = [o for o in outs if self._hooked(o[0])]
        # the style stage: once, with every row of the call's layers when a chain run consumes them
        styles = [(k, t) for k, t in enumerate(self._style_layers()) if t[1] <= n_run and t[2] <= n_rgb]
        S = None
        if any(self._hooked(t[0]) for _, t in styles):
            want = [(k, t) for k, t in styles if hooked or image or self._hooked(t[0])]
            S = self._chain(n_run).styles(w_layers, [k for k, _ in want])
            for k, t in want:
                if self._hooked(t[0]):
                    S[k] = self._hand_style(self._module(t[0]), S[k], t[0])

        def run(n_run, n_rgb, want_act):
            # the chains' last argument: StyleGAN2's ToRGB count, StyleGAN's want_rgb (its one torgb after the last layer)
            chain = self._chain(n_run)
            if S is None:
                return (chain, *chain.forward(w_layers, n_run, None, want_act, n_rgb))
            return (chain, *chain.forward_styled(S, n_run, None, want_act, n_rgb))

        def hand(o, chain, act, img):
            # an edit raises when the run goes on past the output: before the last output, or when the image is made
            downstream = image is not None or o is not outs[-1]
            if o[2]:
                self._hand_off(self._module(o[0]), img, img.shape[1], 3, downstream, o[0])
            else:
                self._hand_off(self._module(o[0]), act, *chain.shapes[o[1] - 1], downstream, o[0])
        # the image's run also serves the outputs it ends at: the last activation, and the image itself
        served = [o for o in hooked if image and (o[1], o[2]) in (image, (image[0], 0))]
        for o in hooked:
            if o not in served:
                hand(o, *run(o[1], o[2], o[2] == 0))
        if image is None:
            return None
        chain, act, img = run(*image, any(o[2] == 0 for o in served))
        for o in served:
            hand(o, chain, act, img)
        return img

    def draw_z_async(self, n_samples, seed):
        """The Z stream of ``sample_latent(n_samples, seed=seed)`` generated on a side stream; returns a callable that makes
        the current stream wait for it and hands back z [n_samples, 512]."""
        side = getattr(self, "_side_stream", None)
        if side is None:
            with torch.cuda.device(self.device):
                side = self._side_stream = torch.cuda.Stream(device=self.device)
        with torch.cuda.device(self.device):
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                z = self._draw_z(n_samples, seed)

        def result():
            with torch.cuda.device(self.device):
                torch.cuda.current_stream().wait_stream(side)
            z.record_stream(torch.cuda.current_stream())
            return z
        return result


class StyleGAN2(_StyledGenerator):
    _MAPPING_LAYER = "style"
    CONFIGS = {"ffhq": 1024, "car": 512, "cat": 256, "church": 256, "horse": 256,
               "bedrooms": 256, "kitchen": 256, "places": 256}
    # deepest feature maps get_or_compute decomposes: convs.8 / convs.9, 128 x 128 x 256.  At c = 80 and a 2000-row batch the large-d
    # engine's stacked matrix is 2112 x d fp32 -- 35.4 GB there -- and convs.10 (d = 8,388,608) would need 71 GB for it alone
    MAX_DECOMPOSITION_DIMS = 4_194_304
    # largest synthesis workspace one activations_into call allocates: bigger batches run in slices of rows (the chain's workspace
    # holds four fp16 planes of the widest input map, 8.4 GB per 1000 samples into convs.8)
    SYNTH_WORKSPACE_BUDGET = 4 << 30

    def __init__(self, device, class_name, truncation=1.0, use_w=False, random_init=None):
        super().__init__("StyleGAN2", class_name or "ffhq")
        self.device = _native.require_cuda(device)
        self.truncation = truncation
        self.latent_avg = None
        self.w_primary = use_w
        assert self.outclass in self.CONFIGS, \
            f'Invalid StyleGAN2 class {self.outclass}, should be one of [{", ".join(self.CONFIGS.keys())}]'
        self.resolution = self.CONFIGS[self.outclass]
        self.name = f"StyleGAN2-{self.outclass}"
        self.has_latent_residual = True
        self._random_init = random_init
        self._synth, self._synth_keys = _native.Repacked(), ()
        self.load_model()
        self.set_noise_seed(0)

    def load_model(self):
        source = self._weight_source(_checkpoint(f"stylegan2/stylegan2_{self.outclass}_{self.resolution}.pt"))
        if isinstance(source, int):
            # the reference's default init, bit-for-bit: parameters are created on the host in the
            # reference's order under one manual seed, then moved to the device
            torch.manual_seed(source)
            self.model = stylegan2.Generator(self.resolution, 512, 8).to(self.device)
            self.latent_avg = torch.zeros(512, device=self.device)
        else:
            self.model = stylegan2.Generator(self.resolution, 512, 8)
            ckpt = torch.load(source, map_location="cpu")
            self.model.load_state_dict(ckpt["g_ema"], strict=False)
            self.model = self.model.to(self.device)
            self.latent_avg = ckpt["latent_avg"].to(self.device)

    def _mapping(self):
        return self.model.style

    def z_to_latent(self, z):
        """What sample_latent does after drawing z (wrappers.py:176-179): the mapping network in W mode."""
        return self.model.style(z) if self.w_primary else z

    def sample_latents_multi(self, n_samples, seeds, out=None, lazy=False):
        """Several ``sample_latent(n_samples, seed=s)`` calls in ONE launch (one CTA per seed);
        ``out`` is an optional [len(seeds)*n_samples, 512] device buffer.  Used by the decomposition
        driver so that a whole run's ~100 independent streams fill the machine.
        ``lazy=True`` (W space): returns (z, ensure) where ``ensure(row_end)`` maps rows [0, row_end) to W in
        place, chunk by chunk, so that the consumer of the first rows does not wait for the last ones."""
        S = len(seeds)
        parts = _native.split_parts(512 * n_samples)
        if not lazy:
            z = _native.legacy_normal(list(seeds), 512 * n_samples, self.device,
                                      out=None if out is None else out.view(S, 512 * n_samples), parts=parts)
            z = z.view(S * n_samples, 512)
            if not self.w_primary:
                return z
            return self.model.style(z) if out is None else self.model.style.packed().forward(z, out=z)
        # lazy: the streams are generated in launch groups on a side stream (a small first group, so that the first
        # partial_fit group exists after ~1.5 ms instead of after the whole run's RNG); ensure(row_end) waits for the groups
        # that cover rows [0, row_end) and, in W mode, maps them group by group in place.
        z = torch.empty((S * n_samples, 512), dtype=torch.float32, device=self.device) if out is None else out.view(S * n_samples, 512)
        # group sizes in streams (x parts CTAs each).  The merge chain's 16-CTA cluster launches need free SMs at every step, so
        # the producers share the machine statically: the persistent GEMM launches leave GANSPACE_B200_LAZY_FREE_SMS SMs to the
        # 7 x 8 = 56 RNG CTAs and the chain.  Config 2 on one H100 (132 SMs), ms per job: 72 free 69, 56 free 66, 44 free 63,
        # 32 free 60 -- the mapping network is the critical path there, the chain (28 -> 35 ms) is not
        sizes = [int(v) for v in os.environ.get("GANSPACE_B200_RNG_GROUPS", "4,7").split(",")]
        bounds, g0 = [], 0
        while g0 < S:
            g1 = min(S, g0 + sizes[min(len(bounds), len(sizes) - 1)])
            bounds.append((g0, g1))
            g0 = g1
        side = getattr(self, "_rng_stream", None)
        if side is None:
            with torch.cuda.device(self.device):
                side = self._rng_stream = torch.cuda.Stream(device=self.device)
        events = []
        seeds_dev = _native.seeds_tensor(list(seeds), self.device)       # ONE host->device copy, before any long kernel is queued
        # the first group decides when the first partial_fit statistics exist (the merge chain, the critical path of a small-d
        # run, waits for them): its streams are split over twice as many CTAs (GANSPACE_B200_RNG_FIRST_PARTS)
        parts0 = parts
        if parts > 1:
            parts0 = max(parts, min(16, int(os.environ.get("GANSPACE_B200_RNG_FIRST_PARTS", 2 * parts))))
            _native.jump_polys(512 * n_samples, parts, self.device)     # (first use: host computation + upload)
            _native.jump_polys(512 * n_samples, parts0, self.device)
            # one scratch buffer for the largest group, so that no launch re-allocates it while an earlier one is running
            gmax = max(b - a for a, b in bounds)
            wsb = _native.load().gsb_legacy_normal_split_workspace_bytes
            need = max(wsb(gmax, 512 * n_samples, parts), wsb(bounds[0][1] - bounds[0][0], 512 * n_samples, parts0))
            _native.scratch.get("rng_split_lazy", need, _native.require_cuda(self.device)).record_stream(side)
        with torch.cuda.device(self.device):
            side.wait_stream(torch.cuda.current_stream())
            with torch.cuda.stream(side):
                for gi, (a, b) in enumerate(bounds):
                    _native.legacy_normal(seeds_dev[a:b], 512 * n_samples, self.device,
                                          out=z[a * n_samples:b * n_samples].view(b - a, 512 * n_samples),
                                          parts=parts0 if gi == 0 else parts, scratch_key="rng_split_lazy")
                    ev = torch.cuda.Event()
                    ev.record(side)
                    events.append(ev)
            z.record_stream(side)
            seeds_dev.record_stream(side)          # read by launches that run long after this function has returned
        packed = self.model.style.packed() if self.w_primary else None
        state = {"g": 0, "keep": seeds_dev}
        free_sms = int(os.environ.get("GANSPACE_B200_LAZY_FREE_SMS", 32 if parts > 1 else 48))

        def ensure(row_end):
            # later groups run next to the IPCA chain and leave a GPC's worth of SMs to it
            while state["g"] < len(bounds) and bounds[state["g"]][0] * n_samples < row_end:
                g = state["g"]
                a, b = bounds[g][0] * n_samples, bounds[g][1] * n_samples
                torch.cuda.current_stream().wait_event(events[g])
                if packed is not None:
                    packed.forward(z[a:b], out=z[a:b], leave_free_sms=0 if g == 0 else free_sms)
                state["g"] = g + 1
        return z, ensure

    def check_numerics(self):
        """Raise if a kernel flagged an out-of-range activation since the weights were packed (synchronises)."""
        self.model.style.packed().check()
        if self._synth.current() is not None:
            self._synth.current().check()

    def get_max_latents(self):
        return self.model.n_latent

    # ---- the fused chain conv1, to_rgb1, convs.0, convs.1, to_rgbs.0, ... (wrappers.py:188-255) ------------------------
    def _chain_outputs(self):
        """StyledConv l runs as (l + 1, 0); ToRGB j, which follows StyledConv 2j, as (2j + 1, j + 1)."""
        convs, rgbs = self.model.chain_layers()
        out = []
        for l, (name, _) in enumerate(convs):
            out.append((name, l + 1, 0))
            if l % 2 == 0:
                out.append((rgbs[l // 2][0], l + 1, l // 2 + 1))
        return out

    def _style_layers(self):
        """The modulation layer of each chain output, in the order of ``Generator.style_layers()``."""
        return [(f"{name}.conv.modulation", n_run, n_rgb) for name, n_run, n_rgb in self._chain_outputs()]

    def _image_run(self):
        return len(self.model.convs) + 1, len(self.model.to_rgbs) + 1

    def _stops_before_chain(self, layer_name, ws):
        if "style" in layer_name:
            # (the reference builds the [N, n_latent, 512] repeat + StridedStyle stack before this early exit, wrappers.py:202-222 --
            # 328 MB of traffic per 10k batch that nothing reads; skipped here)
            return True
        if layer_name == "input":
            self.model.input(self.model.latents_per_layer(ws)[:, 0])
            return True
        return False

    def _w_layers(self, ws, truncate):
        """One latent, a pair (style mixing at a random index, as the reference) or one latent per layer; ``forward`` truncates."""
        if truncate and self.truncation < 1:
            ws = [self.latent_avg + self.truncation * (s - self.latent_avg) for s in ws]       # model.py:511-552
        if len(ws) == 1 and ws[0].dim() < 3:
            return ws[0].reshape(1, -1, 512)
        return self.model.latents_per_layer(ws).permute(1, 0, 2).contiguous()

    def _unhookable_message(self, name):
        return (f"StyleGAN2: a hook on '{name}' is not supported: the StyledConv and ToRGB layers run as one fused chain; the "
                "hookable synthesis layers are conv1, convs.k, to_rgb1, to_rgbs.j and their style layers '<layer>.conv.modulation'")

    def _stop(self, layer_name):
        """The StyledConv or ToRGB named, or the one that contains the style layer named (wrappers.py:228-255)."""
        base = layer_name[:-len(".conv.modulation")] if layer_name.endswith(".conv.modulation") else layer_name
        names = [o[0] for o in self._chain_outputs()]
        if base not in names:
            raise RuntimeError(f"Unknown layer '{layer_name}'")
        return names.index(base)

    def synthesis_layer_names(self):
        return ["conv1"] + [f"convs.{i}" for i in range(len(self.model.convs))]

    def _chain(self, n_run):
        return self._synthesis(n_run)

    def _synthesis(self, n_run):
        """PackedSynthesis covering at least the first ``n_run`` StyledConv layers and the ToRGBs that follow them.  A pack of more
        layers serves as long as the constant and the parameters and noise maps of these layers and ToRGBs are the ones it was
        packed from."""
        mods = [self.model.conv1] + list(self.model.convs)
        rgbs = [self.model.to_rgb1] + list(self.model.to_rgbs)
        rgb_params = lambda r: [r.conv.weight, r.conv.modulation.weight, r.conv.modulation.bias, r.bias]
        keys = (_native.source_key([self.model.input.input]),) + tuple(
            _native.source_key([m.conv.weight, m.conv.modulation.weight, m.conv.modulation.bias, m.noise.weight, m.activate.bias,
                                self.noise[i]] + (rgb_params(rgbs[i // 2]) if i % 2 == 0 else []))
            for i, m in enumerate(mods[:n_run]))
        if self._synth_keys[:len(keys)] != keys:
            self._synth_keys = keys               # a stale or too short pack: the get() below packs n_run layers

        def build():
            layers, res = [], 4
            for i, m in enumerate(mods[:n_run]):
                layers.append(m.describe(self.noise[i], res))
                res = 2 * res if m.conv.upsample else res
            return _native.PackedSynthesis(self.model.input.input.detach()[0], layers,
                                           [r.describe() for r in rgbs[:(n_run + 1) // 2]], self.model.style_dim)
        return self._synth.get([], build, self._synth_keys)

    def feature_layout(self, layer_name):
        names = self.synthesis_layer_names()
        if layer_name not in names:
            return None
        i = names.index(layer_name)
        return self._nhwc_layout(layer_name, *self._synthesis(i + 1).shapes[i])

    def activations_into(self, x, layer_name, out):
        """Hooked-layer activations of latents x [n,512] (in the current primary space) written as fp32 NHWC rows into
        ``out`` [n, H*W*C] (may be row-strided): the decomposition driver's producer for conv layers."""
        names = self.synthesis_layer_names()
        n_run = names.index(layer_name) + 1
        w = (x if self.w_primary else self.model.style(x)).reshape(-1, 512)
        synth = self._synthesis(n_run)
        step = synth.rows_within(n_run, w.shape[0], self.SYNTH_WORKSPACE_BUDGET)
        if step >= w.shape[0]:
            return synth.forward(w, n_run, out=out)[0]
        # every kernel of the chain treats each sample on its own, so slices of rows give the bits of one call
        if out is None:
            out = torch.empty((w.shape[0], synth.out_dims(n_run)), dtype=torch.float32, device=self.device)
        for r0 in range(0, w.shape[0], step):
            synth.forward(w[r0:r0 + step], n_run, out=out[r0:r0 + step])
        return out

    def activations_workspace_bytes(self, layer_name, n):
        """Device scratch that ``activations_into`` of ``n`` rows to ``layer_name`` allocates (at most SYNTH_WORKSPACE_BUDGET)."""
        n_run = self.synthesis_layer_names().index(layer_name) + 1
        synth = self._synthesis(n_run)
        return synth.workspace_bytes(n_run, synth.rows_within(n_run, n, self.SYNTH_WORKSPACE_BUDGET))

    def set_noise_seed(self, seed):
        # same generator stream as the reference (torch.manual_seed(seed); torch.randn per noise map),
        # drawn on the host so that it does not depend on the device RNG implementation
        torch.manual_seed(seed)
        self.noise = [torch.randn(1, 1, 2 ** 2, 2 ** 2).to(self.device)]
        for i in range(3, self.model.log_size + 1):
            for _ in range(2):
                self.noise.append(torch.randn(1, 1, 2 ** i, 2 ** i).to(self.device))


class ProGAN(_DeviceGenerator):
    """wrappers.py:469-522 on the fused chain of csrc/progan.cu.  Z space only; hookable layers are the blocks
    ``layer1 .. layer14`` and ``output_256x256``.  Checkpoint: ``$GANCONTROL_CHECKPOINT_DIR/progan/<class>_lsun.pth`` (there is no
    network to download it); without one, ``random_init=<seed>`` (or env GANSPACE_B200_RANDOM_INIT) builds
    ``progan.random_init(seed)``."""

    CLASSES = ["bedroom", "churchoutdoor", "conferenceroom", "diningroom", "kitchen", "livingroom", "restaurant"]
    # deepest feature map get_or_compute decomposes (layer10, 128 x 64 x 64): the large-d engine's stacked matrix takes
    # (components + max(B, 2000, 3 components) + 1) x d x 4 bytes -- 4.4 GB there, 17.5 GB at layer13/14 with its fp16 operand
    # copies on top -- and has been run up to this size only
    MAX_DECOMPOSITION_DIMS = 524_288

    def __init__(self, device, lsun_class=None, random_init=None):
        super().__init__("ProGAN", lsun_class)
        self.device = _native.require_cuda(device)
        assert self.outclass in self.CLASSES, f"Invalid LSUN class {self.outclass}, should be one of {self.CLASSES}"
        self._random_init = random_init
        self.load_model()
        self.name = f"ProGAN-{self.outclass}"
        self.has_latent_residual = False

    def load_model(self):
        from . import progan
        source = self._weight_source(_checkpoint(f"progan/{self.outclass}_lsun.pth"))
        if isinstance(source, int):
            self.model = progan.random_init(source).to(self.device)
        else:
            self.model = progan.from_state_dict(torch.load(source, map_location="cpu")).to(self.device)
        self.z_dim = self.model.layer1.conv.in_channels
        self._latent_shape = (1, self.z_dim, 1, 1)

    def sample_latent(self, n_samples=1, seed=None, truncation=None):
        """zdataset.py:26-40: ``RandomState(seed).standard_normal(n * z_dim)`` as float32 [n, z_dim, 1, 1], drawn on the device."""
        if seed is None:
            seed = _global_seed()
        return _native.legacy_normal([seed], self.z_dim * n_samples, self.device).view(n_samples, self.z_dim, 1, 1)

    def sample_latents_multi(self, n_samples, seeds, out=None):
        """Several ``sample_latent(n_samples, seed=s)`` calls in one launch (the decomposition driver's producer)."""
        z = _native.legacy_normal(list(seeds), self.z_dim * n_samples, self.device,
                                  out=None if out is None else out.view(len(seeds), self.z_dim * n_samples),
                                  parts=_native.split_parts(self.z_dim * n_samples))
        return z.view(len(seeds) * n_samples, self.z_dim, 1, 1)

    def check_numerics(self):
        """Raise if a kernel flagged an out-of-range operand since the weights were packed (synchronises)."""
        self.model.packed().check()

    @staticmethod
    def _single(x):
        if isinstance(x, list):
            assert len(x) == 1, "ProGAN only supports a single global latent"
            x = x[0]
        return x.reshape(x.shape[0], -1).float()

    def _run(self, x, target, want_rgb):
        """The chain up to block ``target`` (index into layer1 .. layerK; K = the output block, which needs ``want_rgb``) with the
        forward hooks of every block on the way: a hooked earlier block gets its own run of the chain."""
        z = self._single(x)
        names = self.model.block_names()
        mods = list(self.model._modules.values())
        packed = self.model.packed()
        n_conv = len(mods) - 1
        last = min(target, n_conv - 1)
        for i in [i for i in range(last) if len(mods[i]._forward_hooks)]:
            self._hand_off(mods[i], packed.forward(z, i + 1)[0], *packed.shapes[i], i < target, names[i])
        want_act = len(mods[last]._forward_hooks) > 0 or not want_rgb
        act, rgb = packed.forward(z, last + 1, want_act=want_act, want_rgb=want_rgb)
        if want_act:
            self._hand_off(mods[last], act, *packed.shapes[last], last < target, names[last])
        if want_rgb:
            return mods[n_conv](_result=rgb.permute(0, 3, 1, 2))
        return None

    def forward(self, x):
        return 0.5 * (self._run(x, len(self.model) - 1, True) + 1)

    def partial_forward(self, x, layer_name):
        names = self.model.block_names()
        if layer_name not in names:
            raise RuntimeError(f"Layer {layer_name} not encountered in partial_forward")
        target = names.index(layer_name)
        self._run(x, target, want_rgb=(target == len(names) - 1))

    def feature_layout(self, layer_name):
        names = self.model.block_names()
        if layer_name not in names[:-1]:
            return None
        return self._nhwc_layout(layer_name, *self.model.packed().shapes[names.index(layer_name)])

    def activations_into(self, x, layer_name, out):
        """Activations of block ``layer_name`` for latents x [n, z_dim(,1,1)] written as fp32 NHWC rows into ``out`` [n, H*W*C]
        (may be row-strided): the decomposition driver's producer."""
        n_run = self.model.block_names().index(layer_name) + 1
        return self.model.packed().forward(self._single(x), n_run, out=out)[0]


class StyleGAN(_StyledGenerator):
    """wrappers.py:270-436 (StyleGAN v1).  ``g_mapping`` runs the packed mapping kernels, the synthesis blocks the fused chain of
    csrc/stylegan.cu.  Hookable layers: ``g_mapping``, the blocks ``g_synthesis.blocks.RxR`` and their style layers
    ``g_synthesis.blocks.RxR.epi{1,2}.style_mod.lin`` (the StyleMod rows [n, 2C], which an edit replaces).  Checkpoint:
    ``$GANCONTROL_CHECKPOINT_DIR/stylegan/stylegan_<class>_<res>.pt`` (the reference's ``StyleGAN_G`` state dict; there is no network
    to download it and no TensorFlow to convert a ``.pkl``); without one, ``random_init=<seed>`` (or env GANSPACE_B200_RANDOM_INIT)
    builds ``stylegan.random_init(seed)``."""

    _MAPPING_LAYER = "g_mapping"
    CONFIGS = {"ffhq": 1024, "celebahq": 1024, "bedrooms": 256, "cars": 512, "cats": 256, "vases": 1024, "wikiart": 512,
               "fireworks": 512, "abstract": 512, "anime": 512, "ukiyo-e": 512}
    # deepest feature map get_or_compute decomposes (blocks.32x32, 512 x 32 x 32), the bound ProGAN uses: the large-d engine's
    # stacked matrix takes (components + max(B, 2000, 3 components) + 1) x d x 4 bytes in HBM
    MAX_DECOMPOSITION_DIMS = 524_288

    def __init__(self, device, class_name, truncation=1.0, use_w=False, random_init=None):
        super().__init__("StyleGAN", class_name or "ffhq")
        assert self.outclass in self.CONFIGS, \
            f'Invalid StyleGAN class {self.outclass}, should be one of [{", ".join(self.CONFIGS.keys())}]'
        self.device = _native.require_cuda(device)
        self.w_primary = use_w
        self.resolution = self.CONFIGS[self.outclass]
        self.name = f"StyleGAN-{self.outclass}"
        self.has_latent_residual = True
        self._random_init = random_init
        self.load_model()
        self.set_noise_seed(0)

    def load_model(self):
        from . import stylegan
        checkpoint = _checkpoint(f"stylegan/stylegan_{self.outclass}_{self.resolution}.pt")
        try:
            source = self._weight_source(checkpoint)
        except RuntimeError:
            if checkpoint.with_suffix(".pkl").is_file():
                raise RuntimeError(f"StyleGAN: {checkpoint.with_suffix('.pkl')} is a TensorFlow checkpoint; converting it needs "
                                   "TensorFlow (the reference's StyleGAN_G.export_from_tf), which is not part of this package: "
                                   f"convert it to {checkpoint}") from None
            raise
        if isinstance(source, int):
            self.model = stylegan.random_init(source, self.resolution).to(self.device)
        else:
            self.model = stylegan.StyleGAN_G(self.resolution)
            self.model.load_state_dict(torch.load(source, map_location="cpu"))
            self.model = self.model.to(self.device)

    def get_max_latents(self):
        return 18

    def set_noise_seed(self, seed):
        """wrappers.py:419-434: every NoiseLayer gets ``torch.randn(1, 1, H, W)`` right after ``manual_seed(seed)`` (so all maps of
        one resolution are equal), drawn on the host and then moved to the device."""
        for name, m in self.model.g_synthesis.named_modules(prefix="g_synthesis"):
            if type(m).__name__ == "NoiseLayer":
                H, W = [int(s) for s in name.split(".")[2].split("x")]
                torch.random.manual_seed(seed)
                m.noise = torch.randn(1, 1, H, W, dtype=torch.float32).to(self.device)

    # ---- latents ----------------------------------------------------------------------------------------
    def _mapping(self):
        return self.model.g_mapping

    def z_to_latent(self, z):
        return self.model.g_mapping.packed().forward(z) if self.w_primary else z

    def sample_latents_multi(self, n_samples, seeds, out=None, lazy=False):
        """Several ``sample_latent(n_samples, seed=s)`` calls in one RNG launch (the decomposition driver's producer); no hooks fire.
        ``lazy=True``: returns (latents, ensure) where ``ensure(row_end)`` maps rows [0, row_end) to W in place (W mode)."""
        S = len(seeds)
        z = _native.legacy_normal(list(seeds), 512 * n_samples, self.device,
                                  out=None if out is None else out.view(S, 512 * n_samples),
                                  parts=_native.split_parts(512 * n_samples)).view(S * n_samples, 512)
        packed = self.model.g_mapping.packed() if self.w_primary else None
        if not lazy:
            return z if packed is None else packed.forward(z, out=z)
        state = {"done": 0}

        def ensure(row_end):
            a, b = state["done"], min(row_end, z.shape[0])
            if packed is not None and b > a:
                packed.forward(z[a:b], out=z[a:b])
            state["done"] = max(a, b)
        return z, ensure

    def check_numerics(self):
        """Raise if a kernel flagged an out-of-range operand since the weights were packed (synchronises)."""
        self.model.g_mapping.packed().check()
        if self.model.g_synthesis.pack_cache.current() is not None:
            self.model.g_synthesis.pack_cache.current().check()

    # ---- the fused chain: two layers per block, torgb after the last ----------------------------------------------------------
    def _chain_outputs(self):
        """Block i ends the run of its two layers."""
        return [(name, 2 * (i + 1), 0) for i, name in enumerate(self.model.block_names())]

    def _style_layers(self):
        """Style layer l is reached by the run of chain layers 0 .. l."""
        return [(t[0], t[1] + 1, 0) for t in self.model.style_layers()]

    def _image_run(self):
        return 2 * len(self.model.g_synthesis.blocks), 1

    def _chain(self, n_run):
        return self.model.g_synthesis.packed()

    def _stops_before_chain(self, layer_name, ws):
        return "g_mapping" in layer_name or layer_name == "truncation"

    def _w_layers(self, ws, truncate):
        """[18, n, 512] per-layer dlatents (wrappers.py:382-387 / model.py:382-393) from a list of 18, else [1, n, 512]."""
        if len(ws) == 1:
            return ws[0].reshape(1, -1, 512).float()
        assert len(ws) == 18, "Must provide 1 or 18 latents"
        return torch.stack([w.reshape(-1, 512).float() for w in ws])

    def _unhookable_message(self, name):
        return (f"StyleGAN: a hook on '{name}' is not supported: g_mapping and the synthesis blocks run as fused kernels; the "
                f"hookable layers are {', '.join(self._hookable())}")

    def _hookable(self):
        return self.model.hookable_layers()

    def _stop(self, layer_name):
        """The reference's stop rule (wrappers.py:394-417): the first block one of whose leaf modules' names contains ``layer_name``."""
        for i, (n, blk) in enumerate(self.model.g_synthesis.blocks.items()):
            leaves = [f"g_synthesis.blocks.{n}.{c}" for c, m in blk.named_modules(remove_duplicate=False) if c and not m._modules]
            if any(layer_name in c for c in leaves):
                return i
        raise RuntimeError(f"Layer {layer_name} not encountered in partial_forward")

    def feature_layout(self, layer_name):
        names = self.model.block_names()
        if layer_name not in names:
            return None
        return self._nhwc_layout(layer_name, *self.model.g_synthesis.packed().shapes[2 * names.index(layer_name) + 1])

    def activations_into(self, x, layer_name, out):
        """Output of block ``layer_name`` for latents x [n, 512] (in the current primary space) written as fp32 NHWC rows into
        ``out`` [n, H*W*C] (may be row-strided): the decomposition driver's producer."""
        n_run = 2 * (self.model.block_names().index(layer_name) + 1)
        x = x.reshape(-1, 512)
        w = x if self.w_primary else self.model.g_mapping.packed().forward(x)
        return self.model.g_synthesis.packed().forward(w, n_run, out=out)[0]


# ---- factories (wrappers.py:651-735) ---------------------------------------------------------------
@singledispatch
def get_model(name, output_class, device, **kwargs):
    inst = kwargs.get("inst", None)
    model = kwargs.get("model", None)
    if inst or model:
        cached = model or inst.model
        network_same = cached.model_name == name
        outclass_same = cached.outclass == output_class
        can_change_class = "BigGAN" in name
        if network_same and (outclass_same or can_change_class):
            cached.set_output_class(output_class)
            return cached
    if name == "StyleGAN2":
        model = StyleGAN2(device, class_name=output_class, random_init=kwargs.get("random_init"))
    elif "BigGAN" in name:
        assert "-" in name, "Please specify BigGAN resolution, e.g. BigGAN-512"
        from .biggan import BigGAN
        model = BigGAN(device, name.split("-")[-1], class_name=output_class, random_init=kwargs.get("random_init"))
    elif name == "ProGAN":
        model = ProGAN(device, lsun_class=output_class, random_init=kwargs.get("random_init"))
    elif name == "StyleGAN":
        model = StyleGAN(device, class_name=output_class, random_init=kwargs.get("random_init"))
    elif name == "DCGAN":
        raise RuntimeError(f"{name} is outside the GPU hot path (SURVEY.md section 2: not in any BASELINE config)")
    else:
        raise RuntimeError(f"Unknown model {name}")
    return model


@get_model.register(Config)
def _(cfg, device, **kwargs):
    kwargs["use_w"] = kwargs.get("use_w", cfg.use_w)
    return get_model(cfg.model, cfg.output_class, device, **kwargs)


def _annotate_shapes(inst, model, layers):
    """The reference runs one full forward on zeros to record shapes (modelconfig.py:110-144).  Only the
    hooked layers' shapes and the latent shape are consumed by GANSpace, so a partial forward suffices."""
    input_shape = model.get_latent_shape()
    inst.retain_layers(layers)
    with torch.no_grad():
        dry = torch.zeros(input_shape, device=model.device)
        for layer in layers:
            model.partial_forward(dry, layer)
    inst.input_shape = input_shape
    inst.feature_shape = {layer: feat.shape for layer, feat in inst.retained_features().items()}
    inst.output_shape = None   # full image synthesis: SURVEY.md section 8(f) item 2
    return inst


@singledispatch
def get_instrumented_model(name, output_class, layers, device, **kwargs):
    model = get_model(name, output_class, device, **kwargs)
    model.eval()
    inst = kwargs.get("inst", None)
    if inst:
        inst.close()
    if not isinstance(layers, list):
        layers = [layers]
    module_names = [n for (n, _) in model.named_modules()]
    for layer_name in layers:
        if layer_name not in module_names:
            print(f"Layer '{layer_name}' not found in model!")
            print("Available layers:", "\n".join(module_names))
            raise RuntimeError(f"Unknown layer '{layer_name}''")
    if hasattr(model, "use_z"):
        model.use_z()
    inst = InstrumentedModel(model)
    try:
        _annotate_shapes(inst, model, layers)
    except Exception:
        inst.close()                # a refused layer leaves no hook behind on the (cached) model
        raise
    if kwargs.get("use_w", False):
        model.use_w()
    return inst


@get_instrumented_model.register(Config)
def _(cfg, device, **kwargs):
    kwargs["use_w"] = kwargs.get("use_w", cfg.use_w)
    return get_instrumented_model(cfg.model, cfg.output_class, cfg.layer, device, **kwargs)
