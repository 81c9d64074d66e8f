"""ctypes binding of the C-ABI shared library (include/ganspace_b200.h).

There is no CPU fallback: if the library is missing, or a compute entry point is called without a CUDA
device, this module raises.  torch is used only for device memory and streams.
"""
from __future__ import annotations

import contextlib
import ctypes as C
import os
from pathlib import Path

import torch

_LIB_PATH = Path(__file__).resolve().parent / "libganspace_b200.so"
_lib = None

# name -> (restype, argtypes); mirrors include/ganspace_b200.h one to one
_P, _I, _L, _Z, _D, _F = C.c_void_p, C.c_int, C.c_int64, C.c_size_t, C.c_double, C.c_float
SIGNATURES = {
    "gsb_abi_version": (_I, []),
    "gsb_last_error": (C.c_char_p, []),
    "gsb_state_layout_version": (_I, [_I]),
    "gsb_legacy_normal_f32": (_I, [_P, _I, _L, _P, _L, _P]),
    "gsb_legacy_truncnorm_f32": (_I, [_P, _I, _L, _D, _D, _F, _P, _L, _P]),
    "gsb_mt19937_raw_u32": (_I, [_P, _I, _L, _P, _L, _P]),
    "gsb_mt19937_jump_polys": (_I, [_L, _I, _P]),
    "gsb_mt19937_jump_state_host": (_I, [C.c_uint32, _P, _P]),
    "gsb_legacy_normal_split_step_words": (_L, [_L, _I]),
    "gsb_legacy_normal_split_workspace_bytes": (_Z, [_I, _L, _I]),
    "gsb_legacy_normal_f32_split": (_I, [_P, _I, _L, _P, _L, _I, _P, _P, _Z, _P]),
    "gsb_legacy_normal_split_status": (_I, [_P, _I, _L, _I, _P, _P]),
    "gsb_mapping_packed_bytes": (_Z, [_I, _I]),
    "gsb_mapping_pack": (_I, [_P, _P, _I, _I, _F, _P, _P]),
    "gsb_mapping_workspace_bytes": (_Z, [_L, _I]),
    "gsb_mapping_forward": (_I, [_P, _I, _I, _P, _P, _L, _I, _P, _Z, _P]),
    "gsb_mapping_status": (_I, [_P, _I, _I, _P]),
    "gsb_linear_forward": (_I, [_P, _P, _P, _P, _L, _I, _I, _I, _P, _Z, _P]),
    "gsb_linear_workspace_bytes": (_Z, [_L, _I, _I, _I]),
    "gsb_batch_stats_workspace_bytes": (_Z, [_L, _I]),
    "gsb_batch_stats": (_I, [_P, _L, _I, _L, _P, _P, _P, _Z, _P]),
    "gsb_batch_stats_multi_workspace_bytes": (_Z, [_I, _L, _I]),
    "gsb_batch_stats_multi": (_I, [_P, _I, _L, _I, _L, _P, _P, _P, _Z, _P]),
    "gsb_batch_stats_grouped_workspace_bytes": (_Z, [_P, _I]),
    "gsb_batch_stats_grouped": (_I, [_P, _I, _P, _Z, _P]),
    "gsb_ipca_state_bytes": (_Z, [_I, _I]),
    "gsb_ipca_workspace_bytes": (_Z, [_I, _I]),
    "gsb_ipca_reset": (_I, [_P, _I, _I, _P]),
    "gsb_ipca_chain_step": (_I, [_P, _I, _I, _L, _L, _P, _P, _P, _Z, _P]),
    "gsb_ipca_export": (_I, [_P, _I, _I, _L, _P, _P, _P, _P, _P, _P, _P]),
    "gsb_sym_eig_top": (_I, [_P, _I, _I, _P, _P, _P, _Z, _P]),
    "gsb_eig_status": (_I, [_P, _P]),
    "gsb_project_std_workspace_bytes": (_Z, [_I]),
    "gsb_project_std": (_I, [_P, _L, _I, _L, _P, _I, _P, _P, _P, _Z, _P]),
    "gsb_linreg_state_bytes": (_Z, [_I, _I]),
    "gsb_linreg_reset": (_I, [_P, _I, _I, _P]),
    "gsb_linreg_feature_splits": (_I, [_L, _I, _I]),
    "gsb_linreg_workspace_bytes": (_Z, [_L, _I, _I]),
    "gsb_linreg_accumulate": (_I, [_P, _I, _I, _P, _L, _I, _P, _P, _P, _P, _P, _Z, _P]),
    "gsb_linreg_solve": (_I, [_P, _I, _I, _L, _P, _P, _P]),
    "gsb_linreg_solve_status": (_I, [_P, _I, _I, _P, _P]),
    "gsb_linreg_normal_matrix": (_P, [_P, _I, _I]),
    "gsb_linreg_solve_pinv": (_I, [_P, _I, _I, _P, _P, _D, _P, _P]),
    "gsb_ipca_set_chain_mode": (_I, [_I]),
    "gsb_synthesis_packed_bytes": (_Z, [_P, _I, _I]),
    "gsb_synthesis_pack": (_I, [_P, _I, _I, _P, _P, _P, _Z, _P]),
    "gsb_synthesis_workspace_bytes": (_Z, [_P, _I, _I, _L]),
    "gsb_synthesis_forward": (_I, [_P, _P, _I, _I, _I, _I, _P, _I, _L, _P, _L, _P, _P, _Z, _P]),
    "gsb_synthesis_status": (_I, [_P, _P, _I, _I, _P]),
    "gsb_synthesis_styles": (_I, [_P, _P, _I, _I, _P, _I, _L, _P, _P, _P]),
    "gsb_synthesis_forward_styled_workspace_bytes": (_Z, [_P, _I, _I, _L]),
    "gsb_synthesis_forward_styled": (_I, [_P, _P, _I, _I, _I, _I, _P, _P, _L, _P, _L, _P, _P, _Z, _P]),
    "gsb_progan_packed_bytes": (_Z, [_P, _I]),
    "gsb_progan_pack": (_I, [_P, _I, _P, _P, _P, _Z, _P]),
    "gsb_progan_workspace_bytes": (_Z, [_P, _I, _L]),
    "gsb_progan_forward": (_I, [_P, _P, _I, _I, _P, _L, _P, _L, _P, _P, _Z, _P]),
    "gsb_progan_status": (_I, [_P, _P, _I, _P]),
    "gsb_stylegan_packed_bytes": (_Z, [_P, _I, _I]),
    "gsb_stylegan_pack": (_I, [_P, _I, _I, _P, _P, _P, _P, _Z, _P]),
    "gsb_stylegan_workspace_bytes": (_Z, [_P, _I, _L]),
    "gsb_stylegan_forward": (_I, [_P, _P, _I, _I, _I, _P, _I, _L, _P, _L, _P, _P, _Z, _P]),
    "gsb_stylegan_status": (_I, [_P, _P, _I, _I, _P]),
    "gsb_stylegan_styles": (_I, [_P, _P, _I, _I, _P, _I, _L, _P, _I, _P, _P]),
    "gsb_stylegan_forward_styled_workspace_bytes": (_Z, [_P, _I, _L]),
    "gsb_stylegan_forward_styled": (_I, [_P, _P, _I, _I, _I, _P, _L, _P, _L, _P, _P, _Z, _P]),
    "gsb_biggan_conv_forward": (_I, [_P, _L, _P]),
    "gsb_biggan_bn_table": (_I, [_P, _L, _I, _P, _P, _P, _F, _I, _P, _P, _P]),
    "gsb_biggan_bn_rows": (_I, [_P, _L, _I, _P, _I, _P]),
    "gsb_biggan_bn_table_rows": (_I, [_P, _L, _P, _L, _L, _P, _F, _I, _P, _P, _P]),
    "gsb_biggan_attn_pool": (_I, [_P, _L, _I, _I, _P, _P, _P]),
    "gsb_biggan_softmax_rows": (_I, [_P, _L, _I, _P]),
    "gsb_biggan_rgb": (_I, [_P, _L, _I, _I, _P, _P, _P, _P, _P, _P, _P]),
    "gsb_bigd_rows": (_I, [_I, _I]),
    "gsb_bigd_state_bytes": (_Z, [_L, _I]),
    "gsb_bigd_workspace_bytes": (_Z, [_L, _I, _I, _I]),
    "gsb_bigd_reset": (_I, [_P, _P, _L, _I, _I, _P]),
    "gsb_bigd_chain_step": (_I, [_P, _P, _L, _I, _I, _L, _I, _I, _P, _P, _Z, _P]),
    "gsb_bigd_export": (_I, [_P, _P, _L, _I, _L, _P, _P, _P, _P, _P, _P, _P]),
    "gsb_bigd_gram_matrix": (_P, [_P, _L, _I, _I]),
    "gsb_bigd_step_gram": (_I, [_P, _P, _L, _I, _I, _L, _I, _I, _P, _P, _Z, _P]),
    "gsb_bigd_step_solve": (_I, [_P, _P, _L, _I, _I, _L, _I, _I, _P, _P, _Z, _P]),
    "gsb_bigd_step_commit": (_I, [_P, _P, _L, _I, _I, _L, _I, _I, _P, _P, _Z, _P]),
    "gsb_nhwc_to_nchw_rows": (_I, [_P, _L, _P, _L, _L, _I, _I, _I, _P]),
    "gsb_fbpca_state_bytes": (_Z, [_I]),
    "gsb_fbpca_reset": (_I, [_P, _I, _P]),
    "gsb_fbpca_accumulate": (_I, [_P, _I, _I, _L, _P, _P, _P]),
    "gsb_fbpca_add_zero_rows": (_I, [_P, _I, _L, _P]),
    "gsb_fbpca_workspace_bytes": (_Z, [_I, _I, _I]),
    "gsb_fbpca_solve": (_I, [_P, _I, _I, _I, _I, _P, _P, _P, _P, _P, _P, _Z, _P]),
    "gsb_fbpca_status": (_I, [_P, _I, _P, _P]),
    "gsb_fbpca_project_omega": (_I, [_P, _I, _I, _P, _I, _P, _P]),
}


class StatsDesc(C.Structure):
    """``gsb_stats_desc`` of include/ganspace_b200.h."""
    _fields_ = [("x", C.c_void_p), ("ld", C.c_int64), ("d", C.c_int), ("n_groups", C.c_int), ("rows_per_group", C.c_int64),
                ("mean_out", C.c_void_p), ("gram_out", C.c_void_p)]


class StyledConvDesc(C.Structure):
    """``gsb_styled_conv`` of include/ganspace_b200.h (device pointers to the module's fp32 parameters)."""
    _fields_ = [("conv_weight", C.c_void_p), ("mod_weight", C.c_void_p), ("mod_bias", C.c_void_p),
                ("act_bias", C.c_void_p), ("noise", C.c_void_p), ("noise_weight", C.c_void_p),
                ("cin", C.c_int), ("cout", C.c_int), ("upsample", C.c_int), ("res_in", C.c_int)]


class ToRGBDesc(C.Structure):
    """``gsb_to_rgb`` of include/ganspace_b200.h."""
    _fields_ = [("conv_weight", C.c_void_p), ("mod_weight", C.c_void_p), ("mod_bias", C.c_void_p), ("bias", C.c_void_p),
                ("cin", C.c_int)]


class ProGANBlockDesc(C.Structure):
    """``gsb_progan_block`` of include/ganspace_b200.h."""
    _fields_ = [("conv_weight", C.c_void_p), ("bias", C.c_void_p), ("cin", C.c_int), ("cout", C.c_int), ("upsample", C.c_int),
                ("res_in", C.c_int), ("ksize", C.c_int)]


class StyleGANLayerDesc(C.Structure):
    """``gsb_stylegan_layer`` of include/ganspace_b200.h."""
    _fields_ = [("conv_weight", C.c_void_p), ("bias", C.c_void_p), ("noise", C.c_void_p), ("noise_weight", C.c_void_p),
                ("style_weight", C.c_void_p), ("style_bias", C.c_void_p), ("cin", C.c_int), ("cout", C.c_int), ("upsample", C.c_int),
                ("res_out", C.c_int)]


class BigGANConvDesc(C.Structure):
    """``gsb_biggan_conv`` of include/ganspace_b200.h."""
    _fields_ = [("x", C.c_void_p), ("ldx", C.c_int64), ("cin", C.c_int), ("res_in", C.c_int), ("upsample", C.c_int),
                ("ksize", C.c_int), ("bn_mean", C.c_void_p), ("bn_scale", C.c_void_p), ("bn_offset", C.c_void_p),
                ("weight", C.c_void_p), ("w_sample_stride", C.c_int64), ("cout", C.c_int), ("bias", C.c_void_p),
                ("alpha", C.c_float), ("res", C.c_void_p), ("ldres", C.c_int64), ("res_upsample", C.c_int), ("out", C.c_void_p),
                ("ldo", C.c_int64)]


class BigGANBnRowsDesc(C.Structure):
    """``gsb_biggan_bn_rows_desc`` of include/ganspace_b200.h."""
    _fields_ = [("w_scale", C.c_void_p), ("w_offset", C.c_void_p), ("c", C.c_int), ("scale_rows", C.c_void_p),
                ("offset_rows", C.c_void_p)]


class NativeError(RuntimeError):
    pass


def lib_path() -> Path:
    return _LIB_PATH


def load():
    """Load libganspace_b200.so (built in-tree by ``__graft_entry__.build()`` / csrc/Makefile)."""
    global _lib
    if _lib is None:
        if not _LIB_PATH.exists():
            raise NativeError(
                f"{_LIB_PATH} not found: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
                "(nvcc, sm_90a). ganspace_b200 has no CPU fallback.")
        lib = C.CDLL(str(_LIB_PATH))
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(lib, name)          # AttributeError if the header and the library drift apart
            fn.restype, fn.argtypes = res, args
        if lib.gsb_abi_version() != 2:
            raise NativeError("ABI version mismatch between ganspace_b200/_native.py and the library")
        _lib = lib
    return _lib


STATE_KINDS = {"ipca": 0, "bigd": 1, "fbpca": 2}        # GSB_STATE_* of include/ganspace_b200.h


def state_layout_version(kind: str) -> int:
    """The layout version the library reports for an engine's state blob ('ipca', 'bigd' or 'fbpca')."""
    return int(load().gsb_state_layout_version(STATE_KINDS[kind]))


def _to_host(t: torch.Tensor):
    """One device -> host copy of a saved blob, as a NumPy array."""
    return t.detach().cpu().numpy()


def _load_blob(dst: torch.Tensor, src, what: str):
    """Copy a saved host blob into the device tensor ``dst``; its size must be the tensor's."""
    src = torch.as_tensor(src)
    if src.numel() != dst.numel() or src.dtype != dst.dtype:
        raise ValueError(f"{what}: saved blob of {src.numel()} x {src.dtype} does not fit {dst.numel()} x {dst.dtype}")
    dst.copy_(src.reshape(dst.shape))


def require_cuda(device=None) -> torch.device:
    if not torch.cuda.is_available():
        raise NativeError("ganspace_b200 needs a CUDA device (H100, sm_90a); there is no CPU fallback")
    dev = torch.device(device if device is not None else "cuda")
    if dev.type != "cuda":
        raise NativeError(f"ganspace_b200 runs on CUDA devices only, got {dev}")
    return dev


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def _ptr(t):
    if t is None:
        return C.c_void_p(0)
    assert t.is_cuda and t.is_contiguous(), "device-contiguous tensor expected"
    return C.c_void_p(t.data_ptr())


def _check(rc: int, what: str):
    if rc != 0:
        raise NativeError(f"{what} failed ({rc}): {load().gsb_last_error().decode()}")


class _Instrument:
    """Launch counter and optional per-section CUDA-event timers (used by bench.py for the roofline).

    ``launches`` counts the kernels this library enqueued (each C-ABI call launches a fixed number).
    When ``timing`` is on, sections wrap their C call in a pair of events recorded on the launching
    stream; ``section_ms()`` sums them after a synchronize."""

    def __init__(self):
        self.launches = 0
        self.timing = False
        self._events = {}
        self.rows = {}
        self.timeline = [] if os.environ.get("GANSPACE_B200_TIMELINE") == "1" else None

    def reset(self):
        self.launches = 0
        self._events = {}
        self.rows = {}

    def mark(self, name):
        """GANSPACE_B200_TIMELINE=1: a timed event on the current stream (tools/phase_probe.py prints them)."""
        if self.timeline is not None:
            ev = torch.cuda.Event(enable_timing=True)
            ev.record(torch.cuda.current_stream())
            self.timeline.append((name, ev))

    def timeline_ms(self):
        torch.cuda.synchronize()
        t0 = self.timeline[0][1]
        return [(n, t0.elapsed_time(e)) for n, e in self.timeline]

    def add_rows(self, name, n):
        """rows (samples) a section's kernels processed -- the roofline's unit count (bench.py)."""
        self.rows[name] = self.rows.get(name, 0) + int(n)

    def count(self, n):
        self.launches += n

    class _Sec:
        def __init__(self, outer, name):
            self.o, self.name = outer, name

        def __enter__(self):
            if self.o.timing:
                self.e0 = torch.cuda.Event(enable_timing=True)
                self.e1 = torch.cuda.Event(enable_timing=True)
                self.e0.record(torch.cuda.current_stream())

        def __exit__(self, *a):
            if self.o.timing:
                self.e1.record(torch.cuda.current_stream())
                self.o._events.setdefault(self.name, []).append((self.e0, self.e1))
            self.o.mark(self.name + " done")

    def section(self, name):
        return self._Sec(self, name)

    def section_ms(self):
        torch.cuda.synchronize()
        return {k: (sum(a.elapsed_time(b) for a, b in v), len(v)) for k, v in self._events.items()}


instrument = _Instrument()

# the kernels behind each timed section (bench.py's roofline names the one it reports)
SECTION_KERNELS = {
    "mapping": "mapping MLP: pixelnorm_split + 8 x mapping_layer_tc_kernel (wgmma, fp16 hi/lo x3)",
    "linear": "gen_z linear: mapping_layer_tc_kernel (wgmma, fp16 hi/lo x3, bias epilogue, TMA store) for n >= 128",
    "synthesis": "StyledConv chain: tap-GEMM tc_gemm_plain (wgmma) + gather/scatter/blur epilogues",
    "progan": "ProGAN chain: tap-GEMM tc_gemm_plain (wgmma) + pg_gather_kernel (gather, bias, leaky-ReLU, PixelNorm, RGB)",
    "stylegan": "StyleGAN chain: tap-GEMM tc_gemm_plain (wgmma) + sg_epilogue_kernel (gather / blur, noise, leaky-ReLU, sums) + "
                "sg_finish_kernel + sg_apply_kernel (InstanceNorm + StyleMod, torgb)",
    "biggan": "BigGAN chain: bb_conv_kernel (fp32 implicit GEMM, BN+ReLU prologue, skip / residual epilogue), attention, RGB",
}


def kernel_name(section: str) -> str:
    if section == "mapping" and os.environ.get("GANSPACE_B200_MAPPING", MAPPING_DEFAULT) == "simt":
        return "mapping MLP: pixelnorm + 8 x sgemm_tn_bias_act_kernel (fp32 FMA)"
    return SECTION_KERNELS.get(section, section)


class _Scratch:
    """Grow-only per-device scratch buffers keyed by purpose (the C ABI never allocates)."""

    def __init__(self):
        self._bufs = {}

    def get(self, key, nbytes: int, device) -> torch.Tensor:
        k = (key, str(device))
        buf = self._bufs.get(k)
        if buf is None or buf.numel() < nbytes:
            buf = torch.empty(max(int(nbytes), 256), dtype=torch.uint8, device=device)
            self._bufs[k] = buf
        return buf

    def clear(self):
        self._bufs.clear()


scratch = _Scratch()


# ------------------------------------------------------------------------------------------------
# thin tensor-level wrappers
# ------------------------------------------------------------------------------------------------
_jump_polys = {}        # (step_words, count) -> host table; (step_words, count, device) -> device copy


def jump_polys(n_per_stream: int, parts: int, device) -> torch.Tensor:
    """Device copy of the MT19937 jump polynomials for streams of n_per_stream normals split into `parts` sub-streams
    (computed once per process on the host, ~0.1 s; csrc/rng_jump.cu)."""
    import numpy as np
    lib = load()
    step = int(lib.gsb_legacy_normal_split_step_words(int(n_per_stream), int(parts)))
    key = (step, parts - 1)
    if key not in _jump_polys:
        table = np.zeros((parts - 1, 624), np.uint32)
        _check(lib.gsb_mt19937_jump_polys(step, parts - 1, table.ctypes.data_as(C.c_void_p)), "gsb_mt19937_jump_polys")
        _jump_polys[key] = table
    dkey = key + (str(device),)
    if dkey not in _jump_polys:
        _jump_polys[dkey] = torch.from_numpy(_jump_polys[key].view(np.int32)).to(device)
    return _jump_polys[dkey]


def split_parts(n_per_stream: int) -> int:
    """CTAs per stream: long streams (a 10k-row batch = 5.12M normals = 8.6 ms on one SM) are generated by up to 8 CTAs."""
    env = os.environ.get("GANSPACE_B200_RNG_PARTS")
    if env:
        return max(1, min(16, int(env)))
    if n_per_stream % 2:
        return 1
    return max(1, min(8, n_per_stream // 600_000))


def legacy_normal(seeds, n_per_stream: int, device, out=None, parts: int = 1, scratch_key: str = "rng_split") -> torch.Tensor:
    """RandomState(seed).standard_normal(n_per_stream).astype(float32) for every seed -> [S, n].
    ``parts`` > 1: every stream is generated by that many CTAs (MT19937 jump-ahead), bit-identical output."""
    lib = load()
    dev = require_cuda(device)
    # ``seeds``: a list of ints, or an int32 device tensor from seeds_tensor() (no host->device copy on this call: a copy
    # issued behind a long kernel would block the host until that kernel has finished)
    seeds_dev = seeds if isinstance(seeds, torch.Tensor) else _seeds_tensor(seeds, dev)
    assert seeds_dev.is_cuda and seeds_dev.dtype == torch.int32 and seeds_dev.is_contiguous()
    S = seeds_dev.numel()
    if out is None:
        out = torch.empty((S, n_per_stream), dtype=torch.float32, device=dev)
    assert out.is_cuda and out.is_contiguous() and out.numel() >= S * n_per_stream
    if parts > 1 and S > 0 and n_per_stream >= 2 and n_per_stream % 2 == 0:
        polys = jump_polys(n_per_stream, parts, dev)
        ws = scratch.get(scratch_key, lib.gsb_legacy_normal_split_workspace_bytes(S, n_per_stream, parts), dev)
        with torch.cuda.device(dev), instrument.section("rng"):
            _check(lib.gsb_legacy_normal_f32_split(_ptr(seeds_dev), S, n_per_stream, _ptr(out), n_per_stream, parts, _ptr(polys),
                                                   _ptr(ws), ws.numel(), _stream()), "gsb_legacy_normal_f32_split")
        instrument.count(2)
        return out
    with torch.cuda.device(dev), instrument.section("rng"):
        _check(lib.gsb_legacy_normal_f32(_ptr(seeds_dev), S, n_per_stream, _ptr(out), n_per_stream, _stream()),
               "gsb_legacy_normal_f32")
    instrument.count(1)
    return out


def seeds_tensor(seeds, dev):
    return _seeds_tensor(seeds, dev)


def rng_split_status(n_streams: int, n_per_stream: int, parts: int, device) -> int:
    """Status word of the last split launch of this shape on ``device`` (0 = fine; synchronises)."""
    lib = load()
    dev = require_cuda(device)
    ws = scratch.get("rng_split", lib.gsb_legacy_normal_split_workspace_bytes(n_streams, n_per_stream, parts), dev)
    flags = C.c_uint(0)
    with torch.cuda.device(dev):
        _check(lib.gsb_legacy_normal_split_status(_ptr(ws), n_streams, n_per_stream, parts, C.byref(flags), _stream()),
               "gsb_legacy_normal_split_status")
    return int(flags.value)


def _seeds_tensor(seeds, dev):
    """uint32 seeds carried in an int32 tensor (two's-complement reinterpretation)."""
    vals = [(int(s) & 0xFFFFFFFF) for s in seeds]
    vals = [v - (1 << 32) if v >= (1 << 31) else v for v in vals]
    return torch.tensor(vals, dtype=torch.int32, device=dev)


def legacy_truncnorm(seeds, n_per_stream: int, lo: float, hi: float, scale: float, device) -> torch.Tensor:
    lib = load()
    dev = require_cuda(device)
    sd = _seeds_tensor(seeds, dev)
    out = torch.empty((sd.numel(), n_per_stream), dtype=torch.float32, device=dev)
    with torch.cuda.device(dev):
        _check(lib.gsb_legacy_truncnorm_f32(_ptr(sd), sd.numel(), n_per_stream, lo, hi, scale, _ptr(out),
                                            n_per_stream, _stream()), "gsb_legacy_truncnorm_f32")
    return out


def mt19937_raw(seeds, n_per_stream: int, device) -> torch.Tensor:
    lib = load()
    dev = require_cuda(device)
    sd = _seeds_tensor(seeds, dev)
    out = torch.empty((sd.numel(), n_per_stream), dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _check(lib.gsb_mt19937_raw_u32(_ptr(sd), sd.numel(), n_per_stream, _ptr(out), n_per_stream, _stream()),
               "gsb_mt19937_raw_u32")
    return out


# default mapping-network path: "tc" = tensor-core (wgmma) fp16x3 split (fp32-grade), "simt" = fp32 FMA kernels
MAPPING_DEFAULT = "tc"


def source_key(tensors, *extra) -> tuple:
    """What a packed copy of ``tensors`` depends on: ``(t._version, t.data_ptr())`` of each tensor (``None`` entries skipped),
    so that an in-place edit and a replaced storage both show, followed by the ``extra`` values."""
    return tuple((t._version, t.data_ptr()) for t in tensors if t is not None) + extra


class Repacked:
    """The last object built from a set of source tensors (a packed generator, a folded weight); ``get`` rebuilds it when
    ``source_key`` of the sources changes."""

    def __init__(self):
        self._key = self._obj = None

    def get(self, tensors, build, *extra):
        key = source_key(tensors, *extra)
        if self._obj is None or self._key != key:
            self._obj, self._key = build(), key
        return self._obj

    def current(self):
        """The last object built, or None; never builds."""
        return self._obj


class PackedMapping:
    """Pre-scaled mapping-network weights in the layout the kernels read (gsb_mapping_pack)."""

    def __init__(self, weight: torch.Tensor, bias: torch.Tensor, lr_mul: float):
        lib = load()
        dev = require_cuda(weight.device)
        self.n_layers, self.dim = int(weight.shape[0]), int(weight.shape[1])
        assert weight.shape == (self.n_layers, self.dim, self.dim) and bias.shape == (self.n_layers, self.dim)
        self.device = dev
        self.packed = torch.empty(lib.gsb_mapping_packed_bytes(self.n_layers, self.dim), dtype=torch.uint8, device=dev)
        w = weight.detach().to(dev, torch.float32).contiguous()
        b = bias.detach().to(dev, torch.float32).contiguous()
        with torch.cuda.device(dev):
            _check(lib.gsb_mapping_pack(_ptr(w), _ptr(b), self.n_layers, self.dim, float(lr_mul),
                                        _ptr(self.packed), _stream()), "gsb_mapping_pack")

    def check(self):
        """Raise if the tensor-core path saw an activation outside fp16's range (synchronises)."""
        flags = C.c_uint(0)
        with torch.cuda.device(self.device):
            _check(load().gsb_mapping_status(_ptr(self.packed), self.n_layers, self.dim, C.byref(flags)),
                   "gsb_mapping_status")
        if flags.value & 1:
            raise NativeError("mapping network: an activation exceeded fp16 range in the tensor-core path; "
                              "results are invalid (set GANSPACE_B200_MAPPING=simt)")

    def forward(self, z: torch.Tensor, out: torch.Tensor = None, pixelnorm: bool = True,
                force_simt: bool = None, leave_free_sms: int = 0) -> torch.Tensor:
        lib = load()
        if force_simt is None:
            force_simt = os.environ.get("GANSPACE_B200_MAPPING", MAPPING_DEFAULT) == "simt"
        assert z.is_cuda and z.dtype == torch.float32 and z.shape[-1] == self.dim
        z2 = z.reshape(-1, self.dim)
        if not z2.is_contiguous():
            z2 = z2.contiguous()
        n = z2.shape[0]
        if out is None:
            out = torch.empty_like(z2)
        ws_bytes = lib.gsb_mapping_workspace_bytes(n, self.dim)
        ws = scratch.get("mapping", ws_bytes, z.device)
        flags = (1 if pixelnorm else 0) | (2 if force_simt else 0) | ((int(leave_free_sms) & 0xff) << 8)
        with torch.cuda.device(z.device), instrument.section("mapping"):
            _check(lib.gsb_mapping_forward(_ptr(self.packed), self.n_layers, self.dim, _ptr(z2), _ptr(out), n,
                                           flags, _ptr(ws), ws.numel(), _stream()), "gsb_mapping_forward")
        instrument.count(self.n_layers + (1 if pixelnorm else 0))
        instrument.add_rows("mapping", n)
        return out.reshape(z.shape)


def linear(x: torch.Tensor, w: torch.Tensor, bias: torch.Tensor = None, lrelu: bool = False, bounded: bool = False) -> torch.Tensor:
    """y = x @ w.T (+ bias); x [n,K], w [N,K] (N % 128 == 0, K % 16 == 0).  ``bounded`` (|x| < 6e4 guaranteed by the caller)
    lets n >= 128, N % 256 == 0, K % 64 == 0 run on the tensor cores (fp32-grade); otherwise the fp32 FMA GEMM kernel."""
    lib = load()
    assert x.is_cuda and x.dtype == torch.float32 and w.dtype == torch.float32 and x.shape[-1] == w.shape[1]
    x2 = x.reshape(-1, x.shape[-1]).contiguous()
    w = w.contiguous()
    n, K = x2.shape
    N = w.shape[0]
    y = torch.empty((n, N), dtype=torch.float32, device=x.device)
    flags = (1 if lrelu else 0) | (2 if bounded else 0)
    ws = scratch.get("linear", lib.gsb_linear_workspace_bytes(n, N, K, flags), x.device)
    with torch.cuda.device(x.device), instrument.section("linear"):
        _check(lib.gsb_linear_forward(_ptr(x2), _ptr(w), _ptr(bias.contiguous() if bias is not None else None), _ptr(y),
                                      n, N, K, flags, _ptr(ws), ws.numel(), _stream()), "gsb_linear_forward")
    instrument.count(5 if (bounded and n >= 128 and N % 256 == 0 and K % 64 == 0) else 1)
    instrument.add_rows("linear", n)
    return y.reshape(*x.shape[:-1], N)


def mapping_pixelnorm(z: torch.Tensor) -> torch.Tensor:
    """PixelNorm alone (stylegan2-pytorch/model.py:14-19)."""
    lib = load()
    assert z.is_cuda and z.dtype == torch.float32
    dim = z.shape[-1]
    z2 = z.reshape(-1, dim).contiguous()
    out = torch.empty_like(z2)
    ws = scratch.get("mapping", lib.gsb_mapping_workspace_bytes(z2.shape[0], dim), z.device)
    with torch.cuda.device(z.device):
        _check(lib.gsb_mapping_forward(C.c_void_p(0), 0, dim, _ptr(z2), _ptr(out), z2.shape[0], 1, _ptr(ws),
                                       ws.numel(), _stream()), "gsb_mapping_forward")
    return out.reshape(z.shape)


def batch_stats(x: torch.Tensor, mean_out: torch.Tensor = None, gram_out: torch.Tensor = None):
    """(mean[d] fp64, centred Gram[d,d] fp64) of x[n,d] fp32."""
    lib = load()
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    n, d = x.shape
    ld = x.stride(0)
    if mean_out is None:
        mean_out = torch.empty(d, dtype=torch.float64, device=x.device)
    if gram_out is None:
        gram_out = torch.empty((d, d), dtype=torch.float64, device=x.device)
    ws_bytes = lib.gsb_batch_stats_workspace_bytes(n, d)
    ws = scratch.get("stats", ws_bytes, x.device)
    with torch.cuda.device(x.device), instrument.section("stats"):
        _check(lib.gsb_batch_stats(C.c_void_p(x.data_ptr()), n, d, ld, _ptr(mean_out), _ptr(gram_out), _ptr(ws),
                                   ws.numel(), _stream()), "gsb_batch_stats")
    instrument.count(3)
    return mean_out, gram_out


def batch_stats_multi(x: torch.Tensor, n_groups: int, rows_per_group: int, mean_out: torch.Tensor = None,
                      gram_out: torch.Tensor = None):
    """(mean[G,d] fp64, centred Gram[G,d,d] fp64) of G consecutive groups of rows of x[G*rows, d] fp32, one set of launches."""
    lib = load()
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    assert x.shape[0] >= n_groups * rows_per_group
    d, ld = x.shape[1], x.stride(0)
    mean = mean_out if mean_out is not None else torch.empty((n_groups, d), dtype=torch.float64, device=x.device)
    gram = gram_out if gram_out is not None else torch.empty((n_groups, d, d), dtype=torch.float64, device=x.device)
    assert mean.shape == (n_groups, d) and gram.shape == (n_groups, d, d) and mean.dtype == gram.dtype == torch.float64
    ws_bytes = lib.gsb_batch_stats_multi_workspace_bytes(n_groups, rows_per_group, d)
    ws = scratch.get("stats", ws_bytes, x.device)
    with torch.cuda.device(x.device), instrument.section("stats"):
        _check(lib.gsb_batch_stats_multi(C.c_void_p(x.data_ptr()), n_groups, rows_per_group, d, ld, _ptr(mean), _ptr(gram),
                                         _ptr(ws), ws.numel(), _stream()), "gsb_batch_stats_multi")
    instrument.count(4 if (d % 128 == 0 and d <= 1024) else 3 * n_groups)
    return mean, gram


def stats_grouped_width(d: int) -> bool:
    """Whether ``batch_stats_multi`` takes the tensor-core path at width d, i.e. whether ``batch_stats_grouped`` gives its bits
    (GANSPACE_B200_STATS=simt moves every width to the fp32 FMA kernels, which the grouped entry does not run)."""
    return d % 128 == 0 and 128 <= d <= 1024 and os.environ.get("GANSPACE_B200_STATS") != "simt"


def batch_stats_grouped(items):
    """``batch_stats_multi`` of several inputs at once: ``items`` is a list of (x [>= G*rows, d] fp32 with unit column stride,
    n_groups G, rows_per_group, mean_out [G, d] fp64 or None, gram_out [G, d, d] fp64 or None); returns [(mean, gram), ...] in
    the same order, bit-identical to calling ``batch_stats_multi`` on each.  Every width must be a multiple of 128 up to 1024
    (NativeError otherwise, before anything runs)."""
    lib = load()
    if not items:
        return []
    descs = (StatsDesc * len(items))()
    outs = []
    dev = items[0][0].device
    for i, (x, n_groups, rows, mean, gram) in enumerate(items):
        assert x.is_cuda and x.device == dev and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
        assert x.shape[0] >= n_groups * rows
        d = x.shape[1]
        mean = mean if mean is not None else torch.empty((n_groups, d), dtype=torch.float64, device=dev)
        gram = gram if gram is not None else torch.empty((n_groups, d, d), dtype=torch.float64, device=dev)
        assert mean.shape == (n_groups, d) and gram.shape == (n_groups, d, d) and mean.dtype == gram.dtype == torch.float64
        descs[i] = StatsDesc(x.data_ptr(), x.stride(0), d, int(n_groups), int(rows), _ptr(mean).value, _ptr(gram).value)
        outs.append((mean, gram))
    ws_bytes = lib.gsb_batch_stats_grouped_workspace_bytes(descs, len(items))
    if ws_bytes == 0:
        _check(lib.gsb_batch_stats_grouped(descs, len(items), C.c_void_p(0), 0, _stream()), "gsb_batch_stats_grouped")
    ws = scratch.get("stats", ws_bytes, dev)
    with torch.cuda.device(dev), instrument.section("stats"):
        _check(lib.gsb_batch_stats_grouped(descs, len(items), _ptr(ws), ws.numel(), _stream()), "gsb_batch_stats_grouped")
    instrument.count(5 * (-(-len(items) // 32)))
    return outs


class IPCAChain:
    """Device-resident IncrementalPCA state + the Gram-form chain step (small-d engine).

    The chain is the sequential part of a run (K dependent eigensolves), so its steps are enqueued on a
    dedicated high-priority stream: step k waits only for the statistics of group k (an event on the
    producing stream) and runs while the main stream already generates / reduces the next groups."""

    def __init__(self, d: int, c: int, device, side_stream: bool = True):
        lib = load()
        self.dev = require_cuda(device)
        self.d, self.c = int(d), int(c)
        self.state = torch.empty(lib.gsb_ipca_state_bytes(self.d, self.c), dtype=torch.uint8, device=self.dev)
        self.ws = torch.empty(lib.gsb_ipca_workspace_bytes(self.d, self.c), dtype=torch.uint8, device=self.dev)
        self.n_seen = 0
        self.stream = None
        if side_stream and os.environ.get("GANSPACE_B200_CHAIN_STREAM", "1") != "0":
            with torch.cuda.device(self.dev):
                self.stream = torch.cuda.Stream(device=self.dev, priority=-1)
        with torch.cuda.device(self.dev):
            _check(lib.gsb_ipca_reset(_ptr(self.state), self.d, self.c, _stream()), "gsb_ipca_reset")
            if self.stream is not None:
                self.stream.wait_stream(torch.cuda.current_stream())

    def step(self, n_batch: int, mean_b: torch.Tensor, gram_b: torch.Tensor):
        lib = load()
        assert mean_b.dtype == torch.float64 and gram_b.dtype == torch.float64
        with torch.cuda.device(self.dev):
            if self.stream is not None:
                self.stream.wait_stream(torch.cuda.current_stream())      # statistics of this group are ready
                mean_b.record_stream(self.stream)
                gram_b.record_stream(self.stream)
                ctx = torch.cuda.stream(self.stream)
            else:
                ctx = contextlib.nullcontext()
            with ctx, instrument.section("chain"):
                _check(lib.gsb_ipca_chain_step(_ptr(self.state), self.d, self.c, self.n_seen, int(n_batch),
                                               _ptr(mean_b), _ptr(gram_b), _ptr(self.ws), self.ws.numel(), _stream()),
                       "gsb_ipca_chain_step")
        # kernels per step: first step = direct solve (8) + seeding of the subspace form (1); later steps = one cluster
        # launch (orthogonal iteration, csrc/subspace.cu).  Shapes outside the subspace kernel's range: direct solve (8).
        instrument.count((1 if self.n_seen > 0 else 9) if chain_iterates(self.d, self.c) else 8)
        self.n_seen += int(n_batch)

    def join(self):
        """Make the current stream wait for every chain step enqueued so far."""
        if self.stream is not None:
            with torch.cuda.device(self.dev):
                torch.cuda.current_stream().wait_stream(self.stream)

    def state_dict(self):
        """The chain after the steps enqueued so far: the fp64 state blob (with the iterated chain's (H, Q)) and n_seen."""
        self.join()
        with torch.cuda.device(self.dev):
            return {"state": _to_host(self.state), "n_seen": self.n_seen}

    def load_state_dict(self, sd):
        """Continue from a ``state_dict`` of a chain of the same (d, c) and chain mode; later steps see what they would have
        seen after the saved steps."""
        self.join()
        with torch.cuda.device(self.dev):
            _load_blob(self.state, sd["state"], "IPCAChain.load_state_dict")
            if self.stream is not None:
                self.stream.wait_stream(torch.cuda.current_stream())
        self.n_seen = int(sd["n_seen"])

    def export(self):
        lib = load()
        self.join()
        f64 = dict(dtype=torch.float64, device=self.dev)
        out = {
            "components": torch.empty((self.c, self.d), **f64), "singular_values": torch.empty(self.c, **f64),
            "mean": torch.empty(self.d, **f64), "var": torch.empty(self.d, **f64),
            "explained_variance": torch.empty(self.c, **f64),
            "explained_variance_ratio": torch.empty(self.c, **f64),
        }
        with torch.cuda.device(self.dev):
            _check(lib.gsb_ipca_export(_ptr(self.state), self.d, self.c, self.n_seen, _ptr(out["components"]),
                                       _ptr(out["singular_values"]), _ptr(out["mean"]), _ptr(out["var"]),
                                       _ptr(out["explained_variance"]), _ptr(out["explained_variance_ratio"]),
                                       _stream()), "gsb_ipca_export")
            check_eig_status("IPCAChain.export")
        instrument.count(1)
        return out


def chain_iterates(d: int, c: int) -> bool:
    """Whether chain steps after the first enqueued now run the orthogonal iteration of csrc/subspace.cu rather than the direct
    solve.  The library reserves (H, Q) and an export workspace in the state exactly then, so the state is larger than its eigen
    form: header, mean, unnormalised variance, S and V (csrc/ipca.cu, ``state_view``), in fp64 and rounded up to 256 bytes."""
    key = (int(d), int(c), _chain_forced_direct)      # GANSPACE_B200_CHAIN is read once by the library
    if key not in _chain_iterates:
        eigen_form = (8 * (24 + 2 * d + c + c * d) + 255) // 256 * 256
        _chain_iterates[key] = load().gsb_ipca_state_bytes(d, c) > eigen_form
    return _chain_iterates[key]


_chain_iterates = {}


class ChainNotConverged(NativeError):
    """A chain step reached its iteration cap before its residual tolerance (no spectral gap after component c)."""


_chain_forced_direct = False


def set_chain_mode(direct: bool):
    """Every chain step enqueued from now on is the exact direct eigen-solve (True) / the default solver (False)."""
    global _chain_forced_direct
    _check(load().gsb_ipca_set_chain_mode(1 if direct else 0), "gsb_ipca_set_chain_mode")
    _chain_forced_direct = bool(direct)


def check_eig_status(what: str):
    """Raise if a chain kernel reported a failure since the last check (synchronises the current stream)."""
    flags = C.c_uint(0)
    _check(load().gsb_eig_status(C.byref(flags), _stream()), "gsb_eig_status")
    if flags.value:
        raise ChainNotConverged(f"{what}: a chain step hit its iteration cap without reaching the residual tolerance "
                                f"(status {flags.value}): the spectrum has no gap after component c (numerical rank below "
                                "n_components?); the exact route is GANSPACE_B200_CHAIN=direct (decomposition.compute re-runs "
                                "through it by itself)")


def sym_eig_top(a: torch.Tensor, c: int):
    lib = load()
    assert a.is_cuda and a.dtype == torch.float64 and a.dim() == 2 and a.shape[0] == a.shape[1]
    d = a.shape[0]
    a = a.contiguous().clone()
    evals = torch.empty(c, dtype=torch.float64, device=a.device)
    evecs = torch.empty((c, d), dtype=torch.float64, device=a.device)
    ws = torch.empty(lib.gsb_ipca_workspace_bytes(d, c), dtype=torch.uint8, device=a.device)
    with torch.cuda.device(a.device):
        _check(lib.gsb_sym_eig_top(_ptr(a), d, c, _ptr(evals), _ptr(evecs), _ptr(ws), ws.numel(), _stream()),
               "gsb_sym_eig_top")
        check_eig_status("sym_eig_top")
    return evals, evecs


def project_std(x: torch.Tensor, dirs: torch.Tensor, sub: torch.Tensor = None) -> torch.Tensor:
    lib = load()
    assert x.is_cuda and x.dtype == torch.float32 and x.dim() == 2 and x.stride(1) == 1
    n, d = x.shape
    dirs = dirs.to(x.device, torch.float32).contiguous()
    c = dirs.shape[0]
    assert dirs.shape[1] == d
    if sub is not None:
        sub = sub.to(x.device, torch.float64).contiguous()
    out = torch.empty(c, dtype=torch.float32, device=x.device)
    ws = scratch.get("projstd", lib.gsb_project_std_workspace_bytes(c), x.device)
    with torch.cuda.device(x.device):
        _check(lib.gsb_project_std(C.c_void_p(x.data_ptr()), n, d, x.stride(0), _ptr(dirs), c, _ptr(sub), _ptr(out),
                                   _ptr(ws), ws.numel(), _stream()), "gsb_project_std")
    instrument.count(2)
    return out


class LinregAccumulator:
    """Normal-equation accumulators of the latent regression (decomposition.py:77-139)."""

    def __init__(self, c: int, latent_dim: int, device):
        lib = load()
        self.dev = require_cuda(device)
        self.c, self.L = int(c), int(latent_dim)
        self.state = torch.empty(lib.gsb_linreg_state_bytes(self.c, self.L), dtype=torch.uint8, device=self.dev)
        self.n_total = 0
        with torch.cuda.device(self.dev):
            _check(lib.gsb_linreg_reset(_ptr(self.state), self.c, self.L, _stream()), "gsb_linreg_reset")

    def accumulate(self, act, comp32, mean32, stdev32, z):
        lib = load()
        n, d = act.shape
        act, comp32, mean32, stdev32, z = (t.contiguous() for t in (act, comp32, mean32, stdev32, z))
        assert z.shape == (n, self.L) and comp32.shape == (self.c, d)
        ws = scratch.get("linreg", lib.gsb_linreg_workspace_bytes(n, self.c, d), self.dev)
        with torch.cuda.device(self.dev):
            _check(lib.gsb_linreg_accumulate(_ptr(self.state), self.c, self.L, _ptr(act), n, d, _ptr(comp32),
                                             _ptr(mean32), _ptr(stdev32), _ptr(z), _ptr(ws), ws.numel(), _stream()),
                   "gsb_linreg_accumulate")
        instrument.count(2 if lib.gsb_linreg_feature_splits(n, self.c, d) == 1 else 3)     # + the split sum
        self.n_total += n

    RCOND = 1e-6        # eigenvalues of A^T A below RCOND * largest count as zero in the minimum-norm fallback

    def solve(self):
        """(M_t [c, L], Z_mean [L]) fp64.  Well-conditioned normal equations (the usual case: the columns of A are unit-variance
        PC coordinates) are solved by Cholesky; if a pivot fails, the minimum-norm least-squares solution is formed from the
        eigen-decomposition of A^T A -- what scipy's gelsd (decomposition.py:133) returns for a rank-deficient A."""
        lib = load()
        M = torch.zeros((self.c, self.L), dtype=torch.float64, device=self.dev)
        zmean = torch.empty(self.L, dtype=torch.float64, device=self.dev)
        info = C.c_int(0)
        with torch.cuda.device(self.dev):
            _check(lib.gsb_linreg_solve(_ptr(self.state), self.c, self.L, self.n_total, _ptr(M), _ptr(zmean), _stream()),
                   "gsb_linreg_solve")
            _check(lib.gsb_linreg_solve_status(_ptr(self.state), self.c, self.L, C.byref(info), _stream()), "gsb_linreg_solve_status")
        instrument.count(1)
        self.rank_deficient_at = int(info.value)
        if info.value != 0:
            n = (self.c + 31) // 32 * 32                      # the eigensolver wants a multiple of 32: pad with a -1 diagonal
            off = int(lib.gsb_linreg_normal_matrix(_ptr(self.state), self.c, self.L)) - self.state.data_ptr()
            ata = self.state[off:off + self.c * self.c * 8].view(torch.float64).view(self.c, self.c)
            if not bool(torch.isfinite(ata).all()):
                raise NativeError("latent regression: the normal equations contain non-finite entries (a zero or NaN stdev "
                                  "column?); scipy's lstsq raises on such input as well")
            pad = torch.zeros((n, n), dtype=torch.float64, device=self.dev)
            pad[:self.c, :self.c] = ata
            if n > self.c:
                pad[self.c:, self.c:] = -torch.eye(n - self.c, dtype=torch.float64, device=self.dev)
            evals, evecs = sym_eig_top(pad, self.c)           # padding eigenvalues (-1) sort last and are not returned
            evecs = evecs[:, :self.c].contiguous()
            with torch.cuda.device(self.dev):
                _check(lib.gsb_linreg_solve_pinv(_ptr(self.state), self.c, self.L, _ptr(evals), _ptr(evecs), self.RCOND, _ptr(M),
                                                 _stream()), "gsb_linreg_solve_pinv")
            instrument.count(9)
        return M, zmean


class _PackedTapGenerator:
    """What the tap-GEMM generators (PackedSynthesis, PackedProGAN, PackedStyleGAN) share: the packed device buffer, ``shapes``
    ((res_out, cout) per layer), the activation and image outputs, and the fp16-overflow status.  ``NAME`` is the family's
    prefix in the C entry points; each subclass makes its own C calls."""

    NAME = ""

    def _pack(self, nbytes: int, pack):
        """Allocates ``nbytes`` (the family's gsb_*_packed_bytes) and runs ``pack(d_packed, packed_bytes, stream)`` into it."""
        if nbytes == 0:
            raise NativeError(f"gsb_{self.NAME}_packed_bytes: {load().gsb_last_error().decode()}")
        self.packed = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
        with torch.cuda.device(self.device):
            _check(pack(_ptr(self.packed), self.packed.numel(), _stream()), f"gsb_{self.NAME}_pack")
            torch.cuda.current_stream().synchronize()      # the fp32 parameter copies may be freed after this returns

    def out_dims(self, n_run: int) -> int:
        r, co = self.shapes[n_run - 1]
        return r * r * co

    def _rgb_after(self, n_rgb: int) -> int:
        """The layer whose resolution the image after ``n_rgb`` ToRGBs has: the last one (one ToRGB after the last layer)."""
        return -1

    def _outputs(self, n: int, n_run: int, out, want_act: bool, n_rgb: int, device):
        """(activation rows [n, out_dims] -- ``out`` if given -- or None, image [n, res, res, 3] after ``n_rgb`` ToRGBs or None).
        The generators with one ToRGB after the last layer pass their ``want_rgb``."""
        act = rgb = None
        if want_act:
            d = self.out_dims(n_run)
            act = torch.empty((n, d), dtype=torch.float32, device=device) if out is None else out
            assert act.is_cuda and act.dtype == torch.float32 and act.shape == (n, d) and act.stride(1) == 1
        if n_rgb:
            res = self.shapes[self._rgb_after(n_rgb)][0]
            rgb = torch.empty((n, res, res, 3), dtype=torch.float32, device=device)
        return act, rgb

    @staticmethod
    def _latents(w: torch.Tensor, dim: int) -> torch.Tensor:
        """[Lw, n, dim] contiguous latents from ``w`` [n, dim] (one latent for every layer) or [Lw, n, dim] (per-layer latents)."""
        assert w.is_cuda and w.dtype == torch.float32 and w.shape[-1] == dim and w.dim() in (2, 3)
        return (w[None] if w.dim() == 2 else w).contiguous()

    def _style_rows(self, S, keys):
        """(the rows S[k] of the style layers ``keys``, contiguous; their row count n), each checked to be [n, style_width(k)] fp32
        on the device."""
        rows = [S[k] for k in keys]
        n = int(rows[0].shape[0])
        for k, t in zip(keys, rows):
            assert t.is_cuda and t.dtype == torch.float32 and tuple(t.shape) == (n, self.style_width(k)), \
                f"style layer {k}: rows [{n}, {self.style_width(k)}] fp32 on the device expected, got {tuple(t.shape)} {t.dtype}"
        return [t.contiguous() for t in rows], n

    def check(self):
        flags = C.c_uint(0)
        with torch.cuda.device(self.device):
            _check(self._status(C.byref(flags)), f"gsb_{self.NAME}_status")
        if flags.value & 1:
            raise NativeError(f"{self.NAME}: an operand exceeded fp16 range in the tensor-core path; results are invalid")


class PackedSynthesis(_PackedTapGenerator):
    """StyleGAN2 synthesis layers conv1, convs.0 .. convs.k and the ToRGBs that follow them, packed for the tap-GEMM kernels
    (gsb_synthesis_pack).

    ``layers``: dicts with conv_weight [co,ci,3,3], mod_weight [ci,S], mod_bias [ci], act_bias [co], noise [r,r],
    noise_weight [1] (fp32 CUDA tensors) and upsample (bool), res_in (int), in execution order.  ``rgbs``: dicts with conv_weight
    [3,ci], mod_weight [ci,S], mod_bias [ci] and bias [3] of to_rgb1, to_rgbs.0, ...: the (len(layers) + 1) // 2 that follow the
    layers (ToRGB j follows layer 2j).  Style layers are keyed by their position in execution order (conv1, to_rgb1, convs.0,
    convs.1, to_rgbs.0, ...), the order of ``Generator.style_layers()``."""

    NAME = "synthesis"

    def __init__(self, const_input: torch.Tensor, layers, rgbs, style_dim: int):
        lib = load()
        self.device = require_cuda(const_input.device)
        self.style_dim = int(style_dim)
        self.n_layers, self.n_rgb = len(layers), (len(layers) + 1) // 2
        assert len(rgbs) == self.n_rgb, f"{self.n_layers} layers are followed by {self.n_rgb} ToRGBs, got {len(rgbs)}"
        self.desc = (StyledConvDesc * self.n_layers)()
        self.rgb_desc = (ToRGBDesc * self.n_rgb)()
        self.shapes = []                        # (res_out, cout) per layer
        self.slots = []                         # style layer -> ("conv", l) or ("rgb", j), in execution order
        f32 = lambda t: t.detach().to(self.device, torch.float32).contiguous()
        keep = []
        for i, L in enumerate(layers):
            ts = {k: f32(L[k]) for k in ("conv_weight", "mod_weight", "mod_bias", "act_bias", "noise", "noise_weight")}
            keep.append(ts)
            co, ci = ts["conv_weight"].shape[0], ts["conv_weight"].shape[1]
            assert ts["conv_weight"].shape == (co, ci, 3, 3) and ts["mod_weight"].shape == (ci, self.style_dim)
            res_in, up = int(L["res_in"]), bool(L["upsample"])
            res_out = 2 * res_in if up else res_in
            assert ts["noise"].numel() == res_out * res_out and ts["noise_weight"].numel() == 1
            d = self.desc[i]
            for k, t in ts.items():
                setattr(d, k, t.data_ptr())
            d.cin, d.cout, d.upsample, d.res_in = ci, co, int(up), res_in
            self.shapes.append((res_out, co))
            self.slots.append(("conv", i))
            if i % 2 == 0:
                self.slots.append(("rgb", i // 2))
        for j, R in enumerate(rgbs):
            ts = {k: f32(R[k]) for k in ("conv_weight", "mod_weight", "mod_bias", "bias")}
            keep.append(ts)
            ci = self.shapes[2 * j][1]
            assert ts["conv_weight"].numel() == 3 * ci and ts["mod_weight"].shape == (ci, self.style_dim) and ts["bias"].numel() == 3
            for k, t in ts.items():
                setattr(self.rgb_desc[j], k, t.data_ptr())
            self.rgb_desc[j].cin = ci
        self.slot_of = {s: k for k, s in enumerate(self.slots)}
        cst = f32(const_input).reshape(-1, 4, 4)
        self._pack(lib.gsb_synthesis_packed_bytes(self.desc, self.n_layers, self.style_dim),
                   lambda packed, nbytes, st: lib.gsb_synthesis_pack(self.desc, self.n_layers, self.style_dim, self.rgb_desc, _ptr(cst),
                                                                     packed, nbytes, st))

    def _rgb_after(self, n_rgb: int) -> int:
        return 2 * (n_rgb - 1)

    def workspace_bytes(self, n_run: int, n: int) -> int:
        """Workspace of ``forward`` to layer n_run - 1 for n rows, without ToRGBs."""
        return int(load().gsb_synthesis_workspace_bytes(self.desc, n_run, 0, int(n)))

    def rows_within(self, n_run: int, n: int, budget: int) -> int:
        """The most rows (n, or a power of two below it) whose ``forward`` to layer n_run - 1 needs at most ``budget`` bytes of
        workspace; at least 1."""
        rows = int(n)
        while rows > 1 and self.workspace_bytes(n_run, rows) > budget:
            rows = 1 << ((rows - 1).bit_length() - 1)
        return rows

    def style_width(self, k: int) -> int:
        """Width of style layer ``k``'s rows: the input channels of its StyledConv or ToRGB."""
        chain, i = self.slots[k]
        return self.desc[i].cin if chain == "conv" else self.shapes[2 * i][1]

    def forward(self, w: torch.Tensor, n_run: int, out: torch.Tensor = None, want_act: bool = True, n_rgb: int = 0):
        """Layers 0 .. n_run-1 and ToRGBs 0 .. n_rgb-1 (n_rgb <= (n_run + 1) // 2) for latents ``w`` [n, style_dim] (one latent for
        every layer) or [Lw, n, style_dim] (layer l reads latent min(l, Lw-1), ToRGB j latent min(2j+1, Lw-1)).  Returns (activation
        of layer n_run-1 as fp32 NHWC rows [n, res*res*cout] or None, skip image after ToRGB n_rgb-1 as fp32 NHWC [n, res, res, 3]
        or None).  ``out`` may be a row-strided 2-D view, e.g. the batch rows of the large-d IPCA buffer."""
        lib = load()
        w3 = self._latents(w, self.style_dim)
        Lw, n = int(w3.shape[0]), int(w3.shape[1])
        act, rgb = self._outputs(n, n_run, out, want_act, n_rgb, self.device)
        ws = scratch.get("synthesis", lib.gsb_synthesis_workspace_bytes(self.desc, n_run, n_rgb, n), self.device)
        with torch.cuda.device(self.device), instrument.section("synthesis"):
            _check(lib.gsb_synthesis_forward(_ptr(self.packed), self.desc, self.n_layers, n_run, n_rgb, self.style_dim, _ptr(w3), Lw, n,
                                             C.c_void_p(act.data_ptr() if act is not None else 0), act.stride(0) if act is not None else 0,
                                             _ptr(rgb), _ptr(ws), ws.numel(), _stream()), "gsb_synthesis_forward")
        self._count(n, n_run, n_rgb)
        return act, rgb

    def styles(self, w: torch.Tensor, keys):
        """The style-space rows (gsb_synthesis_styles): for latents ``w`` as in ``forward``, the modulation output [n, width] of every
        style layer in ``keys`` (positions in execution order).  Returns {key: rows}.  The launches are the chain's own style stage,
        so at the same n the rows are the ones it consumes."""
        lib = load()
        w3 = self._latents(w, self.style_dim)
        Lw, n = int(w3.shape[0]), int(w3.shape[1])
        keys = sorted(set(int(k) for k in keys))
        assert all(0 <= k < len(self.slots) for k in keys), keys
        S = {k: torch.empty((n, self.style_width(k)), dtype=torch.float32, device=self.device) for k in keys}
        ptrs = {"conv": [None] * self.n_layers, "rgb": [None] * self.n_rgb}
        for k in keys:
            chain, i = self.slots[k]
            ptrs[chain][i] = S[k].data_ptr()
        with torch.cuda.device(self.device), instrument.section("styles"):
            _check(lib.gsb_synthesis_styles(_ptr(self.packed), self.desc, self.n_layers, self.style_dim, _ptr(w3), Lw, n,
                                            (C.c_void_p * self.n_layers)(*ptrs["conv"]), (C.c_void_p * self.n_rgb)(*ptrs["rgb"]),
                                            _stream()), "gsb_synthesis_styles")
        instrument.count(len(keys))
        instrument.add_rows("styles", n)
        return S

    def forward_styled(self, S, n_run: int, out: torch.Tensor = None, want_act: bool = True, n_rgb: int = 0):
        """``forward`` on caller-given styles (gsb_synthesis_forward_styled): ``S`` {style layer: rows [n, width] fp32} holding the
        layers 0 .. n_run-1 and the ToRGBs 0 .. n_rgb-1.  Same outputs as ``forward``."""
        lib = load()
        keys = [self.slot_of["conv", l] for l in range(n_run)] + [self.slot_of["rgb", j] for j in range(n_rgb)]
        rows, n = self._style_rows(S, keys)
        act, rgb = self._outputs(n, n_run, out, want_act, n_rgb, self.device)
        S_ptrs = (C.c_void_p * n_run)(*[t.data_ptr() for t in rows[:n_run]])
        R_ptrs = (C.c_void_p * max(1, n_rgb))(*[t.data_ptr() for t in rows[n_run:]])
        ws = scratch.get("synthesis", lib.gsb_synthesis_forward_styled_workspace_bytes(self.desc, n_run, n_rgb, n), self.device)
        with torch.cuda.device(self.device), instrument.section("synthesis"):
            _check(lib.gsb_synthesis_forward_styled(_ptr(self.packed), self.desc, self.n_layers, n_run, n_rgb, self.style_dim, S_ptrs,
                                                    R_ptrs, n, C.c_void_p(act.data_ptr() if act is not None else 0),
                                                    act.stride(0) if act is not None else 0, _ptr(rgb), _ptr(ws), ws.numel(), _stream()),
                   "gsb_synthesis_forward_styled")
        self._count(n, n_run, n_rgb)
        return act, rgb

    def _count(self, n, n_run, n_rgb):
        # per layer: 4 style/demod launches; per chunk of samples: 1 GEMM + 1 (stride-1) or 2 (upsample) epilogue launches;
        # per ToRGB: its style and its skip-image launch
        launches = 1 + 2 * n_rgb
        for i in range(n_run):
            res_in = self.desc[i].res_in
            chunks = -(-n // max(1, 4096 // (res_in * res_in)))
            launches += 4 + chunks * (3 if self.desc[i].upsample else 2)
        instrument.count(launches)
        instrument.add_rows("synthesis", n)

    def _status(self, flags):
        return load().gsb_synthesis_status(_ptr(self.packed), self.desc, self.n_layers, self.style_dim, flags)


class PackedProGAN(_PackedTapGenerator):
    """ProGAN blocks layer1 .. layerK and the RGB output block packed for the tap-GEMM kernels (gsb_progan_pack).

    ``blocks``: dicts with conv_weight [co,ci,k,k], bias [co] (fp32 tensors) and upsample (bool), in execution order;
    ``out_weight`` [3,c,1,1] / ``out_bias`` [3]: the output block."""

    NAME = "progan"

    def __init__(self, blocks, out_weight: torch.Tensor, out_bias: torch.Tensor):
        lib = load()
        self.device = require_cuda(out_weight.device)
        self.n_blocks = len(blocks)
        self.desc = (ProGANBlockDesc * self.n_blocks)()
        self.shapes = []                        # (res_out, cout) per block
        f32 = lambda t: t.detach().to(self.device, torch.float32).contiguous()
        keep, res = [], 1
        for i, L in enumerate(blocks):
            w, b = f32(L["conv_weight"]), f32(L["bias"])
            keep += [w, b]
            co, ci, k = w.shape[0], w.shape[1], w.shape[2]
            assert w.shape == (co, ci, k, k) and b.shape == (co,) and k == (4 if i == 0 else 3)
            d = self.desc[i]
            d.conv_weight, d.bias = w.data_ptr(), b.data_ptr()
            d.cin, d.cout, d.upsample, d.res_in, d.ksize = ci, co, int(bool(L["upsample"])), res, k
            res = 4 if i == 0 else (2 * res if L["upsample"] else res)
            self.shapes.append((res, co))
        self.z_dim = int(self.desc[0].cin)
        ow, ob = f32(out_weight).reshape(3, -1), f32(out_bias).reshape(3)
        assert ow.shape[1] == self.shapes[-1][1]
        self._pack(lib.gsb_progan_packed_bytes(self.desc, self.n_blocks),
                   lambda packed, nbytes, st: lib.gsb_progan_pack(self.desc, self.n_blocks, _ptr(ow), _ptr(ob), packed, nbytes, st))

    def forward(self, z: torch.Tensor, n_run: int, out: torch.Tensor = None, want_act: bool = True, want_rgb: bool = False):
        """Blocks 0 .. n_run-1 on z [n, z_dim].  Returns (activation of block n_run-1 as fp32 NHWC rows [n, res*res*cout] or None,
        image as fp32 NHWC [n, res, res, 3] or None; the image needs n_run == n_blocks).  ``out`` may be a row-strided 2-D view,
        e.g. the batch rows of the large-d IPCA buffer."""
        lib = load()
        assert z.is_cuda and z.dtype == torch.float32 and z.dim() == 2 and z.shape[1] == self.z_dim
        z = z.contiguous()
        n = z.shape[0]
        act, rgb = self._outputs(n, n_run, out, want_act, want_rgb, z.device)
        if n == 0:
            return act, rgb
        ws_bytes = lib.gsb_progan_workspace_bytes(self.desc, n_run, n)
        ws = scratch.get("progan", ws_bytes, z.device)
        with torch.cuda.device(z.device), instrument.section("progan"):
            _check(lib.gsb_progan_forward(_ptr(self.packed), self.desc, self.n_blocks, n_run, _ptr(z), n,
                                          C.c_void_p(act.data_ptr() if act is not None else 0), act.stride(0) if act is not None else 0,
                                          _ptr(rgb), _ptr(ws), ws.numel(), _stream()), "gsb_progan_forward")
        instrument.count(1)
        instrument.add_rows("progan", n)
        return act, rgb

    def _status(self, flags):
        return load().gsb_progan_status(_ptr(self.packed), self.desc, self.n_blocks, flags)


class PackedStyleGAN(_PackedTapGenerator):
    """StyleGAN (v1) synthesis layers (two per block) and torgb packed for the tap-GEMM kernels (gsb_stylegan_pack).

    ``layers``: dicts with conv_weight [co,ci,3,3] (None for the first layer), bias [co], noise [r,r], noise_weight [co],
    style_weight [2co, dlatent], style_bias [2co] (fp32 tensors), upsample (bool) and res_out (int), in execution order;
    ``const`` [c0,4,4]: the InputBlock's constant; ``rgb_weight`` [3,c,1,1] / ``rgb_bias`` [3]: torgb."""

    NAME = "stylegan"

    def __init__(self, layers, const: torch.Tensor, rgb_weight: torch.Tensor, rgb_bias: torch.Tensor, dlatent: int = 512):
        lib = load()
        self.device = require_cuda(rgb_weight.device)
        self.n_layers, self.dlatent = len(layers), int(dlatent)
        self.desc = (StyleGANLayerDesc * self.n_layers)()
        self.shapes = []                        # (res_out, cout) per layer
        f32 = lambda t: t.detach().to(self.device, torch.float32).contiguous()
        keep = []
        for i, L in enumerate(layers):
            ts = {k: f32(L[k]) for k in ("bias", "noise", "noise_weight", "style_weight", "style_bias")}
            if L["conv_weight"] is not None:
                ts["conv_weight"] = f32(L["conv_weight"])
            keep.append(ts)
            co, r = ts["bias"].shape[0], int(L["res_out"])
            ci = ts["conv_weight"].shape[1] if "conv_weight" in ts else co
            assert ("conv_weight" in ts) == (i > 0) and ts["noise"].numel() == r * r and ts["noise_weight"].shape == (co,)
            assert ts["style_weight"].shape == (2 * co, self.dlatent) and ts["style_bias"].shape == (2 * co,)
            d = self.desc[i]
            for k, t in ts.items():
                setattr(d, k, t.data_ptr())
            d.cin, d.cout, d.upsample, d.res_out = ci, co, int(bool(L["upsample"])), r
            self.shapes.append((r, co))
        cst = f32(const).reshape(self.shapes[0][1], 4, 4)
        rw, rb = f32(rgb_weight).reshape(3, -1), f32(rgb_bias).reshape(3)
        assert rw.shape[1] == self.shapes[-1][1]
        self._pack(lib.gsb_stylegan_packed_bytes(self.desc, self.n_layers, self.dlatent),
                   lambda packed, nbytes, st: lib.gsb_stylegan_pack(self.desc, self.n_layers, self.dlatent, _ptr(cst), _ptr(rw), _ptr(rb),
                                                                    packed, nbytes, st))

    def forward(self, w: torch.Tensor, n_run: int, out: torch.Tensor = None, want_act: bool = True, want_rgb: bool = False):
        """Layers 0 .. n_run-1 for dlatents ``w`` [n, dlatent] (one latent for every layer) or [Lw, n, dlatent] (layer l reads
        latent l).  Returns (output of layer n_run-1 as fp32 NHWC rows [n, res*res*cout] or None, image as fp32 NHWC
        [n, res, res, 3] or None; the image needs n_run == n_layers).  ``out`` may be a row-strided 2-D view, e.g. the batch rows
        of the large-d IPCA buffer."""
        lib = load()
        w3 = self._latents(w, self.dlatent)
        Lw, n = int(w3.shape[0]), int(w3.shape[1])
        act, rgb = self._outputs(n, n_run, out, want_act, want_rgb, w.device)
        if n == 0:
            return act, rgb
        ws = scratch.get("stylegan", lib.gsb_stylegan_workspace_bytes(self.desc, n_run, n), w.device)
        with torch.cuda.device(w.device), instrument.section("stylegan"):
            _check(lib.gsb_stylegan_forward(_ptr(self.packed), self.desc, self.n_layers, n_run, self.dlatent, _ptr(w3), Lw, n,
                                            C.c_void_p(act.data_ptr() if act is not None else 0), act.stride(0) if act is not None else 0,
                                            _ptr(rgb), _ptr(ws), ws.numel(), _stream()), "gsb_stylegan_forward")
        instrument.count(1)
        instrument.add_rows("stylegan", n)
        return act, rgb

    def style_width(self, l: int) -> int:
        """Width 2 cout of layer ``l``'s style rows ([s0 | s1] of its StyleMod)."""
        return 2 * self.shapes[l][1]

    def styles(self, w: torch.Tensor, layers):
        """The style-space rows (gsb_stylegan_styles): for dlatents ``w`` as in ``forward``, the StyleMod output [n, 2 cout] of every
        layer in ``layers``.  Returns {layer: rows}.  The launch is the chain's own style GEMM, so the rows are bit-identical to the
        ones ``forward`` consumes."""
        lib = load()
        w3 = self._latents(w, self.dlatent)
        Lw, n = int(w3.shape[0]), int(w3.shape[1])
        layers = sorted(set(int(l) for l in layers))
        assert layers and all(0 <= l < self.n_layers and (Lw == 1 or l < Lw) for l in layers), layers
        S = {l: torch.empty((n, self.style_width(l)), dtype=torch.float32, device=self.device) for l in layers}
        idx = (C.c_int * len(layers))(*layers)
        ptrs = (C.c_void_p * len(layers))(*[S[l].data_ptr() for l in layers])
        with torch.cuda.device(self.device), instrument.section("styles"):
            _check(lib.gsb_stylegan_styles(_ptr(self.packed), self.desc, self.n_layers, self.dlatent, _ptr(w3), Lw, n, idx, len(layers),
                                           ptrs, _stream()), "gsb_stylegan_styles")
        instrument.count(1)
        instrument.add_rows("styles", n)
        return S

    def forward_styled(self, S, n_run: int, out: torch.Tensor = None, want_act: bool = True, want_rgb: bool = False):
        """``forward`` on caller-given styles (gsb_stylegan_forward_styled): ``S[l]`` [n, 2 cout] fp32 for the layers 0 .. n_run-1
        (a list or a dict by layer).  Same outputs as ``forward``."""
        lib = load()
        rows, n = self._style_rows(S, range(n_run))
        act, rgb = self._outputs(n, n_run, out, want_act, want_rgb, self.device)
        if n == 0:
            return act, rgb
        S_run = torch.cat(rows, dim=1).contiguous()              # [n, s_run]: the chain's column order
        ws = scratch.get("stylegan", lib.gsb_stylegan_forward_styled_workspace_bytes(self.desc, n_run, n), self.device)
        with torch.cuda.device(self.device), instrument.section("stylegan"):
            _check(lib.gsb_stylegan_forward_styled(_ptr(self.packed), self.desc, self.n_layers, n_run, self.dlatent, _ptr(S_run), n,
                                                   C.c_void_p(act.data_ptr() if act is not None else 0),
                                                   act.stride(0) if act is not None else 0, _ptr(rgb), _ptr(ws), ws.numel(), _stream()),
                   "gsb_stylegan_forward_styled")
        instrument.count(1)
        instrument.add_rows("stylegan", n)
        return act, rgb

    def _status(self, flags):
        return load().gsb_stylegan_status(_ptr(self.packed), self.desc, self.n_layers, self.dlatent, flags)


def _f32_dev(t, what):
    assert t.is_cuda and t.dtype == torch.float32 and t.is_contiguous(), f"{what}: contiguous fp32 device tensor expected"
    return C.c_void_p(t.data_ptr())


def biggan_conv(x, n, cin, res_in, ksize, weight, cout, out, ldx=None, ldo=None, upsample=False, bn=None, w_sample_stride=0,
                bias=None, alpha=1.0, res=None, ldres=None, res_upsample=False):
    """One gsb_biggan_conv_forward launch (csrc/biggan.cu): implicit-GEMM conv of NHWC ``x`` (``n`` samples at res_in^2 pixels with
    pixel stride ``ldx``) with ``weight`` [ksize^2 cin, cout] into ``out``; ``bn`` = (mean [cin], scale [n, cin], offset [n, cin])
    is the BatchNorm + ReLU applied to the operand, ``res`` the residual added after ``alpha * (conv + bias)``."""
    d = BigGANConvDesc()
    d.x, d.ldx, d.cin, d.res_in, d.upsample, d.ksize = x.data_ptr(), ldx or cin, cin, res_in, int(upsample), ksize
    if bn is not None:
        d.bn_mean, d.bn_scale, d.bn_offset = (_f32_dev(t, "biggan_conv bn").value for t in bn)
    d.weight, d.w_sample_stride, d.cout = _f32_dev(weight, "biggan_conv weight").value, w_sample_stride, cout
    d.bias = _f32_dev(bias, "biggan_conv bias").value if bias is not None else None
    d.alpha = alpha
    if res is not None:
        d.res, d.ldres, d.res_upsample = res.data_ptr(), ldres or cout, int(res_upsample)
    d.out, d.ldo = out.data_ptr(), ldo or cout
    for t in (x, out) + ((res,) if res is not None else ()):
        assert t.is_cuda and t.dtype == torch.float32
    with torch.cuda.device(out.device):
        _check(load().gsb_biggan_conv_forward(C.byref(d), n, _stream()), "gsb_biggan_conv_forward")
    instrument.count(1)


def biggan_bn_table(cond, w_scale, w_offset, var, eps, scale_out, offset_out):
    n, cdim = cond.shape
    with torch.cuda.device(cond.device):
        _check(load().gsb_biggan_bn_table(_f32_dev(cond, "cond"), n, cdim, _f32_dev(w_scale, "w_scale"), _f32_dev(w_offset, "w_offset"),
                                          _f32_dev(var, "var"), float(eps), var.numel(), _f32_dev(scale_out, "scale"),
                                          _f32_dev(offset_out, "offset"), _stream()), "gsb_biggan_bn_table")
    instrument.count(1)


def biggan_bn_rows(cond, bns):
    """One gsb_biggan_bn_rows launch: for each (w_scale [C, cdim], w_offset [C, cdim]) of ``bns`` (at most 4, the BatchNorms of one
    block), the rows (cond w_scale^T, cond w_offset^T) [n, C] each, in the dot-product order of gsb_biggan_bn_table."""
    n, cdim = cond.shape
    descs = (BigGANBnRowsDesc * len(bns))()
    out = []
    for d, (ws, wo) in zip(descs, bns):
        s, o = (torch.empty((n, ws.shape[0]), dtype=torch.float32, device=cond.device) for _ in range(2))
        d.w_scale, d.w_offset = _f32_dev(ws, "w_scale").value, _f32_dev(wo, "w_offset").value
        d.c, d.scale_rows, d.offset_rows = ws.shape[0], s.data_ptr(), o.data_ptr()
        out.append((s, o))
    with torch.cuda.device(cond.device):
        _check(load().gsb_biggan_bn_rows(_f32_dev(cond, "cond"), n, cdim, C.cast(descs, C.c_void_p), len(bns), _stream()), "gsb_biggan_bn_rows")
    instrument.count(1)
    return out


def _bn_rows_operand(rows, n, c, what):
    """(tensor, row stride) of BatchNorm rows [n, c] or [1, c] (stride 0: the one row applies to every sample)."""
    assert rows.is_cuda and rows.dtype == torch.float32 and rows.dim() == 2 and rows.shape[1] == c and rows.shape[0] in (1, n) \
        and rows.stride(1) == 1, f"{what}: fp32 device rows [{n}, {c}] or [1, {c}] with unit column stride expected"
    return C.c_void_p(rows.data_ptr()), (rows.stride(0) if rows.shape[0] == n and n > 1 else 0)


def biggan_bn_table_rows(scale_rows, offset_rows, var, eps, scale_out, offset_out):
    """gsb_biggan_bn_table_rows: the BatchNorm tables [n, C] from given rows [n, C] (row-strided) or [1, C]."""
    n, c = scale_out.shape
    ps, ls = _bn_rows_operand(scale_rows, n, c, "scale rows")
    po, lo = _bn_rows_operand(offset_rows, n, c, "offset rows")
    with torch.cuda.device(scale_out.device):
        _check(load().gsb_biggan_bn_table_rows(ps, ls, po, lo, n, _f32_dev(var, "var"), float(eps), c, _f32_dev(scale_out, "scale"),
                                               _f32_dev(offset_out, "offset"), _stream()), "gsb_biggan_bn_table_rows")
    instrument.count(1)


def biggan_attn_pool(tpg, n, res, c, phi_t, g):
    with torch.cuda.device(tpg.device):
        _check(load().gsb_biggan_attn_pool(_f32_dev(tpg, "tpg"), n, res, c, _f32_dev(phi_t, "phi_t"), _f32_dev(g, "g"), _stream()),
               "gsb_biggan_attn_pool")
    instrument.count(1)


def biggan_softmax_rows(s, rows, cols):
    with torch.cuda.device(s.device):
        _check(load().gsb_biggan_softmax_rows(_f32_dev(s, "s"), rows, cols, _stream()), "gsb_biggan_softmax_rows")
    instrument.count(1)


def biggan_rgb(x, n, res, c, mean, scale, offset, weight, bias, img):
    with torch.cuda.device(x.device):
        _check(load().gsb_biggan_rgb(_f32_dev(x, "x"), n, res, c, _f32_dev(mean, "mean"), _f32_dev(scale, "scale"),
                                     _f32_dev(offset, "offset"), _f32_dev(weight, "weight"), _f32_dev(bias, "bias"),
                                     _f32_dev(img, "img"), _stream()), "gsb_biggan_rgb")
    instrument.count(1)


def pick_global_signs(rowmax_all: torch.Tensor) -> torch.Tensor:
    """svd_flip across feature shards: rowmax_all [W, c, 2] = per shard (max |.|, its signed value); the sign of the
    global maximum wins, ties go to the lowest shard (= lowest feature index, np.argmax's first-occurrence rule)."""
    idx = torch.argmax(rowmax_all[:, :, 0], dim=0)                      # first maximal shard per row
    val = rowmax_all[idx, torch.arange(rowmax_all.shape[1], device=rowmax_all.device), 1]
    return torch.where(val < 0, -torch.ones_like(val), torch.ones_like(val)).contiguous()


def exchange_rows(stage: torch.Tensor, out: torch.Tensor, world: int, group=None):
    """Row-parallel -> feature-sharded exchange of one IPCA batch (SURVEY.md section 8e).  ``stage`` [q, d]: the q rows
    this rank produced, all d features; ``out`` [world*q, d/world]: every rank's rows for THIS rank's feature block,
    in rank (= sample) order.  One all-to-all; the send side is packed by a strided copy."""
    import torch.distributed as dist
    q, d = stage.shape
    dl = d // world
    assert d % world == 0 and out.shape == (world * q, dl) and out.is_contiguous()
    send = stage.view(q, world, dl).permute(1, 0, 2).contiguous()       # [world, q, dl]: block s goes to rank s
    dist.all_to_all_single(out.view(world, q, dl), send, group=group)
    return out


class DeviceMemoryError(NativeError, MemoryError):
    """A planned allocation does not fit the device's free memory (raised before anything is allocated or launched)."""


def check_device_memory(nbytes: int, device, what: str):
    """Raises DeviceMemoryError if ``nbytes`` exceed the free memory of ``device`` (blocks cached by torch's allocator count
    as free)."""
    dev = require_cuda(device)
    free, total = torch.cuda.mem_get_info(dev)
    free += torch.cuda.memory_reserved(dev) - torch.cuda.memory_allocated(dev)
    if int(nbytes) > free:
        raise DeviceMemoryError(f"{what} needs {int(nbytes):,} bytes of device memory, but {dev} has {free:,} of {total:,} "
                                "bytes free; use fewer components or a smaller batch size")


def nhwc_to_nchw_rows(x: torch.Tensor, hw: int, c: int, out: torch.Tensor = None) -> torch.Tensor:
    """Rows [n, hw*c] in NHWC feature order (the producers' order) permuted to NCHW ([n, c*hw], the reference's flattening) on
    the device (gsb_nhwc_to_nchw_rows); bit-exact.  fp32 or fp64; ``x`` and ``out`` may be row-strided and must not overlap."""
    assert x.is_cuda and x.dtype in (torch.float32, torch.float64) and x.dim() == 2 and x.shape[1] == hw * c and x.stride(1) == 1
    n = int(x.shape[0])
    out = torch.empty((n, hw * c), dtype=x.dtype, device=x.device) if out is None else out
    assert out.dtype == x.dtype and out.shape == x.shape and out.stride(1) == 1
    with torch.cuda.device(x.device):
        for r0 in range(0, n, 65535):
            r1 = min(n, r0 + 65535)
            _check(load().gsb_nhwc_to_nchw_rows(C.c_void_p(x[r0:r1].data_ptr()), x.stride(0), C.c_void_p(out[r0:r1].data_ptr()),
                                                out.stride(0), r1 - r0, int(hw),
                                                int(c), x.element_size(), _stream()), "gsb_nhwc_to_nchw_rows")
    instrument.count(-(-n // 65535))
    return out


class BigIPCA:
    """Large-d IncrementalPCA engine (csrc/bigd.cu): the stacked matrix M = [S*Vt; batch; correction] lives in HBM,
    producers write the batch rows in place (``batch_rows``), ``step`` runs one partial_fit.

    ``shard=(rank, world)``: feature-sharded over a torch.distributed job -- this object holds the column block
    d/world of M; ``step`` all-reduces the small-side Gram (fp64, (c+nb+1)^2) and agrees on the svd_flip signs."""

    def __init__(self, d: int, c: int, nb_max: int, device, shard=None, gram: str = None, reserve: int = 0):
        """``reserve``: bytes that must stay free next to the engine (e.g. the synthesis workspace of its producer); the
        constructor raises DeviceMemoryError before it allocates or launches anything if the device cannot hold both."""
        lib = load()
        self.dev = require_cuda(device)
        # small-side Gram kernel: "tc" = tensor cores (wgmma) with a promoted accumulator (gram_tc.cu; default -- measured error vs fp64
        # 1.6e-6 against 2.4e-6 for the fp32 FMA kernel, and 2.1x faster per step), "simt" = fp32 FMA kernel (bigd.cu);
        # widths that are not a multiple of 64 fall back to the FMA kernel inside the library
        gram = gram or os.environ.get("GANSPACE_B200_BIGD_GRAM", "tc")
        if gram not in ("simt", "tc"):
            raise NativeError(f"unknown Gram kernel '{gram}' (simt | tc)")
        self.flags = 1 if gram == "tc" else 0
        self.shard = shard if (shard is not None and shard[1] > 1) else None
        self.d_full = int(d)
        if self.shard is not None:
            if d % (16 * self.shard[1]) != 0:
                raise NativeError(f"feature sharding needs d % (16*world) == 0 (d={d}, world={self.shard[1]})")
            d = d // self.shard[1]
        self.d, self.c, self.nb_max = int(d), int(c), int(nb_max)
        need = BigIPCA.device_bytes(self.d, self.c, self.nb_max, self.flags)
        ws_bytes = lib.gsb_bigd_workspace_bytes(self.d, self.c, self.nb_max, self.flags)
        self.rows = lib.gsb_bigd_rows(self.c, self.nb_max)
        check_device_memory(need + int(reserve), self.dev, f"the large-d IPCA engine (d = {self.d}, {self.c} components, "
                            f"batches of {self.nb_max} rows: {need / 1e9:.2f} GB, plus {int(reserve) / 1e9:.2f} GB for its producer)")
        self.M = torch.empty((self.rows, self.d), dtype=torch.float32, device=self.dev)
        self.state = torch.empty(lib.gsb_bigd_state_bytes(self.d, self.c), dtype=torch.uint8, device=self.dev)
        self.ws = torch.empty(ws_bytes, dtype=torch.uint8, device=self.dev)
        self.batch_mean = torch.zeros(self.d, dtype=torch.float64, device=self.dev)
        self.n_seen = 0
        self.last_nb = 0
        with torch.cuda.device(self.dev):
            _check(lib.gsb_bigd_reset(_ptr(self.state), _ptr(self.M), self.d, self.c, self.nb_max, _stream()), "gsb_bigd_reset")
        t_ptr = lib.gsb_bigd_gram_matrix(_ptr(self.ws), self.d, self.c, self.nb_max)
        off = int(t_ptr) - self.ws.data_ptr()
        self._T = self.ws[off:off + self.rows * self.rows * 8].view(torch.float64)      # small-side Gram [rows, rows]
        self._rowmax = torch.empty((self.c, 2), dtype=torch.float32, device=self.dev)

    @staticmethod
    def device_bytes(d: int, c: int, nb_max: int, flags: int = 1) -> int:
        """Device memory the engine allocates: the stacked matrix M (gsb_bigd_rows x d fp32), state, workspace, batch mean."""
        lib = load()
        ws = lib.gsb_bigd_workspace_bytes(int(d), int(c), int(nb_max), int(flags))
        if ws == 0:
            raise NativeError(f"gsb_bigd_workspace_bytes: {lib.gsb_last_error().decode()}")
        return int(lib.gsb_bigd_rows(int(c), int(nb_max))) * int(d) * 4 + int(lib.gsb_bigd_state_bytes(int(d), int(c))) + ws + 8 * int(d)

    def batch_rows(self, nb: int) -> torch.Tensor:
        assert 1 <= nb <= self.nb_max
        return self.M[self.c:self.c + nb]

    def state_dict(self):
        """What the next step reads: S*Vt (rows [0, c) of M), the fp64 state blob (mean, unnormalised variance, S), n_seen,
        and the last batch's mean and size (for its centred rows)."""
        with torch.cuda.device(self.dev):
            return {"M": _to_host(self.M[:self.c]), "state": _to_host(self.state), "batch_mean": _to_host(self.batch_mean),
                    "n_seen": self.n_seen, "last_nb": self.last_nb}

    def load_state_dict(self, sd):
        """Continue from a ``state_dict`` of an engine of the same (d, c); this engine's nb_max may be larger."""
        with torch.cuda.device(self.dev):
            _load_blob(self.M[:self.c], sd["M"], "BigIPCA.load_state_dict")
            _load_blob(self.state, sd["state"], "BigIPCA.load_state_dict")
            _load_blob(self.batch_mean, sd["batch_mean"], "BigIPCA.load_state_dict")
        self.n_seen, self.last_nb = int(sd["n_seen"]), int(sd["last_nb"])

    def _args(self, nb):
        return (_ptr(self.state), _ptr(self.M), self.d, self.c, self.nb_max, self.n_seen, int(nb), self.flags)

    def gram_only(self, nb: int) -> torch.Tensor:
        """Test hook: phase 1 alone (centres the batch rows!); returns the small-side Gram [rows, rows] fp64."""
        with torch.cuda.device(self.dev):
            _check(load().gsb_bigd_step_gram(*self._args(nb), _ptr(self.batch_mean), _ptr(self.ws), self.ws.numel(), _stream()),
                   "gsb_bigd_step_gram")
        return self._T.view(self.rows, self.rows)

    def step(self, nb: int):
        lib = load()
        tail = (_ptr(self.ws), self.ws.numel(), _stream())
        with torch.cuda.device(self.dev), instrument.section("chain"):
            if self.shard is None:
                _check(lib.gsb_bigd_chain_step(*self._args(nb), _ptr(self.batch_mean), *tail), "gsb_bigd_chain_step")
            else:
                import torch.distributed as dist
                _check(lib.gsb_bigd_step_gram(*self._args(nb), _ptr(self.batch_mean), *tail), "gsb_bigd_step_gram")
                dist.all_reduce(self._T)                                   # small-side Gram summed over the feature shards
                _check(lib.gsb_bigd_step_solve(*self._args(nb), _ptr(self._rowmax), *tail), "gsb_bigd_step_solve")
                allmax = torch.empty((self.shard[1] * self.c, 2), dtype=torch.float32, device=self.dev)
                dist.all_gather_into_tensor(allmax, self._rowmax)          # concatenated along dim 0 in rank order
                signs = pick_global_signs(allmax.view(self.shard[1], self.c, 2))
                _check(lib.gsb_bigd_step_commit(*self._args(nb), _ptr(signs), *tail), "gsb_bigd_step_commit")
        instrument.count(7 + 5 + (2 if self.flags & 1 else 0))
        self.n_seen += int(nb)
        self.last_nb = int(nb)

    def export(self):
        """sklearn's attributes; under feature sharding every rank returns the full-width arrays (one all-gather)."""
        lib = load()
        f64 = dict(dtype=torch.float64, device=self.dev)
        out = {
            "components": torch.empty((self.c, self.d), dtype=torch.float32, device=self.dev),
            "singular_values": torch.empty(self.c, **f64), "mean": torch.empty(self.d, **f64),
            "var": torch.empty(self.d, **f64), "explained_variance": torch.empty(self.c, **f64),
            "explained_variance_ratio": torch.empty(self.c, **f64),
        }
        with torch.cuda.device(self.dev):
            _check(lib.gsb_bigd_export(_ptr(self.state), _ptr(self.M), self.d, self.c, self.n_seen, _ptr(out["components"]),
                                       _ptr(out["singular_values"]), _ptr(out["mean"]), _ptr(out["var"]),
                                       _ptr(out["explained_variance"]), _ptr(out["explained_variance_ratio"]), _stream()),
                   "gsb_bigd_export")
        instrument.count(3)
        if self.shard is not None:
            import torch.distributed as dist
            W = self.shard[1]
            comp = torch.empty((W * self.c, self.d), dtype=torch.float32, device=self.dev)
            dist.all_gather_into_tensor(comp, out["components"])
            out["components"] = comp.view(W, self.c, self.d).permute(1, 0, 2).reshape(self.c, W * self.d).contiguous()
            for k in ("mean", "var"):
                full = torch.empty(W * self.d, **f64)
                dist.all_gather_into_tensor(full, out[k])
                out[k] = full
            # explained_variance_ratio_ = S^2 / sum(var * n) over ALL features (_incremental_pca.py:366-367)
            out["explained_variance_ratio"] = out["singular_values"] ** 2 / (out["var"].sum() * self.n_seen)
        return out

    def gathered(self, local: torch.Tensor) -> torch.Tensor:
        """[n, d_local] column blocks of every rank -> [n, d_full] (identity without sharding)."""
        if self.shard is None:
            return local
        import torch.distributed as dist
        W = self.shard[1]
        local = local.contiguous()
        n, dl = local.shape
        full = torch.empty((W * n, dl), dtype=local.dtype, device=local.device)
        dist.all_gather_into_tensor(full, local)
        return full.view(W, n, dl).permute(1, 0, 2).reshape(n, W * dl).contiguous()


def fbpca_project_omega(Q: torch.Tensor, omega: torch.Tensor) -> torch.Tensor:
    """Q^T Omega [r, l] fp64 for Q [d, r] fp64 and fbpca's test matrix Omega [d, l] fp32 (csrc/rsvd.cu, fp64 tensor cores)."""
    assert Q.is_cuda and Q.dtype == torch.float64 and omega.dtype == torch.float32 and Q.dim() == omega.dim() == 2
    assert omega.device == Q.device and omega.shape[0] == Q.shape[0]
    Q, omega = Q.contiguous(), omega.contiguous()
    (d, r), l = Q.shape, omega.shape[1]
    out = torch.empty((r, l), dtype=torch.float64, device=Q.device)
    with torch.cuda.device(Q.device), instrument.section("fbpca_project_omega"):
        _check(load().gsb_fbpca_project_omega(_ptr(Q), d, r, _ptr(omega), l, _ptr(out), _stream()), "gsb_fbpca_project_omega")
    instrument.count(1)
    return out


class FBPCARankError(NativeError):
    """fbpca's range finder needs data of numerical rank >= l = 2 n_components; the solve met a non-positive pivot."""


class FBPCAPool:
    """Pooled (n, mean, centred scatter) of a sample matrix built from per-group statistics, and the fbpca solve on it
    (csrc/rsvd.cu; small-d engine, 32 <= d <= 1024, d % 32 == 0).  Groups are folded in the order they are passed."""

    def __init__(self, d: int, device):
        lib = load()
        self.dev = require_cuda(device)
        self.d = int(d)
        self.n = 0
        self.state = torch.empty(lib.gsb_fbpca_state_bytes(self.d), dtype=torch.uint8, device=self.dev)
        with torch.cuda.device(self.dev):
            _check(lib.gsb_fbpca_reset(_ptr(self.state), self.d, _stream()), "gsb_fbpca_reset")

    def accumulate(self, rows_per_group: int, means: torch.Tensor, grams: torch.Tensor):
        """Fold G groups: means [G, d], grams [G, d, d] (fp64, device), rows_per_group rows each."""
        means = means.reshape(-1, self.d)
        assert means.dtype == grams.dtype == torch.float64 and grams.numel() == means.shape[0] * self.d * self.d
        assert means.is_contiguous() and grams.is_contiguous()
        g = means.shape[0]
        with torch.cuda.device(self.dev), instrument.section("fbpca_pool"):
            _check(load().gsb_fbpca_accumulate(_ptr(self.state), self.d, g, int(rows_per_group), _ptr(means), _ptr(grams),
                                               _stream()), "gsb_fbpca_accumulate")
        instrument.count(2)
        self.n += g * int(rows_per_group)

    def state_dict(self):
        """The pool so far: its state blob (n, mean, centred scatter) and row count."""
        with torch.cuda.device(self.dev):
            return {"state": _to_host(self.state), "n": self.n}

    def load_state_dict(self, sd):
        with torch.cuda.device(self.dev):
            _load_blob(self.state, sd["state"], "FBPCAPool.load_state_dict")
        self.n = int(sd["n"])

    def add_zero_rows(self, n_zero: int):
        if n_zero <= 0:
            return
        with torch.cuda.device(self.dev), instrument.section("fbpca_pool"):
            _check(load().gsb_fbpca_add_zero_rows(_ptr(self.state), self.d, int(n_zero), _stream()), "gsb_fbpca_add_zero_rows")
        instrument.count(2)
        self.n += int(n_zero)

    def solve(self, c: int, l: int, omega: torch.Tensor = None, raw: bool = False):
        """-> dict(components [c, d], stdev [c], var_ratio [c], mean [d]) as fp64 device tensors.  ``omega`` [d, l] selects the
        randomized branch (None: exact).  Raises FBPCARankError when the data's numerical rank is below l."""
        lib = load()
        f64 = dict(dtype=torch.float64, device=self.dev)
        out = {"components": torch.empty((c, self.d), **f64), "stdev": torch.empty(c, **f64),
               "var_ratio": torch.empty(c, **f64), "mean": torch.empty(self.d, **f64)}
        if omega is not None:
            omega = omega.to(self.dev, torch.float64).contiguous()
            assert omega.shape == (self.d, l)
        ws = scratch.get("fbpca", lib.gsb_fbpca_workspace_bytes(self.d, int(c), int(l)), self.dev)
        with torch.cuda.device(self.dev):
            with instrument.section("fbpca_solve"):
                _check(lib.gsb_fbpca_solve(_ptr(self.state), self.d, int(c), int(l), 1 if raw else 0, _ptr(omega),
                                           _ptr(out["components"]), _ptr(out["stdev"]), _ptr(out["var_ratio"]), _ptr(out["mean"]),
                                           _ptr(ws), ws.numel(), _stream()), "gsb_fbpca_solve")
            flags = C.c_uint(0)
            _check(lib.gsb_fbpca_status(_ptr(self.state), self.d, C.byref(flags), _stream()), "gsb_fbpca_status")
        if flags.value & 1:
            raise FBPCARankError(f"fbpca: the samples have numerical rank below l = {l} (a Cholesky pivot of the range finder "
                                 "was not positive); use fewer components or more varied samples")
        return out
