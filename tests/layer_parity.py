"""Per-layer parity of the generator chains against fp64 (test infrastructure, imported by the *_gpu.py family tests and by
tests/test_layer_parity.py).

``check`` compares a chain's layer output with an fp64 restatement of that layer fed the chain's own previous output, on every
element of every sample: per sample max|got - ref| / max|ref_s| must stay under the bar.  A failure names the worst element
(sample, channel, y, x), whether it lies on the one-pixel border ring, and the sample chunk it fell in, so that a defect in the
far border of a gather, in one chunk of samples or in one latent index points at its cause.

The chunk rules restate how each chain splits a batch into launches (the C sources are the authority; the constants mirror
them).  A defect that depends on a sample's position inside its chunk (a chunk-local latent, style or noise index) passes any
test whose batch fits one chunk, so every per-layer test runs a batch that spans two chunks and, where a chunk holds more than
one sample, ends in a partly filled one (``parity_batch``)."""
import numpy as np

# csrc/tap_conv.cuh TAP_CHUNK_ELEMS / progan.cu pg_chunk_samples: fp32 tap-plane elements per GEMM launch
PG_CHUNK_ELEMS = 2048 * 9 * 512
# csrc/tap_conv.cuh TAP_CHUNK_ELEMS / stylegan.cu sg_chunk_samples: elements of the largest per-chunk buffer
SG_CHUNK_ELEMS = 2048 * 9 * 512
# csrc/synthesis.cu SY_CHUNK_ROWS / chunk_samples: GEMM rows (input pixels) per launch
SY_CHUNK_ROWS = 2048
# csrc/biggan.cu BB_BM: output rows (n * H * W, sample-major) per tile of the implicit-GEMM convolutions
BB_BM = 128


def progan_chunk_samples(res_in, ksize, cout):
    """Samples per GEMM launch of a ProGAN block: its Y tap planes (res_in^2 pixels x ksize^2 taps x cout) fill the chunk."""
    return max(1, PG_CHUNK_ELEMS // (res_in * res_in * ksize * ksize * cout))


def stylegan_chunk_samples(res_out, cout, upsample, conv):
    """Samples per chunk of a StyleGAN (v1) layer: the larger of its pre-norm activation (res_out^2 cout) and, for a conv layer,
    its tap planes at the input resolution (res_in^2 x 9 cout padded to a multiple of 32) fills the chunk."""
    res_in = res_out // 2 if upsample else res_out
    per = res_out * res_out * cout
    if conv:
        per = max(per, res_in * res_in * ((9 * cout + 31) // 32 * 32))
    return max(1, SG_CHUNK_ELEMS // per)


def stylegan2_chunk_samples(res_in):
    """Samples per chunk of a StyleGAN2 StyledConv (and of the ToRGB fused into its epilogue): SY_CHUNK_ROWS input pixels."""
    return max(1, SY_CHUNK_ROWS // (res_in * res_in))


def biggan_chunk_samples(res):
    """Samples per 128-row tile of a BigGAN convolution at output resolution ``res`` (1 when one sample spans several tiles)."""
    return max(1, BB_BM // (res * res))


def biggan_tile(s, res):
    """Tile of the first output row of sample ``s`` at resolution ``res``."""
    return s * res * res // BB_BM


def parity_batch(spc):
    """The smallest batch that spans two chunks of ``spc`` samples and, when ``spc`` > 1, ends in a partly filled one."""
    return 2 if spc == 1 else spc + 1


def assert_spans_chunks(n, spc):
    assert n > spc, f"batch of {n} fits one chunk of {spc} samples"
    assert spc == 1 or n % spc != 0, f"batch of {n} fills its last chunk of {spc} samples"


class Report:
    """The outcome of one comparison: ``err`` (worst per-sample relative error), ``per_sample``, ``frob`` (whole-tensor
    relative Frobenius error) and the worst element's coordinates."""

    def __init__(self, name, per_sample, frob, worst, shape, chunk_of):
        self.name, self.per_sample, self.frob, self.shape = name, per_sample, frob, shape
        self.err = float(per_sample.max())
        self.worst = worst                               # (sample, channel, y, x); y, x are None for a flat tensor
        s, _, y, x = worst
        self.on_border = y is not None and (y in (0, shape[2] - 1) or x in (0, shape[3] - 1))
        self.chunk = None if chunk_of is None else int(chunk_of(s))

    def __str__(self):
        s, c, y, x = self.worst
        where = f"sample {s} channel {c}" + ("" if y is None else f" y {y} x {x} ({'border ring' if self.on_border else 'interior'})")
        chunk = "" if self.chunk is None else f", chunk {self.chunk}"
        return (f"{self.name}: max rel err {self.err:.3e} (relative Frobenius {self.frob:.3e}) over {self.shape[0]} samples; "
                f"worst at {where}{chunk}")


def compare(got, ref, name="", chunk_of=None):
    """``got`` / ``ref``: [n, C, H, W] (or [n, C]) arrays, any float type; the comparison runs in fp64.  ``chunk_of``: int
    (samples per chunk) or a callable sample -> chunk index, for the report."""
    got = np.asarray(got, np.float64)
    ref = np.asarray(ref, np.float64)
    assert got.shape == ref.shape, (name, got.shape, ref.shape)
    n = got.shape[0]
    diff = np.abs(got - ref).reshape(n, -1)
    scale = np.abs(ref).reshape(n, -1).max(axis=1)
    assert (scale > 0).all(), f"{name}: a sample's reference is identically zero"
    per_sample = diff.max(axis=1) / scale
    frob = float(np.sqrt(((got - ref) ** 2).sum() / (ref ** 2).sum()))
    s = int(per_sample.argmax())
    idx = np.unravel_index(int(diff[s].argmax()), got.shape[1:])
    worst = (s, int(idx[0]), int(idx[1]), int(idx[2])) if len(idx) == 3 else (s, int(idx[0]), None, None)
    if isinstance(chunk_of, int):
        spc = chunk_of
        chunk_of = lambda i: i // spc
    return Report(name, per_sample, frob, worst, got.shape, chunk_of)


def check(got, ref, bar, name="", chunk_of=None):
    """``compare`` and assert the worst per-sample error is under ``bar``; prints the measurement (pytest -s shows it)."""
    r = compare(got, ref, name, chunk_of)
    print(f"[layer parity] {r}")
    assert r.err < bar, f"{r} exceeds the bar {bar:.1e}"
    return r


def nhwc_to_nchw(rows, n, res, c):
    """A chain's fp32 NHWC rows [n, res*res*c] (device or host tensor) as an fp64 NCHW NumPy array."""
    import torch
    t = torch.as_tensor(rows).reshape(n, res, res, c).permute(0, 3, 1, 2)
    return t.double().cpu().numpy()
