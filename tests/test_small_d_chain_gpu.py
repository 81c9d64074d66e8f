"""The small-d IPCA chain (csrc/ipca.cu, the orthogonal-iteration step of csrc/subspace.cu and the direct eigensolver of
csrc/eig.cu) against fp64 references after every step, at one shape per branch of the step, with edge batch sizes, at the
iteration cap and under the process-wide switches.

Steps 2..K run the orthogonal iteration ("iterated") where ``subspace_applicable(d, c)`` holds: d in {128, 256, 384, 512},
c % 8 == 0, 8 <= c <= 128, 2c <= 1.25 d and the kernel's shared memory <= 227 KiB.  Its Cholesky runs on a 7 x 5 register
tile per thread (``<7,5>``) when c <= 80 and c + d/16 <= 112, on a 10 x 8 tile (``<10,8>``) otherwise.  Every other shape,
every first step and every step under ``set_chain_mode(True)`` is the direct solve: G built on the device, then ``eig_top``
(tridiag_reg_kernel for d <= 512, with 256 threads for d <= 256; tridiag_kernel<Cols::Cluster> for d <= 640;
tridiag_kernel<Cols::Grid> with d/8 CTAs for d <= 1024).

Three comparisons per step:
  chain only  -- the device's own (mean_b, gram_b) into both the device chain and ``oracle.ipca_gram_step`` (fp64 eigh);
  end to end  -- device statistics + chain against ``oracle.ipca_partial_fit`` (sklearn's SVD form) on the same fp32 rows;
  iterated vs direct -- each iterated case again under ``set_chain_mode(True)``, against the iterated run and the oracles.

The data come from tests/ipca_rows.py (known "gapped" sigma_k^2 = 0.97^k or "power" 1/(k+1) spectra), and for one case from
the StyleGAN2 mapping network (random-init weights, seed 1234), whose spectrum has 0.3 % gaps near component 80.  The
synthetic iterated cases have c - 1 signal directions rather than c + 16: from the second batch on, the alternating mean
adds one more, the top component, and it has to fit in the top c.  With c + 16 signal directions it pushes signal direction
c - 1 out of the top c, across a 3 % gap; the orthogonal iteration gains a factor 0.97 per multiplication there, hits its
cap of 60 iterations and export raises ChainNotConverged (the host then re-runs the direct solve).

Measured on an H100 80GB HBM3 (700 W), worst over every case, step and run, against the bars (>= 4x margin except where
noted):
  chain only, direct solve (FP64)     1 - cos 1.8e-15, S 3.7e-14 (c = d), ratio 7.8e-16, mean 3.3e-16, var 2.8e-15
  chain only, iterated (ITER)         1 - cos 5.6e-10 (edge batches: 4.2e-8), S 3.0e-7 (edge: 5.0e-7), ratio 5.6e-8
  iterated vs direct on the device    the same as chain only, iterated
  end to end (TIGHT)                  1 - cos 7.0e-7, S 1.8e-6, explained variance 3.6e-6, var 2.4e-6; ratio 3.3e-7
                                      ("power", d = 512, c = 32: 3x below the bar, which is the large-d suite's)
  mapping rows beyond the leading 20  1 - cos 8.1e-7 (chain only 7.9e-7)
The ITER bars follow from the residual tolerance of 1e-4: the S error of 3e-7 is second order in the residual, the
components agree to 1e-9.  At GANSPACE_B200_SUBSPACE_TOL=1e-2, six of the nine iterated cases fail them (all but d = 384,
c = 40 and 88, and d = 512, c = 32; the mapping rows by a flipped component 79).  The file runs in about 65 s."""
import json
import os
import subprocess
import sys
import time
from contextlib import contextmanager
from pathlib import Path

import numpy as np
import pytest
import torch
from ipca_rows import Data

pytestmark = pytest.mark.gpu

ROOT = Path(__file__).resolve().parents[1]

COS_TOL = 0.999        # BASELINE.json north_star tolerances
RATIO_TOL = 1e-3
N_LEAD = 20            # leading components of "power" spectra and of the mapping rows held to the tight bars
# 1 - cos, relative S, relative explained variance, absolute ratio; mean: max |error| / max |mean|; var: relative per feature
FP64 = dict(cos=1e-12, sv=1e-12, ev=2e-12, ratio=1e-13, mean=1e-13, var=1e-13)   # chain only, direct solve
ITER = dict(cos=2e-7, sv=2e-6, ev=4e-6, ratio=1e-6, mean=1e-13, var=1e-13)       # chain only, orthogonal iteration
TIGHT = dict(cos=1e-5, sv=2e-5, ev=4e-5, ratio=1e-6, mean=1e-6, var=1e-5)        # end to end against sklearn's SVD form

CASES = {
    #              d     c    nb    steps  spectrum    path of steps 2..K
    "i128_8":    (128,   8,   64,   8,  "gapped"),   # iterated <7,5>: one row tile, one column tile (c = 8)
    "i128_80":   (128,  80,  240,   5,  "gapped"),   # iterated <7,5>: 2c = 1.25 d, the limit
    "i256_16":   (256,  16,  100,   6,  "power"),    # iterated <7,5>: BigGAN-like shape
    "i256_96":   (256,  96,  300,   5,  "gapped"),   # iterated <10,8> (c > 80)
    "i384_40":   (384,  40,  150,   5,  "gapped"),   # iterated <7,5>: three row tiles
    "i384_88":   (384,  88,  300,   5,  "gapped"),   # iterated <10,8>: three row tiles
    "i512_32":   (512,  32,  200,   6,  "power"),    # iterated <7,5>: config 1's shape
    "i512_80":   (512,  80,  300,   6,  "gapped"),   # iterated <7,5>: config 2's shape, c = 80 fills the 7 x 16 rows
    "i512_80m":  (512,  80, 2000,  12,  "mapping"),  # iterated <7,5>: config 2, mapping-network rows
    "d512_88":   (512,  88,  300,   5,  "gapped"),   # direct: the iterated kernel's shared memory exceeds 227 KiB
    "d128_88":   (128,  88,  270,   5,  "gapped"),   # direct: 2c > 1.25 d
    "d384_36":   (384,  36,  120,   5,  "gapped"),   # direct: c % 8 != 0
    "d160_20":   (160,  20,   80,   6,  "gapped"),   # direct: tridiag_reg_kernel with 256 threads, FMA batch statistics
    "d640_80":   (640,  80,  300,   4,  "gapped"),   # direct: tridiag_kernel<Cols::Cluster>
    "d1024_80":  (1024, 80,  300,   4,  "gapped"),   # direct: tridiag_kernel<Cols::Grid>, 128 CTAs
    "d64_64":    (64,   64,  200,   5,  "gapped"),   # direct: c = d (signal rank capped at d)
}


def _nat():
    from ganspace_b200 import _native
    _native.load()
    return _native


def _iterated(name):
    return name.startswith("i")


@contextmanager
def _direct_mode():
    """Every chain step enqueued inside is the direct solve (process-wide; restored on the way out)."""
    nat = _nat()
    nat.set_chain_mode(True)
    try:
        yield
    finally:
        nat.set_chain_mode(False)


def _state_has_subspace_form(d, c):
    """A state in subspace form reserves H, Q and an export workspace: larger than the same state under the direct mode."""
    lib = _nat().load()
    with _direct_mode():
        eigen_form = lib.gsb_ipca_state_bytes(d, c)
    return lib.gsb_ipca_state_bytes(d, c) > eigen_form


def _mapping_rows(nb, steps, weights=None):
    """fp32 rows of the StyleGAN2 mapping network (the mapping_weights fixture: random-init, seed 1234) from the packed
    kernels; the same rows go to the device and to the oracle."""
    from oracle import ganspace_oracle as orc
    nat = _nat()
    ws, bs = weights if weights is not None else orc.mapping_random_init(1234)
    pm = nat.PackedMapping(torch.tensor(np.stack(ws)).cuda(), torch.tensor(np.stack(bs)).cuda(), 0.01)
    rows = []
    for i in range(steps):
        z = np.random.RandomState(3000 + i).standard_normal((nb, 512)).astype(np.float32)
        rows.append(pm.forward(torch.from_numpy(z).cuda()).cpu().numpy())
    pm.check()
    return rows


def _case_rows(name, weights=None):
    d, c, nb, steps, spectrum = CASES[name]
    if spectrum == "mapping":
        return _mapping_rows(nb, steps, weights)
    data = Data(d, c, nb, spectrum, seed=2000 + 7 * d + c, rank=c - 1 if _iterated(name) else None)
    return [data.batch(i, nb) for i in range(steps)]


def _stats(rows):
    """Device batch statistics (n, mean_b fp64, gram_b fp64) of each fp32 batch."""
    nat = _nat()
    out = []
    for X in rows:
        m, G = nat.batch_stats(torch.from_numpy(np.ascontiguousarray(X)).cuda())
        out.append((X.shape[0], m, G))
    return out


def _oracle_state(st):
    return dict(components=st.components.copy(), singular_values=st.singular_values.copy(),
                explained_variance=st.explained_variance.copy(), explained_variance_ratio=st.explained_variance_ratio.copy(),
                mean=np.array(st.mean, copy=True), var=np.array(st.var, copy=True))


def _references(oracle, c, rows, stats):
    """Per step: the fp64 Gram-form chain on the device's statistics, and sklearn's SVD form on the fp32 rows."""
    st_g, st_s = oracle.IPCAState(c), oracle.IPCAState(c)
    gram, svd = [], []
    for X, (n, m, G) in zip(rows, stats):
        oracle.ipca_gram_step(st_g, n, m.cpu().numpy(), G.cpu().numpy())
        oracle.ipca_partial_fit(st_s, X)
        gram.append(_oracle_state(st_g))
        svd.append(_oracle_state(st_s))
    return gram, svd


def _host(out):
    return {k: v.cpu().numpy().astype(np.float64) for k, v in out.items()}


def _run_chain(d, c, stats, export_every=True, side_stream=True):
    """A fresh chain over the statistics; its exports after every step (or only after the last)."""
    chain = _nat().IPCAChain(d, c, "cuda", side_stream=side_stream)
    outs = []
    for k, (n, m, G) in enumerate(stats):
        chain.step(n, m, G)
        if export_every or k == len(stats) - 1:
            outs.append(_host(chain.export()))
    return outs


def _check(got, ref, bars, nt, what, n=None):
    """Components [:nt] at ``bars``, components [:n] (default all) at the BASELINE bars, mean and var at ``bars``.
    Cosines are signed: both sides apply svd_flip.  Returns the worst values seen."""
    n = len(ref["singular_values"]) if n is None else n
    nt = min(nt, n)
    cos = np.sum(got["components"][:n] * ref["components"][:n], axis=1)
    err = dict(cos=np.abs(1 - cos),
               sv=np.abs(got["singular_values"][:n] / ref["singular_values"][:n] - 1),
               ev=np.abs(got["explained_variance"][:n] / ref["explained_variance"][:n] - 1),
               ratio=np.abs(got["explained_variance_ratio"][:n] - ref["explained_variance_ratio"][:n]))
    for k, e in err.items():
        assert e[:nt].max() <= bars[k], (what, k, int(np.argmax(e[:nt])), e[:nt].max())
    assert cos.min() >= COS_TOL, (what, "cos (baseline)", int(np.argmin(cos)), cos.min())
    assert err["ratio"].max() <= RATIO_TOL, (what, "ratio (baseline)", err["ratio"].max())
    mean = np.abs(got["mean"] - ref["mean"]).max() / np.abs(ref["mean"]).max()
    var = np.abs(got["var"] / ref["var"] - 1).max()
    assert mean <= bars["mean"], (what, "mean", mean)
    assert var <= bars["var"], (what, "var", var)
    worst = {k: e[:nt].max() for k, e in err.items()}
    worst.update(mean=mean, var=var)
    if nt < n:
        worst.update(cos_rest=err["cos"][nt:].max(), ratio_rest=err["ratio"][nt:].max())
    return worst


def _merge_worst(acc, w, prefix=""):
    for k, v in w.items():
        acc[prefix + k] = max(acc.get(prefix + k, 0.0), float(v))


def _fmt(worst):
    return {k: f"{v:.1e}" for k, v in worst.items()}


def run_case(name, oracle=None, weights=None, direct_too=False):
    """Case ``name`` through the chain with every check of test_chain_vs_fp64; returns the worst values per run.  Also the
    body of the subprocess runs (the SUBSPACE_* switches are read once per process)."""
    if oracle is None:
        from oracle import ganspace_oracle as oracle
    nat = _nat()
    d, c, nb, steps, spectrum = CASES[name]
    rows = _case_rows(name, weights)
    stats = _stats(rows)
    ref_gram, ref_svd = _references(oracle, c, rows, stats)
    nt = c if spectrum == "gapped" else min(N_LEAD, c)
    runs = {"default": _run_chain(d, c, stats)}
    if direct_too:
        with _direct_mode():
            runs["direct"] = _run_chain(d, c, stats)
    worst = {}
    for mode, outs in runs.items():
        w = worst.setdefault(mode, {})
        exact = mode == "direct" or not _iterated(name)
        for k, got in enumerate(outs):
            what = (name, mode, k)
            # synthetic iterated cases: the first batch has c - 1 signal directions, its c-th component is noise
            n = c - 1 if k == 0 and _iterated(name) and spectrum != "mapping" else c
            # the direct solve is fp64 throughout: every component at the fp64 bars
            _merge_worst(w, _check(got, ref_gram[k], FP64 if exact else ITER, n if exact else nt, what + ("chain",), n), "chain_")
            _merge_worst(w, _check(got, ref_svd[k], TIGHT, nt, what + ("e2e",), n), "e2e_")
            if mode == "direct":
                _merge_worst(w, _check(got, runs["default"][k], ITER, nt, what + ("vs iterated",), n), "vs_iter_")
    assert nat.chain_iterates(d, c) == _iterated(name)
    return {m: {k: float(v) for k, v in w.items()} for m, w in worst.items()}


# ---- 1. every branch of the step against fp64, after every step ---------------------------------------------------------
@pytest.mark.parametrize("name", list(CASES))
def test_chain_vs_fp64(oracle, mapping_weights, name):
    """Chain only (device statistics into both sides) at the FP64 bars for the direct solve and at the ITER bars for the
    orthogonal iteration; end to end against sklearn's SVD form at the TIGHT bars; each iterated case again in direct mode, against
    the iterated run at the ITER bars and against both oracles.  "gapped": every component at the tight bars; "power" and
    the mapping rows: the leading 20, the rest at cos >= 0.999 and ratio within 1e-3.  Measured values: module docstring."""
    d, c = CASES[name][:2]
    # the table checks itself: a state in subspace form is larger exactly when steps 2..K iterate
    assert _state_has_subspace_form(d, c) == _iterated(name), (name, "path")
    t0 = time.time()
    worst = run_case(name, oracle, mapping_weights, direct_too=_iterated(name))
    print(f"\n[{name} d={d} c={c}] {time.time() - t0:.1f}s", {m: _fmt(w) for m, w in worst.items()})


# ---- 2. bit-for-bit invariants ---------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name", [k for k in CASES if k != "i512_80m"])
def test_chain_bit_invariants(name):
    """Exporting after every step ends bit-identical to exporting only at the end (export does not disturb (Q, H)); the
    side-stream chain and ``IPCAChain(side_stream=False)`` give the same bits (the cluster reductions are fixed-order, so two
    runs on the same inputs agree)."""
    d, c = CASES[name][:2]
    stats = _stats(_case_rows(name))
    every = _run_chain(d, c, stats)[-1]
    end = _run_chain(d, c, stats, export_every=False)[-1]
    inline = _run_chain(d, c, stats, export_every=False, side_stream=False)[-1]
    for k in every:
        assert np.array_equal(every[k], end[k]), (name, k, "export every step vs at the end")
        assert np.array_equal(end[k], inline[k]), (name, k, "side stream vs current stream")


# ---- 3. edge batch sizes ---------------------------------------------------------------------------------------------------
EDGE = {"iterated": (512, 32), "direct": (160, 20)}     # tensor-core / FMA batch statistics


@pytest.mark.parametrize("shape", list(EDGE))
def test_edge_batches(oracle, shape):
    """A first batch of exactly c rows (centred rank c - 1: the c-th direction is arbitrary and carries S = 0), then 1 row,
    c - 5 rows, a larger batch of 4c rows, 1 row and a ragged 2c + 7 rows, against both oracles after every step.  The
    1-row batches run the batch statistics on a 1-row group (tensor-core path at d = 512, FMA path at d = 160).  The rows
    have c - 1 signal directions, so the first batch's centred rank is c - 1 in exact arithmetic: the device's c-th S is
    the rounding of its fp32 Gram (measured 1.6e-4 S_0, bar 1e-3 S_0; H100 80GB HBM3, 700 W)."""
    d, c = EDGE[shape]
    assert _nat().chain_iterates(d, c) == (shape == "iterated")
    nbs = (c, 1, c - 5, 4 * c, 1, 2 * c + 7)
    data = Data(d, c, 4 * c, "gapped", seed=4000 + d, rank=c - 1)
    rows = [data.batch(i, 4 * c)[:nb] for i, nb in enumerate(nbs)]
    stats = _stats(rows)
    ref_gram, ref_svd = _references(oracle, c, rows, stats)
    outs = _run_chain(d, c, stats)
    exact = shape == "direct"
    worst = {}
    for k, got in enumerate(outs):
        n = c - 1 if k == 0 else c
        what = (shape, k, nbs[k])
        _merge_worst(worst, _check(got, ref_gram[k], FP64 if exact else ITER, n, what + ("chain",), n), "chain_")
        _merge_worst(worst, _check(got, ref_svd[k], TIGHT, n, what + ("e2e",), n), "e2e_")
        if k == 0:
            s0 = ref_svd[0]["singular_values"][0]
            assert ref_svd[0]["singular_values"][c - 1] <= 3e-5 * s0, ref_svd[0]["singular_values"][c - 1] / s0
            assert got["singular_values"][c - 1] <= 1e-3 * s0, got["singular_values"][c - 1] / s0
            _merge_worst(worst, dict(first_tail_s=got["singular_values"][c - 1] / s0))
            V = got["components"]
            assert np.abs(V @ V.T - np.eye(c)).max() < 1e-9
    print(f"\n[edge {shape} d={d} c={c} nbs={nbs}]", _fmt(worst))


# ---- 4. the iteration cap and the direct fallback --------------------------------------------------------------------------
def test_rank_deficient_hits_cap_then_direct_mode_matches(oracle):
    """Rows in an affine r-dimensional subspace (r = 40 < c = 80, no noise) at d = 512: G has no gap after component c, so
    every step after the first (always the direct solve) hits the iteration cap and ``export`` raises ChainNotConverged,
    which consumes the status.  A fresh chain under ``set_chain_mode(True)`` matches sklearn on the signal components (r on
    the first step, r + 1 from the second on: the mean-correction row adds the direction of the alternating mean); its
    trailing rows are orthonormal and orthogonal to the leading ones (measured 1.3e-15), and its trailing S sit at the
    rounding noise of its statistics: S^2 <= 1e-6 S_0^2 (measured S 1.9e-4 S_0, the fp32 products of the Gram), while
    sklearn's SVD of the fp32 rows leaves S <= 3e-5 S_0 (measured 6.7e-6 S_0).  H100 80GB HBM3, 700 W."""
    nat = _nat()
    d, c, r, nb, steps = 512, 80, 40, 300, 4
    data = Data(d, c, nb, "gapped", seed=5000, rank=r, noise=False)
    rows = [data.batch(i, nb) for i in range(steps)]
    stats = _stats(rows)
    chain = nat.IPCAChain(d, c, "cuda")
    for k, (n, m, G) in enumerate(stats):
        chain.step(n, m, G)
        if k == 0:
            chain.export()
        else:
            with pytest.raises(nat.ChainNotConverged):
                chain.export()
    _, ref_svd = _references(oracle, c, rows, stats)
    with _direct_mode():
        outs = _run_chain(d, c, stats)
    worst = {}
    for k, got in enumerate(outs):
        ref = ref_svd[k]
        s0 = ref["singular_values"][0]
        ks = int(np.sum(ref["singular_values"] > 1e-5 * s0))
        assert ks == (r if k == 0 else r + 1), (k, ks)
        _merge_worst(worst, _check(got, ref, TIGHT, ks, ("rank-deficient", k), ks))
        V = got["components"]
        orth = np.abs(V @ V.T - np.eye(c)).max()
        assert orth < 1e-9, (k, orth)
        # sklearn's SVD works on the fp32 rows; the device's S^2 are eigenvalues of a Gram accumulated from fp32 products
        assert ref["singular_values"][ks:].max() <= 3e-5 * s0, (k, ref["singular_values"][ks:].max() / s0)
        assert got["singular_values"][ks:].max() <= 1e-3 * s0, (k, got["singular_values"][ks:].max() / s0)
        _merge_worst(worst, dict(orth=orth, tail_s=got["singular_values"][ks:].max() / s0,
                                 tail_s_sklearn=ref["singular_values"][ks:].max() / s0))
    nat.check_eig_status("after the direct run")
    print("\n[rank-deficient d=512 c=80 r=40]", _fmt(worst))


def test_direct_mode_switch_between_runs(oracle):
    """What decomposition.compute does after a ChainNotConverged: default -> direct -> default in one process.  Each run
    matches sklearn at the TIGHT bars, and the third run is bit-identical to the first."""
    nat = _nat()
    name = "i384_40"
    d, c = CASES[name][:2]
    rows = _case_rows(name)
    stats = _stats(rows)
    _, ref_svd = _references(oracle, c, rows, stats)
    first = _run_chain(d, c, stats)
    with _direct_mode():
        assert not nat.chain_iterates(d, c)
        direct = _run_chain(d, c, stats)
    assert nat.chain_iterates(d, c)
    third = _run_chain(d, c, stats)
    for run in (first, direct, third):
        for k, got in enumerate(run):
            _check(got, ref_svd[k], TIGHT, c, (name, k), c - 1 if k == 0 else c)
    for k in first[-1]:
        assert np.array_equal(first[-1][k], third[-1][k]), k
    assert not all(np.array_equal(first[-1][k], direct[-1][k]) for k in first[-1])


# ---- 5. switches read once per process: run in a subprocess ---------------------------------------------------------------
def _run_in_subprocess(name, env):
    code = (f"import json, runpy, sys; sys.path[:0] = [{str(ROOT)!r}, {str(ROOT / 'tests')!r}]; "
            f"run_case = runpy.run_path({__file__!r})['run_case']; "
            "from ganspace_b200 import _native\n"
            f"try:\n    out = run_case({name!r})\n"
            "except _native.ChainNotConverged as e:\n    out = {'not_converged': str(e)}\n"
            "print('RESULT ' + json.dumps(out))")
    cmd = [sys.executable] + (["-s"] if sys.flags.no_user_site else []) + ["-c", code]
    p = subprocess.run(cmd, env={**os.environ, **env}, cwd=str(ROOT), capture_output=True, text=True, timeout=900)
    assert p.returncode == 0, (p.stdout[-2000:], p.stderr[-4000:])
    return json.loads([ln for ln in p.stdout.splitlines() if ln.startswith("RESULT ")][-1][len("RESULT "):])


def test_maxit_1_raises_not_converged():
    """GANSPACE_B200_SUBSPACE_MAXIT=1 on well-gapped data: the first iterated step hits the cap and export raises."""
    out = _run_in_subprocess("i512_80", {"GANSPACE_B200_SUBSPACE_MAXIT": "1"})
    assert "not_converged" in out, out


def test_no_double_step_meets_iterated_bars():
    """GANSPACE_B200_SUBSPACE_DBL=0 (never multiply by G twice per iteration) still meets every bar of test_chain_vs_fp64."""
    out = _run_in_subprocess("i512_80", {"GANSPACE_B200_SUBSPACE_DBL": "0"})
    assert "default" in out, out
    print("\n[i512_80, no double step]", _fmt(out["default"]))
