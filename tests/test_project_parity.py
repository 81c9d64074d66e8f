"""The bars of tests/project_parity.py separate a correct csrc/project.cu from a subtly wrong one (CPU only).

The NumPy model of the kernels' tiling (64-row x 32-component tiles, 32-feature steps, feature slabs summed in order,
256-row normal-equation slabs) runs the driver's call shape -- 20 rows per call -- at a width that splits and ends in a short
slab and a partly filled 32-feature chunk (d = 8192 + 16, two slabs), and a 100-row call shape that spans two row tiles.
Without a defect it stays under a quarter of every bar the GPU tests apply (DEFECT_FREE_MARGIN); each planted defect lands
at least 10x over the bar of every level named in its row -- A^T A and A^T Z for the coordinate defects, A^T Z and M for the
two that leave A^T A unchanged (a call's A^T Z lost, a call's rows permuted), z_mean for the column means."""
import numpy as np
import pytest

import project_parity as pp

D, SPLITS, C, L = 8192 + 16, 2, 40, 100


def _case(rows, calls, seed=0):
    rng = np.random.RandomState(seed)
    n = rows * calls
    act = rng.standard_normal((n, D)).astype(np.float32)
    comp = np.ascontiguousarray(np.linalg.qr(rng.standard_normal((D, C)))[0].T.astype(np.float32))
    mean = (0.1 * rng.standard_normal(D)).astype(np.float32)
    sd = (1 + rng.rand(C)).astype(np.float32)
    A64, absdots = pp.reference_coords(act, comp, mean, sd)
    Z = (0.3 * A64 @ rng.standard_normal((C, L)) + rng.standard_normal((n, L)) + 0.5).astype(np.float32)
    ref = pp.LinregReference(A64, absdots, Z, sd, D, SPLITS, rows)
    return act, Z, comp, mean, sd, ref


_CASES = {}

# How far under each bar the defect-free model must land.  Measured: coordinates 1.5 %, A^T A and A^T Z under 1 %, M about
# 0.01 % (its componentwise bound adds |G^+| and |M| terms whose signs would cancel, on top of the coordinate bar's own
# sqrt(m) slack), z_mean up to 12 % (fp32 partial sums that grow linearly with a non-zero column mean).
DEFECT_FREE_MARGIN = {"AtA": 0.02, "AtZ": 0.02, "M": 0.01, "z_mean": 0.25}


def _cached(rows, calls):
    if (rows, calls) not in _CASES:
        _CASES[rows, calls] = _case(rows, calls)
    return _CASES[rows, calls]


def test_slab_arithmetic():
    assert pp.slab_len(D, 2) == 4128 and D - pp.slab_len(D, 2) == 4080          # ragged: the last slab is short
    assert pp.slab_len(32768, 8) == 4096 and pp.slab_len(524288, 64) == 8192
    assert pp.slab_len(100, 1) == 128 and pp.coord_terms(100, 1) == 101


@pytest.mark.parametrize("rows,calls", [(20, 4), (100, 2)])
def test_defect_free_model_is_far_under_every_bar(rows, calls):
    act, Z, comp, mean, sd, ref = _cached(rows, calls)
    reports = ref.reports(*pp.model_run(act, Z, comp, mean, sd, rows, SPLITS), f"{rows} rows / call")
    for level, r in reports.items():
        print(f"[project parity] {r}")
        assert r.ratio < DEFECT_FREE_MARGIN[level], str(r)
    # the per-coordinate bar itself, on the first call
    A = pp.model_coords(act[:rows], comp, mean, sd, SPLITS)
    r = pp.Report("coordinates", A, ref.A[:rows], ref.E[:rows])
    print(f"[project parity] {r}")
    assert r.ratio < 0.02, str(r)


@pytest.mark.parametrize("defect,rows,calls,levels", [
    ("drop_last_slab", 20, 4, "AtA+AtZ"),
    ("slab_twice", 20, 4, "AtA+AtZ"),
    ("drop_last_chunk", 20, 4, "AtA+AtZ"),
    ("row_tile_alias", 100, 2, "AtA+AtZ"),
    ("stdev_shift", 20, 4, "AtA+AtZ"),
    ("zmean_short", 20, 4, "z_mean"),
    ("atz_call_missing", 20, 4, "AtZ+M"),        # A^T A and z_mean are intact: only A^T Z and M can see it
    ("rows_permuted", 20, 4, "AtZ+M"),           # A^T A is invariant under a row permutation
])
def test_planted_defect_is_ten_times_over_its_bar(defect, rows, calls, levels):
    act, Z, comp, mean, sd, ref = _cached(rows, calls)
    reports = ref.reports(*pp.model_run(act, Z, comp, mean, sd, rows, SPLITS, defect), defect)
    for r in reports.values():
        print(f"[project parity] {r}")
    for lv in levels.split("+"):
        assert reports[lv].ratio >= 10, str(reports[lv])


def test_report_names_the_worst_element():
    ref = np.zeros((3, 4))
    got = ref.copy()
    got[2, 1] = 5.0
    r = pp.Report("x", got, ref, np.ones((3, 4)))
    assert r.ratio == 5.0 and r.worst == (2, 1)
    with pytest.raises(AssertionError):
        pp.check(got, ref, 1.0)
    got[0, 0] = np.nan
    assert pp.Report("nan", got, ref, 1.0).ratio == np.inf
