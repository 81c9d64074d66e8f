"""csrc/project.cu against fp64 at the launch shapes the decomposition driver uses (the regression feeds 20 rows per call).

Every case compares with the same operation in fp64 on the exact fp32 inputs the kernels read, against bars derived from
those inputs (tests/project_parity.py): A^T A read through gsb_linreg_normal_matrix and A^T Z next to it in the state (the
coordinates and the normal-equation kernel in isolation), M and z_mean from LinregAccumulator.solve (scipy's gelsd on the fp64
coordinates), and project_std's output.  Every regression case also shows that its M bar is tight enough to matter: an M 10 %
off in every element fails it.  Products too large for CPU BLAS are formed in torch.float64 on the device.  Every split of the feature axis the
regression can take (1 to 64) is reached, and asserted through gsb_linreg_feature_splits, the rule the library itself uses.
All inputs are seeded here."""
import ctypes as C

import numpy as np
import pytest
import torch

import project_parity as pp

pytestmark = pytest.mark.gpu

DEV = "cuda"


@pytest.fixture(scope="module")
def nat():
    from ganspace_b200 import _native
    _native.load()
    return _native


def _gen(seed):
    g = torch.Generator(device=DEV)
    g.manual_seed(seed)
    return g


def _randn(g, *shape):
    return torch.randn(*shape, generator=g, device=DEV, dtype=torch.float32)


def _orthonormal_rows(g, c, d):
    q = torch.linalg.qr(torch.randn(d, c, generator=g, device=DEV, dtype=torch.float64))[0]
    return q.T.float().contiguous()


def _normal_equations(nat, acc):
    """(A^T A [c, c], A^T Z [c, L]) fp64 of the accumulator: A^T A where gsb_linreg_normal_matrix points, A^T Z right after
    it at the next 256-byte boundary (the state layout of csrc/project.cu linreg_view)."""
    ptr = nat.load().gsb_linreg_normal_matrix(C.c_void_p(acc.state.data_ptr()), acc.c, acc.L)
    off = int(ptr) - acc.state.data_ptr()
    ata_bytes, atz_bytes = acc.c * acc.c * 8, acc.c * acc.L * 8
    off_z = off + (ata_bytes + 255) // 256 * 256
    AtA = acc.state[off:off + ata_bytes].view(torch.float64).view(acc.c, acc.c).clone()
    AtZ = acc.state[off_z:off_z + atz_bytes].view(torch.float64).view(acc.c, acc.L).clone()
    return AtA, AtZ


class _Linreg:
    """Seeded inputs of one regression: act [rows * calls, d], comp (orthonormal rows), mean, stdev, and Z correlated with the
    coordinates (so M is O(1)).  ``dup`` = (p, q): component p is an exact copy of component q, stdev too."""

    def __init__(self, rows, calls, c, L, d, seed, dup=None, zero_sd=None):
        g = _gen(seed)
        n = rows * calls
        self.rows, self.c, self.L, self.d = rows, c, L, d
        self.act = _randn(g, n, d)
        self.comp = _orthonormal_rows(g, c, d)
        self.mean = 0.1 * _randn(g, d)
        self.sd = 1 + torch.rand(c, generator=g, device=DEV)
        if dup is not None:
            p, q = dup
            self.comp[p] = self.comp[q]
            self.sd[p] = self.sd[q]
        xt = (self.act - self.mean).double()                         # the kernel's fp32 subtraction, widened exactly
        c64 = self.comp.double()
        self.A64 = xt @ c64.T / self.sd.double()
        self.absdots = xt.abs() @ c64.abs().T
        del xt
        W = torch.randn(c, L, generator=g, device=DEV, dtype=torch.float64)
        self.Z = (0.3 * self.A64 @ W + _randn(g, n, L).double() + 0.5).float()
        if zero_sd is not None:
            self.sd[zero_sd] = 0.0

    def run(self, nat):
        acc = nat.LinregAccumulator(self.c, self.L, DEV)
        for r0 in range(0, self.act.shape[0], self.rows):
            acc.accumulate(self.act[r0:r0 + self.rows], self.comp, self.mean, self.sd, self.Z[r0:r0 + self.rows])
        M, z_mean = acc.solve()
        return (acc, *_normal_equations(nat, acc), M, z_mean)

    def reference(self, splits, cond=None):
        ref = pp.LinregReference(self.A64.cpu().numpy(), self.absdots.cpu().numpy(), self.Z.double().cpu().numpy(),
                                 self.sd.cpu().numpy(), self.d, splits, self.rows)
        if cond is not None:               # an exact duplicate: its singular value is fp64 rounding noise, not signal
            import scipy.linalg
            ref.M = scipy.linalg.lstsq(ref.A, ref.Z, lapack_driver="gelsd", cond=cond)[0]
            ref.B_M = pp.m_bar(ref.G, ref.B_ata, ref.B_atz, ref.M)
        return ref


def _splits(nat, rows, c, d):
    return nat.load().gsb_linreg_feature_splits(rows, c, d)


def _check_linreg(nat, case, expect_splits, tag):
    splits = _splits(nat, case.rows, case.c, case.d)
    assert splits == expect_splits, (tag, splits)
    acc, AtA, AtZ, M, z_mean = case.run(nat)
    assert acc.rank_deficient_at == 0, (tag, acc.rank_deficient_at)       # the Cholesky route
    ref = case.reference(splits)
    ref.check(AtA.cpu().numpy(), AtZ.cpu().numpy(), M.cpu().numpy(), z_mean.cpu().numpy(), tag)
    _assert_m_bar_discriminates(ref, tag)
    return ref


def _assert_m_bar_discriminates(ref, tag):
    r = pp.Report(f"{tag} 0.9 M", 0.9 * ref.M, ref.M, ref.B_M)
    print(f"[project parity] {r}")
    assert r.ratio > 1, f"{r}: the M bar would pass an M 10 % off"


# ---------------------------------------------------------------------------------------------------------------------------
# accumulate + solve, widths that never split: every value of every axis, and the tile edges together
# ---------------------------------------------------------------------------------------------------------------------------
NARROW = [  # rows per call, calls, c, L, d
    (1, 40, 1, 100, 96),
    (20, 25, 80, 512, 512),          # the driver's call shape at the mapping width
    (63, 4, 31, 100, 1000),
    (64, 4, 32, 128, 96),
    (65, 4, 33, 100, 1000),          # a second row tile, a second component tile, c + L across a 32-column tile, d % 32 != 0
    (256, 2, 80, 128, 512),
    (257, 2, 33, 512, 1000),         # a second 256-row normal-equation slab holding one row
    (1000, 3, 24, 512, 512),         # n = 3000 in 1000-row calls, c = 24, L = 512
    (1000, 3, 512, 100, 1000),       # the largest c the Cholesky kernel takes
]


@pytest.mark.parametrize("rows,calls,c,L,d", NARROW)
def test_linreg_narrow_widths(nat, rows, calls, c, L, d):
    case = _Linreg(rows, calls, c, L, d, seed=rows * 7 + c)
    assert float(torch.linalg.cond(case.A64)) < 10                          # well clear of the min-norm cut
    _check_linreg(nat, case, 1, f"rows {rows} x {calls}, c {c}, L {L}, d {d}")


# ---------------------------------------------------------------------------------------------------------------------------
# the split-feature coordinates: 20 rows per call, c = 80, L = 512 (config 5's shape).  100 calls: the coordinate bar grows
# with sqrt(slab) * sum |x~ c|, and n_total = 2000 keeps the M bar of the widest case under its "M 10 % off" check
# ---------------------------------------------------------------------------------------------------------------------------
SPLIT_WIDTHS = [(8192, 2), (8192 + 16, 2), (16384, 4), (32768, 8), (65536, 16), (131072, 32), (262144, 64), (524288, 64)]


@pytest.mark.parametrize("d,splits", SPLIT_WIDTHS)
def test_linreg_every_split_count(nat, d, splits):
    case = _Linreg(20, 100, 80, 512, d, seed=d)
    if d % pp.PJ_K:
        assert d - (splits - 1) * pp.slab_len(d, splits) < pp.slab_len(d, splits)          # a short last slab
    _check_linreg(nat, case, splits, f"d {d}")


def test_linreg_long_run_at_conv_width(nat):
    """500 calls x 20 rows at d = 32768 (convs.1): n_total = 10^4, as the driver's regression."""
    case = _Linreg(20, 500, 80, 512, 32768, seed=11)
    _check_linreg(nat, case, 8, "500 x 20 rows, d 32768")


@pytest.mark.parametrize("d", [512] + [d for d, _ in SPLIT_WIDTHS if d % pp.PJ_K == 0])
def test_linreg_is_deterministic(nat, d):
    """Two accumulators fed the same 20-row calls give bit-identical A^T A, A^T Z, M and z_mean, at every split count: each
    split's partial coordinates have their own workspace slot and are summed in a fixed order.  Only the rows with 4 or more
    splits (d >= 16384) can tell this from adding the partials with fp32 atomics into a zeroed A: with 1 split there is no
    sum, and with 2 the two orders of 0 + a + b give the same fp32 result."""
    case = _Linreg(20, 20, 80, 512, d, seed=3 + d)
    splits = _splits(nat, 20, 80, d)
    a = case.run(nat)
    b = case.run(nat)
    for name, x, y in zip(("A^T A", "A^T Z", "M", "z_mean"), a[1:], b[1:]):
        assert torch.equal(x, y), f"d {d} (splits {splits}): {name} differs between two runs"


# ---------------------------------------------------------------------------------------------------------------------------
# solve: the minimum-norm route
# ---------------------------------------------------------------------------------------------------------------------------
MIN_NORM_SHAPE = {12: (2000, 1, 256), 32: (20, 25, 512), 80: (257, 2, 512)}   # c -> rows per call, calls, d


@pytest.mark.parametrize("where", ["first", "middle", "last"])
@pytest.mark.parametrize("c", sorted(MIN_NORM_SHAPE))
def test_linreg_duplicated_column_takes_the_min_norm_route(nat, c, where):
    """An exactly duplicated column makes A rank-deficient: the Cholesky pivot of the later copy fails, and the eigen route
    (the normal matrix padded to a multiple of 32 when c is not one) returns gelsd's minimum-norm solution, which gives the
    two copies equal weights."""
    rows, calls, d = MIN_NORM_SHAPE[c]
    p = {"first": 0, "middle": c // 2, "last": c - 1}[where]
    q = 1 if p == 0 else p - 1
    case = _Linreg(rows, calls, c, 128, d, seed=100 + c + p, dup=(p, q))
    assert _splits(nat, rows, c, d) == 1
    acc, AtA, AtZ, M, z_mean = case.run(nat)
    assert acc.rank_deficient_at == max(p, q) + 1, acc.rank_deficient_at
    ref = case.reference(1, cond=pp.NULL_CUT)
    M = M.cpu().numpy()
    ref.check(AtA.cpu().numpy(), AtZ.cpu().numpy(), M, z_mean.cpu().numpy(), f"c {c}, copy at {p}")
    _assert_m_bar_discriminates(ref, f"c {c}, copy at {p}")
    assert np.max(np.abs(M[p] - M[q])) <= 1e-9 * np.abs(M).max(), np.max(np.abs(M[p] - M[q]))


def test_linreg_zero_stdev_raises(nat):
    case = _Linreg(20, 10, 12, 128, 512, seed=5, zero_sd=4)
    with pytest.raises(nat.NativeError, match="non-finite"):
        case.run(nat)


# ---------------------------------------------------------------------------------------------------------------------------
# project_std
# ---------------------------------------------------------------------------------------------------------------------------
def _std_reference(x, dirs, sub):
    """(fp64 std, [c] bar, [c] cancellation bar) of project_std on the exact inputs (SUBMODE 1: fp32(fp64(x) - sub))."""
    xt = (x.double() - sub).float().double() if sub is not None else x.double()
    d64 = dirs.double()
    p = xt @ d64.T
    absdots = xt.abs() @ d64.abs().T
    del xt
    ref = p.std(dim=0, unbiased=False).cpu().numpy()
    bar, cancel = pp.std_bars(p.cpu().numpy(), absdots.cpu().numpy(), x.shape[1])
    return ref, bar, cancel


STD_SHAPES = [(1, 512, 80), (63, 96, 1), (64, 100, 31), (65, 513, 33), (5000, 512, 80), (5000, 32768, 80), (256, 524288, 80)]


@pytest.mark.parametrize("submode", [0, 1])
@pytest.mark.parametrize("n,d,c", STD_SHAPES)
def test_project_std_shapes(nat, n, d, c, submode):
    g = _gen(n + d + c)
    x = 2 * _randn(g, n, d) + 1
    dirs = _randn(g, c, d)
    sub = torch.randn(d, generator=g, device=DEV, dtype=torch.float64) if submode else None
    ref, bar, _ = _std_reference(x, dirs, sub)
    out = nat.project_std(x, dirs, sub).cpu().numpy()
    pp.check(out, ref, bar, f"project_std n {n} d {d} c {c} submode {submode}")


def test_project_std_row_strided(nat):
    g = _gen(17)
    n, d, c = 300, 1000, 80
    big = _randn(g, n, d + 64)
    x = big[:, :d]
    assert x.stride(0) == d + 64
    dirs = _randn(g, c, d)
    sub = torch.randn(d, generator=g, device=DEV, dtype=torch.float64)
    ref, bar, _ = _std_reference(x, dirs, sub)
    pp.check(nat.project_std(x, dirs, sub).cpu().numpy(), ref, bar, "project_std ld = d + 64")


def test_project_std_uncentred(nat):
    """A mean projection ~10^3 x its spread: the fp64 moments keep E[p^2] - E[p]^2 from cancelling away the variance."""
    g = _gen(19)
    n, d, c = 5000, 512, 80
    dirs = _randn(g, c, d)
    x = 1000 * torch.sign(_randn(g, 1, d)) + _randn(g, n, d)
    ref, bar, _ = _std_reference(x, dirs, None)
    p_mean = (x.double().mean(0) @ dirs.double().T).abs().cpu().numpy()
    assert np.median(p_mean / ref) > 300
    pp.check(nat.project_std(x, dirs).cpu().numpy(), ref, bar, "project_std uncentred")


def test_project_std_identical_rows(nat):
    """Identical rows project identically: the std is the fp64 cancellation residue alone, within its absolute bar."""
    g = _gen(23)
    n, d, c = 1000, 512, 80
    x = _randn(g, 1, d).repeat(n, 1) + 3
    dirs = _randn(g, c, d)
    sub = torch.randn(d, generator=g, device=DEV, dtype=torch.float64)
    ref, _, cancel = _std_reference(x, dirs, sub)
    assert np.all(ref < 1e-9 * cancel.max() + cancel)
    out = nat.project_std(x, dirs, sub).cpu().numpy()
    assert np.all(out <= cancel), (out.max(), cancel.min())


# ---------------------------------------------------------------------------------------------------------------------------
# refusals: the C entry points return their error before launching anything
# ---------------------------------------------------------------------------------------------------------------------------
def _p(t):
    return C.c_void_p(t.data_ptr())


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def test_refusals_before_any_launch(nat):
    lib = nat.load()
    L, n, d = 128, 20, 96
    # c = 513: over the Cholesky kernel's limit
    c = 513
    state = torch.zeros(lib.gsb_linreg_state_bytes(c, L), dtype=torch.uint8, device=DEV)
    act, comp = torch.ones(n, d, device=DEV), torch.ones(c, d, device=DEV)
    mean, sd, z = torch.zeros(d, device=DEV), torch.ones(c, device=DEV), torch.ones(n, L, device=DEV)
    ws = torch.zeros(lib.gsb_linreg_workspace_bytes(n, c, d), dtype=torch.uint8, device=DEV)
    assert lib.gsb_linreg_accumulate(_p(state), c, L, _p(act), n, d, _p(comp), _p(mean), _p(sd), _p(z), _p(ws), ws.numel(),
                                     _stream()) == -1
    M, zm = torch.zeros(c, L, dtype=torch.float64, device=DEV), torch.zeros(L, dtype=torch.float64, device=DEV)
    assert lib.gsb_linreg_solve(_p(state), c, L, n, _p(M), _p(zm), _stream()) == -1
    # a workspace one byte short, without and with a feature split; the split workspace holds A and every partial
    c = 80
    for d, splits in ((512, 1), (32768, 8)):
        assert _splits(nat, n, c, d) == splits
        need = lib.gsb_linreg_workspace_bytes(n, c, d)
        assert need >= n * c * 4 * (1 + (splits if splits > 1 else 0))
        state = torch.zeros(lib.gsb_linreg_state_bytes(c, L), dtype=torch.uint8, device=DEV)
        act, comp = torch.ones(n, d, device=DEV), torch.ones(c, d, device=DEV)
        mean, sd = torch.zeros(d, device=DEV), torch.ones(c, device=DEV)
        ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
        assert lib.gsb_linreg_accumulate(_p(state), c, L, _p(act), n, d, _p(comp), _p(mean), _p(sd), _p(z), _p(ws), need - 1,
                                         _stream()) == -3
        assert b"workspace" in lib.gsb_last_error()
        torch.cuda.synchronize()
        assert int(state.count_nonzero()) == 0 and int(ws.count_nonzero()) == 0
    # project_std: ld < d, and a workspace one byte short
    n, d, c = 64, 100, 31
    x, dirs = torch.ones(n, d, device=DEV), torch.ones(c, d, device=DEV)
    out = torch.full((c,), -1.0, device=DEV)
    need = lib.gsb_project_std_workspace_bytes(c)
    ws = torch.zeros(need, dtype=torch.uint8, device=DEV)
    assert lib.gsb_project_std(_p(x), n, d, d - 1, _p(dirs), c, None, _p(out), _p(ws), need, _stream()) == -1
    assert lib.gsb_project_std(_p(x), n, d, d, _p(dirs), c, None, _p(out), _p(ws), need - 1, _stream()) == -3
    torch.cuda.synchronize()
    assert bool((out == -1).all()) and int(ws.count_nonzero()) == 0
