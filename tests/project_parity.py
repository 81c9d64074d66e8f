"""fp64 parity of csrc/project.cu: bars derived from the inputs, and a NumPy model of the kernels' tiling (test infrastructure,
imported by tests/test_project_gpu.py and tests/test_project_parity.py).

The reference of every comparison is the same operation in fp64 on the exact fp32 inputs the kernels read: the subtraction
rounded as the kernel rounds it (``act - mean`` in fp32 for the regression; ``fp32(fp64(x) - sub)`` for project_std), then the
dot products, moments, A^T A, A^T Z and column sums in fp64, and scipy's gelsd for M.

Bars are computed per element from the inputs, never picked as round numbers:

* a coordinate (a sequential fp32 fma chain of m terms, then the split sum and the division by stdev) is within
  ``K_COORD * sqrt(m) * U * sum_i |x~_i c_i| / |sd|``;
* A^T A and A^T Z carry those coordinate errors (independent roundings, so they add in quadrature over rows) plus the fp32
  in-slab accumulation of the normal-equation kernel, ``sqrt(rows per slab) * U * sum_r |a_r b_r|``;
* each element of M = G^+ A^T Z moves by at most ``|G^+| (B_AtZ + B_AtA |M|)`` (componentwise first-order perturbation of
  the normal equations; for a rank-deficient G also the part dG moves into the cut null space), plus the fp64 solve;
* a std moves by at most the RMS of its projections' errors (std is 1-Lipschitz in that norm), plus the fp64 cancellation of
  ``E[p^2] - E[p]^2``.

The model (``model_coords`` / ``model_normal_eq``) restates the kernels' arithmetic order: per (row, component) one fp32 fma
chain over the features of a slab, 32 at a time; slabs of a multiple of 32 features; partials summed in slab order; 256-row
normal-equation slabs accumulated in fp32 and added into fp64.  It takes the split count as an argument: the rule that picks
it lives in the library alone (gsb_linreg_feature_splits).  The ``defect`` argument plants one of the mistakes the tiling
invites, so that tests/test_project_parity.py can show that each one lands far over its bar."""
import numpy as np

U = 2.0 ** -24                          # fp32 unit roundoff
EPS64 = 2.0 ** -53                      # fp64 unit roundoff
PJ_ROWS, PJ_COMPS, PJ_K = 64, 32, 32    # csrc/project.cu: rows x components per coordinate tile, features per step
NE_ROWS = 256                           # csrc/project.cu: rows per normal-equation slab

# Constants of the bars.  A factor 2 on the first-order forms leaves room for the fp32 <-> fp64 conversions and the
# division they do not count, and for the second-order terms of the M bound.  How far under each bar the defect-free model
# lands is asserted in tests/test_project_parity.py.
K_COORD = 2.0       # per coordinate / per projection
K_NE = 2.0          # the normal-equation accumulation and the z_mean column sums
K_SOLVE = 2.0       # the componentwise perturbation bound of M
NULL_CUT = 1e-9     # eigenvalues of the fp64 reference G below this share of the largest are an exact duplicate's zero:
                    # the reference G of a full-rank case (cond(A) < 10) has none within 1e-2, a duplicate's is ~1e-16

DEFECTS = ("drop_last_slab", "slab_twice", "drop_last_chunk", "row_tile_alias", "stdev_shift", "zmean_short",
           "atz_call_missing", "rows_permuted")


def slab_len(d, splits):
    """Features per slab of linreg_coords_kernel: ceil(d / splits) rounded up to a multiple of PJ_K."""
    return ((d + splits - 1) // splits + PJ_K - 1) // PJ_K * PJ_K


def coord_terms(d, splits):
    """Sequential fp32 roundings a coordinate sees: its slab's fma chain, the z-ordered sum of the partials, the division."""
    return min(d, slab_len(d, splits)) + (splits if splits > 1 else 0) + 1


# ---------------------------------------------------------------------------------------------------------------------------
# bars
# ---------------------------------------------------------------------------------------------------------------------------
def coord_bar(absdots, sd, m):
    """[n, c] bar of the coordinates; ``absdots`` = |x~| @ |comp|^T in fp64."""
    return K_COORD * np.sqrt(m) * U * absdots / np.abs(np.asarray(sd, np.float64))


def ata_bar(A, E, rows_per_slab):
    """[c, c] bar of A^T A from the fp64 reference coordinates ``A`` [n, c] and their bar ``E``."""
    A2, E2 = A * A, E * E
    return K_NE * (np.sqrt(E2.T @ A2 + A2.T @ E2) + np.sqrt(rows_per_slab) * U * (np.abs(A).T @ np.abs(A)))


def atz_bar(A, E, Z, rows_per_slab):
    """[c, L] bar of A^T Z."""
    return K_NE * (np.sqrt((E * E).T @ (Z * Z)) + np.sqrt(rows_per_slab) * U * (np.abs(A).T @ np.abs(Z)))


def zmean_bar(Z, rows_per_slab):
    """[L] bar of the column means: fp32 sums over a slab's rows, fp64 across slabs."""
    n = Z.shape[0]
    return K_NE * (np.sqrt(rows_per_slab) * U + n * EPS64) * np.abs(Z).sum(axis=0) / n


def m_bar(G, B_ata, B_atz, M):
    """[c, L] bar of M = G^+ AtZ, element by element.

    First order, dM = G^+ (dAtZ - dG M) - P dG G^+ M, with G^+ over the spectrum above NULL_CUT and P the projector on the
    cut null space (zero for a full-rank G; for an exact duplicate, the part dG moves into the direction the min-norm solve
    drops).  With |dAtZ| <= B_atz and |dG| <= B_ata elementwise:  |dM| <= K_SOLVE (|G^+| (B_atz + B_ata |M|) +
    |P| B_ata |G^+ M|).

    The fp64 solve adds Higham's componentwise forward-error bound of a Cholesky solve, gamma_{3c+1} |G^-1| |R^T| |R| |M|
    (Accuracy and Stability of Numerical Algorithms, Thm 10.4), where |R^T| |R| <= s s^T with s_i = sqrt(G_ii) by
    Cauchy-Schwarz (column i of R has norm sqrt(G_ii)); the same form is applied to the eigen route."""
    c = G.shape[0]
    lam, V = np.linalg.eigh(G)
    keep = lam > NULL_CUT * lam[-1]
    Gp = (V[:, keep] / lam[keep]) @ V[:, keep].T
    P = V[:, ~keep] @ V[:, ~keep].T
    aGp, aM = np.abs(Gp), np.abs(M)
    first = aGp @ (B_atz + B_ata @ aM) + np.abs(P) @ (B_ata @ np.abs(Gp @ M))
    gamma = (3 * c + 1) * EPS64 / (1 - (3 * c + 1) * EPS64)
    s = np.sqrt(np.diag(G))
    solve = gamma * np.outer(aGp @ s, s @ aM)
    return K_SOLVE * first + solve


def std_bars(p, absdots, m):
    """([c] bar of the population std, [c] bar of the cancellation alone) from the fp64 projections ``p`` [n, c] and
    |x~| @ |dirs|^T; ``m`` = the features of one fma chain (d)."""
    n = p.shape[0]
    e = K_COORD * np.sqrt(m) * U * absdots
    cancel = np.sqrt(4.0 * n * EPS64 * (p * p).mean(axis=0))
    return np.sqrt((e * e).mean(axis=0)) + cancel, cancel


# ---------------------------------------------------------------------------------------------------------------------------
# the comparator
# ---------------------------------------------------------------------------------------------------------------------------
class Report:
    """max |got - ref| / bar of one comparison, and where it is worst."""

    def __init__(self, name, got, ref, bar):
        got, ref = np.asarray(got, np.float64), np.asarray(ref, np.float64)
        assert got.shape == ref.shape, (name, got.shape, ref.shape)
        bar = np.broadcast_to(np.asarray(bar, np.float64), ref.shape)
        assert (bar > 0).all(), f"{name}: a bar is not positive"
        ratio = np.abs(got - ref) / bar
        ratio = np.where(np.isnan(ratio), np.inf, ratio)
        self.name, self.ratio = name, float(ratio.max())
        self.worst = np.unravel_index(int(ratio.argmax()), ratio.shape) if ratio.size else ()
        self.err = float(np.abs(got - ref).reshape(-1)[int(ratio.argmax())]) if ratio.size else 0.0

    def __str__(self):
        return f"{self.name}: max error / bar {self.ratio:.3g} (error {self.err:.3e} at {tuple(int(i) for i in self.worst)})"


def check(got, ref, bar, name=""):
    """Compare and assert the worst element is under its bar; prints the measurement (pytest -s shows it)."""
    r = Report(name, got, ref, bar)
    print(f"[project parity] {r}")
    assert r.ratio < 1.0, f"{r} exceeds its bar"
    return r


class LinregReference:
    """fp64 reference of gsb_linreg_accumulate / solve over calls of ``rows`` rows, and the bars of A^T A, A^T Z, M and z_mean.
    ``A`` / ``absdots``: the fp64 coordinates (x~ . comp^T / sd) and |x~| . |comp|^T [n_total, c]; ``Z`` [n_total, L]."""

    def __init__(self, A, absdots, Z, sd, d, splits, rows):
        import scipy.linalg
        self.A, self.Z = np.asarray(A, np.float64), np.asarray(Z, np.float64)
        self.E = coord_bar(absdots, sd, coord_terms(d, splits))
        slab_rows = min(rows, NE_ROWS)
        self.G = self.A.T @ self.A
        self.AtZ = self.A.T @ self.Z
        self.z_mean = self.Z.mean(axis=0)
        self.M = scipy.linalg.lstsq(self.A, self.Z, lapack_driver="gelsd")[0]
        self.B_ata = ata_bar(self.A, self.E, slab_rows)
        self.B_atz = atz_bar(self.A, self.E, self.Z, slab_rows)
        self.B_zmean = zmean_bar(self.Z, slab_rows)
        self.B_M = m_bar(self.G, self.B_ata, self.B_atz, self.M)

    def reports(self, AtA, AtZ, M, z_mean, tag=""):
        return {"AtA": Report(f"{tag} A^T A", AtA, self.G, self.B_ata),
                "AtZ": Report(f"{tag} A^T Z", AtZ, self.AtZ, self.B_atz),
                "M": Report(f"{tag} M", M, self.M, self.B_M),
                "z_mean": Report(f"{tag} z_mean", z_mean, self.z_mean, self.B_zmean)}

    def check(self, AtA, AtZ, M, z_mean, tag=""):
        out = self.reports(AtA, AtZ, M, z_mean, tag)
        for r in out.values():
            print(f"[project parity] {r}")
        for r in out.values():
            assert r.ratio < 1.0, f"{r} exceeds its bar"
        return out


def reference_coords(act, comp, mean, sd):
    """fp64 (A, |x~| . |comp|^T) from the fp32 inputs of linreg_coords_kernel (fp32 subtraction, SUBMODE 2)."""
    xt = (np.asarray(act, np.float32) - np.asarray(mean, np.float32)).astype(np.float64)
    c64 = np.asarray(comp, np.float64)
    return xt @ c64.T / np.asarray(sd, np.float64), np.abs(xt) @ np.abs(c64).T


# ---------------------------------------------------------------------------------------------------------------------------
# the model of the kernels
# ---------------------------------------------------------------------------------------------------------------------------
def _fma32(acc, a, b):
    """fp32 fmaf(a, b, acc), elementwise: the fp32 x fp32 product is exact in fp64."""
    return (acc.astype(np.float64) + a.astype(np.float64) * b.astype(np.float64)).astype(np.float32)


def model_coords(act, comp, mean, sd, splits, defect=None):
    """A [n, c] fp32 as linreg_coords_kernel (+ linreg_split_sum_kernel when splits > 1) computes it for one call."""
    act, comp = np.asarray(act, np.float32), np.asarray(comp, np.float32)
    sd = np.asarray(sd, np.float32)
    n, d = act.shape
    c = comp.shape[0]
    xt = act - np.asarray(mean, np.float32)
    slab = slab_len(d, splits)
    parts = []
    for z in range(splits):
        i0, i1 = z * slab, min(d, (z + 1) * slab)
        if defect == "drop_last_chunk" and z == splits - 1 and d % PJ_K:
            i1 = d // PJ_K * PJ_K                            # the partly filled last 32-feature chunk is skipped
        acc = np.zeros((n, c), np.float32)
        if not (defect == "drop_last_slab" and z == splits - 1):
            for i in range(i0, i1):
                acc = _fma32(acc, xt[:, i:i + 1], comp[None, :, i])
        parts.append(acc)
    if defect == "slab_twice":
        parts.append(parts[-1])
    if splits == 1 and defect != "slab_twice":
        s = parts[0]
    else:
        s = np.zeros((n, c), np.float32)
        for p in parts:
            s = s + p
    div = sd.copy()
    if defect == "stdev_shift":
        div[PJ_COMPS - 1] = sd[PJ_COMPS]                     # component 31 reads the stdev of component 32
    A = s / div
    if defect == "rows_permuted":
        A = A[::-1].copy()                                   # every row's coordinates land on another row of the call
    if defect == "row_tile_alias":
        A[:min(PJ_ROWS, n - PJ_ROWS)] = A[PJ_ROWS:2 * PJ_ROWS]   # tile 1's rows land on tile 0's; its own rows stay stale
        A[PJ_ROWS:2 * PJ_ROWS] = 0.0
    return A


def model_normal_eq(A, Z, state=None, skip_atz=False):
    """Adds one call's A^T [A | Z] and sum(Z) into the fp64 ``state`` (AtA, AtZ, sumZ), as linreg_normal_eq_kernel does
    (``skip_atz``: the A^T Z part of the call is lost)."""
    A, Z = np.asarray(A, np.float32), np.asarray(Z, np.float32)
    n, c = A.shape
    L = Z.shape[1]
    if state is None:
        state = (np.zeros((c, c)), np.zeros((c, L)), np.zeros(L))
    AtA, AtZ, sumZ = state
    B = np.concatenate([A, Z], axis=1)
    for r0 in range(0, n, NE_ROWS):
        acc = np.zeros((c, c + L), np.float32)
        zs = np.zeros(L, np.float32)
        for r in range(r0, min(n, r0 + NE_ROWS)):
            acc = _fma32(acc, A[r][:, None], B[r][None, :])
            zs = zs + Z[r]
        AtA += acc[:, :c]
        if not skip_atz:
            AtZ += acc[:, c:]
        sumZ += zs
    return AtA, AtZ, sumZ


def model_run(act, Z, comp, mean, sd, rows, splits, defect=None):
    """(AtA, AtZ, M, z_mean) of LinregAccumulator fed ``act`` / ``Z`` in calls of ``rows`` rows, solved in fp64."""
    state = None
    n = act.shape[0]
    for r0 in range(0, n, rows):
        A = model_coords(act[r0:r0 + rows], comp, mean, sd, splits, defect)
        last = r0 + rows >= n
        state = model_normal_eq(A, Z[r0:r0 + rows], state, skip_atz=defect == "atz_call_missing" and last)
    AtA, AtZ, sumZ = state
    M = np.linalg.solve(AtA, AtZ)
    z_mean = sumZ / (n - rows if defect == "zmean_short" else n)   # n_total short by one call
    return AtA, AtZ, M, z_mean
