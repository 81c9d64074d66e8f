"""The large-d IPCA engine (csrc/bigd.cu, the small-side eigensolver ``eig_top`` in csrc/eig.cu and the tensor-core Gram in
csrc/gram_tc.cu) against the fp64 restatement of sklearn's IncrementalPCA.partial_fit, at shapes up to config 5's small side
(c = 80, b = 2000: 2081 rows padded to 2112) and at the 4096-row cap, for every tridiagonalisation branch of ``eig_top``.

The data have a known spectrum: X = Z diag(sigma) B^T + noise + shift, with B an orthonormal d x r basis (r = c + 16) and
Z centred with orthogonal columns of norm sqrt(nb), so every batch's centred scatter is exactly diag(sigma^2) nb in B.
The noise floor sits 10x below the smallest signal eigenvalue of a batch.  The mean alternates by +-delta u between batches
(u orthogonal to B, delta^2 = 1.5 sigma_0^2): only the mean-correction row carries that direction into the state, and from
the second batch on it is the top component, 33 % above the next one."""
import time

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

COS_TOL = 0.999        # BASELINE.json north_star tolerances
RATIO_TOL = 1e-3
TIGHT = dict(cos=1e-5, sv=2e-5, ev=4e-5, ratio=1e-6)      # 1 - cos, rtol, rtol, absolute
N_TIGHT_POWER = 20     # leading components of the "power" spectrum held to the tight bars

# np = roundup32(c + nb + 1) decides the eigensolver branch of eig_top (csrc/eig.cu):
#   np <= 512: tridiag_reg_kernel (256 threads for np <= 256); 512 < np <= 640 (the 16-CTA cluster's column blocks fit
#   227 KiB): tridiag_kernel<Cols::Cluster>; np <= 1024: tridiag_kernel<Cols::Grid> with P = np/8 CTAs;
#   np > 1024: tridiag_kernel<Cols::L2>.  Back-transform: <4> for np <= 128, <8> <= 256, <16> <= 512, <32> <= 1024, then
#   backtransform_big_kernel.  The branch of each case below was also seen in torch.profiler traces of its first step; the
#   profiler drops kernel records now and then, so the suite does not assert on them.
CASES = {
    #        c    nb     d     steps     np    tridiagonalisation, back-transform
    "H":  (1,   64,   1024,   6),     # 96    tridiag_reg_kernel (256 threads), <4>; c = 1
    "A":  (8,   100,  1040,   5),     # 128   tridiag_reg_kernel (256 threads), <4>; d % 64 != 0: the tc Gram falls back to FMA
    "B":  (16,  239,  2048,   5),     # 256   tridiag_reg_kernel (256 threads), <8>; n_rows = 2 x 128
    "C":  (24,  300,  18496,  4),     # 352   tridiag_reg_kernel, <16>; d = 289 x 64: ragged K-chunks in both Gram kernels
    "D":  (80,  559,  8192,   4),     # 640   tridiag_kernel<Cols::Cluster> (230,912 B of shared memory), <32>
    "D2": (80,  591,  8192,   4),     # 672   tridiag_kernel<Cols::Grid> (P = 84), <32>
    "E":  (80,  900,  8192,   4),     # 992   tridiag_kernel<Cols::Grid> (P = 124), <32>
    "F":  (80,  2000, 8192,   25),    # 2112  tridiag_kernel<Cols::L2>, backtransform_big_kernel; config 5's c, b and np
    "G":  (128, 3967, 4096,   2),     # 4096  tridiag_kernel<Cols::L2>, backtransform_big_kernel; the cap, c = PJ_CMAX
}
# case F's basis has components whose largest entry lies in the last quarter of the features and whose largest entry in the
# first quarter has the opposite sign, so a feature-sharded step must overrule shard 0's own svd_flip choice for them
F_SPIKES = (2, 5, 9)


class _Data:
    """Batches with a known spectrum ("gapped": sigma_k^2 = 0.97^k; "power": sigma_k^2 = 1/(k+1)), generated on the host
    from fixed RandomState seeds so that the engine and the oracle see the same fp32 rows; batch i depends on (seed, i)."""

    def __init__(self, d, c, nb, spectrum, seed, spikes=()):
        rng = np.random.RandomState(seed)
        self.d, self.seed, self.r = d, seed, c + 16
        k = np.arange(self.r, dtype=np.float64)
        self.sig2 = 0.97 ** k if spectrum == "gapped" else 1.0 / (k + 1.0)
        G = rng.standard_normal((d, self.r)) / np.sqrt(d)
        for i, col in enumerate(spikes):
            G[d - 1 - 97 * i, col] = 0.25                 # global maximum: last feature quarter
            G[11 + 97 * i, col] = -0.15                   # shard 0's maximum, opposite sign
        self.B = np.linalg.qr(G)[0]
        u = rng.standard_normal(d)
        u -= self.B @ (self.B.T @ u)
        self.u = u / np.linalg.norm(u)
        self.shift = 2.0 * rng.standard_normal(d)
        # a batch's noise eigenvalues (Marchenko-Pastur edge nu^2 (sqrt d + sqrt nb)^2) 10x below nb sigma_{r-1}^2
        self.nu = np.sqrt(0.1 * self.sig2[-1] * nb / (np.sqrt(d) + np.sqrt(nb)) ** 2)
        self.delta = np.sqrt(1.5 * self.sig2[0])

    def batch(self, i, nb):
        rng = np.random.RandomState([self.seed, i])
        Z = rng.standard_normal((nb, self.r))
        Z -= Z.mean(axis=0)
        Z = np.linalg.qr(Z)[0] * np.sqrt(nb)              # centred, Z^T Z = nb I
        X = (Z * np.sqrt(self.sig2)) @ self.B.T
        X += self.nu * rng.standard_normal((nb, self.d))
        X += self.shift + (1.0 if i % 2 == 0 else -1.0) * self.delta * self.u
        return X.astype(np.float32)


def _case_data(case, spectrum):
    c, nb, d = CASES[case][:3]
    return _Data(d, c, nb, spectrum, seed=1000 + d + nb + (7 if spectrum == "power" else 0),
                 spikes=F_SPIKES if case == "F" else ())


def _oracle_state(st):
    return dict(components=st.components.copy(), singular_values=st.singular_values.copy(),
                explained_variance=st.explained_variance.copy(), explained_variance_ratio=st.explained_variance_ratio.copy(),
                mean=np.array(st.mean, copy=True), var=np.array(st.var, copy=True))


def _host(out):
    return {k: (v.cpu().numpy() if torch.is_tensor(v) else np.asarray(v)).astype(np.float64) for k, v in out.items()}


def _errors(got, ref):
    """Per-component errors of an export against the oracle: signed cosine (the device applies svd_flip), relative errors of
    S and of the explained variance, absolute error of the ratio."""
    cos = np.sum(got["components"] * ref["components"], axis=1)
    sv = np.abs(got["singular_values"] - ref["singular_values"]) / ref["singular_values"]
    ev = np.abs(got["explained_variance"] - ref["explained_variance"]) / ref["explained_variance"]
    ratio = np.abs(got["explained_variance_ratio"] - ref["explained_variance_ratio"])
    return cos, sv, ev, ratio


def _check(got, ref, spectrum, what):
    """The bars: "gapped" -- every component at the tight bars; "power" -- cos >= 0.999 and ratio within 1e-3 for all, the
    leading N_TIGHT_POWER components at the tight bars.  Returns the worst values seen."""
    cos, sv, ev, ratio = _errors(got, ref)
    nt = len(cos) if spectrum == "gapped" else min(N_TIGHT_POWER, len(cos))
    assert cos[:nt].min() >= 1 - TIGHT["cos"], (what, "cos", int(np.argmin(cos)), cos[:nt].min())
    assert sv[:nt].max() <= TIGHT["sv"], (what, "singular values", int(np.argmax(sv)), sv[:nt].max())
    assert ev[:nt].max() <= TIGHT["ev"], (what, "explained variance", int(np.argmax(ev)), ev[:nt].max())
    assert ratio[:nt].max() <= TIGHT["ratio"], (what, "ratio", int(np.argmax(ratio)), ratio[:nt].max())
    assert cos.min() >= COS_TOL, (what, "cos", int(np.argmin(cos)), cos.min())
    assert ratio.max() <= RATIO_TOL, (what, "ratio", ratio.max())
    assert np.allclose(got["mean"], ref["mean"], rtol=1e-6, atol=1e-6), (what, "mean")
    assert np.allclose(got["var"], ref["var"], rtol=1e-5), (what, "var", np.abs(got["var"] / ref["var"] - 1).max())
    return dict(cos=np.abs(1 - cos).max(), sv=sv.max(), ev=ev.max(), ratio=ratio.max())


def _merge_worst(acc, w):
    for k, v in w.items():
        acc[k] = max(acc.get(k, 0.0), float(v))


# ---- raw C-ABI phases (what BigIPCA.step does under feature sharding, without torch.distributed) ------------------------
def _args(eng, nb):
    from ganspace_b200 import _native
    return (_native._ptr(eng.state), _native._ptr(eng.M), eng.d, eng.c, eng.nb_max, eng.n_seen, int(nb), eng.flags)


def _tail(eng):
    from ganspace_b200 import _native
    return (_native._ptr(eng.ws), eng.ws.numel(), _native._stream())


def _phase_gram(eng, nb):
    from ganspace_b200 import _native
    _native._check(_native.load().gsb_bigd_step_gram(*_args(eng, nb), _native._ptr(eng.batch_mean), *_tail(eng)),
                   "gsb_bigd_step_gram")


def _phase_solve(eng, nb, rowmax=None):
    from ganspace_b200 import _native
    _native._check(_native.load().gsb_bigd_step_solve(*_args(eng, nb), _native._ptr(rowmax), *_tail(eng)), "gsb_bigd_step_solve")


def _phase_commit(eng, nb, signs=None):
    from ganspace_b200 import _native
    _native._check(_native.load().gsb_bigd_step_commit(*_args(eng, nb), _native._ptr(signs), *_tail(eng)), "gsb_bigd_step_commit")
    eng.n_seen += int(nb)
    eng.last_nb = int(nb)


# ---- 1. the engine against fp64 sklearn at every eigensolver branch ---------------------------------------------------
@pytest.mark.parametrize("case,spectrum", [(k, "gapped") for k in CASES] + [("C", "power"), ("E", "power"), ("F", "power")])
def test_engine_vs_fp64_sklearn(oracle, case, spectrum):
    """BigIPCA with both Gram kernels against ``oracle.ipca_partial_fit_small_side`` after every step.  For case A
    (d = 1040) the tensor-core Gram is requested but d % 64 != 0, so the library runs the FMA kernel.

    Measured on an H100 80GB HBM3 (700 W), worst over all cases, steps and both spectra, against the bars:
      |1 - cos|       tc 9.5e-7, FMA 2.4e-6 (case F, 25 steps)      bar 1e-5 (all c "gapped", leading 20 "power")
      S rel. error    tc 1.1e-6, FMA 2.4e-6 (F)                     bar 2e-5 (explained variance: 4.7e-6, bar 4e-5)
      ratio abs.      "gapped" 1.5e-7 (H); "power" 6.5e-7 (F)       bar 1e-6 ("power": 1e-3 beyond the leading 20)
    The Gram's error against fp64 (1.6e-6 tc, 2.4e-6 FMA relative to sqrt(T_ii T_jj), test_gram_tc_matches_fp64) enters
    S, and through Vt = U^T M / S the components' norms, at about that size; with relative gaps of >= 1.8 % between the
    components, the rotation it causes is second order.  The bars leave a margin of 4x or more."""
    from ganspace_b200 import _native
    c, nb, d, steps = CASES[case]
    dev = torch.device("cuda:0")
    data = _case_data(case, spectrum)
    engines = {g: _native.BigIPCA(d, c, nb, dev, gram=g) for g in ("tc", "simt")}
    st = oracle.IPCAState(c)
    worst = {g: {} for g in engines}
    t0 = time.time()
    for i in range(steps):
        X = data.batch(i, nb)
        Xd = torch.from_numpy(X).to(dev)
        for g, eng in engines.items():
            eng.batch_rows(nb).copy_(Xd)
            eng.step(nb)
        oracle.ipca_partial_fit_small_side(st, X)
        ref = _oracle_state(st)
        for g, eng in engines.items():
            _merge_worst(worst[g], _check(_host(eng.export()), ref, spectrum, (case, spectrum, g, i)))
    print(f"\n[{case} {spectrum} c={c} nb={nb} d={d} np={engines['tc'].rows} steps={steps}] {time.time() - t0:.1f}s",
          {g: {k: f"{v:.2e}" for k, v in w.items()} for g, w in worst.items()})


# ---- 2. the three-phase step equals the fused step; the eigensolver on the engine's own matrices -----------------------
@pytest.mark.parametrize("case", ["D", "D2", "E", "F", "G"])
def test_split_step_and_eigensolver_on_engine_gram(case):
    """``gsb_bigd_step_gram`` + ``gsb_bigd_step_solve`` + ``gsb_bigd_step_commit(signs=NULL)`` reproduce
    ``gsb_bigd_chain_step`` bit for bit on two steps (FMA Gram: d <= 8192 is one K-chunk, so every entry of T is one fp64
    add onto zero and T does not depend on the order of the atomics).  The T each split step built -- zero-padded to np,
    rank-deficient on the first step (c zero rows and a zero correction row) -- goes through ``sym_eig_top`` against
    ``numpy.linalg.eigh`` at the bars of test_sym_eig_large."""
    from ganspace_b200 import _native
    c, nb, d = CASES[case][:3]
    dev = torch.device("cuda:0")
    data = _case_data(case, "gapped")
    fused = _native.BigIPCA(d, c, nb, dev, gram="simt")
    split = _native.BigIPCA(d, c, nb, dev, gram="simt")
    worst = {}
    for i in range(2):
        Xd = torch.from_numpy(data.batch(i, nb)).to(dev)
        fused.batch_rows(nb).copy_(Xd)
        split.batch_rows(nb).copy_(Xd)
        fused.step(nb)
        _phase_gram(split, nb)
        T = split._T.view(split.rows, split.rows).clone()
        _phase_solve(split, nb)
        _phase_commit(split, nb)
        assert torch.equal(fused.M, split.M), (case, i, float((fused.M - split.M).abs().max()))
        assert torch.equal(fused.state, split.state), (case, i)

        evals, evecs = _native.sym_eig_top(T, c)
        Th = T.cpu().numpy()
        n = c + nb + 1
        assert np.array_equal(Th, Th.T) and not np.any(Th[n:]) and not np.any(Th[:, n:])
        if i == 0:
            assert not np.any(Th[:c]) and not np.any(Th[c + nb])       # no state and no correction row yet
        ref = np.linalg.eigvalsh(Th)[::-1][:c]
        ev, V = evals.cpu().numpy(), evecs.cpu().numpy()
        lam_err = np.abs(ev - ref).max() / ref[0]
        resid = np.linalg.norm(Th @ V.T - V.T * ev, axis=0).max() / ref[0]
        orth = np.abs(V @ V.T - np.eye(c)).max()
        assert np.allclose(ev, ref, rtol=1e-10, atol=1e-10 * ref[0]), (case, i, lam_err)
        assert resid < 1e-10, (case, i, resid)
        assert orth < 1e-9, (case, i, orth)
        _merge_worst(worst, dict(lam=lam_err, resid=resid, orth=orth))
    print(f"\n[{case} np={split.rows}] eig_top on T vs eigh:", {k: f"{v:.1e}" for k, v in worst.items()})


# ---- 3. batch-size changes through the public API ----------------------------------------------------------------------
@pytest.mark.parametrize("gram", ["tc", "simt"])
def test_batch_size_changes_public_api(oracle, monkeypatch, gram):
    """IPCAEstimator.fit_partial at d = 4096, c = 16 with batches of 703 (nb % 4 = 3: the tail loops of the centring
    kernel), 700 and 300 (rows c + nb + 1 .. np hold an earlier, larger batch), 1000 (the buffer grows and keeps the state)
    and 200, against ``oracle.ipca_partial_fit`` (gesdd) after every call."""
    from ganspace_b200.estimators import get_estimator
    monkeypatch.setenv("GANSPACE_B200_BIGD_GRAM", gram)
    d, c = 4096, 16
    data = _Data(d, c, 700, "gapped", seed=77)
    est = get_estimator("ipca", c, 1.0)
    st = oracle.IPCAState(c)
    worst = {}
    for i, nb in enumerate((703, 700, 300, 1000, 200)):
        X = data.batch(i, nb)
        assert est.fit_partial(torch.from_numpy(X).cuda() if i % 2 else X.copy())
        oracle.ipca_partial_fit(st, X.copy())
        tr = est.transformer
        got = dict(components=tr.components_, singular_values=tr.singular_values_, explained_variance=tr.explained_variance_,
                   explained_variance_ratio=tr.explained_variance_ratio_, mean=tr.mean_, var=tr.var_)
        _merge_worst(worst, _check(_host(got), _oracle_state(st), "gapped", (gram, i, nb)))
        assert int(tr.n_samples_seen_) == st.n_samples_seen
    assert est.transformer.is_large_d and est.transformer._chain.nb_max == 1000
    print(f"\n[batch sizes, {gram}]", {k: f"{v:.2e}" for k, v in worst.items()})


# ---- 4. the feature-sharded step, emulated on one GPU -------------------------------------------------------------------
@pytest.mark.parametrize("W", [2, 4])
def test_feature_sharded_step_on_one_gpu(oracle, W):
    """Case F's data for 4 steps with one BigIPCA(d/W) per feature shard on one device: phase 1 on every shard, the shards'
    T summed here in place of the all-reduce, phase 2, ``pick_global_signs`` on the stacked row maxima, phase 3 with those
    signs.  Some components (F_SPIKES) have their largest entry in the last shard and shard 0's largest entry of the opposite
    sign, so the agreed sign overrules shard 0's own choice on every step.  The assembled export (components concatenated
    over the shards, ratio = S^2 / (sum var n)) matches the unsharded engine to cos >= 1 - 1e-6 and the oracle at the
    "gapped" bars."""
    from ganspace_b200 import _native
    c, nb, d = CASES["F"][:3]
    dl = d // W
    dev = torch.device("cuda:0")
    data = _case_data("F", "gapped")
    full = _native.BigIPCA(d, c, nb, dev, gram="tc")
    shards = [_native.BigIPCA(dl, c, nb, dev, gram="tc") for _ in range(W)]
    st = oracle.IPCAState(c)
    worst = {}
    for i in range(4):
        X = data.batch(i, nb)
        Xd = torch.from_numpy(X).to(dev)
        full.batch_rows(nb).copy_(Xd)
        full.step(nb)
        for s, eng in enumerate(shards):
            eng.batch_rows(nb).copy_(Xd[:, s * dl:(s + 1) * dl])
            _phase_gram(eng, nb)
        T = torch.stack([eng._T for eng in shards]).sum(dim=0)
        for eng in shards:
            eng._T.copy_(T)
        rowmax = torch.empty((W, c, 2), dtype=torch.float32, device=dev)
        for s, eng in enumerate(shards):
            _phase_solve(eng, nb, rowmax[s])
        signs = _native.pick_global_signs(rowmax)
        own0 = torch.where(rowmax[0, :, 1] < 0, -1.0, 1.0)
        overruled = int((signs != own0).sum())
        assert overruled >= len(F_SPIKES), (W, i, overruled)
        for eng in shards:
            _phase_commit(eng, nb, signs)

        parts = [eng.export() for eng in shards]
        got = dict(components=torch.cat([p["components"] for p in parts], dim=1),
                   singular_values=parts[0]["singular_values"], explained_variance=parts[0]["explained_variance"],
                   mean=torch.cat([p["mean"] for p in parts]), var=torch.cat([p["var"] for p in parts]))
        got["explained_variance_ratio"] = got["singular_values"] ** 2 / (got["var"].sum() * shards[0].n_seen)
        got = _host(got)
        ref_full = _host(full.export())
        cos_full = np.sum(got["components"] * ref_full["components"], axis=1)
        assert cos_full.min() >= 1 - 1e-6, (W, i, int(np.argmin(cos_full)), cos_full.min())
        oracle.ipca_partial_fit_small_side(st, X)
        _merge_worst(worst, _check(got, _oracle_state(st), "gapped", (W, i)))
        _merge_worst(worst, dict(cos_vs_unsharded=np.abs(1 - cos_full).max(), overruled=overruled))
    print(f"\n[sharded W={W}]", {k: f"{v:.2e}" for k, v in worst.items()})
