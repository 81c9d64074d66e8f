"""Parity of each CUDA kernel (called through the C ABI) against the oracle, on seeded inputs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def nat():
    from ganspace_b200 import _native
    _native.load()
    return _native


def test_mt19937_raw_bit_exact(nat, oracle):
    seeds = [1791095845, 5, 0, 2147483646, 4294967295]
    n = 30_000   # > 3 super-blocks of 9984 words
    out = nat.mt19937_raw(seeds, n, "cuda").cpu().numpy().view(np.uint32)
    for i, s in enumerate(seeds):
        assert np.array_equal(out[i], oracle.raw_u32(s, n)), f"seed {s}"


@pytest.mark.parametrize("n", [2, 7, 512, 4993, 512 * 1000])
def test_legacy_normal_matches_numpy_stream(nat, oracle, n):
    seeds = [1791095845, 2135392491, 7]
    out = nat.legacy_normal(seeds, n, "cuda").cpu().numpy()
    for i, s in enumerate(seeds):
        ref = oracle.standard_normal_f32(s, n)
        # integer work (MT19937 + rejection decisions) is bit-exact; fp64 log may differ from glibc by
        # 1 ulp, visible after the float32 cast on ~1e-9 of the elements only
        mism = np.flatnonzero(out[i] != ref)
        assert mism.size <= max(1, n // 1_000_000), f"seed {s}: {mism.size} mismatches of {n}"
        if mism.size:
            assert np.max(np.abs(out[i][mism] - ref[mism]) / np.abs(ref[mism])) < 2e-7


def test_legacy_normal_golden_heads(nat, golden):
    g = golden("mapping_known_answers.npz")
    out = nat.legacy_normal(list(g["head_seeds"]), 64, "cuda").cpu().numpy()
    assert np.array_equal(out, g["heads"])
    tail = nat.legacy_normal([1791095845], 512 * 1000, "cuda").cpu().numpy()[0, -64:]
    assert np.array_equal(tail, g["tail_1791095845_512000"])


def test_truncnorm_matches_scipy(nat):
    from scipy.stats import truncnorm
    for seed in (3, 1791095845):
        ref = truncnorm.rvs(-2, 2, size=(1000, 128), random_state=np.random.RandomState(seed)).astype(np.float32)
        out = nat.legacy_truncnorm([seed], 128 * 1000, -2.0, 2.0, 1.0, "cuda").cpu().numpy().reshape(1000, 128)
        assert np.max(np.abs(out - ref)) < 1e-6


@pytest.mark.parametrize("n", [1, 16, 130, 1000])
def test_mapping_forward_vs_oracle(nat, oracle, mapping_weights, golden, n):
    ws, bs = mapping_weights
    W = torch.tensor(np.stack(ws)).cuda()
    Bv = torch.tensor(np.stack(bs)).cuda()
    pm = nat.PackedMapping(W, Bv, 0.01)
    if n == 16:
        g = golden("mapping_known_answers.npz")
        z, ref = g["z"], g["w"]                      # reference Generator.style output
    else:
        z = oracle.standard_normal_f32(123 + n, 512 * n).reshape(n, 512)
        ref = oracle.mapping_forward(z, ws, bs)
    out = pm.forward(torch.tensor(z).cuda()).cpu().numpy()
    # fp32 FMA vs MKL/OpenBLAS fp32: summation-order differences only
    assert np.max(np.abs(out - ref)) < 2e-5 * max(1.0, np.max(np.abs(ref)))


@pytest.mark.parametrize("n", [1, 130, 1000, 10_000])
def test_mapping_tensor_core_path_vs_simt_and_oracle(nat, oracle, mapping_weights, n):
    """Tensor-core fp16x3-split path (22-bit operands; the tensor core truncates when it aligns addends, so the
    96 accumulation steps per layer leave ~1e-5 relative error against ~5e-7 for the fp32 FMA kernels)."""
    ws, bs = mapping_weights
    pm = nat.PackedMapping(torch.tensor(np.stack(ws)).cuda(), torch.tensor(np.stack(bs)).cuda(), 0.01)
    z = oracle.standard_normal_f32(77 + n, 512 * n).reshape(n, 512)
    zt = torch.tensor(z).cuda()
    simt = pm.forward(zt, force_simt=True).cpu().numpy()
    tc = pm.forward(zt, force_simt=False).cpu().numpy()
    pm.check()
    ref = oracle.mapping_forward(z[:1000], ws, bs)
    scale = np.max(np.abs(ref))
    assert np.max(np.abs(simt[:1000] - ref)) < 2e-5 * scale
    assert np.max(np.abs(tc[:1000] - ref)) < 2e-5 * scale
    assert np.max(np.abs(tc - simt)) < 2e-5 * scale
    # error against an fp64 evaluation: far below single-pass fp16 (2^-12 per operand would give ~1e-3)
    def f64(zz):
        x = zz.astype(np.float64)
        x = x / np.sqrt(np.mean(x * x, axis=1, keepdims=True) + 1e-8)
        for w, b in zip(ws, bs):
            y = x @ (w.astype(np.float64) * np.float64(np.float32((1 / np.sqrt(512)) * 0.01))).T + b * 0.01
            x = np.sqrt(2.0) * np.where(y >= 0, y, 0.2 * y)
        return x
    exact = f64(z[:256])
    e_tc, e_simt = np.abs(tc[:256] - exact).max(), np.abs(simt[:256] - exact).max()
    assert e_simt < 2e-6 * scale and e_tc < 3e-5 * scale, (e_tc, e_simt, scale)


def test_mapping_tensor_core_overflow_is_flagged(nat):
    rng = np.random.RandomState(1)
    ws = [(rng.standard_normal((512, 512)) * 1e7).astype(np.float32) for _ in range(2)]
    bs = [np.zeros(512, np.float32) for _ in range(2)]
    pm = nat.PackedMapping(torch.tensor(np.stack(ws)).cuda(), torch.tensor(np.stack(bs)).cuda(), 0.01)
    pm.forward(torch.tensor(rng.standard_normal((64, 512)).astype(np.float32)).cuda(), force_simt=False)
    with pytest.raises(nat.NativeError, match="fp16 range"):
        pm.check()


def test_mapping_nonzero_bias(nat, oracle):
    rng = np.random.RandomState(0)
    ws = [(rng.standard_normal((512, 512)) * 100).astype(np.float32) for _ in range(3)]
    bs = [(rng.standard_normal(512) * 50).astype(np.float32) for _ in range(3)]
    pm = nat.PackedMapping(torch.tensor(np.stack(ws)).cuda(), torch.tensor(np.stack(bs)).cuda(), 0.01)
    z = rng.standard_normal((77, 512)).astype(np.float32)
    ref = oracle.mapping_forward(z, ws, bs)
    out = pm.forward(torch.tensor(z).cuda()).cpu().numpy()
    assert np.max(np.abs(out - ref)) < 2e-5 * np.max(np.abs(ref))


@pytest.mark.parametrize("n,d", [(2000, 512), (300, 96), (1237, 128), (10000, 512)])
def test_batch_stats_vs_oracle(nat, oracle, n, d):
    rng = np.random.RandomState(n + d)
    X = (rng.standard_normal((n, d)) * (1 + rng.rand(d)) + 3 * rng.standard_normal(d)).astype(np.float32)
    _, m_ref, g_ref = oracle.batch_stats(X)
    m, g = nat.batch_stats(torch.tensor(X).cuda())
    m, g = m.cpu().numpy(), g.cpu().numpy()
    assert np.max(np.abs(m - m_ref)) < 1e-12 * max(1, np.max(np.abs(m_ref))) + 1e-13
    assert np.max(np.abs(g - g.T)) == 0.0
    assert np.max(np.abs(g - g_ref)) < 3e-6 * np.max(np.abs(g_ref))


@pytest.mark.parametrize("n,parts", [(20_000, 4), (512 * 1000, 2), (512 * 4000, 3), (512 * 10_000, 8), (512 * 10_000, 16)])
def test_legacy_normal_split_streams_bit_exact(nat, oracle, n, parts):
    """A stream generated by several CTAs (MT19937 jump-ahead + order-preserving compaction across sub-streams) is
    bit-identical to the one-CTA stream, which is bit-identical to NumPy's RandomState.standard_normal."""
    seeds = [1791095845, 7, 2147483646]
    one = nat.legacy_normal(seeds, n, "cuda", parts=1)
    many = nat.legacy_normal(seeds, n, "cuda", parts=parts)
    torch.cuda.synchronize()
    assert torch.equal(one, many)
    if n <= 512 * 1000:
        for i, s in enumerate(seeds):
            assert np.array_equal(many[i].cpu().numpy(), oracle.standard_normal_f32(s, n))
    assert nat.rng_split_status(len(seeds), n, parts, "cuda") == 0


@pytest.mark.parametrize("groups,nb,d", [(3, 2000, 512), (5, 777, 256), (2, 10000, 512), (4, 300, 96), (2, 64, 1024)])
def test_batch_stats_multi_vs_fp64(nat, groups, nb, d):
    """Several partial_fit groups in one call (tensor-core Gram for d % 128 == 0, fp32 FMA kernels otherwise): every group's
    statistics against an fp64 evaluation; groups with very different scales exercise the per-group operand exponent."""
    rng = np.random.RandomState(groups * nb + d)
    X = (rng.standard_normal((groups * nb, d)) * (1 + rng.rand(d)) + 3 * rng.standard_normal(d)).astype(np.float32)
    for g in range(groups):
        X[g * nb:(g + 1) * nb] *= np.float32(10.0 ** (2 * g - 2))
    xd = torch.tensor(X).cuda()
    m, G = nat.batch_stats_multi(xd, groups, nb)
    m, G = m.cpu().numpy(), G.cpu().numpy()
    for g in range(groups):
        Xg = X[g * nb:(g + 1) * nb].astype(np.float64)
        m_ref = Xg.mean(0)
        Xc = (X[g * nb:(g + 1) * nb] - m_ref.astype(np.float32)).astype(np.float64)     # the kernels centre in fp32
        G_ref = Xc.T @ Xc
        assert np.max(np.abs(m[g] - m_ref)) < 1e-12 * max(1, np.max(np.abs(m_ref))) + 1e-13
        assert np.max(np.abs(G[g] - G[g].T)) == 0.0
        assert np.max(np.abs(G[g] - G_ref)) < 3e-6 * np.max(np.abs(G_ref)), (g, np.max(np.abs(G[g] - G_ref)) / np.max(np.abs(G_ref)))
    # a single group through the one-group entry point gives the same numbers
    m1, G1 = nat.batch_stats(xd[nb:2 * nb])
    assert np.array_equal(m1.cpu().numpy(), m[1]) and np.array_equal(G1.cpu().numpy(), G[1])


@pytest.mark.parametrize("d,c", [(96, 12), (512, 80), (512, 512), (256, 1), (1024, 40)])
def test_sym_eig_top_vs_lapack(nat, d, c):
    rng = np.random.RandomState(d + c)
    B = rng.standard_normal((d, 3 * d)) * (0.97 ** np.arange(d))[:, None]
    A = B @ B.T
    lam, Q = np.linalg.eigh(A)
    lam, Q = lam[::-1][:c], Q[:, ::-1][:, :c].T
    ev, evec = nat.sym_eig_top(torch.tensor(A).cuda(), c)
    ev, evec = ev.cpu().numpy(), evec.cpu().numpy()
    assert np.max(np.abs(ev - lam)) < 1e-12 * lam[0]
    # residual and orthonormality
    R = A @ evec.T - evec.T * ev[None, :]
    assert np.max(np.linalg.norm(R, axis=0)) < 1e-11 * lam[0]
    assert np.max(np.abs(evec @ evec.T - np.eye(c))) < 1e-9
    # sign rule: largest-|.| entry of each row positive
    idx = np.argmax(np.abs(evec), axis=1)
    assert np.all(evec[np.arange(c), idx] > 0)


def test_ipca_chain_vs_sklearn_golden(nat, golden):
    g = golden("ipca_chain_d96_c12.npz")
    Xs = g["X"]
    chain = nat.IPCAChain(96, 12, "cuda")
    for k in range(Xs.shape[0]):
        m, G = nat.batch_stats(torch.tensor(Xs[k]).cuda())
        chain.step(Xs.shape[1], m, G)
        out = {kk: v.cpu().numpy() for kk, v in chain.export().items()}
        comp_ref = g[f"comp_{k}"]
        cos = np.sum(out["components"] * comp_ref, axis=1)
        assert np.min(cos) > 1 - 1e-6, f"step {k}: min signed cosine {np.min(cos)}"
        assert np.allclose(out["singular_values"], g[f"sv_{k}"], rtol=2e-5)
        assert np.allclose(np.sqrt(out["explained_variance"]), g[f"stdev_{k}"], rtol=2e-5)
        assert np.max(np.abs(out["explained_variance_ratio"] - g[f"ratio_{k}"])) < 1e-6
        assert np.allclose(out["mean"], g[f"mean_{k}"], rtol=1e-9, atol=1e-9)
        assert np.allclose(out["var"], g[f"var_{k}"], rtol=1e-5)


def test_ipca_chain_vs_oracle_gram_d512(nat, oracle, mapping_weights):
    ws, bs = mapping_weights
    st = oracle.IPCAState(80)
    chain = nat.IPCAChain(512, 80, "cuda")
    for k in range(4):
        z = oracle.standard_normal_f32(1000 + k, 512 * 2500).reshape(2500, 512)
        X = oracle.mapping_forward(z, ws, bs)
        oracle.ipca_partial_fit(st, X)
        m, G = nat.batch_stats(torch.tensor(X).cuda())
        chain.step(2500, m, G)
    out = {kk: v.cpu().numpy() for kk, v in chain.export().items()}
    cos = np.sum(out["components"] * st.components, axis=1)
    assert np.min(cos) > 0.99999, np.min(cos)
    assert np.max(np.abs(out["explained_variance_ratio"] - st.explained_variance_ratio)) < 1e-6


def test_project_std(nat):
    rng = np.random.RandomState(5)
    X = rng.standard_normal((5000, 512)).astype(np.float32) * 2 + 1
    dirs = rng.standard_normal((80, 512)).astype(np.float32)
    sub = rng.standard_normal(512)
    Xc = (X.astype(np.float64) - sub).astype(np.float32)
    ref = np.dot(dirs, Xc.T).std(axis=1)
    out = nat.project_std(torch.tensor(X).cuda(), torch.tensor(dirs), torch.tensor(sub)).cpu().numpy()
    assert np.allclose(out, ref, rtol=2e-5)
    ref0 = np.dot(dirs, X.T).std(axis=1)
    out0 = nat.project_std(torch.tensor(X).cuda(), torch.tensor(dirs)).cpu().numpy()
    assert np.allclose(out0, ref0, rtol=2e-5)


def test_linreg_accumulate_solve(nat):
    import scipy.linalg
    rng = np.random.RandomState(9)
    n, d, c, L = 3000, 512, 24, 512
    act = rng.standard_normal((n, d)).astype(np.float32)
    comp = np.ascontiguousarray(np.linalg.qr(rng.standard_normal((d, c)))[0].T.astype(np.float32))
    mean = rng.standard_normal(d).astype(np.float32)
    stdev = (1 + rng.rand(c)).astype(np.float32)
    Z = rng.standard_normal((n, L)).astype(np.float32)
    A = ((act - mean) @ comp.T) / stdev
    M_ref = scipy.linalg.lstsq(A, Z, lapack_driver="gelsd")[0]
    acc = nat.LinregAccumulator(c, L, "cuda")
    for s in range(0, n, 1000):
        acc.accumulate(torch.tensor(act[s:s + 1000]).cuda(), torch.tensor(comp).cuda(), torch.tensor(mean).cuda(),
                       torch.tensor(stdev).cuda(), torch.tensor(Z[s:s + 1000]).cuda())
    M, zmean = acc.solve()
    assert np.max(np.abs(M.cpu().numpy() - M_ref)) < 1e-5
    assert np.allclose(zmean.cpu().numpy(), Z.mean(axis=0), atol=1e-6)


def test_linreg_rank_deficient_matches_gelsd_min_norm(nat):
    """Two identical projection directions make A rank-deficient: the reference's gelsd (decomposition.py:133) returns the
    minimum-norm solution; the Cholesky route must notice and the eigen route must reproduce it (ADVICE round 1)."""
    import scipy.linalg
    rng = np.random.RandomState(10)
    n, d, c, L = 2000, 256, 12, 128
    act = rng.standard_normal((n, d)).astype(np.float32)
    comp = np.ascontiguousarray(np.linalg.qr(rng.standard_normal((d, c)))[0].T.astype(np.float32))
    comp[7] = comp[3]                                         # duplicated component -> duplicated column of A
    mean = rng.standard_normal(d).astype(np.float32)
    stdev = np.ones(c, np.float32)
    Z = rng.standard_normal((n, L)).astype(np.float32)
    A = ((act - mean) @ comp.T) / stdev
    M_ref = scipy.linalg.lstsq(A.astype(np.float64), Z.astype(np.float64), lapack_driver="gelsd", cond=1e-4)[0]
    acc = nat.LinregAccumulator(c, L, "cuda")
    acc.accumulate(torch.tensor(act).cuda(), torch.tensor(comp).cuda(), torch.tensor(mean).cuda(), torch.tensor(stdev).cuda(),
                   torch.tensor(Z).cuda())
    M, zmean = acc.solve()
    M = M.cpu().numpy()
    assert acc.rank_deficient_at > 0
    assert np.all(np.isfinite(M)) and np.max(np.abs(M - M_ref)) < 1e-4, np.max(np.abs(M - M_ref))
    assert np.max(np.abs(M[3] - M[7])) < 1e-6                 # minimum norm: the duplicated columns share the weight equally


def test_estimator_accepts_host_arrays_and_cuda_tensors(golden):
    """IPCAEstimator keeps the reference's ndarray interface (estimators.py:68-81) and takes CUDA tensors as is."""
    from ganspace_b200.estimators import get_estimator
    g = golden("ipca_chain_d96_c12.npz")
    Xs = g["X"]
    e_host, e_dev = get_estimator("ipca", 12, 1.0), get_estimator("ipca", 12, 1.0)
    for X in Xs:
        assert e_host.fit_partial(X.copy())                       # float32 ndarray, copied to the device
        assert e_dev.fit_partial(torch.tensor(X).cuda())          # stays in HBM
    ch, sh, rh = e_host.get_components()
    cd, sd, rd = e_dev.get_components()
    assert isinstance(ch, np.ndarray) and ch.shape == (12, 96) and ch.dtype == np.float64
    assert np.allclose(ch, cd, atol=1e-9) and np.allclose(sh, sd, rtol=1e-9) and np.allclose(rh, rd, atol=1e-12)
    k = Xs.shape[0] - 1
    assert np.min(np.sum(ch * g[f"comp_{k}"], axis=1)) > 1 - 1e-6
    assert int(e_host.transformer.n_samples_seen_) == Xs.shape[0] * Xs.shape[1]
    assert e_host.transformer.mean_.shape == (96,)
    # first batch smaller than n_components: sklearn raises ValueError -> fit_partial reports False
    assert get_estimator("ipca", 12, 1.0).fit_partial(Xs[0][:5].copy()) is False


def test_estimator_fit_runs_sklearn_batching(golden):
    from ganspace_b200.estimators import get_estimator
    from sklearn.decomposition import IncrementalPCA
    g = golden("ipca_chain_d96_c12.npz")
    X = np.concatenate(list(g["X"]), axis=0)
    est = get_estimator("ipca", 12, 1.0)
    est.fit(X)
    ref = IncrementalPCA(12, whiten=False, batch_size=max(100, 24)).fit(X)
    comp, stdev, ratio = est.get_components()
    assert np.min(np.sum(comp * ref.components_, axis=1)) > 1 - 1e-6
    assert np.allclose(stdev, np.sqrt(ref.explained_variance_), rtol=2e-5)
