"""CPU-side checks: the C-ABI library loads and exports every declared symbol; host logic mirrors the
reference (Config, plan arithmetic, cache naming, estimator surface, hooks); the product never touches
the oracle."""
import ctypes
import re
from pathlib import Path

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]


def test_library_exports_every_declared_symbol():
    from ganspace_b200 import _native
    header = (ROOT / "include" / "ganspace_b200.h").read_text()
    declared = set(re.findall(r"\b(gsb_[a-z0-9_]+)\s*\(", header))
    assert declared == set(_native.SIGNATURES), declared ^ set(_native.SIGNATURES)
    lib = ctypes.CDLL(str(_native.lib_path()))
    for name in declared:
        assert hasattr(lib, name), name
    assert _native.load().gsb_abi_version() == 2


def test_ctypes_signatures_match_header_prototypes():
    """Every prototype of include/ganspace_b200.h against the ctypes signature the host mirror binds: same arity and
    the same C scalar class per argument (pointer / int / int64 / size_t / double / float) and return type."""
    import ctypes as C
    from ganspace_b200 import _native
    header = (ROOT / "include" / "ganspace_b200.h").read_text()
    header = re.sub(r"/\*.*?\*/", " ", header, flags=re.S)                     # strip comments
    protos = re.findall(r"([A-Za-z_][A-Za-z0-9_ \*]*?)\b(gsb_[a-z0-9_]+)\s*\(([^;{}]*?)\)\s*;", header, flags=re.S)
    assert len(protos) == len(_native.SIGNATURES)

    def classify(decl):
        decl = decl.strip()
        if decl in ("void", ""):
            return None
        if "*" in decl or "gsb_stream_t" in decl:
            return C.c_void_p
        for key, ct in (("int64_t", C.c_int64), ("uint32_t", C.c_uint32), ("size_t", C.c_size_t), ("double", C.c_double), ("float", C.c_float),
                        ("unsigned", C.c_uint), ("int", C.c_int)):
            if re.search(rf"\b{key}\b", decl):
                return ct
        raise AssertionError(f"unclassified C type: {decl!r}")

    for ret, name, args in protos:
        res, argtypes = _native.SIGNATURES[name]
        want = [classify(a) for a in args.split(",")]
        want = [w for w in want if w is not None]
        assert len(want) == len(argtypes), (name, len(want), len(argtypes))
        for i, (w, a) in enumerate(zip(want, argtypes)):
            assert w is a, (name, i, w, a)
        rw = classify(ret)
        if name == "gsb_last_error":
            assert res is C.c_char_p
        else:
            assert rw is res, (name, rw, res)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU behaviour")
def test_no_cpu_fallback():
    from ganspace_b200 import _native
    with pytest.raises(_native.NativeError):
        _native.require_cuda("cuda")
    with pytest.raises(_native.NativeError):
        _native.require_cuda("cpu")
    from ganspace_b200.models import StyleGAN2
    with pytest.raises(_native.NativeError):
        StyleGAN2(torch.device("cpu"), "ffhq", random_init=1234)
    lib = _native.load()
    rc = lib.gsb_ipca_reset(ctypes.c_void_p(256), 512, 80, ctypes.c_void_p(0))
    assert rc == -2 and b"cuda" in lib.gsb_last_error().lower()


def test_product_never_imports_oracle():
    for p in (ROOT / "ganspace_b200").rglob("*.py"):
        txt = p.read_text()
        assert not re.search(r"^\s*(from|import)\s+oracle", txt, re.M), p
        assert "ganspace_oracle" not in txt, p
    for p in (ROOT / "ganspace_b200" / "csrc").glob("*.cu*"):
        assert "oracle/" not in p.read_text(), p


def test_config_defaults_and_flags():
    from ganspace_b200.config import Config
    c = Config()
    assert (c.model, c.layer, c.estimator, c.components, c.n, c.use_w) == ("StyleGAN", "g_mapping", "ipca", 80, 300_000, False)
    assert c.batch_size is None and c.seed is None and c.sparsity == 1.0 and c.sigma == 2.0
    c = Config(model="StyleGAN2", n=10, use_w=True, extra=3)
    assert c.model == "StyleGAN2" and c.n == 10 and c.use_w and c.extra == 3
    c = Config().from_args(["--model", "BigGAN-512", "--class", "husky", "-b", "7", "-c", "3", "-n", "9", "--use_w",
                            "--est", "ipca", "--seed", "4", "--layer", "generator.gen_z"])
    assert (c.model, c.output_class, c.batch_size, c.components, c.n, c.use_w, c.seed) == \
        ("BigGAN-512", "husky", 7, 3, 9, True, 4)
    assert '"custom"' in str(c)


@pytest.mark.parametrize("n,B,c,expect", [
    (10_000, 1_000, 32, (10_000, 2_000, 12_000, 5)),
    (1_000_000, 10_000, 80, (1_000_000, 10_000, 1_010_000, 100)),
    (5_000, 700, 20, (4_900, 2_000, 7_000, 3)),
    (300_000, 20, 80, (300_000, 2_000, 302_000, 150)),
    (9_000, 1_000, 800, (9_000, 2_400, 12_000, 4)),
])
def test_plan_matches_reference_arithmetic(oracle, n, B, c, expect):
    from ganspace_b200 import plan
    p = plan.make_plan(n, B, c)
    assert (p.N, p.NB, p.n_lat, p.K) == expect
    assert (p.N, p.NB, p.n_lat, p.K) == oracle.plan(n, B, c)
    # every group's rows are covered by the generated batches
    for k in range(p.K):
        r0, r1 = p.group_rows(k)
        b0, b1 = p.batches_covering(r0, r1)
        assert b0 * B <= r0 and b1 * B >= r1 and b1 <= p.n_calls


def test_sharding_partitions_groups():
    from ganspace_b200 import plan
    p = plan.make_plan(1_000_000, 10_000, 80)
    for world in (1, 2, 4, 8):
        owned = [[k for k in plan.groups_to_process(p, r, world) if plan.owner(k, world, p.K) == r] for r in range(world)]
        assert sorted(sum(owned, [])) == list(range(p.K))
        for r in range(world):
            assert p.K - 1 in plan.groups_to_process(p, r, world)
        # rounds cover every group once, in order; every rank owns at most ceil(len/world) groups of a round
        rs = plan.rounds(0, p.K, world, 4, 10)
        assert [k for r in rs for k in r] == list(range(p.K)) and len(rs[0]) == min(p.K, 4 * world)
        for rnd in rs:
            for r in range(world):
                own = [k for k in rnd if plan.owner(k, world) == r]
                assert len(own) <= -(-len(rnd) // world)
                assert [(k - rnd[0]) // world for k in own] == list(range(len(own)))
    assert plan.contiguous_runs([0, 1, 2, 5, 6, 9]) == [[0, 1, 2], [5, 6], [9]]
    # a rank's groups need one contiguous set of sample_latent calls (+ the final group's)
    p2 = plan.make_plan(5_000, 700, 20)          # ragged: B does not divide NB
    for world in (1, 2, 3):
        for r in range(world):
            runs = plan.contiguous_runs(plan.groups_to_process(p2, r, world))
            needed, offs = plan.batch_slots(p2, runs)
            assert needed == sorted(set(needed)) and max(needed) < p2.n_calls
            for run, off in zip(runs, offs):
                r0 = p2.group_rows(run[0])[0]
                assert needed[off // p2.B] * p2.B + off % p2.B == r0


def test_estimator_surface_and_cache_name():
    from ganspace_b200.estimators import get_estimator
    est = get_estimator("ipca", 80, 1.0)
    assert est.batch_support and est.get_param_str() == "ipca_c80"
    assert est.transformer.batch_size == 160 and int(est.transformer.n_samples_seen_) == 0
    with pytest.raises(RuntimeError, match="Unknown estimator"):
        get_estimator("nope", 3, 1.0)
    with pytest.raises(RuntimeError):
        get_estimator("pca", 3, 1.0)


def test_get_random_dirs_matches_reference_formula():
    from ganspace_b200.decomposition import get_random_dirs, SEED_RANDOM_DIRS
    d = get_random_dirs(5, 64)
    g = np.random.RandomState(SEED_RANDOM_DIRS).normal(size=(5, 64))
    g /= np.sqrt(np.sum(g ** 2, axis=1, keepdims=True))
    assert d.dtype == np.float32 and np.array_equal(d, g.astype(np.float32))


class _Toy(torch.nn.Module):
    def __init__(self):
        super().__init__()
        self.a = torch.nn.Linear(4, 4)
        self.b = torch.nn.Sequential(torch.nn.ReLU(), torch.nn.Linear(4, 2))

    def forward(self, x):
        return self.b(self.a(x))


def test_instrumented_model_retain_edit_close():
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    torch.manual_seed(0)
    toy = _Toy()
    x = torch.randn(3, 4)
    base = toy(x)
    ax = torch.nn.functional.linear(x, toy.a.weight, toy.a.bias)      # un-hooked value of layer 'a'
    tail = lambda h: torch.nn.functional.linear(torch.relu(h), toy.b[1].weight, toy.b[1].bias)
    inst = InstrumentedModel(toy)
    inst.retain_layer("a")
    assert inst.retained_features()["a"] is None
    out = inst(x)
    assert torch.equal(out, base) and torch.equal(inst.retained_layer("a"), ax)
    inst.edit_layer("a", offset=torch.ones(4))
    assert torch.allclose(inst(x), tail(ax + 1))
    assert torch.equal(inst.retained_layer(), ax)                     # retained before the edit
    inst.edit_layer("a", ablation=1.0, replacement=torch.zeros(4))
    assert torch.allclose(inst(x), tail(torch.ones(3, 4)))            # x*(1-1) + 0*1, then +offset
    inst.remove_edits("a", remove_offset=False)
    assert torch.allclose(inst(x), tail(ax + 1))
    inst.remove_edits()
    assert torch.equal(inst(x), base)
    with pytest.raises(ValueError, match="not found"):
        inst.retain_layer("nope")
    inst.close()
    assert torch.equal(toy(x), base) and not inst.retained_features()


def test_generator_module_tree_and_init_order(golden):
    from ganspace_b200.models import stylegan2
    torch.manual_seed(1234)
    g = stylegan2.Generator(1024, 512, 8)
    names = [n for n, _ in g.named_modules()]
    assert len(names) == 163 and g.n_latent == 18
    for must in ("style", "style.8", "input", "conv1", "to_rgb1", "convs.0", "convs.15", "to_rgbs.7", "convs.4.conv.modulation"):
        assert must in names, must
    gold = golden("mapping_known_answers.npz")
    sd = g.state_dict()
    assert np.allclose([float(sd[f"style.{i + 1}.weight"].double().sum()) for i in range(8)], gold["style_weight_sums"])
    if "synth_param_sums" in gold:
        keys = [str(k) for k in gold["synth_param_keys"]]
        assert np.allclose([float(sd[k].double().sum()) for k in keys], gold["synth_param_sums"])


def test_mt19937_jump_polynomials_match_numpy_state():
    """Host side of the split RNG (csrc/rng_jump.cu): characteristic polynomial by Berlekamp-Massey, x^J mod phi, and the
    jumped state as the XOR of state windows -- against NumPy's generator advanced J words (no GPU needed)."""
    import ctypes as C
    from ganspace_b200 import _native as nat
    lib = nat.load()
    step = int(lib.gsb_legacy_normal_split_step_words(512 * 1000, 4))
    assert step > 0 and step % 624 == 0
    polys = np.zeros((3, 624), np.uint32)
    assert lib.gsb_mt19937_jump_polys(step, 3, polys.ctypes.data_as(C.c_void_p)) == 0
    for seed, j in ((1791095845, 1), (5, 3)):
        st = np.zeros(624, np.uint32)
        assert lib.gsb_mt19937_jump_state_host(seed, polys[j - 1].ctypes.data_as(C.c_void_p), st.ctypes.data_as(C.c_void_p)) == 0
        rs = np.random.RandomState(seed)
        rs.randint(0, 2 ** 32, size=step * j, dtype=np.uint32)          # one word per draw
        _, key, pos = rs.get_state()[:3]
        assert pos == 624 and np.array_equal(key[1:], st[1:]) and (key[0] >> 31) == (st[0] >> 31)


def test_named_direction_pkl_round_trip_and_reference_file(tmp_path):
    """The named-direction .pkl format (interactive.py:88-127, 526-571): the file the reference ships loads through
    load_named_components; a direction exported from an .npz has the reference's keys, value types and file name."""
    import pickle
    from ganspace_b200 import directions
    from ganspace_b200.config import Config
    ref_file = Path(__file__).parent / "golden" / "ref_named_direction.pkl"      # the reference's shipped artefact (data fixture)
    with open(ref_file, "rb") as f:
        ref = pickle.load(f)
    assert set(directions.KEYS) <= set(ref)
    d = tmp_path / "dirs"
    d.mkdir()
    (d / "StyleGAN2-Light_direction-ffhq-ipca-w-style-comp15-range8-9.pkl").write_bytes(ref_file.read_bytes())
    comp = directions.load_named_components(str(d), "StyleGAN2", "ffhq", "W")
    assert comp.names == ["Light direction: 15 (8-8)"] or comp.names[0].endswith("15 (8-8)")
    assert comp.ranges == [(8, 9)] and comp.latent_types == ["W"] and comp.layer_names == ["style"]
    assert comp.Z_comp[0].shape == (1, 512) and abs(comp.Z_stdev[0] - ref["lat_stdev"]) == 0
    with pytest.raises(RuntimeError, match="No valid components"):
        directions.load_named_components(str(d), "StyleGAN2", "car", "W")
    # export from an .npz and read it back
    rng = np.random.RandomState(0)
    arrays = {"act_comp": rng.standard_normal((4, 1, 512)).astype(np.float32), "act_mean": np.zeros((1, 512), np.float32),
              "act_stdev": rng.rand(4).astype(np.float32), "lat_comp": rng.standard_normal((4, 1, 512)).astype(np.float32),
              "lat_mean": np.zeros((1, 512), np.float32), "lat_stdev": rng.rand(4).astype(np.float32),
              "var_ratio": rng.rand(4).astype(np.float32), "random_stdevs": rng.rand(4).astype(np.float32)}
    npz = tmp_path / "c.npz"
    np.savez(npz, **arrays)
    cfg = Config(model="StyleGAN2", layer="style", output_class="ffhq", components=4, n=1000, use_w=True, estimator="ipca")
    out = directions.export_direction(npz, d, cfg, 2, "Light direction", "W", 8, 9, sigma_range=2.5, truncation=0.9, example_seed=7)
    assert out.name == "StyleGAN2-Light_direction-ffhq-ipca-w-style-comp2-range8-9.pkl"
    with open(out, "rb") as f:
        mine = pickle.load(f)
    for k in directions.KEYS:
        assert type(mine[k]) is type(ref[k]) or (k == "sigma_range" and isinstance(mine[k], float)), k
    assert mine["act_comp"].shape == ref["act_comp"].shape and mine["act_comp"].dtype == ref["act_comp"].dtype
    assert set(mine["decomposition"]) == set(ref["decomposition"])
    comp2 = directions.load_named_components(str(d), "StyleGAN2", "ffhq", "W")
    assert len(comp2.names) == 2 and np.array_equal(comp2.Z_comp[1], arrays["lat_comp"][2])       # sorted: comp15 < comp2


def test_compute_reruns_with_direct_chain_when_the_iteration_reports_no_gap(tmp_path, monkeypatch):
    """decomposition.compute: a ChainNotConverged from the first pass (gsb_eig_status bit 1) switches the library to the exact
    direct step for ONE re-run and back (gsb_ipca_set_chain_mode is host-only state: callable without a GPU)."""
    from types import SimpleNamespace
    from ganspace_b200 import _native, decomposition
    seen = []

    def fake_compute_arrays(config, inst, state=None):
        seen.append(_native._chain_forced_direct)
        if len(seen) == 1:
            raise _native.ChainNotConverged("a chain step hit its iteration cap")
        state["N"] = 10
        return {"act_comp": np.zeros((1, 1, 2), np.float32)}

    monkeypatch.setattr(decomposition, "compute_arrays", fake_compute_arrays)
    out = tmp_path / "cache" / "x_n10.npz"
    decomposition.compute(SimpleNamespace(), out, None)
    assert seen == [False, True] and _native._chain_forced_direct is False
    assert out.is_file() and np.load(out)["act_comp"].shape == (1, 1, 2)
    with pytest.raises(_native.NativeError):
        _native._check(_native.load().gsb_ipca_set_chain_mode(7), "gsb_ipca_set_chain_mode")


def test_plan_and_rounds_properties_hypothesis():
    """Property test of the host plan: the reference's sizing rules (decomposition.py:198-232,245) for arbitrary (n, B, c), and the
    sharding invariants the drivers rely on for any world size -- rounds cover every group exactly once and in order, ownership
    partitions a round with at most ceil(len / world) groups per rank, batch_slots addresses exactly the rows of each owned run."""
    from hypothesis import given, settings, strategies as st
    from ganspace_b200 import plan

    @settings(max_examples=300, deadline=None)
    @given(n=st.integers(1, 3_000_000), B=st.integers(1, 20_000), c=st.integers(1, 1024), world=st.integers(1, 16),
           g1=st.integers(1, 6), g2=st.integers(1, 12))
    def check(n, B, c, world, g1, g2):
        p = plan.make_plan(n, B, c)
        N = n // B * B
        NB = max(B, max(2_000, 3 * c))
        assert (p.N, p.NB, p.n_lat, p.K) == (N, NB, ((N + NB - 1) // B + 1) * B, len(range(0, N, NB)))
        assert p.n_calls * B == p.n_lat and p.n_lat >= p.K * NB           # the drawn latents cover every (full) group
        rs = plan.rounds(0, p.K, world, g1, g2)
        assert [k for r in rs for k in r] == list(range(p.K))
        for i, rnd in enumerate(rs):
            assert len(rnd) <= world * (g1 if i == 0 else g2)
            per = [sum(1 for k in rnd if plan.owner(k, world) == r) for r in range(world)]
            assert sum(per) == len(rnd) and max(per) <= -(-len(rnd) // world)
        if p.K and p.K <= 400:
            for r in range(min(world, 3)):
                ks = plan.groups_to_process(p, r, world)
                assert (p.K - 1) in ks and all(plan.owner(k, world) == r or k == p.K - 1 for k in ks)
                runs = plan.contiguous_runs(ks)
                needed, offs = plan.batch_slots(p, runs)
                assert needed == sorted(set(needed)) and all(0 <= b < p.n_calls for b in needed)
                for run, off in zip(runs, offs):
                    r0, r1 = p.group_rows(run[0])[0], p.group_rows(run[-1])[1]
                    # the run's rows are contiguous inside the concatenation of the needed calls, starting at `off`
                    first_call = r0 // B
                    assert off == needed.index(first_call) * B + (r0 - first_call * B)
                    assert needed.index((r1 - 1) // B) - needed.index(first_call) == (r1 - 1) // B - first_call

    check()
