"""decomposition.get_or_extend on the CPU stand-ins of the device layer (tests/fakes.py): extending a saved run from N1 to N2
samples gives the fresh N2 file array for array (small-d chain, large-d engine, W latents, the same number of groups); Ctrl-C
leaves the partial file and a state the next call continues; a state that does not match the run (weights, B, c, seed, W
space, a switch, the layout version) is not continued; ChainNotConverged falls back to a fresh run; and the refusals come
before anything runs."""
import copy
import pickle
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
B, C_COMP = 500, 6
SMALL = dict(C=3, H=4, W=4)          # d = 48: the small-d chain
LARGE = dict(C=8, H=16, W=16)        # d = 2048: the large-d engine


def _fakes():
    sys.path.insert(0, str(ROOT / "tests"))
    import fakes
    return fakes


class _Engines:
    """The stand-in engines with the state_dict / load_state_dict of _native.IPCAChain and _native.BigIPCA."""

    @staticmethod
    def make():
        fakes = _fakes()

        class Chain(fakes.FakeChain):
            def state_dict(self):
                return {"state": np.frombuffer(pickle.dumps(self.st), dtype=np.uint8).copy(), "n_seen": self.n_seen}

            def load_state_dict(self, sd):
                self.st = pickle.loads(sd["state"].tobytes())
                self.n_seen = int(sd["n_seen"])

        class Big(fakes.FakeBig):
            def state_dict(self):
                return {"M": self.M[:self.c].numpy().copy(), "state": np.concatenate([self.mean, self.unnorm, self.S]),
                        "batch_mean": self.batch_mean.numpy().copy(), "n_seen": self.n_seen, "last_nb": self.last_nb}

            def load_state_dict(self, sd):
                d = self.d
                self.M[:self.c] = torch.from_numpy(sd["M"])
                self.mean, self.unnorm, self.S = sd["state"][:d].copy(), sd["state"][d:2 * d].copy(), sd["state"][2 * d:].copy()
                self.batch_mean = torch.from_numpy(sd["batch_mean"].copy())
                self.n_seen, self.last_nb = int(sd["n_seen"]), int(sd["last_nb"])

        return Chain, Big


@pytest.fixture
def env(monkeypatch):
    fakes = _fakes()
    from ganspace_b200 import _native, decomposition, estimators
    from ganspace_b200.config import Config
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    Chain, Big = _Engines.make()
    for name, value in (("BigIPCA", Big), ("IPCAChain", Chain), ("batch_stats", fakes.fake_batch_stats),
                        ("batch_stats_multi", fakes.fake_batch_stats_multi), ("LinregAccumulator", fakes.FakeLinreg),
                        ("project_std", fakes.fake_project_std), ("require_cuda", lambda device=None: torch.device("cpu"))):
        monkeypatch.setattr(_native, name, value)
    loads = {"n": 0}
    real_load = estimators.IPCAEstimator.load_state_dict

    def counting(self, *a, **k):
        loads["n"] += 1
        return real_load(self, *a, **k)
    monkeypatch.setattr(estimators.IPCAEstimator, "load_state_dict", counting)

    def make(kind="small", **over):
        if kind == "style":
            model = fakes.FakeStyleModel()
            layer, name, use_w = "style", "FakeStyleGAN", True
        else:
            model = fakes.FakeFeatureModel(**(SMALL if kind == "small" else LARGE))
            layer, name, use_w = "feat", "Fake", False
            if kind == "small":
                model.feature_layout = lambda layer_name: None      # the small-d engine reads the hook
        model.weight_source = 5
        inst = InstrumentedModel(model)
        inst.retain_layer(layer)
        args = dict(model=name, layer=layer, output_class="none", components=C_COMP, n=4000, batch_size=B, use_w=use_w,
                    estimator="ipca")
        args.update(over)
        return inst, Config(**args)
    return SimpleNamespace(d=decomposition, native=_native, estimators=estimators, make=make, loads=loads)


def _sub(tmp):
    return SimpleNamespace(run_dir=str(tmp), run_dir_root=str(tmp))


def _load(path):
    with np.load(path) as f:
        return {k: f[k] for k in f.files}


def _fresh(env, kind, tmp, **cfg):
    inst, c = env.make(kind, **cfg)
    return _load(env.d.get_or_compute(c, inst, submit_config=_sub(tmp), force_recompute=True))


def _extend(env, kind, tmp, n, **cfg):
    inst, c = env.make(kind, n=n, **cfg)
    return env.d.get_or_extend(c, inst, submit_config=_sub(tmp))


def _same(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), k


def _state(tmp):
    return list((Path(tmp) / "cache" / "components" / "state").glob("*.gsbstate"))


@pytest.mark.parametrize("kind,n1,n2", [("small", 4000, 8000), ("small", 3000, 7300), ("large", 4000, 8000),
                                        ("style", 2000, 6000), ("small", 3000, 4000), ("large", 3000, 4000)])
def test_extension_equals_a_fresh_run(env, tmp_path, kind, n1, n2):
    """N1 -> N2 continues from the N1 run's state (one load) and writes the fresh N2 file; n1 = 3000 and n2 = 4000 have the
    same number of groups (the last group is replayed for random_stdevs only)."""
    want = _fresh(env, kind, tmp_path / "fresh", n=n2)
    first = _extend(env, kind, tmp_path / "ext", n1)
    assert env.loads["n"] == 0 and first.is_file() and len(_state(tmp_path / "ext")) == 1
    path = _extend(env, kind, tmp_path / "ext", n2)
    assert env.loads["n"] == 1
    assert path.name == env.d._dump_path(tmp_path, env.make(kind, n=n2)[1]).name
    _same(_load(path), want)
    st = env.d.StateFile(_state(tmp_path / "ext")[0])
    assert st.groups == -(-(n2 // B * B) // 2000)
    # cached: returned as it is, nothing loaded
    again = _extend(env, kind, tmp_path / "ext", n2)
    assert again == path and env.loads["n"] == 1


def test_fewer_groups_than_the_state_runs_from_scratch(env, tmp_path):
    want = _fresh(env, "small", tmp_path / "fresh", n=4000)
    _extend(env, "small", tmp_path / "ext", 8000)
    _same(_load(_extend(env, "small", tmp_path / "ext", 4000)), want)
    assert env.loads["n"] == 0


def test_interrupt_leaves_partial_file_and_state(env, tmp_path, monkeypatch):
    want = _fresh(env, "small", tmp_path / "fresh", n=8000)
    calls = {"n": 0}
    orig = env.estimators.IPCAEstimator.fit_partial_stats

    def interrupting(self, *a):
        calls["n"] += 1
        if calls["n"] == 3:
            raise KeyboardInterrupt
        return orig(self, *a)
    monkeypatch.setattr(env.estimators.IPCAEstimator, "fit_partial_stats", interrupting)
    with pytest.raises(SystemExit) as ex:
        _extend(env, "small", tmp_path / "ext", 8000)
    assert ex.value.code == 1
    files = list((tmp_path / "ext" / "cache" / "components").glob("*.npz"))
    assert [f.name for f in files] == [env.d._dump_path(tmp_path, env.make("small", n=8000)[1]).name.replace("_n8000", "_n4000")]
    assert env.d.StateFile(_state(tmp_path / "ext")[0]).groups == 2
    monkeypatch.setattr(env.estimators.IPCAEstimator, "fit_partial_stats", orig)
    _same(_load(_extend(env, "small", tmp_path / "ext", 8000)), want)
    assert env.loads["n"] == 1


@pytest.mark.parametrize("change", ["weights", "B", "c", "seed", "use_w", "chain", "layout"])
def test_a_mismatching_state_is_not_continued(env, tmp_path, monkeypatch, change):
    kind = "style" if change == "use_w" else "small"
    over = {"B": dict(batch_size=400), "c": dict(components=C_COMP + 2), "seed": dict(seed=7),
            "use_w": dict(use_w=False)}.get(change, {})
    want = _fresh(env, kind, tmp_path / "fresh", n=8000, **over)
    inst, cfg = env.make(kind, n=4000)
    real_version = env.native.state_layout_version
    if change == "weights":
        inst.model.weight_source = 6
    if change == "chain":
        monkeypatch.setenv("GANSPACE_B200_CHAIN", "direct")      # the key only: the stand-in chain has no modes
    if change == "layout":
        monkeypatch.setattr(env.native, "state_layout_version", lambda kind: real_version(kind) + 1)
    env.d.get_or_extend(cfg, inst, submit_config=_sub(tmp_path / "ext"))
    assert len(_state(tmp_path / "ext")) == 1
    monkeypatch.delenv("GANSPACE_B200_CHAIN", raising=False)
    monkeypatch.setattr(env.native, "state_layout_version", real_version)
    path = _extend(env, kind, tmp_path / "ext", 8000, **over)
    assert env.loads["n"] == 0
    _same(_load(path), want)


def test_chain_not_converged_in_an_extension_runs_from_scratch(env, tmp_path, monkeypatch):
    want = _fresh(env, "small", tmp_path / "fresh", n=8000)
    _extend(env, "small", tmp_path / "ext", 4000)
    seen = {"n": 0}
    orig = env.d._export_components

    def failing(*a, **k):
        seen["n"] += 1
        if seen["n"] == 1:
            raise env.native.ChainNotConverged("no gap")
        return orig(*a, **k)
    monkeypatch.setattr(env.d, "_export_components", failing)
    modes = []
    monkeypatch.setattr(env.native, "set_chain_mode", lambda direct: modes.append(direct))
    path = _extend(env, "small", tmp_path / "ext", 8000)
    assert seen["n"] == 2 and modes == [True, False] and env.loads["n"] == 1      # the retry did not load the state
    _same(_load(path), want)


def test_refusals_come_before_anything_runs(env, tmp_path, monkeypatch):
    inst, cfg = env.make("small")
    ran = {"n": 0}
    real = inst.model.partial_forward

    def counting(*a, **k):
        ran["n"] += 1
        return real(*a, **k)
    inst.model.partial_forward = counting
    bad = copy.copy(cfg)
    bad.batch_size = None
    with pytest.raises(ValueError, match="batch_size"):
        env.d.get_or_extend(bad, inst, submit_config=_sub(tmp_path))
    monkeypatch.setattr(env.d, "_dist", lambda: (0, 2, True))
    with pytest.raises(NotImplementedError, match="single process"):
        env.d.get_or_extend(cfg, inst, submit_config=_sub(tmp_path))
    monkeypatch.setattr(env.d, "_dist", lambda: (0, 1, False))
    # a state file cut short
    env.d.get_or_extend(cfg, inst, submit_config=_sub(tmp_path / "ok"))
    state = _state(tmp_path / "ok")[0]
    target = env.d._state_path(env.d._dump_path(tmp_path, cfg), cfg)
    target.parent.mkdir(parents=True)
    target.write_bytes(state.read_bytes()[:-100])
    ran["n"] = 0
    with pytest.raises(ValueError, match="cut short"):
        env.d.get_or_extend(cfg, inst, submit_config=_sub(tmp_path))
    target.write_bytes(state.read_bytes()[:20])
    with pytest.raises(ValueError, match="cut short"):
        env.d.get_or_extend(cfg, inst, submit_config=_sub(tmp_path))
    assert ran["n"] == 0 and not list((tmp_path / "cache" / "components").glob("*.npz"))


def test_state_file_round_trip(env, tmp_path):
    sd = {"state": np.arange(37, dtype=np.uint8), "M": np.random.RandomState(0).standard_normal((3, 5)).astype(np.float32),
          "n_seen": 6000, "engine": "bigd"}
    key = {"model": "x", "weights": {"random_init": 1}, "seed": None}
    path = tmp_path / "s" / "a.gsbstate"
    env.d.StateFile.write(path, key, 3, sd, {"first": torch.ones(2, 4)})
    st = env.d.StateFile(path)
    assert st.groups == 3 and st.meta["key"] == key and st.mismatch(key, 3) == "" and "more than" in st.mismatch(key, 2)
    assert "weights" in st.mismatch(dict(key, weights={"random_init": 2}), 5)
    got = st.load()
    assert got["n_seen"] == 6000 and got["engine"] == "bigd"
    for k in ("state", "M"):
        assert got[k].dtype == sd[k].dtype and np.array_equal(got[k], sd[k])
    assert np.array_equal(got["first"], np.ones((2, 4), np.float32))
    assert path.stat().st_size % 64 == 0 and not list(path.parent.glob("*.tmp"))
