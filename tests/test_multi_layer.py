"""decomposition.get_or_compute_layers on the CPU stand-ins of the device layer (tests/fakes.py): a two-layer model whose layers
take both statistics routes (grouped, d = 128; per layer, d = 48) gives the per-layer files array for array, reuses the cache,
falls back to per-layer runs on ChainNotConverged, and refuses what it does not take."""
import sys
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

ROOT = Path(__file__).resolve().parents[1]
N, B, C_COMP = 4000, 500, 6


def _fake_layer():
    sys.path.insert(0, str(ROOT / "tests"))
    import fakes

    class TwoLayerModel(fakes.FakeFeatureModel):
        """latent -> 'a' [128] -> 'feat' [3, 4, 4]; partial_forward stops after its target, hooks fire on the way."""

        def __init__(self):
            super().__init__(C=3, H=4, W=4, latent=32, seed=5)
            self.model.a = fakes._Identity()
            g = torch.Generator().manual_seed(11)
            self.Aa = torch.randn(128, 32, generator=g) * (0.8 ** torch.arange(32, dtype=torch.float32))[None, :]

        def partial_forward(self, x, layer_name):
            assert layer_name in ("a", "feat")
            a = self.model.a(torch.tanh(x.reshape(-1, self.latent) @ self.Aa.T))
            if layer_name == "feat":
                self.model.feat(self.act_nchw_flat(x + 0.01 * a[:, :32]).view(-1, self.C, self.H, self.W))

        def feature_layout(self, layer_name):
            return None

    return fakes, TwoLayerModel


def _fake_grouped(items):
    sys.path.insert(0, str(ROOT / "tests"))
    import fakes
    return [fakes.fake_batch_stats_multi(x, g, r, m, gr) for x, g, r, m, gr in items]


@pytest.fixture
def env(monkeypatch):
    fakes, TwoLayerModel = _fake_layer()
    from ganspace_b200 import _native, decomposition, estimators
    from ganspace_b200.config import Config
    from ganspace_b200.netdissect.nethook import InstrumentedModel
    for name, value in (("BigIPCA", fakes.FakeBig), ("IPCAChain", fakes.FakeChain), ("batch_stats", fakes.fake_batch_stats),
                        ("batch_stats_multi", fakes.fake_batch_stats_multi), ("LinregAccumulator", fakes.FakeLinreg),
                        ("project_std", fakes.fake_project_std), ("require_cuda", lambda device=None: torch.device("cpu")),
                        ("batch_stats_grouped", _fake_grouped), ("stats_grouped_width", lambda d: d % 128 == 0)):
        monkeypatch.setattr(_native, name, value)
    calls = {"grouped": 0}
    grouped = _native.batch_stats_grouped

    def counting(items):
        calls["grouped"] += 1
        return grouped(items)
    monkeypatch.setattr(_native, "batch_stats_grouped", counting)
    inst = InstrumentedModel(TwoLayerModel())
    cfg = Config(model="Fake", layer="a", output_class="none", components=C_COMP, n=N, batch_size=B, use_w=False, estimator="ipca")
    return SimpleNamespace(decomposition=decomposition, native=_native, inst=inst, cfg=cfg, Config=Config, calls=calls)


def _sub(tmp):
    return SimpleNamespace(run_dir=str(tmp), run_dir_root=str(tmp))


def _per_layer(env, layer, tmp):
    import copy
    cfg = copy.copy(env.cfg)
    cfg.layer = layer
    path = env.decomposition.get_or_compute(cfg, env.inst, submit_config=_sub(tmp), force_recompute=True)
    with np.load(path) as f:
        return path.name, {k: f[k] for k in f.files}


def test_joint_pass_gives_the_per_layer_files(env, tmp_path):
    ref = {l: _per_layer(env, l, tmp_path / "single") for l in ("a", "feat")}
    paths = env.decomposition.get_or_compute_layers(env.cfg, ["feat", "a"], env.inst, submit_config=_sub(tmp_path / "joint"))
    assert list(paths) == ["feat", "a"] and env.calls["grouped"] > 0
    assert env.cfg.layer == "a" and env.cfg.components == C_COMP          # the caller's config is left as it was
    for layer, path in paths.items():
        name, want = ref[layer]
        assert path.name == name and path.parent == tmp_path / "joint" / "cache" / "components"
        with np.load(path) as f:
            assert sorted(f.files) == sorted(want)
            for k in want:
                assert f[k].dtype == want[k].dtype and np.array_equal(f[k], want[k]), (layer, k)


def test_cache_skip_and_force(env, tmp_path):
    paths = env.decomposition.get_or_compute_layers(env.cfg, ["a", "feat"], env.inst, submit_config=_sub(tmp_path))
    stamp = {l: p.stat().st_mtime_ns for l, p in paths.items()}
    n = env.calls["grouped"]
    again = env.decomposition.get_or_compute_layers(env.cfg, ["a", "feat"], env.inst, submit_config=_sub(tmp_path))
    assert again == paths and env.calls["grouped"] == n and all(p.stat().st_mtime_ns == stamp[l] for l, p in paths.items())
    env.decomposition.get_or_compute_layers(env.cfg, ["a", "feat"], env.inst, submit_config=_sub(tmp_path), force_recompute=True)
    assert env.calls["grouped"] > n


def test_chain_not_converged_falls_back_to_per_layer_runs(env, tmp_path, monkeypatch):
    ref = {l: _per_layer(env, l, tmp_path / "single")[1] for l in ("a", "feat")}
    state = {"raised": 0}
    from ganspace_b200 import decomposition

    orig = decomposition._export_components

    def failing(*a, **k):
        if state["raised"] == 0:
            state["raised"] = 1
            raise env.native.ChainNotConverged("no gap")
        return orig(*a, **k)
    monkeypatch.setattr(decomposition, "_export_components", failing)
    paths = decomposition.get_or_compute_layers(env.cfg, ["a", "feat"], env.inst, submit_config=_sub(tmp_path / "joint"),
                                                force_recompute=True)
    assert state["raised"] == 1
    for layer, path in paths.items():
        with np.load(path) as f:
            for k in ref[layer]:
                assert np.array_equal(f[k], ref[layer][k]), (layer, k)


def test_guards(env, tmp_path):
    d, cfg, sub = env.decomposition, env.cfg, _sub(tmp_path)
    with pytest.raises(ValueError, match="repeated"):
        d.get_or_compute_layers(cfg, ["a", "a"], env.inst, submit_config=sub)
    import copy
    bad = copy.copy(cfg)
    bad.estimator = "fbpca"
    with pytest.raises(NotImplementedError, match="fbpca"):
        d.get_or_compute_layers(bad, ["a"], env.inst, submit_config=sub)
    bad = copy.copy(cfg)
    bad.batch_size = None
    with pytest.raises(ValueError, match="batch_size"):
        d.get_or_compute_layers(bad, ["a"], env.inst, submit_config=sub)
    bad = copy.copy(cfg)
    bad.model, bad.use_w = "StyleGAN2", True
    with pytest.raises(ValueError, match="W latents"):
        d.get_or_compute_layers(bad, ["style", "a"], env.inst, submit_config=sub)
    assert not (tmp_path / "cache").exists()


def test_conv_feature_map_is_refused(env, tmp_path):
    """d = 32 * 40 > 1024: the large-d engine's layers are not taken."""
    env.inst.model.C, env.inst.model.H, env.inst.model.W = 1, 32, 40
    g = torch.Generator().manual_seed(3)
    env.inst.model.A = torch.randn(1280, 32, generator=g)
    env.inst.model.b = torch.zeros(1280)
    with pytest.raises(NotImplementedError, match="conv feature map"):
        env.decomposition.get_or_compute_layers(env.cfg, ["a", "feat"], env.inst, submit_config=_sub(tmp_path))
    assert not (tmp_path / "cache").exists()
