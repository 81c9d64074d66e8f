"""get_or_extend on the device: extending a saved run from N1 to N2 samples writes a file whose every array equals the fresh N2
get_or_compute file (StyleGAN2 `style` in W and in Z with the regression and a ragged N, `convs.2.conv.modulation` in W, the
large-d engine at `convs.1`, BigGAN-128 `generator.gen_z` on the affine path, fbpca's randomized and exact branches, and
extensions that add no group); Ctrl-C leaves the reference's partial file and a state that the next call continues (fbpca: a
state and no file); a state that does not match the run is not continued; ChainNotConverged falls back to a fresh run; and the
refusals come before any launch."""
import copy
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")


@pytest.fixture(scope="module")
def stylegan2():
    from ganspace_b200.models import StyleGAN2
    return StyleGAN2(DEV, "cat", random_init=3)


@pytest.fixture(scope="module")
def biggan():
    from ganspace_b200.models.biggan import BigGAN
    return BigGAN(DEV, 128, "husky", random_init=4321)


@pytest.fixture
def loads(monkeypatch):
    """Counts the resumes: every continued run loads its saved state into the estimator exactly once."""
    from ganspace_b200 import estimators
    n = {"n": 0}
    for cls in (estimators.IPCAEstimator, estimators.FacebookPCAEstimator):
        real = cls.load_state_dict

        def counting(self, *a, _real=real, **k):
            n["n"] += 1
            return _real(self, *a, **k)
        monkeypatch.setattr(cls, "load_state_dict", counting)
    return n


def _cfg(model_name, cls, layer, n, c, b, use_w, est="ipca", **kw):
    from ganspace_b200.config import Config
    return Config(model=model_name, layer=layer, output_class=cls, components=c, n=n, batch_size=b, use_w=use_w, estimator=est,
                  **kw)


def _sub(tmp):
    return SimpleNamespace(run_dir=str(tmp), run_dir_root=str(tmp))


def _load(path):
    with np.load(path) as f:
        return {k: f[k] for k in f.files}


def _run(model, cfg, tmp, extend=True, force=False):
    from ganspace_b200.decomposition import get_or_compute, get_or_extend
    from ganspace_b200.models import get_instrumented_model
    if hasattr(model, "use_w"):
        model.use_w() if cfg.use_w else model.use_z()
    inst = get_instrumented_model(cfg.model, cfg.output_class, cfg.layer, DEV, model=model)
    try:
        fn = get_or_extend if extend else get_or_compute
        return fn(copy.copy(cfg), inst, submit_config=_sub(tmp), force_recompute=force)
    finally:
        inst.close()


def _same(a, b):
    assert sorted(a) == sorted(b)
    for k in a:
        assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), k


def _states(tmp):
    return list((Path(tmp) / "cache" / "components" / "state").glob("*.gsbstate"))


CASES = {
    # name: (model, class, layer, n1, n2, c, B, use_w, estimator)
    "style_w": ("StyleGAN2", "cat", "style", 4000, 10_000, 32, 1000, True, "ipca"),
    "style_z_ragged": ("StyleGAN2", "cat", "style", 4500, 7500, 16, 500, False, "ipca"),
    "modulation_w": ("StyleGAN2", "cat", "convs.2.conv.modulation", 4000, 8000, 16, 500, True, "ipca"),
    "convs1_large_d": ("StyleGAN2", "cat", "convs.1", 2000, 6000, 8, 500, False, "ipca"),
    "biggan_gen_z": ("BigGAN-128", "husky", "generator.gen_z", 4000, 8000, 16, 500, False, "ipca"),
    "fbpca_randomized": ("StyleGAN2", "cat", "style", 4000, 10_000, 32, 1000, True, "fbpca"),
    "fbpca_exact": ("StyleGAN2", "cat", "style", 4000, 8000, 210, 1000, True, "fbpca"),
    "same_groups": ("StyleGAN2", "cat", "style", 3000, 4000, 32, 1000, True, "ipca"),
    "same_groups_large_d": ("StyleGAN2", "cat", "convs.1", 3000, 4000, 8, 500, False, "ipca"),
}


@pytest.mark.parametrize("case", list(CASES))
def test_extension_equals_a_fresh_run(stylegan2, biggan, loads, tmp_path, case):
    name, cls, layer, n1, n2, c, b, use_w, est = CASES[case]
    model = biggan if name.startswith("BigGAN") else stylegan2
    if est == "fbpca":
        from ganspace_b200.estimators import FacebookPCAEstimator
        pl_n = n2 // b * b + max(b, 2000, 3 * c)
        assert FacebookPCAEstimator(c).randomized(pl_n, 512) == (case == "fbpca_randomized")
    want = _load(_run(model, _cfg(name, cls, layer, n2, c, b, use_w, est), tmp_path / "fresh", extend=False, force=True))
    first = _run(model, _cfg(name, cls, layer, n1, c, b, use_w, est), tmp_path / "ext")
    assert first.is_file() and len(_states(tmp_path / "ext")) == 1 and loads["n"] == 0
    path = _run(model, _cfg(name, cls, layer, n2, c, b, use_w, est), tmp_path / "ext")
    assert loads["n"] == 1
    _same(_load(path), want)


def test_interrupted_ipca_run_continues(stylegan2, loads, tmp_path, monkeypatch):
    from ganspace_b200 import decomposition, estimators
    cfg = _cfg("StyleGAN2", "cat", "style", 8000, 16, 500, False)
    want = _load(_run(stylegan2, cfg, tmp_path / "fresh", extend=False, force=True))
    calls = {"n": 0}
    orig = estimators.IPCAEstimator.fit_partial_stats

    def interrupting(self, *a):
        calls["n"] += 1
        if calls["n"] == 3:
            raise KeyboardInterrupt
        return orig(self, *a)
    monkeypatch.setattr(estimators.IPCAEstimator, "fit_partial_stats", interrupting)
    with pytest.raises(SystemExit) as ex:
        _run(stylegan2, cfg, tmp_path / "ext")
    assert ex.value.code == 1
    monkeypatch.setattr(estimators.IPCAEstimator, "fit_partial_stats", orig)
    full = decomposition._dump_path(tmp_path / "ext", cfg)
    files = list(full.parent.glob("*.npz"))
    assert [f.name for f in files] == [full.name.replace("_n8000", "_n4000")]          # the reference's partial file
    assert decomposition.StateFile(_states(tmp_path / "ext")[0]).groups == 2
    _same(_load(_run(stylegan2, cfg, tmp_path / "ext")), want)
    assert loads["n"] == 1


def test_interrupted_fbpca_run_leaves_a_state_and_no_file(stylegan2, loads, tmp_path, monkeypatch):
    from ganspace_b200 import decomposition, estimators
    cfg = _cfg("StyleGAN2", "cat", "style", 10_000, 32, 1000, True, "fbpca")
    want = _load(_run(stylegan2, cfg, tmp_path / "fresh", extend=False, force=True))
    calls = {"n": 0}
    orig = estimators.FacebookPCAEstimator.fit_partial_stats

    def interrupting(self, *a):
        calls["n"] += 1
        if calls["n"] == 3:
            raise KeyboardInterrupt
        return orig(self, *a)
    monkeypatch.setattr(estimators.FacebookPCAEstimator, "fit_partial_stats", interrupting)
    with pytest.raises(SystemExit) as ex:
        _run(stylegan2, cfg, tmp_path / "ext")
    assert ex.value.code == 1
    monkeypatch.setattr(estimators.FacebookPCAEstimator, "fit_partial_stats", orig)
    assert not list((tmp_path / "ext").rglob("*.npz"))
    assert decomposition.StateFile(_states(tmp_path / "ext")[0]).groups == 2
    _same(_load(_run(stylegan2, cfg, tmp_path / "ext")), want)
    assert loads["n"] == 1


@pytest.mark.parametrize("change", ["weights", "B", "c", "seed", "use_w", "chain", "layout"])
def test_a_mismatching_state_is_not_continued(stylegan2, loads, tmp_path, monkeypatch, change):
    from ganspace_b200 import _native
    from ganspace_b200.models import StyleGAN2
    base = dict(c=16, b=500, use_w=False)
    over = {"B": dict(b=1000), "c": dict(c=24), "use_w": dict(use_w=True)}.get(change, {})
    extra = dict(seed=7) if change == "seed" else {}
    cfg2 = _cfg("StyleGAN2", "cat", "style", 8000, **dict(base, **over), **extra)
    want = _load(_run(stylegan2, cfg2, tmp_path / "fresh", extend=False, force=True))
    # the earlier run, written under the other setting
    model1 = StyleGAN2(DEV, "cat", random_init=4) if change == "weights" else stylegan2
    if change == "chain":
        monkeypatch.setenv("GANSPACE_B200_CHAIN", "direct")     # read by the key (the library read its mode at its first step)
    real_version = _native.state_layout_version
    if change == "layout":
        monkeypatch.setattr(_native, "state_layout_version", lambda kind: real_version(kind) + 1)
    _run(model1, _cfg("StyleGAN2", "cat", "style", 4000, **base), tmp_path / "ext")
    monkeypatch.delenv("GANSPACE_B200_CHAIN", raising=False)
    monkeypatch.setattr(_native, "state_layout_version", real_version)
    assert len(_states(tmp_path / "ext")) == 1
    path = _run(stylegan2, cfg2, tmp_path / "ext")
    assert loads["n"] == 0
    _same(_load(path), want)


def test_chain_not_converged_in_an_extension_gives_the_fresh_run(stylegan2, loads, tmp_path, monkeypatch):
    """The extension's retry through the direct chain step starts from scratch: its file is the one a fresh N2 run writes when
    its chain reports no gap (the same retry), not a continuation of the iterated chain's state."""
    from ganspace_b200 import _native
    cfg1, cfg2 = (_cfg("StyleGAN2", "cat", "style", n, 16, 500, True) for n in (4000, 8000))
    real, seen = _native.check_eig_status, []

    def once(what):
        seen.append(what)
        if len(seen) == 1:
            raise _native.ChainNotConverged(f"{what}: raised by the test")
        return real(what)
    monkeypatch.setattr(_native, "check_eig_status", once)
    want = _load(_run(stylegan2, cfg2, tmp_path / "fresh", extend=False, force=True))
    assert len(seen) >= 2
    monkeypatch.setattr(_native, "check_eig_status", real)
    _run(stylegan2, cfg1, tmp_path / "ext")
    seen.clear()
    monkeypatch.setattr(_native, "check_eig_status", once)
    path = _run(stylegan2, cfg2, tmp_path / "ext")
    monkeypatch.setattr(_native, "check_eig_status", real)
    assert len(seen) >= 2 and loads["n"] == 1
    _same(_load(path), want)
    # the retry left a state written under the direct chain step: a later call with the default chain does not continue it
    from ganspace_b200 import decomposition
    st = decomposition.StateFile(_states(tmp_path / "ext")[0])
    assert st.groups == 4 and st.meta["key"]["switches"].get("CHAIN") == "direct"


def test_refusals_come_before_any_launch(stylegan2, tmp_path, monkeypatch):
    from ganspace_b200 import _native, decomposition
    cfg = _cfg("StyleGAN2", "cat", "style", 4000, 16, 500, False)
    _run(stylegan2, cfg, tmp_path / "ok")
    state = _states(tmp_path / "ok")[0]
    target = decomposition._state_path(decomposition._dump_path(tmp_path, cfg), cfg)
    target.parent.mkdir(parents=True)
    target.write_bytes(state.read_bytes()[:-4096])
    from ganspace_b200.models import get_instrumented_model
    stylegan2.use_z()
    inst = get_instrumented_model("StyleGAN2", "cat", "style", DEV, model=stylegan2)
    try:
        torch.cuda.synchronize()
        before = _native.instrument.launches
        with pytest.raises(ValueError, match="cut short"):
            decomposition.get_or_extend(copy.copy(cfg), inst, submit_config=_sub(tmp_path))
        bad = copy.copy(cfg)
        bad.batch_size = None
        with pytest.raises(ValueError, match="batch_size"):
            decomposition.get_or_extend(bad, inst, submit_config=_sub(tmp_path))
        monkeypatch.setattr(decomposition, "_dist", lambda: (0, 2, True))
        with pytest.raises(NotImplementedError, match="single process"):
            decomposition.get_or_extend(copy.copy(cfg), inst, submit_config=_sub(tmp_path))
        assert _native.instrument.launches == before
    finally:
        inst.close()
    assert not list((tmp_path / "cache" / "components").glob("*.npz"))
