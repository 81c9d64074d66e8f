"""get_or_compute_layers on the device: every array of every layer's file equals the per-layer get_or_compute file (StyleGAN2
style layers in Z and W space, StyleGAN v1 style layers across resolutions, BigGAN-128 gen_z with an affine and a materialised
row layer), the cache is shared with get_or_compute both ways, a ChainNotConverged falls back to per-layer runs with the same
files, and the layers the joint pass does not take are refused."""
import tempfile
from pathlib import Path
from types import SimpleNamespace

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
N, B, C = 4000, 500, 16


def _cfg(model, cls, layer, use_w=False, **kw):
    from ganspace_b200.config import Config
    args = dict(model=model, layer=layer, output_class=cls, components=C, n=N, batch_size=B, use_w=use_w, estimator="ipca")
    args.update(kw)
    return Config(**args)


def _sub(tmp):
    return SimpleNamespace(run_dir=str(tmp), run_dir_root=str(tmp))


def _inst(name, cls, model, layers, use_w=False):
    from ganspace_b200.models import get_instrumented_model
    return get_instrumented_model(name, cls, layers, DEV, model=model, use_w=use_w)


def _load(path):
    with np.load(path) as f:
        return {k: f[k] for k in f.files}


def _per_layer(name, cls, model, layers, tmp, use_w=False):
    from ganspace_b200.decomposition import get_or_compute
    out = {}
    for layer in layers:
        inst = _inst(name, cls, model, layer, use_w)
        try:
            out[layer] = get_or_compute(_cfg(name, cls, layer, use_w), inst, submit_config=_sub(tmp), force_recompute=True)
        finally:
            inst.close()
    return out


def _joint(name, cls, model, layers, tmp, use_w=False, **kw):
    from ganspace_b200.decomposition import get_or_compute_layers
    inst = _inst(name, cls, model, layers, use_w)
    try:
        return get_or_compute_layers(_cfg(name, cls, layers[0], use_w), layers, inst, submit_config=_sub(tmp), **kw)
    finally:
        inst.close()


def _assert_same_files(single, joint):
    assert list(single) == list(joint)
    for layer in single:
        assert single[layer].name == joint[layer].name
        a, b = _load(single[layer]), _load(joint[layer])
        assert sorted(a) == sorted(b)
        for k in a:
            assert a[k].dtype == b[k].dtype and a[k].shape == b[k].shape and np.array_equal(a[k], b[k]), (layer, k)


@pytest.fixture(scope="module")
def stylegan2():
    from ganspace_b200.models import StyleGAN2
    return StyleGAN2(DEV, "cat", random_init=3)


@pytest.mark.parametrize("use_w", [False, True])
def test_stylegan2_all_style_layers(stylegan2, use_w):
    layers = [t[0] for t in stylegan2.model.style_layers()]
    assert len(layers) == 20
    with tempfile.TemporaryDirectory() as tmp:
        single = _per_layer("StyleGAN2", "cat", stylegan2, layers, Path(tmp) / "single", use_w)
        joint = _joint("StyleGAN2", "cat", stylegan2, layers, Path(tmp) / "joint", use_w)
        _assert_same_files(single, joint)
    stylegan2.use_z()


def test_stylegan_v1_layers_across_resolutions():
    from ganspace_b200.models import StyleGAN
    m = StyleGAN(DEV, "bedrooms", random_init=1234)
    table = [t[0] for t in m.model.style_layers()]
    layers = [table[0], table[3], table[8], table[13]]          # 4x4 epi1, 8x8 epi2, 64x64 epi1, 128x128 epi2 (mixed widths)
    with tempfile.TemporaryDirectory() as tmp:
        single = _per_layer("StyleGAN", "bedrooms", m, layers, Path(tmp) / "single")
        joint = _joint("StyleGAN", "bedrooms", m, layers, Path(tmp) / "joint")
        _assert_same_files(single, joint)


def test_biggan_gen_z_and_row_layers():
    from ganspace_b200.models.biggan import BigGAN
    m = BigGAN(DEV, 128, "husky", random_init=4321)
    widths = m.model.style_layers()
    wide = next(n for n, c in widths if c > 128)
    narrow = next(n for n, c in reversed(widths) if c <= 128)
    assert m.affine_layer(wide) is not None and m.affine_layer(narrow) is None
    layers = ["generator.gen_z", wide, narrow]
    with tempfile.TemporaryDirectory() as tmp:
        single = _per_layer("BigGAN-128", "husky", m, layers, Path(tmp) / "single")
        joint = _joint("BigGAN-128", "husky", m, layers, Path(tmp) / "joint")
        _assert_same_files(single, joint)


def test_cache_is_shared_with_get_or_compute(stylegan2):
    from ganspace_b200.decomposition import get_or_compute
    layers = [t[0] for t in stylegan2.model.style_layers()][:3]
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        # one layer computed per layer first: the joint call computes the other two only
        first = _per_layer("StyleGAN2", "cat", stylegan2, layers[:1], tmp)[layers[0]]
        t_first = first.stat().st_mtime_ns
        paths = _joint("StyleGAN2", "cat", stylegan2, layers, tmp)
        assert paths[layers[0]] == first and first.stat().st_mtime_ns == t_first
        stamps = {l: p.stat().st_mtime_ns for l, p in paths.items()}
        # cached: nothing is rewritten
        assert _joint("StyleGAN2", "cat", stylegan2, layers, tmp) == paths
        assert all(p.stat().st_mtime_ns == stamps[l] for l, p in paths.items())
        # a later per-layer get_or_compute finds the joint pass's file
        inst = _inst("StyleGAN2", "cat", stylegan2, layers[2])
        try:
            assert get_or_compute(_cfg("StyleGAN2", "cat", layers[2]), inst, submit_config=_sub(tmp)) == paths[layers[2]]
        finally:
            inst.close()
        assert paths[layers[2]].stat().st_mtime_ns == stamps[layers[2]]
        # force_recompute rewrites every file, with the same arrays
        before = {l: _load(p) for l, p in paths.items()}
        again = _joint("StyleGAN2", "cat", stylegan2, layers, tmp, force_recompute=True)
        for l, p in again.items():
            assert p.stat().st_mtime_ns > stamps[l]
            after = _load(p)
            assert all(np.array_equal(before[l][k], after[k]) for k in after)


def test_chain_not_converged_falls_back_to_per_layer_runs(stylegan2, monkeypatch):
    from ganspace_b200 import _native
    layers = [t[0] for t in stylegan2.model.style_layers()][4:7]
    real, seen = _native.check_eig_status, []

    def once(what):
        seen.append(what)
        if len(seen) == 1:
            raise _native.ChainNotConverged(f"{what}: raised by the test")
        return real(what)
    with tempfile.TemporaryDirectory() as tmp:
        single = _per_layer("StyleGAN2", "cat", stylegan2, layers, Path(tmp) / "single")
        monkeypatch.setattr(_native, "check_eig_status", once)
        joint = _joint("StyleGAN2", "cat", stylegan2, layers, Path(tmp) / "joint")
        monkeypatch.undo()
        assert len(seen) > len(layers)
        _assert_same_files(single, joint)


def test_guards(stylegan2, monkeypatch):
    from ganspace_b200 import decomposition
    style = [t[0] for t in stylegan2.model.style_layers()][:2]
    with tempfile.TemporaryDirectory() as tmp:
        tmp = Path(tmp)
        with pytest.raises(NotImplementedError, match="conv feature map"):
            _joint("StyleGAN2", "cat", stylegan2, style + ["convs.1"], tmp)
        with pytest.raises(NotImplementedError, match="fbpca"):
            decomposition.get_or_compute_layers(_cfg("StyleGAN2", "cat", style[0], estimator="fbpca"), style, None,
                                                submit_config=_sub(tmp))
        with pytest.raises(ValueError, match="W latents"):
            decomposition.get_or_compute_layers(_cfg("StyleGAN2", "cat", "style", use_w=True), ["style"] + style, None,
                                                submit_config=_sub(tmp))
        with pytest.raises(ValueError, match="batch_size"):
            decomposition.get_or_compute_layers(_cfg("StyleGAN2", "cat", style[0], batch_size=None), style, None,
                                                submit_config=_sub(tmp))
        with pytest.raises(ValueError, match="repeated"):
            decomposition.get_or_compute_layers(_cfg("StyleGAN2", "cat", style[0]), style + style[:1], None, submit_config=_sub(tmp))
        monkeypatch.setattr(decomposition, "_dist", lambda: (0, 2, True))
        with pytest.raises(NotImplementedError, match="single process"):
            decomposition.get_or_compute_layers(_cfg("StyleGAN2", "cat", style[0]), style, None, submit_config=_sub(tmp))
        monkeypatch.undo()
        assert not (tmp / "cache").exists()
    stylegan2.use_z()
