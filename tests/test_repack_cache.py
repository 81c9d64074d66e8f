"""The re-pack cache of the device generators (``_native.source_key`` / ``_native.Repacked``): an unchanged source serves the
packed object it was built from; an in-place edit, a replaced storage or a changed extra value rebuilds it; ``current()``
never builds."""
import torch

from ganspace_b200 import _native
from ganspace_b200.models import stylegan2


class _Build:
    def __init__(self):
        self.calls = 0

    def __call__(self):
        self.calls += 1
        return object()


def _tensors():
    return [torch.nn.Parameter(torch.randn(4, 4)), torch.nn.Parameter(torch.zeros(4)), torch.randn(1, 1, 4, 4)]


def test_unchanged_sources_return_the_same_object():
    ts, build, cache = _tensors(), _Build(), _native.Repacked()
    first = cache.get(ts, build)
    assert cache.get(ts, build) is first and cache.get(ts + [None], build) is first
    assert build.calls == 1


def test_an_in_place_edit_of_any_source_rebuilds():
    ts, build, cache = _tensors(), _Build(), _native.Repacked()
    last = cache.get(ts, build)
    for t in ts:
        with torch.no_grad():
            t.add_(1.0)
        again = cache.get(ts, build)
        assert again is not last
        last = again
    assert build.calls == 1 + len(ts)


def test_a_replaced_bias_storage_rebuilds(monkeypatch):
    # an EqualLinear bias whose storage is swapped keeps its version counter: only the data pointer shows the change
    monkeypatch.setattr(_native, "PackedMapping", lambda w, b, lr_mul: object())
    net = stylegan2.MappingNetwork(8, 2, 0.01)
    first = net.packed()
    assert net.packed() is first
    bias = net[2].bias
    version, old = bias._version, bias.data
    bias.data = old.clone()
    assert bias._version == version
    assert net.packed() is not first


def test_a_changed_extra_value_rebuilds():
    ts, build, cache = _tensors(), _Build(), _native.Repacked()
    a = cache.get(ts, build, 0.5)
    assert cache.get(ts, build, 0.5) is a
    b = cache.get(ts, build, 0.7)
    assert b is not a and cache.get(ts, build, 0.5) is not b
    assert build.calls == 3


def test_current_never_builds():
    ts, build, cache = _tensors(), _Build(), _native.Repacked()
    assert cache.current() is None and build.calls == 0
    obj = cache.get(ts, build)
    with torch.no_grad():
        ts[0].mul_(2.0)
    assert cache.current() is obj and build.calls == 1
