"""Host rules of the activation modes of ganspace_b200.strips: which layers take an activation edit, refused before ``inst`` is
touched, and the argument checks that run before any launch, with CPU stand-ins for the instrumented model."""
import pytest
import torch

from ganspace_b200 import strips
from ganspace_b200.netdissect.nethook import InstrumentedModel


class _Untouchable:
    """An instrumented model stand-in whose ``close`` must not run: the refusal comes first."""

    def __init__(self, model):
        self.model = model

    def close(self):
        raise AssertionError("closed before the layer was checked")


class _Refusing:
    """A model whose edits reach the image on no layer (what ProGAN and every conv map answer)."""

    def edit_reaches_image(self, layer):
        return False


class _RowModel(torch.nn.Module):
    """A CPU model with one row layer 'rows' [n, 6] whose edit reaches the image: enough for the checks before rendering."""

    device = torch.device("cpu")

    def __init__(self):
        super().__init__()
        self.rows = torch.nn.Linear(4, 6)

    def get_max_latents(self):
        return 3

    def edit_reaches_image(self, layer):
        return layer == "rows"

    def partial_forward(self, x, layer):
        self.rows(x)

    def forward(self, x):
        raise AssertionError("rendered before the arguments were checked")


def _args(W=6, D=4, n_comp=1):
    return dict(latents=[torch.zeros(1, D), torch.ones(1, D)], x_comp=torch.ones(n_comp, W), z_comp=torch.ones(n_comp, D),
                act_stdev=1.0, lat_stdev=1.0)


@pytest.mark.parametrize("mode", ["activation", "both"])
@pytest.mark.parametrize("model", [None, _Refusing(), _RowModel()], ids=["no-model", "refusing", "other-layer"])
def test_refused_before_close(mode, model):
    a = _args()
    with pytest.raises(NotImplementedError, match="cannot be propagated"):
        strips.create_strip(_Untouchable(model), mode, "convs.4", a["latents"], a["x_comp"], a["z_comp"], 1.0, 1.0, 2.0, 0, -1, 5)
    with pytest.raises(NotImplementedError, match="cannot be propagated"):
        strips.create_strip_centered(_Untouchable(model), mode, "convs.4", a["latents"], a["x_comp"], a["z_comp"], 1.0, 1.0,
                                     torch.zeros(6), torch.zeros(4), 2.0, 0, -1, 5)


def _assert_closed(inst):
    assert not inst._handles and not inst._offset and not inst._retained
    assert all(not m._forward_hooks for m in inst.model.modules())


@pytest.mark.parametrize("mode", ["activation", "both"])
def test_bad_widths_raise_before_rendering(mode):
    inst = InstrumentedModel(_RowModel())
    a = _args()
    bad = [
        (dict(x_comp=torch.ones(1, 5)), "x_comp rows of 5"),
        (dict(act_stdev=torch.ones(2)), "2 stdevs for 1 components"),
    ]
    for change, msg in bad:
        kw = {**a, **change}
        with pytest.raises(ValueError, match=msg):
            strips.create_strip(inst, mode, "rows", kw["latents"], kw["x_comp"], kw["z_comp"], kw["act_stdev"], 1.0, 2.0, 0, -1, 3)
        _assert_closed(inst)
    if mode == "activation":
        with pytest.raises(ValueError, match="act_mean has 5 values"):
            strips.create_strip_centered(inst, mode, "rows", a["latents"], a["x_comp"], None, 1.0, None, torch.zeros(5), None, 2.0,
                                         0, -1, 3)
        _assert_closed(inst)
    else:
        with pytest.raises(ValueError, match="2 x_comp components and 1 z_comp"):
            strips.create_strip(inst, mode, "rows", a["latents"], torch.ones(2, 6), a["z_comp"][:1], 1.0, 1.0, 2.0, 0, -1, 3,
                                per_component=True)
        _assert_closed(inst)
