"""gsb_batch_stats_grouped: the statistics of several inputs of different widths in one set of launches are bit-identical to
gsb_batch_stats_multi on each input, and within fp64 tolerance of a torch fp64 reference; widths off the tensor-core path are
refused before anything runs."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
WIDTHS = (128, 256, 384, 512, 1024)


def _inputs(rows, groups, strided, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    items = []
    for i, (d, n_groups) in enumerate(zip(WIDTHS, groups)):
        ld = d + (36 if strided else 0)
        # a non-zero mean, a spread of column scales and one group with larger values (its own scale exponent)
        base = torch.randn((n_groups * rows, ld), generator=g, device=DEV) * torch.logspace(0, -2, ld, device=DEV)
        base += 0.5 * (i + 1)
        base[:rows] *= 40.0
        items.append(base[:, :d])
    return items


@pytest.mark.parametrize("rows", [500, 703])
@pytest.mark.parametrize("strided", [False, True])
def test_grouped_matches_per_descriptor_and_fp64(rows, strided):
    from ganspace_b200 import _native
    groups = (1, 3, 10, 2, 4) if rows == 500 else (7, 1, 2, 10, 5)
    xs = _inputs(rows, groups, strided, seed=rows + strided)
    got = _native.batch_stats_grouped([(x, g, rows, None, None) for x, g in zip(xs, groups)])
    for x, g, (mean, gram) in zip(xs, groups, got):
        assert x.stride(0) == (x.shape[1] + 36 if strided else x.shape[1])
        m1, g1 = _native.batch_stats_multi(x, g, rows)
        assert torch.equal(mean, m1) and torch.equal(gram, g1), x.shape
        x64 = x.double().reshape(g, rows, -1)
        m64 = x64.mean(1)
        xc = x64 - m64[:, None, :]
        g64 = xc.transpose(1, 2) @ xc
        assert torch.allclose(mean, m64, rtol=1e-12, atol=1e-12 * float(x64.abs().max()))
        scale = torch.linalg.matrix_norm(g64, ord="fro").reshape(-1, 1, 1)
        # fp32-grade products (fp16 hi/lo split, three MMAs) with promoted accumulation
        assert float(((gram - g64).abs() / scale).max()) < 1e-6, x.shape
        assert torch.equal(gram, gram.transpose(1, 2))


def test_more_descriptors_than_one_launch_set_and_caller_outputs():
    """40 descriptors (two sets of launches sharing the workspace), results written into caller-given tensors."""
    from ganspace_b200 import _native
    g = torch.Generator(device=DEV).manual_seed(7)
    xs = [torch.randn((2 * 300, WIDTHS[i % 5]), generator=g, device=DEV) + i for i in range(40)]
    outs = [(torch.empty((2, x.shape[1]), dtype=torch.float64, device=DEV),
             torch.empty((2, x.shape[1], x.shape[1]), dtype=torch.float64, device=DEV)) for x in xs]
    got = _native.batch_stats_grouped([(x, 2, 300, m, gr) for x, (m, gr) in zip(xs, outs)])
    for x, (m, gr), (m2, g2) in zip(xs, outs, got):
        assert m2 is m and g2 is gr
        m1, g1 = _native.batch_stats_multi(x, 2, 300)
        assert torch.equal(m, m1) and torch.equal(gr, g1)


@pytest.mark.parametrize("bad", [64, 96, 200, 1152, 2048])
def test_bad_width_is_refused_and_nothing_runs(bad):
    from ganspace_b200 import _native
    good = torch.randn((500, 256), device=DEV)
    mean = torch.full((1, 256), -7.0, dtype=torch.float64, device=DEV)
    gram = torch.full((1, 256, 256), -7.0, dtype=torch.float64, device=DEV)
    with pytest.raises(_native.NativeError, match="d %% 128|d % 128"):
        _native.batch_stats_grouped([(good, 1, 500, mean, gram), (torch.randn((500, bad), device=DEV), 1, 500, None, None)])
    torch.cuda.synchronize()
    assert bool((mean == -7.0).all()) and bool((gram == -7.0).all())      # the valid descriptor was not computed either


def test_abi_symbols():
    from ganspace_b200 import _native
    lib = _native.load()
    assert lib.gsb_batch_stats_grouped_workspace_bytes(None, 0) == 0
    assert lib.gsb_batch_stats_grouped(None, 0, None, 0, None) == -1
