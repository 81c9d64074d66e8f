"""The persistent mapping-layer kernel splits its rows into whole 128-row tiles or into single 128 x 256 tiles, whichever
leaves the shorter last round on the CTAs it may use.  Every output element is computed the same way in both cases."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_mapping_work_unit_choice_does_not_change_results(oracle, mapping_weights):
    from ganspace_b200 import _native as nat
    nat.load()
    ws, bs = mapping_weights
    pm = nat.PackedMapping(torch.tensor(np.stack(ws)).cuda(), torch.tensor(np.stack(bs)).cuda(), 0.01)
    n = 70_000                       # one launch group of a W-space run: 547 row tiles
    z = torch.randn((n, 512), generator=torch.Generator(device="cuda").manual_seed(2024), device="cuda")
    # on 132 SMs: 22 SMs left free -> 110 CTAs, whole row tiles (5 rounds of two tiles = 10 single-tile rounds);
    # 32 free -> 100 CTAs, single tiles (11 rounds instead of 6 x 2)
    outs = [pm.forward(z, leave_free_sms=free).cpu().numpy() for free in (22, 32, 0)]
    pm.check()
    assert np.array_equal(outs[0], outs[1]) and np.array_equal(outs[0], outs[2])
    ref = oracle.mapping_forward(z[:500].cpu().numpy(), ws, bs)
    assert np.max(np.abs(outs[1][:500] - ref)) < 2e-5 * np.max(np.abs(ref))
