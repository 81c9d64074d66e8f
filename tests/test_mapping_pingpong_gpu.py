"""The persistent mapping-layer kernel hands out single 128 x 128 tiles (N fastest; with dim 512, 4 tiles per 128-row tile),
and the two consumer warpgroups of a CTA take its tiles in turns: CTA b's i-th unit b + i * grid belongs to warpgroup i & 1.
Row counts that leave a CTA one tile, an odd or an even number of tiles, or a partial last row tile must all give the same
per-row results, and the rows computed by either warpgroup must match the oracle."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def test_mapping_rows_independent_of_tile_schedule(oracle, mapping_weights):
    from ganspace_b200 import _native as nat
    nat.load()
    ws, bs = mapping_weights
    pm = nat.PackedMapping(torch.tensor(np.stack(ws)).cuda(), torch.tensor(np.stack(bs)).cuda(), 0.01)
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n_full = 20_000                                    # 157 row tiles = 628 units, more than two rounds on any current GPU
    z = torch.randn((n_full, 512), generator=torch.Generator(device="cuda").manual_seed(7), device="cuda")
    full = pm.forward(z, leave_free_sms=0).cpu().numpy()
    # 100 rows: one partial row tile (4 units, one per CTA); 1000 rows: 32 units; 20k rows with 16 / 32 SMs left free: 628
    # units over sms - 16 / sms - 32 CTAs, uneven counts per CTA, so either warpgroup takes some CTA's last unit; 5000 rows
    # on the 16-CTA minimum: 160 units, a partial last row tile
    for n, free in ((100, 0), (1000, 0), (n_full, 16), (n_full, 32), (5000, sms)):
        out = pm.forward(z[:n], leave_free_sms=free).cpu().numpy()
        assert np.array_equal(out, full[:n]), (n, free)
    pm.check()
    # the full run uses one CTA per SM (grid = sms): units 0 .. sms-1 are warpgroup 0's first tiles, sms .. 2 sms - 1 warpgroup
    # 1's; row tile t holds units 4t .. 4t+3, so the first row tile wholly inside the second round is warpgroup 1's
    t1 = (sms + 3) // 4
    assert 4 * t1 + 3 < 2 * sms and (t1 + 1) * 128 <= n_full
    for r0 in (0, t1 * 128):
        ref = oracle.mapping_forward(z[r0:r0 + 128].cpu().numpy(), ws, bs)
        assert np.max(np.abs(full[r0:r0 + 128] - ref)) < 2e-5 * np.max(np.abs(ref)), r0
