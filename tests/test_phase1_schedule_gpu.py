"""forward_bags on batches whose 128-row tile counts sit at the edges of the phase-1 kernel's persistent schedule
(one CTA per SM, tile t then t + grid, the load state carried across tile and bag boundaries): a single one-row bag,
totals of grid - 1, grid and grid + 1 tiles, an odd total, a bag table too large for shared memory (> 96 bags), and
bags whose last tile is partial, at D = 512 (eight chunks per tile) and D = 128 (two).  Each bag must equal the
per-bag forward bit for bit and the fp64 oracle within the tolerances of tests/test_gpu_parity.py.

These check the schedule and the row masking, not the L2 prefetch: a prefetch is a hint, so a wrong prefetch address
changes no output.  The prefetch is kept inside the bag's rows by the same row test the loads use."""
import numpy as np
import pytest
import torch

from helpers import build_net
from oracle import dsmil_oracle as orc
from test_gpu_parity import _check_forward

pytestmark = pytest.mark.gpu

TILE = 128


def _grid():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _sizes_for_tiles(total, nbags, seed):
    """nbags bag sizes that use `total` tiles in all; every bag's last tile is partial (1..127 rows)."""
    rng = np.random.default_rng(seed)
    cuts = np.sort(rng.choice(np.arange(1, total), nbags - 1, replace=False)) if nbags > 1 else np.array([], int)
    tiles = np.diff(np.concatenate([[0], cuts, [total]]))
    return [int((t - 1) * TILE + rng.integers(1, TILE)) for t in tiles]


def _case_sizes(case):
    g = _grid()
    if case == "one_row":
        return [1]
    if case == "grid_minus_1":
        return _sizes_for_tiles(g - 1, 5, 1)
    if case == "grid":
        return _sizes_for_tiles(g, 7, 2)
    if case == "grid_plus_1":
        return _sizes_for_tiles(g + 1, 3, 3)
    if case == "odd_total":
        return _sizes_for_tiles(2 * g + 3, 9, 4)
    if case == "many_bags":                  # > 96 bags: the bag table stays in global memory
        rng = np.random.default_rng(5)
        return [int(n) for n in rng.integers(1, 3 * TILE, 101)]
    raise ValueError(case)


@pytest.mark.parametrize("D", [512, 128])
@pytest.mark.parametrize("case", ["one_row", "grid_minus_1", "grid", "grid_plus_1", "odd_total", "many_bags"])
def test_forward_bags_tile_schedule_edges(case, D):
    sizes = _case_sizes(case)
    C = 2
    p = orc.random_params(D, C, 3100 + D, scale=2.0)
    net = build_net(p).eval()
    Xs = [orc.synthetic_bag(n, D, 3200 + i, "uniform") for i, n in enumerate(sizes)]
    xs = [torch.from_numpy(x).cuda() for x in Xs]
    with torch.no_grad():
        outs = net.forward_bags(xs)
        singles = [net(x) for x in xs]
    assert len(outs) == len(sizes)
    for i, (o, s, X) in enumerate(zip(outs, singles, Xs)):
        for u, v in zip(o, s):
            assert u.shape == v.shape and torch.equal(u, v), (case, i, sizes[i])
        t = orc.forward(X, p)
        _check_forward(o, t.classes, t.prediction_bag, t.A, t.B, t.idx, p, None, f"{case} bags[{i}] N={sizes[i]}")
