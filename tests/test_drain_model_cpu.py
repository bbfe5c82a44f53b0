"""tools/drain_model.py's what-if dealing of scan positions to tiles: a bijection of the scanned range that
gives no CTA more than ceil(mean) + 1 of the tiles that gossip at a tick (kernel split: contiguous positions,
floor or ceil of tiles / warps each, 8 warps per CTA)."""
import os
import sys

import numpy as np
import pytest

sys.path.insert(0, os.path.join(os.path.dirname(os.path.dirname(os.path.abspath(__file__))), "tools"))
from drain_model import deal_tiles  # noqa: E402

# (lo, hi, P, phase_shift, GI, CTAs)
SHAPES = {
    "bench 1M": (0, 7813, 10, 0, 2, 528),
    "whole blocks only": (0, 7800, 10, 0, 2, 528),
    "fewer tiles than a block": (0, 13, 10, 0, 2, 528),
    "capped grid 3": (0, 157, 10, 0, 2, 3),
    "phase_group 256": (0, 7813, 10, 1, 2, 528),
    "GI 3": (0, 7813, 6, 0, 3, 528),
    "GI 1": (0, 7813, 10, 0, 1, 528),
    "rank 1 of 4": (1953, 3906, 10, 0, 2, 528),
}


@pytest.mark.parametrize("shape", SHAPES, ids=list(SHAPES))
def test_dealing_is_a_balanced_bijection(shape):
    lo, hi, P, shift, GI, ctas = SHAPES[shape]
    tiles = deal_tiles(lo, hi, P, shift, GI)
    assert sorted(tiles.tolist()) == list(range(lo, hi))
    if GI == 1:
        assert tiles.tolist() == list(range(lo, hi))
    n, warps = hi - lo, ctas * 8
    bounds = ((np.arange(warps + 1, dtype=np.int64) * n) // warps)[::8]
    phase = ((tiles >> shift) // P) % GI
    for k in range(GI):
        m = (phase == k).astype(np.int64)
        per_cta = np.array([m[a:b].sum() for a, b in zip(bounds[:-1], bounds[1:])])
        assert per_cta.max() <= -(-m.sum() // ctas) + 1, (k, per_cta.max())
