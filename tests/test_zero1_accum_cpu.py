"""FT-ZeRO-1 gradient accumulation, host side (no GPU): the accumulator's slice geometry and size, and the reduce mode
of each micro-batch."""

from __future__ import annotations

import pytest

from torchft_b200.parallel.zero1 import (ShardLayout, Zero1Optimizer, accum_elements, accum_mode, accum_offsets,
                                         merge_ranges, total)


def _tile(vectors):
    out, at = [], 0
    for n in vectors:
        out.append((at, at + 8 * n))
        at += 8 * n
    return tuple(out)


# odd unit sizes: 1 vector, 7 vectors (some ranks get an empty slice at large worlds), odd and prime vector counts
UNITS = _tile([1, 7, 1001, 4099, 13])


@pytest.mark.parametrize("k", [1, 2, 3])
@pytest.mark.parametrize("world", range(1, 9))
def test_offsets_tile_the_primary_slices(world, k):
    L = ShardLayout(UNITS, k)
    for rank in range(world):
        offsets, n = accum_offsets(L, rank, world)
        assert len(offsets) == len(UNITS)
        slices = [L.slice_bounds(u, world, rank) for u in range(len(UNITS))]
        # back to back in unit order, each offset 8-element (32 B) aligned
        at = 0
        for off, (lo, hi) in zip(offsets, slices):
            assert off == at and off % 8 == 0
            at += hi - lo
        assert at == n
        assert merge_ranges(slices) == L.primary(rank, world)
        assert n == total(L.primary(rank, world))
    # the ranks' slices together are the whole buffer, once
    assert sum(accum_offsets(L, r, world)[1] for r in range(world)) == UNITS[-1][1]


@pytest.mark.parametrize("min_world", range(1, 9))
def test_allocation_for_min_world_bounds_every_larger_world(min_world):
    L = ShardLayout(UNITS, 2)
    n = accum_elements(L, min_world)
    numel = UNITS[-1][1]
    for w in range(min_world, 9):
        assert all(accum_offsets(L, r, w)[1] <= n for r in range(w))
    assert n == max(accum_offsets(L, r, min_world)[1] for r in range(min_world))
    # about numel / min_world: at most one vector of rounding per unit more
    assert n <= numel // min_world + 8 * len(UNITS)
    if min_world > 1:
        assert max(accum_offsets(L, r, min_world - 1)[1] for r in range(min_world - 1)) > n
    with pytest.raises(ValueError):
        accum_elements(L, 0)


def test_mode_sequence():
    assert [accum_mode(m, 1) for m in range(1)] == [0]
    assert [accum_mode(m, 2) for m in range(2)] == [1, 3]
    assert [accum_mode(m, 3) for m in range(3)] == [1, 2, 3]
    assert [accum_mode(m, 5) for m in range(5)] == [1, 2, 2, 2, 3]
    for bad in ((-1, 2), (2, 2), (0, 0)):
        with pytest.raises(ValueError):
            accum_mode(*bad)


@pytest.mark.parametrize("bad", [0, -1, 1.5])
def test_bad_step_count_raises_before_touching_the_device(bad):
    with pytest.raises(ValueError, match="grad_accum_steps"):
        Zero1Optimizer(None, 8, grad_accum_steps=bad)
