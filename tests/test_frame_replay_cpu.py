"""Sizing of the single-frame Atari replay (jorldy_b200/core/buffer/frame_store.py), computed from shapes: no allocation."""
import pytest

from jorldy_b200.core.buffer.frame_store import FRAME_BYTES, frames_per_lane, store_bytes

GB = 1e9


@pytest.mark.parametrize("capacity,lanes,n_step,limit_gb", [
    (2_000_000, 128, 3, 16.0),      # config.ape_x.atari (num_workers 128)
    (2_000_000, 256, 3, 16.0),      # the same replay behind 256 actors
    (1_000_000, 64, 3, 8.0),        # config.rainbow.atari replay behind 64 actors
])
def test_frame_store_fits_the_reference_replays(capacity, lanes, n_step, limit_gb):
    F = frames_per_lane(capacity, lanes, n_step)
    per_lane = -(-capacity // lanes)
    assert F == per_lane + n_step + 4 + -(-per_lane // 16)
    total = store_bytes(capacity, lanes, n_step)
    assert total == lanes * F * FRAME_BYTES
    assert total <= limit_gb * GB, total / GB
    # against 2 x 28,224 B of stacks per slot in the duplicated layout
    assert total < capacity * 2 * 4 * FRAME_BYTES / 7


def test_frame_store_margin():
    assert frames_per_lane(100, 10, 3, margin=0) == 10 + 3 + 4
    assert frames_per_lane(101, 10, 3, margin=0) == 11 + 3 + 4
    assert frames_per_lane(160, 1, 0) == 160 + 4 + 10
