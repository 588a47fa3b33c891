"""Flag packing of the render-layout debug lever (engine.pack_render_layout; MP_RENDER_LAYOUT in include/mp_engine.h)."""

import pytest

from meltingpot_b200 import engine


def test_render_layout_round_trips_through_the_flags():
  for layout in engine.render_layout_candidates():
    bits = engine.pack_render_layout(*layout)
    assert bits & ~engine.MP_FLAG_LAYOUT_MASK == 0
    assert engine.unpack_render_layout(bits | engine.MP_FLAG_DEFAULT | engine.MP_FLAG_DEBUG_NO_PREMERGE) == layout
  assert engine.unpack_render_layout(engine.MP_FLAG_DEFAULT | engine.MP_FLAG_DEBUG_SCATTER_LANE_MAP) is None


def test_render_layout_bits_do_not_overlap_the_other_flags():
  others = (engine.MP_FLAG_DEFAULT | engine.MP_FLAG_DEBUG_PLAIN_LANE_MAP | engine.MP_FLAG_DEBUG_SCATTER_LANE_MAP
            | engine.MP_FLAG_DEBUG_NO_PREMERGE | 0x1f0)  # 0x1f0: the renderer's per-launch diagnostics (bits 4-8)
  assert others & engine.MP_FLAG_LAYOUT_MASK == 0
  assert engine.pack_render_layout(4, 16, 2) | engine.MP_FLAG_LAYOUT_MASK == engine.MP_FLAG_LAYOUT_MASK


def test_render_layout_candidates_are_the_engines_search_space():
  cands = engine.render_layout_candidates()
  assert len(cands) == len(set(cands)) == 50  # teams 2: 13 warp counts, 3: 7, 4: 5; two strip heights each
  assert all(t * w <= 32 for t, w, _ in cands)


@pytest.mark.parametrize('layout', [(1, 8, 2), (5, 4, 1), (2, 3, 2), (2, 17, 1), (3, 8, 0), (3, 8, 3), (2, 8.5, 1), (-2, 8, 1)])
def test_render_layout_out_of_range_is_rejected(layout):
  with pytest.raises(ValueError):
    engine.pack_render_layout(*layout)
