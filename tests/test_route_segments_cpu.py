"""CPU test: row segments of mp_player_outputs (struct layout, describe_players, no-device refusal), the tensors of
PlayerRoutes / DrawnRoutes.group_outputs and the shapes of a ScenarioTrajectory."""

import ctypes
import os
import shutil
import subprocess
import types

import numpy as np
import pytest
import torch

from meltingpot_b200 import engine
from meltingpot_b200 import scenario
from meltingpot_b200 import substrate

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
B, P, H, W, N = 3, 4, 16, 24, 2
NAMES = ['READY_TO_SHOOT', 'NUM_OTHERS_WHO_CLEANED_THIS_STEP']
GROUPS = np.array([[1, 0, -1, 1],
                   [0, 0, 2, -1],
                   [1, -1, 0, 2]])  # rows: group 0 [0, 4), group 1 [4, 7), group 2 [7, 9)


def _routes(groups=GROUPS, world=None):
  return substrate.PlayerRoutes(groups, B, P, (H, W, 3), NAMES, 'cpu', world)


@pytest.mark.skipif(not (shutil.which('cc') or shutil.which('gcc')), reason='needs a C compiler')
def test_row_segment_struct_matches_the_header(tmp_path):
  cls = engine.MpRowSegment
  fields = [name for name, _ in cls._fields_]
  src = tmp_path / 'layout.c'
  src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "mp_engine.h"\nint main(void) {\n'
                 '  printf("%zu %d", sizeof(mp_row_segment), MP_MAX_ROW_SEGMENTS);\n'
                 + ''.join(f'  printf(" %zu", offsetof(mp_row_segment, {f}));\n' for f in fields)
                 + '  printf(" %zu %zu", offsetof(mp_player_outputs, n_segments), offsetof(mp_player_outputs, segments));\n'
                 '  return 0;\n}\n')
  exe = tmp_path / 'layout'
  subprocess.check_call([shutil.which('cc') or shutil.which('gcc'), '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
  got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
  assert got[:2] == [ctypes.sizeof(cls), engine.MP_MAX_ROW_SEGMENTS]
  assert got[2:-2] == [getattr(cls, f).offset for f in fields]
  assert got[-2:] == [engine.MpPlayerOutputs.n_segments.offset, engine.MpPlayerOutputs.segments.offset]


def _layout(shape, dtype, ptr, stride=None):
  if stride is None:
    stride = tuple(int(s) for s in torch.empty(shape, dtype=dtype, device='meta').stride()) if shape else ()
  return engine.TensorLayout(tuple(shape), tuple(stride), dtype, torch.device('cuda', 0), ptr)


def _describe(players):
  return engine.describe_players(players, (H, W, 3), B, P, N, 0, (32, 40, 3))


def _segment_targets(rows, ptr):
  return {'rgb': _layout((rows, H, W, 3), torch.uint8, ptr), 'reward': _layout((rows,), torch.float64, ptr + (1 << 24)),
          'scalar_obs': _layout((N, rows), torch.float64, ptr + (2 << 24))}


def test_describe_players_builds_the_segment_table():
  rmap = _layout((B, P), torch.int32, 1 << 40)
  s = _describe({'row_of_player': rmap, 'n_rows': 9,
                 'segments': [(0, 4, _segment_targets(4, 1 << 32)), (7, 9, _segment_targets(2, 2 << 32))]})
  assert s.n_rows == 9 and s.n_segments == 2 and not s.rgb and not s.reward and not s.scalar_obs
  a, b = s.segments[0], s.segments[1]
  assert (a.row_begin, a.row_end, b.row_begin, b.row_end) == (0, 4, 7, 9)
  assert a.rgb == 1 << 32 and a.rgb_row_stride == H * W * 3 and a.reward == (1 << 32) + (1 << 24) and a.reward_row_stride == 8
  assert b.scalar_obs == (2 << 32) + (2 << 24) and b.scalar_obs_row_stride == 8 and b.scalar_obs_stride == 2 * 8
  assert s.segments[2].row_end == 0  # the rest of the table stays zero
  plain = _describe({'row_of_player': rmap, 'reward': _layout((9,), torch.float64, 1 << 32)})
  assert plain.n_segments == 0 and plain.n_rows == 9


@pytest.mark.parametrize('edit,match', [
    (lambda p: p.pop('n_rows'), 'n_rows'),
    (lambda p: p.update(segments=[]), '0 segments'),
    (lambda p: p.update(segments=[(0, 1, _segment_targets(1, 1 << 32))] * 17), '17 segments'),
    (lambda p: p.update(rgb=_layout((9, H, W, 3), torch.uint8, 3 << 32)), 'unknown entries'),
    (lambda p: p.update(segments=[(2, 2, _segment_targets(1, 1 << 32))]), 'empty'),
    (lambda p: p.update(segments=[(0, 3, _segment_targets(4, 1 << 32))]), '4 rows'),
    (lambda p: p.update(segments=[(0, 4, {'reward': _layout((4,), torch.float32, 1 << 32)})]), 'dtype'),
])
def test_describe_players_refuses_malformed_segments(edit, match):
  players = {'row_of_player': _layout((B, P), torch.int32, 1 << 40), 'n_rows': 9,
             'segments': [(0, 4, _segment_targets(4, 1 << 32))]}
  edit(players)
  with pytest.raises(ValueError, match=match):
    _describe(players)


def _segments_request(**segment_edits):
  s = engine.MpPlayerOutputs(row_of_player=1 << 40, n_rows=9, n_segments=1)
  s.segments[0].row_begin, s.segments[0].row_end = 0, 4
  s.segments[0].reward, s.segments[0].reward_row_stride = 1 << 32, 8
  for k, v in segment_edits.items():
    setattr(s, k, v)
  return s


@pytest.mark.parametrize('edit', [
    {}, {'n_segments': 17}, {'n_segments': -1}, {'reward': 1 << 33},
])
def test_a_request_with_segments_fails_without_a_handle(edit):
  lib = engine.load_library()
  players = _segments_request(**edit)
  for req in (engine.MpRequest(players=ctypes.pointer(players)), engine.MpRequest(reset=1, players=ctypes.pointer(players))):
    assert lib.mp_run(None, ctypes.byref(req), None) == -1
    assert b'null handle' in lib.mp_last_error()


def test_group_outputs_shapes_views_and_slots():
  r = _routes()
  go = r.group_outputs({0: 5, 2: None})
  assert sorted(go.groups) == [0, 2]
  g0, g2 = go.group(0), go.group(2)
  assert g0['RGB'].shape == (5, 4, H, W, 3) and g0['REWARD'].shape == (5, 4) and g0[NAMES[1]].shape == (5, 4)
  assert g2['RGB'].shape == (2, H, W, 3) and g2['REWARD'].shape == (2,)
  s = go.at(3)
  assert s.slots == {0: None, 2: None}
  assert s.group(0)['RGB'].data_ptr() == g0['RGB'][3].data_ptr() and s.group(2)['RGB'] is g2['RGB']
  assert s.group(0)[NAMES[1]].data_ptr() == g0[NAMES[1]][3].data_ptr()
  segs = s.segments()
  assert [(a, b) for a, b, _ in segs] == [(0, 4), (7, 9)]
  assert segs[0][2]['scalar_obs'].shape == (N, 4) and segs[0][2]['scalar_obs'].data_ptr() == g0[NAMES[0]][3].data_ptr()
  batch = r.group_outputs({1: 6}, time_major=False)
  assert batch.group(1)['RGB'].shape == (3, 6, H, W, 3) and batch.group(1)['REWARD'].shape == (3, 6)
  one = batch.at(-1)
  assert one.group(1)['REWARD'].stride() == (6,) and one.group(1)['REWARD'].data_ptr() == batch.group(1)['REWARD'][:, 5].data_ptr()
  sb = one.groups[1][1]
  assert sb.shape == (N, 3) and sb[1].data_ptr() == batch.group(1)[NAMES[1]][:, 5].data_ptr()
  with pytest.raises(KeyError):
    go.group(1)
  with pytest.raises(IndexError):
    go.at(5)
  with pytest.raises(ValueError, match='slots'):
    r.group_outputs({2: None}).at(0)


def test_group_outputs_world_rows_and_drawn_routes():
  r = _routes(world=(8, 10, 3))
  go = r.group_outputs({0: 4, 1: 2}, world_envs=[2, 0])
  assert go.world_rgb.shape == (4, 2, 8, 10, 3) and go.world_row_of_env.tolist() == [1, -1, 0]
  assert go.at(1).world_rgb.data_ptr() == go.world_rgb[1].data_ptr()
  d = substrate.DrawnRoutes([(0,), (1, 2), (2,), ()], B, P, (H, W, 3), NAMES, 'cpu')
  dg = d.group_outputs({2: 3}, time_major=False)
  assert dg.group(2)['RGB'].shape == (B * 2, 3, H, W, 3)
  assert [(a, b) for a, b, _ in dg.at(0).segments()] == [(d.rows(2).start, d.rows(2).stop)]


@pytest.mark.parametrize('slots,match', [
    ({}, 'at least one'), ([0], 'at least one'), ({3: 1}, 'outside'), ({-1: 1}, 'outside'), ({0: 0}, 'T >= 1'),
    ({0: 2.0}, 'T >= 1'), ({True: 1}, 'outside'),
])
def test_group_outputs_argument_errors(slots, match):
  with pytest.raises(ValueError, match=match):
    _routes().group_outputs(slots)
  with pytest.raises(ValueError, match='no rows'):
    substrate.PlayerRoutes(np.full((B, P), 1), B, P, (H, W, 3), NAMES, 'cpu').group_outputs({0: 1})


def _fake_scenario(world=None):
  groups = np.tile(np.array([0, 1, 0, 0]), (B, 1))
  routes = substrate.PlayerRoutes(groups, B, P, (H, W, 3), NAMES, 'cpu', (8, 10, 3))
  sc = types.SimpleNamespace(_routes=routes, num_envs=B, num_focal=3,
                             _world=None if world is None else substrate.world_row_map(world, B, 'cpu'))
  return sc


@pytest.mark.parametrize('time_major', [True, False])
def test_scenario_trajectory_shapes(time_major):
  T = 5
  traj = scenario.ScenarioTrajectory(_fake_scenario(world=[1]), T, time_major)
  lead, per_env = ((T, B, 3), (T, B)) if time_major else ((B, 3, T), (B, T))
  assert traj.reward.shape == lead and traj.observation['RGB'].shape == lead + (H, W, 3)
  assert traj.observation[NAMES[0]].shape == lead
  assert traj.step_type.shape == per_env and traj.step_type.dtype == torch.int64
  assert traj.discount.shape == per_env and traj.observation['COLLECTIVE_REWARD'].shape == per_env
  assert traj.observation['WORLD.RGB'].shape == ((T, 1) if time_major else (1, T)) + (8, 10, 3)
  slot = traj.at(2)
  assert slot.reward.shape == (B, 3) and slot.observation['RGB'].shape == (B, 3, H, W, 3)
  assert slot.step_type.shape == (B,) and slot.observation['WORLD.RGB'].shape == (1, 8, 10, 3)
  rows = slot.rows.group(0)
  assert rows['RGB'].data_ptr() == slot.observation['RGB'].data_ptr() and rows['RGB'].shape == (B * 3, H, W, 3)
  assert rows['REWARD'].data_ptr() == slot.reward.data_ptr()
  with pytest.raises(IndexError):
    traj.at(T)
  with pytest.raises(ValueError, match='T >= 1'):
    scenario.ScenarioTrajectory(_fake_scenario(), 0, time_major)
