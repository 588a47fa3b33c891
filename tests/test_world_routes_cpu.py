"""CPU test: WORLD.RGB routed per env (PlayerRoutes / DrawnRoutes outputs(world_envs=)): validation of world_envs, the
row map and the [T, n, ...] layouts, group() leaving WORLD.RGB out, the refusal on a batch without WORLD.RGB and the
describe_players checks of 'world_row_of_env' / 'world_rgb'."""

import numpy as np
import pytest
import torch

from meltingpot_b200 import engine
from meltingpot_b200 import substrate

B, P, H, W, N = 6, 3, 16, 24, 1
WH, WW = 40, 56
NAMES = ['READY_TO_SHOOT']


def _routes(world=True):
  return substrate.PlayerRoutes(np.array([[0, 1, -1]] * B), B, P, (H, W, 3), NAMES, 'cpu',
                                (WH, WW, 3) if world else None)


def _drawn(world=True):
  return substrate.DrawnRoutes([(0,), (1, 2), ()], B, P, (H, W, 3), NAMES, 'cpu', (WH, WW, 3) if world else None)


@pytest.mark.parametrize('envs', [[4, 0, 2], np.array([4, 0, 2], np.int16), torch.tensor([4, 0, 2]),
                                  torch.tensor([4, 0, 2], dtype=torch.int32)])
def test_row_map_and_layout(envs):
  po = _routes().outputs(world_envs=envs)
  assert po.world_envs.dtype == torch.int64 and po.world_envs.tolist() == [4, 0, 2]
  m = po.world_row_of_env
  assert m.dtype == torch.int32 and m.shape == (B,) and m.is_contiguous()
  assert m.tolist() == [1, -1, 2, -1, 0, -1]
  assert po['WORLD.RGB'].shape == (3, WH, WW, 3) and po['WORLD.RGB'].dtype == torch.uint8
  assert 'WORLD.RGB' in po.keys() and po['RGB'].shape == (_routes().n_rows, H, W, 3)


def test_trajectory_slots_carry_world_rgb():
  T = 4
  po = _routes().outputs(T, world_envs=[5, 1])
  assert po['WORLD.RGB'].shape == (T, 2, WH, WW, 3)
  s = po.at(2)
  assert s.T is None and s['WORLD.RGB'].shape == (2, WH, WW, 3)
  assert s['WORLD.RGB'].data_ptr() == po['WORLD.RGB'][2].data_ptr()
  assert s.world_row_of_env is po.world_row_of_env and s.world_envs is po.world_envs
  s['WORLD.RGB'].fill_(7)
  assert po['WORLD.RGB'][2].eq(7).all() and po['WORLD.RGB'][1].eq(0).all()


def test_group_leaves_world_rgb_out():
  po = _routes().outputs(world_envs=[0])
  assert 'WORLD.RGB' not in po.group(0) and set(po.group(1)) == {'RGB', 'REWARD'} | set(NAMES)
  poT = _routes().outputs(3, world_envs=[0])
  assert 'WORLD.RGB' not in poT.group(1)


def test_without_world_envs_nothing_changes():
  po = _routes().outputs()
  assert 'WORLD.RGB' not in po.keys() and po.world_envs is None and po.world_row_of_env is None
  assert po.at(0).world_row_of_env is None if po.T else True
  s = _routes().outputs(2).at(1)
  assert s.world_row_of_env is None and 'WORLD.RGB' not in s.keys()


def test_drawn_routes_outputs():
  po = _drawn().outputs(2, world_envs=(3,))
  assert po['WORLD.RGB'].shape == (2, 1, WH, WW, 3) and po.world_row_of_env.tolist() == [-1, -1, -1, 0, -1, -1]
  assert 'WORLD.RGB' not in po.group(2)


@pytest.mark.parametrize('envs,match', [
    ([1, 3, 1], 'twice'),
    ([0, B], r'\[0, 6\)'),
    ([-1], r'\[0, 6\)'),
    ([], 'no env'),
    (np.array([True, False]), 'integer'),
    (torch.tensor([True, False]), 'integer'),
    ([0.0, 1.0], 'integer'),
    (torch.tensor([0.0, 1.0]), 'integer'),
    ([[0, 1]], 'one-dimensional'),
    (torch.tensor([0, 1], device='meta'), 'is on meta'),
])
def test_world_envs_refusals(envs, match):
  with pytest.raises(ValueError, match=match):
    _routes().outputs(world_envs=envs)


def test_refused_without_world_rgb():
  with pytest.raises(ValueError, match='world_rgb=False'):
    _routes(world=False).outputs(world_envs=[0])
  with pytest.raises(ValueError, match='world_rgb=False'):
    _drawn(world=False).outputs(4, world_envs=[0])


# -- describe_players ---------------------------------------------------------------------------------------------------
def _layout(t, device='cuda:0', ptr=1 << 20):
  return engine.TensorLayout(tuple(t.shape), tuple(t.stride()), t.dtype, torch.device(device),
                             ptr + t.storage_offset() * t.element_size())


def _describe(world_shape=(WH, WW, 3), **players):
  players.setdefault('row_of_player', _layout(torch.zeros((B, P), dtype=torch.int32), ptr=1 << 30))
  players.setdefault('reward', _layout(torch.zeros(4, dtype=torch.float64), ptr=1 << 32))
  return engine.describe_players(players, (H, W, 3), B, P, N, 0, world_shape)


def _wmap(device='cuda:0'):
  return _layout(torch.zeros(B, dtype=torch.int32), device, ptr=1 << 31)


def test_describe_world_rows():
  d = _describe(world_row_of_env=_wmap(), world_rgb=_layout(torch.zeros((3, WH, WW, 3), dtype=torch.uint8)))
  assert d.world_row_of_env == 1 << 31 and d.world_n_rows == 3 and d.world_rgb == 1 << 20
  assert d.world_rgb_row_stride == WH * WW * 3 and d.n_rows == 4
  slot = torch.zeros((5, 2, WH, WW, 3), dtype=torch.uint8)[3]
  d = _describe(world_row_of_env=_wmap(), world_rgb=_layout(slot))
  assert d.world_rgb == (1 << 20) + 6 * WH * WW * 3 and d.world_n_rows == 2
  one = torch.zeros((4, WH, WW, 3), dtype=torch.uint8)[1:2]  # one row: the stride is never used
  assert _describe(world_row_of_env=_wmap(), world_rgb=_layout(one)).world_rgb_row_stride == WH * WW * 3
  d = _describe()
  assert not d.world_rgb and not d.world_row_of_env and d.world_n_rows == 0


@pytest.mark.parametrize('players,match', [
    (dict(world_rgb=torch.zeros((2, WH, WW, 3), dtype=torch.uint8)), 'go together'),
    (dict(world_row_of_env=torch.zeros(B, dtype=torch.int32)), 'go together'),
    (dict(world_row_of_env=torch.zeros(B, dtype=torch.int64)), 'int32'),
    (dict(world_row_of_env=torch.zeros(B + 1, dtype=torch.int32)), 'int32'),
    (dict(world_row_of_env=torch.zeros((B, 2), dtype=torch.int32)[:, 0]), 'contiguous'),
    (dict(world_rgb=torch.zeros((2, WH, WW, 4), dtype=torch.uint8)), 'shape'),
    (dict(world_rgb=torch.zeros((WH, WW, 3), dtype=torch.uint8)), 'shape'),
    (dict(world_rgb=torch.zeros((2, WH, WW, 3), dtype=torch.int16)), 'dtype'),
    (dict(world_rgb=torch.zeros((0, WH, WW, 3), dtype=torch.uint8)), 'no rows'),
    (dict(world_rgb=torch.zeros((2, WH, 2 * WW, 3), dtype=torch.uint8)[:, :, :WW]), 'axis 1'),
    (dict(world_rgb=torch.zeros((2 * WH * WW * 3 + 8,), dtype=torch.uint8)[8:].view(2, WH, WW, 3)), '16 bytes'),
    (dict(world_rgb=torch.zeros((3, WH * WW * 3 + 4), dtype=torch.uint8)[:, :WH * WW * 3].view(3, WH, WW, 3)), '16 bytes'),
    (dict(world_events=torch.zeros(4, dtype=torch.int32)), 'unknown'),
])
def test_describe_world_refusals(players, match):
  lay = {k: _layout(v) for k, v in players.items()}
  if 'world_rgb' in players and 'world_row_of_env' not in players and match != 'go together':
    lay['world_row_of_env'] = _wmap()
  if 'world_row_of_env' in players and 'world_rgb' not in players and match != 'go together':
    lay['world_rgb'] = _layout(torch.zeros((2, WH, WW, 3), dtype=torch.uint8))
  with pytest.raises(ValueError, match=match):
    _describe(**lay)


def test_describe_world_devices_and_engine_without_world():
  rows = _layout(torch.zeros((2, WH, WW, 3), dtype=torch.uint8))
  with pytest.raises(ValueError, match='on cpu'):
    _describe(world_row_of_env=_wmap('cpu'), world_rgb=rows)
  with pytest.raises(ValueError, match='on cuda:1'):
    _describe(world_row_of_env=_wmap(), world_rgb=_layout(torch.zeros((2, WH, WW, 3), dtype=torch.uint8), 'cuda:1'))
  with pytest.raises(ValueError, match='renders no WORLD.RGB'):
    _describe(world_shape=None, world_row_of_env=_wmap(), world_rgb=rows)
