"""CPU test: the row layout and outputs of PlayerRoutes, the tensor -> mp_player_outputs conversion, and the no-GPU
failure of a step and a reset with player rows (no device)."""

import ctypes

import numpy as np
import pytest
import torch

from meltingpot_b200 import engine
from meltingpot_b200 import substrate

B, P, H, W, N = 3, 4, 16, 24, 2
NAMES = ['READY_TO_SHOOT', 'NUM_OTHERS_WHO_CLEANED_THIS_STEP']


def _routes(groups, names=NAMES):
  return substrate.PlayerRoutes(groups, B, P, (H, W, 3), names, 'cpu')


def test_rows_are_group_major_then_env_then_player():
  groups = np.array([[1, 0, -1, 1],
                     [0, 0, 2, -1],
                     [1, -1, 0, 2]])
  r = _routes(groups)
  assert r.n_rows == 9 and r.num_groups == 3
  # group 0: (0,1) (1,0) (1,1) (2,2); group 1: (0,0) (0,3) (2,0); group 2: (1,2) (2,3)
  want = [(0, 1), (1, 0), (1, 1), (2, 2), (0, 0), (0, 3), (2, 0), (1, 2), (2, 3)]
  assert list(zip(r.env_of_row.tolist(), r.player_of_row.tolist())) == want
  rows = r.row_of_player.tolist()
  for k, (b, p) in enumerate(want):
    assert rows[b][p] == k
  assert rows[0][2] == -1 and rows[1][3] == -1 and rows[2][1] == -1
  assert r.row_of_player.dtype == torch.int32 and r.row_of_player.shape == (B, P) and r.row_of_player.is_contiguous()
  assert r.rows(0) == slice(0, 4) and r.rows(1) == slice(4, 7) and r.rows(2) == slice(7, 9)
  with pytest.raises(IndexError):
    r.rows(3)


def test_unused_group_ids_give_empty_blocks_and_tensor_input_works():
  groups = torch.full((B, P), 3, dtype=torch.int64)
  groups[0, 0] = -1
  r = _routes(groups)
  assert r.num_groups == 4 and r.n_rows == B * P - 1
  assert r.rows(0) == slice(0, 0) and r.rows(3) == slice(0, B * P - 1)


def test_routes_are_immutable():
  r = _routes(np.zeros((B, P), np.int64))
  with pytest.raises(AttributeError):
    r.n_rows = 3
  with pytest.raises(AttributeError):
    r.row_of_player = None


@pytest.mark.parametrize('groups,match', [
    (np.zeros((B, P + 1), np.int64), 'shape'),
    (np.zeros((B * P,), np.int64), 'shape'),
    (np.zeros((B, P), np.float32), 'integer'),
    (np.zeros((B, P), np.bool_), 'integer'),
    (np.full((B, P), -2, np.int64), '>= 0'),
    (np.full((B, P), -1, np.int64), 'routes no player'),
])
def test_refusals(groups, match):
  with pytest.raises(ValueError, match=match):
    _routes(groups)


def test_outputs_without_T():
  r = _routes(np.array([[0, 1, 0, 1]] * B))
  po = r.outputs()
  assert po.T is None
  assert po['RGB'].shape == (B * P, H, W, 3) and po['RGB'].dtype == torch.uint8
  assert po['REWARD'].shape == (B * P,) and po['REWARD'].dtype == torch.float64
  for k, name in enumerate(NAMES):
    assert po[name].shape == (B * P,) and po[name].dtype == torch.float64
    assert po[name].data_ptr() == po.scalar_block[k].data_ptr()
  assert po.scalar_block.shape == (N, B * P)
  g1 = po.group(1)
  assert g1['RGB'].shape == (B * 2, H, W, 3) and g1['REWARD'].shape == (B * 2,)
  g1['REWARD'].fill_(5.0)
  assert po['REWARD'][r.rows(1)].eq(5.0).all() and po['REWARD'][r.rows(0)].eq(0.0).all()
  with pytest.raises(ValueError):
    po.at(0)


def test_outputs_with_T():
  r = _routes(np.array([[0, -1, 0, 1]] * B))
  T = 5
  po = r.outputs(T)
  n = r.n_rows
  assert po['RGB'].shape == (T, n, H, W, 3) and po['REWARD'].shape == (T, n)
  assert po[NAMES[0]].shape == (T, n) and po.scalar_block.shape == (N, T, n)
  s = po.at(2)
  assert s.T is None and s['RGB'].shape == (n, H, W, 3) and s['REWARD'].shape == (n,)
  assert s.scalar_block.shape == (N, n) and s.scalar_block.stride() == (T * n, 1)
  s['REWARD'].fill_(2.0)
  assert po['REWARD'][2].eq(2.0).all() and po['REWARD'][1].eq(0.0).all()
  assert po.group(1)['RGB'].shape == (T, B, H, W, 3)
  with pytest.raises(IndexError):
    po.at(T)
  with pytest.raises(ValueError):
    r.outputs(0)


def test_outputs_without_scalar_observations():
  po = _routes(np.zeros((B, P), np.int64), names=[]).outputs()
  assert set(po.keys()) == {'RGB', 'REWARD'} and po.scalar_block is None


# -- mp_player_outputs --------------------------------------------------------------------------------------------------
def _layout(t, device='cuda:0', ptr=1 << 20):
  return engine.TensorLayout(tuple(t.shape), tuple(t.stride()), t.dtype, torch.device(device),
                             ptr + t.storage_offset() * t.element_size())


def _describe(**players):
  players.setdefault('row_of_player', _layout(torch.zeros((B, P), dtype=torch.int32), ptr=1 << 30))
  return engine.describe_players(players, (H, W, 3), B, P, N, 0)


def test_describe_dense_and_slot_targets():
  po = _routes(np.array([[0, 1, 0, 1]] * B)).outputs(4)
  s = po.at(1)
  d = _describe(rgb=_layout(s['RGB']), reward=_layout(s['REWARD']), scalar_obs=_layout(s.scalar_block))
  n = B * P
  assert d.n_rows == n and d.row_of_player == 1 << 30
  assert d.rgb == (1 << 20) + n * H * W * 3 and d.rgb_row_stride == H * W * 3
  assert d.reward_row_stride == 8 and d.scalar_obs_row_stride == 8 and d.scalar_obs_stride == 4 * n * 8
  d = _describe(reward=_layout(torch.zeros((7, 3), dtype=torch.float64)[:, 1]))
  assert d.reward_row_stride == 24 and d.n_rows == 7 and not d.rgb and not d.scalar_obs


@pytest.mark.parametrize('players,match', [
    (dict(), 'at least one'),
    (dict(row_of_player=None, reward=torch.zeros(4, dtype=torch.float64)), 'missing'),
    (dict(row_of_player=torch.zeros((B, P), dtype=torch.int64), reward=torch.zeros(4, dtype=torch.float64)), 'int32'),
    (dict(row_of_player=torch.zeros((P, B), dtype=torch.int32).t(), reward=torch.zeros(4, dtype=torch.float64)), 'contiguous'),
    (dict(reward=torch.zeros(4, dtype=torch.float32)), 'dtype'),
    (dict(reward=torch.zeros((4, 1), dtype=torch.float64)), 'shape'),
    (dict(rgb=torch.zeros((4, H, W, 4), dtype=torch.uint8)), 'shape'),
    (dict(rgb=torch.zeros((4, H, 2 * W, 3), dtype=torch.uint8)[:, :, :W]), 'axis 1'),
    (dict(scalar_obs=torch.zeros((N + 1, 4), dtype=torch.float64)), 'shape'),
    (dict(reward=torch.zeros(4, dtype=torch.float64), rgb=torch.zeros((5, H, W, 3), dtype=torch.uint8)), 'rows'),
    (dict(reward=torch.zeros(0, dtype=torch.float64)), 'no rows'),
    (dict(events=torch.zeros(4, dtype=torch.int32)), 'unknown'),
])
def test_describe_refusals(players, match):
  lay = {k: (None if v is None else _layout(v)) for k, v in players.items()}
  if 'row_of_player' not in players:
    lay['row_of_player'] = _layout(torch.zeros((B, P), dtype=torch.int32), ptr=1 << 30)
  with pytest.raises(ValueError, match=match):
    engine.describe_players(lay, (H, W, 3), B, P, N, 0)


def test_describe_refuses_other_devices_and_missing_scalars():
  with pytest.raises(ValueError, match='on cpu'):
    _describe(reward=_layout(torch.zeros(4, dtype=torch.float64), 'cpu'))
  with pytest.raises(ValueError, match='on cuda:1'):
    _describe(reward=_layout(torch.zeros(4, dtype=torch.float64)),
              row_of_player=_layout(torch.zeros((B, P), dtype=torch.int32), 'cuda:1'))
  with pytest.raises(ValueError, match='no scalar observations'):
    engine.describe_players({'row_of_player': _layout(torch.zeros((B, P), dtype=torch.int32)),
                             'scalar_obs': _layout(torch.zeros((0, 4), dtype=torch.float64))}, (H, W, 3), B, P, 0, 0)


# -- C ABI ----------------------------------------------------------------------------------------------------------------
def _cuda_available():
  return torch.cuda.is_available()


@pytest.mark.skipif(_cuda_available(), reason='checks the no-GPU failure mode')
def test_entry_points_raise_without_gpu(clean_up_blob):
  lib = engine.load_library()
  players = ctypes.pointer(engine.MpPlayerOutputs())
  for req in (engine.MpRequest(players=players), engine.MpRequest(reset=1, players=players)):
    assert lib.mp_run(None, ctypes.byref(req), None) == -1
    assert b'null handle' in lib.mp_last_error()
  with pytest.raises(engine.EngineError):
    substrate.BatchedSubstrate(clean_up_blob, 2, seed=1)
  with pytest.raises(engine.EngineError):
    engine.Engine(clean_up_blob, 2)
