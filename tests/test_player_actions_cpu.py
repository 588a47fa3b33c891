"""CPU test: PlayerActions (routes.actions(T)) shapes, slots and groups, the tensor -> mp_player_actions conversion and
its refusals, the argument errors of step(player_actions=), and the no-GPU failure of a step with player_actions."""

import ctypes
import types

import numpy as np
import pytest
import torch

from meltingpot_b200 import engine
from meltingpot_b200 import substrate

B, P, H, W = 3, 4, 16, 24
NAMES = ['READY_TO_SHOOT']


def _routes(groups, num_envs=B, num_players=P, device='cpu'):
  return substrate.PlayerRoutes(groups, num_envs, num_players, (H, W, 3), NAMES, device)


def test_actions_without_T():
  r = _routes(np.array([[0, 1, -1, 1]] * B))
  pa = r.actions()
  assert pa.T is None and pa.routes is r
  assert pa.tensor.shape == (r.n_rows,) and pa.tensor.dtype == torch.int32 and pa.tensor.eq(0).all()
  g1 = pa.group(1)
  assert g1.shape == (2 * B,)
  g1.fill_(7)
  assert pa.tensor[r.rows(1)].eq(7).all() and pa.tensor[r.rows(0)].eq(0).all()
  with pytest.raises(ValueError, match='T slots'):
    pa.at(0)
  with pytest.raises(IndexError):
    pa.group(2)


def test_actions_with_T():
  r = _routes(np.array([[0, 1, 0, 1]] * B))
  T = 5
  pa = r.actions(T)
  n = r.n_rows
  assert pa.tensor.shape == (T, n) and pa.tensor.dtype == torch.int32
  s = pa.at(2)
  assert s.T is None and s.tensor.shape == (n,) and s.tensor.data_ptr() == pa.tensor[2].data_ptr()
  s.tensor.fill_(3)
  assert pa.tensor[2].eq(3).all() and pa.tensor[1].eq(0).all()
  assert pa.at(-1).tensor.data_ptr() == pa.tensor[T - 1].data_ptr()
  assert pa.group(1).shape == (T, 2 * B)
  # group(0) of [B, n_focal] has the layout the outputs' group(0) has: env-major, then player in slot order
  assert torch.equal(r.env_of_row[r.rows(0)].view(B, 2), torch.arange(B).view(B, 1).expand(B, 2))
  with pytest.raises(IndexError):
    pa.at(T)
  with pytest.raises(ValueError, match='T >= 1'):
    r.actions(0)


# -- mp_player_actions --------------------------------------------------------------------------------------------------
def _layout(t, device='cuda:0', ptr=1 << 20):
  return engine.TensorLayout(tuple(t.shape), tuple(t.stride()), t.dtype, torch.device(device),
                             ptr + t.storage_offset() * t.element_size())


def _rmap(device='cuda:0'):
  return _layout(torch.zeros((B, P), dtype=torch.int32), device, ptr=1 << 30)


def test_describe_dense_strided_and_single_row():
  d = engine.describe_player_actions({'row_of_player': _rmap(), 'action': _layout(torch.zeros(9, dtype=torch.int32))}, B, P, 0)
  assert d.row_of_player == 1 << 30 and d.n_rows == 9 and d.action == 1 << 20 and d.action_row_stride == 4
  col = torch.zeros((9, 6), dtype=torch.int32)[:, 2]  # a column of [n_rows, T]
  d = engine.describe_player_actions({'row_of_player': _rmap(), 'action': _layout(col)}, B, P, 0)
  assert d.n_rows == 9 and d.action_row_stride == 24 and d.action == (1 << 20) + 8
  slot = torch.zeros((6, 9), dtype=torch.int32)[4]  # at(t) of [T, n_rows]
  d = engine.describe_player_actions({'row_of_player': _rmap(), 'action': _layout(slot)}, B, P, 0)
  assert d.action_row_stride == 4 and d.action == (1 << 20) + 4 * 9 * 4
  one = torch.zeros((1, 5), dtype=torch.int32)[:, 0]
  d = engine.describe_player_actions({'row_of_player': _rmap(), 'action': _layout(one)}, B, P, 0)
  assert d.n_rows == 1 and d.action_row_stride == 4


@pytest.mark.parametrize('entries,match', [
    (dict(action=torch.zeros(4, dtype=torch.int32)), 'both'),
    (dict(row_of_player=torch.zeros((B, P), dtype=torch.int32)), 'both'),
    (dict(row_of_player=None, action=torch.zeros(4, dtype=torch.int32)), 'both'),
    (dict(row_of_player=torch.zeros((B, P), dtype=torch.int64), action=torch.zeros(4, dtype=torch.int32)), 'contiguous int32'),
    (dict(row_of_player=torch.zeros((P, B), dtype=torch.int32).t(), action=torch.zeros(4, dtype=torch.int32)), 'contiguous'),
    (dict(row_of_player=torch.zeros((B, P + 1), dtype=torch.int32), action=torch.zeros(4, dtype=torch.int32)), 'contiguous'),
    (dict(row_of_player=torch.zeros((B, P), dtype=torch.int32), action=torch.zeros(4, dtype=torch.int64)), 'int32 tensor'),
    (dict(row_of_player=torch.zeros((B, P), dtype=torch.int32), action=torch.zeros((4, 1), dtype=torch.int32)), 'int32 tensor'),
    (dict(row_of_player=torch.zeros((B, P), dtype=torch.int32), action=torch.zeros(0, dtype=torch.int32)), 'no rows'),
    (dict(row_of_player=torch.zeros((B, P), dtype=torch.int32), action=torch.zeros(4, dtype=torch.int32),
          reward=torch.zeros(4, dtype=torch.float64)), 'unknown'),
])
def test_describe_refusals(entries, match):
  lay = {k: (None if v is None else _layout(v)) for k, v in entries.items()}
  with pytest.raises(ValueError, match=match):
    engine.describe_player_actions(lay, B, P, 0)


def test_describe_refuses_other_devices():
  action = torch.zeros(4, dtype=torch.int32)
  with pytest.raises(ValueError, match='on cpu'):
    engine.describe_player_actions({'row_of_player': _rmap(), 'action': _layout(action, 'cpu')}, B, P, 0)
  with pytest.raises(ValueError, match='on cuda:1'):
    engine.describe_player_actions({'row_of_player': _rmap('cuda:1'), 'action': _layout(action)}, B, P, 0)


# -- argument errors of step(player_actions=) (raised before the engine is called) ----------------------------------------
def _engine_stub():
  e = object.__new__(engine.Engine)
  e.num_envs, e.num_players, e.device = B, P, 0
  return e


def test_engine_step_argument_errors():
  e = _engine_stub()
  pa = {'row_of_player': torch.zeros((B, P), dtype=torch.int32), 'action': torch.zeros(4, dtype=torch.int32)}
  with pytest.raises(ValueError, match='not both'):
    e.step(torch.zeros((B, P), dtype=torch.int32), player_actions=pa)
  with pytest.raises(ValueError, match='actions is None'):
    e.step(None)
  with pytest.raises(ValueError, match='on cpu'):
    e.step(None, player_actions=pa)


def _substrate_stub():
  s = object.__new__(substrate.BatchedSubstrate)
  s.num_envs, s.num_players, s._engine = B, P, types.SimpleNamespace(device=0)  # pylint: disable=protected-access
  return s


def test_substrate_step_argument_errors():
  s = _substrate_stub()
  on_gpu = lambda n=B: types.SimpleNamespace(num_envs=n, num_players=P, device=torch.device('cuda', 0))
  with pytest.raises(ValueError, match='not both'):
    s.step(torch.zeros((B, P), dtype=torch.int32), player_actions=object())
  with pytest.raises(ValueError, match='actions is None'):
    s.step()
  with pytest.raises(ValueError, match='must be a PlayerActions'):
    s.step(player_actions={'row_of_player': torch.zeros((B, P), dtype=torch.int32), 'action': torch.zeros(B * P, dtype=torch.int32)})
  with pytest.raises(ValueError, match='routes of 2 envs'):
    s.step(player_actions=substrate.PlayerActions(on_gpu(2), None, torch.zeros(2 * P, dtype=torch.int32)))
  with pytest.raises(ValueError, match='on cpu'):
    s.step(player_actions=_routes(np.zeros((B, P), np.int64)).actions())
  with pytest.raises(ValueError, match='pick one slot'):
    s.step(player_actions=substrate.PlayerActions(on_gpu(), 3, torch.zeros((3, B * P), dtype=torch.int32)))


# -- C ABI ----------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_entry_point_raises_without_gpu():
  lib = engine.load_library()
  req = engine.MpRequest(player_actions=ctypes.pointer(engine.MpPlayerActions()))
  assert lib.mp_run(None, ctypes.byref(req), None) == -1
  assert b'null handle' in lib.mp_last_error()
