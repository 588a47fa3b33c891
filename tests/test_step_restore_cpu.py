"""CPU test: the argument checks of Engine.step(restore=, bank=) and the mp_run request it makes, on tensor layouts
alone (no device). Tensors pose as CUDA tensors through a subclass; the C library is replaced by a recorder."""

import types

import pytest
import torch

from meltingpot_b200 import distributed
from meltingpot_b200 import engine
from meltingpot_b200 import substrate

B, P, R = 6, 3, 64
STREAM = types.SimpleNamespace(cuda_stream=0)


class _OnDevice(torch.Tensor):
  """A CPU tensor that reports itself as living on cuda:`_index` (layout checks only; its memory is never read)."""
  _index = 0

  @property
  def is_cuda(self):
    return True

  @property
  def device(self):
    return torch.device('cuda', self._index)


class _OnDevice1(_OnDevice):
  _index = 1


def _cuda(t, cls=_OnDevice):
  return t.as_subclass(cls)


class _Recorder:
  def __init__(self):
    self.calls = []

  def __getattr__(self, name):
    def call(*args):
      self.calls.append((name, args))
      return 0
    return call


class _Engine(engine.Engine):
  """Only what Engine.step reads, with a recorder in place of the library."""
  state_record_bytes = R

  def __init__(self):  # pylint: disable=super-init-not-called
    self._torch = torch
    self._lib = _Recorder()
    self._h = None
    self.num_envs, self.num_players, self.device = B, P, 0

  def _check_actions(self, actions):
    pass


def _args(**kw):
  base = dict(restore=_cuda(torch.full((B,), -1, dtype=torch.int32)), bank=_cuda(torch.zeros((4, R), dtype=torch.uint8)))
  base.update(kw)
  return base


ACTIONS = torch.zeros((B, P), dtype=torch.int32)


@pytest.mark.parametrize('kw,match', [
    (dict(restore=_cuda(torch.zeros((B + 1,), dtype=torch.int32))), 'restore must be'),
    (dict(restore=_cuda(torch.zeros((B, 1), dtype=torch.int32))), 'restore must be'),
    (dict(restore=_cuda(torch.zeros((B,), dtype=torch.int64))), 'restore must be'),
    (dict(restore=torch.zeros((B,), dtype=torch.int32)), 'restore must be'),  # host memory
    (dict(restore=_cuda(torch.zeros((2 * B,), dtype=torch.int32))[::2]), 'restore must be'),  # not contiguous
    (dict(restore=_cuda(torch.zeros((B,), dtype=torch.int32), _OnDevice1)), 'restore is on cuda:1'),
    (dict(restore=[0] * B), 'restore must be'),
    (dict(bank=_cuda(torch.zeros((4, R + 16), dtype=torch.uint8))), 'bank must be'),
    (dict(bank=_cuda(torch.zeros((4, R), dtype=torch.int8))), 'bank must be'),
    (dict(bank=_cuda(torch.zeros((0, R), dtype=torch.uint8))), 'bank must be'),
    (dict(bank=_cuda(torch.zeros((4 * R,), dtype=torch.uint8))), 'bank must be'),
    (dict(bank=torch.zeros((4, R), dtype=torch.uint8)), 'bank must be'),  # host memory
    (dict(bank=_cuda(torch.zeros((4, 2 * R), dtype=torch.uint8))[:, :R]), 'bank must be'),  # not contiguous
    (dict(bank=_cuda(torch.zeros((4, R), dtype=torch.uint8), _OnDevice1)), 'bank is on cuda:1'),
    (dict(bank=None), 'go together'),
    (dict(restore=None), 'go together'),
    (dict(restore=None, bank=None, rekey=True), 'rekey needs'),
])
def test_engine_step_refuses_restore_layouts(kw, match):
  eng = _Engine()
  with pytest.raises(ValueError, match=match):
    eng.step(ACTIONS, stream=STREAM, **_args(**kw))
  assert not eng._lib.calls, 'a refused call reached the library'  # pylint: disable=protected-access


def test_engine_step_passes_restore_to_the_library():
  eng = _Engine()
  eng.step(ACTIONS, stream=STREAM, **_args(rekey=True))
  eng.step(ACTIONS, stream=STREAM, **_args())
  eng.step(ACTIONS, stream=STREAM)
  calls = eng._lib.calls  # pylint: disable=protected-access
  assert [name for name, _ in calls] == ['mp_run'] * 3
  r0, r1, r2 = (args[1]._obj for _, args in calls)  # the MpRequest behind each byref
  assert r0.n_slots == 4 and r0.restore_flags == engine.MP_RESTORE_REKEY and r1.restore_flags == 0
  assert r0.slot_of_env and r0.bank and r1.slot_of_env and r1.bank
  assert not r0.out and not r0.players  # no `out`: the engine's own buffers
  assert r2.actions and not (r2.slot_of_env or r2.bank or r2.n_slots or r2.restore_flags or r2.reset)


class _StepRecorder:
  def __init__(self):
    self.kw = None

  def step(self, actions, **kw):
    self.kw = kw


def test_batched_and_sharded_substrates_pass_restore_through():
  bs = substrate.BatchedSubstrate.__new__(substrate.BatchedSubstrate)
  bs._engine = _StepRecorder()  # pylint: disable=protected-access
  bs._timestep = lambda: 'ts'  # pylint: disable=protected-access
  idx, bank = object(), object()
  assert bs.step(ACTIONS, restore=idx, bank=bank, rekey=True) == 'ts'
  assert bs._engine.kw == dict(restore=idx, bank=bank, rekey=True)  # pylint: disable=protected-access
  bs.step(ACTIONS)
  assert bs._engine.kw == dict(restore=None, bank=None, rekey=False)  # pylint: disable=protected-access
  sh = distributed.ShardedSubstrate.__new__(distributed.ShardedSubstrate)
  seen = {}
  sh.local = types.SimpleNamespace(step=lambda a, **kw: seen.update(kw) or 'local')
  assert sh.step(ACTIONS, restore=idx, bank=bank) == 'local'
  assert seen == dict(out=None, restore=idx, bank=bank, rekey=False)
