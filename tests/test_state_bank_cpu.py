"""The parts of the per-env state bank that need no device: the index arrays BatchedSubstrate builds, the tag check,
the C ABI declarations, and the oracle's switchable key that rekeyed restores are checked against."""

import os
import re

import numpy as np
import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_bank_index_places_each_source_at_its_destination():
  import torch
  from meltingpot_b200 import substrate
  idx = substrate.bank_index([3, 0, 5], [1, 1, 4], 6, 5, 'envs', 'slots', device='cpu')
  assert idx.dtype == torch.int32 and idx.device.type == 'cpu'
  assert idx.tolist() == [1, -1, -1, 1, -1, 4]  # one source to many destinations (fan-out) is allowed
  idx = substrate.bank_index(torch.tensor([2, 0]), torch.tensor([0, 2]), 3, 3, 'slots', 'envs', device='cpu')
  assert idx.tolist() == [2, -1, 0]
  assert substrate.bank_index([], [], 4, 4, 'envs', 'slots', device='cpu').tolist() == [-1] * 4


@pytest.mark.parametrize('dest,src,match', [
    ([0, 1], [0], 'same length'),
    ([0, 4], [0, 1], 'envs must lie in 0..3'),
    ([-1], [0], 'envs must lie in 0..3'),
    ([0], [2], 'slots must lie in 0..1'),
    ([0], [-1], 'slots must lie in 0..1'),
    ([1, 2, 1], [0, 0, 1], 'twice'),
])
def test_bank_index_refuses(dest, src, match):
  from meltingpot_b200 import substrate
  with pytest.raises(ValueError, match=match):
    substrate.bank_index(dest, src, 4, 2, 'envs', 'slots', device='cpu')


def test_bank_tags_catch_unwritten_and_foreign_rows():
  import torch
  from meltingpot_b200 import substrate
  tag = bytes(range(1, 17))
  bank = torch.zeros((4, 64), dtype=torch.uint8)
  bank[0, :16] = torch.tensor(list(tag), dtype=torch.uint8)
  bank[2, :16] = torch.tensor(list(tag), dtype=torch.uint8)
  substrate.check_bank_tags(bank, [0, 2, 0], tag)
  substrate.check_bank_tags(bank, [], tag)
  with pytest.raises(ValueError, match=r'\[1\]'):
    substrate.check_bank_tags(bank, [0, 1], tag)
  bank[3, :16] = torch.tensor(list(tag), dtype=torch.uint8)
  bank[3, 15] ^= 1  # another engine's tag (another blob hash)
  with pytest.raises(ValueError, match=r'\[3\]'):
    substrate.check_bank_tags(bank, torch.tensor([3]), tag)


def test_c_abi_declares_the_state_bank():
  from meltingpot_b200 import engine
  with open(os.path.join(ROOT, 'include', 'mp_engine.h')) as f:
    header = f.read()
  for fn in ('mp_state_record_bytes', 'mp_state_store', 'mp_state_restore'):
    assert re.search(rf'\bint {fn}\(', header), fn
    assert fn in engine.EXPORTED_SYMBOLS
  assert int(re.search(r'#define MP_RESTORE_REKEY (\d+)u', header).group(1)) == engine.MP_RESTORE_REKEY


def _trace(env, acts):
  out = []
  for a in acts:
    env.step(a)
    out.append((env.step_type(), env.rewards().tolist(), env.avatars().tolist(), env.grid().tobytes()))
  return out


@pytest.fixture(scope='module')
def keyed():
  from oracle import binding
  binding.build()
  from tests import oracle_keys
  return oracle_keys


def test_oracle_set_key_before_reset_equals_that_key(keyed, clean_up_blob):
  a, b = 11, 20
  switched = keyed.KeyedOracleEnv(clean_up_blob, a)
  switched.set_key(b)
  plain = keyed.KeyedOracleEnv(clean_up_blob, b)
  rng = np.random.default_rng(4)
  acts = rng.integers(0, plain.n_actions, size=(30, plain.P)).astype(np.int32)
  switched.reset(); plain.reset()
  np.testing.assert_array_equal(switched.grid(), plain.grid())
  np.testing.assert_array_equal(switched.avatars(), plain.avatars())
  assert _trace(switched, acts) == _trace(plain, acts)
  np.testing.assert_array_equal(switched.world_rgb(), plain.world_rgb())


def test_oracle_set_key_after_a_store_point_changes_the_continuation(keyed, clean_up_blob):
  seed = 5
  rng = np.random.default_rng(9)
  x = keyed.KeyedOracleEnv(clean_up_blob, seed)
  y = keyed.KeyedOracleEnv(clean_up_blob, seed)
  warm = rng.integers(0, x.n_actions, size=(20, x.P)).astype(np.int32)
  tail = rng.integers(0, x.n_actions, size=(60, x.P)).astype(np.int32)
  x.reset(); y.reset()
  assert _trace(x, warm) == _trace(y, warm)
  y.set_key(seed + 3)  # the store point: same state, another key from here on
  assert _trace(x, tail) != _trace(y, tail)
