"""The per-env state layout that state-bank records and snapshots share (engine.cu, layout_state).

Records must keep their format: a bank stored by an earlier build restores into this one. And a snapshot must carry
exactly the state a record carries: an engine loaded from a snapshot stores the same records, byte for byte, as the
engine the snapshot was taken from.
"""

import numpy as np
import pytest

from tests import env_variants as EV

pytestmark = pytest.mark.gpu

FAMILIES = ['clean_up_blob', 'commons_blob', 'territory_blob', 'coins_blob', 'coop_mining_blob',
            'territory_inside_out_blob']
SEED, BASE = 5, 100


def _run(eng, steps, seed):
  import torch
  gen = torch.Generator(device='cuda').manual_seed(seed)
  eng.reset()
  for _ in range(steps):
    eng.step(torch.randint(0, eng.num_actions, (eng.num_envs, eng.num_players), generator=gen, device='cuda',
                           dtype=torch.int32))


def _store_all(eng):
  """A bank holding the record of every env, row b = env b."""
  import torch
  bank = torch.zeros((eng.num_envs, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.arange(eng.num_envs, dtype=torch.int32, device='cuda'))
  torch.cuda.synchronize()
  return bank.cpu().numpy()


@pytest.mark.parametrize('fixture, players, record_bytes', [('clean_up_blob', 7, 18544), ('commons16_blob', 16, 17856)])
def test_record_format(fixture, players, record_bytes, request):
  from meltingpot_b200 import engine
  B = 6
  eng = engine.Engine(request.getfixturevalue(fixture), B, device=0, seed=SEED, env_index_base=BASE)
  assert eng.num_players == players
  assert eng.state_record_bytes == record_bytes
  assert eng.state_tag[:4] == b'MPR1'
  _run(eng, 12, 1)
  bank = _store_all(eng)
  grid = eng.grid.cpu().numpy()
  for b in range(B):
    assert bytes(bank[b, :16]) == eng.state_tag
    assert int.from_bytes(bytes(bank[b, 16:24]), 'little') == SEED + BASE + b
    assert bytes(bank[b, 32:32 + grid[b].nbytes]) == grid[b].tobytes(), f'grid row of env {b}'
  eng.close()


def _snapshot_carries_the_records(make):
  a = make()
  bank_a = _store_all(a)
  snap = a.save_state()
  c = make(fresh=True)
  c.load_state(snap)
  bank_c = _store_all(c)
  for b in range(a.num_envs):
    np.testing.assert_array_equal(bank_c[b], bank_a[b], err_msg=f'record of env {b} after the snapshot round trip')
  a.close(); c.close()


@pytest.mark.parametrize('fixture', FAMILIES)
def test_snapshot_carries_what_records_carry(fixture, request):
  from meltingpot_b200 import engine
  blob = request.getfixturevalue(fixture)

  def make(fresh=False):
    eng = engine.Engine(blob, 9, device=0, seed=SEED, env_index_base=BASE)
    if not fresh:
      _run(eng, 30, 2)
    return eng
  _snapshot_carries_the_records(make)


def test_variant_snapshot_carries_what_records_carry():
  from meltingpot_b200 import engine
  blobs = list(EV.blobs(EV.NAMES[0]))
  B = 9
  assign = np.arange(B) % len(blobs)

  def make(fresh=False):
    eng = engine.Engine(blobs, B, device=0, seed=SEED, env_index_base=BASE, env_variant=assign)
    if not fresh:
      _run(eng, 30, 3)
      eng.set_env_variant((assign + 1) % len(blobs))  # pending differs from active in every env
    return eng
  _snapshot_carries_the_records(make)
