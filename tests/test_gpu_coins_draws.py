"""A batched coins engine over a set of draws of the config builder: env b plays the map size and coin colours of its
own draw (substrate.build_batched(..., build_seeds=...), mp_create_variants with map variants).

The draws are the stored ones of tests/coins_draws.py, compiled as one draw set on one sprite table, with a 40-frame
episode cap so that every run of more than 40 steps crosses an auto-reset. Env b of a mixed batch must equal, byte
for byte, env b of the CPU oracle run on its draw's blob, and env b of a homogeneous engine of that blob.
"""

import copy

import numpy as np
import pytest

from tests import coins_draws as CD
from tests import parity
from tests.test_gpu_env_variants import _MixedOracle, _actions, _lockstep, _replace, _sms, _VIEWS

pytestmark = pytest.mark.gpu

SEED = 31


def _blocks(B, n):
  return (np.arange(B) * n // B).astype(np.int64)


def _interleaved(B, n):
  return (np.arange(B) % n).astype(np.int64)


@pytest.mark.parametrize('layout', ['blocks', 'interleaved'])
def test_every_env_of_a_draw_batch_matches_the_oracle(oracle, layout):
  import torch
  from meltingpot_b200 import engine
  B, steps = 2048, 45
  blobs = CD.draw_set()
  assign = {'blocks': _blocks, 'interleaved': _interleaved}[layout](B, len(blobs))
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  assert eng.num_variants == len(blobs)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  ref = _MixedOracle(oracle, blobs, assign, SEED)
  rng = np.random.default_rng(3)
  eng.reset()
  lasts = 0
  for t in range(steps + 1):
    if t:
      acts = _actions(rng, B, eng.num_players, eng.num_actions)
      eng.step(acts)
      ref.step(acts.cpu().numpy())
    px = t in (0, 1, 20, 39, 40, 41, 42, 45)  # every image byte around the auto-reset at frame 40
    got = parity.device_outputs(eng, ('rgb', 'world') if px else ())
    parity.check_outputs(got, ref.dump(shapes, px, max_ev), f'coins draws {layout} step {t}')
    lasts += int((got['step_type'] == 2).sum())
  assert lasts == B  # every env crossed the 40-frame cap
  assert torch.equal(eng.active_variant.cpu(), torch.from_numpy(assign.astype(np.uint8)))
  ref.close()
  eng.close()


def test_a_draw_batch_equals_homogeneous_engines_in_lockstep():
  blobs = CD.draw_set()
  sms = _sms()
  for B in (1, 7, sms - 1, sms + 1, 2 * sms + 5):
    differ = _lockstep(blobs, blobs, _interleaved(B, len(blobs)), B, 45, seed=SEED)
  # reach: on the largest batch, the homogeneous engines of any two draws differ
  assert differ[~np.eye(len(blobs), dtype=bool)].all(), differ


def test_reassignment_moves_an_env_to_another_map_at_its_next_first(oracle):
  import torch
  from meltingpot_b200 import engine
  blobs = CD.draw_set()
  n = len(blobs)
  B = 12
  first = _interleaved(B, n)
  second = (first + 5) % n
  third = (first + 9) % n
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=first)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  envs = [oracle.OracleEnv(blobs[first[b]], SEED + b) for b in range(B)]
  pending = first.copy()
  rng = np.random.default_rng(11)
  eng.reset()
  for e in envs:
    e.reset()
  mask_b = np.arange(B) % 3 == 0
  switched = {'auto': 0, 'mask': 0}
  for t in range(1, 101):
    if t == 10:  # mid-episode: no env changes its map before its LAST
      eng.set_env_variant(second)
      pending = second.copy()
    if t == 60:  # a masked reset moves the masked envs at once, the others at their next LAST
      eng.set_env_variant(third)
      pending = third.copy()
      eng.reset(torch.from_numpy(mask_b.astype(np.uint8)).cuda())
      for b in np.flatnonzero(mask_b):
        switched['mask'] += 1
        envs[b] = _replace(oracle, envs[b], blobs[pending[b]], SEED + b)
    else:
      acts = rng.integers(0, eng.num_actions, size=(B, eng.num_players)).astype(np.int32)
      eng.step(torch.from_numpy(acts).cuda())
      for b in range(B):
        if envs[b].step_type() == 2:  # this step starts the next episode, on the pending draw's map
          switched['auto'] += int(envs[b]._blob != blobs[pending[b]])
          envs[b] = _replace(oracle, envs[b], blobs[pending[b]], SEED + b)
        else:
          envs[b].step(acts[b])
    px = t % 5 == 0 or t in (41, 42, 61)
    parity.check_outputs(parity.device_outputs(eng, ('rgb', 'world') if px else ()),
                         parity.env_dump(envs, shapes, pixels=px, max_events=max_ev), f'coins draws step {t}')
    active = eng.active_variant.cpu().numpy()
    assert all(envs[b]._blob == blobs[active[b]] for b in range(B)), f'active draws at step {t}: {active}'
  assert switched['auto'] >= B and switched['mask'] == int(mask_b.sum())
  eng.close()


def test_a_clone_continues_on_its_source_map_and_a_snapshot_keeps_every_map():
  import torch
  from meltingpot_b200 import engine
  blobs = CD.draw_set()
  n = len(blobs)
  B = 2 * n
  assign = _interleaved(B, n)
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  rng = np.random.default_rng(13)
  eng.reset()
  for _ in range(7):
    eng.step(_actions(rng, B, eng.num_players, eng.num_actions))
  # clone env 0 (draw 0, a 10x10 interior) into env 3 (draw 3, 15x15) and env 2 (draw 2) into env n + 3 (draw 3)
  src, dst = [0, 2], [3, n + 3]
  bank = torch.zeros((len(src), eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.tensor(src, dtype=torch.int32, device='cuda'))
  slot = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  slot[dst] = torch.arange(len(src), dtype=torch.int32, device='cuda')
  eng.restore_states(bank, slot)
  torch.cuda.synchronize()
  active = eng.active_variant.cpu().numpy()
  assert [int(active[j]) for j in dst] == [int(assign[i]) for i in src]
  for t in range(60):  # across the auto-reset: a clone keeps its source's draw (and key) through its next episode
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    acts[dst] = acts[src]
    eng.step(acts)
    torch.cuda.synchronize()
    for name in _VIEWS:
      g = getattr(eng, name)
      if name == 'scalar_obs':
        assert torch.equal(g[:, dst], g[:, src]), f'{name} at step {t}'
      else:
        assert torch.equal(g[dst], g[src]), f'{name} at step {t}'
  # snapshot round trip: an engine loaded from a snapshot continues as the engine it came from, on every env's map
  snap = eng.save_state()
  loaded = engine.Engine(list(blobs), B, seed=SEED)  # every env on draw 0 until the snapshot says otherwise
  loaded.load_state(snap)
  assert torch.equal(loaded.active_variant, eng.active_variant)
  assert [int(loaded.active_variant[j]) for j in dst] == [int(assign[i]) for i in src]
  for t in range(45):
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    eng.step(acts); loaded.step(acts)
    torch.cuda.synchronize()
    for name in _VIEWS + ('active_variant', 'pending_variant'):
      assert torch.equal(getattr(loaded, name), getattr(eng, name)), f'{name} {t} steps after the load'
  for e in (eng, loaded):
    e.close()


def _wider(s):
  """A draw on a map padded one cell further (another maximum map size)."""
  rows = s['simulation']['map'].split('\n')
  s['simulation']['map'] = '\n'.join(r + ' ' for r in rows)


def _edited(blob, section, index, value):
  """The blob with one value of an int32 section replaced."""
  from meltingpot_b200 import blob as blob_lib
  sec = blob_lib.unpack(blob)
  sec[section] = sec[section].copy()
  sec[section][index] = value
  return blob_lib.pack(sec)


def _three_players(blob):
  """A third player in the metadata (the compiler itself refuses coins with other than two players)."""
  return _edited(blob, 'meta', 4, 3)


def _avatar_layer(blob):
  """Avatar 1 on another layer: of an avatar, only its sprite (av_table column 1) may differ between draws."""
  return _edited(blob, 'av_table', (0, 2), 3)


def _avatar_spawn_group(blob):
  return _edited(blob, 'av_table', (0, 3), 5)


@pytest.mark.parametrize('row', [('map_size', _wider, "section 'meta' differs in field 'W'"),
                                 ('players', _three_players, "section 'meta' differs in field 'players'"),
                                 ('avatar_layer', _avatar_layer, r"section 'av_table' differs in value 2 \(column 2\)"),
                                 ('avatar_spawn_group', _avatar_spawn_group, r"section 'av_table' differs in value 3 \(column 3\)"),
                                 ('sprite_table', None, "section '(atlas|sprite_opaque|sprite_map)'")], ids=lambda r: r[0])
def test_incompatible_draws_are_refused_at_create(row):
  import torch
  from meltingpot_b200 import compiler, engine
  _, edit, what = row
  seeds = CD.seeds()[:2]
  if edit is None:  # two draws compiled apart: each on its own sprite table
    blobs = [CD.alone(seeds[0]), CD.alone(seeds[1])]
  elif edit in (_three_players, _avatar_layer, _avatar_spawn_group):
    blobs = [CD.draw_set()[0], edit(CD.draw_set()[1])]
  else:
    blobs = compiler.compile_settings_set([CD.settings(seeds[0], CD.CAP_40), CD.settings(seeds[1], CD.CAP_40 + (edit,))],
                                          CD.config(), list(seeds))
  torch.cuda.synchronize()
  with pytest.raises(ValueError, match=f'variant 1: {what}'):
    engine.Engine(list(blobs), 8, seed=SEED)


def test_batched_substrate_over_a_draw_set_equals_the_engine():
  import torch
  from meltingpot_b200 import engine, substrate
  blobs = CD.draw_set()
  B = 40
  assign = substrate.draw_of_env(0, B, len(blobs))
  sub = substrate.BatchedSubstrate(list(blobs), B, seed=SEED, env_variant=assign)
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  rng = np.random.default_rng(17)
  sub.reset(); eng.reset()
  for _ in range(45):
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    ts = sub.step(acts)
    eng.step(acts)
    torch.cuda.synchronize()
    assert torch.equal(ts.reward, eng.reward) and torch.equal(ts.step_type, eng.step_type)
    assert torch.equal(ts.observation['RGB'], eng.rgb) and torch.equal(ts.observation['WORLD.RGB'], eng.world_rgb)
  sub.close(); eng.close()
