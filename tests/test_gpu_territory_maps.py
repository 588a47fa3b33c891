"""Map sets of territory__rooms (TORUS), territory__open (BOUNDED) and coop_mining in one engine (map variants,
tests/territory_maps.py).

Each set holds four maps of one size: the substrate's own, walls moved, resources (ores) added or removed so that the
counts differ, and spawn points moved. Env b of a mixed batch must equal, byte for byte, env b of the CPU oracle run on
its map's blob and env b of a homogeneous engine of that blob. The blobs carry a 40-frame episode cap, so every run of
more than 40 steps crosses an auto-reset.
"""

import numpy as np
import pytest

from tests import parity
from tests import territory_maps as TM
from tests.test_gpu_commons_maps import _without_event_rows
from tests.test_gpu_env_variants import _MixedOracle, _VIEWS, _actions, _lockstep, _replace

pytestmark = pytest.mark.gpu

SEED = 41


def _interleaved(B, n):
  return (np.arange(B) % n).astype(np.int64)


@pytest.mark.parametrize('name', TM.NAMES)
def test_every_env_of_a_map_set_batch_matches_the_oracle(oracle, name):
  import torch
  from meltingpot_b200 import engine
  B, steps = 515, 45  # 4k + 3: every CTA holds the four maps
  blobs = TM.map_set(name)
  assign = _interleaved(B, 4)
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
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
    px = t in (0, 1, 20, 39, 40, 41, 42, 45)
    got = parity.device_outputs(eng, ('rgb', 'world') if px else ())
    parity.check_outputs(got, ref.dump(shapes, px, max_ev), f'{name} maps step {t}')
    lasts += int((got['step_type'] == 2).sum())
  assert lasts == B
  assert torch.equal(eng.active_variant.cpu(), torch.from_numpy(assign.astype(np.uint8)))
  ref.close()
  eng.close()


@pytest.mark.parametrize('name', TM.NAMES)
def test_a_map_set_batch_equals_homogeneous_engines_in_lockstep(name):
  blobs = TM.map_set(name)
  for B in (9, 134, 263):  # 4k + 1, 4k + 2, 4k + 3
    differ = _lockstep(blobs, blobs, _interleaved(B, 4), B, 45, seed=SEED)
  assert differ[~np.eye(4, dtype=bool)].all(), differ  # reach: every two maps play differently


@pytest.mark.parametrize('name', TM.NAMES)
def test_reassignment_moves_an_env_to_another_map_at_its_next_first(oracle, name):
  import torch
  from meltingpot_b200 import engine
  blobs = TM.map_set(name)
  B = 12
  first = _interleaved(B, 4)
  second, third = (first + 1) % 4, (first + 2) % 4
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=first)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  envs = [oracle.OracleEnv(blobs[first[b]], SEED + b) for b in range(B)]
  pending = first.copy()
  rng = np.random.default_rng(11)
  eng.reset()
  for e in envs:
    e.reset()
  mask_b = np.arange(B) % 4 == 0
  moves = 0
  for t in range(1, 101):
    if t == 10:  # mid-episode: no env changes its map before its LAST
      eng.set_env_variant(second)
      pending = second.copy()
    if t == 60:  # a masked reset moves the masked envs at once, the others at their next LAST
      eng.set_env_variant(third)
      pending = third.copy()
      eng.reset(torch.from_numpy(mask_b.astype(np.uint8)).cuda())
      for b in np.flatnonzero(mask_b):
        envs[b] = _replace(oracle, envs[b], blobs[pending[b]], SEED + b)
    else:
      acts = rng.integers(0, eng.num_actions, size=(B, eng.num_players)).astype(np.int32)
      eng.step(torch.from_numpy(acts).cuda())
      for b in range(B):
        if envs[b].step_type() == 2:
          moves += envs[b]._blob != blobs[pending[b]]
          envs[b] = _replace(oracle, envs[b], blobs[pending[b]], SEED + b)
        else:
          envs[b].step(acts[b])
    px = t % 5 == 0 or t in (41, 42, 61)
    parity.check_outputs(parity.device_outputs(eng, ('rgb', 'world') if px else ()),
                         parity.env_dump(envs, shapes, pixels=px, max_events=max_ev), f'{name} maps step {t}')
    active = eng.active_variant.cpu().numpy()
    assert all(envs[b]._blob == blobs[active[b]] for b in range(B)), f'active maps at step {t}: {active}'
    if t < 41:
      assert np.array_equal(active, first), t
  assert moves >= B
  eng.close()


@pytest.mark.parametrize('name', TM.NAMES)
def test_a_clone_keeps_its_source_map_and_a_snapshot_continues_byte_for_byte(name):
  import torch
  from meltingpot_b200 import engine
  blobs = TM.map_set(name)
  B = 12
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=_interleaved(B, 4))
  rng = np.random.default_rng(13)
  eng.reset()
  for _ in range(7):
    eng.step(_actions(rng, B, eng.num_players, eng.num_actions))
  src, dst = [2, 5], [0, 3]  # the resource (ore) count map's env into the own map's, walls into spawns
  bank = torch.zeros((len(src), eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.tensor(src, dtype=torch.int32, device='cuda'))
  slot = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  slot[dst] = torch.arange(len(src), dtype=torch.int32, device='cuda')
  eng.restore_states(bank, slot)
  torch.cuda.synchronize()
  assert [int(eng.active_variant[j]) for j in dst] == [2, 1]
  for t in range(60):  # across the auto-reset: a clone plays its source's map through its next episode
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    acts[dst] = acts[src]
    eng.step(acts)
    torch.cuda.synchronize()
    for view in _VIEWS:
      g = getattr(eng, view)
      if view == 'scalar_obs':
        assert torch.equal(g[:, dst], g[:, src]), f'{view} at step {t}'
      else:
        assert torch.equal(g[dst], g[src]), f'{view} at step {t}'
  snap = eng.save_state()
  loaded = engine.Engine(list(blobs), B, seed=SEED)
  loaded.load_state(snap)
  assert torch.equal(loaded.active_variant, eng.active_variant)
  for t in range(45):
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    eng.step(acts); loaded.step(acts)
    torch.cuda.synchronize()
    for view in _VIEWS + ('active_variant', 'pending_variant'):
      assert torch.equal(getattr(loaded, view), getattr(eng, view)), f'{view} {t} steps after the load'
  eng.close(); loaded.close()


@pytest.mark.parametrize('name', TM.NAMES)
def test_an_env_that_moved_from_a_larger_map_stores_the_record_of_an_env_that_was_always_there(name):
  import torch
  from meltingpot_b200 import engine
  blobs = TM.map_set(name)
  table = 'cm_ore' if name == 'coop_mining' else 'tr_res'
  from meltingpot_b200 import blob as blob_lib
  counts = [len(blob_lib.unpack(b)[table]) for b in blobs]
  big, small = int(np.argmax(counts)), int(np.argmin(counts))
  B = 8
  moved = engine.Engine(list(blobs), B, seed=SEED, env_variant=np.full(B, big, np.int64))
  always = engine.Engine(list(blobs), B, seed=SEED, env_variant=np.full(B, small, np.int64))
  max_ev = int(moved.buffers.max_events)
  rng = np.random.default_rng(23)
  moved.reset(); always.reset()
  for t in range(1, 41):
    if t == 5:
      moved.set_env_variant(np.full(B, small, np.int64))
    acts = _actions(rng, B, moved.num_players, moved.num_actions)
    moved.step(acts); always.step(acts)
  torch.cuda.synchronize()
  assert (moved.step_type == 2).all() and (always.step_type == 2).all()
  idx = torch.arange(B, dtype=torch.int32, device='cuda')
  for t in range(6):  # the FIRST step on the smaller map, then five more
    acts = _actions(rng, B, moved.num_players, moved.num_actions)
    moved.step(acts); always.step(acts)
    a = torch.zeros((B, moved.state_record_bytes), dtype=torch.uint8, device='cuda')
    b = torch.zeros_like(a)
    moved.store_states(a, idx); always.store_states(b, idx)
    torch.cuda.synchronize()
    assert torch.equal(moved.active_variant, always.active_variant)
    assert torch.equal(_without_event_rows(a, max_ev), _without_event_rows(b, max_ev)), f'records differ at step {t}'
  moved.close(); always.close()


@pytest.mark.parametrize('name', TM.NAMES)
def test_drawn_and_fixed_player_routes_over_a_map_set_equal_each_other(name):
  from tests.test_gpu_drawn_routes import _lockstep as drawn_lockstep
  blobs = list(TM.map_set(name))
  B = 37
  drawn_lockstep(blobs, B, env_variant=_interleaved(B, 4), steps=48)


def _maps_substrate(monkeypatch, name, B, **kw):
  """build_batched(name, maps=...) over the four maps, compiled from the recorded settings as compile_maps would
  compile them from a reference checkout."""
  from meltingpot_b200 import compiler, substrate, substrates

  def compile_maps(n, roles, maps):
    settings = []
    for m in maps:
      s = TM.settings(n)
      s['simulation']['map'] = m
      settings.append(s)
    return compiler.compile_settings_set(settings, TM.config(n))
  monkeypatch.setattr(substrates, 'compile_maps', compile_maps)
  maps = [TM.ascii_map(name, k) for k in range(4)]
  return substrate.build_batched(name, roles=('default',) * TM.PLAYERS[name], num_envs=B, seed=SEED, maps=maps, **kw)


@pytest.mark.parametrize('name', TM.NAMES)
def test_build_batched_with_maps_equals_the_engine_and_steps_into_a_trajectory(monkeypatch, name):
  import torch
  from meltingpot_b200 import engine
  B, T = 30, 44
  sub = _maps_substrate(monkeypatch, name, B, env_index_base=3)
  into = _maps_substrate(monkeypatch, name, B, env_index_base=3)
  assign = (np.arange(3, 3 + B) % 4).astype(np.int64)
  eng = engine.Engine(list(TM.map_set(name)), B, seed=SEED, env_index_base=3, env_variant=assign)
  assert np.array_equal(sub.engine.active_variant.cpu().numpy(), assign)
  traj = into.trajectory(T)
  rng = np.random.default_rng(17)
  want = sub.reset(); eng.reset()
  into.reset(out=traj.at(0))
  for t in range(T):
    if t:
      acts = _actions(rng, B, eng.num_players, eng.num_actions)
      want = sub.step(acts)
      eng.step(acts)
      into.step(acts, out=traj.at(t))
    torch.cuda.synchronize()
    for view in _VIEWS:
      assert torch.equal(getattr(sub.engine, view), getattr(eng, view)), (view, t)
    slot = traj.at(t)
    for k in ('step_type', 'reward', 'discount'):
      assert torch.equal(getattr(slot, k), getattr(want, k)), (k, t)
    for k, v in want.observation.items():
      assert torch.equal(slot.observation[k], v), (k, t)
  sub.close(); into.close(); eng.close()


@pytest.mark.parametrize('name', TM.NAMES)
def test_shard_slices_with_their_env_index_base_equal_one_map_set_engine(name):
  import torch
  from meltingpot_b200 import distributed, engine
  blobs = list(TM.map_set(name))
  B = 46
  full = engine.Engine(blobs, B, seed=SEED, env_variant=_interleaved(B, 4))
  shards = []
  for r in range(2):
    base, count = distributed.shard_envs(B, r, 2)
    shards.append((base, count, engine.Engine(blobs, count, seed=SEED, env_index_base=base,
                                              env_variant=(np.arange(base, base + count) % 4).astype(np.int64))))
  rng = np.random.default_rng(19)
  full.reset()
  for *_, s in shards:
    s.reset()
  for _ in range(45):
    acts = _actions(rng, B, full.num_players, full.num_actions)
    full.step(acts)
    for base, count, s in shards:
      s.step(acts[base:base + count].contiguous())
  torch.cuda.synchronize()
  for base, count, s in shards:
    assert torch.equal(full.active_variant[base:base + count], s.active_variant)
    for view in ('rgb', 'world_rgb', 'reward', 'grid', 'avatar_state', 'timestep_packed'):
      assert torch.equal(getattr(full, view)[base:base + count], getattr(s, view)), view


def test_maps_of_another_size_are_still_refused():
  from meltingpot_b200 import engine, substrate, substrates
  with pytest.raises(ValueError, match="'territory__open' differs from 'territory__rooms' in its timestep_spec"):
    substrate.build_batched(('territory__rooms', 'territory__open'), roles=('default',) * 9, num_envs=8, seed=SEED)
  with pytest.raises(ValueError, match="variant 1: section 'meta' differs in field 'W'"):
    engine.Engine([substrates.load_blob('territory__rooms'), substrates.load_blob('territory__open')], 8, seed=SEED)
