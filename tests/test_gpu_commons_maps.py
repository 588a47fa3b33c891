"""commons_harvest__open, __closed and __partnership side by side in one engine (map variants, tests/commons_maps.py).

Env b of a mixed batch must equal, byte for byte, env b of the CPU oracle run on its map's blob, and env b of a
homogeneous engine of that blob. The maps differ in their walls (BeamBlocker bits), kind and state tables, apple
piece ids and Zapper: open's beam reaches 3 cells ahead, closed's and partnership's 4. The blobs carry a 40-frame
episode cap, so every run of more than 40 steps crosses an auto-reset.
"""

import numpy as np
import pytest

from tests import commons_maps as CM
from tests import parity
from tests.test_gpu_env_variants import _MixedOracle, _actions, _lockstep, _replace, _sms, _VIEWS

pytestmark = pytest.mark.gpu

SEED = 37
_DIR = {0: (0, -1), 1: (1, 0), 2: (0, 1), 3: (-1, 0)}  # orientation -> forward step (N, E, S, W)


@pytest.fixture
def any_event_width(monkeypatch):
  """Lets _lockstep compare the events of engines whose event rows differ in width (max_events follows the largest
  beam footprint): the sorted keys of the rows in use, padded to one width."""
  keys = parity._event_keys

  def padded(events, counts):
    k = keys(events, counts)
    return np.pad(k, ((0, 0), (0, 1024 - k.shape[1])), constant_values=np.iinfo(np.int64).max)
  monkeypatch.setattr(parity, '_event_keys', padded)


def _blocks(B, n):
  return (np.arange(B) * n // B).astype(np.int64)


def _interleaved(B, n):
  return (np.arange(B) % n).astype(np.int64)


def _zaps_ahead(before, after, events, counts):
  """[(env, forward distance)] of every zap whose target stood straight ahead of its shooter. `before`: avatar_state
  before the step (a zapping avatar neither moves nor turns), `after`: after it (a zapped avatar stays where it was hit)."""
  out = []
  for b in np.flatnonzero(counts):
    for code, src, tgt in events[b, :counts[b]]:
      if code != 1:  # EV_ZAP
        continue
      sx, sy, so = before[b, src - 1, :3]
      tx, ty = after[b, tgt - 1, :2]
      fx, fy = _DIR[int(so)]
      fwd, lat = (tx - sx) * fx + (ty - sy) * fy, (tx - sx) * -fy + (ty - sy) * fx
      if lat == 0:
        out.append((int(b), int(fwd)))
  return out


@pytest.mark.parametrize('layout', ['blocks', 'interleaved'])
def test_every_env_of_a_map_set_batch_matches_the_oracle(oracle, layout):
  import torch
  from meltingpot_b200 import engine
  B, steps = 2048, 45
  blobs = CM.map_set()
  assign = {'blocks': _blocks, 'interleaved': _interleaved}[layout](B, len(blobs))
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  assert eng.num_variants == 3
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  ref = _MixedOracle(oracle, blobs, assign, SEED)
  rng = np.random.default_rng(3)
  eng.reset()
  lasts, zaps, ahead = 0, np.zeros(3, np.int64), {}
  for t in range(steps + 1):
    before = eng.avatar_state.cpu().numpy()
    if t:
      acts = _actions(rng, B, eng.num_players, eng.num_actions)
      eng.step(acts)
      ref.step(acts.cpu().numpy())
    px = t in (0, 1, 20, 39, 40, 41, 42, 45)  # every image byte around the auto-reset at frame 40
    got = parity.device_outputs(eng, ('rgb', 'world') if px else ())
    parity.check_outputs(got, ref.dump(shapes, px, max_ev), f'commons maps {layout} step {t}')
    lasts += int((got['step_type'] == 2).sum())
    events, counts = eng.events.cpu().numpy(), eng.event_count.cpu().numpy()
    for v in range(3):
      zaps[v] += int((events[assign == v, :, 0] == 1).sum())
    for b, fwd in _zaps_ahead(before, eng.avatar_state.cpu().numpy(), events, counts):
      ahead.setdefault(int(assign[b]), set()).add(fwd)
  assert lasts == B  # every env crossed the 40-frame cap
  assert (zaps > 0).all(), zaps
  # reach: the longer beam of closed and partnership hits 4 cells ahead; open's never does
  assert 4 in ahead.get(1, set()) | ahead.get(2, set()), ahead
  assert max(ahead.get(0, {0})) <= 3, ahead
  assert torch.equal(eng.active_variant.cpu(), torch.from_numpy(assign.astype(np.uint8)))
  ref.close()
  eng.close()


def test_a_map_set_batch_equals_homogeneous_engines_in_lockstep(any_event_width):
  blobs = CM.map_set()
  sms = _sms()
  for B in (1, 7, sms - 1, sms + 1, 2 * sms + 5):
    differ = _lockstep(blobs, blobs, _interleaved(B, 3), B, 45, seed=SEED)
  # reach: on the largest batch, the homogeneous engines of any two maps differ
  assert differ[~np.eye(3, dtype=bool)].all(), differ


def test_reassignment_moves_an_env_to_another_map_at_its_next_first(oracle):
  import torch
  from meltingpot_b200 import engine
  blobs = CM.map_set()
  B = 12
  first = _interleaved(B, 3)
  second = (first + 1) % 3  # partnership -> open (other kind tables), open -> closed (longer beam)
  third = (first + 2) % 3
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=first)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  envs = [oracle.OracleEnv(blobs[first[b]], SEED + b) for b in range(B)]
  pending = first.copy()
  rng = np.random.default_rng(11)
  eng.reset()
  for e in envs:
    e.reset()
  mask_b = np.arange(B) % 4 == 0
  moves = set()
  for t in range(1, 101):
    if t == 10:  # mid-episode: no env changes its map before its LAST
      eng.set_env_variant(second)
      pending = second.copy()
    if t == 60:  # a masked reset moves the masked envs at once, the others at their next LAST
      eng.set_env_variant(third)
      pending = third.copy()
      eng.reset(torch.from_numpy(mask_b.astype(np.uint8)).cuda())
      for b in np.flatnonzero(mask_b):
        moves.add(('mask', blobs.index(envs[b]._blob), int(pending[b])))
        envs[b] = _replace(oracle, envs[b], blobs[pending[b]], SEED + b)
    else:
      acts = rng.integers(0, eng.num_actions, size=(B, eng.num_players)).astype(np.int32)
      eng.step(torch.from_numpy(acts).cuda())
      for b in range(B):
        if envs[b].step_type() == 2:  # this step starts the next episode, on the pending map
          moves.add(('auto', blobs.index(envs[b]._blob), int(pending[b])))
          envs[b] = _replace(oracle, envs[b], blobs[pending[b]], SEED + b)
        else:
          envs[b].step(acts[b])
    px = t % 5 == 0 or t in (41, 42, 61)
    parity.check_outputs(parity.device_outputs(eng, ('rgb', 'world') if px else ()),
                         parity.env_dump(envs, shapes, pixels=px, max_events=max_ev), f'commons maps step {t}')
    active = eng.active_variant.cpu().numpy()
    assert all(envs[b]._blob == blobs[active[b]] for b in range(B)), f'active maps at step {t}: {active}'
  assert {('auto', 2, 0), ('auto', 0, 1), ('mask', 2, 0)} <= moves, moves
  eng.close()


def test_a_clone_keeps_its_source_map_and_a_snapshot_continues_byte_for_byte():
  import torch
  from meltingpot_b200 import engine
  blobs = CM.map_set()
  B = 12
  assign = _interleaved(B, 3)
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  rng = np.random.default_rng(13)
  eng.reset()
  for _ in range(7):
    eng.step(_actions(rng, B, eng.num_players, eng.num_actions))
  src, dst = [1, 4], [0, 3]  # closed envs into open envs' slots
  bank = torch.zeros((len(src), eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.tensor(src, dtype=torch.int32, device='cuda'))
  slot = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  slot[dst] = torch.arange(len(src), dtype=torch.int32, device='cuda')
  eng.restore_states(bank, slot)
  torch.cuda.synchronize()
  assert [int(eng.active_variant[j]) for j in dst] == [1, 1]
  for t in range(60):  # across the auto-reset: a clone plays its source's map (and key) through its next episode
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
  snap = eng.save_state()
  loaded = engine.Engine(list(blobs), B, seed=SEED)  # every env on open until the snapshot says otherwise
  loaded.load_state(snap)
  assert torch.equal(loaded.active_variant, eng.active_variant)
  for t in range(45):
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    eng.step(acts); loaded.step(acts)
    torch.cuda.synchronize()
    for name in _VIEWS + ('active_variant', 'pending_variant'):
      assert torch.equal(getattr(loaded, name), getattr(eng, name)), f'{name} {t} steps after the load'
  # records and snapshots only load into an engine of the same maps in the same order
  other = engine.Engine([blobs[1], blobs[0], blobs[2]], B, seed=SEED)
  with pytest.raises(ValueError, match='different compiled substrate'):
    other.load_state(snap)
  from meltingpot_b200 import substrate
  bank = torch.zeros((1, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.tensor([0], dtype=torch.int32, device='cuda'))
  assert other.state_tag != eng.state_tag
  with pytest.raises(ValueError, match='hold no record of this engine'):
    substrate.check_bank_tags(bank, [0], other.state_tag)
  other.reset()
  grid = other.grid.clone()
  other.restore_states(bank, torch.zeros(B, dtype=torch.int32, device='cuda'))  # a row without its tag is skipped
  torch.cuda.synchronize()
  assert torch.equal(other.grid, grid)
  for e in (eng, loaded, other):
    e.close()


def test_maps_with_other_apple_layouts_run_in_lockstep_and_match_the_oracle(oracle):
  from meltingpot_b200 import blob as blob_lib
  from meltingpot_b200 import engine
  blobs = CM.apple_set()
  n_apples = [len(blob_lib.unpack(b)['ch_apple']) for b in blobs]
  assert n_apples[1] < n_apples[0]
  sms = _sms()
  for B in (7, sms + 1):
    _lockstep(blobs, blobs, _interleaved(B, 2), B, 45, seed=SEED)
  B = 256
  assign = _blocks(B, 2)
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  ref = _MixedOracle(oracle, blobs, assign, SEED)
  rng = np.random.default_rng(7)
  eng.reset()
  for t in range(1, 46):
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    eng.step(acts)
    ref.step(acts.cpu().numpy())
    px = t in (20, 40, 41)
    parity.check_outputs(parity.device_outputs(eng, ('rgb', 'world') if px else ()), ref.dump(shapes, px, max_ev),
                         f'apple layouts step {t}')
  ref.close()
  eng.close()


def _without_event_rows(bank, max_events):
  """State records without their event rows, which also hold the rows of earlier steps past the step's count (no
  reader sees those): a record ends with the events [max_events][3] i32 and the event count, padded to 16 bytes."""
  r = bank.clone()
  n = r.shape[1]
  r[:, n - 16 - max_events * 12:n - 16] = 0
  return r


def test_an_env_that_moved_to_a_map_with_fewer_apples_stores_the_record_of_an_env_that_was_always_there():
  import torch
  from meltingpot_b200 import engine
  blobs = CM.apple_set()
  B = 8
  moved = engine.Engine(list(blobs), B, seed=SEED, env_variant=np.zeros(B, np.int64))
  always = engine.Engine(list(blobs), B, seed=SEED, env_variant=np.ones(B, np.int64))
  max_ev = int(moved.buffers.max_events)
  rng = np.random.default_rng(23)
  moved.reset(); always.reset()
  for t in range(1, 41):
    if t == 5:  # takes effect at the next FIRST
      moved.set_env_variant(np.ones(B, np.int64))
    acts = _actions(rng, B, moved.num_players, moved.num_actions)
    moved.step(acts); always.step(acts)
  torch.cuda.synchronize()
  assert (moved.step_type == 2).all() and (always.step_type == 2).all()
  # reach: when the episode on the larger map ended, an apple past the smaller map's count had been eaten, so its byte
  # in the env's apple row was not zero
  from meltingpot_b200 import blob as blob_lib
  big, small = (blob_lib.unpack(b) for b in blobs)
  layer, cells = int(big['ch_ip'][1]), int(moved.buffers.grid_cells)
  tail = big['ch_apple'][len(small['ch_apple']):, 1]
  init = big['init_grid'].reshape(-1, cells)[layer, tail]
  now = moved.grid.cpu().numpy()[:, layer, tail]
  assert (now != init[None]).any(), 'no apple past the smaller map\'s count was ever eaten'
  idx = torch.arange(B, dtype=torch.int32, device='cuda')
  for t in range(6):  # the FIRST step on the smaller map, then five more
    acts = _actions(rng, B, moved.num_players, moved.num_actions)
    moved.step(acts); always.step(acts)
    a = torch.zeros((B, moved.state_record_bytes), dtype=torch.uint8, device='cuda')
    b = torch.zeros_like(a)
    moved.store_states(a, idx); always.store_states(b, idx)
    torch.cuda.synchronize()
    assert torch.equal(moved.active_variant, always.active_variant)
    assert torch.equal(_without_event_rows(a, max_ev), _without_event_rows(b, max_ev)), f'records differ at step {t} on the smaller map'
    ge = parity._event_keys(moved.events.cpu().numpy(), moved.event_count.cpu().numpy())
    we = parity._event_keys(always.events.cpu().numpy(), always.event_count.cpu().numpy())
    assert np.array_equal(ge, we), f'events differ at step {t} on the smaller map'
  moved.close(); always.close()


def test_beam_variants_run_in_lockstep_and_size_the_event_rows_for_the_largest_footprint(any_event_width):
  from meltingpot_b200 import engine
  blobs = CM.beam_set()
  sms = _sms()
  differ = None
  for B in (7, sms + 1):
    differ = _lockstep(blobs, blobs, _interleaved(B, 3), B, 45, seed=SEED)
  assert differ[~np.eye(3, dtype=bool)].all(), differ
  # max_events = P * (3 * footprint cells + 4 + P), rounded up to 16: 9, 12 and 8 cells
  single = [int(engine.Engine(b, 4, seed=SEED).buffers.max_events) for b in blobs]
  assert single == [272, 336, 256], single
  assert int(engine.Engine(list(blobs), 4, seed=SEED).buffers.max_events) == max(single)
  # an engine of open alone keeps its single-map value; the map set is sized for closed's longer beam
  assert int(engine.Engine(CM.alone(CM.NAMES[0], capped=False), 4, seed=SEED).buffers.max_events) == 272
  assert int(engine.Engine(list(CM.map_set()), 4, seed=SEED).buffers.max_events) == 336


def test_maps_the_set_cannot_hold_are_refused_at_create():
  from meltingpot_b200 import engine, substrate, substrates
  wide = CM.compile_set([CM.settings(CM.NAMES[0], CM.CAP_40),
                         CM.settings(CM.NAMES[1], CM.CAP_40 + (CM.V.map_rows(lambda rows: [r + 'W' if r else r for r in rows]),))])
  with pytest.raises(ValueError, match="variant 1: section 'meta' differs in field 'W'"):
    engine.Engine(list(wide), 8, seed=SEED)
  with pytest.raises(ValueError, match="variant 1: .*field 'players'"):
    engine.Engine([substrates.load_blob(CM.NAMES[0], ('default',) * 16), substrates.load_blob(CM.NAMES[1], CM.ROLES)], 8, seed=SEED)
  with pytest.raises(ValueError, match='differs from'):
    substrate.build_batched(('clean_up', CM.NAMES[0]), roles=CM.ROLES, num_envs=8, seed=SEED)
  with pytest.raises(ValueError, match='variant 1: '):
    engine.Engine([substrates.load_blob('clean_up'), substrates.load_blob(CM.NAMES[0])], 8, seed=SEED)


def test_build_batched_over_names_equals_the_engine_and_routes_and_scenarios_over_it_equal_direct_stepping():
  import torch
  from meltingpot_b200 import engine, substrate, substrates
  B = 40
  sub = substrate.build_batched(CM.NAMES, roles=CM.ROLES, num_envs=B, seed=SEED, env_index_base=5)
  blobs = [substrates.load_blob(n, CM.ROLES) for n in CM.NAMES]
  assign = (np.arange(5, 5 + B) % 3).astype(np.int64)
  eng = engine.Engine(blobs, B, seed=SEED, env_index_base=5, env_variant=assign)
  assert np.array_equal(sub.engine.active_variant.cpu().numpy(), assign)
  rng = np.random.default_rng(17)
  sub.reset(); eng.reset()
  for _ in range(30):
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    ts = sub.step(acts)
    eng.step(acts)
    torch.cuda.synchronize()
    for name in _VIEWS:
      assert torch.equal(getattr(sub.engine, name), getattr(eng, name)), name
    assert torch.equal(ts.observation['READY_TO_SHOOT'], eng.scalar_obs[0])
  sub.set_env_variant(np.zeros(B, np.int64))
  assert int(sub.engine.pending_variant.sum()) == 0
  sub.close(); eng.close()
  # a repeated name weights the default assignment
  sub = substrate.build_batched(CM.NAMES[:2] + CM.NAMES[:1], roles=CM.ROLES, num_envs=6, seed=SEED)
  assert sub.engine.active_variant.cpu().tolist() == [0, 1, 2, 0, 1, 2]
  sub.close()


def test_player_routes_and_scenarios_over_a_map_set_batch_equal_direct_stepping():
  import torch
  from meltingpot_b200 import scenario, substrate
  from tests.test_gpu_scenario_routes import _hash_policy
  B = 24
  build = lambda: substrate.build_batched(CM.NAMES, roles=CM.ROLES, num_envs=B, seed=SEED)
  twin, env = build(), build()
  P = env.num_players
  rng = np.random.default_rng(2)
  routes = env.player_routes(rng.integers(-1, 3, size=(B, P)))
  traj = routes.outputs(T=46)
  env.reset(players=traj.at(0))
  twin.reset()
  for t in range(1, 46):
    a = _actions(rng, B, P, env.num_actions)
    ts = env.step(a, players=traj.at(t))
    want = twin.step(a)
    e, p = routes.env_of_row, routes.player_of_row
    assert torch.equal(ts.step_type, want.step_type) and torch.equal(ts.observation['WORLD.RGB'], want.observation['WORLD.RGB'])
    assert torch.equal(traj['RGB'][t], want.observation['RGB'][e, p]), t
    assert torch.equal(traj['REWARD'][t], want.reward[e, p]), t
    assert torch.equal(traj['READY_TO_SHOOT'][t], want.observation['READY_TO_SHOOT'][e, p]), t
  twin.close(); env.close()
  # BatchedScenario (focal players 0, 2, 3, 5; the rest background) against a substrate stepped with the merged actions
  is_focal = (True, False, True, True, False, True, False)
  focal = [i for i, f in enumerate(is_focal) if f]
  background = [i for i, f in enumerate(is_focal) if not f]
  seen = []
  direct = build()
  sc = scenario.BatchedScenario(build(), _hash_policy(direct.num_actions, seen), is_focal,
                                permitted_observations={'RGB', 'READY_TO_SHOOT'})
  sc.reset(); direct.reset()
  for t in range(1, 46):
    fa = _actions(rng, B, len(focal), direct.num_actions)
    ts = sc.step(fa)
    full = torch.zeros((B, P), dtype=torch.int32, device='cuda')
    full[:, focal] = fa
    full[:, background] = seen[-1]
    ref = direct.step(full)
    assert torch.equal(ts.step_type, ref.step_type) and torch.equal(ts.reward, ref.reward[:, focal]), t
    assert torch.equal(sc.background_timestep.reward, ref.reward[:, background]), t
    for key in ('RGB', 'READY_TO_SHOOT'):
      assert torch.equal(ts.observation[key], ref.observation[key][:, focal]), (key, t)
  direct.close()


def test_shard_slices_with_their_env_index_base_equal_one_map_set_engine():
  import torch
  from meltingpot_b200 import distributed, substrate
  B = 48
  full = substrate.build_batched(CM.NAMES, roles=CM.ROLES, num_envs=B, seed=SEED)
  shards = []
  for r in range(2):
    base, count = distributed.shard_envs(B, r, 2)
    shards.append((base, count, substrate.build_batched(CM.NAMES, roles=CM.ROLES, num_envs=count, seed=SEED,
                                                        env_index_base=base)))
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
    assert torch.equal(full.engine.active_variant[base:base + count], s.engine.active_variant)
    for name in ('rgb', 'world_rgb', 'reward', 'grid', 'avatar_state', 'timestep_packed'):
      assert torch.equal(getattr(full.engine, name)[base:base + count], getattr(s.engine, name)), name
