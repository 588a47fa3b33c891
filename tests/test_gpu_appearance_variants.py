"""Appearance overrides in one heterogeneous batch: envs whose pieces look different (recoloured or reshaped sprites, one
set on one sprite table) side by side in one engine, on every kernel family.

Env b of a mixed batch must equal, byte for byte, env b of the CPU oracle run on its variant's blob and env b of a
homogeneous engine of that blob. The variants (tests/appearance_variants.py) share a 40-frame cap, so every run of more
than 40 steps crosses an auto-reset.
"""

import numpy as np
import pytest

from tests import appearance_variants as AV
from tests import parity
from tests.test_gpu_env_variants import SEED, _VIEWS, _MixedOracle, _actions, _lockstep, _sms

pytestmark = pytest.mark.gpu


def _interleaved(B, n):
  return (np.arange(B) % n).astype(np.int64)


@pytest.mark.parametrize('name', AV.NAMES)
def test_every_env_of_a_mixed_appearance_batch_matches_the_oracle(oracle, name):
  import torch
  from meltingpot_b200 import engine
  B, steps = 2048, 45
  blobs = AV.blobs(name)
  assign = _interleaved(B, len(blobs))
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
    px = t in (0, 1, 20, 40, 41, 45)
    got = parity.device_outputs(eng, ('rgb', 'world') if px else ())
    parity.check_outputs(got, ref.dump(shapes, px, max_ev), f'{name} step {t}')
    lasts += int((got['step_type'] == 2).sum())
  assert lasts == B
  assert torch.equal(eng.active_variant.cpu(), torch.from_numpy(assign.astype(np.uint8)))
  ref.close()
  eng.close()


@pytest.mark.parametrize('name', AV.NAMES)
def test_a_mixed_appearance_batch_equals_homogeneous_engines_and_the_images_differ(name):
  import torch
  from meltingpot_b200 import engine
  blobs = AV.blobs(name)
  sms = _sms()
  for B in (1, 7, sms - 1, sms + 1, 2 * sms + 5, 2048):
    _lockstep(blobs, blobs, _interleaved(B, 4), B, 45)
  # reach: each appearance variant's images differ from the stock variant's, in WORLD.RGB and in the players' views,
  # while its grid only differs in sprite ids (same seed, same actions, same pieces)
  B = 16
  homo = [engine.Engine(b, B, seed=SEED) for b in blobs]
  rng = np.random.default_rng(8)
  world_differs, rgb_differs = np.zeros(4, bool), np.zeros(4, bool)
  for e in homo:
    e.reset()
  for t in range(45):
    acts = _actions(rng, B, homo[0].num_players, homo[0].num_actions)
    for e in homo:
      e.step(acts)
    torch.cuda.synchronize()
    for v in range(1, 4):
      world_differs[v] |= not torch.equal(homo[v].world_rgb, homo[0].world_rgb)
      rgb_differs[v] |= not torch.equal(homo[v].rgb, homo[0].rgb)
  assert world_differs[1:].all() and rgb_differs[1:].all(), (world_differs, rgb_differs)
  for e in homo:
    e.close()


@pytest.mark.parametrize('name', ['clean_up', 'territory__rooms', 'coop_mining'])
def test_set_env_variant_changes_the_appearance_at_the_next_episode_start_only(name):
  import torch
  from meltingpot_b200 import engine
  blobs = AV.blobs(name)
  B = 8
  mixed = engine.Engine(list(blobs), B, seed=SEED, env_variant=np.zeros(B, np.int64))
  homo = [engine.Engine(b, B, seed=SEED) for b in blobs[:2]]
  rng = np.random.default_rng(4)
  for e in [mixed] + homo:
    e.reset()
  for t in range(1, 61):
    if t == 5:
      mixed.set_env_variant(torch.ones(B, dtype=torch.uint8, device='cuda'))
    acts = _actions(rng, B, mixed.num_players, mixed.num_actions)
    for e in [mixed] + homo:
      e.step(acts)
    torch.cuda.synchronize()
    want = homo[0] if t <= 40 else homo[1]  # the 40-frame cap: step 41 starts the next episode
    for view in ('rgb', 'world_rgb', 'grid', 'reward'):
      assert torch.equal(getattr(mixed, view), getattr(want, view)), f'{view} at step {t}'
  for e in [mixed] + homo:
    e.close()


@pytest.mark.parametrize('name', ['clean_up', 'territory__inside_out'])
def test_a_clone_keeps_its_source_appearance_and_a_snapshot_continues_byte_for_byte(name):
  import torch
  from meltingpot_b200 import engine
  blobs = AV.blobs(name)
  B = 12
  assign = _interleaved(B, 4)
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  rng = np.random.default_rng(13)
  eng.reset()
  for _ in range(7):
    eng.step(_actions(rng, B, eng.num_players, eng.num_actions))
  src, dst = [1, 2, 3], [4, 8, 0]  # recoloured, reshaped and recolour + knob envs into other variants' slots
  bank = torch.zeros((len(src), eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.tensor(src, dtype=torch.int32, device='cuda'))
  slot = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  slot[dst] = torch.arange(len(src), dtype=torch.int32, device='cuda')
  eng.restore_states(bank, slot)
  torch.cuda.synchronize()
  assert [int(eng.active_variant[j]) for j in dst] == [1, 2, 3]
  for t in range(60):  # across the auto-reset: a clone keeps its source's appearance (and key) into its next episode
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
  loaded = engine.Engine(list(blobs), B, seed=SEED)  # every env stock until the snapshot says otherwise
  loaded.load_state(snap)
  for t in range(45):
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    eng.step(acts); loaded.step(acts)
    torch.cuda.synchronize()
    for view in _VIEWS + ('active_variant', 'pending_variant'):
      assert torch.equal(getattr(loaded, view), getattr(eng, view)), f'{view} {t} steps after the load'
  for e in (eng, loaded):
    e.close()


def test_routes_step_out_and_restores_in_a_step_on_a_mixed_appearance_batch():
  import torch
  from meltingpot_b200 import substrate
  blobs = list(AV.blobs('clean_up'))
  B, T = 24, 46
  assign = _interleaved(B, 4)
  build = lambda: substrate.BatchedSubstrate(blobs, B, seed=SEED, env_variant=assign)
  # player routes: each player's view, reward and scalars delivered to its row
  twin, env = build(), build()
  P = env.num_players
  rng = np.random.default_rng(2)
  routes = env.player_routes(rng.integers(-1, 3, size=(B, P)))
  traj = routes.outputs(T=T)
  env.reset(players=traj.at(0))
  twin.reset()
  for t in range(1, T):
    a = _actions(rng, B, P, env.num_actions)
    ts = env.step(a, players=traj.at(t))
    want = twin.step(a)
    e, p = routes.env_of_row, routes.player_of_row
    assert torch.equal(ts.observation['WORLD.RGB'], want.observation['WORLD.RGB']), t
    assert torch.equal(traj['RGB'][t], want.observation['RGB'][e, p]), t
    assert torch.equal(traj['REWARD'][t], want.reward[e, p]), t
  twin.close(); env.close()
  # step(out=) into a trajectory, with restores inside the step from stored states of other appearances
  into, twin = build(), build()
  out = into.trajectory(T)
  into.reset(); twin.reset()
  bank = into.state_bank(4)
  starts = torch.arange(B, device='cuda', dtype=torch.int32) % 4
  for t in range(T):
    a = _actions(rng, B, P, into.num_actions)
    if t == 3:
      into.store(bank, [0, 5, 10, 15], [0, 1, 2, 3])  # one env of each variant
    if t > 3:
      idx = torch.where(into.engine.step_type == 2, (starts + 1) % 4, -1).to(torch.int32)
      got = into.step(a, out=out.at(t), restore=idx, bank=bank)
      twin.step(a)
      twin.engine.restore_states(bank, idx)
      want = twin._timestep()  # pylint: disable=protected-access
    else:
      got = into.step(a, out=out.at(t))
      want = twin.step(a)
    torch.cuda.synchronize()
    for k in ('step_type', 'reward', 'discount'):
      assert torch.equal(getattr(got, k), getattr(want, k)) and torch.equal(getattr(out.at(t), k), getattr(want, k)), (k, t)
    for k, v in want.observation.items():
      assert torch.equal(out.at(t).observation[k], v), (k, t)
    assert torch.equal(into.engine.active_variant, twin.engine.active_variant), t
  into.close(); twin.close()


def test_shape_changes_next_to_an_appearance_override_are_refused_with_todays_messages():
  from meltingpot_b200 import compiler, engine
  from tests import env_variants as EV
  from tests import variants as V
  s = AV.settings('clean_up')
  recolour = {'potential_apple': AV.recoloured(s, 'potential_apple')}
  for edit, what in ((V.kw('Zapper', beamLength=9, beamRadius=0), "Params field 'zap.geom' differs"),
                     (V.kw('Cleaner', beamLength=2), 'beam footprints differ')):
    bad = EV.settings('clean_up', [edit])
    blobs = compiler.compile_settings_set([s, bad], AV.config('clean_up'), [None, None], [recolour, {}])
    with pytest.raises(ValueError, match=f'variant 1: .*{what}'):
      engine.Engine(blobs, 8, seed=SEED)


def test_a_union_too_large_for_shared_memory_is_refused_at_create_and_leaves_nothing_behind():
  import torch
  from meltingpot_b200 import compiler, engine
  s = AV.settings('territory__rooms')
  prefabs = [p for p, pf in s['simulation']['prefabs'].items()
             if any(c['component'] == 'Appearance' and c['kwargs'].get('spriteNames') for c in pf['components'])]
  overrides = [{}]
  for k in range(1, 4):  # every piece recoloured, three times over: far more than 96 sprites in the union
    o = {}
    for p in prefabs:
      for _ in range(k):
        s2 = compiler.apply_prefab_overrides(s, o)
        o[p] = AV.recoloured(s2, p)
    overrides.append(o)
  blobs = compiler.compile_settings_set([s] * 4, AV.config('territory__rooms'), [None] * 4, overrides)
  engine.Engine(AV.blobs('territory__rooms')[0], 4, seed=SEED).close()  # the context and the module are loaded
  torch.cuda.synchronize()
  free0 = torch.cuda.mem_get_info()[0]
  with pytest.raises(ValueError, match=r'sprites \(max 96\)'):
    engine.Engine(blobs, 64, seed=SEED, env_variant=_interleaved(64, 4))
  torch.cuda.synchronize()
  assert torch.cuda.mem_get_info()[0] == free0
