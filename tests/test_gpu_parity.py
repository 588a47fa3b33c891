"""GPU (CUDA engine through the C ABI) == CPU oracle, bit for bit, on identical seeds/actions."""

import numpy as np
import pytest

from tests import parity

pytestmark = pytest.mark.gpu


def test_clean_up_random_rollout(clean_up_blob, oracle):
  stats = parity.compare_rollout(clean_up_blob, oracle, num_envs=16, steps=300, seed=1)
  assert stats['zaps'] > 0 and stats['cleaned'] > 0


def _cleaning_policy(t, B, P, A, rng):
  # Mostly clean/move so that the river gets clean, apples grow and get eaten.
  probs = np.array([0.05, 0.25, 0.05, 0.05, 0.05, 0.1, 0.1, 0.05, 0.3])
  return rng.choice(A, size=(B, P), p=probs)


def test_clean_up_cleaning_policy_grows_and_eats_apples(clean_up_blob, oracle):
  stats = parity.compare_rollout(clean_up_blob, oracle, num_envs=8, steps=700, seed=77,
                                 actions_fn=_cleaning_policy, pixels_every=7)
  assert stats['cleaned'] > 0


def test_clean_up_sharding_invariance(clean_up_blob, oracle):
  # env b of a shard that starts at env_index_base behaves like global env base+b.
  parity.compare_rollout(clean_up_blob, oracle, num_envs=4, steps=40, seed=5, env_index_base=1000)


def test_clean_up_clean_river_apples_grow_and_get_eaten(clean_river_blob, oracle):
  # Variant map (tools/make_test_blobs.py): river starts clean, so AppleGrow / Edible are exercised.
  stats = parity.compare_rollout(clean_river_blob, oracle, num_envs=12, steps=400, seed=9, pixels_every=5)
  assert stats['eaten'] > 20 and stats['rewards'] > 20


def test_clean_up_full_batch_size_invariants(clean_up_blob, oracle):
  # BASELINE.json config 2 size: 4096 envs. EVERY env is compared with the oracle (state, rewards, events on every
  # step; every RGB byte every 10 steps); the batch is also checked through size-independent properties.
  import torch
  from meltingpot_b200 import engine
  B = 4096
  stats = parity.compare_batch(clean_up_blob, oracle, num_envs=B, steps=60, seed=21, pixels_every=10)
  assert stats['pixel_checks'] == 7 and stats['events'] > 1000
  eng = engine.Engine(clean_up_blob, B, seed=21)
  eng.reset()
  first = eng.world_rgb.clone()
  # every env renders a full frame: no pixel of WORLD.RGB is left at the allocation's zero fill inside the walls
  assert int((eng.world_rgb[:, 8:-8, 8:-8] == 0).all(dim=-1).sum()) == 0
  # walls never change: the border ring is identical across envs and across steps
  ring = eng.world_rgb[:, :8].clone()
  assert bool((ring == ring[0]).all())
  gen = torch.Generator(device='cuda').manual_seed(0)
  for _ in range(30):
    eng.step(torch.randint(0, 9, (B, 7), generator=gen, device='cuda', dtype=torch.int32))
  assert bool((eng.world_rgb[:, :8] == ring).all())
  assert bool((eng.step_type == 1).all()) and bool((eng.discount == 1.0).all())
  assert bool((eng.reward >= 0).all())
  # envs with different seeds diverge, identical seeds stay identical
  assert not bool((eng.world_rgb == first).all())
  twin = engine.Engine(clean_up_blob, 64, seed=21)
  twin.reset()
  gen = torch.Generator(device='cuda').manual_seed(0)
  for _ in range(30):
    a = torch.randint(0, 9, (B, 7), generator=gen, device='cuda', dtype=torch.int32)
    twin.step(a[:64].contiguous())
  assert bool((twin.rgb == eng.rgb[:64]).all()) and bool((twin.world_rgb == eng.world_rgb[:64]).all())


def test_clean_up_episode_boundary_auto_reset(clean_up_blob, oracle):
  # Runs past the first possible episode end (frame 1099) so LAST -> FIRST transitions are compared.
  stats = parity.compare_rollout(clean_up_blob, oracle, num_envs=24, steps=1320, seed=300, pixels_every=97)
  assert stats['lasts'] > 0


def test_dm_env_substrate_api(clean_up_blob):
  from meltingpot_b200 import shims, substrate
  shims.install()
  import dm_env
  with substrate.build('clean_up', roles=('default',) * 7, env_seed=5) as env:
    ts = env.reset()
    assert ts.step_type == dm_env.StepType.FIRST and ts.discount == 0.0 and ts.reward == [0.0] * 7
    assert len(ts.observation) == 7
    keys = {'RGB', 'READY_TO_SHOOT', 'NUM_OTHERS_WHO_CLEANED_THIS_STEP', 'WORLD.RGB', 'COLLECTIVE_REWARD'}
    assert set(ts.observation[0]) == keys
    assert ts.observation[0]['WORLD.RGB'] is ts.observation[6]['WORLD.RGB']
    # assert_step_matches_specs (meltingpot/testing/substrates.py:22-68)
    for obs, spec in zip(ts.observation, env.observation_spec()):
      for k, v in obs.items():
        spec[k].validate(v)
    actions = [spec.maximum for spec in env.action_spec()]
    ts = env.step(actions)
    assert ts.step_type == dm_env.StepType.MID and ts.discount == 1.0
    for r, spec in zip(ts.reward, env.reward_spec()):
      spec.validate(r)
    env.discount_spec().validate(ts.discount)
    with pytest.raises(ValueError):
      env.step([0] * 6)
    with pytest.raises(ValueError):
      env.step([9] * 7)
  # same env_seed => identical first frame (builder_test.py:47-70)
  a = substrate.build('clean_up', roles=('default',) * 7, env_seed=5)
  b = substrate.build('clean_up', roles=('default',) * 7, env_seed=6)
  fa, fb = a.reset().observation[0]['WORLD.RGB'], b.reset().observation[0]['WORLD.RGB']
  assert np.array_equal(fa, ts_first_world(5)) and not np.array_equal(fa, fb)
  assert not np.array_equal(a.reset().observation[0]['WORLD.RGB'], fa)  # next episode differs
  a.close(); b.close()


def ts_first_world(seed):
  from meltingpot_b200 import substrate
  with substrate.build('clean_up', roles=('default',) * 7, env_seed=seed) as env:
    return env.reset().observation[0]['WORLD.RGB']


def test_commons_harvest_random_rollout(commons_blob, oracle):
  stats = parity.compare_rollout(commons_blob, oracle, num_envs=16, steps=500, seed=3, pixels_every=3)
  assert stats['eaten'] > 50 and stats['zaps'] > 0


def test_commons_harvest_16_players(commons16_blob, oracle):
  # BASELINE.json config 3 shape: 16 players (2 inside spawn points + 60 outside).
  stats = parity.compare_rollout(commons16_blob, oracle, num_envs=8, steps=400, seed=11, pixels_every=5)
  assert stats['eaten'] > 50


def test_territory_rooms_random_rollout(territory_blob, oracle):
  # TORUS map, 9 players: claims, zaps on resources, graduated sanctions, removals.
  stats = parity.compare_rollout(territory_blob, oracle, num_envs=16, steps=600, seed=4, pixels_every=3)
  assert stats['rewards'] > 50


def _zap_heavy(t, B, P, A, rng):
  probs = np.array([0.05, 0.3, 0.05, 0.05, 0.05, 0.1, 0.1, 0.2, 0.1])
  return rng.choice(A, size=(B, P), p=probs)


def test_territory_rooms_zap_heavy(territory_blob, oracle):
  stats = parity.compare_rollout(territory_blob, oracle, num_envs=12, steps=500, seed=17, actions_fn=_zap_heavy, pixels_every=5)
  assert stats['zaps'] > 20


def test_territory_open_random_rollout(territory_open_blob, oracle):
  # SURVEY.md section 8f N1: BOUNDED 39x23 map (wider than 32 cells: 5 cells per lane per WORLD.RGB strip).
  stats = parity.compare_rollout(territory_open_blob, oracle, num_envs=12, steps=500, seed=6, pixels_every=3)
  assert stats['rewards'] > 50


def test_commons_harvest_closed_random_rollout(commons_closed_blob, oracle):
  # SURVEY.md section 8f N1: same components as commons_harvest__open on a walled map.
  stats = parity.compare_rollout(commons_closed_blob, oracle, num_envs=16, steps=500, seed=8, pixels_every=3)
  assert stats['eaten'] > 20


def test_territory_inside_out_random_rollout(territory_inside_out_blob, oracle):
  # SURVEY.md section 8f N1: 5 players; the map's 'choice' prefabs are drawn once per blob (policy A.20).
  stats = parity.compare_rollout(territory_inside_out_blob, oracle, num_envs=12, steps=500, seed=12, pixels_every=3)
  assert stats['rewards'] > 50


def test_commons_harvest_partnership_random_rollout(commons_partnership_blob, oracle):
  # SURVEY.md section 8f N1: adds the (inert for default roles) Role / RoleBasedRewardTile components.
  stats = parity.compare_rollout(commons_partnership_blob, oracle, num_envs=16, steps=500, seed=14, pixels_every=3)
  assert stats['eaten'] > 20


def test_events_reach_the_dm_env_api(clean_up_blob):
  # SURVEY.md section 8f N3: substrate.events() / observables().events carry the hot path's events:add calls.
  from meltingpot_b200 import substrate
  seen = []
  with substrate.build('clean_up', roles=('default',) * 7, env_seed=4) as env:
    env.observables().events.subscribe(seen.append)
    env.reset()
    rng = np.random.default_rng(0)
    names = set()
    for _ in range(400):
      env.step(rng.integers(0, 9, 7))
      for name, payload in env.events():
        names.add(name)
        assert payload[0] == b'dict' and payload[1] in (b'source', b'player_index')
        assert 1 <= int(payload[2]) <= 7
  assert 'player_cleaned' in names and 'zap' in names
  assert len(seen) > 0 and all(isinstance(e, tuple) for e in seen)


def test_coins_random_rollout(coins_blob, oracle):
  # SURVEY.md section 8f N1: the eighth substrate of the sweep; two players, no beams, coin_consumed events.
  # (64 envs: a coin appears during the start update of an episode in about one env in twenty)
  stats = parity.compare_rollout(coins_blob, oracle, num_envs=64, steps=700, seed=31, pixels_every=7)
  assert stats['events'] > 30


def _mine_heavy(t, B, P, A, rng):
  probs = np.array([0.05, 0.15, 0.1, 0.1, 0.1, 0.1, 0.1, 0.3])
  return rng.choice(A, size=(B, P), p=probs)


def test_coop_mining_rollout(coop_mining_blob, oracle):
  # SURVEY.md section 8f N1: ninth substrate; beams fired from component updates, two Ore components per ore object.
  stats = parity.compare_rollout(coop_mining_blob, oracle, num_envs=16, steps=1300, seed=41, actions_fn=_mine_heavy, pixels_every=5)
  assert stats['events'] > 200 and stats['rewards'] > 50


def test_commons_harvest_config3_batch_size(commons16_blob, oracle):
  # BASELINE.json config 3 size: 16 players x 8192 envs on one GPU; every env against the oracle.
  stats = parity.compare_batch(commons16_blob, oracle, num_envs=8192, steps=40, seed=51, pixels_every=20)
  assert stats['events'] > 1000 and stats['pixel_checks'] == 3


def test_territory_rooms_config4_shard_size(territory_blob, oracle):
  # BASELINE.json config 4: 16384 envs sharded 2048 per GPU; this is rank 5's shard (env_index_base = 5 * 2048).
  # Every env of the shard against the oracle.
  stats = parity.compare_batch(territory_blob, oracle, num_envs=2048, steps=40, seed=61, pixels_every=8, env_index_base=5 * 2048)
  assert stats['events'] > 0 and stats['pixel_checks'] == 6


@pytest.mark.parametrize('name,players', [
    ('clean_up', 7), ('commons_harvest__open', 7), ('commons_harvest__closed', 7), ('commons_harvest__partnership', 7),
    ('territory__rooms', 9), ('territory__open', 9), ('territory__inside_out', 5), ('coins', 2), ('coop_mining', 6)])
def test_config5_sweep_at_2048_envs(name, players, oracle):
  # BASELINE.json config 5: the substrates of the sweep at 2048 envs each; every env against the oracle.
  from meltingpot_b200 import substrates
  blob = substrates.load_blob(name, ('default',) * players)
  stats = parity.compare_batch(blob, oracle, num_envs=2048, steps=30, seed=71, pixels_every=6)
  assert stats['pixel_checks'] == 6


def test_inside_out_envs_of_one_batch_have_their_own_layouts(territory_inside_out_blob):
  # Deviation A.20 is gone for 'choice' prefabs: every env (and episode) draws its own resources / spawn points.
  import torch
  from meltingpot_b200 import blob as blob_lib, compiler, engine
  sec = blob_lib.unpack(territory_inside_out_blob)
  cells = torch.as_tensor(sec['tr_res'][:, 1].astype(np.int64), device='cuda')
  res_layer = compiler.family_params(sec)['RES_LAYER']
  eng = engine.Engine(territory_inside_out_blob, 256, seed=3)
  eng.reset()
  torch.cuda.synchronize()
  present = eng.grid[:, res_layer][:, cells] != 0
  assert len({tuple(row.tolist()) for row in present.cpu()}) > 250          # (almost) every env its own layout
  first = present.clone()
  eng.reset()
  torch.cuda.synchronize()
  assert not torch.equal(eng.grid[:, res_layer][:, cells] != 0, first)      # and a new one every episode
  frac = float(first.float().mean())
  cond = sec['tr_res_cond']
  assert (cond[:, 0] < 0).mean() < frac < 1.0
