"""Oracle semantics for the coop_mining family (lua/levels/coop_mining/components.lua), SURVEY.md section 8f row N1."""

import json

import numpy as np

from meltingpot_b200 import blob as mpb
from meltingpot_b200 import compiler


def _tables(blob):
  sec = mpb.unpack(blob)
  return sec, json.loads(mpb.section_text(sec, 'info_json'))


def _ore_in_front(env, sec, info, player, state_name):
  """Puts `player` on a free cell facing an ore and sets that ore's state; returns the ore's object id."""
  W = int(sec['meta'][1])
  walls = {int(o[2]) * W + int(o[1]) for o in sec['objects'] if info['kinds'][int(o[0])] == 'wall'}
  ores = {int(c): int(o) for o, c in sec['cm_ore']}
  names = info['kind_states'][info['kinds'].index('ore')]
  for cell, oid in sorted(ores.items()):
    stand = cell + W  # stand south of the ore, facing north (orientation 0)
    if stand in ores and stand not in walls and cell not in walls:
      env.debug_set_avatar(player, stand % W, stand // W, 0)
      env.debug_set_object_state(oid, names.index(state_name))
      return oid
  raise AssertionError('no ore with a free cell below it')


def test_layout(coop_mining_blob):
  sec, info = _tables(coop_mining_blob)
  meta = sec['meta']
  assert int(meta[0]) == 5 and int(meta[4]) == 6 and (int(meta[1]), int(meta[2])) == (27, 27)
  assert info['hits'] == ['mine'] and info['layers'][-1] == 'beamMine'   # MineBeam:addHits (:191-197)
  assert info['individual_observation_names'] == ['RGB', 'READY_TO_SHOOT']
  params = compiler.family_params(sec)
  assert [params[k] for k in ('MINE_REWARD_0', 'MINE_REWARD_1', 'EXTRACT_REWARD_0', 'EXTRACT_REWARD_1')] == [0.0, 0.0, 1.0, 8.0]  # role 'none': mining pays 0, extracting 1 / 8


def test_iron_is_extracted_by_one_miner_and_the_beam_cools_down(oracle, coop_mining_blob):
  sec, info = _tables(coop_mining_blob)
  names = info['kind_states'][info['kinds'].index('ore')]
  env = oracle.OracleEnv(coop_mining_blob, 2)
  env.reset()
  oid = _ore_in_front(env, sec, info, 0, 'ironRaw')
  mine = np.zeros(6, np.int32); mine[0] = 7
  env.step(mine)
  assert env.rewards()[0] == 1.0 and sorted(n for n, _, _ in env.events()) == ['extraction', 'mining']
  assert names[env.object_state(oid)] == 'oreWait'
  assert env.scalar_obs()[0][0] == 0.0                      # READY_TO_SHOOT right after firing (cooldown 3)
  env.step(mine)                                            # still cooling: nothing happens
  assert env.rewards()[0] == 0.0 and env.events() == []
  assert abs(env.scalar_obs()[0][0] - 1.0 / 3.0) < 1e-12


def test_gold_needs_two_miners_inside_the_window(oracle, coop_mining_blob):
  sec, info = _tables(coop_mining_blob)
  names = info['kind_states'][info['kinds'].index('ore')]
  W = int(sec['meta'][1])
  env = oracle.OracleEnv(coop_mining_blob, 5)
  env.reset()
  oid = _ore_in_front(env, sec, info, 0, 'goldRaw')
  cell = int([c for o, c in sec['cm_ore'] if int(o) == oid][0])
  idle = np.zeros(6, np.int32)
  one = idle.copy(); one[0] = 7
  env.step(one)                                            # first miner: partial, no reward for role 'none'
  assert names[env.object_state(oid)] == 'goldPartial' and env.rewards().sum() == 0.0
  assert [n for n, _, _ in env.events()] == ['mining']
  for _ in range(3):                                        # miningWindow = 3: the claim lapses, back to raw
    env.step(idle)
  assert names[env.object_state(oid)] == 'goldRaw'
  # second attempt with a partner standing two cells below, shooting through the first miner (avatars do not block 'mine')
  env.debug_set_avatar(1, cell % W, cell // W + 2, 0)
  env.step(idle); env.step(idle)                            # player 0's beam finishes cooling
  both = idle.copy(); both[0] = 7; both[1] = 7
  env.step(both)
  r = env.rewards()
  assert r[0] == 8.0 and r[1] == 8.0
  ev = sorted(env.events())
  assert [e[0] for e in ev] == ['extraction', 'extraction', 'extraction_pair', 'extraction_pair', 'mining', 'mining']
  assert names[env.object_state(oid)] == 'oreWait'


def test_random_play_pays_only_through_extraction(oracle, coop_mining_blob):
  env = oracle.OracleEnv(coop_mining_blob, 9)
  env.reset()
  rng = np.random.default_rng(3)
  probs = np.array([0.05, 0.15, 0.1, 0.1, 0.1, 0.1, 0.1, 0.3])
  total, extracted = 0.0, 0.0
  for _ in range(1500):
    env.step(rng.choice(8, size=6, p=probs))
    total += env.rewards().sum()
    for name, _, ore_type in env.events():
      if name == 'extraction':
        extracted += 1.0 if ore_type == 1 else 8.0
  assert total == extracted and total > 10
