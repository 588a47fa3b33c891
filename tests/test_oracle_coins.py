"""Oracle semantics for the coins family (lua/levels/coins/components.lua), SURVEY.md section 8f row N1."""

import json

import numpy as np

from meltingpot_b200 import blob as mpb
from meltingpot_b200 import compiler
from meltingpot_b200 import substrates
from tests import settings_golden


def _tables(blob):
  sec = mpb.unpack(blob)
  return sec, json.loads(mpb.section_text(sec, 'info_json'))


def test_layout_and_specs(coins_blob):
  sec, info = _tables(coins_blob)
  meta = sec['meta']
  assert int(meta[0]) == 4 and int(meta[4]) == 2           # family coins, two players (components.lua:93-96)
  assert info['world_rgb_shape'] == [136, 136, 3]           # padded to the maximum map (coins.py:45-84, timestep_spec)
  assert info['individual_observation_names'] == ['RGB', 'MISMATCHED_COIN_COLLECTED_BY_PARTNER']
  assert len(info['action_set']) == 7                       # no zapping in coins
  params = compiler.family_params(sec)
  assert sorted((params['COIN_TYPE_0'], params['COIN_TYPE_1'])) == [0, 1]  # the two players own different coin types
  # player 1's self match, self mismatch, other match, other mismatch
  assert [params[f'REWARD_0_{r}'] for r in ('SELF_MATCH', 'SELF_MISMATCH', 'OTHER_MATCH', 'OTHER_MISMATCH')] == [1.0, 1.0, 0.0, -2.0]


def test_build_seed_fixes_the_python_side_randomness():
  a = settings_golden.compile('coins', 2, 3)
  assert a == settings_golden.compile('coins', 2, 3)
  shapes = {compiler.family_params(mpb.unpack(settings_golden.compile('coins', 2, s)))['N_COINS'] for s in range(6)}
  assert len(shapes) > 1  # different seeds draw different map sizes (coin counts)
  assert settings_golden.compile('coins', 2, substrates.BUILD_SEEDS['coins']) == substrates.load_blob('coins', ('default',) * 2)


def test_coins_appear_are_collected_and_pay_by_type(oracle, coins_blob):
  sec, info = _tables(coins_blob)
  types = [compiler.family_params(sec)[f'COIN_TYPE_{p}'] for p in range(2)]
  coin_kind = info['kinds'].index('coin')
  names = info['kind_states'][coin_kind]
  env = oracle.OracleEnv(coins_blob, 7)
  env.reset()
  assert all(names[env.object_state(int(o))] == 'coinWait' for o, _ in sec['co_coin'])  # every coin starts waiting
  rng = np.random.default_rng(0)
  seen = 0
  for _ in range(4000):
    if env.step(rng.integers(0, 7, 2)) == 2:
      break
    r = env.rewards()
    obs = env.scalar_obs()  # [P][n_scalar]
    mismatch_by = [False, False]
    expect = np.zeros(2)
    for name, player, matched in env.events():
      assert name == 'coin_consumed'
      seen += 1
      p = player - 1
      expect[p] += 1.0                      # rewardSelfForMatch == rewardSelfForMismatch == 1
      if not matched:
        expect[1 - p] += -2.0               # rewardOtherForMismatch
        mismatch_by[p] = True
    np.testing.assert_array_equal(r, expect)
    # MISMATCHED_COIN_COLLECTED_BY_PARTNER: set on the partner of whoever took a coin of the wrong type
    assert [bool(obs[0][0]), bool(obs[1][0])] == [mismatch_by[1], mismatch_by[0]]
  assert seen > 20
  assert sorted(types) == [0, 1]
