"""The substrate variants of tests/variants.py on the CPU: what the compiler makes of them, and what the oracle does.

Every 'parity' variant must compile into a blob that carries its override; every 'refused' one must be refused by the
compiler with NotImplementedError / ValueError (never another exception), or compile and be left to mp_create, as the
table says. The oracle steps each accepted variant and its reach predicate must hold there; the behaviours the
reference's Lua states are pinned with citations, as in test_oracle_semantics.py.
"""

import numpy as np
import pytest

from meltingpot_b200 import compiler
from tests import variants as V

ENV_SEED = 7


def _family_sections(sec):
  return {k: v for k, v in sec.items() if k[:3] in ('cu_', 'ch_', 'tr_', 'co_', 'cm_') or k == 'meta' or k == 'comps_f'}


def _differs_from_stock(variant, sec):
  stock = V.sections(V.stock(variant.substrate, variant.players, variant.seed))
  mine = _family_sections(sec)
  return any(k not in stock or stock[k].shape != v.shape or not np.array_equal(stock[k], v) for k, v in mine.items())


def _has(**want):
  """The blob's family parameters (compiler.family_params) include `want`."""
  return lambda s: all(compiler.family_params(s)[k] == v for k, v in want.items())


# Decoded family fields for the variants whose knob has a slot of its own (include/mpb_format.h).
CARRIES = {
    'clean_up/zap_cooldown_1': _has(ZAP_COOLDOWN=1),
    'clean_up/zap_lateral_28': _has(ZAP_LENGTH=6, ZAP_RADIUS=2),
    'clean_up/zap_line_32': _has(ZAP_LENGTH=32, ZAP_RADIUS=0),
    'clean_up/respawn_1': _has(ZAP_RESPAWN=1),
    'clean_up/keep_hit_player': _has(ZAP_REMOVE=0),
    'clean_up/non_dyadic_rewards': _has(EAT_REWARD=0.1, ZAP_PENALTY=0.3, ZAP_REWARD=0.7),
    'clean_up/clean_cooldown_0': _has(CLEAN_COOLDOWN=0),
    'clean_up/clean_line_32': _has(CLEAN_LENGTH=32, CLEAN_RADIUS=0),
    'clean_up/dirt_fills_river': _has(DIRT_DELAY=0, DIRT_PROB=1.0),
    'clean_up/apple_growth_rate_1': _has(GROW_RATE=1.0),
    'clean_up/apple_thresholds_equal': _has(GROW_DEPLETION=0.0, GROW_RESTORATION=0.0),
    'clean_up/animation_every_frame_random_start_True': _has(ANIM_FRAMES=1, ANIM_RANDOM=1),
    'clean_up/animation_every_frame_random_start_False': _has(ANIM_FRAMES=1, ANIM_RANDOM=0),
    'commons_harvest/zap_line_32': _has(ZAP_LENGTH=32, ZAP_RADIUS=0),
    'commons_harvest/zap_lateral_28': _has(ZAP_LENGTH=6, ZAP_RADIUS=2),
    'commons_harvest/respawn_1': _has(ZAP_RESPAWN=1),
    'commons_harvest/keep_hit_player': _has(ZAP_REMOVE=0),
    'commons_harvest/non_dyadic_rewards': _has(EAT_REWARD=0.1, ZAP_PENALTY=0.3, ZAP_REWARD=0.7),
    'commons/regrow_always': _has(PROB_0=1.0, PROB_1=1.0, PROB_2=1.0, PROB_3=1.0),
    'commons/regrow_never': _has(PROB_0=0.0, PROB_1=0.0, PROB_2=0.0, PROB_3=0.0),
    'commons/radius_1': _has(N_WAIT=5),
    'commons/radius_2_98': lambda s: _has(N_WAIT=29)(s) and (s['ch_nbr'] >= 0).sum(axis=1).max() >= 12,
    'territory/zap_lateral_28': _has(ZAP_LENGTH=6, ZAP_RADIUS=2),
    'territory/health_1': _has(RES_HEALTH=1),
    'territory/health_200': _has(RES_HEALTH=200),
    'territory/fast_rewards': _has(RES_REWARD_DELAY=0, RES_REPAIR_DELAY=0, RES_REWARD=0.3, RES_RATE=1.0, RES_REPAIR_PROB=1.0),
    'territory/reward_delay_65535': _has(RES_REWARD_DELAY=65535),
    'territory/claim_wait_5': _has(CLAIM_WAIT=5),
    'territory/open_beams_32': _has(ZAP_LENGTH=32, ZAP_RADIUS=0, CLAIM_LENGTH=32, CLAIM_RADIUS=0),
    'territory/rooms_zap_20': _has(ZAP_LENGTH=20, ZAP_RADIUS=0),
    'territory/rooms_zap_radius_10': _has(ZAP_LENGTH=1, ZAP_RADIUS=10),
    'territory/sanctions_1_level': _has(MARK_N_LEVELS=1, MARK_RECOVERY=1, MARK_FREEZE_0=2),
    'territory/sanctions_3_levels': _has(MARK_N_LEVELS=3, MARK_REMOVE_2=1, MARK_FREEZE_2=0),
    'territory/sanctions_recovery_1': _has(MARK_RECOVERY=1),
    'coins/regrow_rate_1': _has(REGROW_RATE=1.0),
    'coins/terminate_at_3': _has(TERMINATE=1, TERMINATE_N=3),
    'coins/non_dyadic_rewards': lambda s: (abs(compiler.family_params(s)['REWARD_0_SELF_MATCH'] - 0.3 * 1.1) < 1e-15 and
                                           abs(compiler.family_params(s)['REWARD_0_OTHER_MATCH'] + 0.1 * 3.0) < 1e-15),
    'coop_mining/live_rates_1': _has(RATE_0=1.0, RATE_1=1.0),
    'coop_mining/mining_window_1': _has(MINE_WINDOW=1),
    'coop_mining/mining_window_255': _has(MINE_WINDOW=255),
    'coop_mining/mine_cooldown_1': _has(MINE_COOLDOWN=1),
    'coop_mining/mine_line_32': _has(MINE_LENGTH=32),
}
for _fam in ('clean_up', 'commons_harvest', 'territory'):
  CARRIES.setdefault(f'{_fam}/zap_cooldown_1', _has(ZAP_COOLDOWN=1))
for _v in V.PARITY:
  if '/end_every_frame' in _v.name:
    CARRIES[_v.name] = lambda s: True  # StochasticIntervalEpisodeEnding lives in the comps tables (checked below)
  if '/hard_cap_' in _v.name:
    CARRIES[_v.name] = lambda s, cap=int(_v.name.rsplit('_', 1)[1]): s['meta'][compiler.META['MAX_FRAMES']] == cap
  if '/view_' in _v.name:
    CARRIES[_v.name] = lambda s: True  # the view window is checked by the reach predicate (meta VIEW_*)


def test_every_parity_variant_has_a_decoded_check():
  assert sorted(set(v.name for v in V.PARITY) - set(CARRIES)) == []


@pytest.mark.parametrize('name', [v.name for v in V.PARITY])
def test_parity_variant_compiles_and_carries_its_override(name):
  variant = V.BY_NAME[name]
  sec = V.sections(V.compile(name))
  assert _differs_from_stock(variant, sec), f'{name}: the compiled blob equals the stock one'
  assert CARRIES[name](sec), name
  if '/end_every_frame' in name:
    row = [c for c in sec['comps'] if int(c[0]) == 18][0]  # MPB_C_STOCHASTIC_INTERVAL_EPISODE_ENDING: min frames, interval
    assert (int(row[1]), int(row[2])) == (0, 1)


@pytest.mark.parametrize('name', [v.name for v in V.REFUSED])
def test_refused_variant_is_refused_cleanly(name):
  variant = V.BY_NAME[name]
  if variant.refused_by == 'compiler':
    with pytest.raises((NotImplementedError, ValueError)) as e:
      V.compile(name)
    if name == 'commons/dense_disc':
      assert 'more than 16 other apples' in str(e.value)
  else:
    V.compile(name)  # the compiler accepts it; mp_create refuses it (test_create_checks_cpu.py, test_gpu_param_envelope.py)
    assert variant.refused_by == 'engine'


def _rollout(blob, oracle, num_envs, steps, keep=(), seed=ENV_SEED):
  sec = V.sections(blob)
  m = sec['meta']
  P, A = int(m[4]), int(m[19])
  shapes = dict(P=P, L=int(m[3]), cells=int(m[1]) * int(m[2]), n_scalar=int(m[23]), rgb=(1, 1), world=(1, 1))
  batch = oracle.OracleBatch(blob, num_envs, seed=seed)
  stats = V.new_stats(num_envs, int(m[12]))
  rng = np.random.default_rng(0)
  for t in range(steps + 1):
    if t:
      batch.step_actions(rng.integers(0, A, size=(num_envs, P)).astype(np.int32), 4)
    d = batch.dump(4, shapes, pixels=False, max_events=1024, kinds=())
    V.observe(stats, t, d['reward'], d['step_type'], d['grid'], d['events'], d['n_events'], keep)
  batch.close()
  return stats, sec


@pytest.mark.parametrize('name', [v.name for v in V.PARITY])
def test_oracle_reaches_what_the_variant_is_for(name, oracle):
  variant = V.BY_NAME[name]
  blob = V.compile(name)
  stats, sec = _rollout(blob, oracle, 16, variant.steps, V.probe_sprites(variant, blob))
  assert variant.reach(stats, sec), f'{name}: {V.summary(stats)}'


# ---- behaviours the Lua states --------------------------------------------------------------------------------------

def test_hard_cap_ends_the_episode_on_its_last_frame(oracle):
  # base_simulation.lua: the episode ends once the frame counter reaches maxEpisodeLengthFrames; the next step is the
  # FIRST step of the next episode (policy A.17). With no stochastic ending every env ends on steps 40, 81, 122.
  stats, _ = _rollout(V.compile('territory/hard_cap_40'), oracle, 4, 125)
  assert sorted(stats['last_steps']) == [40, 81, 122] and set(stats['last_steps'].values()) == {4}
  assert sorted(stats['first_steps']) == [41, 82, 123]


def _coin_sprites(sec):
  params = compiler.family_params(sec)
  return params['COIN_SPRITE_0'], params['COIN_SPRITE_1']


def test_coin_regrow_rate_1_regrows_every_waiting_coin_on_the_next_frame(oracle):
  # coins/components.lua:189-199: ChoiceCoinRegrow registers an updater on the wait state with probability regrowRate;
  # at 1.0 it fires on the first frame a coin spends waiting, so a coin collected on one step is back on the next.
  blob = V.compile('coins/regrow_rate_1')
  sec = V.sections(blob)
  n_coins = compiler.family_params(sec)['N_COINS']
  env = oracle.OracleEnv(blob, ENV_SEED)
  env.reset()
  rng = np.random.default_rng(3)
  collected = 0
  a, b = _coin_sprites(sec)
  for _ in range(200):
    env.step(rng.integers(0, env.n_actions, size=env.P).astype(np.int32))
    now = sum(1 for name, _, _ in env.events() if name == 'coin_consumed')
    g = env.grid().astype(np.int64)
    live = int((((g - 1) >> 2 == a) & (g > 0)).sum() + (((g - 1) >> 2 == b) & (g > 0)).sum())
    assert live == n_coins - now, (live, n_coins, now)  # only this step's coins are waiting
    collected += now
  assert collected > 0


def test_coins_end_the_episode_when_a_player_has_collected_three(oracle):
  # coins/components.lua:149-162: Coin:onEnter adds one to the collecting player's cumulativeCoinsCollected and calls
  # endEpisode once it reaches coinsToTerminateEpisode, so the step on which some player collects its third coin of the
  # episode is LAST.
  blob = V.compile('coins/terminate_at_3')
  env = oracle.OracleEnv(blob, ENV_SEED)
  env.reset()
  rng = np.random.default_rng(5)
  per_player = np.zeros(env.P, np.int64)
  ends = 0
  for _ in range(400):
    env.step(rng.integers(0, env.n_actions, size=env.P).astype(np.int32))
    st = env.step_type()
    if st == 0:
      per_player[:] = 0
      continue
    for name, player, _ in env.events():
      if name == 'coin_consumed':
        per_player[player - 1] += 1
    assert (st == 2) == bool((per_player >= 3).any()), (st, per_player)
    ends += st == 2
  assert ends >= 3


def test_apple_growth_with_equal_thresholds_is_nan_and_grows_nothing(oracle):
  # clean_up/components.lua:64-80: interpolation = (dirtFraction - depletion) / (restoration - depletion) is 0/0 = NaN
  # when the thresholds and the fraction are equal; math.min(NaN, 1.0) keeps the NaN in Lua 5.1's lmathlib (its first
  # argument wins unless another is smaller), and random:uniform() < NaN is false: no apple grows (policy A.22). With a
  # clean river and no dirt spawning the fraction is 0 on every frame.
  stats, sec = _rollout(V.compile('clean_up/apple_thresholds_equal'), oracle, 8, 200)
  assert stats['sprite_max'][compiler.family_params(sec)['APPLE_SPRITE']] == 0
  # with the shipped thresholds (depletion 0.4, restoration 0) the same clean river grows apples at the full rate
  stats, sec = _rollout(V.compile('clean_up/apple_growth_rate_1'), oracle, 8, 200)
  assert stats['sprite_grew'][compiler.family_params(sec)['APPLE_SPRITE']] > 0
