"""The substrate variants of tests/variants.py on the CPU: what the compiler makes of them, and what the oracle does.

Every 'parity' variant must compile into a blob that carries its override; every 'refused' one must be refused by the
compiler with NotImplementedError / ValueError (never another exception), or compile and be left to mp_create, as the
table says. The oracle steps each accepted variant and its reach predicate must hold there; the behaviours the
reference's Lua states are pinned with citations, as in test_oracle_semantics.py.
"""

import numpy as np
import pytest

from tests import variants as V

ENV_SEED = 7


def _family_sections(sec):
  return {k: v for k, v in sec.items() if k[:3] in ('cu_', 'ch_', 'tr_', 'co_', 'cm_') or k == 'meta' or k == 'comps_f'}


def _differs_from_stock(variant, sec):
  stock = V.sections(V.stock(variant.substrate, variant.players, variant.seed))
  mine = _family_sections(sec)
  return any(k not in stock or stock[k].shape != v.shape or not np.array_equal(stock[k], v) for k, v in mine.items())


# Decoded family fields for the variants whose knob has a slot of its own (compiler.py _*_tables).
CARRIES = {
    'clean_up/zap_cooldown_1': lambda s: s['cu_ip'][12] == 1,
    'clean_up/zap_lateral_28': lambda s: tuple(s['cu_ip'][13:15]) == (6, 2),
    'clean_up/zap_line_32': lambda s: tuple(s['cu_ip'][13:15]) == (32, 0),
    'clean_up/respawn_1': lambda s: s['cu_ip'][15] == 1,
    'clean_up/keep_hit_player': lambda s: s['cu_ip'][16] == 0,
    'clean_up/non_dyadic_rewards': lambda s: (s['cu_dp'][3], s['cu_dp'][4], s['cu_dp'][5]) == (0.1, 0.3, 0.7),
    'clean_up/clean_cooldown_0': lambda s: s['cu_ip'][18] == 0,
    'clean_up/clean_line_32': lambda s: tuple(s['cu_ip'][19:21]) == (32, 0),
    'clean_up/dirt_fills_river': lambda s: s['cu_ip'][25] == 0 and s['cu_dp'][6] == 1.0,
    'clean_up/apple_growth_rate_1': lambda s: s['cu_dp'][0] == 1.0,
    'clean_up/apple_thresholds_equal': lambda s: s['cu_dp'][1] == s['cu_dp'][2] == 0.0,
    'clean_up/animation_every_frame_random_start_True': lambda s: tuple(s['cu_ip'][10:12]) == (1, 1),
    'clean_up/animation_every_frame_random_start_False': lambda s: tuple(s['cu_ip'][10:12]) == (1, 0),
    'commons_harvest/zap_line_32': lambda s: tuple(s['ch_ip'][13:15]) == (32, 0),
    'commons_harvest/zap_lateral_28': lambda s: tuple(s['ch_ip'][13:15]) == (6, 2),
    'commons_harvest/respawn_1': lambda s: s['ch_ip'][15] == 1,
    'commons_harvest/keep_hit_player': lambda s: s['ch_ip'][16] == 0,
    'commons_harvest/non_dyadic_rewards': lambda s: (s['ch_dp'][4], s['ch_dp'][5], s['ch_dp'][6]) == (0.1, 0.3, 0.7),
    'commons/regrow_always': lambda s: list(s['ch_dp'][:4]) == [1.0] * 4,
    'commons/regrow_never': lambda s: list(s['ch_dp'][:4]) == [0.0] * 4,
    'commons/radius_1': lambda s: s['ch_ip'][5] == 5,
    'commons/radius_2_98': lambda s: s['ch_ip'][5] == 29 and (s['ch_nbr'] >= 0).sum(axis=1).max() >= 12,
    'territory/zap_lateral_28': lambda s: tuple(s['tr_ip'][13:15]) == (6, 2),
    'territory/health_1': lambda s: s['tr_ip'][28] == 1,
    'territory/health_200': lambda s: s['tr_ip'][28] == 200,
    'territory/fast_rewards': lambda s: tuple(s['tr_ip'][29:31]) == (0, 0) and tuple(s['tr_dp'][:3]) == (0.3, 1.0, 1.0),
    'territory/reward_delay_65535': lambda s: s['tr_ip'][29] == 65535,
    'territory/claim_wait_5': lambda s: s['tr_ip'][20] == 5,
    'territory/open_beams_32': lambda s: tuple(s['tr_ip'][13:15]) == (32, 0) and tuple(s['tr_ip'][18:20]) == (32, 0),
    'territory/rooms_zap_20': lambda s: tuple(s['tr_ip'][13:15]) == (20, 0),
    'territory/rooms_zap_radius_10': lambda s: tuple(s['tr_ip'][13:15]) == (1, 10),
    'territory/sanctions_1_level': lambda s: s['tr_ip'][11] == 1 and s['tr_ip'][10] == 1 and s['tr_ip'][34] == 2,
    'territory/sanctions_3_levels': lambda s: s['tr_ip'][11] == 3 and s['tr_ip'][41] == 1 and s['tr_ip'][42] == 0,
    'territory/sanctions_recovery_1': lambda s: s['tr_ip'][10] == 1,
    'coins/regrow_rate_1': lambda s: s['co_dp'][0] == 1.0,
    'coins/terminate_at_3': lambda s: tuple(s['co_ip'][4:6]) == (1, 3),
    'coins/non_dyadic_rewards': lambda s: abs(s['co_dp'][4] - 0.3 * 1.1) < 1e-15 and abs(s['co_dp'][6] + 0.1 * 3.0) < 1e-15,
    'coop_mining/live_rates_1': lambda s: tuple(s['cm_dp'][:2]) == (1.0, 1.0),
    'coop_mining/mining_window_1': lambda s: s['cm_ip'][6] == 1,
    'coop_mining/mining_window_255': lambda s: s['cm_ip'][6] == 255,
    'coop_mining/mine_cooldown_1': lambda s: s['cm_ip'][7] == 1,
    'coop_mining/mine_line_32': lambda s: s['cm_ip'][8] == 32,
}
for _fam, _ip in (('clean_up', 'cu_ip'), ('commons_harvest', 'ch_ip'), ('territory', 'tr_ip')):
  CARRIES.setdefault(f'{_fam}/zap_cooldown_1', lambda s, _ip=_ip: s[_ip][12] == 1)
for _v in V.PARITY:
  if '/end_every_frame' in _v.name:
    CARRIES[_v.name] = lambda s: True  # StochasticIntervalEpisodeEnding lives in the comps tables (checked below)
  if '/hard_cap_' in _v.name:
    CARRIES[_v.name] = lambda s, cap=int(_v.name.rsplit('_', 1)[1]): s['meta'][7] == cap
  if '/view_' in _v.name:
    CARRIES[_v.name] = lambda s: True  # the view window is checked by the reach predicate (meta 15..18)


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
    V.compile(name)  # the compiler accepts it; mp_create refuses it (test_gpu_param_envelope.py)
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
  return int(sec['co_ip'][2]), int(sec['co_ip'][3])


def test_coin_regrow_rate_1_regrows_every_waiting_coin_on_the_next_frame(oracle):
  # coins/components.lua:189-199: ChoiceCoinRegrow registers an updater on the wait state with probability regrowRate;
  # at 1.0 it fires on the first frame a coin spends waiting, so a coin collected on one step is back on the next.
  blob = V.compile('coins/regrow_rate_1')
  sec = V.sections(blob)
  n_coins = int(sec['co_ip'][0])
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
  assert stats['sprite_max'][int(sec['cu_ip'][4])] == 0
  # with the shipped thresholds (depletion 0.4, restoration 0) the same clean river grows apples at the full rate
  stats, sec = _rollout(V.compile('clean_up/apple_growth_rate_1'), oracle, 8, 200)
  assert stats['sprite_grew'][int(sec['cu_ip'][4])] > 0
