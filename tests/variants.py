"""TEST INFRASTRUCTURE: substrate variants at the edges of what the compiler and mp_create accept.

Every shipped blob sits at one point of each substrate parameter (11x11 views, 5000-frame episodes, one beam shape per
substrate, probabilities strictly between 0 and 1, integer rewards). The variants below move one knob, or one coherent
group of knobs, of the stored lab2d settings (tests/golden/settings_*.json.gz) and compile the result at test time, so
no reference checkout is needed. Each entry says whether the engine must match the oracle bit for bit ('parity') or
refuse the variant ('refused', by the compiler or by mp_create), and carries a reach predicate on the rollout
statistics: it proves that the knob changed what happened, so that no parity variant passes vacuously.

Checks of mp_create (meltingpot_b200/csrc/engine.cu) with a value on each side in the table:
  zap / mine cooldown >= 1 ............. zap_cooldown_1 / zap_cooldown_0, mine_cooldown_1 / mine_cooldown_0
  clean cooldown >= 0 .................. clean_cooldown_0 / clean_cooldown_negative
  beam footprint <= 32 cells ........... zap_line_32, zap_lateral_28 / zap_33_cells
  TORUS beam < min(W, H) ............... rooms_zap_20, rooms_zap_radius_10 / rooms_zap_21, rooms_claim_21, rooms_zap_radius_11
  DensityRegrow wait states <= 29 ...... radius_2_98 / radius_3
  resource health 1..200 ............... health_1, health_200 / health_201
  rewardDelay / delayTillSelfRepair .... reward_delay_65535 / reward_delay_65536, repair_delay_65536
  mining window 1..255 ................. mining_window_1, mining_window_255 / mining_window_256
  marking levels 1..3 .................. sanctions_1_level, sanctions_3_levels
  territory never respawns ............. (shipped 1e6 frames) / territory/respawn_1
  view <= 16 cells wide ................ view_16 / view_17
"""

import collections
import functools
import types

import numpy as np

from tests import settings_golden

# ---- settings overrides -----------------------------------------------------------------------------------------------


def _components(settings):
  sim = settings['simulation']
  objs = list(sim.get('gameObjects', [])) + [sim.get('scene', {})] + list(sim.get('prefabs', {}).values())
  for obj in objs:
    for c in obj.get('components', []) or []:
      yield c


def set_kwargs(settings, component, **kw):
  """Sets `kw` on every component named `component` (avatars, scene and prefabs alike). Returns how many it changed."""
  n = 0
  for c in _components(settings):
    if c['component'] == component:
      c.setdefault('kwargs', {}).update(kw)
      n += 1
  if not n:
    raise KeyError(f'no {component} component in these settings')
  return n


def states_of(settings, prefab):
  """The stateConfigs list of a prefab's StateManager (edited in place)."""
  for c in settings['simulation']['prefabs'][prefab]['components']:
    if c['component'] == 'StateManager':
      return c['kwargs']['stateConfigs']
  raise KeyError(prefab)


def kw(component, **values):
  return lambda s: set_kwargs(s, component, **values)


def top(**values):
  return lambda s: s.update(values)


def map_replace(old, new):
  def edit(s):
    assert old in s['simulation']['map']
    s['simulation']['map'] = s['simulation']['map'].replace(old, new)
  return edit


def map_rows(fn):
  def edit(s):
    rows = s['simulation']['map'].split('\n')
    s['simulation']['map'] = '\n'.join(fn(rows))
  return edit


def view(left, right, forward, backward):
  return kw('Avatar', view=dict(left=left, right=right, forward=forward, backward=backward, centered=False))


def density_radius(radius):
  """DensityRegrow radius with the appleWait_<k> states the reference's apple prefab builds for it
  (commons_harvest__open.py:336-338: floor(pi r^2 + 1) + 1 of them)."""
  def edit(s):
    set_kwargs(s, 'DensityRegrow', radius=radius)
    sts = states_of(s, 'apple')
    template = next(st for st in sts if st['state'] == 'appleWait_0')
    keep = [st for st in sts if not st['state'].startswith('appleWait_')]
    upper = int(np.floor(np.pi * radius ** 2 + 1)) + 1
    s['simulation']['prefabs']['apple']['components'][0]['kwargs']['stateConfigs'] = keep + [
        dict(template, state=f'appleWait_{i}') for i in range(upper)]
  return edit


def marking_levels(hit_logic, recovery):
  """GraduatedSanctionsMarking with len(hit_logic) levels; adds the level_<k> states the marking objects lack."""
  def edit(s):
    set_kwargs(s, 'GraduatedSanctionsMarking', hitLogic=hit_logic, recoveryTime=recovery)
    for obj in s['simulation']['gameObjects']:
      comps = obj['components']
      if not any(c['component'] == 'GraduatedSanctionsMarking' for c in comps):
        continue
      sts = comps[0]['kwargs']['stateConfigs']
      have = {st['state'] for st in sts}
      level = next(st for st in sts if st['state'] == 'level_2')
      for i in range(1, len(hit_logic) + 1):
        if f'level_{i}' not in have:
          sts.insert(i - 1, dict(level, state=f'level_{i}'))
  return edit


# ---- rollout statistics -----------------------------------------------------------------------------------------------

EVENT_NAMES = {1: 'zap', 2: 'edible_consumed', 3: 'player_cleaned', 4: 'claimed_resource', 5: 'destroyed_resource',
               6: 'sanctioning', 7: 'removal_due_to_sanctioning', 8: 'coin_consumed', 9: 'mining', 10: 'extraction',
               11: 'extraction_pair'}


def new_stats(num_envs, n_sprites):
  return dict(envs=num_envs, steps=0, rewards=0.0, reward_values=set(), lasts=0, last_steps=collections.Counter(),
              first_steps=collections.Counter(), events=collections.Counter(),
              sprite_max=np.zeros(n_sprites, np.int64), sprite_grew=np.zeros(n_sprites, np.int64),
              sprite_fell=np.zeros(n_sprites, np.int64), sprites_seen=[], _prev=None)


def observe(stats, t, reward, step_type, grid, events, n_events, keep_sprites=()):
  """Folds step t (0 = the reset) of a batch into `stats`. grid: uint16 [B, L, cells] (0 empty, else 1 + sprite * 4 +
  orientation); events: [B, M, 3]. `sprite_grew[s]` / `sprite_fell[s]` count (env, MID step) pairs in which the number
  of cells showing sprite s went up / down; `sprites_seen` keeps env 0's count of each sprite in `keep_sprites`."""
  B = grid.shape[0]
  S = stats['sprite_max'].shape[0]
  v = grid.reshape(B, -1).astype(np.int64)
  sprite = np.where(v > 0, (v - 1) >> 2, S)
  counts = np.bincount((sprite + (S + 1) * np.arange(B)[:, None]).ravel(), minlength=B * (S + 1)).reshape(B, S + 1)[:, :S]
  stats['sprite_max'] = np.maximum(stats['sprite_max'], counts.max(axis=0))
  prev = stats['_prev']
  if prev is not None:
    mid = (step_type == 1)[:, None]
    stats['sprite_grew'] += ((counts > prev) & mid).sum(axis=0)
    stats['sprite_fell'] += ((counts < prev) & mid).sum(axis=0)
  stats['_prev'] = counts
  if keep_sprites:
    stats['sprites_seen'].append(tuple(int(counts[0, s]) for s in keep_sprites))
  if t > 0:
    stats['steps'] += 1
    stats['rewards'] += float(reward.sum())
    stats['reward_values'].update(float(r) for r in np.unique(reward))
    n_last = int((step_type == 2).sum())
    stats['lasts'] += n_last
    if n_last:
      stats['last_steps'][t] += n_last
    n_first = int((step_type == 0).sum())
    if n_first:
      stats['first_steps'][t] += n_first
  for b in range(B):
    for row in events[b, :int(n_events[b])]:
      stats['events'][EVENT_NAMES[int(row[0])]] += 1


def summary(stats):
  """Stats without the bulky fields, for assertion messages."""
  return {k: (dict(v) if isinstance(v, collections.Counter) else v) for k, v in stats.items()
          if k not in ('sprite_max', 'sprite_grew', 'sprite_fell', 'sprites_seen', '_prev', 'reward_values')} | {
              'reward_values': sorted(stats['reward_values'])[:12]}


# ---- the variants -----------------------------------------------------------------------------------------------------

Variant = collections.namedtuple('Variant', 'name substrate players seed edits expect refused_by reach steps probe')
Variant.__new__.__defaults__ = (None, None, 200, None)

# What a variant's reach predicate sees: the stats above and the decoded blob sections of the variant.
EV = lambda s, name: s['events'][name]


def _sec(blob):
  from meltingpot_b200 import blob as blob_lib
  return blob_lib.unpack(blob)


def _nondyadic(s):
  """Some per-player reward of some step is not a whole number."""
  return any(abs(v - round(v)) > 1e-12 for v in s['reward_values'])


def _multi_term(terms):
  """Some per-player reward of some step is a sum of two or more non-zero terms (none of the single terms)."""
  single = {0.0} | {float(t) for t in terms}
  return lambda s, sec: any(v not in single for v in s['reward_values'])


_ENDING = 'StochasticIntervalEpisodeEnding'
_FAMILIES = [('clean_up', 7, None), ('commons_harvest__open', 7, None), ('territory__rooms', 9, None), ('coins', 2, 0),
             ('coop_mining', 6, None)]
_ZAPPERS = [('clean_up', 7), ('commons_harvest__open', 7), ('territory__rooms', 9)]


def _cap_pattern(cap):
  """LAST on exactly the steps cap, 2 cap + 1, ... (every env), FIRST on the step after each."""
  def reach(s, sec):
    lasts = sorted(s['last_steps'])
    want = list(range(cap, s['steps'] + 1, cap + 1))
    return (lasts == want and all(s['last_steps'][t] == s['envs'] for t in want)
            and sorted(s['first_steps']) == [t + 1 for t in want if t + 1 <= s['steps']]
            and all(n == s['envs'] for n in s['first_steps'].values()))
  return reach


def _grew(ip_name, ip_index):
  return lambda s, sec: s['sprite_grew'][int(sec[ip_name][ip_index])] > 0


def _never_grew(ip_name, ip_index):
  return lambda s, sec: s['sprite_grew'][int(sec[ip_name][ip_index])] == 0 and s['sprite_fell'][int(sec[ip_name][ip_index])] > 0


def _variants():
  v = []
  add = lambda *a, **k: v.append(Variant(*a, **k))
  # ---- episode ending, every family
  for sub, p, seed in _FAMILIES:
    fam = sub.split('__')[0]
    add(f'{fam}/end_every_frame', sub, p, seed,
        [kw(_ENDING, probabilityTerminationPerInterval=1.0, minimumFramesPerEpisode=0, intervalLength=1)], 'parity',
        reach=_cap_pattern(1), steps=40)
    add(f'{fam}/hard_cap_40', sub, p, seed, [kw(_ENDING, probabilityTerminationPerInterval=0.0), top(maxEpisodeLengthFrames=40)],
        'parity', reach=_cap_pattern(40), steps=130)
    add(f'{fam}/hard_cap_1', sub, p, seed, [top(maxEpisodeLengthFrames=1)], 'parity', reach=_cap_pattern(1), steps=20)
  # ---- Zapper
  for sub, p in _ZAPPERS:
    fam = sub.split('__')[0]
    add(f'{fam}/zap_cooldown_1', sub, p, None, [kw('Zapper', cooldownTime=1)], 'parity',
        reach=lambda s, sec: EV(s, 'zap') > 0)
    add(f'{fam}/zap_cooldown_0', sub, p, None, [kw('Zapper', cooldownTime=0)], 'refused', 'engine')
    add(f'{fam}/zap_lateral_28', sub, p, None, [kw('Zapper', beamLength=6, beamRadius=2)], 'parity',
        reach=lambda s, sec: EV(s, 'zap') > 0)
    add(f'{fam}/zap_33_cells', sub, p, None, [kw('Zapper', beamLength=7, beamRadius=2)], 'refused', 'engine')
  for sub, p in _ZAPPERS[:2]:
    fam = sub.split('__')[0]
    add(f'{fam}/zap_line_32', sub, p, None, [kw('Zapper', beamLength=32, beamRadius=0)], 'parity',
        reach=lambda s, sec: EV(s, 'zap') > 0)
    add(f'{fam}/respawn_1', sub, p, None, [kw('Zapper', framesTillRespawn=1, cooldownTime=1)], 'parity',
        reach=lambda s, sec: EV(s, 'zap') > 0)
    add(f'{fam}/keep_hit_player', sub, p, None, [kw('Zapper', removeHitPlayer=False, cooldownTime=1)], 'parity',
        reach=lambda s, sec: EV(s, 'zap') > 0)
    add(f'{fam}/non_dyadic_rewards', sub, p, None,
        [kw('Zapper', rewardForZapping=0.7, penaltyForBeingZapped=0.3, cooldownTime=1), kw('Edible', rewardForEating=0.1)],
        'parity', reach=lambda s, sec: EV(s, 'zap') > 0 and _nondyadic(s))
  add('territory/respawn_1', 'territory__rooms', 9, None, [kw('Zapper', framesTillRespawn=1)], 'refused', 'engine')
  # ---- clean_up
  river = map_replace('F', 'H')
  add('clean_up/clean_cooldown_0', 'clean_up', 7, None, [kw('Cleaner', cooldownTime=0)], 'parity',
      reach=lambda s, sec: EV(s, 'player_cleaned') > 0)
  add('clean_up/clean_cooldown_negative', 'clean_up', 7, None, [kw('Cleaner', cooldownTime=-1)], 'refused', 'engine')
  add('clean_up/clean_line_32', 'clean_up', 7, None, [kw('Cleaner', beamLength=32, beamRadius=0)], 'parity',
      reach=lambda s, sec: EV(s, 'player_cleaned') > 0)
  add('clean_up/dirt_fills_river', 'clean_up', 7, None, [kw('DirtSpawner', dirtSpawnProbability=1.0, delayStartOfDirtSpawning=0)],
      'parity', reach=lambda s, sec: s['sprite_max'][int(sec['cu_ip'][6])] == int(sec['cu_ip'][1]))
  add('clean_up/apple_growth_rate_1', 'clean_up', 7, None, [river, kw('AppleGrow', maxAppleGrowthRate=1.0)], 'parity',
      reach=lambda s, sec: EV(s, 'edible_consumed') > 0 and _grew('cu_ip', 4)(s, sec))
  add('clean_up/apple_thresholds_equal', 'clean_up', 7, None,
      [river, kw('AppleGrow', thresholdDepletion=0.0, thresholdRestoration=0.0, maxAppleGrowthRate=1.0),
       kw('DirtSpawner', dirtSpawnProbability=0.0)], 'parity',
      # the river stays clean, so the dirt fraction equals both thresholds on every frame: 0/0, and no apple ever grows
      reach=lambda s, sec: s['sprite_max'][int(sec['cu_ip'][6])] == 0 and s['sprite_max'][int(sec['cu_ip'][4])] == 0)
  for rnd in (True, False):
    add(f'clean_up/animation_every_frame_random_start_{rnd}', 'clean_up', 7, None,
        [kw('Animation', gameFramesPerAnimationFrame=1, randomStartFrame=rnd)], 'parity', steps=60,
        probe=lambda sec: [int(x) for x in sec['cu_water_sprites'][:int(sec['cu_ip'][9])]],
        reach=(lambda s, sec: len(s['sprites_seen']) > 2 and all(a != b for a, b in zip(s['sprites_seen'], s['sprites_seen'][1:]))
               and sum(1 for n in s['sprites_seen'][0] if n) > 1) if rnd else
              (lambda s, sec: len(s['sprites_seen']) > 2 and all(sum(1 for n in c if n) == 1 for c in s['sprites_seen'])
               and all(a != b for a, b in zip(s['sprites_seen'], s['sprites_seen'][1:]))))
  # ---- commons_harvest
  ch = 'commons_harvest__open'
  add('commons/regrow_always', ch, 7, None, [kw('DensityRegrow', regrowthProbabilities=[1.0, 1.0, 1.0, 1.0])], 'parity',
      reach=lambda s, sec: EV(s, 'edible_consumed') > 0 and _grew('ch_ip', 2)(s, sec))
  add('commons/regrow_never', ch, 7, None, [kw('DensityRegrow', regrowthProbabilities=[0.0, 0.0, 0.0, 0.0])], 'parity',
      reach=lambda s, sec: EV(s, 'edible_consumed') > 0 and _never_grew('ch_ip', 2)(s, sec))
  grow = kw('DensityRegrow', regrowthProbabilities=[0.0, 0.2, 0.4, 0.8])
  add('commons/radius_1', ch, 7, None, [density_radius(1.0), grow], 'parity',
      reach=lambda s, sec: int(sec['ch_ip'][5]) == 5 and EV(s, 'edible_consumed') > 0 and _grew('ch_ip', 2)(s, sec))
  add('commons/radius_2_98', ch, 7, None, [density_radius(2.98), grow], 'parity',
      reach=lambda s, sec: int(sec['ch_ip'][5]) == 29 and EV(s, 'edible_consumed') > 0 and _grew('ch_ip', 2)(s, sec))
  add('commons/radius_3', ch, 7, None, [density_radius(3.0)], 'refused', 'engine')
  # a 5x5 block of apples: the radius-2.98 disc around its centre holds 24 other apples
  add('commons/dense_disc', ch, 7, None, [density_radius(2.98), map_rows(lambda rows: [
      r[:9] + 'AAAAA' + r[14:] if 10 <= i <= 14 else r for i, r in enumerate(rows)])], 'refused', 'compiler')
  # ---- territory
  tr = 'territory__rooms'
  add('territory/health_1', tr, 9, None, [kw('Resource', initialHealth=1)], 'parity',
      reach=lambda s, sec: EV(s, 'destroyed_resource') > 0)
  add('territory/health_200', tr, 9, None, [kw('Resource', initialHealth=200)], 'parity',
      reach=lambda s, sec: EV(s, 'destroyed_resource') == 0 and s['sprite_max'][int(sec['tr_ip'][7])] > 0)
  add('territory/health_201', tr, 9, None, [kw('Resource', initialHealth=201)], 'refused', 'engine')
  add('territory/fast_rewards', tr, 9, None,
      [kw('Resource', rewardDelay=0, delayTillSelfRepair=0, selfRepairProbability=1.0, rewardRate=1.0, reward=0.3)], 'parity',
      reach=lambda s, sec: EV(s, 'claimed_resource') > 0 and _nondyadic(s))
  add('territory/reward_delay_65535', tr, 9, None, [kw('Resource', rewardDelay=65535)], 'parity',
      reach=lambda s, sec: EV(s, 'claimed_resource') > 0 and s['rewards'] == 0.0)
  add('territory/reward_delay_65536', tr, 9, None, [kw('Resource', rewardDelay=65536)], 'refused', 'engine')
  add('territory/repair_delay_65536', tr, 9, None, [kw('Resource', delayTillSelfRepair=65536)], 'refused', 'engine')
  add('territory/claim_wait_5', tr, 9, None, [kw('ResourceClaimer', beamWait=5)], 'parity',
      reach=lambda s, sec: EV(s, 'claimed_resource') > 0)
  add('territory/open_beams_32', 'territory__open', 9, None,
      [kw('Zapper', beamLength=32, beamRadius=0), kw('ResourceClaimer', beamLength=32, beamRadius=0)], 'parity',
      reach=lambda s, sec: EV(s, 'claimed_resource') > 0)
  add('territory/rooms_zap_20', tr, 9, None, [kw('Zapper', beamLength=20, beamRadius=0)], 'parity',
      reach=lambda s, sec: EV(s, 'sanctioning') > 0)
  add('territory/rooms_zap_radius_10', tr, 9, None, [kw('Zapper', beamLength=1, beamRadius=10)], 'parity',
      reach=lambda s, sec: EV(s, 'sanctioning') > 0)
  add('territory/rooms_zap_21', tr, 9, None, [kw('Zapper', beamLength=21, beamRadius=0)], 'refused', 'engine')
  add('territory/rooms_zap_radius_11', tr, 9, None, [kw('Zapper', beamLength=1, beamRadius=11)], 'refused', 'engine')
  add('territory/rooms_claim_21', tr, 9, None, [kw('ResourceClaimer', beamLength=21, beamRadius=0)], 'refused', 'engine')
  add('territory/rooms_zap_25', tr, 9, None, [kw('Zapper', beamLength=25, beamRadius=0)], 'refused', 'engine')
  add('territory/sanctions_1_level', tr, 9, None,
      [marking_levels([dict(levelIncrement=0, sourceReward=0.25, targetReward=-0.5, freeze=2)], 1), kw('Zapper', cooldownTime=1)],
      'parity', reach=lambda s, sec: int(sec['tr_ip'][11]) == 1 and EV(s, 'sanctioning') > 0 and _nondyadic(s))
  add('territory/sanctions_3_levels', tr, 9, None,
      [marking_levels([dict(levelIncrement=1, freeze=2), dict(levelIncrement=1, freeze=3, sourceReward=0.7),
                       dict(levelIncrement=-2, remove=True, targetReward=-0.3)], 50), kw('Zapper', cooldownTime=1)],
      'parity', reach=lambda s, sec: int(sec['tr_ip'][11]) == 3 and EV(s, 'removal_due_to_sanctioning') > 0 and _nondyadic(s))
  # the shipped two levels, back to level 1 one frame after a hit: a removal needs two hits on consecutive frames
  add('territory/sanctions_recovery_1', tr, 9, None, [kw('GraduatedSanctionsMarking', recoveryTime=1), kw('Zapper', cooldownTime=1)],
      'parity', reach=lambda s, sec: EV(s, 'sanctioning') > 0 and 20 * EV(s, 'removal_due_to_sanctioning') <= EV(s, 'sanctioning'))
  # ---- coins
  add('coins/regrow_rate_1', 'coins', 2, 0, [kw('ChoiceCoinRegrow', regrowRate=1.0)], 'parity',
      reach=lambda s, sec: EV(s, 'coin_consumed') > 0)
  add('coins/terminate_at_3', 'coins', 2, 0,
      [kw('ChoiceCoinRegrow', regrowRate=1.0), kw('Coin', terminateEpisode=True, coinsToTerminateEpisode=3)], 'parity',
      reach=lambda s, sec: s['lasts'] > 0 and EV(s, 'coin_consumed') >= 3)
  add('coins/non_dyadic_rewards', 'coins', 2, 0,
      [kw('ChoiceCoinRegrow', regrowRate=1.0),
       kw('Coin', rewardSelfForMatch=0.3, rewardSelfForMismatch=0.7, rewardOtherForMatch=-0.1, rewardOtherForMismatch=0.2),
       kw('Role', multiplyRewardSelfForMatch=1.1, multiplyRewardSelfForMismatch=0.9, multiplyRewardOtherForMatch=3.0,
          multiplyRewardOtherForMismatch=0.6)], 'parity',
      reach=lambda s, sec: EV(s, 'coin_consumed') > 0 and _nondyadic(s))
  # ---- coop_mining
  cm = 'coop_mining'
  ores = kw('FixedRateRegrow', liveRates=[1.0, 1.0])
  add('coop_mining/live_rates_1', cm, 6, None, [ores], 'parity', reach=lambda s, sec: EV(s, 'mining') > 0 and EV(s, 'extraction') > 0)
  for w in (1, 255):
    add(f'coop_mining/mining_window_{w}', cm, 6, None, [ores, kw('Ore', miningWindow=w)], 'parity',
        reach=lambda s, sec, w=w: int(sec['cm_ip'][6]) == w and EV(s, 'mining') > 0)
  add('coop_mining/mining_window_256', cm, 6, None, [ores, kw('Ore', miningWindow=256)], 'refused', 'engine')
  add('coop_mining/mine_cooldown_1', cm, 6, None, [ores, kw('MineBeam', cooldownTime=1)], 'parity',
      reach=lambda s, sec: EV(s, 'mining') > 0)
  add('coop_mining/mine_cooldown_0', cm, 6, None, [ores, kw('MineBeam', cooldownTime=0)], 'refused', 'engine')
  add('coop_mining/mine_line_32', cm, 6, None, [ores, kw('MineBeam', beamLength=32)], 'parity',
      reach=lambda s, sec: EV(s, 'mining') > 0)
  # ---- view geometry (every avatar gets the same view)
  for sub, p in (('clean_up', 7), ('territory__rooms', 9)):
    fam = sub.split('__')[0]
    for name, geom in (('1x1', (0, 0, 0, 0)), ('5', (2, 2, 2, 2)), ('asymmetric', (0, 7, 2, 6)), ('12', (5, 6, 9, 1)),
                       ('13', (6, 6, 9, 1)), ('16', (7, 8, 9, 1)), ('tall', (5, 5, 14, 1))):
      add(f'{fam}/view_{name}', sub, p, None, [view(*geom)], 'parity', steps=40,
          reach=lambda s, sec, geom=geom: tuple(int(x) for x in sec['meta'][15:19]) == geom)
    add(f'{fam}/view_17', sub, p, None, [view(8, 8, 9, 1)], 'refused', 'engine')
  return v


VARIANTS = _variants()

# One territory__rooms episode of 70,000 frames (tests/test_gpu_param_envelope.py steps it past frame 65,535).
LONG_EPISODE = Variant('territory/long_episode', 'territory__rooms', 9, None,
                       [kw(_ENDING, probabilityTerminationPerInterval=0.0), top(maxEpisodeLengthFrames=70000)], 'parity')
PARITY = [x for x in VARIANTS if x.expect == 'parity']
REFUSED = [x for x in VARIANTS if x.expect == 'refused']
BY_NAME = {x.name: x for x in VARIANTS}
assert len(BY_NAME) == len(VARIANTS)


def settings(variant):
  s = settings_golden.settings(variant.substrate, variant.players, variant.seed)
  for edit in variant.edits:
    edit(s)
  return s


def compile_variant(x):
  from meltingpot_b200 import compiler
  return compiler.compile_settings(settings(x), settings_golden.config(x.substrate, x.players), x.seed)


@functools.lru_cache(maxsize=None)
def compile(name):  # pylint: disable=redefined-builtin
  """The blob of a table variant (cached per test session)."""
  return compile_variant(BY_NAME[name])


@functools.lru_cache(maxsize=None)
def stock(substrate, players, seed):
  return settings_golden.compile(substrate, players, seed)


def sections(blob):
  return _sec(blob)


def view_geometry(blob):
  m = _sec(blob)['meta']
  return types.SimpleNamespace(left=int(m[15]), right=int(m[16]), forward=int(m[17]), backward=int(m[18]),
                               width=int(m[15]) + int(m[16]) + 1, height=int(m[17]) + int(m[18]) + 1)


def probe_sprites(variant, blob):
  return tuple(variant.probe(_sec(blob))) if variant.probe else ()
