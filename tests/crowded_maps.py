"""TEST INFRASTRUCTURE: crowded arenas, where the same-frame interactions of the step kernels are the rule.

On the stock maps avatars are spread out, so the frames in which the kernels do their order-dependent work are rare:
moves into a cell another avatar leaves or wants in the same frame, beams that hit an avatar which also fires, targets
hit by two beams, respawns onto occupied cells, two claims of one resource, several miners on one ore. Each arena below
keeps a stock map's width, height and topology and walls off all but a small block, with exactly as many spawn points as
mp_create needs for its avatars. A "churn" twin fires and respawns faster where the engine accepts it. Every variant has
a hard cap of 100 frames, so rollouts of 250 steps cross auto-resets.

`Reach` counts the interactions from what OracleBatch.dump (or the engine's buffers) hold after each step, plus the
step's actions and the avatar state before it; `FLOORS` says how many a rollout must reach.
"""

import collections
import functools

import numpy as np

from meltingpot_b200 import compiler
from tests import settings_golden
from tests import variants as V

CAP = 100
STEPS = 250

# ---- the arenas -------------------------------------------------------------------------------------------------------


def _arena(fill, block, y0, x0, box=None):
  """A map edit: every cell of `box` (rows y0..y1, columns x0..x1, inclusive; default the whole map) becomes `fill`, then
  `block` (a list of equal-length strings) is pasted with its top-left corner at (y0, x0), wrapping at the map's edges."""
  def edit(s):
    text = s['simulation']['map']
    lead = '\n' if text.startswith('\n') else ''
    rows = [list(r) for r in text[len(lead):].split('\n')]
    if rows and not rows[-1]:
      rows.pop()
      tail = '\n'
    else:
      tail = ''
    by0, bx0, by1, bx1 = box or (0, 0, len(rows) - 1, max(len(r) for r in rows) - 1)
    for y in range(by0, by1 + 1):
      for x in range(bx0, min(bx1 + 1, len(rows[y]))):
        rows[y][x] = fill
    h, w = len(rows), len(rows[0])
    for dy, line in enumerate(block):
      for dx, c in enumerate(line):
        rows[(y0 + dy) % h][(x0 + dx) % w] = c
    s['simulation']['map'] = lead + '\n'.join(''.join(r) for r in rows) + tail
  return edit


# clean_up 7p: one river row (potential and actual dirt, inside the clean beam's reach of every spawn point), 7 spawn
# points on sand, 10 potential apples.
CLEAN_UP = ['WWWWWWWW',
            'WHFHFHFW',
            'WPP PP W',
            'WP P P W',
            'WBBBBBBW',
            'WBBBB  W',
            'WWWWWWWW']
# commons_harvest__open 16p: 8x5 cells, 2 inside spawn points (Q, players 1 and 2) and 14 spawn points (P, every later
# player and every respawn) in two rows, 16 apples; a radius-2 DensityRegrow disc holds at most 12 other apples.
COMMONS_16 = ['WWWWWWWWWW',
              'WAAAAAAAAW',
              'WQPPPPPPQW',
              'WPPPPPPPPW',
              'WAA    AAW',
              'W AAAA   W',
              'WWWWWWWWWW']
# commons_harvest__partnership 7p: 2 inside spawn points, 5 spawn points, 8 apples in 5x4 cells.
PARTNERSHIP = ['WWWWWWW',
               'WAAAAAW',
               'WQP PQW',
               'WP P PW',
               'WA A AW',
               'WWWWWWW']
# territory__rooms 9p: one room of 5x4 cells inside walls of resources, split by a column of resources that avatars on
# both sides can claim in one frame; its top-left corner is at (18, 18), so the TORUS seam runs through it both ways.
ROOMS = ['RRRRRRR',
         'RPPRPPR',
         'RP,R,PR',
         'RPPR,,R',
         'R,,R,PR',
         'RRRRRRR']
# territory__open 9p (BOUNDED): 6x4 floor cells in the map's top-left corner, ringed by resources.
OPEN = ['RRRRRRRR',
        'RP,P,P,R',
        'R,P,,P,R',
        'RP,P,P,R',
        'R,,,P,,R',
        'RRRRRRRR']
# coins 2p: a 4x3 field of 10 coins and 2 spawn points.
COINS = ['WWWWWW',
         'WCCCCW',
         'W_CC_W',
         'WCCCCW',
         'WWWWWW']
# coop_mining 6p: 6 spawn points and ore on every other cell of a 5x4 block; the churn twin also regrows ore at once.
MINING = ['WWWWWWW',
          'WOPOPOW',
          'WOOOOOW',
          'WPOPOPW',
          'WOOPOOW',
          'WWWWWWW']

_CAP_EDITS = (V.top(maxEpisodeLengthFrames=CAP),)
_NO_STOCHASTIC_END = V.kw('StochasticIntervalEpisodeEnding', probabilityTerminationPerInterval=0.0)

Arena = collections.namedtuple('Arena', 'name substrate players seed family map_edit churn spawns free_cells resources')

ARENAS = (
    Arena('clean_up', 'clean_up', 7, None, 'clean_up', _arena('W', CLEAN_UP, 0, 0),
          (V.kw('Zapper', cooldownTime=1, framesTillRespawn=2),), 7, 30, dict(N_DIRT=6, N_APPLES=10)),
    Arena('commons_16p', 'commons_harvest__open', 16, None, 'commons_harvest', _arena('W', COMMONS_16, 0, 0),
          (V.kw('Zapper', cooldownTime=1, framesTillRespawn=2),), 16, 40, dict(N_APPLES=16)),
    Arena('partnership', 'commons_harvest__partnership', 7, None, 'commons_harvest', _arena('W', PARTNERSHIP, 0, 0),
          (V.kw('Zapper', cooldownTime=1, framesTillRespawn=2),), 7, 20, dict(N_APPLES=8)),
    Arena('territory_rooms', 'territory__rooms', 9, None, 'territory', _arena('W', ROOMS, 18, 18),
          (V.kw('Zapper', cooldownTime=1),), 9, 16, dict(N_RES=26)),
    Arena('territory_open', 'territory__open', 9, None, 'territory', _arena('=', OPEN, 0, 0),
          (V.kw('Zapper', cooldownTime=1),), 9, 24, dict(N_RES=24)),
    Arena('coins', 'coins', 2, 0, 'coins', _arena('W', COINS, 0, 0, box=(0, 0, 13, 11)),
          (V.kw('ChoiceCoinRegrow', regrowRate=1.0),), 2, 12, dict(N_COINS=10)),
    Arena('coop_mining', 'coop_mining', 6, None, 'coop_mining', _arena('W', MINING, 0, 0),
          (V.kw('MineBeam', cooldownTime=1), V.kw('FixedRateRegrow', liveRates=[1.0, 1.0])), 6, 20, dict(N_ORES=14)),
)
ARENA_BY_NAME = {a.name: a for a in ARENAS}

Variant = collections.namedtuple('Variant', 'name arena churn')
VARIANTS = tuple(Variant(f'{a.name}/{kind}', a, kind == 'churn') for a in ARENAS for kind in ('arena', 'churn'))
BY_NAME = {v.name: v for v in VARIANTS}
POLICIES = ('uniform', 'beams')
FAMILIES = tuple(dict.fromkeys(a.family for a in ARENAS))


def _ending_edits(s):
  edits = list(_CAP_EDITS)
  if any(c['component'] == 'StochasticIntervalEpisodeEnding' for c in V._components(s)):  # pylint: disable=protected-access
    edits.append(_NO_STOCHASTIC_END)
  return edits


def settings(variant, stock=False):
  """The lab2d settings of a variant: the arena's map and churn edits, or with `stock` the stock settings under the same
  100-frame cap (the baseline of both twins, as the issue's measurements compare them)."""
  a = variant.arena
  s = settings_golden.settings(a.substrate, a.players, a.seed)
  edits = _ending_edits(s) + ([] if stock else [a.map_edit] + (list(a.churn) if variant.churn else []))
  for edit in edits:
    edit(s)
  return s


def config(variant):
  return settings_golden.config(variant.arena.substrate, variant.arena.players)


@functools.lru_cache(maxsize=None)
def compile(name, stock=False):  # pylint: disable=redefined-builtin
  """The blob of a variant (cached per test session); with `stock`, the stock settings under the same cap."""
  v = BY_NAME[name]
  return compiler.compile_settings(settings(v, stock), config(v), v.arena.seed)


# ---- policies ---------------------------------------------------------------------------------------------------------


def beam_actions(sec):
  """Indices of the actions that fire a beam (zap, clean, claim or mine) in a blob's action table."""
  table = sec['action_table']
  fires = (table[:, compiler.ACTION_FIELDS['fireZap']] != 0) | (table[:, compiler.ACTION_FIELDS['fireClean']] != 0)
  return np.nonzero(fires)[0].astype(np.int32)


def policy(name, sec):
  """actions_fn(t, B, P, A, rng) of parity.compare_batch: 'uniform' draws every action alike; 'beams' fires one of the
  family's beams with probability 1/2 and otherwise draws uniformly. Both use only `rng`."""
  beams = beam_actions(sec)
  if name == 'uniform' or not len(beams):  # coins has no beam: both policies are uniform there
    return lambda t, B, P, A, rng: rng.integers(0, A, size=(B, P))

  def act(t, B, P, A, rng):
    uniform = rng.integers(0, A, size=(B, P))
    beam = beams[rng.integers(0, len(beams), size=(B, P))]
    return np.where(rng.random((B, P)) < 0.5, beam, uniform)
  return act


# ---- reach predicates -------------------------------------------------------------------------------------------------

PREDICATES = ('two_zaps', 'double_hit', 'shooter_zapped', 'chain_move', 'blocked_contest', 'delayed_respawn',
              'double_claim', 'double_sanction', 'gold_2_miners', 'gold_3_miners', 'stack_depth', 'max_events')
# The predicates each family can reach (coins and coop_mining have no zapper; territory avatars never respawn).
APPLIES = {
    'clean_up': ('two_zaps', 'double_hit', 'shooter_zapped', 'chain_move', 'blocked_contest', 'delayed_respawn'),
    'commons_harvest': ('two_zaps', 'double_hit', 'shooter_zapped', 'chain_move', 'blocked_contest', 'delayed_respawn'),
    'territory': ('two_zaps', 'double_hit', 'shooter_zapped', 'chain_move', 'blocked_contest', 'double_claim',
                  'double_sanction'),
    'coins': ('chain_move', 'blocked_contest'),
    'coop_mining': ('chain_move', 'blocked_contest', 'gold_2_miners', 'gold_3_miners'),
}
for _f in APPLIES:
  APPLIES[_f] += ('stack_depth', 'max_events')
# Counted per rollout; `stack_depth` and `max_events` are maxima, not counts.
MAXIMA = ('stack_depth', 'max_events')
_DX = np.array([0, 1, 0, -1])
_DY = np.array([-1, 0, 1, 0])
_EV_ZAP, _EV_CLAIM, _EV_SANCTION, _EV_MINING, _EV_EXTRACTION = 1, 4, 6, 9, 10
_GOLD = 2


class Reach:
  """Counts the same-frame interactions of a batch rollout, one step at a time (`observe`).

  two_zaps         env-frames with two or more zap events
  double_hit       (env-frame, avatar) hit by zaps of two or more shooters
  shooter_zapped   (env-frame, avatar) both zapped and the shooter of a zap event
  chain_move       (env-frame, avatar) moving into the cell another avatar left in that frame
  blocked_contest  (env-frame, avatar) that asked to move into a cell free before the frame, stayed, and finds another
                   avatar that moved there
  delayed_respawn  avatars back on the grid after more than framesTillRespawn + 1 frames off it (a respawn that waited for
                   its cell to clear), counted at the frame they return
  double_claim     (env-frame, resource) right ahead of two or more avatars on the grid after the frame: the one-cell
                   directionHit beams every territory avatar fires each frame claim it twice in that frame
  double_sanction  (env-frame, avatar) sanctioned by two or more shooters (with the stock two-level marking every zap of
                   a marked avatar sanctions it, so this equals double_hit there)
  gold_2_miners    gold extractions (two miners each)
  gold_3_miners    env-frames with a gold extraction and three or more gold miners
  stack_depth      the most non-empty layers of one cell
  max_events       the most events of one env-step
  """

  def __init__(self, sec, num_envs):
    p = compiler.family_params(sec)
    m = sec['meta']
    self.W, self.H, self.P = int(m[1]), int(m[2]), int(m[4])
    self.torus = int(m[compiler.META['TOPOLOGY']]) == 1
    self.move = sec['action_table'][:, compiler.ACTION_FIELDS['move']].astype(np.int64)
    self.respawn = int(p['ZAP_RESPAWN']) if 'ZAP_RESPAWN' in p else None
    self.territory = 'tr_res' in sec
    self.resource = np.zeros(self.W * self.H, bool)
    if 'tr_res' in sec:
      self.resource[sec['tr_res'][:, 1]] = True
    self.counts = dict.fromkeys(PREDICATES, 0)
    self.env_steps = 0
    self.off = np.zeros((num_envs, self.P), np.int64)
    self.prev = None

  def observe(self, t, avatars, grid, events, n_events, step_type, actions=None):
    """Step t (0 = the reset): avatars [B, P, 4] (x, y, orientation, on grid), grid [B, L, cells], events [B, M, 3],
    n_events [B], step_type [B], the actions [B, P] that led here (None at t = 0)."""
    c = self.counts
    c['stack_depth'] = max(c['stack_depth'], int((grid != 0).sum(axis=1).max()))
    c['max_events'] = max(c['max_events'], int(n_events.max()))
    if t > 0:
      self.env_steps += len(step_type)
      for b in np.nonzero(step_type == 1)[0]:  # a FIRST step is a reset: nothing moved or fired
        self._frame(self.prev[b], avatars[b], events[b, :int(n_events[b])], actions[b])
      on = avatars[..., 3] != 0
      back = on & (self.off > 0) & (step_type == 1)[:, None]
      if self.respawn is not None:
        c['delayed_respawn'] += int((back & (self.off > self.respawn + 1)).sum())
      self.off = np.where(on | (step_type != 1)[:, None], 0, self.off + 1)
    self.prev = avatars.copy()

  def _cell(self, x, y):
    if self.torus:
      return (y % self.H) * self.W + (x % self.W)
    return np.where((x >= 0) & (x < self.W) & (y >= 0) & (y < self.H), y * self.W + x, -1)

  def _frame(self, before, after, ev, acts):
    c = self.counts
    kind = ev[:, 0]
    zaps = ev[kind == _EV_ZAP]
    if len(zaps) >= 2:
      c['two_zaps'] += 1
    for tgt in np.unique(zaps[:, 2]):
      if len(np.unique(zaps[zaps[:, 2] == tgt, 1])) >= 2:
        c['double_hit'] += 1
    c['shooter_zapped'] += len(np.intersect1d(zaps[:, 1], zaps[:, 2]))
    sanc = ev[kind == _EV_SANCTION]
    for tgt in np.unique(sanc[:, 2]):
      if len(np.unique(sanc[sanc[:, 2] == tgt, 1])) >= 2:
        c['double_sanction'] += 1
    gold_ex = int(((kind == _EV_EXTRACTION) & (ev[:, 2] == _GOLD)).sum())
    c['gold_2_miners'] += gold_ex // 2
    if gold_ex and int(((kind == _EV_MINING) & (ev[:, 2] == _GOLD)).sum()) >= 3:
      c['gold_3_miners'] += 1
    # moves: cells before and after of the avatars on the grid through the whole frame
    stay_on = (before[:, 3] != 0) & (after[:, 3] != 0)
    cb = self._cell(before[:, 0], before[:, 1])
    ca = self._cell(after[:, 0], after[:, 1])
    moved = stay_on & (cb != ca)
    for i in np.nonzero(moved)[0]:
      if np.any(moved & (cb == ca[i]) & (np.arange(self.P) != i)):
        c['chain_move'] += 1
    mv = self.move[acts]
    d = (before[:, 2] + mv - 1) & 3
    tgt = self._cell(before[:, 0] + _DX[d], before[:, 1] + _DY[d])
    occupied_before = set(cb[before[:, 3] != 0].tolist())
    for i in np.nonzero(stay_on & ~moved & (mv != 0))[0]:
      if tgt[i] >= 0 and tgt[i] not in occupied_before and np.any(moved & (ca == tgt[i])):
        c['blocked_contest'] += 1
    if self.territory:
      # every avatar on the grid claims the resource right ahead of it each frame (Paintbrush's directionHit beam,
      # territory/components.lua:362-412); two of them facing one resource claim it in the same frame, and the kernel
      # resolves them in this frame's rank order
      on = np.nonzero(after[:, 3] != 0)[0]
      ahead = self._cell(after[on, 0] + _DX[after[on, 2]], after[on, 1] + _DY[after[on, 2]])
      ahead = ahead[(ahead >= 0)]
      ahead = ahead[self.resource[ahead]]
      c['double_claim'] += int((np.bincount(ahead, minlength=1) >= 2).sum())


# Floors per 1000 env-steps of every (variant, policy) rollout, about half the least the oracle reaches with 16 envs x
# 250 steps; the move floors hold under the uniform policy only (the beam-heavy one moves rarely). delayed_respawn counts
# only where an avatar can come back within an episode (framesTillRespawn + 2 < CAP), gold_3_miners only where ores
# regrow at once (the coop_mining churn twin).
FLOORS = {
    'clean_up': dict(two_zaps=10, double_hit=2, shooter_zapped=4, chain_move=2, blocked_contest=2, delayed_respawn=1),
    'commons_harvest': dict(two_zaps=8, double_hit=1, shooter_zapped=4, chain_move=2, blocked_contest=2,
                            delayed_respawn=50),
    'territory': dict(two_zaps=15, double_hit=0.75, shooter_zapped=3, chain_move=2, blocked_contest=5, double_claim=0.2,
                      double_sanction=0.75),
    'coins': dict(chain_move=4, blocked_contest=4),
    'coop_mining': dict(chain_move=5, blocked_contest=5, gold_2_miners=0.1, gold_3_miners=2),
}
MOVES = ('chain_move', 'blocked_contest')
# Floors of the maxima: the deepest stack of one cell, the most events of one env-step.
MAX_FLOORS = {'clean_up': dict(stack_depth=3, max_events=4), 'commons_harvest': dict(stack_depth=2, max_events=4),
              'territory': dict(stack_depth=4, max_events=8), 'coins': dict(stack_depth=1, max_events=1),
              'coop_mining': dict(stack_depth=2, max_events=3)}
# Every predicate a variant can reach must be reached more often on its arena than on the stock map under the same
# policies and env-steps (rates pooled over both policies): at least 10x where the stock rate is under 1 per 1000
# env-steps, at least 2x otherwise. The moves of the commons_harvest and territory__open arenas and the double zaps of
# the commons_harvest 16p arena fall short of 2x on every layout tried (the stock maps already spawn those avatars side
# by side, and a dense arena zaps its avatars off the grid early in each episode); they are listed here with the 1.4x
# they must keep.
SHORT_OF_2X = {'commons_16p/arena': ('two_zaps', 'blocked_contest'), 'commons_16p/churn': ('blocked_contest',),
               'partnership/arena': ('blocked_contest',), 'territory_open/arena': ('chain_move', 'blocked_contest'),
               'territory_open/churn': ('chain_move', 'blocked_contest')}
SHORT_RATIO = 1.4


def reachable(variant, sec):
  """The counted predicates a variant can reach, by its family and parameters."""
  fam = variant.arena.family
  p = compiler.family_params(sec)
  out = [k for k in APPLIES[fam] if k not in MAXIMA]
  if 'delayed_respawn' in out and not int(p['ZAP_RESPAWN']) + 2 < CAP:
    out.remove('delayed_respawn')
  if 'gold_3_miners' in out and not variant.churn:
    out.remove('gold_3_miners')
  return tuple(out)


def rates(reach):
  """Counts per 1000 env-steps (maxima as they are)."""
  n = max(reach.env_steps, 1)
  return {k: (v if k in MAXIMA else 1000.0 * v / n) for k, v in reach.counts.items()}


def shortfalls(variant, sec, policy_name, r):
  """The predicates a rollout reached less often than its floor (r: rates per 1000 env-steps), as readable strings."""
  floors = FLOORS[variant.arena.family]
  out = [f'{k}: {r[k]:.2f}/1000 < {floors[k]}' for k in reachable(variant, sec)
         if r[k] < floors[k] and (policy_name == 'uniform' or k not in MOVES)]
  out += [f'{k}: {r[k]} < {f}' for k, f in MAX_FLOORS[variant.arena.family].items() if r[k] < f]
  return out


def coverage_failures(variant, sec, arena_rates, stock_rates):
  """The predicates the arena does not reach often enough next to the stock map (rates per 1000 env-steps)."""
  out = []
  for k in reachable(variant, sec):
    a, st = arena_rates[k], stock_rates[k]
    need = 10 * st if st < 1 else (SHORT_RATIO if k in SHORT_OF_2X.get(variant.name, ()) else 2) * st
    if not (a >= need and a > 0):
      out.append(f'{k}: arena {a:.2f} vs stock {st:.2f} per 1000 env-steps')
  return out
