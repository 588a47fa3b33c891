"""The crowded arenas of tests/crowded_maps.py on the CPU: what they compile to, and what the oracle does on them.

Each arena must compile, pass every check mp_create makes before it opens a device, and have the spawn points, free cells
and resources it claims. An OracleBatch rollout of every (variant, policy) must reach every predicate at its floor, and
the arenas must reach the compared predicates far more often than the stock map does under the same policies and the
same number of env-steps; the rates are printed (pytest -s).
"""

import ctypes
import functools

import numpy as np
import pytest

from meltingpot_b200 import blob as mpb
from meltingpot_b200 import compiler
from tests import crowded_maps as C

B = 16
SEED = 7
MP_E_NO_DEVICE = -4


def rollout(blob, policy, num_envs=B, steps=C.STEPS, seed=SEED, oracle=None):
  """An OracleBatch rollout under `policy`, folded into a crowded_maps.Reach."""
  sec = mpb.unpack(blob)
  m = sec['meta']
  P, A = int(m[4]), int(m[19])
  shapes = dict(P=P, L=int(m[3]), cells=int(m[1]) * int(m[2]), n_scalar=int(m[23]), rgb=(1, 1), world=(1, 1))
  batch = oracle.OracleBatch(blob, num_envs, seed=seed)
  reach = C.Reach(sec, num_envs)
  act = C.policy(policy, sec)
  rng = np.random.default_rng(0)
  acts = None
  for t in range(steps + 1):
    if t:
      acts = np.ascontiguousarray(act(t, num_envs, P, A, rng), np.int32)
      batch.step_actions(acts, 4)
    d = batch.dump(4, shapes, pixels=False, max_events=1024, kinds=())
    reach.observe(t, d['avatars'], d['grid'], d['events'], d['n_events'], d['step_type'], acts)
  batch.close()
  return reach


@functools.lru_cache(maxsize=None)
def _rates(name, policy, stock):
  from oracle import binding
  return C.rates(rollout(C.compile(name, stock), policy, oracle=binding))


@pytest.mark.parametrize('name', [v.name for v in C.VARIANTS])
def test_arena_compiles_with_what_it_claims(name):
  from meltingpot_b200 import engine
  v = C.BY_NAME[name]
  a = v.arena
  blob = C.compile(name)
  sec = mpb.unpack(blob)
  stock = mpb.unpack(C.compile(name, stock=True))
  m, ms = sec['meta'], stock['meta']
  for k in ('W', 'H', 'TOPOLOGY', 'P'):
    assert m[compiler.META[k]] == ms[compiler.META[k]], k
  assert int(m[compiler.META['MAX_FRAMES']]) == C.CAP
  assert blob != C.compile(name, stock=True)
  # the arena's text: spawn points and free cells (everything an avatar can stand on)
  text = [r for r in C.settings(v)['simulation']['map'].split('\n') if r]
  spawn_chars = {'P', 'Q', '_'}
  free_chars = spawn_chars | {' ', ',', 'A', 'B', 'C', 'O', 'H', 'F', 'S'}
  wall = {'clean_up': 'W', 'commons_harvest': 'W', 'territory': 'WR=', 'coins': 'W', 'coop_mining': 'W'}[a.family]
  n_spawn = sum(r.count(c) for r in text for c in spawn_chars)
  n_free = sum(1 for r in text for c in r if c in free_chars and c not in wall)
  if a.family == 'coins':  # the stock map's right-hand margin is blank, outside the walled field
    n_free = sum(1 for r in text[:14] for c in r[:12] if c in free_chars)
  assert (n_spawn, n_free) == (a.spawns, a.free_cells), (n_spawn, n_free)
  params = compiler.family_params(sec)
  for k, want in a.resources.items():
    assert params[k] == want, (k, params[k], want)
  spawn_sections = [k for k in sec if k.startswith('spawn_cells_')]
  assert spawn_sections and sum(len(sec[k]) for k in spawn_sections) == a.spawns
  # every check mp_create makes before it opens a device passes
  lib = engine.load_library()
  h = ctypes.c_void_p()
  rc = lib.mp_create(blob, ctypes.c_size_t(len(blob)), 4, 0, ctypes.c_uint64(1), ctypes.c_uint64(0), ctypes.c_uint32(0),
                     ctypes.byref(h))
  if rc == 0:
    lib.mp_destroy(h)
  assert rc in (0, MP_E_NO_DEVICE), lib.mp_last_error().decode()


def test_churn_twins_carry_their_overrides():
  for a in C.ARENAS:
    p = compiler.family_params(mpb.unpack(C.compile(f'{a.name}/churn')))
    if a.family in ('clean_up', 'commons_harvest'):
      assert (p['ZAP_COOLDOWN'], p['ZAP_RESPAWN']) == (1, 2), a.name
    elif a.family == 'territory':
      assert p['ZAP_COOLDOWN'] == 1, a.name
    elif a.family == 'coins':
      assert p['REGROW_RATE'] == 1.0, a.name
    else:
      assert (p['MINE_COOLDOWN'], p['RATE_0'], p['RATE_1']) == (1, 1.0, 1.0), a.name


@pytest.mark.parametrize('policy', C.POLICIES)
@pytest.mark.parametrize('name', [v.name for v in C.VARIANTS])
def test_oracle_reaches_every_predicate(name, policy, oracle):
  v = C.BY_NAME[name]
  sec = mpb.unpack(C.compile(name))
  r = _rates(name, policy, False)
  print(name, policy, {k: round(x, 1) for k, x in r.items()})
  bad = C.shortfalls(v, sec, policy, r)
  assert not bad, bad


@pytest.mark.parametrize('name', [v.name for v in C.VARIANTS])
def test_arena_reaches_more_than_the_stock_map(name, oracle):
  v = C.BY_NAME[name]
  sec = mpb.unpack(C.compile(name))
  pooled = {}
  for stock in (False, True):
    per = [_rates(name, pol, stock) for pol in C.POLICIES]
    pooled[stock] = {k: float(np.mean([p[k] for p in per])) for k in per[0]}
  rows = [f'{k:16s} stock {pooled[True][k]:8.2f}  arena {pooled[False][k]:8.2f}' for k in C.reachable(v, sec)]
  print(f'\n{name} per 1000 env-steps, {B} envs x {C.STEPS} steps per policy\n  ' + '\n  '.join(rows))
  bad = C.coverage_failures(v, sec, pooled[False], pooled[True])
  assert not bad, bad
