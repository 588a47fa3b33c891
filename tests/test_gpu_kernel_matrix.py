"""Every k_step table cell and every routed and gathered k_render, each against the oracle.

The engine picks its state-transition kernel from a table, k_step<Family, Source, kRestore, Actions> (one blob or
ParamVariants; advance or fused restore; dense actions, action rows or drawn routes), and its renderer from three modes
of one k_render<NCP, NCW> instantiation (plain, observation gather, player / WORLD.RGB rows) at a layout chosen per
engine. After every call, Engine.last_launch() (mp_debug_last_launch) names the cell and mode that ran, and each test
asserts it is the one the call meant to reach.

1. One test per family row runs all 12 k_step cells of the row (one-blob and variant engines) against per-env oracle
   envs on every step: rewards bit for bit, discount, step type, scalar observations, avatar state, grid and events,
   and every image byte at the first and middle steps and around every auto-reset. Variant engines interleave map
   variants so that every 4-env k_step CTA holds envs on different maps, at B = 4k + 3 >= 2 * SMs + 5. Records stored
   at MID and LAST steps restore, as clones and rekeyed, into envs on other maps, beside envs that advance in the same
   CTA, while a reassignment is still pending. A restored env's oracle env is its source's, replayed to the store point.
2. RENDER_ROUTED at every feasible layout of the nine substrates, with the debug lane maps and without pre-merged
   sprites, in lockstep with a default-layout plain engine that is checked against the oracle in the same loop; at
   the view geometries of tests/variants.py (k_render<4, 5> among them) against per-env oracle envs; RENDER_GATHER at
   each of the four instantiations against the oracle.
"""

import functools
import os
import types

import numpy as np
import pytest

from tests import coins_draws as CD
from tests import commons_maps as CM
from tests import env_variants as EV
from tests import parity
from tests import territory_maps as TM
from tests import variants as V
from tests.test_gpu_drawn_routes import _Model, _choices, _routes
from tests.test_gpu_player_actions import _action_rows, _dense
from tests.test_gpu_player_routes import _Rows, _row_map
from tests.test_gpu_state_bank import _index as _idx, _keyed
from tests.test_gpu_render_variants import SUBSTRATES, _IDS, _blob as _stock_blob, _feasible_layouts, _layout, _plan
from tests.test_gpu_step_into import _blob as _cap40_blob, _sms
from tests.test_gpu_world_routes import _World

pytestmark = pytest.mark.gpu

THREADS = os.cpu_count() or 1
SEED = 53
FAMILY_IDS = {'clean_up': 1, 'commons_harvest': 2, 'territory': 3, 'coins': 4, 'coop_mining': 5}
# Each row: (family, the variant set of its ParamVariants cells). territory__inside_out, whose 'choice' resources are
# drawn per episode, runs as an extra row: a one-blob engine and an engine of two identical variants.
ROWS = {
    'clean_up': 'clean_up',
    'commons_harvest': 'commons_harvest',
    'coins': 'coins',
    'territory__rooms': 'territory',
    'coop_mining': 'coop_mining',
    'territory__inside_out': 'territory',
}
RESTORE_CELLS = [(r, a) for r in (0, 1) for a in (0, 1, 2)]  # (restore, actions: 0 dense, 1 rows, 2 drawn)
RENDER_INSTS = ((3, 3), (3, 4), (3, 5), (4, 5))
RENDER_MODES = (0, 1, 2)  # plain, gather, routed
VIEWS = ('1x1', '5', 'asymmetric', '12', '13', '16', 'tall')

_RENDER_REACHED = set()   # (ncp, ncw, mode) of oracle-anchored runs in this module
_RENDER_TESTS_RUN = set()


def variant_set(row):
  """The blobs of a row's variant engine: the map or parameter variants it runs side by side."""
  if row == 'clean_up':
    return tuple(EV.blobs('clean_up'))
  if row == 'commons_harvest':
    return tuple(CM.map_set())
  if row == 'coins':
    return tuple(CD.draw_set())
  if row in ('territory__rooms', 'coop_mining'):
    return tuple(TM.map_set(row))
  from tests.test_gpu_entry_points import _inside_out_cap40
  return (_inside_out_cap40(),) * 2


def single_blob(row):
  return _cap40_blob({'territory__rooms': 'territory'}.get(row, row))


# each map set's own entity table: a cross-map restore moves an env to a map with more or fewer of these entities
ENTITY_SECTIONS = {'commons_harvest': 'ch_apple', 'coins': 'co_coin', 'territory__rooms': 'tr_res', 'coop_mining': 'cm_ore'}


def family_of(substrate):
  return FAMILY_IDS[substrate.split('__')[0]]


def step_cells():
  """Every (family id, variants, restore, actions) cell the rows reach."""
  return {(FAMILY_IDS[ROWS[row]], v, r, a) for row in ROWS for v in (0, 1) for r, a in RESTORE_CELLS}


# ---- per-env oracle model ---------------------------------------------------------------------------------------------
class _Env:
  """One env's oracle env, with the recipe that rebuilds it (so a record restores as a replay of its source)."""

  def __init__(self, keyed, blobs, ops, pending):
    self.keyed, self.blobs, self.ops, self.pending = keyed, blobs, [], pending
    self.e = None
    for op in ops:
      self._apply(op)

  def _apply(self, op):
    kind, x = op
    if kind == 'new':        # (variant, key): the env's first episode
      self.v, self.key = x
      self.e = self.keyed.KeyedOracleEnv(self.blobs[self.v], self.key)
      self.e.reset()
    elif kind == 'next':     # the next episode, under variant x (an auto-reset after LAST or a masked reset)
      ep = self.e.counters()['episode']
      self.v = x
      self.e = self.keyed.KeyedOracleEnv(self.blobs[x], self.key)
      self.e.set_episode(ep + 1)
      self.e.reset()
    elif kind == 'step':
      self.e.step(x)
    elif kind == 'key':
      self.key = x
      self.e.set_key(x)
    self.ops.append(op)

  def step(self, acts):
    self._apply(('next', self.pending) if self.e.step_type() == 2 else ('step', np.array(acts, np.int32)))

  def reset(self):
    self._apply(('next', self.pending))

  def record(self):
    return list(self.ops), self.pending

  @classmethod
  def restored(cls, keyed, blobs, rec, rekey_to=None):
    ops, pending = rec
    env = cls(keyed, blobs, ops, pending)
    if rekey_to is not None:
      env._apply(('key', rekey_to))
    return env


def _rows_with_edges(rng, B, P, n_rows, kind):
  """A row map (permuted or partial) that uses row 0 and row n_rows - 1 and holds out-of-range ids and rows."""
  import torch
  m = _row_map(kind, B, P, n_rows, rng).cpu().numpy().reshape(-1)
  first, last = rng.choice(B * P, 2, replace=False)
  m[m == 0] = -1; m[m == n_rows - 1] = -1
  m[first], m[last] = 0, n_rows - 1
  others = [i for i in range(B * P) if i not in (first, last)]
  bad = rng.choice(others, min(len(others), 3), replace=False)
  m[bad] = rng.choice([n_rows, n_rows + 7, -5], len(bad))
  return torch.from_numpy(m.reshape(B, P).astype(np.int32)).cuda()


def _check_launch(eng, family, variants, restore, actions, mode):
  got = eng.last_launch()
  want = dict(family=family, variants=variants, restore=restore, actions=actions, render_mode=mode)
  assert {k: got[k] for k in want} == want, f'launched {got}, meant {want}'
  return got


def _run_step_cells(row, blobs, assign, B, steps=56):
  """Every (restore, actions) cell of one engine (one blob or a variant set) against per-env oracle envs."""
  import torch
  from meltingpot_b200 import engine
  keyed = _keyed()
  fam = FAMILY_IDS[ROWS[row]]
  n_var = len(blobs)
  variants = int(n_var > 1)
  eng = engine.Engine(list(blobs) if variants else blobs[0], B, seed=SEED, env_variant=assign)
  P, A = eng.num_players, eng.num_actions
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  assign = np.zeros(B, np.int64) if assign is None else np.asarray(assign)
  envs = [_Env(keyed, blobs, [('new', (int(assign[b]), SEED + b))], int(assign[b])) for b in range(B)]
  rng = np.random.default_rng(B + 7 * fam)
  r = _routes(eng, _choices(P, rng))
  draws = _Model(B, SEED, r)
  tg = _Rows(eng, r.n_rows)
  n_slots = 2 * n_var + 1  # MID records of every map, LAST records of every map, one slot never written
  bank = torch.zeros((n_slots, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  records, slot_var = {}, {}
  reached = set()
  restored_ever = np.zeros(B, bool)
  if row in ENTITY_SECTIONS and n_var > 1:
    from meltingpot_b200 import blob as blob_lib
    entities = [len(blob_lib.unpack(x)[ENTITY_SECTIONS[row]]) for x in blobs]
    if len(set(entities)) == 1:  # (commons_harvest's three maps hold 64 apples each)
      entities = None
  else:
    entities = None
  directions = set()  # signs of (record's entity count - target's) over the cross-map restores

  def store(t, slot_env):
    eng.store_states(bank, _idx(n_slots, slot_env))
    draws.store(_idx(n_slots, slot_env).cpu().numpy())
    for s, b in slot_env.items():
      records[s] = envs[b].record()
      slot_var[s] = envs[b].v

  def restore_map(t):
    """About a third of the envs, each from a record of a map other than its own, beside envs that advance in its
    CTA; larger entity counts into smaller ones and the reverse, as clones of MID and LAST records."""
    mapping = {}
    for b in range(B):
      if reserved[b]:
        continue
      if b % 4 == (t // 6) % 4 or rng.random() < 0.15:
        cands = [s for s in records if n_var == 1 or slot_var[s] != envs[b].v]
        if cands:
          mapping[b] = int(rng.choice(cands))
    mapping[B - 1] = n_slots - 1  # the row never written: env B - 1 advances
    return mapping

  def check(t, where, restored, routed_map=None):
    """Every output of every env; the images of every env at the first and middle steps, else of the envs whose step
    is FIRST or LAST or that were restored. routed_map: player images went to tg's rows by this map."""
    parity.check_outputs(parity.device_outputs(eng, ()), parity.env_dump([e.e for e in envs], shapes, max_events=max_ev), where)
    if variants:
      assert np.array_equal(eng.active_variant.cpu().numpy(), [e.v for e in envs]), f'active variants {where}'
    px = list(range(B)) if t in (0, steps // 2) else sorted(
        {b for b in range(B) if envs[b].e.step_type() in (0, 2)} | set(restored))
    if not px:
      return
    idx = torch.tensor(px, device='cuda')
    want = parity.env_dump([envs[b].e for b in px], shapes, pixels=True, max_events=max_ev)
    got = {'world': eng.world_rgb[idx].cpu().numpy()}
    if routed_map is None:
      got['rgb'] = eng.rgb[idx].cpu().numpy()
    else:
      m = routed_map[px]
      k, p = np.nonzero(m >= 0)
      got['rgb'] = tg.rgb[torch.from_numpy(m[k, p]).long().cuda()].cpu().numpy()
      want['rgb'] = want['rgb'][k, p]
    parity.check_outputs(got, {'world': want['world'], 'rgb': want['rgb']}, f'{where} images of envs {px[:8]}...')

  reserved = (np.arange(B) // n_var) % 4 == 3  # whole blocks of every map that no restore touches: LAST at step 40
  eng.reset()
  draws.after(eng.step_type, mask=np.ones(B, np.uint8))
  _check_launch(eng, fam, variants, 0, 0, 0)
  reached.add((0, 0))
  check(0, f'{row} reset', [])
  for t in range(1, steps + 1):
    if variants and t == 30:  # pending until each env's next episode start; restores arrive meanwhile
      ids = (assign + 1 + (np.arange(B) % 2)) % n_var
      eng.set_env_variant(ids)
      for b in range(B):
        envs[b].pending = int(ids[b])
    if t in (11, 41):  # records of every map: MID ones after step 10, LAST ones after step 40
      st = eng.step_type.cpu().numpy()
      base = 0 if t == 11 else n_var
      slot_env = {}
      for v in range(n_var):
        pool = [b for b in range(B) if envs[b].v == v and (t == 11 or st[b] == 2)]
        if pool:
          slot_env[base + v] = pool[len(pool) // 2]
      store(t, slot_env)
      want_st = 1 if t == 11 else 2
      assert len(slot_env) == n_var and all(envs[b].e.step_type() == want_st for b in slot_env.values()), slot_env
    restore, act_kind = RESTORE_CELLS[t % 6]
    if restore and not records:
      restore = 0
    if t == steps - 8:
      act_kind, restore = 2, 0   # a masked reset on drawn routes
    mapping = restore_map(t) if restore else {}
    rekey = restore and (t // 6) % 2 == 1
    kw = dict(restore=_idx(B, mapping), bank=bank, rekey=rekey) if restore else {}
    where = f'{row} B={B} variants={variants} t={t} cell=({restore},{act_kind})'
    pre_map = draws.map()
    mode = 0
    if t == steps - 8:
      mask_h = (np.arange(B) % 3 == 1).astype(np.uint8)
      tg.refill()
      eng.reset(torch.from_numpy(mask_h).cuda(), players=tg.players(r.row_of_player), draw=r.draw)
      for b in np.flatnonzero(mask_h):
        envs[b].reset()
      draws.after(eng.step_type, mask=mask_h)
      mode = 2
    elif act_kind == 0:
      acts = np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)
      eng.step(torch.from_numpy(acts).cuda(), **kw)
      dense = acts
    elif act_kind == 1:
      n_rows = B * P + 2
      rmap = _rows_with_edges(rng, B, P, n_rows, 'partial' if t % 2 else 'permuted')
      action = torch.from_numpy(_action_rows(rng, eng, n_rows)).cuda()
      eng.step(None, player_actions={'row_of_player': rmap, 'action': action}, **kw)
      dense = _dense(rmap, action).cpu().numpy()
    else:
      action = torch.from_numpy(_action_rows(rng, eng, r.n_rows)).cuda()
      tg.refill()
      eng.step(None, player_actions={'row_of_player': r.row_of_player, 'action': action},
               players=tg.players(r.row_of_player), draw=r.draw, **kw)
      dense = _dense(torch.from_numpy(pre_map).cuda(), action).cpu().numpy()
      mode = 2
    _check_launch(eng, fam, variants, restore, act_kind, mode)
    reached.add((restore, act_kind))
    if t != steps - 8:
      for b in range(B):
        envs[b].step(dense[b])
      for b, s in mapping.items():
        if s in records:
          if entities is not None:
            directions.add(int(np.sign(entities[slot_var[s]] - entities[envs[b].v])))
          envs[b] = _Env.restored(keyed, blobs, records[s], SEED + b if rekey else None)
          restored_ever[b] = True
      draws.after(eng.step_type, restored=np.array([mapping.get(b, -1) if mapping.get(b, -1) in records else -1
                                                    for b in range(B)], np.int32), rekey=rekey)
    routed_map = None
    if mode == 2:
      routed_map = r.row_of_player.cpu().numpy()
      assert np.array_equal(routed_map, draws.map()), f'row map {where}'
    check(t, where, [b for b, s in mapping.items() if s in records], routed_map)
  assert restored_ever.any()
  if entities is not None:  # larger entity counts restored into smaller ones, and the reverse
    assert {1, -1} <= directions, (entities, directions)
  assert reached == set(RESTORE_CELLS), reached
  eng.close()
  return {(fam, variants, r_, a_) for r_, a_ in reached}


def _step_row_sizes():
  sms = _sms()
  big = 2 * sms + 5
  big += (3 - big % 4) % 4  # 4k + 3: the last k_step CTA holds three envs
  return big, 23


@pytest.mark.parametrize('row', list(ROWS))
def test_every_k_step_cell_of_the_row_matches_the_oracle(row):
  big, small = _step_row_sizes()
  blobs = variant_set(row)
  if row != 'territory__inside_out':
    pairs = [(a, b) for i, a in enumerate(blobs) for b in blobs[i + 1:]]
    assert all(EV.differing_sections(a, b) for a, b in pairs), 'two variants of the set are one blob'
  reached = _run_step_cells(row, blobs, EV.interleaved(big, len(blobs)), big)
  reached |= _run_step_cells(row, (single_blob(row) if row != 'territory__inside_out' else blobs[0],), None, small)
  fam = FAMILY_IDS[ROWS[row]]
  want = {c for c in step_cells() if c[0] == fam}
  print(f'{row}: k_step cells reached {sorted(reached)}')
  assert reached == want, want ^ reached


# ---- 2. k_render: routed at every layout, routed on other views, gathered at every instantiation ----------------------
@functools.lru_cache(maxsize=None)
def _layouts(name, players):
  ok, _ = _feasible_layouts(_stock_blob(name, players))
  return ok


def _routed_targets(eng, rng):
  """Partial player rows and scattered WORLD.RGB rows, each target exactly as large as what is routed to it (no spare
  row, the last row used), for `eng`."""
  import torch
  B, P = eng.num_envs, eng.num_players
  pick = rng.random(B * P) < 0.5
  pick[rng.integers(0, B * P)] = True
  n_rows = int(pick.sum())
  m = np.full(B * P, -1, np.int32)
  m[pick] = rng.permutation(n_rows)
  rmap = torch.from_numpy(m.reshape(B, P)).cuda()
  n_world = max(1, B // 3)
  envs = rng.choice(B, n_world, replace=False)
  wmap = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  wmap[torch.from_numpy(envs).cuda()] = torch.arange(n_world, dtype=torch.int32, device='cuda')
  return rmap, _Rows(eng, n_rows), torch.from_numpy(envs).cuda(), wmap, _World(eng, n_world)


def _routed_lockstep(oracle, blob, family, B, seed, twins_kw, steps=4):
  """A default-layout plain engine checked against the oracle at every step, and routed engines (Engine keyword
  arguments `twins_kw`) in lockstep with it: every routed player and WORLD.RGB row must equal the plain engine's."""
  import torch
  from meltingpot_b200 import engine
  ref = engine.Engine(blob, B, seed=seed)
  batch = oracle.OracleBatch(blob, B, seed=seed)
  shapes, max_ev = parity.shapes_of(ref), int(ref.buffers.max_events)
  rng = np.random.default_rng(B + seed)
  twins = [engine.Engine(blob, B, seed=seed, **kw) for kw in twins_kw]
  targets = [_routed_targets(tw, rng) for tw in twins]
  P, A = ref.num_players, ref.num_actions
  for t in range(steps + 1):
    if t == 0:
      ref.reset()
    else:
      acts = np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)
      ref.step(torch.from_numpy(acts).cuda())
      batch.step_actions(acts, THREADS)
    ll = _check_launch(ref, family, 0, 0, 0, 0)
    px = t in (0, steps // 2, steps)
    parity.check_outputs(parity.device_outputs(ref, ('rgb', 'world') if px else ()),
                         batch.dump(THREADS, shapes, pixels=px, max_events=max_ev), f'plain B={B} t={t}')
    _RENDER_REACHED.add((ll['ncp'], ll['ncw'], 0))
    for kw, tw, (rmap, tg, envs, wmap, world) in zip(twins_kw, twins, targets):
      tg.refill(); world.refill()
      players = dict(tg.players(rmap), world_row_of_env=wmap, world_rgb=world.rows)
      if t == 0:
        tw.reset(players=players)
      else:
        tw.step(torch.from_numpy(acts).cuda(), players=players)
      ll = _check_launch(tw, family, 0, 0, 0, 2)
      plan = tw.render_plan()
      assert (ll['teams'], ll['warps'], ll['wstrip_log2']) == _layout(plan), (kw, ll)
      assert 'render_layout' not in kw or _layout(plan) == kw['render_layout'], (kw, plan)
      where = f'routed {kw} B={B} t={t}'
      world.check(ref.world_rgb, envs, where)
      tg.check(ref, rmap, where)
      assert torch.equal(tw.step_type, ref.step_type), where
      _RENDER_REACHED.add((ll['ncp'], ll['ncw'], 2))
  for e in [ref] + twins:
    e.close()
  batch.close()


@pytest.mark.parametrize('name,players', SUBSTRATES, ids=_IDS)
def test_routed_render_at_every_feasible_layout(name, players, oracle):
  from meltingpot_b200 import engine
  blob = _stock_blob(name, players)
  sm = _sms()
  ok = _layouts(name, players)
  default = _layout(_plan(blob))
  by_size = {}
  for lay in ok:
    ns = sm * lay[0]
    for B in (7, ns + sm + 7, 2 * ns):
      by_size.setdefault(B, []).append(dict(render_layout=lay))
  # the debug levers, at the default layout: plain and scattered lane maps, no pre-merged sprites
  levers = (engine.MP_FLAG_DEBUG_PLAIN_LANE_MAP, engine.MP_FLAG_DEBUG_SCATTER_LANE_MAP, engine.MP_FLAG_DEBUG_NO_PREMERGE)
  by_size.setdefault(sm * default[0] + sm + 7, []).extend(dict(flags=engine.MP_FLAG_DEFAULT | f) for f in levers)
  for B, kws in sorted(by_size.items()):
    _routed_lockstep(oracle, blob, family_of(name), B, 300 + B, kws)
  _RENDER_TESTS_RUN.add(('layouts', name))
  print(f'{name}: routed at {len(ok)} layouts, instantiations reached so far {sorted(_RENDER_REACHED)}')


@pytest.mark.parametrize('view', VIEWS)
@pytest.mark.parametrize('fam', ['clean_up', 'territory'])
def test_routed_render_on_other_views_matches_the_oracle(fam, view, oracle):
  import torch
  from meltingpot_b200 import engine
  blob = V.compile(f'{fam}/view_{view}')
  geom = V.view_geometry(blob)
  ok, _ = _feasible_layouts(blob)
  default = _layout(_plan(blob))
  forced = sorted(l for l in ok if l != default)
  B, seed, steps = 9, 61, 12
  for lay in [None] + forced[len(forced) // 2:][:1]:
    eng = engine.Engine(blob, B, seed=seed, render_layout=lay)
    assert (eng.rgb.shape[2], eng.rgb.shape[3]) == (geom.height * 8, geom.width * 8)
    envs = [oracle.OracleEnv(blob, seed + b) for b in range(B)]
    rng = np.random.default_rng(len(view) + (lay is None))
    rmap, tg, wenvs, wmap, world = _routed_targets(eng, rng)
    if lay is not None:
      assert _layout(eng.render_plan()) == lay
    for t in range(steps + 1):
      tg.refill(); world.refill()
      players = dict(tg.players(rmap), world_row_of_env=wmap, world_rgb=world.rows)
      if t == 0:
        eng.reset(players=players)
        for e in envs:
          e.reset()
      else:
        acts = np.ascontiguousarray(rng.integers(0, eng.num_actions, size=(B, eng.num_players)), np.int32)
        eng.step(torch.from_numpy(acts).cuda(), players=players)
        for b, e in enumerate(envs):
          e.step(acts[b])
      ll = _check_launch(eng, FAMILY_IDS[fam], 0, 0, 0, 2)
      where = f'{fam}/view_{view} layout {lay} t={t}'
      torch.cuda.synchronize()
      n_sc = eng.num_scalar_obs
      want = types.SimpleNamespace(  # the oracle's outputs in the engine's layout, for _Rows.check
          rgb=torch.from_numpy(np.stack([e.rgb() for e in envs])).cuda(),
          reward=torch.from_numpy(np.stack([e.rewards() for e in envs])).cuda(), num_scalar_obs=n_sc,
          scalar_obs=torch.from_numpy(np.stack([e.scalar_obs().T for e in envs], 1) if n_sc else np.zeros((1, B, 1))).cuda())
      tg.check(want, rmap, where)
      world.check(torch.from_numpy(np.stack([e.world_rgb() for e in envs])).cuda(), wenvs, where)
      _RENDER_REACHED.add((ll['ncp'], ll['ncw'], 2))
    eng.close()
  _RENDER_TESTS_RUN.add(('views', fam, view))


def _instantiation_layouts():
  """(substrate blob, layout) that reaches each k_render instantiation, from the nine substrates and a 13-cell view."""
  found = {}
  for name, players in SUBSTRATES:
    for lay, plan in _layouts(name, players).items():
      found.setdefault((plan['ncp'], plan['ncw']), (_stock_blob(name, players), family_of(name), lay))
  wide = V.compile('clean_up/view_13')
  for lay, plan in _feasible_layouts(wide)[0].items():
    found.setdefault((plan['ncp'], plan['ncw']), (wide, FAMILY_IDS['clean_up'], lay))
  return found


def test_gathered_render_at_every_instantiation_matches_the_oracle(oracle):
  import torch
  from meltingpot_b200 import engine
  found = _instantiation_layouts()
  assert set(RENDER_INSTS) <= set(found), sorted(found)
  sm = _sms()
  for inst in RENDER_INSTS:
    blob, family, lay = found[inst]
    B, seed, steps = 2 * sm * lay[0] + sm // 2 + 3, 71, 5  # two balanced rounds and a cooperative tail
    eng = engine.Engine(blob, B, seed=seed, render_layout=lay)
    plain = engine.Engine(blob, B, seed=seed, render_layout=lay)
    ptr, _ = eng.gather_obs_create(0, 1)
    eng.gather_obs_connect([ptr])
    batch = oracle.OracleBatch(blob, B, seed=seed)
    shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
    rng = np.random.default_rng(B)
    for t in range(steps + 1):
      if t == 0:
        eng.reset(); plain.reset()
      else:
        acts = np.ascontiguousarray(rng.integers(0, eng.num_actions, size=(B, eng.num_players)), np.int32)
        eng.step(torch.from_numpy(acts).cuda()); plain.step(torch.from_numpy(acts).cuda())
        batch.step_actions(acts, THREADS)
      lg, lp = _check_launch(eng, family, 0, 0, 0, 1), _check_launch(plain, family, 0, 0, 0, 0)
      assert (lg['ncp'], lg['ncw'], lg['teams'], lg['warps'], lg['wstrip_log2']) == inst + lay, lg
      assert (lp['ncp'], lp['ncw']) == inst, lp
      eng.gather_obs_wait()
      torch.cuda.synchronize()
      where = f'gather <{inst[0]},{inst[1]}> layout {lay} B={B} t={t}'
      rgb, world = eng.gathered_observations()
      assert torch.equal(rgb, eng.rgb) and torch.equal(world, eng.world_rgb), where
      assert torch.equal(plain.rgb, eng.rgb) and torch.equal(plain.world_rgb, eng.world_rgb), where
      px = t in (0, 2, steps)
      parity.check_outputs(parity.device_outputs(eng, ('rgb', 'world') if px else ()),
                           batch.dump(THREADS, shapes, pixels=px, max_events=max_ev), where)
      _RENDER_REACHED.update({inst + (1,), inst + (0,)})
    eng.close(); plain.close(); batch.close()
  _RENDER_TESTS_RUN.add(('gather',))


def test_every_k_render_cell_was_reached_by_an_oracle_anchored_run():
  want_tests = ({('layouts', n) for n in _IDS} | {('views', f, v) for f in ('clean_up', 'territory') for v in VIEWS}
                | {('gather',)})
  if not want_tests <= _RENDER_TESTS_RUN:
    pytest.skip('runs only after every k_render test of this module')
  want = {i + (m,) for i in RENDER_INSTS for m in RENDER_MODES}
  print('k_render cells reached', sorted(_RENDER_REACHED))
  assert want <= _RENDER_REACHED, sorted(want - _RENDER_REACHED)
