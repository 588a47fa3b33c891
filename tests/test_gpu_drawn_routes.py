"""Drawn routes (mp_run's draw, BatchedSubstrate.drawn_routes, BatchedScenario population mode).

A drawn engine steps beside a lockstep twin built with the same seed, which is handed the drawn engine's row maps as
fixed inputs: its actions come from the map the drawn engine held before the call (player_actions) and its outputs go
to the map the drawn engine wrote (players). Both deliver into sentinel-filled targets, which
must then be equal byte for byte, as must every per-env output and, at the end, every env's state record. Each written
map must equal the draw rule (tests/drawn_routes.py, on the oracle's Philox) for every env, with each env's episode and key tracked
on the host across auto-resets, masked resets and in-step restores (clones keep the record's key, rekeyed restores take
their own). Runs use the hard_cap_40 variants of tests/variants.py, so every rollout crosses auto-resets.
"""

import numpy as np
import pytest

from tests import commons_maps as CM
from tests.drawn_routes import route_draw
from tests import env_variants as EV
from tests.test_gpu_player_actions import _action_rows, _records
from tests.test_gpu_player_routes import _Rows, _same_per_env
from tests.test_gpu_step_into import FAMILIES, _blob, _sms

pytestmark = pytest.mark.gpu

STEPS = 60


def _choices(P, rng, n_groups=3):
  """Up to 4 groups per slot (duplicates allowed), one slot without choices when P > 2."""
  out = []
  for p in range(P):
    k = 0 if (P > 2 and p == 1) else int(rng.integers(1, 5))
    out.append(tuple(int(g) for g in rng.integers(0, n_groups, k)))
  if not any(out):
    out[0] = (0,)
  return out


def _routes(eng, choices):
  import torch
  from meltingpot_b200 import substrate
  return substrate.DrawnRoutes(choices, eng.num_envs, eng.num_players, tuple(eng.rgb.shape[2:]), [],
                               torch.device('cuda', eng.device))


class _Model:
  """Each env's episode and key on the host, and the row map the draw rule gives for them."""

  def __init__(self, B, seed, routes, base=0):
    self.ep = np.full(B, -1, np.int64)
    self.key = np.arange(B, dtype=np.int64) + seed + base
    self.seed, self.base, self.r = seed, base, routes
    self.rec = {}

  def map(self):
    d, B, P = self.r.draw, len(self.ep), self.r.num_players
    m = np.full((B, P), -1, np.int32)
    for b in range(B):
      for p in range(P):
        n = d.n_choices[p]
        o = route_draw(int(self.key[b]), int(self.ep[b]), p, n)
        if o >= 0:
          m[b, p] = d.row_base[p][o] + b * d.rows_per_env[p][o]
    return m

  def after(self, step_type, mask=None, restored=None, rekey=False):
    """mask: a reset's envs (None = all); otherwise a step, whose FIRST envs started an episode."""
    st = step_type.cpu().numpy()
    for b in range(len(self.ep)):
      if restored is not None and restored[b] >= 0:
        self.ep[b], key = self.rec[int(restored[b])]
        self.key[b] = self.seed + self.base + b if rekey else key
      elif mask is not None and mask[b]:
        self.ep[b] += 1
      elif mask is None and st[b] == 0:
        self.ep[b] += 1

  def store(self, env_of_slot):
    for s, e in enumerate(env_of_slot):
      if e >= 0:
        self.rec[s] = (int(self.ep[e]), int(self.key[e]))


def _lockstep(blob, B, seed=11, steps=STEPS, env_variant=None, restores=True, rng_seed=0, check_launches=False):
  import torch
  from meltingpot_b200 import engine
  kw = dict(seed=seed, env_variant=env_variant)
  twin, eng = engine.Engine(blob, B, **kw), engine.Engine(blob, B, **kw)
  P = eng.num_players
  rng = np.random.default_rng(rng_seed + B)
  r = _routes(eng, _choices(P, rng))
  model = _Model(B, seed, r)
  tg_e, tg_t = _Rows(eng, r.n_rows), _Rows(twin, r.n_rows)
  bank_e = torch.zeros((6, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  bank_t = bank_e.clone()
  mask_h = np.zeros(B, np.uint8); mask_h[1::3] = 1
  mask = torch.from_numpy(mask_h).cuda()
  prev = None
  for t in range(steps + 1):
    tg_e.refill(); tg_t.refill()
    where = f'B={B} t={t}'
    n0, m0 = eng.launch_count(), twin.launch_count()
    if t in (0, steps // 2):
      m = None if t == 0 else mask
      eng.reset(m, players=tg_e.players(r.row_of_player), draw=r.draw)
      got = r.row_of_player.clone()
      twin.reset(m, players=tg_t.players(got))
      model.after(twin.step_type, mask=np.ones(B, np.uint8) if m is None else mask_h)
    else:
      if restores and t == 8:
        store = torch.full((6,), -1, dtype=torch.int32, device='cuda'); store[:3] = torch.tensor([0, B // 2, B - 1], dtype=torch.int32)
        eng.store_states(bank_e, store); twin.store_states(bank_t, store)
        model.store(store.cpu().numpy())
        n0, m0 = eng.launch_count(), twin.launch_count()
      action = torch.from_numpy(_action_rows(rng, eng, r.n_rows)).cuda()
      kw, idx_h = {}, None
      if restores and t >= 10 and t % 4 == 2:
        idx_h = np.where(rng.random(B) < 0.35, rng.integers(0, 3, B), -1).astype(np.int32)
        kw = dict(restore=torch.from_numpy(idx_h).cuda(), rekey=t % 8 == 2)
      eng.step(None, player_actions={'row_of_player': r.row_of_player, 'action': action},
               players=tg_e.players(r.row_of_player), draw=r.draw, bank=bank_e if kw else None, **kw)
      got = r.row_of_player.clone()
      twin.step(None, player_actions={'row_of_player': prev, 'action': action}, players=tg_t.players(got),
                bank=bank_t if kw else None, **kw)
      model.after(twin.step_type, restored=idx_h, rekey=kw.get('rekey', False))
    if check_launches:
      assert eng.launch_count() - n0 == twin.launch_count() - m0, f'launches {where}'
    assert np.array_equal(got.cpu().numpy(), model.map()), f'row map {where}'
    for name in ('rgb_raw', 'reward_raw', 'scalar_raw'):
      assert torch.equal(getattr(tg_e, name), getattr(tg_t, name)), f'{name} {where}'
    assert torch.equal(eng.reward, twin.reward) and torch.equal(eng.scalar_obs, twin.scalar_obs), where
    _same_per_env(eng, twin, where)
    prev = got
  # unrouted rows kept their sentinel: a routed row holds an image, so not every byte is the sentinel, and rows no
  # player reached this step still are
  used = set(got[got >= 0].tolist())
  free = [k for k in range(r.n_rows) if k not in used]
  assert free and bool((tg_e.rgb[free] == 0xA5).all())
  assert torch.equal(_records(eng), _records(twin)), f'records B={B}'
  return eng, r


@pytest.mark.parametrize('fam', FAMILIES)
def test_drawn_maps_follow_the_rule_and_rows_equal_the_fixed_route_calls(fam):
  blob = _blob(fam)
  for B in (7, _sms() + 3):
    _lockstep(blob, B, check_launches=B == 7)


@pytest.mark.parametrize('which', ['clean_up_variants', 'commons_maps'])
def test_variant_engines(which):
  blobs = list(EV.blobs('clean_up')) if which == 'clean_up_variants' else list(CM.map_set())
  B = _sms() + 5
  _lockstep(blobs, B, env_variant=(np.arange(B) % len(blobs)).astype(np.int64), steps=48)


def test_launch_counts_with_rendering_off():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 16
  eng, twin = engine.Engine(blob, B, seed=1), engine.Engine(blob, B, seed=1)
  r = _routes(eng, _choices(eng.num_players, np.random.default_rng(3)))
  action = torch.zeros(r.n_rows, dtype=torch.int32, device='cuda')
  for e in (eng, twin):
    e.set_flags(0)
  reward_e = torch.zeros(r.n_rows, dtype=torch.float64, device='cuda')
  reward_t = reward_e.clone()

  def added(e, fn):
    n = e.launch_count(); fn(); return e.launch_count() - n

  assert added(eng, lambda: eng.reset(players={'row_of_player': r.row_of_player, 'reward': reward_e}, draw=r.draw)) == \
      added(twin, lambda: twin.reset(players={'row_of_player': r.row_of_player.clone(), 'reward': reward_t}))
  m = r.row_of_player.clone()
  assert added(eng, lambda: eng.step(None, player_actions={'row_of_player': r.row_of_player, 'action': action},
                                     players={'row_of_player': r.row_of_player, 'reward': reward_e}, draw=r.draw)) == \
      added(twin, lambda: twin.step(None, player_actions={'row_of_player': m, 'action': action},
                                    players={'row_of_player': m, 'reward': reward_t}))
  torch.cuda.synchronize()
  assert torch.equal(reward_e, reward_t)


def test_sharded_engines_draw_the_same_groups():
  """One engine of 8 envs and two of 4 (env_index_base 0 and 4) play the same group in every slot of every env."""
  import torch
  from meltingpot_b200 import engine
  blob, seed = _blob('commons_harvest'), 21
  P = engine.Engine(blob, 1, seed=seed).num_players
  choices = _choices(P, np.random.default_rng(5))
  whole = engine.Engine(blob, 8, seed=seed)
  parts = [engine.Engine(blob, 4, seed=seed, env_index_base=4 * i) for i in range(2)]
  routes = [_routes(e, choices) for e in [whole] + parts]

  def groups(r):
    m = r.row_of_player.cpu().numpy()
    starts = np.array([r.rows(g).start for g in range(r.num_groups)] + [r.n_rows])
    return np.where(m >= 0, np.searchsorted(starts, m, side='right') - 1, -1)

  rng = np.random.default_rng(6)
  for t in range(50):
    for e, r in zip([whole] + parts, routes):
      players = {'row_of_player': r.row_of_player, 'reward': torch.zeros(r.n_rows, dtype=torch.float64, device='cuda')}
      if t == 0:
        e.reset(players=players, draw=r.draw)
      else:
        action = torch.from_numpy(rng.integers(0, e.num_actions, r.n_rows).astype(np.int32)).cuda()
        e.step(None, player_actions={'row_of_player': r.row_of_player, 'action': action}, players=players, draw=r.draw)
    g = [groups(r) for r in routes]
    assert np.array_equal(g[0], np.concatenate(g[1:])), f't={t}'


def test_refused_calls_change_nothing():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 8
  eng = engine.Engine(blob, B, seed=1)
  r = _routes(eng, _choices(eng.num_players, np.random.default_rng(2)))
  tg = _Rows(eng, r.n_rows)
  eng.reset(players=tg.players(r.row_of_player), draw=r.draw)
  torch.cuda.synchronize()
  before, n = r.row_of_player.clone(), eng.launch_count()
  action = torch.zeros(r.n_rows, dtype=torch.int32, device='cuda')
  pa = {'row_of_player': r.row_of_player, 'action': action}

  def refused(draw, players, match, actions=pa):
    with pytest.raises(ValueError, match=match):  # MP_E_INVALID
      eng.step(None, player_actions=actions, players=players, draw=draw)

  bad = engine.MpRouteDraw.from_buffer_copy(r.draw)
  bad.n_choices[0] = 9
  refused(bad, tg.players(r.row_of_player), 'player 0 has 9 choices')
  bad = engine.MpRouteDraw.from_buffer_copy(r.draw)
  bad.n_choices[0], bad.row_base[0][0], bad.rows_per_env[0][0] = 1, r.n_rows - 1, 1
  refused(bad, tg.players(r.row_of_player), 'leaves rows')
  bad = engine.MpRouteDraw.from_buffer_copy(r.draw)
  bad.n_rows = r.n_rows - 1
  refused(bad, tg.players(r.row_of_player), "players must deliver through the draw's row map")
  other = r.row_of_player.clone()
  refused(r.draw, tg.players(other), "players must deliver through the draw's row map")
  # the map may not overlap a target or the action rows
  over = torch.zeros(r.n_rows + B * eng.num_players, dtype=torch.int32, device='cuda')
  bad = engine.MpRouteDraw.from_buffer_copy(r.draw)
  bad.row_of_player = over.data_ptr()
  players = dict(tg.players(over[:B * eng.num_players].view(B, -1)))
  refused(bad, players, 'overlap', actions={'row_of_player': over[:B * eng.num_players].view(B, -1), 'action': over[B:B + r.n_rows]})
  torch.cuda.synchronize()
  assert eng.launch_count() == n and torch.equal(r.row_of_player, before)


def test_refused_request_shapes_change_nothing():
  """mp_run refuses a request that mixes a step's and a reset's fields, gives both action sources or neither, or draws
  without the rows the draw delivers to and reads from, before anything is enqueued."""
  import ctypes
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 8
  eng = engine.Engine(blob, B, seed=1)
  P = eng.num_players
  lib = engine.load_library()
  r = _routes(eng, _choices(P, np.random.default_rng(2)))
  tg = _Rows(eng, r.n_rows)
  eng.reset(players=tg.players(r.row_of_player), draw=r.draw)
  a = torch.zeros((B, P), dtype=torch.int32, device='cuda')
  mask = torch.ones(B, dtype=torch.uint8, device='cuda')
  idx = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  bank = torch.zeros((4, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  action = torch.zeros(r.n_rows, dtype=torch.int32, device='cuda')
  other = r.row_of_player.clone()
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

  def rows(rmap, n_rows):
    s = engine.MpPlayerActions()
    s.row_of_player, s.n_rows, s.action, s.action_row_stride = rmap.data_ptr(), n_rows, action.data_ptr(), 4
    return ctypes.pointer(s)

  pa = rows(r.row_of_player, r.n_rows)
  players = ctypes.pointer(eng._player_outputs(tg.players(r.row_of_player)))  # pylint: disable=protected-access
  draw = ctypes.pointer(r.draw)

  def refused(match, **request):
    torch.cuda.synchronize()
    state, n, rmap = eng.save_state(), eng.launch_count(), r.row_of_player.clone()
    rc = lib.mp_run(eng._h, ctypes.byref(engine.MpRequest(**request)), stream)  # pylint: disable=protected-access
    assert rc == -1, (match, rc)
    assert match in lib.mp_last_error().decode(), (match, lib.mp_last_error())
    torch.cuda.synchronize()
    assert eng.launch_count() == n, match
    assert eng.save_state() == state and torch.equal(r.row_of_player, rmap), match

  # a reset with any field of a step
  no_step_fields = 'a reset takes no actions, player_actions, slot_of_env, bank or restore_flags'
  refused(no_step_fields, reset=1, actions=a.data_ptr())
  refused(no_step_fields, reset=1, player_actions=pa, players=players)
  refused(no_step_fields, reset=1, slot_of_env=idx.data_ptr(), bank=bank.data_ptr(), n_slots=4)
  refused(no_step_fields, reset=1, slot_of_env=idx.data_ptr())
  refused(no_step_fields, reset=1, bank=bank.data_ptr())
  refused(no_step_fields, reset=1, restore_flags=engine.MP_RESTORE_REKEY)
  # a step with a reset's mask, with both action sources, or with neither
  refused('env_mask is for a reset', actions=a.data_ptr(), env_mask=mask.data_ptr())
  refused('not both', actions=a.data_ptr(), player_actions=pa)
  refused('has neither', out=None)
  refused('has neither', slot_of_env=idx.data_ptr(), bank=bank.data_ptr(), n_slots=4, players=players)
  # draw without players, on a step or a reset
  refused('draw needs players', reset=1, draw=draw)
  refused('draw needs players', player_actions=pa, draw=draw)
  # a drawn step whose actions do not come from the draw's rows
  through = "a drawn step must read player_actions through the draw's row map and n_rows"
  refused(through, actions=a.data_ptr(), draw=draw, players=players)
  refused(through, player_actions=rows(other, r.n_rows), draw=draw, players=players)
  refused(through, player_actions=rows(r.row_of_player, r.n_rows - 1), draw=draw, players=players)
  # accepted as a control: the same drawn step, reading through the draw's rows
  engine._check(lib.mp_run(eng._h, ctypes.byref(engine.MpRequest(player_actions=pa, draw=draw, players=players)), stream))  # pylint: disable=protected-access
  torch.cuda.synchronize()


def test_batched_scenario_population_equals_manual_stepping():
  """Three constant-action bots: the scenario's focal outputs equal a dense twin stepped with the bots' actions."""
  import torch
  from meltingpot_b200 import scenario, substrate
  blob, B, seed = _blob('clean_up'), 24, 3
  sub = substrate.BatchedSubstrate(blob, B, seed=seed)
  twin = substrate.BatchedSubstrate(blob, B, seed=seed)
  P = sub.num_players
  is_focal = [p < 3 for p in range(P)]
  roles = ['default'] * P
  bot_action = {'a': 1, 'b': 7, 'c': 3}

  def bot(name):
    def policy(ts, active):
      assert ts.reward.shape == active.shape and active.dtype == torch.bool
      return torch.full(active.shape, bot_action[name], dtype=torch.int32, device=active.device)
    return policy

  s = scenario.BatchedScenario(sub, {k: bot(k) for k in bot_action}, is_focal, ['RGB', 'READY_TO_SHOOT'], roles=roles,
                               bots_by_role={'default': ['c', 'a', 'b', 'a']})
  assert s.bot_names == ('a', 'b', 'c')
  rng = np.random.default_rng(0)
  focal_ts, ts = s.reset(), twin.reset()
  lut = torch.tensor([bot_action[n] for n in s.bot_names], dtype=torch.int32, device='cuda')
  bg = [p for p in range(P) if not is_focal[p]]
  seen = set()
  for t in range(60):
    assert torch.equal(focal_ts.reward, ts.reward[:, :3]), f't={t}'
    assert torch.equal(focal_ts.observation['RGB'], ts.observation['RGB'][:, :3]), f't={t}'
    bots = s.background_bots()
    seen |= set(bots.reshape(-1).tolist())
    for k, name in enumerate(s.bot_names):  # each bot's active rows are the slots that play it
      active = s._routes.active(k + 1)  # pylint: disable=protected-access
      slots = s._routes.group(k + 1)  # pylint: disable=protected-access
      want = torch.stack([bots[:, bg.index(p)] == k for p in slots], dim=1)
      assert torch.equal(active, want), f'active {name} t={t}'
    focal = torch.from_numpy(rng.integers(0, sub.num_actions, (B, 3)).astype(np.int32)).cuda()
    dense = torch.zeros((B, P), dtype=torch.int32, device='cuda')
    dense[:, :3] = focal
    dense[:, bg] = lut[bots]
    focal_ts, ts = s.step(focal), twin.step(dense)
  assert seen == {0, 1, 2}
