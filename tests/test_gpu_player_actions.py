"""Actions read from rows (mp_run's player_actions, Engine.step(player_actions=), PlayerRoutes.actions).

A routed engine steps beside a lockstep twin built with the same seed. The twin is stepped with the dense [B, P] actions
the rule gives, composed on the host: player p of env b takes action[row_of_player[b, p]] when that row lies in
0..n_rows-1, and action 0 otherwise. Every output, the per-env state and, at the end, every env's state record (keys and
variant bytes included) must then be equal. Rows hold out-of-range ids too, and the maps change every step. Runs use the
hard_cap_40 variants of tests/variants.py, so every rollout crosses an auto-reset.
"""

import ctypes

import numpy as np
import pytest

from tests import coins_draws as CD
from tests import env_variants as EV
from tests.test_gpu_player_routes import FAMILIES, _Rows, _row_map, _same_per_env
from tests.test_gpu_step_into import _acts, _blob, _cudart, _sms

pytestmark = pytest.mark.gpu

STEPS = 44


def _action_rows(rng, eng, n_rows):
  """int32 [n_rows] action ids, about one in eight out of range (-1, n_actions or larger)."""
  a = rng.integers(0, eng.num_actions, n_rows)
  bad = rng.random(n_rows) < 0.125
  a[bad] = rng.choice([-1, -7, eng.num_actions, eng.num_actions + 3, 1 << 20], int(bad.sum()))
  return a.astype(np.int32)


def _dense(row_map, action):
  """The [B, P] actions the rows give (host-composed)."""
  import torch
  m, a = row_map.cpu().numpy(), action.cpu().numpy()
  ok = (m >= 0) & (m < a.shape[0])
  return torch.from_numpy(np.where(ok, a[np.clip(m, 0, a.shape[0] - 1)], 0).astype(np.int32)).cuda()


class _Source:
  """Action rows in one of three layouts: dense [n_rows], a column of [n_rows, T] or at(t) of [T, n_rows]."""

  def __init__(self, kind, n_rows, T):
    import torch
    self.kind = kind
    shape = {'dense': (n_rows,), 'column': (n_rows, T), 'slot': (T, n_rows)}[kind]
    self.buf = torch.full(shape, 0x5A5A5A5A, dtype=torch.int32, device='cuda')

  def rows(self, t, values):
    import torch
    v = self.buf if self.kind == 'dense' else self.buf[:, t] if self.kind == 'column' else self.buf[t]
    v.copy_(torch.from_numpy(values))
    return v


def _records(eng):
  import torch
  bank = torch.zeros((eng.num_envs, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.arange(eng.num_envs, dtype=torch.int32, device='cuda'))
  return bank


def _same_outputs(eng, twin, where):
  import torch
  for name in ('rgb', 'reward', 'scalar_obs'):
    assert torch.equal(getattr(eng, name), getattr(twin, name)), f'{name} {where}'
  _same_per_env(eng, twin, where)


def _lockstep(blob, B, kind, source, seed=11, steps=STEPS, env_variant=None, blobs=None):
  import torch
  from meltingpot_b200 import engine
  src = blobs if blobs is not None else blob
  kw = dict(seed=seed, env_variant=env_variant)
  twin, eng = engine.Engine(src, B, **kw), engine.Engine(src, B, **kw)
  P = eng.num_players
  n_rows = B * P + 3
  rng = np.random.default_rng(B * 5 + len(kind) + len(source))
  acts = _Source(source, n_rows, steps + 1)
  mask = torch.zeros(B, dtype=torch.uint8, device='cuda'); mask[1::3] = 1
  twin.reset(); eng.reset()
  for t in range(1, steps + 1):
    if t == steps // 2:
      twin.reset(mask); eng.reset(mask)
    rmap = _row_map(kind, B, P, n_rows, rng)  # a new map every step
    action = acts.rows(t, _action_rows(rng, eng, n_rows))
    twin.step(_dense(rmap, action))
    eng.step(None, player_actions={'row_of_player': rmap, 'action': action})
    _same_outputs(eng, twin, f'{kind} {source} B={B} t={t}')
  assert torch.equal(_records(eng), _records(twin)), f'records {kind} {source} B={B}'


@pytest.mark.parametrize('kind', ['identity', 'permuted', 'partial'])
@pytest.mark.parametrize('fam', FAMILIES)
def test_routed_actions_equal_the_twin(fam, kind):
  sms = _sms()
  blob = _blob(fam)
  for i, B in enumerate((1, 7, sms - 1, sms + 1, 2 * sms + 5)):
    _lockstep(blob, B, kind, ('dense', 'column', 'slot')[i % 3])


@pytest.mark.parametrize('family', ['clean_up', 'coins'])
def test_variant_engines_and_coins_draws(family):
  blobs = list(EV.blobs(family)) if family == 'clean_up' else list(CD.draw_set())
  B = 2 * _sms() + 5
  _lockstep(None, B, 'permuted', 'column', blobs=blobs, env_variant=(np.arange(B) % len(blobs)).astype(np.int64), steps=45)


def test_with_players_out_and_bank():
  """players (sharing the action row map), out and a bank, alone and together; restored envs ignore their rows."""
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('commons_harvest'), 37
  twin, eng = engine.Engine(blob, B, seed=5), engine.Engine(blob, B, seed=5)
  P = eng.num_players
  n_rows = B * P
  tg = _Rows(eng, n_rows)
  rng = np.random.default_rng(1)
  bank_t = torch.zeros((8, twin.state_record_bytes), dtype=torch.uint8, device='cuda')
  bank_e = bank_t.clone()
  # (no world_rgb: it would leave the engine's own WORLD.RGB unwritten, which the per-env check reads)
  out = {'discount': torch.zeros_like(eng.discount), 'step_type': torch.zeros_like(eng.step_type),
         'reward': torch.zeros_like(eng.reward)}
  twin.reset(); eng.reset()
  for t in range(60):
    if t == 10:
      store = torch.full((8,), -1, dtype=torch.int32, device='cuda'); store[:4] = torch.tensor([0, 5, 9, 30], dtype=torch.int32)
      twin.store_states(bank_t, store); eng.store_states(bank_e, store)
    rmap = _row_map('partial' if t % 2 else 'permuted', B, P, n_rows, rng)
    action = torch.from_numpy(_action_rows(rng, eng, n_rows)).cuda()
    dense = _dense(rmap, action)
    pa = {'row_of_player': rmap, 'action': action}
    kw, where = {}, f't={t}'
    if t >= 12 and t % 3 == 0:  # restored envs' rows hold actions, which they must ignore
      idx = torch.from_numpy(np.where(rng.random(B) < 0.3, rng.integers(0, 5, B), -1).astype(np.int32)).cuda()
      kw = dict(restore=idx, rekey=t % 2 == 0)
    with_players, with_out = t % 4 in (1, 3), t % 4 in (2, 3)
    tg.refill()
    twin.step(dense, bank=bank_t if kw else None, **kw)
    eng.step(None, player_actions=pa, bank=bank_e if kw else None, out=out if with_out else None,
             players=tg.players(rmap) if with_players else None, **kw)
    if with_players:
      tg.check(twin, rmap, where)
    else:
      assert torch.equal(eng.rgb, twin.rgb), where
    if with_out:
      for name in out:
        assert torch.equal(out[name], getattr(twin, name)), f'{name} {where}'
    assert torch.equal(eng.reward, twin.reward) and torch.equal(eng.scalar_obs, twin.scalar_obs), where
    _same_per_env(eng, twin, where)
  assert torch.equal(_records(eng), _records(twin))


def test_routed_actions_equal_the_oracle(oracle):
  import torch
  from meltingpot_b200 import engine
  blob, B, seed = _blob('clean_up'), 7, 3
  eng = engine.Engine(blob, B, seed=seed)
  P = eng.num_players
  envs = [oracle.OracleEnv(blob, seed + b) for b in range(B)]
  rng = np.random.default_rng(0)
  eng.reset()
  for e in envs:
    e.reset()
  for t in range(45):
    rmap = _row_map('partial', B, P, B * P, rng)
    action = torch.from_numpy(_action_rows(rng, eng, B * P)).cuda()
    eng.step(None, player_actions={'row_of_player': rmap, 'action': action})
    dense = _dense(rmap, action).cpu().numpy()
    torch.cuda.synchronize()
    rgb, reward = eng.rgb.cpu().numpy(), eng.reward.cpu().numpy()
    for b, e in enumerate(envs):
      e.step(dense[b])
      assert np.array_equal(rgb[b], e.rgb()), (t, b)
      assert np.array_equal(reward[b], e.rewards()), (t, b)
    assert np.array_equal(eng.world_rgb.cpu().numpy(), np.stack([e.world_rgb() for e in envs])), t


def test_launch_count_equals_the_composed_call():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 16
  eng = engine.Engine(blob, B, seed=1)
  P = eng.num_players
  tg = _Rows(eng, B * P)
  rmap = _row_map('partial', B, P, B * P, np.random.default_rng(0))
  pa = {'row_of_player': rmap, 'action': torch.zeros(B * P, dtype=torch.int32, device='cuda')}
  out = {'reward': torch.zeros_like(eng.reward)}
  bank = torch.zeros((2, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  idx = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  eng.reset()
  a = torch.zeros((B, P), dtype=torch.int32, device='cuda')

  def added(fn):
    n = eng.launch_count(); fn(); return eng.launch_count() - n

  for flags in (engine.MP_FLAG_DEFAULT, 0):
    eng.set_flags(flags)
    assert added(lambda: eng.step(None, player_actions=pa)) == added(lambda: eng.step(a))
    assert added(lambda: eng.step(None, player_actions=pa, out=out)) == added(lambda: eng.step(a, out=out))
    assert added(lambda: eng.step(None, player_actions=pa, restore=idx, bank=bank)) == added(lambda: eng.step(a, restore=idx, bank=bank))
    players = tg.players(rmap) if flags else {'row_of_player': rmap, 'reward': tg.reward}
    assert (added(lambda: eng.step(None, player_actions=pa, players=players, restore=idx, bank=bank))
            == added(lambda: eng.step(a, players=players, restore=idx, bank=bank)))


def test_refused_calls_change_nothing():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 12
  eng = engine.Engine(blob, B, seed=1)
  P = eng.num_players
  lib = engine.load_library()
  eng.reset()
  rmap = torch.arange(B * P, dtype=torch.int32, device='cuda').view(B, P)
  act = torch.full((4 * B * P,), 3, dtype=torch.int32, device='cuda')
  rew = torch.full((B * P,), 1.5, dtype=torch.float64, device='cuda')
  bank = torch.zeros((4, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  idx = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

  def struct(**kw):
    s = engine.MpPlayerActions()
    s.row_of_player, s.n_rows, s.action, s.action_row_stride = rmap.data_ptr(), B * P, act.data_ptr(), 4
    for k, v in kw.items():
      setattr(s, k, v)
    return s

  def refused(s, match, players=None, restore=False, out=None, flags=0, n_slots=4):
    torch.cuda.synchronize()
    before = [t.clone() for t in (eng.avatar_state, eng.grid, eng.step_type, eng.reward, act, rew)]
    snap = eng.save_state()
    n = eng.launch_count()
    r = engine.MpRequest(n_slots=n_slots, restore_flags=flags)
    if s is not None:
      r.player_actions = ctypes.pointer(s)
    if restore:
      r.slot_of_env, r.bank = idx.data_ptr(), bank.data_ptr()
    if out is not None:
      r.out = ctypes.pointer(out)
    if players is not None:
      r.players = ctypes.pointer(players)
    rc = lib.mp_run(eng._h, ctypes.byref(r), stream)  # pylint: disable=protected-access
    assert rc == -1, (match, rc)
    assert match in lib.mp_last_error().decode(), (match, lib.mp_last_error())
    torch.cuda.synchronize()
    assert eng.launch_count() == n, match
    assert eng.save_state() == snap, match
    for x, y in zip(before, (eng.avatar_state, eng.grid, eng.step_type, eng.reward, act, rew)):
      assert torch.equal(x, y), match

  refused(None, 'has neither')  # a step with neither actions nor player_actions
  refused(struct(n_rows=0), 'n_rows')
  refused(struct(row_of_player=None), 'row_of_player')
  refused(struct(row_of_player=rmap.data_ptr() + 2), 'row_of_player')
  refused(struct(action=None), 'action is null')
  refused(struct(action=act.data_ptr() + 2), 'multiple of 4')
  refused(struct(action_row_stride=6), 'multiple of 4')
  refused(struct(action_row_stride=1 << 31), '2 GiB')
  refused(struct(action_row_stride=0), 'smaller than one row')
  cudart = _cudart()
  ptr = ctypes.c_void_p()
  assert cudart.cudaMalloc(ctypes.byref(ptr), ctypes.c_size_t(1 << 20)) == 0
  try:  # a row map whose B * P i32, and action rows that run past the end of their allocation
    end = ptr.value + (1 << 20)
    refused(struct(row_of_player=end - 16), 'past the end')
    refused(struct(action=end - 8, n_rows=3), 'past the end')
    refused(struct(action=end - 64, action_row_stride=32, n_rows=3), 'past the end')
  finally:
    cudart.cudaFree(ptr)
  refused(struct(action=rmap.data_ptr()), 'overlap')
  refused(struct(action=eng.step_type.data_ptr()), "engine's own buffers")
  refused(struct(row_of_player=eng.grid.data_ptr()), "engine's own buffers")
  refused(struct(action=bank.data_ptr()), 'overlap', restore=True)
  refused(struct(action=idx.data_ptr(), n_rows=B), 'overlap', restore=True)
  o = engine.MpDeviceOutputs(); o.reward, o.reward_env_stride = act.data_ptr(), P * 8
  refused(struct(), 'overlap', out=o)
  p = engine.MpPlayerOutputs(); p.row_of_player, p.n_rows, p.reward, p.reward_row_stride = rmap.data_ptr(), B * P, act.data_ptr(), 8
  refused(struct(), 'overlap', players=p)
  p = engine.MpPlayerOutputs(); p.row_of_player, p.n_rows, p.reward, p.reward_row_stride = rmap.data_ptr() + 4, B * P, rew.data_ptr(), 8
  refused(struct(), 'overlap', players=p)  # two row maps that overlap without being one tensor
  # the refusals of the composed calls
  r = engine.MpRequest(player_actions=ctypes.pointer(struct()), slot_of_env=idx.data_ptr(), n_slots=4)
  assert lib.mp_run(eng._h, ctypes.byref(r), stream) == -1  # pylint: disable=protected-access
  assert 'go together' in lib.mp_last_error().decode()
  refused(struct(), 'n_slots', restore=True, n_slots=0)
  refused(struct(), 'unknown flags', restore=True, flags=2)
  refused(struct(), 'flags without a bank', flags=1)
  refused(struct(), 'n_rows', players=engine.MpPlayerOutputs())
  # accepted: the two row maps are one tensor, and the player outputs take the rows
  p = engine.MpPlayerOutputs(); p.row_of_player, p.n_rows, p.reward, p.reward_row_stride = rmap.data_ptr(), B * P, rew.data_ptr(), 8
  r = engine.MpRequest(player_actions=ctypes.pointer(struct()), players=ctypes.pointer(p))
  assert lib.mp_run(eng._h, ctypes.byref(r), stream) == 0  # pylint: disable=protected-access
  torch.cuda.synchronize()
  assert torch.equal(rew, eng.reward.reshape(-1))


def test_gather_accepted_without_players_and_refused_with_them(clean_up_blob):
  import torch
  from meltingpot_b200 import engine
  B = 40
  twin, eng = engine.Engine(clean_up_blob, B, seed=5), engine.Engine(clean_up_blob, B, seed=5)
  P = eng.num_players
  tg = _Rows(eng, B * P)
  for e in (eng, twin):
    ptr, _ = e.gather_obs_create(0, 1)
    e.gather_obs_connect([ptr])
  twin.reset(); eng.reset()
  rng = np.random.default_rng(3)
  for t in range(45):
    rmap = _row_map('permuted', B, P, B * P, rng)
    action = torch.from_numpy(_action_rows(rng, eng, B * P)).cuda()
    n = eng.launch_count()
    eng.step(None, player_actions={'row_of_player': rmap, 'action': action})
    m = twin.launch_count()
    twin.step(_dense(rmap, action))
    assert eng.launch_count() - n == twin.launch_count() - m
    torch.cuda.synchronize()
    _same_outputs(eng, twin, f'gather t={t}')
  n = eng.launch_count()
  with pytest.raises(ValueError, match='-2.*gather'):
    eng.step(None, player_actions={'row_of_player': rmap, 'action': action}, players=tg.players(rmap))
  assert eng.launch_count() == n


def test_batched_substrate_player_actions():
  """Observations into rows and actions from the same rows, T slots of each, against a twin stepped densely."""
  import torch
  from meltingpot_b200 import substrate
  blob, B = _blob('clean_up'), 9
  twin = substrate.BatchedSubstrate(blob, B, seed=4)
  env = substrate.BatchedSubstrate(blob, B, seed=4)
  P = env.num_players
  rng = np.random.default_rng(2)
  groups = rng.integers(-1, 3, size=(B, P))
  routes = env.player_routes(groups)
  traj, acts = routes.outputs(T=45), routes.actions(T=45)
  env.reset(players=traj.at(0))
  twin.reset()
  for t in range(1, 45):
    for g in range(routes.num_groups):
      acts.group(g)[t].copy_(torch.from_numpy(rng.integers(0, env.num_actions, routes.rows(g).stop - routes.rows(g).start)))
    ts = env.step(players=traj.at(t), player_actions=acts.at(t))
    dense = torch.zeros((B, P), dtype=torch.int32, device='cuda')
    dense[routes.env_of_row, routes.player_of_row] = acts.tensor[t]
    want = twin.step(dense)
    assert torch.equal(ts.step_type, want.step_type) and torch.equal(ts.reward, want.reward), t
    assert torch.equal(traj['RGB'][t], want.observation['RGB'][routes.env_of_row, routes.player_of_row]), t
  with pytest.raises(ValueError, match='not both'):
    env.step(dense, player_actions=acts.at(0))
