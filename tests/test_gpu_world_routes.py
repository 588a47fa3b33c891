"""WORLD.RGB routed per env (mp_player_outputs.world_row_of_env / world_rgb; PlayerRoutes.outputs(world_envs=),
BatchedScenario(world_envs=)).

Each run steps a routed engine beside a lockstep twin of the same blob and seed, fed the same actions. The routed engine
draws WORLD.RGB only for a scattered, non-monotone subset of envs, into padded rows of a sentinel-filled target. Every
routed row must equal the twin's WORLD.RGB of its env byte for byte, the player rows the twin's images; every other
byte of the targets (spare rows, row padding) and the routed engine's own images must keep the sentinel. Runs use the
40-frame-capped blobs of tests/env_variants.py, so every rollout crosses an auto-reset.
"""

import ctypes

import numpy as np
import pytest

from tests import env_variants as EV
from tests import parity
from tests.test_gpu_player_routes import _Rows, _row_map, _same_per_env
from tests.test_gpu_step_into import _SENT, _acts, _cudart, _sms

pytestmark = pytest.mark.gpu

STEPS = 46
PAD = 16   # bytes of padding behind every WORLD.RGB row (keeps the rows 16-byte aligned)
SPARE = 2  # rows of the target no env is routed to


def _blob(fam):
  return EV.blobs(fam)[0]


class _World:
  """A sentinel-filled target of `n_rows` padded WORLD.RGB rows for `eng`."""

  def __init__(self, eng, n_rows):
    import torch
    H, W = eng.world_rgb.shape[1:3]
    per = H * W * 3
    self.raw = torch.full((n_rows * (per + PAD),), _SENT['u8'], dtype=torch.uint8, device='cuda')
    self.rows = torch.as_strided(self.raw, (n_rows, H, W, 3), (per + PAD, W * 3, 3, 1))

  def refill(self):
    self.raw.fill_(_SENT['u8'])

  def check(self, want, envs, where):
    """Row k equals want[envs[k]]; with the routed rows set back to the sentinel, every byte is the sentinel."""
    import torch
    k = len(envs)
    assert torch.equal(self.rows[:k], want[envs]), f'WORLD.RGB {where}'
    self.rows[:k] = _SENT['u8']
    assert bool((self.raw == _SENT['u8']).all()), f'WORLD.RGB {where}: bytes outside the routed rows were written'


def _scattered(B, n_tail, rng):
  """int64 CUDA [n] of distinct envs in a random (non-monotone) order: about a quarter of the balanced part [0, B -
  n_tail) and of the cooperative tail [B - n_tail, B), each part keeping routed and unrouted envs where it has two."""
  import torch
  parts = [np.arange(0, B - n_tail), np.arange(B - n_tail, B)]
  pick = []
  for part in parts:
    if len(part) == 0:
      continue
    n = max(2, len(part) // 4) if len(part) > 2 else 1
    pick.extend(rng.choice(part, size=n, replace=False).tolist())
  pick = rng.permutation(np.array(pick, np.int64))
  if len(pick) > 1 and np.all(np.diff(pick) > 0):
    pick = pick[::-1].copy()
  return torch.from_numpy(pick).cuda()


def _row_map_of(B, envs):
  import torch
  m = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  m[envs] = torch.arange(len(envs), dtype=torch.int32, device='cuda')
  return m


def _tail_batch(eng_like_blob):
  """A batch size whose balanced part holds two rounds and whose cooperative tail holds about half the SMs' envs."""
  from meltingpot_b200 import engine
  e = engine.Engine(eng_like_blob, 8, seed=1)
  teams = e.render_plan()['teams']
  e.close()
  sms = _sms()
  return 2 * sms * teams + sms // 2 + 3, sms // 2 + 3


def _lockstep(blob, B, n_tail, seed=11, steps=STEPS, blobs=None, env_variant=None, player_kind='partial'):
  import torch
  from meltingpot_b200 import engine
  src = blobs if blobs is not None else blob
  kw = dict(seed=seed, env_variant=env_variant)
  twin, eng = engine.Engine(src, B, **kw), engine.Engine(src, B, **kw)
  P = eng.num_players
  rng = np.random.default_rng(B * 13 + seed)
  envs = _scattered(B, n_tail, rng)
  wmap = _row_map_of(B, envs)
  world = _World(eng, len(envs) + SPARE)
  n_rows = B * P + 3
  tg = _Rows(eng, n_rows)
  eng.world_rgb.fill_(_SENT['u8']); eng.rgb.fill_(_SENT['u8'])
  mask = torch.zeros(B, dtype=torch.uint8, device='cuda'); mask[1::3] = 1
  for t in range(steps + 1):
    rmap = _row_map(player_kind, B, P, n_rows, rng)
    players = dict(tg.players(rmap), world_row_of_env=wmap, world_rgb=world.rows)
    tg.refill(); world.refill()
    if t == 0 or t == steps // 2:
      m = None if t == 0 else mask
      twin.reset(m)
      eng.reset(m, players=players)
    else:
      a = _acts(rng, eng)
      twin.step(a)
      eng.step(a, players=players)
    where = f'B={B} t={t}'
    world.check(twin.world_rgb, envs, where)
    tg.check(twin, rmap, where)
    for name in ('discount', 'step_type', 'avatar_state', 'grid', 'event_count'):
      assert torch.equal(getattr(eng, name), getattr(twin, name)), f'{name} {where}'
    assert bool((eng.world_rgb == _SENT['u8']).all()), f'own world_rgb written {where}'
    assert bool((eng.rgb == _SENT['u8']).all()), f'own rgb written {where}'
  return twin, eng


@pytest.mark.parametrize('fam', EV.NAMES)
def test_routed_world_rows_equal_the_dense_engine(fam):
  blob = _blob(fam)
  _lockstep(blob, 5, 0)
  B, n_tail = _tail_batch(blob)
  _lockstep(blob, B, n_tail)


def test_routed_world_rows_equal_the_oracle(oracle):
  import torch
  from meltingpot_b200 import engine
  blob, B, seed = _blob('clean_up'), 9, 3
  eng = engine.Engine(blob, B, seed=seed)
  P = eng.num_players
  envs_of = [oracle.OracleEnv(blob, seed + b) for b in range(B)]
  envs = torch.tensor([7, 2, 5], dtype=torch.int64, device='cuda')
  world = _World(eng, 3)
  tg = _Rows(eng, B * P)
  players = dict(tg.players(_row_map('identity', B, P, B * P, None)), world_row_of_env=_row_map_of(B, envs),
                 world_rgb=world.rows)
  eng.reset(players=players)
  for e in envs_of:
    e.reset()
  rng = np.random.default_rng(0)
  shapes = parity.shapes_of(eng)
  pick = envs.tolist()
  for t in range(45):
    a = _acts(rng, eng)
    eng.step(a, players=players)
    acts = a.cpu().numpy()
    for b, e in enumerate(envs_of):
      e.step(acts[b])
    if t % 11 == 0 or t == 44:
      torch.cuda.synchronize()
      want = parity.env_dump([envs_of[b] for b in pick], shapes, pixels=True, kinds=('world',))
      parity.check_outputs({'world': world.rows.cpu().numpy()}, want, f'routed WORLD.RGB step {t}')


def test_restores_inside_the_step():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('commons_harvest'), 37
  twin, eng = engine.Engine(blob, B, seed=5), engine.Engine(blob, B, seed=5)
  P = eng.num_players
  rng = np.random.default_rng(1)
  envs = _scattered(B, 0, rng)
  world = _World(eng, len(envs) + SPARE)
  tg = _Rows(eng, B * P)
  wmap = _row_map_of(B, envs)
  bank_t = torch.zeros((8, twin.state_record_bytes), dtype=torch.uint8, device='cuda')
  bank_e = bank_t.clone()
  twin.reset(); eng.reset()
  for t in range(50):
    a = _acts(rng, eng)
    if t == 10:
      store = torch.full((8,), -1, dtype=torch.int32, device='cuda'); store[:4] = torch.tensor([0, 5, 9, 30], dtype=torch.int32)
      twin.store_states(bank_t, store); eng.store_states(bank_e, store)
    if t >= 12 and t % 3 == 0:
      idx = torch.from_numpy(np.where(rng.random(B) < 0.3, rng.integers(0, 5, B), -1).astype(np.int32)).cuda()
      rmap = _row_map('partial', B, P, B * P, rng)
      tg.refill(); world.refill()
      twin.step(a, restore=idx, bank=bank_t, rekey=t % 2 == 0)
      eng.step(a, restore=idx, bank=bank_e, rekey=t % 2 == 0,
               players=dict(tg.players(rmap), world_row_of_env=wmap, world_rgb=world.rows))
      world.check(twin.world_rgb, envs, f'restore t={t}')
      tg.check(twin, rmap, f'restore t={t}')
    else:
      twin.step(a); eng.step(a)
      _same_per_env(eng, twin, f't={t}')


def test_variant_engine():
  blobs = list(EV.blobs('clean_up'))
  B = 2 * _sms() + 5
  assign = (np.arange(B) % len(blobs)).astype(np.int64)
  _lockstep(None, B, 5, blobs=blobs, env_variant=assign, player_kind='permuted', steps=45)


def test_drawn_routes_with_world_rows():
  import torch
  from meltingpot_b200 import substrate
  blob, B = _blob('coop_mining'), 23
  sa, sb = substrate.BatchedSubstrate(blob, B, seed=7), substrate.BatchedSubstrate(blob, B, seed=7)
  P = sa.num_players
  choices = [(0,), (1, 2), (2,), (), (1,), (0, 2)][:P]
  ra, rb = sa.drawn_routes(choices), sb.drawn_routes(choices)
  envs = [17, 3, 11, 0, 22]
  poa, pob = ra.outputs(world_envs=envs), rb.outputs()
  paa, pab = ra.actions(), rb.actions()
  sa.engine.world_rgb.fill_(_SENT['u8'])
  ta, tb = sa.reset(players=poa), sb.reset(players=pob)
  rng = np.random.default_rng(5)
  idx = torch.tensor(envs, device='cuda')
  for t in range(46):
    if t:
      acts = torch.from_numpy(rng.integers(0, sa.num_actions, ra.n_rows).astype(np.int32)).cuda()
      paa.tensor.copy_(acts); pab.tensor.copy_(acts)
      ta, tb = sa.step(players=poa, player_actions=paa), sb.step(players=pob, player_actions=pab)
    assert ta.observation['WORLD.RGB'] is poa['WORLD.RGB']
    assert torch.equal(poa['WORLD.RGB'], tb.observation['WORLD.RGB'][idx]), t
    assert torch.equal(poa['RGB'], pob['RGB']) and torch.equal(poa['REWARD'], pob['REWARD']), t
    assert torch.equal(ra.row_of_player, rb.row_of_player) and torch.equal(ta.step_type, tb.step_type), t
    assert bool((sa.engine.world_rgb == _SENT['u8']).all()), t


def test_trajectory_slots():
  import torch
  from meltingpot_b200 import substrate
  blob, B, T = _blob('territory'), 19, 45
  env, twin = substrate.BatchedSubstrate(blob, B, seed=4), substrate.BatchedSubstrate(blob, B, seed=4)
  P = env.num_players
  rng = np.random.default_rng(2)
  routes = env.player_routes(rng.integers(-1, 3, size=(B, P)))
  envs = torch.tensor([12, 0, 18, 5], device='cuda')
  traj = routes.outputs(T, world_envs=envs)
  out = twin.trajectory(T)
  ts = env.reset(players=traj.at(0)); twin.reset(out=out.at(0))
  for t in range(1, T):
    a = torch.from_numpy(rng.integers(0, env.num_actions, (B, P)).astype(np.int32)).cuda()
    # with out= as well: WORLD.RGB goes to the rows, out keeps every other per-env field
    dst = env.trajectory(1).at(0)
    before = dst.observation['WORLD.RGB'].clone()
    ts = env.step(a, out=dst, players=traj.at(t))
    twin.step(a, out=out.at(t))
    assert ts.observation['WORLD.RGB'].data_ptr() == traj['WORLD.RGB'][t].data_ptr()
    assert torch.equal(dst.observation['WORLD.RGB'], before), t
    assert torch.equal(dst.step_type, out.step_type[t]) and torch.equal(dst.reward, out.reward[t]), t
  e, p = routes.env_of_row, routes.player_of_row
  assert torch.equal(traj['WORLD.RGB'][1:], out.observation['WORLD.RGB'][1:, envs])
  assert torch.equal(traj['RGB'][1:], out.observation['RGB'][1:, e, p])


def test_launch_counts_equal_the_call_without_world_rows():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 16
  eng = engine.Engine(blob, B, seed=1)
  P = eng.num_players
  tg = _Rows(eng, B * P)
  world = _World(eng, 4)
  rmap = _row_map('partial', B, P, B * P, np.random.default_rng(0))
  plain = tg.players(rmap)
  routed = dict(plain, world_row_of_env=_row_map_of(B, torch.tensor([3, 9, 0], device='cuda')), world_rgb=world.rows)
  eng.reset()
  a = torch.zeros((B, P), dtype=torch.int32, device='cuda')

  def added(fn):
    n = eng.launch_count(); fn(); return eng.launch_count() - n

  assert added(lambda: eng.step(a, players=routed)) == added(lambda: eng.step(a, players=plain))
  assert added(lambda: eng.reset(players=routed)) == added(lambda: eng.reset(players=plain))
  rows = {'row_of_player': rmap, 'action': torch.zeros(B * P, dtype=torch.int32, device='cuda')}
  assert (added(lambda: eng.step(None, players=routed, player_actions=rows))
          == added(lambda: eng.step(None, players=plain, player_actions=rows)))


def test_refused_calls_change_nothing():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 12
  eng = engine.Engine(blob, B, seed=1)
  P, h, w = eng.num_players, eng.rgb.shape[2], eng.rgb.shape[3]
  H, W = eng.world_rgb.shape[1:3]
  per = H * W * 3
  lib = engine.load_library()
  eng.reset()
  a = torch.zeros((B, P), dtype=torch.int32, device='cuda')
  rmap = torch.arange(B * P, dtype=torch.int32, device='cuda').view(B, P)
  wmap = torch.arange(B, dtype=torch.int32, device='cuda')
  prgb = torch.full((B * P * h * w * 3,), 0xA5, dtype=torch.uint8, device='cuda')
  wrgb = torch.full((B * per + 4096,), 0xA5, dtype=torch.uint8, device='cuda')
  rew = torch.full((4 * B * P,), 1.5, dtype=torch.float64, device='cuda')
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

  def struct(**kw):
    s = engine.MpPlayerOutputs()
    s.row_of_player, s.n_rows = rmap.data_ptr(), B * P
    s.rgb, s.rgb_row_stride = prgb.data_ptr(), h * w * 3
    s.world_row_of_env, s.world_n_rows = wmap.data_ptr(), B
    s.world_rgb, s.world_rgb_row_stride = wrgb.data_ptr(), per
    for k, v in kw.items():
      setattr(s, k, v)
    return s

  def refused(s, match, out=None, flags=None, bank=None):
    torch.cuda.synchronize()
    state = eng.save_state()
    before = [t.clone() for t in (prgb, wrgb, rew, eng.world_rgb)]
    n = eng.launch_count()
    if flags is not None:
      eng.set_flags(flags)
    r = engine.MpRequest(actions=a.data_ptr(), players=ctypes.pointer(s))
    if out is not None:
      r.out = ctypes.pointer(out)
    if bank is not None:
      r.slot_of_env, r.bank, r.n_slots = bank[0].data_ptr(), bank[1].data_ptr(), 4
    rc = lib.mp_run(eng._h, ctypes.byref(r), stream)  # pylint: disable=protected-access
    eng.set_flags(engine.MP_FLAG_DEFAULT)
    assert rc == -1, (match, rc)
    assert match in lib.mp_last_error().decode(), (match, lib.mp_last_error())
    torch.cuda.synchronize()
    assert eng.launch_count() == n, match
    assert eng.save_state() == state, match
    for x, y in zip(before, (prgb, wrgb, rew, eng.world_rgb)):
      assert torch.equal(x, y), match

  # accepted as a control: the struct above is a valid call
  eng.step(a, players={'row_of_player': rmap, 'rgb': prgb.view(B * P, h, w, 3), 'world_row_of_env': wmap,
                       'world_rgb': wrgb[:B * per].view(B, H, W, 3)})
  wrgb.fill_(0xA5); prgb.fill_(0xA5)
  refused(struct(world_row_of_env=None), 'go together')
  refused(struct(world_rgb=None), 'go together')
  refused(struct(world_n_rows=0), 'world_n_rows')
  refused(struct(world_row_of_env=wmap.data_ptr() + 2), '4-byte')
  cudart = _cudart()
  ptr = ctypes.c_void_p()
  assert cudart.cudaMalloc(ctypes.byref(ptr), ctypes.c_size_t(1 << 20)) == 0
  try:  # a row map whose B i32 run past the end of its allocation
    refused(struct(world_row_of_env=ptr.value + (1 << 20) - 16), 'past the end')
  finally:
    cudart.cudaFree(ptr)
  host = torch.zeros(B, dtype=torch.int32).pin_memory()
  refused(struct(world_row_of_env=host.data_ptr()), 'not device memory')
  refused(struct(world_rgb=wrgb.data_ptr() + 8), 'multiple of 16')
  refused(struct(world_rgb_row_stride=per + 8), 'multiple of 16')
  refused(struct(world_rgb_row_stride=per - 16), 'smaller than one row')
  refused(struct(), 'switch WORLD.RGB off', flags=engine.MP_FLAG_RENDER_PLAYERS)
  o = engine.MpDeviceOutputs(); o.world_rgb, o.world_rgb_env_stride = wrgb.data_ptr(), per
  refused(struct(), 'both routed', out=o)
  refused(struct(world_rgb=prgb.data_ptr()), 'overlap')  # the world rows overlap the player rows
  refused(struct(world_row_of_env=wrgb.data_ptr()), 'overlap')  # the map overlaps the world rows
  refused(struct(world_row_of_env=rmap.data_ptr()), 'overlap')  # the map overlaps the player map
  refused(struct(world_rgb=eng.world_rgb.data_ptr()), "engine's own buffers")
  refused(struct(world_row_of_env=eng.reward.data_ptr()), "engine's own buffers")
  o = engine.MpDeviceOutputs(); o.reward, o.reward_env_stride = wrgb.data_ptr(), P * 8
  refused(struct(), 'overlap', out=o)  # out's reward overlaps the world rows
  both = torch.zeros((4 * eng.state_record_bytes + per,), dtype=torch.uint8, device='cuda')  # a bank, then room for a row
  bank = both[:4 * eng.state_record_bytes].view(4, -1)
  idx = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  refused(struct(world_rgb=bank.data_ptr(), world_n_rows=1), 'overlap', bank=(idx, bank))
  refused(struct(world_row_of_env=idx.data_ptr()), 'overlap', bank=(idx, bank))
  # a routed call's action rows
  rows = engine.MpPlayerActions(); rows.row_of_player, rows.n_rows, rows.action, rows.action_row_stride = rmap.data_ptr(), B * P, wrgb.data_ptr(), 4
  state, n = eng.save_state(), eng.launch_count()
  r = engine.MpRequest(player_actions=ctypes.pointer(rows), players=ctypes.pointer(struct()))
  assert lib.mp_run(eng._h, ctypes.byref(r), stream) == -1  # pylint: disable=protected-access
  assert 'overlap' in lib.mp_last_error().decode() and eng.launch_count() == n and eng.save_state() == state
  # the Python layer refuses before any call on a batch without WORLD.RGB
  from meltingpot_b200 import substrate
  env = substrate.BatchedSubstrate(blob, 4, seed=1, world_rgb=False)
  with pytest.raises(ValueError, match='world_rgb=False'):
    env.player_routes(np.zeros((4, P), np.int64)).outputs(world_envs=[1])


def test_batched_scenario_world_envs():
  import torch
  from meltingpot_b200 import scenario, substrate
  blob, B = _blob('clean_up'), 11
  P = 7
  is_focal = [p % 2 == 0 for p in range(P)]
  n_bg = P - sum(is_focal)

  def policy(seed):
    rng = np.random.default_rng(seed)
    return lambda ts: torch.from_numpy(rng.integers(0, 9, (B, n_bg)).astype(np.int32)).cuda()

  envs = [9, 4, 10, 1]
  permitted = {'RGB', 'WORLD.RGB', 'READY_TO_SHOOT'}
  routed = scenario.BatchedScenario(substrate.BatchedSubstrate(blob, B, seed=3), policy(0), is_focal, permitted,
                                    world_envs=envs)
  dense = scenario.BatchedScenario(substrate.BatchedSubstrate(blob, B, seed=3), policy(0), is_focal, permitted)
  ta, tb = routed.reset(), dense.reset()
  rng = np.random.default_rng(1)
  idx = torch.tensor(envs, device='cuda')
  for t in range(46):
    if t:
      a = torch.from_numpy(rng.integers(0, 9, (B, sum(is_focal))).astype(np.int32)).cuda()
      ta, tb = routed.step(a), dense.step(a)
    assert ta.observation['WORLD.RGB'].shape == (len(envs),) + tuple(tb.observation['WORLD.RGB'].shape[1:])
    assert torch.equal(ta.observation['WORLD.RGB'], tb.observation['WORLD.RGB'][idx]), t
    assert torch.equal(ta.observation['RGB'], tb.observation['RGB']) and torch.equal(ta.reward, tb.reward), t
    assert torch.equal(routed.background_timestep.observation['WORLD.RGB'], ta.observation['WORLD.RGB']), t
  no_world = substrate.BatchedSubstrate(blob, B, seed=3, world_rgb=False)
  with pytest.raises(ValueError, match='world_rgb=False'):
    scenario.BatchedScenario(no_world, policy(0), is_focal, permitted, world_envs=envs)
