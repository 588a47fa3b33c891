"""Per-player delivery to caller-chosen rows (mp_run's players, Engine.step(players=),
BatchedSubstrate.player_routes).

Each run steps a routed engine beside a lockstep twin built with the same seed and fed the same actions. Every routed
row must equal the twin's (b, p) image, reward and scalar observations byte for byte. Every other byte of the targets
(unrouted rows, row padding) and the routed engine's own rgb must keep a sentinel. WORLD.RGB, discount and step type
stay per env and must equal the twin's. Runs use the hard_cap_40 variants of tests/variants.py, so every rollout
crosses an auto-reset.
"""

import ctypes

import numpy as np
import pytest

from tests import coins_draws as CD
from tests import env_variants as EV
from tests.test_gpu_step_into import _SENT, _acts, _blob, _cudart, _sms

pytestmark = pytest.mark.gpu

FAMILIES = ['clean_up', 'commons_harvest', 'territory', 'coins', 'coop_mining', 'territory__inside_out']
STEPS = 44
PAD = 16  # bytes of padding behind every image row, 8 behind every scalar row


class _Rows:
  """Sentinel-filled per-player targets of `n_rows` padded rows for `eng`."""

  def __init__(self, eng, n_rows):
    import torch
    self.n_rows = n_rows
    h, w = eng.rgb.shape[2:4]
    per = h * w * 3
    self.rgb_raw = torch.full((n_rows * (per + PAD),), _SENT['u8'], dtype=torch.uint8, device='cuda')
    self.rgb = torch.as_strided(self.rgb_raw, (n_rows, h, w, 3), (per + PAD, w * 3, 3, 1))
    self.reward_raw = torch.full((2 * n_rows,), _SENT['f64'], dtype=torch.float64, device='cuda')
    self.reward = self.reward_raw[::2]
    n = max(eng.num_scalar_obs, 1)
    self.scalar_raw = torch.full((n, 2 * n_rows + 1), _SENT['f64'], dtype=torch.float64, device='cuda')
    self.scalar_obs = self.scalar_raw[:eng.num_scalar_obs, :2 * n_rows:2] if eng.num_scalar_obs else None

  def refill(self):
    for t in (self.rgb_raw, self.reward_raw, self.scalar_raw):
      t.view(torch_u8()).fill_(0xA5)  # (a byte view: the f64 sentinel is 0xA5 in every byte)

  def players(self, row_map):
    out = {'row_of_player': row_map, 'rgb': self.rgb, 'reward': self.reward}
    if self.scalar_obs is not None:
      out['scalar_obs'] = self.scalar_obs
    return out

  def check(self, twin, row_map, where):
    """Routed rows equal the twin's (b, p); then, with those rows set back to the sentinel, every byte is the sentinel."""
    import torch
    bs, ps = torch.nonzero(row_map >= 0, as_tuple=True)
    rows = row_map[bs, ps].long()
    assert torch.equal(self.rgb[rows], twin.rgb[bs, ps]), f'rgb {where}'
    assert torch.equal(self.reward[rows].view(torch.int64), twin.reward[bs, ps].view(torch.int64)), f'reward {where}'
    if self.scalar_obs is not None:
      want = twin.scalar_obs[:twin.num_scalar_obs][:, bs, ps]
      assert torch.equal(self.scalar_obs[:, rows].view(torch.int64), want.view(torch.int64)), f'scalar_obs {where}'
      self.scalar_obs[:, rows] = _SENT['f64']
    self.rgb[rows] = _SENT['u8']
    self.reward[rows] = _SENT['f64']
    for name, t in (('rgb', self.rgb_raw), ('reward', self.reward_raw), ('scalar_obs', self.scalar_raw)):
      assert bool((t.view(torch.uint8) == 0xA5).all()), f'{name} {where}: bytes outside the routed rows were written'


def torch_u8():
  import torch
  return torch.uint8


def _row_map(kind, B, P, n_rows, rng):
  """int32 CUDA [B, P]: identity (row b * P + p), permuted (a random injection into n_rows rows) or partial (about half
  the players, permuted, the rest -1)."""
  import torch
  if kind == 'identity':
    m = np.arange(B * P, dtype=np.int32)
  else:
    m = rng.permutation(n_rows)[:B * P].astype(np.int32)
    if kind == 'partial':
      keep = m[0]
      m[rng.random(B * P) < 0.5] = -1
      if (m < 0).all():
        m[0] = keep
  return torch.from_numpy(m.reshape(B, P)).cuda()


def _same_per_env(a, b, where):
  import torch
  for name in ('world_rgb', 'discount', 'step_type', 'avatar_state', 'grid', 'event_count'):
    assert torch.equal(getattr(a, name), getattr(b, name)), f'{name} {where}'


def _lockstep(blob, B, kind, seed=11, steps=STEPS, env_variant=None, blobs=None):
  import torch
  from meltingpot_b200 import engine
  src = blobs if blobs is not None else blob
  kw = dict(seed=seed, env_variant=env_variant)
  twin, eng = engine.Engine(src, B, **kw), engine.Engine(src, B, **kw)
  P = eng.num_players
  n_rows = B * P + 3
  tg = _Rows(eng, n_rows)
  eng.rgb.fill_(0xA5)
  rng = np.random.default_rng(B * 7 + len(kind))
  mask = torch.zeros(B, dtype=torch.uint8, device='cuda'); mask[::3] = 1
  for t in range(steps + 1):
    rmap = _row_map(kind, B, P, n_rows, rng)  # a new map every step: it takes effect at that step
    tg.refill()
    if t == 0 or t == steps // 2:
      m = None if t == 0 else mask
      twin.reset(m)
      eng.reset(m, players=tg.players(rmap))
    else:
      a = _acts(rng, eng)
      twin.step(a)
      eng.step(a, players=tg.players(rmap))
    where = f'{kind} B={B} t={t}'
    tg.check(twin, rmap, where)
    _same_per_env(eng, twin, where)
    assert bool((eng.rgb == 0xA5).all()), f'own rgb written {where}'
  return twin, eng


@pytest.mark.parametrize('kind', ['identity', 'permuted', 'partial'])
@pytest.mark.parametrize('fam', FAMILIES)
def test_routed_rows_equal_the_twin(fam, kind):
  sms = _sms()
  blob = _blob(fam)
  for B in (1, 7, sms - 1, sms + 1, 2 * sms + 5):
    _lockstep(blob, B, kind)


def test_routed_rows_equal_the_oracle(oracle):
  import torch
  from meltingpot_b200 import engine
  blob, B, seed = _blob('clean_up'), 5, 3
  eng = engine.Engine(blob, B, seed=seed)
  P = eng.num_players
  envs = [oracle.OracleEnv(blob, seed + b) for b in range(B)]
  tg = _Rows(eng, B * P)
  rng = np.random.default_rng(0)
  eng.reset(players=tg.players(_row_map('partial', B, P, B * P, rng)))
  for e in envs:
    e.reset()
  for t in range(45):
    rmap = _row_map('partial', B, P, B * P, rng)
    tg.refill()
    a = _acts(rng, eng)
    eng.step(a, players=tg.players(rmap))
    acts = a.cpu().numpy()
    torch.cuda.synchronize()
    rm = rmap.cpu().numpy()
    rgb, reward = tg.rgb.cpu().numpy(), tg.reward.cpu().numpy()
    for b, e in enumerate(envs):
      e.step(acts[b])
      want_rgb, want_r = e.rgb(), e.rewards()
      for p in range(P):
        if rm[b, p] >= 0:
          assert np.array_equal(rgb[rm[b, p]], want_rgb[p]), (t, b, p)
          assert reward[rm[b, p]] == want_r[p], (t, b, p)
    assert np.array_equal(eng.world_rgb.cpu().numpy(), np.stack([e.world_rgb() for e in envs])), t


def test_restore_composes_with_routing():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('commons_harvest'), 37
  twin, eng = engine.Engine(blob, B, seed=5), engine.Engine(blob, B, seed=5)
  P = eng.num_players
  tg = _Rows(eng, B * P)
  rng = np.random.default_rng(1)
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
      rekey = t % 2 == 0
      rmap = _row_map('partial', B, P, B * P, rng)
      tg.refill()
      twin.step(a, restore=idx, bank=bank_t, rekey=rekey)
      eng.step(a, restore=idx, bank=bank_e, rekey=rekey, players=tg.players(rmap))
      tg.check(twin, rmap, f'restore t={t}')
    else:
      twin.step(a); eng.step(a)
    _same_per_env(eng, twin, f'restore t={t}')


@pytest.mark.parametrize('family', ['clean_up', 'coins'])
def test_variant_engines_and_coins_draws(family):
  blobs = list(EV.blobs(family)) if family == 'clean_up' else list(CD.draw_set())
  B = 2 * _sms() + 5
  assign = (np.arange(B) % len(blobs)).astype(np.int64)
  _lockstep(None, B, 'permuted', blobs=blobs, env_variant=assign, steps=45)


def test_routing_into_out_and_trajectory_slots():
  # players= with out=: WORLD.RGB and the per-env scalars go to out, the images to the rows
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('territory'), 19
  twin, eng = engine.Engine(blob, B, seed=2), engine.Engine(blob, B, seed=2)
  P = eng.num_players
  tg = _Rows(eng, B * P)
  out = {'world_rgb': torch.full_like(eng.world_rgb, 0xA5), 'discount': torch.zeros_like(eng.discount),
         'step_type': torch.zeros_like(eng.step_type), 'reward': torch.zeros_like(eng.reward)}
  rng = np.random.default_rng(4)
  twin.reset(); eng.reset(out=None, players=tg.players(_row_map('identity', B, P, B * P, rng)))
  for t in range(45):
    a = _acts(rng, eng)
    rmap = _row_map('permuted', B, P, B * P, rng)
    tg.refill()
    twin.step(a)
    eng.step(a, out=out, players=tg.players(rmap))
    tg.check(twin, rmap, f't={t}')
    for name in out:
      assert torch.equal(out[name], getattr(twin, name)), f'{name} t={t}'
  with pytest.raises(ValueError, match='both routed'):
    eng.step(_acts(rng, eng), out={'rgb': torch.zeros_like(eng.rgb)}, players=tg.players(rmap))


def test_batched_substrate_player_routes():
  import torch
  from meltingpot_b200 import substrate
  blob, B = _blob('clean_up'), 9
  twin = substrate.BatchedSubstrate(blob, B, seed=4)
  env = substrate.BatchedSubstrate(blob, B, seed=4)
  P = env.num_players
  rng = np.random.default_rng(2)
  groups = rng.integers(-1, 3, size=(B, P))
  routes = env.player_routes(groups)
  traj = routes.outputs(T=45)
  ts = env.reset(players=traj.at(0))
  twin.reset()
  assert 'RGB' not in ts.observation and 'WORLD.RGB' in ts.observation
  for t in range(1, 45):
    a = torch.from_numpy(rng.integers(0, env.num_actions, (B, P)).astype(np.int32)).cuda()
    ts = env.step(a, players=traj.at(t))
    want = twin.step(a)
    assert torch.equal(ts.step_type, want.step_type) and torch.equal(ts.observation['WORLD.RGB'], want.observation['WORLD.RGB'])
    e, p = routes.env_of_row, routes.player_of_row
    assert torch.equal(traj['RGB'][t], want.observation['RGB'][e, p]), t
    assert torch.equal(traj['REWARD'][t], want.reward[e, p]), t
    assert torch.equal(traj['READY_TO_SHOOT'][t], want.observation['READY_TO_SHOOT'][e, p]), t
  for g in range(routes.num_groups):
    sl = routes.rows(g)
    assert bool((torch.from_numpy(groups).cuda()[routes.env_of_row[sl], routes.player_of_row[sl]] == g).all())


def test_launch_count_equals_step_into():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 16
  eng = engine.Engine(blob, B, seed=1)
  P = eng.num_players
  tg = _Rows(eng, B * P)
  rmap = _row_map('partial', B, P, B * P, np.random.default_rng(0))
  out = {'reward': torch.zeros_like(eng.reward)}
  eng.reset()
  a = torch.zeros((B, P), dtype=torch.int32, device='cuda')

  def added(fn):
    n = eng.launch_count(); fn(); return eng.launch_count() - n

  assert added(lambda: eng.step(a, players=tg.players(rmap))) == added(lambda: eng.step(a, out=out))
  assert added(lambda: eng.reset(players=tg.players(rmap))) == added(lambda: eng.reset(out=out))
  # rendering off: the routed scalars travel by one small kernel
  eng.set_flags(0)
  scal = {'row_of_player': rmap, 'reward': tg.reward}
  assert added(lambda: eng.step(a, players=scal)) == added(lambda: eng.step(a, out=out)) + 1


def test_refused_calls_change_nothing():
  import torch
  from meltingpot_b200 import engine
  blob, B = _blob('clean_up'), 12
  eng = engine.Engine(blob, B, seed=1)
  P, h, w = eng.num_players, eng.rgb.shape[2], eng.rgb.shape[3]
  lib = engine.load_library()
  eng.reset()
  a = torch.zeros((B, P), dtype=torch.int32, device='cuda')
  rmap = torch.arange(B * P, dtype=torch.int32, device='cuda').view(B, P)
  big = torch.full((B * P * h * w * 3 + 4096,), 0xA5, dtype=torch.uint8, device='cuda')
  rew = torch.full((4 * B * P,), 1.5, dtype=torch.float64, device='cuda')
  scal = torch.full((2, 4 * B * P), 1.5, dtype=torch.float64, device='cuda')
  stream = ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)

  def struct(**kw):
    s = engine.MpPlayerOutputs()
    s.row_of_player, s.n_rows = rmap.data_ptr(), B * P
    s.rgb, s.rgb_row_stride = big.data_ptr(), h * w * 3
    for k, v in kw.items():
      setattr(s, k, v)
    return s

  def refused(s, match, out=None, flags=None, code=-1):
    torch.cuda.synchronize()
    before = [t.clone() for t in (eng.avatar_state, eng.grid, eng.step_type, eng.reward, big, rew)]
    n = eng.launch_count()
    if flags is not None:
      eng.set_flags(flags)
    r = engine.MpRequest(actions=a.data_ptr(), players=ctypes.pointer(s))
    if out is not None:
      r.out = ctypes.pointer(out)
    rc = lib.mp_run(eng._h, ctypes.byref(r), stream)  # pylint: disable=protected-access
    eng.set_flags(engine.MP_FLAG_DEFAULT)
    assert rc == code, (match, rc)
    assert match in lib.mp_last_error().decode(), (match, lib.mp_last_error())
    torch.cuda.synchronize()
    assert eng.launch_count() == n
    for x, y in zip(before, (eng.avatar_state, eng.grid, eng.step_type, eng.reward, big, rew)):
      assert torch.equal(x, y), match

  refused(struct(n_rows=0), 'n_rows')
  refused(struct(row_of_player=rmap.data_ptr() + 2), 'row_of_player')
  cudart = _cudart()
  ptr = ctypes.c_void_p()
  assert cudart.cudaMalloc(ctypes.byref(ptr), ctypes.c_size_t(1 << 20)) == 0
  try:  # a row map whose B * P i32 run past the end of its allocation
    refused(struct(row_of_player=ptr.value + (1 << 20) - 16), 'past the end')
  finally:
    cudart.cudaFree(ptr)
  refused(struct(), 'switch the player images off', flags=engine.MP_FLAG_RENDER_WORLD)
  o = engine.MpDeviceOutputs(); o.rgb, o.rgb_env_stride = big.data_ptr(), P * h * w * 3
  refused(struct(rgb=big.data_ptr()), 'both routed', out=o)
  refused(struct(rgb=big.data_ptr() + 8), 'multiple of 16')
  refused(struct(rgb_row_stride=h * w * 3 + 8), 'multiple of 16')
  refused(struct(rgb_row_stride=h * w * 3 - 16), 'smaller than one row')
  refused(struct(reward=rew.data_ptr() + 4, reward_row_stride=8), 'multiple of 8')
  refused(struct(reward=rew.data_ptr(), reward_row_stride=4), 'multiple of 8')
  refused(struct(reward=rew.data_ptr(), reward_row_stride=1 << 31), '2 GiB')
  refused(struct(scalar_obs=scal.data_ptr(), scalar_obs_row_stride=8, scalar_obs_stride=8), 'rows overlap')
  refused(struct(scalar_obs=scal.data_ptr(), scalar_obs_row_stride=8, scalar_obs_stride=12), 'multiple of 8')
  refused(struct(reward=big.data_ptr(), reward_row_stride=8), 'overlap')
  refused(struct(reward=rmap.data_ptr(), reward_row_stride=8, rgb=None), 'overlap')
  refused(struct(rgb=eng.rgb.data_ptr()), "engine's own buffers")
  refused(struct(reward=rew.data_ptr(), reward_row_stride=8, rgb=None), 'overlap',
          out=(lambda o: (setattr(o, 'reward', rew.data_ptr()), setattr(o, 'reward_env_stride', P * 8), o)[-1])(engine.MpDeviceOutputs()))
  # a bank that overlaps a routed target
  bank = torch.zeros((4, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  idx = torch.full((B,), -1, dtype=torch.int32, device='cuda')
  s = struct(reward=bank.data_ptr(), reward_row_stride=8, rgb=None)
  r = engine.MpRequest(actions=a.data_ptr(), slot_of_env=idx.data_ptr(), bank=bank.data_ptr(), n_slots=4, players=ctypes.pointer(s))
  assert lib.mp_run(eng._h, ctypes.byref(r), stream) == -1  # pylint: disable=protected-access
  assert 'overlap' in lib.mp_last_error().decode()


def test_gather_refused_and_exchange_accepted(clean_up_blob):
  import torch
  from meltingpot_b200 import engine
  B = 40
  eng = engine.Engine(clean_up_blob, B, seed=5)
  P = eng.num_players
  tg = _Rows(eng, B * P)
  rmap = _row_map('identity', B, P, B * P, np.random.default_rng(0))
  ptr, _ = eng.gather_obs_create(0, 1)
  eng.gather_obs_connect([ptr])
  eng.reset()
  a = torch.zeros((B, P), dtype=torch.int32, device='cuda')
  n = eng.launch_count()
  with pytest.raises(ValueError, match='-2.*gather'):
    eng.step(a, players=tg.players(rmap))
  assert eng.launch_count() == n
  eng.gather_obs_enable(False)
  eng.step(a, players=tg.players(rmap))  # switched off: accepted
  eng.close()
  # the timestep exchange: accepted, and the step is published like any other
  twin = engine.Engine(clean_up_blob, B, seed=5)
  eng = engine.Engine(clean_up_blob, B, seed=5)
  ptr, _ = eng.exchange_create(0, 1)
  eng.exchange_connect([ptr])
  twin.reset(); eng.reset()
  eng.exchange_wait()
  rng = np.random.default_rng(3)
  for t in range(45):
    a = _acts(rng, eng)
    rmap = _row_map('partial', B, P, B * P, rng)
    tg.refill()
    twin.step(a)
    eng.step(a, players=tg.players(rmap))
    eng.exchange_wait()
    torch.cuda.synchronize()
    assert eng.exchange_slot()[1] == t + 2
    assert torch.equal(eng.gathered_timestep(), twin.timestep_packed), t
    tg.check(twin, rmap, f'exchange t={t}')
