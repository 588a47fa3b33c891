"""GPU test: per-player rows delivered through row segments (mp_player_outputs.segments) equal, byte for byte, the same
request with one target, on every kernel family and in every mode a routed step composes with; refused segment tables
change nothing; BatchedScenario.trajectory equals stacking a twin scenario's timesteps."""

import numpy as np
import pytest

from tests import env_variants as EV
from tests.test_gpu_step_into import _SENT, _acts, _blob, _sms

pytestmark = pytest.mark.gpu

FAMILIES = ['clean_up', 'commons_harvest', 'territory', 'coins', 'coop_mining']
STEPS = 44  # > the 40-frame cap of the test blobs: every env crosses an auto-reset
PAD = 16


class _Seg:
  """Sentinel-filled targets of rows [begin, end), padded behind every row."""

  def __init__(self, eng, begin, end, scalars_only=False):
    import torch
    self.begin, self.end, self.scalars_only = begin, end, scalars_only
    n = end - begin
    h, w = eng.rgb.shape[2:4]
    per = h * w * 3
    self.rgb_raw = torch.full((n * (per + PAD),), _SENT['u8'], dtype=torch.uint8, device='cuda')
    self.rgb = torch.as_strided(self.rgb_raw, (n, h, w, 3), (per + PAD, w * 3, 3, 1))
    self.reward_raw = torch.full((3 * n,), _SENT['f64'], dtype=torch.float64, device='cuda')
    self.reward = self.reward_raw[::3]
    k = max(eng.num_scalar_obs, 1)
    self.scalar_raw = torch.full((k, 2 * n + 1), _SENT['f64'], dtype=torch.float64, device='cuda')
    self.scalar_obs = self.scalar_raw[:eng.num_scalar_obs, :2 * n:2] if eng.num_scalar_obs else None

  def targets(self):
    t = {'reward': self.reward} if self.scalars_only else {'rgb': self.rgb, 'reward': self.reward}
    if self.scalar_obs is not None:
      t['scalar_obs'] = self.scalar_obs
    return (self.begin, self.end, t)

  def refill(self):
    import torch
    for t in (self.rgb_raw, self.reward_raw, self.scalar_raw):
      t.view(torch.uint8).fill_(0xA5)

  def check(self, one, where):
    """Rows equal those of the one-target request `one` (a _Seg over every row); the padding stays the sentinel."""
    import torch
    r = slice(self.begin, self.end)
    assert torch.equal(self.rgb, one.rgb[r]), f'rgb {where}'
    assert torch.equal(self.reward.view(torch.int64), one.reward[r].view(torch.int64)), f'reward {where}'
    if self.scalar_obs is not None:
      assert torch.equal(self.scalar_obs.view(torch.int64), one.scalar_obs[:, r].view(torch.int64)), f'scalar_obs {where}'
    self.rgb.fill_(_SENT['u8']); self.reward.fill_(_SENT['f64'])
    if self.scalar_obs is not None:
      self.scalar_obs.fill_(_SENT['f64'])
    for name, t in (('rgb', self.rgb_raw), ('reward', self.reward_raw), ('scalar_obs', self.scalar_raw)):
      assert bool((t.view(torch.uint8) == 0xA5).all()), f'{name} {where}: padding written'


def _bounds(n_rows):
  """Three segments with a gap before, between and after them: rows in no segment are left undelivered."""
  a, b, c = n_rows // 5, n_rows // 2, (4 * n_rows) // 5
  return [(1, a), (a + 3, b), (b, c)]


def _lockstep(blob, B, *, seed=5, steps=STEPS, drawn=False, world=False, restore=False, env_variant=None, flags=None):
  """Two engines: `one` delivers every row of the request to one target, `seg` the same request through row
  segments; the segments' rows equal `one`'s at every step and nothing else is written."""
  import torch
  from meltingpot_b200 import engine
  kw = dict(seed=seed, env_variant=env_variant)
  if flags is not None:
    kw['flags'] = flags
  one_eng, seg_eng = engine.Engine(blob, B, **kw), engine.Engine(blob, B, **kw)
  P = one_eng.num_players
  rng = np.random.default_rng(B + 3 * drawn + 5 * world)
  if drawn:
    choices = [[p % 3, (p + 1) % 3] for p in range(P)]
    n_g = [sum(g in c for c in choices) for g in range(3)]
    starts = np.concatenate([[0], np.cumsum([B * n for n in n_g])])
    base = [[int(starts[g]) + [p for p in range(P) if g in choices[p]].index(p) for g in c] for p, c in enumerate(choices)]
    per_env = [[n_g[g] for g in c] for c in choices]
    n_rows = int(starts[-1])
    maps = [torch.full((B, P), -1, dtype=torch.int32, device='cuda') for _ in range(2)]
    draws = [engine.describe_draw(m, n_rows, base, per_env) for m in maps]
    acts = torch.zeros(n_rows, dtype=torch.int32, device='cuda')
  else:
    n_rows = B * P + 2
    perm = rng.permutation(n_rows)[:B * P].astype(np.int32)
    maps = [torch.from_numpy(perm.reshape(B, P)).cuda()] * 2
  one = _Seg(one_eng, 0, n_rows, scalars_only=flags == 0)
  segs = [_Seg(seg_eng, a, b, scalars_only=flags == 0) for a, b in _bounds(n_rows)]
  wkw = [{}, {}]
  if world:
    wrows = torch.full((B,), -1, dtype=torch.int32, device='cuda'); wrows[::4] = torch.arange((B + 3) // 4, dtype=torch.int32, device='cuda')
    for k, e in enumerate((one_eng, seg_eng)):
      wkw[k] = {'world_row_of_env': wrows, 'world_rgb': torch.full(((B + 3) // 4,) + tuple(e.world_rgb.shape[1:]), 0xA5, dtype=torch.uint8, device='cuda')}
  bank = None
  if restore:
    bank = [torch.zeros((4, e.state_record_bytes), dtype=torch.uint8, device='cuda') for e in (one_eng, seg_eng)]
  mask = torch.zeros(B, dtype=torch.uint8, device='cuda'); mask[1::3] = 1
  for t in range(steps + 1):
    players = [dict(row_of_player=maps[0], **one.targets()[2], **wkw[0]),
               dict(row_of_player=maps[1], n_rows=n_rows, segments=[s.targets() for s in segs], **wkw[1])]
    common = [{}, {}]
    if drawn:
      common = [dict(draw=draws[k]) for k in range(2)]
    if t == 0 or t == steps // 2:
      m = None if t == 0 else mask
      for k, e in enumerate((one_eng, seg_eng)):
        e.reset(m, players=players[k], **common[k])
    else:
      a = _acts(rng, one_eng)
      rkw = [{}, {}]
      if restore and t == 10:
        for k, e in enumerate((one_eng, seg_eng)):
          e.store_states(bank[k], torch.tensor([0, 3, -1, -1], dtype=torch.int32, device='cuda'))
      if restore and t > 10 and t % 5 == 0:
        idx = torch.full((B,), -1, dtype=torch.int32, device='cuda'); idx[t % B] = t % 2; idx[(3 * t) % B] = 1 - t % 2
        rkw = [dict(restore=idx, bank=bank[k]) for k in range(2)]
      for k, e in enumerate((one_eng, seg_eng)):
        if drawn:
          acts.copy_(torch.from_numpy(rng.integers(0, e.num_actions, n_rows).astype(np.int32)).cuda() if k == 0 else acts)
          e.step(None, players=players[k], player_actions={'row_of_player': maps[k], 'action': acts}, **common[k], **rkw[k])
        else:
          e.step(a, players=players[k], **rkw[k])
    where = f'B={B} t={t} drawn={drawn} world={world} restore={restore}'
    if drawn:
      assert torch.equal(maps[0], maps[1]), f'row maps {where}'
    for s in segs:
      s.check(one, where)
    one.refill()
    for name in ('discount', 'step_type', 'avatar_state', 'grid'):
      assert torch.equal(getattr(one_eng, name), getattr(seg_eng, name)), f'{name} {where}'
    if world:
      assert torch.equal(wkw[0]['world_rgb'], wkw[1]['world_rgb']), f'world rows {where}'
    assert one_eng.last_launch() == seg_eng.last_launch(), where
    assert one_eng.launch_count() == seg_eng.launch_count(), where
  return one_eng, seg_eng


@pytest.mark.parametrize('fam', FAMILIES)
def test_segments_equal_one_target(fam):
  blob = _blob(fam)
  for B in (7, 2 * _sms() + 5):  # (the second reaches the cooperative tail of k_render)
    _lockstep(blob, B)


@pytest.mark.parametrize('fam', FAMILIES)
def test_segments_with_drawn_routes_and_world_rows(fam):
  _lockstep(_blob(fam), 2 * _sms() + 3, drawn=True, world=True)


def test_segments_with_restores_and_a_variant_engine():
  blobs = EV.blobs('clean_up')
  B = 2 * _sms() + 5
  _lockstep(list(blobs), B, restore=True, env_variant=EV.interleaved(B, len(blobs)))


def test_segments_with_rendering_off():
  one, seg = _lockstep(_blob('clean_up'), 37, flags=0, steps=12)
  assert one.last_launch()['render_mode'] == -1  # no render: k_exchange_push delivered the rows


def test_refused_segment_tables_change_nothing():
  import torch
  from meltingpot_b200 import engine
  B = 9
  eng = engine.Engine(_blob('clean_up'), B, seed=3)
  P = eng.num_players
  rmap = torch.arange(B * P, dtype=torch.int32, device='cuda').view(B, P)
  eng.reset(players={'row_of_player': rmap, 'reward': torch.zeros(B * P, dtype=torch.float64, device='cuda')})
  torch.cuda.synchronize()
  a = _Seg(eng, 0, 10)
  b = _Seg(eng, 10, 20)

  def request(segments, **extra):
    s = eng._player_outputs({'row_of_player': rmap, 'n_rows': B * P, 'segments': segments[:1]})
    s.n_segments = len(segments)
    for k, (begin, end, t) in enumerate(segments):
      g = s.segments[k]
      g.row_begin, g.row_end = begin, end
      g.rgb, g.rgb_row_stride = (t['rgb'].data_ptr(), t['rgb'].stride(0)) if 'rgb' in t else (None, 0)
      g.reward, g.reward_row_stride = (t['reward'].data_ptr(), t['reward'].stride(0) * 8) if 'reward' in t else (None, 0)
      if 'scalar_obs' in t:
        g.scalar_obs, g.scalar_obs_row_stride, g.scalar_obs_stride = t['scalar_obs'].data_ptr(), t['scalar_obs'].stride(1) * 8, t['scalar_obs'].stride(0) * 8
    for k, v in extra.items():
      setattr(s, k, v)
    return s

  import ctypes
  ta, tb = a.targets()[2], b.targets()[2]
  bad = [
      request([(0, 10, ta), (10, 20, tb)], n_segments=17),
      request([(0, 10, ta), (10, 20, tb)], n_segments=-1),
      request([(0, 10, ta), (10, 20, tb)], reward=tb['reward'].data_ptr()),
      request([(10, 20, tb), (0, 10, ta)]),                          # unsorted
      request([(0, 10, ta), (9, 19, tb)]),                           # overlapping
      request([(0, 10, ta), (12, 12, tb)]),                          # empty
      request([(0, 10, ta), (B * P - 5, B * P + 5, tb)]),            # outside [0, n_rows)
      request([(0, 10, ta), (10, 20, {'reward': tb['reward']})]),    # a different set of outputs
      request([(0, 10, ta), (10, 20, dict(tb, rgb=ta['rgb']))]),     # targets that overlap
  ]
  before = [t.clone() for t in (eng.grid, eng.avatar_state, eng.reward, a.rgb_raw, b.rgb_raw)]
  count = eng.launch_count()
  for k, s in enumerate(bad):
    r = engine.MpRequest(actions=_acts(np.random.default_rng(k), eng).data_ptr(), players=ctypes.pointer(s))
    assert eng._lib.mp_run(eng._h, ctypes.byref(r), None) == -1, f'request {k} accepted'
  torch.cuda.synchronize()
  assert eng.launch_count() == count
  for x, y in zip(before, (eng.grid, eng.avatar_state, eng.reward, a.rgb_raw, b.rgb_raw)):
    assert torch.equal(x, y)


def _scenario_pair(population, world_envs, B=23):
  from meltingpot_b200 import scenario, substrate
  import torch
  blob = _blob('clean_up')
  subs = [substrate.BatchedSubstrate(blob, B, seed=41) for _ in range(2)]
  is_focal = [True, False, True, True, False, True, False]

  def policy(name):
    def act(ts, active=None):  # per row, so that the unplayed rows of a bot (never written) do not reach the others
      n = ts.reward.shape[1]
      return (torch.nan_to_num(ts.reward).abs().clamp(max=1e3).long() + torch.arange(n, device='cuda') + len(name)) % 9
    return act

  kw = {}
  if population:
    kw = dict(roles=['default'] * 7, bots_by_role={'default': ['a', 'b']})
    pol = {'a': policy('a'), 'b': policy('b')}
  else:
    pol = policy('bg')
  permitted = ['RGB', 'READY_TO_SHOOT', 'COLLECTIVE_REWARD', 'WORLD.RGB']
  return [scenario.BatchedScenario(s, pol, is_focal, permitted, world_envs=world_envs, **kw) for s in subs]


def _same_ts(a, b, where, active=None):
  """Equal timesteps; `active` (bool [B, n]): compare per-player fields on those rows only."""
  import torch
  rows = (lambda v: v) if active is None else (lambda v: v[active])
  for f in ('step_type', 'discount'):
    assert torch.equal(getattr(a, f), getattr(b, f)), f'{f} {where}'
  assert torch.equal(rows(a.reward), rows(b.reward)), f'reward {where}'
  assert list(a.observation) == list(b.observation), where
  for k in a.observation:
    x, y = a.observation[k], b.observation[k]
    if k not in ('WORLD.RGB', 'COLLECTIVE_REWARD'):
      x, y = rows(x), rows(y)
    assert torch.equal(x, y), f'{k} {where}'


@pytest.mark.parametrize('time_major', [True, False])
@pytest.mark.parametrize('population,world_envs', [(False, None), (True, None), (False, [0, 5, 22]), (True, [3])])
def test_scenario_trajectory_equals_stacked_timesteps(population, world_envs, time_major):
  import torch
  plain, traj_sc = _scenario_pair(population, world_envs)
  T = 45
  traj = traj_sc.trajectory(T, time_major=time_major)
  rng = np.random.default_rng(7)
  want = []
  for t in range(T):
    if t == 0:
      ts, got = plain.reset(), traj_sc.reset(out=traj.at(0))
    else:
      acts = torch.from_numpy(rng.integers(0, 9, (plain.num_envs, plain.num_focal))).cuda()
      ts, got = plain.step(acts), traj_sc.step(acts, out=traj.at(t))
    where = f't={t} population={population} world={world_envs} time_major={time_major}'
    _same_ts(ts, got, where)
    want.append({'step_type': ts.step_type.clone(), 'discount': ts.discount.clone(), 'reward': ts.reward.clone(),
                 **{k: v.clone() for k, v in ts.observation.items() if k != 'WORLD.RGB' or world_envs is not None}})
    bg_a, bg_b = plain.background_timestep, traj_sc.background_timestep
    if population:
      for k, name in enumerate(plain.bot_names):
        _same_ts(bg_a[name], bg_b[name], f'background {name} {where}', active=traj_sc._routes.active(k + 1))
    else:
      _same_ts(bg_a, bg_b, f'background {where}')
  assert any(bool((w['step_type'] == 0).any()) for w in want[1:]), 'no episode start after the first within T'
  for t, w in enumerate(want):
    slot = traj.at(t)
    for k, v in w.items():
      got = getattr(slot, k) if k in ('step_type', 'discount', 'reward') else slot.observation[k]
      assert torch.equal(got, v), f'slot {t} {k}'
