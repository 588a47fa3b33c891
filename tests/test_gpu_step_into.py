"""Steps and resets into caller-owned device tensors (mp_run's out, Engine.step(out=),
BatchedSubstrate.trajectory).

An engine that steps into a trajectory buffer must give, slot for slot and byte for byte, what an engine stepped plainly
with the same seed and actions holds in its own buffers, and must write nothing else: each trajectory tensor is
pre-filled with a sentinel and has padded env strides, and padding bytes and slots not yet written keep the sentinel.
Runs use the hard_cap_40 variants of tests/variants.py, so every rollout crosses an auto-reset.
"""

import ctypes
import ctypes.util
import glob
import os
import struct

import numpy as np
import pytest

from tests import parity
from tests import variants as V

pytestmark = pytest.mark.gpu

FAMILIES = ['clean_up', 'commons_harvest', 'territory', 'coins', 'coop_mining']
THREADS = os.cpu_count() or 1
STEPS = 48
_SENT = {'u8': 0xA5, 'f64': struct.unpack('<d', b'\xa5' * 8)[0], 'i64': int.from_bytes(b'\xa5' * 8, 'little', signed=True)}


def _blob(fam):
  if fam == 'territory__inside_out':
    from tests.test_gpu_entry_points import _inside_out_cap40
    return _inside_out_cap40()
  return V.compile(f'{fam}/hard_cap_40')


def _sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _acts(rng, eng):
  import torch
  return torch.from_numpy(np.ascontiguousarray(rng.integers(0, eng.num_actions, size=(eng.num_envs, eng.num_players)), np.int32)).cuda()


class _Traj:
  """One padded [T, B, ...] trajectory tensor per output of `eng` (indexed time first whatever the physical layout),
  each over a raw buffer pre-filled with the sentinel."""

  def __init__(self, eng, T, time_major, pad, names):
    import torch
    self.raw, self.view, self.sent = {}, {}, {}
    B = eng.num_envs
    for name in names:
      shape, dtype = eng.output_views()[name]
      kind = {torch.uint8: 'u8', torch.float64: 'f64', torch.int64: 'i64'}[dtype]
      es = torch.empty((), dtype=dtype).element_size()
      n = 1
      if name == 'scalar_obs':
        n, shape = eng.num_scalar_obs, shape[1:]
      inner = shape[1:]
      E = int(np.prod(inner, dtype=np.int64)) if inner else 1
      p = pad // es
      if time_major:
        env_s = E + p
        time_s = B * env_s
        total = T * time_s
      else:
        env_s = T * E + p
        time_s = E
        total = B * env_s
      dense = [int(np.prod(inner[i + 1:], dtype=np.int64)) for i in range(len(inner))]
      raw = torch.full((n * total,), _SENT[kind], dtype=dtype, device='cuda')
      if name == 'scalar_obs':
        v = torch.as_strided(raw, (T, n, B) + tuple(inner), (time_s, total, env_s) + tuple(dense))
      else:
        v = torch.as_strided(raw, (T, B) + tuple(inner), (time_s, env_s) + tuple(dense))
      self.raw[name], self.view[name], self.sent[name] = raw, v, _SENT[kind]

  def at(self, t):
    return {k: v[t] for k, v in self.view.items()}

  def untouched(self, t):
    return all(bool((v[t] == self.sent[k]).all()) for k, v in self.view.items())

  def only_slots_written(self, slots):
    """Overwrites the given slots with the sentinel; every byte of every raw buffer must then be the sentinel."""
    import torch
    for k, v in self.view.items():
      for t in slots:
        v[t].fill_(self.sent[k])
      assert bool((self.raw[k].view(torch.uint8) == 0xA5).all()), f'{k}: bytes outside the written slots were changed'


def _own(eng, name):
  v = getattr(eng, name)
  return v[:eng.num_scalar_obs] if name == 'scalar_obs' else v


def _names(eng, flags=None):
  from meltingpot_b200 import engine
  flags = engine.MP_FLAG_DEFAULT if flags is None else flags
  out = ['reward', 'discount', 'step_type']
  if eng.num_scalar_obs:
    out.append('scalar_obs')
  if flags & engine.MP_FLAG_RENDER_PLAYERS:
    out.append('rgb')
  if flags & engine.MP_FLAG_RENDER_WORLD:
    out.append('world_rgb')
  return out


def _run(blob, B, ops, seed, time_major, pad, names=None, flags=None, env_variant=None, on_slot=None):
  """Runs `ops` (('reset', mask or None) or ('step', actions)) on a plain engine and on one stepping into a trajectory,
  slot t = op t. After each op, slot t must equal the plain engine's outputs and slot t + 1 must be untouched; at the
  end every byte outside the written slots must still be the sentinel. Returns (plain, into, traj)."""
  import torch
  from meltingpot_b200 import engine
  kw = dict(seed=seed, env_variant=env_variant)
  if flags is not None:
    kw['flags'] = flags
  plain, into = engine.Engine(blob, B, **kw), engine.Engine(blob, B, **kw)
  names = _names(into, flags) if names is None else names
  traj = _Traj(into, len(ops), time_major, pad, names)
  for t, (kind, arg) in enumerate(ops):
    if kind == 'reset':
      plain.reset(arg)
      into.reset(arg, out=traj.at(t))
    else:
      plain.step(arg)
      into.step(arg, out=traj.at(t))
    want = parity.device_outputs(plain, kinds=())
    for name in names:
      if name in ('rgb', 'world_rgb'):
        assert torch.equal(traj.view[name][t], getattr(plain, name)), f'{name} slot {t} (B={B}, time_major={time_major})'
      else:
        np.testing.assert_array_equal(traj.view[name][t].cpu().numpy(), want[name], err_msg=f'{name} slot {t} (B={B})')
    for name in parity._STATE_VIEWS:  # pylint: disable=protected-access
      assert torch.equal(getattr(into, name), getattr(plain, name)), f'engine {name} after op {t}'
    if t + 1 < len(ops):
      assert traj.untouched(t + 1), f'slot {t + 1} written before its step'
    if on_slot is not None:
      on_slot(t, plain, into, traj)
  return plain, into, traj


def _script(eng_like, B, P, A, steps, seed, reset_at=None, mask=None):
  rng = np.random.default_rng(seed)
  import torch
  ops = [('reset', None)]
  for t in range(1, steps):
    if t == reset_at:
      ops.append(('reset', torch.from_numpy(mask).cuda()))
    else:
      ops.append(('step', torch.from_numpy(np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)).cuda()))
  return ops


def _shape(blob):
  from meltingpot_b200 import engine
  e = engine.Engine(blob, 1)
  P, A = e.num_players, e.num_actions
  e.close()
  return P, A


# ---- lockstep with a plainly stepped engine ------------------------------------------------------------------------
@pytest.mark.parametrize('layout', ['time_major', 'env_major'])
@pytest.mark.parametrize('B', ['7', 'sms+7', '257'])
@pytest.mark.parametrize('fam', FAMILIES + ['territory__inside_out'])
def test_step_into_trajectory_matches_plain_steps(fam, B, layout):
  blob = _blob(fam)
  B = _sms() + 7 if B == 'sms+7' else int(B)
  P, A = _shape(blob)
  time_major = layout == 'time_major'
  ops = _script(None, B, P, A, STEPS, seed=71)
  plain, into, traj = _run(blob, B, ops, seed=71, time_major=time_major, pad=16 if time_major else 48)
  if fam != 'territory__inside_out':
    lasts = [t for t in range(STEPS) if bool((traj.view['step_type'][t] == 2).any())]
    assert lasts == [40], lasts
  traj.only_slots_written(range(STEPS))
  plain.close()
  into.close()


# ---- the oracle ------------------------------------------------------------------------------------------------------
def test_step_into_matches_the_oracle(oracle):
  from meltingpot_b200 import engine
  blob = _blob('clean_up')
  B, seed = _sms() + 7, 72
  eng = engine.Engine(blob, B, seed=seed)
  batch = oracle.OracleBatch(blob, B, seed=seed)
  traj = _Traj(eng, 45, False, 48, _names(eng))
  rng = np.random.default_rng(seed)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  keys = dict(rgb='rgb', world_rgb='world', reward='reward', discount='discount', step_type='step_type', scalar_obs='scalar_obs')
  eng.reset(out=traj.at(0))
  for t in range(45):
    if t:
      a = _acts(rng, eng)
      eng.step(a, out=traj.at(t))
      batch.step_actions(a.cpu().numpy(), THREADS)
    px = t % 4 == 0 or t in (40, 41)
    got = {keys[k]: v[t].cpu().numpy() for k, v in traj.view.items() if px or k not in ('rgb', 'world_rgb')}
    parity.check_outputs(got, batch.dump(THREADS, shapes, pixels=px, max_events=max_ev), f'slot {t}')
  eng.close()
  batch.close()


# ---- masked reset, two-variant engine --------------------------------------------------------------------------------
def test_masked_reset_into_and_variants():
  from tests import env_variants as EV
  blobs = list(EV.blobs('clean_up')[:2])
  B = 130
  P, A = _shape(blobs[0])
  mask = (np.arange(B) % 3 == 0).astype(np.uint8)
  ops = _script(None, B, P, A, STEPS, seed=73, reset_at=20, mask=mask)
  for time_major in (True, False):
    plain, into, traj = _run(blobs, B, ops, seed=73, time_major=time_major, pad=16, env_variant=EV.interleaved(B, 2))
    st = traj.view['step_type'][20].cpu().numpy()
    assert (st[mask == 1] == 0).all() and (st[mask == 0] == 1).all()
    traj.only_slots_written(range(STEPS))
    plain.close()
    into.close()


# ---- partial targets -------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('mode', ['images', 'scalars', 'players_only', 'world_only'])
def test_partial_targets(mode):
  import torch
  from meltingpot_b200 import engine
  blob = _blob('clean_up')
  B = 64
  P, A = _shape(blob)
  flags = {'players_only': engine.MP_FLAG_RENDER_PLAYERS, 'world_only': engine.MP_FLAG_RENDER_WORLD}.get(mode, engine.MP_FLAG_DEFAULT)
  names = {'images': ['rgb', 'world_rgb'], 'scalars': ['reward', 'discount', 'step_type', 'scalar_obs']}.get(mode)
  ops = _script(None, B, P, A, 44, seed=74)
  own_images = {}

  def on_slot(t, plain, into, traj):
    if t == 0:  # from here on, every image the target takes must leave the engine's own copy alone
      for name in ('rgb', 'world_rgb'):
        if name in traj.view:
          getattr(into, name).fill_(0x5A)
          own_images[name] = True
    for name in own_images:
      assert bool((getattr(into, name) == 0x5A).all()), f'{mode}: the engine\'s own {name} was written at op {t}'
    for name in ('rgb', 'world_rgb'):  # an image the target leaves NULL is rendered into the engine's own set
      if name not in traj.view and name in _names(into, flags):
        assert torch.equal(getattr(into, name), getattr(plain, name)), f'{mode}: own {name} at op {t}'

  # (the own images are filled after op 0's render into the target, so ops 1.. show whether they are written)
  plain, into, traj = _run(blob, B, ops, seed=74, time_major=True, pad=16, names=names, flags=flags, on_slot=on_slot)
  traj.only_slots_written(range(len(ops)))
  if mode in ('players_only', 'world_only'):
    excluded = 'world_rgb' if mode == 'players_only' else 'rgb'
    other = _Traj(into, 1, True, 16, [excluded])
    before = into.save_state()
    with pytest.raises(ValueError, match='render flags'):
      into.step(_acts(np.random.default_rng(0), into), out=other.at(0))
    assert into.save_state() == before
    assert other.untouched(0)
  plain.close()
  into.close()


# ---- host paths and the engine's own buffers -------------------------------------------------------------------------
def test_own_buffers_after_a_target_step():
  import torch
  from meltingpot_b200 import engine
  blob = _blob('territory')
  B = 96
  plain, into = engine.Engine(blob, B, seed=75), engine.Engine(blob, B, seed=75)
  traj = _Traj(into, 1, True, 16, _names(into))
  rng = np.random.default_rng(75)
  plain.reset(); into.reset()
  a = _acts(rng, plain)
  plain.step(a); into.step(a)
  images = (plain.rgb.clone(), plain.world_rgb.clone())
  for _ in range(3):
    a = _acts(rng, plain)
    plain.step(a); into.step(a, out=traj.at(0))
  torch.cuda.synchronize()
  for name in parity._STATE_VIEWS:  # pylint: disable=protected-access
    assert torch.equal(getattr(into, name), getattr(plain, name)), name
  assert torch.equal(into.rgb, images[0]) and torch.equal(into.world_rgb, images[1]), 'own images: not those of the last own render'
  plain.close(); into.close()


def test_target_step_between_async_slot0_and_its_wait(oracle):
  import torch
  from meltingpot_b200 import engine
  blob = _blob('clean_up')
  B, seed = 512, 76
  eng = engine.Engine(blob, B, seed=seed)
  batch = oracle.OracleBatch(blob, B, seed=seed)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  rng = np.random.default_rng(seed)
  a1, a2 = _acts(rng, eng), _acts(rng, eng)
  h1 = eng.make_host_actions()
  h1.copy_(a1.cpu())
  out0 = eng.make_host_outputs()
  traj = _Traj(eng, 1, False, 48, _names(eng))
  eng.reset()
  torch.cuda.synchronize()
  eng.step_host_async(h1, out0, 0)
  eng.step(a2, out=traj.at(0))
  eng.wait(0)
  batch.step_actions(a1.cpu().numpy(), THREADS)
  parity.check_outputs(parity.host_outputs(out0, eng.num_scalar_obs), batch.dump(THREADS, shapes, pixels=True, max_events=max_ev), 'slot 0 host outputs')
  batch.step_actions(a2.cpu().numpy(), THREADS)
  keys = dict(rgb='rgb', world_rgb='world', reward='reward', discount='discount', step_type='step_type', scalar_obs='scalar_obs')
  got = {keys[k]: v[0].cpu().numpy() for k, v in traj.view.items()}
  parity.check_outputs(got, batch.dump(THREADS, shapes, pixels=True, max_events=max_ev), 'target step')
  eng.close()
  batch.close()


# ---- launch count ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('render', [True, False], ids=['render_on', 'render_off'])
def test_target_step_launches_as_many_kernels_as_a_plain_step(render):
  import torch
  from meltingpot_b200 import engine
  blob = _blob('coins')
  B = 64
  flags = engine.MP_FLAG_DEFAULT if render else 0
  plain, into = engine.Engine(blob, B, seed=77, flags=flags), engine.Engine(blob, B, seed=77, flags=flags)
  traj = _Traj(into, 4, True, 16, _names(into, flags))
  rng = np.random.default_rng(77)
  plain.reset(); into.reset(out=traj.at(0))
  assert plain.launch_count() == into.launch_count()
  for t in range(1, 4):
    a = _acts(rng, plain)
    plain.step(a); into.step(a, out=traj.at(t))
    assert plain.launch_count() == into.launch_count(), t
    torch.cuda.synchronize()
    for name in ('reward', 'discount', 'step_type'):
      assert torch.equal(traj.view[name][t], _own(plain, name)), (name, t)
  plain.close(); into.close()


# ---- refusals --------------------------------------------------------------------------------------------------------
def _cudart():
  import torch
  cands = [ctypes.util.find_library('cudart')]
  cands += sorted(glob.glob(os.path.join(os.path.dirname(torch.__file__), '..', 'nvidia', 'cuda_runtime', 'lib', 'libcudart.so*')))
  cands += sorted(glob.glob('/usr/local/cuda/lib64/libcudart.so*'))
  for c in cands:
    if c:
      try:
        return ctypes.CDLL(c)
      except OSError:
        pass
  pytest.skip('no libcudart to allocate with')


def test_refused_outputs_step_no_env():
  import torch
  from meltingpot_b200 import engine
  blob = _blob('clean_up')
  B = 9
  eng = engine.Engine(blob, B, seed=78)
  eng.reset()
  a = _acts(np.random.default_rng(0), eng)
  views = eng.output_views()
  E_rgb = int(np.prod(views['rgb'][0][1:]))
  P, n = eng.num_players, eng.num_scalar_obs
  assert n >= 2
  lib = engine.load_library()
  dev = torch.device('cuda', 0)
  raw = torch.zeros(B * (E_rgb + 64) + 64, dtype=torch.uint8, device=dev)

  def rgb_at(offset, stride):
    return torch.as_strided(raw, views['rgb'][0], (stride,) + tuple(eng.rgb.stride()[1:]), offset)

  scal = torch.zeros(n * B * P + 64, dtype=torch.float64, device=dev)
  cases = [
      ('pointer off by 8 bytes', dict(rgb=rgb_at(8, E_rgb)), 'multiple of 16'),
      ('env stride not a multiple of 16', dict(rgb=rgb_at(0, E_rgb + 8)), 'multiple of 16'),
      ('env stride below one env', dict(rgb=rgb_at(0, E_rgb - 16)), 'smaller than one env'),
      ('overlapping scalar_obs rows', dict(scalar_obs=torch.as_strided(scal, (n, B, P), (1, P, 1))), 'overlap'),
      ('outputs overlapping each other', dict(reward=torch.as_strided(scal, (B, P), (P, 1)),
                                              discount=torch.as_strided(scal, (B,), (P,), 2)), 'overlap'),
      ('the engine\'s own buffers', dict(reward=eng.reward), 'own buffers'),
  ]

  def refused(out, match, raw_call=None):
    before = eng.save_state()
    with pytest.raises(ValueError, match=match):
      if raw_call is None:
        eng.step(a, out=out)
      else:
        engine._check(raw_call())  # pylint: disable=protected-access
    assert eng.save_state() == before, f'a refused call ({match}) changed the state'

  for what, out, match in cases:
    refused(out, match)
  # a host pointer (pinned, so it has a device mapping) and an extent past the end of a cudaMalloc'ed buffer go straight
  # to the C call, past the Python checks
  host = torch.zeros(B * P, dtype=torch.float64).pin_memory()
  s = engine.MpDeviceOutputs()
  s.reward, s.reward_env_stride = host.data_ptr(), P * 8
  step_into = lambda s: lib.mp_run(eng._h, ctypes.byref(engine.MpRequest(actions=a.data_ptr(), out=ctypes.pointer(s))), None)  # pylint: disable=protected-access
  refused(None, 'not device memory', lambda: step_into(s))
  cudart = _cudart()
  ptr = ctypes.c_void_p()
  mib = 1 << 20
  assert cudart.cudaMalloc(ctypes.byref(ptr), ctypes.c_size_t((B - 1) * mib)) == 0
  try:
    s = engine.MpDeviceOutputs()
    s.reward, s.reward_env_stride = ptr.value, mib  # env B - 1's row starts at the end of the allocation
    refused(None, 'past the end', lambda: step_into(s))
    s.reward_env_stride = mib - P * 8  # ... and ends exactly at it: accepted
    torch.cuda.synchronize()
    engine._check(step_into(s))  # pylint: disable=protected-access
    torch.cuda.synchronize()
  finally:
    cudart.cudaFree(ptr)
  eng.close()


# ---- two GPUs: stacked observations while the local images go to a target ------------------------------------------
def test_gather_obs_with_local_images_into_a_target():
  import torch
  from meltingpot_b200 import engine
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  blob = _blob('clean_up')
  B = 150
  ranks = [engine.Engine(blob, B, device=r, seed=79, env_index_base=r * B) for r in range(2)]
  ptrs = [e.gather_obs_create(r, 2)[0] for r, e in enumerate(ranks)]
  engine.enable_peer_access(0, 1); engine.enable_peer_access(1, 0)
  for e in ranks:
    e.gather_obs_connect(ptrs)
  trajs = []
  for r, e in enumerate(ranks):
    with torch.cuda.device(r):
      trajs.append(_Traj(e, 6, r == 0, 16, ['rgb', 'world_rgb']))
  for r, e in enumerate(ranks):
    with torch.cuda.device(r):
      e.reset(out=trajs[r].at(0))
  gen = torch.Generator().manual_seed(2)
  for t in range(6):
    for e in ranks:
      e.gather_obs_wait()
    torch.cuda.synchronize(0); torch.cuda.synchronize(1)
    want_rgb = torch.cat([tr.view['rgb'][t].cpu() for tr in trajs])
    want_world = torch.cat([tr.view['world_rgb'][t].cpu() for tr in trajs])
    for e in ranks:
      rgb, world = e.gathered_observations()
      assert torch.equal(rgb.cpu(), want_rgb) and torch.equal(world.cpu(), want_world), t
    if t + 1 < 6:
      acts = torch.randint(0, ranks[0].num_actions, (2 * B, ranks[0].num_players), generator=gen, dtype=torch.int32)
      for r, e in enumerate(ranks):
        with torch.cuda.device(r):
          e.step(acts[r * B:(r + 1) * B].contiguous().cuda(r), out=trajs[r].at(t + 1))
  for e in ranks:
    e.close()


# ---- BatchedSubstrate.trajectory --------------------------------------------------------------------------------------
@pytest.mark.parametrize('time_major', [True, False], ids=['time_major', 'env_major'])
def test_batched_substrate_steps_into_a_trajectory(time_major):
  import torch
  from meltingpot_b200 import substrate
  blob = _blob('clean_up')
  B, T = 33, 44
  plain = substrate.BatchedSubstrate(blob, B, seed=80)
  into = substrate.BatchedSubstrate(blob, B, seed=80)
  traj = into.trajectory(T, time_major=time_major)
  rng = np.random.default_rng(80)
  want = plain.reset()
  got = into.reset(out=traj.at(0))
  for t in range(T):
    if t:
      a = _acts(rng, plain.engine)
      want = plain.step(a)
      got = into.step(a, out=traj.at(t))
    torch.cuda.synchronize()
    slot = traj.at(t)
    for k in ('step_type', 'reward', 'discount'):
      assert torch.equal(getattr(got, k), getattr(want, k)) and torch.equal(getattr(slot, k), getattr(want, k)), (k, t)
    for k, v in want.observation.items():
      assert torch.equal(slot.observation[k], v), (k, t)
  plain.close(); into.close()
