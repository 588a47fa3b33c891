"""Restores inside a step (mp_run's slot_of_env and bank, Engine.step(restore=, bank=), BatchedSubstrate / ShardedSubstrate.step).

The fused call must give, byte for byte, what a step followed by mp_state_restore with the same arguments gives: every
output, the events, the state, the variant bytes and the mp_state_save snapshot, after the call and on every step that
follows. Two identically seeded engines run in lockstep, one taking the fused call and its twin the two calls. At one
batch size per family the restored envs are also checked against the oracle env of their source, replayed to the store
point, as tests/test_gpu_state_bank.py does for mp_state_restore. Runs use the hard_cap_40 variants, so every run
crosses an auto-reset.
"""

import ctypes

import numpy as np
import pytest

from tests import env_variants as EV
from tests import parity
from tests.test_gpu_state_bank import FAMILIES, SEED, _VIEWS, _batch_size, _blob, _env_outputs, _keyed, _replay
from tests.test_gpu_step_into import _cudart, _names, _Traj

pytestmark = pytest.mark.gpu

_ALL = _VIEWS + ('events',)
N_SLOTS = 6  # slots 0..3: envs 0..3 at step 25; slot 4: env 4 at step 40 (LAST); slot 5: never written (untagged)
STORE_AT = {0: 25, 1: 25, 2: 25, 3: 25, 4: 40}


def _idx(n, mapping):
  import torch
  idx = torch.full((n,), -1, dtype=torch.int32)
  for k, v in mapping.items():
    idx[k] = v
  return idx.cuda()


def _same(a, b, what, snapshot=False):
  import torch
  torch.cuda.synchronize()
  for name in _ALL:
    assert torch.equal(getattr(a, name), getattr(b, name)), f'{name}: {what}'
  if a.active_variant is not None:
    assert torch.equal(a.active_variant, b.active_variant) and torch.equal(a.pending_variant, b.pending_variant), what
  if snapshot:
    assert a.save_state() == b.save_state(), f'mp_state_save snapshot: {what}'


def _fused_and_twin(a, b, acts, idx, bank, rekey=False):
  a.step(acts, restore=idx, bank=bank, rekey=rekey)
  b.step(acts)
  b.restore_states(bank, idx, rekey=rekey)


def _restore_sets(B):
  """(plain restores at step 41, rekeyed restores at step 42): a permutation, an env onto itself, a fan-out of the LAST
  record, out-of-range and untagged rows (stepped as plain envs), and a rekeyed clone. Every env's step 40 is LAST, so
  each restore at step 41 takes the place of an auto-reset."""
  plain = {1: 2, 2: 3, 3: 1, 4: 4, 5: 4, 0: 5, 6: 99}  # env 0: untagged row; env 6: slot out of range
  rekeyed = {6: 0, 3: 3}
  if B > 7:
    plain.update({B - 1: 0, B - 2: 3, B // 2: 4, 7: -5, 8: 2**31 - 1})
  if B >= 64:
    plain.update({j: j % 5 for j in range(16, 48)})
    rekeyed.update({j: j % 4 for j in range(48, 56)})
  return plain, rekeyed


def _run(fam, B, oracle):
  import torch
  from meltingpot_b200 import engine
  blob = _blob(fam)
  a = engine.Engine(blob, B, device=0, seed=SEED)
  b = engine.Engine(blob, B, device=0, seed=SEED)
  P, A = a.num_players, a.num_actions
  rng = np.random.default_rng(B + 3)
  bank = torch.zeros((N_SLOTS, a.state_record_bytes), dtype=torch.uint8, device='cuda')
  hist = []
  a.reset(); b.reset()
  for t in range(1, 41):
    acts = np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)
    hist.append(acts)
    x = torch.from_numpy(acts).cuda()
    a.step(x); b.step(x)
    for t_store, slots in ((25, [0, 1, 2, 3]), (40, [4])):
      if t == t_store:
        a.store_states(bank, _idx(N_SLOTS, {k: k for k in slots}))
  torch.cuda.synchronize()
  assert (a.step_type.cpu().numpy() == 2).all()  # step 40 ends every episode (the 40-frame cap)
  plain, rekeyed = _restore_sets(B)
  tagged = lambda m: {j: s for j, s in m.items() if s in STORE_AT}

  x41 = torch.from_numpy(np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)).cuda()
  _fused_and_twin(a, b, x41, _idx(B, plain), bank)
  _same(a, b, f'after the fused call B={B}', snapshot=True)
  st = a.step_type.cpu().numpy()
  assert st[5] == 2 and st[1] == 1, 'a restored env must show its record\'s timestep'
  assert st[6] == 0 and st[0] == 0, 'an env with an out-of-range index or an untagged row must take its auto-reset'
  x42 = torch.from_numpy(np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)).cuda()
  _fused_and_twin(a, b, x42, _idx(B, rekeyed), bank, rekey=True)
  _same(a, b, f'after the rekeyed fused call B={B}', snapshot=True)

  clones = {}
  if oracle:
    keyed = _keyed()
    shapes = parity.shapes_of(a)
    max_ev = int(a.buffers.max_events)

    def oracle_of(j, slot, rekey):
      e = _replay(keyed, blob, SEED + slot, [hist[t][slot] for t in range(STORE_AT[slot])])
      if rekey:
        e.set_key(SEED + j)
      return e

    clones = {j: oracle_of(j, s, False) for j, s in tagged(plain).items() if j not in rekeyed}
    for j in clones:  # step 42 moved the step-41 clones on with their actions
      clones[j].step(x42[j].cpu().numpy())
    clones.update({j: oracle_of(j, s, True) for j, s in tagged(rekeyed).items()})
    order = sorted(clones)

    def check(t, px):
      got = _env_outputs(a, order, px)
      want = parity.env_dump([clones[j] for j in order], shapes, pixels=px, max_events=max_ev)
      parity.check_outputs(got, want, f'restored envs {order} step {t} B={B}')

    check(42, True)
  trail = []
  for t in range(43, 88):
    x = torch.from_numpy(np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)).cuda()
    if t % 3 == 0:  # no restore: an index of all -1 steps every env as a plain step does
      a.step(x, restore=_idx(B, {}), bank=bank)
      b.step(x)
    else:
      a.step(x); b.step(x)
    _same(a, b, f'step {t} B={B}', snapshot=t == 87)
    for j, e in clones.items():
      e.step(x[j].cpu().numpy())
    if clones:
      check(t, t in (43, 60, 87))
    trail.append(int((a.step_type == 0).sum()))
  assert any(trail), 'the tail never crossed an auto-reset'
  a.close(); b.close()


@pytest.mark.parametrize('which', ['7', 'sms-1', 'sms+1', '2048'])
@pytest.mark.parametrize('fam', FAMILIES)
def test_fused_restore_equals_step_then_restore(fam, which):
  _run(fam, _batch_size(which), oracle=which == '7')


# ---- launch count ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('render', [True, False], ids=['render_on', 'render_off'])
def test_fused_restore_launches_as_many_kernels_as_a_step(render):
  import torch
  from meltingpot_b200 import engine
  blob = _blob('coins')
  B = 64
  flags = engine.MP_FLAG_DEFAULT if render else 0
  eng = engine.Engine(blob, B, seed=81, flags=flags)
  rng = np.random.default_rng(81)
  x = lambda: torch.from_numpy(np.ascontiguousarray(rng.integers(0, eng.num_actions, size=(B, eng.num_players)), np.int32)).cuda()
  eng.reset()
  bank = torch.zeros((B, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.arange(B, dtype=torch.int32, device='cuda'))
  every = torch.arange(B, dtype=torch.int32, device='cuda')
  traj = _Traj(eng, 2, True, 16, _names(eng, flags))

  def added(fn):
    n = eng.launch_count()
    fn()
    return eng.launch_count() - n

  step, fused = added(lambda: eng.step(x())), added(lambda: eng.step(x(), restore=every, bank=bank))
  assert fused == step, (fused, step)
  step, fused = added(lambda: eng.step(x(), out=traj.at(0))), added(lambda: eng.step(x(), out=traj.at(1), restore=every, bank=bank))
  assert fused == step, (fused, step)
  eng.close()


# ---- variants --------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('family', EV.NAMES)
def test_fused_restore_on_a_variant_engine(family):
  import torch
  from meltingpot_b200 import engine
  blobs = list(EV.blobs(family))
  B = 12
  assign = EV.interleaved(B, len(blobs))
  a = engine.Engine(blobs, B, device=0, seed=SEED, env_variant=assign)
  b = engine.Engine(blobs, B, device=0, seed=SEED, env_variant=assign)
  P, A = a.num_players, a.num_actions
  gen = torch.Generator(device='cuda').manual_seed(9)
  a.reset(); b.reset()
  bank = torch.zeros((3, a.state_record_bytes), dtype=torch.uint8, device='cuda')
  for t in range(60):
    x = torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32)
    if t == 20:
      a.store_states(bank, _idx(3, {0: 1, 1: 2}))
      ids = np.asarray(assign).copy(); ids[2] = (ids[2] + 1) % len(blobs)
      a.set_env_variant(ids); b.set_env_variant(ids)
      a.store_states(bank, _idx(3, {2: 2}))  # env 2 with another pending variant
    if t in (25, 40):  # a restore into envs of other variants, once where every env's last step was LAST
      _fused_and_twin(a, b, x, _idx(B, {4: 0, 5: 1, 6: 2, 7: 2, 8: 9}), bank)
      _same(a, b, f'fused call at step {t}', snapshot=True)
    else:
      a.step(x); b.step(x)
      _same(a, b, f'step {t}')
  a.close(); b.close()


# ---- trajectory targets ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('time_major', [True, False], ids=['time_major', 'env_major'])
def test_batched_substrate_restores_into_a_trajectory(time_major):
  import torch
  from meltingpot_b200 import substrate
  blob = _blob('clean_up')
  B, T = 33, 50
  into = substrate.BatchedSubstrate(blob, B, seed=82)
  twin = substrate.BatchedSubstrate(blob, B, seed=82)
  traj = into.trajectory(T, time_major=time_major)
  gen = torch.Generator(device='cuda').manual_seed(82)
  into.reset(); twin.reset()
  bank = into.state_bank(4)
  starts = torch.arange(B, device='cuda', dtype=torch.int32) % 4  # the stored start state each env restarts from
  restored = 0
  for t in range(T):
    a = torch.randint(0, into.num_actions, (B, into.num_players), generator=gen, device='cuda', dtype=torch.int32)
    if t == 3:
      into.store(bank, [0, 5, 9, 20], [0, 1, 2, 3])
    if t > 3:  # restart every finished episode from a stored state, the index built on the device
      idx = torch.where(into.engine.step_type == 2, starts, -1).to(torch.int32)
      restored += int((idx >= 0).sum())
      torch.cuda.set_sync_debug_mode('error')
      try:
        got = into.step(a, out=traj.at(t), restore=idx, bank=bank)
      finally:
        torch.cuda.set_sync_debug_mode(0)
      twin.step(a)
      twin.engine.restore_states(bank, idx)
      want = twin._timestep()  # pylint: disable=protected-access
    else:
      got = into.step(a, out=traj.at(t))
      want = twin.step(a)
    torch.cuda.synchronize()
    slot = traj.at(t)
    for k in ('step_type', 'reward', 'discount'):
      assert torch.equal(getattr(got, k), getattr(want, k)) and torch.equal(getattr(slot, k), getattr(want, k)), (k, t)
    for k, v in want.observation.items():
      assert torch.equal(slot.observation[k], v), (k, t)
    for name in parity._STATE_VIEWS:  # pylint: disable=protected-access
      assert torch.equal(getattr(into.engine, name), getattr(twin.engine, name)), (name, t)
  assert restored > 0, 'no episode ended: nothing was restored'
  into.close(); twin.close()


# ---- sharded engines -------------------------------------------------------------------------------------------------
def _connected_lockstep(devices, fam, B, steps):
  """Rank r on devices[r], exchange and gather connected; each rank has an unconnected twin on the same device that
  runs plain steps and step-then-restore where the rank interleaves plain and fused steps."""
  import torch
  from meltingpot_b200 import engine
  blob = _blob(fam)
  world = len(devices)
  ranks = [engine.Engine(blob, B, device=d, seed=SEED, env_index_base=r * B) for r, d in enumerate(devices)]
  twins = [engine.Engine(blob, B, device=d, seed=SEED, env_index_base=r * B) for r, d in enumerate(devices)]
  if world > 1:
    engine.enable_peer_access(devices[0], devices[1]); engine.enable_peer_access(devices[1], devices[0])
  xp = [e.exchange_create(r, world)[0] for r, e in enumerate(ranks)]
  gp = [e.gather_obs_create(r, world)[0] for r, e in enumerate(ranks)]
  for e in ranks:
    e.exchange_connect(xp); e.gather_obs_connect(gp)
  P, A = ranks[0].num_players, ranks[0].num_actions
  banks = []
  for r, d in enumerate(devices):
    with torch.cuda.device(d):
      banks.append(torch.zeros((B, ranks[r].state_record_bytes), dtype=torch.uint8, device=f'cuda:{d}'))
  gen = torch.Generator().manual_seed(83)
  for r, d in enumerate(devices):
    with torch.cuda.device(d):
      ranks[r].reset(); twins[r].reset()
  fused_steps = 0
  for t in range(steps):
    acts = torch.randint(0, A, (world * B, P), generator=gen, dtype=torch.int32)
    perm = torch.randperm(B, generator=gen).to(torch.int32)
    for r, d in enumerate(devices):
      with torch.cuda.device(d):
        x = acts[r * B:(r + 1) * B].contiguous().cuda(d)
        if t == 10:
          ranks[r].store_states(banks[r], torch.arange(B, dtype=torch.int32, device=f'cuda:{d}'))
        if t > 10 and t % 2:  # fused: a permutation of the stored states on half the envs (rank 1 restores nothing at t = 13)
          idx = torch.where(torch.arange(B) % 2 == 0, perm, -1).to(torch.int32)
          if r == 1 and t == 13:
            idx.fill_(-1)
          idx = idx.cuda(d)
          _fused_and_twin(ranks[r], twins[r], x, idx, banks[r])
          fused_steps += r == 0
        else:
          ranks[r].step(x); twins[r].step(x)
    for r, d in enumerate(devices):
      with torch.cuda.device(d):
        ranks[r].exchange_wait(); ranks[r].gather_obs_wait()
    for d in devices:
      torch.cuda.synchronize(d)
    want_rows = torch.cat([tw.timestep_packed.cpu() for tw in twins])
    want_rgb = torch.cat([tw.rgb.cpu() for tw in twins])
    want_world = torch.cat([tw.world_rgb.cpu() for tw in twins])
    for r, e in enumerate(ranks):
      assert torch.equal(e.gathered_timestep().cpu(), want_rows), f'gathered rows on rank {r} at step {t}'
      rgb, world_rgb = e.gathered_observations()
      assert torch.equal(rgb.cpu(), want_rgb) and torch.equal(world_rgb.cpu(), want_world), f'stacked images on rank {r} at step {t}'
      for name in _ALL:
        assert torch.equal(getattr(e, name).cpu(), getattr(twins[r], name).cpu()), f'{name} of rank {r} at step {t}'
  assert fused_steps > 0
  for e in ranks + twins:
    e.close()


def test_fused_restore_on_a_connected_engine_of_one_rank():
  _connected_lockstep([0], 'clean_up', 40, 30)


def test_fused_restore_between_two_gpus_one_process():
  import torch
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  _connected_lockstep([0, 1], 'territory', 24, 30)


def test_sharded_substrate_world_of_one_passes_restore_through():
  import os
  import torch
  import torch.distributed as dist
  from meltingpot_b200 import distributed
  created = False
  if not dist.is_initialized():
    os.environ.setdefault('MASTER_ADDR', '127.0.0.1'); os.environ.setdefault('MASTER_PORT', '29534')
    dist.init_process_group('nccl', rank=0, world_size=1, device_id=torch.device('cuda', 0))
    created = True
  try:
    sh = distributed.ShardedSubstrate('clean_up', ('default',) * 7, global_num_envs=64, seed=4, device=0)
    sh.connect(observations=True)
    ts = sh.reset()
    bank = sh.local.state_bank(8)
    gen = torch.Generator(device='cuda').manual_seed(0)
    for t in range(8):
      reward, discount, step_type = sh.stacked_timestep()
      rgb, world = sh.stacked_observations()
      torch.cuda.synchronize()
      assert torch.equal(reward, ts.reward) and torch.equal(discount, ts.discount) and torch.equal(step_type, ts.step_type)
      assert torch.equal(rgb, ts.observation['RGB']) and torch.equal(world, ts.observation['WORLD.RGB'])
      if t == 2:
        sh.local.store(bank, list(range(8)), list(range(8)))
        snap = sh.local.engine.rgb[:8].clone()
      acts = torch.randint(0, 9, (64, 7), generator=gen, device='cuda', dtype=torch.int32)
      if t == 5:
        idx = torch.full((64,), -1, dtype=torch.int32, device='cuda')
        idx[56:] = torch.arange(8, dtype=torch.int32, device='cuda')
        ts = sh.step(acts, restore=idx, bank=bank)
        torch.cuda.synchronize()
        assert torch.equal(ts.observation['RGB'][56:], snap), 'the restored envs do not show their records\' images'
      else:
        ts = sh.step(acts)
    sh.close()
  finally:
    if created:
      dist.destroy_process_group()


# ---- refusals --------------------------------------------------------------------------------------------------------
def test_refused_fused_calls_step_no_env(clean_up_blob):
  import torch
  from meltingpot_b200 import engine
  lib = engine.load_library()
  B = 8
  eng = engine.Engine(clean_up_blob, B, device=0, seed=SEED)
  eng.reset()
  R, P = eng.state_record_bytes, eng.num_players
  acts = torch.zeros((B, P), dtype=torch.int32, device='cuda')
  idx = torch.arange(B, dtype=torch.int32, device='cuda')
  big = torch.zeros((2 * R + 64,), dtype=torch.uint8, device='cuda')
  eng.store_states(big[:2 * R].view(2, R), torch.arange(2, dtype=torch.int32, device='cuda'))

  def call(bank, index, n, flags=0, out=None):
    r = engine.MpRequest(actions=acts.data_ptr(), slot_of_env=index, bank=bank, n_slots=n, restore_flags=flags)
    if out is not None:
      r.out = ctypes.pointer(out)
    return lib.mp_run(eng._h, ctypes.byref(r), None)  # pylint: disable=protected-access

  def refused(match, fn):
    torch.cuda.synchronize()
    snap, launches = eng.save_state(), eng.launch_count()
    with pytest.raises(ValueError, match=match):
      engine._check(fn())  # pylint: disable=protected-access
    assert eng.launch_count() == launches, f'a refused call ({match}) launched a kernel'
    assert eng.save_state() == snap, f'a refused call ({match}) moved an env'

  refused('go together', lambda: call(None, idx.data_ptr(), 2))
  refused('go together', lambda: call(big.data_ptr(), None, 2))
  refused('n_slots', lambda: call(big.data_ptr(), idx.data_ptr(), 0))
  refused('flags', lambda: call(big.data_ptr(), idx.data_ptr(), 2, flags=6))
  refused('aligned', lambda: call(big.data_ptr() + 1, idx.data_ptr(), 2))
  host = torch.zeros((2 * R,), dtype=torch.uint8).pin_memory()
  refused('not device memory', lambda: call(host.data_ptr(), idx.data_ptr(), 2))
  host_idx = torch.zeros((B,), dtype=torch.int32).pin_memory()
  refused('not device memory', lambda: call(big.data_ptr(), host_idx.data_ptr(), 2))
  refused('own buffers', lambda: call(eng.grid.data_ptr(), idx.data_ptr(), 1))
  cudart = _cudart()
  ptr = ctypes.c_void_p()
  assert cudart.cudaMalloc(ctypes.byref(ptr), ctypes.c_size_t(2 * R)) == 0
  try:
    refused('past the end', lambda: call(ptr.value, idx.data_ptr(), 3))
  finally:
    cudart.cudaFree(ptr)
  # a bank overlapping a target of `out`, and a refused `out` itself
  region = torch.zeros((2 * R + B * P * 8,), dtype=torch.uint8, device='cuda')
  o = engine.MpDeviceOutputs()
  o.reward, o.reward_env_stride = region.data_ptr() + R, P * 8
  refused('overlap', lambda: call(region.data_ptr(), idx.data_ptr(), 2, out=o))
  o.reward = eng.reward.data_ptr()
  refused('own buffers', lambda: call(big.data_ptr(), idx.data_ptr(), 2, out=o))
  o.reward = region.data_ptr() + 2 * R  # beside the bank: accepted
  engine._check(call(region.data_ptr(), idx.data_ptr(), 2, out=o))  # pylint: disable=protected-access
  torch.cuda.synchronize()
  eng.close()


# ---- host-async interplay --------------------------------------------------------------------------------------------
def test_fused_call_between_async_slot0_and_its_wait(commons_blob):
  import torch
  from meltingpot_b200 import engine
  B = 20
  eng = engine.Engine(commons_blob, B, device=0, seed=SEED)
  twin = engine.Engine(commons_blob, B, device=0, seed=SEED)
  P, A = eng.num_players, eng.num_actions
  rng = np.random.default_rng(7)
  eng.reset(); twin.reset()
  bank = torch.zeros((B, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  for t in range(25):
    x = torch.from_numpy(np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)).cuda()
    eng.step(x); twin.step(x)
    if t == 10:
      eng.store_states(bank, torch.arange(B, dtype=torch.int32, device='cuda'))
  out = eng.make_host_outputs()
  acts = eng.make_host_actions()
  acts.copy_(torch.from_numpy(np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)))
  eng.step_host_async(acts, out, 0)
  x = torch.from_numpy(np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)).cuda()
  eng.step(x, restore=torch.arange(B, dtype=torch.int32, device='cuda'), bank=bank)  # before wait(0)
  eng.wait(0)
  twin.step(acts.cuda())
  torch.cuda.synchronize()
  assert torch.equal(out['rgb'], twin.rgb.cpu()) and torch.equal(out['world_rgb'], twin.world_rgb.cpu())
  assert torch.equal(out['reward'], twin.reward.cpu()) and torch.equal(out['step_type'], twin.step_type.cpu())
  assert torch.equal(out['discount'], twin.discount.cpu())
  twin.step(x)
  twin.restore_states(bank, torch.arange(B, dtype=torch.int32, device='cuda'))
  _same(eng, twin, 'after the fused call')
  eng.close(); twin.close()
