"""Per-env state bank on the device (mp_state_store / mp_state_restore, Engine.store_states / restore_states,
BatchedSubstrate.store / restore).

A restored env must continue exactly as the stored env would have: env j restored from a record of env s equals, bit
for bit, the oracle env keyed seed + s replayed to the store point and stepped on with env j's actions (with
MP_RESTORE_REKEY: that oracle env switched to key seed + j at the store point). Every env a call does not name must
equal its own oracle env. Runs use the hard_cap_40 variants of tests/variants.py (and territory__inside_out, whose
'choice' prefabs are drawn per episode), so every tail crosses an auto-reset.
"""

import ctypes
import os

import numpy as np
import pytest

from tests import env_variants as EV
from tests import parity
from tests import variants as V
from tests.test_gpu_step_into import _cudart

pytestmark = pytest.mark.gpu

FAMILIES = ['clean_up', 'commons_harvest', 'territory', 'coins', 'coop_mining', 'territory__inside_out']
THREADS = os.cpu_count() or 1
SEED = 17
_VIEWS = ('reward', 'discount', 'step_type', 'scalar_obs', 'avatar_state', 'grid', 'event_count', 'timestep_packed',
          'rgb', 'world_rgb')


def _blob(fam):
  if fam == 'territory__inside_out':
    from tests.test_gpu_entry_points import _inside_out_cap40
    return _inside_out_cap40()
  return V.compile(f'{fam}/hard_cap_40')


def _sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _batch_size(which):
  return {'7': 7, 'sms-1': _sms() - 1, 'sms+1': _sms() + 1, '2048': 2048}[which]


def _keyed():
  from oracle import binding
  binding.build()
  from tests import oracle_keys
  return oracle_keys


def _env_outputs(eng, envs, pixels):
  """Outputs of the listed envs keyed like parity.env_dump (images only with `pixels`)."""
  import torch
  torch.cuda.synchronize()
  idx = torch.as_tensor(list(envs), device='cuda', dtype=torch.int64)
  got = dict(step_type=eng.step_type[idx].cpu().numpy(), discount=eng.discount[idx].cpu().numpy(),
             reward=eng.reward[idx].cpu().numpy(), scalar_obs=eng.scalar_obs[:, idx].cpu().numpy()[:eng.num_scalar_obs],
             avatars=eng.avatar_state[idx].cpu().numpy(),
             grid=eng.grid[idx].cpu().numpy().view(np.uint16)[:, :, :int(eng.buffers.grid_cells)],
             n_events=eng.event_count[idx].cpu().numpy(), events=eng.events[idx].cpu().numpy())
  if pixels:
    got['rgb'] = eng.rgb[idx].cpu().numpy()
    got['world'] = eng.world_rgb[idx].cpu().numpy()
  return got


def _rows(d, envs):
  """The rows of `envs` of an OracleBatch.dump / device_outputs dict."""
  return {k: (v[:, envs] if k == 'scalar_obs' else v[envs]) for k, v in d.items()}


def _replay(keyed, blob, key, actions):
  """An oracle env keyed `key`, reset and stepped through `actions` (a list of [P] rows)."""
  e = keyed.KeyedOracleEnv(blob, key)
  e.reset()
  for a in actions:
    e.step(a)
  return e


def _index(n, mapping):
  import torch
  idx = torch.full((n,), -1, dtype=torch.int32)
  for k, v in mapping.items():
    idx[k] = v
  return idx.cuda()


# ---- 1 + 2: clones against the oracle ---------------------------------------------------------------------------------
def _clone_run(fam, B):
  """Stores envs 0..3 at step 25 and env 4 at step 40 (a LAST step), restores at step 40 and steps on 45 more steps.
  Restores: a permutation (envs 1, 2, 3 take the records of 2, 3, 1), env 4 onto itself, a fan-out of env 4's LAST
  record (envs 4, 5), and env 6 from env 0's record with MP_RESTORE_REKEY. Larger batches add a plain clone of env 0's
  record beside the rekeyed one (with the same actions), more fan-out and a block of restores; the rest is untouched.
  Returns, per tail step: the rekeyed clone's oracle state, the GPU states of (plain twin, rekeyed clone) on batches
  that hold the twin, and the un-rekeyed clone's oracle state."""
  import torch
  from meltingpot_b200 import engine
  keyed = _keyed()
  from oracle import binding
  blob = _blob(fam)
  eng = engine.Engine(blob, B, device=0, seed=SEED)
  P, A = eng.num_players, eng.num_actions
  shapes = parity.shapes_of(eng)
  max_ev = int(eng.buffers.max_events)
  batch = binding.OracleBatch(blob, B, seed=SEED)
  rng = np.random.default_rng(B)
  hist = []
  bank = torch.zeros((5, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  store_at = {0: 25, 1: 25, 2: 25, 3: 25, 4: 40}  # slot k holds env k as of step store_at[k]
  plain = {1: 2, 2: 3, 3: 1, 4: 4, 5: 4}
  rekeyed = {6: 0}
  if B > 7:
    plain.update({B - 1: 0, B - 2: 3, B // 2: 4})
  if B >= 64:
    plain.update({j: j % 5 for j in range(16, 48)})
  touched = sorted(set(plain) | set(rekeyed))
  untouched = [b for b in range(B) if b not in touched]

  eng.reset()
  for t in range(1, 41):
    acts = np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)
    hist.append(acts)
    eng.step(torch.from_numpy(acts).cuda())
    batch.step_actions(acts, THREADS)
    for t_store, slots in ((25, [0, 1, 2, 3]), (40, [4])):
      if t == t_store:
        eng.store_states(bank, _index(5, {k: k for k in slots}))
  assert (eng.step_type.cpu().numpy() == 2).all()  # step 40 ends every episode (the 40-frame cap)
  launches = eng.launch_count()
  eng.restore_states(bank, _index(B, plain))
  eng.restore_states(bank, _index(B, rekeyed), rekey=True)
  assert eng.launch_count() == launches + 4  # per restore: k_state_restore and the re-render

  def oracle_of(j, slot, rekey):
    src, at = slot, store_at[slot]
    e = _replay(keyed, blob, SEED + src, [hist[t][src] for t in range(at)])
    if rekey:
      e.set_key(SEED + j)
    return e

  clones = {j: oracle_of(j, s, False) for j, s in plain.items()}
  clones.update({j: oracle_of(j, s, True) for j, s in rekeyed.items()})
  unrekeyed = oracle_of(6, 0, False)
  order = sorted(clones)

  def check(t, px, px_untouched):
    got = _env_outputs(eng, order, px)
    want = parity.env_dump([clones[j] for j in order], shapes, pixels=px, max_events=max_ev)
    parity.check_outputs(got, want, f'clones {order} step {t} B={B}')
    if untouched:
      got = _rows(parity.device_outputs(eng, ('rgb', 'world') if px_untouched else ()), untouched)
      want = _rows(batch.dump(THREADS, shapes, pixels=px_untouched, max_events=max_ev), untouched)
      parity.check_outputs(got, want, f'untouched envs step {t} B={B}')

  check(40, True, True)
  # the restored timestep is the stored one: a LAST record shows LAST, a step-25 record a MID step
  st = eng.step_type.cpu().numpy()
  assert st[5] == 2 and st[1] == 1 and st[6] == 1
  src_of = dict(plain)
  src_of.update(rekeyed)
  trail6, trail_twin, trail_unrekeyed = [], [], []
  for t in range(41, 86):
    base = rng.integers(0, A, size=(B, P))
    acts = base.copy()
    for j, s in src_of.items():
      acts[j] = base[s]  # each clone takes its source's actions
    acts = np.ascontiguousarray(acts, np.int32)
    eng.step(torch.from_numpy(acts).cuda())
    batch.step_actions(acts, THREADS)
    for j in order:
      clones[j].step(acts[j])
    unrekeyed.step(acts[6])
    check(t, t in (41, 55, 70, 85), t == 85)
    trail6.append((clones[6].avatars().tobytes(), clones[6].grid().tobytes(), clones[6].rewards().tobytes()))
    trail_unrekeyed.append((unrekeyed.avatars().tobytes(), unrekeyed.grid().tobytes(), unrekeyed.rewards().tobytes()))
    if B > 7:  # env B - 1: the plain clone of env 0's record, with env 6's actions
      trail_twin.append((eng.grid[B - 1].cpu().numpy().tobytes() + eng.avatar_state[B - 1].cpu().numpy().tobytes(),
                         eng.grid[6].cpu().numpy().tobytes() + eng.avatar_state[6].cpu().numpy().tobytes()))
  eng.close()
  batch.close()
  return trail6, trail_twin, trail_unrekeyed


@pytest.mark.parametrize('which', ['7', 'sms-1', 'sms+1', '2048'])
@pytest.mark.parametrize('fam', FAMILIES)
def test_clone_equals_its_source(fam, which):
  trail6, trail_twin, trail_unrekeyed = _clone_run(fam, _batch_size(which))
  # reach: the rekeyed clone (env 6) leaves the un-rekeyed clone's trajectory somewhere in the tail
  assert trail6 != trail_unrekeyed, 'MP_RESTORE_REKEY made no difference over the whole tail'
  if trail_twin:
    assert any(a != b for a, b in trail_twin), 'the rekeyed clone and its plain twin on the GPU never differed'


# ---- 3: round trip ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fam', FAMILIES)
def test_round_trip_restores_the_stored_timestep_and_continuation(fam):
  import torch
  from meltingpot_b200 import substrate
  B, K = 33, 45
  bs = substrate.BatchedSubstrate(_blob(fam), B, seed=SEED)
  P, A = bs.num_players, bs.num_actions
  gen = torch.Generator(device='cuda').manual_seed(5)
  bs.reset()
  for _ in range(22):
    bs.step(torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32))
  bank = bs.state_bank(B)
  every = list(range(B))
  bs.store(bank, every, every)
  e = bs.engine
  at_store = {name: getattr(e, name).clone() for name in _VIEWS}
  acts = [torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32) for _ in range(K)]
  traj = bs.trajectory(K)
  first = []
  for t in range(K):
    bs.step(acts[t], out=traj.at(t))  # (the images go to the trajectory, not to the engine's own buffers)
    first.append((e.grid.clone(), e.avatar_state.clone()))
  assert int((traj.step_type == 0).sum()) > 0, 'the continuation never crossed an auto-reset'
  ts = bs.restore(bank, every, every)
  for name in _VIEWS:
    assert torch.equal(getattr(e, name), at_store[name]), f'{name} after the restore differs from the stored one'
  assert torch.equal(ts.step_type, at_store['step_type']) and torch.equal(ts.observation['RGB'], at_store['rgb'])
  for t in range(K):
    bs.step(acts[t])
    slot = traj.at(t)
    assert torch.equal(e.step_type, slot.step_type) and torch.equal(e.reward, slot.reward), t
    assert torch.equal(e.discount, slot.discount) and torch.equal(e.rgb, slot.observation['RGB']), t
    assert torch.equal(e.world_rgb, slot.observation['WORLD.RGB']), t
    for k, name in enumerate(bs._scalar_names):  # pylint: disable=protected-access
      assert torch.equal(e.scalar_obs[k], slot.observation[name]), (t, name)
    g, av = first[t]
    assert torch.equal(e.grid, g) and torch.equal(e.avatar_state, av), t
  # restored from the trajectory's run, continuing into a trajectory again gives the same slots
  bs.restore(bank, every, every)
  traj2 = bs.trajectory(K)
  for t in range(K):
    bs.step(acts[t], out=traj2.at(t))
  for name in traj.observation:
    assert torch.equal(traj.observation[name], traj2.observation[name]), name
  assert torch.equal(traj.step_type, traj2.step_type) and torch.equal(traj.reward, traj2.reward)
  bs.close()


# ---- 4: portability ---------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fam', FAMILIES)
def test_record_continues_identically_in_another_engine(fam):
  import torch
  from meltingpot_b200 import engine
  blob = _blob(fam)
  a = engine.Engine(blob, 8, device=0, seed=1)
  c = engine.Engine(blob, 33, device=0, seed=9, env_index_base=100)
  P, A = a.num_players, a.num_actions
  assert a.state_record_bytes == c.state_record_bytes and a.state_tag == c.state_tag
  gen = torch.Generator(device='cuda').manual_seed(2)
  a.reset(); c.reset()
  for _ in range(30):
    a.step(torch.randint(0, A, (8, P), generator=gen, device='cuda', dtype=torch.int32))
    c.step(torch.randint(0, A, (33, P), generator=gen, device='cuda', dtype=torch.int32))
  bank = torch.zeros((2, a.state_record_bytes), dtype=torch.uint8, device='cuda')
  a.store_states(bank, _index(2, {0: 3, 1: 5}))
  c.restore_states(bank, _index(33, {10: 0, 20: 0, 32: 1}))
  pairs = ((10, 3), (20, 3), (32, 5))
  for t in range(50):
    xa = torch.randint(0, A, (8, P), generator=gen, device='cuda', dtype=torch.int32)
    xc = torch.randint(0, A, (33, P), generator=gen, device='cuda', dtype=torch.int32)
    for j, s in pairs:
      xc[j] = xa[s]
    a.step(xa); c.step(xc)
    for j, s in pairs:
      for name in _VIEWS:
        va, vc = getattr(a, name), getattr(c, name)
        ga, gc = (va[:, s], vc[:, j]) if name == 'scalar_obs' else (va[s], vc[j])
        assert torch.equal(ga, gc), f'{name} of env {j} (record of env {s}) at step {t}'
  a.close(); c.close()


# ---- 5: variants ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('family', EV.NAMES)
def test_record_carries_its_variant(family):
  import torch
  from meltingpot_b200 import engine
  blobs = EV.blobs(family)
  B = 8
  assign = np.zeros(B, np.int64); assign[1] = 1
  mixed = engine.Engine(list(blobs), B, device=0, seed=SEED, env_variant=assign)
  homog = engine.Engine(blobs[1], B, device=0, seed=SEED)  # its env 1 runs as the mixed engine's env 1
  P, A = mixed.num_players, mixed.num_actions
  gen = torch.Generator(device='cuda').manual_seed(3)
  mixed.reset(); homog.reset()
  for _ in range(25):
    x = torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32)
    mixed.step(x); homog.step(x)
  bank = torch.zeros((2, mixed.state_record_bytes), dtype=torch.uint8, device='cuda')
  mixed.store_states(bank, _index(2, {0: 1}))
  ids = assign.copy(); ids[1] = 3
  mixed.set_env_variant(ids)   # env 1's next episode: variant 3; the second record carries that pending assignment
  mixed.store_states(bank, _index(2, {1: 1}))
  assert int(mixed.active_variant[4]) == 0
  mixed.restore_states(bank, _index(B, {4: 0, 5: 1}))
  torch.cuda.synchronize()
  assert mixed.active_variant.cpu().tolist()[4:6] == [1, 1]
  assert mixed.pending_variant.cpu().tolist()[4:6] == [1, 3]
  for t in range(40):  # env 4's episode (frame 25 at the store) ends at frame 40 and restarts under variant 1
    x = torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32)
    x[4] = x[1]
    mixed.step(x); homog.step(x)
    for name in _VIEWS:
      vm, vh = getattr(mixed, name), getattr(homog, name)
      gm, gh = (vm[:, 4], vh[:, 1]) if name == 'scalar_obs' else (vm[4], vh[1])
      assert torch.equal(gm, gh), f'{name} of the restored env 4 vs the variant-1 engine at step {t}'
  assert int(mixed.active_variant[4]) == 1 and int(mixed.active_variant[5]) == 3  # env 5 took its pending variant at the reset
  mixed.close(); homog.close()


# ---- 6: skips and refusals --------------------------------------------------------------------------------------------
def test_out_of_range_indices_and_untagged_rows_are_skipped(clean_up_blob):
  import torch
  from meltingpot_b200 import engine
  B = 12
  eng = engine.Engine(clean_up_blob, B, device=0, seed=SEED)
  P, A = eng.num_players, eng.num_actions
  gen = torch.Generator(device='cuda').manual_seed(4)
  eng.reset()
  for _ in range(10):
    eng.step(torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32))
  R = eng.state_record_bytes
  bank = torch.randint(0, 256, (6, R), generator=gen, device='cuda', dtype=torch.int32).to(torch.uint8)
  bank[4] = 0  # a never-written row
  before = bank.clone()
  eng.store_states(bank, torch.tensor([-1, B, 2**31 - 1, -7, -2**31, 2], dtype=torch.int32, device='cuda'))
  torch.cuda.synchronize()
  assert torch.equal(bank[:5], before[:5]), 'a store with an index outside 0..B-1 wrote its row'
  assert bytes(bank[5, :16].cpu().numpy()) == eng.state_tag
  views = {name: getattr(eng, name).clone() for name in _VIEWS}
  eng.restore_states(bank, torch.tensor([-1, 6, -5, 0, 4, 5, 7, 100, -1, 3, 1, 2], dtype=torch.int32, device='cuda'))
  torch.cuda.synchronize()
  for name in _VIEWS:
    now, was = getattr(eng, name), views[name]
    for b in range(B):
      n, w = (now[:, b], was[:, b]) if name == 'scalar_obs' else (now[b], was[b])
      if b == 5:
        src = (views[name][:, 2] if name == 'scalar_obs' else views[name][2])
        assert torch.equal(n, src), f'{name}: env 5 did not receive env 2\'s record'
      else:
        assert torch.equal(n, w), f'{name} of env {b} changed (index out of range or untagged row)'
  eng.close()


def test_refused_banks_touch_nothing(clean_up_blob):
  import torch
  from meltingpot_b200 import engine
  lib = engine.load_library()
  B = 8
  eng = engine.Engine(clean_up_blob, B, device=0, seed=SEED)
  eng.reset()
  R = eng.state_record_bytes
  idx_b = torch.arange(B, dtype=torch.int32, device='cuda')
  idx_2 = torch.arange(2, dtype=torch.int32, device='cuda')
  store = lambda bank, idx, n: lib.mp_state_store(eng._h, ctypes.c_void_p(idx), n, ctypes.c_void_p(bank), None)  # pylint: disable=protected-access
  restore = lambda bank, idx, n: lib.mp_state_restore(eng._h, ctypes.c_void_p(idx), ctypes.c_void_p(bank), n, 0, None)  # pylint: disable=protected-access

  def refused(match, call):
    torch.cuda.synchronize()
    snap, launches = eng.save_state(), eng.launch_count()
    with pytest.raises(ValueError, match=match):
      engine._check(call())  # pylint: disable=protected-access
    assert eng.launch_count() == launches, f'a refused call ({match}) launched a kernel'
    assert eng.save_state() == snap, f'a refused call ({match}) changed the state'

  big = torch.zeros((2 * R + 64,), dtype=torch.uint8, device='cuda')
  for what, call in (('store', store), ('restore', restore)):
    idx = idx_2 if what == 'store' else idx_b
    refused('aligned', lambda: call(big.data_ptr() + 1, idx.data_ptr(), 2))
    refused('null', lambda: call(None, idx.data_ptr(), 2))
    refused('null', lambda: call(big.data_ptr(), None, 2))
    refused('n_slots', lambda: call(big.data_ptr(), idx.data_ptr(), 0))
    refused('own buffers', lambda: call(eng.grid.data_ptr(), idx.data_ptr(), 1))
    host = torch.zeros((2 * R,), dtype=torch.uint8).pin_memory()
    refused('not device memory', lambda: call(host.data_ptr(), idx.data_ptr(), 2))
    host_idx = torch.zeros((B,), dtype=torch.int32).pin_memory()
    refused('not device memory', lambda: call(big.data_ptr(), host_idx.data_ptr(), 2))
    cudart = _cudart()
    ptr = ctypes.c_void_p()
    assert cudart.cudaMalloc(ctypes.byref(ptr), ctypes.c_size_t(2 * R)) == 0
    try:
      refused('past the end', lambda: call(ptr.value, idx.data_ptr(), 3))  # a bank one row too short
      engine._check(call(ptr.value, idx.data_ptr(), 2))  # exactly long enough: accepted  # pylint: disable=protected-access
      torch.cuda.synchronize()
    finally:
      cudart.cudaFree(ptr)
    if torch.cuda.device_count() > 1:
      other = torch.zeros((2 * R,), dtype=torch.uint8, device='cuda:1')
      refused('device 1', lambda: call(other.data_ptr(), idx.data_ptr(), 2))
  with pytest.raises(ValueError, match='flags'):
    engine._check(lib.mp_state_restore(eng._h, ctypes.c_void_p(idx_b.data_ptr()), ctypes.c_void_p(big.data_ptr()), 2, 6, None))  # pylint: disable=protected-access
  eng.close()


def test_restore_is_refused_once_peers_are_connected(clean_up_blob):
  import torch
  from meltingpot_b200 import engine
  for kind in ('exchange', 'gather_obs'):
    eng = engine.Engine(clean_up_blob, 8, device=0, seed=SEED)
    eng.reset()
    bank = torch.zeros((8, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
    eng.store_states(bank, torch.arange(8, dtype=torch.int32, device='cuda'))
    ptr = getattr(eng, f'{kind}_create')(0, 1)[0]
    getattr(eng, f'{kind}_connect')([ptr])
    launches = eng.launch_count()
    with pytest.raises(ValueError, match=f'mp_{kind}_connect'):
      eng.restore_states(bank, torch.arange(8, dtype=torch.int32, device='cuda'))
    assert eng.launch_count() == launches
    eng.store_states(bank, torch.arange(8, dtype=torch.int32, device='cuda'))  # storing stays possible
    eng.close()


def test_restore_is_refused_between_two_gpus_one_process(territory_blob):
  import torch
  from meltingpot_b200 import engine
  if torch.cuda.device_count() < 2:
    pytest.skip('needs 2 GPUs')
  B = 16
  ranks = [engine.Engine(territory_blob, B, device=r, seed=SEED, env_index_base=r * B) for r in range(2)]
  ptrs = [e.exchange_create(r, 2)[0] for r, e in enumerate(ranks)]
  engine.enable_peer_access(0, 1); engine.enable_peer_access(1, 0)
  for e in ranks:
    e.exchange_connect(ptrs)
  for r, e in enumerate(ranks):
    with torch.cuda.device(r):
      bank = torch.zeros((B, e.state_record_bytes), dtype=torch.uint8, device=f'cuda:{r}')
      with pytest.raises(ValueError, match='mp_exchange_connect'):
        e.restore_states(bank, torch.arange(B, dtype=torch.int32, device=f'cuda:{r}'))


def test_python_refusals(clean_up_blob, commons_blob):
  import torch
  from meltingpot_b200 import substrate
  bs = substrate.BatchedSubstrate(clean_up_blob, 6, seed=SEED)
  bs.reset()
  bank = bs.state_bank(4)
  with pytest.raises(ValueError, match='twice'):
    bs.store(bank, [0, 1], [2, 2])
  with pytest.raises(ValueError, match='twice'):
    bs.restore(bank, [3, 3], [0, 1])
  with pytest.raises(ValueError, match='lie in'):
    bs.store(bank, [6], [0])
  with pytest.raises(ValueError, match='lie in'):
    bs.store(bank, [0], [4])
  with pytest.raises(ValueError, match='lie in'):
    bs.restore(bank, [0], [-1])
  with pytest.raises(ValueError, match='no record'):
    bs.restore(bank, [0], [1])  # never written
  bs.store(bank, [0, 1], [0, 1])
  bs.restore(bank, [2, 3], [0, 0])  # fan-out of one record is fine
  other = substrate.BatchedSubstrate(commons_blob, 6, seed=SEED)
  other.reset()
  foreign = bs.state_bank(2)
  foreign[0, :16] = torch.tensor(list(other.engine.state_tag), dtype=torch.uint8)
  with pytest.raises(ValueError, match='no record'):
    bs.restore(foreign, [0], [0])
  with pytest.raises(ValueError, match='bank must be'):
    bs.engine.restore_states(bank.view(torch.int8), torch.zeros(6, dtype=torch.int32, device='cuda'))
  with pytest.raises(ValueError, match='slot_of_env'):
    bs.engine.restore_states(bank, torch.zeros(5, dtype=torch.int32, device='cuda'))
  bs.close(); other.close()


# ---- 7: host-async interplay ------------------------------------------------------------------------------------------
def test_restore_after_host_async_step_leaves_that_slot_alone(commons_blob):
  import torch
  from meltingpot_b200 import engine
  B = 20
  eng = engine.Engine(commons_blob, B, device=0, seed=SEED)
  twin = engine.Engine(commons_blob, B, device=0, seed=SEED)
  P, A = eng.num_players, eng.num_actions
  rng = np.random.default_rng(6)
  eng.reset(); twin.reset()
  bank = torch.zeros((B, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  for _ in range(15):
    x = np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)
    eng.step(torch.from_numpy(x).cuda()); twin.step(torch.from_numpy(x).cuda())
  eng.store_states(bank, torch.arange(B, dtype=torch.int32, device='cuda'))  # every env as of step 15
  for _ in range(10):
    x = np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)
    eng.step(torch.from_numpy(x).cuda()); twin.step(torch.from_numpy(x).cuda())
  out = eng.make_host_outputs()
  acts = eng.make_host_actions()
  acts.copy_(torch.from_numpy(np.ascontiguousarray(rng.integers(0, A, size=(B, P)), np.int32)))
  eng.step_host_async(acts, out, 0)
  eng.restore_states(bank, torch.arange(B, dtype=torch.int32, device='cuda'))  # before wait(0)
  eng.wait(0)
  twin.step(acts.cuda())
  torch.cuda.synchronize()
  assert torch.equal(out['rgb'], twin.rgb.cpu()) and torch.equal(out['world_rgb'], twin.world_rgb.cpu())
  assert torch.equal(out['reward'], twin.reward.cpu()) and torch.equal(out['step_type'], twin.step_type.cpu())
  assert torch.equal(out['discount'], twin.discount.cpu())
  assert not torch.equal(eng.rgb, twin.rgb), 'the restore did not change the images'
  eng.close(); twin.close()


# ---- 8: whole-batch snapshots carry the keys --------------------------------------------------------------------------
@pytest.mark.parametrize('fam', ['clean_up', 'territory__inside_out'])
def test_snapshot_after_a_clone_continues_identically(fam):
  import torch
  from meltingpot_b200 import engine
  blob = _blob(fam)
  B = 10
  eng = engine.Engine(blob, B, device=0, seed=SEED)
  P, A = eng.num_players, eng.num_actions
  gen = torch.Generator(device='cuda').manual_seed(8)
  eng.reset()
  for _ in range(12):
    eng.step(torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32))
  bank = torch.zeros((1, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
  eng.store_states(bank, torch.tensor([1], dtype=torch.int32, device='cuda'))
  eng.restore_states(bank, _index(B, {5: 0}))
  for _ in range(3):
    x = torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32)
    x[5] = x[1]
    eng.step(x)
  snap = eng.save_state()
  fresh = engine.Engine(blob, B, device=0, seed=SEED)
  fresh.load_state(snap)
  for t in range(50):
    x = torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32)
    x[5] = x[1]
    eng.step(x); fresh.step(x)
    for name in _VIEWS:
      assert torch.equal(getattr(eng, name), getattr(fresh, name)), f'{name} at step {t}'
    assert torch.equal(fresh.grid[5], fresh.grid[1]) and torch.equal(fresh.rgb[5], fresh.rgb[1]), f'clone left its source at {t}'
  eng.close(); fresh.close()
