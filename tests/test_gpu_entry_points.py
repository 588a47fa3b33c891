"""The C ABI's other entry points against the oracle, bit for bit, on every kernel family.

The parity suites reach the kernels through mp_run's plain steps and resets on the current stream and read the engine's own
buffers. These tests run the same kernels through the calls that use other buffers, streams or launch sequences: the
pipelined host path (mp_step_host_async / mp_wait), split launches (mp_step_state / mp_render), host-buffer events at
B > 1, snapshots across episode boundaries and render layouts, caller-created streams, and Philox keys whose high word
changes within a batch. Short episodes come from the hard_cap_40 variants of tests/variants.py: LAST falls on steps
40, 81, 122, ... of every env, so each run below crosses an auto-reset within a few dozen steps.
"""

import functools
import os

import numpy as np
import pytest

from tests import parity
from tests import variants as V

pytestmark = pytest.mark.gpu

FAMILIES = ['clean_up', 'commons_harvest', 'territory', 'coins', 'coop_mining']
THREADS = os.cpu_count() or 1


def _cap40(fam):
  return V.compile(f'{fam}/hard_cap_40')


@functools.lru_cache(maxsize=None)
def _inside_out_cap40():
  """territory__inside_out (a 'choice' resource layout drawn per env and episode) with the hard_cap_40 edits."""
  return V.compile_variant(V.BY_NAME['territory/hard_cap_40']._replace(
      name='territory/inside_out_hard_cap_40', substrate='territory__inside_out', players=5))


def _stock(name, players):
  from meltingpot_b200 import substrates
  return substrates.load_blob(name, ('default',) * players)


def _acts(rng, eng):
  return np.ascontiguousarray(rng.integers(0, eng.num_actions, size=(eng.num_envs, eng.num_players)), np.int32)


def _dump(batch, eng, pixels, kinds=('rgb', 'world')):
  return batch.dump(THREADS, parity.shapes_of(eng), pixels=pixels, max_events=int(eng.buffers.max_events), kinds=kinds)


# ---- 1. pipelined host path ------------------------------------------------------------------------------------------
def _separate_scalars(eng):
  """A host output set with the four scalar pointers and no scalar_block (mp_step_host_async's per-pointer copies)."""
  import torch
  B, P, ns = eng.num_envs, eng.num_players, max(eng.num_scalar_obs, 1)
  out = {k: v for k, v in eng.make_host_outputs().items() if k in ('rgb', 'world_rgb')}
  out['reward'] = torch.full((B, P), np.nan, dtype=torch.float64).pin_memory()
  out['discount'] = torch.full((B,), np.nan, dtype=torch.float64).pin_memory()
  out['step_type'] = torch.full((B,), -7, dtype=torch.int64).pin_memory()
  out['scalar_obs'] = torch.full((ns, B, P), np.nan, dtype=torch.float64).pin_memory()
  return out


def _no_images(eng):
  """A full host output set whose image pointers are passed as NULL; the buffers themselves hold a sentinel."""
  out = eng.make_host_outputs()
  for k in ('rgb', 'world_rgb'):
    out[k].fill_(parity._SENTINEL)  # pylint: disable=protected-access
  return out, {k: (None if k in ('rgb', 'world_rgb') else v) for k, v in out.items()}


def _pipelined(blob, oracle, B, steps, seed, outputs='block'):
  """Steps an engine with mp_step_host_async, alternating slots 0 and 1 with one host output set per slot, and an
  OracleBatch with the same actions. After each wait(slot), every host output of that slot's step must equal the
  oracle at that step, images included. Step t+1 is enqueued before wait(t), so each step's kernels run while the
  previous step's outputs are being copied out. `steps` is even: the last step runs on slot 1."""
  from meltingpot_b200 import engine
  assert steps % 2 == 0
  eng = engine.Engine(blob, B, seed=seed)
  batch = oracle.OracleBatch(blob, B, seed=seed)
  if outputs == 'block':
    sets = [eng.make_host_outputs() for _ in range(2)]
    passed = sets
  elif outputs == 'pointers':
    sets = passed = [_separate_scalars(eng) for _ in range(2)]
  else:
    sets, passed = zip(*[_no_images(eng) for _ in range(2)])
  acts_host = [eng.make_host_actions() for _ in range(2)]
  rng = np.random.default_rng(seed)
  eng.reset()
  parity.check_outputs(parity.device_outputs(eng), _dump(batch, eng, True), 'reset')
  lasts = 0

  def check(slot, t, want):
    eng.wait(slot)
    got = parity.host_outputs(passed[slot], eng.num_scalar_obs)
    assert ('rgb' in got) == (outputs != 'none')
    parity.check_outputs(got, want, f'step {t} (slot {slot})')
    for k in ('rgb', 'world_rgb'):
      if outputs == 'none':
        assert bool((sets[slot][k] == parity._SENTINEL).all()), f'step {t}: a NULL image was written'  # pylint: disable=protected-access

  want = None
  for t in range(1, steps + 1):
    slot = (t + 1) % 2
    a = _acts(rng, eng)
    acts_host[slot].numpy()[:] = a  # this slot's previous call was waited for one iteration ago
    eng.step_host_async(acts_host[slot], passed[slot], slot)
    if want is not None:
      check(1 - slot, t - 1, want)
    batch.step_actions(a, THREADS)
    want = _dump(batch, eng, True)
    lasts += int((want['step_type'] == 2).sum())
  check(1, steps, want)
  # After a slot-1 call mp_buffers holds that step's scalars and state, and the images of the last slot-0 step.
  parity.check_outputs(parity.device_outputs(eng, kinds=()), want, f'device buffers after step {steps} (slot 1)')
  if outputs != 'none':
    np.testing.assert_array_equal(eng.rgb.cpu().numpy(), sets[0]['rgb'].numpy())
    np.testing.assert_array_equal(eng.world_rgb.cpu().numpy(), sets[0]['world_rgb'].numpy())
  eng.close()
  batch.close()
  return lasts


@pytest.mark.parametrize('fam', FAMILIES + ['territory__inside_out'])
def test_pipelined_host_path_matches_the_oracle(fam, oracle):
  # B = 257 is not a multiple of 4 and leaves the renderer a cooperative tail.
  blob = _stock('territory__inside_out', 5) if fam == 'territory__inside_out' else _cap40(fam)
  lasts = _pipelined(blob, oracle, 257, 100, seed=61)
  assert lasts == (0 if fam == 'territory__inside_out' else 2 * 257)


@pytest.mark.parametrize('outputs', ['pointers', 'none'])
def test_pipelined_host_path_output_variants(outputs, oracle):
  # 'pointers': reward / discount / step_type / scalar_obs each through their own pointer, at their offsets in the
  # slot's scalar staging; 'none': the image pointers are NULL and only the scalars are copied.
  assert _pipelined(_cap40('commons_harvest'), oracle, 257, 44, seed=62, outputs=outputs) == 257


# ---- 2. a refused async call -----------------------------------------------------------------------------------------
def test_refused_async_call_steps_no_env(oracle):
  def on_step(t, eng):
    if t != 5:
      return
    acts = eng.make_host_actions()
    before = eng.save_state()
    with pytest.raises(ValueError, match='events'):
      eng.step_host_async(acts, eng.make_host_outputs(events=True), 0)
    assert eng.save_state() == before, 'a refused mp_step_host_async changed the state'
    with pytest.raises(ValueError, match='slot'):
      eng.step_host_async(acts, eng.make_host_outputs(), 2)
    assert eng.save_state() == before, 'a refused mp_step_host_async changed the state'
  # the oracle did not take the refused steps: every later step still matches
  stats = parity.compare_batch(_cap40('territory'), oracle, num_envs=64, steps=45, seed=63, pixels_every=5, on_step=on_step)
  assert stats['last_steps'] == [40]


# ---- 3. slot 0's copy-out against later renders into the same images -------------------------------------------------
@functools.lru_cache(maxsize=1)
def _clean_up_after_one_step(oracle, B, seed, acts_bytes):
  blob = _stock('clean_up', 7)
  batch = oracle.OracleBatch(blob, B, seed=seed)
  acts = np.frombuffer(acts_bytes, np.int32).reshape(B, 7)
  batch.step_actions(acts, THREADS)
  from meltingpot_b200 import engine
  eng = engine.Engine(blob, 1, seed=seed)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)  # (max_events does not depend on B)
  eng.close()
  want = batch.dump(THREADS, shapes, pixels=True, max_events=max_ev)
  batch.close()
  return want


@pytest.mark.parametrize('later', ['step', 'step_host', 'render', 'reset', 'load_state'])
def test_slot0_copy_is_not_overwritten_by_a_later_render(later, oracle):
  # Slot 0 renders into the engine's own images and copies them out on the engine's copy stream. Each call below
  # renders into the same images on the caller's stream before mp_wait(0): the host copy must still hold step 1.
  # (2048 clean_up envs: the copy is about 0.6 GB, the next render a fraction of a millisecond.)
  import torch
  from meltingpot_b200 import engine
  blob = _stock('clean_up', 7)
  B, seed = 2048, 64
  eng = engine.Engine(blob, B, seed=seed)
  rng = np.random.default_rng(4)
  a1, a2 = _acts(rng, eng), _acts(rng, eng)
  want = _clean_up_after_one_step(oracle, B, seed, a1.tobytes())
  out0 = eng.make_host_outputs()
  h1, h2 = eng.make_host_actions(), eng.make_host_actions()
  h1.numpy()[:] = a1
  h2.numpy()[:] = a2
  d2 = torch.from_numpy(a2).cuda()
  mask = torch.from_numpy((np.arange(B) % 2).astype(np.uint8)).cuda()
  scalars_only = eng.make_host_outputs(rgb=False, world_rgb=False)
  eng.reset()
  snap = eng.save_state()
  torch.cuda.synchronize()
  eng.step_host_async(h1, out0, 0)
  if later == 'step':
    eng.step(d2)
  elif later == 'step_host':
    eng.step_host(h2, scalars_only)
  elif later == 'render':
    eng.step_state(d2)
    eng.render()
  elif later == 'reset':
    eng.reset(mask)
  else:
    eng.load_state(snap)
  eng.wait(0)
  parity.check_outputs(parity.host_outputs(out0, eng.num_scalar_obs), want, f'slot 0 step 1, then {later}')
  eng.close()


# ---- 4. split launches -----------------------------------------------------------------------------------------------
@pytest.mark.parametrize('fam', ['clean_up', 'coins'])
def test_split_launches_match_the_oracle(fam, oracle):
  import torch
  from meltingpot_b200 import engine
  blob = _cap40(fam)
  B, seed = 96, 65
  eng = engine.Engine(blob, B, seed=seed)
  batch = oracle.OracleBatch(blob, B, seed=seed)
  rng = np.random.default_rng(seed)
  eng.reset()
  t = 0
  while t < 45:
    images = (eng.rgb.clone(), eng.world_rgb.clone())
    for _ in range(3):  # mp_step_state: the state advances, the images stay
      a = _acts(rng, eng)
      eng.step_state(torch.from_numpy(a).cuda())
      batch.step_actions(a, THREADS)
      t += 1
      parity.check_outputs(parity.device_outputs(eng, kinds=()), _dump(batch, eng, False), f'step_state, step {t}')
      assert torch.equal(eng.rgb, images[0]) and torch.equal(eng.world_rgb, images[1]), f'step_state rendered at step {t}'
    eng.render()
    parity.check_outputs(parity.device_outputs(eng), _dump(batch, eng, True), f'render after step {t}')
    rendered = (eng.rgb.clone(), eng.world_rgb.clone())
    eng.render()
    torch.cuda.synchronize()
    assert torch.equal(eng.rgb, rendered[0]) and torch.equal(eng.world_rgb, rendered[1]), f'second render at step {t}'
  # a step rendered without WORLD.RGB, then a full render: WORLD.RGB of the current state, not the stale frame
  eng.set_flags(engine.MP_FLAG_RENDER_PLAYERS)
  a = _acts(rng, eng)
  eng.step(torch.from_numpy(a).cuda())
  batch.step_actions(a, THREADS)
  eng.set_flags(engine.MP_FLAG_DEFAULT)
  eng.render()
  parity.check_outputs(parity.device_outputs(eng), _dump(batch, eng, True), f'full render after a players-only step {t + 1}')
  eng.close()
  batch.close()


# ---- 5. host-buffer events at B > 1 ----------------------------------------------------------------------------------
def _zap_heavy(t, B, P, A, rng):
  from tests import test_gpu_parity
  return test_gpu_parity._zap_heavy(t, B, P, A, rng)  # pylint: disable=protected-access


def _mine_heavy(t, B, P, A, rng):
  from tests import test_gpu_parity
  return test_gpu_parity._mine_heavy(t, B, P, A, rng)  # pylint: disable=protected-access


@pytest.mark.parametrize('name,players,policy', [('territory__rooms', 9, _zap_heavy), ('coop_mining', 6, _mine_heavy)],
                         ids=['territory__rooms', 'coop_mining'])
def test_host_buffer_events_match_the_oracle(name, players, policy, oracle):
  import torch
  from meltingpot_b200 import engine
  blob = _stock(name, players)
  B, seed = 64, 66
  eng = engine.Engine(blob, B, seed=seed)
  batch = oracle.OracleBatch(blob, B, seed=seed)
  out = eng.make_host_outputs(events=True)
  out['events'].fill_(-1)
  out['event_count'].fill_(-1)
  rng = np.random.default_rng(seed)
  eng.reset_host(out)
  parity.check_outputs(parity.host_outputs(out, eng.num_scalar_obs), _dump(batch, eng, True), 'reset_host')
  events = 0
  for t in range(1, 61):
    a = np.ascontiguousarray(policy(t, B, eng.num_players, eng.num_actions, rng), np.int32)
    eng.step_host(torch.from_numpy(a), out)
    batch.step_actions(a, THREADS)
    want = _dump(batch, eng, True)
    parity.check_outputs(parity.host_outputs(out, eng.num_scalar_obs), want, f'step_host step {t}')
    events += int(want['n_events'].sum())
  assert events > 100, events
  eng.close()
  batch.close()


# ---- 6. snapshots across episode boundaries, masked resets and render layouts ----------------------------------------
@pytest.mark.parametrize('fam', FAMILIES + ['territory__inside_out'])
def test_snapshot_restores_into_another_layout_and_matches_the_oracle(fam, oracle):
  # One script: steps 1-45, a masked reset of every third env, steps 46-90 (LAST on 40 and 81, and on 85 for the
  # masked envs). Engine A runs it against a list of OracleEnv (an OracleBatch has no masked reset) and is
  # snapshotted at the LAST step 40, the FIRST step 41 and 5 steps after the masked reset. Each snapshot is loaded
  # into a fresh engine built with another render layout, which then runs the rest of the script against freshly
  # replayed oracle envs, every op checked, and must end where A ended. On territory__inside_out the grid comparison
  # pins each restored env's drawn resource layout until its next episode, and the new draw after it.
  import torch
  from meltingpot_b200 import engine
  from tests.test_gpu_param_envelope import _alternative_layout
  blob = _inside_out_cap40() if fam == 'territory__inside_out' else _cap40(fam)
  B, seed = 64, 67
  a_eng = engine.Engine(blob, B, seed=seed)
  plan = a_eng.render_plan()
  alt = _alternative_layout(blob, (plan['teams'], plan['team_threads'] // 32, plan['wstrip_log2']))
  shapes, max_ev = parity.shapes_of(a_eng), int(a_eng.buffers.max_events)
  rng = np.random.default_rng(seed)
  mask = (np.arange(B) % 3 == 0).astype(np.uint8)
  ops = [('step', _acts(rng, a_eng)) for _ in range(45)] + [('reset', mask)] + [('step', _acts(rng, a_eng)) for _ in range(45)]
  snap_at = (40, 41, 51)  # ops done: step 40, step 41, the masked reset + 5 steps
  pixels_at = {40, 41, 45, 46, 47, 51, 81, 82, 85, 86, 87, 91}

  def apply(eng, envs, op):
    kind, arg = op
    if kind == 'step':
      if eng is not None:
        eng.step(torch.from_numpy(arg).cuda())
      for b, e in enumerate(envs):
        e.step(arg[b])
    else:
      if eng is not None:
        eng.reset(torch.from_numpy(arg).cuda())
      for b in np.nonzero(arg)[0]:
        envs[b].reset()

  def new_envs(n_ops):
    envs = [oracle.OracleEnv(blob, seed + b) for b in range(B)]
    for e in envs:
      e.reset()
    for op in ops[:n_ops]:
      apply(None, envs, op)
    return envs

  def check(eng, envs, done, where):
    px = done in pixels_at or done % 10 == 0
    got = parity.device_outputs(eng, ('rgb', 'world') if px else ())
    parity.check_outputs(got, parity.env_dump(envs, shapes, px, max_ev), f'{where}, {done} ops done')
    return got

  def follow(eng, envs, start, where):
    for i in range(start, len(ops)):
      apply(eng, envs, ops[i])
      check(eng, envs, i + 1, where)
      if i + 1 in snap_at and eng is a_eng:
        snaps[i + 1] = eng.save_state()

  snaps = {}
  a_eng.reset()
  a_envs = new_envs(0)
  check(a_eng, a_envs, 0, 'A')
  follow(a_eng, a_envs, 0, 'A')
  for done in snap_at:
    b_eng = engine.Engine(blob, B, seed=seed, render_layout=alt)
    b_eng.load_state(snaps[done])
    envs = new_envs(done)
    check(b_eng, envs, done, f'B (layout {alt}) loaded after op {done}')
    follow(b_eng, envs, done, f'B (layout {alt}) from op {done}')
    for name in parity._STATE_VIEWS + ('rgb', 'world_rgb'):  # pylint: disable=protected-access
      assert torch.equal(getattr(b_eng, name), getattr(a_eng, name)), f'{name}: B from op {done} did not end where A did'
    b_eng.close()
  a_eng.close()


# ---- 7. caller-created streams ---------------------------------------------------------------------------------------
def test_compare_batch_on_a_caller_stream(oracle):
  import torch
  s = torch.cuda.Stream()
  with torch.cuda.stream(s):
    stats = parity.compare_batch(_cap40('coop_mining'), oracle, num_envs=130, steps=45, seed=68, pixels_every=3)
  assert stats['last_steps'] == [40]


def test_two_engines_in_flight_on_two_streams(oracle):
  import torch
  from meltingpot_b200 import engine
  runs = []
  for fam, B, seed in (('clean_up', 200, 69), ('territory', 150, 70)):
    blob = _cap40(fam)
    runs.append(dict(eng=engine.Engine(blob, B, seed=seed), batch=oracle.OracleBatch(blob, B, seed=seed),
                     stream=torch.cuda.Stream(), rng=np.random.default_rng(seed), fam=fam))
  for r in runs:
    r['eng'].reset(stream=r['stream'])
  for t in range(1, 41):
    for r in runs:  # both steps are enqueued before anything synchronises
      r['acts'] = _acts(r['rng'], r['eng'])
      with torch.cuda.stream(r['stream']):
        dev = torch.from_numpy(r['acts']).pin_memory().cuda(non_blocking=True)
        r['eng'].step(dev, stream=r['stream'])
    for r in runs:
      r['batch'].step_actions(r['acts'], THREADS)
      px = t % 4 == 0
      parity.check_outputs(parity.device_outputs(r['eng'], ('rgb', 'world') if px else ()), _dump(r['batch'], r['eng'], px),
                           f'{r["fam"]} step {t}')
  for r in runs:
    assert (r['batch'].dump(THREADS, parity.shapes_of(r['eng']), max_events=int(r['eng'].buffers.max_events))['step_type'] == 2).all()
    r['eng'].close()
    r['batch'].close()


# ---- 8. the high word of the Philox key ------------------------------------------------------------------------------
@pytest.mark.parametrize('fam', ['clean_up', 'coop_mining'])
@pytest.mark.parametrize('seed', [2**32 - 32, 2**64 - 16], ids=['crosses_2^32', 'wraps_2^64'])
def test_rng_keys_crossing_the_high_word_match_the_oracle(fam, seed, oracle):
  # keys seed + b: the high word changes half way through the batch (2^32 - 32 + b) or the key wraps to 0 (2^64 - 16 + b)
  stats = parity.compare_batch(_cap40(fam), oracle, num_envs=64, steps=42, seed=seed, pixels_at=lambda t: t in (0, 1, 20, 40, 41))
  assert stats['pixel_checks'] == 5 and stats['last_steps'] == [40]


def test_rng_key_high_word_changes_the_rollout():
  # Independent of the oracle: keys k and k + 2^32 differ only in the high word, so a key whose high word the kernels
  # dropped (in the oracle too) would give both the same rollout.
  import torch
  from meltingpot_b200 import engine
  blob = _stock('clean_up', 7)
  B, k = 8, 12345
  engines = [engine.Engine(blob, B, seed=k), engine.Engine(blob, B, seed=k + 2**32)]
  rng = np.random.default_rng(0)
  history = [[], []]
  for e in engines:
    e.reset()
  for t in range(12):
    for e, h in zip(engines, history):
      torch.cuda.synchronize()
      h.append(e.grid.cpu().numpy().reshape(B, -1).copy())
    a = torch.from_numpy(_acts(rng, engines[0])).cuda()
    for e in engines:
      e.step(a)
  lo, hi = np.stack(history[0], 1), np.stack(history[1], 1)
  for b in range(B):
    assert not np.array_equal(lo[b], hi[b]), f'env {b}: keys {k + b} and {k + b + 2**32} gave the same rollout'
  for e in engines:
    e.close()
