"""The CUDA engine against the oracle on substrate variants the shipped blobs never reach (tests/variants.py).

Every 'parity' variant runs 64 envs through parity.compare_batch (every output of every env on every step, pixels
regularly); its reach predicate must hold on what the engine produced, and its outputs must differ from the stock
blob's on the same seed and actions. Every variant mp_create must refuse makes Engine(...) raise at create time and is
never stepped. The long-episode test runs territory__rooms past frame 65,535, where a 16-bit frame stamp wraps.
"""

import hashlib

import numpy as np
import pytest

from tests import parity
from tests import variants as V

pytestmark = pytest.mark.gpu

B = 64
SEED = 4242


def _fingerprint():
  h = hashlib.sha1()

  def on_step(t, eng):
    for name in ('reward', 'step_type', 'grid', 'avatar_state', 'event_count'):
      h.update(getattr(eng, name).cpu().numpy().tobytes())
    if t == 0:
      h.update(repr(tuple(eng.rgb.shape)).encode())
      h.update(eng.rgb.cpu().numpy().tobytes())
  return h, on_step


def _stock_fingerprint(variant, steps):
  import torch
  from meltingpot_b200 import engine
  blob = V.stock(variant.substrate, variant.players, variant.seed)
  eng = engine.Engine(blob, B, seed=SEED)
  rng = np.random.default_rng(0)
  h, on_step = _fingerprint()
  eng.reset()
  on_step(0, eng)
  for t in range(1, steps + 1):
    acts = rng.integers(0, eng.num_actions, size=(B, eng.num_players))
    eng.step(torch.from_numpy(np.ascontiguousarray(acts, np.int32)).cuda())
    on_step(t, eng)
  eng.close()
  return h.hexdigest()


def _alternative_layout(blob, default):
  """The first layout of the engine's search, other than `default`, that mp_create accepts for this blob."""
  from meltingpot_b200 import engine
  for lay in engine.render_layout_candidates():
    if lay == default:
      continue
    try:
      eng = engine.Engine(blob, 1, seed=1, render_layout=lay)
    except ValueError:
      continue
    eng.close()
    return lay
  raise AssertionError('no alternative render layout fits')


def _plan(blob, **kw):
  from meltingpot_b200 import engine
  eng = engine.Engine(blob, 1, seed=1, **kw)
  plan = eng.render_plan()
  eng.close()
  return plan


@pytest.mark.parametrize('name', [v.name for v in V.PARITY])
def test_variant_matches_the_oracle(name, oracle):
  variant = V.BY_NAME[name]
  blob = V.compile(name)
  sec = V.sections(blob)
  stats = V.new_stats(B, int(sec['meta'][12]))
  keep = V.probe_sprites(variant, blob)
  h, fingerprint = _fingerprint()
  cells = int(sec['meta'][1]) * int(sec['meta'][2])

  def on_step(t, eng):
    fingerprint(t, eng)
    V.observe(stats, t, eng.reward.cpu().numpy(), eng.step_type.cpu().numpy(),
              eng.grid.cpu().numpy().view(np.uint16)[:, :, :cells], eng.events.cpu().numpy(),
              eng.event_count.cpu().numpy(), keep)

  every = 2 if variant.steps <= 40 else 10
  out = parity.compare_batch(blob, oracle, num_envs=B, steps=variant.steps, seed=SEED, on_step=on_step,
                             pixels_at=lambda t: t % every == 0 or t == variant.steps)
  assert out['pixel_checks'] > 0
  assert variant.reach(stats, sec), f'{name}: the variant did not reach what it is for: {V.summary(stats)}'
  assert h.hexdigest() != _stock_fingerprint(variant, variant.steps), f'{name}: same outputs as the stock blob'

  if '/view_' in name:  # which renderer instantiation ran, at the default layout and at a forced alternative one
    g = V.view_geometry(blob)
    plan = _plan(blob)
    ncp = -(-g.width // 4)
    assert plan['ncp'] == max(3, ncp), (g, plan)
    if ncp == 4:
      assert (plan['ncp'], plan['ncw']) == (4, 5), plan
    default = (plan['teams'], plan['team_threads'] // 32, plan['wstrip_log2'])
    lay = _alternative_layout(blob, default)
    alt = _plan(blob, render_layout=lay)
    assert (alt['teams'], alt['team_threads'] // 32, alt['wstrip_log2']) == lay
    assert alt['ncp'] == plan['ncp'], (plan, alt)
    parity.compare_batch(blob, oracle, num_envs=B, steps=12, seed=SEED + 1, render_layout=lay, pixels_every=3)
    print(name, 'view', (g.width, g.height), 'k_render<%d,%d>' % (plan['ncp'], plan['ncw']), 'layouts', default, lay)


@pytest.mark.parametrize('name', [v.name for v in V.REFUSED if v.refused_by == 'engine'])
def test_variant_is_refused_at_create(name):
  from meltingpot_b200 import engine
  blob = V.compile(name)
  with pytest.raises(ValueError, match='mp_engine error -2'):  # MP_E_UNSUPPORTED, before anything is launched
    engine.Engine(blob, 4, seed=1)


@pytest.mark.parametrize('substrate,section', [('clean_up', 'cu_dirt'), ('commons_harvest__open', 'ch_apple'),
                                               ('territory__rooms', 'tr_res'), ('coins', 'co_coin'), ('coop_mining', 'cm_ore')])
def test_entity_table_short_or_off_the_map_is_refused_at_create(substrate, section):
  # The kernels read the first n rows of each entity table, and every table's cell column feeds a cell -> entity index.
  from meltingpot_b200 import blob as mpb, engine, substrates
  sec = mpb.unpack(substrates.load_blob(substrate))
  short = dict(sec)
  short[section] = sec[section][:-1]
  off_map = dict(sec)
  off_map[section] = sec[section].copy()
  off_map[section][-1, 1] = int(sec['meta'][1]) * int(sec['meta'][2])  # W * H: one past the last cell
  for bad, what in ((short, r'has \d+ values for'), (off_map, 'puts entity')):
    with pytest.raises(ValueError, match=f"mp_engine error -1: blob: section '{section}' {what}"):  # MP_E_INVALID
      engine.Engine(mpb.pack(bad), 4, seed=1)
  engine.Engine(mpb.pack(sec), 4, seed=1).close()


def test_territory_past_frame_65535_matches_the_oracle(oracle):
  # One episode of 70,000 frames. A resource's age (frames since its last state change) decides when its claim starts
  # paying (rewardDelay) and when the claim of a removed avatar is released (5 frames); past frame 65,535 a 16-bit
  # frame stamp would make every new claim pay at once. Avatars never zap, so all nine stay on the map and keep claiming.
  import os
  import torch
  from meltingpot_b200 import compiler, engine
  blob = V.compile_variant(V.LONG_EPISODE)
  sec = V.sections(blob)
  assert int(sec['meta'][7]) == 70000
  n_envs, steps, chunk = 16, 65536 + 300, 4096
  threads = min(4, os.cpu_count() or 1)  # 16 small envs per step: more host threads cost more than they save
  eng = engine.Engine(blob, n_envs, seed=SEED, flags=0)  # no rendering: the state transition alone
  batch = oracle.OracleBatch(blob, n_envs, seed=SEED)
  bf = eng.buffers
  shapes = dict(P=eng.num_players, L=int(bf.grid_layers), cells=int(bf.grid_cells), n_scalar=eng.num_scalar_obs,
                rgb=(1, 1), world=(1, 1))
  max_ev = int(bf.max_events)
  no_zap = np.nonzero(sec['action_table'][:, compiler.ACTION_FIELDS['fireZap']] == 0)[0].astype(np.int32)
  rng = np.random.default_rng(11)
  totals = dict(checks=0, rewards_late=0.0, claims_late=0)

  def compare(t):
    torch.cuda.synchronize()
    want = batch.dump(threads, shapes, pixels=False, max_events=max_ev, kinds=())
    got = dict(reward=eng.reward.cpu().numpy(), discount=eng.discount.cpu().numpy(), step_type=eng.step_type.cpu().numpy(),
               avatars=eng.avatar_state.cpu().numpy(), grid=eng.grid.cpu().numpy().view(np.uint16)[:, :, :shapes['cells']],
               n_events=eng.event_count.cpu().numpy())
    for k, v in got.items():
      if not np.array_equal(v, want[k]):
        bad = np.argwhere(v != want[k])
        raise AssertionError(f'{k} differs at step {t}: {len(bad)} mismatches, first at {bad[0].tolist()}: '
                             f'gpu {v[tuple(bad[0])]} oracle {want[k][tuple(bad[0])]}')
    assert np.array_equal(parity._event_keys(eng.events.cpu().numpy(), got['n_events']),  # pylint: disable=protected-access
                          parity._event_keys(want['events'], want['n_events'])), f'events differ at step {t}'  # pylint: disable=protected-access
    totals['checks'] += 1
    if t > 65536:
      totals['rewards_late'] += float(want['reward'].sum())
      totals['claims_late'] += int(((want['events'][..., 0] == 4) & (np.arange(max_ev)[None] < want['n_events'][:, None])).sum())
    assert (got['step_type'] == (0 if t == 0 else 1)).all(), f'the episode ended at step {t}'

  eng.reset()
  compare(0)
  for base in range(1, steps + 1, chunk):
    n = min(chunk, steps + 1 - base)
    acts = no_zap[rng.integers(0, len(no_zap), size=(n, n_envs, eng.num_players))]
    dev = torch.from_numpy(acts).cuda()
    for i in range(n):
      t = base + i
      eng.step(dev[i])
      batch.step_actions(acts[i], threads)
      if t % chunk == 0 or t >= 65500:
        compare(t)
  eng.close()
  batch.close()
  print('long episode', totals)
  assert totals['checks'] == 1 + 15 + (steps - 65500 + 1)
  assert totals['claims_late'] > 0 and totals['rewards_late'] > 0, totals
