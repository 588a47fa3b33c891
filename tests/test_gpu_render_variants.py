"""Render layouts, lane maps, render flags, batch-size edges and episode boundaries against the oracle.

The default configuration of each code path is covered by test_gpu_parity.py. These tests reach the others: every
render layout the engine's search can pick (and so every k_render instantiation the shipped substrates use), the
renderer's scheduler edges (no balanced round, one or two rounds, a cooperative tail that gives some CTAs two envs, no
tail), batch sizes that leave the step kernels' last CTA partly empty, both A/B lane maps, the general compositing path
for stacked sprites, partial render flags and the auto-reset / masked reset of every kernel family. Each variant is
compared with the oracle directly, or in lockstep (parity.lockstep) with the default engine that the same test
compares with the oracle at the same B, seed and actions.
"""

import numpy as np
import pytest

from tests import parity

pytestmark = pytest.mark.gpu

SUBSTRATES = [('clean_up', 7), ('commons_harvest__open', 7), ('commons_harvest__closed', 7),
              ('commons_harvest__partnership', 7), ('territory__rooms', 9), ('territory__open', 9),
              ('territory__inside_out', 5), ('coins', 2), ('coop_mining', 6)]
_IDS = [n for n, _ in SUBSTRATES]


def _blob(name, players):
  from meltingpot_b200 import substrates
  return substrates.load_blob(name, ('default',) * players)


def _sm_count():
  import torch
  return int(torch.cuda.get_device_properties(0).multi_processor_count)


def _plan(blob, **kw):
  from meltingpot_b200 import engine
  eng = engine.Engine(blob, 1, seed=1, **kw)
  plan = eng.render_plan()
  eng.close()
  return plan


def _layout(plan):
  return plan['teams'], plan['team_threads'] // 32, plan['wstrip_log2']


def _feasible_layouts(blob):
  """(feasible layouts with their render plans, infeasible layouts): every candidate of the engine's search is tried."""
  from meltingpot_b200 import engine
  ok, bad = {}, []
  for lay in engine.render_layout_candidates():
    try:
      ok[lay] = _plan(blob, render_layout=lay)
    except ValueError as e:
      assert 'mp_engine error -2' in str(e), f'{lay}: {e}'  # MP_E_UNSUPPORTED, never a launch
      bad.append(lay)
  return ok, bad


def _pixels_at(*steps):
  return lambda t: t in steps


# ---- 1. batch-size edges, default layout ---------------------------------------------------------------------------
@pytest.mark.parametrize('name,players', SUBSTRATES, ids=_IDS)
def test_batch_size_edges_match_the_oracle(name, players, oracle):
  # B relative to the SM count and to n_streams = SMs x teams decides the renderer's rounds and cooperative tail; B not
  # a multiple of 4 leaves the step kernels' last CTA partly empty.
  blob = _blob(name, players)
  sm = _sm_count()
  ns = sm * _plan(blob)['teams']
  sizes = sorted({1, 2, 3, 5, sm - 1, sm, sm + 1, ns - 1, ns, ns + 1, 2 * ns + sm + 7})
  for B in sizes:
    stats = parity.compare_batch(blob, oracle, num_envs=B, steps=8, seed=900 + B, action_seed=B,
                                 pixels_at=_pixels_at(0, 4, 8))
    assert stats['pixel_checks'] == 3, B


# ---- 2. every feasible render layout ---------------------------------------------------------------------------------
def test_layout_sweep_reaches_every_instantiation():
  # The shipped substrates all have 11-cell views (NCP = 3): k_render<4, *> needs a view wider than 12 cells and no
  # shipped substrate reaches it. NCW follows the map width and the strip height: <3,3> with 2-row strips, <3,4>
  # (clean_up, coop_mining) and <3,5> (territory__open) with 4-row strips.
  reached, counts = set(), {}
  for name, players in SUBSTRATES:
    blob = _blob(name, players)
    ok, _ = _feasible_layouts(blob)
    counts[name] = len(ok)
    assert _layout(_plan(blob)) in ok, name
    for lay, plan in ok.items():
      assert _layout(plan) == lay
      reached.add((plan['ncp'], plan['ncw']))
  print('feasible layouts per substrate', counts, 'instantiations', sorted(reached))
  assert {(3, 3), (3, 4), (3, 5)} <= reached


@pytest.mark.parametrize('name,players', SUBSTRATES, ids=_IDS)
def test_every_feasible_layout_matches_the_default(name, players, oracle):
  blob = _blob(name, players)
  sm = _sm_count()
  ok, bad = _feasible_layouts(blob)
  default = _layout(_plan(blob))
  assert default in ok and len(ok) + len(bad) == 50
  # per layout: B = 7 (cooperative tail only, 7 CTAs); n_streams + SM + 7 (one balanced round, then CTAs 0-6 render
  # two tail envs and the others one); 2 * n_streams (two rounds, no tail)
  by_size = {}
  for lay in ok:
    ns = sm * lay[0]
    for B in (7, ns + sm + 7, 2 * ns):
      by_size.setdefault(B, []).append(lay)
  for B, lays in sorted(by_size.items()):
    stats = parity.compare_batch(blob, oracle, num_envs=B, steps=4, seed=300 + B, action_seed=B, pixels_at=_pixels_at(0, 2, 4))
    assert stats['pixel_checks'] == 3
    plans = parity.lockstep(blob, B, 4, seed=300 + B, action_seed=B, variants=[dict(render_layout=lay) for lay in lays])
    assert [_layout(p) for p in plans] == lays


# ---- 3. lane maps ----------------------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,players', SUBSTRATES, ids=_IDS)
def test_lane_map_variants_match_the_default(name, players, oracle):
  import ctypes
  from meltingpot_b200 import engine
  blob = _blob(name, players)
  sm = _sm_count()
  B = sm + 7  # cooperative tail only: CTAs 0-6 render two envs, the others one
  plan = _plan(blob)
  parity.compare_batch(blob, oracle, num_envs=B, steps=6, seed=17, pixels_at=_pixels_at(0, 3, 6))
  plain = engine.MP_FLAG_DEFAULT | engine.MP_FLAG_DEBUG_PLAIN_LANE_MAP
  scatter = engine.MP_FLAG_DEFAULT | engine.MP_FLAG_DEBUG_SCATTER_LANE_MAP
  p_plain, p_scatter = parity.lockstep(blob, B, 6, seed=17, variants=[dict(flags=plain), dict(flags=scatter)])
  assert p_plain['lane_map_players'] == p_plain['lane_map_world'] == engine.LANE_MAP_PLAIN
  # the scattered colouring exists for some strip shapes only; otherwise the engine keeps its default dealing
  lib = engine.load_library()
  out = (ctypes.c_uint32 * 32)()
  eng = engine.Engine(blob, 1, seed=1)
  view_w, W = int(eng.buffers.rgb_w) // 8, int(eng.buffers.world_w) // 8
  eng.close()
  ncp, per_turn = -(-view_w // 4), 32 >> plan['wstrip_log2']  # cells per lane as mp_create deals them
  can = (lib.mp_debug_lane_map(8, view_w, 3 * view_w, ncp, 1, out) == 0 and
         lib.mp_debug_lane_map(1 << plan['wstrip_log2'], W, 3 * W, -(-W // per_turn), 1, out) == 0)
  if can:
    assert p_scatter['lane_map_players'] == p_scatter['lane_map_world'] == engine.LANE_MAP_SCATTER
  else:
    assert (p_scatter['lane_map_players'], p_scatter['lane_map_world']) == (plan['lane_map_players'], plan['lane_map_world'])
    assert p_scatter['lane_map_players'] % 16 == 1 and p_scatter['lane_map_world'] % 16 == 1
  print(name, 'scattered lane map built' if can else 'scattered lane map not possible: default dealing kept')


# ---- 4. general compositing path -------------------------------------------------------------------------------------
def _beam_heavy(t, B, P, A, rng):
  # moves and turns, with the fire actions (zap, clean, claim / paint, mine: ids 7 and up) taking 40 % between them, so
  # that beams, markings and overlays stack on resources, apples and dirt
  w = np.array([0.05] + [0.1] * 4 + [0.075] * 2 + [0.4 / max(A - 7, 1)] * max(A - 7, 0))[:A]
  return rng.choice(A, size=(B, P), p=w / w.sum())


@pytest.mark.parametrize('name,players', SUBSTRATES, ids=_IDS)
def test_no_premerge_general_compositing_matches_the_oracle(name, players, oracle):
  from meltingpot_b200 import blob as blob_lib, engine
  blob = _blob(name, players)
  flags = engine.MP_FLAG_DEFAULT | engine.MP_FLAG_DEBUG_NO_PREMERGE
  eng = engine.Engine(blob, 1, seed=1, flags=flags)
  pair, _ = eng.render_tables()
  n_sprites = int(blob_lib.unpack(blob)['meta'][12])
  assert pair.max() == 0 and pair.shape[0] == n_sprites == eng.render_plan()['atlas_sprites']  # no merged sprite
  eng.close()
  stats = parity.compare_batch(blob, oracle, num_envs=40, steps=100, seed=23, flags=flags, actions_fn=_beam_heavy,
                               pixels_every=2)
  assert stats['pixel_checks'] == 51
  parity.lockstep(blob, 40, 100, seed=23, actions_fn=_beam_heavy, variants=[dict(flags=flags)])


# ---- 5. partial render flags -----------------------------------------------------------------------------------------
@pytest.mark.parametrize('name,players', SUBSTRATES, ids=_IDS)
def test_partial_render_flags_match_the_oracle(name, players, oracle):
  from meltingpot_b200 import engine
  blob = _blob(name, players)
  B = _sm_count() + 7  # cooperative tail only: CTAs 0-6 render two envs, the others one
  for flags in (engine.MP_FLAG_RENDER_PLAYERS, engine.MP_FLAG_RENDER_WORLD, 0):
    # (compare_batch fills the images the flags leave out with a sentinel and checks they are never written)
    stats = parity.compare_batch(blob, oracle, num_envs=B, steps=6, seed=29, flags=flags, pixels_every=1)
    assert stats['pixel_checks'] == 7


def test_batched_substrate_without_world_rgb_matches_the_oracle(clean_up_blob, oracle):
  import torch
  from meltingpot_b200 import substrate
  B, seed = 9, 77
  sub = substrate.BatchedSubstrate(clean_up_blob, B, seed=seed, world_rgb=False)
  eng = sub.engine
  eng.world_rgb.fill_(0xA5)
  envs = [oracle.OracleEnv(clean_up_blob, seed + b) for b in range(B)]
  ts = sub.reset()
  for e in envs:
    e.reset()
  rng = np.random.default_rng(3)
  for t in range(4):
    assert 'WORLD.RGB' not in ts.observation
    torch.cuda.synchronize()
    rgb = ts.observation['RGB'].cpu().numpy()
    for b, e in enumerate(envs):
      np.testing.assert_array_equal(e.rgb(), rgb[b], err_msg=f'RGB step {t} env {b}')
      np.testing.assert_array_equal(e.rewards(), ts.reward[b].cpu().numpy(), err_msg=f'reward step {t} env {b}')
    assert bool((eng.world_rgb == 0xA5).all())
    a = rng.integers(0, sub.num_actions, (B, sub.num_players)).astype(np.int32)
    ts = sub.step(torch.from_numpy(a).cuda())
    for b, e in enumerate(envs):
      e.step(a[b])
  sub.close()


# ---- 6. auto-reset of every family -----------------------------------------------------------------------------------
def _episode_ends(blob):
  """(first step that can be LAST, interval between chances) from the blob's StochasticIntervalEpisodeEnding
  (ip0 minimumFramesPerEpisode, ip1 intervalLength): the component's counter is step + 1 and it may end the episode on
  a multiple of the interval once the minimum is reached."""
  from meltingpot_b200 import blob as blob_lib
  comps = blob_lib.unpack(blob)['comps']
  row = [c for c in comps if int(c[0]) == 18][0]  # MPB_C_STOCHASTIC_INTERVAL_EPISODE_ENDING
  minimum, interval = int(row[1]), int(row[2])
  return -(-(minimum + 1) // interval) * interval - 1, interval


def _resource_layout(blob):
  import torch
  from meltingpot_b200 import blob as blob_lib, compiler
  sec = blob_lib.unpack(blob)
  cells = torch.as_tensor(sec['tr_res'][:, 1].astype(np.int64), device='cuda')
  res_layer = compiler.family_params(sec)['RES_LAYER']
  return lambda eng: (eng.grid[:, res_layer][:, cells] != 0).cpu().numpy()


@pytest.mark.parametrize('name,players,B', [
    ('commons_harvest__open', 7, 256), ('territory__rooms', 9, 256), ('territory__inside_out', 5, 256),
    ('coins', 2, 512), ('coop_mining', 6, 256)])
def test_auto_reset_matches_the_oracle(name, players, B, oracle):
  blob = _blob(name, players)
  first, interval = _episode_ends(blob)
  steps = first + 4
  near = lambda t: any(abs(t - e) <= 3 for e in range(first, steps + 4, interval))
  redraws = []
  on_step = None
  if name == 'territory__inside_out':
    layout_of = _resource_layout(blob)
    prev = {}

    def on_step(t, eng):  # envs that auto-reset on step t draw a new resource layout
      cur = layout_of(eng)
      if t > 0:
        st = eng.step_type.cpu().numpy()
        for b in np.nonzero(st == 0)[0]:
          redraws.append(not np.array_equal(cur[b], prev['layout'][b]))
      prev['layout'] = cur

  stats = parity.compare_batch(blob, oracle, num_envs=B, steps=steps, seed=500, pixels_at=lambda t: near(t) or t % 100 == 0,
                               on_step=on_step)
  assert stats['lasts'] > 0 and stats['mids_after_restart'] > 0, stats
  assert all(near(t) for t in stats['last_steps']), stats['last_steps']  # the episode ends fall in the checked windows
  if name == 'territory__inside_out':
    assert len(redraws) > 0 and all(redraws), redraws
