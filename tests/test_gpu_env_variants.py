"""Heterogeneous batches: every env of one engine under its own variant of the substrate parameters (mp_create_variants).

Env b of a mixed batch must equal, byte for byte, env b of a homogeneous batch built from its variant's blob with the
same seed and env_index_base, and so env b of the CPU oracle run on that blob. The variants (tests/env_variants.py)
share a 40-frame episode cap, so every run of more than 40 steps crosses an auto-reset.
"""

import os

import numpy as np
import pytest

from tests import env_variants as EV
from tests import parity
from tests import variants as V

pytestmark = pytest.mark.gpu

SEED = 29
_VIEWS = ('reward', 'discount', 'step_type', 'scalar_obs', 'avatar_state', 'grid', 'event_count', 'timestep_packed', 'rgb',
          'world_rgb')


def _sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _actions(rng, B, P, A):
  import torch
  return torch.from_numpy(rng.integers(0, A, size=(B, P)).astype(np.int32)).cuda()


class _MixedOracle:
  """The oracle of a mixed batch: per variant, one OracleBatch over the env range that holds its envs (env b keyed
  seed + b), of which the rows of the variant's own envs are kept."""

  def __init__(self, oracle, blobs, assign, seed):
    self.assign = np.asarray(assign)
    self.parts = []
    for v, blob in enumerate(blobs):
      idx = np.flatnonzero(self.assign == v)
      if len(idx):
        lo, hi = int(idx[0]), int(idx[-1]) + 1
        self.parts.append((v, lo, hi, idx, oracle.OracleBatch(blob, hi - lo, seed=seed + lo)))
    self.threads = os.cpu_count() or 1

  def step(self, acts):
    for _, lo, hi, _, batch in self.parts:
      batch.step_actions(acts[lo:hi], self.threads)

  def dump(self, shapes, pixels, max_events, kinds=('rgb', 'world')):
    out = None
    for _, lo, _, idx, batch in self.parts:
      d = batch.dump(self.threads, shapes, pixels=pixels, max_events=max_events, kinds=kinds)
      if out is None:
        B = len(self.assign)
        out = {k: np.zeros((v.shape[0], B) + v.shape[2:] if k == 'scalar_obs' else (B,) + v.shape[1:], v.dtype) for k, v in d.items()}
      for k, v in d.items():
        if k == 'scalar_obs':
          out[k][:, idx] = v[:, idx - lo]
        else:
          out[k][idx] = v[idx - lo]
      del d
    return out

  def close(self):
    for part in self.parts:
      part[-1].close()


@pytest.mark.parametrize('layout', ['blocks', 'interleaved'])
@pytest.mark.parametrize('family', EV.NAMES)
def test_every_env_of_a_mixed_batch_matches_the_oracle(oracle, family, layout):
  from meltingpot_b200 import engine
  import torch
  B, steps = 2048, 45
  blobs = EV.blobs(family)
  assign = getattr(EV, layout)(B, len(blobs))
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  assert eng.num_variants == 4
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  ref = _MixedOracle(oracle, blobs, assign, SEED)
  rng = np.random.default_rng(3)
  eng.reset()
  lasts = 0
  for t in range(steps + 1):
    if t:
      acts = _actions(rng, B, eng.num_players, eng.num_actions)
      eng.step(acts)
      ref.step(acts.cpu().numpy())
    px = t in (0, 20, 41, 45)
    got = parity.device_outputs(eng, ('rgb', 'world') if px else ())
    parity.check_outputs(got, ref.dump(shapes, px, max_ev), f'{family} {layout} step {t}')
    lasts += int((got['step_type'] == 2).sum())
  assert lasts == B  # every env crossed the 40-frame cap
  assert torch.equal(eng.active_variant.cpu(), torch.from_numpy(assign.astype(np.uint8)))
  ref.close()
  eng.close()


def _lockstep(blobs, mixed_blobs, assign, B, steps, seed=SEED, env_index_base=0):
  """Steps a mixed engine and one homogeneous engine per variant with the same actions; env b of the mixed engine must
  equal env b of its variant's engine in every view and event. Returns, per pair of variants, whether their engines
  ever differed."""
  import torch
  from meltingpot_b200 import engine
  mixed = engine.Engine(list(mixed_blobs), B, seed=seed, env_index_base=env_index_base, env_variant=assign)
  homo = [engine.Engine(b, B, seed=seed, env_index_base=env_index_base) for b in blobs]
  rows = [torch.from_numpy(np.flatnonzero(assign == v)).cuda() for v in range(len(blobs))]
  n = len(blobs)
  differ = np.zeros((n, n), bool)
  rng = np.random.default_rng(5)

  def check(t):
    for v, h in enumerate(homo):
      if not len(rows[v]):
        continue
      for name in _VIEWS:
        g, w = getattr(mixed, name), getattr(h, name)
        if name == 'scalar_obs':
          g, w = g[:, rows[v]], w[:, rows[v]]
        else:
          g, w = g[rows[v]], w[rows[v]]
        assert torch.equal(g, w), f'{name} of variant {v} envs differs from its homogeneous engine at step {t} (B={B})'
      ge = parity._event_keys(mixed.events.cpu().numpy(), mixed.event_count.cpu().numpy())[rows[v].cpu().numpy()]
      we = parity._event_keys(h.events.cpu().numpy(), h.event_count.cpu().numpy())[rows[v].cpu().numpy()]
      assert np.array_equal(ge, we), f'events of variant {v} envs differ at step {t} (B={B})'
    for i in range(n):
      for j in range(i + 1, n):
        d = any(not torch.equal(getattr(homo[i], k), getattr(homo[j], k)) for k in ('reward', 'grid', 'avatar_state', 'event_count'))
        differ[i, j] |= d
        differ[j, i] |= d

  mixed.reset()
  for h in homo:
    h.reset()
  torch.cuda.synchronize()
  check(0)
  for t in range(1, steps + 1):
    acts = _actions(rng, B, mixed.num_players, mixed.num_actions)
    mixed.step(acts)
    for h in homo:
      h.step(acts)
    torch.cuda.synchronize()
    check(t)
  for e in [mixed] + homo:
    e.close()
  return differ


@pytest.mark.parametrize('family', EV.NAMES)
def test_mixed_batch_equals_homogeneous_engines_in_lockstep(family):
  blobs = EV.blobs(family)
  sms = _sms()
  sizes = (1, 7, sms - 1, sms + 1, 2 * sms + 5)
  for B in sizes:
    differ = _lockstep(blobs, blobs, EV.interleaved(B, 4), B, 45)
  # reach: on the largest batch, the homogeneous engines of any two variants differ, so no variant passes vacuously
  assert differ[~np.eye(4, dtype=bool)].all(), differ


@pytest.mark.parametrize('family', EV.NAMES)
def test_identical_variants_equal_a_single_blob_engine(family):
  import torch
  stock = EV.stock(family)
  B = _sms() + 1
  from meltingpot_b200 import engine
  one = engine.Engine(stock, B, seed=SEED)
  four = engine.Engine([stock] * 4, B, seed=SEED, env_variant=EV.interleaved(B, 4))
  rng = np.random.default_rng(9)
  one.reset(); four.reset()
  for t in range(30):
    acts = _actions(rng, B, one.num_players, one.num_actions)
    one.step(acts); four.step(acts)
    torch.cuda.synchronize()
    for name in _VIEWS:
      assert torch.equal(getattr(one, name), getattr(four, name)), f'{name} at step {t}'


def _replace(oracle, env, blob, seed):
  """The oracle env that starts env `env`'s next episode under `blob`."""
  nxt = oracle.OracleEnv(blob, seed)
  nxt.set_episode(env.counters()['episode'] + 1)
  nxt.reset()
  return nxt


@pytest.mark.parametrize('family', ['clean_up', 'coins', 'territory'])
def test_reassignment_takes_effect_at_the_next_episode_start(oracle, family):
  import torch
  from meltingpot_b200 import engine
  blobs = EV.blobs(family)
  B = 12
  first = EV.interleaved(B, 4)
  second = (first + 1) % 4
  third = (first + 2) % 4
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=first)
  shapes, max_ev = parity.shapes_of(eng), int(eng.buffers.max_events)
  envs = [oracle.OracleEnv(blobs[first[b]], SEED + b) for b in range(B)]
  pending = first.copy()
  rng = np.random.default_rng(11)
  eng.reset()
  for e in envs:
    e.reset()
  mask_b = np.arange(B) % 3 == 0
  switched = {'auto': 0, 'mask': 0}
  for t in range(1, 101):
    if t == 10:  # mid-episode: nothing changes until each env's LAST
      eng.set_env_variant(second)
      pending = second.copy()
    if t == 60:  # a masked reset moves the masked envs at once, the others at their next LAST
      eng.set_env_variant(third)
      pending = third.copy()
      eng.reset(torch.from_numpy(mask_b.astype(np.uint8)).cuda())
      for b in np.flatnonzero(mask_b):
        switched['mask'] += 1
        envs[b] = _replace(oracle, envs[b], blobs[pending[b]], SEED + b)
    else:
      acts = rng.integers(0, eng.num_actions, size=(B, eng.num_players)).astype(np.int32)
      eng.step(torch.from_numpy(acts).cuda())
      for b in range(B):
        if envs[b].step_type() == 2:  # this step starts the next episode, under the pending variant
          if envs[b]._blob != blobs[pending[b]]:
            switched['auto'] += 1
          envs[b] = _replace(oracle, envs[b], blobs[pending[b]], SEED + b)
        else:
          envs[b].step(acts[b])
    px = t % 15 == 0
    parity.check_outputs(parity.device_outputs(eng, ('rgb', 'world') if px else ()),
                         parity.env_dump(envs, shapes, pixels=px, max_events=max_ev), f'{family} step {t}')
    active = eng.active_variant.cpu().numpy()
    assert all(envs[b]._blob == blobs[active[b]] for b in range(B)), f'active variants at step {t}: {active}'
  assert switched['auto'] >= B and switched['mask'] == int(mask_b.sum())
  assert np.array_equal(eng.pending_variant.cpu().numpy(), third)
  eng.close()


def test_snapshots_carry_the_assignments_and_refuse_another_variant_set():
  import torch
  from meltingpot_b200 import engine
  blobs = EV.blobs('clean_up')
  B = 40
  assign = EV.interleaved(B, 4)
  a = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  rng = np.random.default_rng(13)
  a.reset()
  for _ in range(25):
    a.step(_actions(rng, B, a.num_players, a.num_actions))
  a.set_env_variant((assign + 3) % 4)  # pending, not yet active
  snap = a.save_state()
  acts = [_actions(rng, B, a.num_players, a.num_actions) for _ in range(30)]
  for x in acts:
    a.step(x)
  b = engine.Engine(list(blobs), B, seed=SEED)  # every env on variant 0 until the snapshot says otherwise
  b.load_state(snap)
  assert np.array_equal(b.active_variant.cpu().numpy(), assign)
  assert np.array_equal(b.pending_variant.cpu().numpy(), (assign + 3) % 4)
  for x in acts:
    b.step(x)
  torch.cuda.synchronize()
  for name in _VIEWS + ('active_variant', 'pending_variant'):
    assert torch.equal(getattr(a, name), getattr(b, name)), name
  for other in ([blobs[1], blobs[0], blobs[2], blobs[3]], list(blobs[:3]), [blobs[0]] * 4):
    c = engine.Engine(other, B, seed=SEED)
    with pytest.raises(ValueError, match='different compiled substrate'):
      c.load_state(snap)
    c.close()
  single = engine.Engine(blobs[0], B, seed=SEED)
  with pytest.raises(ValueError):
    single.load_state(snap)
  for e in (a, b, single):
    e.close()


def _refusals():
  cu = 'clean_up'
  rows = [
      ('map', cu, V.map_replace('F', 'H'), 'section'),
      ('view', cu, V.view(2, 2, 2, 2), 'section'),
      # the same number of footprint cells (3 forward, radius 1 -> 9 in a line), another shape
      ('zap_beam', cu, V.kw('Zapper', beamLength=9, beamRadius=0), "'zap.geom'"),
      ('clean_beam', cu, V.kw('Cleaner', beamLength=9, beamRadius=0), "'clean_geom'"),
      ('clean_beam_cells', cu, V.kw('Cleaner', beamLength=2), 'beam footprints'),
      ('episode_cap', cu, V.top(maxEpisodeLengthFrames=50), "section 'meta'"),
      ('episode_ending', cu, V.kw('StochasticIntervalEpisodeEnding', probabilityTerminationPerInterval=0.5), 'episode ending'),
      ('density_radius', 'commons_harvest', V.density_radius(1.0), 'section'),
      ('marking_levels', 'territory',
       V.marking_levels([dict(levelIncrement=0, sourceReward=0.25, targetReward=-0.5, freeze=2)], 1), "'mark_n_levels'"),
  ]
  return rows


@pytest.mark.parametrize('row', _refusals(), ids=lambda r: r[0])
def test_incompatible_variants_are_refused_at_create(row):
  from meltingpot_b200 import engine
  _, family, edit, what = row
  blobs = EV.blobs(family)
  bad = EV.compile_settings(family, EV.settings(family, [edit]))
  with pytest.raises(ValueError, match=f'variant 1: .*{what}'):
    engine.Engine([blobs[0], bad], 8, seed=SEED)


def test_a_sprite_colour_override_is_refused_at_create():
  from meltingpot_b200 import engine
  blobs = EV.blobs('clean_up')
  palette = {'x': [0, 0, 0, 0], '*': [12, 80, 57, 255], '#': [173, 66, 47, 255], 'o': [43, 127, 53, 255], '|': [79, 47, 44, 255]}
  bad = EV.compile_settings('clean_up', EV.settings('clean_up'), {'potential_apple': {'Appearance': {'palettes': [palette]}}})
  assert 'atlas' in EV.differing_sections(blobs[0], bad)
  with pytest.raises(ValueError, match="variant 2: section '(atlas|sprite_opaque)'"):
    engine.Engine([blobs[0], blobs[1], bad], 8, seed=SEED)


def test_batched_substrate_of_variants_equals_the_engine():
  import torch
  from meltingpot_b200 import engine, substrate
  blobs = EV.blobs('coop_mining')
  B = 33
  assign = EV.blocks(B, 4)
  sub = substrate.BatchedSubstrate(list(blobs), B, seed=SEED, env_variant=assign)
  eng = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  rng = np.random.default_rng(17)
  sub.reset(); eng.reset()
  for t in range(45):
    acts = _actions(rng, B, eng.num_players, eng.num_actions)
    ts = sub.step(acts)
    eng.step(acts)
    torch.cuda.synchronize()
    assert torch.equal(ts.reward, eng.reward) and torch.equal(ts.step_type, eng.step_type)
    assert torch.equal(ts.observation['RGB'], eng.rgb) and torch.equal(ts.observation['WORLD.RGB'], eng.world_rgb)
  sub.set_env_variant(np.zeros(B, np.int64))
  assert sub.engine.pending_variant.sum().item() == 0
  sub.close(); eng.close()


def test_slices_of_the_assignment_with_their_env_index_base_equal_one_mixed_engine():
  import torch
  from meltingpot_b200 import distributed, engine
  blobs = EV.blobs('territory')
  B = 64
  assign = EV.interleaved(B, 4)
  full = engine.Engine(list(blobs), B, seed=SEED, env_variant=assign)
  shards = []
  for r in range(2):
    base, count = distributed.shard_envs(B, r, 2)
    shards.append((base, count, engine.Engine(list(blobs), count, seed=SEED, env_index_base=base,
                                              env_variant=assign[base:base + count])))
  rng = np.random.default_rng(19)
  full.reset()
  for *_, s in shards:
    s.reset()
  for t in range(45):
    acts = _actions(rng, B, full.num_players, full.num_actions)
    full.step(acts)
    for base, count, s in shards:
      s.step(acts[base:base + count].contiguous())
  torch.cuda.synchronize()
  for base, count, s in shards:
    for name in ('rgb', 'world_rgb', 'reward', 'grid', 'avatar_state', 'timestep_packed'):
      assert torch.equal(getattr(full, name)[base:base + count], getattr(s, name)), name
