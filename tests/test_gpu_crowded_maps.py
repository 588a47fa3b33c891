"""The CUDA engine against the oracle on the crowded arenas of tests/crowded_maps.py.

On these maps the order-dependent work of the step kernels happens on most frames: chains of moves and contested cells
(move_avatars), zapped avatars that still block and fire beams, targets hit by two beams (draw_hit_sprite), respawns onto
occupied cells, two claims of one resource, several miners on one gold ore, and deep stacks of pieces in one cell for
k_render. parity.compare_batch checks every env on every step; the predicates are counted from the engine's own buffers
and must reach their floors, and the raw event count never exceeds max_events. Each family also runs in lockstep with a
twin that skips the render pre-merge and one with a forced render layout.
"""

import numpy as np
import pytest

from meltingpot_b200 import blob as mpb
from tests import crowded_maps as C
from tests import parity

pytestmark = pytest.mark.gpu

SEED = 9001
# one variant per family for the largest batch: the churn twins, where most happens per frame
BIG = {'clean_up': 'clean_up/churn', 'commons_harvest': 'commons_16p/churn', 'territory': 'territory_rooms/churn',
       'coins': 'coins/churn', 'coop_mining': 'coop_mining/churn'}


def _sms():
  import torch
  return torch.cuda.get_device_properties(0).multi_processor_count


def _run(name, policy, oracle, num_envs, steps, pixels_every):
  """compare_batch of one (variant, policy), with the predicates counted from the engine's buffers."""
  blob = C.compile(name)
  sec = mpb.unpack(blob)
  reach = C.Reach(sec, num_envs)
  act = C.policy(policy, sec)
  last = {}

  def actions_fn(t, B, P, A, rng):
    last['acts'] = np.ascontiguousarray(act(t, B, P, A, rng), np.int32)
    return last['acts']

  def on_step(t, eng):
    n_events = eng.event_count.cpu().numpy()
    max_ev = int(eng.buffers.max_events)
    assert int(n_events.max()) <= max_ev, f'step {t}: {int(n_events.max())} events exceed max_events {max_ev}'
    cells = int(eng.buffers.grid_cells)
    reach.observe(t, eng.avatar_state.cpu().numpy(), eng.grid.cpu().numpy().view(np.uint16)[:, :, :cells],
                  eng.events.cpu().numpy(), n_events, eng.step_type.cpu().numpy(), last.get('acts') if t else None)

  stats = parity.compare_batch(blob, oracle, num_envs=num_envs, steps=steps, seed=SEED, actions_fn=actions_fn,
                               pixels_every=pixels_every, on_step=on_step)
  assert stats['lasts'] >= num_envs * (steps // (C.CAP + 1)), stats  # the runs cross auto-resets
  return reach, sec


@pytest.mark.parametrize('policy', C.POLICIES)
@pytest.mark.parametrize('name', [v.name for v in C.VARIANTS])
def test_arena_matches_the_oracle_at_7_envs(name, policy, oracle):
  reach, _ = _run(name, policy, oracle, 7, C.STEPS, 1)
  print(name, policy, {k: round(x, 1) for k, x in C.rates(reach).items()})


@pytest.mark.parametrize('name', [v.name for v in C.VARIANTS])
def test_arena_matches_the_oracle_at_two_waves(name, oracle):
  # 2 * SMs + 5 envs, every pixel on every step, past the first auto-reset; the arena under uniform actions, its churn
  # twin under the beam-heavy policy
  v = C.BY_NAME[name]
  policy = 'beams' if v.churn else 'uniform'
  reach, sec = _run(name, policy, oracle, 2 * _sms() + 5, C.CAP + 5, 1)
  print(name, policy, {k: round(x, 1) for k, x in C.rates(reach).items()})
  bad = C.shortfalls(v, sec, policy, C.rates(reach))
  assert not bad, f'{name} {policy}: the engine did not reach {bad}'


@pytest.mark.parametrize('family', C.FAMILIES)
def test_arena_matches_the_oracle_at_2048_envs(family, oracle):
  # the first 30 frames of 2048 episodes, pixels every 5 steps (the oracle's rendering bounds the run time)
  name = BIG[family]
  reach, _ = _run(name, 'uniform', oracle, 2048, 30, 5)
  print(name, {k: round(x, 1) for k, x in C.rates(reach).items()})


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


@pytest.mark.parametrize('family', C.FAMILIES)
def test_arena_twins_run_in_lockstep(family):
  from meltingpot_b200 import engine
  name = BIG[family]
  blob = C.compile(name)
  sec = mpb.unpack(blob)
  n = 2 * _sms() + 5
  probe = engine.Engine(blob, n, seed=SEED)
  plan = probe.render_plan()
  probe.close()
  lay = _alternative_layout(blob, (plan['teams'], plan['team_threads'] // 32, plan['wstrip_log2']))
  variants = [dict(flags=engine.MP_FLAG_DEFAULT | engine.MP_FLAG_DEBUG_NO_PREMERGE), dict(render_layout=lay)]
  plans = parity.lockstep(blob, n, C.CAP + 10, SEED, variants, actions_fn=C.policy('beams', sec))
  forced = plans[1]
  assert (forced['teams'], forced['team_threads'] // 32, forced['wstrip_log2']) == lay, (lay, forced)
