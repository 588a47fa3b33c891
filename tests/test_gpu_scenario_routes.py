"""BatchedScenario on player routes: focal and background observations are drawn straight into rows, and actions are
read from rows. Each scenario runs beside a BatchedSubstrate stepped directly with the merged [B, P] actions.

The background policy derives its actions from its own observations (a hash of each background player's image and
READY_TO_SHOOT), so a misrouted observation or action row changes the trajectory instead of going unnoticed."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _hash_policy(num_actions, seen):
  def policy(ts):
    import torch
    rgb = ts.observation['RGB']
    h = rgb.to(torch.int64).flatten(2).mul(torch.arange(1, rgb[0, 0].numel() + 1, device='cuda')).sum(dim=2)
    if 'READY_TO_SHOOT' in ts.observation:
      h = h + (ts.observation['READY_TO_SHOOT'] * 7).to(torch.int64)
    a = (h % num_actions).to(torch.int32)
    seen.append(a.clone())
    return a
  return policy


def _run(blob, B, is_focal, steps, permitted, seed=9):
  import torch
  from meltingpot_b200 import scenario, substrate
  focal = [i for i, f in enumerate(is_focal) if f]
  background = [i for i, f in enumerate(is_focal) if not f]
  seen = []
  sub = substrate.BatchedSubstrate(blob, B, seed=seed)
  sc = scenario.BatchedScenario(sub, _hash_policy(sub.num_actions, seen), is_focal, permitted_observations=permitted)
  direct = substrate.BatchedSubstrate(blob, B, seed=seed)
  ts, ref = sc.reset(), direct.reset()
  rng = np.random.default_rng(0)
  firsts = 0
  for t in range(steps):
    if t:
      fa = torch.from_numpy(np.ascontiguousarray(rng.integers(0, sub.num_actions, (B, len(focal))), np.int32)).cuda()
      ts = sc.step(fa)
      full = torch.zeros((B, sub.num_players), dtype=torch.int32, device='cuda')
      full[:, focal] = fa
      if background:
        full[:, background] = seen[-1]
      ref = direct.step(full)
    firsts += int((ref.step_type == 0).sum()) if t else 0
    bg = sc.background_timestep
    assert torch.equal(ts.step_type, ref.step_type) and torch.equal(ts.discount, ref.discount), t
    assert torch.equal(ts.reward, ref.reward[:, focal]), t
    assert torch.equal(bg.reward, ref.reward[:, background]), t
    assert set(ts.observation) == set(permitted) & set(ref.observation), t
    for key, want in ref.observation.items():
      per_player = key not in ('WORLD.RGB', 'COLLECTIVE_REWARD')
      assert torch.equal(bg.observation[key], want[:, background] if per_player else want), (key, t)
      if key in ts.observation:
        assert torch.equal(ts.observation[key], want[:, focal] if per_player else want), (key, t)
  assert firsts > 0, 'the run never crossed an auto-reset'
  return sc


@pytest.mark.parametrize('substrate_name,B,is_focal,permitted', [
    ('clean_up', 64, (True, False, True, True, False, True, True), {'RGB', 'READY_TO_SHOOT', 'COLLECTIVE_REWARD', 'WORLD.RGB'}),
    ('commons_harvest__open_16p', 48, (True,) * 6 + (False,) * 2 + (True,) * 6 + (False,) * 2, {'RGB', 'READY_TO_SHOOT'}),
    ('coins', 33, (True, False), {'RGB', 'COLLECTIVE_REWARD', 'WORLD.RGB'}),
])
def test_routed_scenario_equals_direct_stepping(substrate_name, B, is_focal, permitted):
  _run(_blob(substrate_name), B, is_focal, 45, permitted)


def test_all_focal_and_no_focal_splits():
  blob = _blob('clean_up')
  sc = _run(blob, 9, (True,) * 7, 45, {'RGB', 'READY_TO_SHOOT'})
  assert sc.num_background == 0 and sc.background_timestep.observation['RGB'].shape[:2] == (9, 0)
  sc = _run(blob, 9, (False,) * 7, 45, {'RGB', 'COLLECTIVE_REWARD'})
  assert sc.num_focal == 0


def test_a_held_timestep_keeps_its_step():
  import torch
  from meltingpot_b200 import scenario, substrate
  blob, B = _blob('clean_up'), 16
  seen = []
  sub = substrate.BatchedSubstrate(blob, B, seed=2)
  sc = scenario.BatchedScenario(sub, _hash_policy(sub.num_actions, seen), (True,) * 5 + (False,) * 2, {'RGB', 'READY_TO_SHOOT'})
  sc.reset()
  rng = np.random.default_rng(1)
  held, copies = [], []
  for _ in range(6):
    ts = sc.step(torch.from_numpy(rng.integers(0, 9, (B, 5)).astype(np.int32)).cuda())
    held.append((ts, sc.background_timestep))
    copies.append([x.clone() for x in (ts.observation['RGB'], ts.reward, ts.observation['READY_TO_SHOOT'],
                                       sc.background_timestep.observation['RGB'], sc.background_timestep.reward)])
  for (ts, bg), want in zip(held, copies):
    got = (ts.observation['RGB'], ts.reward, ts.observation['READY_TO_SHOOT'], bg.observation['RGB'], bg.reward)
    for g, w in zip(got, want):
      assert torch.equal(g, w)
  assert not torch.equal(copies[0][0], copies[-1][0])


def _blob(name):
  """hard_cap_40 blobs, so that every run crosses an auto-reset."""
  from tests import variants as V
  from tests.test_gpu_step_into import _blob as cap40
  if name == 'commons_harvest__open_16p':
    return V.compile_variant(V.Variant('commons_harvest/hard_cap_40_16p', 'commons_harvest__open', 16, None,
                                       [V.kw(V._ENDING, probabilityTerminationPerInterval=0.0),  # pylint: disable=protected-access
                                        V.top(maxEpisodeLengthFrames=40)], 'parity'))
  return cap40(name)
