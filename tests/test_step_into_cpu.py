"""CPU test: the tensor -> mp_device_outputs conversion of Engine.step(out=) and the layout of
BatchedSubstrate.trajectory, on tensor layouts alone (no device)."""

import numpy as np
import pytest
import torch

from meltingpot_b200 import engine
from meltingpot_b200 import substrate

B, P, H, W, WH, WW, N = 5, 3, 16, 24, 40, 32, 2
VIEWS = {'rgb': ((B, P, H, W, 3), torch.uint8), 'world_rgb': ((B, WH, WW, 3), torch.uint8),
         'reward': ((B, P), torch.float64), 'discount': ((B,), torch.float64), 'step_type': ((B,), torch.int64),
         'scalar_obs': ((N, B, P), torch.float64)}


def _layout(t, device='cuda:0', ptr=1 << 20):
  return engine.TensorLayout(tuple(t.shape), tuple(t.stride()), t.dtype, torch.device(device),
                             ptr + t.storage_offset() * t.element_size())


def _describe(**out):
  return engine.describe_outputs(out, VIEWS, 0)


def test_dense_outputs_give_dense_strides():
  out = {k: _layout(torch.zeros(shape, dtype=dt)) for k, (shape, dt) in VIEWS.items()}
  s = _describe(**out)
  assert s.rgb == 1 << 20 and s.rgb_env_stride == P * H * W * 3
  assert s.world_rgb_env_stride == WH * WW * 3
  assert s.reward_env_stride == P * 8 and s.discount_env_stride == 8 and s.step_type_env_stride == 8
  assert s.scalar_obs_env_stride == P * 8 and s.scalar_obs_stride == B * P * 8


@pytest.mark.parametrize('time_major', [True, False])
def test_trajectory_slots_describe_strided_envs(time_major):
  T, t = 4, 2
  traj = substrate.Trajectory(T, B, P, (P, H, W, 3), (WH, WW, 3), ['A', 'B'], time_major, 'cpu')
  ts = traj.at(t)
  scal = torch.as_strided(ts.observation['A'], (N, B, P), ((T * B * P), ) + ts.observation['A'].stride())
  out = dict(rgb=_layout(ts.observation['RGB']), world_rgb=_layout(ts.observation['WORLD.RGB']), reward=_layout(ts.reward),
             discount=_layout(ts.discount), step_type=_layout(ts.step_type), scalar_obs=_layout(scal))
  s = _describe(**out)
  per = P * H * W * 3
  if time_major:
    assert s.rgb_env_stride == per and s.rgb == (1 << 20) + t * B * per
    assert s.reward_env_stride == P * 8 and s.discount_env_stride == 8
    assert s.scalar_obs_env_stride == P * 8
  else:
    assert s.rgb_env_stride == T * per and s.rgb == (1 << 20) + t * per
    assert s.reward_env_stride == T * P * 8 and s.discount_env_stride == T * 8 and s.step_type_env_stride == T * 8
    assert s.scalar_obs_env_stride == T * P * 8
  assert s.scalar_obs_stride == T * B * P * 8


def test_padded_env_stride_and_offset():
  raw = torch.zeros(16 + B * (P * H * W * 3 + 48), dtype=torch.uint8)
  rgb = torch.as_strided(raw, (B, P, H, W, 3), (P * H * W * 3 + 48, H * W * 3, W * 3, 3, 1), 16)
  s = _describe(rgb=_layout(rgb))
  assert s.rgb == (1 << 20) + 16 and s.rgb_env_stride == P * H * W * 3 + 48
  assert not s.world_rgb and not s.reward  # outputs not named stay NULL


def test_one_env_passes_the_dense_stride():
  views = dict(VIEWS, reward=((1, P), torch.float64))
  t = torch.zeros((1, 7 * P), dtype=torch.float64)[:, :P]
  s = engine.describe_outputs({'reward': _layout(t)}, views, 0)
  assert s.reward_env_stride == P * 8


@pytest.mark.parametrize('name,tensor,device,match', [
    ('rgb', torch.zeros((B, P, H, W, 4), dtype=torch.uint8), 'cuda:0', 'shape'),
    ('reward', torch.zeros((B, P), dtype=torch.float32), 'cuda:0', 'dtype'),
    ('step_type', torch.zeros((B,), dtype=torch.float64), 'cuda:0', 'dtype'),
    ('reward', torch.zeros((B, P), dtype=torch.float64), 'cpu', 'on cpu'),
    ('reward', torch.zeros((B, P), dtype=torch.float64), 'cuda:1', 'on cuda:1'),
    ('rgb', torch.zeros((B, P, H, W * 2, 3), dtype=torch.uint8)[:, :, :, :W], 'cuda:0', 'axis 2'),
    ('reward', torch.zeros((B, 2 * P), dtype=torch.float64)[:, ::2], 'cuda:0', 'axis 1'),
    ('scalar_obs', torch.zeros((N, B, 2 * P), dtype=torch.float64)[:, :, ::2], 'cuda:0', 'axis 2'),
    ('events', torch.zeros((B,), dtype=torch.int32), 'cuda:0', 'unknown output'),
])
def test_refusals(name, tensor, device, match):
  with pytest.raises(ValueError, match=match):
    _describe(**{name: _layout(tensor, device)})


def test_env_and_observation_axes_may_be_strided():
  base = torch.zeros((3, B, 2, P), dtype=torch.float64)
  scal = base[:N, :, 1]  # obs stride 2 * B * P, env stride 2 * P
  s = _describe(scalar_obs=_layout(scal))
  assert s.scalar_obs_stride == B * 2 * P * 8 and s.scalar_obs_env_stride == 2 * P * 8


@pytest.mark.parametrize('time_major', [True, False])
def test_trajectory_shapes(time_major):
  T = 6
  traj = substrate.Trajectory(T, B, P, (P, H, W, 3), (WH, WW, 3), ['READY_TO_SHOOT'], time_major, 'cpu')
  lead = (T, B) if time_major else (B, T)
  assert traj.step_type.shape == lead and traj.step_type.dtype == torch.int64
  assert traj.reward.shape == lead + (P,) and traj.discount.shape == lead
  assert traj.observation['RGB'].shape == lead + (P, H, W, 3)
  assert traj.observation['WORLD.RGB'].shape == lead + (WH, WW, 3)
  assert traj.observation['READY_TO_SHOOT'].shape == lead + (P,)
  assert traj.observation['COLLECTIVE_REWARD'].shape == lead
  for t in (0, T - 1, -1):
    ts = traj.at(t)
    assert ts.reward.shape == (B, P) and ts.discount.shape == (B,) and ts.step_type.shape == (B,)
    assert ts.observation['RGB'].shape == (B, P, H, W, 3) and ts.observation['COLLECTIVE_REWARD'].shape == (B,)
    ts.reward.fill_(t + 7.0)
    sel = traj.reward[t] if time_major else traj.reward[:, t]
    assert bool((sel == t + 7.0).all())
  env_stride = traj.at(1).observation['RGB'].stride(0)
  assert env_stride == (P * H * W * 3 if time_major else T * P * H * W * 3)
  with pytest.raises(IndexError):
    traj.at(T)


def test_trajectory_without_world_or_scalars():
  traj = substrate.Trajectory(2, B, P, (P, H, W, 3), None, [], True, 'cpu')
  assert set(traj.observation) == {'RGB', 'COLLECTIVE_REWARD'}
  with pytest.raises(ValueError):
    substrate.Trajectory(0, B, P, (P, H, W, 3), None, [], True, 'cpu')
