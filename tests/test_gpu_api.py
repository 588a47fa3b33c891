"""C-ABI behaviours beyond plain stepping: masked resets, host-buffer calls, action validation, render flags."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _cmp(eng, envs, where):
  import torch
  torch.cuda.synchronize()
  rew = eng.reward.cpu().numpy(); st = eng.step_type.cpu().numpy()
  rgb = eng.rgb.cpu().numpy(); world = eng.world_rgb.cpu().numpy()
  for b, e in enumerate(envs):
    assert e.step_type() == st[b], f'step_type {where} env {b}'
    np.testing.assert_array_equal(e.rewards(), rew[b], err_msg=f'reward {where} env {b}')
    np.testing.assert_array_equal(e.rgb(), rgb[b], err_msg=f'RGB {where} env {b}')
    np.testing.assert_array_equal(e.world_rgb(), world[b], err_msg=f'WORLD.RGB {where} env {b}')


def test_masked_reset_restarts_only_the_selected_envs(clean_up_blob, oracle):
  # a reset with env_mask (mp_run): the reference has one env per object, so a "masked reset" is env[i].reset() for some i.
  _masked_reset(clean_up_blob, 'clean_up', oracle)


@pytest.mark.parametrize('name,players', [('commons_harvest__open', 7), ('territory__rooms', 9),
                                          ('territory__inside_out', 5), ('coins', 2), ('coop_mining', 6)])
def test_masked_reset_of_every_kernel_family(name, players, oracle):
  # The other kernel families (territory computes its reset condition apart from the others), plus inside_out, whose
  # reset also redraws the env's 'choice' resource layout.
  from meltingpot_b200 import substrates
  _masked_reset(substrates.load_blob(name, ('default',) * players), name, oracle)


def _masked_reset(blob, name, oracle):
  import torch
  from meltingpot_b200 import engine
  B, seed = 12, 40
  eng = engine.Engine(blob, B, device=0, seed=seed)
  P, A = eng.num_players, eng.num_actions
  envs = [oracle.OracleEnv(blob, seed + b) for b in range(B)]
  eng.reset()
  for e in envs:
    e.reset()
  rng = np.random.default_rng(2)
  def play(k, tag):
    for t in range(k):
      a = np.ascontiguousarray(rng.integers(0, A, (B, P)), np.int32)
      eng.step(torch.from_numpy(a).cuda())
      for b, e in enumerate(envs):
        e.step(a[b])
      if t % 5 == 4:
        _cmp(eng, envs, f'{tag} step {t}')
  play(25, 'before')
  grid_before = eng.grid.cpu().numpy()
  mask = np.zeros(B, np.uint8); mask[[1, 4, 5, 10]] = 1
  eng.reset(torch.from_numpy(mask).cuda())
  for b in np.nonzero(mask)[0]:
    envs[b].reset()  # next episode of that env only
  _cmp(eng, envs, 'after masked reset')
  for b, e in enumerate(envs):
    np.testing.assert_array_equal(e.grid(), eng.grid.cpu().numpy().view(np.uint16)[b][:, :e.grid().shape[1]],
                                  err_msg=f'grid after masked reset env {b}')
  st = eng.step_type.cpu().numpy()
  assert (st[mask == 1] == 0).all() and (st[mask == 0] == 1).all()  # FIRST only where reset
  if name == 'territory__inside_out':
    from meltingpot_b200 import blob as blob_lib, compiler
    sec = blob_lib.unpack(blob)
    cells, res_layer = sec['tr_res'][:, 1].astype(np.int64), compiler.family_params(sec)['RES_LAYER']
    layout = lambda g: g[:, res_layer][:, cells] != 0
    before, after = layout(grid_before), layout(eng.grid.cpu().numpy())
    for b in range(B):  # masked envs redraw their resource layout, the others keep theirs
      assert np.array_equal(before[b], after[b]) == (mask[b] == 0), f'resource layout env {b}'
  play(25, 'after')


def test_host_buffer_calls_return_the_device_buffers(commons_blob):
  import torch
  from meltingpot_b200 import engine
  B = 16
  eng = engine.Engine(commons_blob, B, device=0, seed=5)
  out = eng.make_host_outputs()
  eng.reset_host(out)
  assert (out['step_type'].numpy() == 0).all()
  np.testing.assert_array_equal(out['rgb'].numpy(), eng.rgb.cpu().numpy())
  rng = np.random.default_rng(0)
  for _ in range(20):
    a = torch.from_numpy(np.ascontiguousarray(rng.integers(0, 8, (B, 7)), np.int32)).pin_memory()
    eng.step_host(a, out)
  for name in ('rgb', 'world_rgb', 'reward', 'discount', 'step_type'):
    np.testing.assert_array_equal(out[name].numpy(), getattr(eng, name).cpu().numpy(), err_msg=name)
  np.testing.assert_array_equal(out['scalar_obs'].numpy(), eng.scalar_obs.cpu().numpy())
  scalars_only = {k: v for k, v in out.items() if k not in ('rgb', 'world_rgb')}  # NULL pointers skip those copies
  before = out['rgb'].numpy().copy()
  eng.step_host(torch.zeros((B, 7), dtype=torch.int32).pin_memory(), scalars_only)
  np.testing.assert_array_equal(out['rgb'].numpy(), before)
  np.testing.assert_array_equal(scalars_only['reward'].numpy(), eng.reward.cpu().numpy())


def test_out_of_range_action_ids_are_noops(clean_up_blob, oracle):
  # Both sides clamp an id outside the action table to 0 (NOOP); the Python wrapper rejects them earlier.
  import torch
  from meltingpot_b200 import engine
  B, P, seed = 4, 7, 8
  eng = engine.Engine(clean_up_blob, B, device=0, seed=seed)
  envs = [oracle.OracleEnv(clean_up_blob, seed + b) for b in range(B)]
  eng.reset()
  for e in envs:
    e.reset()
  rng = np.random.default_rng(1)
  for t in range(30):
    a = np.ascontiguousarray(rng.integers(-3, 14, (B, P)), np.int32)
    eng.step(torch.from_numpy(a).cuda())
    for b, e in enumerate(envs):
      e.step(a[b])
  _cmp(eng, envs, 'out-of-range ids')


def test_render_flags_select_the_images(clean_up_blob):
  import torch
  from meltingpot_b200 import engine
  eng = engine.Engine(clean_up_blob, 8, device=0, seed=2)
  eng.reset()
  a = torch.ones((8, 7), dtype=torch.int32, device='cuda')
  eng.step(a)
  world0, rgb0 = eng.world_rgb.clone(), eng.rgb.clone()
  eng.set_flags(engine.MP_FLAG_RENDER_PLAYERS)
  for _ in range(5):
    eng.step(a)
  assert torch.equal(eng.world_rgb, world0) and not torch.equal(eng.rgb, rgb0)  # WORLD.RGB left untouched
  eng.set_flags(engine.MP_FLAG_RENDER_PLAYERS | engine.MP_FLAG_RENDER_WORLD)
  eng.step(a)
  assert not torch.equal(eng.world_rgb, world0)
