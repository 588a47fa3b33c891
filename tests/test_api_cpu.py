"""Host-side logic that must hold without a GPU: shims, config/spec surface, C ABI symbols."""

import ctypes
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from meltingpot_b200 import engine, shims, specs, substrate

shims.install()
import dm_env  # noqa: E402

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_dm_env_surface():
  ts = dm_env.restart({'a': 1})
  assert ts.first() and ts.reward is None and ts.discount is None
  assert dm_env.transition(1.0, {}).mid() and dm_env.transition(1.0, {}).discount == 1.0
  last = dm_env.termination(2.0, {})
  assert last.last() and last.discount == 0.0
  assert int(dm_env.StepType.FIRST) == 0 and int(dm_env.StepType.LAST) == 2


def test_spec_equality_ignores_name_like_dm_env():
  # substrate_test.py:41-47 compares per-player specs with `==`; names differ, shapes do not.
  a = dm_env.specs.Array((88, 88, 3), np.uint8, name='RGB')
  b = dm_env.specs.Array((88, 88, 3), np.uint8, name='1.RGB')
  assert a == b and a != dm_env.specs.Array((88, 88, 3), np.int32)
  d = dm_env.specs.DiscreteArray(9, dtype=np.int64, name='action')
  assert d.num_values == 9 and d.maximum == 8 and d.replace(num_values=8).num_values == 8
  d.validate(np.int64(3))
  with pytest.raises(ValueError):
    d.validate(np.int64(9))
  with pytest.raises(ValueError):
    a.validate(np.zeros((88, 88, 3), np.float32))


def test_config_dict_lock():
  from ml_collections import config_dict
  c = config_dict.ConfigDict()
  c.x = 1
  c.lock()
  with pytest.raises(AttributeError):
    c.y = 2
  with c.unlocked():
    c.y = 2
  assert c.y == 2 and c.is_locked and c.to_dict() == {'x': 1, 'y': 2}


def test_clean_up_config_matches_reference_api():
  config = substrate.get_config('clean_up')
  # clean_up.py:461-483: ids map to NOOP, FORWARD, BACKWARD, STEP_LEFT, STEP_RIGHT, TURN_LEFT, TURN_RIGHT, ZAP, CLEAN
  assert len(config.action_set) == 9
  assert config.action_set[2] == {'move': 3, 'turn': 0, 'fireZap': 0, 'fireClean': 0}
  assert config.action_set[4]['move'] == 2 and config.action_set[5]['turn'] == -1
  assert config.action_set[7]['fireZap'] == 1 and config.action_set[8]['fireClean'] == 1
  assert list(config.individual_observation_names) == ['RGB', 'READY_TO_SHOOT', 'NUM_OTHERS_WHO_CLEANED_THIS_STEP']
  assert list(config.global_observation_names) == ['WORLD.RGB']
  obs = config.timestep_spec.observation
  assert obs['RGB'] == specs.rgb(88, 88) and obs['WORLD.RGB'] == specs.rgb(168, 240)
  assert obs['READY_TO_SHOOT'].dtype == np.float64 and obs['READY_TO_SHOOT'].shape == ()
  assert config.action_spec.num_values == 9 and config.action_spec.dtype == np.int64
  assert config.valid_roles == frozenset({'default'}) and config.default_player_roles == ('default',) * 7
  assert config.timestep_spec.reward.dtype == np.float64
  with pytest.raises(ValueError):
    substrate.get_config('not_a_substrate')


def test_invalid_roles_raise_value_error():
  # configs/substrates/__init__.py:42-45
  with pytest.raises(ValueError, match='Invalid roles'):
    substrate.build('clean_up', roles=('default', 'cleaner'))


def test_c_abi_exports_every_declared_symbol():
  header = open(os.path.join(ROOT, 'include', 'mp_engine.h')).read()
  declared = set(re.findall(r'\b(mp_[a-z_]+)\s*\(', header))
  declared.discard('mp_engine')
  assert declared == set(engine.EXPORTED_SYMBOLS), declared ^ set(engine.EXPORTED_SYMBOLS)
  lib = engine.load_library()
  for sym in declared:
    assert hasattr(lib, sym), sym
  assert b'sm_90a' in lib.mp_version()


def test_c_abi_declares_mp_run():
  with open(os.path.join(ROOT, 'include', 'mp_engine.h')) as f:
    header = f.read()
  decl = [p.strip() for p in re.search(r'\bint mp_run\(([^;]*)\);', header).group(1).split(',')]
  assert decl == ['mp_handle h', 'const mp_request* r', 'void* stream']
  lib = engine.load_library()
  assert lib.mp_run.argtypes == [ctypes.c_void_p, ctypes.POINTER(engine.MpRequest), ctypes.c_void_p]
  for name, value in re.findall(r'#define (MP_MAX_ROUTE_\w+) (\d+)', header):
    assert getattr(engine, name) == int(value)


# every struct the C ABI shares with the ctypes binding, by its C name
ABI_STRUCTS = {'mp_buffers': engine.MpBuffers, 'mp_host_outputs': engine.MpHostOutputs,
               'mp_device_outputs': engine.MpDeviceOutputs, 'mp_player_outputs': engine.MpPlayerOutputs,
               'mp_player_actions': engine.MpPlayerActions, 'mp_route_draw': engine.MpRouteDraw,
               'mp_request': engine.MpRequest}


@pytest.mark.skipif(not (shutil.which('cc') or shutil.which('gcc')), reason='needs a C compiler')
@pytest.mark.parametrize('c_name', sorted(ABI_STRUCTS))
def test_abi_struct_matches_the_header(c_name, tmp_path):
  cls = ABI_STRUCTS[c_name]
  fields = [name for name, _ in cls._fields_]
  src = tmp_path / 'layout.c'
  src.write_text('#include <stddef.h>\n#include <stdio.h>\n#include "mp_engine.h"\nint main(void) {\n'
                 f'  printf("%zu", sizeof({c_name}));\n'
                 + ''.join(f'  printf(" %zu", offsetof({c_name}, {f}));\n' for f in fields) + '  return 0;\n}\n')
  exe = tmp_path / 'layout'
  subprocess.check_call([shutil.which('cc') or shutil.which('gcc'), '-I', os.path.join(ROOT, 'include'), str(src), '-o', str(exe)])
  got = [int(x) for x in subprocess.check_output([str(exe)]).split()]
  assert got[0] == ctypes.sizeof(cls)
  assert got[1:] == [getattr(cls, f).offset for f in fields]


def _cuda_available():
  import torch
  return torch.cuda.is_available()


@pytest.mark.skipif(_cuda_available(), reason='checks the no-GPU failure mode')
def test_engine_fails_loudly_without_gpu(clean_up_blob):
  lib = engine.load_library()
  handle = ctypes.c_void_p()
  rc = lib.mp_create(clean_up_blob, len(clean_up_blob), 4, 0, ctypes.c_uint64(1), ctypes.c_uint64(0),
                     ctypes.c_uint32(3), ctypes.byref(handle))
  assert rc == -4 and not handle.value  # MP_E_NO_DEVICE: there is no CPU path to fall back to
  assert b'no CPU path' in lib.mp_last_error()
  with pytest.raises(engine.EngineError):
    engine.Engine(clean_up_blob, 4)
  with pytest.raises(engine.EngineError):
    substrate.build('clean_up', roles=('default',) * 7)


def test_product_package_never_imports_the_oracle():
  pkg = os.path.join(ROOT, 'meltingpot_b200')
  bad = re.compile(r'^\s*(#\s*include\s*[<"][^>"]*oracle|from\s+oracle\b|import\s+oracle\b)|liboracle|CDLL\([^)]*oracle',
                   re.MULTILINE)
  for dirpath, _, files in os.walk(pkg):
    for f in files:
      if f.endswith(('.py', '.cu', '.cuh', '.h')):
        text = open(os.path.join(dirpath, f), errors='ignore').read()
        assert not bad.search(text), f


def test_dmlab2d_level_views_invert_the_multiplayer_wrapper():
  # observables().dmlab2d carries the raw stream (wrappers/observables.py:32-45). flat_action / flat_timestep build it from
  # the multiplayer TimeStep: {"<i>.<name>"} keys, "<i>.REWARD", reward / discount None on FIRST (multiplayer_wrapper.py:80-130).
  rgb = [np.full((2, 2, 3), i, np.uint8) for i in range(2)]
  world = np.zeros((4, 4, 3), np.uint8)
  obs = [{'RGB': rgb[i], 'READY_TO_SHOOT': np.float64(i), 'WORLD.RGB': world, 'COLLECTIVE_REWARD': np.float64(3.0)} for i in range(2)]
  ts = dm_env.TimeStep(dm_env.StepType.MID, [np.float64(1.0), np.float64(2.0)], 1.0, obs)
  flat = substrate.flat_timestep(ts, ['RGB', 'READY_TO_SHOOT'], ['WORLD.RGB'])
  assert set(flat.observation) == {'1.RGB', '1.READY_TO_SHOOT', '1.REWARD', '2.RGB', '2.READY_TO_SHOOT', '2.REWARD', 'WORLD.RGB'}
  assert flat.observation['2.RGB'] is rgb[1] and flat.observation['WORLD.RGB'] is world
  assert flat.observation['1.REWARD'] == 1.0 and flat.observation['2.REWARD'] == 2.0 and flat.reward == 0.0 and flat.discount == 1.0
  first = substrate.flat_timestep(dm_env.TimeStep(dm_env.StepType.FIRST, [0.0, 0.0], 0.0, obs), ['RGB'], [])
  assert first.reward is None and first.discount is None and set(first.observation) == {'1.RGB', '1.REWARD', '2.RGB', '2.REWARD'}
  action_set = ({'move': 0, 'turn': 0, 'fireZap': 0}, {'move': 1, 'turn': 0, 'fireZap': 0}, {'move': 0, 'turn': -1, 'fireZap': 1})
  act = substrate.flat_action([2, 1], action_set)
  assert {k: int(v) for k, v in act.items()} == {'1.move': 0, '1.turn': -1, '1.fireZap': 1, '2.move': 1, '2.turn': 0, '2.fireZap': 0}
  assert all(v.dtype == np.int32 and v.shape == () for v in act.values())
  fields = {f.name for f in __import__('dataclasses').fields(substrate.SubstrateObservables)}
  assert fields == {'action', 'timestep', 'events', 'dmlab2d'}
  assert all(hasattr(substrate.Substrate, m) for m in ('list_property', 'read_property', 'write_property'))


class _FakeEngine:
  """Stands in for engine.Engine in the host-logic test below: fills the pinned-buffer dict the way mp_reset_host /
  mp_step_host do, with values that depend on the step count (no kernels, no oracle: nothing is computed)."""

  def __init__(self, P, n_scalar, rgb_hw, world_hw, max_events=8):
    self.num_players, self.num_scalar_obs = P, n_scalar
    self.shape = (P, n_scalar, rgb_hw, world_hw, max_events)
    self.t = -1
    self.closed = False

  def make_host_outputs(self, rgb=True, world_rgb=True, events=False):
    import torch
    P, n, (h, w), (H, W), M = self.shape
    block = torch.zeros((P + 2 + max(n, 1) * P,), dtype=torch.float64)
    out = {'scalar_block': block, 'reward': block[:P].view(1, P), 'discount': block[P:P + 1], 'step_type': block[P + 1:P + 2].view(torch.int64),
           'scalar_obs': block[P + 2:].view(max(n, 1), 1, P), 'rgb': torch.zeros((1, P, h, w, 3), dtype=torch.uint8),
           'world_rgb': torch.zeros((1, H, W, 3), dtype=torch.uint8), 'events': torch.zeros((1, M, 3), dtype=torch.int32),
           'event_count': torch.zeros((1,), dtype=torch.int32)}
    return out

  def make_host_actions(self):
    import torch
    return torch.zeros((1, self.num_players), dtype=torch.int32)

  def _fill(self, host, first):
    self.t += 1
    host['step_type'][0] = 0 if first else 1
    host['discount'][0] = 0.0 if first else 1.0
    host['reward'][0] = 0.0 if first else float(self.t)
    host['scalar_obs'][:] = 0.5
    host['rgb'][:] = self.t % 251
    host['world_rgb'][:] = (self.t + 1) % 251
    host['event_count'][0] = 0 if first else 1
    host['events'][0, 0, 0] = 1; host['events'][0, 0, 1] = 1; host['events'][0, 0, 2] = 2   # zap(source 1, target 2)

  def reset_host(self, host):
    self._fill(host, True)

  def step_host(self, actions, host):
    assert tuple(actions.shape) == (1, self.num_players)
    self.last_actions = actions.clone()
    self._fill(host, False)

  def close(self):
    self.closed = True


def test_substrate_host_logic_on_a_fake_engine():
  # Substrate (the dm_env view, B = 1): timestep assembly, fresh arrays per step, shared WORLD.RGB object, COLLECTIVE_REWARD,
  # action validation, events, all three observable levels incl. observables().dmlab2d, close().
  config = substrate.get_config('clean_up')
  env = substrate.Substrate.__new__(substrate.Substrate)
  fake = _FakeEngine(7, 2, (88, 88), (168, 240))

  class _Batched:
    engine = fake
    num_players = 7
    _world_rgb = True
    _scalar_names = ['READY_TO_SHOOT', 'NUM_OTHERS_WHO_CLEANED_THIS_STEP']

    def close(self):
      fake.close()

  import torch
  env._torch = torch
  env._config = config
  env._batched = _Batched()
  env._num_players = 7
  env._individual = list(config.individual_observation_names)
  env._global = list(config.global_observation_names)
  env._action_subject, env._timestep_subject, env._events_subject = substrate.Subject(), substrate.Subject(), substrate.Subject()
  env._raw = substrate.Lab2dObservables(action=substrate.Subject(), timestep=substrate.Subject(), events=substrate.Subject())
  env._observables = substrate.SubstrateObservables(dmlab2d=env._raw, action=env._action_subject, timestep=env._timestep_subject, events=env._events_subject)
  env._closed, env._last_observation, env._last_events, env._host = False, None, np.zeros((0, 3), np.int32), None
  seen = {k: [] for k in ('action', 'timestep', 'events', 'raw_action', 'raw_timestep', 'raw_events')}
  env.observables().action.subscribe(seen['action'].append)
  env.observables().timestep.subscribe(seen['timestep'].append)
  env.observables().events.subscribe(seen['events'].append)
  env.observables().dmlab2d.action.subscribe(seen['raw_action'].append)
  env.observables().dmlab2d.timestep.subscribe(seen['raw_timestep'].append)
  env.observables().dmlab2d.events.subscribe(seen['raw_events'].append)
  ts0 = env.reset()
  assert ts0.step_type == dm_env.StepType.FIRST and ts0.discount == 0.0 and ts0.reward == [0.0] * 7
  assert set(ts0.observation[0]) == {'RGB', 'READY_TO_SHOOT', 'NUM_OTHERS_WHO_CLEANED_THIS_STEP', 'WORLD.RGB', 'COLLECTIVE_REWARD'}
  assert ts0.observation[0]['WORLD.RGB'] is ts0.observation[6]['WORLD.RGB'] and ts0.observation[3]['RGB'].shape == (88, 88, 3)
  ts1 = env.step([0, 1, 2, 3, 4, 5, 6])
  assert ts1.step_type == dm_env.StepType.MID and ts1.discount == 1.0 and ts1.reward == [1.0] * 7 and ts1.observation[0]['COLLECTIVE_REWARD'] == 7.0
  assert fake.last_actions.tolist() == [[0, 1, 2, 3, 4, 5, 6]]
  assert int(ts0.observation[0]['RGB'][0, 0, 0]) == 0 and int(ts1.observation[0]['RGB'][0, 0, 0]) == 1   # fresh arrays each step
  assert env.events() == [('zap', [b'dict', b'source', np.array(1.0), b'target', np.array(2.0)])]
  assert env.observation() is not None and len(env.observation()) == 7
  with pytest.raises(ValueError):
    env.step([0] * 6)
  with pytest.raises(ValueError):
    env.step([9] * 7)
  assert env.list_property('') == []
  with pytest.raises(KeyError):
    env.read_property('x')
  assert len(seen['action']) == 1 and len(seen['timestep']) == 2 and len(seen['events']) == 1
  assert len(seen['raw_timestep']) == 2 and len(seen['raw_action']) == 1 and len(seen['raw_events']) == 1
  raw = seen['raw_timestep'][1]
  assert raw.reward == 0.0 and raw.discount == 1.0 and raw.observation['3.REWARD'] == 1.0 and '7.RGB' in raw.observation and 'WORLD.RGB' in raw.observation
  assert seen['raw_timestep'][0].reward is None and seen['raw_timestep'][0].discount is None
  assert int(seen['raw_action'][0]['2.move']) == config.action_set[1]['move']
  done = []
  env.observables().timestep.subscribe(on_completed=lambda: done.append(1))
  env.close()
  assert fake.closed and done == [1]
