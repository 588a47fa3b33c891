"""ctypes binding for the CPU oracle (oracle/mp_oracle.c). TEST INFRASTRUCTURE ONLY.

Only `tests/`, `__graft_entry__.smoke()` and `bench.py`'s cpu_baseline /
`--impl reference` legs may import this module; nothing under `meltingpot_b200/` does.
"""

from __future__ import annotations

import ctypes
import os
import subprocess

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
_LIB_PATH = os.path.join(_HERE, 'liboracle.so')
_lib = None


def build(force: bool = False) -> str:
  """Compiles liboracle.so with the recipe in oracle/Makefile."""
  src = os.path.join(_HERE, 'mp_oracle.c')
  stale = (not os.path.exists(_LIB_PATH) or
           os.path.getmtime(_LIB_PATH) < os.path.getmtime(src))
  if force or stale:
    subprocess.check_call(['make', '-C', _HERE, '-s', '-B', 'liboracle.so'])
  return _LIB_PATH


def lib() -> ctypes.CDLL:
  global _lib
  if _lib is None:
    if not os.path.exists(_LIB_PATH):
      build()
    L = ctypes.CDLL(_LIB_PATH)
    vp, i32p, u8p, f64p = (ctypes.c_void_p, ctypes.POINTER(ctypes.c_int32),
                           ctypes.POINTER(ctypes.c_uint8), ctypes.POINTER(ctypes.c_double))
    L.oracle_create.restype = vp
    L.oracle_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_uint64]
    L.oracle_destroy.argtypes = [vp]
    L.oracle_reset.argtypes = [vp]
    L.oracle_set_episode.argtypes = [vp, ctypes.c_int]
    L.oracle_step.argtypes = [vp, i32p]
    L.oracle_get_rewards.argtypes = [vp, f64p]
    L.oracle_get_discount.argtypes = [vp]
    L.oracle_get_discount.restype = ctypes.c_double
    L.oracle_get_step_type.argtypes = [vp]
    L.oracle_get_scalar_obs.argtypes = [vp, f64p]
    L.oracle_get_avatars.argtypes = [vp, i32p]
    L.oracle_get_grid.argtypes = [vp, ctypes.POINTER(ctypes.c_uint16)]
    L.oracle_get_events.argtypes = [vp, i32p, ctypes.c_int]
    L.oracle_layer_view.argtypes = [vp, ctypes.c_int, i32p]
    L.oracle_get_object_state.argtypes = [vp, ctypes.c_int]
    L.oracle_get_counters.argtypes = [vp, i32p]
    L.oracle_render_player.argtypes = [vp, ctypes.c_int, u8p]
    L.oracle_render_world.argtypes = [vp, u8p]
    L.oracle_debug_set_avatar.argtypes = [vp] + [ctypes.c_int] * 4
    L.oracle_debug_set_object_state.argtypes = [vp, ctypes.c_int, ctypes.c_int]
    L.oracle_philox.argtypes = [ctypes.POINTER(ctypes.c_uint32)] * 3
    L.oracle_run_random.restype = ctypes.c_long
    L.oracle_run_random.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_int,
                                    ctypes.c_int, ctypes.c_uint64, ctypes.c_int,
                                    ctypes.POINTER(ctypes.c_uint64)]
    L.oracle_batch_create.restype = vp
    L.oracle_batch_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int, ctypes.c_uint64]
    L.oracle_batch_destroy.argtypes = [vp]
    L.oracle_batch_step_random.restype = ctypes.c_long
    L.oracle_batch_step_random.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.c_int]
    L.oracle_batch_step_actions.argtypes = [vp, i32p, ctypes.c_int]
    L.oracle_batch_dump.argtypes = [vp, ctypes.c_int] + [vp] * 8 + [ctypes.c_int, vp, vp]
    L.oracle_batch_checksum.restype = ctypes.c_uint64
    L.oracle_batch_checksum.argtypes = [vp]
    _lib = L
  return _lib


def philox(ctr, key):
  c = (ctypes.c_uint32 * 4)(*ctr)
  k = (ctypes.c_uint32 * 2)(*key)
  o = (ctypes.c_uint32 * 4)()
  lib().oracle_philox(c, k, o)
  return list(o)


def _ptr(arr, ctype):
  return arr.ctypes.data_as(ctypes.POINTER(ctype))


EVENT_NAMES = {1: 'zap', 2: 'edible_consumed', 3: 'player_cleaned', 4: 'claimed_resource',
               5: 'destroyed_resource', 6: 'sanctioning', 7: 'removal_due_to_sanctioning', 8: 'coin_consumed',
               9: 'mining', 10: 'extraction', 11: 'extraction_pair'}


class OracleEnv:
  """One CPU environment instance driven by a compiled blob."""

  def __init__(self, blob: bytes, seed: int):
    from meltingpot_b200 import blob as blob_lib  # layout helpers only
    self._blob = bytes(blob)
    self._h = lib().oracle_create(self._blob, len(self._blob), ctypes.c_uint64(seed))
    if not self._h:
      raise RuntimeError('oracle_create failed')
    sec = blob_lib.unpack(self._blob)
    m = sec['meta']
    self.W, self.H, self.L, self.P, self.S = (int(m[1]), int(m[2]), int(m[3]), int(m[4]), int(m[5]))
    self.view = (int(m[15]), int(m[16]), int(m[17]), int(m[18]))
    self.n_scalar = int(m[23])
    self.n_actions = int(m[19])
    self.rgb_shape = ((self.view[2] + self.view[3] + 1) * self.S,
                      (self.view[0] + self.view[1] + 1) * self.S, 3)
    self.world_shape = (self.H * self.S, self.W * self.S, 3)

  def close(self):
    if self._h:
      lib().oracle_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  def reset(self) -> int:
    return lib().oracle_reset(self._h)

  def set_episode(self, episode: int):
    lib().oracle_set_episode(self._h, episode)

  def step(self, actions) -> int:
    a = np.ascontiguousarray(actions, np.int32)
    assert a.shape == (self.P,)
    return lib().oracle_step(self._h, _ptr(a, ctypes.c_int32))

  def rewards(self):
    out = np.zeros(self.P, np.float64)
    lib().oracle_get_rewards(self._h, _ptr(out, ctypes.c_double))
    return out

  def discount(self) -> float:
    return lib().oracle_get_discount(self._h)

  def step_type(self) -> int:
    return lib().oracle_get_step_type(self._h)

  def scalar_obs(self):
    out = np.zeros((self.P, max(self.n_scalar, 1)), np.float64)
    lib().oracle_get_scalar_obs(self._h, _ptr(out, ctypes.c_double))
    return out[:, :self.n_scalar]

  def avatars(self):
    out = np.zeros((self.P, 4), np.int32)
    lib().oracle_get_avatars(self._h, _ptr(out, ctypes.c_int32))
    return out

  def grid(self):
    out = np.zeros((self.L, self.H * self.W), np.uint16)
    lib().oracle_get_grid(self._h, _ptr(out, ctypes.c_uint16))
    return out

  def events(self):
    out = np.zeros((256, 3), np.int32)
    n = lib().oracle_get_events(self._h, _ptr(out, ctypes.c_int32), 256)
    return [(EVENT_NAMES[int(t)], int(a), int(b)) for t, a, b in out[:min(n, 256)]]

  def layer_view(self):
    vh, vw = self.rgb_shape[0] // self.S, self.rgb_shape[1] // self.S
    out = np.zeros((self.P, vh, vw, self.L), np.int32)
    for p in range(self.P):
      lib().oracle_layer_view(self._h, p, _ptr(out[p], ctypes.c_int32))
    return out

  def object_state(self, oid: int) -> int:
    return lib().oracle_get_object_state(self._h, oid)

  def counters(self):
    out = np.zeros(5, np.int32)
    lib().oracle_get_counters(self._h, _ptr(out, ctypes.c_int32))
    return dict(dirt=int(out[0]), clean=int(out[1]), frame=int(out[2]),
                step=int(out[3]), episode=int(out[4]))

  def rgb(self):
    out = np.zeros((self.P,) + self.rgb_shape, np.uint8)
    for p in range(self.P):
      lib().oracle_render_player(self._h, p, _ptr(out[p], ctypes.c_uint8))
    return out

  def world_rgb(self):
    out = np.zeros(self.world_shape, np.uint8)
    lib().oracle_render_world(self._h, _ptr(out, ctypes.c_uint8))
    return out

  def debug_set_avatar(self, p, x, y, orient):
    lib().oracle_debug_set_avatar(self._h, p, x, y, orient)

  def debug_set_object_state(self, oid, state):
    lib().oracle_debug_set_object_state(self._h, oid, state)


def run_random(blob: bytes, n_envs: int, n_steps: int, n_threads: int,
               seed: int = 1, render: bool = True):
  """CPU baseline loop in C; returns (env_steps, checksum)."""
  chk = ctypes.c_uint64(0)
  n = lib().oracle_run_random(bytes(blob), len(blob), n_envs, n_steps, n_threads,
                              ctypes.c_uint64(seed), int(render), ctypes.byref(chk))
  return int(n), int(chk.value)


class OracleBatch:
  """Persistent set of CPU envs stepped with uniform-random actions on host threads."""

  def __init__(self, blob: bytes, n_envs: int, seed: int = 1):
    self._blob = bytes(blob)
    self.n_envs = n_envs
    self._h = lib().oracle_batch_create(self._blob, len(self._blob), n_envs, ctypes.c_uint64(seed))
    if not self._h:
      raise RuntimeError('oracle_batch_create failed')

  def step_random(self, n_steps: int, n_threads: int, render: bool = True) -> int:
    return int(lib().oracle_batch_step_random(self._h, n_steps, n_threads, int(render)))

  def checksum(self) -> int:
    return int(lib().oracle_batch_checksum(self._h))

  def step_actions(self, actions, n_threads: int) -> None:
    """Steps every env with the given discrete actions (int32 [n_envs, P]) on host threads."""
    a = np.ascontiguousarray(actions, np.int32)
    assert a.ndim == 2 and a.shape[0] == self.n_envs
    lib().oracle_batch_step_actions(self._h, _ptr(a, ctypes.c_int32), n_threads)

  def dump(self, n_threads: int, shapes, pixels: bool = False, max_events: int = 256, kinds=('rgb', 'world')):
    """Every output of every env, laid out like the engine's buffers. `shapes` = dict(P, L, cells, n_scalar,
    rgb=(h, w), world=(h, w)). Event rows are sorted per env. With `pixels`, the images named in `kinds` too."""
    B, P = self.n_envs, shapes['P']
    out = {
        'reward': np.zeros((B, P), np.float64), 'discount': np.zeros((B,), np.float64),
        'step_type': np.zeros((B,), np.int64), 'scalar_obs': np.zeros((max(shapes['n_scalar'], 1), B, P), np.float64),
        'avatars': np.zeros((B, P, 4), np.int32), 'grid': np.zeros((B, shapes['L'], shapes['cells']), np.uint16),
        'events': np.zeros((B, max_events, 3), np.int32), 'n_events': np.zeros((B,), np.int32),
    }
    if pixels and 'rgb' in kinds:
      out['rgb'] = np.zeros((B, P) + tuple(shapes['rgb']) + (3,), np.uint8)
    if pixels and 'world' in kinds:
      out['world'] = np.zeros((B,) + tuple(shapes['world']) + (3,), np.uint8)
    vp = lambda k: out[k].ctypes.data if k in out else None
    lib().oracle_batch_dump(self._h, n_threads, vp('reward'), vp('discount'), vp('step_type'), vp('scalar_obs'),
                            vp('avatars'), vp('grid'), vp('events'), vp('n_events'), max_events, vp('rgb'), vp('world'))
    return out

  def close(self):
    if self._h:
      lib().oracle_batch_destroy(self._h)
      self._h = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass
