"""ctypes binding of libmpengine.so (include/mp_engine.h) + zero-copy torch views.

PyTorch is used only to wrap the engine's device buffers as tensors and to supply
streams; all compute is in the library's CUDA kernels. There is no CPU path: if
the library or a CUDA device is missing, construction raises.
"""

from __future__ import annotations

import ctypes
import os
from typing import Any, Dict, Mapping, NamedTuple, Optional, Tuple

import numpy as np

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get('MP_ENGINE_LIB') or os.path.join(_HERE, 'libmpengine.so')

MP_FLAG_RENDER_WORLD = 1
MP_FLAG_RENDER_PLAYERS = 2
MP_FLAG_DEFAULT = 3
MP_FLAG_DEBUG_PLAIN_LANE_MAP = 1 << 9
MP_FLAG_DEBUG_SCATTER_LANE_MAP = 1 << 10
MP_FLAG_DEBUG_NO_PREMERGE = 1 << 11
MP_FLAG_LAYOUT_MASK = 0x3ff << 16
# mp_debug_render_plan's lane-map kinds (the default whole-cell dealing is 1 + 16 * spare wavefronts)
LANE_MAP_PLAIN, LANE_MAP_SCATTER = 0, 2

# Ranges of a forced render layout (include/mp_engine.h, MP_RENDER_LAYOUT): teams per CTA, warps per team, log2 of
# the pixel rows per WORLD.RGB strip.
RENDER_LAYOUT_RANGES = ((2, 4), (4, 16), (1, 2))


def pack_render_layout(teams: int, warps: int, wstrip_log2: int) -> int:
  """Flag bits that make mp_create use this render layout instead of the one it scores best."""
  vals = (teams, warps, wstrip_log2)
  for name, v, (lo, hi) in zip(('teams', 'warps', 'wstrip_log2'), vals, RENDER_LAYOUT_RANGES):
    if int(v) != v or not lo <= v <= hi:
      raise ValueError(f'render layout {name}={v!r} outside {lo}..{hi}')
  return (int(teams) << 16) | (int(warps) << 19) | (int(wstrip_log2) << 24)


def unpack_render_layout(flags: int):
  """(teams, warps, wstrip_log2) forced by `flags`, or None when the engine chooses."""
  if not flags & MP_FLAG_LAYOUT_MASK:
    return None
  return (flags >> 16) & 7, (flags >> 19) & 31, (flags >> 24) & 3


def render_layout_candidates():
  """Every (teams, warps, wstrip_log2) the engine's layout search considers (teams * warps <= 32 warps per CTA)."""
  (t0, t1), (w0, w1), (l0, l1) = RENDER_LAYOUT_RANGES
  return [(t, w, l) for t in range(t0, t1 + 1) for w in range(w0, w1 + 1) for l in range(l0, l1 + 1) if t * w <= 32]

EXPORTED_SYMBOLS = (
    'mp_create', 'mp_destroy', 'mp_set_flags', 'mp_run', 'mp_step_state', 'mp_render', 'mp_get_buffers', 'mp_step_host',
    'mp_reset_host', 'mp_launch_count', 'mp_algorithmic_bytes', 'mp_debug_render_tables', 'mp_debug_render_plan', 'mp_state_size', 'mp_state_save', 'mp_state_load',
    'mp_step_host_async', 'mp_wait', 'mp_exchange_create', 'mp_ipc_export', 'mp_ipc_open', 'mp_enable_peer_access',
    'mp_exchange_connect', 'mp_exchange_wait', 'mp_exchange_slot', 'mp_debug_lane_map', 'mp_debug_observations',
    'mp_gather_obs_create', 'mp_gather_obs_connect', 'mp_gather_obs_enable', 'mp_gather_obs_wait', 'mp_gather_obs_slot',
    'mp_create_variants', 'mp_set_env_variants', 'mp_env_variants', 'mp_last_error',
    'mp_version', 'mp_state_record_bytes', 'mp_state_store', 'mp_state_restore', 'mp_debug_last_launch',
)

MP_RESTORE_REKEY = 1


class MpBuffers(ctypes.Structure):
  _fields_ = [
      ('num_envs', ctypes.c_int32), ('num_players', ctypes.c_int32),
      ('rgb_h', ctypes.c_int32), ('rgb_w', ctypes.c_int32),
      ('world_h', ctypes.c_int32), ('world_w', ctypes.c_int32),
      ('num_actions', ctypes.c_int32), ('num_scalar_obs', ctypes.c_int32),
      ('rgb', ctypes.c_void_p), ('world_rgb', ctypes.c_void_p),
      ('reward', ctypes.c_void_p), ('discount', ctypes.c_void_p),
      ('step_type', ctypes.c_void_p), ('scalar_obs', ctypes.c_void_p),
      ('avatar_state', ctypes.c_void_p), ('grid', ctypes.c_void_p),
      ('grid_layers', ctypes.c_int32), ('grid_cells', ctypes.c_int32),
      ('grid_cells_padded', ctypes.c_int32),
      ('timestep_packed', ctypes.c_void_p),
      ('events', ctypes.c_void_p), ('event_count', ctypes.c_void_p), ('max_events', ctypes.c_int32),
      ('scalar_block', ctypes.c_void_p), ('scalar_block_bytes', ctypes.c_uint64),
      ('gathered', ctypes.c_void_p), ('gathered_world', ctypes.c_int32),
      ('gathered_rgb', ctypes.c_void_p), ('gathered_world_rgb', ctypes.c_void_p), ('gathered_obs_slot_bytes', ctypes.c_uint64),
  ]


class MpHostOutputs(ctypes.Structure):
  _fields_ = [
      ('rgb', ctypes.c_void_p), ('world_rgb', ctypes.c_void_p),
      ('reward', ctypes.c_void_p), ('discount', ctypes.c_void_p),
      ('step_type', ctypes.c_void_p), ('scalar_obs', ctypes.c_void_p),
      ('scalar_block', ctypes.c_void_p), ('events', ctypes.c_void_p), ('event_count', ctypes.c_void_p),
  ]


class MpDeviceOutputs(ctypes.Structure):
  _fields_ = [
      ('rgb', ctypes.c_void_p), ('rgb_env_stride', ctypes.c_uint64),
      ('world_rgb', ctypes.c_void_p), ('world_rgb_env_stride', ctypes.c_uint64),
      ('reward', ctypes.c_void_p), ('reward_env_stride', ctypes.c_uint64),
      ('discount', ctypes.c_void_p), ('discount_env_stride', ctypes.c_uint64),
      ('step_type', ctypes.c_void_p), ('step_type_env_stride', ctypes.c_uint64),
      ('scalar_obs', ctypes.c_void_p), ('scalar_obs_env_stride', ctypes.c_uint64), ('scalar_obs_stride', ctypes.c_uint64),
  ]


# The outputs a step can deliver into caller-owned tensors (mp_request.out).
DEVICE_OUTPUTS = ('rgb', 'world_rgb', 'reward', 'discount', 'step_type', 'scalar_obs')


def _strides(label: str, t, lead: int, unit: str, item: int) -> Tuple[int, ...]:
  """The byte strides of the first `lead` axes of `t` (a TensorLayout), which must be dense in every other axis. An
  axis of length 1 gets the stride it would have if dense (its stride is never used)."""
  dense = 1
  for axis in range(len(t.shape) - 1, lead - 1, -1):
    if t.shape[axis] != 1 and t.stride[axis] != dense:
      raise ValueError(f'{label}: axis {axis} has stride {t.stride[axis]}, must be {dense} (only the {unit} axis'
                       f'{" and the observation axis" if lead > 1 else ""} may be strided)')
    dense *= t.shape[axis]
  strides = []
  for axis in range(lead - 1, -1, -1):
    strides.insert(0, (t.stride[axis] if t.shape[axis] > 1 else dense) * item)
    dense *= t.shape[axis]
  return tuple(strides)


MP_MAX_ROW_SEGMENTS = 16


class MpRowSegment(ctypes.Structure):
  _fields_ = [
      ('row_begin', ctypes.c_int32), ('row_end', ctypes.c_int32),
      ('rgb', ctypes.c_void_p), ('rgb_row_stride', ctypes.c_uint64),
      ('reward', ctypes.c_void_p), ('reward_row_stride', ctypes.c_uint64),
      ('scalar_obs', ctypes.c_void_p), ('scalar_obs_row_stride', ctypes.c_uint64), ('scalar_obs_stride', ctypes.c_uint64),
  ]


class MpPlayerOutputs(ctypes.Structure):
  _fields_ = [
      ('row_of_player', ctypes.c_void_p), ('n_rows', ctypes.c_int32),
      ('rgb', ctypes.c_void_p), ('rgb_row_stride', ctypes.c_uint64),
      ('reward', ctypes.c_void_p), ('reward_row_stride', ctypes.c_uint64),
      ('scalar_obs', ctypes.c_void_p), ('scalar_obs_row_stride', ctypes.c_uint64), ('scalar_obs_stride', ctypes.c_uint64),
      ('world_row_of_env', ctypes.c_void_p), ('world_n_rows', ctypes.c_int32),
      ('world_rgb', ctypes.c_void_p), ('world_rgb_row_stride', ctypes.c_uint64),
      ('n_segments', ctypes.c_int32), ('segments', MpRowSegment * MP_MAX_ROW_SEGMENTS),
  ]


# The per-player outputs a step can deliver into rows of caller-owned tensors (mp_request.players).
PLAYER_OUTPUTS = ('rgb', 'reward', 'scalar_obs')
# WORLD.RGB routed per env in the same call: the row map and the rows, given together.
WORLD_OUTPUTS = ('world_row_of_env', 'world_rgb')


def describe_players(players: Mapping[str, Any], rgb_shape: Tuple[int, ...], num_envs: int, num_players: int,
                     num_scalar_obs: int, device: int, world_shape: Optional[Tuple[int, ...]] = None,
                     _rows_only: bool = False) -> MpPlayerOutputs:
  """The mp_player_outputs of `players`: 'row_of_player' (TensorLayout of a contiguous int32 CUDA [B, P]) and any of
  'rgb' (uint8 [n_rows, *rgb_shape], dense inside a row), 'reward' (float64 [n_rows]) and 'scalar_obs' (float64
  [num_scalar_obs, n_rows]); the row axis (and the observation axis of scalar_obs) may have any stride. Every target
  must have the same n_rows. WORLD.RGB rows, optional: 'world_row_of_env' (contiguous int32 CUDA [B]) with 'world_rgb'
  (uint8 [n, *world_shape], dense inside a row, 16-byte aligned rows; world_shape None: the engine renders no
  WORLD.RGB). Only shapes, dtypes, devices and layouts are checked, never the row maps' values.

  Row segments instead of the per-player targets: 'n_rows' (the row map's row count) and 'segments', a sequence of up to
  MP_MAX_ROW_SEGMENTS (row_begin, row_end, {name: TensorLayout}) whose targets are those above for rows
  [row_begin, row_end) only (row r in the segment's row r - row_begin). A row in no segment is not delivered."""
  import torch  # pylint: disable=g-import-not-at-top
  if 'segments' in players:
    return _describe_segments(players, rgb_shape, num_envs, num_players, num_scalar_obs, device, world_shape)
  unknown = set(players) - set(PLAYER_OUTPUTS) - set(WORLD_OUTPUTS) - {'row_of_player'}
  if unknown:
    raise ValueError(f'players: unknown entries {sorted(unknown)} (row_of_player and any of {", ".join(PLAYER_OUTPUTS)}, '
                     f'or {" with ".join(WORLD_OUTPUTS)})')

  def on_device(name, t):
    dev = torch.device(t.device)
    if dev.type != 'cuda' or dev.index != device:
      raise ValueError(f'players[{name!r}]: on {dev}, the engine runs on cuda:{device}')

  rmap = players.get('row_of_player')
  if rmap is None:
    raise ValueError('players: row_of_player is missing')
  if (tuple(rmap.shape) != (num_envs, num_players) or rmap.dtype != torch.int32
      or tuple(rmap.stride) != (num_players, 1)):
    raise ValueError(f'players[\'row_of_player\']: must be a contiguous int32 tensor [{num_envs}, {num_players}]')
  on_device('row_of_player', rmap)
  s = MpPlayerOutputs()
  s.row_of_player = ctypes.c_void_p(int(rmap.data_ptr))
  n_rows = None
  targets = {k: v for k, v in players.items() if k in PLAYER_OUTPUTS and v is not None}
  if not targets and not _rows_only:  # (_rows_only: the row map and WORLD.RGB of a request whose segments hold the rest)
    raise ValueError(f'players: give at least one of {", ".join(PLAYER_OUTPUTS)}')
  for name, t in targets.items():
    row_axis = 1 if name == 'scalar_obs' else 0
    if name == 'scalar_obs' and num_scalar_obs == 0:
      raise ValueError('players[\'scalar_obs\']: this substrate has no scalar observations')
    dtype = torch.uint8 if name == 'rgb' else torch.float64
    inner = tuple(rgb_shape) if name == 'rgb' else ()
    lead = (num_scalar_obs,) if name == 'scalar_obs' else ()
    if len(t.shape) != len(lead) + 1 + len(inner) or tuple(t.shape[:row_axis]) != lead or tuple(t.shape[row_axis + 1:]) != inner:
      raise ValueError(f'players[{name!r}]: shape {tuple(t.shape)}, must be {lead + ("n_rows",) + inner}')
    if t.dtype != dtype:
      raise ValueError(f'players[{name!r}]: dtype {t.dtype}, must be {dtype}')
    on_device(name, t)
    rows = int(t.shape[row_axis])
    if rows < 1:
      raise ValueError(f'players[{name!r}]: no rows')
    if n_rows is None:
      n_rows = rows
    elif rows != n_rows:
      raise ValueError(f'players[{name!r}]: {rows} rows, another target has {n_rows}')
    strides = _strides(f'players[{name!r}]', t, row_axis + 1, 'row', torch.empty((), dtype=dtype).element_size())
    setattr(s, name, ctypes.c_void_p(int(t.data_ptr)))
    setattr(s, f'{name}_row_stride', strides[-1])
    if name == 'scalar_obs':
      s.scalar_obs_stride = strides[0]
  s.n_rows = n_rows or 0
  wmap, world = players.get('world_row_of_env'), players.get('world_rgb')
  if (wmap is None) != (world is None):
    raise ValueError('players: world_row_of_env and world_rgb go together')
  if world is not None:
    if world_shape is None:
      raise ValueError('players[\'world_rgb\']: this engine renders no WORLD.RGB')
    if tuple(wmap.shape) != (num_envs,) or wmap.dtype != torch.int32 or (num_envs > 1 and tuple(wmap.stride) != (1,)):
      raise ValueError(f'players[\'world_row_of_env\']: must be a contiguous int32 tensor [{num_envs}]')
    on_device('world_row_of_env', wmap)
    inner = tuple(world_shape)
    if len(world.shape) != 1 + len(inner) or tuple(world.shape[1:]) != inner:
      raise ValueError(f'players[\'world_rgb\']: shape {tuple(world.shape)}, must be {("n",) + inner}')
    if world.dtype != torch.uint8:
      raise ValueError(f'players[\'world_rgb\']: dtype {world.dtype}, must be torch.uint8')
    on_device('world_rgb', world)
    rows = int(world.shape[0])
    if rows < 1:
      raise ValueError('players[\'world_rgb\']: no rows')
    (row_stride,) = _strides('players[\'world_rgb\']', world, 1, 'row', 1)
    if world.data_ptr % 16 or row_stride % 16:
      raise ValueError('players[\'world_rgb\']: the pointer and the row stride must be multiples of 16 bytes')
    s.world_row_of_env = ctypes.c_void_p(int(wmap.data_ptr))
    s.world_n_rows = rows
    s.world_rgb = ctypes.c_void_p(int(world.data_ptr))
    s.world_rgb_row_stride = row_stride
  return s


def _describe_segments(players, rgb_shape, num_envs, num_players, num_scalar_obs, device, world_shape) -> MpPlayerOutputs:
  """describe_players with row segments: each segment's targets are described as a players dict of its own rows, so
  they take exactly the checks of top-level targets; the C call checks the table (order, range, one set of outputs)."""
  unknown = set(players) - set(WORLD_OUTPUTS) - {'row_of_player', 'n_rows', 'segments'}
  if unknown:
    raise ValueError(f'players: unknown entries {sorted(unknown)} with segments (row_of_player, n_rows, segments, '
                     f'optionally {" with ".join(WORLD_OUTPUTS)})')
  segments = list(players['segments'])
  if not 1 <= len(segments) <= MP_MAX_ROW_SEGMENTS:
    raise ValueError(f'players: {len(segments)} segments, must be 1..{MP_MAX_ROW_SEGMENTS}')
  n_rows = players.get('n_rows')
  if n_rows is None or int(n_rows) < 1:
    raise ValueError('players: segments need n_rows >= 1, the row count of the row map')
  base = {k: players.get(k) for k in ('row_of_player',) + WORLD_OUTPUTS if players.get(k) is not None}
  s = describe_players(base, rgb_shape, num_envs, num_players, num_scalar_obs, device, world_shape, _rows_only=True)
  s.n_rows = int(n_rows)
  s.n_segments = len(segments)
  for k, (begin, end, targets) in enumerate(segments):
    begin, end = int(begin), int(end)
    if end - begin < 1:
      raise ValueError(f'players: segment {k} rows [{begin}, {end}) are empty')
    one = describe_players(dict(targets, row_of_player=players['row_of_player']), rgb_shape, num_envs, num_players,
                           num_scalar_obs, device, world_shape)
    if one.n_rows != end - begin:
      raise ValueError(f'players: segment {k} targets have {one.n_rows} rows, rows [{begin}, {end}) are {end - begin}')
    g = s.segments[k]
    g.row_begin, g.row_end = begin, end
    for name in ('rgb', 'rgb_row_stride', 'reward', 'reward_row_stride', 'scalar_obs', 'scalar_obs_row_stride',
                 'scalar_obs_stride'):
      setattr(g, name, getattr(one, name))
  return s


class MpPlayerActions(ctypes.Structure):
  _fields_ = [
      ('row_of_player', ctypes.c_void_p), ('n_rows', ctypes.c_int32),
      ('action', ctypes.c_void_p), ('action_row_stride', ctypes.c_uint64),
  ]


MP_MAX_ROUTE_CHOICES = 8
MP_MAX_ROUTE_PLAYERS = 16


class MpRouteDraw(ctypes.Structure):
  _fields_ = [
      ('row_of_player', ctypes.c_void_p), ('n_rows', ctypes.c_int32),
      ('n_choices', ctypes.c_int32 * MP_MAX_ROUTE_PLAYERS),
      ('row_base', (ctypes.c_int32 * MP_MAX_ROUTE_CHOICES) * MP_MAX_ROUTE_PLAYERS),
      ('rows_per_env', (ctypes.c_int32 * MP_MAX_ROUTE_CHOICES) * MP_MAX_ROUTE_PLAYERS),
  ]


def describe_draw(row_of_player, n_rows: int, row_base, rows_per_env) -> MpRouteDraw:
  """The mp_route_draw of drawn routes: row_of_player is the CUDA int32 [B, P] map the engine writes, row_base[p] and
  rows_per_env[p] list the row base and rows per env of each of slot p's choices (as many as it has)."""
  d = MpRouteDraw()
  d.row_of_player = ctypes.c_void_p(int(row_of_player.data_ptr()))
  d.n_rows = int(n_rows)
  for p, (bases, per_env) in enumerate(zip(row_base, rows_per_env)):
    d.n_choices[p] = len(bases)
    for j, (r, n) in enumerate(zip(bases, per_env)):
      d.row_base[p][j], d.rows_per_env[p][j] = int(r), int(n)
  return d


class MpRequest(ctypes.Structure):
  _fields_ = [
      ('reset', ctypes.c_int32), ('env_mask', ctypes.c_void_p), ('actions', ctypes.c_void_p),
      ('player_actions', ctypes.POINTER(MpPlayerActions)), ('draw', ctypes.POINTER(MpRouteDraw)),
      ('slot_of_env', ctypes.c_void_p), ('bank', ctypes.c_void_p), ('n_slots', ctypes.c_int32), ('restore_flags', ctypes.c_uint32),
      ('out', ctypes.POINTER(MpDeviceOutputs)), ('players', ctypes.POINTER(MpPlayerOutputs)),
  ]


def describe_player_actions(player_actions: Mapping[str, Any], num_envs: int, num_players: int, device: int) -> MpPlayerActions:
  """The mp_player_actions of `player_actions`: 'row_of_player' (TensorLayout of a contiguous int32 CUDA [B, P]) and
  'action' (int32 [n_rows], any row stride). Only shapes, dtypes, devices and layouts are checked, never the values."""
  import torch  # pylint: disable=g-import-not-at-top
  unknown = set(player_actions) - {'row_of_player', 'action'}
  if unknown:
    raise ValueError(f'player_actions: unknown entries {sorted(unknown)} (row_of_player and action)')
  rmap, action = player_actions.get('row_of_player'), player_actions.get('action')
  if rmap is None or action is None:
    raise ValueError('player_actions: needs both row_of_player and action')
  if (tuple(rmap.shape) != (num_envs, num_players) or rmap.dtype != torch.int32
      or tuple(rmap.stride) != (num_players, 1)):
    raise ValueError(f'player_actions[\'row_of_player\']: must be a contiguous int32 tensor [{num_envs}, {num_players}]')
  if len(action.shape) != 1 or action.dtype != torch.int32:
    raise ValueError(f'player_actions[\'action\']: must be an int32 tensor [n_rows], got {action.dtype} {tuple(action.shape)}')
  if action.shape[0] < 1:
    raise ValueError('player_actions[\'action\']: no rows')
  for name, t in (('row_of_player', rmap), ('action', action)):
    dev = torch.device(t.device)
    if dev.type != 'cuda' or dev.index != device:
      raise ValueError(f'player_actions[{name!r}]: on {dev}, the engine runs on cuda:{device}')
  s = MpPlayerActions()
  s.row_of_player = ctypes.c_void_p(int(rmap.data_ptr))
  s.n_rows = int(action.shape[0])
  s.action = ctypes.c_void_p(int(action.data_ptr))
  s.action_row_stride = (action.stride[0] if action.shape[0] > 1 else 1) * 4  # with one row the stride is never used
  return s


class TensorLayout(NamedTuple):
  """What describe_outputs needs of a tensor: shape and strides in elements, dtype, device and address."""
  shape: Tuple[int, ...]
  stride: Tuple[int, ...]
  dtype: Any
  device: Any
  data_ptr: int


def layout_of(t) -> TensorLayout:
  return TensorLayout(tuple(t.shape), tuple(t.stride()), t.dtype, t.device, int(t.data_ptr()))


def describe_outputs(out: Mapping[str, TensorLayout], views: Mapping[str, Tuple[Tuple[int, ...], Any]], device: int) -> MpDeviceOutputs:
  """The mp_device_outputs of `out` (name -> TensorLayout of a CUDA tensor). `views` maps each output name to the shape
  and dtype of the engine's own view of it; each tensor must have that shape and dtype, live on cuda:`device`, and be
  dense in every axis but the env axis (axis 0; axes 0 and 1 for scalar_obs, whose axis 1 indexes envs). Alignment,
  allocation bounds and overlaps are checked by the C call."""
  import torch  # pylint: disable=g-import-not-at-top
  s = MpDeviceOutputs()
  for name, t in out.items():
    if t is None:
      continue
    if name not in DEVICE_OUTPUTS:
      raise ValueError(f'out: unknown output {name!r} (one of {", ".join(DEVICE_OUTPUTS)})')
    shape, dtype = views[name]
    if tuple(t.shape) != tuple(shape):
      raise ValueError(f'out[{name!r}]: shape {tuple(t.shape)}, the engine\'s is {tuple(shape)}')
    if t.dtype != dtype:
      raise ValueError(f'out[{name!r}]: dtype {t.dtype}, the engine\'s is {dtype}')
    dev = torch.device(t.device)
    if dev.type != 'cuda' or dev.index != device:
      raise ValueError(f'out[{name!r}]: on {dev}, the engine runs on cuda:{device}')
    strides = _strides(f'out[{name!r}]', t, 2 if name == 'scalar_obs' else 1, 'env', torch.empty((), dtype=dtype).element_size())
    setattr(s, name, ctypes.c_void_p(int(t.data_ptr)))
    setattr(s, f'{name}_env_stride', strides[-1])
    if name == 'scalar_obs':
      s.scalar_obs_stride = strides[0]
  return s


_lib = None


def load_library() -> ctypes.CDLL:
  """Loads libmpengine.so; raises if it has not been built (no fallback)."""
  global _lib
  if _lib is not None:
    return _lib
  if not os.path.exists(LIB_PATH):
    raise RuntimeError(
        f'{LIB_PATH} is missing: build it with `python -m meltingpot_b200.build` '
        '(the engine has no CPU or PyTorch fallback)')
  lib = ctypes.CDLL(LIB_PATH)
  vp = ctypes.c_void_p
  lib.mp_create.argtypes = [ctypes.c_char_p, ctypes.c_size_t, ctypes.c_int,
                            ctypes.c_int, ctypes.c_uint64, ctypes.c_uint64,
                            ctypes.c_uint32, ctypes.POINTER(vp)]
  lib.mp_create_variants.argtypes = [ctypes.POINTER(ctypes.c_char_p), ctypes.POINTER(ctypes.c_size_t), ctypes.c_int, vp,
                                     ctypes.c_int, ctypes.c_int, ctypes.c_uint64, ctypes.c_uint64, ctypes.c_uint32,
                                     ctypes.POINTER(vp)]
  lib.mp_set_env_variants.argtypes = [vp, vp, vp]
  lib.mp_env_variants.argtypes = [vp, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(vp), ctypes.POINTER(vp)]
  lib.mp_destroy.argtypes = [vp]
  lib.mp_set_flags.argtypes = [vp, ctypes.c_uint32]
  lib.mp_run.argtypes = [vp, ctypes.POINTER(MpRequest), vp]
  lib.mp_step_state.argtypes = [vp, vp, vp]
  lib.mp_render.argtypes = [vp, vp]
  lib.mp_get_buffers.argtypes = [vp, ctypes.POINTER(MpBuffers)]
  lib.mp_step_host.argtypes = [vp, vp, ctypes.POINTER(MpHostOutputs), vp]
  lib.mp_reset_host.argtypes = [vp, ctypes.POINTER(MpHostOutputs), vp]
  lib.mp_launch_count.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64)]
  lib.mp_algorithmic_bytes.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64),
                                       ctypes.POINTER(ctypes.c_uint64)]
  lib.mp_state_size.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64)]
  lib.mp_state_save.argtypes = [vp, vp, vp]
  lib.mp_state_load.argtypes = [vp, vp, ctypes.c_uint64, vp]
  lib.mp_state_record_bytes.argtypes = [vp, ctypes.POINTER(ctypes.c_uint64), vp]
  lib.mp_state_store.argtypes = [vp, vp, ctypes.c_int, vp, vp]
  lib.mp_state_restore.argtypes = [vp, vp, vp, ctypes.c_int, ctypes.c_uint32, vp]
  lib.mp_debug_render_plan.argtypes = [vp, ctypes.POINTER(ctypes.c_int32)]
  lib.mp_debug_last_launch.argtypes = [vp, ctypes.POINTER(ctypes.c_int32)]
  lib.mp_debug_render_tables.argtypes = [vp, ctypes.POINTER(ctypes.c_int32), vp, vp]
  lib.mp_step_host_async.argtypes = [vp, vp, ctypes.POINTER(MpHostOutputs), ctypes.c_int, vp]
  lib.mp_wait.argtypes = [vp, ctypes.c_int]
  lib.mp_exchange_create.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_uint64)]
  lib.mp_ipc_export.argtypes = [vp, vp, ctypes.POINTER(ctypes.c_uint64)]
  lib.mp_ipc_open.argtypes = [ctypes.c_int, vp, ctypes.c_uint64, ctypes.POINTER(vp)]
  lib.mp_enable_peer_access.argtypes = [ctypes.c_int, ctypes.c_int]
  lib.mp_exchange_connect.argtypes = [vp, ctypes.POINTER(vp)]
  lib.mp_exchange_wait.argtypes = [vp, vp]
  lib.mp_exchange_slot.argtypes = [vp, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_uint64)]
  lib.mp_gather_obs_create.argtypes = [vp, ctypes.c_int, ctypes.c_int, ctypes.POINTER(vp), ctypes.POINTER(ctypes.c_uint64)]
  lib.mp_gather_obs_connect.argtypes = [vp, ctypes.POINTER(vp)]
  lib.mp_gather_obs_enable.argtypes = [vp, ctypes.c_int]
  lib.mp_gather_obs_wait.argtypes = [vp, vp]
  lib.mp_gather_obs_slot.argtypes = [vp, ctypes.POINTER(ctypes.c_int), ctypes.POINTER(ctypes.c_uint64)]
  lib.mp_debug_observations.argtypes = [vp] * 6
  lib.mp_debug_lane_map.argtypes = [ctypes.c_int] * 5 + [ctypes.POINTER(ctypes.c_uint32)]
  lib.mp_last_error.restype = ctypes.c_char_p
  lib.mp_version.restype = ctypes.c_char_p
  _lib = lib
  return lib


EVENT_NAMES = {1: 'zap', 2: 'edible_consumed', 3: 'player_cleaned', 4: 'claimed_resource',
               5: 'destroyed_resource', 6: 'sanctioning', 7: 'removal_due_to_sanctioning', 8: 'coin_consumed',
               9: 'mining', 10: 'extraction', 11: 'extraction_pair'}
# argument names of each event's dict payload (second one unused for single-argument events)
EVENT_FIELDS = {1: ('source', 'target'), 2: ('player_index',), 3: ('player_index',), 4: ('player_index',),
                5: ('player_index',), 6: ('source', 'target'), 7: ('source', 'target'), 8: ('player_index', 'matched'),
                9: ('player', 'ore_type'), 10: ('player', 'ore_type'), 11: ('player_a', 'player_b_and_ore_type')}


class EngineError(RuntimeError):
  pass


def _check(rc: int) -> None:
  if rc != 0:
    msg = load_library().mp_last_error().decode('utf-8', 'replace')
    if rc in (-1, -2):
      raise ValueError(f'mp_engine error {rc}: {msg}')
    raise EngineError(f'mp_engine error {rc}: {msg}')


class _Handle:
  """Owns one mp_handle. Every tensor view of the engine's buffers holds a reference, so the device memory is
  released (mp_destroy) only once the Engine has been closed AND the last view is gone: a retained observation
  tensor can never dangle."""

  def __init__(self, lib, handle):
    self._lib = lib
    self.h = handle

  def __del__(self):
    try:
      if self.h:
        self._lib.mp_destroy(self.h)
        self.h = None
    except Exception:  # pylint: disable=broad-except
      pass


class _CudaView:
  """Exposes a raw device pointer through __cuda_array_interface__ (v2)."""

  def __init__(self, ptr: int, shape, typestr: str, owner):
    self._owner = owner  # the _Handle: keeps the device memory alive while tensors exist
    self.__cuda_array_interface__ = {
        'shape': tuple(int(s) for s in shape), 'typestr': typestr,
        'data': (int(ptr), False), 'version': 2, 'strides': None,
    }


class Engine:
  """One engine handle = `num_envs` env instances on one GPU."""

  def __init__(self, blob, num_envs: int, device: int = 0, seed: int = 1,
               env_index_base: int = 0, flags: int = MP_FLAG_DEFAULT, render_layout=None, env_variant=None):
    """blob: one compiled substrate, or a list of compatible variants of one (mp_create_variants), e.g. compiled with
    different `prefab_overrides`; env b then starts under variant env_variant[b] (default 0 for every env).
    render_layout: (teams, warps per team, wstrip_log2) to force instead of the engine's choice (diagnostic)."""
    if render_layout is not None:
      flags = (flags & ~MP_FLAG_LAYOUT_MASK) | pack_render_layout(*render_layout)
    import torch  # pylint: disable=g-import-not-at-top
    if not torch.cuda.is_available():
      raise EngineError('CUDA is not available: the CUDA engine has no CPU path')
    self._torch = torch
    self._lib = load_library()
    blobs = [bytes(b) for b in blob] if isinstance(blob, (list, tuple)) else None
    self._blob = blobs[0] if blobs else bytes(blob)
    self.device = int(device)
    self.num_envs = int(num_envs)
    torch.cuda.init()
    with torch.cuda.device(self.device):
      torch.cuda.current_stream()  # make sure the primary context exists
    handle = ctypes.c_void_p()
    if blobs is None:
      if env_variant is not None:
        raise ValueError('env_variant needs a list of blobs')
      _check(self._lib.mp_create(self._blob, len(self._blob), self.num_envs,
                                 self.device, ctypes.c_uint64(seed),
                                 ctypes.c_uint64(env_index_base),
                                 ctypes.c_uint32(flags), ctypes.byref(handle)))
    else:
      assign = None
      if env_variant is not None:
        ids = np.asarray(env_variant, np.int64).reshape(-1)
        if ids.shape != (self.num_envs,) or ids.min(initial=0) < 0 or ids.max(initial=0) >= len(blobs):
          raise ValueError(f'env_variant must hold {self.num_envs} variant indices in 0..{len(blobs) - 1}')
        assign = np.ascontiguousarray(ids, np.uint8)
      arr = (ctypes.c_char_p * len(blobs))(*blobs)
      sizes = (ctypes.c_size_t * len(blobs))(*[len(b) for b in blobs])
      _check(self._lib.mp_create_variants(arr, sizes, len(blobs), assign.ctypes.data if assign is not None else None,
                                          self.num_envs, self.device, ctypes.c_uint64(seed),
                                          ctypes.c_uint64(env_index_base), ctypes.c_uint32(flags),
                                          ctypes.byref(handle)))
    self._owner = _Handle(self._lib, handle)
    self._h = handle
    bufs = MpBuffers()
    _check(self._lib.mp_get_buffers(self._h, ctypes.byref(bufs)))
    self.buffers = bufs
    self.num_players = int(bufs.num_players)
    self.num_actions = int(bufs.num_actions)
    self.num_scalar_obs = int(bufs.num_scalar_obs)
    B, P = self.num_envs, self.num_players
    dev = torch.device('cuda', self.device)

    def view(ptr, shape, typestr, dtype):
      return torch.as_tensor(_CudaView(ptr, shape, typestr, self._owner), device=dev, dtype=dtype)

    self.rgb = view(bufs.rgb, (B, P, bufs.rgb_h, bufs.rgb_w, 3), '|u1', torch.uint8)
    self.world_rgb = view(bufs.world_rgb, (B, bufs.world_h, bufs.world_w, 3), '|u1', torch.uint8)
    self.reward = view(bufs.reward, (B, P), '<f8', torch.float64)
    self.discount = view(bufs.discount, (B,), '<f8', torch.float64)
    self.step_type = view(bufs.step_type, (B,), '<i8', torch.int64)
    self.scalar_obs = view(bufs.scalar_obs, (max(self.num_scalar_obs, 1), B, P), '<f8', torch.float64)
    self.avatar_state = view(bufs.avatar_state, (B, P, 4), '<i4', torch.int32)
    self.grid = view(bufs.grid, (B, bufs.grid_layers, bufs.grid_cells_padded), '<i2', torch.int16)
    self.timestep_packed = view(bufs.timestep_packed, (B, P + 2), '<f8', torch.float64)
    self.events = view(bufs.events, (B, bufs.max_events, 3), '<i4', torch.int32)
    self.event_count = view(bufs.event_count, (B,), '<i4', torch.int32)
    n, active, pending = ctypes.c_int(1), ctypes.c_void_p(), ctypes.c_void_p()
    _check(self._lib.mp_env_variants(self._h, ctypes.byref(n), ctypes.byref(active), ctypes.byref(pending)))
    self.num_variants = int(n.value)
    # uint8 [B]: the variant each env's current episode runs / its next episode will run (None with one variant)
    self.active_variant = view(active.value, (B,), '|u1', torch.uint8) if active.value else None
    self.pending_variant = view(pending.value, (B,), '|u1', torch.uint8) if pending.value else None

  # -- lifecycle -----------------------------------------------------------------
  _VIEWS = ('rgb', 'world_rgb', 'reward', 'discount', 'step_type', 'scalar_obs', 'avatar_state', 'grid',
            'timestep_packed', 'events', 'event_count', 'gathered', 'gathered_rgb', 'gathered_world_rgb',
            'active_variant', 'pending_variant')

  def set_env_variant(self, ids, stream=None) -> None:
    """Assigns env b to variant ids[b] from its next episode start on (the auto-reset after LAST or a reset); an
    episode under way keeps its parameters. Reset envs with a mask to switch them at once."""
    torch = self._torch
    ids = torch.as_tensor(ids)
    if self.num_variants < 2:
      raise ValueError('set_env_variant needs an engine built from a list of blobs')
    if ids.shape != (self.num_envs,) or bool((ids < 0).any()) or bool((ids >= self.num_variants).any()):
      raise ValueError(f'ids must hold {self.num_envs} variant indices in 0..{self.num_variants - 1}')
    ids = ids.to(device=torch.device('cuda', self.device), dtype=torch.uint8).contiguous()
    stream = torch.cuda.current_stream(self.device) if stream is None else stream
    _check(self._lib.mp_set_env_variants(self._h, ctypes.c_void_p(ids.data_ptr()), ctypes.c_void_p(stream.cuda_stream)))
    ids.record_stream(stream)  # the copy reads `ids` on `stream`

  def close(self) -> None:
    """Drops this object's references. mp_destroy runs when the last tensor view handed out has been released too
    (tensors a caller still holds stay readable; the engine itself can no longer be stepped)."""
    if getattr(self, '_h', None):
      self._h = None
      for name in self._VIEWS:
        self.__dict__.pop(name, None)
      self._owner = None

  def __del__(self):
    try:
      self.close()
    except Exception:  # pylint: disable=broad-except
      pass

  def _stream(self, stream) -> ctypes.c_void_p:
    if stream is None:
      stream = self._torch.cuda.current_stream(self.device)
    return ctypes.c_void_p(stream.cuda_stream)

  # -- device-resident API ---------------------------------------------------------
  def set_flags(self, flags: int) -> None:
    _check(self._lib.mp_set_flags(self._h, ctypes.c_uint32(flags)))

  def reset(self, mask=None, stream=None, out=None, players=None, draw=None) -> None:
    """out, players, draw: as for step."""
    r = MpRequest(reset=1)
    if mask is not None:
      assert mask.dtype == self._torch.uint8 and mask.is_cuda and mask.numel() == self.num_envs
      r.env_mask = mask.data_ptr()
    if draw is not None and players is None:
      raise ValueError('draw needs players')
    self._run(r, stream, out, players, draw)

  def step(self, actions, stream=None, out=None, restore=None, bank=None, rekey: bool = False, players=None,
           player_actions=None, draw=None) -> None:
    """actions: int32 CUDA tensor [B, P] of discrete action ids, or None with player_actions.

    One mp_run request (include/mp_engine.h, mp_request) carries the step and everything below.

    out: {name: CUDA tensor} for any of DEVICE_OUTPUTS: the step's images are rendered straight into
    out['rgb'] / out['world_rgb'] instead of this engine's own image buffers, and its scalars are written into the
    others as well as into this engine's buffers. Shapes and dtypes are those of the engine's views (rgb, reward, ...);
    the env axis may have any stride (and the observation axis of scalar_obs), every other axis is dense.

    restore, bank: restore envs within the step. restore is a contiguous CUDA int32 tensor [B] and
    bank a state bank (see restore_states). Env b takes bank row restore[b] instead of stepping, ignoring its action,
    when that index is in 0..n_slots-1 and the row holds one of this engine's records; -1, any other out-of-range index
    and rows without this engine's tag step env b as usual. The result is that of a step followed by
    restore_states(bank, restore, rekey), without the second render. Only the tensors' shape, dtype, device and
    layout are checked, never their values, so the call never synchronises: build the index on the device, e.g.
    `torch.where(step_type == 2, row, -1)`. rekey: as for restore_states.

    players: per-player rows, {'row_of_player': contiguous CUDA int32 [B, P]} plus any of 'rgb'
    (uint8 [n_rows, h, w, 3]), 'reward' (float64 [n_rows]) and 'scalar_obs' (float64 [num_scalar_obs, n_rows]). Player p
    of env b is delivered to row row_of_player[b, p] when that lies in 0..n_rows-1, and nowhere otherwise; with 'rgb'
    the images are drawn straight into the rows, an unrouted player is not drawn at all and this engine's own rgb is
    not written. Combines with out (whose rgb it replaces) and with restore / bank. The row map's values are never
    checked on the host; two players routed to one row leave one of them there. WORLD.RGB may be routed per env in
    the same call: 'world_row_of_env' (contiguous CUDA int32 [B]) with 'world_rgb' (uint8 [n, H, W, 3]); env b's image
    is drawn into row world_row_of_env[b] when that lies in 0..n-1, and not at all otherwise, and this engine's own
    world_rgb is not written (out's world_rgb must then be absent). Instead of 'rgb' / 'reward' / 'scalar_obs', players
    may give 'n_rows' and 'segments': up to 16 sorted, disjoint (row_begin, row_end, {name: tensor}) whose tensors hold
    rows [row_begin, row_end) only, e.g. one trajectory buffer per group; a row in no segment is not delivered.

    player_actions: actions read from rows, {'row_of_player': contiguous CUDA int32 [B, P],
    'action': CUDA int32 [n_rows], any stride}, with actions None. Player p of env b takes action[row_of_player[b, p]]
    when that row lies in 0..n_rows-1, and action 0 (NOOP) otherwise. The row map may be players' own. Combines with
    out, players and restore / bank; the result is that of the same call with the dense actions those rows give.

    draw: drawn routes (an MpRouteDraw from describe_draw), with players and player_actions whose
    row_of_player is the draw's map: the step writes the map (each player's row for the episode its env is in
    afterwards) and reads each player's action from the row of the episode it is in before the step."""
    if draw is not None and (players is None or player_actions is None):
      raise ValueError('draw needs players and player_actions')
    r = MpRequest()
    if player_actions is not None:
      if actions is not None:
        raise ValueError('give actions or player_actions, not both')
      r.player_actions = ctypes.pointer(describe_player_actions(
          {k: (None if v is None else layout_of(v)) for k, v in player_actions.items()}, self.num_envs, self.num_players,
          self.device))
    elif actions is None:
      raise ValueError('actions is None: give actions, or player_actions')
    else:
      self._check_actions(actions)
      r.actions = actions.data_ptr()
    r.restore_flags, r.slot_of_env, r.bank, r.n_slots = self._restore_args(restore, bank, rekey)
    self._run(r, stream, out, players, draw)

  def _run(self, r: MpRequest, stream, out, players, draw) -> None:
    """Adds the targets and drawn routes to request `r` and runs it: one mp_run call."""
    if out is not None:
      r.out = ctypes.pointer(self._device_outputs(out))
    if players is not None:
      r.players = ctypes.pointer(self._player_outputs(players))
    if draw is not None:
      r.draw = ctypes.pointer(draw)
    _check(self._lib.mp_run(self._h, ctypes.byref(r), self._stream(stream)))

  def _restore_args(self, restore, bank, rekey):
    """flags, index pointer, bank pointer and slot count of restore / bank (0, None, None, 0 without them)."""
    if restore is None and bank is None:
      if rekey:
        raise ValueError('rekey needs restore and bank')
      return 0, None, None, 0
    if restore is None or bank is None:
      raise ValueError('restore and bank go together')
    bank = self._bank(bank)
    idx = self._indices(restore, self.num_envs, 'restore')
    for name, t in (('bank', bank), ('restore', idx)):
      if t.device.index != self.device:
        raise ValueError(f'{name} is on {t.device}, the engine runs on cuda:{self.device}')
    return (MP_RESTORE_REKEY if rekey else 0), idx.data_ptr(), bank.data_ptr(), int(bank.shape[0])

  def output_views(self):
    """name -> (shape, dtype) of the engine's own view of each output a step can deliver into caller tensors."""
    return {name: (tuple(getattr(self, name).shape), getattr(self, name).dtype) for name in DEVICE_OUTPUTS}

  def _device_outputs(self, out) -> MpDeviceOutputs:
    return describe_outputs({k: (None if v is None else layout_of(v)) for k, v in out.items()}, self.output_views(), self.device)

  def _player_outputs(self, players) -> MpPlayerOutputs:
    layouts = lambda d: {k: (None if v is None else layout_of(v)) for k, v in d.items()}
    described = layouts({k: v for k, v in players.items() if k not in ('n_rows', 'segments')})
    if 'segments' in players:
      described.update(n_rows=players.get('n_rows'),
                       segments=[(begin, end, layouts(targets)) for begin, end, targets in players['segments']])
    return describe_players(described, tuple(self.rgb.shape[2:]),
                            self.num_envs, self.num_players, self.num_scalar_obs, self.device,
                            tuple(self.world_rgb.shape[1:]))

  def step_state(self, actions, stream=None) -> None:
    self._check_actions(actions)
    _check(self._lib.mp_step_state(self._h, ctypes.c_void_p(actions.data_ptr()), self._stream(stream)))

  def render(self, stream=None) -> None:
    _check(self._lib.mp_render(self._h, self._stream(stream)))

  def _check_actions(self, actions) -> None:
    torch = self._torch
    if (actions.dtype != torch.int32 or not actions.is_cuda or not actions.is_contiguous()
        or actions.shape != (self.num_envs, self.num_players)
        or actions.device.index != self.device):
      raise ValueError('actions must be a contiguous int32 CUDA tensor [B, P] on the engine device')

  # -- host-buffer API (end-to-end path) -----------------------------------------
  def make_host_outputs(self, rgb=True, world_rgb=True, events=False) -> Dict[str, 'np.ndarray']:
    """Pinned host tensors for mp_step_host / mp_step_host_async, as a dict of torch CPU tensors.

    reward / discount / step_type / scalar_obs are views of one pinned block laid out like mp_buffers.scalar_block,
    so the engine moves all scalar outputs of a step with a single device->host copy.
    """
    torch = self._torch
    b = self.buffers
    B, P = self.num_envs, self.num_players
    ns = max(self.num_scalar_obs, 1)
    n_words = int(b.scalar_block_bytes) // 8
    assert n_words == B * P + 2 * B + ns * B * P
    block = torch.empty((n_words,), dtype=torch.float64).pin_memory()
    o = 0
    out = {'scalar_block': block}
    out['reward'] = block[o:o + B * P].view(B, P); o += B * P
    out['discount'] = block[o:o + B]; o += B
    out['step_type'] = block[o:o + B].view(torch.int64); o += B
    out['scalar_obs'] = block[o:o + ns * B * P].view(ns, B, P)
    if rgb:
      out['rgb'] = torch.empty((B, P, b.rgb_h, b.rgb_w, 3), dtype=torch.uint8).pin_memory()
    if world_rgb:
      out['world_rgb'] = torch.empty((B, b.world_h, b.world_w, 3), dtype=torch.uint8).pin_memory()
    if events:
      out['events'] = torch.empty((B, b.max_events, 3), dtype=torch.int32).pin_memory()
      out['event_count'] = torch.empty((B,), dtype=torch.int32).pin_memory()
    return out

  def make_host_actions(self):
    """Pinned int32 [B, P] host tensor for the actions of mp_step_host / mp_step_host_async."""
    return self._torch.zeros((self.num_envs, self.num_players), dtype=self._torch.int32).pin_memory()

  @staticmethod
  def _host_struct(outputs) -> MpHostOutputs:
    s = MpHostOutputs()
    for name in ('rgb', 'world_rgb', 'reward', 'discount', 'step_type', 'scalar_obs', 'scalar_block', 'events', 'event_count'):
      t = outputs.get(name) if outputs else None
      setattr(s, name, ctypes.c_void_p(t.data_ptr()) if t is not None else None)
    return s

  def step_host(self, actions_host, outputs, stream=None) -> None:
    """actions_host: int32 CPU tensor [B, P] (pinned for full speed)."""
    assert actions_host.dtype == self._torch.int32 and not actions_host.is_cuda
    assert actions_host.is_contiguous() and actions_host.shape == (self.num_envs, self.num_players)
    s = self._host_struct(outputs)
    _check(self._lib.mp_step_host(self._h, ctypes.c_void_p(actions_host.data_ptr()),
                                  ctypes.byref(s), self._stream(stream)))

  def step_host_async(self, actions_host, outputs, slot: int, stream=None) -> None:
    """Pipelined step (mp_step_host_async): returns at once; `wait(slot)` before reading `outputs` or reusing
    `actions_host`. Alternate slot 0 / 1 between consecutive calls."""
    assert actions_host.dtype == self._torch.int32 and not actions_host.is_cuda
    assert actions_host.is_contiguous() and actions_host.shape == (self.num_envs, self.num_players)
    s = self._host_struct(outputs)
    _check(self._lib.mp_step_host_async(self._h, ctypes.c_void_p(actions_host.data_ptr()), ctypes.byref(s),
                                        int(slot), self._stream(stream)))

  def wait(self, slot: int) -> None:
    _check(self._lib.mp_wait(self._h, int(slot)))

  # -- stacked timestep across GPUs (mp_exchange_*) ------------------------------------
  def exchange_create(self, rank: int, world: int):
    """Allocates this rank's exchange block; returns (device pointer, bytes)."""
    ptr, n = ctypes.c_void_p(), ctypes.c_uint64(0)
    _check(self._lib.mp_exchange_create(self._h, int(rank), int(world), ctypes.byref(ptr), ctypes.byref(n)))
    self._x_world, self._x_rank = int(world), int(rank)
    bufs = MpBuffers()
    _check(self._lib.mp_get_buffers(self._h, ctypes.byref(bufs)))
    self.buffers = bufs
    torch = self._torch
    self.gathered = torch.as_tensor(
        _CudaView(bufs.gathered, (2, world * self.num_envs, self.num_players + 2), '<f8', self._owner),
        device=torch.device('cuda', self.device), dtype=torch.float64)
    return int(ptr.value), int(n.value)

  def exchange_connect(self, peer_blocks) -> None:
    """peer_blocks: every rank's block pointer (ints) as mapped into this process, in rank order."""
    arr = (ctypes.c_void_p * len(peer_blocks))(*[ctypes.c_void_p(int(p)) for p in peer_blocks])
    _check(self._lib.mp_exchange_connect(self._h, arr))

  def exchange_wait(self, stream=None) -> None:
    _check(self._lib.mp_exchange_wait(self._h, self._stream(stream)))

  def exchange_slot(self):
    slot, step = ctypes.c_int(0), ctypes.c_uint64(0)
    _check(self._lib.mp_exchange_slot(self._h, ctypes.byref(slot), ctypes.byref(step)))
    return int(slot.value), int(step.value)

  def gathered_timestep(self):
    """The stacked [world * B, P + 2] timestep rows of the most recent step (call exchange_wait first)."""
    return self.gathered[self.exchange_slot()[0]]

  # -- stacked observations across GPUs (mp_gather_obs_*) ----------------------------------
  def gather_obs_create(self, rank: int, world: int):
    """Allocates this rank's stacked-observation block; returns (device pointer, bytes)."""
    ptr, n = ctypes.c_void_p(), ctypes.c_uint64(0)
    _check(self._lib.mp_gather_obs_create(self._h, int(rank), int(world), ctypes.byref(ptr), ctypes.byref(n)))
    bufs = MpBuffers()
    _check(self._lib.mp_get_buffers(self._h, ctypes.byref(bufs)))
    self.buffers = bufs
    torch = self._torch
    dev = torch.device('cuda', self.device)
    B, P = self.num_envs, self.num_players
    slot = int(bufs.gathered_obs_slot_bytes)
    self.gathered_rgb = [torch.as_tensor(_CudaView(bufs.gathered_rgb + k * slot, (world * B, P, bufs.rgb_h, bufs.rgb_w, 3), '|u1', self._owner),
                                         device=dev, dtype=torch.uint8) for k in range(2)]
    self.gathered_world_rgb = [torch.as_tensor(_CudaView(bufs.gathered_world_rgb + k * slot, (world * B, bufs.world_h, bufs.world_w, 3), '|u1', self._owner),
                                               device=dev, dtype=torch.uint8) for k in range(2)]
    return int(ptr.value), int(n.value)

  def gather_obs_connect(self, peer_blocks) -> None:
    arr = (ctypes.c_void_p * len(peer_blocks))(*[ctypes.c_void_p(int(p)) for p in peer_blocks])
    _check(self._lib.mp_gather_obs_connect(self._h, arr))

  def gather_obs_enable(self, on: bool) -> None:
    _check(self._lib.mp_gather_obs_enable(self._h, int(bool(on))))

  def gather_obs_wait(self, stream=None) -> None:
    _check(self._lib.mp_gather_obs_wait(self._h, self._stream(stream)))

  def gathered_observations(self):
    """(rgb [world * B, P, h, w, 3], world_rgb [world * B, H, W, 3]) of the most recent render (gather_obs_wait first)."""
    slot = ctypes.c_int(0)
    _check(self._lib.mp_gather_obs_slot(self._h, ctypes.byref(slot), None))
    return self.gathered_rgb[slot.value], self.gathered_world_rgb[slot.value]

  def debug_observations(self, layer: bool = True, zap_matrix: bool = True, stream=None):
    """{'POSITION' [B,P,2], 'ORIENTATION' [B,P], 'LAYER' [B,P,vh,vw,L], 'ZAP_MATRIX' [B,P,P]} int32 CUDA tensors of the
    current timestep (mp_debug_observations)."""
    torch = self._torch
    dev = torch.device('cuda', self.device)
    b = self.buffers
    B, P = self.num_envs, self.num_players
    out = {'POSITION': torch.empty((B, P, 2), dtype=torch.int32, device=dev),
           'ORIENTATION': torch.empty((B, P), dtype=torch.int32, device=dev)}
    if layer:
      out['LAYER'] = torch.empty((B, P, b.rgb_h // 8, b.rgb_w // 8, b.grid_layers), dtype=torch.int32, device=dev)
    if zap_matrix:
      out['ZAP_MATRIX'] = torch.empty((B, P, P), dtype=torch.int32, device=dev)
    ptr = lambda k: ctypes.c_void_p(out[k].data_ptr()) if k in out else None
    _check(self._lib.mp_debug_observations(self._h, ptr('POSITION'), ptr('ORIENTATION'), ptr('LAYER'), ptr('ZAP_MATRIX'),
                                           self._stream(stream)))
    return out

  def reset_host(self, outputs, stream=None) -> None:
    s = self._host_struct(outputs)
    _check(self._lib.mp_reset_host(self._h, ctypes.byref(s), self._stream(stream)))

  # -- introspection -----------------------------------------------------------------
  def launch_count(self) -> int:
    n = ctypes.c_uint64(0)
    _check(self._lib.mp_launch_count(self._h, ctypes.byref(n)))
    return int(n.value)

  def save_state(self, stream=None) -> bytes:
    """Snapshot of every env instance (mp_state_save); restore with load_state on an identically built engine."""
    n = ctypes.c_uint64(0)
    _check(self._lib.mp_state_size(self._h, ctypes.byref(n)))
    buf = ctypes.create_string_buffer(n.value)
    _check(self._lib.mp_state_save(self._h, buf, self._stream(stream)))
    return buf.raw

  def load_state(self, snapshot: bytes, stream=None) -> None:
    snapshot = bytes(snapshot)
    buf = ctypes.create_string_buffer(snapshot, len(snapshot))
    _check(self._lib.mp_state_load(self._h, buf, ctypes.c_uint64(len(snapshot)), self._stream(stream)))

  # -- per-env state bank (mp_state_store / mp_state_restore) ------------------------------
  @property
  def state_record_bytes(self) -> int:
    """Bytes of one env's record in a state bank (a multiple of 16)."""
    n = ctypes.c_uint64(0)
    _check(self._lib.mp_state_record_bytes(self._h, ctypes.byref(n), None))
    return int(n.value)

  @property
  def state_tag(self) -> bytes:
    """The 16 bytes every record this engine stores starts with; a restore skips rows that do not start with them."""
    tag = ctypes.create_string_buffer(16)
    _check(self._lib.mp_state_record_bytes(self._h, None, tag))
    return tag.raw

  def _bank(self, bank):
    torch = self._torch
    if (not isinstance(bank, torch.Tensor) or bank.dtype != torch.uint8 or not bank.is_cuda or bank.dim() != 2
        or bank.shape[1] != self.state_record_bytes or bank.shape[0] < 1 or not bank.is_contiguous()):
      raise ValueError(f'bank must be a contiguous CUDA uint8 tensor [n_slots, {self.state_record_bytes}]')
    return bank

  def _indices(self, idx, n: int, what: str):
    torch = self._torch
    if (not isinstance(idx, torch.Tensor) or idx.dtype != torch.int32 or not idx.is_cuda or idx.shape != (n,)
        or not idx.is_contiguous()):
      raise ValueError(f'{what} must be a contiguous CUDA int32 tensor [{n}]')
    return idx

  def store_states(self, bank, env_of_slot, stream=None) -> None:
    """Bank row k receives env env_of_slot[k] (mp_state_store); rows whose index is outside 0..B-1 are left as they
    are. bank: CUDA uint8 [n_slots, state_record_bytes]; env_of_slot: CUDA int32 [n_slots]. Asynchronous."""
    bank = self._bank(bank)
    idx = self._indices(env_of_slot, bank.shape[0], 'env_of_slot')
    _check(self._lib.mp_state_store(self._h, ctypes.c_void_p(idx.data_ptr()), int(bank.shape[0]),
                                    ctypes.c_void_p(bank.data_ptr()), self._stream(stream)))

  def restore_states(self, bank, slot_of_env, rekey: bool = False, stream=None) -> None:
    """Env b receives bank row slot_of_env[b] (mp_state_restore) when that index is in range and the row carries this
    engine's tag; other envs are left as they are. The batch is then re-rendered. rekey: restored envs draw their random
    numbers under their own key instead of the stored env's. slot_of_env: CUDA int32 [B]. Asynchronous."""
    bank = self._bank(bank)
    idx = self._indices(slot_of_env, self.num_envs, 'slot_of_env')
    _check(self._lib.mp_state_restore(self._h, ctypes.c_void_p(idx.data_ptr()), ctypes.c_void_p(bank.data_ptr()),
                                      int(bank.shape[0]), ctypes.c_uint32(MP_RESTORE_REKEY if rekey else 0),
                                      self._stream(stream)))

  def render_plan(self):
    """Layout the renderer chose for this substrate, the lane maps it built and its k_render<ncp, ncw> (diagnostic)."""
    keys = ('teams', 'team_threads', 'wstrip_log2', 'smem_bytes', 'atlas_sprites', 'rec_stride', 'stage_bytes', 'grid_bytes',
            'lane_map_players', 'lane_map_world', 'ncp', 'ncw')
    out = (ctypes.c_int32 * len(keys))()
    _check(self._lib.mp_debug_render_plan(self._h, out))
    return dict(zip(keys, (int(v) for v in out)))

  # mp_debug_last_launch's fields, in order
  LAST_LAUNCH_FIELDS = ('family', 'variants', 'restore', 'actions', 'render_mode', 'ncp', 'ncw', 'teams', 'warps',
                        'wstrip_log2')

  def last_launch(self):
    """The k_step cell and the k_render mode and layout of the last call that launched either, -1 for a part it did
    not launch (diagnostic): family (MpbFamily), variants (0/1), restore (0/1), actions (0 dense, 1 rows, 2 drawn),
    render_mode (0 plain, 1 gather, 2 routed), the k_render<ncp, ncw> instantiation, teams, warps per team and
    wstrip_log2."""
    out = (ctypes.c_int32 * len(self.LAST_LAUNCH_FIELDS))()
    _check(self._lib.mp_debug_last_launch(self._h, out))
    return dict(zip(self.LAST_LAUNCH_FIELDS, (int(v) for v in out)))

  def render_tables(self):
    """(pair[n, n], flags[n]) uint8 numpy arrays of the renderer's sprite tables (diagnostic)."""
    import numpy as np
    n = ctypes.c_int32(0)
    _check(self._lib.mp_debug_render_tables(self._h, ctypes.byref(n), None, None))
    pair = np.zeros((n.value, n.value), np.uint8)
    flags = np.zeros((n.value,), np.uint8)
    _check(self._lib.mp_debug_render_tables(self._h, ctypes.byref(n), pair.ctypes.data, flags.ctypes.data))
    return pair, flags

  def algorithmic_bytes(self):
    a, r = ctypes.c_uint64(0), ctypes.c_uint64(0)
    _check(self._lib.mp_algorithmic_bytes(self._h, ctypes.byref(a), ctypes.byref(r)))
    return int(a.value), int(r.value)


def ipc_export(device_ptr: int):
  """(64-byte CUDA IPC handle, offset) naming `device_ptr` for another process (mp_ipc_export)."""
  handle = ctypes.create_string_buffer(64)
  off = ctypes.c_uint64(0)
  _check(load_library().mp_ipc_export(ctypes.c_void_p(int(device_ptr)), handle, ctypes.byref(off)))
  return handle.raw, int(off.value)


def ipc_open(device: int, handle: bytes, offset: int) -> int:
  ptr = ctypes.c_void_p()
  buf = ctypes.create_string_buffer(bytes(handle), 64)
  _check(load_library().mp_ipc_open(int(device), buf, ctypes.c_uint64(int(offset)), ctypes.byref(ptr)))
  return int(ptr.value)


def enable_peer_access(device: int, peer_device: int) -> None:
  _check(load_library().mp_enable_peer_access(int(device), int(peer_device)))
