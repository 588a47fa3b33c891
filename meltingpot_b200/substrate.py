"""Public API: drop-in for `meltingpot.substrate` backed by the CUDA engine.

Mirrors `meltingpot/substrate.py:38-113`:
  SUBSTRATES, get_config(name), build(name, *, roles), build_from_config(config, *, roles),
  get_factory(name), get_factory_from_config(config)
and adds `build_batched(...)` for thousands of env instances as torch tensors.

`build(...)` returns a `Substrate` with the reference's dm_env surface and timestep layout
(`meltingpot/utils/substrates/substrate.py:47-104`, wrapper stack `:107-139`):
  * `step(actions)` takes one discrete action id per player (DiscreteActionWrapper);
  * `timestep.reward` is a list of P float64 scalars, `discount` 0.0 on FIRST/LAST else 1.0
    (MultiplayerWrapper, multiplayer_wrapper.py:108-118);
  * `timestep.observation` is a list of P dicts with the configured per-player and global
    observations plus `COLLECTIVE_REWARD` (collective_reward_wrapper.py:39-50);
  * a step after LAST starts a new episode and returns FIRST.
All state transition and rendering runs in the CUDA engine; there is no CPU path.
"""

from __future__ import annotations

import dataclasses
import json
from typing import Any, Callable, Collection, Dict, List, Mapping, Optional, Sequence, Tuple

import numpy as np

from meltingpot_b200 import blob as blob_lib
from meltingpot_b200 import shims
from meltingpot_b200 import specs as specs_lib
from meltingpot_b200 import substrates as substrate_blobs

shims.install()
import dm_env  # noqa: E402  pylint: disable=g-import-not-at-top,g-bad-import-order
from ml_collections import config_dict  # noqa: E402  pylint: disable=g-import-not-at-top,g-bad-import-order

SUBSTRATES = frozenset(substrate_blobs.PRECOMPILED)
_COLLECTIVE_REWARD_OBS = 'COLLECTIVE_REWARD'
_SCALAR_NAMES = {0: 'READY_TO_SHOOT', 1: 'NUM_OTHERS_WHO_CLEANED_THIS_STEP',
                 2: 'MISMATCHED_COIN_COLLECTED_BY_PARTNER'}  # include/mpb_format.h MpbScalarObs
_MAX_SEED = 2**32 - 1


# ---------------------------------------------------------------------------------------------
# Config
# ---------------------------------------------------------------------------------------------
def _info(blob: bytes) -> Dict[str, Any]:
  return json.loads(blob_lib.section_text(blob_lib.unpack(blob), 'info_json'))


def _config_from_info(name: str, info: Mapping[str, Any]) -> config_dict.ConfigDict:
  config = config_dict.ConfigDict()
  config.substrate_name = name
  config.action_set = tuple(dict(a) for a in info['action_set'])
  config.individual_observation_names = list(info['individual_observation_names'])
  config.global_observation_names = list(info['global_observation_names'])
  config.action_spec = specs_lib.action(len(info['action_set']))
  obs = {}
  for key in info['individual_observation_names']:
    obs[key] = specs_lib.rgb(*info['rgb_shape'][:2]) if key == 'RGB' else specs_lib.float64()
  for key in info['global_observation_names']:
    obs[key] = specs_lib.rgb(*info['world_rgb_shape'][:2])
  config.timestep_spec = specs_lib.timestep(obs)
  config.valid_roles = frozenset(info['valid_roles'])
  config.default_player_roles = tuple(info['default_player_roles'])
  return config


def get_config(name: str) -> config_dict.ConfigDict:
  """Returns the locked configuration for the specified substrate (substrate.py:41-54)."""
  if name not in SUBSTRATES:
    raise ValueError(f'{name} not in {sorted(SUBSTRATES)}.')
  blob = substrate_blobs.load_blob(name)
  return _config_from_info(name, _info(blob)).lock()


# ---------------------------------------------------------------------------------------------
# Observables (reactivex is not available here; this is the small subset Substrate exposes)
# ---------------------------------------------------------------------------------------------
class Subject:
  """Minimal hot observable: subscribe(on_next, on_error, on_completed)."""

  def __init__(self):
    self._observers: List[Any] = []

  def subscribe(self, on_next=None, on_error=None, on_completed=None):
    if on_next is not None and not callable(on_next):  # observer object
      observer = on_next
      entry = (getattr(observer, 'on_next', None), getattr(observer, 'on_error', None),
               getattr(observer, 'on_completed', None))
    else:
      entry = (on_next, on_error, on_completed)
    self._observers.append(entry)
    return entry

  def on_next(self, value):
    for fn, _, _ in list(self._observers):
      if fn:
        fn(value)

  def on_completed(self):
    for _, _, fn in list(self._observers):
      if fn:
        fn()
    self._observers.clear()


@dataclasses.dataclass(frozen=True)
class Lab2dObservables:
  """Same fields as the reference's Lab2dObservables (wrappers/observables.py:32-45): the raw dmlab2d-level stream."""
  action: Subject      # {"1.move": ..., "1.turn": ..., ...} per step
  timestep: Subject    # dm_env.TimeStep with the flat {"1.RGB", "1.REWARD", ..., "WORLD.RGB"} observation dict
  events: Subject


@dataclasses.dataclass(frozen=True)
class SubstrateObservables:
  """Same fields as the reference's SubstrateObservables (substrate.py:32-44)."""
  action: Subject
  timestep: Subject
  events: Subject
  dmlab2d: Optional[Lab2dObservables] = None


def flat_action(action: Sequence[int], action_set: Sequence[Mapping[str, int]]) -> Dict[str, np.ndarray]:
  """What the wrapper stack would hand to dmlab2d for these discrete actions (discrete_action_wrapper.py:97-100,
  multiplayer_wrapper.py:120-130): {"<player>.<field>": int32 scalar}."""
  out = {}
  for i, a in enumerate(action):
    for key, value in action_set[int(a)].items():
      out[f'{i + 1}.{key}'] = np.array(value, dtype=np.int32)
  return out


def flat_timestep(timestep: 'dm_env.TimeStep', individual: Sequence[str], global_names: Sequence[str]) -> 'dm_env.TimeStep':
  """The dmlab2d-level view of a multiplayer TimeStep: flat observation dict with "{i}.REWARD" entries, reward None on
  FIRST else 0.0, discount None on FIRST (the inverse of multiplayer_wrapper.py:80-118)."""
  obs = {}
  for i, (player, reward) in enumerate(zip(timestep.observation, timestep.reward)):
    for name in individual:
      obs[f'{i + 1}.{name}'] = player[name]
    obs[f'{i + 1}.REWARD'] = np.float64(reward)
  for name in global_names:
    obs[name] = timestep.observation[0][name]
  first = timestep.step_type == dm_env.StepType.FIRST
  return dm_env.TimeStep(step_type=timestep.step_type, reward=None if first else 0.0,
                         discount=None if first else timestep.discount, observation=obs)


# ---------------------------------------------------------------------------------------------
# Batched substrate (tensors)
# ---------------------------------------------------------------------------------------------
@dataclasses.dataclass
class BatchedTimeStep:
  """One timestep of B env instances; all fields are CUDA tensors viewing engine buffers."""
  step_type: Any   # int64 [B]
  reward: Any      # float64 [B, P]
  discount: Any    # float64 [B]
  observation: Dict[str, Any]


def bank_index(dest, src, n_dest: int, n_src: int, dest_name: str, src_name: str, device=None):
  """The index array of a state-bank call: int32 [n_dest] holding src[i] at dest[i] and -1 everywhere else, built on
  `device`. dest / src are matching sequences or integer tensors; raises ValueError on a length mismatch, an index
  outside 0..n_dest-1 / 0..n_src-1 or a destination named twice."""
  import torch  # pylint: disable=g-import-not-at-top
  d = torch.as_tensor(dest, dtype=torch.int64, device=device).reshape(-1)
  s = torch.as_tensor(src, dtype=torch.int64, device=device).reshape(-1)
  if d.shape != s.shape:
    raise ValueError(f'{dest_name} and {src_name} must have the same length ({d.numel()} vs {s.numel()})')
  if d.numel():
    if bool(((d < 0) | (d >= n_dest)).any()):
      raise ValueError(f'{dest_name} must lie in 0..{n_dest - 1}')
    if bool(((s < 0) | (s >= n_src)).any()):
      raise ValueError(f'{src_name} must lie in 0..{n_src - 1}')
    if torch.unique(d).numel() != d.numel():
      raise ValueError(f'{dest_name} names a destination twice')
  idx = torch.full((n_dest,), -1, dtype=torch.int32, device=device)
  idx[d] = s.to(torch.int32)
  return idx


def check_bank_tags(bank, slots, tag: bytes) -> None:
  """Raises ValueError unless every bank row in `slots` starts with `tag` (the engine's state_tag): a row that was never
  stored, or was stored by an engine of another substrate, would be skipped by the restore. One compare on the bank's
  device."""
  import torch  # pylint: disable=g-import-not-at-top
  s = torch.as_tensor(slots, dtype=torch.int64, device=bank.device).reshape(-1)
  if not s.numel():
    return
  want = torch.frombuffer(bytearray(tag), dtype=torch.uint8).to(bank.device)
  bad = (bank[s, :16] != want).any(dim=1)
  if bool(bad.any()):
    raise ValueError(f'bank rows {s[bad].tolist()} hold no record of this engine (never stored, or stored by an engine '
                     'of another substrate)')


class BatchedSubstrate:
  """`num_envs` independent instances of a substrate on one GPU.

  Observations are zero-copy views of the engine's output buffers and are overwritten by the
  next `step`/`reset`; clone what must be kept, or step into tensors of your own with
  `step(actions, out=traj.at(t))` (see `trajectory`), which costs no copy.

  Single envs can be stored into and restored from a device state bank (`state_bank`, `store`, `restore`), e.g. to
  branch rollouts from one state or restart episodes from stored start states. A clone is a store followed by a
  restore: `store(bank, [i], [0]); restore(bank, [j, k], [0, 0])` makes envs j and k twins of env i, drawing the same
  random numbers as env i would (with `rekey=True` they draw their own).
  """

  def __init__(self, blob, num_envs: int, device: int = 0, seed: Optional[int] = None,
               env_index_base: int = 0, world_rgb: bool = True, env_variant=None):
    """blob: a compiled substrate, or a list of variants of one (e.g. compiled with different `prefab_overrides`),
    env b starting under variant env_variant[b] (see Engine)."""
    from meltingpot_b200 import engine as engine_lib  # pylint: disable=g-import-not-at-top
    if seed is None:
      seed = int(np.random.randint(1, _MAX_SEED))
    first = blob[0] if isinstance(blob, (list, tuple)) else blob
    self._info = _info(first)
    flags = engine_lib.MP_FLAG_RENDER_PLAYERS | (engine_lib.MP_FLAG_RENDER_WORLD if world_rgb else 0)
    self._engine = engine_lib.Engine(blob, num_envs, device=device, seed=seed,
                                     env_index_base=env_index_base, flags=flags, env_variant=env_variant)
    self.num_envs = num_envs
    self.num_players = self._engine.num_players
    self.num_actions = self._engine.num_actions
    self.seed = seed
    sections = blob_lib.unpack(first)
    self._scalar_names = [_SCALAR_NAMES[int(k)] for k in sections['scalar_obs']]
    self._world_rgb = world_rgb

  @property
  def engine(self):
    return self._engine

  def _timestep(self) -> BatchedTimeStep:
    e = self._engine
    obs = {'RGB': e.rgb}
    for k, name in enumerate(self._scalar_names):
      obs[name] = e.scalar_obs[k]
    if self._world_rgb:
      obs['WORLD.RGB'] = e.world_rgb
    obs[_COLLECTIVE_REWARD_OBS] = e.reward.sum(dim=1)
    return BatchedTimeStep(step_type=e.step_type, reward=e.reward, discount=e.discount, observation=obs)

  def reset(self, mask=None, out: Optional[BatchedTimeStep] = None, players: Optional['PlayerOutputs'] = None) -> BatchedTimeStep:
    """out, players: as for step."""
    if players is not None:
      routes = getattr(players, 'routes', None)
      self._engine.reset(mask, out=None if out is None else self._engine_outputs(out, routed=players),
                         players=self._routed_outputs(players),
                         draw=routes.draw if isinstance(routes, DrawnRoutes) else None)
      return self._routed_timestep(self._timestep() if out is None else self._fill_collective(out), players)
    if out is None:
      self._engine.reset(mask)
      return self._timestep()
    self._engine.reset(mask, out=self._engine_outputs(out))
    return self._fill_collective(out)

  def player_routes(self, groups) -> 'PlayerRoutes':
    """Rows for per-player delivery: groups is an integer [B, P] array of group ids (e.g. the policy of each player
    slot), -1 for a player nobody reads. See PlayerRoutes."""
    import torch  # pylint: disable=g-import-not-at-top
    return PlayerRoutes(groups, self.num_envs, self.num_players, tuple(self._engine.rgb.shape[2:]), self._scalar_names,
                        torch.device('cuda', self._engine.device), self._world_shape())

  def drawn_routes(self, choices) -> 'DrawnRoutes':
    """Rows for per-player delivery that are drawn again at every episode start: choices[p] is a sequence of group ids
    (e.g. the bots that may fill slot p), empty for a player nobody reads. See DrawnRoutes."""
    import torch  # pylint: disable=g-import-not-at-top
    return DrawnRoutes(choices, self.num_envs, self.num_players, tuple(self._engine.rgb.shape[2:]), self._scalar_names,
                       torch.device('cuda', self._engine.device), self._world_shape())

  def _world_shape(self):
    """One env's WORLD.RGB shape [H, W, 3], or None when this batch renders no WORLD.RGB."""
    return tuple(self._engine.world_rgb.shape[1:]) if self._world_rgb else None

  def step(self, actions=None, out: Optional[BatchedTimeStep] = None, restore=None, bank=None,
           rekey: bool = False, players: Optional['PlayerOutputs'] = None,
           player_actions: Optional['PlayerActions'] = None) -> BatchedTimeStep:
    """actions: integer tensor [B, P] on the engine's device (int32 preferred), or None with player_actions.

    out: a BatchedTimeStep of caller-owned tensors to fill and return instead of views of the engine's buffers, e.g.
    `trajectory(T).at(t)`: the engine renders the images straight into it and delivers the scalars there too, so a
    learner keeps T steps without copying them.

    restore, bank: restarts or clones envs within this step, at no extra render. restore is a CUDA int32 tensor [B]:
    env b takes bank row restore[b] (a `state_bank` row written by `store`) instead of stepping, and shows that
    record's timestep and images. -1, other out-of-range indices and rows that hold no record of this substrate step
    env b as usual. The values are not checked, so nothing synchronises; e.g. restart finished episodes from stored
    start states with `restore = torch.where(ts.step_type == 2, rows, -1)`. rekey: as for `restore`.

    players: a PlayerOutputs (`player_routes(groups).outputs()`, or `.at(t)` of one with T slots): each routed
    player's image, reward and scalar observations go to its row, the images drawn straight there; unrouted players are
    not drawn. The returned timestep then has no 'RGB'; every other field is as without players. Combines with out and
    restore / bank. With outputs made with world_envs (`outputs(world_envs=envs)`), WORLD.RGB is drawn only for those
    envs, straight into players['WORLD.RGB'] (row k: env envs[k]), and the timestep's 'WORLD.RGB' is that tensor; out's
    'WORLD.RGB' is then left alone. players may also be a GroupOutputs (`group_outputs(slots)`, or `.at(t)` of one with
    slots): each listed group's players go to that group's own tensors, the other groups' players nowhere.

    player_actions: a PlayerActions (`player_routes(groups).actions()`, or `.at(t)` of one with T slots), with actions
    None: each routed player takes the action in its row, an unrouted player action 0 (NOOP). The routes may be the
    players' own, so a learner reads observations from rows and writes actions into the same rows. Combines with out,
    players and restore / bank.

    players and player_actions of one DrawnRoutes (`drawn_routes(choices)`) go together: the step draws each player's
    row again at every episode start (see DrawnRoutes)."""
    import torch  # pylint: disable=g-import-not-at-top
    kw = dict(restore=restore, bank=bank, rekey=rekey)
    routes, action_routes = getattr(players, 'routes', None), getattr(player_actions, 'routes', None)
    if isinstance(routes, DrawnRoutes) or isinstance(action_routes, DrawnRoutes):
      if routes is not action_routes:
        raise ValueError('drawn routes: give players and player_actions of the same DrawnRoutes')
      kw['draw'] = routes.draw
    if player_actions is not None:
      if actions is not None:
        raise ValueError('give actions or player_actions, not both')
      kw['player_actions'] = self._routed_actions(player_actions)
    else:
      if actions is None:
        raise ValueError('actions is None: give actions, or player_actions')
      if actions.dtype != torch.int32:
        actions = actions.to(torch.int32)
      actions = actions.contiguous()
    if players is not None:
      self._engine.step(actions, out=None if out is None else self._engine_outputs(out, routed=players),
                        players=self._routed_outputs(players), **kw)
      return self._routed_timestep(self._timestep() if out is None else self._fill_collective(out), players)
    if out is None:
      self._engine.step(actions, **kw)
      return self._timestep()
    self._engine.step(actions, out=self._engine_outputs(out), **kw)
    return self._fill_collective(out)

  def trajectory(self, T: int, time_major: bool = True) -> 'Trajectory':
    """Tensors for T timesteps of every output, COLLECTIVE_REWARD included, laid out [T, B, ...] (time_major) or
    [B, T, ...]; `at(t)` is slot t as a BatchedTimeStep for step(..., out=) / reset(..., out=)."""
    import torch  # pylint: disable=g-import-not-at-top
    e = self._engine
    return Trajectory(int(T), self.num_envs, self.num_players, e.rgb.shape[1:], e.world_rgb.shape[1:] if self._world_rgb else None,
                      self._scalar_names, bool(time_major), torch.device('cuda', e.device))

  def _routed_outputs(self, po: 'PlayerOutputs'):
    """The engine's per-player targets of a PlayerOutputs (the scalar observations as one [n, n_rows] view), or the
    row segments of a GroupOutputs."""
    if isinstance(po, GroupOutputs):
      self._check_routes(po.routes, 'players')
      if any(T is not None for T in po.slots.values()):
        raise ValueError('players: pick one slot of a GroupOutputs with slots (group_outputs(slots).at(t))')
      targets = {'row_of_player': po.routes.row_of_player, 'n_rows': po.routes.n_rows, 'segments': po.segments()}
      if _routes_world(po):
        if not self._world_rgb:
          raise ValueError('players: WORLD.RGB is routed, but this batch was built with world_rgb=False')
        targets.update(world_row_of_env=po.world_row_of_env, world_rgb=po.world_rgb)
      return targets
    if not isinstance(po, PlayerOutputs):
      raise ValueError('players must be a PlayerOutputs (player_routes(groups).outputs() or drawn_routes(choices).outputs())')
    r = po.routes
    self._check_routes(r, 'players')
    if po.T is not None:
      raise ValueError('players: pick one slot of a PlayerOutputs with T slots (outputs(T).at(t))')
    targets = {'row_of_player': r.row_of_player, 'rgb': po['RGB'], 'reward': po['REWARD'], 'scalar_obs': po.scalar_block}
    if _routes_world(po):
      if not self._world_rgb:
        raise ValueError('players: WORLD.RGB is routed, but this batch was built with world_rgb=False')
      targets.update(world_row_of_env=po.world_row_of_env, world_rgb=po['WORLD.RGB'])
    return targets

  def _check_routes(self, r: 'PlayerRoutes', what: str) -> None:
    import torch  # pylint: disable=g-import-not-at-top
    if (r.num_envs, r.num_players) != (self.num_envs, self.num_players) or r.device != torch.device('cuda', self._engine.device):
      raise ValueError(f'{what}: routes of {r.num_envs} envs x {r.num_players} players on {r.device}, this batch has '
                       f'{self.num_envs} x {self.num_players} on cuda:{self._engine.device}')

  def _routed_actions(self, pa: 'PlayerActions'):
    """The engine's player_actions of a PlayerActions."""
    if not isinstance(pa, PlayerActions):
      raise ValueError('player_actions must be a PlayerActions (player_routes(groups).actions())')
    self._check_routes(pa.routes, 'player_actions')
    if pa.T is not None:
      raise ValueError('player_actions: pick one slot of a PlayerActions with T slots (actions(T).at(t))')
    return {'row_of_player': pa.routes.row_of_player, 'action': pa.tensor}

  @staticmethod
  def _routed_timestep(ts: BatchedTimeStep, po: 'PlayerOutputs') -> BatchedTimeStep:
    """ts without 'RGB' (the rows hold the images), its 'WORLD.RGB' the routed rows when po routes it."""
    obs = {k: v for k, v in ts.observation.items() if k != 'RGB'}
    if _routes_world(po):
      obs['WORLD.RGB'] = po.world_rgb if isinstance(po, GroupOutputs) else po['WORLD.RGB']
    return BatchedTimeStep(step_type=ts.step_type, reward=ts.reward, discount=ts.discount, observation=obs)

  def _engine_outputs(self, ts: BatchedTimeStep, routed=None):
    """The engine's output tensors of a BatchedTimeStep (the scalar observations as one [n, B, P] view). routed: the
    images go to those rows instead, so ts's 'RGB' is left alone (and its 'WORLD.RGB' when routed routes it)."""
    import torch  # pylint: disable=g-import-not-at-top
    obs = ts.observation
    world = self._world_rgb and not (routed is not None and _routes_world(routed))
    out = {'rgb': None if routed is not None else obs.get('RGB'), 'world_rgb': obs.get('WORLD.RGB') if world else None,
           'reward': ts.reward, 'discount': ts.discount, 'step_type': ts.step_type}
    scalars = [obs[name] for name in self._scalar_names if name in obs]
    if scalars:
      if len(scalars) != len(self._scalar_names):
        raise ValueError(f'out: give all of {self._scalar_names} or none')
      first = scalars[0]
      step = (scalars[1].data_ptr() - first.data_ptr()) // first.element_size() if len(scalars) > 1 else first.numel()
      for k, s in enumerate(scalars):  # views of one tensor, evenly spaced, as trajectory() makes them
        if (s.shape != first.shape or s.stride() != first.stride() or s.dtype != first.dtype or s.device != first.device
            or s.untyped_storage().data_ptr() != first.untyped_storage().data_ptr()
            or s.data_ptr() != first.data_ptr() + k * step * first.element_size()):
          raise ValueError('out: the scalar observations must be evenly spaced views of one tensor (see trajectory())')
      out['scalar_obs'] = torch.as_strided(first, (len(scalars),) + tuple(first.shape), (step,) + tuple(first.stride()))
    return out

  def _fill_collective(self, ts: BatchedTimeStep) -> BatchedTimeStep:
    import torch  # pylint: disable=g-import-not-at-top
    collective = ts.observation.get(_COLLECTIVE_REWARD_OBS)
    if collective is not None:
      torch.sum(ts.reward, dim=1, out=collective)
    return ts

  def set_env_variant(self, ids) -> None:
    """Moves env b to variant ids[b] from its next episode start on (reset(mask) to switch at once)."""
    self._engine.set_env_variant(ids)

  def debug_observations(self, layer: bool = True, zap_matrix: bool = True):
    """The reference's debug observations of the current timestep as int32 tensors: 'POSITION' [B, P, 2],
    'ORIENTATION' [B, P] (specs.py:39-44), 'LAYER' [B, P, view_h, view_w, layers], 'ZAP_MATRIX' [B, P, P]."""
    return self._engine.debug_observations(layer=layer, zap_matrix=zap_matrix)

  def events(self):
    """(event_count int32 [B], events int32 [B, max_events, 3]) of the last step; rows are (type, a, b), unordered."""
    return self._engine.event_count, self._engine.events

  def save_state(self) -> bytes:
    """Snapshot of every env instance (no reference counterpart; SURVEY.md section 8f N4)."""
    return self._engine.save_state()

  def load_state(self, snapshot: bytes) -> BatchedTimeStep:
    """Restores a snapshot taken from an identically built BatchedSubstrate; returns the timestep it held."""
    self._engine.load_state(snapshot)
    return self._timestep()

  def state_bank(self, capacity: int):
    """A zeroed CUDA uint8 bank [capacity, record_bytes] for `store` / `restore`. A record restores into any
    BatchedSubstrate built from the same substrate (or the same variants, in the same order), whatever its num_envs,
    seed or device (copy the bank there)."""
    import torch  # pylint: disable=g-import-not-at-top
    if capacity < 1:
      raise ValueError(f'a state bank needs capacity >= 1, got {capacity}')
    e = self._engine
    return torch.zeros((int(capacity), e.state_record_bytes), dtype=torch.uint8, device=torch.device('cuda', e.device))

  def store(self, bank, envs, slots) -> None:
    """Stores env envs[i] into bank row slots[i] for every i (asynchronous, on the current stream). The record holds
    the env's state, its current timestep and its random stream, not its images."""
    e = self._engine
    idx = bank_index(slots, envs, int(bank.shape[0]), self.num_envs, 'slots', 'envs', device=bank.device)
    e.store_states(bank, idx)

  def restore(self, bank, envs, slots, rekey: bool = False) -> BatchedTimeStep:
    """Restores bank row slots[i] into env envs[i] for every i and re-renders; returns the timestep, in which each
    restored env shows the stored env's timestep and images at store time. The other envs are untouched. A restored env
    continues exactly as the stored env would have (given the same actions), from an auto-reset if its stored step was
    LAST, and under the stored env's variant; rekey=True gives it its own random stream instead."""
    e = self._engine
    idx = bank_index(envs, slots, self.num_envs, int(bank.shape[0]), 'envs', 'slots', device=bank.device)
    check_bank_tags(bank, slots, e.state_tag)
    e.restore_states(bank, idx, rekey=rekey)
    return self._timestep()

  def action_spec(self):
    return tuple(specs_lib.action(self.num_actions) for _ in range(self.num_players))

  def close(self):
    self._engine.close()

  def __enter__(self):
    return self

  def __exit__(self, *unused):
    self.close()


class Trajectory:
  """T timesteps of a BatchedSubstrate's outputs in caller-owned CUDA tensors (BatchedSubstrate.trajectory).

  Fields mirror BatchedTimeStep with a time axis: step_type int64, reward float64 [.., P], discount float64 and
  observation {name: tensor}, each [T, B, ...] when time_major else [B, T, ...]."""

  def __init__(self, T: int, num_envs: int, num_players: int, rgb_shape, world_rgb_shape, scalar_names: Sequence[str],
               time_major: bool, device):
    """rgb_shape: one env's [P, h, w, 3]; world_rgb_shape: one env's [H, W, 3], or None without WORLD.RGB."""
    import torch  # pylint: disable=g-import-not-at-top
    if T < 1:
      raise ValueError(f'a trajectory needs T >= 1 slots, got {T}')
    self.T, self.time_major = T, time_major
    B, P = num_envs, num_players

    def new(shape, dtype):
      return torch.zeros(((T, B) if time_major else (B, T)) + tuple(shape), dtype=dtype, device=device)

    self.step_type = new((), torch.int64)
    self.reward = new((P,), torch.float64)
    self.discount = new((), torch.float64)
    self.observation = {'RGB': new(tuple(rgb_shape), torch.uint8)}
    if scalar_names:  # one tensor, so that slot t of every scalar observation is one [n, B, P] view for the engine
      scalars = torch.zeros((len(scalar_names),) + tuple(self.reward.shape), dtype=torch.float64, device=device)
      for k, name in enumerate(scalar_names):
        self.observation[name] = scalars[k]
    if world_rgb_shape is not None:
      self.observation['WORLD.RGB'] = new(tuple(world_rgb_shape), torch.uint8)
    self.observation[_COLLECTIVE_REWARD_OBS] = new((), torch.float64)

  def at(self, t: int) -> BatchedTimeStep:
    """Slot t as a BatchedTimeStep of views ([B, ...] each)."""
    if not -self.T <= t < self.T:
      raise IndexError(f'slot {t} of a trajectory of {self.T}')
    pick = (lambda x: x[t]) if self.time_major else (lambda x: x[:, t])
    return BatchedTimeStep(step_type=pick(self.step_type), reward=pick(self.reward), discount=pick(self.discount),
                           observation={k: pick(v) for k, v in self.observation.items()})


class PlayerRoutes:
  """Where each player's outputs go (BatchedSubstrate.player_routes): an immutable assignment of player slots to rows.

  groups[b, p] is the group of player p of env b (e.g. the policy that plays that slot), -1 for a player whose
  observations nobody reads. Rows are laid out group-major, then env, then player, so each group's rows are one
  contiguous block, `rows(g)`. The assignment is validated once, here, on the host; the device tensors are then used as
  they are by every step.
    row_of_player  int32 CUDA [B, P]: the row of each player, -1 if unrouted (what the engine reads);
    env_of_row, player_of_row  int64 CUDA [n_rows]: the env and player of each row.
  WORLD.RGB can be routed per env along with them: `outputs(world_envs=envs)` draws it only for envs, into rows of its
  own (see PlayerOutputs).
  Actions go the same way: `actions(T)` gives rows a step reads its actions from (step(player_actions=)), laid out
  like the outputs' rows, so nothing is scattered back into [B, P].
  Do not write to these tensors: they are shared by every PlayerOutputs and PlayerActions made from this object."""

  __slots__ = ('num_envs', 'num_players', 'num_groups', 'n_rows', 'device', 'row_of_player', 'env_of_row', 'player_of_row',
               '_starts', '_rgb_shape', '_scalar_names', '_world_shape')

  def __init__(self, groups, num_envs: int, num_players: int, rgb_shape, scalar_names: Sequence[str], device,
               world_rgb_shape=None):
    """rgb_shape: one player's [h, w, 3]; device: where the tensors live (a CUDA device for the engine);
    world_rgb_shape: one env's WORLD.RGB [H, W, 3], or None when the batch renders none."""
    import torch  # pylint: disable=g-import-not-at-top
    g = groups.detach().cpu().numpy() if isinstance(groups, torch.Tensor) else np.asarray(groups)
    if g.shape != (num_envs, num_players):
      raise ValueError(f'groups must have shape [{num_envs}, {num_players}], got {list(g.shape)}')
    if g.dtype == np.bool_ or not np.issubdtype(g.dtype, np.integer):
      raise ValueError(f'groups must hold integer group ids, got dtype {g.dtype}')
    g = g.astype(np.int64)
    if (g < -1).any():
      raise ValueError('group ids must be >= 0, or -1 for a player that is not delivered')
    routed = np.flatnonzero(g.reshape(-1) >= 0)
    if routed.size == 0:
      raise ValueError('groups routes no player (every id is -1)')
    if routed.size >= 2**31:
      raise ValueError('more than 2^31 - 1 rows')
    flat = routed[np.argsort(g.reshape(-1)[routed], kind='stable')]  # group-major; env, then player within a group
    rows = np.full(num_envs * num_players, -1, np.int32)
    rows[flat] = np.arange(flat.size, dtype=np.int32)
    n_groups = int(g.max()) + 1
    counts = np.bincount(g.reshape(-1)[routed], minlength=n_groups)
    dev = torch.device(device)
    set_ = lambda k, v: object.__setattr__(self, k, v)
    set_('num_envs', int(num_envs)); set_('num_players', int(num_players)); set_('num_groups', n_groups)
    set_('n_rows', int(flat.size)); set_('device', dev)
    set_('_starts', tuple(int(x) for x in np.concatenate([[0], np.cumsum(counts)])))
    set_('_rgb_shape', tuple(int(x) for x in rgb_shape)); set_('_scalar_names', tuple(scalar_names))
    set_('_world_shape', None if world_rgb_shape is None else tuple(int(x) for x in world_rgb_shape))
    set_('row_of_player', torch.from_numpy(rows.reshape(num_envs, num_players)).to(dev))
    set_('env_of_row', torch.from_numpy(flat // num_players).to(dev))
    set_('player_of_row', torch.from_numpy(flat % num_players).to(dev))

  def __setattr__(self, name, value):
    raise AttributeError('PlayerRoutes is immutable; build a new one with player_routes(groups)')

  def rows(self, g: int) -> slice:
    """The rows of group g (empty for a group id nobody has)."""
    if not 0 <= g < self.num_groups:
      raise IndexError(f'group {g} outside 0..{self.num_groups - 1}')
    return slice(self._starts[g], self._starts[g + 1])

  def outputs(self, T: Optional[int] = None, world_envs=None) -> 'PlayerOutputs':
    """Zeroed CUDA tensors for the routed outputs: 'RGB' uint8 [n_rows, h, w, 3], 'REWARD' float64 [n_rows] and each
    scalar observation float64 [n_rows] (views of one tensor); with T, each gets a leading time axis [T, n_rows, ...]
    and `at(t)` is slot t. world_envs: distinct env indices (a sequence or 1-D integer tensor) whose WORLD.RGB is
    rendered, into 'WORLD.RGB' uint8 [n, H, W, 3] ([T, n, H, W, 3] with T), row k holding env world_envs[k]; no other
    env's WORLD.RGB is rendered."""
    return PlayerOutputs(self, T, world_envs=world_envs)

  def group_outputs(self, slots: Mapping[int, Optional[int]], time_major: bool = True, world_envs=None) -> 'GroupOutputs':
    """Zeroed CUDA tensors of their own for each group listed in slots (group -> T_g, or None for no time axis); see
    GroupOutputs. A group not listed is not delivered."""
    return GroupOutputs(self, slots, time_major, world_envs=world_envs)

  def actions(self, T: Optional[int] = None) -> 'PlayerActions':
    """A zeroed int32 CUDA tensor of actions, one per row: [n_rows], or [T, n_rows] with T, whose `at(t)` is slot t."""
    return PlayerActions(self, T)


class DrawnRoutes:
  """Where each player's outputs go when the rows are drawn per env and episode (BatchedSubstrate.drawn_routes).

  choices[p] lists the groups player slot p may play in (up to 8, e.g. the bots that may fill a background slot; empty
  for a player nobody reads). At every episode start of every env, each slot draws one of its choices, uniformly with
  replacement and independently per slot and episode, on the device (the draw is addressed by the env's key and episode,
  like every other draw of the engine, so it does not depend on num_envs or env_index_base, and a restored clone plays
  its source's draw). It is not Python's `random` stream. Listing a group twice for one slot doubles its weight.

  Rows are laid out group-major: group g has capacity n_g, the number of slots that list g, and its block `rows(g)` is
  [B, n_g] in env, then slot order; `group(g)` names those n_g slots. Player p of env b sits in row
  start_g + b * n_g + rank_g(p) of the group it drew, rank_g(p) being p's position in group(g); the other rows of the
  block are inactive this episode: not rendered, their actions not read. Every step and reset writes
    row_of_player  int32 CUDA [B, P]: each player's row for the episode its env is in, -1 if it has no choices;
  `active(g)` derives which rows of group g are played from it. outputs(T) and actions(T) are as for PlayerRoutes; pass
  both to BatchedSubstrate.step (players=, player_actions=) and the outputs to reset (players=)."""

  __slots__ = ('num_envs', 'num_players', 'num_groups', 'n_rows', 'device', 'row_of_player', 'choices', 'draw',
               '_starts', '_members', '_rgb_shape', '_scalar_names', '_world_shape')

  def __init__(self, choices, num_envs: int, num_players: int, rgb_shape, scalar_names: Sequence[str], device,
               world_rgb_shape=None):
    """rgb_shape: one player's [h, w, 3]; device: where the tensors live (a CUDA device for the engine);
    world_rgb_shape: one env's WORLD.RGB [H, W, 3], or None when the batch renders none."""
    import torch  # pylint: disable=g-import-not-at-top
    from meltingpot_b200 import engine as engine_lib  # pylint: disable=g-import-not-at-top
    if isinstance(choices, (str, bytes)) or len(choices) != num_players:
      raise ValueError(f'choices must list the groups of each of the {num_players} player slots')
    norm = []
    for p, c in enumerate(choices):
      if isinstance(c, (str, bytes)) or not isinstance(c, Sequence) and not isinstance(c, np.ndarray):
        raise ValueError(f'choices[{p}] must be a sequence of group ids')
      c = tuple(c)
      if len(c) > engine_lib.MP_MAX_ROUTE_CHOICES:
        raise ValueError(f'choices[{p}] lists {len(c)} groups, at most {engine_lib.MP_MAX_ROUTE_CHOICES}')
      for g in c:
        if isinstance(g, (bool, np.bool_)) or not isinstance(g, (int, np.integer)) or g < 0:
          raise ValueError(f'choices[{p}]: group ids must be integers >= 0, got {g!r}')
      norm.append(tuple(int(g) for g in c))
    if not any(norm):
      raise ValueError('choices routes no player (every slot lists no group)')
    n_groups = max(max(c) for c in norm if c) + 1
    members = tuple(tuple(p for p, c in enumerate(norm) if g in c) for g in range(n_groups))
    starts = [0]
    for g in range(n_groups):
      starts.append(starts[-1] + num_envs * len(members[g]))
    if starts[-1] >= 2**31:
      raise ValueError('more than 2^31 - 1 rows')
    row_base = [[starts[g] + members[g].index(p) for g in c] for p, c in enumerate(norm)]
    rows_per_env = [[len(members[g]) for g in c] for c in norm]
    dev = torch.device(device)
    set_ = lambda k, v: object.__setattr__(self, k, v)
    set_('num_envs', int(num_envs)); set_('num_players', int(num_players)); set_('num_groups', n_groups)
    set_('n_rows', starts[-1]); set_('device', dev); set_('choices', tuple(norm))
    set_('_starts', tuple(starts)); set_('_members', members)
    set_('_rgb_shape', tuple(int(x) for x in rgb_shape)); set_('_scalar_names', tuple(scalar_names))
    set_('_world_shape', None if world_rgb_shape is None else tuple(int(x) for x in world_rgb_shape))
    set_('row_of_player', torch.full((num_envs, num_players), -1, dtype=torch.int32, device=dev))
    set_('draw', engine_lib.describe_draw(self.row_of_player, self.n_rows, row_base, rows_per_env))

  def __setattr__(self, name, value):
    raise AttributeError('DrawnRoutes is immutable; build a new one with drawn_routes(choices)')

  def _check_group(self, g: int) -> None:
    if not 0 <= g < self.num_groups:
      raise IndexError(f'group {g} outside 0..{self.num_groups - 1}')

  def rows(self, g: int) -> slice:
    """The rows of group g, [B, n_g] in env-major order (empty for a group id no slot lists)."""
    self._check_group(g)
    return slice(self._starts[g], self._starts[g + 1])

  def group(self, g: int) -> Tuple[int, ...]:
    """The player slots that list group g, in rank order: column k of rows(g) viewed as [B, n_g] belongs to slot
    group(g)[k] whenever that slot drew g."""
    self._check_group(g)
    return self._members[g]

  def active(self, g: int):
    """bool CUDA [B, n_g]: which rows of group g are played in the episode each env is in (from row_of_player, with
    torch ops on the current stream)."""
    import torch  # pylint: disable=g-import-not-at-top
    r = self.rows(g)
    n = r.stop - r.start
    flat = self.row_of_player.reshape(-1).to(torch.int64)
    inside = (flat >= r.start) & (flat < r.stop)
    act = torch.zeros(n + 1, dtype=torch.bool, device=self.device)  # the last entry takes every other player
    act.scatter_(0, torch.where(inside, flat - r.start, n), True)
    return act[:n].view(self.num_envs, len(self._members[g]))

  def outputs(self, T: Optional[int] = None, world_envs=None) -> 'PlayerOutputs':
    """As PlayerRoutes.outputs."""
    return PlayerOutputs(self, T, world_envs=world_envs)

  def group_outputs(self, slots: Mapping[int, Optional[int]], time_major: bool = True, world_envs=None) -> 'GroupOutputs':
    """As PlayerRoutes.group_outputs: group g's tensors hold its whole block rows(g), [B, n_g] in env-major order."""
    return GroupOutputs(self, slots, time_major, world_envs=world_envs)

  def actions(self, T: Optional[int] = None) -> 'PlayerActions':
    """As PlayerRoutes.actions."""
    return PlayerActions(self, T)


def world_row_map(world_envs, num_envs: int, device):
  """(world_envs int64 [n], world_row_of_env int32 [B]) on `device` for routed WORLD.RGB: row k holds env
  world_envs[k], an env not listed has row -1 and is not rendered. world_envs is a sequence or 1-D integer tensor of
  distinct env indices in [0, num_envs), validated here, on the host."""
  import torch  # pylint: disable=g-import-not-at-top
  dev = torch.device(device)
  if isinstance(world_envs, torch.Tensor):
    if world_envs.device.type != 'cpu' and world_envs.device != dev:
      raise ValueError(f'world_envs is on {world_envs.device}, the routes are on {dev}')
    if world_envs.dtype == torch.bool or world_envs.is_floating_point() or world_envs.is_complex():
      raise ValueError(f'world_envs must hold integer env indices, got dtype {world_envs.dtype}')
    e = world_envs.detach().cpu().numpy()
  else:
    e = np.asarray(world_envs)
  if e.ndim != 1:
    raise ValueError(f'world_envs must be one-dimensional, got shape {list(e.shape)}')
  if e.size == 0:
    raise ValueError('world_envs lists no env')
  if e.dtype == np.bool_ or not np.issubdtype(e.dtype, np.integer):
    raise ValueError(f'world_envs must hold integer env indices, got dtype {e.dtype}')
  e = e.astype(np.int64)
  if (e < 0).any() or (e >= num_envs).any():
    raise ValueError(f'world_envs must lie in [0, {num_envs}), got {e.min()}..{e.max()}')
  if np.unique(e).size != e.size:
    raise ValueError('world_envs lists an env twice')
  rows = np.full(num_envs, -1, np.int32)
  rows[e] = np.arange(e.size, dtype=np.int32)
  return torch.from_numpy(e).to(dev), torch.from_numpy(rows).to(dev)


def _routes_world(po) -> bool:
  """Whether a PlayerOutputs routes WORLD.RGB."""
  return getattr(po, 'world_row_of_env', None) is not None


class PlayerOutputs:
  """Caller-owned CUDA tensors for the routed outputs of PlayerRoutes (routes.outputs(T)); `po[name]` is one of them.
  Pass it (or, with T slots, `at(t)`) to BatchedSubstrate.step / reset as players=.
  Made with world_envs, it also holds 'WORLD.RGB' (row k: env world_envs[k]) and
    world_envs  int64 CUDA [n]: the env of each WORLD.RGB row;
    world_row_of_env  int32 CUDA [B]: the WORLD.RGB row of each env, -1 if it is not rendered (what the engine reads);
  both None otherwise."""

  def __init__(self, routes: PlayerRoutes, T: Optional[int] = None, tensors=None, scalar_block=None, world_envs=None,
               world=None):
    """tensors, scalar_block, world: a view (at / group) or rows made by the caller, world being the (world_envs,
    world_row_of_env) pair of world_row_map when tensors holds 'WORLD.RGB'."""
    import torch  # pylint: disable=g-import-not-at-top
    self.routes, self.T = routes, T
    if tensors is not None:  # a view (at / group), or rows made by the caller
      self.tensors, self.scalar_block = tensors, scalar_block
      self.world_envs, self.world_row_of_env = world if world is not None else (None, None)
      return
    if T is not None and T < 1:
      raise ValueError(f'outputs need T >= 1 slots, got {T}')
    lead = (routes.n_rows,) if T is None else (int(T), routes.n_rows)
    dev = routes.device
    self.tensors = {'RGB': torch.zeros(lead + routes._rgb_shape, dtype=torch.uint8, device=dev),  # pylint: disable=protected-access
                    'REWARD': torch.zeros(lead, dtype=torch.float64, device=dev)}
    names = routes._scalar_names  # pylint: disable=protected-access
    self.scalar_block = torch.zeros((len(names),) + lead, dtype=torch.float64, device=dev) if names else None
    for k, name in enumerate(names):  # one tensor, so that a slot's scalar observations are one [n, n_rows] view
      self.tensors[name] = self.scalar_block[k]
    self.world_envs = self.world_row_of_env = None
    if world_envs is not None:
      if routes._world_shape is None:  # pylint: disable=protected-access
        raise ValueError('world_envs: this batch renders no WORLD.RGB (it was built with world_rgb=False)')
      self.world_envs, self.world_row_of_env = world_row_map(world_envs, routes.num_envs, dev)
      n = int(self.world_envs.shape[0])
      self.tensors['WORLD.RGB'] = torch.zeros(((n,) if T is None else (int(T), n)) + routes._world_shape,  # pylint: disable=protected-access
                                              dtype=torch.uint8, device=dev)

  def __getitem__(self, name):
    return self.tensors[name]

  def keys(self):
    return self.tensors.keys()

  def at(self, t: int) -> 'PlayerOutputs':
    """Slot t of outputs made with T slots, as views."""
    if self.T is None:
      raise ValueError('at() needs outputs made with T slots')
    if not -self.T <= t < self.T:
      raise IndexError(f'slot {t} of {self.T}')
    sb = None if self.scalar_block is None else self.scalar_block[:, t]
    tensors = {k: v[t] for k, v in self.tensors.items()}
    for k, name in enumerate(self.routes._scalar_names):  # pylint: disable=protected-access
      tensors[name] = sb[k]
    return PlayerOutputs(self.routes, None, tensors, sb, world=(self.world_envs, self.world_row_of_env))

  def group(self, g: int) -> Dict[str, Any]:
    """{name: view of group g's rows} ([rows, ...], or [T, rows, ...] with T slots); WORLD.RGB, which is per env, is
    not among them."""
    r = self.routes.rows(g)
    per_player = {k: v for k, v in self.tensors.items() if k != 'WORLD.RGB'}
    if self.T is None:
      return {k: v[r] for k, v in per_player.items()}
    return {k: v[:, r] for k, v in per_player.items()}


def _group_tensors(routes, g: int, lead: Tuple[int, ...], alloc):
  """({name: tensor}, scalar block) of group g's routed outputs: 'RGB', 'REWARD' and each scalar observation, with
  `lead` in front of each ((n_g,), (T, n_g) or (n_g, T)) and the scalar observations views of one block
  [n_scalar, *lead]. alloc: torch.zeros or torch.empty."""
  import torch  # pylint: disable=g-import-not-at-top
  dev = routes.device
  tensors = {'RGB': alloc(lead + routes._rgb_shape, dtype=torch.uint8, device=dev),  # pylint: disable=protected-access
             'REWARD': alloc(lead, dtype=torch.float64, device=dev)}
  names = routes._scalar_names  # pylint: disable=protected-access
  block = alloc((len(names),) + lead, dtype=torch.float64, device=dev) if names else None
  for k, name in enumerate(names):
    tensors[name] = block[k]
  return tensors, block


class GroupOutputs:
  """Caller-owned CUDA tensors of routed outputs, one set per group (routes.group_outputs(slots)), so that each group's
  rows land in a buffer of its own, e.g. one trajectory buffer per learning group of a population, with its own T.

  Group g of `slots` gets 'RGB' uint8, 'REWARD' float64 and each scalar observation float64 (views of one block),
  each [T_g, n_g, ...] (time_major) or [n_g, T_g, ...], or [n_g, ...] with T_g None; n_g is the size of rows(g), row k
  of the group being row rows(g).start + k of the routes. Groups not listed are not delivered: their players are
  neither rendered nor given scalars. Pass it (or `at(t)`) to BatchedSubstrate.step / reset as players=: the step
  delivers each listed group into its tensors through one row segment per group, in the same kernels as outputs().
  Made with world_envs, it also holds WORLD.RGB as outputs() does, with a slot axis when some group has slots (T the
  largest T_g, laid out like the groups'): `world_rgb`, `world_envs`, `world_row_of_env`; all None otherwise."""

  def __init__(self, routes, slots: Mapping[int, Optional[int]], time_major: bool = True, world_envs=None, groups=None,
               world=None):
    """groups, world: a view (at), or tensors made by the caller: groups maps g to ({name: tensor}, scalar block) and
    world is (world_envs, world_row_of_env, world_rgb) or None."""
    import torch  # pylint: disable=g-import-not-at-top
    self.routes, self.time_major = routes, bool(time_major)
    if not isinstance(slots, Mapping) or not slots:
      raise ValueError('slots must map at least one group id to its number of slots (or None)')
    norm = {}
    for g, T in slots.items():
      if isinstance(g, (bool, np.bool_)) or not isinstance(g, (int, np.integer)) or not 0 <= g < routes.num_groups:
        raise ValueError(f'slots: group {g!r} outside 0..{routes.num_groups - 1}')
      if T is not None and (isinstance(T, (bool, np.bool_)) or not isinstance(T, (int, np.integer)) or T < 1):
        raise ValueError(f'slots: group {g} needs T >= 1 slots or None, got {T!r}')
      norm[int(g)] = None if T is None else int(T)
    self.slots = dict(sorted(norm.items()))
    if all(routes.rows(g).stop == routes.rows(g).start for g in self.slots):
      raise ValueError('slots: every group listed has no rows')
    if groups is not None:
      self.groups = groups
      self.world_envs, self.world_row_of_env, self.world_rgb = world if world is not None else (None, None, None)
      return
    self.groups = {}
    for g, T in self.slots.items():
      n = routes.rows(g).stop - routes.rows(g).start
      lead = (n,) if T is None else ((T, n) if self.time_major else (n, T))
      self.groups[g] = _group_tensors(routes, g, lead, torch.zeros)
    self.world_envs = self.world_row_of_env = self.world_rgb = None
    if world_envs is not None:
      if routes._world_shape is None:  # pylint: disable=protected-access
        raise ValueError('world_envs: this batch renders no WORLD.RGB (it was built with world_rgb=False)')
      self.world_envs, self.world_row_of_env = world_row_map(world_envs, routes.num_envs, routes.device)
      n = int(self.world_envs.shape[0])
      T = max((t for t in self.slots.values() if t is not None), default=None)
      lead = (n,) if T is None else ((T, n) if self.time_major else (n, T))
      self.world_rgb = torch.zeros(lead + routes._world_shape, dtype=torch.uint8, device=routes.device)  # pylint: disable=protected-access

  def group(self, g: int) -> Dict[str, Any]:
    """{name: tensor} of group g."""
    if g not in self.groups:
      raise KeyError(f'group {g} is not delivered (slots lists {sorted(self.groups)})')
    return dict(self.groups[g][0])

  def at(self, t: int) -> 'GroupOutputs':
    """Slot t of every group that has slots (and of WORLD.RGB), as views; groups without slots keep their tensors."""
    timed = [T for T in self.slots.values() if T is not None]
    if not timed:
      raise ValueError('at() needs a group with slots')
    if not all(-T <= t < T for T in timed):
      raise IndexError(f'slot {t} of groups with {min(timed)} slots or more')
    pick = (lambda x: x[t]) if self.time_major else (lambda x: x[:, t])
    groups = {}
    for g, (tensors, block) in self.groups.items():
      if self.slots[g] is None:
        groups[g] = (tensors, block)
        continue
      sb = None if block is None else (block[:, t] if self.time_major else block[:, :, t])
      view = {k: pick(v) for k, v in tensors.items()}
      for k, name in enumerate(self.routes._scalar_names):  # pylint: disable=protected-access
        view[name] = sb[k]
      groups[g] = (view, sb)
    world = None
    if self.world_rgb is not None:
      world = (self.world_envs, self.world_row_of_env, pick(self.world_rgb))
    return GroupOutputs(self.routes, {g: None for g in self.slots}, self.time_major, groups=groups, world=world)

  def segments(self):
    """The engine's row segments of a view without slots: [(row_begin, row_end, {target: tensor})], one per group
    that has rows."""
    out = []
    for g, (tensors, block) in self.groups.items():
      r = self.routes.rows(g)
      if r.stop > r.start:
        out.append((r.start, r.stop, {'rgb': tensors['RGB'], 'reward': tensors['REWARD'], 'scalar_obs': block}))
    return out


class PlayerActions:
  """Caller-owned CUDA rows of actions for PlayerRoutes (routes.actions(T)): `tensor` is int32 [n_rows], or
  [T, n_rows] with T slots. Write row r's action id into tensor[r] and pass this (or, with T slots, `at(t)`) to
  BatchedSubstrate.step as player_actions=; `group(g)` is the view of group g's rows."""

  def __init__(self, routes: PlayerRoutes, T: Optional[int] = None, tensor=None):
    import torch  # pylint: disable=g-import-not-at-top
    self.routes, self.T = routes, T
    if tensor is not None:  # a view (at)
      self.tensor = tensor
      return
    if T is not None and T < 1:
      raise ValueError(f'actions need T >= 1 slots, got {T}')
    lead = (routes.n_rows,) if T is None else (int(T), routes.n_rows)
    self.tensor = torch.zeros(lead, dtype=torch.int32, device=routes.device)

  def at(self, t: int) -> 'PlayerActions':
    """Slot t of actions made with T slots, as a view."""
    if self.T is None:
      raise ValueError('at() needs actions made with T slots')
    if not -self.T <= t < self.T:
      raise IndexError(f'slot {t} of {self.T}')
    return PlayerActions(self.routes, None, self.tensor[t])

  def group(self, g: int):
    """View of group g's rows ([rows], or [T, rows] with T slots)."""
    r = self.routes.rows(g)
    return self.tensor[r] if self.T is None else self.tensor[:, r]


# ---------------------------------------------------------------------------------------------
# dm_env substrate (one env, numpy)
# ---------------------------------------------------------------------------------------------
class Substrate(dm_env.Environment):
  """dm_env view of a single env instance (the reference's `Substrate`)."""

  def __init__(self, blob: bytes, config: config_dict.ConfigDict, device: int = 0,
               env_seed: Optional[int] = None):
    import torch  # pylint: disable=g-import-not-at-top
    self._torch = torch
    self._config = config
    self._batched = BatchedSubstrate(blob, 1, device=device, seed=env_seed)
    self._num_players = self._batched.num_players
    self._individual = list(config.individual_observation_names)
    self._global = list(config.global_observation_names)
    self._action_subject, self._timestep_subject, self._events_subject = Subject(), Subject(), Subject()
    self._raw = Lab2dObservables(action=Subject(), timestep=Subject(), events=Subject())
    self._observables = SubstrateObservables(dmlab2d=self._raw, action=self._action_subject, timestep=self._timestep_subject,
                                             events=self._events_subject)
    self._closed = False
    self._last_observation = None
    self._last_events = np.zeros((0, 3), np.int32)
    self._host = None

  # -- helpers --------------------------------------------------------------------------------
  def _host_buffers(self):
    """Pinned host buffers of the B = 1 view: one host-buffer C-ABI call per step fills them (three device->host
    copies: images, WORLD.RGB, and the packed scalar block; plus the events), then the stream is synchronised once."""
    if self._host is None:
      eng = self._batched.engine
      self._host = eng.make_host_outputs(rgb=True, world_rgb=self._batched._world_rgb, events=True)  # pylint: disable=protected-access
      self._host_actions = eng.make_host_actions()
      self._scalar_index = {name: k for k, name in enumerate(self._batched._scalar_names)}  # pylint: disable=protected-access
    return self._host

  def _to_timestep(self) -> dm_env.TimeStep:
    host = self._host
    step_type = dm_env.StepType(int(host['step_type'][0]))
    rewards = [np.float64(r) for r in host['reward'][0].numpy()]
    # fresh arrays every step, as the reference returns (the pinned buffers are overwritten by the next call)
    rgb = host['rgb'][0].numpy().copy()
    shared = {}
    for name in self._global:
      shared[name] = host['world_rgb'][0].numpy().copy()
    collective = np.sum(rewards)
    observations = []
    for i in range(self._num_players):
      obs = {_COLLECTIVE_REWARD_OBS: collective}
      for name in self._individual:
        obs[name] = rgb[i] if name == 'RGB' else np.float64(host['scalar_obs'][self._scalar_index[name], 0, i])
      for name in self._global:
        obs[name] = shared[name]  # the same array object in every player's dict
      observations.append(obs)
    self._last_observation = observations
    n = int(host['event_count'][0])
    if n > host['events'].shape[1]:
      raise RuntimeError(f'{n} events in one step exceed the engine\'s max_events {host["events"].shape[1]}')
    self._last_events = host['events'][0, :n].numpy().copy()
    return dm_env.TimeStep(step_type=step_type, reward=rewards, discount=float(host['discount'][0]),
                           observation=observations)

  # -- dm_env API -------------------------------------------------------------------------------
  def _emit_raw(self, timestep, action=None) -> None:
    """observables().dmlab2d: the dmlab2d-level stream the reference's innermost ObservablesWrapper emits
    (observables_wrapper.py:43-58), built only while somebody is subscribed."""
    raw = self._raw
    if action is not None and raw.action._observers:  # pylint: disable=protected-access
      raw.action.on_next(flat_action(action, self._config.action_set))
    if raw.timestep._observers:  # pylint: disable=protected-access
      raw.timestep.on_next(flat_timestep(timestep, self._individual, self._global))
    if raw.events._observers:  # pylint: disable=protected-access
      for event in self.events():
        raw.events.on_next(event)

  def reset(self) -> dm_env.TimeStep:
    self._batched.engine.reset_host(self._host_buffers())
    timestep = self._to_timestep()
    self._emit_raw(timestep)
    self._timestep_subject.on_next(timestep)
    for event in self.events():
      self._events_subject.on_next(event)
    return timestep

  def step(self, action: Sequence[int]) -> dm_env.TimeStep:
    if len(action) != self._num_players:
      raise ValueError(f'expected {self._num_players} actions, got {len(action)}')
    specs = self.action_spec()
    for a, spec in zip(action, specs):
      if not 0 <= int(a) < spec.num_values:
        raise ValueError(f'action {a} out of range [0, {spec.num_values})')
    self._action_subject.on_next(action)
    host = self._host_buffers()
    self._host_actions[0] = self._torch.as_tensor(np.asarray(action, np.int32))
    self._batched.engine.step_host(self._host_actions, host)
    timestep = self._to_timestep()
    self._emit_raw(timestep, action)
    self._timestep_subject.on_next(timestep)
    for event in self.events():
      self._events_subject.on_next(event)
    return timestep

  def observation(self) -> Sequence[Mapping[str, np.ndarray]]:
    return self._last_observation

  def events(self) -> Sequence[tuple]:
    """Events of the last reset/step in dmlab2d's shape: (name, [b'dict', b'key', array(value), ...]).

    Covers the events:add calls on the hot path (include/mp_engine.h, mp_buffers.events). dmlab2d's own
    order within a step is engine-defined and unpinned; here they are sorted by (type, arguments).
    """
    from meltingpot_b200 import engine as engine_lib  # pylint: disable=g-import-not-at-top
    rows = sorted(tuple(int(v) for v in row) for row in self._last_events)
    out = []
    for kind, a, b in rows:
      payload = [b'dict']
      for key, value in zip(engine_lib.EVENT_FIELDS[kind], (a, b)):
        payload += [key.encode(), np.array(float(value))]
      out.append((engine_lib.EVENT_NAMES[kind], payload))
    return out

  def action_spec(self) -> Sequence['dm_env.specs.DiscreteArray']:
    return tuple(self._config.action_spec for _ in range(self._num_players))

  def observation_spec(self) -> Sequence[Mapping[str, 'dm_env.specs.Array']]:
    spec = dict(self._config.timestep_spec.observation)
    spec[_COLLECTIVE_REWARD_OBS] = dm_env.specs.Array(shape=(), dtype=np.float64, name=_COLLECTIVE_REWARD_OBS)
    return tuple(dict(spec) for _ in range(self._num_players))

  def reward_spec(self) -> Sequence['dm_env.specs.Array']:
    return tuple(self._config.timestep_spec.reward for _ in range(self._num_players))

  def discount_spec(self):
    return self._config.timestep_spec.discount

  def observables(self) -> SubstrateObservables:
    return self._observables

  # dmlab2d's key-value debugging interface (wrappers/base.py:66-80): the engine exposes no properties.
  def list_property(self, key: str = ''):
    del key
    return []

  def read_property(self, key: str):
    raise KeyError(key)

  def write_property(self, key: str, value: str):
    del value
    raise KeyError(key)

  def close(self) -> None:
    if not self._closed:
      self._closed = True
      self._batched.close()
      for subject in (self._raw.action, self._raw.timestep, self._raw.events):
        subject.on_completed()
      self._action_subject.on_completed()
      self._timestep_subject.on_completed()
      self._events_subject.on_completed()


# ---------------------------------------------------------------------------------------------
# Factories
# ---------------------------------------------------------------------------------------------
def _validate_roles(config, roles: Sequence[str]) -> None:
  invalid = set(roles) - set(config.valid_roles)
  if invalid:  # configs/substrates/__init__.py:42-45
    raise ValueError(f'Invalid roles: {invalid!r}. Must be one of {config.valid_roles!r}')


class SubstrateFactory:
  """Mirrors `meltingpot/utils/substrates/substrate_factory.py:24-95`."""

  def __init__(self, name: str, config: config_dict.ConfigDict, device: int = 0):
    self._name = name
    self._config = config
    self._device = device

  def valid_roles(self) -> Collection[str]:
    return frozenset(self._config.valid_roles)

  def default_player_roles(self) -> Sequence[str]:
    return tuple(self._config.default_player_roles)

  def timestep_spec(self):
    return self._config.timestep_spec

  def action_spec(self):
    return self._config.action_spec

  def build(self, roles: Sequence[str], env_seed: Optional[int] = None) -> Substrate:
    _validate_roles(self._config, roles)
    blob = substrate_blobs.load_blob(self._name, tuple(roles))
    return Substrate(blob, self._config, device=self._device, env_seed=env_seed)

  def build_batched(self, roles: Sequence[str], num_envs: int, seed: Optional[int] = None,
                    env_index_base: int = 0, world_rgb: bool = True, prefab_overrides=None,
                    env_variant=None, build_seeds=None, maps=None) -> BatchedSubstrate:
    _validate_roles(self._config, roles)
    if maps is not None:  # one map set: the substrate under each ASCII map
      if prefab_overrides is not None or build_seeds is not None:
        raise ValueError('maps take neither prefab_overrides nor build_seeds')
      maps = substrate_blobs.checked_maps(self._name, maps)
      if env_variant is None:
        env_variant = draw_of_env(env_index_base, num_envs, len(maps))
      else:
        env_variant = _checked_env_variant(env_variant, num_envs, len(maps), 'maps')
      blob = substrate_blobs.compile_maps(self._name, tuple(roles), maps)
    elif build_seeds is not None:  # one draw of the config builder per seed
      if prefab_overrides is not None:
        raise ValueError('pass build_seeds or prefab_overrides, not both')
      build_seeds = [int(s) for s in build_seeds]
      if not build_seeds:
        raise ValueError('build_seeds is empty')
      blob = substrate_blobs.compile_draws(self._name, tuple(roles), build_seeds)
      if env_variant is None:
        env_variant = draw_of_env(env_index_base, num_envs, len(build_seeds))
    elif prefab_overrides is None:
      if env_variant is not None:
        raise ValueError('env_variant needs a sequence of prefab_overrides')
      blob = substrate_blobs.load_blob(self._name, tuple(roles))
    elif isinstance(prefab_overrides, Mapping):  # one parameter set for every env
      if env_variant is not None:
        raise ValueError('env_variant needs a sequence of prefab_overrides')
      blob = substrate_blobs.compile_with_overrides(self._name, tuple(roles), prefab_overrides)
    else:  # one variant per entry, compiled as one set on one sprite table
      prefab_overrides = list(prefab_overrides)
      if not prefab_overrides:
        raise ValueError('the sequence of prefab_overrides is empty')
      for i, o in enumerate(prefab_overrides):
        if o is not None and not isinstance(o, Mapping):
          raise ValueError(f'prefab_overrides[{i}] is a {type(o).__name__}, not a mapping')
      if env_variant is not None:
        env_variant = _checked_env_variant(env_variant, num_envs, len(prefab_overrides), 'prefab_overrides')
      blob = substrate_blobs.compile_with_overrides(self._name, tuple(roles), prefab_overrides)
    return BatchedSubstrate(blob, num_envs, device=self._device, seed=seed,
                            env_index_base=env_index_base, world_rgb=world_rgb, env_variant=env_variant)


def get_factory(name: str, device: int = 0) -> SubstrateFactory:
  return SubstrateFactory(name, get_config(name), device=device)


def get_factory_from_config(config: config_dict.ConfigDict, device: int = 0) -> SubstrateFactory:
  return SubstrateFactory(config.substrate_name, config, device=device)


def build(name: str, *, roles: Sequence[str], env_seed: Optional[int] = None, device: int = 0) -> Substrate:
  """Builds an instance of the specified substrate (substrate.py:57-70)."""
  return get_factory(name, device).build(roles, env_seed=env_seed)


def build_from_config(config: config_dict.ConfigDict, *, roles: Sequence[str],
                      env_seed: Optional[int] = None, device: int = 0) -> Substrate:
  return get_factory_from_config(config, device).build(roles, env_seed=env_seed)


def draw_of_env(env_index_base: int, num_envs: int, num_draws: int) -> np.ndarray:
  """The default draw of each env of a build_seeds batch: global env g plays draw g % num_draws."""
  return (np.arange(env_index_base, env_index_base + num_envs) % num_draws).astype(np.int64)


def build_batched(name, *, roles: Sequence[str], num_envs: int, device: int = 0,
                  seed: Optional[int] = None, env_index_base: int = 0,
                  world_rgb: bool = True, prefab_overrides=None, env_variant=None, build_seeds=None,
                  maps=None) -> BatchedSubstrate:
  """Builds `num_envs` instances on one GPU; see `BatchedSubstrate`.

  `name` is a substrate name, or a sequence of substrate names whose maps the engine runs side by side, e.g.
  ('commons_harvest__open', 'commons_harvest__closed', 'commons_harvest__partnership'): each name's blob is
  load_blob(name, roles), and env b plays names[env_variant[b]], by default (env_index_base + b) % len(name). The names
  are variants, so active_variant / pending_variant / set_env_variant index into the sequence and set_env_variant moves
  an env to another map at its next episode. A name may repeat, which weights the default assignment. The names must
  share the action set, observation names and timestep spec, and their blobs must form one map set (mp_create_variants
  refuses another family, player count or map size); not combined with prefab_overrides or build_seeds.

  `prefab_overrides` (the reference builder's, builder.py:70-87) is one mapping for every env, or a sequence of
  mappings: a heterogeneous batch whose env b runs variant env_variant[b] (default 0). The sequence is compiled as one
  set on one sprite table, so its entries may also change how pieces look (an `Appearance` palette or sprite shape),
  e.g. [{}, {'potential_apple': {'Appearance': {'palettes': [recoloured]}}}]. Compiling overrides needs a reference
  checkout.

  `build_seeds` (coins): one draw of the substrate's config builder per seed, as separate reference builds would
  make (coins draws its map size and its two coin colours on every build), compiled as one draw set. Env b plays
  draw env_variant[b], by default (env_index_base + b) % len(build_seeds); a draw is a variant, so set_env_variant
  moves an env to another draw at its next episode. Needs a reference checkout; not combined with prefab_overrides.

  `maps` (territory__rooms, __open, __inside_out and coop_mining): a sequence of ASCII maps, each replacing the
  substrate's own (territory's `config.layout.ascii_map`, coop_mining's level map), compiled as one map set on one
  sprite table. Every map keeps the substrate's rows and row width; its walls, resources or ores and spawn points may
  move, and their counts may differ. Env b plays maps[env_variant[b]], by default (env_index_base + b) % len(maps),
  and set_env_variant moves an env to another map at its next episode. Needs a reference checkout; not combined with
  prefab_overrides or build_seeds, nor with a sequence of names."""
  if not isinstance(name, str):
    if maps is not None:
      raise ValueError('maps take one substrate name, not a sequence of names')
    return _build_map_set(tuple(name), roles=roles, num_envs=num_envs, device=device, seed=seed,
                          env_index_base=env_index_base, world_rgb=world_rgb, prefab_overrides=prefab_overrides,
                          env_variant=env_variant, build_seeds=build_seeds)
  return get_factory(name, device).build_batched(roles, num_envs, seed=seed, env_index_base=env_index_base,
                                                 world_rgb=world_rgb, prefab_overrides=prefab_overrides,
                                                 env_variant=env_variant, build_seeds=build_seeds, maps=maps)


def _checked_env_variant(env_variant, num_envs: int, num_variants: int, what: str) -> np.ndarray:
  """env_variant as an int64 array of num_envs entries, each indexing the num_variants `what`."""
  env_variant = np.asarray(env_variant, np.int64).reshape(-1)
  if env_variant.shape != (num_envs,):
    raise ValueError(f'env_variant has {env_variant.size} entries for {num_envs} envs')
  if env_variant.size and (env_variant.min() < 0 or env_variant.max() >= num_variants):
    raise ValueError(f'env_variant must index the {num_variants} {what} (0..{num_variants - 1})')
  return env_variant


_SHARED_CONFIG_FIELDS = ('action_set', 'individual_observation_names', 'global_observation_names', 'timestep_spec')


def _build_map_set(names: Sequence[str], *, roles, num_envs, device, seed, env_index_base, world_rgb, prefab_overrides,
                   env_variant, build_seeds) -> BatchedSubstrate:
  """build_batched over a sequence of substrate names: every argument is checked here, before an engine exists."""
  if not names:
    raise ValueError('the sequence of substrate names is empty')
  if prefab_overrides is not None or build_seeds is not None:
    raise ValueError('a sequence of substrate names takes neither prefab_overrides nor build_seeds')
  configs = [get_config(n) for n in names]
  for config in configs:
    _validate_roles(config, roles)
  for n, config in zip(names[1:], configs[1:]):
    for field in _SHARED_CONFIG_FIELDS:
      if config[field] != configs[0][field]:
        raise ValueError(f'{n!r} differs from {names[0]!r} in its {field}')
  if env_variant is None:
    env_variant = draw_of_env(env_index_base, num_envs, len(names))
  else:
    env_variant = _checked_env_variant(env_variant, num_envs, len(names), 'names')
  blobs = [substrate_blobs.load_blob(n, tuple(roles)) for n in names]
  return BatchedSubstrate(blobs, num_envs, device=device, seed=seed, env_index_base=env_index_base,
                          world_rgb=world_rgb, env_variant=env_variant)
