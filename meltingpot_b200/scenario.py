"""Scenario layer: a substrate in which some player slots are filled by background players.

SURVEY.md section 8f, row N2. Mirrors `meltingpot/utils/scenarios/scenario.py`:
  * `Scenario` (`scenario.py:101-263`) — the dm_env wrapper, same constructor arguments, same
    focal / background partition (`_partition` :55-68, `_merge` :71-81), same restriction of
    focal observations to `permitted_observations` (`_restrict_observation(s)` :33-52), same
    error texts. The background population is any object with the reference `Population`
    surface used here: `await_action()`, `send_timestep(timestep)`, `reset()`, `close()`
    (`utils/policies/...` SavedModel bots are out of scope and stay external).
  * `BatchedScenario` — the same split over B env instances on player routes: focal players are
    group 0 and background players group 1 of `BatchedSubstrate.player_routes`, so each step draws
    their observations straight into focal and background rows and reads their actions from rows
    laid out the same way. The background policy is a callable on the background `BatchedTimeStep`.
    With `roles` and `bots_by_role` it plays a background population instead, as the reference's `Population`
    (`utils/scenarios/population.py`) does: each background slot draws one of its role's bots at every episode start,
    on the device (`BatchedSubstrate.drawn_routes`), and each bot's policy acts on its own rows.

Scenario configs (`meltingpot/configs/scenarios`) name SavedModel bots and are not compiled here.
"""

from __future__ import annotations

import dataclasses
from typing import Any, Collection, Dict, Mapping, Sequence, Tuple

from meltingpot_b200 import substrate as substrate_lib

# Observations that exist once per env instance, not once per player, in a BatchedTimeStep.
_GLOBAL_KEYS = ('WORLD.RGB', 'COLLECTIVE_REWARD')


def _restrict_observation(observation: Mapping[str, Any], permitted: Collection[str]) -> Dict[str, Any]:
  return {key: observation[key] for key in observation if key in permitted}


def _restrict_observations(observations, permitted):
  return tuple(_restrict_observation(o, permitted) for o in observations)


def _partition(values: Sequence[Any], is_focal: Sequence[bool]) -> Tuple[tuple, tuple]:
  focal, background = [], []
  for f, v in zip(is_focal, values):
    (focal if f else background).append(v)
  return tuple(focal), tuple(background)


def _merge(focal_values: Sequence[Any], background_values: Sequence[Any], is_focal: Sequence[bool]) -> tuple:
  focal_values, background_values = iter(focal_values), iter(background_values)
  return tuple(next(focal_values if f else background_values) for f in is_focal)


@dataclasses.dataclass(frozen=True)
class ScenarioObservables:
  """Fields of the reference's ScenarioObservables that exist here (`scenario.py:84-98`)."""
  action: substrate_lib.Subject
  timestep: substrate_lib.Subject
  events: substrate_lib.Subject      # never emits (`scenario.py:216-220`)
  substrate: Any


class Scenario:
  """A substrate where a number of player slots are filled by bots (dm_env surface, one env)."""

  def __init__(self, substrate, background_population, is_focal: Sequence[bool],
               permitted_observations: Collection[str]) -> None:
    num_players = len(substrate.action_spec())
    if len(is_focal) != num_players:
      raise ValueError(f'is_focal is length {len(is_focal)} but substrate is '
                       f'{num_players}-player.')
    self._substrate = substrate
    self._background_population = background_population
    self._is_focal = tuple(bool(f) for f in is_focal)
    self._permitted_observations = frozenset(permitted_observations)
    self._focal_action_subject = substrate_lib.Subject()
    self._focal_timestep_subject = substrate_lib.Subject()
    self._events_subject = substrate_lib.Subject()
    self._observables = ScenarioObservables(
        action=self._focal_action_subject, timestep=self._focal_timestep_subject,
        events=self._events_subject, substrate=self._substrate.observables())

  def close(self) -> None:
    self._background_population.close()
    self._substrate.close()
    self._focal_action_subject.on_completed()
    self._focal_timestep_subject.on_completed()
    self._events_subject.on_completed()

  def __enter__(self):
    return self

  def __exit__(self, *unused):
    self.close()

  def _await_full_action(self, focal_action: Sequence[int]) -> Sequence[int]:
    expected = sum(self._is_focal)
    if len(focal_action) != expected:
      raise ValueError(f'Expected {expected} focal actions, got {len(focal_action)}.')
    self._focal_action_subject.on_next(focal_action)
    background_action = self._background_population.await_action()
    return _merge(focal_action, background_action, self._is_focal)

  def _split_timestep(self, timestep):
    focal_rewards, background_rewards = _partition(timestep.reward, self._is_focal)
    focal_obs, background_obs = _partition(timestep.observation, self._is_focal)
    focal_obs = _restrict_observations(focal_obs, self._permitted_observations)
    return (timestep._replace(reward=focal_rewards, observation=focal_obs),
            timestep._replace(reward=background_rewards, observation=background_obs))

  def _send_full_timestep(self, timestep):
    focal_timestep, background_timestep = self._split_timestep(timestep)
    self._background_population.send_timestep(background_timestep)
    self._focal_timestep_subject.on_next(focal_timestep)
    return focal_timestep

  def reset(self):
    timestep = self._substrate.reset()
    self._background_population.reset()
    return self._send_full_timestep(timestep)

  def step(self, action: Sequence[int]):
    action = self._await_full_action(focal_action=action)
    timestep = self._substrate.step(action)
    if timestep.step_type.first():
      self._background_population.reset()
    return self._send_full_timestep(timestep)

  def observation(self):
    focal, _ = _partition(self._substrate.observation(), self._is_focal)
    return _restrict_observations(focal, self._permitted_observations)

  def events(self):
    return ()  # substrate events would carry substrate player indices (`scenario.py:216-220`)

  def action_spec(self):
    return _partition(self._substrate.action_spec(), self._is_focal)[0]

  def observation_spec(self):
    focal, _ = _partition(self._substrate.observation_spec(), self._is_focal)
    return _restrict_observations(focal, self._permitted_observations)

  def reward_spec(self):
    return _partition(self._substrate.reward_spec(), self._is_focal)[0]

  def discount_spec(self, *args, **kwargs):
    return self._substrate.discount_spec(*args, **kwargs)

  def observables(self) -> ScenarioObservables:
    return self._observables


class BatchedScenario:
  """The focal / background split over a `BatchedSubstrate` (all tensors stay on the device).

  `background_policy(background_timestep) -> int tensor [B, n_background]` is called once per
  step with the timestep the background players see (all their observations, unrestricted).

  Focal and background players are routed (`BatchedSubstrate.player_routes`): every step renders their images, rewards
  and scalar observations straight into rows of new tensors, focal rows first, each group laid out [B, n, ...] in slot
  order, and reads their actions from rows laid out the same way. A returned timestep's per-player tensors therefore
  stay valid after the next step.

  Population mode (`roles` and `bots_by_role` given): `roles[p]` is the role of player slot p and `bots_by_role` maps
  each background slot's role to the names of the bots that may fill it; `background_policy` maps each bot name to a
  callable `policy(timestep, active) -> int tensor [B, n_k]`. At every episode start of every env, each background slot
  plays a bot drawn uniformly with replacement from its role's bots, as the reference's `Population.reset` does
  (`population.py:114-128`), though not from Python's `random` stream. Bot k's rows hold every slot that may play it,
  [B, n_k] in slot order; its callable gets their timestep and `active` (bool [B, n_k]: the rows played this episode)
  and returns an action for each row. Inactive rows are neither rendered nor read. `background_bots()` tells which bot
  each background slot plays. Focal players are routed as without a population.

  world_envs: distinct env indices whose WORLD.RGB is rendered (e.g. the few envs of a video); every other env's is
  not. The timesteps' 'WORLD.RGB', where permitted, is then uint8 [n, H, W, 3], row k holding env world_envs[k].
  """

  def __init__(self, substrate: substrate_lib.BatchedSubstrate, background_policy, is_focal: Sequence[bool],
               permitted_observations: Collection[str], *, roles: Sequence[str] = None,
               bots_by_role: Mapping[str, Collection[str]] = None, world_envs=None) -> None:
    import numpy as np  # pylint: disable=g-import-not-at-top
    if len(is_focal) != substrate.num_players:
      raise ValueError(f'is_focal is length {len(is_focal)} but substrate is '
                       f'{substrate.num_players}-player.')
    self._substrate = substrate
    self._policy = background_policy
    self._is_focal = tuple(bool(f) for f in is_focal)
    self._permitted = frozenset(permitted_observations)
    self._background_timestep = None
    self.num_envs = substrate.num_envs
    self.num_focal = sum(self._is_focal)
    self.num_background = substrate.num_players - self.num_focal
    self.bot_names: Tuple[str, ...] = ()
    if bots_by_role is None:
      if roles is not None:
        raise ValueError('roles needs bots_by_role')
      groups = np.tile(np.array([0 if f else 1 for f in self._is_focal], np.int64), (self.num_envs, 1))
      self._routes = substrate.player_routes(groups)
      n = self._routes.n_rows  # every player is routed: B * P rows, focal rows first
      self._background_rows = slice(self.num_envs * self.num_focal, n)
    else:
      self._routes = substrate.drawn_routes(self._population_choices(background_policy, roles, bots_by_role))
    self._actions = self._routes.actions()
    self._focal_rows = slice(0, self.num_envs * self.num_focal)
    self._world = None  # (world_envs, world_row_of_env) when WORLD.RGB is routed
    if world_envs is not None:
      if substrate._world_shape() is None:  # pylint: disable=protected-access
        raise ValueError('world_envs: this batch renders no WORLD.RGB (it was built with world_rgb=False)')
      self._world = substrate_lib.world_row_map(world_envs, self.num_envs, self._routes.device)

  def _population_choices(self, policies, roles, bots_by_role):
    """Validates population mode and returns each slot's groups for drawn_routes: group 0 for focal slots, group
    1 + k for bot k of bot_names (the bots that some background slot may play, sorted)."""
    if roles is None:
      raise ValueError('bots_by_role needs roles, the role of each player slot')
    if isinstance(roles, str) or len(roles) != len(self._is_focal):
      raise ValueError('roles and is_focal must be the same length.')
    names_by_role = {role: tuple(sorted(set(names))) for role, names in bots_by_role.items()}
    background_roles = [role for role, f in zip(roles, self._is_focal) if not f]
    for role in background_roles:
      if role not in names_by_role:
        raise ValueError(f'no bots for role {role!r}: bots_by_role has roles {sorted(names_by_role)}')
      if not names_by_role[role]:
        raise ValueError(f'bots_by_role[{role!r}] is empty')
      if len(names_by_role[role]) > 8:
        raise ValueError(f'bots_by_role[{role!r}] lists {len(names_by_role[role])} bots, at most 8')
    self.bot_names = tuple(sorted({n for role in background_roles for n in names_by_role[role]}))
    if not isinstance(policies, Mapping):
      raise ValueError('with bots_by_role, background_policy must map each bot name to a callable')
    for name in self.bot_names:
      if not callable(policies.get(name)):
        raise ValueError(f'background_policy has no callable for bot {name!r}')
    index = {n: k for k, n in enumerate(self.bot_names)}
    return [(0,) if f else tuple(1 + index[n] for n in names_by_role[role]) for role, f in zip(roles, self._is_focal)]

  def _outputs(self):
    """Fresh row tensors for one step (every row is written, so they are not zeroed)."""
    import torch  # pylint: disable=g-import-not-at-top
    r = self._routes
    dev = r.device
    tensors = {'RGB': torch.empty((r.n_rows,) + tuple(self._substrate.engine.rgb.shape[2:]), dtype=torch.uint8, device=dev),
               'REWARD': torch.empty((r.n_rows,), dtype=torch.float64, device=dev)}
    names = self._substrate._scalar_names  # pylint: disable=protected-access
    block = torch.empty((len(names), r.n_rows), dtype=torch.float64, device=dev) if names else None
    for k, name in enumerate(names):
      tensors[name] = block[k]
    if self._world is not None:
      shape = (int(self._world[0].shape[0]),) + self._substrate._world_shape()  # pylint: disable=protected-access
      tensors['WORLD.RGB'] = torch.empty(shape, dtype=torch.uint8, device=dev)
    return substrate_lib.PlayerOutputs(r, None, tensors, block, world=self._world)

  def _select(self, timestep, tensors, n, permitted):
    """The timestep of one group: `tensors` holds its rows ({name: [B * n, ...]})."""
    def view(v):
      return v.view((self.num_envs, n) + tuple(v.shape[1:]))
    obs = {}
    for key in ('RGB',) + tuple(timestep.observation):  # a routed timestep has no 'RGB': the rows hold the images
      if permitted is not None and key not in permitted:
        continue
      obs[key] = timestep.observation[key] if key in _GLOBAL_KEYS else view(tensors[key])
    return substrate_lib.BatchedTimeStep(step_type=timestep.step_type, reward=view(tensors['REWARD']),
                                         discount=timestep.discount, observation=obs)

  def _split(self, timestep, tensors):
    """tensors(g): {name: tensor} of group g's rows (0 focal, then the background groups)."""
    if self.bot_names:
      r = self._routes
      self._background_timestep = {n: self._select(timestep, tensors(k + 1), len(r.group(k + 1)), None)
                                   for k, n in enumerate(self.bot_names)}
    else:
      self._background_timestep = self._select(timestep, tensors(1), self.num_background, None)
    return self._select(timestep, tensors(0), self.num_focal, self._permitted)

  def _rows_of(self, po):
    """tensors(g) for _split of a PlayerOutputs holding every row."""
    rows = {0: self._focal_rows}
    if self.bot_names:
      rows.update({k + 1: self._routes.rows(k + 1) for k in range(len(self.bot_names))})
    else:
      rows[1] = self._background_rows
    return lambda g: {k: v[rows[g]] for k, v in po.tensors.items() if k != 'WORLD.RGB'}

  def trajectory(self, T: int, time_major: bool = True) -> 'ScenarioTrajectory':
    """Tensors for T focal timesteps; `reset(out=traj.at(t))` and `step(focal_actions, out=traj.at(t))` deliver the
    focal players straight into slot t. See ScenarioTrajectory."""
    return ScenarioTrajectory(self, int(T), bool(time_major))

  def _slot(self, out):
    """(GroupOutputs of one step into slot `out`, engine targets of its per-env outputs)."""
    import torch  # pylint: disable=g-import-not-at-top
    if not isinstance(out, ScenarioSlot) or out.rows.routes is not self._routes:
      raise ValueError('out must be a slot of this scenario\'s trajectory (trajectory(T).at(t))')
    r = self._routes
    groups = {0: out.rows.groups[0]}
    for g in range(1, r.num_groups):  # the background rows go to fresh tensors, as without out
      rows = r.rows(g)
      groups[g] = substrate_lib._group_tensors(r, g, (rows.stop - rows.start,), torch.empty)  # pylint: disable=protected-access
    world = None
    if self._world is not None:
      world = (out.rows.world_envs, out.rows.world_row_of_env, out.rows.world_rgb)
    po = substrate_lib.GroupOutputs(r, {g: None for g in groups}, groups=groups, world=world)
    targets = substrate_lib.BatchedTimeStep(step_type=out.step_type, reward=None, discount=out.discount, observation={})
    return po, targets

  def _slot_timestep(self, timestep, po, out):
    """_split of a step into slot `out`, its COLLECTIVE_REWARD summed into the slot from the engine's rewards."""
    import torch  # pylint: disable=g-import-not-at-top
    sub = self._substrate
    collective = out.observation[substrate_lib._COLLECTIVE_REWARD_OBS]  # pylint: disable=protected-access
    sub._fill_collective(substrate_lib.BatchedTimeStep(  # pylint: disable=protected-access
        step_type=out.step_type, reward=sub.engine.reward, discount=out.discount,
        observation={substrate_lib._COLLECTIVE_REWARD_OBS: collective}))  # pylint: disable=protected-access
    # the keys of a routed timestep, in its order; _select reads per-player values from the rows, not from here
    obs = {name: None for name in sub._scalar_names}  # pylint: disable=protected-access
    if sub._world_shape() is not None:  # pylint: disable=protected-access
      obs['WORLD.RGB'] = timestep.observation.get('WORLD.RGB', sub.engine.world_rgb)  # unrouted: per env, as without out
    obs[substrate_lib._COLLECTIVE_REWARD_OBS] = collective  # pylint: disable=protected-access
    ts = substrate_lib.BatchedTimeStep(step_type=timestep.step_type, reward=None, discount=timestep.discount, observation=obs)
    background = lambda g: (po.groups[g][0] if g < self._routes.num_groups else  # (no background players)
                            substrate_lib._group_tensors(self._routes, g, (0,), torch.empty)[0])  # pylint: disable=protected-access
    return self._split(ts, background)

  def reset(self, out=None):
    """out: a slot of trajectory(T) (`traj.at(t)`) to reset into; the returned focal timestep is then views of it."""
    if out is not None:
      po, targets = self._slot(out)
      return self._slot_timestep(self._substrate.reset(out=targets, players=po), po, out)
    po = self._outputs()
    return self._split(self._substrate.reset(players=po), self._rows_of(po))

  def step(self, focal_actions, out=None):
    """focal_actions: int tensor [B, num_focal]; returns the focal players' BatchedTimeStep. out: as for reset."""
    if tuple(focal_actions.shape) != (self.num_envs, self.num_focal):
      raise ValueError(f'Expected {self.num_focal} focal actions per env, got shape {tuple(focal_actions.shape)}.')
    rows = self._actions.tensor
    rows[self._focal_rows].view(self.num_envs, self.num_focal).copy_(focal_actions)
    if self.bot_names:
      r = self._routes
      for k, name in enumerate(self.bot_names):
        g = k + 1
        actions = self._policy[name](self._background_timestep[name], r.active(g))
        rows[r.rows(g)].view(self.num_envs, len(r.group(g))).copy_(actions)
    elif self.num_background:
      background_actions = self._policy(self._background_timestep)
      rows[self._background_rows].view(self.num_envs, self.num_background).copy_(background_actions)
    if out is not None:
      po, targets = self._slot(out)
      return self._slot_timestep(self._substrate.step(out=targets, players=po, player_actions=self._actions), po, out)
    po = self._outputs()
    return self._split(self._substrate.step(players=po, player_actions=self._actions), self._rows_of(po))

  @property
  def background_timestep(self):
    """What the background players saw last (unrestricted observations); in population mode, a dict of each bot's."""
    return self._background_timestep

  def background_bots(self):
    """Population mode: int64 CUDA [B, num_background], the index in bot_names of the bot each background slot plays
    in the episode its env is in (from the routes' row map, with torch ops on the current stream)."""
    import torch  # pylint: disable=g-import-not-at-top
    if not self.bot_names:
      raise ValueError('background_bots needs population mode (roles and bots_by_role)')
    r = self._routes
    slots = [p for p, f in enumerate(self._is_focal) if not f]
    starts = torch.tensor([r.rows(g).start for g in range(1, r.num_groups)], dtype=torch.int64, device=r.device)
    rows = r.row_of_player[:, slots].to(torch.int64)
    return torch.bucketize(rows, starts, right=True) - 1

  def close(self):
    self._substrate.close()


@dataclasses.dataclass
class ScenarioSlot(substrate_lib.BatchedTimeStep):
  """Slot t of a ScenarioTrajectory: the focal timestep's fields as views of the slot, and `rows`, the focal group's
  rows of the slot (a GroupOutputs) that the engine writes."""
  rows: Any = None


class ScenarioTrajectory:
  """T focal timesteps of a BatchedScenario in caller-owned CUDA tensors (BatchedScenario.trajectory).

  Per focal player: `reward` float64 and observation 'RGB' uint8 and each scalar observation float64, each
  [T, B, num_focal, ...] (time_major) or [B, num_focal, T, ...]; the step renders them straight into slot t through
  the focal group's row segment, so keeping a trajectory costs no copy. Per env: `step_type` int64, `discount` float64
  and observation 'COLLECTIVE_REWARD' float64, [T, B] or [B, T]. With the scenario's world_envs, observation
  'WORLD.RGB' uint8 is [T, n, H, W, 3] ([n, T, H, W, 3] when not time_major), row k holding env world_envs[k]. Without
  world_envs, WORLD.RGB stays per env in the engine's buffer, where the background players see it too. The background
  players' rows go to fresh tensors every step, as without a trajectory."""

  def __init__(self, scenario: BatchedScenario, T: int, time_major: bool):
    import torch  # pylint: disable=g-import-not-at-top
    if T < 1:
      raise ValueError(f'a trajectory needs T >= 1 slots, got {T}')
    r = scenario._routes  # pylint: disable=protected-access
    world = scenario._world  # pylint: disable=protected-access
    self.T, self.time_major = T, time_major
    self.num_envs, self.num_focal = scenario.num_envs, scenario.num_focal
    self.rows = r.group_outputs({0: T}, time_major, world_envs=None if world is None else world[0])
    B, n = self.num_envs, self.num_focal
    tensors, block = self.rows.groups[0]

    def per_player(v, lead):  # [T, B * n, ...] -> [T, B, n, ...]; [B * n, T, ...] -> [B, n, T, ...]
      shape = tuple(v.shape)
      if time_major:
        return v.view(shape[:lead + 1] + (B, n) + shape[lead + 2:])
      return v.view(shape[:lead] + (B, n) + shape[lead + 1:])

    def new(dtype):
      return torch.zeros((T, B) if time_major else (B, T), dtype=dtype, device=r.device)

    self.step_type = new(torch.int64)
    self.discount = new(torch.float64)
    self.reward = per_player(tensors['REWARD'], 0)
    self.observation = {k: per_player(v, 0) for k, v in tensors.items() if k != 'REWARD'}
    if self.rows.world_rgb is not None:
      self.observation['WORLD.RGB'] = self.rows.world_rgb
    self.observation[substrate_lib._COLLECTIVE_REWARD_OBS] = new(torch.float64)  # pylint: disable=protected-access

  def at(self, t: int) -> ScenarioSlot:
    """Slot t, for BatchedScenario.reset(out=) / step(out=)."""
    if not -self.T <= t < self.T:
      raise IndexError(f'slot {t} of a trajectory of {self.T}')
    pick = (lambda x: x[t]) if self.time_major else (lambda x: x[:, t])
    pick_player = (lambda x: x[t]) if self.time_major else (lambda x: x[:, :, t])
    obs = {}
    for k, v in self.observation.items():
      obs[k] = pick(v) if k in _GLOBAL_KEYS else pick_player(v)
    return ScenarioSlot(step_type=pick(self.step_type), reward=pick_player(self.reward), discount=pick(self.discount),
                        observation=obs, rows=self.rows.at(t))
