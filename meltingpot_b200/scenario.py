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

Scenario configs (`meltingpot/configs/scenarios`) name SavedModel bots and are not compiled here.
"""

from __future__ import annotations

import dataclasses
from typing import Any, Callable, Collection, Dict, Mapping, Sequence, Tuple

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
  """

  def __init__(self, substrate: substrate_lib.BatchedSubstrate, background_policy: Callable[[Any], Any],
               is_focal: Sequence[bool], permitted_observations: Collection[str]) -> None:
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
    groups = np.tile(np.array([0 if f else 1 for f in self._is_focal], np.int64), (self.num_envs, 1))
    self._routes = substrate.player_routes(groups)
    self._actions = self._routes.actions()
    n = self._routes.n_rows  # every player is routed: B * P rows, focal rows first
    self._focal_rows, self._background_rows = slice(0, self.num_envs * self.num_focal), slice(self.num_envs * self.num_focal, n)

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
    return substrate_lib.PlayerOutputs(r, None, tensors, block)

  def _select(self, timestep, po, rows, n, permitted):
    def view(v):
      return v[rows].view((self.num_envs, n) + tuple(v.shape[1:]))
    obs = {}
    for key in ('RGB',) + tuple(timestep.observation):  # a routed timestep has no 'RGB': the rows hold the images
      if permitted is not None and key not in permitted:
        continue
      obs[key] = timestep.observation[key] if key in _GLOBAL_KEYS else view(po[key])
    return substrate_lib.BatchedTimeStep(step_type=timestep.step_type, reward=view(po['REWARD']),
                                         discount=timestep.discount, observation=obs)

  def _split(self, timestep, po):
    self._background_timestep = self._select(timestep, po, self._background_rows, self.num_background, None)
    return self._select(timestep, po, self._focal_rows, self.num_focal, self._permitted)

  def reset(self):
    po = self._outputs()
    return self._split(self._substrate.reset(players=po), po)

  def step(self, focal_actions):
    """focal_actions: int tensor [B, num_focal]; returns the focal players' BatchedTimeStep."""
    if tuple(focal_actions.shape) != (self.num_envs, self.num_focal):
      raise ValueError(f'Expected {self.num_focal} focal actions per env, got shape {tuple(focal_actions.shape)}.')
    rows = self._actions.tensor
    rows[self._focal_rows].view(self.num_envs, self.num_focal).copy_(focal_actions)
    if self.num_background:
      background_actions = self._policy(self._background_timestep)
      rows[self._background_rows].view(self.num_envs, self.num_background).copy_(background_actions)
    po = self._outputs()
    return self._split(self._substrate.step(players=po, player_actions=self._actions), po)

  @property
  def background_timestep(self):
    """What the background players saw last (unrestricted observations)."""
    return self._background_timestep

  def close(self):
    self._substrate.close()
