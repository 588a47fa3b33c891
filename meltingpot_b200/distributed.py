"""Env-instance data parallelism: shard envs over ranks, return the stacked timestep / observations to every rank.

Env instances never interact (each `dmlab2d.Lab2d` is an isolated world,
`meltingpot/utils/substrates/builder.py:179-187`), so the hot path itself needs
no collective: rank r simply steps envs [base, base + count). Env b's RNG key is
`seed + b` with b the GLOBAL env index, so results do not depend on the number of ranks.
The only exchange is returning one stacked tensor per timestep field (and, optionally, the stacked observations) to
every rank. On GPUs this is done by the engine itself: `connect_exchange` / `connect_gather_obs` hand every rank's
buffers to every rank once (CUDA IPC handles over torch.distributed) and from then on the kernels deliver with
peer-memory stores over NVLink (include/mp_engine.h, mp_exchange_* / mp_gather_obs_*). The plain collectives below
(`all_gather_stacked`, `gather_timestep_scalars`; NCCL or gloo) remain for host-side logic and the CPU tests.
"""

from __future__ import annotations

from typing import Optional, Tuple


def shard_envs(global_num_envs: int, rank: int, world_size: int) -> Tuple[int, int]:
  """Returns (env_index_base, count) of the contiguous shard owned by `rank`."""
  if not 0 <= rank < world_size:
    raise ValueError(f'rank {rank} outside world of {world_size}')
  if global_num_envs % world_size:
    raise ValueError(f'{global_num_envs} envs do not split evenly over {world_size} ranks')
  count = global_num_envs // world_size
  return rank * count, count


def all_gather_stacked(tensor, group=None):
  """Stacks equal-shaped per-rank tensors along dim 0 on every rank (rank order = env order)."""
  import torch  # pylint: disable=g-import-not-at-top
  import torch.distributed as dist  # pylint: disable=g-import-not-at-top
  world = dist.get_world_size(group)
  tensor = tensor.contiguous()
  out = torch.empty((world * tensor.shape[0],) + tuple(tensor.shape[1:]), dtype=tensor.dtype, device=tensor.device)
  if dist.get_backend(group) == 'nccl':
    dist.all_gather_into_tensor(out, tensor, group=group)
  else:
    chunks = list(out.chunk(world, dim=0))
    dist.all_gather(chunks, tensor, group=group)
  return out


def gather_timestep_scalars(reward, discount, step_type, group=None):
  """All-gathers (reward [b,P], discount [b], step_type [b]) into global [B,...] tensors.

  The three fields travel in one float64 buffer so that a step costs a single collective.
  """
  import torch  # pylint: disable=g-import-not-at-top
  b, p = reward.shape
  packed = torch.empty((b, p + 2), dtype=torch.float64, device=reward.device)
  packed[:, :p] = reward
  packed[:, p] = discount
  packed[:, p + 1] = step_type.to(torch.float64)
  full = all_gather_stacked(packed, group)
  return full[:, :p], full[:, p], full[:, p + 1].to(torch.int64)


def connect_exchange(eng, group=None) -> None:
  """Wires `eng` (this rank's engine.Engine) into the cross-GPU timestep exchange (mp_exchange_*).

  torch.distributed only carries the 64-byte CUDA IPC handles between the ranks, once; from then on every
  state-transition kernel writes its packed timestep rows straight into every rank's `gathered` buffer over
  NVLink peer mappings, with no collective kernel per step.
  """
  import torch.distributed as dist  # pylint: disable=g-import-not-at-top
  from meltingpot_b200 import engine as engine_lib  # pylint: disable=g-import-not-at-top
  rank, world = dist.get_rank(group), dist.get_world_size(group)
  ptr, _ = eng.exchange_create(rank, world)
  mine = engine_lib.ipc_export(ptr)
  everyone = [None] * world
  dist.all_gather_object(everyone, mine, group=group)
  blocks = [ptr if r == rank else engine_lib.ipc_open(eng.device, everyone[r][0], everyone[r][1]) for r in range(world)]
  eng.exchange_connect(blocks)
  dist.barrier(group=group)  # nobody publishes before everyone is mapped


def connect_gather_obs(eng, group=None) -> None:
  """Wires `eng` into the stacked-observation gather (mp_gather_obs_*): from then on its renderer also delivers every
  strip into every rank's stacked buffer over NVLink. torch.distributed only carries the IPC handles, once."""
  import torch.distributed as dist  # pylint: disable=g-import-not-at-top
  from meltingpot_b200 import engine as engine_lib  # pylint: disable=g-import-not-at-top
  rank, world = dist.get_rank(group), dist.get_world_size(group)
  ptr, _ = eng.gather_obs_create(rank, world)
  mine = engine_lib.ipc_export(ptr)
  everyone = [None] * world
  dist.all_gather_object(everyone, mine, group=group)
  blocks = [ptr if r == rank else engine_lib.ipc_open(eng.device, everyone[r][0], everyone[r][1]) for r in range(world)]
  eng.gather_obs_connect(blocks)
  dist.barrier(group=group)


class ShardedSubstrate:
  """One rank's shard of a globally indexed batch of env instances."""

  def __init__(self, name: str, roles, global_num_envs: int, seed: int, device: Optional[int] = None,
               world_rgb: bool = True, group=None, prefab_overrides=None, env_variant=None, build_seeds=None, maps=None):
    """name / prefab_overrides / build_seeds / maps / env_variant: as substrate.build_batched, with env_variant indexed
    by GLOBAL env; each rank takes the slice of its own envs (with build_seeds, maps or a sequence of names, and no
    env_variant, global env g plays variant g % len(build_seeds), g % len(maps) or g % len(name))."""
    import torch.distributed as dist  # pylint: disable=g-import-not-at-top
    from meltingpot_b200 import substrate  # pylint: disable=g-import-not-at-top
    self._group = group
    rank, world = dist.get_rank(group), dist.get_world_size(group)
    self.env_index_base, self.local_num_envs = shard_envs(global_num_envs, rank, world)
    self.global_num_envs = global_num_envs
    if device is None:
      import torch  # pylint: disable=g-import-not-at-top
      device = torch.cuda.current_device()
    local_variant = None
    if env_variant is not None:
      if len(env_variant) != global_num_envs:
        raise ValueError(f'env_variant has {len(env_variant)} entries for {global_num_envs} envs')
      local_variant = list(env_variant[self.env_index_base:self.env_index_base + self.local_num_envs])
    self.local = substrate.build_batched(name, roles=roles, num_envs=self.local_num_envs, device=device, seed=seed,
                                         env_index_base=self.env_index_base, world_rgb=world_rgb,
                                         prefab_overrides=prefab_overrides, env_variant=local_variant,
                                         build_seeds=build_seeds, maps=maps)

  def reset(self, out=None):
    """out: a BatchedTimeStep of this rank's envs to fill (BatchedSubstrate.step)."""
    return self.local.reset(out=out)

  def step(self, local_actions, out=None, restore=None, bank=None, rekey: bool = False):
    """restore / bank / rekey: as BatchedSubstrate.step, with restore indexed by LOCAL env. On a connected shard the
    restored envs' rows and images are published like any step's; every rank steps when the others do (passing an
    index of all -1 when it restores nothing)."""
    return self.local.step(local_actions, out=out, restore=restore, bank=bank, rekey=rekey)

  # -- engine-level exchanges (peer-memory stores from the kernels; no collective per step) ---------------------------
  def connect(self, observations: bool = False) -> None:
    """Wires this rank's engine into the stacked-timestep exchange (and the stacked-observation gather)."""
    connect_exchange(self.local.engine, self._group)
    if observations:
      connect_gather_obs(self.local.engine, self._group)
    self._connected = True

  def stacked_timestep(self):
    """(reward [G, P], discount [G], step_type [G]) of ALL ranks' envs for the step just taken (G = global envs).

    Collective: every rank calls it once per step. The rows were written into this rank's buffer by the other ranks'
    kernels; this enqueues the publish-and-wait kernel on the current stream and returns views of the buffer
    (valid until two steps later)."""
    import torch  # pylint: disable=g-import-not-at-top
    eng = self.local.engine
    eng.exchange_wait()
    rows = eng.gathered_timestep()
    p = eng.num_players
    return rows[:, :p], rows[:, p], rows[:, p + 1].to(torch.int64)

  def stacked_observations(self):
    """(RGB [G, P, h, w, 3], WORLD.RGB [G, H, W, 3]) of all ranks' envs (needs connect(observations=True))."""
    eng = self.local.engine
    eng.gather_obs_wait()
    return eng.gathered_observations()

  def gather_scalars(self, timestep):
    return gather_timestep_scalars(timestep.reward, timestep.discount, timestep.step_type, self._group)

  def gather_observation(self, timestep, key: str = 'RGB'):
    return all_gather_stacked(timestep.observation[key], self._group)

  def close(self):
    self.local.close()
