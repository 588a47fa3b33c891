"""Locates / builds compiled substrate blobs."""

from __future__ import annotations

import os
from typing import Mapping, Optional, Sequence

_DATA = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'data')

# substrate -> player counts with a committed blob (default roles repeated).
PRECOMPILED = {
    'clean_up': (7,),
    'commons_harvest__open': (7, 16),
    'territory__rooms': (9,),
    'territory__open': (9,),
    'territory__inside_out': (5,),
    'commons_harvest__closed': (7,),
    'commons_harvest__partnership': (7,),
    'coins': (2,),
    'coop_mining': (6,),
}

# Substrates whose CONFIG BUILDER draws from Python's `random` (coins.py:45-84,488: map size, coin colours): the
# reference makes one draw per `build()` call; a compiled blob fixes one draw, made with this seed (policy A.20).
# ('choice' prefabs -- territory__inside_out -- are NOT fixed at compile time: the engine draws them per env and per
# episode, as the reference's prefab_utils.lua:63-65 does at every env build.)
BUILD_SEEDS = {'coins': 0}


def blob_path(name: str, num_players: int) -> str:
  return os.path.join(_DATA, f'{name}__{num_players}p.mpb')


def load_blob(name: str, roles: Optional[Sequence[str]] = None) -> bytes:
  """Returns the compiled blob for `name` with `roles`.

  Uses the committed blob when the roles are the substrate's default role
  repeated; otherwise compiles from a reference checkout (compiler.reference_root()).
  """
  from meltingpot_b200 import compiler  # pylint: disable=g-import-not-at-top
  num_players = len(roles) if roles is not None else None
  if roles is None or len(set(roles)) == 1:
    counts = PRECOMPILED.get(name, ())
    n = num_players if num_players is not None else (counts[0] if counts else None)
    if n is not None and os.path.exists(blob_path(name, n)):
      if roles is None or _is_default_role(name, roles[0]):
        with open(blob_path(name, n), 'rb') as f:
          return f.read()
  if compiler.reference_root() is None:
    raise FileNotFoundError(
        f'no precompiled blob for {name!r} with roles {roles!r} and no Melting Pot '
        'reference checkout to compile from (set MELTINGPOT_REFERENCE_ROOT)')
  return compiler.compile_substrate(name, roles, build_seed=BUILD_SEEDS.get(name))


def compile_with_overrides(name: str, roles: Sequence[str], prefab_overrides):
  """The blob of `name` with `roles` and the reference's `prefab_overrides` (compiled from a reference checkout).

  One mapping gives one blob. A sequence of mappings gives one blob per entry, compiled as one set on one sprite table
  (compiler.compile_substrate_set), so that entries whose overrides change how pieces look can run side by side in one
  engine; without such overrides each blob equals the entry compiled alone."""
  from meltingpot_b200 import compiler  # pylint: disable=g-import-not-at-top
  if compiler.reference_root() is None:
    raise FileNotFoundError(
        f'prefab_overrides for {name!r} need a Melting Pot reference checkout to compile from '
        '(set MELTINGPOT_REFERENCE_ROOT)')
  if isinstance(prefab_overrides, Mapping):
    return compiler.compile_substrate(name, roles, build_seed=BUILD_SEEDS.get(name), prefab_overrides=prefab_overrides)
  overrides = list(prefab_overrides)
  return compiler.compile_substrate_set(name, roles, [BUILD_SEEDS.get(name)] * len(overrides), prefab_overrides=overrides)


def compile_draws(name: str, roles: Sequence[str], build_seeds: Sequence[int]) -> list:
  """The draws of `name` with `roles` under `build_seeds`, one blob per seed on one sprite table
  (compiler.compile_substrate_set; compiled from a reference checkout)."""
  from meltingpot_b200 import compiler  # pylint: disable=g-import-not-at-top
  if compiler.reference_root() is None:
    raise FileNotFoundError(
        f'build_seeds for {name!r} need a Melting Pot reference checkout to compile from '
        '(set MELTINGPOT_REFERENCE_ROOT)')
  return compiler.compile_substrate_set(name, roles, list(build_seeds))


# Substrates whose ASCII map build_batched(maps=...) replaces: every map of a set keeps the substrate's size, topology,
# players and view, so the engine runs the set side by side (map variants).
MAP_SUBSTRATES = ('territory__rooms', 'territory__open', 'territory__inside_out', 'coop_mining')


def checked_maps(name: str, maps: Sequence[str]) -> list:
  """`maps` as a list of ASCII maps of `name`, each with the rows and row width of the substrate's own map."""
  from meltingpot_b200 import blob as blob_lib  # pylint: disable=g-import-not-at-top
  from meltingpot_b200 import compiler  # pylint: disable=g-import-not-at-top
  if name not in MAP_SUBSTRATES:
    raise ValueError(f'maps replace the map of {", ".join(MAP_SUBSTRATES)}, not of {name!r}')
  if isinstance(maps, str):
    raise ValueError('maps is a sequence of ASCII maps, not one map')
  maps = list(maps)
  if not maps:
    raise ValueError('the sequence of maps is empty')
  with open(blob_path(name, PRECOMPILED[name][0]), 'rb') as f:
    meta = blob_lib.unpack(f.read())['meta']
  W, H = int(meta[1]), int(meta[2])
  for i, ascii_map in enumerate(maps):
    if not isinstance(ascii_map, str):
      raise ValueError(f'maps[{i}] is a {type(ascii_map).__name__}, not a str')
    rows = compiler._map_rows(ascii_map)  # pylint: disable=protected-access
    if len(rows) != H:
      raise ValueError(f'maps[{i}] has {len(rows)} rows; {name} has {H}')
    for y, row in enumerate(rows):
      if len(row) != W:
        raise ValueError(f'row {y} of maps[{i}] is {len(row)} wide; {name} is {W} wide')
  return maps


def compile_maps(name: str, roles: Sequence[str], maps: Sequence[str]) -> list:
  """The blobs of `name` with `roles` and each of `maps` as its ASCII map, compiled as one map set on one sprite table
  (compiler.compile_substrate_maps; compiled from a reference checkout)."""
  from meltingpot_b200 import compiler  # pylint: disable=g-import-not-at-top
  if compiler.reference_root() is None:
    raise FileNotFoundError(
        f'maps for {name!r} need a Melting Pot reference checkout to compile from '
        '(set MELTINGPOT_REFERENCE_ROOT)')
  return compiler.compile_substrate_maps(name, roles, list(maps))


def _is_default_role(name: str, role: str) -> bool:
  del name
  return role == 'default'
