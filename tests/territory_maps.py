"""TEST INFRASTRUCTURE: map sets of territory__rooms (TORUS), territory__open (BOUNDED) and coop_mining.

Each substrate gets four maps of one size: its own and three edits of it, one that moves walls, one that adds or removes
resources (ores) so that the counts differ, and one that moves spawn points. The maps are compiled as one set on one
sprite table (compiler.compile_settings_set, what substrate.build_batched(maps=...) does from a reference checkout), from
the recorded lab2d settings (tests/golden/settings_*.json.gz) under the 40-frame cap of tests/env_variants.py, so no
reference checkout is needed.
"""

import functools

from meltingpot_b200 import compiler
from tests import env_variants as EV
from tests import settings_golden
from tests import variants as V

PLAYERS = {'territory__rooms': 9, 'territory__open': 9, 'coop_mining': 6}
NAMES = tuple(PLAYERS)


def _put(rows, y, x, text):
  rows[y] = rows[y][:x] + text + rows[y][x + len(text):]


def _edit(fn):
  """A map_rows edit; `fn` edits the map's rows in place, numbered from the first row of the map (the settings' map
  text starts with a newline)."""
  def rows_edit(rows):
    lead = 1 if rows and rows[0] == '' else 0
    body = list(rows[lead:])
    fn(body)
    return list(rows[:lead]) + body
  return V.map_rows(rows_edit)


def _rooms_walls(r):  # the top-left corner piece moves into the room below it
  _put(r, 1, 0, 'J'); _put(r, 3, 2, 'W'); _put(r, 12, 4, 'WW')


def _rooms_resources(r):  # doors between the rooms (-12 resources), a resource row inside each room (+15): 183
  for y in (3, 10, 17):
    _put(r, y, 6, ',,'); _put(r, y, 13, ',,')
  for y in (9, 16):
    for x in (1, 8, 15):
      _put(r, y, x, 'RRRRR')


def _rooms_spawns(r):  # every spawn point one cell down and right
  for y in (3, 10, 17):
    for x in (3, 10, 17):
      _put(r, y, x, ','); _put(r, y + 1, x + 1, 'P')


def _open_walls(r):  # wall segments inside the open field
  _put(r, 11, 5, '======'); _put(r, 20, 30, '||')


def _open_resources(r):  # the top rows lose their resources (-20), the bottom row gains 37: 105
  for y in (1, 2, 3, 4):
    r[y] = r[y][0] + r[y][1:-1].replace('R', ',') + r[y][-1]
  _put(r, 21, 1, 'R' * 37)


def _open_spawns(r):  # the spawn points of row 19 move up to row 11
  r[11] = r[11][0] + r[19][1:-1] + r[11][-1]
  r[19] = r[19].replace('P', ',')


def _mining_walls(r):  # one wall segment moves, ore count unchanged
  _put(r, 3, 9, 'O'); _put(r, 3, 15, 'W')


def _mining_ores(r):  # the ores of the bottom rows and the right column become wall, a wall segment becomes ore
  for y in range(20, 26):
    r[y] = r[y][0] + r[y][1:-1].replace('O', 'W') + r[y][-1]
  for y in range(2, 20):
    _put(r, y, 25, 'W')
  _put(r, 12, 6, 'OOO')


def _mining_spawns(r):  # every spawn point one row down
  ps = [(y, x) for y, row in enumerate(r) for x, c in enumerate(row) if c == 'P']
  for y, x in ps:
    _put(r, y, x, 'O')
  for y, x in ps:
    _put(r, y + 1, x, 'P')


EDITS = {
    'territory__rooms': (_rooms_walls, _rooms_resources, _rooms_spawns),
    'territory__open': (_open_walls, _open_resources, _open_spawns),
    'coop_mining': (_mining_walls, _mining_ores, _mining_spawns),
}


def settings(name, k=0):
  """The capped settings of map k of `name`: 0 its own, 1 walls moved, 2 resource (ore) count changed, 3 spawns moved."""
  s = settings_golden.settings(name, PLAYERS[name])
  for edit in EV._CAP_40:  # pylint: disable=protected-access
    edit(s)
  if k:
    _edit(EDITS[name][k - 1])(s)
  return s


def config(name):
  return settings_golden.config(name, PLAYERS[name])


def ascii_map(name, k=0):
  return settings(name, k)['simulation']['map']


@functools.lru_cache(maxsize=None)
def map_set(name):
  """The four maps of `name` compiled as one set."""
  return tuple(compiler.compile_settings_set([settings(name, k) for k in range(4)], config(name)))


@functools.lru_cache(maxsize=None)
def alone(name, k):
  """Map k of `name` compiled on its own."""
  return compiler.compile_settings(settings(name, k), config(name))
