"""TEST INFRASTRUCTURE: commons_harvest__open, __closed and __partnership (7 players) compiled as one map set.

The three substrates share one player interface and one sprite table, so an engine runs them side by side as map
variants (substrate.build_batched with a sequence of names, mp_create_variants). Everything here compiles from the
recorded lab2d settings (tests/golden/settings_commons_harvest__*__7p.json.gz), so no reference checkout is needed.
"""

import functools

from meltingpot_b200 import compiler
from tests import settings_golden
from tests import variants as V

NAMES = ('commons_harvest__open', 'commons_harvest__closed', 'commons_harvest__partnership')
PLAYERS = 7
ROLES = ('default',) * PLAYERS
# the 40-frame episode cap of the GPU tests: every rollout of more than 40 steps crosses an auto-reset
CAP_40 = (V.kw('StochasticIntervalEpisodeEnding', probabilityTerminationPerInterval=0.0), V.top(maxEpisodeLengthFrames=40))


def settings(name, edits=()):
  s = settings_golden.settings(name, PLAYERS)
  for edit in edits:
    edit(s)
  return s


def config():
  return settings_golden.config(NAMES[0], PLAYERS)


def compile_set(settings_list):
  return tuple(compiler.compile_settings_set(list(settings_list), config()))


@functools.lru_cache(maxsize=None)
def map_set(capped=True):
  """The blobs of the three substrates compiled as one set, optionally with the 40-frame cap."""
  return compile_set([settings(n, CAP_40 if capped else ()) for n in NAMES])


@functools.lru_cache(maxsize=None)
def alone(name, capped=True):
  """The blob of one substrate compiled on its own."""
  return compiler.compile_settings(settings(name, CAP_40 if capped else ()), config())


def _fewer_apples(rows):
  """The open map without the apples of its right half, plus three apples moved to the middle of the empty row 12."""
  out = [r[:12] + r[12:].replace('A', ' ') if 0 < i < len(rows) - 1 else r for i, r in enumerate(rows)]
  out[12] = out[12][:10] + 'AAA' + out[12][13:]
  return out


FEWER_APPLES = V.map_rows(_fewer_apples)


@functools.lru_cache(maxsize=None)
def apple_set():
  """The capped open map and a copy of it with apples removed and moved, compiled as one set: the maps differ in their
  apple count (nA) and regrowth discs (ch_nbr)."""
  return compile_set([settings(NAMES[0], CAP_40), settings(NAMES[0], CAP_40 + (FEWER_APPLES,))])


@functools.lru_cache(maxsize=None)
def beam_set():
  """The capped open map under three Zapper footprints (beamLength 3 radius 1, 4 / 1, 2 / 2): variants that differ only
  in the zap beam, as prefab_overrides on Zapper.beamLength / beamRadius give them."""
  shapes = ((3, 1), (4, 1), (2, 2))
  return tuple(compiler.compile_settings(settings(NAMES[0], CAP_40 + (V.kw('Zapper', beamLength=l, beamRadius=r),)), config())
               for l, r in shapes)
