"""TEST INFRASTRUCTURE: a stored set of coins draws (tests/golden/settings_coins_draws__2p.json.gz).

coins' config builder draws a map size and an ordered pair of coin colours on every build. The fixture holds the lab2d
settings the reference builder returned for sixteen build seeds (tools/make_coins_draws_golden.py), covering the
smallest and the largest map and eleven colour pairs, five in both orders. Everything here compiles from those
settings, so no reference checkout is needed.
"""

import functools
import gzip
import json
import os
import types

from meltingpot_b200 import compiler
from tests import variants as V

PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), 'golden', 'settings_coins_draws__2p.json.gz')
# the 40-frame episode cap of the GPU tests: every rollout of more than 40 steps crosses an auto-reset
CAP_40 = (V.kw('StochasticIntervalEpisodeEnding', probabilityTerminationPerInterval=0.0), V.top(maxEpisodeLengthFrames=40))


@functools.lru_cache(maxsize=None)
def _record():
  with gzip.open(PATH, 'rt') as f:
    return json.load(f)


def seeds():
  return tuple(_record()['seeds'])


def config():
  return types.SimpleNamespace(**_record()['config'])


def settings(seed, edits=()):
  """A fresh copy of the settings of draw `seed`, with `edits` (settings -> None) applied."""
  s = json.loads(json.dumps(_record()['settings'][str(seed)]))
  for edit in edits:
    edit(s)
  return s


@functools.lru_cache(maxsize=None)
def draw_set(capped=True, draw_seeds=None):
  """The blobs of the stored draws (or of `draw_seeds`) compiled as one draw set, optionally with the 40-frame cap."""
  chosen = seeds() if draw_seeds is None else tuple(draw_seeds)
  edits = CAP_40 if capped else ()
  return tuple(compiler.compile_settings_set([settings(s, edits) for s in chosen], config(), list(chosen)))


@functools.lru_cache(maxsize=None)
def alone(seed, capped=True):
  """The blob of draw `seed` compiled on its own (what compile_substrate gives for that build seed)."""
  return compiler.compile_settings(settings(seed, CAP_40 if capped else ()), config(), seed)
