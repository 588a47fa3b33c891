"""TEST INFRASTRUCTURE: appearance overrides (prefab_overrides of an `Appearance` component) of the five kernel families.

Each substrate gets four variants of its stored lab2d settings (tests/golden/settings_*.json.gz), all under the 40-frame
cap of tests/env_variants.py: the stock settings, a recoloured map piece, a reshaped map piece, and a recolour combined
with a knob override. The overrides are derived from the stored Appearance kwargs (every colour moved, every shape
rolled by a row), compiled as one set on one sprite table (compiler.compile_settings_set), so no reference checkout is needed.
"""

import copy
import functools

from meltingpot_b200 import compiler
from tests import env_variants as EV
from tests import settings_golden

# substrate -> (players, settings seed, recoloured prefabs, reshaped prefabs, (recoloured prefabs, knob override))
SUBSTRATES = {
    'clean_up': (7, None, ['potential_dirt', 'actual_dirt'], ['river'],
                 (['potential_apple'], {'potential_apple': {'AppleGrow': {'maxAppleGrowthRate': 1.0, 'thresholdDepletion': 0.9,
                                                                          'thresholdRestoration': 0.0}}})),
    'commons_harvest__open': (7, None, ['apple'], ['grass'],
                              (['apple'], {'apple': {'Edible': {'rewardForEating': 2.5}}})),
    'territory__rooms': (9, None, ['resource'], ['resource_texture'],
                         (['reward_indicator', 'damage_indicator'], {'resource': {'Resource': {'initialHealth': 1}}})),
    'territory__inside_out': (5, None, ['resource'], ['resource_texture'],
                              (['reward_indicator'], {'resource': {'Resource': {'rewardDelay': 0, 'reward': 0.5}}})),
    'coins': (2, 0, ['coin'], ['wall'], (['coin'], {'coin': {'ChoiceCoinRegrow': {'regrowRate': 1.0}}})),
    'coop_mining': (6, None, ['ore'], ['ore'], (['wall'], {'ore': {'FixedRateRegrow': {'liveRates': [1.0, 1.0]}}})),
}
NAMES = tuple(SUBSTRATES)


def _recolour(color):
  c = list(color)
  return [(c[0] + 97) % 256, (c[1] + 41) % 256, c[2]] + c[3:]


def _roll(shape):
  if isinstance(shape, (list, tuple)):  # four explicit facings
    return [_roll(s) for s in shape]
  rows = shape.strip('\n').split('\n')
  return '\n'.join(rows[-1:] + rows[:-1])


def appearance(s, prefab):
  """The kwargs of the first Appearance component of `prefab` in settings `s`."""
  return next(c['kwargs'] for c in s['simulation']['prefabs'][prefab]['components'] if c['component'] == 'Appearance')


def recoloured(s, prefab):
  """{'Appearance': {...}}: every colour of the prefab's sprites moved (palette entries or square colours)."""
  kw = appearance(s, prefab)
  if kw.get('renderMode') == 'ascii_shape':
    return {'Appearance': {'palettes': [{k: (_recolour(v) if len(v) < 4 or v[3] else v) for k, v in p.items()}
                                        for p in kw['palettes']]}}
  return {'Appearance': {'spriteRGBColors': [_recolour(c) for c in kw['spriteRGBColors']]}}


def reshaped(s, prefab):
  """{'Appearance': {...}}: every sprite shape of the prefab moved down one row (the bottom row wraps to the top)."""
  return {'Appearance': {'spriteShapes': [_roll(x) for x in appearance(s, prefab)['spriteShapes']]}}


def merge(*overrides):
  out = {}
  for o in overrides:
    for prefab, comps in o.items():
      for comp, kw in comps.items():
        out.setdefault(prefab, {}).setdefault(comp, {}).update(copy.deepcopy(kw))
  return out


def settings(name):
  players, seed = SUBSTRATES[name][:2]
  s = settings_golden.settings(name, players, seed)
  for edit in EV._CAP_40:  # pylint: disable=protected-access
    edit(s)
  return s


def config(name):
  return settings_golden.config(name, SUBSTRATES[name][0])


def overrides(name):
  """The four prefab_overrides of `name`: stock, recolour, reshape, recolour + knob."""
  s = settings(name)
  _, _, colour, shape, (colour2, knob) = SUBSTRATES[name]
  return [
      {},
      merge(*[{p: recoloured(s, p)} for p in colour]),
      merge(*[{p: reshaped(s, p)} for p in shape]),
      merge(knob, *[{p: recoloured(s, p)} for p in colour2]),
  ]


@functools.lru_cache(maxsize=None)
def blobs(name):
  """The four variant blobs of `name`, compiled as one set."""
  seed = SUBSTRATES[name][1]
  o = overrides(name)
  return tuple(compiler.compile_settings_set([settings(name)] * len(o), config(name), [seed] * len(o), o))


@functools.lru_cache(maxsize=None)
def alone(name):
  """Each variant compiled on its own (compile_settings), with its own sprite table."""
  seed = SUBSTRATES[name][1]
  return tuple(compiler.compile_settings(settings(name), config(name), seed, o) for o in overrides(name))
