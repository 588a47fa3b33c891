"""TEST INFRASTRUCTURE: per-env parameter variants (heterogeneous batches) of the five kernel families.

Each family gets four variants of its stored lab2d settings (tests/golden/settings_*.json.gz), compiled at test time
as tests/variants.py does, so no reference checkout is needed: the stock parameters, two sets of `prefab_overrides` on
map pieces (applied with compiler.apply_prefab_overrides, as the reference builder applies them) and one avatar-level
knob (set with variants.set_kwargs: the reference's overrides do not reach avatars). All four share a 40-frame episode
cap, so that every rollout of more than 40 steps crosses an auto-reset.
"""

import functools

import numpy as np

from meltingpot_b200 import compiler
from tests import settings_golden
from tests import variants as V

_CAP_40 = [V.kw('StochasticIntervalEpisodeEnding', probabilityTerminationPerInterval=0.0), V.top(maxEpisodeLengthFrames=40)]

# family -> (substrate, players, settings seed, [(prefab_overrides, avatar-level edits)] for variants 0..3)
FAMILIES = {
    'clean_up': ('clean_up', 7, None, [
        ({}, []),
        ({'potential_apple': {'AppleGrow': {'maxAppleGrowthRate': 1.0, 'thresholdDepletion': 0.9, 'thresholdRestoration': 0.0}}}, []),
        ({'potential_apple': {'Edible': {'rewardForEating': 4.0},
                              'AppleGrow': {'maxAppleGrowthRate': 0.5, 'thresholdDepletion': 0.9, 'thresholdRestoration': 0.0}}}, []),
        ({}, [V.kw('Zapper', cooldownTime=1, penaltyForBeingZapped=-2.0)]),
    ]),
    'commons_harvest': ('commons_harvest__open', 7, None, [
        ({}, []),
        ({'apple': {'DensityRegrow': {'regrowthProbabilities': [0.0, 0.5, 0.8, 1.0]}}}, []),
        ({'apple': {'Edible': {'rewardForEating': 2.5}, 'DensityRegrow': {'regrowthProbabilities': [0.0, 0.2, 0.4, 0.6]}}}, []),
        ({}, [V.kw('Zapper', cooldownTime=1, rewardForZapping=0.5)]),
    ]),
    'territory': ('territory__rooms', 9, None, [
        ({}, []),
        ({'resource': {'Resource': {'initialHealth': 1}}}, []),
        ({'resource': {'Resource': {'rewardDelay': 0, 'reward': 0.5, 'rewardRate': 1.0, 'selfRepairProbability': 1.0}}}, []),
        ({}, [V.kw('ResourceClaimer', beamWait=5)]),
    ]),
    'coins': ('coins', 2, 0, [
        ({}, []),
        ({'coin': {'ChoiceCoinRegrow': {'regrowRate': 1.0}}}, []),
        ({'coin': {'Coin': {'rewardSelfForMatch': 2.0, 'rewardOtherForMismatch': -3.0}, 'ChoiceCoinRegrow': {'regrowRate': 0.5}}}, []),
        ({'coin': {'ChoiceCoinRegrow': {'regrowRate': 1.0}}},
         [V.kw('Role', multiplyRewardSelfForMatch=3.0, multiplyRewardSelfForMismatch=3.0, multiplyRewardOtherForMatch=3.0,
               multiplyRewardOtherForMismatch=3.0)]),
    ]),
    'coop_mining': ('coop_mining', 6, None, [
        ({}, []),
        ({'ore': {'FixedRateRegrow': {'liveRates': [1.0, 1.0]}}}, []),
        ({'ore': {'Ore': {'miningWindow': 3}, 'FixedRateRegrow': {'liveRates': [0.5, 0.5]}}}, []),
        ({}, [V.kw('MineBeam', cooldownTime=1)]),
    ]),
}
NAMES = tuple(FAMILIES)


def settings(family, edits=()):
  """The family's stored settings with the 40-frame cap and `edits` (settings -> None) applied."""
  sub, players, seed, _ = FAMILIES[family]
  s = settings_golden.settings(sub, players, seed)
  for edit in list(_CAP_40) + list(edits):
    edit(s)
  return s


def compile_settings(family, s, prefab_overrides=None):
  sub, players, seed, _ = FAMILIES[family]
  return compiler.compile_settings(s, settings_golden.config(sub, players), seed, prefab_overrides)


@functools.lru_cache(maxsize=None)
def blobs(family):
  """The family's four variant blobs, in order."""
  return tuple(compile_settings(family, settings(family, edits), overrides) for overrides, edits in FAMILIES[family][3])


@functools.lru_cache(maxsize=None)
def stock(family):
  """The stock blob of the family's substrate (no cap, no override)."""
  sub, players, seed, _ = FAMILIES[family]
  return settings_golden.compile(sub, players, seed)


def blocks(num_envs, n):
  """Variant of each env in n contiguous blocks."""
  return (np.arange(num_envs) * n // num_envs).astype(np.int64)


def interleaved(num_envs, n):
  """Variant of each env cycling per env, so the four env warps of a CTA run different variants."""
  return (np.arange(num_envs) % n).astype(np.int64)


def differing_sections(a, b):
  """Names of the blob sections that differ between two blobs."""
  from meltingpot_b200 import blob as blob_lib
  sa, sb = blob_lib.unpack(a), blob_lib.unpack(b)
  out = sorted(k for k in set(sa) ^ set(sb))
  for k in set(sa) & set(sb):
    x, y = sa[k], sb[k]
    same = (np.array_equal(x, y) and x.dtype == y.dtype) if isinstance(x, np.ndarray) else x == y
    if not same:
      out.append(k)
  return sorted(set(out))
