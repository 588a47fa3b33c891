"""Substrate compiler: reference lab2d settings dict -> flat numeric tables (MPB blob).

Replaces, for the hot path only, what the reference does at build time:
  * `builder.builder` (`meltingpot/utils/substrates/builder.py:142-192`)
    flattens the settings for Lua; we flatten them into tables instead.
  * `BaseSimulation.__init__` / `prefab_utils.buildGameObjectConfigs` walk the ASCII
    map row-major and instantiate prefabs
    (`meltingpot/lua/modules/base_simulation.lua:102-134`,
    `prefab_utils.lua:92-109,163-176`): object creation order = scene, configured
    game objects (avatars), then map objects row-major.
  * `BaseSimulation:worldConfig` (`base_simulation.lua:253-320`) builds layers
    (render order), states, hits; `_addShapesToTileSet`
    (`component_library.lua:567-597`) builds sprites.

The compiler CONSUMES the reference configs as data (imported from a reference
checkout when available); compiled blobs for the supported substrates are
committed under `meltingpot_b200/data/` so that running them needs no reference
checkout.
"""

from __future__ import annotations

import collections
import copy
import json
import os
import random
import sys
import types
from typing import Any, Dict, List, Mapping, Optional, Sequence

import numpy as np

from meltingpot_b200 import blob as blob_lib

# ---------------------------------------------------------------------------
# Enumerations mirrored from include/mpb_format.h
# ---------------------------------------------------------------------------
META = dict(FAMILY=0, W=1, H=2, L=3, P=4, SPRITE_SIZE=5, TOPOLOGY=6,
            MAX_FRAMES=7, N_OBJECTS=8, N_KINDS=9, N_STATES=10, N_COMPS=11,
            N_SPRITES=12, N_HITS=13, N_GROUPS=14, VIEW_LEFT=15, VIEW_RIGHT=16,
            VIEW_FORWARD=17, VIEW_BACKWARD=18, N_ACTIONS=19,
            N_ACTION_FIELDS=20, OOB_SPRITE=21, OOV_SPRITE=22, N_SCALAR_OBS=23)
META_COUNT = 32
FAMILY = {'clean_up': 1, 'commons_harvest': 2, 'territory': 3, 'coins': 4,
          'coop_mining': 5}
COMP = dict(StateManager=1, Transform=2, Appearance=3, BeamBlocker=4, Edible=5,
            AppleGrow=6, DirtTracker=7, DirtCleaning=8, Avatar=9, Zapper=10,
            ReadyToShootObservation=11, Cleaner=12, Taste=13,
            AllNonselfCumulants=14, AvatarMetricReporter=15, RiverMonitor=16,
            DirtSpawner=17, StochasticIntervalEpisodeEnding=18, GlobalData=19,
            Animation=20, AdditionalSprites=21, Neighborhoods=22,
            DensityRegrow=23, LocationObserver=24, AllBeamBlocker=25,
            Resource=26, ResourceClaimer=27, RewardIndicator=28, Paintbrush=29,
            GraduatedSanctionsMarking=30, TerritoryTaste=31, Role=32,
            RoleBasedRewardTile=33, Coin=34, ChoiceCoinRegrow=35,
            GlobalCoinCollectionTracker=36, PlayerCoinType=37, CoinsRole=38,
            PartnerTracker=39, FixedRateRegrow=40, Ore=41, MineBeam=42,
            MiningTracker=43)
COMP_NI, COMP_ND = 16, 6
ACTION_FIELDS = {'move': 0, 'turn': 1, 'fireZap': 2, 'mine': 2, 'fireClean': 3,
                 'fireClaim': 3}
SCALAR_OBS = {'READY_TO_SHOOT': 0, 'NUM_OTHERS_WHO_CLEANED_THIS_STEP': 1,
              'MISMATCHED_COIN_COLLECTED_BY_PARTNER': 2}
# Family parameter blocks: MPB_FP_* (shared by the int32 blocks of clean_up, commons_harvest and territory) and
# MPB_<CU|CH|TR|CO|CM>_<I|D>_*; COUNT is the block's size.
FP = dict(ZAP_COOLDOWN=12, ZAP_LENGTH=13, ZAP_RADIUS=14, ZAP_RESPAWN=15, ZAP_REMOVE=16, ZAP_LAYER=21, ZAP_SPRITE=22,
          END_MIN_FRAMES=26, END_INTERVAL=27)
CU_I = dict(N_APPLES=0, N_DIRT=1, N_WATER=2, APPLE_LAYER=3, APPLE_SPRITE=4, DIRT_LAYER=5, DIRT_SPRITE=6,
            DIRT_WAIT_LAYER=7, WATER_LAYER=8, N_ANIM=9, ANIM_FRAMES=10, ANIM_RANDOM=11, CLEAN_COOLDOWN=18,
            CLEAN_LENGTH=19, CLEAN_RADIUS=20, CLEAN_LAYER=23, CLEAN_SPRITE=24, DIRT_DELAY=25, TASTE_ROLE=28, COUNT=48)
CU_D = dict(GROW_RATE=0, GROW_DEPLETION=1, GROW_RESTORATION=2, EAT_REWARD=3, ZAP_PENALTY=4, ZAP_REWARD=5,
            DIRT_PROB=6, END_PROB=7, TASTE_AMOUNT=8, COUNT=16)
CH_I = dict(N_APPLES=0, APPLE_LAYER=1, APPLE_SPRITE=2, WAIT_LAYER=3, WAIT_SPRITE=4, N_WAIT=5, N_PROBS=6,
            GRASS_LAYER=7, GRASS_SPRITE=8, DESS_SPRITE=9, COUNT=48)
CH_D = dict(PROB_0=0, PROB_1=1, PROB_2=2, PROB_3=3, EAT_REWARD=4, ZAP_PENALTY=5, ZAP_REWARD=6, END_PROB=7, COUNT=16)
TR_I = dict(N_RES=0, RES_LAYER=1, UNCLAIMED_SPRITE=2, TEX_LAYER=3, TEX_SPRITE=4, IND_LAYER=5, DMG_LAYER=6,
            DMG_SPRITE=7, MARK_LAYER=8, MARK_INITIAL_LEVEL=9, MARK_RECOVERY=10, MARK_N_LEVELS=11, CLAIM_LENGTH=18,
            CLAIM_RADIUS=19, CLAIM_WAIT=20, BRUSH_LAYER=23, CLAIM_LAYER=24, RES_HEALTH=28, RES_REWARD_DELAY=29,
            RES_REPAIR_DELAY=30, TASTE_ROLE=31, COUNT=64,
            **{f'MARK_{f}_{l}': 32 + 4 * l + k for l in range(3)
               for k, f in enumerate(('INC', 'REMOVE', 'FREEZE', 'SPRITE'))})
TR_D = dict(RES_REWARD=0, RES_RATE=1, RES_REPAIR_PROB=2, ZAP_PENALTY=3, ZAP_REWARD=4, END_PROB=5, TASTE_AMOUNT=6,
            TASTE_MULT=7, COUNT=16,
            **{f'MARK_{f}_REWARD_{l}': 8 + 2 * l + k for l in range(3) for k, f in enumerate(('SRC', 'TGT'))})
CO_I = dict(N_COINS=0, COIN_LAYER=1, COIN_SPRITE_0=2, COIN_SPRITE_1=3, TERMINATE=4, TERMINATE_N=5,
            END_MIN_FRAMES=6, END_INTERVAL=7, COIN_TYPE_0=8, COIN_TYPE_1=9, COUNT=48)
_COIN_REWARDS = ('SELF_MATCH', 'SELF_MISMATCH', 'OTHER_MATCH', 'OTHER_MISMATCH')
CO_D = dict(REGROW_RATE=0, END_PROB=1, COUNT=16,
            **{f'REWARD_{p}_{r}': 4 + 4 * p + k for p in range(2) for k, r in enumerate(_COIN_REWARDS)})
CM_I = dict(N_ORES=0, ORE_LAYER=1, ORE_SPRITE_0=2, ORE_SPRITE_1=3, ORE_SPRITE_2=4, ORE_SPRITE_3=5, MINE_WINDOW=6,
            MINE_COOLDOWN=7, MINE_LENGTH=8, MINE_LAYER=9, MINE_SPRITE=10, END_MIN_FRAMES=11, END_INTERVAL=12,
            MINE_HIT=13, COUNT=48)
CM_D = dict(RATE_0=0, RATE_1=1, END_PROB=2, MINE_REWARD_0=4, MINE_REWARD_1=5, EXTRACT_REWARD_0=6,
            EXTRACT_REWARD_1=7, COUNT=16)
# family -> (section prefix, int32 block layout, f64 block layout)
FAMILY_PARAMS = {'clean_up': ('cu', {**FP, **CU_I}, CU_D), 'commons_harvest': ('ch', {**FP, **CH_I}, CH_D),
                 'territory': ('tr', {**FP, **TR_I}, TR_D), 'coins': ('co', CO_I, CO_D),
                 'coop_mining': ('cm', CM_I, CM_D)}
COMPASS = {'N': 0, 'E': 1, 'S': 2, 'W': 3}
BASE_LAYERS = ['logic', 'alternateLogic', 'background', 'lowerPhysical',
               'upperPhysical', 'overlay', 'superOverlay']
_TASTE_ROLES = {'free': 0, 'cleaner': 1, 'consumer': 2}
_TERRITORY_TASTE_ROLES = {'none': 0, 'rewarded_per_claim': 1, 'rewarded_per_claim_only': 2}
_HIT_OF = {'Zapper': ('zapHit', 'beamZap', 'BeamZap'),
           'Cleaner': ('cleanHit', 'beamClean', 'BeamClean'),
           'MineBeam': ('mine', 'beamMine', 'beamMine')}  # coop_mining/components.lua:191-201


# ---------------------------------------------------------------------------
# Loading reference configs without executing meltingpot/__init__.py
# ---------------------------------------------------------------------------
def reference_root() -> Optional[str]:
  """The Melting Pot checkout to compile from: ONLY the one named by MELTINGPOT_REFERENCE_ROOT.

  Compiling imports and executes the checkout's config modules, so no location is ever guessed: without the
  variable (or an explicit `root` argument) there is no reference, and `substrates.load_blob` serves committed
  blobs only.
  """
  cand = os.environ.get('MELTINGPOT_REFERENCE_ROOT')
  if cand and os.path.isdir(os.path.join(cand, 'meltingpot', 'configs')):
    return cand
  return None


import contextlib  # pylint: disable=g-import-not-at-top,g-bad-import-order


@contextlib.contextmanager
def reference_packages(root: Optional[str] = None):
  """Temporarily makes `meltingpot.*` import from a reference checkout, without running its package __init__.

  The reference's `meltingpot/__init__.py` pulls in dmlab2d / chex / reactivex (absent here;
  `meltingpot/__init__.py:18`), so namespace stubs stand in for the parent packages. Whatever
  `meltingpot*` modules were loaded before (this repo's own `meltingpot` alias package, or a real dm-meltingpot
  install) are put back on exit and every module imported from the checkout is dropped again, so the process is
  not left with shadowing stubs.
  """
  from meltingpot_b200 import shims  # pylint: disable=g-import-not-at-top
  shims.install()
  root = root or reference_root()
  if root is None:
    raise FileNotFoundError('no Melting Pot reference checkout: set MELTINGPOT_REFERENCE_ROOT (nothing is guessed)')
  base = os.path.join(root, 'meltingpot')
  mine = lambda k: k == 'meltingpot' or k.startswith('meltingpot.')
  saved = {k: v for k, v in sys.modules.items() if mine(k)}
  for k in saved:
    del sys.modules[k]
  try:
    for name, path in (('meltingpot', base), ('meltingpot.utils', os.path.join(base, 'utils')),
                       ('meltingpot.utils.substrates', os.path.join(base, 'utils', 'substrates')),
                       ('meltingpot.utils.substrates.wrappers', os.path.join(base, 'utils', 'substrates', 'wrappers')),
                       ('meltingpot.configs', os.path.join(base, 'configs'))):
      module = types.ModuleType(name)
      module.__path__ = [path]
      sys.modules[name] = module
    yield base
  finally:
    for k in [k for k in sys.modules if mine(k)]:
      del sys.modules[k]
    sys.modules.update(saved)


def load_reference_config(name: str, root: Optional[str] = None):
  """Imports `meltingpot.configs.substrates.<name>` from a reference checkout and returns its config."""
  import importlib  # pylint: disable=g-import-not-at-top
  with reference_packages(root):
    configs = importlib.import_module('meltingpot.configs.substrates')
    return configs.get_config(name)


def _plain(value: Any) -> Any:
  """ConfigDict / tuples -> plain dict / list, recursively."""
  if hasattr(value, 'to_dict') and not isinstance(value, dict):
    value = value.to_dict()
  if isinstance(value, Mapping):
    return {k: _plain(v) for k, v in value.items()}
  if isinstance(value, (list, tuple)):
    return [_plain(v) for v in value]
  return value


# ---------------------------------------------------------------------------
# Sprites
# ---------------------------------------------------------------------------
def _rgba(color: Sequence[int]) -> List[int]:
  color = [int(c) for c in color]
  if len(color) == 3:
    color.append(255)
  return color


def text_to_image(text: str, palette: Mapping[str, Sequence[int]]) -> np.ndarray:
  """ASCII shape + palette -> uint8 [h, w, 4] (component_library.lua:567-597)."""
  # Lines are trimmed: territory.py:512-521 indents its sprite text.
  rows = [r.strip() for r in text.strip().split('\n')]
  rows = [r for r in rows if r]
  h, w = len(rows), len(rows[0])
  img = np.zeros((h, w, 4), np.uint8)
  for y, row in enumerate(rows):
    if len(row) != w:
      raise ValueError('ragged sprite text')
    for x, ch in enumerate(row):
      if ch not in palette:
        raise KeyError(f'palette has no entry for {ch!r}')
      img[y, x] = _rgba(palette[ch])
  return img


def downscale_box(img: np.ndarray, size: int) -> np.ndarray:
  """Integer box average with round-half-up (policy A.15; parity unpinned)."""
  h, w, _ = img.shape
  if h == size and w == size:
    return img
  if h % size or w % size:
    raise ValueError(f'cannot box-scale {h}x{w} to {size}')
  fy, fx = h // size, w // size
  acc = img.astype(np.uint32).reshape(size, fy, size, fx, 4).sum(axis=(1, 3))
  n = fy * fx
  return ((acc * 2 + n) // (2 * n)).astype(np.uint8)


def four_facings(img: np.ndarray, no_rotate: bool) -> np.ndarray:
  """[4, s, s, 4]: facing N, E, S, W. Rotating sprites turn clockwise (A.12)."""
  if no_rotate:
    return np.stack([img] * 4)
  return np.stack([np.rot90(img, k=-k) for k in range(4)])


class SpriteSet:
  """Name -> [4, s, s, 4] images, in first-registration order."""

  def __init__(self, size: int):
    self.size = size
    self.names: List[str] = []
    self.images: Dict[str, np.ndarray] = {}

  def _ensure(self, name: str) -> None:
    if name not in self.images:
      self.names.append(name)
      self.images[name] = np.zeros((4, self.size, self.size, 4), np.uint8)

  def add_color(self, name: str, color: Sequence[int]) -> None:
    self._ensure(name)
    self.images[name][:] = np.array(_rgba(color), np.uint8)

  def add_shape(self, name: str, text, palette, no_rotate: bool) -> None:
    if isinstance(text, (list, tuple)) and len(text) == 4:
      if not no_rotate:
        raise ValueError('explicit 4-facing sprites need noRotate=True')
      self._ensure(name)
      for k in range(4):
        img = downscale_box(text_to_image(text[k], palette), self.size)
        self.images[name][k] = img
      return
    img = downscale_box(text_to_image(text, palette), self.size)
    self._ensure(name)
    self.images[name][:] = four_facings(img, bool(no_rotate))

  def add_from_appearance(self, kw: Mapping[str, Any], prefix: str = 'sprite'):
    mode = kw.get('renderMode', 'colored_square')
    names = kw.get(prefix + 'Names', [])
    key = lambda s: ('custom' + s[0].upper() + s[1:]) if prefix == 'customSprite' else s
    if prefix == 'customSprite':
      colors = kw.get('customSpriteRGBColors', [])
      shapes = kw.get('customSpriteShapes', [])
      palettes = kw.get('customPalettes', [])
      no_rot = kw.get('customNoRotates', [])
    else:
      colors = kw.get('spriteRGBColors', [])
      shapes = kw.get('spriteShapes', [])
      palettes = kw.get('palettes', [])
      no_rot = kw.get('noRotates', [])
    del key
    for i, name in enumerate(names):
      if mode == 'colored_square':
        self.add_color(name, colors[i])
      elif mode == 'ascii_shape':
        self.add_shape(name, shapes[i], palettes[i],
                       bool(no_rot[i]) if i < len(no_rot) else False)
      elif mode == 'invisible':
        pass
      else:
        raise ValueError(mode)

  def index(self, name: str) -> int:
    return self.names.index(name)

  def atlas(self) -> np.ndarray:
    return np.stack([self.images[n] for n in self.names])


class SharedSprites:
  """The one sprite table of a draw set (compile_settings_set): every entry's sprites, deduplicated by name and pixels,
  in first-appearance order. Two entries may register one name with different pixels (coins' avatars take the palette
  of their draw's coin colours); each pair is a sprite of its own. `view(sprites)` is the table as one entry sees it."""

  def __init__(self, size: int):
    self.size = size
    self.names: List[str] = []
    self._images: List[np.ndarray] = []

  def _find(self, name: str, image: np.ndarray) -> int:
    for i, (n, img) in enumerate(zip(self.names, self._images)):
      if n == name and np.array_equal(img, image):
        return i
    return -1

  def add(self, sprites: SpriteSet) -> None:
    for name in sprites.names:
      if self._find(name, sprites.images[name]) < 0:
        self.names.append(name)
        self._images.append(sprites.images[name])

  def view(self, sprites: SpriteSet) -> 'SpriteView':
    return SpriteView(self, {name: self._find(name, sprites.images[name]) for name in sprites.names})

  def atlas(self) -> np.ndarray:
    return np.stack(self._images)


class SpriteView:
  """A SharedSprites table indexed by the sprite names of one entry of the set."""

  def __init__(self, shared: SharedSprites, ids: Mapping[str, int]):
    self.size = shared.size
    self.names = shared.names
    self._shared = shared
    self._ids = ids

  def index(self, name: str) -> int:
    return self._ids[name]

  def atlas(self) -> np.ndarray:
    return self._shared.atlas()


# ---------------------------------------------------------------------------
# World model
# ---------------------------------------------------------------------------
def _first(components, name):
  for c in components:
    if c['component'] == name:
      return c
  return None


def _map_rows(ascii_map: str) -> List[str]:
  # prefab_utils.lua:92-109 strips leading newlines only; a trailing newline
  # terminates the last row.
  text = ascii_map.lstrip('\n')
  rows = text.split('\n')
  while rows and rows[-1] == '':
    rows.pop()
  return rows


def _flatten_option(spec) -> List[str]:
  """Prefab names of one option of a 'choice' ('all' lists are expanded; a nested 'choice' is refused)."""
  if isinstance(spec, Mapping):
    if spec['type'] != 'all':
      raise NotImplementedError("a 'choice' prefab nested inside a 'choice'")
    out: List[str] = []
    for p in spec['list']:
      out += _flatten_option(p)
    return out
  return [spec]


def _expand_prefab(spec, prefabs, out, x, y, rng, choices=None):
  """prefab_utils.lua:44-72 (_createPrefabsFromSpec): a name, or {'type': 'all' | 'choice', 'list': [...]}.

  The reference draws a 'choice' with the env's own random stream when the env is built -- i.e. for every env
  instance and, because the ResetWrapper rebuilds the env, for every episode. Without a build seed the draw is left
  to the engine: the prefabs common to all options are emitted as usual, the others become CONDITIONAL objects
  tagged (choice group, bit mask of the tickets 0..n_options-1 on which they exist); every env draws one ticket per
  group at each episode start (kernels and oracle alike). `out` entries are (prefab, x, y, condition or None).
  With a build seed (`rng`) one draw is fixed at compile time for all envs (the old behaviour, policy A.20).
  """
  if isinstance(spec, Mapping):
    if spec['type'] == 'all':
      for p in spec['list']:
        _expand_prefab(p, prefabs, out, x, y, rng, choices)
    elif spec['type'] == 'choice':
      options = list(spec['list'])
      if rng is not None:
        _expand_prefab(options[rng.randrange(len(options))], prefabs, out, x, y, rng, choices)
        return
      if choices is None or len(options) > 31:
        raise NotImplementedError("charPrefabMap type 'choice' with more than 31 options")
      flat = [_flatten_option(o) for o in options]
      common = list(flat[0])
      for f in flat[1:]:
        rest = list(f)
        kept = []
        for name in common:
          if name in rest:
            rest.remove(name)
            kept.append(name)
        common = kept
      for name in common:
        _expand_prefab(name, prefabs, out, x, y, rng, choices)
      group = len(choices)
      choices.append(len(options))
      extras: Dict[str, int] = {}  # prefab name (with multiplicity index) -> ticket mask
      for t, f in enumerate(flat):
        rest = list(f)
        for name in common:
          rest.remove(name)
        seen: Dict[str, int] = {}
        for name in rest:
          k = seen.get(name, 0)
          seen[name] = k + 1
          extras[(name, k)] = extras.get((name, k), 0) | (1 << t)
      for (name, _), mask in extras.items():
        if name not in prefabs:
          raise KeyError(f"Prefab with name '{name}' not found in prefabs.")
        out.append((prefabs[name], x, y, (group, mask)))
    else:
      raise NotImplementedError(f"charPrefabMap type {spec['type']!r} is not supported by the CUDA engine")
  else:
    if spec not in prefabs:
      raise KeyError(f"Prefab with name '{spec}' not found in prefabs.")
    out.append((prefabs[spec], x, y, None))


class WorldModel:
  """Everything the engines need, as python lists prior to packing."""

  def __init__(self, settings: Mapping[str, Any], build_seed: Optional[int] = None,
               shared_sprites: Optional[SharedSprites] = None):
    s = _plain(settings)
    sim = s['simulation']
    self.level = s['levelName']
    fam = self.level
    for key in FAMILY:
      if fam.startswith(key):
        fam = key
    if fam not in FAMILY:
      raise NotImplementedError(f'substrate family {self.level!r} is not '
                                'supported by the CUDA engine')
    self.family = fam
    self.num_players = int(s['numPlayers'])
    self.sprite_size = int(s.get('spriteSize', 8))
    self.topology = {'BOUNDED': 0, 'TORUS': 1}[s.get('topology', 'BOUNDED')]
    self.max_frames = int(s.get('maxEpisodeLengthFrames', 3600))
    rows = _map_rows(sim['map'])
    self.H, self.W = len(rows), max(len(r) for r in rows)

    # ---- objects in creation order (base_simulation.lua:102-134) ----------
    objs = []  # (config, x, y)
    if sim.get('scene') is not None:
      objs.append((sim['scene'], 0, 0, None))
    for go in sim.get('gameObjects', []):
      objs.append((go, 0, 0, None))
    cpm = {str(k): v for k, v in sim['charPrefabMap'].items()}
    rng = random.Random(build_seed) if build_seed is not None else None
    self.choice_options: List[int] = []   # options per 'choice' group (drawn per env and episode by the engine)
    for y, row in enumerate(rows):
      for x, ch in enumerate(row):
        if ch in cpm:
          _expand_prefab(cpm[ch], sim['prefabs'], objs, x, y, rng, self.choice_options)
    self.objects_cfg = objs
    self._prefabs = sim.get('prefabs', {})
    self.avatar_roles = set()
    self.rewarded_roles = set()

    # ---- layers, hits (base_simulation.lua:263-271; addHits) ---------------
    self.layers = list(BASE_LAYERS)
    self.hits: List[tuple] = []  # (name, layer, sprite)
    def add_hit(hit, layer, sprite, insert_layer):
      if hit not in [h[0] for h in self.hits]:
        self.hits.append((hit, layer, sprite))
      if insert_layer and layer not in self.layers:
        self.layers.append(layer)
    for cfg, _, _, _ in objs:
      for c in cfg['components']:
        kw = c.get('kwargs', {}) or {}
        if c['component'] in _HIT_OF:
          hit, layer, sprite = _HIT_OF[c['component']]
          add_hit(hit, layer, sprite, True)
        elif c['component'] == 'ResourceClaimer':  # territory/components.lua:241-246
          i = int(kw['playerIndex'])
          add_hit(f'claimBeam_{i}', 'superDirectionIndicatorLayer', f'claimBeamSprite_{i}', False)
        elif c['component'] == 'Paintbrush':       # territory/components.lua:387-396
          i = int(kw['playerIndex'])
          add_hit(f'directionHit{i}', 'directionIndicatorLayer', f'brush{i}', False)
    if self.family == 'territory':
      # lua/levels/territory/init.lua:30-37 appends two render layers after BaseSimulation's own
      # (which by then include the hit layers added by Zapper:addHits).
      self.layers += ['directionIndicatorLayer', 'superDirectionIndicatorLayer']

    # ---- sprites (base_simulation.lua:322-329) -----------------------------
    sp = SpriteSet(self.sprite_size)
    sp.add_color('OutOfBounds', (0, 0, 0))
    sp.add_color('OutOfView', (80, 80, 80))
    for cfg, _, _, _ in objs:
      for c in cfg['components']:
        kw = c.get('kwargs', {}) or {}
        if c['component'] == 'Appearance':
          sp.add_from_appearance(kw)
        elif c['component'] == 'AdditionalSprites':
          sp.add_from_appearance(kw, prefix='customSprite')
        elif c['component'] == 'Zapper':
          sp.add_color('BeamZap', kw.get('beamColor', (252, 252, 106)))
        elif c['component'] == 'Cleaner':
          sp.add_color('BeamClean', (99, 223, 242, 175))
        elif c['component'] == 'MineBeam':
          sp.add_color('beamMine', (255, 202, 202))
        elif c['component'] == 'ResourceClaimer':
          sp.add_color(f"claimBeamSprite_{int(kw['playerIndex'])}", kw['color'])
        elif c['component'] == 'Paintbrush':  # four explicit facings, noRotate (components.lua:374-385)
          sp.add_shape(f"brush{int(kw['playerIndex'])}", list(kw['shape']), kw['palette'], True)
    self.own_sprites = sp  # this build's sprites alone
    self.sprites = shared_sprites.view(sp) if shared_sprites is not None else sp

    # ---- groups -------------------------------------------------------------
    self.groups: List[str] = []
    for cfg, _, _, _ in objs:
      sm = _first(cfg['components'], 'StateManager')
      for st in sm['kwargs']['stateConfigs']:
        for g in st.get('groups', []) or []:
          if g not in self.groups:
            self.groups.append(g)
    if len(self.groups) > 31:
      raise ValueError('too many groups')

    # ---- kinds / states / comps / objects ----------------------------------
    self.kinds: List[List[int]] = []
    self.states: List[List[int]] = []
    self.comps_i: List[List[int]] = []
    self.comps_d: List[List[float]] = []
    self.objects: List[List[int]] = []
    self.kind_names: List[str] = []
    self._needs_grass: List[int] = []
    self.state_names: List[List[str]] = []
    kind_of: Dict[str, int] = {}
    self.avatar_objs: List[int] = []
    self.view = None
    self.sprite_maps: Dict[int, Dict[str, str]] = {}
    self.obj_choice: List[List[int]] = []
    for oid, (cfg, x, y, cond) in enumerate(objs):
      comps = cfg['components']
      tr = _first(comps, 'Transform')
      tkw = (tr or {}).get('kwargs', {}) or {}
      orient = COMPASS[tkw.get('orientation', 'N')]
      if 'position' in tkw and tkw['position'] not in ([0, 0], None):
        x, y = tkw['position']
      stripped = copy.deepcopy(comps)
      for c in stripped:
        if c['component'] == 'Transform':
          c.pop('kwargs', None)
      key = json.dumps([cfg.get('name', ''), stripped], sort_keys=True,
                       default=str)
      if key not in kind_of:
        kind_of[key] = self._add_kind(cfg)
      kid = kind_of[key]
      sm = _first(comps, 'StateManager')['kwargs']
      init = self.state_names[kid].index(sm['initialState'])
      self.objects.append([kid, int(x), int(y), orient, init])
      self.obj_choice.append([cond[0], cond[1]] if cond else [-1, 0])
      if cond:
        # What may depend on the per-env draw: invisible component-free pieces (spawn points), and territory's resource
        # bundle (resource + its texture / reward indicator / damage indicator on the same cell, all on one condition),
        # which the territory kernel and the oracle both treat as "this resource does not exist in this episode".
        names = {c['component'] for c in comps}
        states = self.states[self.kinds[kid][0]:self.kinds[kid][0] + self.kinds[kid][1]]
        inert = names <= {'StateManager', 'Transform', 'Appearance'} and all(st[1] < 0 and st[2] < 0 for st in states)
        bundle = cfg.get('name') in ('resource', 'resource_texture', 'reward_indicator', 'damage_indicator')
        if not (inert or (bundle and self.family == 'territory')):
          raise NotImplementedError(f"'choice' prefab {cfg.get('name')!r} cannot depend on the per-env draw in the CUDA engine "
                                    '(supported: invisible component-free pieces, territory resource bundles); pass a build_seed '
                                    'to fix one draw at compile time')
      if self.kinds[kid][4]:
        self.avatar_objs.append(oid)
    if len(self.avatar_objs) != self.num_players:
      raise ValueError('number of avatar objects != numPlayers')
    for ci, comp in enumerate(self.comps_i):
      if comp[0] == COMP['Resource']:  # territory/components.lua:177-182 (queryPosition layers are hard-coded)
        tex = self.state_names[self.kind_names.index('resource_texture')]
        dmg = self.state_names[self.kind_names.index('damage_indicator')]
        comp[1 + 7] = self.layers.index('lowerPhysical')
        comp[1 + 8] = self.layers.index('superDirectionIndicatorLayer')
        comp[1 + 9] = tex.index('destroyed')
        comp[1 + 10] = dmg.index('inactive')
        comp[1 + 11] = dmg.index('damaged')
      elif comp[0] == COMP['RewardIndicator']:  # :293-300
        comp[1 + 2] = self.layers.index('upperPhysical')
    for ci in self._needs_grass:  # DensityRegrow toggles the underlying grass (components.lua:181-193)
      grass = [n for n in self.state_names if 'grass' in n and 'dessicated' in n]
      if not grass:
        raise ValueError('DensityRegrow needs a prefab with states grass/dessicated')
      self.comps_i[ci][1 + 9] = grass[0].index('grass')
      self.comps_i[ci][1 + 10] = grass[0].index('dessicated')
    self.world_sprite_map = sim.get('worldSpriteMap') or {}

  # -------------------------------------------------------------------------
  def _state_index(self, names: List[str], state: str) -> int:
    if state not in names:
      raise KeyError(f'state {state!r} not in {names}')
    return names.index(state)

  def _add_kind(self, cfg) -> int:
    comps = cfg['components']
    sm = _first(comps, 'StateManager')['kwargs']
    names = [st['state'] for st in sm['stateConfigs']]
    state0 = len(self.states)
    for st in sm['stateConfigs']:
      layer = self.layers.index(st['layer']) if isinstance(st.get('layer'), str) else -1
      sprite = self.sprites.index(st['sprite']) if isinstance(st.get('sprite'), str) else -1
      contact = 0 if isinstance(st.get('contact'), str) else -1
      if isinstance(st.get('contact'), str) and st['contact'] != 'avatar':
        raise NotImplementedError('only the "avatar" contact is supported')
      mask = 0
      for g in st.get('groups', []) or []:
        mask |= 1 << self.groups.index(g)
      self.states.append([layer, sprite, contact, mask])
    comp0 = len(self.comps_i)
    is_avatar = 0
    for c in comps:
      name = c['component']
      kw = c.get('kwargs', {}) or {}
      if name not in COMP:
        raise NotImplementedError(
            f'component {name!r} is not supported by the CUDA engine')
      ip = [0] * COMP_NI
      dp = [0.0] * COMP_ND
      si = lambda s: self._state_index(names, s)
      hit_id = lambda h: [x[0] for x in self.hits].index(h)
      if name == 'BeamBlocker':
        ip[0] = hit_id(kw['beamType']) if kw['beamType'] in [h[0] for h in self.hits] else -1
      elif name == 'Edible':
        ip[0], ip[1] = si(kw['liveState']), si(kw['waitState'])
        dp[0] = float(kw['rewardForEating'])
      elif name == 'AppleGrow':
        ip[0] = si('apple')
        dp[0] = float(kw['maxAppleGrowthRate'])
        dp[1] = float(kw['thresholdDepletion'])
        dp[2] = float(kw['thresholdRestoration'])
      elif name == 'DirtTracker':
        ip[0] = si(kw.get('activeState', 'dirt'))
        ip[1] = si(kw.get('inactiveState', 'dirtWait'))
      elif name == 'DirtCleaning':
        ip[0], ip[1], ip[2] = si('dirt'), si('dirtWait'), hit_id('cleanHit')
      elif name == 'Avatar':
        is_avatar = 1
        idx0 = int(kw['index']) - 1
        ip[0] = idx0
        ip[1], ip[2] = si(kw['aliveState']), si(kw['waitState'])
        ip[3] = self.groups.index(kw['spawnGroup'])
        post = kw.get('postInitialSpawnGroup', '_DEFAULT')
        ip[4] = -1 if post == '_DEFAULT' else self.groups.index(post)
        view = kw['view']
        for i, side in enumerate(('left', 'right', 'forward', 'backward')):
          ip[5 + i] = int(view[side])
        if view.get('centered', False):
          raise NotImplementedError('centered views')
        if self.view is None:
          self.view = tuple(ip[5:9])
        elif self.view != tuple(ip[5:9]):
          raise NotImplementedError('per-avatar view sizes')
        ip[9] = int(kw.get('skipWaitStateRewards', True))
        ip[10] = int(kw.get('randomizeInitialOrientation', True))
        dp[0] = float(kw.get('speed', 1.0))
        if kw.get('useAbsoluteCoordinates', False):
          raise NotImplementedError('useAbsoluteCoordinates')
        if kw.get('additionalLiveStates'):
          raise NotImplementedError('additionalLiveStates')
        order = list(kw.get('actionOrder', ['move', 'turn']))
        for a in order:
          if a not in ACTION_FIELDS:
            raise NotImplementedError(f'action {a!r}')
        self.sprite_maps[idx0] = dict(kw.get('spriteMap', {}) or {})
      elif name == 'Zapper':
        ip[0], ip[1], ip[2] = int(kw['cooldownTime']), int(kw['beamLength']), int(kw['beamRadius'])
        ip[3] = int(kw['framesTillRespawn'])
        ip[4] = int(kw.get('removeHitPlayer', True))
        ip[5] = hit_id('zapHit')
        dp[0] = float(kw['penaltyForBeingZapped'])
        dp[1] = float(kw['rewardForZapping'])
      elif name == 'Cleaner':
        ip[0], ip[1], ip[2] = int(kw['cooldownTime']), int(kw['beamLength']), int(kw['beamRadius'])
        ip[3] = hit_id('cleanHit')
      elif name == 'MineBeam':  # coop_mining/components.lua:160-262
        ip[0], ip[1], ip[2] = int(kw['cooldownTime']), int(kw['beamLength']), int(kw['beamRadius'])
        ip[3] = hit_id('mine')
        role = kw['agentRole']
        mining, extracting = list(kw['roleRewardForMining'][role]), list(kw['roleRewardForExtracting'][role])
        if len(mining) != 2 or len(extracting) != 2:
          raise NotImplementedError('coop_mining with other than two ore types')
        dp[0], dp[1], dp[2], dp[3] = (float(v) for v in mining + extracting)
      elif name == 'Ore':  # coop_mining/components.lua:60-157
        ip[0], ip[1], ip[2] = si(kw['waitState']), si(kw['rawState']), si(kw['partialState'])
        ip[3], ip[4] = int(kw['minNumMiners']), int(kw['miningWindow'])
      elif name == 'FixedRateRegrow':  # coop_mining/components.lua:25-58
        live, rates = list(kw['liveStates']), list(kw['liveRates'])
        if len(live) != len(rates) or len(live) > 4:
          raise NotImplementedError('FixedRateRegrow with more than four live states')
        ip[0] = len(live)
        for i, st_name in enumerate(live):
          ip[1 + i] = si(st_name)
          dp[i] = float(rates[i])
        ip[5] = si(kw['waitState'])
      elif name == 'Taste' and self.family != 'territory':
        ip[0] = _TASTE_ROLES[kw.get('role', 'free')]
        dp[0] = float(kw.get('rewardAmount', 1))
      elif name == 'DirtSpawner':
        ip[0] = int(kw.get('delayStartOfDirtSpawning', 0))
        dp[0] = float(kw['dirtSpawnProbability'])
      elif name == 'StochasticIntervalEpisodeEnding':
        ip[0] = int(kw['minimumFramesPerEpisode'])
        ip[1] = int(kw['intervalLength'])
        dp[0] = float(kw['probabilityTerminationPerInterval'])
      elif name == 'Animation':
        sts = list(kw['states'])
        if len(sts) > 8:
          raise NotImplementedError('Animation with > 8 states')
        ip[0] = len(sts)
        for i, s in enumerate(sts):
          ip[1 + i] = si(s)
        ip[9] = int(kw['gameFramesPerAnimationFrame'])
        ip[10] = int(kw['loop'])
        ip[11] = int(kw.get('randomStartFrame', False))
      elif name == 'Role' and self.family == 'coins':
        # coins/components.lua Role: multipliers on the four Coin rewards.
        name = 'CoinsRole'
        dp[0] = float(kw.get('multiplyRewardSelfForMatch', 1.0))
        dp[1] = float(kw.get('multiplyRewardSelfForMismatch', 1.0))
        dp[2] = float(kw.get('multiplyRewardOtherForMatch', 1.0))
        dp[3] = float(kw.get('multiplyRewardOtherForMismatch', 1.0))
      elif name == 'Coin':  # coins/components.lua Coin
        ip[0] = si(kw['waitState'])
        ip[1] = int(bool(kw.get('terminateEpisode', False)))
        ip[2] = int(kw.get('coinsToTerminateEpisode', -1))
        dp[0] = float(kw['rewardSelfForMatch'])
        dp[1] = float(kw['rewardSelfForMismatch'])
        dp[2] = float(kw['rewardOtherForMatch'])
        dp[3] = float(kw['rewardOtherForMismatch'])
      elif name == 'ChoiceCoinRegrow':  # coins/components.lua ChoiceCoinRegrow
        ip[0], ip[1], ip[2] = si(kw['liveStateA']), si(kw['liveStateB']), si(kw['waitState'])
        dp[0] = float(kw['regrowRate'])
      elif name == 'PlayerCoinType':
        # 0 / 1 = the coin prefab's liveStateA / liveStateB (Coin:onEnter compares the type with the coin's state name)
        regrow = _first(self._prefabs['coin']['components'], 'ChoiceCoinRegrow')['kwargs']
        ip[0] = [regrow['liveStateA'], regrow['liveStateB']].index(kw['coinType'])
      elif name == 'Role':
        # component_library.lua Role: a string the avatar carries; only RoleBasedRewardTile reads it.
        self.avatar_roles.add(str(kw.get('role', 'none')))
      elif name == 'RoleBasedRewardTile':
        # component_library.lua:1098-1136: pays rolesToRewards[role] to an avatar that steps on the
        # tile. Emitted as an inert component; _check_role_tiles() rejects configs in which some
        # avatar's role is actually rewarded (not the case for any default-role build).
        self.rewarded_roles.update(str(k) for k in (kw.get('rolesToRewards') or {}))
      elif name == 'Taste' and self.family == 'territory':
        name = 'TerritoryTaste'
        ip[0] = _TERRITORY_TASTE_ROLES[kw.get('role', 'none')]
        dp[0] = float(kw.get('rewardAmount', 0))
        dp[1] = float(kw.get('firstClaimRewardMultiplier', 1.0))
      elif name == 'Resource':
        ip[0] = int(kw['initialHealth'])
        ip[1] = si(kw['destroyedState'])
        ip[2] = int(kw['rewardDelay'])
        ip[3] = int(kw.get('delayTillSelfRepair', 15))
        ip[4] = si('claimed_by_1')
        ip[5] = si(sm['initialState'])
        ip[6] = self.groups.index('claimedResources')
        dp[0] = float(kw['reward']); dp[1] = float(kw['rewardRate'])
        dp[2] = float(kw.get('selfRepairProbability', 0.1))
      elif name == 'ResourceClaimer':
        ip[0] = int(kw['playerIndex']) - 1
        ip[1], ip[2], ip[3] = int(kw['beamLength']), int(kw['beamRadius']), int(kw['beamWait'])
        ip[4] = hit_id(f"claimBeam_{int(kw['playerIndex'])}")
      elif name == 'RewardIndicator':
        ip[0] = si('inactive')
        ip[1] = si('dry_claimed_by_1')
      elif name == 'Paintbrush':
        ip[0] = int(kw['playerIndex']) - 1
        ip[1] = hit_id(f"directionHit{int(kw['playerIndex'])}")
      elif name == 'GraduatedSanctionsMarking':
        logic = list(kw['hitLogic'])
        if len(logic) > 3:
          raise NotImplementedError('GraduatedSanctionsMarking with > 3 levels')
        ip[0] = int(kw['playerIndex']) - 1
        ip[1] = si(kw['waitState'])
        ip[2] = int(kw.get('initialLevel', 1))
        rec = kw.get('recoveryTime', False)
        ip[3] = int(rec) if rec else -1
        ip[4] = hit_id(kw['hitName'])
        ip[5] = len(logic)
        ip[6] = si('level_1')
        for li, lg in enumerate(logic):
          ip[7 + 3 * li] = int(lg.get('levelIncrement', 0))
          ip[8 + 3 * li] = int(bool(lg.get('remove', False)))
          fr = lg.get('freeze', None)
          ip[9 + 3 * li] = int(fr) if fr else 0
          dp[2 * li] = float(lg.get('sourceReward', 0))
          dp[2 * li + 1] = float(lg.get('targetReward', 0))
      elif name == 'DensityRegrow':
        ip[0] = si(kw['liveState'])
        ip[3] = si(kw['waitState'])
        radius = float(kw['radius'])
        upper = int(np.floor(np.pi * radius**2 + 1)) + 1 if radius >= 0 else 0
        ip[1] = si(kw['waitState'] + '_0')
        ip[2] = upper
        probs = [float(p) for p in kw['regrowthProbabilities']]
        if len(probs) > COMP_ND - 1:
          raise NotImplementedError('too many regrowthProbabilities')
        ip[4] = len(probs)
        ip[5] = int(kw.get('canRegrowIfOccupied', True))
        dp[0] = radius
        dp[1:1 + len(probs)] = probs
        # Layer names are hard-coded in the Lua (commons_harvest/components.lua:149,196-199).
        ip[6] = self.layers.index('logic')
        ip[7] = self.layers.index('lowerPhysical')
        ip[8] = self.layers.index('background')
        self._needs_grass.append(len(self.comps_i))
      self.comps_i.append([COMP[name]] + ip)
      self.comps_d.append(dp)
    kid = len(self.kinds)
    self.kinds.append([state0, len(names), comp0, len(comps), is_avatar, 0])
    self.kind_names.append(cfg.get('name', ''))
    self.state_names.append(names)
    return kid

  # -------------------------------------------------------------------------
  def sprite_map_table(self) -> np.ndarray:
    """[P+1, n_sprites]: viewer -> displayed sprite (row P = WORLD.RGB)."""
    n = len(self.sprites.names)
    table = np.tile(np.arange(n, dtype=np.int32), (self.num_players + 1, 1))
    for idx0, mapping in self.sprite_maps.items():
      for src, dst in mapping.items():
        table[idx0, self.sprites.index(src)] = self.sprites.index(dst)
    for src, dst in self.world_sprite_map.items():
      table[self.num_players, self.sprites.index(src)] = self.sprites.index(dst)
    return table

  def init_grid(self) -> np.ndarray:
    """uint16 [L, H*W]: sprites of all non-avatar objects in their initial state."""
    L = len(self.layers)
    grid = np.zeros((L, self.H * self.W), np.uint16)
    occupied = np.zeros((L, self.H * self.W), bool)
    for (kid, x, y, orient, st) in self.objects:
      if self.kinds[kid][4]:
        continue
      layer, sprite, _, _ = self.states[self.kinds[kid][0] + st]
      if layer < 0:
        continue
      cell = y * self.W + x
      if occupied[layer, cell]:
        raise ValueError(f'two pieces on layer {self.layers[layer]} at {x},{y}')
      occupied[layer, cell] = True
      if sprite >= 0:
        grid[layer, cell] = 1 + sprite * 4 + orient
    return grid


# ---------------------------------------------------------------------------
# Family tables for the CUDA engine
# ---------------------------------------------------------------------------
def _objects_with(model: WorldModel, comp: str):
  out = []
  for oid, (kid, x, y, orient, st) in enumerate(model.objects):
    k = model.kinds[kid]
    for ci in range(k[2], k[2] + k[3]):
      if model.comps_i[ci][0] == COMP[comp]:
        out.append((oid, ci))
        break
  return out


_Entity = collections.namedtuple('_Entity', 'oid cell state kind comp')


def _entities(model: WorldModel, comp: str) -> List[_Entity]:
  """The objects with component `comp`, in object order: id, cell, initial state, kind and the component's row."""
  rows = []
  for oid, ci in _objects_with(model, comp):
    kid, x, y, _, st = model.objects[oid]
    rows.append(_Entity(oid, y * model.W + x, st, kid, ci))
  return rows


def _one_kind(rows: List[_Entity], what: str) -> int:
  """The kind all of `rows` share."""
  kid = rows[0].kind
  if any(r.kind != kid for r in rows):
    raise NotImplementedError(f'heterogeneous {what} prefabs')
  return kid


def _kind_comps(model: WorldModel, kid: int, comp: str) -> List[int]:
  """Rows of the components `comp` of kind `kid`."""
  k = model.kinds[kid]
  return [c for c in range(k[2], k[2] + k[3]) if model.comps_i[c][0] == COMP[comp]]


def _comp_params(model: WorldModel, ci: int):
  """(int params, f64 params) of component row `ci`."""
  return model.comps_i[ci][1:], model.comps_d[ci]


def _avatar_comps(model: WorldModel, comp: str):
  """The parameters of component `comp` of every avatar, in avatar object order."""
  return [_comp_params(model, _kind_comps(model, model.objects[oid][0], comp)[0]) for oid in model.avatar_objs]


def _avatar_comp(model: WorldModel, comp: str):
  """The parameters of component `comp`, which must be identical across avatars."""
  rows = _avatar_comps(model, comp)
  if any(r != rows[0] for r in rows[1:]):
    raise NotImplementedError(f'per-avatar {comp} parameters')
  return rows[0]


def _scene_comp(model: WorldModel, comp: str):
  """The parameters of the scene's component `comp` (the scene is object 0)."""
  rows = _kind_comps(model, model.objects[0][0], comp)
  if not rows:
    raise KeyError(comp)
  return _comp_params(model, rows[0])


def _hits(model: WorldModel) -> Dict[str, tuple]:
  """Hit name -> (layer, sprite) of its beam."""
  return {h[0]: (model.layers.index(h[1]), model.sprites.index(h[2])) for h in model.hits}


def _zapper_params(zap, hits, ending) -> Dict[str, int]:
  """The MPB_FP_* slots from the Zapper and StochasticIntervalEpisodeEnding int params."""
  return dict(ZAP_COOLDOWN=zap[0], ZAP_LENGTH=zap[1], ZAP_RADIUS=zap[2], ZAP_RESPAWN=zap[3], ZAP_REMOVE=zap[4],
              ZAP_LAYER=hits['zapHit'][0], ZAP_SPRITE=hits['zapHit'][1], END_MIN_FRAMES=ending[0],
              END_INTERVAL=ending[1])


def _store_params(sections: Dict[str, np.ndarray], family: str, ints: Mapping[str, Any], floats: Mapping[str, Any]):
  """Writes the family's "<prefix>_ip" and "<prefix>_dp" blocks: each value in the slot of its name, 0 elsewhere."""
  prefix, int_layout, float_layout = FAMILY_PARAMS[family]
  for suffix, layout, values, dtype in (('_ip', int_layout, ints, np.int32), ('_dp', float_layout, floats, np.float64)):
    block = np.zeros(layout['COUNT'], dtype)
    for name, value in values.items():
      if name == 'COUNT' or name not in layout:
        raise KeyError(f'{prefix}{suffix} has no slot {name!r}')
      block[layout[name]] = value
    sections[prefix + suffix] = block


def family_params(sections: Mapping[str, np.ndarray]) -> Dict[str, Any]:
  """Slot name -> value of both parameter blocks of a blob's family; `sections` is the unpacked blob."""
  family = {v: k for k, v in FAMILY.items()}[int(sections['meta'][META['FAMILY']])]
  prefix, int_layout, float_layout = FAMILY_PARAMS[family]
  out = {k: int(sections[prefix + '_ip'][i]) for k, i in int_layout.items() if k != 'COUNT'}
  out.update({k: float(sections[prefix + '_dp'][i]) for k, i in float_layout.items() if k != 'COUNT'})
  return out


def _avatar_tables(model: WorldModel, sections: Dict[str, np.ndarray]):
  """Tables shared by all families: avatars, spawn points, blockers."""
  P = model.num_players
  av = np.zeros((P, 8), np.int32)  # obj id, live sprite, layer, spawn group, post group
  for oid in model.avatar_objs:
    kid = model.objects[oid][0]
    ip = model.comps_i[_kind_comps(model, kid, 'Avatar')[0]][1:]
    idx0 = ip[0]
    alive = model.states[model.kinds[kid][0] + ip[1]]
    av[idx0] = [oid, alive[1], alive[0], ip[3], ip[4], 0, 0, 0]
  sections['av_table'] = av
  # Spawn cells per group, in object (piece) order.
  for gi, g in enumerate(model.groups):
    cells, conds = [], []
    for oid, (kid, x, y, orient, st) in enumerate(model.objects):
      state = model.states[model.kinds[kid][0] + st]
      if state[3] & (1 << gi) and not model.kinds[kid][4]:
        cells.append(y * model.W + x)
        conds.append(model.obj_choice[oid])
    if g in ('spawnPoints', 'insideSpawnPoints'):
      sections['spawn_cells_' + str(gi)] = np.array(cells, np.int32)
      if any(c[0] >= 0 for c in conds):  # members that exist only on some tickets of their 'choice' group
        sections['spawn_cond_' + str(gi)] = np.array(conds, np.int32).reshape(-1, 2)
      users = int((av[:, 3] == gi).sum())
      if sum(1 for c in conds if c[0] < 0) < users:
        raise ValueError(f'{users} avatars start in group {g!r} but the map guarantees only '
                         f'{sum(1 for c in conds if c[0] < 0)} such cells')
  # Static beam blockers: bit h set if a BeamBlocker for hit h sits on the cell.
  flags = np.zeros(model.H * model.W, np.uint8)
  for oid, ci in _objects_with(model, 'BeamBlocker'):
    kid, x, y, _, _ = model.objects[oid]
    for c in _kind_comps(model, kid, 'BeamBlocker'):
      if model.comps_i[c][1] >= 0:
        flags[y * model.W + x] |= 1 << model.comps_i[c][1]
  sections['cell_flags'] = flags


def _clean_up_tables(model: WorldModel, sections: Dict[str, np.ndarray]):
  """SoA tables for the clean_up step kernel (SURVEY.md Appendix B.1)."""
  apples = _entities(model, 'AppleGrow')
  dirts = _entities(model, 'DirtTracker')
  waters = _entities(model, 'Animation')
  kid_a = _one_kind(apples, 'apple')
  ka = model.kinds[kid_a]
  grow_i, grow_d = _comp_params(model, apples[0].comp)
  apple_state = model.states[ka[0] + grow_i[0]]
  edible = _kind_comps(model, kid_a, 'Edible')[0]
  sections['cu_apple'] = np.array([[r.oid, r.cell, int(r.state == grow_i[0])] for r in apples], np.int32)
  # Dirt: both prefabs share states; column 2 = initially dirty.
  dirt_rows = []
  dirt_layer = dirt_sprite = wait_layer = None
  for r in dirts:
    k = model.kinds[r.kind]
    active, inactive = model.comps_i[r.comp][1:3]
    sa, sw = model.states[k[0] + active], model.states[k[0] + inactive]
    if dirt_layer is None:
      dirt_layer, dirt_sprite, wait_layer = sa[0], sa[1], sw[0]
    elif (dirt_layer, dirt_sprite, wait_layer) != (sa[0], sa[1], sw[0]):
      raise NotImplementedError('heterogeneous dirt prefabs')
    dirt_rows.append([r.oid, r.cell, int(r.state == active)])
  sections['cu_dirt'] = np.array(dirt_rows, np.int32)
  kw_ = model.kinds[waters[0].kind]
  anim = model.comps_i[waters[0].comp][1:]
  n_anim = anim[0]
  water_sprites = [model.states[kw_[0] + anim[1 + i]][1] for i in range(n_anim)]
  sections['cu_water'] = np.array([[r.oid, r.cell] for r in waters], np.int32)
  sections['cu_water_sprites'] = np.array(water_sprites, np.int32)
  zi, zd = _avatar_comp(model, 'Zapper')
  cl, _ = _avatar_comp(model, 'Cleaner')
  ti, td = _avatar_comp(model, 'Taste')
  di, dd = _scene_comp(model, 'DirtSpawner')
  ei, ed = _scene_comp(model, 'StochasticIntervalEpisodeEnding')
  hits = _hits(model)
  _store_params(sections, 'clean_up', dict(
      N_APPLES=len(apples), N_DIRT=len(dirts), N_WATER=len(waters), APPLE_LAYER=apple_state[0],
      APPLE_SPRITE=apple_state[1], DIRT_LAYER=dirt_layer, DIRT_SPRITE=dirt_sprite, DIRT_WAIT_LAYER=wait_layer,
      WATER_LAYER=model.states[kw_[0] + anim[1]][0], N_ANIM=n_anim, ANIM_FRAMES=anim[9], ANIM_RANDOM=anim[11],
      **_zapper_params(zi, hits, ei), CLEAN_COOLDOWN=cl[0], CLEAN_LENGTH=cl[1], CLEAN_RADIUS=cl[2],
      CLEAN_LAYER=hits['cleanHit'][0], CLEAN_SPRITE=hits['cleanHit'][1], DIRT_DELAY=di[0], TASTE_ROLE=ti[0]), dict(
      GROW_RATE=grow_d[0], GROW_DEPLETION=grow_d[1], GROW_RESTORATION=grow_d[2], EAT_REWARD=model.comps_d[edible][0],
      ZAP_PENALTY=zd[0], ZAP_REWARD=zd[1], DIRT_PROB=dd[0], END_PROB=ed[0], TASTE_AMOUNT=td[0]))


def _commons_tables(model: WorldModel, sections: Dict[str, np.ndarray]):
  """SoA tables for the commons_harvest step kernel (SURVEY.md Appendix B.2)."""
  W = model.W
  apples = _entities(model, 'DensityRegrow')
  kid_a = _one_kind(apples, 'apple')
  ka = model.kinds[kid_a]
  dr, drd = _comp_params(model, apples[0].comp)
  live_state, wait0, n_wait, plain_wait, n_probs = dr[0], dr[1], dr[2], dr[3], dr[4]
  if not dr[5]:
    raise NotImplementedError('canRegrowIfOccupied=False')
  live = model.states[ka[0] + live_state]
  waitk = model.states[ka[0] + wait0]
  plain = model.states[ka[0] + plain_wait]
  if plain[0] != waitk[0] or plain[1] != waitk[1]:
    raise NotImplementedError('wait states with different layers/sprites')
  edible = _kind_comps(model, kid_a, 'Edible')[0]
  if model.comps_i[edible][1] != live_state or model.comps_i[edible][2] != plain_wait:
    raise NotImplementedError('Edible states differ from DensityRegrow states')
  # grass under each apple (background layer)
  grass_kind = [i for i, n in enumerate(model.state_names) if 'grass' in n and 'dessicated' in n][0]
  gk = model.kinds[grass_kind]
  gnames = model.state_names[grass_kind]
  grass_state = model.states[gk[0] + gnames.index('grass')]
  dess_state = model.states[gk[0] + gnames.index('dessicated')]
  grass_at = {}
  for oid, (kid, x, y, orient, st) in enumerate(model.objects):
    if kid == grass_kind:
      grass_at[y * W + x] = oid
  radius = drd[0]
  cell_to_apple = {r.cell: i for i, r in enumerate(apples)}
  nbr = np.full((len(apples), 16), -1, np.int32)
  r_int = int(radius)
  for i, row in enumerate(apples):
    cx, cy = row.cell % W, row.cell // W
    k = 0
    for dy in range(-r_int, r_int + 1):   # same scan order as the oracle (irrelevant to results)
      for dx in range(-r_int, r_int + 1):
        if dx * dx + dy * dy > radius * radius or (dx == 0 and dy == 0):
          continue
        x, y = cx + dx, cy + dy
        if model.topology == 1:
          x %= W; y %= model.H
        elif not (0 <= x < W and 0 <= y < model.H):
          continue
        j = cell_to_apple.get(y * W + x)
        if j is not None:
          if k == nbr.shape[1]:
            raise NotImplementedError(f'DensityRegrow radius {radius}: the disc around the apple at ({cx}, {cy}) holds '
                                      f'more than {nbr.shape[1]} other apples (the kernel keeps at most '
                                      f'{nbr.shape[1]} neighbours per apple)')
          nbr[i, k] = j
          k += 1
  zi, zd = _avatar_comp(model, 'Zapper')
  ei, ed = _scene_comp(model, 'StochasticIntervalEpisodeEnding')
  probs = drd[1:1 + min(n_probs, 4)]  # mp_create refuses more than four
  _store_params(sections, 'commons_harvest', dict(
      N_APPLES=len(apples), APPLE_LAYER=live[0], APPLE_SPRITE=live[1], WAIT_LAYER=waitk[0], WAIT_SPRITE=waitk[1],
      N_WAIT=n_wait, N_PROBS=n_probs, GRASS_LAYER=grass_state[0], GRASS_SPRITE=grass_state[1],
      DESS_SPRITE=dess_state[1], **_zapper_params(zi, _hits(model), ei)), dict(
      {f'PROB_{i}': p for i, p in enumerate(probs)}, EAT_REWARD=model.comps_d[edible][0], ZAP_PENALTY=zd[0],
      ZAP_REWARD=zd[1], END_PROB=ed[0]))
  sections['ch_apple'] = np.array([[r.oid, r.cell, int(r.state == live_state), grass_at.get(r.cell, -1)] for r in apples],
                                  np.int32)
  sections['ch_nbr'] = nbr


def _coins_tables(model: WorldModel, sections: Dict[str, np.ndarray]):
  """SoA tables for the coins step kernel (lua/levels/coins/components.lua)."""
  if model.num_players != 2:
    raise NotImplementedError('coins supports exactly two players (coins/components.lua:93-96)')
  coins = _entities(model, 'Coin')
  kid_c = _one_kind(coins, 'coin')
  kc = model.kinds[kid_c]
  coin_i, coin_d = _comp_params(model, coins[0].comp)
  ri, rd = _comp_params(model, _kind_comps(model, kid_c, 'ChoiceCoinRegrow')[0])
  if ri[2] != coin_i[0]:
    raise NotImplementedError('Coin and ChoiceCoinRegrow wait states differ')
  if any(c.state != coin_i[0] for c in coins):
    raise NotImplementedError('coins that do not start in the wait state')
  live_a, live_b = model.states[kc[0] + ri[0]], model.states[kc[0] + ri[1]]
  if live_a[0] != live_b[0]:
    raise NotImplementedError('coin types on different layers')
  types = [i[0] for i, _ in _avatar_comps(model, 'PlayerCoinType')]
  roles = [d for _, d in _avatar_comps(model, 'CoinsRole')]
  ei, ed = _scene_comp(model, 'StochasticIntervalEpisodeEnding')
  _store_params(sections, 'coins', dict(
      N_COINS=len(coins), COIN_LAYER=live_a[0], COIN_SPRITE_0=live_a[1], COIN_SPRITE_1=live_b[1], TERMINATE=coin_i[1],
      TERMINATE_N=coin_i[2], END_MIN_FRAMES=ei[0], END_INTERVAL=ei[1], COIN_TYPE_0=types[0], COIN_TYPE_1=types[1]), dict(
      REGROW_RATE=rd[0], END_PROB=ed[0],
      # the four rewards as each collecting player pays them: base reward x that player's Role multiplier
      **{f'REWARD_{p}_{name}': coin_d[k] * roles[p][k] for p in range(2) for k, name in enumerate(_COIN_REWARDS)}))
  sections['co_coin'] = np.array([[c.oid, c.cell] for c in coins], np.int32)


def _mining_tables(model: WorldModel, sections: Dict[str, np.ndarray]):
  """SoA tables for the coop_mining step kernel (lua/levels/coop_mining/components.lua)."""
  ores = _entities(model, 'FixedRateRegrow')
  kid_o = _one_kind(ores, 'ore')
  ko = model.kinds[kid_o]
  ri, rd = _comp_params(model, ores[0].comp)
  ore_comps = _kind_comps(model, kid_o, 'Ore')
  if ri[0] != 2 or len(ore_comps) != 2:
    raise NotImplementedError('coop_mining needs two ore types (two Ore components, two live states)')
  wait = ri[5]
  if any(o.state != wait for o in ores):
    raise NotImplementedError('ores that do not start in the wait state')
  # which Ore component owns which live state; "single" ore: one miner extracts, "joint" ore: two miners within the window
  by_raw = {model.comps_i[c][2]: model.comps_i[c][1:] for c in ore_comps}
  single, joint = by_raw[ri[1]], by_raw[ri[2]]
  if single[3] != 1 or joint[3] != 2 or single[0] != wait or joint[0] != wait or single[2] != single[1]:
    raise NotImplementedError('ore types other than (1 miner, no partial state) and (2 miners, partial state)')
  st = lambda i: model.states[ko[0] + i]
  layers = {st(i)[0] for i in (wait, single[1], joint[1], joint[2])}
  if len(layers) != 1:
    raise NotImplementedError('ore states on different layers')
  bi, bd = _avatar_comp(model, 'MineBeam')
  if bi[2] != 0:
    raise NotImplementedError('mine beams with a radius')
  ei, ed = _scene_comp(model, 'StochasticIntervalEpisodeEnding')
  hits = _hits(model)
  _store_params(sections, 'coop_mining', dict(
      N_ORES=len(ores), ORE_LAYER=st(wait)[0], ORE_SPRITE_0=st(wait)[1], ORE_SPRITE_1=st(single[1])[1],
      ORE_SPRITE_2=st(joint[1])[1], ORE_SPRITE_3=st(joint[2])[1], MINE_WINDOW=joint[4], MINE_COOLDOWN=bi[0],
      MINE_LENGTH=bi[1], MINE_LAYER=hits['mine'][0], MINE_SPRITE=hits['mine'][1], END_MIN_FRAMES=ei[0],
      END_INTERVAL=ei[1], MINE_HIT=bi[3]), dict(
      RATE_0=rd[0], RATE_1=rd[1], END_PROB=ed[0], MINE_REWARD_0=bd[0], MINE_REWARD_1=bd[1], EXTRACT_REWARD_0=bd[2],
      EXTRACT_REWARD_1=bd[3]))
  sections['cm_ore'] = np.array([[o.oid, o.cell] for o in ores], np.int32)


def _territory_tables(model: WorldModel, sections: Dict[str, np.ndarray]):
  """SoA tables for the territory step kernel (SURVEY.md Appendix B.3)."""
  W, P = model.W, model.num_players
  L = model.layers.index
  res = _entities(model, 'Resource')
  kid_r = _one_kind(res, 'resource')
  kr = model.kinds[kid_r]
  rnames = model.state_names[kid_r]
  rc, rd = _comp_params(model, res[0].comp)
  if rnames.index('unclaimed') != 0 or rnames.index('destroyed') != 1 or rc[4] != 2:
    raise NotImplementedError('resource states must be unclaimed, destroyed, claimed_by_1..P')
  def st_of(kind_name, state):
    kid = model.kind_names.index(kind_name)
    return model.states[model.kinds[kid][0] + model.state_names[kid].index(state)]
  unclaimed = st_of('resource', 'unclaimed')
  tex = st_of('resource_texture', 'unclaimed')
  dmg = st_of('damage_indicator', 'damaged')
  zap = _avatar_comps(model, 'Zapper')
  claim = _avatar_comps(model, 'ResourceClaimer')
  taste = _avatar_comps(model, 'TerritoryTaste')
  for rows, skip in ((zap, ()), (claim, (0, 4)), (taste, ())):
    for r in rows[1:]:
      a = [v for i, v in enumerate(r[0]) if i not in skip]; b = [v for i, v in enumerate(rows[0][0]) if i not in skip]
      if a != b or r[1] != rows[0][1]:
        raise NotImplementedError('per-avatar beam / taste parameters')
  zi, zd = zap[0]
  cli = claim[0][0]
  ti, td = taste[0]
  # markings: one per avatar, in avatar order
  marks = _objects_with(model, 'GraduatedSanctionsMarking')
  if len(marks) != P:
    raise NotImplementedError('territory needs one GraduatedSanctionsMarking object per avatar')
  mk, mkd = _comp_params(model, marks[0][1])
  for i, (oid, ci) in enumerate(marks):
    if model.comps_i[ci][1] != i or model.comps_i[ci][2:] != list(model.comps_i[marks[0][1]][2:]):
      raise NotImplementedError('per-avatar marking parameters')
  mkind = model.objects[marks[0][0]][0]
  mnames = model.state_names[mkind]
  level_states = [model.states[model.kinds[mkind][0] + mnames.index(f'level_{l + 1}')] for l in range(mk[5])]
  ei, ed = _scene_comp(model, 'StochasticIntervalEpisodeEnding')
  hits = _hits(model)
  ints = dict(N_RES=len(res), RES_LAYER=unclaimed[0], UNCLAIMED_SPRITE=unclaimed[1], TEX_LAYER=tex[0],
              TEX_SPRITE=tex[1], IND_LAYER=L('overlay'), DMG_LAYER=dmg[0], DMG_SPRITE=dmg[1],
              MARK_LAYER=level_states[0][0], MARK_INITIAL_LEVEL=mk[2], MARK_RECOVERY=mk[3], MARK_N_LEVELS=mk[5],
              **_zapper_params(zi, hits, ei), CLAIM_LENGTH=cli[1], CLAIM_RADIUS=cli[2], CLAIM_WAIT=cli[3],
              BRUSH_LAYER=L('directionIndicatorLayer'), CLAIM_LAYER=L('superDirectionIndicatorLayer'),
              RES_HEALTH=rc[0], RES_REWARD_DELAY=rc[2], RES_REPAIR_DELAY=rc[3], TASTE_ROLE=ti[0])
  floats = dict(RES_REWARD=rd[0], RES_RATE=rd[1], RES_REPAIR_PROB=rd[2], ZAP_PENALTY=zd[0], ZAP_REWARD=zd[1],
                END_PROB=ed[0], TASTE_AMOUNT=td[0], TASTE_MULT=td[1])
  for l in range(mk[5]):
    ints.update({f'MARK_INC_{l}': mk[7 + 3 * l], f'MARK_REMOVE_{l}': mk[8 + 3 * l], f'MARK_FREEZE_{l}': mk[9 + 3 * l],
                 f'MARK_SPRITE_{l}': level_states[l][1]})
    floats.update({f'MARK_SRC_REWARD_{l}': mkd[2 * l], f'MARK_TGT_REWARD_{l}': mkd[2 * l + 1]})
  _store_params(sections, 'territory', ints, floats)
  sections['tr_res'] = np.array([[r.oid, r.cell, r.state] for r in res], np.int32)
  if model.choice_options:  # resources that exist only on some tickets of their 'choice' group (territory__inside_out's A / B cells)
    cond = np.array([model.obj_choice[r.oid] for r in res], np.int32).reshape(-1, 2)
    by_cell = {}
    for oid, (kid, x, y, orient, st) in enumerate(model.objects):
      if model.obj_choice[oid][0] >= 0 and model.kind_names[kid] in ('resource', 'resource_texture', 'reward_indicator', 'damage_indicator'):
        by_cell.setdefault(y * model.W + x, set()).add(tuple(model.obj_choice[oid]))
    for r in res:  # the four pieces of a resource cell come and go together
      if len(by_cell.get(r.cell, {tuple(model.obj_choice[r.oid])})) != 1 or (model.obj_choice[r.oid][0] >= 0) != (r.cell in by_cell):
        raise NotImplementedError('a resource and its texture / indicators must share one choice condition')
    sections['tr_res_cond'] = cond
  per_player = np.zeros((P, 4), np.int32)
  ind_kind = model.kind_names.index('reward_indicator')
  for i in range(P):
    per_player[i] = [
        model.states[kr[0] + 2 + i][1],
        model.states[model.kinds[ind_kind][0] + model.state_names[ind_kind].index(f'dry_claimed_by_{i + 1}')][1],
        hits[f'directionHit{i + 1}'][1], hits[f'claimBeam_{i + 1}'][1]]
  sections['tr_player_sprites'] = per_player
  # cells whose avatar layer is statically blocked by an AllBeamBlocker piece (walls)
  wall = np.zeros(model.H * W, np.uint8)
  for oid, ci in _objects_with(model, 'AllBeamBlocker'):
    kid, x, y, _, _ = model.objects[oid]
    wall[y * W + x] = 1
  sections['tr_wall'] = wall


# ---------------------------------------------------------------------------
# Entry points
# ---------------------------------------------------------------------------
def apply_prefab_overrides(settings: Mapping[str, Any],
                           overrides: Optional[Mapping[str, Mapping[str, Mapping[str, Any]]]]) -> Dict[str, Any]:
  """`builder.apply_prefab_overrides` (builder.py:70-87) on a plain settings dict: {prefab: {component: {kwarg: value}}}
  sets each kwarg on the FIRST component of that name in `simulation.prefabs[prefab]`. Returns a new settings dict;
  neither argument is modified. Only prefabs are reached, so avatars (built into `gameObjects`) keep their kwargs."""
  settings = copy.deepcopy(dict(settings))
  prefabs = settings['simulation'].get('prefabs', {})
  for prefab, override in (overrides or {}).items():
    for component, arg_overrides in override.items():
      for arg_name, arg_override in arg_overrides.items():
        if prefab not in prefabs:
          raise ValueError(f"Prefab override for '{prefab}' given, but not available in `prefabs`.")
        named = [c for c in prefabs[prefab].get('components', []) if c.get('component') == component]
        if not named:  # game_object_utils.get_first_named_component
          raise ValueError(f"No component with name '{component}' found.")
        named[0]['kwargs'][arg_name] = copy.deepcopy(arg_override)
  return settings


def compile_settings(settings: Mapping[str, Any],
                     config: Optional[Any] = None,
                     build_seed: Optional[int] = None,
                     prefab_overrides: Optional[Mapping[str, Any]] = None) -> bytes:
  """lab2d settings (+ optional substrate config for API metadata) -> blob.

  `build_seed` resolves 'choice' prefabs (see _expand_prefab); configs without them ignore it. `prefab_overrides` are
  applied first, as the reference builder applies them (apply_prefab_overrides).
  """
  if prefab_overrides:
    settings = apply_prefab_overrides(settings, prefab_overrides)
  return _compile_model(WorldModel(settings, build_seed), config)


def compile_settings_set(settings_list: Sequence[Mapping[str, Any]],
                         config: Optional[Any] = None,
                         build_seeds: Optional[Sequence[Optional[int]]] = None,
                         prefab_overrides: Optional[Sequence[Optional[Mapping[str, Any]]]] = None) -> List[bytes]:
  """A draw set: one blob per entry of `settings_list` (e.g. the builds of one substrate under several build seeds, or
  one build under several `prefab_overrides`), all on one sprite table. That table is the union of every entry's
  sprites, deduplicated by name and pixels, in first-appearance order (SharedSprites), so the sprite-side sections
  (atlas, sprite_opaque, sprite_map, the OutOfBounds / OutOfView ids) are byte-identical across the set, and an engine
  can run the blobs as per-env variants (mp_create_variants). What differs is which sprite ids the states, avatars and
  family tables refer to, and whatever the map decides. When no entry adds a sprite of its own (no appearance
  override), each blob equals the entry compiled alone. A set of one is compile_settings' blob, byte for byte.
  `build_seeds[i]` resolves entry i's 'choice' prefabs; `prefab_overrides[i]` is applied to entry i as
  compile_settings applies it."""
  settings_list = list(settings_list)
  if not settings_list:
    raise ValueError('compile_settings_set needs at least one settings entry')
  seeds = list(build_seeds) if build_seeds is not None else [None] * len(settings_list)
  if len(seeds) != len(settings_list):
    raise ValueError(f'{len(seeds)} build seeds for {len(settings_list)} settings entries')
  if prefab_overrides is not None:
    prefab_overrides = list(prefab_overrides)
    if len(prefab_overrides) != len(settings_list):
      raise ValueError(f'{len(prefab_overrides)} prefab_overrides for {len(settings_list)} settings entries')
    settings_list = [apply_prefab_overrides(s, o) if o else s for s, o in zip(settings_list, prefab_overrides)]
  own = [WorldModel(s, seed) for s, seed in zip(settings_list, seeds)]
  shared = SharedSprites(own[0].sprite_size)
  for model in own:
    if model.sprite_size != shared.size:
      raise ValueError('the entries of a draw set need one sprite size')
    shared.add(model.own_sprites)
  return [_compile_model(WorldModel(s, seed, shared), config) for s, seed in zip(settings_list, seeds)]


def _compile_model(model: WorldModel, config: Optional[Any]) -> bytes:
  """The blob of one world model."""
  rewarded = model.avatar_roles & model.rewarded_roles
  if rewarded:
    raise NotImplementedError(f'RoleBasedRewardTile paying roles {sorted(rewarded)} is not supported by the CUDA engine')
  P = model.num_players
  meta = np.zeros(META_COUNT, np.int32)
  atlas = model.sprites.atlas()
  action_set = [dict(a) for a in _plain(config.action_set)] if config is not None else []
  fields = sorted({ACTION_FIELDS[k] for a in action_set for k in a}) or [0, 1]
  n_fields = max(fields) + 1
  action_table = np.zeros((max(len(action_set), 1), 4), np.int32)
  for i, a in enumerate(action_set):
    for k, v in a.items():
      action_table[i, ACTION_FIELDS[k]] = int(v)
  indiv = list(config.individual_observation_names) if config is not None else ['RGB']
  globs = list(config.global_observation_names) if config is not None else ['WORLD.RGB']
  scalar_obs = []
  for name in indiv:
    if name == 'RGB':
      continue
    if name not in SCALAR_OBS:
      raise NotImplementedError(f'observation {name!r}')
    scalar_obs.append(SCALAR_OBS[name])
  for name in globs:
    if name != 'WORLD.RGB':
      raise NotImplementedError(f'global observation {name!r}')
  vals = dict(FAMILY=FAMILY[model.family], W=model.W, H=model.H,
              L=len(model.layers), P=P, SPRITE_SIZE=model.sprite_size,
              TOPOLOGY=model.topology, MAX_FRAMES=model.max_frames,
              N_OBJECTS=len(model.objects), N_KINDS=len(model.kinds),
              N_STATES=len(model.states), N_COMPS=len(model.comps_i),
              N_SPRITES=len(model.sprites.names), N_HITS=len(model.hits),
              N_GROUPS=len(model.groups), VIEW_LEFT=model.view[0],
              VIEW_RIGHT=model.view[1], VIEW_FORWARD=model.view[2],
              VIEW_BACKWARD=model.view[3], N_ACTIONS=len(action_set),
              N_ACTION_FIELDS=n_fields,
              OOB_SPRITE=model.sprites.index('OutOfBounds'),
              OOV_SPRITE=model.sprites.index('OutOfView'),
              N_SCALAR_OBS=len(scalar_obs))
  for k, v in vals.items():
    meta[META[k]] = v
  opaque = (atlas[..., 3] == 255).all(axis=(1, 2, 3)).astype(np.uint8)
  sections: Dict[str, Any] = {
      'meta': meta,
      'atlas': atlas.reshape(len(model.sprites.names), 4, -1),
      'sprite_opaque': opaque,
      'states': np.array(model.states, np.int32),
      'kinds': np.array(model.kinds, np.int32),
      'comps': np.array(model.comps_i, np.int32),
      'comps_f': np.array(model.comps_d, np.float64),
      'objects': np.array(model.objects, np.int32),
      'hits': np.array([[model.layers.index(h[1]), model.sprites.index(h[2])]
                        for h in model.hits], np.int32).reshape(-1, 2),
      'action_table': action_table,
      'sprite_map': model.sprite_map_table(),
      'scalar_obs': np.array(scalar_obs, np.int32),
      'init_grid': model.init_grid(),
  }
  if model.choice_options:
    sections['choice_groups'] = np.array(model.choice_options, np.int32)
    sections['obj_choice'] = np.array(model.obj_choice, np.int32).reshape(-1, 2)
  _avatar_tables(model, sections)
  if model.family == 'clean_up':
    _clean_up_tables(model, sections)
  elif model.family == 'commons_harvest':
    _commons_tables(model, sections)
  elif model.family == 'territory':
    _territory_tables(model, sections)
  elif model.family == 'coins':
    _coins_tables(model, sections)
  elif model.family == 'coop_mining':
    _mining_tables(model, sections)
  info = dict(
      level=model.level, family=model.family, layers=model.layers,
      sprites=model.sprites.names, groups=model.groups,
      hits=[h[0] for h in model.hits], kinds=model.kind_names,
      kind_states=model.state_names, num_players=P,
      individual_observation_names=indiv, global_observation_names=globs,
      action_set=action_set,
      world_rgb_shape=[model.H * model.sprite_size, model.W * model.sprite_size, 3],
      rgb_shape=[(model.view[2] + model.view[3] + 1) * model.sprite_size,
                 (model.view[0] + model.view[1] + 1) * model.sprite_size, 3],
      valid_roles=sorted(config.valid_roles) if config is not None else [],
      default_player_roles=list(config.default_player_roles) if config is not None else [],
  )
  sections['info_json'] = json.dumps(info)
  return blob_lib.pack(sections)


def compile_substrate(name: str, roles: Optional[Sequence[str]] = None,
                      root: Optional[str] = None,
                      build_seed: Optional[int] = None,
                      prefab_overrides: Optional[Mapping[str, Any]] = None) -> bytes:
  """Compiles a named reference substrate (needs a reference checkout), with the reference's `prefab_overrides`."""
  config = load_reference_config(name, root)
  roles = tuple(roles) if roles is not None else tuple(config.default_player_roles)
  # Some builders draw from Python's global `random` (coins.py:45-84,488: map size and the two coin types):
  # with a build seed the draw is reproducible (policy A.20), without one it is the reference's behaviour.
  state = random.getstate()
  try:
    if build_seed is not None:
      random.seed(build_seed)
    settings = config.lab2d_settings_builder(roles=roles, config=config)
  finally:
    random.setstate(state)
  return compile_settings(settings, config, build_seed, prefab_overrides)


def compile_substrate_set(name: str, roles: Optional[Sequence[str]] = None,
                          build_seeds: Sequence[Optional[int]] = (0,),
                          root: Optional[str] = None,
                          prefab_overrides: Optional[Sequence[Optional[Mapping[str, Any]]]] = None) -> List[bytes]:
  """The builds of a named reference substrate under `build_seeds` and `prefab_overrides` (what compile_substrate
  returns for each pair) as a draw set on one sprite table (compile_settings_set). Needs a reference checkout."""
  config = load_reference_config(name, root)
  roles = tuple(roles) if roles is not None else tuple(config.default_player_roles)
  settings_list = []
  state = random.getstate()
  try:
    for seed in build_seeds:
      if seed is not None:
        random.seed(seed)
      settings_list.append(config.lab2d_settings_builder(roles=roles, config=config))
  finally:
    random.setstate(state)
  return compile_settings_set(settings_list, config, list(build_seeds), prefab_overrides)


def compile_substrate_maps(name: str, roles: Optional[Sequence[str]], maps: Sequence[str],
                           root: Optional[str] = None) -> List[bytes]:
  """The builds of a named reference substrate with each of `maps` as its ASCII map, as one map set on one sprite table
  (compile_settings_set). A territory map replaces `config.layout.ascii_map`, which territory.py's builder turns into
  the level's map; any other substrate's (coop_mining) replaces the map of its lab2d settings. Needs a reference
  checkout."""
  config = load_reference_config(name, root)
  roles = tuple(roles) if roles is not None else tuple(config.default_player_roles)
  settings_list = []
  for ascii_map in maps:
    if 'layout' in config and 'ascii_map' in config.layout:
      config.layout.ascii_map = ascii_map
      settings_list.append(config.lab2d_settings_builder(roles=roles, config=config))
    else:
      settings = config.lab2d_settings_builder(roles=roles, config=config)
      settings['simulation']['map'] = ascii_map
      settings_list.append(settings)
  return compile_settings_set(settings_list, config)
