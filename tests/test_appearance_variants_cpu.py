"""Appearance overrides in one heterogeneous batch: prefab_overrides that change how pieces look, compiled as one set on
one sprite table (compiler.compile_settings_set), and the compatibility check of mp_create_variants, which runs before
any device is touched."""

import ctypes
import re

import numpy as np
import pytest

from meltingpot_b200 import blob as blob_lib
from meltingpot_b200 import compiler
from tests import appearance_variants as AV
from tests import env_variants as EV
from tests import variants as V

SPRITE_SIDE = ('atlas', 'sprite_opaque', 'sprite_map', 'hits')


def _sections(blob):
  return blob_lib.unpack(blob)


@pytest.mark.parametrize('family', EV.NAMES)
def test_the_env_variant_lists_compile_byte_identically_as_a_set_and_apart(family):
  sub, players, seed, rows = EV.FAMILIES[family]
  settings = [EV.settings(family, edits) for _, edits in rows]
  got = compiler.compile_settings_set(settings, EV.settings_golden.config(sub, players), [seed] * len(rows),
                                      [o for o, _ in rows])
  assert tuple(got) == EV.blobs(family)


@pytest.mark.parametrize('name', AV.NAMES)
def test_a_set_of_one_is_compile_settings(name):
  seed = AV.SUBSTRATES[name][1]
  for o, alone in zip(AV.overrides(name), AV.alone(name)):
    assert compiler.compile_settings_set([AV.settings(name)], AV.config(name), [seed], [o]) == [alone]


def _sprite_refs(sec):
  """Every sprite id a blob's tables refer to, as (what, id) pairs: states, avatars, beam hits, the family's sprite slots
  and its tables of sprite ids."""
  refs = [('state', int(s)) for s in sec['states'][:, 1] if s >= 0]
  refs += [('avatar', int(s)) for s in sec['av_table'][:, 1]]
  refs += [('hit', int(s)) for s in sec['hits'][:, 1]]
  refs += [(k, int(v)) for k, v in sorted(compiler.family_params(sec).items()) if 'SPRITE' in k and v >= 0]
  for k in ('cu_water_sprites', 'tr_player_sprites'):
    if k in sec:
      refs += [(k, int(v)) for v in np.asarray(sec[k]).reshape(-1)]
  return refs


@pytest.mark.parametrize('name', AV.NAMES)
def test_an_appearance_set_shares_its_sprite_table_and_every_entry_shows_its_own_pixels(name):
  sets = [_sections(b) for b in AV.blobs(name)]
  alone = [_sections(b) for b in AV.alone(name)]
  for sec in sets[1:]:
    for k in SPRITE_SIDE:
      assert np.array_equal(sec[k], sets[0][k]), k
    for f in ('N_SPRITES', 'OOB_SPRITE', 'OOV_SPRITE'):
      assert sec['meta'][compiler.META[f]] == sets[0]['meta'][compiler.META[f]], f
  for v, (s, a) in enumerate(zip(sets, alone)):
    rs, ra = _sprite_refs(s), _sprite_refs(a)
    assert [w for w, _ in rs] == [w for w, _ in ra]
    for (what, i), (_, j) in zip(rs, ra):
      assert np.array_equal(s['atlas'][i], a['atlas'][j]), f'variant {v}: {what} sprite {i} / {j}'
    gs, ga = s['init_grid'].reshape(-1), a['init_grid'].reshape(-1)
    assert np.array_equal(np.flatnonzero(gs), np.flatnonzero(ga)) and np.array_equal((gs - 1) & 3, (ga - 1) & 3)
    for i, j in np.unique(np.stack([gs, ga], 1)[gs != 0], axis=0):
      assert np.array_equal(s['atlas'][(i - 1) >> 2], a['atlas'][(j - 1) >> 2]), f'variant {v}: initial cell sprite {i} / {j}'
  # the overrides really change pixels: each entry refers to a sprite no other entry refers to
  ids = [{i for _, i in _sprite_refs(s)} | {int(g - 1) >> 2 for g in np.unique(s['init_grid']) if g} for s in sets]
  for v in range(1, len(sets)):
    assert ids[v] - ids[0], f'variant {v} shows nothing stock does not'
  # the stock entry's blob is its stand-alone blob apart from the sprite table the others add to
  assert sets[0]['atlas'].shape[0] > alone[0]['atlas'].shape[0]
  assert EV.differing_sections(AV.blobs(name)[0], AV.alone(name)[0]) == ['atlas', 'info_json', 'meta', 'sprite_map',
                                                                          'sprite_opaque']


def test_compile_settings_set_checks_the_length_of_prefab_overrides():
  with pytest.raises(ValueError, match='2 prefab_overrides for 1 settings entries'):
    compiler.compile_settings_set([AV.settings('coins')], AV.config('coins'), [0], [{}, {}])


# --- the section check of mp_create_variants (no device needed: it runs before the device is opened, as do the Params
# checks that follow it, tests/test_create_checks_cpu.py) ---
MP_E_UNSUPPORTED, MP_E_NO_DEVICE = -2, -4


def _create(blobs):
  """mp_create_variants' return code and message."""
  from meltingpot_b200 import engine
  lib = engine.load_library()
  arr = (ctypes.c_char_p * len(blobs))(*blobs)
  sizes = (ctypes.c_size_t * len(blobs))(*[len(b) for b in blobs])
  h = ctypes.c_void_p()
  rc = lib.mp_create_variants(arr, sizes, len(blobs), None, 4, 0, ctypes.c_uint64(1), ctypes.c_uint64(0),
                              ctypes.c_uint32(0), ctypes.byref(h))
  if rc == 0:
    lib.mp_destroy(h)
  return rc, lib.mp_last_error().decode()


def _no_gpu():
  import torch
  if torch.cuda.is_available():
    pytest.skip('a GPU is present: tests/test_gpu_appearance_variants.py covers the engine')


@pytest.mark.parametrize('name', AV.NAMES)
def test_the_check_passes_an_appearance_set(name):
  _no_gpu()
  rc, msg = _create(list(AV.blobs(name)))
  assert rc == MP_E_NO_DEVICE, msg


_CU_APPLE = {'potential_apple': {'Appearance': {'palettes': [{'x': [0, 0, 0, 0], '*': [12, 80, 57, 255]}]}}}


def _refused():
  cu = 'clean_up'
  return [
      # today's messages: a shape difference next to an appearance override
      ('map', cu, V.map_replace('F', 'H'), r"section '\w+' differs \(variants may differ only in the family's parameters\)"),
      ('view', cu, V.view(2, 2, 2, 2), "section 'meta' differs"),
      ('episode_cap', cu, V.top(maxEpisodeLengthFrames=50), "section 'meta' differs in|section 'meta' differs"),
  ]


@pytest.mark.parametrize('row', _refused(), ids=lambda r: r[0])
def test_shape_changes_are_still_refused_with_todays_messages(row):
  _no_gpu()
  _, family, edit, what = row
  sub, players, seed, _ = EV.FAMILIES[family]
  s = [EV.settings(family), EV.settings(family, [edit])]
  recolour = {'potential_apple': AV.recoloured(s[0], 'potential_apple')} if family == 'clean_up' else {}
  blobs = compiler.compile_settings_set(s, EV.settings_golden.config(sub, players), [seed] * 2, [recolour, {}])
  rc, msg = _create(blobs)
  assert rc == MP_E_UNSUPPORTED
  assert re.search(f'variant 1: .*{what}', msg), msg


def test_blobs_compiled_apart_are_still_refused():
  _no_gpu()
  rc, msg = _create([AV.alone('clean_up')[0], AV.alone('clean_up')[1]])
  assert rc == MP_E_UNSUPPORTED and re.search("variant 1: section '(atlas|sprite_opaque)'", msg), msg


# --- build_batched: argument errors come before an engine (or a compile) exists ---
def _build(**kw):
  from meltingpot_b200 import substrate
  args = dict(roles=['default'] * 7, num_envs=4, prefab_overrides=[{}, _CU_APPLE])
  args.update(kw)
  return substrate.build_batched('clean_up', **args)


@pytest.mark.parametrize('kw, what', [
    (dict(prefab_overrides=[]), 'the sequence of prefab_overrides is empty'),
    (dict(prefab_overrides=[{}, 'apple']), r'prefab_overrides\[1\] is a str, not a mapping'),
    (dict(env_variant=[0, 1, 0]), 'env_variant has 3 entries for 4 envs'),
    (dict(env_variant=[0, 1, 2, 0]), r'env_variant must index the 2 prefab_overrides \(0..1\)'),
    (dict(env_variant=[0, -1, 0, 0]), 'env_variant must index'),
    (dict(prefab_overrides={'apple': {}}, env_variant=[0, 0, 0, 0]), 'env_variant needs a sequence of prefab_overrides'),
], ids=['empty', 'not_a_mapping', 'env_variant_length', 'env_variant_range', 'env_variant_negative', 'mapping_with_env_variant'])
def test_build_batched_checks_its_arguments_before_creating_an_engine(kw, what, monkeypatch):
  from meltingpot_b200 import substrates

  def no_compile(*a, **k):
    raise AssertionError('compiled before the arguments were checked')

  monkeypatch.setattr(substrates, 'compile_with_overrides', no_compile)
  with pytest.raises(ValueError, match=what):
    _build(**kw)


def test_build_batched_compiles_a_sequence_as_one_set(monkeypatch):
  from meltingpot_b200 import substrate, substrates
  seen = {}
  monkeypatch.setattr(compiler, 'reference_root', lambda: '/nonexistent')
  monkeypatch.setattr(compiler, 'compile_substrate_set',
                      lambda name, roles, seeds, prefab_overrides=None: seen.update(set=(name, seeds, prefab_overrides)) or [b'a', b'b'])
  monkeypatch.setattr(compiler, 'compile_substrate',
                      lambda name, roles, build_seed=None, prefab_overrides=None: seen.update(one=(name, prefab_overrides)) or b'c')

  class Stop(Exception):
    pass

  def fake(blob, num_envs, **kw):
    seen['blob'] = blob
    raise Stop

  monkeypatch.setattr(substrate, 'BatchedSubstrate', fake)
  with pytest.raises(Stop):
    _build(env_variant=[1, 0, 1, 0])
  assert seen['set'] == ('clean_up', [None, None], [{}, _CU_APPLE]) and seen['blob'] == [b'a', b'b']
  with pytest.raises(Stop):
    _build(prefab_overrides=_CU_APPLE)
  assert seen['one'] == ('clean_up', _CU_APPLE) and seen['blob'] == b'c'
  assert substrates.compile_with_overrides('coins', ('default',) * 2, [{}]) == [b'a', b'b']
  assert seen['set'] == ('coins', [0], [{}])
