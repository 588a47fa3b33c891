"""mp_create and mp_create_variants check every blob before they open a device, so a refused blob is refused with its own
code and message on any machine, with or without a GPU. Valid blobs get as far as the device: without one, mp_create
returns MP_E_NO_DEVICE. The GPU tests (test_gpu_param_envelope.py, test_gpu_env_variants.py,
test_gpu_appearance_variants.py) check the same refusals through the Python engine."""

import ctypes
import re

import numpy as np
import pytest

from meltingpot_b200 import blob as mpb
from meltingpot_b200 import compiler
from tests import appearance_variants as AV
from tests import commons_maps as CM
from tests import env_variants as EV
from tests import variants as V

MP_E_INVALID, MP_E_UNSUPPORTED, MP_E_NO_DEVICE = -1, -2, -4


def _create(blobs):
  """The return code and message of mp_create (one blob) or mp_create_variants (a list)."""
  from meltingpot_b200 import engine
  lib = engine.load_library()
  h = ctypes.c_void_p()
  args = (4, 0, ctypes.c_uint64(1), ctypes.c_uint64(0), ctypes.c_uint32(0), ctypes.byref(h))
  if isinstance(blobs, bytes):
    rc = lib.mp_create(blobs, ctypes.c_size_t(len(blobs)), *args)
  else:
    arr = (ctypes.c_char_p * len(blobs))(*blobs)
    sizes = (ctypes.c_size_t * len(blobs))(*[len(b) for b in blobs])
    rc = lib.mp_create_variants(arr, sizes, len(blobs), None, *args)
  if rc == 0:
    lib.mp_destroy(h)
  return rc, lib.mp_last_error().decode()


# The render-kernel instantiation refuses a view wider than 16 cells. It is chosen with the render layout, after the
# device is checked, so without a device that variant gets MP_E_NO_DEVICE.
_AFTER_THE_DEVICE = ('view_17',)


@pytest.mark.parametrize('name', [v.name for v in V.REFUSED if v.refused_by == 'engine'
                                  and not v.name.endswith(_AFTER_THE_DEVICE)])
def test_a_refused_variant_is_refused_before_the_device(name):
  rc, msg = _create(V.compile(name))
  assert rc == MP_E_UNSUPPORTED, msg


@pytest.mark.parametrize('substrate,players,seed,section', [('clean_up', 7, None, 'cu_dirt'),
                                                            ('commons_harvest__open', 7, None, 'ch_apple'),
                                                            ('territory__rooms', 9, None, 'tr_res'), ('coins', 2, 0, 'co_coin'),
                                                            ('coop_mining', 6, None, 'cm_ore')])
def test_an_entity_table_short_or_off_the_map_is_refused_before_the_device(substrate, players, seed, section):
  sec = mpb.unpack(V.stock(substrate, players, seed))
  short = dict(sec)
  short[section] = sec[section][:-1]
  off_map = dict(sec)
  off_map[section] = sec[section].copy()
  off_map[section][-1, 1] = int(sec['meta'][1]) * int(sec['meta'][2])  # W * H: one past the last cell
  for bad, what in ((short, r'has \d+ values for'), (off_map, 'puts entity')):
    rc, msg = _create(mpb.pack(bad))
    assert rc == MP_E_INVALID and re.match(f"blob: section '{section}' {what}", msg), msg


def _params_refusals():
  cu = 'clean_up'
  return [
      ('zap_beam', cu, V.kw('Zapper', beamLength=9, beamRadius=0), "Params field 'zap.geom' differs"),
      ('clean_beam', cu, V.kw('Cleaner', beamLength=9, beamRadius=0), "Params field 'clean_geom' differs"),
      ('clean_beam_cells', cu, V.kw('Cleaner', beamLength=2), 'beam footprints differ'),
      ('episode_ending', cu, V.kw('StochasticIntervalEpisodeEnding', probabilityTerminationPerInterval=0.5),
       'episode ending differs'),
      ('marking_levels', 'territory',
       V.marking_levels([dict(levelIncrement=0, sourceReward=0.25, targetReward=-0.5, freeze=2)], 1),
       "Params field 'mark_n_levels' differs"),
      ('own_loader', cu, V.kw('Zapper', cooldownTime=0), 'non-positive zap cooldown'),
  ]


@pytest.mark.parametrize('row', _params_refusals(), ids=lambda r: r[0])
def test_a_variant_whose_params_do_not_fit_is_refused_before_the_device(row):
  _, family, edit, what = row
  bad = EV.compile_settings(family, EV.settings(family, [edit]))
  rc, msg = _create([EV.blobs(family)[0], bad])
  assert rc == MP_E_UNSUPPORTED and msg.startswith(f'variant 1: {what}'), msg


@pytest.mark.parametrize('edit, what', [(V.kw('Zapper', beamLength=9, beamRadius=0), "Params field 'zap.geom' differs"),
                                        (V.kw('Cleaner', beamLength=2), 'beam footprints differ')], ids=['zap_beam', 'beam_cells'])
def test_a_shape_change_next_to_an_appearance_override_is_refused_before_the_device(edit, what):
  s = AV.settings('clean_up')
  recolour = {'potential_apple': AV.recoloured(s, 'potential_apple')}
  blobs = compiler.compile_settings_set([s, EV.settings('clean_up', [edit])], AV.config('clean_up'), [None, None],
                                        [recolour, {}])
  rc, msg = _create(blobs)
  assert rc == MP_E_UNSUPPORTED and msg.startswith(f'variant 1: {what}'), msg


def test_a_variant_loader_refusal_comes_after_the_checks_of_blob_0():
  # Blob 0's own checks run through to its render tables first; a variant's loader refusal is reported after them, with
  # the variant's other checks. Here blob 0 carries 'choice' prefabs, which only territory supports.
  good = EV.blobs('clean_up')[0]
  bad = EV.compile_settings('clean_up', EV.settings('clean_up', [V.kw('Zapper', cooldownTime=0)]))
  with_choice = []
  for b in (good, bad):
    sec = mpb.unpack(b)
    sec['choice_groups'] = np.array([2], np.int32)
    with_choice.append(mpb.pack(sec))
  rc, msg = _create(with_choice)
  assert rc == MP_E_UNSUPPORTED and msg.startswith("per-env 'choice' prefabs are implemented for the territory family"), msg
  rc, msg = _create([good, bad])
  assert rc == MP_E_UNSUPPORTED and msg == 'variant 1: non-positive zap cooldown', msg


def _no_gpu():
  import torch
  if torch.cuda.is_available():
    pytest.skip('a GPU is present: the GPU tests create these engines')


@pytest.mark.parametrize('blobs', [lambda: V.stock('clean_up', 7, None), lambda: list(EV.blobs('coop_mining')),
                                   lambda: list(CM.map_set())], ids=['single_blob', 'variant_set', 'map_set'])
def test_valid_blobs_get_as_far_as_the_device(blobs):
  _no_gpu()
  rc, msg = _create(blobs())
  assert rc == MP_E_NO_DEVICE, msg
