"""commons_harvest__open, __closed and __partnership as one map set (tests/commons_maps.py), without a GPU: the committed
blobs form the set, the sections they differ in are pinned, and build_batched over a sequence of names checks its
arguments before any engine exists."""

import numpy as np
import pytest

from meltingpot_b200 import substrate, substrates
from tests import commons_maps as CM
from tests import env_variants as EV

# What the maps of the set differ in (every other section is byte-identical across the set).
DIFFERS_FROM_OPEN = {
    'commons_harvest__closed': ['cell_flags', 'ch_dp', 'ch_ip', 'comps', 'comps_f', 'init_grid', 'objects'],
    'commons_harvest__partnership': ['cell_flags', 'ch_apple', 'ch_dp', 'ch_ip', 'comps', 'comps_f', 'info_json', 'init_grid',
                                     'kinds', 'meta', 'objects', 'states'],
}


def test_the_recorded_settings_compiled_as_one_set_are_the_committed_blobs():
  blobs = CM.map_set(capped=False)
  for name, blob in zip(CM.NAMES, blobs):
    assert blob == substrates.load_blob(name, CM.ROLES), name


def test_the_sections_the_maps_differ_in_are_pinned():
  from meltingpot_b200 import blob as blob_lib
  committed = [substrates.load_blob(n, CM.ROLES) for n in CM.NAMES]
  for name, blob in zip(CM.NAMES[1:], committed[1:]):
    assert EV.differing_sections(committed[0], blob) == DIFFERS_FROM_OPEN[name], name
  sec = [blob_lib.unpack(b) for b in committed]
  # partnership: one more kind (an inert reward tile) and state; the apples stand on the same cells
  assert [int(s['meta'][9]) for s in sec] == [14, 14, 15] and [int(s['meta'][10]) for s in sec] == [37, 37, 38]
  assert all(np.array_equal(s['ch_apple'][:, [1, 2]], sec[0]['ch_apple'][:, [1, 2]]) for s in sec)
  assert all(np.array_equal(s['ch_nbr'], sec[0]['ch_nbr']) for s in sec)
  # the Zapper: open's beam is 3 cells long, closed's and partnership's 4
  assert [int(s['ch_ip'][13]) for s in sec] == [3, 4, 4]


def _build(**kw):
  args = dict(roles=CM.ROLES, num_envs=4)
  args.update(kw)
  return substrate.build_batched(args.pop('name', CM.NAMES), **args)


@pytest.mark.parametrize('kw,what', [
    (dict(name=()), 'empty'),
    (dict(name=list(CM.NAMES)[:1], prefab_overrides={}), 'neither prefab_overrides nor build_seeds'),
    (dict(build_seeds=[0]), 'neither prefab_overrides nor build_seeds'),
    (dict(env_variant=[0, 1, 2]), 'env_variant has 3 entries for 4 envs'),
    (dict(env_variant=[0, 1, 2, 3]), r'env_variant must index the 3 names \(0..2\)'),
    (dict(env_variant=[0, -1, 2, 1]), r'env_variant must index the 3 names'),
    (dict(roles=('other',) * 7), 'Invalid roles'),
    (dict(name=('commons_harvest__open', 'clean_up')), "'clean_up' differs from 'commons_harvest__open' in its action_set"),
    (dict(name=('commons_harvest__open', 'no_such_substrate')), 'no_such_substrate not in'),
], ids=['empty', 'overrides', 'build_seeds', 'env_variant_length', 'env_variant_range', 'env_variant_negative', 'roles',
        'action_set', 'unknown_name'])
def test_build_batched_over_names_checks_its_arguments_before_creating_an_engine(kw, what):
  with pytest.raises(ValueError, match=what):
    _build(**kw)


def test_a_mixed_batch_fails_loudly_without_gpu():
  import torch
  if torch.cuda.is_available():
    pytest.skip('a GPU is present')
  from meltingpot_b200 import engine
  with pytest.raises(engine.EngineError, match='no CPU path'):
    _build()
  with pytest.raises(engine.EngineError, match='no CPU path'):
    _build(name=CM.NAMES + CM.NAMES[:1], env_variant=[3, 2, 1, 0])
