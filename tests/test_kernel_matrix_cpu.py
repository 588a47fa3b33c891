"""What tests/test_gpu_kernel_matrix.py enumerates, checked without a device: the launch ledger's C ABI, the k_step
cells against the engine's kernel table, and the variant sets whose cells are meant to run different maps."""

import os
import re

import pytest

from meltingpot_b200 import blob as blob_lib
from meltingpot_b200 import engine
from tests import env_variants as EV
from tests import test_gpu_kernel_matrix as KM

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _read(*path):
  with open(os.path.join(ROOT, *path)) as f:
    return f.read()


def test_last_launch_abi():
  header = _read('include', 'mp_engine.h')
  assert re.search(r'int mp_debug_last_launch\(mp_handle h, int32_t out\[MP_LAST_LAUNCH_FIELDS\]\);', header)
  n = int(re.search(r'#define MP_LAST_LAUNCH_FIELDS (\d+)', header).group(1))
  assert n == len(engine.Engine.LAST_LAUNCH_FIELDS) == 10
  assert 'mp_debug_last_launch' in engine.EXPORTED_SYMBOLS
  assert hasattr(engine.load_library(), 'mp_debug_last_launch')


def test_enumerated_cells_are_the_kernel_table_plus_the_inside_out_row():
  src = _read('meltingpot_b200', 'csrc', 'engine.cu')
  dims = tuple(int(d) for d in re.search(r'const void\* step\[(\d+)\]\[(\d+)\]\[(\d+)\];', src).groups())
  assert dims == (2, 2, 3)
  table = re.search(r'const FamilyEntry kFamilies\[\] = \{(.*?)\};', src, re.S).group(1)
  names = re.findall(r'family_entry<\w+>\((MPB_FAMILY_\w+)\)', table)
  ids = dict(re.findall(r'(MPB_FAMILY_\w+) = (\d+)', _read('include', 'mpb_format.h')))
  families = {int(ids[n]) for n in names}
  assert len(families) == len(names) == 5
  want = {(f, v, r, a) for f in families for v in range(dims[0]) for r in range(dims[1]) for a in range(dims[2])}
  assert KM.step_cells() == want and len(want) == 60
  assert set(KM.FAMILY_IDS.values()) == families
  # one test per row: the five families and territory__inside_out, a territory row of its own
  assert len(KM.ROWS) == 6 and KM.ROWS['territory__inside_out'] == KM.ROWS['territory__rooms'] == 'territory'
  assert sorted(set(KM.ROWS.values())) == sorted(KM.FAMILY_IDS)
  assert {(n, w) for n, w in KM.RENDER_INSTS} == {(3, 3), (3, 4), (3, 5), (4, 5)}
  for ncp, ncw in KM.RENDER_INSTS:
    assert f'MP_RENDER_INST({ncp}, {ncw})' in src


@pytest.mark.parametrize('row', sorted(KM.ENTITY_SECTIONS))
def test_every_map_set_differs_in_its_map_sections(row):
  blobs = KM.variant_set(row)
  assert len(blobs) >= 3
  maps = set()
  for i, a in enumerate(blobs):
    for b in blobs[i + 1:]:
      assert EV.differing_sections(a, b), f'{row}: two variants are one blob'
    sec = blob_lib.unpack(a)
    maps.add(b''.join(sec[k].tobytes() for k in ('init_grid', 'objects', KM.ENTITY_SECTIONS[row])))
  # every variant plays a map of its own; coins' draws repeat a map size with other coin colours, so there at least
  # the smallest and the largest map
  assert len(maps) == len(blobs) if row != 'coins' else len(maps) >= 2, f'{row}: {len(blobs)} variants on {len(maps)} maps'
