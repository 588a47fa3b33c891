"""The blob layout is declared once, in include/mpb_format.h: the compiler's mirrors of it must agree with the header,
and every value the compiler writes into a family parameter block must sit in a named slot."""

import glob
import os
import re

import pytest

from meltingpot_b200 import blob as blob_lib
from meltingpot_b200 import compiler

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_HEADER = os.path.join(_ROOT, 'include', 'mpb_format.h')
_BLOBS = sorted(glob.glob(os.path.join(_ROOT, 'meltingpot_b200', 'data', '*.mpb')) +
                glob.glob(os.path.join(_ROOT, 'tests', 'golden', '*.mpb')))
_BLOCKS = {'FP': compiler.FP, 'CU_I': compiler.CU_I, 'CU_D': compiler.CU_D, 'CH_I': compiler.CH_I,
           'CH_D': compiler.CH_D, 'TR_I': compiler.TR_I, 'TR_D': compiler.TR_D, 'CO_I': compiler.CO_I,
           'CO_D': compiler.CO_D, 'CM_I': compiler.CM_I, 'CM_D': compiler.CM_D}


def _header():
  """MPB_<NAME> -> value of every `MPB_<NAME> = <n>` enumerator and `#define MPB_<NAME> <n>` of the header."""
  with open(_HEADER) as f:
    text = re.sub(r'/\*.*?\*/', '', f.read(), flags=re.S)
  out = {m[0]: int(m[1]) for m in re.findall(r'\b(MPB_\w+)\s*=\s*(-?\d+)', text)}
  out.update({m[0]: int(m[1]) for m in re.findall(r'#define\s+(MPB_\w+)\s+(\d+)u?\b', text)})
  return out


def _with_prefix(prefix):
  return {k[len(prefix):]: v for k, v in _header().items() if k.startswith(prefix)}


def _snake(camel):
  return re.sub(r'(?<!^)(?=[A-Z])', '_', camel).upper()


def test_named_mirrors_match_the_header():
  assert _with_prefix('MPB_META_') == dict(compiler.META, COUNT=compiler.META_COUNT)
  assert _with_prefix('MPB_FAMILY_') == {k.upper(): v for k, v in compiler.FAMILY.items()}
  for block, layout in _BLOCKS.items():
    assert _with_prefix(f'MPB_{block}_') == layout, block
  h = _header()
  assert (h['MPB_COMP_NI'], h['MPB_COMP_ND']) == (compiler.COMP_NI, compiler.COMP_ND)


def test_lua_keyed_mirrors_have_the_header_ids():
  names = {'ReadyToShootObservation': 'READY_TO_SHOOT'}
  assert {names.get(k, _snake(k)): v for k, v in compiler.COMP.items()} == _with_prefix('MPB_C_')
  fields = _with_prefix('MPB_ACT_')
  field_of = {'move': 'MOVE', 'turn': 'TURN', 'fireZap': 'FIRE_ZAP', 'mine': 'FIRE_ZAP', 'fireClean': 'FIRE_2',
              'fireClaim': 'FIRE_2'}
  assert {k: fields[field_of[k]] for k in compiler.ACTION_FIELDS} == compiler.ACTION_FIELDS
  obs = _with_prefix('MPB_OBS_')
  obs_of = {'READY_TO_SHOOT': 'READY_TO_SHOOT', 'NUM_OTHERS_WHO_CLEANED_THIS_STEP': 'NUM_OTHERS_WHO_CLEANED',
            'MISMATCHED_COIN_COLLECTED_BY_PARTNER': 'MISMATCHED_COIN_BY_PARTNER'}
  assert {k: obs[obs_of[k]] for k in compiler.SCALAR_OBS} == compiler.SCALAR_OBS
  assert sorted(obs.values()) == sorted(compiler.SCALAR_OBS.values())


@pytest.mark.parametrize('family', sorted(compiler.FAMILY_PARAMS))
def test_family_slots_are_distinct_and_fit_their_blocks(family):
  _, ints, floats = compiler.FAMILY_PARAMS[family]
  for layout in (ints, floats):
    slots = [v for k, v in layout.items() if k != 'COUNT']
    assert len(set(slots)) == len(slots), f'{family}: two names share a slot'
    assert all(0 <= v < layout['COUNT'] for v in slots), family
  assert not (set(ints) - {'COUNT'}) & (set(floats) - {'COUNT'}), f'{family}: a name in both blocks'


@pytest.mark.parametrize('path', _BLOBS, ids=os.path.basename)
def test_every_written_slot_of_a_blob_has_a_name(path):
  with open(path, 'rb') as f:
    sec = blob_lib.unpack(f.read())
  family = {v: k for k, v in compiler.FAMILY.items()}[int(sec['meta'][compiler.META['FAMILY']])]
  prefix, ints, floats = compiler.FAMILY_PARAMS[family]
  for suffix, layout in (('_ip', ints), ('_dp', floats)):
    block = sec[prefix + suffix]
    assert block.shape == (layout['COUNT'],)
    named = {v for k, v in layout.items() if k != 'COUNT'}
    assert [i for i in range(len(block)) if block[i] != 0 and i not in named] == [], prefix + suffix
  assert set(compiler.family_params(sec)) == (set(ints) | set(floats)) - {'COUNT'}
