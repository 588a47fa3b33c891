"""prefab_overrides in the compiler, the variant blobs of tests/env_variants.py and the sharded slicing of env_variant."""

import copy

import numpy as np
import pytest

from meltingpot_b200 import blob as blob_lib
from meltingpot_b200 import compiler
from tests import env_variants as EV
from tests import settings_golden

_PARAM_SECTIONS = {'comps', 'comps_f', 'info_json'}


def test_apply_prefab_overrides_sets_the_first_named_component_only():
  s = settings_golden.settings('coop_mining', 6)
  before = copy.deepcopy(s)
  overrides = {'ore': {'Ore': {'miningWindow': 7}}}
  frozen = copy.deepcopy(overrides)
  out = compiler.apply_prefab_overrides(s, overrides)
  ores = [c for c in out['simulation']['prefabs']['ore']['components'] if c['component'] == 'Ore']
  assert len(ores) == 2
  assert ores[0]['kwargs']['miningWindow'] == 7
  assert ores[1]['kwargs'] == [c for c in before['simulation']['prefabs']['ore']['components'] if c['component'] == 'Ore'][1]['kwargs']
  assert s == before and overrides == frozen  # neither argument is modified
  # avatars live in gameObjects: overrides never reach them
  assert out['simulation']['gameObjects'] == before['simulation']['gameObjects']


def test_apply_prefab_overrides_refuses_unknown_prefabs_and_components():
  s = settings_golden.settings('clean_up', 7)
  with pytest.raises(ValueError, match="Prefab override for 'apple' given, but not available in `prefabs`."):
    compiler.apply_prefab_overrides(s, {'apple': {'Edible': {'rewardForEating': 2.0}}})
  with pytest.raises(ValueError, match="No component with name 'DensityRegrow' found."):
    compiler.apply_prefab_overrides(s, {'potential_apple': {'DensityRegrow': {'radius': 2}}})
  assert compiler.apply_prefab_overrides(s, None) == s


def test_compile_settings_applies_overrides_before_the_world_model():
  s = settings_golden.settings('clean_up', 7)
  stock = compiler.compile_settings(s, settings_golden.config('clean_up', 7))
  over = {'potential_apple': {'Edible': {'rewardForEating': 3.5}}}
  blob = compiler.compile_settings(s, settings_golden.config('clean_up', 7), None, over)
  s2 = compiler.apply_prefab_overrides(s, over)
  assert blob == compiler.compile_settings(s2, settings_golden.config('clean_up', 7))
  assert compiler.family_params(blob_lib.unpack(blob))['EAT_REWARD'] == 3.5
  assert blob != stock


@pytest.mark.parametrize('family', EV.NAMES)
def test_variants_differ_only_in_the_parameter_sections(family):
  blobs = EV.blobs(family)
  prefix = compiler.FAMILY_PARAMS[EV.FAMILIES[family][0].split('__')[0]][0]
  allowed = _PARAM_SECTIONS | {f'{prefix}_ip', f'{prefix}_dp'}
  for v, b in enumerate(blobs[1:], 1):
    diff = set(EV.differing_sections(blobs[0], b))
    assert diff and diff <= allowed, (v, diff)
    assert diff & {f'{prefix}_ip', f'{prefix}_dp'}, (v, diff)  # the kernel sees the change


def test_oracle_envs_of_a_mixed_batch_follow_their_own_variant():
  """A mixed batch on the oracle, as the GPU tests build it: per variant one OracleBatch over the variant's env range
  (env b keyed seed + b); each kept row equals an OracleEnv of that variant's blob."""
  from oracle import binding
  binding.build()
  blobs = EV.blobs('clean_up')
  B, seed = 8, 41
  assign = EV.interleaved(B, 4)
  rng = np.random.default_rng(0)
  envs = [binding.OracleEnv(blobs[assign[b]], seed + b) for b in range(B)]
  for e in envs:
    e.reset()
  batches = []
  for v in range(4):
    idx = np.flatnonzero(assign == v)
    lo, hi = idx[0], idx[-1] + 1
    batches.append((idx, lo, hi, binding.OracleBatch(blobs[v], hi - lo, seed=seed + lo)))
  for _ in range(45):
    acts = rng.integers(0, envs[0].n_actions, size=(B, envs[0].P)).astype(np.int32)
    for b, e in enumerate(envs):
      e.step(acts[b])
    for idx, lo, hi, batch in batches:
      batch.step_actions(acts[lo:hi], 2)
  shapes = dict(P=envs[0].P, L=envs[0].L, cells=envs[0].W * envs[0].H, n_scalar=envs[0].n_scalar, rgb=(1, 1), world=(1, 1))
  for idx, lo, _, batch in batches:
    d = batch.dump(2, shapes)
    for b in idx:
      assert np.array_equal(d['grid'][b - lo], envs[b].grid()) and np.array_equal(d['reward'][b - lo], envs[b].rewards())


def test_sharded_substrate_hands_each_rank_its_slice_of_env_variant(monkeypatch):
  import torch.distributed as dist
  from meltingpot_b200 import distributed, substrate
  calls = []
  monkeypatch.setattr(substrate, 'build_batched', lambda name, **kw: calls.append(kw) or object())
  assign = list(range(4)) * 4
  overrides = [{}, {'potential_apple': {'Edible': {'rewardForEating': 2.0}}}]
  for rank in range(2):
    monkeypatch.setattr(dist, 'get_rank', lambda group=None, r=rank: r)
    monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 2)
    distributed.ShardedSubstrate('clean_up', ['default'] * 7, 16, seed=3, device=0, prefab_overrides=overrides,
                                 env_variant=assign)
  assert [c['env_index_base'] for c in calls] == [0, 8] and [c['num_envs'] for c in calls] == [8, 8]
  assert calls[0]['env_variant'] == assign[:8] and calls[1]['env_variant'] == assign[8:]
  assert all(c['prefab_overrides'] is overrides for c in calls)
  with pytest.raises(ValueError):
    distributed.ShardedSubstrate('clean_up', ['default'] * 7, 16, seed=3, device=0, env_variant=assign[:5])


def test_build_batched_with_overrides_needs_a_reference_checkout(monkeypatch):
  from meltingpot_b200 import substrate
  monkeypatch.setattr(compiler, 'reference_root', lambda: None)
  with pytest.raises(FileNotFoundError):
    substrate.build_batched('clean_up', roles=['default'] * 7, num_envs=4,
                            prefab_overrides=[{}, {'potential_apple': {'Edible': {'rewardForEating': 2.0}}}])
  with pytest.raises(ValueError):
    substrate.build_batched('clean_up', roles=['default'] * 7, num_envs=4, env_variant=[0, 0, 0, 0])
