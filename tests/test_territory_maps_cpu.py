"""Map sets of territory and coop_mining (tests/territory_maps.py) without a GPU: what the compiler makes of a set, the
refusals mp_create_variants gives before it opens a device, build_batched(maps=...)'s argument checks, and the oracle of
a mixed batch."""

import numpy as np
import pytest

from meltingpot_b200 import blob as mpb
from meltingpot_b200 import compiler, substrate, substrates
from tests import territory_maps as TM
from tests import variants as V
from tests.test_create_checks_cpu import MP_E_NO_DEVICE, MP_E_UNSUPPORTED, _create


@pytest.mark.parametrize('name', TM.NAMES)
def test_a_set_of_one_map_is_the_committed_blob(name):
  from tests import settings_golden
  s = settings_golden.settings(name, TM.PLAYERS[name])
  assert compiler.compile_settings_set([s], TM.config(name)) == [substrates.load_blob(name, ('default',) * TM.PLAYERS[name])]


@pytest.mark.parametrize('name', TM.NAMES)
def test_each_map_of_a_set_is_the_map_compiled_alone(name):
  blobs = TM.map_set(name)
  sec = [mpb.unpack(b) for b in blobs]
  table = 'cm_ore' if name == 'coop_mining' else 'tr_res'
  counts = [len(s[table]) for s in sec]
  assert len(set(counts)) > 1, counts  # the resource (ore) counts differ
  for k, b in enumerate(blobs):
    assert b == TM.alone(name, k), k
  spawns = [next(v for n, v in s.items() if n.startswith('spawn_cells_')) for s in sec]
  assert not np.array_equal(spawns[3], spawns[0])
  walls = 'cell_flags' if name == 'coop_mining' else 'tr_wall'
  assert not np.array_equal(sec[1][walls], sec[0][walls])


@pytest.mark.parametrize('name', TM.NAMES)
def test_a_map_set_gets_as_far_as_the_device(name):
  import torch
  if torch.cuda.is_available():
    pytest.skip('a GPU is present: the GPU tests create these engines')
  rc, msg = _create(list(TM.map_set(name)))
  assert rc == MP_E_NO_DEVICE, msg


def _refusals():
  return [
      ('other_size', 'territory__rooms', None, "variant 1: section 'meta' differs in field 'W'"),
      ('view', 'territory__rooms', V.view(2, 2, 2, 2), "variant 1: section 'meta' differs in field 'view left'"),
      ('episode_cap', 'territory__open', V.top(maxEpisodeLengthFrames=50), "variant 1: section 'meta' differs in field 'max frames'"),
      ('zap_beam', 'territory__rooms', V.kw('Zapper', beamLength=2, beamRadius=0), "variant 1: Params field 'zap.geom' differs"),
      ('claim_beam', 'territory__open', V.kw('ResourceClaimer', beamLength=1, beamRadius=0), "variant 1: Params field 'claim_geom' differs"),
      ('mine_beam', 'coop_mining', V.kw('MineBeam', beamLength=2), "variant 1: Params field 'mine_length' differs"),
      ('episode_ending', 'coop_mining', V.kw('StochasticIntervalEpisodeEnding', probabilityTerminationPerInterval=0.5),
       'variant 1: episode ending differs'),
  ]


@pytest.mark.parametrize('row', _refusals(), ids=lambda r: r[0])
def test_what_maps_may_not_differ_in_is_refused_before_the_device(row):
  _, name, edit, what = row
  if edit is None:  # rooms (21 x 21, TORUS) next to open (39 x 23, BOUNDED)
    blobs = [substrates.load_blob('territory__rooms'), substrates.load_blob('territory__open')]
  else:
    s = TM.settings(name, 1)
    edit(s)
    blobs = compiler.compile_settings_set([TM.settings(name, 0), s], TM.config(name))
  rc, msg = _create(blobs)
  assert rc == MP_E_UNSUPPORTED and msg.startswith(what), msg


def test_inside_out_maps_are_refused_by_their_choice_groups():
  from tests import settings_golden
  s0 = settings_golden.settings('territory__inside_out', 5)
  s1 = settings_golden.settings('territory__inside_out', 5)
  rows = s1['simulation']['map'].split('\n')
  y = next(i for i, r in enumerate(rows) if ',A,' in r)  # a 'choice' cell moves one cell to the right
  x = rows[y].index(',A,') + 1
  rows[y] = rows[y][:x] + ',A' + rows[y][x + 2:]
  s1['simulation']['map'] = '\n'.join(rows)
  blobs = compiler.compile_settings_set([s0, s1], settings_golden.config('territory__inside_out', 5))
  assert 'choice_groups' in mpb.unpack(blobs[0])
  rc, msg = _create(blobs)
  assert rc == MP_E_UNSUPPORTED and msg.startswith('variant 1: section '), msg


def _build(name='territory__rooms', **kw):
  args = dict(roles=('default',) * TM.PLAYERS.get(name, 9), num_envs=4, maps=[TM.ascii_map('territory__rooms', k) for k in range(2)])
  args.update(kw)
  return substrate.build_batched(name, **args)


@pytest.mark.parametrize('kw,what', [
    (dict(maps=[]), 'the sequence of maps is empty'),
    (dict(maps='W'), 'not one map'),
    (dict(maps=[3]), r'maps\[0\] is a int, not a str'),
    (dict(maps=['\n'.join(['W' * 21] * 20)]), r'maps\[0\] has 20 rows; territory__rooms has 21'),
    (dict(maps=['\n'.join(['W' * 21] * 20 + ['W' * 22])]), r'row 20 of maps\[0\] is 22 wide; territory__rooms is 21 wide'),
    (dict(name='clean_up', roles=('default',) * 7), "not of 'clean_up'"),
    (dict(name=('territory__rooms', 'territory__open')), 'maps take one substrate name'),
    (dict(prefab_overrides=[{}]), 'maps take neither prefab_overrides nor build_seeds'),
    (dict(build_seeds=[0]), 'maps take neither prefab_overrides nor build_seeds'),
    (dict(env_variant=[0, 1, 2, 0]), r'env_variant must index the 2 maps \(0..1\)'),
    (dict(roles=('other',) * 9), 'Invalid roles'),
], ids=['empty', 'str', 'not_str', 'rows', 'width', 'other_substrate', 'names', 'overrides', 'build_seeds', 'env_variant',
        'roles'])
def test_build_batched_with_maps_checks_its_arguments_before_compiling(kw, what, monkeypatch):
  monkeypatch.setattr(substrates, 'compile_maps', lambda *a: pytest.fail('compiled'))
  with pytest.raises(ValueError, match=what):
    _build(**kw)


def test_build_batched_with_maps_needs_a_reference_checkout(monkeypatch):
  monkeypatch.setattr(compiler, 'reference_root', lambda: None)
  with pytest.raises(FileNotFoundError, match='maps for .territory__rooms. need a Melting Pot reference checkout'):
    _build()


def test_build_batched_with_maps_compiles_the_set_and_assigns_maps_by_global_env(monkeypatch):
  calls = []
  monkeypatch.setattr(substrates, 'compile_maps', lambda name, roles, maps: calls.append((name, roles, maps)) or ['a', 'b', 'c'])
  monkeypatch.setattr(substrate, 'BatchedSubstrate', lambda blob, n, **kw: (blob, n, kw))
  maps = [TM.ascii_map('coop_mining', k) for k in range(3)]
  blob, n, kw = substrate.build_batched('coop_mining', roles=('default',) * 6, num_envs=5, env_index_base=7, maps=maps)
  assert calls == [('coop_mining', ('default',) * 6, maps)] and blob == ['a', 'b', 'c'] and n == 5
  assert kw['env_variant'].tolist() == [1, 2, 0, 1, 2]


def test_compile_substrate_maps_replaces_the_map_the_builder_reads(monkeypatch):
  from meltingpot_b200.shims.config_dict_shim import ConfigDict

  def builder(roles, config):
    return {'simulation': {'map': config.layout.ascii_map if 'layout' in config else 'STOCK'}}
  monkeypatch.setattr(compiler, 'compile_settings_set', lambda settings, config: [s['simulation']['map'] for s in settings])
  for with_layout, want in ((True, ['A', 'B']), (False, ['A', 'B'])):
    cfg = ConfigDict({'default_player_roles': ['default'], 'lab2d_settings_builder': builder})
    if with_layout:
      cfg.layout = ConfigDict({'ascii_map': 'STOCK'})
    monkeypatch.setattr(compiler, 'load_reference_config', lambda name, root=None, c=cfg: c)
    assert compiler.compile_substrate_maps('x', None, ['A', 'B']) == want


def test_sharded_substrate_passes_maps_through(monkeypatch):
  import torch.distributed as dist
  from meltingpot_b200 import distributed
  calls = []
  monkeypatch.setattr(substrate, 'build_batched', lambda name, **kw: calls.append(kw) or object())
  monkeypatch.setattr(dist, 'get_rank', lambda group=None: 1)
  monkeypatch.setattr(dist, 'get_world_size', lambda group=None: 2)
  maps = ['m0', 'm1']
  distributed.ShardedSubstrate('coop_mining', ['default'] * 6, 16, seed=3, device=0, maps=maps)
  assert calls[0]['maps'] is maps and calls[0]['env_index_base'] == 8 and calls[0]['env_variant'] is None


@pytest.mark.parametrize('name', TM.NAMES)
def test_the_oracle_of_a_mixed_batch_equals_single_map_oracle_envs(name, oracle):
  from tests.test_gpu_env_variants import _MixedOracle, _replace
  blobs = TM.map_set(name)
  B, seed = 10, 5
  assign = (np.arange(B) % 4).astype(np.int64)
  mixed = _MixedOracle(oracle, blobs, assign, seed)
  envs = [oracle.OracleEnv(blobs[assign[b]], seed + b) for b in range(B)]
  for e in envs:
    e.reset()
  rng = np.random.default_rng(1)
  P = envs[0].P
  shapes = dict(P=P, L=envs[0].L, cells=envs[0].W * envs[0].H, n_scalar=envs[0].n_scalar, rgb=(1, 1), world=(1, 1))
  for t in range(45):
    acts = rng.integers(0, envs[0].n_actions, size=(B, P)).astype(np.int32)
    mixed.step(acts)
    for b, e in enumerate(envs):
      if e.step_type() == 2:  # the batch starts the next episode in this step
        envs[b] = _replace(oracle, e, blobs[assign[b]], seed + b)
      else:
        e.step(acts[b])
    d = mixed.dump(shapes, False, 256)
    for b, e in enumerate(envs):
      assert np.array_equal(d['grid'][b], e.grid()) and np.array_equal(d['reward'][b], e.rewards()), (t, b)
      assert int(d['step_type'][b]) == e.step_type(), (t, b)
  mixed.close()
