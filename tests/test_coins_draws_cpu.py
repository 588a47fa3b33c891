"""Draw sets (compiler.compile_settings_set): several builds of one substrate on one sprite table, so that one engine
can run them as per-env variants. Checked on the stored coins draws (tests/coins_draws.py) without a GPU."""

import json

import numpy as np
import pytest

from meltingpot_b200 import blob as blob_lib
from meltingpot_b200 import compiler
from meltingpot_b200 import substrates
from tests import coins_draws as CD
from tests import settings_golden

SPRITE_SECTIONS = ('atlas', 'sprite_opaque', 'sprite_map', 'hits', 'cell_flags')


def _sections(blob):
  return blob_lib.unpack(blob)


def test_a_set_of_one_is_the_stand_alone_blob():
  for seed in (0, 3):
    s = settings_golden.settings('coins', 2, seed)
    alone = compiler.compile_settings(s, settings_golden.config('coins', 2), seed)
    (one,) = compiler.compile_settings_set([s], settings_golden.config('coins', 2), [seed])
    assert one == alone
  committed = substrates.load_blob('coins', ('default',) * 2)
  seed = substrates.BUILD_SEEDS['coins']
  assert compiler.compile_settings_set([settings_golden.settings('coins', 2, seed)], settings_golden.config('coins', 2), [seed])[0] == committed
  for seed in CD.seeds()[:3]:
    assert CD.draw_set(False, (seed,))[0] == CD.alone(seed, False)


def test_the_sprite_sections_are_identical_across_the_set():
  blobs = CD.draw_set(False)
  secs = [_sections(b) for b in blobs]
  for name in SPRITE_SECTIONS:
    for k, s in enumerate(secs[1:], 1):
      assert np.array_equal(s[name], secs[0][name]), f'{name} of draw {k}'
  for field in ('N_SPRITES', 'OOB_SPRITE', 'OOV_SPRITE', 'W', 'H', 'P', 'L'):
    assert len({int(s['meta'][compiler.META[field]]) for s in secs}) == 1, field
  # the union holds every draw's sprites: per-name pixel variants of the avatars, and the five coin colours
  names = json.loads(blob_lib.section_text(secs[0], 'info_json'))['sprites']
  assert sorted({n for n in names if n.startswith('coin_')}) == ['coin_blue', 'coin_green', 'coin_purple', 'coin_red', 'coin_yellow']
  assert names.count('Avatar1') > 1 and names.count('Avatar2') > 1
  assert len(names) == len(set((n, secs[0]['atlas'][i].tobytes()) for i, n in enumerate(names)))  # deduplicated by name and pixels


def test_each_set_blob_draws_the_pixels_of_its_stand_alone_blob():
  blobs = CD.draw_set(False)
  for seed, blob in zip(CD.seeds(), blobs):
    a, u = _sections(CD.alone(seed, False)), _sections(blob)
    atlas_a, atlas_u = a['atlas'], u['atlas']
    # every sprite id the draw refers to shows the same pixels in the union
    ids = lambda s: list(s['states'][:, 1]) + list(s['av_table'][:, 1]) + [int(s['meta'][compiler.META['OOB_SPRITE']])]
    for i, j in zip(ids(a), ids(u)):
      if i >= 0:
        assert np.array_equal(atlas_a[i], atlas_u[j]), seed
    for name in ('objects', 'kinds', 'comps', 'comps_f', 'co_coin', 'co_dp', 'spawn_cells_2', 'action_table'):
      assert np.array_equal(a[name], u[name]), (seed, name)


def test_the_stored_draws_differ_in_map_size_and_in_colours():
  secs = [_sections(b) for b in CD.draw_set(False)]
  coins = [int(compiler.family_params(s)['N_COINS']) for s in secs]
  assert min(coins) == 10 * 10 - 2 and max(coins) == 15 * 15 - 2  # the smallest and the largest interior
  pairs = []
  for s in secs:
    names = json.loads(blob_lib.section_text(s, 'info_json'))['sprites']
    p = compiler.family_params(s)
    pairs.append((names[p['COIN_SPRITE_0']], names[p['COIN_SPRITE_1']]))
  assert len(set(pairs)) >= 6
  assert any((b, a) in pairs for a, b in pairs)  # some pair in both orders
  assert len({s['init_grid'].tobytes() for s in secs}) >= 8  # (the walls of a map: its interior's width and height)


@pytest.mark.parametrize('seed', CD.seeds()[:4] + CD.seeds()[-2:])
def test_the_oracle_on_a_set_blob_equals_the_oracle_on_its_stand_alone_blob(oracle, seed):
  blobs = dict(zip(CD.seeds(), CD.draw_set(True)))
  a, u = oracle.OracleEnv(CD.alone(seed), 7), oracle.OracleEnv(blobs[seed], 7)
  rng = np.random.default_rng(seed)
  a.reset(); u.reset()
  lasts = 0
  for t in range(200):
    if a.step_type() == 2:
      a.reset(); u.reset()
    else:
      acts = rng.integers(0, a.n_actions, size=a.P)
      a.step(acts); u.step(acts)
    where = f'draw {seed} step {t}'
    assert a.step_type() == u.step_type() and a.discount() == u.discount(), where
    lasts += a.step_type() == 2
    np.testing.assert_array_equal(a.rewards(), u.rewards(), err_msg=where)
    np.testing.assert_array_equal(a.scalar_obs(), u.scalar_obs(), err_msg=where)
    assert a.events() == u.events(), where
    np.testing.assert_array_equal(a.avatars(), u.avatars(), err_msg=where)
    np.testing.assert_array_equal(a.rgb(), u.rgb(), err_msg=where)
    np.testing.assert_array_equal(a.world_rgb(), u.world_rgb(), err_msg=where)
  assert lasts >= 4  # across auto-resets (40-frame cap)


def test_a_draw_set_is_not_combined_with_prefab_overrides(monkeypatch):
  from meltingpot_b200 import substrate
  with pytest.raises(ValueError, match='build_seeds or prefab_overrides'):
    substrate.build_batched('coins', roles=('default',) * 2, num_envs=4, build_seeds=[0, 1], prefab_overrides=[{}])
  monkeypatch.delenv('MELTINGPOT_REFERENCE_ROOT', raising=False)
  with pytest.raises(FileNotFoundError):
    substrate.build_batched('coins', roles=('default',) * 2, num_envs=4, build_seeds=[0, 1])


def test_the_default_draw_of_each_env_counts_global_envs():
  from meltingpot_b200 import substrate
  assert substrate.draw_of_env(0, 5, 2).tolist() == [0, 1, 0, 1, 0]
  assert substrate.draw_of_env(3, 4, 3).tolist() == [0, 1, 2, 0]


def test_set_entries_and_seeds_must_match():
  with pytest.raises(ValueError):
    compiler.compile_settings_set([], None)
  with pytest.raises(ValueError):
    compiler.compile_settings_set([CD.settings(CD.seeds()[0])], CD.config(), [1, 2])
