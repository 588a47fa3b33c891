"""CPU test: the row layout of DrawnRoutes, every refusal of drawn_routes and of BatchedScenario's population mode, the
mp_route_draw struct and entry points against the header, and the draw rule (tests/drawn_routes.py, on the oracle's
Philox: uniform, and a function of (key, episode, slot) only)."""

import ctypes

import numpy as np
import pytest
import torch
from scipy import stats

from meltingpot_b200 import engine
from meltingpot_b200 import scenario
from meltingpot_b200 import substrate
from oracle import binding as oracle
from tests.drawn_routes import route_draw

B, P, H, W = 3, 5, 16, 24
NAMES = ['READY_TO_SHOOT']


def _drawn(choices, num_envs=B, num_players=P):
  return substrate.DrawnRoutes(choices, num_envs, num_players, (H, W, 3), NAMES, 'cpu')


def test_rows_are_group_major_with_capacity_per_listing_slot():
  # slot 0 focal (group 0); slots 1..3 draw from groups 1 and 2; slot 4 draws from group 2 only
  r = _drawn([(0,), (1, 2), (2, 1), (1, 2), (2,)])
  assert r.num_groups == 3
  assert [r.group(g) for g in range(3)] == [(0,), (1, 2, 3), (1, 2, 3, 4)]  # rank_g(p) = position in group(g)
  assert r.rows(0) == slice(0, B) and r.rows(1) == slice(B, 4 * B) and r.rows(2) == slice(4 * B, 8 * B)
  assert r.n_rows == 8 * B
  d = r.draw
  assert d.n_rows == r.n_rows and d.row_of_player == r.row_of_player.data_ptr()
  assert list(d.n_choices)[:P] == [1, 2, 2, 2, 1] and list(d.n_choices)[P:] == [0] * (16 - P)
  starts, cap = {0: 0, 1: B, 2: 4 * B}, {0: 1, 1: 3, 2: 4}
  for p, choices in enumerate(r.choices):
    for j, g in enumerate(choices):
      assert d.row_base[p][j] == starts[g] + r.group(g).index(p)
      assert d.rows_per_env[p][j] == cap[g]
  # every (b, p, choice) has a row of its own inside its group's block
  seen = set()
  for p, choices in enumerate(r.choices):
    for j, g in enumerate(choices):
      for b in range(B):
        row = d.row_base[p][j] + b * d.rows_per_env[p][j]
        assert r.rows(g).start <= row < r.rows(g).stop
        assert row not in seen
        seen.add(row)
  assert len(seen) == r.n_rows
  assert r.row_of_player.shape == (B, P) and r.row_of_player.dtype == torch.int32
  assert (r.row_of_player == -1).all()


def test_unlisted_groups_and_slots_without_choices():
  r = _drawn([(), (3,), (3, 3), (), (1,)])
  assert r.num_groups == 4
  assert r.group(0) == () and r.group(2) == () and r.rows(0) == slice(0, 0) and r.rows(2) == slice(B, B)
  assert r.group(3) == (1, 2) and r.rows(3) == slice(B, 3 * B)
  assert list(r.draw.n_choices)[:P] == [0, 1, 2, 0, 1]
  # a group listed twice by one slot is one row of that slot, drawn with twice the weight
  assert r.draw.row_base[2][0] == r.draw.row_base[2][1] == B + 1
  with pytest.raises(IndexError):
    r.rows(4)
  with pytest.raises(IndexError):
    r.group(-1)


def test_active_follows_the_row_map():
  r = _drawn([(0,), (1, 2), (2, 1), (1, 2), (2,)])
  d = r.draw
  m = torch.tensor([[0, d.row_base[1][0] + 0 * 3, d.row_base[2][0], d.row_base[3][1], d.row_base[4][0]],
                    [1, d.row_base[1][1] + 1 * 4, d.row_base[2][1] + 1 * 3, d.row_base[3][0] + 1 * 3, d.row_base[4][0] + 4],
                    [2, d.row_base[1][0] + 2 * 3, d.row_base[2][1] + 2 * 3, d.row_base[3][0] + 2 * 3, d.row_base[4][0] + 8]],
                   dtype=torch.int32)
  r.row_of_player.copy_(m)
  assert r.active(0).tolist() == [[True], [True], [True]]
  # group 1 = slots (1, 2, 3): env 0 slot 1; env 1 slots 2, 3; env 2 slots 1, 2, 3
  assert r.active(1).tolist() == [[True, False, False], [False, True, True], [True, True, True]]
  # group 2 = slots (1, 2, 3, 4)
  assert r.active(2).tolist() == [[False, True, True, True], [True, False, False, True], [False, False, False, True]]


def test_drawn_routes_are_immutable():
  r = _drawn([(0,), (1,), (1,), (1,), (1,)])
  with pytest.raises(AttributeError, match='immutable'):
    r.n_rows = 3


@pytest.mark.parametrize('choices, match', [
    ([(0,)] * (P - 1), 'each of the 5 player slots'),
    ('abcde', 'each of the 5 player slots'),
    ([(0,), (1,), 2, (1,), (1,)], r'choices\[2\] must be a sequence'),
    ([(0,), (1,), 'ab', (1,), (1,)], r'choices\[2\] must be a sequence'),
    ([(0,), tuple(range(9)), (1,), (1,), (1,)], r'choices\[1\] lists 9 groups, at most 8'),
    ([(0,), (-1,), (1,), (1,), (1,)], r'choices\[1\]: group ids must be integers >= 0'),
    ([(0,), (True,), (1,), (1,), (1,)], r'choices\[1\]: group ids must be integers >= 0'),
    ([(0,), (1.0,), (1,), (1,), (1,)], r'choices\[1\]: group ids must be integers >= 0'),
    ([()] * P, 'routes no player'),
])
def test_drawn_routes_refusals(choices, match):
  with pytest.raises(ValueError, match=match):
    _drawn(choices)


def test_too_many_rows_are_refused():
  with pytest.raises(ValueError, match='2\\^31'):
    substrate.DrawnRoutes([(0,)] * 16, 2**27, 16, (H, W, 3), NAMES, 'meta')


# -- BatchedScenario population mode --------------------------------------------------------------------------------------
class FakeBatched:
  """What BatchedScenario's constructor reads of a BatchedSubstrate."""

  num_envs, num_players = B, P

  def drawn_routes(self, choices):
    return _drawn(choices)

  def player_routes(self, groups):
    return substrate.PlayerRoutes(groups, B, P, (H, W, 3), NAMES, 'cpu')


def _noop(ts, active):
  return torch.zeros(active.shape, dtype=torch.int32)


ROLES = ('focal', 'a', 'b', 'a', 'b')
IS_FOCAL = (True, False, False, False, False)
BOTS = {'a': ['x', 'y'], 'b': ['z', 'y', 'y']}
POLICIES = {'x': _noop, 'y': _noop, 'z': _noop}


def test_population_choices_follow_sorted_bot_names():
  s = scenario.BatchedScenario(FakeBatched(), POLICIES, IS_FOCAL, ['RGB'], roles=ROLES, bots_by_role=BOTS)
  assert s.bot_names == ('x', 'y', 'z')
  r = s._routes  # pylint: disable=protected-access
  assert r.choices == ((0,), (1, 2), (2, 3), (1, 2), (2, 3))  # roles' bots sorted and deduplicated, as Population does
  assert r.group(0) == (0,) and r.group(1) == (1, 3) and r.group(2) == (1, 2, 3, 4) and r.group(3) == (2, 4)
  with pytest.raises(ValueError, match='population mode'):
    scenario.BatchedScenario(FakeBatched(), _noop, IS_FOCAL, ['RGB']).background_bots()


@pytest.mark.parametrize('kwargs, match', [
    (dict(is_focal=IS_FOCAL[:-1]), 'is_focal is length 4 but substrate is 5-player.'),
    (dict(roles=ROLES[:-1]), 'roles and is_focal must be the same length.'),
    (dict(roles=None), 'bots_by_role needs roles'),
    (dict(bots_by_role=None), 'roles needs bots_by_role'),
    (dict(bots_by_role={'a': ['x']}), "no bots for role 'b'"),
    (dict(bots_by_role={'a': ['x'], 'b': []}), r"bots_by_role\['b'\] is empty"),
    (dict(bots_by_role={'a': ['x'], 'b': [f'n{i}' for i in range(9)]}), r"bots_by_role\['b'\] lists 9 bots, at most 8"),
    (dict(policy={'x': _noop, 'y': _noop}), "no callable for bot 'z'"),
    (dict(policy={'x': _noop, 'y': _noop, 'z': 3}), "no callable for bot 'z'"),
    (dict(policy=_noop), 'must map each bot name to a callable'),
])
def test_population_refusals(kwargs, match):
  args = dict(policy=POLICIES, is_focal=IS_FOCAL, roles=ROLES, bots_by_role=BOTS)
  args.update(kwargs)
  with pytest.raises(ValueError, match=match):
    scenario.BatchedScenario(FakeBatched(), args['policy'], args['is_focal'], ['RGB'], roles=args['roles'],
                             bots_by_role=args['bots_by_role'])


def test_roles_of_focal_slots_need_no_bots():
  s = scenario.BatchedScenario(FakeBatched(), {'x': _noop}, IS_FOCAL, ['RGB'], roles=('nobody', 'a', 'a', 'a', 'a'),
                               bots_by_role={'a': ['x']})
  assert s.bot_names == ('x',)


# -- the draw rule --------------------------------------------------------------------------------------------------------
def test_draw_depends_on_key_episode_and_slot_only():
  # the rule: pick(philox(counter {0, episode, p, RS_ROUTE = 6}, key).x, n), written out with the oracle's philox
  for key, episode, p, n in [(1, 1, 0, 2), (2**40 + 7, 3, 4, 5), (123456789, 0, 15, 8), (99, 1000, 7, 3)]:
    w = oracle.philox([0, episode, p, 6], [key & 0xffffffff, key >> 32])[0]
    assert route_draw(key, episode, p, n) == (w * n) >> 32
    assert route_draw(key, episode, p, n) == route_draw(key, episode, p, n)
  assert route_draw(5, 1, 2, 0) == -1
  # other streams at the same address draw other numbers (RS_ROUTE leaves every existing draw alone)
  key, n = 77, 1 << 16
  draws = {s: (oracle.philox([0, 1, 2, s], [key, 0])[0] * n) >> 32 for s in range(7)}
  assert draws[6] == route_draw(key, 1, 2, n) and len(set(draws.values())) == 7


@pytest.mark.parametrize('n', [2, 3, 5, 8])
def test_draw_is_uniform(n):
  counts = np.zeros(n, np.int64)
  for key in range(1, 41):
    for episode in range(1, 26):
      for p in range(16):
        counts[route_draw(1000 + key, episode, p, n)] += 1
  _, pvalue = stats.chisquare(counts)
  assert pvalue > 1e-4, counts
  # and independent between the slots of one env and episode: pairs of slots are uniform over n * n
  pairs = np.zeros((n, n), np.int64)
  for key in range(1, 201):
    for episode in range(1, 11):
      pairs[route_draw(key, episode, 0, n), route_draw(key, episode, 1, n)] += 1
  _, pvalue = stats.chisquare(pairs.reshape(-1))
  assert pvalue > 1e-4, pairs


# -- C ABI ----------------------------------------------------------------------------------------------------------------
@pytest.mark.skipif(torch.cuda.is_available(), reason='checks the no-GPU failure mode')
def test_entry_points_refuse_a_null_handle_without_gpu():
  lib = engine.load_library()
  d, players = ctypes.pointer(engine.MpRouteDraw()), ctypes.pointer(engine.MpPlayerOutputs())
  pa = ctypes.pointer(engine.MpPlayerActions())
  for req in (engine.MpRequest(player_actions=pa, draw=d, players=players), engine.MpRequest(reset=1, draw=d, players=players)):
    assert lib.mp_run(None, ctypes.byref(req), None) == -1
    assert b'mp_run: null handle or request' in lib.mp_last_error()
