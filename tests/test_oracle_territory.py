"""territory__rooms on the CPU oracle vs what the Lua states
(meltingpot/lua/levels/territory/components.lua,
 meltingpot/lua/modules/avatar_library.lua:948-1121)."""

import json

import numpy as np

from meltingpot_b200 import blob as blob_lib
from meltingpot_b200 import compiler

NOOP, FORWARD, BACKWARD, STEP_LEFT, STEP_RIGHT, TURN_LEFT, TURN_RIGHT, ZAP, CLAIM = range(9)
N, E, S, W = range(4)
P = 9
WC = 21


def _tables(blob):
  sec = blob_lib.unpack(blob)
  return sec, json.loads(blob_lib.section_text(sec, 'info_json'))


def _sprite(env, info, layer, x, y):
  v = int(env.grid()[info['layers'].index(layer)][y * WC + x])
  return info['sprites'][(v - 1) // 4] if v else None


def _fresh(oracle, blob, seed=1):
  env = oracle.OracleEnv(blob, seed)
  env.reset()
  return env


def act(**kw):
  a = [NOOP] * P
  for k, v in kw.items():
    a[int(k[1:])] = v
  return np.array(a, np.int32)


def test_layers_and_reset(oracle, territory_blob):
  _, info = _tables(territory_blob)
  # territory/init.lua:30-37 appends the two indicator layers after BaseSimulation's (incl. beamZap).
  assert info['layers'][-3:] == ['beamZap', 'directionIndicatorLayer', 'superDirectionIndicatorLayer']
  env = _fresh(oracle, territory_blob)
  av = env.avatars()
  assert (av[:, 3] == 1).all()
  assert {(int(x) % 7, int(y) % 7) for x, y, _, _ in av} == {(3, 3)}  # the nine room centres ('P')
  for x, y, o, _ in av:  # the marking overlay sits on its avatar from frame 0 (avatar_library.lua:1033-1047)
    assert _sprite(env, info, 'superOverlay', int(x), int(y)) == 'sprite_for_level_1'
    fx, fy = int(x) + (o == E) - (o == W), int(y) + (o == S) - (o == N)
    assert _sprite(env, info, 'directionIndicatorLayer', fx, fy).startswith('brush')  # Paintbrush fires in api:start too
  assert env.scalar_obs().shape == (P, 1)


def test_facing_a_resource_claims_it_and_pays_after_delay(oracle, territory_blob):
  _, info = _tables(territory_blob)
  total = 0.0
  env = _fresh(oracle, territory_blob, seed=3)
  for p in range(1, P):
    env.debug_set_avatar(p, 2 + 7 * (p % 3), 2 + 7 * (p // 3), N)  # far from any wall of resources
  env.debug_set_avatar(0, 3, 1, N)                                   # facing the room's north wall of resources at (3, 0)
  assert _sprite(env, info, 'upperPhysical', 3, 0) == 'UnclaimedResourceSprite'
  env.step(act())
  assert ('claimed_resource', 1, 0) in env.events()                 # directionHit -> Resource:_claim (components.lua:114-137)
  assert _sprite(env, info, 'upperPhysical', 3, 0) == 'Color1ResourceSprite'
  env.step(act(p0=FORWARD))
  assert tuple(env.avatars()[0][:2]) == (3, 1)                      # resources stand on the avatar layer and block
  paid = 0
  for t in range(1500):
    env.step(act())
    paid += env.rewards()[0]
    if t == 20:
      assert paid == 0                                              # rewardDelay = 25 frames in the claimed state
  assert 5 <= paid <= 30                                            # rewardRate 0.01 per frame: Binomial(~1475, 0.01)
  assert _sprite(env, info, 'overlay', 3, 0) == 'Color1DryPaintSprite'  # RewardIndicator shows dry paint once paying


def test_claim_beam_reaches_two_cells_and_skips_resource_cells_for_its_sprite(oracle, territory_blob):
  _, info = _tables(territory_blob)
  env = _fresh(oracle, territory_blob)
  for p in range(1, P):
    env.debug_set_avatar(p, 2 + 7 * (p % 3), 2 + 7 * (p // 3), S)
  env.debug_set_avatar(0, 3, 2, N)
  env.step(act(p0=CLAIM))                                           # beamLength 2, radius 0 (territory.py:731-738)
  assert _sprite(env, info, 'upperPhysical', 3, 0) == 'Color1ResourceSprite'
  assert _sprite(env, info, 'superDirectionIndicatorLayer', 3, 1) == 'claimBeamSprite_1'
  assert _sprite(env, info, 'superDirectionIndicatorLayer', 3, 0) is None   # the damage indicator occupies that layer there
  env.step(act())
  assert _sprite(env, info, 'superDirectionIndicatorLayer', 3, 1) is None   # hit sprites last one frame


def test_two_zaps_destroy_a_resource_and_damage_self_repairs(oracle, territory_blob):
  _, info = _tables(territory_blob)
  env = _fresh(oracle, territory_blob, seed=2)
  for p in range(1, P):
    env.debug_set_avatar(p, 2 + 7 * (p % 3), 2 + 7 * (p // 3), S)
  env.debug_set_avatar(0, 3, 1, N)
  env.step(act(p0=ZAP))                                             # health 2 -> 1, the zap stops at it
  assert _sprite(env, info, 'upperPhysical', 3, 0) is not None
  env.step(act())
  assert _sprite(env, info, 'superDirectionIndicatorLayer', 3, 0) == 'DamagedResource'  # one frame later (Resource:update)
  for _ in range(4):
    env.step(act())                                                 # cooldownTime = 4
  env.step(act(p0=ZAP))
  assert ('destroyed_resource', 1, 0) in env.events()
  assert _sprite(env, info, 'upperPhysical', 3, 0) is None and _sprite(env, info, 'lowerPhysical', 3, 0) is None
  assert _sprite(env, info, 'superDirectionIndicatorLayer', 3, 0) is None
  env.step(act(p0=FORWARD))
  assert tuple(env.avatars()[0][:2]) == (3, 0)                      # a destroyed resource no longer blocks
  # a resource hit once repairs itself: p = 0.1 per frame after 15 frames
  env2 = _fresh(oracle, territory_blob, seed=9)
  for p in range(1, P):
    env2.debug_set_avatar(p, 2 + 7 * (p % 3), 2 + 7 * (p // 3), S)
  env2.debug_set_avatar(0, 3, 1, N)
  env2.step(act(p0=ZAP))
  for _ in range(15):
    env2.step(act())
    assert _sprite(env2, info, 'superDirectionIndicatorLayer', 3, 0) == 'DamagedResource'
  for _ in range(150):
    env2.step(act())
  assert _sprite(env2, info, 'superDirectionIndicatorLayer', 3, 0) is None


def test_graduated_sanctions_freeze_then_remove(oracle, territory_blob):
  _, info = _tables(territory_blob)
  env = _fresh(oracle, territory_blob)
  for p in range(2, P):
    env.debug_set_avatar(p, 2 + 7 * (p % 3), 9 + 7 * (p // 6), S)
  env.debug_set_avatar(0, 2, 3, E)
  env.debug_set_avatar(1, 4, 3, W)
  env.step(act())                                                   # let the markings follow the moved avatars
  env.step(act(p0=ZAP))                                             # hit 1: level 1 -> 2, frozen for 25 frames
  assert ('sanctioning', 1, 2) in env.events() and env.avatars()[1, 3] == 1
  assert _sprite(env, info, 'superOverlay', 4, 3) == 'sprite_for_level_2'
  env.step(act(p1=FORWARD))
  assert tuple(env.avatars()[1][:2]) == (4, 3)                      # disallowMovementUntil(25)
  for _ in range(3):
    env.step(act())
  assert env.scalar_obs()[1, 0] == 0.0                              # disallowZappingUntil: cooling timer held above cooldown
  env.step(act(p0=ZAP))                                             # hit 2 at level 2: removal, one frame later
  assert ('removal_due_to_sanctioning', 1, 2) in env.events() and env.avatars()[1, 3] == 1
  env.step(act())
  assert env.avatars()[1, 3] == 0 and (env.rgb()[1] == 80).all()
  env.step(act())
  assert _sprite(env, info, 'superOverlay', 4, 3) is None            # the marking leaves with its avatar
  for _ in range(200):
    env.step(act())
  assert env.avatars()[1, 3] == 0                                    # framesTillRespawn = 1e6: out for the episode


def test_marking_recovers_after_50_frames(oracle, territory_blob):
  _, info = _tables(territory_blob)
  env = _fresh(oracle, territory_blob)
  for p in range(2, P):
    env.debug_set_avatar(p, 2 + 7 * (p % 3), 9 + 7 * (p // 6), S)
  env.debug_set_avatar(0, 2, 3, E)
  env.debug_set_avatar(1, 4, 3, W)
  env.step(act())
  env.step(act(p0=ZAP))
  seen = []
  for _ in range(55):
    env.step(act())
    seen.append(_sprite(env, info, 'superOverlay', 4, 3))
  assert seen[48] == 'sprite_for_level_2' and seen[49] == 'sprite_for_level_1'  # recoveryTime = 50 (territory.py:804-819)
  env.step(act(p1=FORWARD))
  assert tuple(env.avatars()[1][:2]) == (3, 3)                      # thawed after 25 frames


def test_torus_wraps_movement_and_views(oracle, territory_blob):
  env = _fresh(oracle, territory_blob)
  for p in range(1, P):
    env.debug_set_avatar(p, 2 + 7 * (p % 3), 2 + 7 * (p // 3), S)
  # destroy the resources at (3, 0) and (3, 20) so that the torus seam can be crossed
  sec, _ = _tables(territory_blob)
  for k, (oid, cell, st) in enumerate(sec['tr_res']):
    if int(cell) in (0 * WC + 3, 20 * WC + 3):
      env.debug_set_object_state(int(oid), 1)
  env.debug_set_avatar(0, 3, 1, N)
  env.step(act(p0=FORWARD))
  env.step(act(p0=FORWARD))
  assert tuple(env.avatars()[0][:2]) == (3, 20)                     # territory__rooms.py:91 topology TORUS
  cells = env.rgb()[0].reshape(11, 8, 11, 8, 3).transpose(0, 2, 1, 3, 4).reshape(121, -1)
  assert (cells != 0).any(axis=1).all()                             # no OutOfBounds (all-black) cell in a torus view


def test_inside_out_choice_prefabs_are_drawn_per_env_and_per_episode(territory_inside_out_blob, oracle):
  # prefab_utils.lua:63-65: a 'choice' prefab is drawn with the env's random stream at every env build, so every env
  # instance -- and, through the ResetWrapper, every episode -- has its own map: territory__inside_out's 'A' / 'B'
  # cells are resources with odds 2:1 / 1:3, its 'Q' cells spawn points with odds 1:6 (territory__inside_out.py:72-86).
  from meltingpot_b200 import blob as blob_lib
  sec = blob_lib.unpack(territory_inside_out_blob)
  cond = sec['tr_res_cond']
  n_cond = int((cond[:, 0] >= 0).sum())
  assert n_cond > 50 and len(sec['choice_groups']) >= n_cond and 'spawn_cond_' + str(0) in sec or any(k.startswith('spawn_cond_') for k in sec)
  counts, layouts = [], []
  for seed in range(12):
    e = oracle.OracleEnv(territory_inside_out_blob, 100 + seed)
    e.reset()
    g = e.grid()
    res_layer = compiler.family_params(sec)['RES_LAYER']
    layouts.append(g[res_layer].copy())
    unclaimed = g[res_layer][0 * 0 + sec['tr_res'][:, 1]] == g[res_layer][int(sec['tr_res'][np.argmax(cond[:, 0] < 0), 1])]
    counts.append(int(unclaimed.sum()))  # resource cells that show the 'unclaimed' resource sprite
    if seed == 0:
      e.reset()
      assert not np.array_equal(e.grid()[res_layer][sec['tr_res'][:, 1]] != 0, layouts[0][sec['tr_res'][:, 1]] != 0)  # next episode: another draw
  assert len({c for c in counts}) > 3               # envs differ
  n_always = int((cond[:, 0] < 0).sum())
  mean = np.mean(counts)
  # expectation: always-present resources + 2/3 of the A cells + 1/4 of the B cells; a loose band around it
  assert n_always + 0.2 * n_cond < mean < n_always + 0.7 * n_cond
