"""The kernels one call of each step and reset request (mp_run) and of the other step and reset entry points launches
(mp_launch_count): rendering on or off, with or without the timestep exchange connected (world 1).

A state transition that the renderer follows on the stream lets k_render raise the exchange flags. A call that
publishes its step without that (a step request without `out` and `players`, mp_step_state) launches k_exchange_push of
its own, before k_render when rendering is on. With rendering off, k_exchange_push also delivers per-player scalars;
scalars into `out` are copies, not kernels.
"""

import pytest

pytestmark = pytest.mark.gpu

B = 16

# mp_run request (by its fields) or entry point -> launches in the settings
# (render on, render on + exchange, render off, render off + exchange)
EXPECTED = {
    'reset': (2, 2, 1, 2),
    'reset out': (2, 2, 1, 2),
    'reset players': (2, 2, 2, 2),
    'mp_step_state': (1, 2, 1, 2),
    'step': (2, 3, 1, 2),
    'step out': (2, 2, 1, 2),
    'step restore': (2, 3, 1, 2),
    'step restore out': (2, 2, 1, 2),
    'step players': (2, 2, 2, 2),
    'step players restore': (2, 2, 2, 2),
    'step player_actions': (2, 3, 1, 2),
    'step player_actions out': (2, 2, 1, 2),
    'step player_actions players': (2, 2, 2, 2),
    'step player_actions restore': (2, 3, 1, 2),
    'step player_actions restore out players': (2, 2, 2, 2),
    'mp_step_host': (2, 2, 1, 2),
    'mp_reset_host': (2, 2, 1, 2),
    'mp_step_host_async': (2, 2, 1, 2),
}


def _calls(eng):
  import torch
  P = eng.num_players
  a = torch.zeros((B, P), dtype=torch.int32, device='cuda')
  rows = torch.arange(B * P, dtype=torch.int32, device='cuda').view(B, P)
  pa = {'row_of_player': rows, 'action': torch.zeros(B * P, dtype=torch.int32, device='cuda')}
  players = {'row_of_player': rows, 'reward': torch.zeros(B * P, dtype=torch.float64, device='cuda')}
  out = {'reward': torch.zeros_like(eng.reward)}
  rs = dict(restore=torch.full((B,), -1, dtype=torch.int32, device='cuda'),
            bank=torch.zeros((2, eng.state_record_bytes), dtype=torch.uint8, device='cuda'))
  host_a = eng.make_host_actions()

  def host_async():
    eng.step_host_async(host_a, None, 0)
    eng.wait(0)

  return {
      'reset': lambda: eng.reset(),
      'reset out': lambda: eng.reset(out=out),
      'reset players': lambda: eng.reset(players=players),
      'mp_step_state': lambda: eng.step_state(a),
      'step': lambda: eng.step(a),
      'step out': lambda: eng.step(a, out=out),
      'step restore': lambda: eng.step(a, **rs),
      'step restore out': lambda: eng.step(a, out=out, **rs),
      'step players': lambda: eng.step(a, players=players),
      'step players restore': lambda: eng.step(a, players=players, **rs),
      'step player_actions': lambda: eng.step(None, player_actions=pa),
      'step player_actions out': lambda: eng.step(None, player_actions=pa, out=out),
      'step player_actions players': lambda: eng.step(None, player_actions=pa, players=players),
      'step player_actions restore': lambda: eng.step(None, player_actions=pa, **rs),
      'step player_actions restore out players': lambda: eng.step(None, player_actions=pa, out=out, players=players, **rs),
      'mp_step_host': lambda: eng.step_host(host_a, None),
      'mp_reset_host': lambda: eng.reset_host(None),
      'mp_step_host_async': host_async,
  }


def test_every_entry_point_launches_its_sequence(clean_up_blob):
  import torch
  from meltingpot_b200 import engine
  seen = {name: [] for name in EXPECTED}
  for exchange in (False, True):
    eng = engine.Engine(clean_up_blob, B, seed=3)
    if exchange:
      ptr, _ = eng.exchange_create(0, 1)
      eng.exchange_connect([ptr])
    calls = _calls(eng)
    assert set(calls) == set(EXPECTED)
    for flags in (engine.MP_FLAG_DEFAULT, 0):
      eng.set_flags(flags)
      eng.reset()
      for name, fn in calls.items():
        n = eng.launch_count()
        fn()
        seen[name].append((flags, exchange, eng.launch_count() - n))
    torch.cuda.synchronize()
    eng.close()
  for name, want in EXPECTED.items():
    got = {(f, x): d for f, x, d in seen[name]}
    got = (got[engine.MP_FLAG_DEFAULT, False], got[engine.MP_FLAG_DEFAULT, True], got[0, False], got[0, True])
    assert got == want, (name, got, want)
