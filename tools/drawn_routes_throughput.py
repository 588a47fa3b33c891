"""What drawing player routes on the device (mp_run's draw) costs against fixed routes and against rerouting in torch.

For each workload, alternating in rounds:

  a_fixed:  a step with player_actions and players: fixed routes (the row map of the drawn reset that starts the run, as input);
  b_drawn:  a drawn step on the same DrawnRoutes: the step draws each slot's bot at every episode start;
  c_torch:  a step with player_actions and players, after rerouting in torch between steps: envs whose step was FIRST draw their
            slots' bots anew (torch.randint) and the row map is rebuilt from the drawn choices with torch ops.

Workloads: clean_up x 4096 with clean_up_0's split (3 focal slots, 4 background slots drawing from 2 bots), and
commons_harvest__open 16p x 8192 with 12 focal slots and 4 background slots drawing from 2 bots. Every player is routed;
each bot's block has the full capacity B * n_k, so half the background rows are inactive in every episode.

Step ms: CUDA events around --reps calls of each, in --rounds alternating rounds after a warm-up of every call; the
median and spread (min..max) over the rounds. Prints one JSON line per (workload, call) with the GPU's name and power
limit, read in the same run.

  python tools/drawn_routes_throughput.py [--reps 20] [--rounds 5]
"""

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

# (substrate, players, envs, focal slots); the background slots come after the focal ones
WORKLOADS = (('clean_up', 7, 4096, 3), ('commons_harvest__open', 16, 8192, 12))
CALLS = ('a_fixed', 'b_drawn', 'c_torch')


def _gpu():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    return 'unknown'


def _calls(sub, eng, routes):
  import torch
  dev = routes.device
  B, P = eng.num_envs, eng.num_players
  h, w = eng.rgb.shape[2:4]
  players = {'row_of_player': routes.row_of_player, 'rgb': torch.empty((routes.n_rows, h, w, 3), dtype=torch.uint8, device=dev),
             'reward': torch.empty((routes.n_rows,), dtype=torch.float64, device=dev)}
  gen = torch.Generator(device=dev).manual_seed(0)
  action = torch.randint(0, eng.num_actions, (routes.n_rows,), generator=gen, device=dev, dtype=torch.int32)
  eng.reset(players=players, draw=routes.draw)
  fixed = routes.row_of_player.clone()
  fixed_players = dict(players, row_of_player=fixed)
  # the layout of c_torch: row_base / rows_per_env of each slot's choices, as DrawnRoutes laid them out
  d = routes.draw
  n = torch.tensor([d.n_choices[p] for p in range(P)], dtype=torch.int64, device=dev)
  base = torch.tensor([[d.row_base[p][j] for j in range(8)] for p in range(P)], dtype=torch.int64, device=dev)
  per_env = torch.tensor([[d.rows_per_env[p][j] for j in range(8)] for p in range(P)], dtype=torch.int64, device=dev)
  env = torch.arange(B, dtype=torch.int64, device=dev).view(B, 1)
  choice = torch.zeros((B, P), dtype=torch.int64, device=dev)
  torch_map = fixed.clone()
  torch_players = dict(players, row_of_player=torch_map)

  def torch_step():
    first = (eng.step_type == 0).view(B, 1)
    drawn = torch.randint(0, 1 << 30, (B, P), generator=gen, device=dev) % n.clamp(min=1)
    choice.copy_(torch.where(first, drawn, choice))
    rows = base.gather(1, choice.t()).t() + env * per_env.gather(1, choice.t()).t()
    torch_map.copy_(torch.where(n > 0, rows, -1).to(torch.int32))
    eng.step(None, player_actions={'row_of_player': torch_map, 'action': action}, players=torch_players)

  return {'a_fixed': lambda: eng.step(None, player_actions={'row_of_player': fixed, 'action': action}, players=fixed_players),
          'b_drawn': lambda: eng.step(None, player_actions={'row_of_player': routes.row_of_player, 'action': action},
                                      players=players, draw=routes.draw),
          'c_torch': torch_step}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--only', default='', help='run only this substrate')
  args = ap.parse_args()
  import torch
  from meltingpot_b200 import substrate, substrates
  gpu = _gpu()
  for name, P, B, n_focal in WORKLOADS:
    if args.only and name != args.only:
      continue
    sub = substrate.BatchedSubstrate(substrates.load_blob(name, ('default',) * P), B, seed=1, world_rgb=False)
    eng = sub.engine
    routes = sub.drawn_routes([(0,) if p < n_focal else (1, 2) for p in range(P)])
    calls = _calls(sub, eng, routes)
    for fn in calls.values():  # warm-up of every call
      fn(); fn()
    torch.cuda.synchronize()
    times = {k: [] for k in calls}
    start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for _ in range(args.rounds):
      for k, fn in calls.items():
        start.record()
        for _ in range(args.reps):
          fn()
        end.record()
        end.synchronize()
        times[k].append(start.elapsed_time(end) / args.reps)
    for k in calls:
      t = sorted(times[k])
      print(json.dumps({'gpu': gpu, 'workload': f'{name} {P}p x {B}, {n_focal} focal, {P - n_focal} background of 2 bots',
                        'call': k, 'step_ms': round(t[len(t) // 2], 4), 'step_ms_min': round(t[0], 4),
                        'step_ms_max': round(t[-1], 4), 'rows': routes.n_rows}), flush=True)
    sub.close()
    del calls
    torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
