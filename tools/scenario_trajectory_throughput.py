"""Cost of keeping a BatchedScenario trajectory: four arms, alternated over rounds, per scenario step.

  (a) sc.step(actions)                               the step alone, focal rows in fresh tensors
  (b) sc.step(actions) + copy into a [T, ...] buffer  how a trajectory was kept before BatchedScenario.trajectory
  (c) sc.step(actions, out=traj.at(t))               the focal rows rendered straight into slot t
  (d) outputs(T) over every row, one target           every row kept T times (focal and background)

Workloads: clean_up x 4096 (5 focal / 2 background) and commons_harvest__open 16p x 8192 (12 / 4). Prints the card
and its power limit, then per workload and arm the median and min-max ms per step over the rounds, as JSON lines.
Usage: python tools/scenario_trajectory_throughput.py [--rounds 5] [--steps 20] [--T 8]
"""

import argparse
import json
import os
import subprocess
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WORKLOADS = [('clean_up', 7, 4096, 5), ('commons_harvest__open', 16, 8192, 12)]


def card():
  try:
    out = subprocess.check_output(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader'], text=True)
    return out.strip().splitlines()[0]
  except (OSError, subprocess.CalledProcessError):
    return 'unknown'


def main():
  import torch
  from meltingpot_b200 import scenario, substrate, substrates
  ap = argparse.ArgumentParser()
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--steps', type=int, default=20)
  ap.add_argument('--T', type=int, default=8, help='trajectory slots (the timed steps cycle through them)')
  ap.add_argument('--scale', type=float, default=1.0, help='fraction of each workload\'s envs (for a quick run)')
  args = ap.parse_args()
  print(json.dumps({'card': card()}), flush=True)
  for name, players, envs, n_focal in WORKLOADS:
    B = max(1, int(envs * args.scale))
    blob = substrates.load_blob(name, ('default',) * players)
    sub = substrate.BatchedSubstrate(blob, B, seed=3, world_rgb=False)
    is_focal = [p < n_focal for p in range(players)]
    n_bg = players - n_focal
    bg = lambda ts: torch.randint(0, sub.num_actions, (B, n_bg), device='cuda')
    sc = scenario.BatchedScenario(sub, bg, is_focal, ['RGB', 'READY_TO_SHOOT'])
    T = args.T
    traj = sc.trajectory(T)
    keep = {'RGB': torch.empty((T, B, n_focal) + tuple(sub.engine.rgb.shape[2:]), dtype=torch.uint8, device='cuda'),
            'reward': torch.empty((T, B, n_focal), dtype=torch.float64, device='cuda')}
    routes = sub.player_routes(torch.zeros((B, players), dtype=torch.int64))
    full = routes.outputs(T)
    acts = torch.randint(0, sub.num_actions, (B, n_focal), device='cuda')
    route_acts = routes.actions()
    rows = {'a': lambda t: sc.step(acts),
            'b': None, 'c': lambda t: sc.step(acts, out=traj.at(t)),
            'd': lambda t: sub.step(players=full.at(t), player_actions=route_acts)}

    def copy_arm(t):
      ts = sc.step(acts)
      keep['RGB'][t].copy_(ts.observation['RGB'])
      keep['reward'][t].copy_(ts.reward)
    rows['b'] = copy_arm
    sc.reset()
    sub.reset(players=full.at(0))
    times = {k: [] for k in rows}
    for k, fn in rows.items():  # warm-up
      for t in range(2):
        fn(t)
    torch.cuda.synchronize()
    for _ in range(args.rounds):
      for k, fn in rows.items():
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for i in range(args.steps):
          fn(i % T)
        end.record()
        torch.cuda.synchronize()
        times[k].append(start.elapsed_time(end) / args.steps)
    for k, v in times.items():
      v = sorted(v)
      print(json.dumps({'workload': f'{name} x {B} ({n_focal} focal / {n_bg} background), T={T}', 'arm': k,
                        'ms_per_step_median': round(v[len(v) // 2], 4), 'min': round(v[0], 4), 'max': round(v[-1], 4)}),
            flush=True)
    del sc, sub, traj, keep, full
    torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
