"""What per-player routing (mp_run's players) costs against a dense step and against gathering players after the step.

For each workload (clean_up x 4096 and commons_harvest__open 16p x 8192), alternating in rounds:

  a_step_into:    a step with `out`: a dense [B, P, h, w, 3] image target and reward;
  b_identity:     a step with players, row of player p of env b = b * P + p (the same bytes as a);
  c_permuted:     a step with players, a random permutation of those rows;
  d_half:         a step with players, a random half of the players unrouted (neither drawn nor stored);
  e_index_select: a plain step followed by BatchedScenario's split: index_select of the images and rewards on the player
                  axis, once for the focal and once for the background players (first / second half of the slots).

Step ms: CUDA events around --reps calls of each, in --rounds alternating rounds after a warm-up of every call; the
median and spread (min..max) over the rounds. k_render ms: torch.profiler over --prof calls of each, in a run of its own.
Prints one JSON line per (workload, call) with the GPU's name and power limit.

  python tools/player_routes_throughput.py [--reps 20] [--rounds 5] [--prof 10]
"""

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = (('clean_up', 7, 4096), ('commons_harvest__open', 16, 8192))
CALLS = ('a_step_into', 'b_identity', 'c_permuted', 'd_half', 'e_index_select')


def _gpu():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    return 'unknown'


def _calls(eng, B, P):
  import torch
  dev = torch.device('cuda', eng.device)
  gen = torch.Generator(device=dev).manual_seed(0)
  acts = torch.randint(0, eng.num_actions, (B, P), generator=gen, device=dev, dtype=torch.int32)
  h, w = eng.rgb.shape[2:4]
  dense = {'rgb': torch.empty((B, P, h, w, 3), dtype=torch.uint8, device=dev), 'reward': torch.empty((B, P), dtype=torch.float64, device=dev)}
  rows = torch.empty((B * P, h, w, 3), dtype=torch.uint8, device=dev)
  reward = torch.empty((B * P,), dtype=torch.float64, device=dev)
  rng = np.random.default_rng(0)
  ident = torch.arange(B * P, dtype=torch.int32, device=dev).view(B, P)
  perm = torch.from_numpy(rng.permutation(B * P).astype(np.int32)).to(dev).view(B, P)
  half = np.arange(B * P, dtype=np.int32)
  half[rng.random(B * P) < 0.5] = -1
  half = torch.from_numpy(half).to(dev).view(B, P)
  focal = torch.arange(0, P // 2, device=dev)
  background = torch.arange(P // 2, P, device=dev)

  def routed(m):
    return lambda: eng.step(acts, players={'row_of_player': m, 'rgb': rows, 'reward': reward})

  def split():
    eng.step(acts)
    for idx in (focal, background):
      eng.rgb.index_select(1, idx)
      eng.reward.index_select(1, idx)

  return {'a_step_into': lambda: eng.step(acts, out=dense), 'b_identity': routed(ident), 'c_permuted': routed(perm),
          'd_half': routed(half), 'e_index_select': split}, int((half >= 0).sum())


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--prof', type=int, default=10)
  ap.add_argument('--only', default='', help='run only this substrate')
  args = ap.parse_args()
  import torch
  from meltingpot_b200 import engine, substrates
  gpu = _gpu()
  for name, P, B in WORKLOADS:
    if args.only and name != args.only:
      continue
    eng = engine.Engine(substrates.load_blob(name, ('default',) * P), B, seed=1)
    eng.reset()
    calls, n_half = _calls(eng, B, P)
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
    render = {}
    for k, fn in calls.items():
      with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.prof):
          fn()
        torch.cuda.synchronize()
      us = [e.device_time_total for e in prof.key_averages() if 'k_render' in e.key]
      render[k] = sum(us) / args.prof / 1000.0
    for k in calls:
      t = sorted(times[k])
      print(json.dumps({'gpu': gpu, 'workload': f'{name} {P}p x {B}', 'call': k, 'step_ms': round(t[len(t) // 2], 4),
                        'step_ms_min': round(t[0], 4), 'step_ms_max': round(t[-1], 4), 'k_render_ms': round(render[k], 4),
                        'routed_players': n_half if k == 'd_half' else B * P}), flush=True)
    eng.close()
    del calls
    torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
