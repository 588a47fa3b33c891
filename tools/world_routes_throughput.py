"""What routing WORLD.RGB to a few envs (mp_player_outputs.world_row_of_env) costs against not rendering it and against
rendering it for every env.

For each workload (clean_up x 4096 and commons_harvest__open 16p x 8192), every player routed to its own row
(a step with players, identity rows), alternating in rounds:

  a_world_off:   the engine built without WORLD.RGB (render flags: player images only);
  b_world_dense: WORLD.RGB rendered for every env into the engine's own buffer;
  c_world_8:     WORLD.RGB routed to 8 scattered envs, the others not rendered;
  d_world_q:     WORLD.RGB routed to B / 4 scattered envs.

Step ms: CUDA events around --reps calls of each, in --rounds alternating rounds after a warm-up of every call; the
median and spread (min..max) over the rounds. k_render ms: torch.profiler over --prof calls of each, in a run of its own.
Prints one JSON line per (workload, call) with the GPU's name and power limit.

  python tools/world_routes_throughput.py [--reps 20] [--rounds 5] [--prof 10]
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
CALLS = ('a_world_off', 'b_world_dense', 'c_world_8', 'd_world_q')


def _gpu():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    return 'unknown'


def _calls(eng_off, eng, B, P):
  import torch
  dev = torch.device('cuda', eng.device)
  gen = torch.Generator(device=dev).manual_seed(0)
  acts = torch.randint(0, eng.num_actions, (B, P), generator=gen, device=dev, dtype=torch.int32)
  h, w = eng.rgb.shape[2:4]
  rows = torch.empty((B * P, h, w, 3), dtype=torch.uint8, device=dev)
  reward = torch.empty((B * P,), dtype=torch.float64, device=dev)
  ident = torch.arange(B * P, dtype=torch.int32, device=dev).view(B, P)
  players = {'row_of_player': ident, 'rgb': rows, 'reward': reward}
  rng = np.random.default_rng(0)

  def world(n):
    envs = torch.from_numpy(rng.choice(B, size=n, replace=False)).to(dev)
    m = torch.full((B,), -1, dtype=torch.int32, device=dev)
    m[envs] = torch.arange(n, dtype=torch.int32, device=dev)
    target = torch.empty((n,) + tuple(eng.world_rgb.shape[1:]), dtype=torch.uint8, device=dev)
    return dict(players, world_row_of_env=m, world_rgb=target)

  w8, wq = world(8), world(B // 4)
  return {'a_world_off': lambda: eng_off.step(acts, players=players),
          'b_world_dense': lambda: eng.step(acts, players=players),
          'c_world_8': lambda: eng.step(acts, players=w8),
          'd_world_q': lambda: eng.step(acts, players=wq)}, {'a_world_off': 0, 'b_world_dense': B, 'c_world_8': 8,
                                                             'd_world_q': B // 4}


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
    blob = substrates.load_blob(name, ('default',) * P)
    eng_off = engine.Engine(blob, B, seed=1, flags=engine.MP_FLAG_RENDER_PLAYERS)
    eng = engine.Engine(blob, B, seed=1)
    eng_off.reset(); eng.reset()
    calls, n_world = _calls(eng_off, eng, B, P)
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
                        'world_envs': n_world[k]}), flush=True)
    eng.close(); eng_off.close()
    del calls
    torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
