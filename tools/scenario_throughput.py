"""What actions read from rows (mp_run's player_actions) cost against dense actions, and what BatchedScenario's step costs on
player routes against the index_select / index_copy_ split it replaced.

For each workload (clean_up 7p x 4096 with 5 focal / 2 background players, commons_harvest__open 16p x 8192 with
12 / 4), alternating in rounds:

  a_dense:            a step with dense [B, P] actions;
  b_rows_identity:    a step with player_actions, row of player p of env b = b * P + p (the same actions as a);
  c_rows_permuted:    a step with player_actions, a random permutation of those rows;
  d_scenario_split:   the scenario step of the previous BatchedScenario, reproduced here: index_copy_ of the focal and
                      background actions into [B, P], a plain step, then index_select of every per-player output, once
                      for the focal and once for the background players;
  e_scenario_routes:  BatchedScenario.step (player routes: observations drawn into rows, actions read from rows).

The background policy returns a constant tensor, so the scenario calls time the engine and the routing alone.
Step ms: CUDA events around --reps calls of each, in --rounds alternating rounds after a warm-up of every call; the
median and spread (min..max) over the rounds. k_step and k_render ms: torch.profiler over --prof calls of each, in a run
of its own. Prints one JSON line per (workload, call) with the GPU's name and power limit.

  python tools/scenario_throughput.py [--reps 20] [--rounds 5] [--prof 10] [--only clean_up]
"""

import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = (('clean_up', 7, 5, 4096), ('commons_harvest__open', 16, 12, 8192))
CALLS = ('a_dense', 'b_rows_identity', 'c_rows_permuted', 'd_scenario_split', 'e_scenario_routes')


def _gpu():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    return 'unknown'


def _calls(sub, sc, B, P, n_focal):
  import torch
  eng = sub.engine
  dev = torch.device('cuda', eng.device)
  gen = torch.Generator(device=dev).manual_seed(0)
  acts = torch.randint(0, eng.num_actions, (B, P), generator=gen, device=dev, dtype=torch.int32)
  rng = np.random.default_rng(0)
  ident = torch.arange(B * P, dtype=torch.int32, device=dev).view(B, P)
  perm = torch.from_numpy(rng.permutation(B * P).astype(np.int32)).to(dev).view(B, P)
  rows_ident = acts.reshape(-1).clone()
  rows_perm = torch.empty_like(rows_ident)
  rows_perm[perm.reshape(-1).long()] = acts.reshape(-1)  # the same [B, P] actions as a_dense
  focal_actions = acts[:, :n_focal].contiguous()
  focal_idx = torch.arange(0, n_focal, device=dev)
  background_idx = torch.arange(n_focal, P, device=dev)
  background_actions = acts[:, n_focal:].contiguous()
  full = torch.zeros((B, P), dtype=torch.int32, device=dev)

  def split():
    full.index_copy_(1, focal_idx, focal_actions)
    full.index_copy_(1, background_idx, background_actions)
    ts = sub.step(full)
    for idx in (background_idx, focal_idx):
      for key, value in ts.observation.items():
        if key not in ('WORLD.RGB', 'COLLECTIVE_REWARD'):
          value.index_select(1, idx)
      ts.reward.index_select(1, idx)

  return {'a_dense': lambda: eng.step(acts),
          'b_rows_identity': lambda: eng.step(None, player_actions={'row_of_player': ident, 'action': rows_ident}),
          'c_rows_permuted': lambda: eng.step(None, player_actions={'row_of_player': perm, 'action': rows_perm}),
          'd_scenario_split': split,
          'e_scenario_routes': lambda: sc.step(focal_actions)}


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=20)
  ap.add_argument('--rounds', type=int, default=5)
  ap.add_argument('--prof', type=int, default=10)
  ap.add_argument('--only', default='', help='run only this substrate')
  args = ap.parse_args()
  import torch
  import torch._inductor  # pylint: disable=unused-import  (the profiler imports it; before the dm_env shims' stand-in modules)
  from meltingpot_b200 import scenario, substrate, substrates
  gpu = _gpu()
  for name, P, n_focal, B in WORKLOADS:
    if args.only and name != args.only:
      continue
    sub = substrate.BatchedSubstrate(substrates.load_blob(name, ('default',) * P), B, seed=1)
    background = torch.ones((B, P - n_focal), dtype=torch.int32, device='cuda')
    sc = scenario.BatchedScenario(sub, lambda ts, a=background: a, (True,) * n_focal + (False,) * (P - n_focal),
                                  permitted_observations={'RGB', 'READY_TO_SHOOT', 'COLLECTIVE_REWARD'})
    sc.reset()
    calls = _calls(sub, sc, B, P, n_focal)
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
    kernels = {}
    for k, fn in calls.items():
      with torch.profiler.profile(activities=[torch.profiler.ProfilerActivity.CUDA]) as prof:
        for _ in range(args.prof):
          fn()
        torch.cuda.synchronize()
      avg = prof.key_averages()
      kernels[k] = {kern: sum(e.device_time_total for e in avg if kern in e.key) / args.prof / 1000.0 for kern in ('k_step', 'k_render')}
    for k in calls:
      t = sorted(times[k])
      print(json.dumps({'gpu': gpu, 'workload': f'{name} {P}p x {B} ({n_focal} focal)', 'call': k,
                        'step_ms': round(t[len(t) // 2], 4), 'step_ms_min': round(t[0], 4), 'step_ms_max': round(t[-1], 4),
                        'k_step_ms': round(kernels[k]['k_step'], 4), 'k_render_ms': round(kernels[k]['k_render'], 4)}), flush=True)
    sub.close()
    del calls, sc, sub
    torch.cuda.empty_cache()


if __name__ == '__main__':
  main()
