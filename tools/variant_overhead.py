"""Cost of per-env parameter variants (mp_create_variants) on the GPU.

For each workload it times three engines in one process, alternating them in rounds: a single-blob engine, the same
blob passed as 4 identical variants (the variant kernel, envs interleaved over the four copies) and 4 different
variants (tests/env_variants.py: the stored settings with a 40-frame episode cap, prefab overrides on map pieces and
one avatar-level knob). CUDA events bracket the state transition (mp_step_state) and whole steps (state transition +
render) of each round; the medians over rounds are printed with the card's name and power limit.

  python tools/variant_overhead.py [--steps 600] [--warmup 50] [--rounds 6]
"""

import argparse
import os
import subprocess
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

WORKLOADS = (('clean_up', 4096), ('territory', 2048))


def _card():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                          capture_output=True, text=True, check=True).stdout.strip().splitlines()[0]
  except (OSError, subprocess.CalledProcessError):
    import torch
    return torch.cuda.get_device_name(0) + ', power limit not readable'


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=600, help='timed steps per engine (split over the rounds)')
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--rounds', type=int, default=6)
  args = ap.parse_args()
  import torch
  from meltingpot_b200 import engine
  from tests import env_variants as EV
  print(f'card: {_card()}')
  per_round = max(1, args.steps // args.rounds)
  for family, B in WORKLOADS:
    blobs = EV.blobs(family)
    assign = EV.interleaved(B, 4)
    engines = {'single blob': engine.Engine(blobs[0], B, seed=7),
               '4 identical variants': engine.Engine([blobs[0]] * 4, B, seed=7, env_variant=assign),
               '4 different variants': engine.Engine(list(blobs), B, seed=7, env_variant=assign)}
    P, A = engines['single blob'].num_players, engines['single blob'].num_actions
    gen = torch.Generator(device='cuda').manual_seed(0)
    acts = [torch.randint(0, A, (B, P), device='cuda', dtype=torch.int32, generator=gen) for _ in range(16)]
    for e in engines.values():
      e.reset()
      for i in range(args.warmup):
        e.step(acts[i % 16])
    torch.cuda.synchronize()
    times = {k: ([], []) for k in engines}
    for _ in range(args.rounds):
      for name, e in engines.items():
        marks = [(torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)) for _ in range(per_round)]
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        for i, (a, b) in enumerate(marks):
          a.record()
          e.step_state(acts[i % 16])
          b.record()
          e.render()
        end.record()
        end.synchronize()
        times[name][0].append(sum(a.elapsed_time(b) for a, b in marks) / per_round)
        times[name][1].append(start.elapsed_time(end) / per_round)
    print(f'\n{family} x {B}: {args.rounds} rounds x {per_round} steps per engine, after {args.warmup} warm-up steps')
    print(f'{"engine":<24}{"mp_step_state ms":>18}{"whole step ms":>16}   (median over rounds; min..max)')
    base = np.median(times['single blob'][0])
    for name, (st, whole) in times.items():
      print(f'{name:<24}{np.median(st):>18.4f}{np.median(whole):>16.4f}   state {min(st):.4f}..{max(st):.4f}, '
            f'step {min(whole):.4f}..{max(whole):.4f}, state vs single blob {100 * (np.median(st) / base - 1):+.1f} %')
    for e in engines.values():
      e.close()


if __name__ == '__main__':
  main()
