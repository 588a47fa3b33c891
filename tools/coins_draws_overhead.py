"""Cost of a coins batch over a set of draws (build_seeds: per-env map sizes and coin colours) on the GPU.

Times, in one process and alternating in rounds, coins x 2048 as a single-blob engine (the committed coins blob) and
as a mixed batch over the 16 stored draws of tests/coins_draws.py (envs interleaved over the draws, no episode cap).
CUDA events bracket the state transition (mp_step_state) and the render (mp_render) of every step; the medians over
rounds are printed with the card's name and power limit.

  python tools/coins_draws_overhead.py [--steps 600] [--warmup 50] [--rounds 6]
"""

import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.variant_overhead import _card  # noqa: E402

B = 2048


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=600, help='timed steps per engine (split over the rounds)')
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--rounds', type=int, default=6)
  args = ap.parse_args()
  import torch
  from meltingpot_b200 import engine, substrates
  from tests import coins_draws as CD
  print(f'card: {_card()}')
  per_round = max(1, args.steps // args.rounds)
  draws = CD.draw_set(capped=False)
  engines = {'single blob': engine.Engine(substrates.load_blob('coins', ('default',) * 2), B, seed=7),
             f'{len(draws)} draws': engine.Engine(list(draws), B, seed=7, env_variant=np.arange(B) % len(draws))}
  P, A = 2, engines['single blob'].num_actions
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
      ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(per_round)]
      for i, (a, b, c) in enumerate(ev):
        a.record()
        e.step_state(acts[i % 16])
        b.record()
        e.render()
        c.record()
      torch.cuda.synchronize()
      times[name][0].append(sum(a.elapsed_time(b) for a, b, _ in ev) / per_round)
      times[name][1].append(sum(b.elapsed_time(c) for _, b, c in ev) / per_round)
  print(f'\ncoins x {B}: {args.rounds} rounds x {per_round} steps per engine, after {args.warmup} warm-up steps')
  print(f'{"engine":<16}{"step ms":>10}{"render ms":>12}   (median over rounds; min..max)')
  base = [np.median(times['single blob'][k]) for k in (0, 1)]
  for name, (st, rd) in times.items():
    print(f'{name:<16}{np.median(st):>10.4f}{np.median(rd):>12.4f}   step {min(st):.4f}..{max(st):.4f} '
          f'({100 * (np.median(st) / base[0] - 1):+.1f} %), render {min(rd):.4f}..{max(rd):.4f} '
          f'({100 * (np.median(rd) / base[1] - 1):+.1f} %)')
  for e in engines.values():
    e.close()


if __name__ == '__main__':
  main()
