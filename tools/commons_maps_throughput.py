"""Throughput of commons_harvest__open, __closed and __partnership run side by side, on the GPU.

Times, in one process and alternating in rounds, B = 4096 envs of
  (a) the single-blob commons_harvest__open engine,
  (b) one engine over the three maps (map variants), envs interleaved,
  (c) three homogeneous engines of ceil(B/3) / floor(B/3) envs, stepped in turn into slices of one set of output tensors
      with step(out=...): what running the three maps took before they could share an engine.
CUDA events bracket the state transition (mp_step_state) and the render (mp_render) of (a) and (b), and the three
step(out=...) calls of (c), which step and render. The committed blobs are used (5000-frame episodes). Medians over
rounds are printed with min..max and the card's name and power limit.

  python tools/commons_maps_throughput.py [--steps 600] [--warmup 50] [--rounds 6]
"""

import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.variant_overhead import _card  # noqa: E402

B = 4096
NAMES = ('commons_harvest__open', 'commons_harvest__closed', 'commons_harvest__partnership')
ROLES = ('default',) * 7


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=600, help='timed steps per configuration (split over the rounds)')
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--rounds', type=int, default=6)
  args = ap.parse_args()
  import torch
  from meltingpot_b200 import engine, substrates
  print(f'card: {_card()}')
  per_round = max(1, args.steps // args.rounds)
  blobs = [substrates.load_blob(n, ROLES) for n in NAMES]
  single = engine.Engine(blobs[0], B, seed=7)
  mixed = engine.Engine(blobs, B, seed=7, env_variant=np.arange(B) % 3)
  sizes = [(B + 2 - v) // 3 for v in range(3)]  # ceil, then floor
  bounds = np.cumsum([0] + sizes)
  three = [engine.Engine(b, n, seed=7, env_index_base=int(lo)) for b, n, lo in zip(blobs, sizes, bounds)]
  out = {k: torch.empty_like(getattr(single, k)) for k in engine.DEVICE_OUTPUTS}
  slices = [{k: (v[:, lo:hi] if k == 'scalar_obs' else v[lo:hi]) for k, v in out.items()} for lo, hi in zip(bounds, bounds[1:])]
  P, A = single.num_players, single.num_actions
  gen = torch.Generator(device='cuda').manual_seed(0)
  acts = [torch.randint(0, A, (B, P), device='cuda', dtype=torch.int32, generator=gen) for _ in range(16)]
  acts_of = [[a[lo:hi].contiguous() for lo, hi in zip(bounds, bounds[1:])] for a in acts]

  def step_split(e, i, ev):
    ev[0].record()
    e.step_state(acts[i % 16])
    ev[1].record()
    e.render()
    ev[2].record()

  def step_three(i, ev):
    ev[0].record()
    for e, a, o in zip(three, acts_of[i % 16], slices):
      e.step(a, out=o)
    ev[2].record()

  runs = {'(a) open alone': lambda i, ev: step_split(single, i, ev),
          '(b) 3 maps, 1 engine': lambda i, ev: step_split(mixed, i, ev),
          '(c) 3 engines, out=': step_three}
  for e in [single, mixed] + three:
    e.reset()
  for i in range(args.warmup):
    for run in runs.values():
      run(i, [torch.cuda.Event(enable_timing=True) for _ in range(3)])
  torch.cuda.synchronize()
  times = {k: ([], [], []) for k in runs}
  for _ in range(args.rounds):
    for name, run in runs.items():
      ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(per_round)]
      for i, e3 in enumerate(ev):
        run(i, e3)
      torch.cuda.synchronize()
      split = name != '(c) 3 engines, out='
      times[name][0].append(sum(a.elapsed_time(b) for a, b, _ in ev) / per_round if split else float('nan'))
      times[name][1].append(sum(b.elapsed_time(c) for _, b, c in ev) / per_round if split else float('nan'))
      times[name][2].append(sum(a.elapsed_time(c) for a, _, c in ev) / per_round)
  print(f'\ncommons_harvest x {B}, 7 players: {args.rounds} rounds x {per_round} steps each, after {args.warmup} warm-up steps')
  print(f'{"configuration":<24}{"step ms":>10}{"render ms":>12}{"total ms":>11}   (median over rounds; total min..max)')
  base = np.median(times['(a) open alone'][2])
  for name, (st, rd, tot) in times.items():
    print(f'{name:<24}{np.median(st):>10.4f}{np.median(rd):>12.4f}{np.median(tot):>11.4f}   {min(tot):.4f}..{max(tot):.4f} '
          f'({100 * (np.median(tot) / base - 1):+.1f} % vs (a))')
  for e in [single, mixed] + three:
    e.close()


if __name__ == '__main__':
  main()
