"""What running territory and coop_mining maps side by side costs, on the GPU.

Times, in one process and alternating in rounds, territory__rooms x 2048 and coop_mining x 2048, each in three
configurations:
  (a) one blob: the substrate's own map,
  (b) four copies of that map as a map set: the map-variant kernel (territory: tables staged per warp) on one layout,
  (c) the four maps of tests/territory_maps.py (own, walls moved, resource / ore count changed, spawns moved) as one
      map set, envs interleaved, so the four envs of a CTA run four maps.
CUDA events bracket the state transition (mp_step_state) and the render (mp_render). The settings are the recorded ones
with the 40-frame cap of the tests, so the timed window crosses many episode starts. Medians over rounds are printed
with min..max and the card's name and power limit.

  python tools/territory_maps_throughput.py [--steps 600] [--warmup 50] [--rounds 6]
"""

import argparse
import os
import sys

import numpy as np

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
from tools.variant_overhead import _card  # noqa: E402

WORKLOADS = (('territory__rooms', 2048), ('coop_mining', 2048))


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--steps', type=int, default=600, help='timed steps per configuration (split over the rounds)')
  ap.add_argument('--warmup', type=int, default=50)
  ap.add_argument('--rounds', type=int, default=6)
  args = ap.parse_args()
  import torch
  from meltingpot_b200 import engine
  from tests import territory_maps as TM
  print(f'card: {_card()}')
  per_round = max(1, args.steps // args.rounds)
  for name, B in WORKLOADS:
    blobs = TM.map_set(name)
    assign = np.arange(B) % 4
    engines = {'(a) one blob': engine.Engine(blobs[0], B, seed=7),
               '(b) own map x 4 as a set': engine.Engine([blobs[0]] * 4, B, seed=7, env_variant=assign),
               '(c) 4 maps, interleaved': engine.Engine(list(blobs), B, seed=7, env_variant=assign)}
    P, A = engines['(a) one blob'].num_players, engines['(a) one blob'].num_actions
    gen = torch.Generator(device='cuda').manual_seed(0)
    acts = [torch.randint(0, A, (B, P), device='cuda', dtype=torch.int32, generator=gen) for _ in range(16)]

    def run(e, i, ev):
      ev[0].record()
      e.step_state(acts[i % 16])
      ev[1].record()
      e.render()
      ev[2].record()

    for e in engines.values():
      e.reset()
    for i in range(args.warmup):
      for e in engines.values():
        run(e, i, [torch.cuda.Event(enable_timing=True) for _ in range(3)])
    torch.cuda.synchronize()
    times = {k: ([], [], []) for k in engines}
    for _ in range(args.rounds):
      for k, e in engines.items():
        ev = [[torch.cuda.Event(enable_timing=True) for _ in range(3)] for _ in range(per_round)]
        for i, e3 in enumerate(ev):
          run(e, i, e3)
        torch.cuda.synchronize()
        times[k][0].append(sum(a.elapsed_time(b) for a, b, _ in ev) / per_round)
        times[k][1].append(sum(b.elapsed_time(c) for _, b, c in ev) / per_round)
        times[k][2].append(sum(a.elapsed_time(c) for a, _, c in ev) / per_round)
    print(f'\n{name} x {B}, {P} players: {args.rounds} rounds x {per_round} steps each, after {args.warmup} warm-up steps')
    print(f'{"configuration":<28}{"step ms":>10}{"render ms":>12}{"total ms":>11}   (median over rounds; min..max)')
    base = {j: np.median(times['(a) one blob'][j]) for j in range(3)}
    for k, (st, rd, tot) in times.items():
      print(f'{k:<28}{np.median(st):>10.4f}{np.median(rd):>12.4f}{np.median(tot):>11.4f}   '
            f'step {min(st):.4f}..{max(st):.4f}, render {min(rd):.4f}..{max(rd):.4f} '
            f'(step {100 * (np.median(st) / base[0] - 1):+.1f} %, render {100 * (np.median(rd) / base[1] - 1):+.1f} % vs (a))')
    for e in engines.values():
      e.close()


if __name__ == '__main__':
  main()
