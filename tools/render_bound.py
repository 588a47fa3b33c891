"""Where k_render's time goes on this GPU: the write ceiling next to the kernel with and without its halves.

For each workload (substrate, players, envs) it times, with CUDA events over --launches back-to-back launches:
  fill_           torch fill_ of as many bytes as one render writes (the write-only HBM ceiling);
  copy_           torch copy_ of those bytes (read + write);
  full            k_render as it runs (render flags 3);
  stores_only     the strips are stored without being composed (flags 3 | MP_FLAG_DEBUG_NO_COMPOSE);
  compose_only    the strips are composed and never stored (flags 3 | MP_FLAG_DEBUG_NO_STORE);
  neither         only the skeleton: grid loads, per-cell pass, barriers, strip claims (both debug flags).
The render is timed on the state after --steps steps of uniform-random actions. GB/s are observation bytes written
per second. One JSON line per workload, the first line names the card and its power limit.

  python tools/render_bound.py [--launches 60] [--create-flags 0] [--out FILE]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bench import device_info  # noqa: E402
from meltingpot_b200 import engine, substrates  # noqa: E402

WORKLOADS = (('clean_up', 7, 4096), ('territory__rooms', 9, 2048), ('commons_harvest__open', 16, 8192))
NO_COMPOSE, NO_STORE = 16, 32


def timeit(fn, n):
  for _ in range(3):
    fn()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(n):
    fn()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / n


def measure(name, players, B, launches, steps, create_flags):
  blob = substrates.load_blob(name, ('default',) * players)
  eng = engine.Engine(blob, B, seed=1, flags=engine.MP_FLAG_DEFAULT | create_flags)
  eng.reset()
  gen = torch.Generator(device='cuda').manual_seed(0)
  for _ in range(steps):
    eng.step_state(torch.randint(0, eng.num_actions, (B, players), generator=gen, device='cuda', dtype=torch.int32))
  nbytes = eng.rgb.numel() + eng.world_rgb.numel()
  row = {'substrate': name, 'players': players, 'envs': B, 'launches': launches, 'obs_bytes': nbytes,
         'plan': {k: eng.render_plan().get(k) for k in ('teams', 'team_threads', 'wstrip_log2', 'slots', 'smem_bytes', 'atlas_sprites')}}
  ms = {}
  for label, fl in (('full', 0), ('stores_only', NO_COMPOSE), ('compose_only', NO_STORE), ('neither', NO_COMPOSE | NO_STORE)):
    eng.set_flags(engine.MP_FLAG_DEFAULT | fl)
    ms[label] = timeit(eng.render, launches)
  eng.set_flags(engine.MP_FLAG_DEFAULT)
  eng.close()
  x = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
  y = torch.empty(nbytes, dtype=torch.uint8, device='cuda')
  ms['fill_'] = timeit(lambda: x.fill_(7), launches)
  ms['copy_'] = timeit(lambda: y.copy_(x), launches)
  del x, y
  row['ms'] = {k: round(v, 4) for k, v in ms.items()}
  row['GBps'] = {k: round(nbytes / v / 1e6, 1) for k, v in ms.items()}
  row['full_over_fill'] = round(ms['full'] / ms['fill_'], 3)
  return row


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--launches', type=int, default=60)
  ap.add_argument('--steps', type=int, default=20, help='random steps before the render is timed')
  ap.add_argument('--create-flags', type=lambda s: int(s, 0), default=0, help='extra mp_create flags (e.g. a slot cap)')
  ap.add_argument('--out', help='also append the lines to this file')
  args = ap.parse_args()
  assert args.launches >= 50
  lines = [{'device': device_info(0), 'create_flags': args.create_flags}]
  for name, players, B in WORKLOADS:
    lines.append(measure(name, players, B, args.launches, args.steps, args.create_flags))
  for ln in lines:
    print(json.dumps(ln), flush=True)
  if args.out:
    with open(args.out, 'a') as f:
      for ln in lines:
        f.write(json.dumps(ln) + '\n')


if __name__ == '__main__':
  main()
