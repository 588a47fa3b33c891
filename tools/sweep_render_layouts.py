"""Times k_render at every feasible render layout of every shipped substrate (the data build_plan's score is fitted to).

For each substrate at its benchmark size it forces each (teams, warps, wstrip_log2) of the engine's search
(MP_RENDER_LAYOUT), skips the ones mp_create rejects as not fitting in shared memory, and times the render of the state
after --steps random steps with CUDA events over --launches launches. One JSON line per (substrate, layout), marked
`chosen` where it is the layout the engine picks by itself; the first line names the card and its power limit.

  python tools/sweep_render_layouts.py [--out profiles/render_layouts_h100.jsonl]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch  # noqa: E402

from bench import device_info  # noqa: E402
from meltingpot_b200 import engine, substrates  # noqa: E402

# (substrate, players, envs): bench.py config 5's sweep (2048 envs each), coop_mining, and the config 2-4 headline sizes
WORKLOADS = (('clean_up', 7, 2048), ('commons_harvest__open', 7, 2048), ('commons_harvest__closed', 7, 2048),
             ('commons_harvest__partnership', 7, 2048), ('territory__rooms', 9, 2048), ('territory__open', 9, 2048),
             ('territory__inside_out', 5, 2048), ('coins', 2, 2048), ('coop_mining', 6, 2048),
             ('clean_up', 7, 4096), ('commons_harvest__open', 16, 8192))


def time_render(eng, launches):
  for _ in range(3):
    eng.render()
  torch.cuda.synchronize()
  a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  a.record()
  for _ in range(launches):
    eng.render()
  b.record()
  torch.cuda.synchronize()
  return a.elapsed_time(b) / launches


def sweep(name, players, B, launches, steps):
  blob = substrates.load_blob(name, ('default',) * players)
  gen = torch.Generator(device='cuda').manual_seed(0)
  actions = [torch.randint(0, 64, (B, players), generator=gen, device='cuda', dtype=torch.int32) for _ in range(steps)]
  probe = engine.Engine(blob, 1, seed=1)
  plan = probe.render_plan()
  chosen = (plan['teams'], plan['team_threads'] // 32, plan['wstrip_log2'])
  probe.close()
  rows = []
  for lay in engine.render_layout_candidates():
    try:
      eng = engine.Engine(blob, B, seed=1, render_layout=lay)
    except ValueError:
      continue  # does not fit in shared memory
    eng.reset()
    for a in actions:
      eng.step_state(a % eng.num_actions)
    p = eng.render_plan()
    ms = time_render(eng, launches)
    eng.close()
    rows.append({'substrate': name, 'players': players, 'envs': B, 'teams': lay[0], 'warps': lay[1], 'wstrip_log2': lay[2],
                 'slots': p.get('slots', 1), 'smem_bytes': p['smem_bytes'], 'render_ms': round(ms, 4), 'chosen': lay == chosen})
  return rows


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--launches', type=int, default=50)
  ap.add_argument('--steps', type=int, default=10)
  ap.add_argument('--out', help='write the lines to this file as well')
  args = ap.parse_args()
  lines = [{'device': device_info(0)}]
  for w in WORKLOADS:
    lines += sweep(*w, args.launches, args.steps)
  for ln in lines:
    print(json.dumps(ln), flush=True)
  if args.out:
    os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
    with open(args.out, 'w') as f:
      for ln in lines:
        f.write(json.dumps(ln) + '\n')


if __name__ == '__main__':
  main()
