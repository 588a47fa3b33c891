"""What storing and restoring every env of a batch costs: ms per call and bytes per second of the state-bank kernels.

For each workload (clean_up x 4096 and commons_harvest__open 16p x 8192, each with and without WORLD.RGB):

  store:           mp_state_store of all B envs into a bank of B rows (one kernel);
  restore_kernel:  mp_state_restore of all B envs with rendering switched off (the kernel alone);
  render:          mp_render (what a restore re-renders);
  restore:         mp_state_restore with rendering on (kernel + render);
  step:            a plain step with uniform-random actions, for scale;
  d2d_copy:        a device-to-device copy of the same 2 x record_bytes x B bytes (read + write), the bandwidth yardstick;
  step_restore:    a step that restores a fraction of the envs instead of advancing them (mp_run's slot_of_env and bank);
  step+restore:    a step followed by mp_state_restore of the same envs (what step_restore replaces).
The last two run at restored fractions 0, 1/64, 1/8 and 1 of B (field `restored`: envs restored per call, spread evenly
over the batch).

Timed with CUDA events over --reps calls after a warm-up of every call. The kernels' rate is reported against the bytes
they have to move, 2 x record_bytes x B (each record is read once and written once). Prints one JSON line per
(workload, call) with the GPU's name and power limit.

  python tools/state_bank_throughput.py [--reps 50] [--only clean_up]
"""

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = (('clean_up', 7, 4096), ('commons_harvest__open', 16, 8192))
FRACTIONS = ((0, 1), (1, 64), (1, 8), (1, 1))


def _gpu():
  try:
    return subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                          capture_output=True, text=True, timeout=30).stdout.strip()
  except (OSError, subprocess.SubprocessError):
    return 'unknown'


def _time(fn, reps):
  import torch
  start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
  start.record()
  for _ in range(reps):
    fn()
  end.record()
  end.synchronize()
  return start.elapsed_time(end) / reps


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--reps', type=int, default=50)
  ap.add_argument('--only', default='', help='run only this substrate')
  args = ap.parse_args()
  import torch
  from meltingpot_b200 import engine, substrates
  if not torch.cuda.is_available():
    raise SystemExit('needs a CUDA device')
  gpu = _gpu()
  for name, players, B in WORKLOADS:
    if args.only and name != args.only:
      continue
    blob = substrates.load_blob(name, ('default',) * players)
    for world in (True, False):
      flags = engine.MP_FLAG_RENDER_PLAYERS | (engine.MP_FLAG_RENDER_WORLD if world else 0)
      eng = engine.Engine(blob, B, device=0, seed=1, flags=flags)
      P, A, R = eng.num_players, eng.num_actions, eng.state_record_bytes
      gen = torch.Generator(device='cuda').manual_seed(0)
      actions = [torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32) for _ in range(8)]
      bank = torch.zeros((B, R), dtype=torch.uint8, device='cuda')
      every = torch.arange(B, dtype=torch.int32, device='cuda')
      eng.reset()
      for a in actions:
        eng.step(a)
      k = [0]

      def step():
        eng.step(actions[k[0] % len(actions)])
        k[0] += 1

      def restore_kernel():
        eng.set_flags(0)
        eng.restore_states(bank, every)
        eng.set_flags(flags)

      copy_src = torch.empty((B * R,), dtype=torch.uint8, device='cuda')
      copy_dst = torch.empty_like(copy_src)
      calls = {'store': lambda: eng.store_states(bank, every), 'restore_kernel': restore_kernel, 'render': eng.render,
               'restore': lambda: eng.restore_states(bank, every), 'step': step, 'd2d_copy': lambda: copy_dst.copy_(copy_src)}
      restored = {}
      for num, den in FRACTIONS:
        n = B * num // den
        idx = torch.full((B,), -1, dtype=torch.int32, device='cuda')
        if n:
          envs = torch.arange(0, B, B // n, device='cuda')[:n]
          idx[envs] = envs.to(torch.int32)

        def step_restore(idx=idx):
          eng.step(actions[k[0] % len(actions)], restore=idx, bank=bank)
          k[0] += 1

        def step_then_restore(idx=idx):
          step()
          eng.restore_states(bank, idx)

        tag = f'{num}/{den}'
        calls[f'step_restore {tag}'] = step_restore
        calls[f'step+restore {tag}'] = step_then_restore
        restored[f'step_restore {tag}'] = restored[f'step+restore {tag}'] = n
      for fn in calls.values():  # warm-up
        for _ in range(3):
          fn()
      torch.cuda.synchronize()
      moved = 2 * R * B
      for call, fn in calls.items():
        ms = _time(fn, args.reps)
        row = dict(substrate=name, players=P, envs=B, world_rgb=world, call=call, ms=round(ms, 4), record_bytes=R,
                   reps=args.reps, gpu=gpu)
        if call in restored:
          row['restored'] = restored[call]
        if call in ('store', 'restore_kernel', 'd2d_copy'):
          row['bytes'] = moved
          row['GB_per_s'] = round(moved / (ms * 1e-3) / 1e9, 1)
        print(json.dumps(row), flush=True)
      eng.close()


if __name__ == '__main__':
  main()
