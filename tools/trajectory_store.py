"""What keeping a learner's trajectory costs per step: ms per step of three loops over T slots, in both layouts.

  (a) copy:  step(), then copy_ of every output into slot t of the trajectory (what a loop had to do before step(out=));
  (b) into:  step(out=traj.at(t)): the engine renders and delivers straight into slot t;
  (c) plain: step() keeping nothing.

Timed with CUDA events over alternated rounds after a warm-up of every loop, on clean_up x 4096, T = 8 by default.
Prints one JSON line per (layout, loop) and the GPU's name and power limit with them.

  python tools/trajectory_store.py [--envs 4096] [--T 8] [--rounds 6] [--substrate clean_up]
"""

import argparse
import json
import os
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def _gpu():
  try:
    q = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit', '--format=csv,noheader', '-i', '0'],
                       capture_output=True, text=True, timeout=30).stdout.strip()
    return q
  except (OSError, subprocess.SubprocessError):
    return 'unknown'


def main():
  ap = argparse.ArgumentParser()
  ap.add_argument('--substrate', default='clean_up')
  ap.add_argument('--envs', type=int, default=4096)
  ap.add_argument('--T', type=int, default=8)
  ap.add_argument('--rounds', type=int, default=6, help='alternated rounds of T steps per loop and layout')
  args = ap.parse_args()
  import torch
  from meltingpot_b200 import substrate
  if not torch.cuda.is_available():
    raise SystemExit('needs a CUDA device')
  cfg = substrate.get_config(args.substrate)
  sub = substrate.build_batched(args.substrate, roles=cfg.default_player_roles, num_envs=args.envs, seed=1)
  B, P, A, T = sub.num_envs, sub.num_players, sub.num_actions, args.T
  gen = torch.Generator(device='cuda').manual_seed(0)
  actions = [torch.randint(0, A, (B, P), generator=gen, device='cuda', dtype=torch.int32) for _ in range(T)]
  trajs = {'time_major': sub.trajectory(T, True), 'env_major': sub.trajectory(T, False)}
  sub.reset()

  def copy_loop(traj):
    for t in range(T):
      ts = sub.step(actions[t])
      slot = traj.at(t)
      slot.step_type.copy_(ts.step_type); slot.reward.copy_(ts.reward); slot.discount.copy_(ts.discount)
      for k, v in ts.observation.items():
        slot.observation[k].copy_(v)

  def into_loop(traj):
    for t in range(T):
      sub.step(actions[t], out=traj.at(t))

  def plain_loop(traj):
    del traj
    for t in range(T):
      sub.step(actions[t])

  loops = {'a_copy': copy_loop, 'b_into': into_loop, 'c_plain': plain_loop}
  for traj in trajs.values():  # warm-up: every loop and layout
    for fn in loops.values():
      fn(traj)
  torch.cuda.synchronize()
  times = {(lay, name): [] for lay in trajs for name in loops}
  for _ in range(args.rounds):
    for lay, traj in trajs.items():
      for name, fn in loops.items():
        start, end = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        start.record()
        fn(traj)
        end.record()
        end.synchronize()
        times[(lay, name)].append(start.elapsed_time(end) / T)
  gpu = _gpu()
  for (lay, name), ms in times.items():
    ms = sorted(ms)
    print(json.dumps(dict(substrate=args.substrate, envs=B, T=T, layout=lay, loop=name, ms_per_step_median=ms[len(ms) // 2],
                          ms_per_step_min=ms[0], ms_per_step_max=ms[-1], rounds=len(ms), gpu=gpu)))
  sub.close()


if __name__ == '__main__':
  main()
