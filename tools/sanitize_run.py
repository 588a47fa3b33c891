"""Small workload for compute-sanitizer (memcheck / racecheck / synccheck) on the engine's kernels.

  compute-sanitizer --tool memcheck  python tools/sanitize_run.py
  compute-sanitizer --tool racecheck python tools/sanitize_run.py
"""
import os, sys
sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import torch
from meltingpot_b200 import engine, substrates

CASES = (('clean_up', 7, 9, 700), ('commons_harvest__open', 16, 8, 700), ('territory__rooms', 9, 9, 400),
         ('territory__open', 9, 9, 400), ('territory__inside_out', 5, 9, 300), ('coins', 2, 7, 700), ('coop_mining', 6, 8, 500))
only = sys.argv[1:]
for name, players, n_act, B in CASES:
  if only and name not in only:
    continue
  roles = ('default',) * players
  blob = substrates.load_blob(name, roles)
  eng = engine.Engine(blob, B, seed=3)   # more envs than render teams, so that teams process several envs each
  if name in ('clean_up', 'territory__rooms'):  # world-of-one exchange + observation gather: the peer stores land locally
    ptr, _ = eng.exchange_create(0, 1); eng.exchange_connect([ptr])
    ptr, _ = eng.gather_obs_create(0, 1); eng.gather_obs_connect([ptr])
  eng.reset()
  gen = torch.Generator(device='cuda').manual_seed(0)
  for _ in range(8):
    eng.step(torch.randint(0, n_act, (B, len(roles)), generator=gen, device='cuda', dtype=torch.int32))
    if name in ('clean_up', 'territory__rooms'):
      eng.exchange_wait(); eng.gather_obs_wait()
  eng.debug_observations()
  if name not in ('clean_up', 'territory__rooms'):  # state bank (a restore is refused once peers are connected)
    bank = torch.zeros((4, eng.state_record_bytes), dtype=torch.uint8, device='cuda')
    eng.store_states(bank, torch.tensor([0, B - 1, -1, B], dtype=torch.int32, device='cuda'))  # rows 2, 3 skipped
    slots = torch.full((B,), -1, dtype=torch.int32, device='cuda')
    slots[1::3] = 0; slots[2::5] = 1; slots[3::7] = 2   # fan-out, and row 2 is untagged
    eng.restore_states(bank, slots); eng.restore_states(bank, slots, rekey=True)
    eng.step(torch.randint(0, n_act, (B, len(roles)), generator=gen, device='cuda', dtype=torch.int32))
  torch.cuda.synchronize()
  if name in ('clean_up', 'territory__rooms'):
    assert torch.equal(eng.gathered_timestep(), eng.timestep_packed) and torch.equal(eng.gathered_observations()[0], eng.rgb)
  snap = eng.save_state(); eng.load_state(snap)
  print(name, 'ok', int(eng.rgb.sum()) % 1000, eng.launch_count(), int(eng.event_count.sum()), eng.render_plan())
  eng.close()
