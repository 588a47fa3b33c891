"""Snapshot / restore of the batched engine state (SURVEY.md section 8f, row N4)."""

import numpy as np
import pytest

pytestmark = pytest.mark.gpu


def _play(eng, acts):
  import torch
  out = []
  for a in acts:
    eng.step(torch.from_numpy(a).cuda())
    torch.cuda.synchronize()
    out.append((eng.reward.cpu().numpy().copy(), eng.step_type.cpu().numpy().copy(), eng.discount.cpu().numpy().copy()))
  return out, eng.rgb.cpu().numpy().copy(), eng.world_rgb.cpu().numpy().copy(), eng.grid.cpu().numpy().copy()


@pytest.mark.parametrize('fixture', ['clean_up_blob', 'commons_blob', 'territory_blob', 'coins_blob', 'coop_mining_blob',
                                     'territory_inside_out_blob'])
def test_restore_replays_identically(fixture, request):
  import torch
  from meltingpot_b200 import engine
  blob = request.getfixturevalue(fixture)
  B = 24
  eng = engine.Engine(blob, B, device=0, seed=21)
  P, A = eng.num_players, eng.num_actions
  rng = np.random.default_rng(3)
  warm = [np.ascontiguousarray(rng.integers(0, A, (B, P)), np.int32) for _ in range(60)]
  tail = [np.ascontiguousarray(rng.integers(0, A, (B, P)), np.int32) for _ in range(80)]
  eng.reset()
  _play(eng, warm)
  snap = eng.save_state()
  at_snapshot = (eng.rgb.cpu().numpy().copy(), eng.world_rgb.cpu().numpy().copy(), eng.reward.cpu().numpy().copy())
  first = _play(eng, tail)

  eng.load_state(snap)  # same engine, rewound
  torch.cuda.synchronize()
  np.testing.assert_array_equal(eng.rgb.cpu().numpy(), at_snapshot[0])  # observations are re-rendered on load
  np.testing.assert_array_equal(eng.world_rgb.cpu().numpy(), at_snapshot[1])
  np.testing.assert_array_equal(eng.reward.cpu().numpy(), at_snapshot[2])
  second = _play(eng, tail)

  other = engine.Engine(blob, B, device=0, seed=21)  # a fresh engine built the same way
  other.load_state(snap)
  third = _play(other, tail)
  for run in (second, third):
    for (r0, s0, d0), (r1, s1, d1) in zip(first[0], run[0]):
      np.testing.assert_array_equal(r0, r1); np.testing.assert_array_equal(s0, s1); np.testing.assert_array_equal(d0, d1)
    for k in (1, 2, 3):
      np.testing.assert_array_equal(first[k], run[k])


def test_snapshot_of_another_shape_is_refused(clean_up_blob):
  from meltingpot_b200 import engine
  a = engine.Engine(clean_up_blob, 4, device=0, seed=1)
  b = engine.Engine(clean_up_blob, 8, device=0, seed=1)
  a.reset(); b.reset()
  with pytest.raises(ValueError, match='does not fit'):
    b.load_state(a.save_state())
  with pytest.raises(ValueError, match='not a snapshot'):
    b.load_state(b'\0' * 64)


def test_load_rejects_truncated_and_foreign_snapshots(clean_up_blob, commons_blob):
  # mp_state_load takes the buffer length and the header names what the snapshot belongs to: env count, payload size,
  # RNG key (seed + env_index_base) and a hash of the compiled blob.
  from meltingpot_b200 import engine
  eng = engine.Engine(clean_up_blob, 8, seed=5)
  eng.reset()
  snap = eng.save_state()
  eng.load_state(snap)  # round trip is fine
  with pytest.raises(ValueError, match='truncated|shorter'):
    eng.load_state(snap[:len(snap) // 2])
  with pytest.raises(ValueError, match='shorter'):
    eng.load_state(snap[:8])
  other_seed = engine.Engine(clean_up_blob, 8, seed=6)
  with pytest.raises(ValueError, match='seed'):
    other_seed.load_state(snap)
  other_base = engine.Engine(clean_up_blob, 8, seed=5, env_index_base=8)
  with pytest.raises(ValueError, match='seed'):
    other_base.load_state(snap)
  other_blob = engine.Engine(commons_blob, 8, seed=5)
  with pytest.raises(ValueError):
    other_blob.load_state(snap)
  bigger = engine.Engine(clean_up_blob, 16, seed=5)
  with pytest.raises(ValueError, match='does not fit'):
    bigger.load_state(snap)


def test_tensor_views_outlive_close(clean_up_blob):
  # Engine.close() drops the engine's own references; the device memory is released (mp_destroy) only when the last
  # tensor view of its buffers is gone, so a retained observation can still be read and never dangles.
  import gc
  import torch
  from meltingpot_b200 import engine
  eng = engine.Engine(clean_up_blob, 4, seed=2)
  eng.reset()
  torch.cuda.synchronize()
  kept = eng.world_rgb            # a zero-copy view, as a BatchedTimeStep hands out
  want = kept.clone()
  eng.close()
  del eng
  gc.collect()
  filler = [torch.zeros(1 << 22, device='cuda') for _ in range(8)]  # would reuse the memory had it been freed
  torch.cuda.synchronize()
  assert torch.equal(kept, want)
  closed = engine.Engine(clean_up_blob, 4, seed=2)
  closed.close()
  with pytest.raises(ValueError, match='null handle'):   # a closed engine can no longer be stepped
    closed.step(torch.zeros((4, 7), dtype=torch.int32, device='cuda'))
  del filler
