"""Shared GPU-vs-oracle comparison loop (used by the -m gpu tests)."""

import numpy as np


def compare_rollout(blob, oracle, num_envs, steps, seed, check_envs=None, action_seed=0,
                    pixels_every=1, actions_fn=None, env_index_base=0):
  import torch
  from meltingpot_b200 import engine
  eng = engine.Engine(blob, num_envs, device=0, seed=seed, env_index_base=env_index_base)
  P, A = eng.num_players, eng.num_actions
  check_envs = list(range(num_envs)) if check_envs is None else list(check_envs)
  envs = {b: oracle.OracleEnv(blob, seed + env_index_base + b) for b in check_envs}
  rng = np.random.default_rng(action_seed)
  eng.reset()
  for e in envs.values():
    e.reset()
  stats = dict(rewards=0.0, lasts=0, zaps=0, cleaned=0, eaten=0, events=0)
  code_of = {v: k for k, v in oracle.EVENT_NAMES.items()}

  def check(t, acts):
    torch.cuda.synchronize()
    rew = eng.reward.cpu().numpy(); disc = eng.discount.cpu().numpy(); st = eng.step_type.cpu().numpy()
    sc = eng.scalar_obs.cpu().numpy(); av = eng.avatar_state.cpu().numpy()
    grid = eng.grid.cpu().numpy().view(np.uint16)
    nev = eng.event_count.cpu().numpy(); evs = eng.events.cpu().numpy()
    do_px = (t % pixels_every) == 0
    if do_px:
      idx = torch.as_tensor(check_envs, device='cuda')
      rgb = eng.rgb[idx].cpu().numpy(); world = eng.world_rgb[idx].cpu().numpy()
    for i, b in enumerate(check_envs):
      e = envs[b]
      where = f'step {t} env {b}'
      assert e.step_type() == st[b], f'step_type {where}: {e.step_type()} vs {st[b]}'
      assert e.discount() == disc[b], f'discount {where}'
      np.testing.assert_array_equal(e.rewards(), rew[b], err_msg=f'reward {where}')
      np.testing.assert_array_equal(e.scalar_obs().T, sc[:e.n_scalar, b, :], err_msg=f'scalar obs {where}')
      np.testing.assert_array_equal(e.avatars(), av[b], err_msg=f'avatars {where}')
      og = e.grid()
      gg = grid[b][:, :og.shape[1]]
      if not np.array_equal(og, gg):
        bad = np.argwhere(og != gg)
        raise AssertionError(f'grid {where}: first diffs (layer, cell) {bad[:8].tolist()} '
                             f'oracle {og[tuple(bad[0])]} gpu {gg[tuple(bad[0])]}')
      if do_px:
        np.testing.assert_array_equal(e.rgb(), rgb[i], err_msg=f'RGB {where}')
        np.testing.assert_array_equal(e.world_rgb(), world[i], err_msg=f'WORLD.RGB {where}')
      stats['rewards'] += float(rew[b].sum())
      stats['lasts'] += int(st[b] == 2)
      want = sorted((code_of[name], a, b2) for name, a, b2 in e.events())
      assert nev[b] == len(want), f'event count {where}: oracle {len(want)} gpu {nev[b]}'
      assert nev[b] <= evs.shape[1], f'events {where}: {nev[b]} events exceed max_events {evs.shape[1]} (the bound of mp_create is wrong)'
      got = sorted(tuple(int(v) for v in row) for row in evs[b][:int(nev[b])])
      assert got == want, f'events {where}: oracle {want} gpu {got}'
      stats['events'] += len(want)
      for name, _, _ in e.events():
        key = {'zap': 'zaps', 'player_cleaned': 'cleaned', 'edible_consumed': 'eaten'}.get(name)
        if key:
          stats[key] += 1

  check(-1, None)
  for t in range(steps):
    if actions_fn is not None:
      acts = actions_fn(t, num_envs, P, A, rng)
    else:
      acts = rng.integers(0, A, size=(num_envs, P))
    acts = np.ascontiguousarray(acts, np.int32)
    eng.step(torch.from_numpy(acts).cuda())
    for b, e in envs.items():
      e.step(acts[b])
    check(t, acts)
  eng.close()
  return stats


def _event_keys(events, counts):
  """Sorted int64 keys of each env's event rows ([B, M, 3] -> [B, M], unused rows = int64 max)."""
  ev = events.astype(np.int64)
  key = (ev[..., 0] << 44) | ((ev[..., 1] & 0x3fffff) << 22) | (ev[..., 2] & 0x3fffff)
  mask = np.arange(ev.shape[1])[None, :] >= counts[:, None]
  key[mask] = np.iinfo(np.int64).max
  key.sort(axis=1)
  return key


def shapes_of(eng):
  """The output shapes OracleBatch.dump / env_dump lay their arrays out with, for this engine."""
  bf = eng.buffers
  return dict(P=eng.num_players, L=int(bf.grid_layers), cells=int(bf.grid_cells), n_scalar=eng.num_scalar_obs,
              rgb=(int(bf.rgb_h), int(bf.rgb_w)), world=(int(bf.world_h), int(bf.world_w)))


def device_outputs(eng, kinds=('rgb', 'world')):
  """Every output in the engine's own buffers (mp_buffers) as host arrays keyed like OracleBatch.dump; of the images,
  those named in `kinds`. Synchronises the device first."""
  import torch
  torch.cuda.synchronize()
  got = dict(step_type=eng.step_type.cpu().numpy(), discount=eng.discount.cpu().numpy(), reward=eng.reward.cpu().numpy(),
             scalar_obs=eng.scalar_obs.cpu().numpy()[:eng.num_scalar_obs], avatars=eng.avatar_state.cpu().numpy(),
             grid=eng.grid.cpu().numpy().view(np.uint16)[:, :, :int(eng.buffers.grid_cells)],
             n_events=eng.event_count.cpu().numpy(), events=eng.events.cpu().numpy())
  if 'rgb' in kinds:
    got['rgb'] = eng.rgb.cpu().numpy()
  if 'world' in kinds:
    got['world'] = eng.world_rgb.cpu().numpy()
  return got


_HOST_KEYS = dict(rgb='rgb', world_rgb='world', reward='reward', discount='discount', step_type='step_type',
                  scalar_obs='scalar_obs', events='events', event_count='n_events')


def host_outputs(out, n_scalar):
  """The arrays of a host output set (Engine.make_host_outputs names) keyed like OracleBatch.dump."""
  got = {_HOST_KEYS[k]: v.numpy() for k, v in out.items() if k in _HOST_KEYS and v is not None}
  if 'scalar_obs' in got:
    got['scalar_obs'] = got['scalar_obs'][:n_scalar]
  return got


def env_dump(envs, shapes, pixels=False, max_events=256, kinds=('rgb', 'world')):
  """OracleBatch.dump for a list of OracleEnv (env b of the batch = envs[b]), for runs an OracleBatch cannot follow."""
  from oracle import binding
  code_of = {v: k for k, v in binding.EVENT_NAMES.items()}
  B, P = len(envs), shapes['P']
  out = {'reward': np.stack([e.rewards() for e in envs]), 'discount': np.array([e.discount() for e in envs]),
         'step_type': np.array([e.step_type() for e in envs], np.int64),
         'scalar_obs': np.zeros((max(shapes['n_scalar'], 1), B, P), np.float64),
         'avatars': np.stack([e.avatars() for e in envs]), 'grid': np.stack([e.grid() for e in envs]),
         'events': np.zeros((B, max_events, 3), np.int32), 'n_events': np.zeros((B,), np.int32)}
  for b, e in enumerate(envs):
    out['scalar_obs'][:shapes['n_scalar'], b] = e.scalar_obs().T
    rows = [(code_of[name], x, y) for name, x, y in e.events()]
    out['n_events'][b] = len(rows)
    out['events'][b, :len(rows)] = np.array(rows, np.int32).reshape(-1, 3)
  if pixels and 'rgb' in kinds:
    out['rgb'] = np.stack([e.rgb() for e in envs])
  if pixels and 'world' in kinds:
    out['world'] = np.stack([e.world_rgb() for e in envs])
  return out


def check_outputs(got, want, where):
  """Each array of `got` (device_outputs / host_outputs) must equal the same entry of `want` (OracleBatch.dump /
  env_dump) bit for bit; event rows are compared as sorted keys, since the rows of one step are in no particular order."""

  def same(name, g, exp):
    assert g.shape == exp.shape, f'{name} {where}: shape {g.shape}, oracle {exp.shape}'
    if not np.array_equal(g, exp):
      bad = np.argwhere(g != exp)
      raise AssertionError(f'{name} {where}: {len(bad)} mismatches, first at {bad[0].tolist()} (env first): gpu {g[tuple(bad[0])]} oracle {exp[tuple(bad[0])]}')

  for key, name in (('step_type', 'step_type'), ('discount', 'discount'), ('reward', 'reward'), ('avatars', 'avatars'),
                    ('grid', 'grid')):
    if key in got:
      same(name, got[key], want[key])
  if 'scalar_obs' in got:
    same('scalar_obs', got['scalar_obs'], want['scalar_obs'][:len(got['scalar_obs'])])
  if 'n_events' in got:
    nev = got['n_events']
    same('event count', nev, want['n_events'])
    if 'events' in got:
      max_ev = got['events'].shape[1]
      assert int(nev.max(initial=0)) <= max_ev, f'{where}: {int(nev.max())} events exceed max_events {max_ev}'
      same('events', _event_keys(got['events'], nev), _event_keys(want['events'], want['n_events']))
  for key, name in (('rgb', 'RGB'), ('world', 'WORLD.RGB')):
    if key in got:
      same(name, got[key], want[key])


def compare_batch(blob, oracle, num_envs, steps, seed, action_seed=0, pixels_every=10, actions_fn=None,
                  env_index_base=0, threads=None, flags=None, render_layout=None, pixels_at=None, on_step=None):
  """EVERY env of the batch against the oracle: rewards, discount, step type, scalar observations, avatar state, the
  whole sprite grid and the events on every step, every RGB byte of every env every `pixels_every` steps (or on the
  steps t where `pixels_at(t)` holds; t = 0 is the reset). `flags` / `render_layout` go to the Engine; only the images
  the flags produce are compared, and an image buffer the flags leave out is filled with a sentinel before the reset
  and must still hold it on every pixel check. `on_step(t, eng)` runs after each check."""
  import os
  import torch
  from meltingpot_b200 import engine
  threads = threads or os.cpu_count() or 1
  flags = engine.MP_FLAG_DEFAULT if flags is None else flags
  eng = engine.Engine(blob, num_envs, device=0, seed=seed, env_index_base=env_index_base, flags=flags,
                      render_layout=render_layout)
  P, A = eng.num_players, eng.num_actions
  shapes = shapes_of(eng)
  max_ev = int(eng.buffers.max_events)
  kinds = [k for k, bit in (('rgb', engine.MP_FLAG_RENDER_PLAYERS), ('world', engine.MP_FLAG_RENDER_WORLD)) if flags & bit]
  absent = [t for k, t in (('rgb', eng.rgb), ('world', eng.world_rgb)) if k not in kinds]
  for t in absent:
    t.fill_(_SENTINEL)
  batch = oracle.OracleBatch(blob, num_envs, seed=seed + env_index_base)  # oracle_batch_create starts episode 0
  rng = np.random.default_rng(action_seed)
  eng.reset()
  stats = dict(rewards=0.0, lasts=0, events=0, pixel_checks=0, envs=num_envs, last_steps=[], mids_after_restart=0)
  restarted = np.zeros(num_envs, bool)

  def check(t):
    px = pixels_at(t) if pixels_at is not None else (t % pixels_every) == 0
    got = device_outputs(eng, kinds if px else ())
    want = batch.dump(threads, shapes, pixels=px, max_events=max_ev, kinds=kinds)
    check_outputs(got, want, f'step {t}')
    st = got['step_type']
    if px:
      for img in absent:
        assert bool((img == _SENTINEL).all()), f'step {t}: an image the flags leave out was written'
      stats['pixel_checks'] += 1
    stats['rewards'] += float(want['reward'].sum())
    stats['lasts'] += int((st == 2).sum())
    if (st == 2).any():
      stats['last_steps'].append(t)
    stats['mids_after_restart'] += int(((st == 1) & restarted).sum())
    if t > 0:
      restarted[st == 0] = True
    stats['events'] += int(want['n_events'].sum())
    if on_step is not None:
      on_step(t, eng)

  check(0)
  for t in range(1, steps + 1):
    acts = actions_fn(t, num_envs, P, A, rng) if actions_fn is not None else rng.integers(0, A, size=(num_envs, P))
    acts = np.ascontiguousarray(acts, np.int32)
    eng.step(torch.from_numpy(acts).cuda())
    batch.step_actions(acts, threads)
    check(t)
  eng.close()
  batch.close()
  return stats


_SENTINEL = 0xA5
# the engine's per-env state and timestep buffers (everything a later step depends on or a caller reads)
# (event rows are compared as sorted keys: the rows of one step are in no particular order)
_STATE_VIEWS = ('reward', 'discount', 'step_type', 'scalar_obs', 'avatar_state', 'grid', 'event_count', 'timestep_packed')


def lockstep(blob, num_envs, steps, seed, variants, action_seed=0, actions_fn=None, env_index_base=0):
  """Steps an engine with the default options and one engine per entry of `variants` (Engine keyword arguments such as
  `flags` / `render_layout`), all built from the same blob, seed and B, with the same actions. After the reset and
  after every step each variant's images (those its flags produce) and state buffers must equal the default engine's,
  compared on the device. The default engine follows the same action stream as compare_batch with the same
  `action_seed` / `actions_fn`, so a compare_batch run anchors the chain to the oracle. Returns each variant's
  render_plan()."""
  import torch
  from meltingpot_b200 import engine
  ref = engine.Engine(blob, num_envs, device=0, seed=seed, env_index_base=env_index_base)
  twins = [engine.Engine(blob, num_envs, device=0, seed=seed, env_index_base=env_index_base, **v) for v in variants]
  P, A = ref.num_players, ref.num_actions
  rng = np.random.default_rng(action_seed)

  def check(t):
    ref_events = _event_keys(ref.events.cpu().numpy(), ref.event_count.cpu().numpy())
    for v, tw in zip(variants, twins):
      f = v.get('flags', engine.MP_FLAG_DEFAULT)
      names = list(_STATE_VIEWS) + (['rgb'] if f & engine.MP_FLAG_RENDER_PLAYERS else []) + (['world_rgb'] if f & engine.MP_FLAG_RENDER_WORLD else [])
      for name in names:
        if not torch.equal(getattr(tw, name), getattr(ref, name)):
          raise AssertionError(f'{name} differs from the default engine at step {t} (B={num_envs}, {v}, plan {tw.render_plan()})')
      if not np.array_equal(_event_keys(tw.events.cpu().numpy(), tw.event_count.cpu().numpy()), ref_events):
        raise AssertionError(f'events differ from the default engine at step {t} (B={num_envs}, {v})')

  ref.reset()
  for tw in twins:
    tw.reset()
  check(0)
  for t in range(1, steps + 1):
    acts = actions_fn(t, num_envs, P, A, rng) if actions_fn is not None else rng.integers(0, A, size=(num_envs, P))
    acts = torch.from_numpy(np.ascontiguousarray(acts, np.int32)).cuda()
    ref.step(acts)
    for tw in twins:
      tw.step(acts)
    check(t)
  plans = [tw.render_plan() for tw in twins]
  for e in [ref] + twins:
    e.close()
  return plans
