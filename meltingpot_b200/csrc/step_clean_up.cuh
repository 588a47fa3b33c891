// step_clean_up.cuh -- state transition of the clean_up family, one warp per env instance.
//
// Restates, in closed form over SoA state, one frame of
//   api:advance            meltingpot/lua/modules/api_factory.lua:104-111
//   BaseSimulation:update  meltingpot/lua/modules/base_simulation.lua:476-486
//   grid:update            (engine; DESIGN.md "Engine policy ledger")
// for the components of meltingpot/lua/levels/clean_up/components.lua and the
// Avatar / Zapper components of meltingpot/lua/modules/avatar_library.lua.
// Lanes are avatars (arbitration, timers), beam cells (ray scan) or entities (apples, dirt,
// water) depending on the phase; envs never interact, so nothing leaves the warp.
#pragma once

#include "common.cuh"

__host__ __device__ inline size_t scratch_round16(size_t n) { return (n + 15) & ~(size_t)15; }

struct WarpScratch {  // per-warp shared memory, carved from the dynamic allocation
  uint8_t* occ;       // [cells_pad] 0 free, 1..P avatar p-1, 255 static piece on the avatar layer
  uint8_t* apple;     // [nA_pad] bit0 live this frame, bit1 eaten this frame
  uint8_t* dirt;      // [nD_pad] bit0 dirty this frame, bit1 cleaned this frame
  uint32_t* beam_zap; // [cells/32+1] cells that already carry a zap sprite
  uint32_t* beam_2;   // same for the second beam
  int16_t* tmp;       // [64]
  // per-CTA copies of static lookup tables (clean_up family): they sit on the serial avatar-by-avatar chain, where a
  // shared-memory read costs ~30 cycles and an L2 round trip ~600
  const int16_t* apple_of;  // [cells_pad] apple index or -1
  const int16_t* dirt_of;   // [cells_pad] dirt index or -1
  const uint8_t* flags;     // [cells_pad] BeamBlocker bits
  const uint8_t* solid;     // [cells_pad] 255 where the avatar layer is statically occupied
  const int32_t* act_table; // [n_actions][4]
};

__host__ __device__ inline size_t clean_up_table_bytes(const Tables& T) { return scratch_round16((size_t)T.cells_pad * 6) + scratch_round16((size_t)T.n_actions * 16); }

// Every region starts 16-byte aligned (the per-entity state is moved with 128-bit accesses).
__host__ __device__ inline size_t warp_scratch_bytes(const Tables& T) {
  size_t words = (size_t)(T.cells + 31) / 32 + 1;
  return scratch_round16(T.cells_pad) + scratch_round16(T.nA_pad) + scratch_round16(T.nD_pad) + 2 * scratch_round16(words * 4) + 64 * 2;
}

__device__ __forceinline__ WarpScratch carve_scratch(const Tables& T, uint8_t* base) {
  WarpScratch s;
  size_t words = (size_t)(T.cells + 31) / 32 + 1;
  s.occ = base; base += scratch_round16(T.cells_pad);
  s.apple = base; base += scratch_round16(T.nA_pad);
  s.dirt = base; base += scratch_round16(T.nD_pad);
  s.beam_zap = (uint32_t*)base; base += scratch_round16(words * 4);
  s.beam_2 = (uint32_t*)base; base += scratch_round16(words * 4);
  s.tmp = (int16_t*)base;
  return s;
}

// ---------------------------------------------------------------------------------------------
// Episode start: api:start (api_factory.lua:85-102) + BaseSimulation:start/_avatarStart
// (base_simulation.lua:396-471) + the frame-0 grid:update.
// ---------------------------------------------------------------------------------------------
__device__ void clean_up_reset(const Tables& T, const State& S, int b, int lane, WarpScratch& sc) {
  int32_t* env = S.env + (size_t)b * ENV_COLS;
  const int episode = env[ENV_EPISODE] + 1;
  const uint64_t key = S.seed + (uint64_t)b;
  const uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
  uint16_t* grid = S.grid + (size_t)b * T.L * T.cells_pad;
  __syncwarp();
  {  // static pieces + initial states
    const uint4* src = reinterpret_cast<const uint4*>(T.init_grid);
    uint4* dst = reinterpret_cast<uint4*>(grid);
    const int n16 = T.L * T.cells_pad / 8;
    for (int i = lane; i < n16; i += 32) dst[i] = src[i];
  }
  for (int k = lane; k < T.nA; k += 32) S.apple[(size_t)b * T.nA_pad + k] = (uint8_t)T.apple[k * 3 + 2];
  for (int j = lane; j < T.nD; j += 32) S.dirt[(size_t)b * T.nD_pad + j] = (uint8_t)T.dirt[j * 3 + 2];
  __syncwarp();
  // Animation:postStart random start frame (component_library.lua:1064-1068).
  for (int k = lane; k < T.nW; k += 32) {
    int phase = 0;
    if (T.anim_random) {
      uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)T.water[k * 2], RS_OBJECT_RESET, k0, k1);
      phase = (int)pick(w.x, (uint32_t)T.n_anim);
    }
    S.water[(size_t)b * T.nW_pad + k] = (uint8_t)phase;
    grid[(size_t)T.water_layer * T.cells_pad + T.water[k * 2 + 1]] = cell_value(T.water_sprite[phase], 0);
  }
  // _avatarStart: groupShuffledWithCount(random, spawnGroup, P) as a partial Fisher-Yates.
  for (int i = lane; i < T.n_spawn && i < 64; i += 32) sc.tmp[i] = (int16_t)T.spawn_cell[i];
  __syncwarp();
  if (lane == 0) {
    for (int p = 0; p < T.P; ++p) {
      uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)p, RS_AVATAR_RESET, k0, k1);
      int r = p + (int)pick(w.x, (uint32_t)(T.n_spawn - p));
      int16_t t = sc.tmp[p]; sc.tmp[p] = sc.tmp[r]; sc.tmp[r] = t;
    }
  }
  __syncwarp();
  if (lane < T.P) {
    uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)lane, RS_AVATAR_RESET, k0, k1);
    int cell = sc.tmp[lane], orient = (int)(w.y & 3u);  // Avatar:start, avatar_library.lua:299-304
    int32_t* av = S.avatar + ((size_t)b * T.P + lane) * 4;
    av[AV_X] = cell % T.W; av[AV_Y] = cell / T.W; av[AV_ORIENT] = orient; av[AV_ALIVE] = 1;
    int32_t* tm = S.av_timer + ((size_t)b * T.P + lane) * 4;
    tm[TM_ZAP] = 0; tm[TM_BEAM2] = 0; tm[TM_FRAME] = 0; tm[3] = 0;
    grid[(size_t)T.avatar_layer * T.cells_pad + cell] = cell_value(T.avatar_sprite[lane], orient);
    S.reward[(size_t)b * T.P + lane] = 0.0;
    S.packed[(size_t)b * (T.P + 2) + lane] = 0.0;
    for (int k = 0; k < T.n_scalar; ++k)
      S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = T.scalar_obs[k] == 0 ? 1.0 : 0.0;
  }
  if (lane == 0) {
    env[ENV_STEP] = 0; env[ENV_EPISODE] = episode; env[ENV_DONE] = 0; env[ENV_DIRT] = T.dirt_count0;
    env[ENV_CLEANED] = 0; env[ENV_ATE] = 0; env[ENV_BEAM] = 0;
    S.discount[b] = 0.0;   // multiplayer_wrapper.py:117 (None -> 0.)
    S.step_type[b] = 0;    // dm_env.StepType.FIRST
    S.packed[(size_t)b * (T.P + 2) + T.P] = 0.0; S.packed[(size_t)b * (T.P + 2) + T.P + 1] = 0.0;
  }
  __syncwarp();
}

// One beam: lanes are footprint cells. A cell is visited iff its parent was visited and did not
// block; resolved by `depth` rounds of warp shuffles along the parent links.
__device__ __forceinline__ void beam_scan(const BeamGeom& G, int lane, bool self_blocked, bool& vis) {
  bool ok = lane < G.n;
  int parent = ok ? G.parent[lane] : -1;
  vis = ok;
  bool open = ok && !self_blocked;  // this cell lets the ray continue
  for (int d = 0; d < G.depth; ++d) {
    int src = parent < 0 ? lane : parent;
    bool pv = __shfl_sync(MP_FULL, vis, src);
    bool po = __shfl_sync(MP_FULL, open, src);
    if (ok && parent >= 0) { vis = pv && po; }
    open = vis && !self_blocked;
  }
}

__device__ void clean_up_step(const Tables& T, const State& S, int b, int lane, const int32_t* __restrict__ actions, WarpScratch& sc) {
  int32_t* env = S.env + (size_t)b * ENV_COLS;
  const int n = env[ENV_STEP] + 1;  // frame number of this advance
  const int episode = env[ENV_EPISODE];
  const uint64_t key = S.seed + (uint64_t)b;
  const uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
  uint16_t* grid = S.grid + (size_t)b * T.L * T.cells_pad;
  int dirt_count = env[ENV_DIRT];
  const unsigned cleaned_prev = (unsigned)env[ENV_CLEANED];
  unsigned cleaned_now = 0, ate_now = 0;
  const bool is_av = lane < T.P;

  // ---- load ---------------------------------------------------------------------------------
  int x = 0, y = 0, orient = 0, alive = 0, zap_cool = 0, clean_cool = 0, state_frame = 0;
  int act_move = 0, act_turn = 0, act_zap = 0, act_clean = 0;
  if (is_av) {
    const int4 a = *reinterpret_cast<const int4*>(S.avatar + ((size_t)b * T.P + lane) * 4);
    const int4 t = *reinterpret_cast<const int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4);
    x = a.x; y = a.y; orient = a.z; alive = a.w; zap_cool = t.x; clean_cool = t.y; state_frame = t.z;
    int id = actions[(size_t)b * T.P + lane];
    if (id < 0 || id >= T.n_actions) id = 0;
    const int4 at = *reinterpret_cast<const int4*>(sc.act_table + id * 4);  // discrete_action_wrapper.py:97-100
    act_move = at.x; act_turn = at.y; act_zap = at.z; act_clean = at.w;
  }
  const int x0 = x, y0 = y, orient0 = orient, alive0 = alive;
  double reward = 0.0;  // Avatar:preUpdate (avatar_library.lua:330-332)

  for (int i = lane; i < T.cells_pad / 8; i += 32)
    reinterpret_cast<uint2*>(sc.occ)[i] = reinterpret_cast<const uint2*>(sc.solid)[i];
  // per-entity state, 16 entities per lane and access; bit 3 keeps the state the frame started with (round 2 compares
  // against it instead of re-reading global memory)
  for (int i = lane; i < T.nA_pad / 16; i += 32) {
    uint4 v = reinterpret_cast<const uint4*>(S.apple + (size_t)b * T.nA_pad)[i];
    v.x |= (v.x & 0x01010101u) << 3; v.y |= (v.y & 0x01010101u) << 3; v.z |= (v.z & 0x01010101u) << 3; v.w |= (v.w & 0x01010101u) << 3;
    reinterpret_cast<uint4*>(sc.apple)[i] = v;
  }
  for (int i = lane; i < T.nD_pad / 16; i += 32) {
    uint4 v = reinterpret_cast<const uint4*>(S.dirt + (size_t)b * T.nD_pad)[i];
    v.x |= (v.x & 0x01010101u) << 3; v.y |= (v.y & 0x01010101u) << 3; v.z |= (v.z & 0x01010101u) << 3; v.w |= (v.w & 0x01010101u) << 3;
    reinterpret_cast<uint4*>(sc.dirt)[i] = v;
  }
  const int words = (T.cells + 31) / 32 + 1;
  for (int i = lane; i < words; i += 32) { sc.beam_zap[i] = 0; sc.beam_2[i] = 0; }
  __syncwarp();
  if (is_av && alive) sc.occ[y * T.W + x] = (uint8_t)(lane + 1);
  // Hit sprites live for one frame (policy A.8): clear both beam layers if the last frame drew any.
  if (env[ENV_BEAM]) {
    uint4 z = make_uint4(0, 0, 0, 0);
    uint4* lz = reinterpret_cast<uint4*>(grid + (size_t)T.zap_layer * T.cells_pad);
    uint4* lc = reinterpret_cast<uint4*>(grid + (size_t)T.clean_layer * T.cells_pad);
    for (int i = lane; i < T.cells_pad / 8; i += 32) { lz[i] = z; lc[i] = z; }
  }
  __syncwarp();
  int beam_dirty = 0;

  // ---- simulation:update --------------------------------------------------------------------
  // DirtSpawner:update (clean_up/components.lua:329-340); its _timeStep equals n here.
  int spawn_dirt = -1;
  if (n > T.dirt_delay) {
    uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, SCENE_DRAW_DIRT, RS_SCENE, k0, k1);
    int n_inactive = T.nD - dirt_count;
    if (u01(w.x, w.y) < T.dirt_prob && n_inactive > 0) {
      int kth = (int)pick(w.z, (uint32_t)n_inactive);  // k-th inactive dirt in piece order
      for (int base = 0; base < T.nD; base += 32) {
        int j = base + lane;
        bool inactive = j < T.nD && !(sc.dirt[j] & 1);
        unsigned m = __ballot_sync(MP_FULL, inactive);
        int c = __popc(m);
        if (kth < c) {
          // position of the kth set bit
          unsigned mm = m;
          for (int q = 0; q < kth; ++q) mm &= mm - 1;
          spawn_dirt = base + __ffs(mm) - 1;
          break;
        }
        kth -= c;
      }
    }
  }
  // AppleGrow:update (clean_up/components.lua:64-80): one uniform per potential apple per frame.
  {
    const double dirt = (double)dirt_count, clean = (double)(T.nD - dirt_count);
    const double fraction = dirt / (dirt + clean);
    double interpolation = (fraction - T.grow_depletion) / (T.grow_restoration - T.grow_depletion);
    interpolation = 1.0 < interpolation ? 1.0 : interpolation;  // Lua 5.1 math.min: a NaN (0/0) stays NaN, no growth (policy A.22)
    const double probability = T.grow_rate * interpolation;
    if (probability > 0.0) {  // u >= 0 can never be below a non-positive (or NaN) probability
      for (int k = lane; k < T.nA; k += 32) {
        uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)T.apple[k * 3], RS_OBJECT, k0, k1);
        if (u01(w.x, w.y) < probability && !(sc.apple[k] & 1)) sc.apple[k] |= 4;  // grows this frame
      }
    }
  }
  __syncwarp();

  // ---- updaters (priority order) ------------------------------------------------------------
  // Avatars are visited in a fresh random order each frame (policy A.7).
  int rank = 0;
  {
    uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)lane, RS_AVATAR, k0, k1);
    uint32_t mykey = w.x;
    for (int q = 0; q < T.P; ++q) {
      uint32_t kq = __shfl_sync(MP_FULL, mykey, q);
      if (is_av && (kq < mykey || (kq == mykey && q < lane))) ++rank;
    }
    if (!is_av) rank = 99;
  }
  // 150 Avatar move (avatar_library.lua:156-171): intents are act_turn / act_move.
  // 140 Zapper zap (:613-631) and Cleaner clean (clean_up/components.lua:201-219).
  bool fire_zap = false, fire_clean = false;
  if (is_av && alive) {
    if (zap_cool > 0) --zap_cool; else if (act_zap == 1) { zap_cool = T.zap_cooldown; fire_zap = true; }
    if (clean_cool > 0) --clean_cool; else if (act_clean == 1) { clean_cool = T.clean_cooldown; fire_clean = true; }
  }
  // 135 Zapper respawn (:638-649): state = waitState, startFrame = framesTillRespawn.
  const bool want_respawn = is_av && !alive && (n - state_frame) >= T.zap_respawn;
  // 100 StochasticIntervalEpisodeEnding (component_library.lua:927-948); its _t equals n + 1.
  bool cont = true;
  if (n >= T.end_min_frames && ((n + 1) % T.end_interval) == 0) {
    uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, SCENE_DRAW_EPISODE_END, RS_SCENE, k0, k1);
    if (u01(w.x, w.y) < T.end_prob) cont = false;
  }
  // 4 AllNonselfCumulants:getCumulants (clean_up/components.lua:535-545); 2 GlobalData reset.
  const int num_others_cleaned = is_av ? __popc(cleaned_prev & ~(1u << lane)) : 0;

  // ---- queue drain, round 1 -----------------------------------------------------------------
  // (a) setState('dirt') from the spawner.
  if (spawn_dirt >= 0) { if (lane == 0) sc.dirt[spawn_dirt] |= 1; ++dirt_count; }
  __syncwarp();
  // (b) setState('apple'); an avatar standing there triggers Edible:onEnter immediately.
  for (int base = 0; base < T.nA; base += 32) {
    int k = base + lane;
    bool grows = k < T.nA && (sc.apple[k] & 4);
    int eater = -1;
    if (grows) {
      sc.apple[k] = (sc.apple[k] & ~4) | 1;
      int o = sc.occ[T.apple[k * 3 + 1]];
      if (o >= 1 && o <= T.P) { eater = o - 1; sc.apple[k] |= 2; }
    }
    unsigned m = __ballot_sync(MP_FULL, eater >= 0);
    while (m) {  // in apple (object) order
      int src = __ffs(m) - 1; m &= m - 1;
      int e = __shfl_sync(MP_FULL, eater, src);
      if (lane == e) { reward += T.eat_reward; emit_event(S, b, EV_EDIBLE_CONSUMED, e + 1, 0); }
      ate_now |= 1u << e;
    }
  }
  __syncwarp();
  // (c) turns and moves, avatar by avatar in this frame's order.
  for (int r = 0; r < T.P; ++r) {
    unsigned m = __ballot_sync(MP_FULL, is_av && rank == r);
    int src = __ffs(m) - 1;
    // one shuffle instead of six: alive | turn + 1 | move | orient | y | x
    const uint32_t packed = __shfl_sync(MP_FULL, (uint32_t)(alive & 1) | ((uint32_t)(act_turn + 1) << 1) | ((uint32_t)act_move << 3) |
                                                     ((uint32_t)orient << 6) | ((uint32_t)y << 8) | ((uint32_t)x << 20), src);
    if (!(packed & 1u)) continue;
    const int s_turn = (int)((packed >> 1) & 3u) - 1, s_move = (int)((packed >> 3) & 7u);
    int so = (int)((packed >> 6) & 3u), sy = (int)((packed >> 8) & 0xfffu), sx = (int)(packed >> 20);
    if (s_turn != 0) so = (so + s_turn) & 3;
    bool ate = false;
    if (s_move != 0) {
      int d = (so + s_move - 1) & 3;
      int nx = sx + dir_dx(d), ny = sy + dir_dy(d);
      bool inb = wrap_or_reject(T, nx, ny);
      if (inb && sc.occ[ny * T.W + nx] == 0) {
        __syncwarp();
        if (lane == 0) { sc.occ[sy * T.W + sx] = 0; sc.occ[ny * T.W + nx] = (uint8_t)(src + 1); }
        sx = nx; sy = ny;
      }
      // place -> contact enter on the final cell, even when blocked (policy A.5)
      int fcell = sy * T.W + sx;
      int ai = sc.apple_of[fcell];
      ate = ai >= 0 && (sc.apple[ai] & 1);
      __syncwarp();
      if (ate && lane == 0) sc.apple[ai] |= 2;
    }
    if (lane == src) { x = sx; y = sy; orient = so; if (ate) { reward += T.eat_reward; emit_event(S, b, EV_EDIBLE_CONSUMED, src + 1, 0); } }
    if (ate) ate_now |= 1u << src;
    __syncwarp();
  }
  // (d) zap beams, then (e) clean beams, shooter by shooter.
  unsigned zapped = 0;
  for (int pass = 0; pass < 2; ++pass) {
    const BeamGeom& G = pass == 0 ? T.zap_geom : T.clean_geom;
    for (int r = 0; r < T.P; ++r) {
      unsigned m = __ballot_sync(MP_FULL, is_av && rank == r && (pass == 0 ? fire_zap : fire_clean));
      if (!m) continue;
      int src = __ffs(m) - 1;
      int sx = __shfl_sync(MP_FULL, x, src), sy = __shfl_sync(MP_FULL, y, src), so = __shfl_sync(MP_FULL, orient, src);
      // geometry of my footprint cell
      int cell = -1; bool blocked = false; int hit_avatar = -1, hit_dirt = -1;
      if (lane < G.n) {
        int f = so, rgt = (so + 1) & 3;
        int cx = sx + dir_dx(f) * G.fwd[lane] + dir_dx(rgt) * G.lat[lane];
        int cy = sy + dir_dy(f) * G.fwd[lane] + dir_dy(rgt) * G.lat[lane];
        if (!wrap_or_reject(T, cx, cy)) { blocked = true; }
        else {
          cell = cy * T.W + cx;
          int hit = pass == 0 ? T.zap_hit : T.clean_hit;
          if (sc.flags[cell] & (1 << hit)) blocked = true;  // BeamBlocker:onHit
          if (pass == 0) {
            int o = sc.occ[cell];
            if (o >= 1 && o <= T.P && o - 1 != src) { hit_avatar = o - 1; blocked = true; }  // Zapper:onHit
          } else {
            int dj = sc.dirt_of[cell];
            if (dj >= 0 && (sc.dirt[dj] & 1)) { hit_dirt = dj; blocked = true; }  // DirtCleaning:onHit
          }
        }
      }
      bool vis;
      beam_scan(G, lane, blocked, vis);
      // effects, in footprint order
      if (pass == 0) {
        unsigned hm = __ballot_sync(MP_FULL, vis && hit_avatar >= 0);
        while (hm) {
          int c = __ffs(hm) - 1; hm &= hm - 1;
          int t = __shfl_sync(MP_FULL, hit_avatar, c);
          if (lane == t) reward += T.zap_penalty;   // zapped avatar is still alive in this round
          if (lane == src) { reward += T.zap_reward; emit_event(S, b, EV_ZAP, src + 1, t + 1); }
          if (T.zap_remove) zapped |= 1u << t;
        }
      } else {
        bool cleaned = vis && hit_dirt >= 0;
        if (cleaned) { sc.dirt[hit_dirt] |= 2; emit_event(S, b, EV_PLAYER_CLEANED, src + 1, 0); }
        if (__any_sync(MP_FULL, cleaned)) cleaned_now |= 1u << src;  // Cleaner:setCumulant
      }
      if (vis && !blocked && cell >= 0) {
        uint32_t* bm = pass == 0 ? sc.beam_zap : sc.beam_2;
        uint32_t bit = 1u << (cell & 31);
        uint32_t old = atomicOr(&bm[cell >> 5], bit);
        if (!(old & bit)) {
          int layer = pass == 0 ? T.zap_layer : T.clean_layer, sprite = pass == 0 ? T.zap_sprite : T.clean_sprite;
          grid[(size_t)layer * T.cells_pad + cell] = cell_value(sprite, so);
        }
        beam_dirty = 1;
      }
      __syncwarp();
    }
  }
  beam_dirty = __any_sync(MP_FULL, beam_dirty);
  // (f) teleportToGroup for respawning avatars (policy A.9).
  for (int r = 0; r < T.P; ++r) {
    unsigned m = __ballot_sync(MP_FULL, is_av && rank == r && want_respawn);
    if (!m) continue;
    int src = __ffs(m) - 1;
    uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)src, RS_AVATAR, k0, k1);
    int target = T.spawn_cell[pick(w.y, (uint32_t)T.n_spawn)];
    if (sc.occ[target] != 0) continue;  // blocked: the updater fires again next frame
    __syncwarp();
    if (lane == 0) sc.occ[target] = (uint8_t)(src + 1);
    int ai = sc.apple_of[target];
    bool ate = ai >= 0 && (sc.apple[ai] & 1);
    __syncwarp();
    if (ate && lane == 0) sc.apple[ai] |= 2;
    if (lane == src) {
      x = target % T.W; y = target / T.W; orient = (int)(w.z & 3u); alive = 1; state_frame = n;
      if (ate) { reward += T.eat_reward; emit_event(S, b, EV_EDIBLE_CONSUMED, src + 1, 0); }
    }
    if (ate) ate_now |= 1u << src;
    __syncwarp();
  }

  // ---- round 2: the setStates queued by callbacks --------------------------------------------
  if (is_av && (zapped >> lane & 1u)) { alive = 0; state_frame = n; }
  for (int k = lane; k < T.nA; k += 32) {
    uint8_t v = sc.apple[k];
    uint8_t was = (v >> 3) & 1;
    uint8_t now = (v & 1) && !(v & 2);
    if (now != was) {
      S.apple[(size_t)b * T.nA_pad + k] = now;
      grid[(size_t)T.apple_layer * T.cells_pad + T.apple[k * 3 + 1]] = now ? cell_value(T.apple_sprite, 0) : (uint16_t)0;
    }
  }
  int d_delta = 0;
  for (int j = lane; j < T.nD; j += 32) {
    uint8_t v = sc.dirt[j];
    uint8_t was = (v >> 3) & 1;
    uint8_t now = (v & 1) && !(v & 2);
    if ((v & 1) && (v & 2)) --d_delta;  // DirtTracker:onStateChange (clean_up/components.lua:118-129)
    if (now != was) {
      S.dirt[(size_t)b * T.nD_pad + j] = now;
      grid[(size_t)T.dirt_layer * T.cells_pad + T.dirt[j * 3 + 1]] = now ? cell_value(T.dirt_sprite, 0) : (uint16_t)0;
    }
  }
  for (int o = 16; o > 0; o >>= 1) d_delta += __shfl_xor_sync(MP_FULL, d_delta, o);
  dirt_count += d_delta;
  // water Animation (component_library.lua:1070-1094): every piece flips every anim_frames frames.
  if (n % T.anim_frames == 0) {
    const int turn = (n / T.anim_frames) % T.n_anim;  // (uniform: the divisions are done once, not per piece)
    for (int k = lane; k < T.nW; k += 32) {
      int phase = (int)S.water[(size_t)b * T.nW_pad + k] + turn;
      if (phase >= T.n_anim) phase -= T.n_anim;
      grid[(size_t)T.water_layer * T.cells_pad + T.water[k * 2 + 1]] = cell_value(T.water_sprite[phase], 0);
    }
  }
  // avatar sprites: clear old cells, then write new ones.
  const bool changed = is_av && (x != x0 || y != y0 || orient != orient0 || alive != alive0);
  if (changed && alive0) grid[(size_t)T.avatar_layer * T.cells_pad + y0 * T.W + x0] = 0;
  __syncwarp();
  if (changed && alive) grid[(size_t)T.avatar_layer * T.cells_pad + y * T.W + x] = cell_value(T.avatar_sprite[lane], orient);

  // ---- store ---------------------------------------------------------------------------------
  const bool done = !cont || n >= T.max_frames;
  if (is_av) {
    *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(x, y, orient, alive);
    *reinterpret_cast<int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4) = make_int4(zap_cool, clean_cool, state_frame, 0);
    S.reward[(size_t)b * T.P + lane] = reward;
    S.packed[(size_t)b * (T.P + 2) + lane] = reward;
    for (int k = 0; k < T.n_scalar; ++k) {
      double v;
      if (T.scalar_obs[k] == 0)  // Zapper:readyToShoot (avatar_library.lua:737-744)
        v = alive ? fmax(1.0 - (double)zap_cool / (double)T.zap_cooldown, 0.0) : 0.0;
      else
        v = (double)num_others_cleaned;
      S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = v;
    }
  }
  if (lane == 0) {
    env[ENV_STEP] = n; env[ENV_DONE] = done ? 1 : 0; env[ENV_DIRT] = dirt_count;
    env[ENV_CLEANED] = (int)cleaned_now; env[ENV_ATE] = (int)ate_now; env[ENV_BEAM] = beam_dirty;
    S.discount[b] = done ? 0.0 : 1.0;
    S.step_type[b] = done ? 2 : 1;
    S.packed[(size_t)b * (T.P + 2) + T.P] = done ? 0.0 : 1.0;
    S.packed[(size_t)b * (T.P + 2) + T.P + 1] = done ? 2.0 : 1.0;
  }
}

// mode 0: step (envs whose last step was LAST start a new episode instead, policy A.17)
// mode 1: reset envs selected by `mask` (all if null)
__global__ void __launch_bounds__(128, 8) k_step_clean_up(Tables T, State S, const int32_t* __restrict__ actions,
                                                       const uint8_t* __restrict__ mask, int mode) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Programmatic dependent launch, both ways: let the renderer that follows in the stream stage its tables while this
  // grid drains, and do not touch env state before the kernel that precedes this one (the previous render) is complete.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // static lookup tables into shared memory, once per CTA (before the dependency wait: they never change)
  int16_t* s_apple_of = reinterpret_cast<int16_t*>(smem + 4 * warp_scratch_bytes(T));
  int16_t* s_dirt_of = s_apple_of + T.cells_pad;
  uint8_t* s_solid = reinterpret_cast<uint8_t*>(s_dirt_of + T.cells_pad);   // (8-byte aligned: cells_pad is a multiple of 8)
  uint8_t* s_flags = s_solid + T.cells_pad;
  int32_t* s_act = reinterpret_cast<int32_t*>(smem + 4 * warp_scratch_bytes(T) + scratch_round16((size_t)T.cells_pad * 6));
  for (int i = threadIdx.x; i < T.cells_pad; i += (int)blockDim.x) { s_apple_of[i] = T.apple_of_cell[i]; s_dirt_of[i] = T.dirt_of_cell[i]; s_flags[i] = T.cell_flags[i]; s_solid[i] = T.solid[i]; }
  for (int i = threadIdx.x; i < T.n_actions * 4; i += (int)blockDim.x) s_act[i] = T.action_table[i];
  asm volatile("griddepcontrol.wait;" ::: "memory");
  __syncthreads();
  const int b = blockIdx.x * 4 + warp;
  if (b >= S.B) return;
  WarpScratch sc = carve_scratch(T, smem + warp * warp_scratch_bytes(T));
  sc.apple_of = s_apple_of; sc.dirt_of = s_dirt_of; sc.flags = s_flags; sc.solid = s_solid; sc.act_table = s_act;
  if (!(mode == 1 && !(mask == nullptr || mask[b]))) {
    event_begin(lane);
    if (mode == 1 || S.env[(size_t)b * ENV_COLS + ENV_DONE]) clean_up_reset(T, S, b, lane, sc);
    else clean_up_step(T, S, b, lane, actions, sc);
    event_end(S, b, lane);
  }
}
