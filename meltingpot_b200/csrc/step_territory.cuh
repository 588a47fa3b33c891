// step_territory.cuh -- state transition of the territory family, one warp per env instance.
//
// Restates one frame of api:advance (api_factory.lua:104-111) for
//   meltingpot/lua/levels/territory/components.lua
//     (AllBeamBlocker, Resource, ResourceClaimer, RewardIndicator, Taste, Paintbrush)
//   meltingpot/lua/modules/avatar_library.lua
//     (Avatar :39-526, Zapper :570-850, GraduatedSanctionsMarking :948-1121)
// in closed form. Queue order of one frame (DESIGN.md policy ledger):
//   update():  Avatar (freeze / scheduled removal), Zapper (timed zapping prevention),
//              Resource (damage indicator, self repair), RewardIndicator          -> queued setStates
//   updaters:  150 move, 140 zap, 130 paintbrush, 100 episode end / claim / provideRewards,
//              3 marking recovery, 2 releaseClaimOfDeadAgent
//   round 1:   the queue in that order; callbacks (claims, destruction, sanctions) queue setStates
//   round 2:   those setStates, in enqueue order.
// Every episode start runs frame 0 through the same code with no-op actions (the paintbrush beam
// already fires during api:start's grid:update).
#pragma once

#include "common.cuh"
#include "step_clean_up.cuh"  // beam_scan

// Resource state codes: 0 unclaimed, 1 destroyed, 2 + i claimed_by_(i+1).
enum { RF_ACTIVE = 1, RF_NEVER_CLAIMED = 2, RF_DESTROYED = 4, RF_ABSENT = 8 /* not drawn into this episode's map ('choice' prefab) */ };
// fam_u8 sub-arrays (each nR_pad long), fam_u16 sub-arrays.
enum { RU_STATE = 0, RU_HEALTH = 1, RU_FLAGS = 2, RU_CLAIMER = 3, RU_IND = 4, RU_DMG = 5, RU_TEX = 6, RU_COUNT = 7 };
// RS_AGE is the resource's age in the frame about to run: frames since its last state change, which the updaters'
// startFrame (components.lua:101,115) is compared with and the oracle computes as frame - state_frame; saturated at 65535. mp_create refuses delays above that, so the
// comparisons with rewardDelay / delayTillSelfRepair / 5 stay exact in episodes of any length.
enum { RS_FSZ = 0, RS_AGE = 1, RS_COUNT = 2 };
// av_extra columns
enum { AX_FREEZE = 0, AX_REMOVAL = 1, AX_FLAGS = 2 /* bit0 movement allowed, bit1 zapping disallowed, bit2 marking on grid */,
       AX_NOZAP = 3, AX_LEVEL = 4, AX_MARK_T = 5, AX_SHOWN = 6 /* level whose sprite the marking shows */, AX_CLAIM_COOL = 7 };

struct TerritoryScratch {
  uint8_t* occ;            // [cells_pad] 0 free, 1..P avatar, 253 orphaned marking, 254 resource, 255 wall
  uint8_t* r[RU_COUNT];    // resource bytes
  uint8_t* r2_state;       // state after the queued setStates (simulated in enqueue order)
  uint8_t* r2_changed;
  uint8_t* was[4];         // state / reward indicator / damage indicator / texture as the frame started (round 2 writes the grid on change)
  uint16_t* fsz;
  uint16_t* age;
  uint32_t* bm_zap; uint32_t* bm_brush; uint32_t* bm_claim;  // cells already carrying a hit sprite
  int* cnt;                // [MP_MAX_PLAYERS] rewards provided this frame per avatar
  // per-CTA copies of static tables that sit on the frame's serial chain (an L2 round trip each otherwise)
  const uint8_t* wall255;  // [cells_pad] 255 where an AllBeamBlocker stands, else 0 (the initial occupancy)
  const int16_t* res_of;   // [cells_pad] resource index of a cell or -1
  const int16_t* res_cell; // [nR_pad] cell of a resource
  const int32_t* res_obj;  // [nR_pad] object id of a resource (RNG address)
};

__host__ __device__ inline size_t tr_round16(size_t n);
__host__ __device__ inline size_t territory_table_bytes(const Tables& T) {
  return ((size_t)T.cells_pad + 15) / 16 * 16 + ((size_t)T.cells_pad * 2 + 15) / 16 * 16 + (size_t)T.nR_pad * 2 + (size_t)T.nR_pad * 4;
}

__host__ __device__ inline size_t tr_round16(size_t n) { return (n + 15) & ~(size_t)15; }

// Layout: [fsz | age] (as in fam_u16) then [r[0..RU_COUNT)] (as in fam_u8), both 16-byte aligned and contiguous so that
// a frame moves them between HBM and shared memory with 128-bit accesses; then r2_state, r2_changed, the four
// frame-start copies round 2 compares against, occ, the hit-sprite bitmaps and the reward counters.
__host__ __device__ inline size_t territory_scratch_bytes(const Tables& T) {
  size_t words = (size_t)(T.cells + 31) / 32 + 1;
  return 2 * 2 * (size_t)T.nR_pad + (RU_COUNT + 2 + 4) * (size_t)T.nR_pad + tr_round16(T.cells_pad) + 3 * tr_round16(words * 4) + MP_MAX_PLAYERS * 4;
}

__device__ __forceinline__ TerritoryScratch carve_territory(const Tables& T, uint8_t* base) {
  TerritoryScratch s;
  size_t words = (size_t)(T.cells + 31) / 32 + 1;
  s.fsz = (uint16_t*)base; base += 2 * T.nR_pad;
  s.age = (uint16_t*)base; base += 2 * T.nR_pad;
  for (int i = 0; i < RU_COUNT; ++i) { s.r[i] = base; base += T.nR_pad; }
  s.r2_state = base; base += T.nR_pad;
  s.r2_changed = base; base += T.nR_pad;
  for (int i = 0; i < 4; ++i) { s.was[i] = base; base += T.nR_pad; }
  s.occ = base; base += tr_round16(T.cells_pad);
  s.bm_zap = (uint32_t*)base; base += tr_round16(words * 4);
  s.bm_brush = (uint32_t*)base; base += tr_round16(words * 4);
  s.bm_claim = (uint32_t*)base; base += tr_round16(words * 4);
  s.cnt = (int*)base;
  return s;
}

__device__ __forceinline__ uint16_t resource_sprite_value(const Tables& T, int state) {
  if (state == 0) return cell_value(T.unclaimed_sprite, 0);
  if (state == 1) return 0;
  return cell_value(T.claimed_sprite[state - 2], 0);
}

// Raw state of a new episode (before frame 0 runs).
__device__ void territory_init(const Tables& T, const State& S, int b, int lane, TerritoryScratch& sc, int episode, uint32_t k0, uint32_t k1) {
  uint16_t* grid = S.grid + (size_t)b * T.L * T.cells_pad;
  uint8_t* u8 = S.fam_u8 + (size_t)b * S.fam_u8_stride;
  uint16_t* u16 = S.fam_u16 + (size_t)b * S.fam_u16_stride;
  {
    const uint4* src = reinterpret_cast<const uint4*>(T.init_grid);
    uint4* dst = reinterpret_cast<uint4*>(grid);
    const int n16 = T.L * T.cells_pad / 8;
    for (int i = lane; i < n16; i += 32) dst[i] = src[i];
  }
  for (int k = lane; k < T.nR; k += 32) {  // Resource:reset (components.lua:73-80)
    u8[RU_STATE * T.nR_pad + k] = (uint8_t)T.tr_res[k * 3 + 2];
    u8[RU_HEALTH * T.nR_pad + k] = (uint8_t)T.res_health0;
    u8[RU_FLAGS * T.nR_pad + k] = RF_NEVER_CLAIMED;
    u8[RU_CLAIMER * T.nR_pad + k] = 0xFF;
    u8[RU_IND * T.nR_pad + k] = 0; u8[RU_DMG * T.nR_pad + k] = 0; u8[RU_TEX * T.nR_pad + k] = 0;
    u16[RS_FSZ * T.nR_pad + k] = 0; u16[RS_AGE * T.nR_pad + k] = 0;
    if (T.tr_res_cond && !choice_present(T, T.tr_res_cond[k * 2], (uint32_t)T.tr_res_cond[k * 2 + 1], episode, k0, k1)) {
      // This episode's map has plain floor here: the resource, its texture and its two indicators were not created.
      // Kept as a destroyed resource that never had a texture: nothing stands on the cell, nothing is drawn, nothing updates.
      const int cell = T.tr_res[k * 3 + 1];
      u8[RU_STATE * T.nR_pad + k] = 1; u8[RU_FLAGS * T.nR_pad + k] = RF_DESTROYED | RF_ABSENT; u8[RU_TEX * T.nR_pad + k] = 1;
      grid[(size_t)T.res_layer * T.cells_pad + cell] = 0; grid[(size_t)T.tex_layer * T.cells_pad + cell] = 0;
      grid[(size_t)T.ind_layer * T.cells_pad + cell] = 0; grid[(size_t)T.dmg_layer * T.cells_pad + cell] = 0;
    }
  }
  // spawn: partial Fisher-Yates over the spawn group (base_simulation.lua:396-445); with 'choice' spawn points the
  // group's members are this episode's draw, kept in piece order
  int16_t* tmp = reinterpret_cast<int16_t*>(sc.r2_state);  // scratch, reused later
  int n_spawn = T.n_spawn;
  if (T.spawn_cond) {
    n_spawn = 0;
    for (int base = 0; base < T.n_spawn && base < 64; base += 32) {
      const int i = base + lane;
      const bool on = i < T.n_spawn && choice_present(T, T.spawn_cond[i * 2], (uint32_t)T.spawn_cond[i * 2 + 1], episode, k0, k1);
      const unsigned m = __ballot_sync(MP_FULL, on);
      if (on) tmp[n_spawn + __popc(m & ((1u << lane) - 1u))] = (int16_t)T.spawn_cell[i];
      n_spawn += __popc(m);
    }
  } else {
    for (int i = lane; i < T.n_spawn && i < 64; i += 32) tmp[i] = (int16_t)T.spawn_cell[i];
  }
  __syncwarp();
  if (lane == 0) {
    for (int p = 0; p < T.P; ++p) {
      uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)p, RS_AVATAR_RESET, k0, k1);
      int r = p + (int)pick(w.x, (uint32_t)(n_spawn - p));
      int16_t t = tmp[p]; tmp[p] = tmp[r]; tmp[r] = t;
    }
  }
  __syncwarp();
  if (lane < T.P) {
    uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)lane, RS_AVATAR_RESET, k0, k1);
    int cell = tmp[lane], orient = (int)(w.y & 3u);
    *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(cell % T.W, cell / T.W, orient, 1);
    *reinterpret_cast<int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4) = make_int4(0, 0, 0, 0);
    int32_t* ax = S.av_extra + ((size_t)b * T.P + lane) * 8;
    ax[AX_FREEZE] = 0; ax[AX_REMOVAL] = 0; ax[AX_FLAGS] = 1; ax[AX_NOZAP] = 0;
    ax[AX_LEVEL] = T.mark_initial_level; ax[AX_MARK_T] = 0; ax[AX_SHOWN] = T.mark_initial_level; ax[AX_CLAIM_COOL] = 0;
    grid[(size_t)T.avatar_layer * T.cells_pad + cell] = cell_value(T.avatar_sprite[lane], orient);
  }
  __syncwarp();
}

// One frame. `actions` may be null (frame 0 of an episode: every avatar does nothing).
__device__ void territory_frame(const Tables& T, const State& S, int b, int lane, const int32_t* __restrict__ actions,
                                TerritoryScratch& sc, int n, int episode, uint32_t k0, uint32_t k1) {
  int32_t* env = S.env + (size_t)b * ENV_COLS;
  uint16_t* grid = S.grid + (size_t)b * T.L * T.cells_pad;
  uint8_t* u8 = S.fam_u8 + (size_t)b * S.fam_u8_stride;
  uint16_t* u16 = S.fam_u16 + (size_t)b * S.fam_u16_stride;
  const bool is_av = lane < T.P;
  const int words = (T.cells + 31) / 32 + 1;

  // ---- load ------------------------------------------------------------------------------------
  int x = 0, y = 0, orient = 0, alive = 0, zap_cool = 0, claim_cool = 0, state_frame = 0;
  int freeze = 0, removal = 0, move_ok = 1, nozap = 0, nozap_cnt = 0, mk_on = 0, level = 1, mark_t = 0, shown = 1;
  int act_move = 0, act_turn = 0, act_zap = 0, act_claim = 0;
  if (is_av) {
    const int4 a = *reinterpret_cast<const int4*>(S.avatar + ((size_t)b * T.P + lane) * 4);
    const int4 t = *reinterpret_cast<const int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4);
    const int32_t* ax = S.av_extra + ((size_t)b * T.P + lane) * 8;
    x = a.x; y = a.y; orient = a.z; alive = a.w; zap_cool = t.x; state_frame = t.z;
    freeze = ax[AX_FREEZE]; removal = ax[AX_REMOVAL]; move_ok = ax[AX_FLAGS] & 1; nozap = (ax[AX_FLAGS] >> 1) & 1; mk_on = (ax[AX_FLAGS] >> 2) & 1;
    nozap_cnt = ax[AX_NOZAP]; level = ax[AX_LEVEL]; mark_t = ax[AX_MARK_T]; shown = ax[AX_SHOWN]; claim_cool = ax[AX_CLAIM_COOL];
    if (actions) {
      int id = actions[(size_t)b * T.P + lane];
      if (id < 0 || id >= T.n_actions) id = 0;
      const int4 at = *reinterpret_cast<const int4*>(T.action_table + id * 4);
      act_move = at.x; act_turn = at.y; act_zap = at.z; act_claim = at.w;
    }
  }
  const int x0 = x, y0 = y, orient0 = orient, alive0 = alive, mk_on0 = mk_on, shown0 = shown;
  double reward = 0.0;  // Avatar:preUpdate
  {  // per-resource state, 16 resources per lane and access (fam_u8 / fam_u16 rows and the scratch have the same layout)
    const uint4* src8 = reinterpret_cast<const uint4*>(u8);
    uint4* dst8 = reinterpret_cast<uint4*>(sc.r[0]);
    for (int i = lane; i < RU_COUNT * T.nR_pad / 16; i += 32) dst8[i] = src8[i];
    const uint4* src16 = reinterpret_cast<const uint4*>(u16);
    uint4* dst16 = reinterpret_cast<uint4*>(sc.fsz);
    for (int i = lane; i < RS_COUNT * T.nR_pad / 8; i += 32) dst16[i] = src16[i];
    __syncwarp();
    for (int i = lane; i < T.nR_pad / 16; i += 32) {
      const uint4 st = reinterpret_cast<const uint4*>(sc.r[RU_STATE])[i];
      reinterpret_cast<uint4*>(sc.r2_state)[i] = st; reinterpret_cast<uint4*>(sc.was[0])[i] = st;
      reinterpret_cast<uint4*>(sc.was[1])[i] = reinterpret_cast<const uint4*>(sc.r[RU_IND])[i];
      reinterpret_cast<uint4*>(sc.was[2])[i] = reinterpret_cast<const uint4*>(sc.r[RU_DMG])[i];
      reinterpret_cast<uint4*>(sc.was[3])[i] = reinterpret_cast<const uint4*>(sc.r[RU_TEX])[i];
      reinterpret_cast<uint4*>(sc.r2_changed)[i] = make_uint4(0, 0, 0, 0);
    }
  }
  for (int i = lane; i < T.cells_pad / 8; i += 32) reinterpret_cast<uint2*>(sc.occ)[i] = reinterpret_cast<const uint2*>(sc.wall255)[i];
  for (int i = lane; i < words; i += 32) { sc.bm_zap[i] = 0; sc.bm_brush[i] = 0; sc.bm_claim[i] = 0; }
  if (lane < MP_MAX_PLAYERS) sc.cnt[lane] = 0;
  __syncwarp();
  for (int k = lane; k < T.nR; k += 32) if (sc.r[RU_STATE][k] != 1) sc.occ[sc.res_cell[k]] = 254;  // resources stand on the avatar layer
  if (is_av && alive) sc.occ[y * T.W + x] = (uint8_t)(lane + 1);
  // hit sprites live one frame (policy A.8)
  if (env[ENV_BEAM] & 1) { uint4 z = make_uint4(0, 0, 0, 0); uint4* l = reinterpret_cast<uint4*>(grid + (size_t)T.zap_layer * T.cells_pad); for (int i = lane; i < T.cells_pad / 8; i += 32) l[i] = z; }
  if (env[ENV_BEAM] & 2) { uint4 z = make_uint4(0, 0, 0, 0); uint4* l = reinterpret_cast<uint4*>(grid + (size_t)T.brush_layer * T.cells_pad); for (int i = lane; i < T.cells_pad / 8; i += 32) l[i] = z; }
  if (env[ENV_BEAM] & 4) for (int c = lane; c < T.cells; c += 32) { const int rr = sc.res_of[c]; if (rr < 0 || (sc.r[RU_FLAGS][rr] & RF_ABSENT)) grid[(size_t)T.claim_layer * T.cells_pad + c] = 0; }
  __syncwarp();
  int beam_dirty = 0;

  // ---- simulation:update ---------------------------------------------------------------------
  bool removed_now = false;
  if (is_av) {
    // Avatar:update (avatar_library.lua:334-354)
    if (freeze == 1) move_ok = 1;
    freeze = freeze > 0 ? freeze - 1 : 0;
    if (removal == 1) removed_now = alive != 0;  // setState(waitState): first item of this frame's queue
    removal = removal > 0 ? removal - 1 : 0;
    // Zapper:update (:713-724)
    if (nozap) zap_cool = T.zap_cooldown + 1;
    const int old = nozap_cnt;
    nozap_cnt = nozap_cnt > 0 ? nozap_cnt - 1 : 0;
    if (old == 1) nozap = 0;
  }
  for (int k = lane; k < T.nR; k += 32) {
    // Resource:update (components.lua:184-197) -> damage indicator setStates (applied in round 1)
    int health = sc.r[RU_HEALTH][k];
    if (health < T.res_health0) {
      int dmg = 1;
      int fsz = sc.fsz[k];
      if (fsz >= T.res_repair_delay) {
        uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)sc.res_obj[k], RS_OBJECT, k0, k1);
        if (u01(w.x, w.y) < T.res_repair_prob) { ++health; if (health == T.res_health0) dmg = 0; }
      }
      sc.r[RU_HEALTH][k] = (uint8_t)health;
      sc.r[RU_DMG][k] = (uint8_t)dmg;
      sc.fsz[k] = (uint16_t)min(fsz + 1, 65535);
    }
    // RewardIndicator:update (:303-312)
    const int st = sc.r[RU_STATE][k];
    sc.r[RU_IND][k] = ((sc.r[RU_FLAGS][k] & RF_ACTIVE) && st >= 2) ? (uint8_t)(st - 1) : 0;
  }
  __syncwarp();

  // ---- updaters --------------------------------------------------------------------------------
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
  const bool want_move = is_av && move_ok;                        // 150 Avatar move
  bool fire_zap = false, fire_claim = false;
  if (is_av && alive) { if (zap_cool > 0) --zap_cool; else if (act_zap == 1) { zap_cool = T.zap_cooldown; fire_zap = true; } }  // 140
  if (is_av && T.claim_wait >= 0) { if (claim_cool > 0) --claim_cool; else if (act_claim == 1) { claim_cool = T.claim_wait; fire_claim = true; } }  // 100 (no alive check)
  bool cont = true;
  if (n >= T.end_min_frames && ((n + 1) % T.end_interval) == 0) {
    uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, SCENE_DRAW_EPISODE_END, RS_SCENE, k0, k1);
    if (u01(w.x, w.y) < T.end_prob) cont = false;
  }
  const unsigned alive_mask0 = __ballot_sync(MP_FULL, is_av && alive);
  // 100 Resource provideRewards (:82-99) and 2 releaseClaimOfDeadAgent (:100-112), on frame-start state
  for (int k = lane; k < T.nR; k += 32) {
    const int st = sc.r[RU_STATE][k];
    if (st < 2) continue;
    const int age = sc.age[k];
    const int claimer = sc.r[RU_CLAIMER][k];
    if (age >= T.res_reward_delay) {
      uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)sc.res_obj[k], RS_OBJECT, k0, k1);
      if (u01(w.z, w.w) < T.res_rate && claimer != 0xFF) {
        if (alive_mask0 >> claimer & 1u) atomicAdd(&sc.cnt[claimer], 1);  // Avatar:addReward skips avatars in their wait state
        sc.r[RU_FLAGS][k] |= RF_ACTIVE;
      }
    }
    if (age >= 5 && claimer != 0xFF && !(alive_mask0 >> claimer & 1u) && !(sc.r[RU_FLAGS][k] & RF_DESTROYED)) {
      sc.r2_state[k] = 0; sc.r2_changed[k] = 1;  // setState(initialState): last item of round 1
      sc.r[RU_FLAGS][k] &= ~RF_ACTIVE; sc.r[RU_CLAIMER][k] = 0xFF;
    }
  }
  __syncwarp();
  if (is_av) {
    const double amount = T.tr_taste_role == 2 ? 0.0 : T.res_reward;  // Taste:addDefaultReward (:348-356)
    for (int i = 0; i < sc.cnt[lane]; ++i) reward += amount;
  }
  // 3 GraduatedSanctionsMarking resetToInitialLevel (avatar_library.lua:1009-1026)
  if (is_av && alive && level != T.mark_initial_level) {
    ++mark_t;
    if (mark_t == T.mark_recovery) { level = T.mark_initial_level; shown = level; mark_t = 0; }
  }

  // ---- round 1 ---------------------------------------------------------------------------------
  if (n == 0 && is_av) mk_on = 1;  // marking postStart: setState(level), teleport, setOrientation (:1033-1047)
  if (removed_now) { alive = 0; state_frame = n; }  // scheduled removal (queued by Avatar:update)
  __syncwarp();
  // The marking of a removed avatar stays on its cell until round 2: the cell cannot be entered this
  // frame (connected pieces move only if every member can), but beams treat it as empty.
  if (removed_now) sc.occ[y * T.W + x] = mk_on ? 253 : 0;
  __syncwarp();
  // moves
  for (int r = 0; r < T.P; ++r) {
    unsigned m = __ballot_sync(MP_FULL, is_av && rank == r);
    int src = __ffs(m) - 1;
    int s_ok = __shfl_sync(MP_FULL, (int)(alive && want_move), src);
    if (!s_ok) continue;
    int s_turn = __shfl_sync(MP_FULL, act_turn, src), s_move = __shfl_sync(MP_FULL, act_move, src);
    int sx = __shfl_sync(MP_FULL, x, src), sy = __shfl_sync(MP_FULL, y, src), so = __shfl_sync(MP_FULL, orient, src);
    if (s_turn != 0) so = (so + s_turn) & 3;
    if (s_move != 0) {
      int d = (so + s_move - 1) & 3;
      int nx = sx + dir_dx(d), ny = sy + dir_dy(d);
      bool inb = wrap_or_reject(T, nx, ny);
      if (inb && sc.occ[ny * T.W + nx] == 0) {
        __syncwarp();
        if (lane == 0) { sc.occ[sy * T.W + sx] = 0; sc.occ[ny * T.W + nx] = (uint8_t)(src + 1); }
        sx = nx; sy = ny;
      }
    }
    if (lane == src) { x = sx; y = sy; orient = so; }
    __syncwarp();
  }
  // beams: pass 0 zap (140), pass 1 paintbrush (130), pass 2 claim (100)
  for (int pass = 0; pass < 3; ++pass) {
    const BeamGeom& G = pass == 0 ? T.zap_geom : (pass == 1 ? T.brush_geom : T.claim_geom);
    if (pass == 1 && G.n == 1 && G.fwd[0] == 1 && G.lat[0] == 0) {
      // Paintbrush (territory/components.lua:362-412): every living avatar fires a one-cell beam every frame. The nine
      // beams are resolved together, one lane per avatar, with exactly the outcome of visiting them in this frame's
      // order: per resource the LAST claimant in order becomes the claimer; every claimant whose colour the resource does
      // not already show emits its event; the queued state is that of the last such claimant; the hit sprite of a
      // cell is the FIRST painter's (the sprite layer already holds one for later painters).
      int cell = -1, res = -1; bool cond = false;
      if (is_av && alive) {
        int cx = x + dir_dx(orient), cy = y + dir_dy(orient);
        if (wrap_or_reject(T, cx, cy)) {
          const int c = cy * T.W + cx, o = sc.occ[c];
          if (o != 255) cell = c;                       // AllBeamBlocker: no sprite, no hit
          if (o == 254) {
            res = sc.res_of[c];
            cond = sc.r[RU_STATE][res] != 2 + lane && !(sc.r[RU_FLAGS][res] & RF_DESTROYED);
          }
        }
      }
      int last_all = rank, last_cond = cond ? rank : -1, n_cond = cond ? 1 : 0, first_cell = rank;
      for (int q = 0; q < T.P; ++q) {
        const int q_res = __shfl_sync(MP_FULL, res, q), q_cell = __shfl_sync(MP_FULL, cell, q), q_rank = __shfl_sync(MP_FULL, rank, q);
        const bool q_cond = __shfl_sync(MP_FULL, (int)cond, q) != 0;
        if (q == lane) continue;
        if (res >= 0 && q_res == res) {
          last_all = max(last_all, q_rank);
          if (q_cond) { last_cond = max(last_cond, q_rank); ++n_cond; }
        }
        if (cell >= 0 && q_cell == cell) first_cell = min(first_cell, q_rank);
      }
      if (res >= 0) {
        if (last_all == rank) sc.r[RU_CLAIMER][res] = (uint8_t)lane;
        if (cond) emit_event(S, b, EV_CLAIMED_RESOURCE, lane + 1, 0);
        if (cond && last_cond == rank) {
          if (n_cond > 1 || sc.r2_state[res] != 2 + lane) { sc.r2_state[res] = (uint8_t)(2 + lane); sc.r2_changed[res] = 1; }
          sc.r[RU_FLAGS][res] &= ~(RF_ACTIVE | RF_NEVER_CLAIMED);
        }
      }
      if (cell >= 0 && first_cell == rank) {
        atomicOr(&sc.bm_brush[cell >> 5], 1u << (cell & 31));
        grid[(size_t)T.brush_layer * T.cells_pad + cell] = cell_value(T.brush_sprite[lane], orient);
        beam_dirty |= 2;
      }
      __syncwarp();
      continue;
    }
    for (int r = 0; r < T.P; ++r) {
      const bool fires = pass == 0 ? fire_zap : (pass == 1 ? true : fire_claim);
      unsigned m = __ballot_sync(MP_FULL, is_av && rank == r && fires && alive);  // off-grid shooters: hitBeam is a no-op
      if (!m) continue;
      int src = __ffs(m) - 1;
      int sx = __shfl_sync(MP_FULL, x, src), sy = __shfl_sync(MP_FULL, y, src), so = __shfl_sync(MP_FULL, orient, src);
      int cell = -1, res = -1, hit_avatar = -1; bool blocked = false;
      if (lane < G.n) {
        int f = so, rgt = (so + 1) & 3;
        int cx = sx + dir_dx(f) * G.fwd[lane] + dir_dx(rgt) * G.lat[lane];
        int cy = sy + dir_dy(f) * G.fwd[lane] + dir_dy(rgt) * G.lat[lane];
        if (!wrap_or_reject(T, cx, cy)) blocked = true;
        else {
          cell = cy * T.W + cx;
          const int o = sc.occ[cell];
          if (o == 255) blocked = true;  // AllBeamBlocker:onHit
          else if (o == 254) {
            res = sc.res_of[cell];
            if (pass == 0 && (int)sc.r[RU_HEALTH][res] - 1 != 0) blocked = true;  // zaps stop at an undestroyed resource
          } else if (o >= 1 && o <= T.P && o - 1 != src && pass == 0) { hit_avatar = o - 1; blocked = true; }  // Zapper:onHit
        }
      }
      bool vis;
      beam_scan(G, lane, blocked, vis);
      if (pass == 0) {
        // effects in footprint order
        unsigned em = __ballot_sync(MP_FULL, vis && (res >= 0 || hit_avatar >= 0));
        while (em) {
          const int c = __ffs(em) - 1; em &= em - 1;
          const int rr = __shfl_sync(MP_FULL, res, c), t = __shfl_sync(MP_FULL, hit_avatar, c);
          if (rr >= 0) {  // Resource:onHit zapHit (:148-170)
            if (lane == 0) {
              int h = (int)sc.r[RU_HEALTH][rr] - 1;
              sc.fsz[rr] = 0;
              if (h == 0) {
                h = T.res_health0;
                sc.r2_state[rr] = 1; sc.r2_changed[rr] = 1;
                sc.r[RU_FLAGS][rr] = (sc.r[RU_FLAGS][rr] & ~RF_ACTIVE) | RF_DESTROYED;
                sc.r[RU_TEX][rr] = 1; sc.r[RU_DMG][rr] = 0;  // texture 'destroyed', damage indicator 'inactive' (round 2)
                emit_event(S, b, EV_DESTROYED_RESOURCE, src + 1, 0);
              }
              sc.r[RU_HEALTH][rr] = (uint8_t)h;
            }
          } else {
            // Zapper:onHit (avatar_library.lua:652-681), then the marking on the same cell (:1049-1093)
            if (lane == t) reward += T.zap_penalty;
            if (lane == src) { reward += T.zap_reward; emit_event(S, b, EV_ZAP, src + 1, t + 1); }
            const int t_mk = __shfl_sync(MP_FULL, mk_on, t), t_level = __shfl_sync(MP_FULL, level, t);
            if (t_mk && t_level >= 1 && t_level <= T.mark_n_levels) {
              const int l = t_level - 1;
              if (lane == src) reward += T.mark_src_reward[l];
              if (lane == t) {
                reward += T.mark_tgt_reward[l];
                level += T.mark_inc[l];
                if (T.mark_remove[l]) { removal = 1; move_ok = 0; freeze = 1; nozap = 1; nozap_cnt = 1; emit_event(S, b, EV_REMOVAL, src + 1, t + 1); }
                else {
                  shown = level;  // _setLevel (round 2)
                  if (T.mark_freeze[l] > 0) { move_ok = 0; freeze = T.mark_freeze[l]; nozap = 1; nozap_cnt = T.mark_freeze[l]; }
                }
                mark_t = 0;
                emit_event(S, b, EV_SANCTIONING, src + 1, t + 1);
              }
            }
          }
          __syncwarp();
        }
      } else if (vis && res >= 0) {
        // Resource:_claim (:114-131) via directionHit* / claimBeam_*
        sc.r[RU_CLAIMER][res] = (uint8_t)src;
        const int flags_r = sc.r[RU_FLAGS][res];
        if (sc.r[RU_STATE][res] != 2 + src && !(flags_r & RF_DESTROYED)) {
          if (sc.r2_state[res] != 2 + src) { sc.r2_state[res] = (uint8_t)(2 + src); sc.r2_changed[res] = 1; }
          sc.r[RU_FLAGS][res] = flags_r & ~(RF_ACTIVE | RF_NEVER_CLAIMED);
          emit_event(S, b, EV_CLAIMED_RESOURCE, src + 1, 0);
        }
      }
      if (vis && !blocked && cell >= 0) {
        uint32_t* bm = pass == 0 ? sc.bm_zap : (pass == 1 ? sc.bm_brush : sc.bm_claim);
        const int layer = pass == 0 ? T.zap_layer : (pass == 1 ? T.brush_layer : T.claim_layer);
        const int sprite = pass == 0 ? T.zap_sprite : (pass == 1 ? T.brush_sprite[src] : T.claimbeam_sprite[src]);
        const int rr_here = pass == 2 ? sc.res_of[cell] : -1;
        const bool layer_free = rr_here < 0 || (sc.r[RU_FLAGS][rr_here] & RF_ABSENT);  // a resource's damage indicator occupies the claim layer
        if (layer_free) {
          const uint32_t bit = 1u << (cell & 31);
          const uint32_t old = atomicOr(&bm[cell >> 5], bit);
          if (!(old & bit)) grid[(size_t)layer * T.cells_pad + cell] = cell_value(sprite, so);
          beam_dirty |= 1 << pass;
        }
      }
      __syncwarp();
    }
  }
  beam_dirty = __reduce_or_sync(MP_FULL, (unsigned)beam_dirty);

  // ---- round 2 + write back -----------------------------------------------------------------
  if (is_av && !alive && alive0) mk_on = 0;  // avatarStateChange('die') -> marking setState(waitState)
  for (int k = lane; k < T.nR; k += 32) {
    const int cell = sc.res_cell[k];
    const int st_new = sc.r2_state[k];
    sc.age[k] = sc.r2_changed[k] ? (uint16_t)1 : (uint16_t)min((int)sc.age[k] + 1, 65535);  // age in frame n + 1
    const uint8_t was_state = sc.was[0][k], was_ind = sc.was[1][k], was_dmg = sc.was[2][k], was_tex = sc.was[3][k];
    sc.r[RU_STATE][k] = (uint8_t)st_new;
    if (st_new != was_state) grid[(size_t)T.res_layer * T.cells_pad + cell] = resource_sprite_value(T, st_new);
    if (sc.r[RU_IND][k] != was_ind) grid[(size_t)T.ind_layer * T.cells_pad + cell] = sc.r[RU_IND][k] ? cell_value(T.dry_sprite[sc.r[RU_IND][k] - 1], 0) : (uint16_t)0;
    if (sc.r[RU_DMG][k] != was_dmg) grid[(size_t)T.dmg_layer * T.cells_pad + cell] = sc.r[RU_DMG][k] ? cell_value(T.dmg_sprite, 0) : (uint16_t)0;
    if (sc.r[RU_TEX][k] != was_tex) grid[(size_t)T.tex_layer * T.cells_pad + cell] = sc.r[RU_TEX][k] ? (uint16_t)0 : cell_value(T.tex_sprite, 0);
  }
  __syncwarp();
  {
    uint4* dst8 = reinterpret_cast<uint4*>(u8);
    const uint4* src8 = reinterpret_cast<const uint4*>(sc.r[0]);
    for (int i = lane; i < RU_COUNT * T.nR_pad / 16; i += 32) dst8[i] = src8[i];
    uint4* dst16 = reinterpret_cast<uint4*>(u16);
    const uint4* src16 = reinterpret_cast<const uint4*>(sc.fsz);
    for (int i = lane; i < RS_COUNT * T.nR_pad / 8; i += 32) dst16[i] = src16[i];
  }
  // avatars and their markings
  const bool av_changed = is_av && (x != x0 || y != y0 || orient != orient0 || alive != alive0);
  const bool mk_changed = is_av && (av_changed || mk_on != mk_on0 || shown != shown0);
  if (av_changed && alive0) grid[(size_t)T.avatar_layer * T.cells_pad + y0 * T.W + x0] = 0;
  if (mk_changed && mk_on0) grid[(size_t)T.mark_layer * T.cells_pad + y0 * T.W + x0] = 0;
  __syncwarp();
  if (av_changed && alive) grid[(size_t)T.avatar_layer * T.cells_pad + y * T.W + x] = cell_value(T.avatar_sprite[lane], orient);
  if (mk_changed && mk_on) grid[(size_t)T.mark_layer * T.cells_pad + y * T.W + x] = cell_value(T.mark_sprite[shown - 1], orient);

  const bool done = n > 0 && (!cont || n >= T.max_frames);
  if (is_av) {
    *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(x, y, orient, alive);
    *reinterpret_cast<int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4) = make_int4(zap_cool, 0, state_frame, 0);
    int32_t* ax = S.av_extra + ((size_t)b * T.P + lane) * 8;
    ax[AX_FREEZE] = freeze; ax[AX_REMOVAL] = removal; ax[AX_FLAGS] = move_ok | (nozap << 1) | (mk_on << 2); ax[AX_NOZAP] = nozap_cnt;
    ax[AX_LEVEL] = level; ax[AX_MARK_T] = mark_t; ax[AX_SHOWN] = shown; ax[AX_CLAIM_COOL] = claim_cool;
    const double out = n == 0 ? 0.0 : reward;
    S.reward[(size_t)b * T.P + lane] = out;
    S.packed[(size_t)b * (T.P + 2) + lane] = out;
    for (int k = 0; k < T.n_scalar; ++k)
      S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = alive ? fmax(1.0 - (double)zap_cool / (double)T.zap_cooldown, 0.0) : 0.0;
  }
  if (lane == 0) {
    env[ENV_STEP] = n; env[ENV_DONE] = done ? 1 : 0; env[ENV_BEAM] = beam_dirty;
    const double disc = (n == 0 || done) ? 0.0 : 1.0;
    const int stype = n == 0 ? 0 : (done ? 2 : 1);
    S.discount[b] = disc; S.step_type[b] = stype;
    S.packed[(size_t)b * (T.P + 2) + T.P] = disc; S.packed[(size_t)b * (T.P + 2) + T.P + 1] = (double)stype;
  }
}

__global__ void __launch_bounds__(128, 8) k_step_territory(Tables T, State S, const int32_t* __restrict__ actions,
                                                       const uint8_t* __restrict__ mask, int mode) {
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Programmatic dependent launch, both ways: let the renderer that follows in the stream stage its tables while this
  // grid drains, and do not touch env state before the kernel that precedes this one (the previous render) is complete.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  // static tables into shared memory, once per CTA (before the dependency wait: they never change)
  uint8_t* tb = smem + 4 * territory_scratch_bytes(T);
  uint8_t* s_wall = tb; tb += ((size_t)T.cells_pad + 15) / 16 * 16;
  int16_t* s_res_of = reinterpret_cast<int16_t*>(tb); tb += ((size_t)T.cells_pad * 2 + 15) / 16 * 16;
  int16_t* s_res_cell = reinterpret_cast<int16_t*>(tb); tb += (size_t)T.nR_pad * 2;
  int32_t* s_res_obj = reinterpret_cast<int32_t*>(tb);
  for (int i = threadIdx.x; i < T.cells_pad; i += (int)blockDim.x) { s_wall[i] = T.wall[i] ? 255 : 0; s_res_of[i] = T.res_of_cell[i]; }
  for (int i = threadIdx.x; i < T.nR_pad; i += (int)blockDim.x) { s_res_cell[i] = i < T.nR ? (int16_t)T.tr_res[i * 3 + 1] : (int16_t)0; s_res_obj[i] = i < T.nR ? T.tr_res[i * 3] : 0; }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  __syncthreads();
  const int b = blockIdx.x * 4 + warp;
  if (b >= S.B) return;
  TerritoryScratch sc = carve_territory(T, smem + warp * territory_scratch_bytes(T));
  sc.wall255 = s_wall; sc.res_of = s_res_of; sc.res_cell = s_res_cell; sc.res_obj = s_res_obj;
  int32_t* env = S.env + (size_t)b * ENV_COLS;
  const uint64_t key = S.seed + (uint64_t)b;
  const uint32_t k0 = (uint32_t)key, k1 = (uint32_t)(key >> 32);
  const bool reset = mode == 1 ? (mask == nullptr || mask[b]) : (env[ENV_DONE] != 0);
  if (!(mode == 1 && !reset)) {
    event_begin(lane);
    if (reset) {
      const int episode = env[ENV_EPISODE] + 1;
      __syncwarp();
      territory_init(T, S, b, lane, sc, episode, k0, k1);
      if (lane == 0) { env[ENV_EPISODE] = episode; env[ENV_BEAM] = 0; }
      __syncwarp();
      territory_frame(T, S, b, lane, nullptr, sc, 0, episode, k0, k1);
    } else {
      territory_frame(T, S, b, lane, actions, sc, env[ENV_STEP] + 1, env[ENV_EPISODE], k0, k1);
    }
    event_end(S, b, lane);
  }
}
