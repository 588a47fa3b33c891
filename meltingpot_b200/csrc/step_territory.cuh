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

#include "family_load.h"
#include "step_common.cuh"

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

__host__ __device__ inline size_t territory_table_bytes(const Tables& T) {
  return scratch_round16(T.cells_pad) + scratch_round16((size_t)T.cells_pad * 2) + (size_t)T.nR_pad * 2 + (size_t)T.nR_pad * 4;
}

// Layout: [fsz | age] (as in fam_u16) then [r[0..RU_COUNT)] (as in fam_u8), both 16-byte aligned and contiguous so that
// a frame moves them between HBM and shared memory with 128-bit accesses; then r2_state, r2_changed, the four
// frame-start copies round 2 compares against, occ, the hit-sprite bitmaps and the reward counters.
__host__ __device__ inline size_t territory_scratch_bytes(const Tables& T) {
  size_t words = (size_t)(T.cells + 31) / 32 + 1;
  return 2 * 2 * (size_t)T.nR_pad + (RU_COUNT + 2 + 4) * (size_t)T.nR_pad + scratch_round16(T.cells_pad) + 3 * scratch_round16(words * 4) + MP_MAX_PLAYERS * 4;
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
  s.occ = base; base += scratch_round16(T.cells_pad);
  s.bm_zap = (uint32_t*)base; base += scratch_round16(words * 4);
  s.bm_brush = (uint32_t*)base; base += scratch_round16(words * 4);
  s.bm_claim = (uint32_t*)base; base += scratch_round16(words * 4);
  s.cnt = (int*)base;
  return s;
}

struct Territory {
  struct Params {
    Zapper zap;
    int res_layer, unclaimed_sprite, tex_layer, tex_sprite, ind_layer, dmg_layer, dmg_sprite, mark_layer;
    int mark_initial_level, mark_recovery, mark_n_levels, mark_inc[3], mark_remove[3], mark_freeze[3], mark_sprite[3];
    double mark_src_reward[3], mark_tgt_reward[3];
    int claim_wait, brush_layer, claim_layer, res_health0, res_reward_delay, res_repair_delay, tr_taste_role;
    double res_reward, res_rate, res_repair_prob;
    int claimed_sprite[MP_MAX_PLAYERS], dry_sprite[MP_MAX_PLAYERS], brush_sprite[MP_MAX_PLAYERS], claimbeam_sprite[MP_MAX_PLAYERS];
    BeamGeom claim_geom, brush_geom;
    const int32_t* tr_res;       // [nR][3] obj id, cell, initial state
    const int16_t* res_of_cell;  // [cells_pad] resource index or -1
    const uint8_t* wall;         // [cells_pad] 1 where an AllBeamBlocker piece stands
    const int32_t* tr_res_cond;  // [nR][2] (group or -1, ticket mask) of each resource ('choice' prefabs, Tables::choice_n), or null
  };

  __device__ __forceinline__ static uint16_t resource_sprite_value(const Params& F, int state) {
    if (state == 0) return cell_value(F.unclaimed_sprite, 0);
    if (state == 1) return 0;
    return cell_value(F.claimed_sprite[state - 2], 0);
  }

  // Host: the territory tables of the blob (compiler.py _territory_tables): tr_ip / tr_dp, resources, per-player
  // sprites, walls and the 'choice' conditions of the resources.
  static int load(FamilyLoad& ld, const Tables& T, Params& F) {
    const int32_t* ip;
    const double* dp;
    Section<int32_t> res, player_sprites;
    Section<uint8_t> wall_sec;
    int rc;
    if ((rc = ld.params("tr", MPB_TR_I_COUNT, MPB_TR_D_COUNT, &ip, &dp)) || (rc = ld.need("tr_res", MPB_I32, &res)) ||
        (rc = ld.need("tr_player_sprites", MPB_I32, &player_sprites)) || (rc = ld.need("tr_wall", MPB_U8, &wall_sec)))
      return rc;
    ld.nR = ip[MPB_TR_I_N_RES]; ld.nR_pad = round_up(std::max(ld.nR, 64), 16);
    F.res_layer = ip[MPB_TR_I_RES_LAYER]; F.unclaimed_sprite = ip[MPB_TR_I_UNCLAIMED_SPRITE];
    F.tex_layer = ip[MPB_TR_I_TEX_LAYER]; F.tex_sprite = ip[MPB_TR_I_TEX_SPRITE]; F.ind_layer = ip[MPB_TR_I_IND_LAYER];
    F.dmg_layer = ip[MPB_TR_I_DMG_LAYER]; F.dmg_sprite = ip[MPB_TR_I_DMG_SPRITE]; F.mark_layer = ip[MPB_TR_I_MARK_LAYER];
    F.mark_initial_level = ip[MPB_TR_I_MARK_INITIAL_LEVEL]; F.mark_recovery = ip[MPB_TR_I_MARK_RECOVERY];
    F.mark_n_levels = ip[MPB_TR_I_MARK_N_LEVELS];
    if (F.res_layer != T.avatar_layer) return fail(MP_E_UNSUPPORTED, "territory: resources and avatars must share a layer");
    if (F.mark_n_levels < 1 || F.mark_n_levels > 3) return fail(MP_E_UNSUPPORTED, "%d marking levels (1..3)", F.mark_n_levels);
    if ((rc = load_zapper(ld, T, ip, dp[MPB_TR_D_ZAP_PENALTY], dp[MPB_TR_D_ZAP_REWARD], F.zap))) return rc;
    if (F.zap.respawn <= T.max_frames) return fail(MP_E_UNSUPPORTED, "territory kernel assumes avatars never respawn (framesTillRespawn %d)", F.zap.respawn);
    const int length = ip[MPB_TR_I_CLAIM_LENGTH], radius = ip[MPB_TR_I_CLAIM_RADIUS];
    if (!make_beam_geom(length, radius, &F.claim_geom) || !make_beam_geom(1, 0, &F.brush_geom)) return fail(MP_E_UNSUPPORTED, "beam footprint larger than %d cells", MP_MAX_BEAM_CELLS);
    if (!beam_fits_torus(T, length, radius)) return fail(MP_E_UNSUPPORTED, "claim beam (length %d, radius %d) does not fit the %dx%d TORUS map", length, radius, T.W, T.H);
    ld.beam_cells = F.zap.geom.n + F.claim_geom.n + F.brush_geom.n;
    F.claim_wait = ip[MPB_TR_I_CLAIM_WAIT]; F.brush_layer = ip[MPB_TR_I_BRUSH_LAYER]; F.claim_layer = ip[MPB_TR_I_CLAIM_LAYER];
    if (F.claim_layer != F.dmg_layer) return fail(MP_E_UNSUPPORTED, "territory: claim beam layer must be the damage indicator layer");
    F.res_health0 = ip[MPB_TR_I_RES_HEALTH]; F.res_reward_delay = ip[MPB_TR_I_RES_REWARD_DELAY];
    F.res_repair_delay = ip[MPB_TR_I_RES_REPAIR_DELAY]; F.tr_taste_role = ip[MPB_TR_I_TASTE_ROLE];
    if (F.tr_taste_role != 0) return fail(MP_E_UNSUPPORTED, "territory Taste roles other than 'none'");
    if (F.res_health0 < 1 || F.res_health0 > 200) return fail(MP_E_UNSUPPORTED, "resource health %d", F.res_health0);
    // the resource age and frames-since-zapped counters saturate at 65535 (see RS_AGE)
    if (F.res_reward_delay > 65535 || F.res_repair_delay > 65535)
      return fail(MP_E_UNSUPPORTED, "rewardDelay %d / delayTillSelfRepair %d (max 65535)", F.res_reward_delay, F.res_repair_delay);
    const int istride = MPB_TR_I_MARK_INC_1 - MPB_TR_I_MARK_INC_0, dstride = MPB_TR_D_MARK_SRC_REWARD_1 - MPB_TR_D_MARK_SRC_REWARD_0;
    for (int l = 0; l < F.mark_n_levels; ++l) {
      const int32_t* li = ip + istride * l;
      const double* dl = dp + dstride * l;
      F.mark_inc[l] = li[MPB_TR_I_MARK_INC_0]; F.mark_remove[l] = li[MPB_TR_I_MARK_REMOVE_0];
      F.mark_freeze[l] = li[MPB_TR_I_MARK_FREEZE_0]; F.mark_sprite[l] = li[MPB_TR_I_MARK_SPRITE_0];
      F.mark_src_reward[l] = dl[MPB_TR_D_MARK_SRC_REWARD_0]; F.mark_tgt_reward[l] = dl[MPB_TR_D_MARK_TGT_REWARD_0];
    }
    F.res_reward = dp[MPB_TR_D_RES_REWARD]; F.res_rate = dp[MPB_TR_D_RES_RATE]; F.res_repair_prob = dp[MPB_TR_D_RES_REPAIR_PROB];
    ld.end_prob = dp[MPB_TR_D_END_PROB];
    for (int p = 0; p < T.P; ++p) {
      const int32_t* ps = player_sprites.data + p * 4;
      F.claimed_sprite[p] = ps[0]; F.dry_sprite[p] = ps[1]; F.brush_sprite[p] = ps[2]; F.claimbeam_sprite[p] = ps[3];
    }
    for (int p = 0; p < T.P; ++p) {  // wet paint on the resource texture, then dry paint on top: what most resource cells show
      ld.hint_stacks.push_back({F.tex_sprite, F.claimed_sprite[p]});
      ld.hint_stacks.push_back({F.tex_sprite, F.claimed_sprite[p], F.dry_sprite[p]});
    }
    std::vector<int32_t> v_res(res.data, res.data + res.count);
    std::vector<uint8_t> wall(T.cells_pad, 0);
    memcpy(wall.data(), wall_sec.data, std::min<size_t>(wall_sec.count, T.cells));
    ld.table(&F.tr_res, v_res);
    if ((rc = cell_index(ld, T, "tr_res", res, ld.nR, 3, &F.res_of_cell))) return rc;
    ld.table(&F.wall, wall);
    Section<int32_t> res_cond;
    if (get_section(ld.blob, ld.n, "tr_res_cond", MPB_I32, &res_cond)) {
      if ((int)res_cond.count != ld.nR * 2) return fail(MP_E_INVALID, "blob: tr_res_cond has %zu values for %d resources", res_cond.count, ld.nR);
      std::vector<int32_t> v(res_cond.data, res_cond.data + res_cond.count);
      ld.table(&F.tr_res_cond, v);
    }
    return MP_OK;
  }

  // Host: per-env variants may differ in the Zapper knobs, the marking's initial level, recovery, per-level increments,
  // removals, freezes and rewards, the claim wait, the Resource knobs and the resource, texture, damage, marking and
  // per-player claimed / dry sprites (appearance overrides); layers, beam hit sprites, beams, the number of marking
  // levels and the Taste role agree.
  static int same_shape(const Params& a, const Params& b) {
    MP_SAME_ZAPPER MP_SAME(res_layer) MP_SAME(tex_layer) MP_SAME(ind_layer) MP_SAME(dmg_layer)
    MP_SAME(mark_layer) MP_SAME(mark_n_levels) MP_SAME(brush_layer) MP_SAME(claim_layer)
    MP_SAME(tr_taste_role) MP_SAME(brush_sprite) MP_SAME(claimbeam_sprite)
    MP_SAME(claim_geom) MP_SAME(brush_geom)
    return MP_OK;
  }

  using Scratch = TerritoryScratch;
  // Maps of one set (same size, topology, players and 'choice' groups) may differ in their walls, resources and spawn
  // points: the resource table, the walls and the resources' 'choice' conditions are their entity tables, and the resource
  // count is the nR of each variant's Tables (nR_pad is the largest map's, setup_variants).
  static constexpr bool kMapVariants = true;
  static constexpr const char* kMapSections[] = {"tr_res", "tr_wall", "tr_res_cond", nullptr};
  // Its tables that hold only sprite ids (per player: claimed, dry, brush and claim-beam sprites): variants of one set may
  // differ there (mp_create_variants), as far as same_shape allows.
  static constexpr const char* kSpriteSections[] = {"tr_player_sprites", nullptr};
  static constexpr bool kStagesTables = true;
  __host__ __device__ static size_t scratch_bytes(const Tables& T) { return territory_scratch_bytes(T); }
  __host__ __device__ static size_t table_bytes(const Tables& T) { return territory_table_bytes(T); }

  // Per-CTA tables: wall255, res_of (int16 per cell), res_cell (int16) and res_obj (int32 per resource).
  __device__ static void stage(const Tables& T, const Params& F, uint8_t* tb) {
    uint8_t* s_wall = tb; tb += scratch_round16(T.cells_pad);
    int16_t* s_res_of = reinterpret_cast<int16_t*>(tb); tb += scratch_round16((size_t)T.cells_pad * 2);
    int16_t* s_res_cell = reinterpret_cast<int16_t*>(tb); tb += (size_t)T.nR_pad * 2;
    int32_t* s_res_obj = reinterpret_cast<int32_t*>(tb);
    for (int i = threadIdx.x; i < T.cells_pad; i += (int)blockDim.x) { s_wall[i] = F.wall[i] ? 255 : 0; s_res_of[i] = F.res_of_cell[i]; }
    for (int i = threadIdx.x; i < T.nR_pad; i += (int)blockDim.x) { s_res_cell[i] = i < T.nR ? (int16_t)F.tr_res[i * 3 + 1] : (int16_t)0; s_res_obj[i] = i < T.nR ? F.tr_res[i * 3] : 0; }
  }

  // The same tables for one env of a map-variant engine, by its warp, from its own map (T: that map's Tables, whose
  // nR_pad is the largest map's). stage() keeps its own copy of these lines: sharing them changed the SASS of the
  // single-blob kernels.
  __device__ static void stage_warp(const Tables& T, const Params& F, uint8_t* tb, int lane) {
    uint8_t* s_wall = tb; tb += scratch_round16(T.cells_pad);
    int16_t* s_res_of = reinterpret_cast<int16_t*>(tb); tb += scratch_round16((size_t)T.cells_pad * 2);
    int16_t* s_res_cell = reinterpret_cast<int16_t*>(tb); tb += (size_t)T.nR_pad * 2;
    int32_t* s_res_obj = reinterpret_cast<int32_t*>(tb);
    for (int i = lane; i < T.cells_pad; i += 32) { s_wall[i] = F.wall[i] ? 255 : 0; s_res_of[i] = F.res_of_cell[i]; }
    for (int i = lane; i < T.nR_pad; i += 32) { s_res_cell[i] = i < T.nR ? (int16_t)F.tr_res[i * 3 + 1] : (int16_t)0; s_res_obj[i] = i < T.nR ? F.tr_res[i * 3] : 0; }
  }

  __device__ static TerritoryScratch carve(const Tables& T, uint8_t* base, const uint8_t* tb) {
    TerritoryScratch sc = carve_territory(T, base);
    sc.wall255 = tb; tb += scratch_round16(T.cells_pad);
    sc.res_of = reinterpret_cast<const int16_t*>(tb); tb += scratch_round16((size_t)T.cells_pad * 2);
    sc.res_cell = reinterpret_cast<const int16_t*>(tb); tb += (size_t)T.nR_pad * 2;
    sc.res_obj = reinterpret_cast<const int32_t*>(tb);
    return sc;
  }

  // Raw state of a new episode (before frame 0 runs).
  __device__ static void init(const Tables& T, const Params& F, const State& S, int b, int lane, TerritoryScratch& sc, uint16_t* grid, int episode, uint32_t k0, uint32_t k1) {
    uint8_t* u8 = S.fam_u8 + (size_t)b * S.fam_u8_stride;
    uint16_t* u16 = S.fam_u16 + (size_t)b * S.fam_u16_stride;
    copy_init_grid(T, grid, lane);
    for (int k = lane; k < T.nR; k += 32) {  // Resource:reset (components.lua:73-80)
      u8[RU_STATE * T.nR_pad + k] = (uint8_t)F.tr_res[k * 3 + 2];
      u8[RU_HEALTH * T.nR_pad + k] = (uint8_t)F.res_health0;
      u8[RU_FLAGS * T.nR_pad + k] = RF_NEVER_CLAIMED;
      u8[RU_CLAIMER * T.nR_pad + k] = 0xFF;
      u8[RU_IND * T.nR_pad + k] = 0; u8[RU_DMG * T.nR_pad + k] = 0; u8[RU_TEX * T.nR_pad + k] = 0;
      u16[RS_FSZ * T.nR_pad + k] = 0; u16[RS_AGE * T.nR_pad + k] = 0;
      if (F.tr_res_cond && !choice_present(T, F.tr_res_cond[k * 2], (uint32_t)F.tr_res_cond[k * 2 + 1], episode, k0, k1)) {
        // This episode's map has plain floor here: the resource, its texture and its two indicators were not created.
        // Kept as a destroyed resource that never had a texture: nothing stands on the cell, nothing is drawn, nothing updates.
        const int cell = F.tr_res[k * 3 + 1];
        u8[RU_STATE * T.nR_pad + k] = 1; u8[RU_FLAGS * T.nR_pad + k] = RF_DESTROYED | RF_ABSENT; u8[RU_TEX * T.nR_pad + k] = 1;
        grid[(size_t)F.res_layer * T.cells_pad + cell] = 0; grid[(size_t)F.tex_layer * T.cells_pad + cell] = 0;
        grid[(size_t)F.ind_layer * T.cells_pad + cell] = 0; grid[(size_t)F.dmg_layer * T.cells_pad + cell] = 0;
      }
    }
    // spawn: with 'choice' spawn points the group's members are this episode's draw
    spawn_group(T, S, b, lane, grid, reinterpret_cast<int16_t*>(sc.r2_state) /* scratch, reused later */, T.spawn_cell, T.n_spawn,
                [](int) { return true; },
                [&](int i) { return !T.spawn_cond || choice_present(T, T.spawn_cond[i * 2], (uint32_t)T.spawn_cond[i * 2 + 1], episode, k0, k1); },
                episode, k0, k1, [&](int) {
      int32_t* ax = S.av_extra + ((size_t)b * T.P + lane) * 8;
      ax[AX_FREEZE] = 0; ax[AX_REMOVAL] = 0; ax[AX_FLAGS] = 1; ax[AX_NOZAP] = 0;
      ax[AX_LEVEL] = F.mark_initial_level; ax[AX_MARK_T] = 0; ax[AX_SHOWN] = F.mark_initial_level; ax[AX_CLAIM_COOL] = 0;
    });
  }

  // One frame. `actions` is null on frame 0 of an episode: every avatar does nothing.
  template <class Actions>
  __device__ static void frame(const Tables& T, const Params& F, const State& S, int b, int lane, const Actions& actions, TerritoryScratch& sc,
                               const Frame& f) {
    const auto [env, grid, k0, k1, n, episode] = f;
    uint8_t* u8 = S.fam_u8 + (size_t)b * S.fam_u8_stride;
    uint16_t* u16 = S.fam_u16 + (size_t)b * S.fam_u16_stride;
    const bool is_av = lane < T.P;
    const int words = (T.cells + 31) / 32 + 1;

    // ---- load ------------------------------------------------------------------------------------
    int4 a, t, act;
    load_avatar(T, S, b, lane, actions, T.action_table, a, t, act);
    int x = a.x, y = a.y, orient = a.z, alive = a.w, zap_cool = t.x, claim_cool = 0, state_frame = t.z;
    int freeze = 0, removal = 0, move_ok = 1, nozap = 0, nozap_cnt = 0, mk_on = 0, level = 1, mark_t = 0, shown = 1;
    const int act_move = act.x, act_turn = act.y, act_zap = act.z, act_claim = act.w;
    if (is_av) {
      const int32_t* ax = S.av_extra + ((size_t)b * T.P + lane) * 8;
      freeze = ax[AX_FREEZE]; removal = ax[AX_REMOVAL]; move_ok = ax[AX_FLAGS] & 1; nozap = (ax[AX_FLAGS] >> 1) & 1; mk_on = (ax[AX_FLAGS] >> 2) & 1;
      nozap_cnt = ax[AX_NOZAP]; level = ax[AX_LEVEL]; mark_t = ax[AX_MARK_T]; shown = ax[AX_SHOWN]; claim_cool = ax[AX_CLAIM_COOL];
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
    init_occupancy(T, sc.occ, sc.wall255, lane);
    for (int i = lane; i < words; i += 32) { sc.bm_zap[i] = 0; sc.bm_brush[i] = 0; sc.bm_claim[i] = 0; }
    if (lane < MP_MAX_PLAYERS) sc.cnt[lane] = 0;
    __syncwarp();
    for (int k = lane; k < T.nR; k += 32) if (sc.r[RU_STATE][k] != 1) sc.occ[sc.res_cell[k]] = 254;  // resources stand on the avatar layer
    if (is_av && alive) sc.occ[y * T.W + x] = (uint8_t)(lane + 1);
    // hit sprites live one frame (policy A.8)
    if (env[ENV_BEAM] & 1) clear_layer(T, grid, F.zap.layer, lane);
    if (env[ENV_BEAM] & 2) clear_layer(T, grid, F.brush_layer, lane);
    if (env[ENV_BEAM] & 4) for (int c = lane; c < T.cells; c += 32) { const int rr = sc.res_of[c]; if (rr < 0 || (sc.r[RU_FLAGS][rr] & RF_ABSENT)) grid[(size_t)F.claim_layer * T.cells_pad + c] = 0; }
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
      if (nozap) zap_cool = F.zap.cooldown + 1;
      const int old = nozap_cnt;
      nozap_cnt = nozap_cnt > 0 ? nozap_cnt - 1 : 0;
      if (old == 1) nozap = 0;
    }
    for (int k = lane; k < T.nR; k += 32) {
      // Resource:update (components.lua:184-197) -> damage indicator setStates (applied in round 1)
      int health = sc.r[RU_HEALTH][k];
      if (health < F.res_health0) {
        int dmg = 1;
        int fsz = sc.fsz[k];
        if (fsz >= F.res_repair_delay) {
          uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)sc.res_obj[k], RS_OBJECT, k0, k1);
          if (u01(w.x, w.y) < F.res_repair_prob) { ++health; if (health == F.res_health0) dmg = 0; }
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
    const int rank = visit_rank(T, lane, n, episode, k0, k1);
    bool fire_zap = false, fire_claim = false;
    if (is_av && alive) { if (zap_cool > 0) --zap_cool; else if (act_zap == 1) { zap_cool = F.zap.cooldown; fire_zap = true; } }  // 140
    if (is_av && F.claim_wait >= 0) { if (claim_cool > 0) --claim_cool; else if (act_claim == 1) { claim_cool = F.claim_wait; fire_claim = true; } }  // 100 (no alive check)
    const bool cont = episode_continues(T, n, episode, k0, k1);
    const unsigned alive_mask0 = __ballot_sync(MP_FULL, is_av && alive);
    // 100 Resource provideRewards (:82-99) and 2 releaseClaimOfDeadAgent (:100-112), on frame-start state
    for (int k = lane; k < T.nR; k += 32) {
      const int st = sc.r[RU_STATE][k];
      if (st < 2) continue;
      const int age = sc.age[k];
      const int claimer = sc.r[RU_CLAIMER][k];
      if (age >= F.res_reward_delay) {
        uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)sc.res_obj[k], RS_OBJECT, k0, k1);
        if (u01(w.z, w.w) < F.res_rate && claimer != 0xFF) {
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
      const double amount = F.tr_taste_role == 2 ? 0.0 : F.res_reward;  // Taste:addDefaultReward (:348-356)
      for (int i = 0; i < sc.cnt[lane]; ++i) reward += amount;
    }
    // 3 GraduatedSanctionsMarking resetToInitialLevel (avatar_library.lua:1009-1026)
    if (is_av && alive && level != F.mark_initial_level) {
      ++mark_t;
      if (mark_t == F.mark_recovery) { level = F.mark_initial_level; shown = level; mark_t = 0; }
    }

    // ---- round 1 ---------------------------------------------------------------------------------
    if (n == 0 && is_av) mk_on = 1;  // marking postStart: setState(level), teleport, setOrientation (:1033-1047)
    if (removed_now) { alive = 0; state_frame = n; }  // scheduled removal (queued by Avatar:update)
    __syncwarp();
    // The marking of a removed avatar stays on its cell until round 2: the cell cannot be entered this
    // frame (connected pieces move only if every member can), but beams treat it as empty.
    if (removed_now) sc.occ[y * T.W + x] = mk_on ? 253 : 0;
    __syncwarp();
    // 150 Avatar move
    move_avatars(T, lane, rank, is_av && alive && move_ok, act_turn, act_move, x, y, orient, sc.occ, [](int, int) {});
    // beams: pass 0 zap (140), pass 1 paintbrush (130), pass 2 claim (100)
    for (int pass = 0; pass < 3; ++pass) {
      const BeamGeom& G = pass == 0 ? F.zap.geom : (pass == 1 ? F.brush_geom : F.claim_geom);
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
          grid[(size_t)F.brush_layer * T.cells_pad + cell] = cell_value(F.brush_sprite[lane], orient);
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
        const int cell = beam_cell(T, G, lane, sx, sy, so);
        int res = -1, hit_avatar = -1;
      bool blocked = cell < 0 && lane < G.n;  // off the map
        if (cell >= 0) {
          const int o = sc.occ[cell];
          if (o == 255) blocked = true;  // AllBeamBlocker:onHit
          else if (o == 254) {
            res = sc.res_of[cell];
            if (pass == 0 && (int)sc.r[RU_HEALTH][res] - 1 != 0) blocked = true;  // zaps stop at an undestroyed resource
          } else if (o >= 1 && o <= T.P && o - 1 != src && pass == 0) { hit_avatar = o - 1; blocked = true; }  // Zapper:onHit
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
                  h = F.res_health0;
                  sc.r2_state[rr] = 1; sc.r2_changed[rr] = 1;
                  sc.r[RU_FLAGS][rr] = (sc.r[RU_FLAGS][rr] & ~RF_ACTIVE) | RF_DESTROYED;
                  sc.r[RU_TEX][rr] = 1; sc.r[RU_DMG][rr] = 0;  // texture 'destroyed', damage indicator 'inactive' (round 2)
                  emit_event(S, b, EV_DESTROYED_RESOURCE, src + 1, 0);
                }
                sc.r[RU_HEALTH][rr] = (uint8_t)h;
              }
            } else {
              // Zapper:onHit (avatar_library.lua:652-681), then the marking on the same cell (:1049-1093)
              if (lane == t) reward += F.zap.penalty;
              if (lane == src) { reward += F.zap.reward; emit_event(S, b, EV_ZAP, src + 1, t + 1); }
              const int t_mk = __shfl_sync(MP_FULL, mk_on, t), t_level = __shfl_sync(MP_FULL, level, t);
              if (t_mk && t_level >= 1 && t_level <= F.mark_n_levels) {
                const int l = t_level - 1;
                if (lane == src) reward += F.mark_src_reward[l];
                if (lane == t) {
                  reward += F.mark_tgt_reward[l];
                  level += F.mark_inc[l];
                  if (F.mark_remove[l]) { removal = 1; move_ok = 0; freeze = 1; nozap = 1; nozap_cnt = 1; emit_event(S, b, EV_REMOVAL, src + 1, t + 1); }
                  else {
                    shown = level;  // _setLevel (round 2)
                    if (F.mark_freeze[l] > 0) { move_ok = 0; freeze = F.mark_freeze[l]; nozap = 1; nozap_cnt = F.mark_freeze[l]; }
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
        if (vis && !blocked) {
          uint32_t* bm = pass == 0 ? sc.bm_zap : (pass == 1 ? sc.bm_brush : sc.bm_claim);
          const int layer = pass == 0 ? F.zap.layer : (pass == 1 ? F.brush_layer : F.claim_layer);
          const int sprite = pass == 0 ? F.zap.sprite : (pass == 1 ? F.brush_sprite[src] : F.claimbeam_sprite[src]);
          const int rr_here = pass == 2 ? sc.res_of[cell] : -1;
          const bool layer_free = rr_here < 0 || (sc.r[RU_FLAGS][rr_here] & RF_ABSENT);  // a resource's damage indicator occupies the claim layer
          if (layer_free) { draw_hit_sprite(T, grid, bm, layer, cell, cell_value(sprite, so)); beam_dirty |= 1 << pass; }
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
      if (st_new != was_state) grid[(size_t)F.res_layer * T.cells_pad + cell] = resource_sprite_value(F, st_new);
      if (sc.r[RU_IND][k] != was_ind) grid[(size_t)F.ind_layer * T.cells_pad + cell] = sc.r[RU_IND][k] ? cell_value(F.dry_sprite[sc.r[RU_IND][k] - 1], 0) : (uint16_t)0;
      if (sc.r[RU_DMG][k] != was_dmg) grid[(size_t)F.dmg_layer * T.cells_pad + cell] = sc.r[RU_DMG][k] ? cell_value(F.dmg_sprite, 0) : (uint16_t)0;
      if (sc.r[RU_TEX][k] != was_tex) grid[(size_t)F.tex_layer * T.cells_pad + cell] = sc.r[RU_TEX][k] ? (uint16_t)0 : cell_value(F.tex_sprite, 0);
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
    const bool av_changed = draw_avatars(T, grid, lane, x0, y0, orient0, alive0, x, y, orient, alive);
    const bool mk_changed = is_av && (av_changed || mk_on != mk_on0 || shown != shown0);
    if (mk_changed && mk_on0) grid[(size_t)F.mark_layer * T.cells_pad + y0 * T.W + x0] = 0;
    __syncwarp();
    if (mk_changed && mk_on) grid[(size_t)F.mark_layer * T.cells_pad + y * T.W + x] = cell_value(F.mark_sprite[shown - 1], orient);

    const bool done = n > 0 && (!cont || n >= T.max_frames);
    if (is_av) {
      *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(x, y, orient, alive);
      *reinterpret_cast<int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4) = make_int4(zap_cool, 0, state_frame, 0);
      int32_t* ax = S.av_extra + ((size_t)b * T.P + lane) * 8;
      ax[AX_FREEZE] = freeze; ax[AX_REMOVAL] = removal; ax[AX_FLAGS] = move_ok | (nozap << 1) | (mk_on << 2); ax[AX_NOZAP] = nozap_cnt;
      ax[AX_LEVEL] = level; ax[AX_MARK_T] = mark_t; ax[AX_SHOWN] = shown; ax[AX_CLAIM_COOL] = claim_cool;
      for (int k = 0; k < T.n_scalar; ++k)
        S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = alive ? fmax(1.0 - (double)zap_cool / (double)F.zap.cooldown, 0.0) : 0.0;
    }
    store_timestep(T, S, b, lane, n, n == 0 ? 0.0 : reward, n == 0 ? 0 : (done ? 2 : 1), beam_dirty);
  }

  // Every episode starts with the raw state of init, then runs frame 0.
  __device__ static void reset(const Tables& T, const Params& F, const State& S, int b, int lane, TerritoryScratch& sc) {
    const Frame f = begin_frame(T, S, b, true);
    __syncwarp();
    init(T, F, S, b, lane, sc, f.grid, f.episode, f.k0, f.k1);
    reset_env_row(T, S, b, lane, f.episode, 0);
    frame<DenseActions>(T, F, S, b, lane, nullptr, sc, f);
  }

  // Episode start of an env of a map-variant engine: also zeroes the env's resource bytes past this map's resources, up
  // to the padding of the largest map, so that an env that moved from a map with more resources keeps none of their
  // bytes (records and snapshots of equal envs stay equal byte for byte). A single-map engine never writes there.
  __device__ static void reset_map(const Tables& T, const Params& F, const State& S, int b, int lane, TerritoryScratch& sc) {
    uint8_t* u8 = S.fam_u8 + (size_t)b * S.fam_u8_stride;
    uint16_t* u16 = S.fam_u16 + (size_t)b * S.fam_u16_stride;
    for (int k = T.nR + lane; k < T.nR_pad; k += 32) {
      for (int r = 0; r < RU_COUNT; ++r) u8[r * T.nR_pad + k] = 0;
      for (int r = 0; r < RS_COUNT; ++r) u16[r * T.nR_pad + k] = 0;
    }
    reset(T, F, S, b, lane, sc);
  }

  template <class Actions>
  __device__ static void step(const Tables& T, const Params& F, const State& S, int b, int lane, const Actions& actions, TerritoryScratch& sc) {
    frame<Actions>(T, F, S, b, lane, actions, sc, begin_frame(T, S, b, false));
  }
};
