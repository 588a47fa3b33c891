// step_commons.cuh -- state transition of the commons_harvest family, one warp per env instance.
//
// Restates one frame of api:advance (api_factory.lua:104-111) for the components of
//   meltingpot/lua/levels/commons_harvest/components.lua (Neighborhoods, DensityRegrow)
//   meltingpot/lua/modules/component_library.lua:953-1002 (Edible)
//   meltingpot/lua/modules/avatar_library.lua (Avatar, Zapper)
// in the closed form of step_common.cuh: lanes are avatars, beam footprint cells, apples or
// the disc neighbours of one apple, depending on the phase.
//
// Apple state codes (State.apple): 0 live ('apple', lowerPhysical), 1 'appleWait', 2 + k 'appleWait_k'.
// State.apple_count is DensityRegrow's pieceToNumNeighbors, maintained with the reference's own
// incremental (and order dependent) bookkeeping -- see _beginLive / _endLive below.
#pragma once

#include "family_load.h"
#include "step_common.cuh"

__device__ __forceinline__ bool ch_is_wait(uint8_t s) { return s != 0; }

struct Commons {
  struct Params {
    Zapper zap;
    int apple_layer, apple_sprite, wait_layer, wait_sprite, grass_layer, grass_sprite, dess_sprite, ch_n_wait, ch_n_probs;
    double ch_probs[4], eat_reward;
    const int32_t* ch_apple;       // [nA][4] obj id, cell, initially live, grass obj id
    const int32_t* ch_nbr;         // [nA][16] apples inside the regrowth disc (excluding self), -1 padded
    const int16_t* apple_of_cell;  // [cells_pad] apple index or -1
  };

  // Host: the commons_harvest tables of the blob (compiler.py _commons_tables): ch_ip / ch_dp, apples and their
  // regrowth-disc neighbours.
  static int load(FamilyLoad& ld, const Tables& T, Params& F) {
    const int32_t* ip;
    const double* dp;
    Section<int32_t> apple, nbr;
    int rc;
    if ((rc = ld.params("ch", MPB_CH_I_COUNT, MPB_CH_D_COUNT, &ip, &dp)) || (rc = ld.need("ch_apple", MPB_I32, &apple)) ||
        (rc = ld.need("ch_nbr", MPB_I32, &nbr)))
      return rc;
    ld.nA = ip[MPB_CH_I_N_APPLES]; F.apple_layer = ip[MPB_CH_I_APPLE_LAYER]; F.apple_sprite = ip[MPB_CH_I_APPLE_SPRITE];
    F.wait_layer = ip[MPB_CH_I_WAIT_LAYER]; F.wait_sprite = ip[MPB_CH_I_WAIT_SPRITE];
    F.ch_n_wait = ip[MPB_CH_I_N_WAIT]; F.ch_n_probs = ip[MPB_CH_I_N_PROBS]; F.grass_layer = ip[MPB_CH_I_GRASS_LAYER];
    F.grass_sprite = ip[MPB_CH_I_GRASS_SPRITE]; F.dess_sprite = ip[MPB_CH_I_DESS_SPRITE];
    if (F.ch_n_wait < 1 || F.ch_n_wait > 29 || F.ch_n_probs < 1 || F.ch_n_probs > 4) return fail(MP_E_UNSUPPORTED, "DensityRegrow with %d wait states / %d probabilities", F.ch_n_wait, F.ch_n_probs);
    if (ld.nA > 2048) return fail(MP_E_UNSUPPORTED, "%d apples (max 2048)", ld.nA);
    if ((rc = load_zapper(ld, T, ip, dp[MPB_CH_D_ZAP_PENALTY], dp[MPB_CH_D_ZAP_REWARD], F.zap))) return rc;
    ld.beam_cells = F.zap.geom.n;
    for (int i = 0; i < 4; ++i) F.ch_probs[i] = dp[MPB_CH_D_PROB_0 + i];
    F.eat_reward = dp[MPB_CH_D_EAT_REWARD]; ld.end_prob = dp[MPB_CH_D_END_PROB];
    std::vector<int32_t> v_apple(apple.data, apple.data + apple.count), v_nbr(nbr.data, nbr.data + nbr.count);
    ld.table(&F.ch_apple, v_apple); ld.table(&F.ch_nbr, v_nbr);
    return cell_index(ld, T, "ch_apple", apple, ld.nA, 4, &F.apple_of_cell);
  }

  // Host: per-env variants may differ in the Zapper knobs and its beam footprint (length and radius), the DensityRegrow
  // probabilities and the Edible reward, and, as maps of one set (map variants: commons_harvest__open, __closed and
  // __partnership), in the apples, their regrowth discs and the walls. The apple, wait, grass and desert sprites are
  // knobs too (appearance overrides).
  static int same_shape(const Params& a, const Params& b) {
    MP_SAME(zap.layer) MP_SAME(zap.sprite) MP_SAME(zap.hit) MP_SAME(apple_layer) MP_SAME(wait_layer) MP_SAME(grass_layer)
    MP_SAME(ch_n_wait) MP_SAME(ch_n_probs)
    return MP_OK;
  }

  using Scratch = WarpScratch;
  // Maps of one set may differ in their walls and apples (mp_create_variants): the apple table and the regrowth discs are
  // their entity tables, and the apple count is the nA of each variant's Tables (setup_variants).
  static constexpr bool kMapVariants = true;
  static constexpr const char* kMapSections[] = {"ch_apple", "ch_nbr", nullptr};
  static constexpr const char* const* kSpriteSections = nullptr;
  static constexpr bool kStagesTables = false;
  __host__ __device__ static size_t scratch_bytes(const Tables& T) { return warp_scratch_bytes(T); }
  __host__ __device__ static size_t table_bytes(const Tables&) { return 0; }
  __device__ static void stage(const Tables&, const Params&, uint8_t*) {}
  __device__ static WarpScratch carve(const Tables& T, uint8_t* base, const uint8_t*) { return carve_scratch(T, base); }

  // Episode start for commons_harvest: one spawn group per initial group of avatars.
  __device__ static void reset(const Tables& T, const Params& F, const State& S, int b, int lane, WarpScratch& sc) {
    const auto [env, grid, k0, k1, n, episode] = begin_frame(T, S, b, true);
    __syncwarp();
    copy_init_grid(T, grid, lane);
    for (int k = lane; k < T.nA; k += 32) {  // DensityRegrow:start -> count 0; all apples start live
      S.apple[(size_t)b * T.nA_pad + k] = F.ch_apple[k * 4 + 2] ? 0 : 1;
      S.apple_count[(size_t)b * T.nA_pad + k] = 0;
    }
    __syncwarp();
    for (int g = 0; g < 2; ++g) {
      if (T.n_spawn_init[g] == 0) continue;
      spawn_group(T, S, b, lane, grid, sc.tmp, T.spawn_init_cell[g], T.n_spawn_init[g], [&](int p) { return T.avatar_init_group[p] == g; },
                  [](int) { return true; }, episode, k0, k1, [&](int) {
        for (int k = 0; k < T.n_scalar; ++k) S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = T.scalar_obs[k] == 0 ? 1.0 : 0.0;
      });
    }
    reset_env_row(T, S, b, lane, episode, 0);
  }

  // Episode start of an env of a map-variant engine: also zeroes the env's apple rows past this map's apples, up to the
  // padding of the largest map, so that an env that moved from a map with more apples keeps none of their bytes (records
  // and snapshots of equal envs stay equal byte for byte). A single-map engine never writes there.
  __device__ static void reset_map(const Tables& T, const Params& F, const State& S, int b, int lane, WarpScratch& sc) {
    for (int k = T.nA + lane; k < T.nA_pad; k += 32) { S.apple[(size_t)b * T.nA_pad + k] = 0; S.apple_count[(size_t)b * T.nA_pad + k] = 0; }
    reset(T, F, S, b, lane, sc);
  }

  template <class Actions>
  __device__ static void step(const Tables& T, const Params& F, const State& S, int b, int lane, const Actions& actions, WarpScratch& sc) {
    const auto [env, grid, k0, k1, n, episode] = begin_frame(T, S, b, false);
    const bool is_av = lane < T.P;
    uint8_t* s_state = sc.apple;  // [nA_pad] bits 0-4 state code, bit 5 sprouts, bit 6 eaten
    uint8_t* s_count = sc.dirt;   // [nA_pad]
    int16_t* s_events = sc.tmp;   // eaten-apple queue (round 2), in event order

    int4 a, t, act;
    load_avatar(T, S, b, lane, actions, T.action_table, a, t, act);
    int x = a.x, y = a.y, orient = a.z, alive = a.w, zap_cool = t.x, state_frame = t.z;
    const int act_move = act.x, act_turn = act.y, act_zap = act.z;
    const int x0 = x, y0 = y, orient0 = orient, alive0 = alive;
    double reward = 0.0;

    init_occupancy(T, sc.occ, T.solid, lane);
    for (int k = lane; k < T.nA; k += 32) { s_state[k] = S.apple[(size_t)b * T.nA_pad + k]; s_count[k] = S.apple_count[(size_t)b * T.nA_pad + k]; }
    const int words = (T.cells + 31) / 32 + 1;
    for (int i = lane; i < words; i += 32) sc.beam_zap[i] = 0;
    __syncwarp();
    if (is_av && alive) sc.occ[y * T.W + x] = (uint8_t)(lane + 1);
    if (env[ENV_BEAM]) clear_layer(T, grid, F.zap.layer, lane);
    __syncwarp();
    int beam_dirty = 0;

    // ---- simulation:update: DensityRegrow:update -> _updateWaitState (components.lua:147-193) ------
    // and the priority-10 sprout updaters (:92-123), evaluated on the state the apple has NOW.
    for (int k = lane; k < T.nA; k += 32) {
      const uint8_t st = s_state[k];
      if (!ch_is_wait(st)) continue;
      if (st >= 2) {  // in some appleWait_j: its updater fires with probability probs[min(j, n-1)]
        const int j = st - 2;
        const double p = F.ch_probs[j < F.ch_n_probs ? j : F.ch_n_probs - 1];
        if (p > 0.0) {
          uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)F.ch_apple[k * 4], RS_OBJECT, k0, k1);
          if (u01(w.x, w.y) < p) s_state[k] |= 32;
        }
      }
      // relabel to appleWait_count and toggle the grass below (processed first in the queue)
      int c = s_count[k]; if (c >= F.ch_n_wait) c = F.ch_n_wait - 1;
      s_state[k] = (s_state[k] & 32) | (uint8_t)(2 + c);
      const int cell = F.ch_apple[k * 4 + 1];
      if (F.ch_apple[k * 4 + 3] >= 0)
        grid[(size_t)F.grass_layer * T.cells_pad + cell] = cell_value(c == 0 ? F.dess_sprite : F.grass_sprite, 0);
    }
    __syncwarp();

    // ---- updaters ------------------------------------------------------------------------------------
    const int rank = visit_rank(T, lane, n, episode, k0, k1);
    bool fire_zap = false;
    if (is_av && alive) { if (zap_cool > 0) --zap_cool; else if (act_zap == 1) { zap_cool = F.zap.cooldown; fire_zap = true; } }
    const bool want_respawn = is_av && !alive && (n - state_frame) >= F.zap.respawn;
    const bool cont = episode_continues(T, n, episode, k0, k1);

    // ---- round 1 ---------------------------------------------------------------------------------------
    int n_events = 0;  // uniform across the warp
    // Edible:onEnter of an avatar arriving on `cell` with a live apple (component_library.lua:990-1002); a second
    // setState(appleWait) of the same apple would be a no-op, so the queue holds each apple once.
    const auto eat = [&](int src, int cell) {
      const int ai = F.apple_of_cell[cell];
      const bool ate = ai >= 0 && (s_state[ai] & 31) == 0;
      const bool fresh = ate && !(s_state[ai] & 64);
      __syncwarp();
      if (fresh) {
        if (lane == 0) { s_state[ai] |= 64; s_events[n_events] = (int16_t)ai; }
        ++n_events;
      }
      if (ate && lane == src) { reward += F.eat_reward; emit_event(S, b, EV_EDIBLE_CONSUMED, src + 1, 0); }
    };
    move_avatars(T, lane, rank, is_av && alive, act_turn, act_move, x, y, orient, sc.occ, eat);
    // zap beams
    unsigned zapped = 0;
    for (int r = 0; r < T.P; ++r) {
      unsigned m = __ballot_sync(MP_FULL, is_av && rank == r && fire_zap);
      if (!m) continue;
      int src = __ffs(m) - 1;
      int sx = __shfl_sync(MP_FULL, x, src), sy = __shfl_sync(MP_FULL, y, src), so = __shfl_sync(MP_FULL, orient, src);
      const BeamGeom& G = F.zap.geom;
      const int cell = beam_cell(T, G, lane, sx, sy, so);
      int hit_avatar = -1;
    bool blocked = cell < 0 && lane < G.n;  // off the map
      if (cell >= 0) {
        if (T.cell_flags[cell] & (1 << F.zap.hit)) blocked = true;
        int o = sc.occ[cell];
        if (o >= 1 && o <= T.P && o - 1 != src) { hit_avatar = o - 1; blocked = true; }
      }
      bool vis;
      beam_scan(G, lane, blocked, vis);
      unsigned hm = __ballot_sync(MP_FULL, vis && hit_avatar >= 0);
      while (hm) {
        int c = __ffs(hm) - 1; hm &= hm - 1;
        int t = __shfl_sync(MP_FULL, hit_avatar, c);
        if (lane == t) reward += F.zap.penalty;
        if (lane == src) { reward += F.zap.reward; emit_event(S, b, EV_ZAP, src + 1, t + 1); }
        if (F.zap.remove) zapped |= 1u << t;
      }
      if (vis && !blocked) { draw_hit_sprite(T, grid, sc.beam_zap, F.zap.layer, cell, cell_value(F.zap.sprite, so)); beam_dirty = 1; }
      __syncwarp();
    }
    beam_dirty = __any_sync(MP_FULL, beam_dirty);
    // respawns (teleportToGroup to the post-initial spawn group)
    respawn_avatars(T, lane, rank, want_respawn, n, episode, k0, k1, sc.occ, x, y, orient, alive, state_frame, eat);
    // sprouts, in object order: setState(live) -> _beginLive (components.lua:206-219) -> contact.
    for (int base = 0; base < T.nA; base += 32) {
      int k = base + lane;
      unsigned sm = __ballot_sync(MP_FULL, k < T.nA && (s_state[k] & 32));
      while (sm) {
        const int i = base + __ffs(sm) - 1; sm &= sm - 1;
        __syncwarp();
        if (lane == 0) s_state[i] = 0;  // live
        __syncwarp();
        if (lane < 16) {  // every wait neighbour inside the disc gains one
          const int j = F.ch_nbr[i * 16 + lane];
          if (j >= 0 && ch_is_wait(s_state[j] & 31)) s_count[j] += 1;
        }
        const int cell = F.ch_apple[i * 4 + 1];
        const int o = sc.occ[cell];
        if (o >= 1 && o <= T.P) {  // an avatar stands here: eaten at once
          if (lane == o - 1) { reward += F.eat_reward; emit_event(S, b, EV_EDIBLE_CONSUMED, o, 0); }
          __syncwarp();
          if (lane == 0) { s_state[i] |= 64; s_events[n_events] = (int16_t)i; }
          ++n_events;
        }
        __syncwarp();
      }
    }

    // ---- round 2: setState(appleWait) of eaten apples -> _endLive (components.lua:221-240) ----------
    for (int e = 0; e < n_events; ++e) {
      const int i = s_events[e];
      __syncwarp();
      if (lane == 0) s_state[i] = 1;  // plain 'appleWait' (layer logic)
      __syncwarp();
      int live = 0;
      if (lane < 16) {
        const int j = F.ch_nbr[i * 16 + lane];
        if (j >= 0) {
          if (ch_is_wait(s_state[j] & 31)) s_count[j] -= 1; else live = 1;
        }
      }
      const unsigned lm = __ballot_sync(MP_FULL, live);
      if (lane == 0) s_count[i] = (uint8_t)__popc(lm);  // liveNeighbors inside the disc (self is no longer live)
      __syncwarp();
    }
    if (is_av && (zapped >> lane & 1u)) { alive = 0; state_frame = n; }

    // ---- write back -----------------------------------------------------------------------------------
    for (int k = lane; k < T.nA; k += 32) {
      const uint8_t now = s_state[k] & 31;
      const uint8_t was = S.apple[(size_t)b * T.nA_pad + k];
      if (now != was) {
        S.apple[(size_t)b * T.nA_pad + k] = now;
        const int cell = F.ch_apple[k * 4 + 1];
        if ((now == 0) != (was == 0)) {  // moved between lowerPhysical and logic
          grid[(size_t)F.apple_layer * T.cells_pad + cell] = now == 0 ? cell_value(F.apple_sprite, 0) : (uint16_t)0;
          grid[(size_t)F.wait_layer * T.cells_pad + cell] = now == 0 ? (uint16_t)0 : cell_value(F.wait_sprite, 0);
        }
      }
      S.apple_count[(size_t)b * T.nA_pad + k] = s_count[k];
    }
    draw_avatars(T, grid, lane, x0, y0, orient0, alive0, x, y, orient, alive);

    const bool done = !cont || n >= T.max_frames;
    if (is_av) {
      *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(x, y, orient, alive);
      *reinterpret_cast<int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4) = make_int4(zap_cool, 0, state_frame, 0);
      for (int k = 0; k < T.n_scalar; ++k)
        S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = alive ? fmax(1.0 - (double)zap_cool / (double)F.zap.cooldown, 0.0) : 0.0;
    }
    store_timestep(T, S, b, lane, n, reward, done ? 2 : 1, beam_dirty);
  }
};
