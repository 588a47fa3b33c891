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

#include "family_load.h"
#include "step_common.cuh"

struct CleanUp {
  struct Params {
    Zapper zap;
    int apple_layer, apple_sprite, dirt_layer, dirt_sprite, water_layer, n_anim, anim_frames, anim_random;
    int water_sprite[8];
    int clean_cooldown, clean_layer, clean_sprite, clean_hit;
    BeamGeom clean_geom;
    int dirt_delay, dirt_count0;
    double grow_rate, grow_depletion, grow_restoration, eat_reward, dirt_prob;
    const int32_t* apple;          // [nA][3] obj id, cell, initially live
    const int32_t* dirt;           // [nD][3] obj id, cell, initially dirty
    const int32_t* water;          // [nW][2] obj id, cell
    const int16_t* apple_of_cell;  // [cells_pad] apple index or -1
    const int16_t* dirt_of_cell;   // [cells_pad] dirt index or -1
  };

  // Host: the clean_up tables of the blob (compiler.py _clean_up_tables): cu_ip / cu_dp, apples, dirt and water.
  static int load(FamilyLoad& ld, const Tables& T, Params& F) {
    const int32_t* ip;
    const double* dp;
    Section<int32_t> apple, dirt, water, water_sprites;
    int rc;
    if ((rc = ld.params("cu", MPB_CU_I_COUNT, MPB_CU_D_COUNT, &ip, &dp)) || (rc = ld.need("cu_apple", MPB_I32, &apple)) ||
        (rc = ld.need("cu_dirt", MPB_I32, &dirt)) || (rc = ld.need("cu_water", MPB_I32, &water)) ||
        (rc = ld.need("cu_water_sprites", MPB_I32, &water_sprites)))
      return rc;
    ld.nA = ip[MPB_CU_I_N_APPLES]; ld.nD = ip[MPB_CU_I_N_DIRT]; ld.nW = ip[MPB_CU_I_N_WATER];
    F.apple_layer = ip[MPB_CU_I_APPLE_LAYER]; F.apple_sprite = ip[MPB_CU_I_APPLE_SPRITE];
    F.dirt_layer = ip[MPB_CU_I_DIRT_LAYER]; F.dirt_sprite = ip[MPB_CU_I_DIRT_SPRITE];
    F.water_layer = ip[MPB_CU_I_WATER_LAYER]; F.n_anim = ip[MPB_CU_I_N_ANIM];
    F.anim_frames = ip[MPB_CU_I_ANIM_FRAMES]; F.anim_random = ip[MPB_CU_I_ANIM_RANDOM];
    if (F.n_anim < 1 || F.n_anim > 8 || F.anim_frames < 1) return fail(MP_E_UNSUPPORTED, "animation with %d states / %d frames", F.n_anim, F.anim_frames);
    for (int i = 0; i < F.n_anim; ++i) F.water_sprite[i] = water_sprites.data[i];
    if ((rc = load_zapper(ld, T, ip, dp[MPB_CU_D_ZAP_PENALTY], dp[MPB_CU_D_ZAP_REWARD], F.zap))) return rc;
    F.clean_cooldown = ip[MPB_CU_I_CLEAN_COOLDOWN]; F.clean_layer = ip[MPB_CU_I_CLEAN_LAYER]; F.clean_sprite = ip[MPB_CU_I_CLEAN_SPRITE];
    F.clean_hit = 1;
    for (int h = 0; h < (int)ld.hits.count / 2; ++h) if (ld.hits.data[h * 2] == F.clean_layer) F.clean_hit = h;
    const int length = ip[MPB_CU_I_CLEAN_LENGTH], radius = ip[MPB_CU_I_CLEAN_RADIUS];
    if (F.clean_cooldown < 0) return fail(MP_E_UNSUPPORTED, "negative clean cooldown");
    if (!make_beam_geom(length, radius, &F.clean_geom)) return fail(MP_E_UNSUPPORTED, "beam footprint larger than %d cells", MP_MAX_BEAM_CELLS);
    if (!beam_fits_torus(T, length, radius)) return fail(MP_E_UNSUPPORTED, "clean beam (length %d, radius %d) does not fit the %dx%d TORUS map", length, radius, T.W, T.H);
    ld.beam_cells = F.zap.geom.n + F.clean_geom.n;
    F.dirt_delay = ip[MPB_CU_I_DIRT_DELAY];
    if (ip[MPB_CU_I_TASTE_ROLE] != 0) return fail(MP_E_UNSUPPORTED, "Taste roles other than 'free'");
    F.grow_rate = dp[MPB_CU_D_GROW_RATE]; F.grow_depletion = dp[MPB_CU_D_GROW_DEPLETION];
    F.grow_restoration = dp[MPB_CU_D_GROW_RESTORATION]; F.eat_reward = dp[MPB_CU_D_EAT_REWARD];
    F.dirt_prob = dp[MPB_CU_D_DIRT_PROB]; ld.end_prob = dp[MPB_CU_D_END_PROB];
    std::vector<int32_t> v_apple(apple.data, apple.data + apple.count), v_dirt(dirt.data, dirt.data + dirt.count);
    std::vector<int32_t> v_water(water.data, water.data + water.count);
    ld.table(&F.apple, v_apple); ld.table(&F.dirt, v_dirt); ld.table(&F.water, v_water);
    if ((rc = cell_index(ld, T, "cu_apple", apple, ld.nA, 3, &F.apple_of_cell)) || (rc = cell_index(ld, T, "cu_dirt", dirt, ld.nD, 3, &F.dirt_of_cell)))
      return rc;
    F.dirt_count0 = 0;
    for (int j = 0; j < ld.nD; ++j) F.dirt_count0 += v_dirt[j * 3 + 2];
    return MP_OK;
  }

  // Host: per-env variants may differ in the Zapper and Cleaner cooldowns and rewards, DirtSpawner, AppleGrow, Edible
  // and the water Animation's timing, and in the apple, dirt and water sprites (appearance overrides); layers, beam hit
  // sprites, hits, beam footprints and the number of animation states agree.
  static int same_shape(const Params& a, const Params& b) {
    MP_SAME_ZAPPER MP_SAME(apple_layer) MP_SAME(dirt_layer) MP_SAME(water_layer) MP_SAME(n_anim)
    MP_SAME(clean_layer) MP_SAME(clean_sprite) MP_SAME(clean_hit) MP_SAME(clean_geom) MP_SAME(dirt_count0)
    return MP_OK;
  }

  using Scratch = WarpScratch;
  static constexpr bool kMapVariants = false;
  static constexpr const char* const* kMapSections = nullptr;
  // Its tables that hold only sprite ids: variants of one set (appearance overrides) may differ there (mp_create_variants).
  static constexpr const char* kSpriteSections[] = {"cu_water_sprites", nullptr};
  static constexpr bool kStagesTables = true;
  __host__ __device__ static size_t scratch_bytes(const Tables& T) { return warp_scratch_bytes(T); }
  __host__ __device__ static size_t table_bytes(const Tables& T) { return scratch_round16((size_t)T.cells_pad * 6) + (size_t)T.n_actions * 16 + 2 * sizeof(BeamGeom); }

  // Per-CTA tables: apple_of and dirt_of (int16), solid and flags (8-byte aligned: cells_pad is a multiple of 8), the
  // action table, then the zap and clean beam footprints. Each lane reads its own footprint cell; read from the kernel
  // parameters instead, the two footprints cost this kernel 24 B more stack and 32 / 48 B more spill stores / loads.
  __device__ static void stage(const Tables& T, const Params& F, uint8_t* tb) {
    int16_t* s_apple_of = reinterpret_cast<int16_t*>(tb);
    int16_t* s_dirt_of = s_apple_of + T.cells_pad;
    uint8_t* s_solid = reinterpret_cast<uint8_t*>(s_dirt_of + T.cells_pad);
    uint8_t* s_flags = s_solid + T.cells_pad;
    int32_t* s_act = reinterpret_cast<int32_t*>(tb + scratch_round16((size_t)T.cells_pad * 6));
    for (int i = threadIdx.x; i < T.cells_pad; i += (int)blockDim.x) { s_apple_of[i] = F.apple_of_cell[i]; s_dirt_of[i] = F.dirt_of_cell[i]; s_flags[i] = T.cell_flags[i]; s_solid[i] = T.solid[i]; }
    for (int i = threadIdx.x; i < T.n_actions * 4; i += (int)blockDim.x) s_act[i] = T.action_table[i];
    BeamGeom* s_beams = reinterpret_cast<BeamGeom*>(s_act + T.n_actions * 4);
    if (threadIdx.x == 0) { s_beams[0] = F.zap.geom; s_beams[1] = F.clean_geom; }
  }

  __device__ static WarpScratch carve(const Tables& T, uint8_t* base, const uint8_t* tb) {
    WarpScratch sc = carve_scratch(T, base);
    sc.apple_of = reinterpret_cast<const int16_t*>(tb);
    sc.dirt_of = sc.apple_of + T.cells_pad;
    sc.solid = reinterpret_cast<const uint8_t*>(sc.dirt_of + T.cells_pad);
    sc.flags = sc.solid + T.cells_pad;
    sc.act_table = reinterpret_cast<const int32_t*>(tb + scratch_round16((size_t)T.cells_pad * 6));
    return sc;
  }
  // The zap and clean beam footprints, right after the action table (found from act_table: one more pointer in the
  // scratch struct spills as well).
  __device__ static const BeamGeom* beams(const Tables& T, const WarpScratch& sc) { return reinterpret_cast<const BeamGeom*>(sc.act_table + T.n_actions * 4); }

  __device__ static void reset(const Tables& T, const Params& F, const State& S, int b, int lane, WarpScratch& sc) {
    const auto [env, grid, k0, k1, n, episode] = begin_frame(T, S, b, true);
    __syncwarp();
    copy_init_grid(T, grid, lane);
    for (int k = lane; k < T.nA; k += 32) S.apple[(size_t)b * T.nA_pad + k] = (uint8_t)F.apple[k * 3 + 2];
    for (int j = lane; j < T.nD; j += 32) S.dirt[(size_t)b * T.nD_pad + j] = (uint8_t)F.dirt[j * 3 + 2];
    __syncwarp();
    // Animation:postStart random start frame (component_library.lua:1064-1068).
    for (int k = lane; k < T.nW; k += 32) {
      int phase = 0;
      if (F.anim_random) {
        uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)F.water[k * 2], RS_OBJECT_RESET, k0, k1);
        phase = (int)pick(w.x, (uint32_t)F.n_anim);
      }
      S.water[(size_t)b * T.nW_pad + k] = (uint8_t)phase;
      grid[(size_t)F.water_layer * T.cells_pad + F.water[k * 2 + 1]] = cell_value(F.water_sprite[phase], 0);
    }
    const auto all = [](int) { return true; };
    spawn_group(T, S, b, lane, grid, sc.tmp, T.spawn_cell, T.n_spawn, all, all, episode, k0, k1, [&](int) {
      for (int k = 0; k < T.n_scalar; ++k) S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = T.scalar_obs[k] == 0 ? 1.0 : 0.0;
    });
    reset_env_row(T, S, b, lane, episode, F.dirt_count0);
  }

  template <class Actions>
  __device__ static void step(const Tables& T, const Params& F, const State& S, int b, int lane, const Actions& actions, WarpScratch& sc) {
    const auto [env, grid, k0, k1, n, episode] = begin_frame(T, S, b, false);
    int dirt_count = env[ENV_DIRT];
    const unsigned cleaned_prev = (unsigned)env[ENV_CLEANED];
    unsigned cleaned_now = 0, ate_now = 0;
    const bool is_av = lane < T.P;

    // ---- load ---------------------------------------------------------------------------------
    int4 a, t, act;
    load_avatar(T, S, b, lane, actions, sc.act_table, a, t, act);
    int x = a.x, y = a.y, orient = a.z, alive = a.w, zap_cool = t.x, clean_cool = t.y, state_frame = t.z;
    const int act_move = act.x, act_turn = act.y, act_zap = act.z, act_clean = act.w;
    const int x0 = x, y0 = y, orient0 = orient, alive0 = alive;
    double reward = 0.0;  // Avatar:preUpdate (avatar_library.lua:330-332)

    init_occupancy(T, sc.occ, sc.solid, lane);
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
    if (env[ENV_BEAM]) { clear_layer(T, grid, F.zap.layer, lane); clear_layer(T, grid, F.clean_layer, lane); }
    __syncwarp();
    int beam_dirty = 0;

    // ---- simulation:update --------------------------------------------------------------------
    // DirtSpawner:update (clean_up/components.lua:329-340); its _timeStep equals n here.
    int spawn_dirt = -1;
    if (n > F.dirt_delay) {
      uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, SCENE_DRAW_DIRT, RS_SCENE, k0, k1);
      int n_inactive = T.nD - dirt_count;
      if (u01(w.x, w.y) < F.dirt_prob && n_inactive > 0) {
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
      double interpolation = (fraction - F.grow_depletion) / (F.grow_restoration - F.grow_depletion);
      interpolation = 1.0 < interpolation ? 1.0 : interpolation;  // Lua 5.1 math.min: a NaN (0/0) stays NaN, no growth (policy A.22)
      const double probability = F.grow_rate * interpolation;
      if (probability > 0.0) {  // u >= 0 can never be below a non-positive (or NaN) probability
        for (int k = lane; k < T.nA; k += 32) {
          uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)F.apple[k * 3], RS_OBJECT, k0, k1);
          if (u01(w.x, w.y) < probability && !(sc.apple[k] & 1)) sc.apple[k] |= 4;  // grows this frame
        }
      }
    }
    __syncwarp();

    // ---- updaters (priority order) ------------------------------------------------------------
    // Avatars are visited in a fresh random order each frame (policy A.7).
    const int rank = visit_rank(T, lane, n, episode, k0, k1);
    // 150 Avatar move (avatar_library.lua:156-171): intents are act_turn / act_move.
    // 140 Zapper zap (:613-631) and Cleaner clean (clean_up/components.lua:201-219).
    bool fire_zap = false, fire_clean = false;
    if (is_av && alive) {
      if (zap_cool > 0) --zap_cool; else if (act_zap == 1) { zap_cool = F.zap.cooldown; fire_zap = true; }
      if (clean_cool > 0) --clean_cool; else if (act_clean == 1) { clean_cool = F.clean_cooldown; fire_clean = true; }
    }
    // 135 Zapper respawn (:638-649): state = waitState, startFrame = framesTillRespawn.
    const bool want_respawn = is_av && !alive && (n - state_frame) >= F.zap.respawn;
    // 100 StochasticIntervalEpisodeEnding
    const bool cont = episode_continues(T, n, episode, k0, k1);
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
        int o = sc.occ[F.apple[k * 3 + 1]];
        if (o >= 1 && o <= T.P) { eater = o - 1; sc.apple[k] |= 2; }
      }
      unsigned m = __ballot_sync(MP_FULL, eater >= 0);
      while (m) {  // in apple (object) order
        int src = __ffs(m) - 1; m &= m - 1;
        int e = __shfl_sync(MP_FULL, eater, src);
        if (lane == e) { reward += F.eat_reward; emit_event(S, b, EV_EDIBLE_CONSUMED, e + 1, 0); }
        ate_now |= 1u << e;
      }
    }
    __syncwarp();
    // Edible:onEnter of an avatar arriving on `cell` (by a move, even a blocked one, or by a respawn).
    const auto eat = [&](int src, int cell) {
      const int ai = sc.apple_of[cell];
      const bool ate = ai >= 0 && (sc.apple[ai] & 1);
      __syncwarp();
      if (ate && lane == 0) sc.apple[ai] |= 2;
      if (ate && lane == src) { reward += F.eat_reward; emit_event(S, b, EV_EDIBLE_CONSUMED, src + 1, 0); }
      if (ate) ate_now |= 1u << src;
    };
    // (c) turns and moves, avatar by avatar in this frame's order.
    move_avatars(T, lane, rank, is_av && alive, act_turn, act_move, x, y, orient, sc.occ, eat);
    // (d) zap beams, then (e) clean beams, shooter by shooter.
    unsigned zapped = 0;
    for (int pass = 0; pass < 2; ++pass) {
      const BeamGeom& G = beams(T, sc)[pass];
      for (int r = 0; r < T.P; ++r) {
        unsigned m = __ballot_sync(MP_FULL, is_av && rank == r && (pass == 0 ? fire_zap : fire_clean));
        if (!m) continue;
        int src = __ffs(m) - 1;
        int sx = __shfl_sync(MP_FULL, x, src), sy = __shfl_sync(MP_FULL, y, src), so = __shfl_sync(MP_FULL, orient, src);
        const int cell = beam_cell(T, G, lane, sx, sy, so);
        int hit_avatar = -1, hit_dirt = -1;
      bool blocked = cell < 0 && lane < G.n;  // off the map
        if (cell >= 0) {
          int hit = pass == 0 ? F.zap.hit : F.clean_hit;
          if (sc.flags[cell] & (1 << hit)) blocked = true;  // BeamBlocker:onHit
          if (pass == 0) {
            int o = sc.occ[cell];
            if (o >= 1 && o <= T.P && o - 1 != src) { hit_avatar = o - 1; blocked = true; }  // Zapper:onHit
          } else {
            int dj = sc.dirt_of[cell];
            if (dj >= 0 && (sc.dirt[dj] & 1)) { hit_dirt = dj; blocked = true; }  // DirtCleaning:onHit
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
            if (lane == t) reward += F.zap.penalty;   // zapped avatar is still alive in this round
            if (lane == src) { reward += F.zap.reward; emit_event(S, b, EV_ZAP, src + 1, t + 1); }
            if (F.zap.remove) zapped |= 1u << t;
          }
        } else {
          bool cleaned = vis && hit_dirt >= 0;
          if (cleaned) { sc.dirt[hit_dirt] |= 2; emit_event(S, b, EV_PLAYER_CLEANED, src + 1, 0); }
          if (__any_sync(MP_FULL, cleaned)) cleaned_now |= 1u << src;  // Cleaner:setCumulant
        }
        if (vis && !blocked) {
          draw_hit_sprite(T, grid, pass == 0 ? sc.beam_zap : sc.beam_2, pass == 0 ? F.zap.layer : F.clean_layer, cell,
                          cell_value(pass == 0 ? F.zap.sprite : F.clean_sprite, so));
          beam_dirty = 1;
        }
        __syncwarp();
      }
    }
    beam_dirty = __any_sync(MP_FULL, beam_dirty);
    // (f) teleportToGroup for respawning avatars.
    respawn_avatars(T, lane, rank, want_respawn, n, episode, k0, k1, sc.occ, x, y, orient, alive, state_frame, eat);

    // ---- round 2: the setStates queued by callbacks --------------------------------------------
    if (is_av && (zapped >> lane & 1u)) { alive = 0; state_frame = n; }
    for (int k = lane; k < T.nA; k += 32) {
      uint8_t v = sc.apple[k];
      uint8_t was = (v >> 3) & 1;
      uint8_t now = (v & 1) && !(v & 2);
      if (now != was) {
        S.apple[(size_t)b * T.nA_pad + k] = now;
        grid[(size_t)F.apple_layer * T.cells_pad + F.apple[k * 3 + 1]] = now ? cell_value(F.apple_sprite, 0) : (uint16_t)0;
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
        grid[(size_t)F.dirt_layer * T.cells_pad + F.dirt[j * 3 + 1]] = now ? cell_value(F.dirt_sprite, 0) : (uint16_t)0;
      }
    }
    for (int o = 16; o > 0; o >>= 1) d_delta += __shfl_xor_sync(MP_FULL, d_delta, o);
    dirt_count += d_delta;
    // water Animation (component_library.lua:1070-1094): every piece flips every anim_frames frames.
    if (n % F.anim_frames == 0) {
      const int turn = (n / F.anim_frames) % F.n_anim;  // (uniform: the divisions are done once, not per piece)
      for (int k = lane; k < T.nW; k += 32) {
        int phase = (int)S.water[(size_t)b * T.nW_pad + k] + turn;
        if (phase >= F.n_anim) phase -= F.n_anim;
        grid[(size_t)F.water_layer * T.cells_pad + F.water[k * 2 + 1]] = cell_value(F.water_sprite[phase], 0);
      }
    }
    draw_avatars(T, grid, lane, x0, y0, orient0, alive0, x, y, orient, alive);

    // ---- store ---------------------------------------------------------------------------------
    const bool done = !cont || n >= T.max_frames;
    if (is_av) {
      *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(x, y, orient, alive);
      *reinterpret_cast<int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4) = make_int4(zap_cool, clean_cool, state_frame, 0);
      for (int k = 0; k < T.n_scalar; ++k) {
        double v;
        if (T.scalar_obs[k] == 0)  // Zapper:readyToShoot (avatar_library.lua:737-744)
          v = alive ? fmax(1.0 - (double)zap_cool / (double)F.zap.cooldown, 0.0) : 0.0;
        else
          v = (double)num_others_cleaned;
        S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = v;
      }
    }
    if (lane == 0) { env[ENV_DIRT] = dirt_count; env[ENV_CLEANED] = (int)cleaned_now; env[ENV_ATE] = (int)ate_now; }
    store_timestep(T, S, b, lane, n, reward, done ? 2 : 1, beam_dirty);
  }
};
