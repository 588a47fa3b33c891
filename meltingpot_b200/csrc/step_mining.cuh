// step_mining.cuh -- state transition of the coop_mining family, one warp per env instance.
//
// Restates one frame of api:advance (api_factory.lua:104-111) for the components of
//   meltingpot/lua/levels/coop_mining/components.lua
//     FixedRateRegrow :25-58, Ore :60-157, MineBeam :160-262
//   meltingpot/lua/modules/avatar_library.lua (Avatar movement)
//   meltingpot/lua/modules/component_library.lua:900-950 (StochasticIntervalEpisodeEnding)
// in the closed form of the other families. Ore state codes (State.apple): 0 'oreWait', 1 the
// single-miner ore ('ironRaw'), 2 the two-miner ore ('goldRaw'), 3 its partial state
// ('goldPartial'). State.dirt holds the two-miner Ore component's _miners as a bit per player and
// State.apple_count its _miningCountdown while positive (the single-miner component never keeps
// either beyond a hit). Avatars never leave the map; there is no zapping.
//
// Order inside a frame (DESIGN.md policies A.2-A.8): the component updates run first -- Ore:update
// (count-down, possibly a reset) and MineBeam:update, which fires the beam into the action queue --
// then the updaters queue the regrowth (priority 200), the moves (150) and the episode check (100).
// The queue is drained in that order: beams in avatar (object) order against the ore states the
// frame started with, the resets and the regrowth, the moves; the state changes the hits asked for
// land in the next round.
#pragma once

#include "family_load.h"
#include "step_common.cuh"

struct Mining {
  struct Params {
    int ore_layer;
    int ore_sprite[4];            // wait, single-miner raw, two-miner raw, two-miner partial
    int mine_window;              // frames a partly mined two-miner ore waits for its second miner
    int mine_cooldown, mine_length, mine_layer, mine_sprite, mine_hit;  // MineBeam
    double mine_rate[2];          // FixedRateRegrow liveRates
    double mine_reward[2], extract_reward[2];  // per ore type (1 miner, 2 miners)
    const int32_t* ore;           // [nA][2] obj id, cell
    const int16_t* ore_of_cell;   // [cells_pad] ore index or -1
  };

  // Host: the coop_mining tables of the blob (compiler.py _mining_tables): cm_ip / cm_dp and the ores.
  static int load(FamilyLoad& ld, const Tables& T, Params& F) {
    const int32_t* ip;
    const double* dp;
    Section<int32_t> ore;
    int rc;
    if ((rc = ld.params("cm", MPB_CM_I_COUNT, MPB_CM_D_COUNT, &ip, &dp)) || (rc = ld.need("cm_ore", MPB_I32, &ore))) return rc;
    ld.nA = ip[MPB_CM_I_N_ORES]; F.ore_layer = ip[MPB_CM_I_ORE_LAYER];
    for (int i = 0; i < 4; ++i) F.ore_sprite[i] = ip[MPB_CM_I_ORE_SPRITE_0 + i];
    F.mine_window = ip[MPB_CM_I_MINE_WINDOW]; F.mine_cooldown = ip[MPB_CM_I_MINE_COOLDOWN]; F.mine_length = ip[MPB_CM_I_MINE_LENGTH];
    F.mine_layer = ip[MPB_CM_I_MINE_LAYER]; F.mine_sprite = ip[MPB_CM_I_MINE_SPRITE];
    ld.end_min_frames = ip[MPB_CM_I_END_MIN_FRAMES]; ld.end_interval = ip[MPB_CM_I_END_INTERVAL]; F.mine_hit = ip[MPB_CM_I_MINE_HIT];
    if (T.P > 8) return fail(MP_E_UNSUPPORTED, "coop_mining with %d players (max 8: miners are kept as a bit mask)", T.P);
    if (ld.nA > 2048) return fail(MP_E_UNSUPPORTED, "%d ores (max 2048)", ld.nA);
    if (F.mine_cooldown < 1 || F.mine_window < 1 || F.mine_window > 255 || F.mine_length < 1) return fail(MP_E_UNSUPPORTED, "MineBeam / Ore parameters out of range");
    if (ld.end_interval < 1) return fail(MP_E_INVALID, "episode interval < 1");
    if (F.mine_hit < 0 || F.mine_hit > 7) return fail(MP_E_UNSUPPORTED, "mine hit id %d", F.mine_hit);
    if (!beam_fits_torus(T, F.mine_length, 0)) return fail(MP_E_UNSUPPORTED, "mine beam (length %d) does not fit the %dx%d TORUS map", F.mine_length, T.W, T.H);
    F.mine_rate[0] = dp[MPB_CM_D_RATE_0]; F.mine_rate[1] = dp[MPB_CM_D_RATE_1]; ld.end_prob = dp[MPB_CM_D_END_PROB];
    F.mine_reward[0] = dp[MPB_CM_D_MINE_REWARD_0]; F.mine_reward[1] = dp[MPB_CM_D_MINE_REWARD_1];
    F.extract_reward[0] = dp[MPB_CM_D_EXTRACT_REWARD_0]; F.extract_reward[1] = dp[MPB_CM_D_EXTRACT_REWARD_1];
    std::vector<int32_t> v_ore(ore.data, ore.data + ore.count);
    ld.table(&F.ore, v_ore);
    return cell_index(ld, T, "cm_ore", ore, ld.nA, 2, &F.ore_of_cell);
  }

  // Host: per-env variants may differ in the mining window, the mine cooldown, the regrowth rates, the rewards and the
  // ore sprites (appearance overrides).
  static int same_shape(const Params& a, const Params& b) {
    MP_SAME(ore_layer) MP_SAME(mine_length) MP_SAME(mine_layer) MP_SAME(mine_sprite) MP_SAME(mine_hit)
    return MP_OK;
  }

  using Scratch = WarpScratch;
  // Maps of one set may differ in their walls, ores and spawn points: the ore table is their entity table, and the ore
  // count is the nA of each variant's Tables (setup_variants).
  static constexpr bool kMapVariants = true;
  static constexpr const char* kMapSections[] = {"cm_ore", nullptr};
  static constexpr const char* const* kSpriteSections = nullptr;
  static constexpr bool kStagesTables = false;
  __host__ __device__ static size_t scratch_bytes(const Tables& T) { return warp_scratch_bytes(T); }
  __host__ __device__ static size_t table_bytes(const Tables&) { return 0; }
  __device__ static void stage(const Tables&, const Params&, uint8_t*) {}
  __device__ static WarpScratch carve(const Tables& T, uint8_t* base, const uint8_t*) { return carve_scratch(T, base); }

  // Episode start: the avatars draw their spawn points (policy A.10); MineBeam:start (:254-261) leaves them ready to shoot.
  __device__ static void reset(const Tables& T, const Params& F, const State& S, int b, int lane, WarpScratch& sc) {
    const auto [env, grid, k0, k1, n, episode] = begin_frame(T, S, b, true);
    __syncwarp();
    copy_init_grid(T, grid, lane);
    for (int k = lane; k < T.nA; k += 32) {  // Ore:reset (:96-103): every ore waits, nobody is mining
      S.apple[(size_t)b * T.nA_pad + k] = 0;
      S.dirt[(size_t)b * T.nD_pad + k] = 0;
      S.apple_count[(size_t)b * T.nA_pad + k] = 0;
    }
    __syncwarp();
    const auto all = [](int) { return true; };
    spawn_group(T, S, b, lane, grid, sc.tmp, T.spawn_init_cell[0], T.n_spawn_init[0], all, all, episode, k0, k1, [&](int) {
      for (int k = 0; k < T.n_scalar; ++k) S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = T.scalar_obs[k] == 0 ? 1.0 : 0.0;
    });
    // api:start ends with one grid:update (api_factory.lua:101): the FixedRateRegrow updaters already fire at frame 0
    // (the component updates do not run then). Spawn points are not ore cells; the avatar check is kept for symmetry.
    for (int k = lane; k < T.nA; k += 32) {
      uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)F.ore[k * 2], RS_OBJECT, k0, k1);
      const bool first = u01(w.x, w.y) < F.mine_rate[0], second = u01(w.z, w.w) < F.mine_rate[1];
      const int cell = F.ore[k * 2 + 1];
      if ((first || second) && grid[(size_t)T.avatar_layer * T.cells_pad + cell] == 0) {
        const int now = second ? 2 : 1;
        S.apple[(size_t)b * T.nA_pad + k] = (uint8_t)now;
        grid[(size_t)F.ore_layer * T.cells_pad + cell] = cell_value(F.ore_sprite[now], 0);
      }
    }
    reset_env_row(T, S, b, lane, episode, 0);
  }

  // Episode start of an env of a map-variant engine: also zeroes the env's ore bytes past this map's ores, up to the
  // padding of the largest map (as Commons::reset_map does for apples).
  __device__ static void reset_map(const Tables& T, const Params& F, const State& S, int b, int lane, WarpScratch& sc) {
    for (int k = T.nA + lane; k < T.nA_pad; k += 32) { S.apple[(size_t)b * T.nA_pad + k] = 0; S.apple_count[(size_t)b * T.nA_pad + k] = 0; }
    for (int k = T.nA + lane; k < T.nD_pad; k += 32) S.dirt[(size_t)b * T.nD_pad + k] = 0;
    reset(T, F, S, b, lane, sc);
  }

  template <class Actions>
  __device__ static void step(const Tables& T, const Params& F, const State& S, int b, int lane, const Actions& actions, WarpScratch& sc) {
    const auto [env, grid, k0, k1, n, episode] = begin_frame(T, S, b, false);
    const bool is_av = lane < T.P;
    // bits 0-1 state code; bits 2-3 state set in round 1 (1 single-miner ore, 2 two-miner ore; by a reset or by
    // regrowth, never both); bits 4-5 what the frame's last hit asked for (1 partial state, 2 wait state)
    uint8_t* s_state = sc.apple;
    uint8_t* s_miners = sc.dirt;
    uint8_t* cd = S.apple_count + (size_t)b * T.nA_pad;  // count-down, touched by its own lane or by lane 0 between barriers

    int4 a, t, act;
    load_avatar(T, S, b, lane, actions, T.action_table, a, t, act);
    int x = a.x, y = a.y, orient = a.z, cool = t.x;
    const int act_move = act.x, act_turn = act.y, act_mine = act.z;
    const int x0 = x, y0 = y, orient0 = orient;
    double reward = 0.0;  // Avatar:preUpdate (avatar_library.lua:330-332)

    init_occupancy(T, sc.occ, T.solid, lane);
    for (int k = lane; k < T.nA; k += 32) { s_state[k] = S.apple[(size_t)b * T.nA_pad + k]; s_miners[k] = S.dirt[(size_t)b * T.nD_pad + k]; }
    const int words = (T.cells + 31) / 32 + 1;
    for (int i = lane; i < words; i += 32) sc.beam_zap[i] = 0;
    __syncwarp();
    if (is_av) sc.occ[y * T.W + x] = (uint8_t)(lane + 1);
    if (env[ENV_BEAM]) clear_layer(T, grid, F.mine_layer, lane);
    __syncwarp();

    // ---- component updates -----------------------------------------------------------------------------
    // MineBeam:update (:236-252): cool down, then fire if asked to and ready.
    bool fire = false;
    if (is_av) { if (cool > 0) --cool; if (act_mine == 1 && cool == 0) { cool = F.mine_cooldown; fire = true; } }
    // Ore:update (:104-109): the window of a partly mined ore runs out -> reset: forget the miners, back to raw.
    for (int k = lane; k < T.nA; k += 32) {
      if (cd[k] > 0 && --cd[k] == 0) {
        s_miners[k] = 0;
        if ((s_state[k] & 3) != 0) s_state[k] |= 2 << 2;
      }
    }
    // ---- updaters --------------------------------------------------------------------------------------
    // 200 FixedRateRegrow (:41-57): one updater per live state, each with its own draw, only where no avatar stands
    // (positions as the frame started); if both fire the second setState wins.
    for (int k = lane; k < T.nA; k += 32) {
      if ((s_state[k] & 3) != 0) continue;
      uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)F.ore[k * 2], RS_OBJECT, k0, k1);
      const bool first = u01(w.x, w.y) < F.mine_rate[0], second = u01(w.z, w.w) < F.mine_rate[1];
      if ((first || second) && sc.occ[F.ore[k * 2 + 1]] == 0) s_state[k] |= (second ? 2 : 1) << 2;
    }
    // 150 Avatar movement: the frame's random visiting order (policy A.7).
    const int rank = visit_rank(T, lane, n, episode, k0, k1);
    // 100 StochasticIntervalEpisodeEnding
    const bool cont = episode_continues(T, n, episode, k0, k1);
    __syncwarp();

    // ---- round 1a: the beams, shooter by shooter in avatar order (they entered the queue during the updates) ----
    int beam_dirty = 0;
    for (int src = 0; src < T.P; ++src) {
      if (!__shfl_sync(MP_FULL, (int)fire, src)) continue;
      const int sx = __shfl_sync(MP_FULL, x, src), sy = __shfl_sync(MP_FULL, y, src), so = __shfl_sync(MP_FULL, orient, src);
      for (int i = 1; i <= F.mine_length; ++i) {  // radius 0: one ray (every lane walks it)
        int cx = sx + dir_dx(so) * i, cy = sy + dir_dy(so) * i;
        if (!wrap_or_reject(T, cx, cy)) break;
        const int cell = cy * T.W + cx;
        bool blocked = (T.cell_flags[cell] >> F.mine_hit) & 1;  // BeamBlocker 'mine' (walls)
        const int k = F.ore_of_cell[cell];
        const int st = k >= 0 ? (s_state[k] & 3) : 0;
        if (st != 0) {  // Ore:onHit (:118-150): a raw or partial ore takes the hit and stops the beam
          blocked = true;
          if (st == 1) {
            // single-miner ore: mined and extracted by the same hit; partial, raw (reset), wait are queued -> wait
            if (lane == src) {
              reward += F.mine_reward[0] + F.extract_reward[0];
              emit_event(S, b, EV_MINING, src + 1, 1);
              emit_event(S, b, EV_EXTRACTION, src + 1, 1);
            }
            __syncwarp();  // every lane has read the ore's state byte before lane 0 rewrites it
            if (lane == 0) s_state[k] = (uint8_t)((s_state[k] & ~(3 << 4)) | (2 << 4));
          } else {
            const unsigned miners = s_miners[k] | (1u << src);  // Ore:addMiner (:110-114)
            if (lane == src) { reward += F.mine_reward[1]; emit_event(S, b, EV_MINING, src + 1, 2); }
            if (__popc(miners) == 2) {  // enough miners: both extract, then Ore:reset and the wait state
              if (is_av && ((miners >> lane) & 1u)) {
                reward += F.extract_reward[1];
                emit_event(S, b, EV_EXTRACTION, lane + 1, 2);
                emit_event(S, b, EV_EXTRACTION_PAIR, lane + 1, (__ffs(miners & ~(1u << lane))) | (2 << 8));
              }
              __syncwarp();
              if (lane == 0) { s_miners[k] = 0; cd[k] = 0; s_state[k] = (uint8_t)((s_state[k] & ~(3 << 4)) | (2 << 4)); }
            } else {
              __syncwarp();
              if (lane == 0) { s_miners[k] = (uint8_t)miners; cd[k] = (uint8_t)F.mine_window; s_state[k] = (uint8_t)((s_state[k] & ~(3 << 4)) | (1 << 4)); }
            }
          }
          __syncwarp();
        }
        if (blocked) break;
        if (lane == 0 && grid[(size_t)F.mine_layer * T.cells_pad + cell] == 0 && !((sc.beam_zap[cell >> 5] >> (cell & 31)) & 1u)) {
          sc.beam_zap[cell >> 5] |= 1u << (cell & 31);
          grid[(size_t)F.mine_layer * T.cells_pad + cell] = cell_value(F.mine_sprite, so);
        }
        beam_dirty = 1;
        __syncwarp();
      }
    }
    // ---- round 1b: resets and regrowth take effect (no contact callbacks on these pieces) ---------------------
    for (int k = lane; k < T.nA; k += 32) {
      const int r1 = (s_state[k] >> 2) & 3;
      if (r1) s_state[k] = (uint8_t)((s_state[k] & ~0x0f) | r1);
    }
    __syncwarp();
    // ---- round 1c: moves in the frame's order ------------------------------------------------------------------
    move_avatars(T, lane, rank, true, act_turn, act_move, x, y, orient, sc.occ, [](int, int) {});

    // ---- round 2 + write back ------------------------------------------------------------------------------
    for (int k = lane; k < T.nA; k += 32) {
      const int q2 = (s_state[k] >> 4) & 3;
      const uint8_t now = q2 == 2 ? 0 : (q2 == 1 ? 3 : (s_state[k] & 3));
      const uint8_t was = S.apple[(size_t)b * T.nA_pad + k];
      if (now != was) {
        S.apple[(size_t)b * T.nA_pad + k] = now;
        grid[(size_t)F.ore_layer * T.cells_pad + F.ore[k * 2 + 1]] = cell_value(F.ore_sprite[now], 0);
      }
      S.dirt[(size_t)b * T.nD_pad + k] = s_miners[k];
    }
    draw_avatars(T, grid, lane, x0, y0, orient0, 1, x, y, orient, 1);

    const bool done = !cont || n >= T.max_frames;
    if (is_av) {
      *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(x, y, orient, 1);
      S.av_timer[((size_t)b * T.P + lane) * 4] = cool;
      for (int k = 0; k < T.n_scalar; ++k)  // READY_TO_SHOOT = MineBeam:readyToShoot (:186-189)
        S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = T.scalar_obs[k] == 0 ? 1.0 - (double)cool / (double)F.mine_cooldown : 0.0;
    }
    store_timestep(T, S, b, lane, n, reward, done ? 2 : 1, beam_dirty);
  }
};
