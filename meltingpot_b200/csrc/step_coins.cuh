// step_coins.cuh -- state transition of the coins family (two players), one warp per env instance.
//
// Restates one frame of api:advance (api_factory.lua:104-111) for the components of
//   meltingpot/lua/levels/coins/components.lua
//     Coin:onEnter :87-160, ChoiceCoinRegrow :183-194, Role :213-258, PartnerTracker :283-330
//   meltingpot/lua/modules/avatar_library.lua (Avatar movement)
//   meltingpot/lua/modules/component_library.lua:900-950 (StochasticIntervalEpisodeEnding)
// in the closed form of the other families: lanes are the two avatars or the coins, depending on
// the phase. Coin state codes (State.apple): 0 'coinWait' (layer logic), 1 / 2 the two coin types
// (liveStateA / liveStateB, superOverlay). There are no beams and avatars never leave the map.
#pragma once

#include "family_load.h"
#include "step_common.cuh"

struct Coins {
  struct Params {
    int coin_layer;
    int coin_sprite[2];           // sprite of coin type 0 / 1 (liveStateA / liveStateB)
    int coin_type[2];             // PlayerCoinType of each player
    double coin_reward[2][4];     // per collecting player: self match, self mismatch, other match, other mismatch
    double coin_rate;             // ChoiceCoinRegrow regrowRate
    int terminate, terminate_n;   // the episode ends once a player has collected terminate_n coins (if terminate)
    const int32_t* coin;          // [nA][2] obj id, cell
    const int16_t* coin_of_cell;  // [cells_pad] coin index or -1
  };

  // Host: the coins tables of the blob (compiler.py _coins_tables): co_ip / co_dp and the coins.
  static int load(FamilyLoad& ld, const Tables& T, Params& F) {
    const int32_t* ip;
    const double* dp;
    Section<int32_t> coin;
    int rc;
    if ((rc = ld.params("co", MPB_CO_I_COUNT, MPB_CO_D_COUNT, &ip, &dp)) || (rc = ld.need("co_coin", MPB_I32, &coin))) return rc;
    if (T.P != 2) return fail(MP_E_UNSUPPORTED, "coins needs exactly two players (got %d)", T.P);
    ld.nA = ip[MPB_CO_I_N_COINS]; F.coin_layer = ip[MPB_CO_I_COIN_LAYER];
    F.coin_sprite[0] = ip[MPB_CO_I_COIN_SPRITE_0]; F.coin_sprite[1] = ip[MPB_CO_I_COIN_SPRITE_1];
    F.terminate = ip[MPB_CO_I_TERMINATE]; F.terminate_n = ip[MPB_CO_I_TERMINATE_N];
    ld.end_min_frames = ip[MPB_CO_I_END_MIN_FRAMES]; ld.end_interval = ip[MPB_CO_I_END_INTERVAL];
    F.coin_type[0] = ip[MPB_CO_I_COIN_TYPE_0]; F.coin_type[1] = ip[MPB_CO_I_COIN_TYPE_1];
    if (ld.nA > 2048) return fail(MP_E_UNSUPPORTED, "%d coins (max 2048)", ld.nA);
    if (ld.end_interval < 1) return fail(MP_E_INVALID, "episode interval < 1");
    F.coin_rate = dp[MPB_CO_D_REGROW_RATE]; ld.end_prob = dp[MPB_CO_D_END_PROB];
    for (int p = 0; p < 2; ++p) for (int k = 0; k < 4; ++k) F.coin_reward[p][k] = dp[MPB_CO_D_REWARD_0_SELF_MATCH + 4 * p + k];
    std::vector<int32_t> v_coin(coin.data, coin.data + coin.count);
    ld.table(&F.coin, v_coin);
    return cell_index(ld, T, "co_coin", coin, ld.nA, 2, &F.coin_of_cell);
  }

  // Host: per-env variants may differ in the coin rewards, the regrowth rate and the termination rule, and, as draws of
  // the builder (map variants), in the coins, their cells and the coin sprites (the draw's colours).
  static int same_shape(const Params& a, const Params& b) {
    MP_SAME(coin_layer) MP_SAME(coin_type)
    return MP_OK;
  }

  using Scratch = WarpScratch;
  // Draws of the builder may differ in their map (mp_create_variants): the coin table is their entity table, and the coin
  // count is the nA of each variant's Tables (setup_variants).
  static constexpr bool kMapVariants = true;
  static constexpr const char* kMapSections[] = {"co_coin", nullptr};
  static constexpr const char* const* kSpriteSections = nullptr;
  static constexpr bool kStagesTables = false;
  __host__ __device__ static size_t scratch_bytes(const Tables& T) { return warp_scratch_bytes(T); }
  __host__ __device__ static size_t table_bytes(const Tables&) { return 0; }
  __device__ static void stage(const Tables&, const Params&, uint8_t*) {}
  __device__ static WarpScratch carve(const Tables& T, uint8_t* base, const uint8_t*) { return carve_scratch(T, base); }

  // Episode start for coins: every coin waits, the two avatars draw their spawn points (policy A.10).
  __device__ static void reset(const Tables& T, const Params& F, const State& S, int b, int lane, WarpScratch& sc) {
    const auto [env, grid, k0, k1, n, episode] = begin_frame(T, S, b, true);
    __syncwarp();
    copy_init_grid(T, grid, lane);
    // the whole padded row, so that an env that moved from a draw with more coins keeps no bytes of it (records and
    // snapshots of equal envs stay equal byte for byte)
    for (int k = lane; k < T.nA_pad / 16; k += 32) reinterpret_cast<uint4*>(S.apple + (size_t)b * T.nA_pad)[k] = make_uint4(0, 0, 0, 0);
    __syncwarp();
    const auto all = [](int) { return true; };
    spawn_group(T, S, b, lane, grid, sc.tmp, T.spawn_init_cell[0], T.n_spawn_init[0], all, all, episode, k0, k1, [&](int) {
      S.av_extra[((size_t)b * T.P + lane) * 8] = 0;  // cumulativeCoinsCollected (GlobalCoinCollectionTracker:reset :203-207)
      for (int k = 0; k < T.n_scalar; ++k) S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = 0.0;
    });
    // api:start ends with one grid:update (api_factory.lua:101): the ChoiceCoinRegrow updaters already fire at frame 0.
    // (Spawn points are not coin cells, so no avatar can be standing on a coin that appears now.)
    for (int k = lane; k < T.nA; k += 32) {
      uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)F.coin[k * 2], RS_OBJECT, k0, k1);
      if (u01(w.x, w.y) < F.coin_rate) {
        const int type = (int)pick(w.z, 2u);
        S.apple[(size_t)b * T.nA_pad + k] = (uint8_t)(1 + type);
        grid[(size_t)F.coin_layer * T.cells_pad + F.coin[k * 2 + 1]] = cell_value(F.coin_sprite[type], 0);
      }
    }
    reset_env_row(T, S, b, lane, episode, 0);
  }

  template <class Actions>
  __device__ static void step(const Tables& T, const Params& F, const State& S, int b, int lane, const Actions& actions, WarpScratch& sc) {
    const auto [env, grid, k0, k1, n, episode] = begin_frame(T, S, b, false);
    const bool is_av = lane < T.P;
    uint8_t* s_state = sc.apple;  // [nA_pad] bits 0-1 state code, bits 4-5 state queued by ChoiceCoinRegrow, bit 6 collected

    int4 a, t, act;
    load_avatar(T, S, b, lane, actions, T.action_table, a, t, act);
    int x = a.x, y = a.y, orient = a.z, cumulative = is_av ? S.av_extra[((size_t)b * T.P + lane) * 8] : 0;
    const int act_move = act.x, act_turn = act.y;
    const int x0 = x, y0 = y, orient0 = orient;
    double reward = 0.0;     // Avatar:preUpdate (avatar_library.lua:330-332)
    int partner_mismatch = 0;  // PartnerTracker:preUpdate (coins/components.lua:303-306)
    bool cont = true;

    init_occupancy(T, sc.occ, T.solid, lane);
    for (int k = lane; k < T.nA; k += 32) s_state[k] = S.apple[(size_t)b * T.nA_pad + k];
    __syncwarp();
    if (is_av) sc.occ[y * T.W + x] = (uint8_t)(lane + 1);
    __syncwarp();

    // ---- updaters -------------------------------------------------------------------------------------
    // 150 Avatar movement: the frame's random visiting order (policy A.7).
    const int rank = visit_rank(T, lane, n, episode, k0, k1);
    // 100 StochasticIntervalEpisodeEnding (the scene registers first), then ChoiceCoinRegrow on every waiting coin:
    // probability regrowRate, then random:choice of the two live states (coins/components.lua:183-194).
    cont = episode_continues(T, n, episode, k0, k1);
    for (int k = lane; k < T.nA; k += 32) {
      if ((s_state[k] & 3) != 0) continue;
      uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)F.coin[k * 2], RS_OBJECT, k0, k1);
      if (u01(w.x, w.y) < F.coin_rate) s_state[k] |= (uint8_t)((1 + pick(w.z, 2u)) << 4);
    }
    __syncwarp();

    // Coin:onEnter for collector `who` on coin `k` (every lane calls this with the same arguments).
    auto collect = [&](int who, int k) {
      const int type = (s_state[k] & 3) - 1;
      const bool match = type == F.coin_type[who];
      const double* R = F.coin_reward[who];  // self match, self mismatch, other match, other mismatch (Role multipliers folded in)
      if (lane == who) {
        reward += match ? R[0] : R[1];
        ++cumulative;
        if (F.terminate && cumulative >= F.terminate_n) cont = false;
        emit_event(S, b, EV_COIN_CONSUMED, who + 1, match ? 1 : 0);
      } else if (is_av) {  // Coin:rewardOthers (:74-85) and PartnerTracker:reportMatch / reportMismatch (:324-330)
        reward += match ? R[2] : R[3];
        if (!match) partner_mismatch = 1;
      }
      __syncwarp();
      if (lane == 0) s_state[k] |= 64;  // setState(waitState) is queued: the coin stays where it is until round 2
      __syncwarp();
    };

    // ---- round 1: moves in the frame's order, then the queued coin states in object order -----------------
    // policy A.5: `enter` fires on the final cell, moved or blocked
    move_avatars(T, lane, rank, true, act_turn, act_move, x, y, orient, sc.occ, [&](int src, int cell) {
      const int ci = F.coin_of_cell[cell];
      if (ci >= 0 && (s_state[ci] & 3) != 0 && !(s_state[ci] & 64)) collect(src, ci);
    });
    const int partner_cont = __all_sync(MP_FULL, cont);  // (cont is per lane so far: either collector may end the episode)
    cont = partner_cont;
    for (int base = 0; base < T.nA; base += 32) {
      const int k = base + lane;
      const int queued = k < T.nA ? (s_state[k] >> 4) & 3 : 0;
      if (queued) s_state[k] = (uint8_t)queued;  // now live (placed on superOverlay)
      __syncwarp();
      // a coin that appears under a standing avatar is entered at once (contact is symmetric on placement, policy A.5)
      const int o = queued ? sc.occ[F.coin[k * 2 + 1]] : 0;
      unsigned gm = __ballot_sync(MP_FULL, o >= 1 && o <= T.P);
      while (gm) {
        const int c = __ffs(gm) - 1; gm &= gm - 1;
        collect(__shfl_sync(MP_FULL, o, c) - 1, base + c);
      }
    }
    cont = __all_sync(MP_FULL, cont);

    // ---- round 2 + write back ------------------------------------------------------------------------------
    for (int k = lane; k < T.nA; k += 32) {
      const uint8_t now = (s_state[k] & 64) ? 0 : (s_state[k] & 3);
      const uint8_t was = S.apple[(size_t)b * T.nA_pad + k];
      if (now != was) {
        S.apple[(size_t)b * T.nA_pad + k] = now;
        grid[(size_t)F.coin_layer * T.cells_pad + F.coin[k * 2 + 1]] = now ? cell_value(F.coin_sprite[now - 1], 0) : (uint16_t)0;
      }
    }
    draw_avatars(T, grid, lane, x0, y0, orient0, 1, x, y, orient, 1);

    const bool done = !cont || n >= T.max_frames;
    if (is_av) {
      *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(x, y, orient, 1);
      S.av_extra[((size_t)b * T.P + lane) * 8] = cumulative;
      for (int k = 0; k < T.n_scalar; ++k)  // MISMATCHED_COIN_COLLECTED_BY_PARTNER (coins.py AvatarMetricReporter)
        S.scalar_obs[((size_t)k * S.B + b) * T.P + lane] = T.scalar_obs[k] == 2 ? (double)partner_mismatch : 0.0;
    }
    store_timestep(T, S, b, lane, n, reward, done ? 2 : 1, 0);
  }
};
