// common.cuh -- device-side tables, per-env state layout and RNG shared by the kernels.
//
// Data layout in HBM (struct-of-arrays, env instance on the leading axis):
//   grid        u16 [B][L][cells_pad]   sprite grid: 0 empty, else 1 + sprite*4 + orientation.
//                                       This is the engine's view of "which piece is on
//                                       (x, y, layer)" (SURVEY.md A.1) reduced to what the
//                                       renderer and the collision tests need.
//   avatar      i32 [B][P][4]           x, y, orientation, alive
//   av_timer    i32 [B][P][4]           zap cooldown, second-beam cooldown, frame of last state
//                                       change, spare
//   apple/dirt/water/apple_count u8 [B][n_pad]  per-entity state (family specific)
//   env         i32 [B][8]              step, episode, done, dirt count, cleaned flags, ate flags,
//                                       beam-dirty, spare
// cells_pad keeps every layer row 16-byte aligned so rows can be moved with 128-bit accesses.
#pragma once

#include <cuda_runtime.h>
#include <stdint.h>

#define MP_MAX_PLAYERS 16
#define MP_MAX_LAYERS 16
#define MP_MAX_BEAM_CELLS 32
#define MP_FULL 0xffffffffu
#define MP_MAX_PEERS 8   // ranks of one NVSwitch domain that exchange their timesteps (mp_exchange_*)

enum { ENV_STEP = 0, ENV_EPISODE = 1, ENV_DONE = 2, ENV_DIRT = 3, ENV_CLEANED = 4, ENV_ATE = 5, ENV_BEAM = 6, ENV_COLS = 8 };
enum { AV_X = 0, AV_Y = 1, AV_ORIENT = 2, AV_ALIVE = 3 };
enum { TM_ZAP = 0, TM_BEAM2 = 1, TM_FRAME = 2 };
// RNG streams: must match oracle/mp_oracle.c (the RNG addressing is part of the engine policy).
enum { RS_SCENE = 0, RS_AVATAR = 1, RS_OBJECT = 2, RS_AVATAR_RESET = 3, RS_OBJECT_RESET = 4, RS_CHOICE = 5 };
enum { SCENE_DRAW_DIRT = 0, SCENE_DRAW_EPISODE_END = 1 };

struct BeamGeom {  // one beam footprint, cells in visiting order (policy A.8)
  int n;
  int depth;
  int8_t lat[MP_MAX_BEAM_CELLS];     // lateral offset, negative = left of the shooter
  int8_t fwd[MP_MAX_BEAM_CELLS];     // forward distance
  int8_t parent[MP_MAX_BEAM_CELLS];  // cell that must be visited and unblocked first, or -1
};

struct Tables {
  // geometry
  int W, H, cells, cells_pad, L, P, topology, max_frames;
  int view_l, view_r, view_f, view_b, n_sprites, oob_sprite, oov_sprite, n_actions, n_scalar;
  int scalar_obs[4];
  // shared avatar machinery
  int avatar_layer, n_spawn;
  int avatar_sprite[MP_MAX_PLAYERS];
  int zap_cooldown, zap_respawn, zap_remove, zap_layer, zap_sprite, zap_hit;
  double zap_penalty, zap_reward;
  BeamGeom zap_geom;
  // clean_up family
  int nA, nD, nW, nA_pad, nD_pad, nW_pad;
  int apple_layer, apple_sprite, dirt_layer, dirt_sprite, water_layer, n_anim, anim_frames, anim_random;
  int water_sprite[8];
  int clean_cooldown, clean_layer, clean_sprite, clean_hit;
  BeamGeom clean_geom;
  int dirt_delay, end_min_frames, end_interval, taste_role, dirt_count0;
  double grow_rate, grow_depletion, grow_restoration, eat_reward, dirt_prob, end_prob, taste_amount;
  // commons_harvest family
  int wait_layer, wait_sprite, grass_layer, grass_sprite, dess_sprite, ch_n_wait, ch_n_probs;
  double ch_probs[4];
  // initial spawn groups (Avatar spawnGroup vs postInitialSpawnGroup, avatar_library.lua:121-125,322-328)
  int n_spawn_init[2];
  int avatar_init_group[MP_MAX_PLAYERS];
  const int32_t* spawn_init_cell[2];
  const int32_t* ch_apple;     // [nA][4] obj id, cell, initially live, grass obj id
  // territory family
  int nR, nR_pad, res_layer, unclaimed_sprite, tex_layer, tex_sprite, ind_layer, dmg_layer, dmg_sprite, mark_layer;
  int mark_initial_level, mark_recovery, mark_n_levels, mark_inc[3], mark_remove[3], mark_freeze[3], mark_sprite[3];
  double mark_src_reward[3], mark_tgt_reward[3];
  int claim_wait, brush_layer, claim_layer, res_health0, res_reward_delay, res_repair_delay, tr_taste_role;
  double res_reward, res_rate, res_repair_prob, tr_taste_amount, tr_taste_mult;
  int claimed_sprite[MP_MAX_PLAYERS], dry_sprite[MP_MAX_PLAYERS], brush_sprite[MP_MAX_PLAYERS], claimbeam_sprite[MP_MAX_PLAYERS];
  BeamGeom claim_geom, brush_geom;
  const int32_t* tr_res;       // [nR][3] obj id, cell, initial state
  const int16_t* res_of_cell;  // [cells_pad] resource index or -1
  const uint8_t* wall;         // [cells_pad] 1 where an AllBeamBlocker piece stands
  // 'choice' prefabs drawn per env and episode (prefab_utils.lua:63-65): ticket of group g = pick(philox(0, episode, g, RS_CHOICE).x, choice_n[g])
  int n_choice;
  const int32_t* choice_n;     // [n_choice] options per group
  const int32_t* spawn_cond;   // [n_spawn][2] (group or -1, ticket mask) of each spawn candidate, or null
  const int32_t* tr_res_cond;  // [nR][2] same for each resource, or null
  const int32_t* ch_nbr;       // [nA][16] apples inside the regrowth disc (excluding self), -1 padded
  // device tables
  const uint16_t* init_grid;   // [L][cells_pad]
  const int32_t* action_table; // [n_actions][4]
  const int32_t* apple;        // [nA][3] obj id, cell, initially live
  const int32_t* dirt;         // [nD][3] obj id, cell, initially dirty
  const int32_t* water;        // [nW][2] obj id, cell
  const int32_t* spawn_cell;   // [n_spawn]
  const uint8_t* solid;        // [cells_pad] 255 where the avatar layer is statically occupied
  const uint8_t* cell_flags;   // [cells_pad] bit h: a BeamBlocker for hit h sits here
  const int16_t* apple_of_cell;  // [cells_pad] apple index or -1
  const int16_t* dirt_of_cell;   // [cells_pad] dirt index or -1
  // render tables
  const uint8_t* atlas;        // [n_total][4][2][8][16]: facing, half (px 0-3 | 4-7), row, 16 B (n_total includes pre-merged sprites)
  const int16_t* sprite_map;   // [P+1][n_total]
  const uint8_t* sprite_opaque;  // [n_total] bit 0: every pixel alpha 255 and never remapped; bit 1: remapped for some viewer
  const uint8_t* sprite_pair;    // [n_total][n_total] pre-merged sprite for (opaque base, sprite on top) or 0
  // coins family (step_coins.cuh); the coins reuse ch_apple / apple_of_cell / apple_layer
  int coin_sprite[2];          // sprite of coin type 0 / 1 (liveStateA / liveStateB)
  int coin_type[2];            // PlayerCoinType of each player
  double coin_reward[2][4];    // per collecting player: self match, self mismatch, other match, other mismatch
  double coin_rate;            // ChoiceCoinRegrow regrowRate
  int coin_terminate, coin_terminate_n;
  // coop_mining family (step_mining.cuh); ores reuse ch_apple / apple_of_cell / apple_layer, the beam reuses zap_*
  int ore_sprite[4];           // wait, single-miner raw, two-miner raw, two-miner partial
  int mine_window, mine_length;
  double mine_rate[2];         // FixedRateRegrow liveRates
  double mine_reward[2], extract_reward[2];  // per ore type (1 miner, 2 miners)
};

struct State {
  int B;
  uint64_t seed;  // key of env b = seed + b (env_index_base already folded in)
  uint16_t* grid;
  int32_t* avatar;
  int32_t* av_timer;
  uint8_t* apple;
  uint8_t* dirt;
  uint8_t* water;
  uint8_t* apple_count;
  uint8_t* fam_u8;     // family-specific per-env bytes  [B][fam_u8_stride]
  uint16_t* fam_u16;   // family-specific per-env shorts [B][fam_u16_stride]
  int32_t* av_extra;   // i32 [B][P][8] family-specific avatar state
  int fam_u8_stride, fam_u16_stride;
  int32_t* env;
  // outputs
  double* reward;
  double* discount;
  int64_t* step_type;
  double* scalar_obs;  // [n_scalar][B][P]
  double* packed;      // [B][P+2] reward..., discount, step type: one buffer for the per-step all-gather
  uint8_t* rgb;
  uint8_t* world_rgb;
  int32_t* events;     // [B][max_events][3] (type, a, b) of the current step, unordered (see emit_event)
  int32_t* n_events;   // [B] events emitted this step
  int max_events;      // rows per env: the family's worst case for one step (mp_create), so nothing is ever dropped
  // Cross-GPU exchange of the stacked timestep (mp_exchange_*, include/mp_engine.h). Off when x_world == 0. Every rank
  // owns gathered[2][x_world * B][P + 2] and flags[MP_MAX_PEERS]; x_gathered / x_flags are those buffers of every rank,
  // mapped into this process (NVLink peer memory; entry x_rank is the local one).
  int x_world, x_rank;
  unsigned long long x_step;               // sequence number of this launch; slot = x_step & 1
  double* x_gathered[MP_MAX_PEERS];
  unsigned long long* x_flags[MP_MAX_PEERS];
  int x_raise;                             // render launches only: 1 = deliver this step's rows (exchange_push / exchange_finish)
  // Stacked observations across GPUs (mp_gather_obs_*): when g_world > 0 the renderer stores every strip not only to
  // this rank's rgb / world_rgb but also, straight from its staging buffer (TMA bulk stores over NVLink peer mappings),
  // into this rank's slab of EVERY rank's stacked buffer. g_rgb / g_wrgb already point at (slot, x_rank's slab).
  int g_world;
  unsigned long long g_step;               // sequence number of this render launch; slot = g_step & 1
  uint8_t* g_rgb[MP_MAX_PEERS];
  uint8_t* g_wrgb[MP_MAX_PEERS];
  const unsigned long long* g_flags;       // local flags[r] = last render rank r has fully delivered here
};

// Events of the current step (the reference's events:add calls on the hot path). Types follow
// the order of oracle/mp_oracle.c; player indices are 1-based as in Lua.
#define MP_MIN_EVENTS 64  // floor of State::max_events
enum { EV_ZAP = 1, EV_EDIBLE_CONSUMED = 2, EV_PLAYER_CLEANED = 3, EV_CLAIMED_RESOURCE = 4, EV_DESTROYED_RESOURCE = 5,
       EV_SANCTIONING = 6, EV_REMOVAL = 7, EV_COIN_CONSUMED = 8 /* a = player, b = 1 match / 0 mismatch */,
       EV_MINING = 9 /* a = player, b = ore type */, EV_EXTRACTION = 10 /* a = player, b = ore type */,
       EV_EXTRACTION_PAIR = 11 /* a = player_a, b = player_b | ore type << 8 */ };

// Called by the one lane that owns the event. Lanes append concurrently, so the order within a step is unspecified
// (hosts sort). One warp owns an env, so the step's event count lives in shared memory (a global atomic per event
// would put its round trip on the warp's critical path); event_end publishes it once.
__device__ __forceinline__ int* event_counter() {
  __shared__ int s_event_count[4];  // one per env warp of a state-transition CTA
  return &s_event_count[(threadIdx.x >> 5) & 3];
}
__device__ __forceinline__ void event_begin(int lane) {
  if (lane == 0) *event_counter() = 0;
  __syncwarp();
}
__device__ __forceinline__ void emit_event(const State& S, int b, int type, int a0, int a1) {
  const int i = atomicAdd(event_counter(), 1);
  if (i < S.max_events) {  // (always true: max_events bounds what one step can emit; kept as a memory-safety guard)
    int32_t* e = S.events + ((size_t)b * S.max_events + i) * 3;
    e[0] = type; e[1] = a0; e[2] = a1;
  }
}
__device__ __forceinline__ void event_end(const State& S, int b, int lane) {
  __syncwarp();
  if (lane == 0) S.n_events[b] = *event_counter();
}

__device__ __forceinline__ uint4 philox4x32_10(uint32_t c0, uint32_t c1, uint32_t c2, uint32_t c3, uint32_t k0, uint32_t k1) {
#pragma unroll
  for (int r = 0; r < 10; ++r) {
    uint32_t h0 = __umulhi(0xD2511F53u, c0), l0 = 0xD2511F53u * c0;
    uint32_t h1 = __umulhi(0xCD9E8D57u, c2), l1 = 0xCD9E8D57u * c2;
    uint32_t n0 = h1 ^ c1 ^ k0, n2 = h0 ^ c3 ^ k1;
    c0 = n0; c1 = l1; c2 = n2; c3 = l0;
    k0 += 0x9E3779B9u; k1 += 0xBB67AE85u;
  }
  return make_uint4(c0, c1, c2, c3);
}

__device__ __forceinline__ double u01(uint32_t a, uint32_t b) {
  return ((double)(a >> 5) * 67108864.0 + (double)(b >> 6)) / 9007199254740992.0;
}
__device__ __forceinline__ uint32_t pick(uint32_t w, uint32_t n) { return __umulhi(w, n); }

// Does a piece with condition (group, mask) exist in this env's current episode?
__device__ __forceinline__ bool choice_present(const Tables& T, int group, uint32_t mask, int episode, uint32_t k0, uint32_t k1) {
  if (group < 0) return true;
  const uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)group, RS_CHOICE, k0, k1);
  return (mask >> pick(w.x, (uint32_t)T.choice_n[group])) & 1u;
}

__device__ __forceinline__ int dir_dx(int d) { return (d == 1) - (d == 3); }
__device__ __forceinline__ int dir_dy(int d) { return (d == 2) - (d == 0); }
__device__ __forceinline__ uint16_t cell_value(int sprite, int orient) { return (uint16_t)(1 + sprite * 4 + (orient & 3)); }

// Maps (x, y) into the map; returns false if it falls outside a BOUNDED map.
// On a TORUS every caller stays within one map width / height of the map (moves, beam footprints and
// view windows are all smaller than the map: mp_create refuses views and beams that are not, see beam_fits_torus),
// so a conditional add wraps.
__device__ __forceinline__ bool wrap_or_reject(const Tables& T, int& x, int& y) {
  if (T.topology == 1) {
    x += x < 0 ? T.W : (x >= T.W ? -T.W : 0);
    y += y < 0 ? T.H : (y >= T.H ? -T.H : 0);
    return true;
  }
  return x >= 0 && x < T.W && y >= 0 && y < T.H;
}

// Delivery of this rank's packed timestep rows (reward[0..P), discount, step type per env) into every rank's gathered
// buffer: plain stores through the NVLink peer mappings, P + 2 per env and rank -- the "all-gather" of the stacked
// timestep without a collective kernel. It runs in the kernel that FOLLOWS the state transition (the renderer's
// prologue, or k_exchange_push when no render follows): the rows are complete there (kernel boundary), the remote
// round trips hide behind ~200 us of rendering instead of sitting in the tail of the latency-bound transition kernel,
// and no warp of the transition pays a system-scope fence (measured: 15 us per step when every warp fenced, 6 us
// with the stores alone in the transition kernel). Called by every thread of every CTA of the delivering grid.
__device__ __forceinline__ void exchange_push(const Tables& T, const State& S) {
  if (S.x_world == 0) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = (int)blockDim.x >> 5;
  // Two flag rows per rank: done[r] (flags[0..8), raised by rank r's k_exchange_wait: "my rows of step s are complete here")
  // and begun[r] (flags[8..16), raised right here: "rank r has started delivering step s"). Flow control: slot
  // (x_step & 1) still holds step x_step - 2 on every rank, and a rank's consumers of that step are stream-ordered
  // before its next state transition, so the slot is free once the rank has BEGUN step x_step - 1. That is a whole
  // render ago in steady state, so ranks are not lock-stepped; the slowest rank never waits on a faster one (no cycle).
  if (blockIdx.x == 0 && threadIdx.x < S.x_world)
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(S.x_flags[threadIdx.x] + MP_MAX_PEERS + S.x_rank), "l"(S.x_step) : "memory");
  if (lane < S.x_world && S.x_step > 1ull) {
    const volatile unsigned long long* f = S.x_flags[S.x_rank] + MP_MAX_PEERS + lane;
    while (*f + 1ull < S.x_step) __nanosleep(100);
  }
  __syncwarp();
  const int n = T.P + 2;
  const size_t base = ((size_t)(S.x_step & 1ull) * S.x_world + (size_t)S.x_rank) * S.B;
  for (int b = (int)blockIdx.x + warp * (int)gridDim.x; b < S.B; b += n_warps * (int)gridDim.x) {
    if (lane < n) {
      const double v = S.packed[(size_t)b * n + lane];
      for (int r = 0; r < S.x_world; ++r) S.x_gathered[r][(base + b) * n + lane] = v;
    }
  }
}

// Delivery when no render follows the state transition (mp_step_state on its own, or rendering switched off).
__global__ void __launch_bounds__(256) k_exchange_push(Tables T, State S) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  exchange_push(T, S);
}

// The consumer side, enqueued by EVERY rank after its step (mp_exchange_wait; stream-ordered after the kernel that
// delivered, i.e. the renderer): one warp. Lane r first tells rank r "my rows of step `step` are complete in your
// buffer" -- true without any fence, because the delivering kernel has completed before this one started (kernel
// boundary) -- and then waits until rank r has said the same here. Collective in the usual sense: a rank's rows become
// visible to the others when it calls this. Small enough to sit beside a persistent k_render CTA.
__global__ void __launch_bounds__(32) k_exchange_wait(State S, unsigned long long step) {
  const int lane = threadIdx.x;
  if (lane < S.x_world) {
    asm volatile("st.relaxed.sys.global.u64 [%0], %1;" ::"l"(S.x_flags[lane] + S.x_rank), "l"(step) : "memory");
    const unsigned long long* mine = S.x_flags[S.x_rank] + lane;
    unsigned long long v;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(mine) : "memory");
      if (v < step) __nanosleep(200);
    } while (v < step);
  }
}

// One warp: lane r < world waits until local flags[r] has reached `step`.
__global__ void __launch_bounds__(32) k_flag_wait(const unsigned long long* flags, int world, unsigned long long step) {
  const int lane = threadIdx.x;
  if (lane < world) {
    unsigned long long v;
    do {
      asm volatile("ld.acquire.sys.global.u64 %0, [%1];" : "=l"(v) : "l"(flags + lane) : "memory");
      if (v < step) __nanosleep(200);
    } while (v < step);
  }
}

// After a gathering render has completed: flags[rank] = step on every rank (same protocol as exchange_raise).
__global__ void __launch_bounds__(32) k_gather_raise(unsigned long long* const* flags, int world, int rank, unsigned long long step) {
  if (threadIdx.x < world) {
    __threadfence_system();
    asm volatile("st.release.sys.global.u64 [%0], %1;" ::"l"(flags[threadIdx.x] + rank), "l"(step) : "memory");
  }
}
