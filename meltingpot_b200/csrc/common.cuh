// common.cuh -- what the kernels share: the tables every kernel reads (Tables), the per-env state layout (State), the
// step's events and the RNG. Each substrate family's own parameters are in its step_<family>.cuh.
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
//   key         u64 [B]                 Philox key of each env (seed + env_index_base + b at creation)
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
// RNG streams: must match oracle/mp_oracle.c (the RNG addressing is part of the engine policy); RS_ROUTE (drawn routes only) by tests/drawn_routes.py.
enum { RS_SCENE = 0, RS_AVATAR = 1, RS_OBJECT = 2, RS_AVATAR_RESET = 3, RS_OBJECT_RESET = 4, RS_CHOICE = 5, RS_ROUTE = 6 };
enum { SCENE_DRAW_DIRT = 0, SCENE_DRAW_EPISODE_END = 1 };

struct BeamGeom {  // one beam footprint, cells in visiting order (policy A.8)
  int n;
  int depth;
  int8_t lat[MP_MAX_BEAM_CELLS];     // lateral offset, negative = left of the shooter
  int8_t fwd[MP_MAX_BEAM_CELLS];     // forward distance
  int8_t parent[MP_MAX_BEAM_CELLS];  // cell that must be visited and unblocked first, or -1
};

// What every kernel reads: the map, the view, the avatars and their spawn points, the episode ending, the sizes of the
// per-env entity arrays and the render tables. What only one family's state transition reads is in that family's
// Params (step_<family>.cuh).
struct Tables {
  // geometry
  int W, H, cells, cells_pad, L, P, topology, max_frames;
  int view_l, view_r, view_f, view_b, n_sprites, oob_sprite, oov_sprite, n_actions, n_scalar;
  int scalar_obs[4];
  // avatars and spawn points
  int avatar_layer, n_spawn;
  int avatar_sprite[MP_MAX_PLAYERS];
  const int32_t* spawn_cell;   // [n_spawn]
  // initial spawn groups (Avatar spawnGroup vs postInitialSpawnGroup, avatar_library.lua:121-125,322-328)
  int n_spawn_init[2];
  int avatar_init_group[MP_MAX_PLAYERS];
  const int32_t* spawn_init_cell[2];
  // 'choice' prefabs drawn per env and episode (prefab_utils.lua:63-65): ticket of group g = pick(philox(0, episode, g, RS_CHOICE).x, choice_n[g])
  int n_choice;
  const int32_t* choice_n;     // [n_choice] options per group
  const int32_t* spawn_cond;   // [n_spawn][2] (group or -1, ticket mask) of each spawn candidate, or null
  // StochasticIntervalEpisodeEnding (every family)
  int end_min_frames, end_interval;
  double end_prob;
  // per-env entity arrays of State: apple / apple_count [nA_pad], dirt [nD_pad], water [nW_pad], fam_u8 / fam_u16 rows of nR_pad
  int nA, nD, nW, nR, nA_pad, nD_pad, nW_pad, nR_pad;
  // device tables
  const uint16_t* init_grid;   // [L][cells_pad]
  const int32_t* action_table; // [n_actions][4]
  const uint8_t* solid;        // [cells_pad] 255 where the avatar layer is statically occupied
  const uint8_t* cell_flags;   // [cells_pad] bit h: a BeamBlocker for hit h sits here
  // render tables
  const uint8_t* atlas;        // [n_total][4][2][8][16]: facing, half (px 0-3 | 4-7), row, 16 B (n_total includes pre-merged sprites)
  const int16_t* sprite_map;   // [P+1][n_total]
  const uint8_t* sprite_opaque;  // [n_total] bit 0: every pixel alpha 255 and never remapped; bit 1: remapped for some viewer
  const uint8_t* sprite_pair;    // [n_total][n_total] pre-merged sprite for (opaque base, sprite on top) or 0
};

// Caller-owned destinations of a step's scalar outputs (mp_device_outputs): any pointer may be null. Strides in bytes;
// scalar_obs row (k, b) starts at scalar_obs + k * scalar_obs_stride + b * scalar_obs_env_stride.
struct ScalarTargets {
  double* reward;
  double* discount;
  int64_t* step_type;
  double* scalar_obs;
  uint64_t reward_stride, discount_stride, step_type_stride, scalar_obs_env_stride, scalar_obs_stride;
  int on;  // any of the four is set
};

// Caller-owned per-player rows of one step (mp_player_outputs, mp_run's players): player p of env b goes to row
// row_of_player[b][p], delivered through the segment that holds the row (RowSegments) and nowhere when no segment does.
// Env b's WORLD.RGB goes to row world_row_of_env[b] of world_rgb when that is in [0, world_n_rows) and world_rgb is
// set. Read only by k_render<..., RENDER_ROUTED> and k_exchange_push.
struct PlayerTargets {
  const int32_t* row_of_player;  // [B][P]
  int scalars_on;  // the segments carry reward or scalar_obs
  const int32_t* world_row_of_env;  // [B]
  uint8_t* world_rgb;
  uint64_t world_rgb_row_stride;
  int world_n_rows;
};

// The per-player targets of a routed step by row range (mp_row_segment, same layout): row r of segment s
// (row_begin <= r < row_end) goes to target + (r - row_begin) * row_stride; scalar_obs row (k, r) starts at
// scalar_obs + k * scalar_obs_stride + (r - row_begin) * scalar_obs_row_stride. A request without segments is one segment
// [0, n_rows). Segments are sorted and disjoint and all carry the same outputs (checked on the host), so s[0] tells which
// outputs are routed. A __grid_constant__ parameter of k_render and k_exchange_push: the table reaches the kernels with
// their launch, so no copy, synchronise or extra launch is needed, and only the routed code reads it.
#define MP_ROW_SEGMENTS 16
struct RowSegment {
  int32_t row_begin, row_end;
  uint8_t* rgb; uint64_t rgb_row_stride;
  double* reward; uint64_t reward_row_stride;
  double* scalar_obs; uint64_t scalar_obs_row_stride, scalar_obs_stride;
};
struct RowSegments {
  int n;
  RowSegment s[MP_ROW_SEGMENTS];
};

// The segment that holds row `row`, or -1 when none does. A scan with a uniform index: a warp's lanes read the same
// constant-bank entries.
__device__ __forceinline__ int row_segment(const RowSegments& G, int row) {
  int s = -1;
  for (int k = 0; k < G.n; ++k) s = (row >= G.s[k].row_begin && row < G.s[k].row_end) ? k : s;
  return s;
}

struct State {
  int B;
  uint64_t* key;  // [B] Philox key of each env: seed + env_index_base + b at mp_create; state, so a restored env keeps its source's
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
  // Where k_render stores env b's images: rgb + b * rgb_env_stride (player p at + p * player_bytes) and
  // world_rgb + b * world_env_stride, in bytes. The engine's own images are the dense case; mp_run's out points them at
  // a caller's tensors. (Kept behind every field the state-transition kernels read.)
  uint64_t rgb_env_stride, world_env_stride;
  ScalarTargets out;                       // the step's scalar rows into caller-owned memory (mp_run's out), or none
  PlayerTargets pr;                        // the step's per-player rows (mp_run's players), or all zero
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

// Delivery of the step's reward, discount, step type and scalar observations from the engine's scalar block into the
// caller's rows (State::out), by the kernel that follows the state transition, like exchange_push: one warp per env,
// called by every thread of every CTA of the delivering grid.
__device__ __forceinline__ void deliver_scalars(const Tables& T, const State& S) {
  const ScalarTargets& o = S.out;
  if (!o.on) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = (int)blockDim.x >> 5;
  const int P = T.P, n = P + 2 + (o.scalar_obs ? T.n_scalar * P : 0);
  for (int b = (int)blockIdx.x + warp * (int)gridDim.x; b < S.B; b += n_warps * (int)gridDim.x) {
    for (int i = lane; i < n; i += 32) {
      if (i < P) {
        if (o.reward) reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(o.reward) + b * o.reward_stride)[i] = S.reward[(size_t)b * P + i];
      } else if (i == P) {
        if (o.discount) *reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(o.discount) + b * o.discount_stride) = S.discount[b];
      } else if (i == P + 1) {
        if (o.step_type) *reinterpret_cast<int64_t*>(reinterpret_cast<uint8_t*>(o.step_type) + b * o.step_type_stride) = S.step_type[b];
      } else {
        const int k = (i - P - 2) / P, p = i - P - 2 - k * P;
        reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(o.scalar_obs) + k * o.scalar_obs_stride + b * o.scalar_obs_env_stride)[p] =
            S.scalar_obs[((size_t)k * S.B + b) * P + p];
      }
    }
  }
}

// Delivery of the routed players' reward and scalar observations into their rows (State::pr), like deliver_scalars:
// one warp per env, lane i covering (output k = i / P, player p = i % P); output 0 is the reward, output 1 + j
// scalar observation j. A player whose row lies in no segment gets nothing; nothing outside the segments is written.
__device__ __forceinline__ void deliver_player_scalars(const Tables& T, const State& S, const RowSegments& G) {
  if (!S.pr.scalars_on) return;
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5, n_warps = (int)blockDim.x >> 5;
  const int P = T.P, n = P * (1 + (G.s[0].scalar_obs ? T.n_scalar : 0));
  for (int b = (int)blockIdx.x + warp * (int)gridDim.x; b < S.B; b += n_warps * (int)gridDim.x) {
    for (int i = lane; i < n; i += 32) {
      const int k = i / P, p = i - k * P;
      const int row = S.pr.row_of_player[(size_t)b * P + p];
      const int s = row_segment(G, row);
      if (s < 0) continue;
      const RowSegment& o = G.s[s];
      const size_t r = (size_t)(row - o.row_begin);
      if (k == 0) {
        if (o.reward) *reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(o.reward) + r * o.reward_row_stride) = S.reward[(size_t)b * P + p];
      } else {
        *reinterpret_cast<double*>(reinterpret_cast<uint8_t*>(o.scalar_obs) + (size_t)(k - 1) * o.scalar_obs_stride + r * o.scalar_obs_row_stride) =
            S.scalar_obs[((size_t)(k - 1) * S.B + b) * P + p];
      }
    }
  }
}

// Delivery when no render follows the state transition (mp_step_state on its own, or rendering switched off).
// G: the per-player rows' segments (n = 0 when the call routes none).
__global__ void __launch_bounds__(256) k_exchange_push(Tables T, State S, const __grid_constant__ RowSegments G) {
  asm volatile("griddepcontrol.wait;" ::: "memory");
  exchange_push(T, S);
  deliver_scalars(T, S);
  deliver_player_scalars(T, S, G);
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
