// step_common.cuh -- the warp-per-env machinery every state-transition family shares.
//
// One warp advances one env instance; lanes are avatars, beam footprint cells or entities depending on the phase, and
// envs never interact, so nothing leaves the warp. This header holds what does not depend on a substrate's Lua
// components: the kernel skeleton (k_step), episode start, the step prologue, the frame's visiting order, the episode
// ending draw, move arbitration, beam footprints, respawn, the avatar sprites and the timestep store. A family
// (step_<family>.cuh) supplies its component logic through a struct of static functions and plugs per-family
// behaviour into the helpers below as lambdas.
#pragma once

#include <type_traits>

#include "common.cuh"
#include "state_bank.cuh"

__host__ __device__ inline size_t scratch_round16(size_t n) { return (n + 15) & ~(size_t)15; }

struct WarpScratch {  // per-warp shared memory, carved from the dynamic allocation
  uint8_t* occ;       // [cells_pad] 0 free, 1..P avatar p-1, 255 static piece on the avatar layer
  uint8_t* apple;     // [nA_pad] family-specific per-entity state
  uint8_t* dirt;      // [nD_pad] family-specific per-entity state
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

// A map-variant engine of a family that stages tables (territory) stages them per warp, from the env's own map, after the
// dependency wait and the env's variant promotion: the four envs of a CTA may play four maps (see k_step).
template <class Family, class Source>
constexpr bool kWarpTables = Family::kStagesTables && Family::kMapVariants && !std::is_same<Source, typename Family::Params>::value;

// Dynamic shared memory of one step launch: four env warps' scratch, then the family's per-CTA tables (one copy per warp
// with kWarpTables).
template <class Family>
__host__ __device__ inline size_t step_smem_bytes(const Tables& T, bool variants) {
  const bool per_warp = variants && Family::kStagesTables && Family::kMapVariants;
  return 4 * Family::scratch_bytes(T) + (per_warp ? 4 : 1) * Family::table_bytes(T);
}

// mode 0: step (envs whose last step was LAST start a new episode instead, policy A.17)
// mode 1: reset envs selected by `mask` (all if null)
//
// Per-env parameter variants (mp_create_variants): env b runs under params[active[b]]. An episode start first takes the
// env's pending assignment (active[b] = pending[b]), so a reassignment never changes an episode that is under way.
// The variants of a family without map variants stage the same per-CTA tables (the compatibility check of
// mp_create_variants), so stage() reads params[0].
// A family with kMapVariants (coins, commons_harvest, territory, coop_mining) also advances under maps[active[b]]: the
// engine's Tables with that variant's initial grid, static occupancy, BeamBlocker bits, spawn points, avatar sprites and
// entity count (the State's entity arrays are sized for the largest variant). Such a family may provide reset_map, which
// then starts the episodes of map-variant engines instead of reset (it also zeroes the env's entity bytes past its map's
// count). A map-variant family that stages tables (territory) stages them per warp (kWarpTables), from the env's own
// variant, once the dependency wait and the promotion have fixed it. The map is only ever read through the env's active
// variant, which changes at an episode start, so an env's map changes there too and never mid-episode. The Tables are read from the device array through the L1: a
// local copy of the kernel's Tables with the variant's fields swapped in would sit on the stack (392 bytes for coins,
// since avatar_sprite is indexed by lane).
// The variants of any other family may differ in their initial grid (appearance overrides: which sprite each piece
// shows), so their episode starts also read maps[k], whose Tables equal the kernel's except for init_grid; their steps
// read the kernel's Tables. Sprite ids are read from the env's Params, never from the per-CTA tables stage() builds from
// params[0] (which hold cell indices, walls and beam footprints only).
template <class Params>
struct ParamVariants {
  const Params* __restrict__ params;  // [n]
  uint8_t* active;                    // [B]
  const uint8_t* pending;             // [B]
  int n;
  const Tables* __restrict__ maps;    // [n] each variant's Tables (its map; for other families, its initial grid)
};

// The variant env b advances under: on an episode start its pending assignment, which lane 0 makes the active one; an
// index outside the set reads as variant 0.
template <class Params>
__device__ __forceinline__ int env_variant(const ParamVariants<Params>& V, int b, int lane, bool reset) {
  int k = reset ? V.pending[b] : V.active[b];
  if (k >= V.n) k = 0;
  if (reset && lane == 0) V.active[b] = (uint8_t)k;
  return k;
}

// Where a step's actions come from. DenseActions: an id per player, [B][P] (null on territory's frame 0: every avatar
// does nothing). RowActions (player_actions): player p of env b takes the id in row row_of_player[b][p] of `action`,
// rows `stride` bytes apart, or action 0 when that row lies outside [0, n_rows). The row is read on the avatar's lane
// where the action is decoded (load_avatar), so nothing of it stays live across the frame.
using DenseActions = const int32_t* __restrict__;
struct RowActions {
  const int32_t* row_of_player;  // [B][P]
  const uint8_t* action;         // [n_rows] x i32
  uint64_t stride;
  int n_rows;
};

template <class Actions>
__device__ __forceinline__ const Actions& select_actions(const DenseActions& dense, const RowActions& rows) {
  if constexpr (std::is_same<Actions, RowActions>::value) return rows;
  else return dense;
}

// Drawn routes (mp_run's draw, k_step_drawn): each episode, player slot p of env b plays choice
// o = pick(philox(0, episode, p, RS_ROUTE).x, n_choices[p]) under env b's key (uniform with replacement per slot and
// episode, like choice_present), and its row is base[p][o] + b * per_env[p][o]; a slot without choices has no row. The
// step reads player p's action from the row of the episode it is in, and writes every env's row map after the advance
// (row_of_player[b][p]: the row of the episode env b is in now, -1 for no row), which the render that follows reads.
// mp_run checks every row of the table against [0, n_rows) for every env, so a drawn row is always in range.
#define MP_ROUTE_CHOICES 8  // = MP_MAX_ROUTE_CHOICES (include/mp_engine.h)
struct DrawnActions {
  int32_t* row_of_player;  // [B][P], written
  const uint8_t* action;   // [n_rows] x i32
  uint64_t stride;
  int n_rows;
  int32_t n_choices[MP_MAX_PLAYERS];
  int32_t base[MP_MAX_PLAYERS][MP_ROUTE_CHOICES];
  int32_t per_env[MP_MAX_PLAYERS][MP_ROUTE_CHOICES];
};

__device__ __forceinline__ int drawn_row(const DrawnActions& d, int b, int p, int episode, uint32_t k0, uint32_t k1) {
  const int n = d.n_choices[p];
  if (n <= 0) return -1;
  const int o = (int)pick(philox4x32_10(0u, (uint32_t)episode, (uint32_t)p, RS_ROUTE, k0, k1).x, (uint32_t)n);
  return d.base[p][o] + b * d.per_env[p][o];
}

template <class F, class = void>
struct HasResetMap : std::false_type {};
template <class F>
struct HasResetMap<F, std::void_t<decltype(&F::reset_map)>> : std::true_type {};

// A Family provides: Params (what only its kernel reads), the host-side load(FamilyLoad&, T, Params&) that decodes its
// blob sections into Params and host tables (family_load.h), Scratch, kStagesTables, kMapVariants (whether its variants
// may differ in the map), kMapSections and kSpriteSections
// (the sections its variants may differ in, see same_sections in engine.cu; null if none), scratch_bytes(T) per warp, table_bytes(T) per CTA,
// stage(T, F, tables) (copies static tables into shared memory; with kMapVariants also stage_warp(T, F, tables, lane),
// one warp's copy), carve(T, warp_base, tables), reset(T, F, S, b, lane, sc)
// and step(T, F, S, b, lane, actions, sc) for either action source, and on the host same_shape(a, b) for per-env
// variants, which run under their own Params. `Source` is the family's Params (one blob) or ParamVariants<Params>. A single Params is a grid constant:
// without it, the compiler copies a small Params that is indexed with a run-time value (coins' coin_reward[who],
// coop_mining's ore_sprite[state]) to the stack, and passed on as it is, it keeps its constant-bank reads. Variants are
// read through the L1 from the device array.
//
// kRestore (a restoring mp_run, mode 0 only): the warp of an env that `restore` names (restore_env's predicate, read after
// the dependency wait) copies that record instead of advancing, which also takes precedence over the auto-reset after
// LAST; the record carries the timestep and the events, so event_begin / event_end are skipped too. Every other warp
// runs the plain step. With kRestore = false, `restore` is never read and the kernel is the plain step.
// Actions: DenseActions (`actions`; `rows` is never read), or RowActions (`rows`; launched by mp_run's player_actions only, mode 0,
// and `actions` is never read); k_step_drawn reads DrawnActions.
//
// k_step's body as a function, for k_step_drawn: stages the family's tables, waits for the kernel before, then restores
// or advances (or, masked out of a reset, leaves) this warp's env. Returns the env, or -1 for a warp past the batch.
// k_step keeps its own copy of these lines: calling this function from it schedules the 40 k_step instantiations
// differently (32 of them got other SASS, 17 other register or spill counts), which the copy avoids.
template <class Family, class Source, bool kRestore, class Actions>
__device__ __forceinline__ int advance_env(const Tables& T, const Source& src, const State& S, const uint8_t* __restrict__ mask,
                                           int mode, const StepRestore& restore, const Actions& acts) {
  constexpr bool kVariants = !std::is_same<Source, typename Family::Params>::value;
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Programmatic dependent launch, both ways: let the renderer that follows in the stream stage its tables while this
  // grid drains, and do not touch env state before the kernel that precedes this one (the previous render) is complete.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  uint8_t* tables = smem + 4 * Family::scratch_bytes(T);
  constexpr bool kCtaTables = Family::kStagesTables && !kWarpTables<Family, Source>;
  if constexpr (kCtaTables) {  // before the dependency wait: the tables never change
    if constexpr (kVariants) Family::stage(T, src.params[0], tables);
    else Family::stage(T, src, tables);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if constexpr (kCtaTables) __syncthreads();
  const int b = blockIdx.x * 4 + warp;
  if (b >= S.B) return -1;
  if constexpr (kRestore) {
    if (restore_env(*restore.layout, restore.slot_of_env, restore.bank, restore.n_slots, b, lane, restore.rekey, restore.key_base)) return b;
  }
  if constexpr (kWarpTables<Family, Source>) tables += warp * Family::table_bytes(T);
  typename Family::Scratch sc = Family::carve(T, smem + warp * Family::scratch_bytes(T), tables);
  if (!(mode == 1 && !(mask == nullptr || mask[b]))) {
    event_begin(lane);
    if constexpr (kVariants) {
      const bool reset = mode == 1 || S.env[(size_t)b * ENV_COLS + ENV_DONE];
      const int k = env_variant(src, b, lane, reset);
      const typename Family::Params& F = src.params[k];
      if constexpr (Family::kMapVariants) {
        const Tables& Tm = src.maps[k];
        if constexpr (kWarpTables<Family, Source>) {  // this env's map, known only now
          Family::stage_warp(Tm, F, tables, lane);
          __syncwarp();
        }
        if (reset) {
          if constexpr (HasResetMap<Family>::value) Family::reset_map(Tm, F, S, b, lane, sc);
          else Family::reset(Tm, F, S, b, lane, sc);
        } else Family::template step<Actions>(Tm, F, S, b, lane, acts, sc);
      } else {  // the variants differ in their initial grid only (appearance overrides): an episode start reads maps[k]
        if (reset) Family::reset(src.maps[k], F, S, b, lane, sc);
        else Family::template step<Actions>(T, F, S, b, lane, acts, sc);
      }
    } else {
      if (mode == 1 || S.env[(size_t)b * ENV_COLS + ENV_DONE]) Family::reset(T, src, S, b, lane, sc);
      else Family::template step<Actions>(T, src, S, b, lane, acts, sc);
    }
    event_end(S, b, lane);
  }
  return b;
}

template <class Family, class Source = typename Family::Params, bool kRestore = false, class Actions = DenseActions>
__global__ void __launch_bounds__(128, 8) k_step(Tables T, const __grid_constant__ Source src, State S, const int32_t* __restrict__ actions,
                                                 const uint8_t* __restrict__ mask, int mode, const __grid_constant__ StepRestore restore,
                                                 const __grid_constant__ RowActions rows) {
  constexpr bool kVariants = !std::is_same<Source, typename Family::Params>::value;
  const Actions& acts = select_actions<Actions>(actions, rows);
  extern __shared__ __align__(128) uint8_t smem[];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  // Programmatic dependent launch, both ways: let the renderer that follows in the stream stage its tables while this
  // grid drains, and do not touch env state before the kernel that precedes this one (the previous render) is complete.
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");
  uint8_t* tables = smem + 4 * Family::scratch_bytes(T);
  constexpr bool kCtaTables = Family::kStagesTables && !kWarpTables<Family, Source>;
  if constexpr (kCtaTables) {  // before the dependency wait: the tables never change
    if constexpr (kVariants) Family::stage(T, src.params[0], tables);
    else Family::stage(T, src, tables);
  }
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if constexpr (kCtaTables) __syncthreads();
  const int b = blockIdx.x * 4 + warp;
  if (b >= S.B) return;
  if constexpr (kRestore) {
    if (restore_env(*restore.layout, restore.slot_of_env, restore.bank, restore.n_slots, b, lane, restore.rekey, restore.key_base)) return;
  }
  if constexpr (kWarpTables<Family, Source>) tables += warp * Family::table_bytes(T);
  typename Family::Scratch sc = Family::carve(T, smem + warp * Family::scratch_bytes(T), tables);
  if (!(mode == 1 && !(mask == nullptr || mask[b]))) {
    event_begin(lane);
    if constexpr (kVariants) {
      const bool reset = mode == 1 || S.env[(size_t)b * ENV_COLS + ENV_DONE];
      const int k = env_variant(src, b, lane, reset);
      const typename Family::Params& F = src.params[k];
      if constexpr (Family::kMapVariants) {
        const Tables& Tm = src.maps[k];
        if constexpr (kWarpTables<Family, Source>) {  // this env's map, known only now
          Family::stage_warp(Tm, F, tables, lane);
          __syncwarp();
        }
        if (reset) {
          if constexpr (HasResetMap<Family>::value) Family::reset_map(Tm, F, S, b, lane, sc);
          else Family::reset(Tm, F, S, b, lane, sc);
        } else Family::template step<Actions>(Tm, F, S, b, lane, acts, sc);
      } else {  // the variants differ in their initial grid only (appearance overrides): an episode start reads maps[k]
        if (reset) Family::reset(src.maps[k], F, S, b, lane, sc);
        else Family::template step<Actions>(T, F, S, b, lane, acts, sc);
      }
    } else {
      if (mode == 1 || S.env[(size_t)b * ENV_COLS + ENV_DONE]) Family::reset(T, src, S, b, lane, sc);
      else Family::template step<Actions>(T, src, S, b, lane, acts, sc);
    }
    event_end(S, b, lane);
  }
}

// k_step with drawn routes (mp_run's draw: a step, mode 0, or a reset, mode 1): the same advance, with actions from
// the rows of DrawnActions; then every env's row map is written from the episode and key the env now has, whether it
// advanced, started an episode, was restored (a record's key, or its own with rekey) or was masked out of a reset.
// `actions` and `rows` are those of k_step, so one argument list launches either kernel; neither is read here.
template <class Family, class Source = typename Family::Params, bool kRestore = false>
__global__ void __launch_bounds__(128, 8) k_step_drawn(Tables T, const __grid_constant__ Source src, State S, const int32_t* __restrict__ actions,
                                                       const uint8_t* __restrict__ mask, int mode, const __grid_constant__ StepRestore restore,
                                                       const __grid_constant__ DrawnActions drawn) {
  const int b = advance_env<Family, Source, kRestore, DrawnActions>(T, src, S, mask, mode, restore, drawn);
  if (b < 0) return;
  __syncwarp();  // the env row and key were written by lanes of this warp
  const int lane = threadIdx.x & 31;
  if (lane < T.P) {
    const uint64_t key = *reinterpret_cast<volatile const uint64_t*>(S.key + b);
    const int episode = *reinterpret_cast<volatile const int32_t*>(S.env + (size_t)b * ENV_COLS + ENV_EPISODE);
    drawn.row_of_player[(size_t)b * T.P + lane] = drawn_row(drawn, b, lane, episode, (uint32_t)key, (uint32_t)(key >> 32));
  }
}

// What an advance of env b starts from: its env row, its sprite grid, its Philox key (State::key), and the frame number
// and episode it runs (frame 0 of the next episode on a reset).
//
// The key is per-env state (State::key) that no state-transition kernel writes, so each of its two words is read where
// it is used instead of once here: a value loaded up front would stay live in two registers across the whole advance,
// and the step kernels run at their 64-register cap (k_step<CleanUp> spilled 72 bytes more that way). The volatile read
// keeps the compiler from merging the reads back into one.
struct KeyWord {
  const uint32_t* p;
  __device__ __forceinline__ operator uint32_t() const { uint32_t v; asm volatile("ld.global.nc.u32 %0, [%1];" : "=r"(v) : "l"(p)); return v; }
};
struct Frame {
  int32_t* env;
  uint16_t* grid;
  KeyWord k0, k1;
  int n, episode;
};
__device__ __forceinline__ Frame begin_frame(const Tables& T, const State& S, int b, bool reset) {
  Frame f;
  f.env = S.env + (size_t)b * ENV_COLS;
  f.grid = S.grid + (size_t)b * T.L * T.cells_pad;
  f.k0.p = reinterpret_cast<const uint32_t*>(S.key + b); f.k1.p = f.k0.p + 1;
  f.n = reset ? 0 : f.env[ENV_STEP] + 1;
  f.episode = f.env[ENV_EPISODE] + (reset ? 1 : 0);
  return f;
}

// ---------------------------------------------------------------------------------------------
// Episode start: api:start (api_factory.lua:85-102) + BaseSimulation:start/_avatarStart
// (base_simulation.lua:396-471) + the frame-0 grid:update.
// ---------------------------------------------------------------------------------------------
// Static pieces and initial states.
__device__ __forceinline__ void copy_init_grid(const Tables& T, uint16_t* grid, int lane) {
  const uint4* src = reinterpret_cast<const uint4*>(T.init_grid);
  uint4* dst = reinterpret_cast<uint4*>(grid);
  const int n16 = T.L * T.cells_pad / 8;
  for (int i = lane; i < n16; i += 32) dst[i] = src[i];
}

// _avatarStart for one spawn group (base_simulation.lua:396-445): the group's members this episode (`present(i)` of
// candidate i, in piece order; 'choice' spawn points are drawn per episode) are shuffled by groupShuffledWithCount as a
// partial Fisher-Yates, one draw per avatar of the group (`in_group(p)`) in avatar order, and the group's j-th avatar
// takes the j-th cell. Avatar:start (avatar_library.lua:299-304) gives it a random orientation, alive, zeroed timers and
// its sprite; place(lane, cell) then runs on the avatar's lane. tmp holds 64 cells (mp_create refuses larger groups).
template <class InGroup, class Present, class Place>
__device__ __forceinline__ void spawn_group(const Tables& T, const State& S, int b, int lane, uint16_t* grid, int16_t* tmp,
                                            const int32_t* cells, int n_cells, InGroup in_group, Present present,
                                            int episode, uint32_t k0, uint32_t k1, Place place) {
  int n = 0;
  for (int base = 0; base < n_cells && base < 64; base += 32) {
    const int i = base + lane;
    const bool on = i < n_cells && present(i);
    const unsigned m = __ballot_sync(MP_FULL, on);
    if (on) tmp[n + __popc(m & ((1u << lane) - 1u))] = (int16_t)cells[i];
    n += __popc(m);
  }
  __syncwarp();
  const unsigned members = __ballot_sync(MP_FULL, lane < T.P && in_group(lane));
  if (lane == 0) {
    int j = 0;
    for (int p = 0; p < T.P; ++p) {
      if (!(members >> p & 1u)) continue;
      uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)p, RS_AVATAR_RESET, k0, k1);
      int r = j + (int)pick(w.x, (uint32_t)(n - j));
      int16_t t = tmp[j]; tmp[j] = tmp[r]; tmp[r] = t;
      ++j;
    }
  }
  __syncwarp();
  if (members >> lane & 1u) {
    uint4 w = philox4x32_10(0u, (uint32_t)episode, (uint32_t)lane, RS_AVATAR_RESET, k0, k1);
    const int cell = tmp[__popc(members & ((1u << lane) - 1u))], orient = (int)(w.y & 3u);
    *reinterpret_cast<int4*>(S.avatar + ((size_t)b * T.P + lane) * 4) = make_int4(cell % T.W, cell / T.W, orient, 1);
    *reinterpret_cast<int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4) = make_int4(0, 0, 0, 0);
    grid[(size_t)T.avatar_layer * T.cells_pad + cell] = cell_value(T.avatar_sprite[lane], orient);
    place(cell);
  }
  __syncwarp();
}

// Timestep of frame n: every avatar's reward (lanes < P) and, on lane 0, the discount and step type (FIRST 0, MID 1,
// LAST 2) into the outputs and the packed row, and the env row's frame counter, done flag and hit-sprite flags. The
// discount is 1 on MID steps only (multiplayer_wrapper.py:117 turns FIRST's None into 0.).
__device__ __forceinline__ void store_timestep(const Tables& T, const State& S, int b, int lane, int n, double reward,
                                               int step_type, int beam_dirty) {
  if (lane < T.P) {
    S.reward[(size_t)b * T.P + lane] = reward;
    S.packed[(size_t)b * (T.P + 2) + lane] = reward;
  }
  if (lane == 0) {
    int32_t* env = S.env + (size_t)b * ENV_COLS;
    env[ENV_STEP] = n; env[ENV_DONE] = step_type == 2 ? 1 : 0; env[ENV_BEAM] = beam_dirty;
    const double discount = step_type == 1 ? 1.0 : 0.0;
    S.discount[b] = discount; S.step_type[b] = step_type;
    S.packed[(size_t)b * (T.P + 2) + T.P] = discount; S.packed[(size_t)b * (T.P + 2) + T.P + 1] = (double)step_type;
  }
}

// The env row of a new episode, and its FIRST timestep with zero rewards.
__device__ __forceinline__ void reset_env_row(const Tables& T, const State& S, int b, int lane, int episode, int dirt_count) {
  if (lane == 0) {
    int32_t* env = S.env + (size_t)b * ENV_COLS;
    env[ENV_EPISODE] = episode; env[ENV_DIRT] = dirt_count; env[ENV_CLEANED] = 0; env[ENV_ATE] = 0;
  }
  store_timestep(T, S, b, lane, 0, 0.0, 0, 0);
  __syncwarp();
}

// ---------------------------------------------------------------------------------------------
// One frame
// ---------------------------------------------------------------------------------------------
// The action id of player i = b * P + p (see DenseActions / RowActions); null dense actions are no actions. Actions
// are read-only for the whole step, so they are read through the non-coherent path.
__device__ __forceinline__ bool has_actions(DenseActions actions) { return actions != nullptr; }
__device__ __forceinline__ bool has_actions(const RowActions&) { return true; }
__device__ __forceinline__ bool has_actions(const DrawnActions&) { return true; }
__device__ __forceinline__ int action_id(DenseActions actions, const State&, int b, int P, int lane) {
  const size_t i = (size_t)b * P + lane;
  return __ldg(actions + i);
}
__device__ __forceinline__ int action_id(const RowActions& a, const State&, int b, int P, int lane) {
  const size_t i = (size_t)b * P + lane;
  const int row = __ldg(a.row_of_player + i);
  return (uint32_t)row < (uint32_t)a.n_rows ? __ldg(reinterpret_cast<const int32_t*>(a.action + (size_t)row * a.stride)) : 0;
}
// The row of the episode a stepping env is in (its key is never written by a stepping env's warp, see KeyWord).
__device__ __forceinline__ int action_id(const DrawnActions& a, const State& S, int b, int, int lane) {
  const uint64_t key = __ldg(reinterpret_cast<const unsigned long long*>(S.key + b));
  const int row = drawn_row(a, b, lane, S.env[(size_t)b * ENV_COLS + ENV_EPISODE], (uint32_t)key, (uint32_t)(key >> 32));
  return row >= 0 ? __ldg(reinterpret_cast<const int32_t*>(a.action + (size_t)row * a.stride)) : 0;
}

// This lane's avatar (x, y, orientation, alive), its timers, and its action decoded by the action table
// (discrete_action_wrapper.py:97-100; an id out of range is action 0). Zeros on lanes >= P, and for the action when
// `actions` is null (territory's frame 0: every avatar does nothing).
template <class Actions>
__device__ __forceinline__ void load_avatar(const Tables& T, const State& S, int b, int lane, const Actions& actions,
                                            const int32_t* act_table, int4& av, int4& timer, int4& act) {
  av = timer = act = make_int4(0, 0, 0, 0);
  if (lane < T.P) {
    av = *reinterpret_cast<const int4*>(S.avatar + ((size_t)b * T.P + lane) * 4);
    timer = *reinterpret_cast<const int4*>(S.av_timer + ((size_t)b * T.P + lane) * 4);
    if (has_actions(actions)) {
      int id = action_id(actions, S, b, T.P, lane);
      if (id < 0 || id >= T.n_actions) id = 0;
      act = *reinterpret_cast<const int4*>(act_table + id * 4);
    }
  }
}

// Occupancy of the avatar layer as the frame starts: the static pieces (`solid`, cells_pad bytes) plus every avatar on
// the map, written by its own lane. Call __syncwarp before the next reader.
__device__ __forceinline__ void init_occupancy(const Tables& T, uint8_t* occ, const uint8_t* solid, int lane) {
  for (int i = lane; i < T.cells_pad / 8; i += 32) reinterpret_cast<uint2*>(occ)[i] = reinterpret_cast<const uint2*>(solid)[i];
}

// Hit sprites live for one frame (policy A.8): a beam layer the last frame drew into is cleared.
__device__ __forceinline__ void clear_layer(const Tables& T, uint16_t* grid, int layer, int lane) {
  const uint4 z = make_uint4(0, 0, 0, 0);
  uint4* l = reinterpret_cast<uint4*>(grid + (size_t)layer * T.cells_pad);
  for (int i = lane; i < T.cells_pad / 8; i += 32) l[i] = z;
}

// Avatars are visited in a fresh random order each frame (policy A.7): this lane's avatar's rank, 99 on lanes >= P.
__device__ __forceinline__ int visit_rank(const Tables& T, int lane, int n, int episode, uint32_t k0, uint32_t k1) {
  const uint32_t mykey = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)lane, RS_AVATAR, k0, k1).x;
  int rank = 0;
  for (int q = 0; q < T.P; ++q) {
    const uint32_t kq = __shfl_sync(MP_FULL, mykey, q);
    if (kq < mykey || (kq == mykey && q < lane)) ++rank;
  }
  return lane < T.P ? rank : 99;
}

// StochasticIntervalEpisodeEnding (component_library.lua:927-948); its _t equals n + 1. False when the episode ends.
__device__ __forceinline__ bool episode_continues(const Tables& T, int n, int episode, uint32_t k0, uint32_t k1) {
  if (n >= T.end_min_frames && ((n + 1) % T.end_interval) == 0) {
    uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, SCENE_DRAW_EPISODE_END, RS_SCENE, k0, k1);
    if (u01(w.x, w.y) < T.end_prob) return false;
  }
  return true;
}

// Avatar move (avatar_library.lua:156-171), avatar by avatar in this frame's order: turn, then one step if the target
// cell is on the map and free. Only avatars with `may_move` act. When the action moves, contact(src, cell) runs on every
// lane with the final cell, even when the step was blocked (place -> contact enter, policy A.5).
// One shuffle instead of six: may_move | turn + 1 | move | orient | y | x; exact because mp_create refuses maps of 4096
// cells or more, so x and y fit in 12 bits.
template <class Contact>
__device__ __forceinline__ void move_avatars(const Tables& T, int lane, int rank, bool may_move, int act_turn, int act_move,
                                             int& x, int& y, int& orient, uint8_t* occ, Contact contact) {
  for (int r = 0; r < T.P; ++r) {
    const unsigned m = __ballot_sync(MP_FULL, lane < T.P && rank == r);
    const int src = __ffs(m) - 1;
    const uint32_t packed = __shfl_sync(MP_FULL, (uint32_t)may_move | ((uint32_t)(act_turn + 1) << 1) | ((uint32_t)act_move << 3) |
                                                     ((uint32_t)orient << 6) | ((uint32_t)y << 8) | ((uint32_t)x << 20), src);
    if (!(packed & 1u)) continue;
    const int s_turn = (int)((packed >> 1) & 3u) - 1, s_move = (int)((packed >> 3) & 7u);
    int so = (int)((packed >> 6) & 3u), sy = (int)((packed >> 8) & 0xfffu), sx = (int)(packed >> 20);
    if (s_turn != 0) so = (so + s_turn) & 3;
    if (s_move != 0) {
      const int d = (so + s_move - 1) & 3;
      int nx = sx + dir_dx(d), ny = sy + dir_dy(d);
      if (wrap_or_reject(T, nx, ny) && occ[ny * T.W + nx] == 0) {
        __syncwarp();
        if (lane == 0) { occ[sy * T.W + sx] = 0; occ[ny * T.W + nx] = (uint8_t)(src + 1); }
        sx = nx; sy = ny;
      }
      contact(src, sy * T.W + sx);
    }
    if (lane == src) { x = sx; y = sy; orient = so; }
    __syncwarp();
  }
}

// Footprint cell `lane` of beam G fired from (sx, sy) facing so, or -1 past the footprint or off a BOUNDED map.
__device__ __forceinline__ int beam_cell(const Tables& T, const BeamGeom& G, int lane, int sx, int sy, int so) {
  if (lane >= G.n) return -1;
  const int rgt = (so + 1) & 3;
  int cx = sx + dir_dx(so) * G.fwd[lane] + dir_dx(rgt) * G.lat[lane];
  int cy = sy + dir_dy(so) * G.fwd[lane] + dir_dy(rgt) * G.lat[lane];
  return wrap_or_reject(T, cx, cy) ? cy * T.W + cx : -1;
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

// The first beam of the frame to pass a cell draws its hit sprite there; `drawn` marks the cells that carry one.
__device__ __forceinline__ void draw_hit_sprite(const Tables& T, uint16_t* grid, uint32_t* drawn, int layer, int cell, uint16_t value) {
  const uint32_t bit = 1u << (cell & 31);
  if (!(atomicOr(&drawn[cell >> 5], bit) & bit)) grid[(size_t)layer * T.cells_pad + cell] = value;
}

// teleportToGroup for respawning avatars (policy A.9), in this frame's order: a random cell of the respawn group; if it
// is occupied the updater fires again next frame. arrive(src, cell) runs on every lane once the cell is taken.
template <class Arrive>
__device__ __forceinline__ void respawn_avatars(const Tables& T, int lane, int rank, bool want_respawn, int n, int episode,
                                                uint32_t k0, uint32_t k1, uint8_t* occ, int& x, int& y, int& orient,
                                                int& alive, int& state_frame, Arrive arrive) {
  for (int r = 0; r < T.P; ++r) {
    const unsigned m = __ballot_sync(MP_FULL, lane < T.P && rank == r && want_respawn);
    if (!m) continue;
    const int src = __ffs(m) - 1;
    const uint4 w = philox4x32_10((uint32_t)n, (uint32_t)episode, (uint32_t)src, RS_AVATAR, k0, k1);
    const int target = T.spawn_cell[pick(w.y, (uint32_t)T.n_spawn)];
    if (occ[target] != 0) continue;
    __syncwarp();
    if (lane == 0) occ[target] = (uint8_t)(src + 1);
    arrive(src, target);
    if (lane == src) { x = target % T.W; y = target / T.W; orient = (int)(w.z & 3u); alive = 1; state_frame = n; }
    __syncwarp();
  }
}

// Avatar sprites: every changed avatar clears its old cell, then draws its new one (after the barrier, so that an
// avatar that moved onto a cell another one left is not erased). Returns whether this lane's avatar changed.
__device__ __forceinline__ bool draw_avatars(const Tables& T, uint16_t* grid, int lane, int x0, int y0, int orient0, int alive0,
                                             int x, int y, int orient, int alive) {
  const bool changed = lane < T.P && (x != x0 || y != y0 || orient != orient0 || alive != alive0);
  if (changed && alive0) grid[(size_t)T.avatar_layer * T.cells_pad + y0 * T.W + x0] = 0;
  __syncwarp();
  if (changed && alive) grid[(size_t)T.avatar_layer * T.cells_pad + y * T.W + x] = cell_value(T.avatar_sprite[lane], orient);
  return changed;
}
