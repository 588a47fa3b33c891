// engine.cu -- host side of libmpengine.so: blob -> device tables, state allocation, launches, C ABI.
// See include/mp_engine.h for the boundary contract. No CPU implementation of the path exists in
// this library: without a CUDA device every entry point fails with MP_E_NO_DEVICE / MP_E_CUDA.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdio>
#include <cstring>
#include <map>
#include <string>
#include <variant>
#include <vector>

#include "../../include/mp_engine.h"
#include "../../include/mpb_format.h"
#include "common.cuh"
#include "family_load.h"
#include "render.cuh"
#include "step_clean_up.cuh"
#include "step_commons.cuh"
#include "step_territory.cuh"
#include "step_coins.cuh"
#include "step_mining.cuh"
#include "state_bank.cuh"

static_assert(MP_MAX_ROUTE_CHOICES == MP_ROUTE_CHOICES && MP_MAX_ROUTE_PLAYERS == MP_MAX_PLAYERS,
              "mp_route_draw's table is DrawnActions'");
namespace {

constexpr int kRenderSmemLimit = 227 * 1024 - 2560;  // dynamic shared memory: the 227 KB opt-in maximum less k_render's static arrays
constexpr int kMaxAtlasSprites = 96;
#define MP_MAX_DEVICES 64
#define MP_EXCHANGE_HEADER 256  // bytes reserved for the per-rank flags in front of the gathered rows  // sprites incl. pre-merged ones kept in shared memory by k_render

// Deals the cells of one strip to lanes so that the 64-bit staging stores of every half-warp are bank-conflict free.
// A strip is `n_rows` pixel rows (8 for a player cell-row, 4 or 2 for WORLD.RGB) by `n_cells` cells of 24 bytes at a
// row pitch of `pitch_slots` 8-byte slots; lane l draws pixel row l % n_rows in each of its `iters` turns. A 64-bit
// shared store is served per half-warp and lane (row j, cell c) touches bank pair (pitch_slots * j + 3 * c) mod 16,
// so each half-warp turn may hold every residue once and every row 16 / n_rows times: an edge colouring of the
// bipartite multigraph rows x residues with one colour per half-warp turn (Koenig: it exists whenever no residue occurs
// more often than there are half-warp turns). Returns false in that case (the caller keeps the plain dealing).
bool make_lane_map(int n_rows, int n_cells, int pitch_slots, int iters, uint32_t out[32]) {
  const int cap = 16 / n_rows, nH = 2 * iters;
  struct Edge { int u, v, cell, col; };
  std::vector<Edge> edges;
  int cnt[16] = {};
  for (int j = 0; j < n_rows; ++j)
    for (int c = 0; c < n_cells; ++c) {
      const int r = (pitch_slots * j + 3 * c) & 15;
      edges.push_back({j * cap + c % cap, r, c, -1});
      if (++cnt[r] > nH) return false;
    }
  if (n_cells > cap * nH || iters * 6 > 32) return false;
  const int nL = n_rows * cap;
  std::vector<int> colL((size_t)nL * nH, -1), colR((size_t)16 * nH, -1);  // (vertex, colour) -> edge
  auto free_col = [&](const std::vector<int>& tab, int v) { for (int a = 0; a < nH; ++a) if (tab[(size_t)v * nH + a] < 0) return a; return -1; };
  for (int ei = 0; ei < (int)edges.size(); ++ei) {
    Edge& e = edges[ei];
    const int a = free_col(colL, e.u), b = free_col(colR, e.v);
    if (a < 0 || b < 0) return false;
    if (a != b) {  // swap colours a / b along the alternating path that starts at e.v with colour a
      std::vector<int> path;
      int cur = e.v, want = a; bool right = true;
      for (;;) {
        const int pe = right ? colR[(size_t)cur * nH + want] : colL[(size_t)cur * nH + want];
        if (pe < 0) break;
        path.push_back(pe);
        cur = right ? edges[pe].u : edges[pe].v;
        right = !right;
        want = want == a ? b : a;
      }
      for (int pe : path) { colL[(size_t)edges[pe].u * nH + edges[pe].col] = -1; colR[(size_t)edges[pe].v * nH + edges[pe].col] = -1; }
      for (int pe : path) { edges[pe].col = edges[pe].col == a ? b : a; colL[(size_t)edges[pe].u * nH + edges[pe].col] = pe; colR[(size_t)edges[pe].v * nH + edges[pe].col] = pe; }
    }
    e.col = a;
    colL[(size_t)e.u * nH + a] = ei; colR[(size_t)e.v * nH + a] = ei;
  }
  for (int l = 0; l < 32; ++l) { out[l] = 0; for (int i = 0; i < iters; ++i) out[l] |= 63u << (6 * i); }
  for (const Edge& e : edges) {
    const int j = e.u / cap, sub = e.u % cap, it = e.col / 2, half = e.col % 2;
    const int lane = 16 * half + sub * n_rows + j;
    out[lane] = (out[lane] & ~(63u << (6 * it))) | ((uint32_t)e.cell << (6 * it));
  }
  return true;
}

// The dealing used by default: every cell keeps all its pixel rows on `n_rows` consecutive lanes and in ONE turn (so a
// multi-sprite cell sends a warp through the slow compositing path once, not once per turn it was scattered over), and
// only WHICH cell sits on which lane group in which turn is chosen, to minimise the extra wavefronts of the staging
// stores: sum over half-warp turns of (largest number of lanes on one bank pair - 1). Steepest-descent over pair swaps
// from the plain dealing; deterministic. Returns the remaining extra wavefronts per strip.
int make_lane_map_cells(int n_rows, int n_cells, int pitch_slots, int iters, uint32_t out[32]) {
  const int G = 32 / n_rows, n_slots = G * iters, per_half = 16 / n_rows;
  std::vector<int> slot(n_slots, -1);
  for (int c = 0; c < n_cells && c < n_slots; ++c) slot[c] = c;  // plain: slot index = turn * G + group
  auto cost = [&]() {
    int total = 0;
    for (int it = 0; it < iters; ++it)
      for (int h = 0; h < 2; ++h) {
        int cnt[16] = {}, mx = 0;
        for (int g = h * per_half; g < (h + 1) * per_half; ++g) {
          const int c = slot[it * G + g];
          if (c < 0) continue;
          for (int j = 0; j < n_rows; ++j) mx = std::max(mx, ++cnt[(pitch_slots * j + 3 * c) & 15]);
        }
        total += mx > 1 ? mx - 1 : 0;
      }
    return total;
  };
  int best = cost();
  for (bool improved = true; improved && best > 0;) {
    improved = false;
    int bi = -1, bj = -1, bc = best;
    for (int i = 0; i < n_slots; ++i)
      for (int j = i + 1; j < n_slots; ++j) {
        if (slot[i] == slot[j]) continue;
        std::swap(slot[i], slot[j]);
        const int c = cost();
        if (c < bc) { bc = c; bi = i; bj = j; }
        std::swap(slot[i], slot[j]);
      }
    if (bi >= 0) { std::swap(slot[bi], slot[bj]); best = bc; improved = true; }
  }
  for (int l = 0; l < 32; ++l) {
    out[l] = 0;
    for (int it = 0; it < 5; ++it) {
      const int c = it < iters ? slot[it * G + l / n_rows] : -1;
      out[l] |= (uint32_t)(c < 0 ? 63 : c) << (6 * it);
    }
  }
  return best;
}

// One row per substrate family: the blob decode into the family's Params (host, step_<family>.cuh) and the
// state-transition kernel with the dynamic shared memory one launch of it takes. An engine keeps the Params of its
// family in a FamilyParams; only the row's own functions look inside it.
using FamilyParams = std::variant<CleanUp::Params, Commons::Params, Territory::Params, Coins::Params, Mining::Params>;
// The per-env variant set of an engine (mp_create_variants): the device array of Params and the per-env assignments.
struct VariantSet {
  const void* params = nullptr;  // Family::Params [n]
  uint8_t* active = nullptr;     // [B] the variant each env's current episode runs
  uint8_t* pending = nullptr;    // [B] the variant each env's next episode runs
  int n = 1;
  const Tables* maps = nullptr;  // [n] the Tables of each variant (its map, or for other families its initial grid)
};
struct FamilyEntry {
  int id;  // MpbFamily
  bool map_variants;  // Family::kMapVariants: its variants may be draws of different maps (mp_create_variants)
  const char* const* map_sections;  // Family::kMapSections: its own entity tables, which such variants may differ in, or null
  const char* const* sprite_sections;  // Family::kSpriteSections: its int32 tables that hold nothing but sprite ids, or null
  int (*load)(FamilyLoad&, const Tables&, FamilyParams&);
  size_t (*step_smem)(const Tables&, bool variants);
  // per-env variants: same_shape(a, b) (MP_OK or MP_E_UNSUPPORTED naming the field) and the upload of every variant's
  // own Params
  int (*same_shape)(const FamilyParams&, const FamilyParams&);
  int (*upload_variants)(std::vector<void*>&, const std::vector<FamilyParams>&, const void**);
  // Every k_step<Family, ...> an engine may launch, [variants][restore][actions]: Source Params or ParamVariants<Params>
  // (mp_create_variants), kRestore (a step that restores envs from a bank), and the action source: DenseActions,
  // RowActions (mp_run's player_actions) or drawn routes (k_step_drawn: mp_run's draw; a drawn reset without restore).
  const void* step[2][2][3];
  // Launches `kernel`, one of `step`, with the kernel arguments `args` after filling in its Source argument (args[1]):
  // `params` for one blob, or the ParamVariants<Params> of `variants`.
  cudaError_t (*launch)(const cudaLaunchConfig_t&, const void* kernel, void** args, const FamilyParams& params, const VariantSet& variants);
};

template <class Family>
int load_family(FamilyLoad& ld, const Tables& T, FamilyParams& params) {
  return Family::load(ld, T, params.emplace<typename Family::Params>());
}
template <class Family>
int same_shape_family(const FamilyParams& a, const FamilyParams& b) {
  return Family::same_shape(std::get<typename Family::Params>(a), std::get<typename Family::Params>(b));
}
template <class Family>
int upload_variants_family(std::vector<void*>& allocs, const std::vector<FamilyParams>& variants, const void** out) {
  using P = typename Family::Params;
  std::vector<P> host;
  for (const FamilyParams& v : variants) host.push_back(std::get<P>(v));
  const P* d = nullptr;
  int rc = upload(allocs, host, &d);
  *out = d;
  return rc;
}
template <class Family>
cudaError_t launch_family(const cudaLaunchConfig_t& cfg, const void* kernel, void** args, const FamilyParams& params, const VariantSet& V) {
  using P = typename Family::Params;
  ParamVariants<P> variants{static_cast<const P*>(V.params), V.active, V.pending, V.n, V.maps};
  args[1] = V.n > 1 ? static_cast<void*>(&variants) : const_cast<P*>(&std::get<P>(params));
  return cudaLaunchKernelExC(&cfg, kernel, args);
}
template <class Family, class Source, bool kRestore, class Actions>
const void* step_kernel() {
  return reinterpret_cast<const void*>(k_step<Family, Source, kRestore, Actions>);
}
template <class Family, class Source, bool kRestore>
const void* drawn_kernel() {
  return reinterpret_cast<const void*>(k_step_drawn<Family, Source, kRestore>);
}
template <class Family>
FamilyEntry family_entry(int id) {
  using P = typename Family::Params;
  using V = ParamVariants<P>;
  return {id, Family::kMapVariants, Family::kMapSections, Family::kSpriteSections, load_family<Family>, step_smem_bytes<Family>,
          same_shape_family<Family>, upload_variants_family<Family>,
          {{{step_kernel<Family, P, false, DenseActions>(), step_kernel<Family, P, false, RowActions>(), drawn_kernel<Family, P, false>()},
            {step_kernel<Family, P, true, DenseActions>(), step_kernel<Family, P, true, RowActions>(), drawn_kernel<Family, P, true>()}},
           {{step_kernel<Family, V, false, DenseActions>(), step_kernel<Family, V, false, RowActions>(), drawn_kernel<Family, V, false>()},
            {step_kernel<Family, V, true, DenseActions>(), step_kernel<Family, V, true, RowActions>(), drawn_kernel<Family, V, true>()}}},
          launch_family<Family>};
}
const FamilyEntry kFamilies[] = {
    family_entry<CleanUp>(MPB_FAMILY_CLEAN_UP),
    family_entry<Commons>(MPB_FAMILY_COMMONS_HARVEST),
    family_entry<Territory>(MPB_FAMILY_TERRITORY),
    family_entry<Coins>(MPB_FAMILY_COINS),
    family_entry<Mining>(MPB_FAMILY_COOP_MINING),
};
const FamilyEntry* find_family(int id) {
  for (const FamilyEntry& f : kFamilies) if (f.id == id) return &f;
  return nullptr;
}

}  // namespace

struct mp_engine {
  int device = 0;
  int B = 0;
  uint32_t flags = MP_FLAG_DEFAULT;
  const FamilyEntry* family = nullptr;
  int n_total = 0;  // atlas sprites incl. pre-merged
  Tables T{};
  FamilyParams params;
  State S{};
  RenderPlan R{};
  mp_buffers buffers{};
  std::vector<void*> allocs;
  int32_t* d_actions = nullptr;  // staging for mp_step_host
  // one allocation holding reward | discount | step_type | scalar_obs, so the host path moves them with one copy
  uint8_t* scalar_block = nullptr;
  size_t scalar_block_bytes = 0;
  // mp_step_host_async: two slots, each with its own observation images, action staging and scalar staging
  struct AsyncSlot { uint8_t* rgb = nullptr; uint8_t* world_rgb = nullptr; int32_t* actions = nullptr; uint8_t* scalars = nullptr;
                     cudaEvent_t computed = nullptr, copied = nullptr; };
  AsyncSlot slot[2];
  cudaStream_t copy_stream = nullptr;
  bool async_ready = false;
  // mp_exchange_*: this rank's gathered / flags buffers and the launch sequence number
  uint8_t* x_block = nullptr;      // [flags: MP_EXCHANGE_HEADER bytes][gathered f64 [2][world * B][P + 2]]
  uint64_t x_block_bytes = 0;
  unsigned long long x_seq = 0;   // incremented by every state-transition launch once the exchange is connected
  bool x_pending_raise = false;   // a state transition published and the flags are to be raised by the render that follows
  int32_t* d_avatar_dbg = nullptr;
  uint64_t launches = 0;
  int sm_count = 0;
  size_t step_smem = 0;  // dynamic shared memory of one state-transition launch
  // k_render<inst_ncp, inst_ncw, mode> by mode: RENDER_PLAIN, RENDER_GATHER (mp_gather_obs_*), RENDER_ROUTED (player rows)
  void (*render_fns[3])(Tables, State, RenderPlan, uint32_t, RowSegments) = {};
  // mp_gather_obs_*: this rank's stacked-observation block [flags 256 B][2 slots][rgb of all ranks | world_rgb of all ranks]
  uint8_t* g_block = nullptr;
  uint64_t g_block_bytes = 0, g_slot_bytes = 0, g_world_off = 0;
  uint8_t* g_peer[MP_MAX_PEERS] = {};
  unsigned long long** d_g_flag_ptrs = nullptr;  // device array of every rank's flags pointer (for k_gather_raise)
  int g_world = 0, g_rank = 0;
  unsigned long long g_seq = 0;
  uint64_t algo_bytes = 0, render_bytes = 0;
  std::vector<uint8_t> host_pair, host_sflags;  // kept for mp_debug_render_tables
  int black_sprite = -1;
  int lane_map_players = 0, lane_map_world = 0;  // 0 plain, 2 scattered colouring, 1 + 16 * (extra wavefronts left) whole-cell dealing
  int inst_ncp = 0, inst_ncw = 0;                // the k_render<NCP, NCW> instantiation this engine launches
  // mp_debug_last_launch: the k_step cell and the k_render mode and layout of the last call that launched either, -1 for
  // a part it did not launch. Written by launch_state and launch_render from the values that pick the kernel.
  int32_t last_launch[MP_LAST_LAUNCH_FIELDS];
  uint64_t key_base = 0;   // seed + env_index_base: env b's key at creation is key_base + b (State::key)
  uint64_t blob_hash = 0;  // FNV-1a of the compiled blob (of the ordered variant set): a snapshot only loads into an engine built from the same
  VariantSet variants;     // n > 1: per-env parameter variants (mp_create_variants)
  RecordLayout record{};                     // every per-env state array (layout_state): what records and snapshots copy
  RecordLayout* d_record_layout = nullptr;  // device copy of `record`, read by a restoring mp_run's k_step

  template <typename T>
  int alloc(size_t count, T** out) {
    void* p = nullptr;
    size_t bytes = std::max<size_t>(count * sizeof(T), 16);
    CUDA_TRY(cudaMalloc(&p, bytes));
    allocs.push_back(p);
    CUDA_TRY(cudaMemset(p, 0, bytes));
    *out = static_cast<T*>(p);
    return MP_OK;
  }
};

namespace {

// What a map decides of the Tables (load_map).
struct MapVariant {
  const uint16_t* init_grid;  // [L][cells_pad]
  const uint8_t* solid;       // [cells_pad]
  const int32_t* spawn_cell;  // [n_spawn]
  const int32_t* spawn_init_cell[2];
  int n_spawn, n_spawn_init[2];
  int avatar_sprite[MP_MAX_PLAYERS];
  const uint8_t* cell_flags;  // [cells_pad] BeamBlocker bits
};
void apply_map(Tables& T, const MapVariant& M) {
  T.init_grid = M.init_grid; T.solid = M.solid; T.spawn_cell = M.spawn_cell; T.n_spawn = M.n_spawn; T.cell_flags = M.cell_flags;
  for (int k = 0; k < 2; ++k) { T.spawn_init_cell[k] = M.spawn_init_cell[k]; T.n_spawn_init[k] = M.n_spawn_init[k]; }
  memcpy(T.avatar_sprite, M.avatar_sprite, sizeof M.avatar_sprite);
}

// The map of one blob, which apply_map puts into a Tables: its initial grid padded to cells_pad, the static occupancy of
// the avatar layer (non-avatar pieces that start there), the cells of the respawn group and of the initial spawn groups,
// the avatars' sprites and the BeamBlocker bits of each cell (its walls), as host tables aimed at M's fields. `T` holds the
// geometry and the avatar tables of the engine, `groups` the respawn group and the two initial groups (or -1).
// build_tables decodes variant 0's map, which create puts into the Tables; setup_variants decodes every other variant's.
int load_map(const void* blob, size_t n, const Tables& T, const int groups[3], std::vector<HostTable>& tables, MapVariant& M) {
  Section<int32_t> meta, objects, kinds, states, av_table;
  Section<uint16_t> init_grid;
  Section<uint8_t> cell_flags;
  if (!get_section(blob, n, "meta", MPB_I32, &meta) || !get_section(blob, n, "objects", MPB_I32, &objects) ||
      !get_section(blob, n, "kinds", MPB_I32, &kinds) || !get_section(blob, n, "states", MPB_I32, &states) ||
      !get_section(blob, n, "av_table", MPB_I32, &av_table) || !get_section(blob, n, "init_grid", MPB_U16, &init_grid) ||
      !get_section(blob, n, "cell_flags", MPB_U8, &cell_flags))
    return fail(MP_E_INVALID, "blob: missing map sections");
  if (init_grid.count < (size_t)T.L * T.cells) return fail(MP_E_INVALID, "blob: 'init_grid' has %zu cells (expected %d)", init_grid.count, T.L * T.cells);
  char name[64];
  std::vector<int32_t> cells[3];
  for (int k = 0; k < 3; ++k) {
    if (groups[k] < 0) continue;
    snprintf(name, sizeof name, "spawn_cells_%d", groups[k]);
    Section<int32_t> sec;
    if (!get_section(blob, n, name, MPB_I32, &sec)) return fail(MP_E_INVALID, "blob: missing section '%s'", name);
    cells[k].assign(sec.data, sec.data + sec.count);
  }
  M.n_spawn = (int)cells[0].size();
  for (int k = 0; k < 2; ++k) {
    M.n_spawn_init[k] = (int)cells[1 + k].size();
    if (groups[1 + k] < 0) continue;
    int users = 0;
    for (int p = 0; p < T.P; ++p) users += T.avatar_init_group[p] == k;
    if (M.n_spawn_init[k] < users || M.n_spawn_init[k] > 64) return fail(MP_E_UNSUPPORTED, "%d spawn points for %d avatars (need n..64)", M.n_spawn_init[k], users);
  }
  if (M.n_spawn < 1) return fail(MP_E_INVALID, "empty respawn group");
  for (int p = 0; p < T.P; ++p) M.avatar_sprite[p] = av_table.data[p * 8 + 1];
  std::vector<uint16_t> grid0((size_t)T.L * T.cells_pad, 0);
  for (int l = 0; l < T.L; ++l) memcpy(&grid0[(size_t)l * T.cells_pad], init_grid.data + (size_t)l * T.cells, T.cells * sizeof(uint16_t));
  std::vector<uint8_t> solid(T.cells_pad, 0);
  for (int o = 0; o < meta.data[MPB_META_N_OBJECTS]; ++o) {  // non-avatar pieces that start on the avatar layer
    const int32_t* od = objects.data + o * MPB_OBJ_COLS;
    const int32_t* kd = kinds.data + od[MPB_OBJ_KIND] * MPB_KIND_COLS;
    if (kd[MPB_KIND_IS_AVATAR]) continue;
    const int32_t* st = states.data + (kd[MPB_KIND_STATE0] + od[MPB_OBJ_STATE]) * MPB_STATE_COLS;
    if (st[MPB_STATE_LAYER] == T.avatar_layer) solid[od[MPB_OBJ_Y] * T.W + od[MPB_OBJ_X]] = 255;
  }
  std::vector<uint8_t> flags(T.cells_pad, 0);
  memcpy(flags.data(), cell_flags.data, std::min<size_t>(cell_flags.count, T.cells));
  add_table(tables, &M.init_grid, grid0); add_table(tables, &M.spawn_cell, cells[0]); add_table(tables, &M.solid, solid);
  add_table(tables, &M.cell_flags, flags);
  // an initial group without cells of its own spawns on the respawn group's (the same bytes, so the same device table)
  for (int k = 0; k < 2; ++k) add_table(tables, &M.spawn_init_cell[k], cells[1 + k].empty() ? cells[0] : cells[1 + k]);
  return MP_OK;
}

// What create decodes from the blobs before it opens a device (build_tables, setup_variants). The device tables are
// host tables so far, each aimed at a field of `T`, of a variant's Params or of a variant's map; upload_tables uploads
// them once the device is checked. Everything per variant is sized to the set before decoding starts, so no field a
// table is aimed at moves.
struct Decoded {
  const FamilyEntry* family = nullptr;
  Tables T{};
  int spawn_groups[3] = {-1, -1, -1};  // the respawn group and the two initial spawn groups (or -1) of every variant
  int beam_cells = 0;                  // FamilyLoad::beam_cells: sizes State::max_events
  int n_total = 0, black_sprite = -1;
  std::vector<uint8_t> host_pair, host_sflags;
  std::vector<HostTable> tables;     // the Tables' own and those of every map
  std::vector<FamilyParams> params;  // [n] each variant's own Params
  std::vector<FamilyLoad> loads;     // [n] what each variant's loader handed back, with its Params' tables
  std::vector<int> load_rc;          // [n] each loader's refusal: variant 0's is reported at once, the others' by setup_variants
  std::vector<std::string> load_error;
  std::vector<MapVariant> maps;      // [n]
  explicit Decoded(int n) : params(n), loads(n), load_rc(n), load_error(n), maps(n) {}
};

// The engine's tables from blob 0 of `blobs`. The pre-merged sprites cover the cell stacks and the family's hint stacks
// of every blob: the variants of an engine share one sprite table and the renderer's pre-merged pairs, and may differ in
// their maps (map variants) or in the sprites their pieces show (appearance overrides). Variants that differ in neither
// add no stack of their own, so their engine has the pre-merged sprites of blob 0 alone.
int build_tables(Decoded& D, const void* const* blobs, const size_t* blob_sizes, int n_blobs, uint32_t flags) {
  const void* blob = blobs[0];
  const size_t n = blob_sizes[0];
  Section<int32_t> meta, states, kinds, comps, objects, hits, action_table, sprite_map, scalar_obs, av_table;
  Section<double> comps_f;
  Section<uint8_t> atlas, sprite_opaque;
  Section<uint16_t> init_grid;
  if (!get_section(blob, n, "meta", MPB_I32, &meta) || meta.count < MPB_META_COUNT) return fail(MP_E_INVALID, "blob: missing/invalid 'meta' (not an MPB%u blob?)", MPB_VERSION);
#define NEED(sec, dt) if (!get_section(blob, n, #sec, dt, &sec)) return fail(MP_E_INVALID, "blob: missing section '%s'", #sec);
  NEED(states, MPB_I32) NEED(kinds, MPB_I32) NEED(comps, MPB_I32) NEED(comps_f, MPB_F64) NEED(objects, MPB_I32) NEED(hits, MPB_I32)
  NEED(action_table, MPB_I32) NEED(sprite_map, MPB_I32) NEED(scalar_obs, MPB_I32) NEED(av_table, MPB_I32)
  NEED(atlas, MPB_U8) NEED(sprite_opaque, MPB_U8) NEED(init_grid, MPB_U16)
  const int32_t* m = meta.data;
  Tables& T = D.T;
  T.W = m[MPB_META_W]; T.H = m[MPB_META_H]; T.cells = T.W * T.H; T.cells_pad = round_up(T.cells, 8);
  T.L = m[MPB_META_L]; T.P = m[MPB_META_P]; T.topology = m[MPB_META_TOPOLOGY]; T.max_frames = m[MPB_META_MAX_FRAMES];
  T.view_l = m[MPB_META_VIEW_LEFT]; T.view_r = m[MPB_META_VIEW_RIGHT]; T.view_f = m[MPB_META_VIEW_FORWARD]; T.view_b = m[MPB_META_VIEW_BACKWARD];
  T.n_sprites = m[MPB_META_N_SPRITES]; T.oob_sprite = m[MPB_META_OOB_SPRITE]; T.oov_sprite = m[MPB_META_OOV_SPRITE];
  T.n_actions = m[MPB_META_N_ACTIONS]; T.n_scalar = m[MPB_META_N_SCALAR_OBS];
  if (m[MPB_META_SPRITE_SIZE] != 8) return fail(MP_E_UNSUPPORTED, "spriteSize %d (kernels are written for 8x8 sprites)", m[MPB_META_SPRITE_SIZE]);
  if (T.P < 1 || T.P > MP_MAX_PLAYERS) return fail(MP_E_UNSUPPORTED, "%d players (max %d)", T.P, MP_MAX_PLAYERS);
  if (T.L > MP_MAX_LAYERS) return fail(MP_E_UNSUPPORTED, "%d layers (max %d)", T.L, MP_MAX_LAYERS);
  if (T.n_sprites > kMaxAtlasSprites) return fail(MP_E_UNSUPPORTED, "%d sprites (max %d)", T.n_sprites, kMaxAtlasSprites);
  if (T.n_scalar > 4) return fail(MP_E_UNSUPPORTED, "%d scalar observations (max 4)", T.n_scalar);
  if (T.n_actions < 1) return fail(MP_E_INVALID, "blob has no action table (compile with the substrate config)");
  if (T.cells >= 4096) return fail(MP_E_UNSUPPORTED, "map of %d cells (max 4095)", T.cells);
  if (T.topology == 1 && (T.view_l + T.view_r + 1 > T.W || T.view_f + T.view_b + 1 > T.H || T.view_l + T.view_r + 1 > T.H || T.view_f + T.view_b + 1 > T.W))
    return fail(MP_E_UNSUPPORTED, "TORUS map smaller than the view window");
  for (int k = 0; k < T.n_scalar; ++k) T.scalar_obs[k] = scalar_obs.data[k];
  D.family = find_family(m[MPB_META_FAMILY]);
  if (!D.family) return fail(MP_E_UNSUPPORTED, "substrate family %d has no CUDA state-transition kernel yet", m[MPB_META_FAMILY]);

  // ---- avatars ---------------------------------------------------------------------------------
  T.avatar_layer = av_table.data[2];
  int init_groups[2] = {-1, -1};
  int respawn_group = -1;
  for (int p = 0; p < T.P; ++p) {
    const int32_t* a = av_table.data + p * 8;
    T.avatar_sprite[p] = a[1];
    if (a[2] != T.avatar_layer) return fail(MP_E_UNSUPPORTED, "per-avatar layers");
    const int post = a[4] >= 0 ? a[4] : a[3];
    if (respawn_group >= 0 && post != respawn_group) return fail(MP_E_UNSUPPORTED, "per-avatar respawn groups");
    respawn_group = post;
    int g = -1;
    for (int k = 0; k < 2; ++k) if (init_groups[k] == a[3]) g = k;
    if (g < 0) { for (int k = 0; k < 2 && g < 0; ++k) if (init_groups[k] < 0) { init_groups[k] = a[3]; g = k; } }
    if (g < 0) return fail(MP_E_UNSUPPORTED, "more than two initial spawn groups");
    T.avatar_init_group[p] = g;
  }
  D.spawn_groups[0] = respawn_group; D.spawn_groups[1] = init_groups[0]; D.spawn_groups[2] = init_groups[1];
  const MapVariant& map0 = D.maps[0];
  int rc;
  if ((rc = load_map(blob, n, T, D.spawn_groups, D.tables, D.maps[0]))) return rc;

  // ---- family tables: every blob's loader, once. Variant 0's refusal is reported here, every other variant's by
  // setup_variants; the hint stacks of every loader that succeeded go to the pre-merge.
  for (int v = 0; v < n_blobs; ++v) {
    Section<int32_t> v_hits;
    if (!get_section(blobs[v], blob_sizes[v], "hits", MPB_I32, &v_hits)) {
      D.load_rc[v] = fail(MP_E_INVALID, "blob: missing section 'hits'");
    } else {
      D.loads[v] = FamilyLoad{blobs[v], blob_sizes[v], v_hits};
      D.load_rc[v] = D.family->load(D.loads[v], T, D.params[v]);
    }
    if (D.load_rc[v] && v == 0) return D.load_rc[v];
    if (D.load_rc[v]) D.load_error[v] = g_error;
  }
  std::vector<std::vector<int>> hint_stacks;
  for (int v = 0; v < n_blobs; ++v)
    if (!D.load_rc[v]) hint_stacks.insert(hint_stacks.end(), D.loads[v].hint_stacks.begin(), D.loads[v].hint_stacks.end());
#undef NEED
  const FamilyLoad& ld = D.loads[0];
  T.nA = ld.nA; T.nD = ld.nD; T.nW = ld.nW; T.nR = ld.nR; T.nR_pad = ld.nR_pad;
  T.end_min_frames = ld.end_min_frames; T.end_interval = ld.end_interval; T.end_prob = ld.end_prob;
  D.beam_cells = ld.beam_cells;
  {  // 'choice' prefabs left to the engine (drawn per env and episode)
    Section<int32_t> choice_groups, obj_choice, spawn_cond;
    char name[64];
    if (get_section(blob, n, "choice_groups", MPB_I32, &choice_groups)) {
      if (D.family->id != MPB_FAMILY_TERRITORY) return fail(MP_E_UNSUPPORTED, "per-env 'choice' prefabs are implemented for the territory family only (compile with a build_seed)");
      T.n_choice = (int)choice_groups.count;
      for (size_t g = 0; g < choice_groups.count; ++g) if (choice_groups.data[g] < 1 || choice_groups.data[g] > 31) return fail(MP_E_INVALID, "blob: choice group with %d options", choice_groups.data[g]);
      add_table(D.tables, &T.choice_n, std::vector<int32_t>(choice_groups.data, choice_groups.data + choice_groups.count));
      snprintf(name, sizeof name, "spawn_cond_%d", respawn_group);
      if (get_section(blob, n, name, MPB_I32, &spawn_cond)) {
        if ((int)spawn_cond.count != map0.n_spawn * 2 || map0.n_spawn > 64) return fail(MP_E_UNSUPPORTED, "%d conditional spawn candidates (max 64)", map0.n_spawn);
        add_table(D.tables, &T.spawn_cond, std::vector<int32_t>(spawn_cond.data, spawn_cond.data + spawn_cond.count));
      }
    }
  }
  T.nA_pad = round_up(std::max(T.nA, 1), 16); T.nD_pad = round_up(std::max(std::max(T.nD, T.nA), 1), 16); T.nW_pad = round_up(std::max(T.nW, 1), 16);

  add_table(D.tables, &T.action_table, std::vector<int32_t>(action_table.data, action_table.data + action_table.count));

  // ---- render tables ------------------------------------------------------------------------------
  if (atlas.count != (size_t)T.n_sprites * 1024) return fail(MP_E_INVALID, "atlas has %zu bytes, expected %d", atlas.count, T.n_sprites * 1024);
  std::vector<uint8_t> img(atlas.data, atlas.data + atlas.count);  // [sprite][facing][row][px][4]
  std::vector<uint8_t> opq(sprite_opaque.data, sprite_opaque.data + T.n_sprites);
  std::vector<uint8_t> remapped(T.n_sprites, 0);
  for (int v = 0; v <= T.P; ++v)
    for (int s = 0; s < T.n_sprites; ++s)
      if (sprite_map.data[(size_t)v * T.n_sprites + s] != s) { remapped[s] = 1; opq[s] = 0; }  // a remapped sprite must not hide layers
  // Pre-merged sprites. For every stack of map pieces that can occur on a cell, the opaque bottom
  // sprite and the sprites above it are folded pairwise into new opaque sprites using exactly the
  // renderer's arithmetic (policy A.14), so the kernel composes most cells with a single copy.
  std::vector<std::vector<int>> pair_of;  // pair_of[base][top] -> merged id (grown with the atlas)
  auto n_now = [&]() { return (int)opq.size(); };
  pair_of.assign(T.n_sprites, std::vector<int>());
  auto blend = [](uint8_t* d, const uint8_t* s_) {
    unsigned a = s_[3];
    if (a == 255) { d[0] = s_[0]; d[1] = s_[1]; d[2] = s_[2]; }
    else if (a) for (int c = 0; c < 3; ++c) d[c] = (uint8_t)((s_[c] * a + d[c] * (255u - a)) / 255u);
  };
  auto merged_id = [&](int base, int top) -> int {
    if ((int)pair_of[base].size() <= top) pair_of[base].resize(top + 1, 0);
    if (pair_of[base][top]) return pair_of[base][top];
    if (n_now() >= kMaxAtlasSprites) return 0;  // budget: the atlas has to fit in shared memory next to the staging buffers
    if (flags & MP_FLAG_DEBUG_NO_PREMERGE) return 0;  // budget zero: every stack takes the general compositing path
    int id = n_now();
    img.resize((size_t)(id + 1) * 1024);
    for (int f = 0; f < 4; ++f)
      for (int px = 0; px < 64; ++px) {
        uint8_t* d = &img[(size_t)id * 1024 + f * 256 + px * 4];
        memcpy(d, &img[(size_t)base * 1024 + f * 256 + px * 4], 4);
        blend(d, &img[(size_t)top * 1024 + f * 256 + px * 4]);
        d[3] = 255;
      }
    opq.push_back(1); remapped.push_back(0);
    pair_of.push_back(std::vector<int>());
    pair_of[base][top] = id;
    return id;
  };
  {
    // Per blob: the sprites each (cell, layer) can show (opts_of) and the initial grid (init_of).
    struct Opt { std::vector<int> sprites; bool absent = false; int orient = -1; bool bad = false; };
    std::vector<std::vector<Opt>> opts_of(n_blobs, std::vector<Opt>((size_t)T.cells * T.L));
    std::vector<const uint16_t*> init_of(n_blobs);
    for (int v = 0; v < n_blobs; ++v) {
      Section<int32_t> v_meta, v_states, v_kinds, v_objects;
      Section<uint16_t> v_init;
      if (!get_section(blobs[v], blob_sizes[v], "meta", MPB_I32, &v_meta) || !get_section(blobs[v], blob_sizes[v], "states", MPB_I32, &v_states) ||
          !get_section(blobs[v], blob_sizes[v], "kinds", MPB_I32, &v_kinds) || !get_section(blobs[v], blob_sizes[v], "objects", MPB_I32, &v_objects) ||
          !get_section(blobs[v], blob_sizes[v], "init_grid", MPB_U16, &v_init) || v_init.count < (size_t)T.L * T.cells)
        return fail(MP_E_INVALID, "blob %d: missing map sections", v);
      init_of[v] = v_init.data;
      std::vector<Opt>& opts = opts_of[v];
      for (int o = 0; o < v_meta.data[MPB_META_N_OBJECTS]; ++o) {
        const int32_t* od = v_objects.data + o * MPB_OBJ_COLS;
        const int32_t* kd = v_kinds.data + od[MPB_OBJ_KIND] * MPB_KIND_COLS;
        if (kd[MPB_KIND_IS_AVATAR]) continue;
        const int cell = od[MPB_OBJ_Y] * T.W + od[MPB_OBJ_X];
        const int ns = kd[MPB_KIND_NSTATES];
        for (int si = 0; si < ns; ++si) {
          const int32_t* st = v_states.data + (kd[MPB_KIND_STATE0] + si) * MPB_STATE_COLS;
          const int l = st[MPB_STATE_LAYER], sp = st[MPB_STATE_SPRITE];
          if (l < 0 || sp < 0) continue;
          Opt& op = opts[(size_t)cell * T.L + l];
          if (std::find(op.sprites.begin(), op.sprites.end(), sp) == op.sprites.end()) op.sprites.push_back(sp);
          if (op.orient >= 0 && op.orient != od[MPB_OBJ_ORIENT]) op.bad = true;
          op.orient = od[MPB_OBJ_ORIENT];
          // the piece may also be somewhere else (another layer / off grid / sprite-less state)
          for (int sj = 0; sj < ns; ++sj) {
            const int32_t* s2 = v_states.data + (kd[MPB_KIND_STATE0] + sj) * MPB_STATE_COLS;
            if (s2[MPB_STATE_LAYER] != l || s2[MPB_STATE_SPRITE] < 0) op.absent = true;
          }
        }
      }
    }
    for (const auto& hs : hint_stacks) {
      if (hs.empty() || !opq[hs[0]]) continue;
      int cur = hs[0];
      for (size_t q = 1; q < hs.size() && cur; ++q) { if (remapped[hs[q]] || remapped[cur]) break; cur = merged_id(cur, hs[q]); }
    }
    std::vector<int> stack_s, stack_o;
    for (int pass = 0; pass < 2; ++pass)  // pass 0: the maps as they are at reset (most common stacks) get the budget first
    for (int v = 0; v < n_blobs; ++v)        // (the stacks of every variant's map)
    for (int cell = 0; cell < T.cells; ++cell) {
      const std::vector<Opt>& opts = opts_of[v];
      const uint16_t* init_grid = init_of[v];
      // enumerate the cartesian product of per-layer options, bottom up (bounded)
      size_t combos = 1;
      bool bad = false;
      for (int l = 0; l < T.L; ++l) {
        const Opt& op = opts[(size_t)cell * T.L + l];
        bad |= op.bad;
        combos *= std::max<size_t>(1, op.sprites.size() + ((op.absent || op.sprites.empty()) ? 1 : 0));
        if (combos > 4096) { bad = true; break; }
      }
      if (bad) continue;
      std::vector<int> idx(T.L, 0);
      for (size_t k = 0; k < combos; ++k) {
        stack_s.clear(); stack_o.clear();
        bool is_initial = true;
        for (int l = 0; l < T.L; ++l) {
          const Opt& op = opts[(size_t)cell * T.L + l];
          const int i = idx[l];
          const int init_v = init_grid[(size_t)l * T.cells + cell];
          const int init_sprite = init_v ? (init_v - 1) >> 2 : -1;
          if (i < (int)op.sprites.size()) { stack_s.push_back(op.sprites[i]); stack_o.push_back(op.orient); is_initial &= op.sprites[i] == init_sprite; }
          else is_initial &= init_sprite < 0;
        }
        if ((pass == 0) != is_initial) stack_s.clear();  // handled in the other pass
        // the walk the kernel performs: opaque bottom, then fold upwards while possible
        int j = -1;
        for (int q = (int)stack_s.size() - 1; q >= 0; --q) if (opq[stack_s[q]]) { j = q; break; }
        if (j >= 0) {
          int cur = stack_s[j];
          for (int q = j + 1; q < (int)stack_s.size(); ++q) {
            const int t = stack_s[q];
            if (stack_o[q] != stack_o[j] || remapped[t] || remapped[cur]) break;
            cur = merged_id(cur, t);
            if (!cur) break;
          }
        }
        for (int l = 0; l < T.L; ++l) {  // next combination
          const Opt& op = opts[(size_t)cell * T.L + l];
          const int radix = (int)std::max<size_t>(1, op.sprites.size() + ((op.absent || op.sprites.empty()) ? 1 : 0));
          if (++idx[l] < radix) break;
          idx[l] = 0;
        }
      }
    }
  }
  const int n_total = n_now();
  D.n_total = n_total;
  // atlas re-laid out as [sprite][facing][half][row][16 B] so that the 8 rows of one half are 128
  // contiguous bytes (conflict-free 128-bit shared loads).
  std::vector<uint8_t> at((size_t)n_total * 1024);
  for (int s = 0; s < n_total * 4; ++s)
    for (int row = 0; row < 8; ++row)
      for (int half = 0; half < 2; ++half)
        memcpy(&at[(size_t)s * 256 + half * 128 + row * 16], &img[(size_t)s * 256 + row * 32 + half * 16], 16);
  add_table(D.tables, &T.atlas, at);
  std::vector<int16_t> smap((size_t)(T.P + 1) * n_total);
  for (int v = 0; v <= T.P; ++v)
    for (int s = 0; s < n_total; ++s)
      smap[(size_t)v * n_total + s] = (int16_t)(s < T.n_sprites ? sprite_map.data[(size_t)v * T.n_sprites + s] : s);
  std::vector<uint8_t> pair((size_t)n_total * n_total, 0);
  for (int b = 0; b < n_total; ++b)
    for (int t = 0; t < (int)pair_of[b].size(); ++t) pair[(size_t)b * n_total + t] = (uint8_t)pair_of[b][t];
  std::vector<uint8_t> sflags(n_total);  // bit 0 opaque, bit 1 remapped for some viewer, bit 2 binary alpha
  std::vector<uint8_t> binary_alpha(n_total, 1);  // every alpha 0 or 255
  for (int i = 0; i < n_total; ++i)
    for (int px = 0; px < 256; ++px) { const uint8_t a = img[(size_t)i * 1024 + px * 4 + 3]; if (a != 0 && a != 255) { binary_alpha[i] = 0; break; } }
  for (int i = 0; i < n_total; ++i) {
    bool bin = true;  // must hold for whatever sprite a viewer sees in its place
    for (int v = 0; v <= T.P; ++v) bin = bin && binary_alpha[smap[(size_t)v * n_total + i]];
    bool invisible = true;  // every alpha 0, whatever a viewer sees in its place
    for (int v = 0; v <= T.P && invisible; ++v) {
      const int t = smap[(size_t)v * n_total + i];
      for (int px = 0; px < 256 && invisible; ++px) invisible = img[(size_t)t * 1024 + px * 4 + 3] == 0;
    }
    sflags[i] = (uint8_t)((opq[i] ? 1 : 0) | (remapped[i] ? 2 : 0) | (bin ? 4 : 0) | (invisible ? 8 : 0));
  }
  D.host_pair = pair; D.host_sflags = sflags;
  // an opaque, never remapped, all-black sprite (D.black_sprite) stands in for cells with nothing to draw
  for (int i = 0; i < n_total && D.black_sprite < 0; ++i) {
    if (!opq[i] || remapped[i]) continue;
    bool black = true;
    for (int px = 0; px < 256 && black; ++px) { const uint8_t* q = &img[(size_t)i * 1024 + px * 4]; black = q[0] == 0 && q[1] == 0 && q[2] == 0; }
    if (black) D.black_sprite = i;
  }
  add_table(D.tables, &T.sprite_map, smap); add_table(D.tables, &T.sprite_opaque, sflags); add_table(D.tables, &T.sprite_pair, pair);
  return MP_OK;
}

int build_plan(mp_engine* E) {
  const Tables& T = E->T;
  RenderPlan& R = E->R;
  R.view_w = T.view_l + T.view_r + 1; R.view_h = T.view_f + T.view_b + 1;
  R.player_bytes = R.view_w * R.view_h * 192;
  R.world_bytes = T.H * T.W * 192;
  R.grid_bytes = T.L * T.cells_pad * 2;
  R.n_total = E->n_total;
  R.atlas_bytes = R.n_total * 1024;
  R.rec_stride = (int)round_up(T.L + 1, 4);  // header + entries, 8-byte aligned records
  R.magic_view_h = (65536u + R.view_h - 1) / R.view_h;
  int off = 128;  // mbarriers
  R.off_atlas = off; off += round_up(R.atlas_bytes, 128);
  R.off_pair = off; off += round_up(R.n_total * R.n_total, 128);
  R.off_map = off; off += round_up((T.P + 1) * R.n_total * 2, 128);
  R.off_team0 = off;
  // Teams per CTA x warps per team x WORLD.RGB strip height: among the layouts that fit in shared memory, the one
  // with the most useful warps in flight. A team draws one env at a time, so its warps share that env's strips; with
  // few strips per warp the end-of-env barrier and the last straggling strip weigh more (score below).
  // A layout forced through the flags (MP_RENDER_LAYOUT) replaces the search; it must fit like any candidate.
  const int f_teams = (E->flags >> MP_FLAG_LAYOUT_TEAMS_SHIFT) & 7, f_warps = (E->flags >> MP_FLAG_LAYOUT_WARPS_SHIFT) & 31,
            f_wlog = (E->flags >> MP_FLAG_LAYOUT_WLOG_SHIFT) & 3;
  const bool forced = (E->flags & MP_FLAG_LAYOUT_MASK) != 0;
  if (forced) {
    if (f_teams < 2 || f_teams > RENDER_MAX_TEAMS || f_warps < 4 || f_warps > TEAM_THREADS / 32 || f_wlog < 1 || f_wlog > 2)
      return fail(MP_E_INVALID, "render layout (%d teams, %d warps, wstrip_log2 %d) outside 2-%d / 4-%d / 1-2", f_teams, f_warps, f_wlog,
                  RENDER_MAX_TEAMS, TEAM_THREADS / 32);
    if (f_teams * f_warps > RENDER_MAX_THREADS / 32)
      return fail(MP_E_UNSUPPORTED, "render layout of %d teams x %d warps exceeds %d threads per CTA", f_teams, f_warps, RENDER_MAX_THREADS);
  }
  R.smem_bytes = 1 << 30;
  int need_forced = 0;
  double best = -1.0;
  for (int teams = 2; teams <= RENDER_MAX_TEAMS; ++teams)
    for (int warps = TEAM_THREADS / 32; warps >= 4; --warps) {
      if (teams * warps > RENDER_MAX_THREADS / 32) continue;
      if (forced && (teams != f_teams || warps != f_warps)) continue;
      for (int wlog = 2; wlog >= 1; --wlog) {
        if (forced && wlog != f_wlog) continue;
        const int stage = RENDER_SLOTS * round_up(std::max(R.view_w * 192, T.W * 24 * (1 << wlog)), 128);
        const int team_bytes = round_up(R.grid_bytes, 128) + round_up(T.cells * R.rec_stride * 2, 128) + warps * stage;
        const int total = R.off_team0 + teams * team_bytes;
        if (forced) need_forced = total;
        if (total > kRenderSmemLimit) continue;
        const double items = T.P * R.view_h + (8 >> wlog) * T.H, per_warp = items / warps;
        // (constants fitted to a sweep of every feasible layout of the nine substrates on an H100 SXM,
        //  profiles/render_layouts_h100.jsonl: about 18 warps per SM keep the write stream full and more only add idle
        //  time, about four strips' worth of idle time per env and warp at the team barriers, 2-row WORLD.RGB strips
        //  ~15 % slower than 4-row ones, and each extra team ~10 % better: teams out of phase fill each other's per-env
        //  gaps in the write stream)
        const double score = std::min(teams * warps, 18) * per_warp / (per_warp + 4.0) * (wlog == 2 ? 1.0 : 0.85) * (1.0 + 0.1 * teams);
        if (score > best + 1e-9) {
          best = score;
          R.n_teams = teams; R.team_threads = warps * 32; R.wstrip_log2 = wlog; R.stage_bytes = stage;
          R.toff_grid = 0; R.toff_rec = round_up(R.grid_bytes, 128);
          R.toff_stage = R.toff_rec + round_up(T.cells * R.rec_stride * 2, 128);
          R.team_stride = team_bytes; R.smem_bytes = total;
        }
      }
    }
  if (forced && R.smem_bytes > kRenderSmemLimit)
    return fail(MP_E_UNSUPPORTED, "render layout (%d teams, %d warps, wstrip_log2 %d) needs %d B of shared memory (> %d)", f_teams, f_warps,
                f_wlog, need_forced, kRenderSmemLimit);
  if (R.smem_bytes > kRenderSmemLimit) return fail(MP_E_UNSUPPORTED, "render kernel needs %d B of shared memory (> 227 KB)", R.smem_bytes);
  return MP_OK;
}

// Debug observations (SURVEY.md section 8f N3): {i}.POSITION / {i}.ORIENTATION (LocationObserver, component_library.lua:806-855),
// {i}.LAYER (the unrotated view window as per-layer sprite ids, avatar_library.lua:247-257) and the per-step zap matrix
// (who zapped whom, from the step's events; clean_up.py:751-784 builds the same from the 'zap' events).
__global__ void k_debug_obs(Tables T, State S, int32_t* position, int32_t* orientation, int32_t* layer, int32_t* zap, int view_w, int view_h) {
  const int b = blockIdx.x, P = T.P;
  const int32_t* av = S.avatar + (size_t)b * P * 4;
  for (int p = threadIdx.x; p < P; p += blockDim.x) {
    if (position) { position[((size_t)b * P + p) * 2] = av[p * 4 + AV_X]; position[((size_t)b * P + p) * 2 + 1] = av[p * 4 + AV_Y]; }
    if (orientation) orientation[(size_t)b * P + p] = av[p * 4 + AV_ORIENT];
  }
  if (layer) {
    const int per_player = view_h * view_w * T.L;
    const uint16_t* grid = S.grid + (size_t)b * T.L * T.cells_pad;
    for (int i = threadIdx.x; i < P * per_player; i += blockDim.x) {
      const int p = i / per_player, r = i - p * per_player, l = r % T.L, c = r / T.L, vx = c % view_w, vy = c / view_w;
      int x = av[p * 4 + AV_X] - T.view_l + vx, y = av[p * 4 + AV_Y] - T.view_f + vy;  // orientation 'N': window not rotated
      int32_t v = -1;  // outside a BOUNDED map (policy A.21)
      if (wrap_or_reject(T, x, y)) { const uint16_t g = grid[(size_t)l * T.cells_pad + y * T.W + x]; v = g ? ((g - 1) >> 2) + 1 : 0; }
      layer[(size_t)b * P * per_player + i] = v;
    }
  }
  if (zap) {
    for (int i = threadIdx.x; i < P * P; i += blockDim.x) zap[(size_t)b * P * P + i] = 0;
    __syncthreads();
    const int n = min(S.n_events[b], S.max_events);
    for (int i = threadIdx.x; i < n; i += blockDim.x) {
      const int32_t* e = S.events + ((size_t)b * S.max_events + i) * 3;
      if (e[0] == EV_ZAP && e[1] >= 1 && e[1] <= P && e[2] >= 1 && e[2] <= P) atomicAdd(&zap[(size_t)b * P * P + (e[1] - 1) * P + (e[2] - 1)], 1);
    }
  }
}

// For a call that launches no state transition: every field -1 until launch_render records its render.
void clear_last_launch(mp_engine* E) { std::fill_n(E->last_launch, MP_LAST_LAUNCH_FIELDS, -1); }

// `S`: the engine's state with the step's targets applied (apply_outputs), for the scalar rows k_exchange_push delivers;
// `G`: the segments of its per-player rows (apply_players).
int raise_flags(mp_engine* E, cudaStream_t st, const State& S, const RowSegments& G = RowSegments{}) {
  E->x_pending_raise = false;
  k_exchange_push<<<std::min(E->sm_count, (E->B + 7) / 8), 256, 0, st>>>(E->T, S, G);
  ++E->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

// `render_follows`: the caller launches the renderer next on the same stream; it raises the exchange flags.
// `restore`: a step (mode 0) that restores the envs it names instead of advancing them (k_step<..., true>), or null.
// `rows`: the step's actions come from rows (player_actions, k_step<..., RowActions>; `actions` unused), or null.
// `drawn`: drawn routes (k_step_drawn, which writes the row map; `actions` and `rows` unused), or null.
int launch_state(mp_engine* E, const int32_t* actions, const uint8_t* mask, int mode, cudaStream_t st, bool render_follows = true,
                 const StepRestore* restore = nullptr, const RowActions* rows = nullptr, const DrawnActions* drawn = nullptr) {
  const int blocks = (E->B + 3) / 4;
  if (E->S.x_world) E->S.x_step = ++E->x_seq;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(128); cfg.dynamicSmemBytes = E->step_smem; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  StepRestore restore_arg = restore ? *restore : StepRestore{};
  RowActions rows_arg = rows ? *rows : RowActions{};
  void* args[] = {&E->T, nullptr, &E->S, &actions, &mask, &mode, &restore_arg,
                  drawn ? const_cast<DrawnActions*>(drawn) : static_cast<void*>(&rows_arg)};  // k_step's parameters; Source by `launch`
  const int variants = E->variants.n > 1, restoring = restore != nullptr, source = drawn ? 2 : rows != nullptr;
  const void* kernel = E->family->step[variants][restoring][source];
  CUDA_TRY(E->family->launch(cfg, kernel, args, E->params, E->variants));
  const int32_t cell[MP_LAST_LAUNCH_FIELDS] = {E->family->id, variants, restoring, source, -1, -1, -1, -1, -1, -1};
  memcpy(E->last_launch, cell, sizeof cell);
  if (E->S.x_world) {
    E->x_pending_raise = true;
    if (!render_follows) { ++E->launches; return raise_flags(E, st, E->S); }
  }
  ++E->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

// Points a launch's copy of the state at the targets of `o` (checked by check_device_outputs, or the engine's own
// second image set of mp_step_host_async slot 1): the images it names replace the engine's own, its scalar rows are added.
void apply_outputs(const mp_device_outputs& o, State& S) {
  if (o.rgb) { S.rgb = o.rgb; S.rgb_env_stride = o.rgb_env_stride; }
  if (o.world_rgb) { S.world_rgb = o.world_rgb; S.world_env_stride = o.world_rgb_env_stride; }
  S.out = ScalarTargets{o.reward, o.discount, o.step_type, o.scalar_obs, o.reward_env_stride, o.discount_env_stride,
                        o.step_type_env_stride, o.scalar_obs_env_stride, o.scalar_obs_stride, 0};
  S.out.on = o.reward || o.discount || o.step_type || o.scalar_obs;
}

// The scalar rows of a step that no kernel follows (rendering off, no exchange): strided device-to-device copies, so
// that a step into a target launches no more kernels than a plain one.
int copy_scalars(mp_engine* E, const ScalarTargets& o, cudaStream_t st) {
  const size_t B = E->B, P = E->T.P;
  const State& S = E->S;
  if (o.reward) CUDA_TRY(cudaMemcpy2DAsync(o.reward, o.reward_stride, S.reward, P * 8, P * 8, B, cudaMemcpyDeviceToDevice, st));
  if (o.discount) CUDA_TRY(cudaMemcpy2DAsync(o.discount, o.discount_stride, S.discount, 8, 8, B, cudaMemcpyDeviceToDevice, st));
  if (o.step_type) CUDA_TRY(cudaMemcpy2DAsync(o.step_type, o.step_type_stride, S.step_type, 8, 8, B, cudaMemcpyDeviceToDevice, st));
  for (int k = 0; o.scalar_obs && k < E->T.n_scalar; ++k)
    CUDA_TRY(cudaMemcpy2DAsync(reinterpret_cast<uint8_t*>(o.scalar_obs) + k * o.scalar_obs_stride, o.scalar_obs_env_stride,
                               S.scalar_obs + k * B * P, P * 8, P * 8, B, cudaMemcpyDeviceToDevice, st));
  return MP_OK;
}

static_assert(sizeof(RowSegment) == sizeof(mp_row_segment) && offsetof(RowSegment, rgb) == offsetof(mp_row_segment, rgb) &&
                  offsetof(RowSegment, reward) == offsetof(mp_row_segment, reward) &&
                  offsetof(RowSegment, scalar_obs_stride) == offsetof(mp_row_segment, scalar_obs_stride) &&
                  MP_ROW_SEGMENTS == MP_MAX_ROW_SEGMENTS,
              "RowSegment must match mp_row_segment");

// The per-player targets of `p` as segments: its own, or one segment [0, n_rows) of its top-level targets.
RowSegments row_segments(const mp_player_outputs& p) {
  RowSegments G{};
  if (p.n_segments > 0) {
    G.n = p.n_segments;
    memcpy(G.s, p.segments, sizeof(RowSegment) * G.n);
  } else {
    G.n = 1;
    G.s[0] = RowSegment{0, p.n_rows, p.rgb, p.rgb_row_stride, p.reward, p.reward_row_stride, p.scalar_obs,
                        p.scalar_obs_row_stride, p.scalar_obs_stride};
  }
  return G;
}

// Points a launch's copy of the state at the per-player rows of `p` (checked by check_player_outputs); `G` is
// row_segments(p).
void apply_players(const mp_player_outputs& p, const RowSegments& G, State& S) {
  S.pr = PlayerTargets{p.row_of_player, (G.s[0].reward || G.s[0].scalar_obs) ? 1 : 0, p.world_row_of_env, p.world_rgb,
                       p.world_rgb_row_stride, p.world_n_rows};
}

// `out`: where this render's outputs go besides / instead of the engine's own buffers (see apply_outputs), or null.
// `players`: per-player rows (mp_run's players): the render runs k_render<..., RENDER_ROUTED>, or, with rendering off,
// k_exchange_push delivers the routed scalars (one launch).
int launch_render(mp_engine* E, cudaStream_t st, const mp_device_outputs* out = nullptr, const mp_player_outputs* routed = nullptr) {
  const bool players = E->flags & MP_FLAG_RENDER_PLAYERS, world = E->flags & MP_FLAG_RENDER_WORLD;
  const RowSegments G = routed ? row_segments(*routed) : RowSegments{};
  if (!players && !world) {
    State S = E->S;
    if (out) apply_outputs(*out, S);
    if (routed) apply_players(*routed, G, S);
    if (E->x_pending_raise || S.pr.scalars_on) return raise_flags(E, st, S, G);  // (k_exchange_push also delivers S.out)
    return S.out.on ? copy_scalars(E, S.out, st) : MP_OK;
  }
  // The engine's own images are also slot 0's of mp_step_host_async: a render into them must not start before that
  // slot's device->host copy has read them, whichever call issues it. (A render into a target does not touch them.)
  const bool own_images = (players && !(out && out->rgb) && !G.s[0].rgb) ||
                          (world && !(out && out->world_rgb) && !(routed && routed->world_rgb));
  if (E->async_ready && own_images) CUDA_TRY(cudaStreamWaitEvent(st, E->slot[0].copied, 0));
  E->S.x_raise = E->x_pending_raise ? 1 : 0;
  E->x_pending_raise = false;
  const int blocks = std::min(E->B, E->sm_count);  // every CTA has at least one env (balanced rounds + cooperative tail)
  RenderPlan R = E->R;
  const Tables& T = E->T;
  R.n_player_items = (E->flags & MP_FLAG_RENDER_PLAYERS) ? T.P * R.view_h : 0;
  R.n_items = R.n_player_items + ((E->flags & MP_FLAG_RENDER_WORLD) ? (8 >> R.wstrip_log2) * T.H : 0);
  R.prow_bytes = R.view_w * 24; R.wrow_bytes = T.W * 24;
  R.pitem_bytes = R.prow_bytes * 8; R.witem_bytes = R.wrow_bytes << R.wstrip_log2;
  R.h_oob = 0x8000 | (T.oob_sprite * 4); R.h_oov = 0x8000 | (T.oov_sprite * 4);
  R.h_empty = E->black_sprite >= 0 ? (0x8000 | (E->black_sprite * 4)) : 0;
  // Programmatic dependent launch: the renderer's prologue (atlas + table staging, ~3 us) runs under the tail of the
  // state-transition kernel that precedes it in the stream; it reads env state only after griddepcontrol.wait.
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(R.n_teams * R.team_threads); cfg.dynamicSmemBytes = R.smem_bytes; cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  const bool gather = E->g_world > 0 && E->S.g_world > 0;
  if (gather) {
    E->S.g_step = ++E->g_seq;
    const size_t slot = (size_t)(E->g_seq & 1ull) * E->g_slot_bytes;
    for (int r = 0; r < E->g_world; ++r) {
      uint8_t* base = E->g_peer[r] + MP_EXCHANGE_HEADER + slot;
      E->S.g_rgb[r] = base + (size_t)E->g_rank * E->B * T.P * R.player_bytes;
      E->S.g_wrgb[r] = base + E->g_world_off + (size_t)E->g_rank * E->B * R.world_bytes;
    }
  }
  State S = E->S;
  if (out) apply_outputs(*out, S);
  if (routed) apply_players(*routed, G, S);  // (never with gather: mp_run refuses it)
  const int mode = routed ? RENDER_ROUTED : gather ? RENDER_GATHER : RENDER_PLAIN;
  CUDA_TRY(cudaLaunchKernelEx(&cfg, E->render_fns[mode], E->T, S, R, E->flags, G));
  const int32_t layout[6] = {mode, E->inst_ncp, E->inst_ncw, R.n_teams, R.team_threads / 32, R.wstrip_log2};
  memcpy(E->last_launch + 4, layout, sizeof layout);
  if (gather) {
    k_gather_raise<<<1, 32, 0, st>>>(E->d_g_flag_ptrs, E->g_world, E->g_rank, E->g_seq);
    ++E->launches;
  }
  ++E->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

int copy_out(mp_engine* E, const mp_host_outputs* out, cudaStream_t st) {
  if (!out) return MP_OK;
  const mp_buffers& bf = E->buffers;
  const size_t B = E->B, P = E->T.P;
  if (out->rgb) CUDA_TRY(cudaMemcpyAsync(out->rgb, bf.rgb, B * P * E->R.player_bytes, cudaMemcpyDeviceToHost, st));
  if (out->world_rgb) CUDA_TRY(cudaMemcpyAsync(out->world_rgb, bf.world_rgb, B * E->R.world_bytes, cudaMemcpyDeviceToHost, st));
  if (out->events) CUDA_TRY(cudaMemcpyAsync(out->events, bf.events, B * (size_t)bf.max_events * 3 * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (out->event_count) CUDA_TRY(cudaMemcpyAsync(out->event_count, bf.event_count, B * sizeof(int32_t), cudaMemcpyDeviceToHost, st));
  if (out->scalar_block) {  // reward | discount | step_type | scalar_obs in one transfer (layout of mp_buffers.scalar_block)
    CUDA_TRY(cudaMemcpyAsync(out->scalar_block, E->scalar_block, E->scalar_block_bytes, cudaMemcpyDeviceToHost, st));
    return MP_OK;
  }
  if (out->reward) CUDA_TRY(cudaMemcpyAsync(out->reward, bf.reward, B * P * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out->discount) CUDA_TRY(cudaMemcpyAsync(out->discount, bf.discount, B * sizeof(double), cudaMemcpyDeviceToHost, st));
  if (out->step_type) CUDA_TRY(cudaMemcpyAsync(out->step_type, bf.step_type, B * sizeof(int64_t), cudaMemcpyDeviceToHost, st));
  if (out->scalar_obs && E->T.n_scalar) CUDA_TRY(cudaMemcpyAsync(out->scalar_obs, bf.scalar_obs, (size_t)E->T.n_scalar * B * P * sizeof(double), cudaMemcpyDeviceToHost, st));
  return MP_OK;
}

struct DeviceGuard {
  int prev = -1;
  explicit DeviceGuard(int dev) { cudaGetDevice(&prev); if (prev != dev) cudaSetDevice(dev); else prev = -1; }
  ~DeviceGuard() { if (prev >= 0) cudaSetDevice(prev); }
};

uint64_t fnv1a(const void* p, size_t n, uint64_t h = 1469598103934665603ull) {
  const uint8_t* bp = static_cast<const uint8_t*>(p);
  for (size_t i = 0; i < n; ++i) { h ^= bp[i]; h *= 1099511628211ull; }
  return h;
}

// The one list of per-env state arrays, as E->record and its device copy. Env b's row of an array is its `bytes` bytes
// at base + b * bytes: one env's rows make its state-bank record (mp_state_store / mp_state_restore), the arrays whole
// make a snapshot (mp_state_save / mp_state_load). Images are not state; a restore or a load re-renders them. Every
// size follows from the blob (or the variant set) alone, so a record restores into any engine built from it, whatever
// its num_envs, seed, env_index_base or device. A record:
//   [0, 16)   tag: format word, record bytes, blob_hash (the hash of the ordered variant set for a variant engine)
//   [16, 24)  key u64; [24] active, [25] pending variant (0 in a single-blob engine, which has neither array)
//   [32, ..)  every other array in list order, each row at a 16-byte offset
// `allocate` (mp_create): first gives every array that has an allocation of its own its B zeroed rows. reward,
// discount, step_type and scalar_obs are carved from the scalar block; mp_create_variants adds active and pending.
constexpr uint32_t kRecordFormat = 0x3152504du;  // "MPR1"
int layout_state(mp_engine* E, bool allocate) {
  const Tables& T = E->T;
  State& S = E->S;
  const uint32_t P = T.P;
  RecordLayout& R = E->record;
  R = RecordLayout{};  // key_row 0: the key is the first row
  uint32_t off = 16;
  int rc = MP_OK;
  auto row = [&](void* base, uint32_t bytes, uint32_t align) {
    if (R.n_rows == MP_RECORD_MAX_ROWS) { rc = fail(MP_E_UNSUPPORTED, "more than %d per-env state arrays", MP_RECORD_MAX_ROWS); return; }
    off = (off + align - 1) / align * align;
    R.row[R.n_rows++] = {static_cast<uint8_t*>(base), bytes, bytes, off};
    off += bytes;
  };
  auto own = [&](auto*& p, uint32_t bytes, uint32_t align = 16) {
    if (allocate && !rc) rc = E->alloc((size_t)E->B * bytes / sizeof *p, &p);
    row(p, bytes, align);
  };
  own(S.key, 8, 8);
  row(E->variants.active, 1, 1); row(E->variants.pending, 1, 1);
  own(S.grid, T.L * T.cells_pad * 2); own(S.avatar, P * 16); own(S.av_timer, P * 16);
  own(S.apple, T.nA_pad); own(S.dirt, T.nD_pad); own(S.water, T.nW_pad); own(S.apple_count, T.nA_pad);
  own(S.fam_u8, S.fam_u8_stride); own(S.fam_u16, S.fam_u16_stride * 2); own(S.av_extra, P * 32);
  own(S.packed, (P + 2) * 8); own(S.env, ENV_COLS * 4);
  row(S.reward, P * 8, 16); row(S.discount, 8, 16); row(S.step_type, 8, 16);
  for (int k = 0; k < T.n_scalar; ++k) row(S.scalar_obs + (size_t)k * E->B * P, P * 8, 16);
  own(S.events, S.max_events * 12); own(S.n_events, 4);
  if (rc) return rc;
  R.record_bytes = (off + 15) / 16 * 16;
  const uint64_t h = E->blob_hash;
  R.tag = make_uint4(kRecordFormat, (uint32_t)R.record_bytes, (uint32_t)h, (uint32_t)(h >> 32));
  CUDA_TRY(cudaMemcpy(E->d_record_layout, &R, sizeof R, cudaMemcpyHostToDevice));
  return MP_OK;
}

}  // namespace

extern "C" {

const char* mp_last_error(void) { return g_error.c_str(); }
const char* mp_version(void) { return "meltingpot_b200 engine 0.1 (sm_90a)"; }

}  // extern "C"

namespace {
int setup_variants(Decoded& D, const void* const* blobs, const size_t* blob_bytes, int n);
int upload_tables(mp_engine* E, Decoded& D);
int upload_variants(mp_engine* E, const Decoded& D, const void* const* blobs, const size_t* blob_bytes, int n, const uint8_t* env_variant_host);

// mp_create (one blob) and mp_create_variants (a checked variant set of n_blobs > 1, env b starting on env_variant[b]).
// Every check of the blobs runs before the device is opened.
int create(const void* const* blobs, const size_t* blob_sizes, int n_blobs, const uint8_t* env_variant, int num_envs, int device,
           uint64_t seed, uint64_t env_index_base, uint32_t flags, mp_handle* out) {
  Decoded D(n_blobs);
  int rc = build_tables(D, blobs, blob_sizes, n_blobs, flags);
  // before the state is sized: the variants of a map-variant engine size its entity arrays for the largest of them
  if (rc == MP_OK && n_blobs > 1) rc = setup_variants(D, blobs, blob_sizes, n_blobs);
  if (rc != MP_OK) return rc;
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0) return fail(MP_E_NO_DEVICE, "no CUDA device available (%s); this engine has no CPU path", cudaGetErrorString(e));
  if (device < 0 || device >= n_dev || device >= MP_MAX_DEVICES) return fail(MP_E_INVALID, "device %d out of range (0..%d)", device, n_dev - 1);
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(MP_E_NO_DEVICE, "device %d is sm_%d%d; kernels are built for sm_90a only", device, prop.major, prop.minor);
  DeviceGuard guard(device);
  mp_engine* E = new mp_engine();
  clear_last_launch(E);
  E->device = device; E->B = num_envs; E->flags = flags; E->sm_count = prop.multiProcessorCount;
  E->blob_hash = fnv1a(blobs[0], blob_sizes[0]);
  rc = upload_tables(E, D);
  if (rc == MP_OK && n_blobs > 1) rc = upload_variants(E, D, blobs, blob_sizes, n_blobs, env_variant);
  if (rc == MP_OK) rc = build_plan(E);
  if (rc != MP_OK) {
    const std::string msg = g_error;
    mp_destroy(E);
    g_error = msg;
    return rc;
  }
  const Tables& T = E->T;
  State& S = E->S;
  S.B = num_envs; E->key_base = seed + env_index_base;
  const size_t B = num_envs, P = T.P;
  {  // Worst case of events one step can emit per env: per avatar, every cell of every beam footprint can carry a hit
     // with up to three events (zap + sanctioning + removal), plus the contact / regrowth events (<= 4) and the pair
     // events of coop_mining (<= P). Sized so that emit_event never drops a row.
    S.max_events = round_up(std::max(MP_MIN_EVENTS, T.P * (3 * D.beam_cells + 4 + T.P)), 16);
  }
  S.fam_u8_stride = std::max(16, RU_COUNT * T.nR_pad); S.fam_u16_stride = std::max(16, RS_COUNT * T.nR_pad);
  // reward [B][P] | discount [B] | step_type [B] | scalar_obs [n][B][P], all 8-byte elements, one block
  E->scalar_block_bytes = (B * P + B + B + std::max<size_t>(1, T.n_scalar) * B * P) * 8;
  if ((rc = E->alloc(E->scalar_block_bytes, &E->scalar_block)) || (rc = E->alloc(B * P * E->R.player_bytes, &S.rgb)) ||
      (rc = E->alloc(B * (size_t)E->R.world_bytes, &S.world_rgb)) || (rc = E->alloc(B * P, &E->d_actions)) ||
      (rc = E->alloc(1, &E->d_record_layout))) {
    mp_destroy(E);
    return rc;
  }
  S.reward = reinterpret_cast<double*>(E->scalar_block);
  S.discount = S.reward + B * P;
  S.step_type = reinterpret_cast<int64_t*>(S.discount + B);
  S.scalar_obs = reinterpret_cast<double*>(S.step_type + B);
  if ((rc = layout_state(E, /*allocate=*/true))) {
    mp_destroy(E);
    return rc;
  }
  S.rgb_env_stride = P * E->R.player_bytes; S.world_env_stride = E->R.world_bytes;  // the own images: dense
  // episode counter starts at -1 so that the first reset plays episode 0; envs start "done".
  {
    std::vector<int32_t> env0(B * ENV_COLS, 0);
    for (size_t b = 0; b < B; ++b) { env0[b * ENV_COLS + ENV_EPISODE] = -1; env0[b * ENV_COLS + ENV_DONE] = 1; }
    std::vector<uint64_t> key0(B);
    for (size_t b = 0; b < B; ++b) key0[b] = E->key_base + b;
    cudaError_t ce = cudaMemcpy(S.env, env0.data(), env0.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (ce == cudaSuccess) ce = cudaMemcpy(S.key, key0.data(), key0.size() * sizeof(uint64_t), cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) { mp_destroy(E); return fail(MP_E_CUDA, "cudaMemcpy(env / key) failed: %s", cudaGetErrorString(ce)); }
  }
  E->step_smem = E->family->step_smem(T, n_blobs > 1);
  {  // cells per lane per strip: ceil(view_w / 4) for player rows, ceil(W / 8) for world half-rows
    const int ncp = (E->R.view_w + 3) / 4, ncw = (T.W + (32 >> E->R.wstrip_log2) - 1) / (32 >> E->R.wstrip_log2);
#define MP_RENDER_INST(NCP, NCW)                                                                                  \
  {                                                                                                               \
    E->render_fns[RENDER_PLAIN] = k_render<NCP, NCW, RENDER_PLAIN>;                                               \
    E->render_fns[RENDER_GATHER] = k_render<NCP, NCW, RENDER_GATHER>;                                             \
    E->render_fns[RENDER_ROUTED] = k_render<NCP, NCW, RENDER_ROUTED>; E->inst_ncp = NCP; E->inst_ncw = NCW;       \
  }
    if (ncp <= 3 && ncw <= 3) MP_RENDER_INST(3, 3)
    else if (ncp <= 3 && ncw <= 4) MP_RENDER_INST(3, 4)
    else if (ncp <= 3 && ncw <= 5) MP_RENDER_INST(3, 5)
    else if (ncp <= 4 && ncw <= 5) MP_RENDER_INST(4, 5)
#undef MP_RENDER_INST
    else { mp_destroy(E); return fail(MP_E_UNSUPPORTED, "view of %d cells / map of %d cells wide (max 16 / 40)", E->R.view_w, T.W); }
    // lane -> cell dealing (see make_lane_map_cells / make_lane_map): whole cells per lane group with the cell order chosen
    // to minimise store bank conflicts by default; the fully conflict-free scattered colouring or the plain order for A/B.
    const int wrows = 1 << E->R.wstrip_log2;
    if (flags & MP_FLAG_DEBUG_PLAIN_LANE_MAP) {
      for (int l = 0; l < 32; ++l) { E->R.pmap[l] = 0; for (int i = 0; i < 4; ++i) E->R.pmap[l] |= (uint32_t)std::min(63, (l >> 3) + 4 * i) << (6 * i); }
      for (int l = 0; l < 32; ++l) { E->R.wmap[l] = 0; for (int i = 0; i < 5; ++i) E->R.wmap[l] |= (uint32_t)std::min(63, (l >> E->R.wstrip_log2) + (32 >> E->R.wstrip_log2) * i) << (6 * i); }
    } else if ((flags & MP_FLAG_DEBUG_SCATTER_LANE_MAP) && make_lane_map(8, E->R.view_w, 3 * E->R.view_w, ncp, E->R.pmap) &&
               make_lane_map(wrows, T.W, 3 * T.W, ncw, E->R.wmap)) {
      E->lane_map_players = E->lane_map_world = 2;
    } else {
      E->lane_map_players = 1 + 16 * make_lane_map_cells(8, E->R.view_w, 3 * E->R.view_w, ncp, E->R.pmap);
      E->lane_map_world = 1 + 16 * make_lane_map_cells(wrows, T.W, 3 * T.W, ncw, E->R.wmap);
    }
  }
  // The attribute belongs to the kernel function, not to this handle: engines that share an instantiation must not
  // lower each other's limit, so the renderer always gets the opt-in maximum and the step kernels only ever raise theirs.
  cudaError_t ce = cudaSuccess;
  for (auto fn : E->render_fns)
    if (ce == cudaSuccess) ce = cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kRenderSmemLimit);
  {
    static int step_smem_max[MP_MAX_DEVICES] = {};
    const int need = (int)E->step_smem;
    if (ce == cudaSuccess && need > 48 * 1024 && need > step_smem_max[device]) {
      for (const FamilyEntry& f : kFamilies)
        for (const auto& by_restore : f.step)
          for (const auto& by_actions : by_restore)
            for (const void* k : by_actions)
              if (ce == cudaSuccess) ce = cudaFuncSetAttribute(k, cudaFuncAttributeMaxDynamicSharedMemorySize, need);
      if (ce == cudaSuccess) step_smem_max[device] = need;
    }
  }
  if (ce != cudaSuccess) { mp_destroy(E); return fail(MP_E_CUDA, "cudaFuncSetAttribute failed: %s", cudaGetErrorString(ce)); }
  mp_buffers& bf = E->buffers;
  bf.num_envs = num_envs; bf.num_players = T.P; bf.rgb_h = E->R.view_h * 8; bf.rgb_w = E->R.view_w * 8;
  bf.world_h = T.H * 8; bf.world_w = T.W * 8; bf.num_actions = T.n_actions; bf.num_scalar_obs = T.n_scalar;
  bf.rgb = S.rgb; bf.world_rgb = S.world_rgb; bf.reward = S.reward; bf.discount = S.discount; bf.step_type = S.step_type;
  bf.scalar_obs = S.scalar_obs; bf.avatar_state = S.avatar; bf.grid = S.grid; bf.timestep_packed = S.packed;
  bf.grid_layers = T.L; bf.grid_cells = T.cells; bf.grid_cells_padded = T.cells_pad;
  bf.events = S.events; bf.event_count = S.n_events; bf.max_events = S.max_events;
  bf.scalar_block = E->scalar_block; bf.scalar_block_bytes = E->scalar_block_bytes;
  // SURVEY.md section 8d: observations + scalars + actions + one read and one write of the compact grid.
  E->render_bytes = (uint64_t)P * E->R.player_bytes + (uint64_t)E->R.world_bytes + (uint64_t)T.L * T.cells * 2;
  E->algo_bytes = (uint64_t)P * E->R.player_bytes + (uint64_t)E->R.world_bytes + 8ull * ((1 + T.n_scalar) * P + 2) + 8ull * P + 2ull * T.L * T.cells * 2;
  *out = E;
  return MP_OK;
}

// Rule (a) of mp_create_variants: variant `v` has the same sections as variant 0, byte for byte, except the family's
// parameter blocks, the component tables and the metadata string. The variants of a family with map variants (maps
// compiled as one set on one sprite table; `map_sections` lists the family's entity tables, null for other families) may
// also differ in their map: the initial grid, the object table, the kind and state tables, the BeamBlocker bits, the
// spawn points and those entity tables, in the object, kind, state and component counts of 'meta', and in the sprite of
// each avatar. The kind and state tables are only read per blob, by load_map and the pre-merge enumeration of
// build_tables, never from variant 0 for every env. The sprite table itself (atlas, sprite_opaque, sprite_map) stays
// identical.
// Variants of any family (one set on one sprite table: appearance overrides) may also differ in which sprite ids their
// pieces use: the sprite column of 'states', the sprite of each non-empty cell of 'init_grid' (not which cells are
// empty, nor their orientations) and the family's tables of sprite ids (`sprite_sections`), where a sprite may change
// but not whether there is one. A section that differs in anything else is refused as before.
int same_sections(const void* b0, size_t n0, const void* bv, size_t nv, const char* const* map_sections,
                  const char* const* sprite_sections) {
  const bool maps = map_sections != nullptr;
  const MpbHeader* h0 = static_cast<const MpbHeader*>(b0);
  const MpbHeader* hv = static_cast<const MpbHeader*>(bv);
  if (n0 < sizeof(MpbHeader) || nv < sizeof(MpbHeader) || memcmp(hv->magic, MPB_MAGIC, 4) != 0 || hv->version != MPB_VERSION ||
      nv < sizeof(MpbHeader) + (size_t)hv->n_sections * sizeof(MpbSection))
    return fail(MP_E_INVALID, "blob: not an MPB%u blob", MPB_VERSION);
  auto free_to_differ = [maps, map_sections](const char* name) {
    const size_t len = strnlen(name, MPB_NAME_LEN);
    if ((len == 5 && name[2] == '_' && (name[3] == 'i' || name[3] == 'd') && name[4] == 'p') || !strcmp(name, "comps") ||
        !strcmp(name, "comps_f") || !strcmp(name, "info_json"))
      return true;
    if (!maps) return false;
    if (!strcmp(name, "init_grid") || !strcmp(name, "objects") || !strcmp(name, "kinds") || !strcmp(name, "states") ||
        !strcmp(name, "cell_flags") || !strncmp(name, "spawn_cells_", 12))
      return true;
    for (const char* const* t = map_sections; *t; ++t) if (!strcmp(name, *t)) return true;
    return false;
  };
  // map variants: the columns of an int32 section that may differ (a bit per column, of `cols`), or 0
  auto free_columns = [maps](const char* name, int* cols) -> uint64_t {
    if (!maps) return 0;
    if (!strcmp(name, "meta")) {
      *cols = MPB_META_COUNT;
      return 1ull << MPB_META_N_OBJECTS | 1ull << MPB_META_N_KINDS | 1ull << MPB_META_N_STATES | 1ull << MPB_META_N_COMPS;
    }
    if (!strcmp(name, "av_table")) { *cols = 8; return 1ull << 1; }
    return 0;
  };
  static const char* const kMetaNames[] = {"family", "W", "H", "layers", "players", "sprite size", "topology", "max frames", "objects",
                                           "kinds", "states", "comps", "sprites", "hits", "groups", "view left", "view right",
                                           "view forward", "view backward", "actions", "action fields", "OutOfBounds sprite",
                                           "OutOfView sprite", "scalar observations"};
  const MpbSection* s0 = reinterpret_cast<const MpbSection*>(h0 + 1);
  const MpbSection* sv = reinterpret_cast<const MpbSection*>(hv + 1);
  // whether two sections of the same shape differ in sprite ids only
  auto sprite_ids_only = [sprite_sections](const char* name, const MpbSection* s, const void* x, const void* y) {
    const size_t n = s->nbytes / 4;
    const int32_t* a = static_cast<const int32_t*>(x);
    const int32_t* b = static_cast<const int32_t*>(y);
    if (!strcmp(name, "init_grid") && s->dtype == MPB_U16) {
      const uint16_t* p = static_cast<const uint16_t*>(x);
      const uint16_t* q = static_cast<const uint16_t*>(y);
      for (size_t k = 0; k < s->nbytes / 2; ++k)
        if ((p[k] == 0) != (q[k] == 0) || (p[k] && ((p[k] - 1) & 3) != ((q[k] - 1) & 3))) return false;
      return true;
    }
    if (s->dtype != MPB_I32) return false;
    if (!strcmp(name, "states")) {
      for (size_t k = 0; k < n; ++k)
        if (k % MPB_STATE_COLS == MPB_STATE_SPRITE ? (a[k] < 0) != (b[k] < 0) : a[k] != b[k]) return false;
      return true;
    }
    for (const char* const* t = sprite_sections; t && *t; ++t)
      if (!strcmp(name, *t)) {
        for (size_t k = 0; k < n; ++k) if ((a[k] < 0) != (b[k] < 0)) return false;
        return true;
      }
    return false;
  };
  auto check = [&](const MpbSection* s, uint32_t count, const void* other, size_t n_other, const void* own) -> int {
    for (uint32_t i = 0; i < count; ++i) {
      char name[MPB_NAME_LEN + 1] = {};
      memcpy(name, s[i].name, MPB_NAME_LEN);
      if (free_to_differ(name)) continue;
      const MpbSection* t = mpb_find(other, n_other, name);
      const bool same_shape = t && t->dtype == s[i].dtype && t->ndim == s[i].ndim && memcmp(t->shape, s[i].shape, sizeof t->shape) == 0 &&
                              t->nbytes == s[i].nbytes;
      if (same_shape && sprite_ids_only(name, &s[i], mpb_data(own, &s[i]), mpb_data(other, t))) continue;
      int cols = 0;
      const uint64_t free_cols = free_columns(name, &cols);
      if (same_shape && free_cols && s[i].dtype == MPB_I32) {
        const int32_t* x = static_cast<const int32_t*>(mpb_data(own, &s[i]));
        const int32_t* y = static_cast<const int32_t*>(mpb_data(other, t));
        for (size_t k = 0; k < s[i].nbytes / 4; ++k) {
          if ((free_cols >> (k % cols) & 1u) || x[k] == y[k]) continue;
          if (!strcmp(name, "meta") && k < sizeof kMetaNames / sizeof *kMetaNames)
            return fail(MP_E_UNSUPPORTED, "section 'meta' differs in field '%s' (%d vs %d)", kMetaNames[k], x[k], y[k]);
          return fail(MP_E_UNSUPPORTED, "section '%s' differs in value %zu (column %zu)", name, k, k % cols);
        }
        continue;
      }
      if (!same_shape || memcmp(mpb_data(other, t), mpb_data(own, &s[i]), s[i].nbytes) != 0)
        return fail(MP_E_UNSUPPORTED, maps ? "section '%s' differs (map variants may differ only in the family's parameters and their map)"
                                           : "section '%s' differs (variants may differ only in the family's parameters)", name);
    }
    return MP_OK;
  };
  int rc = check(s0, h0->n_sections, bv, nv, b0);
  return rc ? rc : check(sv, hv->n_sections, b0, n0, bv);
}

// Rules (b)-(d) of mp_create_variants for a set whose blob 0 build_tables has decoded: each variant's loader (its
// refusal, kept by build_tables), its entity counts, episode ending, beam footprints and Params (same_shape), then its
// map. A family with map variants keeps each variant's map (MapVariant) and entity tables, and the State's entity
// arrays (T.nA_pad) are sized for the variant with the most. Its variants may also differ in their beam footprints, as
// far as the family's same_shape allows (commons_harvest: the Zapper's length and radius; coins has no beams), and
// State::max_events is sized for the largest footprint. Every variant engine keeps the Tables of each variant
// (VariantSet::maps), from which an episode start reads: the variants of the other families differ there in their
// initial grid only (the sprites of an appearance override).
int setup_variants(Decoded& D, const void* const* blobs, const size_t* blob_bytes, int n) {
  const bool maps = D.family->map_variants;
  Tables& T = D.T;
  const FamilyLoad& a = D.loads[0];
  for (int v = 1; v < n; ++v) {
    const FamilyLoad& b = D.loads[v];
    int rc = D.load_rc[v];
    if (rc) g_error = D.load_error[v];
    else if ((!maps && (a.nA != b.nA || a.nR != b.nR || a.nR_pad != b.nR_pad)) || a.nD != b.nD || a.nW != b.nW) rc = fail(MP_E_UNSUPPORTED, "entity counts differ");
    else if (a.end_min_frames != b.end_min_frames || a.end_interval != b.end_interval || memcmp(&a.end_prob, &b.end_prob, sizeof a.end_prob) != 0)
      rc = fail(MP_E_UNSUPPORTED, "episode ending differs");
    else if (!maps && a.beam_cells != b.beam_cells) rc = fail(MP_E_UNSUPPORTED, "beam footprints differ");
    else rc = D.family->same_shape(D.params[0], D.params[v]);
    if (rc == MP_OK) rc = load_map(blobs[v], blob_bytes[v], T, D.spawn_groups, D.tables, D.maps[v]);
    if (rc) {
      g_error = "variant " + std::to_string(v) + ": " + g_error;
      return rc;
    }
  }
  if (maps) {
    for (const FamilyLoad& l : D.loads) {
      T.nA = std::max(T.nA, l.nA); T.nR = std::max(T.nR, l.nR); T.nR_pad = std::max(T.nR_pad, l.nR_pad);
      D.beam_cells = std::max(D.beam_cells, l.beam_cells);
    }
    T.nA_pad = round_up(std::max(T.nA, 1), 16); T.nD_pad = round_up(std::max(std::max(T.nD, T.nA), 1), 16);
  }
  return MP_OK;
}

// Uploads every table the decode recorded and writes its device address into the field it is aimed at, then puts the
// decoded Tables and variant 0's Params into the engine. No kernel writes these tables, so tables with the same bytes
// share one allocation: the variants of a set point at one copy of every table they may not differ in (rule (a) of
// mp_create_variants), as map variants do at the tables their maps share.
int upload_tables(mp_engine* E, Decoded& D) {
  std::map<std::vector<uint8_t>, const uint8_t*> shared;
  auto put = [&](const std::vector<HostTable>& tables) {
    for (const HostTable& t : tables) {
      const uint8_t*& d = shared[t.bytes];
      int rc;
      if (!d && (rc = upload(E->allocs, t.bytes, &d))) return rc;
      memcpy(t.field, &d, sizeof d);
    }
    return (int)MP_OK;
  };
  int rc = put(D.tables);
  for (const FamilyLoad& l : D.loads) if (rc == MP_OK) rc = put(l.tables);
  if (rc) return rc;
  apply_map(D.T, D.maps[0]);
  E->family = D.family; E->T = D.T; E->params = D.params[0];
  E->n_total = D.n_total; E->black_sprite = D.black_sprite; E->host_pair = D.host_pair; E->host_sflags = D.host_sflags;
  return MP_OK;
}

// The device arrays of a variant set: each variant's Tables (the engine's, with its map and entity count) and own Params,
// and the env assignments.
int upload_variants(mp_engine* E, const Decoded& D, const void* const* blobs, const size_t* blob_bytes, int n, const uint8_t* env_variant_host) {
  int rc;
  {
    std::vector<Tables> tv(n, E->T);  // T is final here: create changes nothing in it after this
    for (int v = 0; v < n; ++v) { apply_map(tv[v], D.maps[v]); tv[v].nA = D.loads[v].nA; tv[v].nR = D.loads[v].nR; }
    const Tables* d = nullptr;
    if ((rc = upload(E->allocs, tv, &d))) return rc;
    E->variants.maps = d;
  }
  if ((rc = E->family->upload_variants(E->allocs, D.params, &E->variants.params))) return rc;
  const size_t B = E->B;
  std::vector<uint8_t> assign(B, 0);
  if (env_variant_host) assign.assign(env_variant_host, env_variant_host + B);
  const uint8_t* d = nullptr;
  if ((rc = upload(E->allocs, assign, &d))) return rc;
  E->variants.active = const_cast<uint8_t*>(d);
  if ((rc = upload(E->allocs, assign, &d))) return rc;
  E->variants.pending = const_cast<uint8_t*>(d);
  E->variants.n = n;
  // records and snapshots carry the assignments, and only load into an engine with the same variants in the same order
  uint64_t h = fnv1a(&n, sizeof n);
  for (int v = 0; v < n; ++v) { const uint64_t hv = fnv1a(blobs[v], blob_bytes[v]); h = fnv1a(&hv, sizeof hv, h); }
  E->blob_hash = h;
  return MP_OK;
}
}  // namespace

extern "C" {

int mp_create(const void* blob, size_t blob_bytes, int num_envs, int device, uint64_t seed, uint64_t env_index_base, uint32_t flags, mp_handle* out) {
  if (!blob || !out || num_envs < 1) return fail(MP_E_INVALID, "mp_create: bad arguments");
  return create(&blob, &blob_bytes, 1, nullptr, num_envs, device, seed, env_index_base, flags, out);
}

int mp_create_variants(const void* const* blobs, const size_t* blob_bytes, int n_variants, const uint8_t* env_variant_host, int num_envs,
                       int device, uint64_t seed, uint64_t env_index_base, uint32_t flags, mp_handle* out) {
  if (!blobs || !blob_bytes || !out || num_envs < 1 || n_variants < 1 || n_variants > MP_MAX_VARIANTS)
    return fail(MP_E_INVALID, "mp_create_variants: bad arguments (1..%d variants)", MP_MAX_VARIANTS);
  *out = nullptr;
  for (int v = 0; v < n_variants; ++v) if (!blobs[v]) return fail(MP_E_INVALID, "mp_create_variants: null blob %d", v);
  if (env_variant_host)
    for (int b = 0; b < num_envs; ++b)
      if (env_variant_host[b] >= n_variants) return fail(MP_E_INVALID, "mp_create_variants: env %d assigned variant %d of %d", b, env_variant_host[b], n_variants);
  // whether the family (of variant 0) takes map variants decides which sections may differ
  const FamilyEntry* family = nullptr;
  if (const MpbSection* m = mpb_find(blobs[0], blob_bytes[0], "meta"))
    if (m->dtype == MPB_I32 && m->nbytes >= 4) family = find_family(static_cast<const int32_t*>(mpb_data(blobs[0], m))[MPB_META_FAMILY]);
  const char* const* map_sections = family ? family->map_sections : nullptr;
  const char* const* sprite_sections = family ? family->sprite_sections : nullptr;
  for (int v = 1; v < n_variants; ++v)
    if (int rc = same_sections(blobs[0], blob_bytes[0], blobs[v], blob_bytes[v], map_sections, sprite_sections)) {
      g_error = "variant " + std::to_string(v) + ": " + g_error;
      return rc;
    }
  return create(blobs, blob_bytes, n_variants, env_variant_host, num_envs, device, seed, env_index_base, flags, out);
}

int mp_set_env_variants(mp_handle h, const uint8_t* env_variant, void* stream) {
  if (!h || !env_variant) return fail(MP_E_INVALID, "mp_set_env_variants: null argument");
  if (h->variants.n < 2) return fail(MP_E_INVALID, "mp_set_env_variants: the engine has one parameter set (create it with mp_create_variants)");
  DeviceGuard guard(h->device);
  CUDA_TRY(cudaMemcpyAsync(h->variants.pending, env_variant, (size_t)h->B, cudaMemcpyDeviceToDevice, (cudaStream_t)stream));
  return MP_OK;
}

int mp_env_variants(mp_handle h, int* n_variants, uint8_t** active, uint8_t** pending) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  if (n_variants) *n_variants = h->variants.n;
  if (active) *active = h->variants.active;
  if (pending) *pending = h->variants.pending;
  return MP_OK;
}

int mp_destroy(mp_handle h) {
  if (!h) return MP_OK;
  {
    DeviceGuard guard(h->device);
    cudaDeviceSynchronize();
    for (auto& sl : h->slot) { if (sl.computed) cudaEventDestroy(sl.computed); if (sl.copied) cudaEventDestroy(sl.copied); }
    if (h->copy_stream) cudaStreamDestroy(h->copy_stream);
    for (void* p : h->allocs) cudaFree(p);
  }
  delete h;
  return MP_OK;
}

int mp_set_flags(mp_handle h, uint32_t flags) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  h->flags = (flags & ~(uint32_t)MP_FLAGS_CREATE_ONLY) | (h->flags & (uint32_t)MP_FLAGS_CREATE_ONLY);
  return MP_OK;
}

int mp_step_state(mp_handle h, const int32_t* actions, void* stream) {
  if (!h || !actions) return fail(MP_E_INVALID, "mp_step_state: null handle or actions");
  DeviceGuard guard(h->device);
  return launch_state(h, actions, nullptr, 0, (cudaStream_t)stream, /*render_follows=*/false);
}

int mp_render(mp_handle h, void* stream) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  DeviceGuard guard(h->device);
  clear_last_launch(h);
  return launch_render(h, (cudaStream_t)stream);
}

}  // extern "C"

namespace {
typedef unsigned __int128 u128;
// A caller-owned device range an entry point reads or writes: `extent` bytes from `p`.
struct DeviceExtent { const char* name; uintptr_t p; u128 extent; };

// Each extent spans less than 2^48 bytes, lies inside one device allocation on the engine's device and overlaps neither
// another extent nor the engine's own buffers (mp_run's targets, row maps and action rows, the bank and index arrays of
// mp_state_store / mp_state_restore / mp_run).
int check_extents(mp_engine* E, const std::vector<DeviceExtent>& outs, const char* fn) {
  const uint64_t B = E->B, P = E->T.P;
  for (const DeviceExtent& x : outs)
    if (x.extent >= ((u128)1 << 48)) return fail(MP_E_INVALID, "%s: %s spans more than 2^48 bytes", fn, x.name);
  // each extent inside one device allocation on the engine's device (cuMemGetAddressRange through the runtime's driver
  // entry point, as mp_ipc_export does, so the library does not link libcuda)
  typedef int (*GetRange)(unsigned long long*, size_t*, unsigned long long);
  void* range_fn = nullptr;
  cudaDriverEntryPointQueryResult qr;
  CUDA_TRY(cudaGetDriverEntryPoint("cuMemGetAddressRange", &range_fn, cudaEnableDefault, &qr));
  if (!range_fn || qr != cudaDriverEntryPointSuccess) return fail(MP_E_CUDA, "cuMemGetAddressRange is not available");
  for (const DeviceExtent& x : outs) {
    cudaPointerAttributes a{};
    if (cudaPointerGetAttributes(&a, (const void*)x.p) != cudaSuccess) {
      cudaGetLastError();
      return fail(MP_E_INVALID, "%s: %s is not a device pointer", fn, x.name);
    }
    if (a.type != cudaMemoryTypeDevice) return fail(MP_E_INVALID, "%s: %s is not device memory", fn, x.name);
    if (a.device != E->device) return fail(MP_E_INVALID, "%s: %s lies on device %d, the engine runs on device %d", fn, x.name, a.device, E->device);
    unsigned long long base = 0;
    size_t size = 0;
    if (reinterpret_cast<GetRange>(range_fn)(&base, &size, (unsigned long long)x.p) != 0)
      return fail(MP_E_INVALID, "%s: %s is not in a device allocation", fn, x.name);
    if ((u128)x.p + x.extent > (u128)base + size)
      return fail(MP_E_INVALID, "%s: %s runs %llu bytes past the end of its allocation", fn, x.name,
                  (unsigned long long)((u128)x.p + x.extent - ((u128)base + size)));
  }
  // no extent overlaps another output or the engine's own buffers
  // (the whole scalar block: it also holds the unused scalar_obs row of a substrate without scalar observations)
  std::vector<std::pair<uintptr_t, uint64_t>> own{{(uintptr_t)E->scalar_block, E->scalar_block_bytes}};
  for (int r = 0; r < E->record.n_rows; ++r)
    if (E->record.row[r].base) own.push_back({(uintptr_t)E->record.row[r].base, B * E->record.row[r].bytes});
  own.push_back({(uintptr_t)E->S.rgb, B * P * E->R.player_bytes});
  own.push_back({(uintptr_t)E->S.world_rgb, B * E->R.world_bytes});
  if (E->async_ready) {
    own.push_back({(uintptr_t)E->slot[1].rgb, B * P * E->R.player_bytes});
    own.push_back({(uintptr_t)E->slot[1].world_rgb, B * E->R.world_bytes});
  }
  for (size_t i = 0; i < outs.size(); ++i) {
    const u128 lo = outs[i].p, hi = lo + outs[i].extent;
    for (size_t j = i + 1; j < outs.size(); ++j)
      if (lo < (u128)outs[j].p + outs[j].extent && (u128)outs[j].p < hi)
        return fail(MP_E_INVALID, "%s: %s and %s overlap", fn, outs[i].name, outs[j].name);
    for (const auto& sp : own)
      if (lo < (u128)sp.first + sp.second && (u128)sp.first < hi) return fail(MP_E_INVALID, "%s: %s overlaps the engine's own buffers", fn, outs[i].name);
  }
  return MP_OK;
}

// A caller-owned target of `count` records (`unit`: "env" or "row") of `per_record` bytes, `stride` bytes apart, plus
// `extra` bytes past the last one (scalar_obs' other observations): checks the pointer and stride against `align` and
// one record, and 8-byte targets' stride against 2 GiB, then appends its extent to `ext` for check_extents. Extents are
// computed in 128 bits, so no stride can wrap them around. A null `p` is not asked for.
int add_strided(std::vector<DeviceExtent>& ext, const char* fn, const char* unit, const char* name, const void* p, uint64_t stride,
                uint64_t count, uint64_t per_record, uint64_t align, u128 extra) {
  if (!p) return MP_OK;
  if ((uintptr_t)p % align || stride % align)
    return fail(MP_E_INVALID, "%s: %s pointer or %s stride is not a multiple of %llu bytes", fn, name, unit, (unsigned long long)align);
  if (stride < per_record)
    return fail(MP_E_INVALID, "%s: %s %s stride of %llu bytes is smaller than one %s's %llu bytes", fn, name, unit,
                (unsigned long long)stride, unit, (unsigned long long)per_record);
  if (align == 8 && stride >= (1ull << 31)) return fail(MP_E_INVALID, "%s: %s %s stride of 2 GiB or more", fn, name, unit);
  ext.push_back({name, (uintptr_t)p, (u128)(count - 1) * stride + per_record + extra});
  return MP_OK;
}

// scalar_obs targets hold n x count rows of `bytes` bytes at k * s + r * e (observation k, env or row r, e >= bytes).
// Rows of one k are e apart; rows j = k' - k apart are |j * s + m * e| apart, m = r' - r in [-(count - 1), count - 1],
// closest at m = -floor(j * s / e) or one below.
int check_scalar_rows(const char* fn, const char* unit, const char* name, uint64_t s, uint64_t e, uint64_t n, uint64_t count,
                      uint64_t bytes) {
  for (uint64_t j = 1; j < n; ++j) {
    const u128 d = (u128)j * s, q = d / e, r = d % e;
    const u128 gap = q > count - 1 ? d - (u128)(count - 1) * e : (q + 1 <= count - 1 ? std::min<u128>(r, e - r) : r);
    if (gap < bytes) return fail(MP_E_INVALID, "%s: %s rows overlap (%s stride %llu, stride %llu bytes)", fn, name, unit,
                                 (unsigned long long)e, (unsigned long long)s);
  }
  return MP_OK;
}

// The checks of mp_run's `out` that need no other argument (include/mp_engine.h), before anything is enqueued: a pointer
// that fails one never reaches a kernel. Its extents are appended to `ext` for check_extents.
int check_device_outputs(mp_engine* E, const mp_device_outputs* o, const char* fn, std::vector<DeviceExtent>& ext) {
  const uint64_t B = E->B, P = E->T.P, n = E->T.n_scalar;
  if (o->rgb && !(E->flags & MP_FLAG_RENDER_PLAYERS)) return fail(MP_E_INVALID, "%s: rgb asked for, but the render flags switch the player images off", fn);
  if (o->world_rgb && !(E->flags & MP_FLAG_RENDER_WORLD)) return fail(MP_E_INVALID, "%s: world_rgb asked for, but the render flags switch WORLD.RGB off", fn);
  if (o->scalar_obs && n == 0) return fail(MP_E_INVALID, "%s: scalar_obs asked for, but this substrate has no scalar observations", fn);
  if (o->scalar_obs && o->scalar_obs_stride % 8) return fail(MP_E_INVALID, "%s: scalar_obs stride is not a multiple of 8 bytes", fn);
  int rc;
  if ((rc = add_strided(ext, fn, "env", "rgb", o->rgb, o->rgb_env_stride, B, P * E->R.player_bytes, 16, 0)) ||
      (rc = add_strided(ext, fn, "env", "world_rgb", o->world_rgb, o->world_rgb_env_stride, B, (uint64_t)E->R.world_bytes, 16, 0)) ||
      (rc = add_strided(ext, fn, "env", "reward", o->reward, o->reward_env_stride, B, P * 8, 8, 0)) ||
      (rc = add_strided(ext, fn, "env", "discount", o->discount, o->discount_env_stride, B, 8, 8, 0)) ||
      (rc = add_strided(ext, fn, "env", "step_type", o->step_type, o->step_type_env_stride, B, 8, 8, 0)) ||
      (rc = add_strided(ext, fn, "env", "scalar_obs", o->scalar_obs, o->scalar_obs_env_stride, B, P * 8, 8,
                        (u128)(n - 1) * o->scalar_obs_stride)))
    return rc;
  return o->scalar_obs ? check_scalar_rows(fn, "env", "scalar_obs", o->scalar_obs_stride, o->scalar_obs_env_stride, n, B, P * 8) : MP_OK;
}
}  // namespace

extern "C" {

int mp_get_buffers(mp_handle h, mp_buffers* out) {
  if (!h || !out) return fail(MP_E_INVALID, "null argument");
  *out = h->buffers;
  return MP_OK;
}

int mp_step_host(mp_handle h, const int32_t* actions_host, const mp_host_outputs* out, void* stream) {
  if (!h || !actions_host) return fail(MP_E_INVALID, "mp_step_host: null handle or actions");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  CUDA_TRY(cudaMemcpyAsync(h->d_actions, actions_host, (size_t)h->B * h->T.P * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  int rc = launch_state(h, h->d_actions, nullptr, 0, st);
  if (!rc) rc = launch_render(h, st);
  if (!rc) rc = copy_out(h, out, st);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(st));
  return MP_OK;
}

int mp_reset_host(mp_handle h, const mp_host_outputs* out, void* stream) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  int rc = launch_state(h, nullptr, nullptr, 1, st);
  if (!rc) rc = launch_render(h, st);
  if (!rc) rc = copy_out(h, out, st);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(st));
  return MP_OK;
}

namespace {
// Lazily sets up the two slots of mp_step_host_async. Slot 0 renders into the engine's own images (mp_buffers.rgb /
// world_rgb); slot 1 gets a second set, so the kernels of one step can run while the previous step's images are
// still being copied out.
int async_setup(mp_engine* E) {
  if (E->async_ready) return MP_OK;
  const size_t B = E->B, P = E->T.P;
  int rc;
  E->slot[0].rgb = E->S.rgb; E->slot[0].world_rgb = E->S.world_rgb;
  if ((rc = E->alloc(B * P * E->R.player_bytes, &E->slot[1].rgb)) || (rc = E->alloc(B * (size_t)E->R.world_bytes, &E->slot[1].world_rgb))) return rc;
  for (auto& sl : E->slot) {
    if ((rc = E->alloc(B * P, &sl.actions)) || (rc = E->alloc(E->scalar_block_bytes, &sl.scalars))) return rc;
    CUDA_TRY(cudaEventCreateWithFlags(&sl.computed, cudaEventDisableTiming));
    CUDA_TRY(cudaEventCreateWithFlags(&sl.copied, cudaEventDisableTiming));
  }
  CUDA_TRY(cudaStreamCreateWithFlags(&E->copy_stream, cudaStreamNonBlocking));
  E->async_ready = true;
  return MP_OK;
}
}  // namespace

int mp_step_host_async(mp_handle h, const int32_t* actions_host, const mp_host_outputs* out, int slot, void* stream) {
  if (!h || !actions_host || slot < 0 || slot > 1) return fail(MP_E_INVALID, "mp_step_host_async: null handle / actions or slot outside 0..1");
  // (every argument is checked before anything is enqueued: a refused call leaves the envs where they were)
  if (out && (out->events || out->event_count)) return fail(MP_E_INVALID, "mp_step_host_async: events are not staged per slot; read them with mp_step_host");
  DeviceGuard guard(h->device);
  int rc = async_setup(h);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  mp_engine::AsyncSlot& sl = h->slot[slot];
  CUDA_TRY(cudaStreamWaitEvent(st, sl.copied, 0));  // the copy-out that last used this slot's device buffers has drained
  CUDA_TRY(cudaMemcpyAsync(sl.actions, actions_host, (size_t)h->B * h->T.P * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if ((rc = launch_state(h, sl.actions, nullptr, 0, st))) return rc;
  mp_device_outputs second{};  // slot 1: a dense target in the engine's second image set
  if (slot == 1) {
    if (h->flags & MP_FLAG_RENDER_PLAYERS) { second.rgb = sl.rgb; second.rgb_env_stride = (uint64_t)h->T.P * h->R.player_bytes; }
    if (h->flags & MP_FLAG_RENDER_WORLD) { second.world_rgb = sl.world_rgb; second.world_rgb_env_stride = (uint64_t)h->R.world_bytes; }
  }
  if ((rc = launch_render(h, st, slot == 1 ? &second : nullptr))) return rc;
  CUDA_TRY(cudaMemcpyAsync(sl.scalars, h->scalar_block, h->scalar_block_bytes, cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaEventRecord(sl.computed, st));
  CUDA_TRY(cudaStreamWaitEvent(h->copy_stream, sl.computed, 0));
  if (out) {
    const size_t B = h->B, P = h->T.P;
    cudaStream_t cs = h->copy_stream;
    if (out->rgb) CUDA_TRY(cudaMemcpyAsync(out->rgb, sl.rgb, B * P * h->R.player_bytes, cudaMemcpyDeviceToHost, cs));
    if (out->world_rgb) CUDA_TRY(cudaMemcpyAsync(out->world_rgb, sl.world_rgb, B * h->R.world_bytes, cudaMemcpyDeviceToHost, cs));
    if (out->scalar_block) CUDA_TRY(cudaMemcpyAsync(out->scalar_block, sl.scalars, h->scalar_block_bytes, cudaMemcpyDeviceToHost, cs));
    else {
      const uint8_t* sb = sl.scalars;
      if (out->reward) CUDA_TRY(cudaMemcpyAsync(out->reward, sb, B * P * 8, cudaMemcpyDeviceToHost, cs));
      if (out->discount) CUDA_TRY(cudaMemcpyAsync(out->discount, sb + B * P * 8, B * 8, cudaMemcpyDeviceToHost, cs));
      if (out->step_type) CUDA_TRY(cudaMemcpyAsync(out->step_type, sb + (B * P + B) * 8, B * 8, cudaMemcpyDeviceToHost, cs));
      if (out->scalar_obs && h->T.n_scalar) CUDA_TRY(cudaMemcpyAsync(out->scalar_obs, sb + (B * P + 2 * B) * 8, (size_t)h->T.n_scalar * B * P * 8, cudaMemcpyDeviceToHost, cs));
    }
  }
  CUDA_TRY(cudaEventRecord(sl.copied, h->copy_stream));
  return MP_OK;
}

int mp_wait(mp_handle h, int slot) {
  if (!h || slot < 0 || slot > 1) return fail(MP_E_INVALID, "mp_wait: null handle or slot outside 0..1");
  if (!h->async_ready) return MP_OK;
  DeviceGuard guard(h->device);
  CUDA_TRY(cudaEventSynchronize(h->slot[slot].copied));
  return MP_OK;
}

// ---- cross-GPU exchange of the stacked timestep ---------------------------------------------------------------------
int mp_exchange_create(mp_handle h, int rank, int world, void** block, uint64_t* block_bytes) {
  if (!h || world < 1 || world > MP_MAX_PEERS || rank < 0 || rank >= world) return fail(MP_E_INVALID, "mp_exchange_create: rank %d / world %d (max %d ranks)", rank, world, MP_MAX_PEERS);
  if (h->x_block) return fail(MP_E_INVALID, "mp_exchange_create: already created for this handle");
  DeviceGuard guard(h->device);
  const size_t n = (size_t)2 * world * h->B * (h->T.P + 2);
  int rc;
  // one allocation: flags (MP_EXCHANGE_HEADER bytes) then gathered, so that one IPC handle shares both
  if ((rc = h->alloc(MP_EXCHANGE_HEADER + n * sizeof(double), &h->x_block))) return rc;
  h->x_block_bytes = MP_EXCHANGE_HEADER + n * sizeof(double);
  h->S.x_rank = rank;  // x_world stays 0 (exchange off) until mp_exchange_connect
  h->buffers.gathered = reinterpret_cast<double*>(h->x_block + MP_EXCHANGE_HEADER); h->buffers.gathered_world = world;
  CUDA_TRY(cudaDeviceSynchronize());
  if (block) *block = h->x_block;
  if (block_bytes) *block_bytes = h->x_block_bytes;
  return MP_OK;
}

int mp_ipc_export(const void* device_ptr, void* handle64, uint64_t* offset) {
  if (!device_ptr || !handle64 || !offset) return fail(MP_E_INVALID, "mp_ipc_export: null argument");
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  cudaIpcMemHandle_t hd;
  CUDA_TRY(cudaIpcGetMemHandle(&hd, const_cast<void*>(device_ptr)));
  memcpy(handle64, &hd, sizeof hd);
  // The handle names the driver allocation that contains the pointer (cudaMalloc sub-allocates small requests), and
  // opening it yields that allocation's base: the receiver needs the pointer's offset from the base as well.
  typedef int (*GetRange)(unsigned long long*, size_t*, unsigned long long);
  void* fn = nullptr;
  cudaDriverEntryPointQueryResult qr;
  CUDA_TRY(cudaGetDriverEntryPoint("cuMemGetAddressRange", &fn, cudaEnableDefault, &qr));
  if (!fn || qr != cudaDriverEntryPointSuccess) return fail(MP_E_CUDA, "cuMemGetAddressRange is not available");
  unsigned long long base = 0; size_t size = 0;
  if (reinterpret_cast<GetRange>(fn)(&base, &size, (unsigned long long)(uintptr_t)device_ptr) != 0) return fail(MP_E_CUDA, "cuMemGetAddressRange failed");
  *offset = (uint64_t)((unsigned long long)(uintptr_t)device_ptr - base);
  return MP_OK;
}

int mp_ipc_open(int device, const void* handle64, uint64_t offset, void** device_ptr) {
  if (!handle64 || !device_ptr) return fail(MP_E_INVALID, "mp_ipc_open: null argument");
  DeviceGuard guard(device);
  cudaIpcMemHandle_t hd;
  memcpy(&hd, handle64, sizeof hd);
  void* base = nullptr;
  CUDA_TRY(cudaIpcOpenMemHandle(&base, hd, cudaIpcMemLazyEnablePeerAccess));
  *device_ptr = static_cast<uint8_t*>(base) + offset;
  return MP_OK;
}

int mp_enable_peer_access(int device, int peer_device) {
  if (device == peer_device) return MP_OK;
  DeviceGuard guard(device);
  int can = 0;
  CUDA_TRY(cudaDeviceCanAccessPeer(&can, device, peer_device));
  if (!can) return fail(MP_E_UNSUPPORTED, "device %d cannot access device %d (no NVLink / P2P path)", device, peer_device);
  cudaError_t e = cudaDeviceEnablePeerAccess(peer_device, 0);
  if (e == cudaErrorPeerAccessAlreadyEnabled) { cudaGetLastError(); return MP_OK; }
  CUDA_TRY(e);
  return MP_OK;
}

int mp_exchange_connect(mp_handle h, void* const* peer_blocks) {
  if (!h || !peer_blocks) return fail(MP_E_INVALID, "mp_exchange_connect: null argument");
  if (!h->x_block) return fail(MP_E_INVALID, "mp_exchange_connect: call mp_exchange_create first");
  const int world = h->buffers.gathered_world;
  if (peer_blocks[h->S.x_rank] != h->x_block) return fail(MP_E_INVALID, "mp_exchange_connect: entry %d must be this rank's own block", h->S.x_rank);
  for (int r = 0; r < world; ++r) {
    if (!peer_blocks[r]) return fail(MP_E_INVALID, "mp_exchange_connect: null pointer for rank %d", r);
    h->S.x_flags[r] = static_cast<unsigned long long*>(peer_blocks[r]);
    h->S.x_gathered[r] = reinterpret_cast<double*>(static_cast<uint8_t*>(peer_blocks[r]) + MP_EXCHANGE_HEADER);
  }
  h->S.x_world = world;
  return MP_OK;
}

// ---- stacked observations across GPUs -------------------------------------------------------------------------------
int mp_gather_obs_create(mp_handle h, int rank, int world, void** block, uint64_t* block_bytes) {
  if (!h || world < 1 || world > MP_MAX_PEERS || rank < 0 || rank >= world) return fail(MP_E_INVALID, "mp_gather_obs_create: rank %d / world %d (max %d ranks)", rank, world, MP_MAX_PEERS);
  if (h->g_block) return fail(MP_E_INVALID, "mp_gather_obs_create: already created for this handle");
  DeviceGuard guard(h->device);
  const size_t rgb_all = (size_t)world * h->B * h->T.P * h->R.player_bytes, world_all = (size_t)world * h->B * h->R.world_bytes;
  h->g_world_off = rgb_all;
  h->g_slot_bytes = (rgb_all + world_all + 255) / 256 * 256;
  h->g_block_bytes = MP_EXCHANGE_HEADER + 2 * h->g_slot_bytes;
  void* p = nullptr;
  CUDA_TRY(cudaMalloc(&p, h->g_block_bytes));  // (not zeroed: gigabytes; only the flags header is)
  h->allocs.push_back(p);
  h->g_block = static_cast<uint8_t*>(p);
  CUDA_TRY(cudaMemset(p, 0, MP_EXCHANGE_HEADER));
  CUDA_TRY(cudaDeviceSynchronize());
  h->g_world = world; h->g_rank = rank;
  h->buffers.gathered_rgb = h->g_block + MP_EXCHANGE_HEADER;
  h->buffers.gathered_world_rgb = h->g_block + MP_EXCHANGE_HEADER + h->g_world_off;
  h->buffers.gathered_obs_slot_bytes = h->g_slot_bytes;
  if (block) *block = h->g_block;
  if (block_bytes) *block_bytes = h->g_block_bytes;
  return MP_OK;
}

int mp_gather_obs_connect(mp_handle h, void* const* peer_blocks) {
  if (!h || !peer_blocks) return fail(MP_E_INVALID, "mp_gather_obs_connect: null argument");
  if (!h->g_block) return fail(MP_E_INVALID, "mp_gather_obs_connect: call mp_gather_obs_create first");
  if (peer_blocks[h->g_rank] != h->g_block) return fail(MP_E_INVALID, "mp_gather_obs_connect: entry %d must be this rank's own block", h->g_rank);
  DeviceGuard guard(h->device);
  std::vector<unsigned long long*> ptrs(MP_MAX_PEERS, nullptr);
  for (int r = 0; r < h->g_world; ++r) {
    if (!peer_blocks[r]) return fail(MP_E_INVALID, "mp_gather_obs_connect: null pointer for rank %d", r);
    h->g_peer[r] = static_cast<uint8_t*>(peer_blocks[r]);
    ptrs[r] = reinterpret_cast<unsigned long long*>(peer_blocks[r]);
  }
  int rc = h->alloc((size_t)MP_MAX_PEERS, &h->d_g_flag_ptrs);
  if (rc) return rc;
  CUDA_TRY(cudaMemcpy(h->d_g_flag_ptrs, ptrs.data(), MP_MAX_PEERS * sizeof(void*), cudaMemcpyHostToDevice));
  h->S.g_flags = reinterpret_cast<const unsigned long long*>(h->g_block);
  h->S.g_world = h->g_world;
  return MP_OK;
}

int mp_gather_obs_enable(mp_handle h, int on) {
  if (!h || !h->g_block || !h->d_g_flag_ptrs) return fail(MP_E_INVALID, "mp_gather_obs_enable: not connected");
  h->S.g_world = on ? h->g_world : 0;
  return MP_OK;
}

int mp_gather_obs_wait(mp_handle h, void* stream) {
  if (!h || !h->g_block) return fail(MP_E_INVALID, "mp_gather_obs_wait: not created");
  DeviceGuard guard(h->device);
  k_flag_wait<<<1, 32, 0, (cudaStream_t)stream>>>(reinterpret_cast<const unsigned long long*>(h->g_block), h->g_world, h->g_seq);
  ++h->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

int mp_gather_obs_slot(mp_handle h, int* slot, uint64_t* step) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  if (slot) *slot = (int)(h->g_seq & 1ull);
  if (step) *step = h->g_seq;
  return MP_OK;
}

int mp_exchange_wait(mp_handle h, void* stream) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  if (!h->S.x_world) return fail(MP_E_INVALID, "mp_exchange_wait: exchange not connected");
  DeviceGuard guard(h->device);
  k_exchange_wait<<<1, 32, 0, (cudaStream_t)stream>>>(h->S, h->x_seq);
  ++h->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

int mp_exchange_slot(mp_handle h, int* slot, uint64_t* step) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  if (slot) *slot = (int)(h->x_seq & 1ull);
  if (step) *step = h->x_seq;
  return MP_OK;
}

namespace {
// A snapshot: this header, then every per-env state array of the engine (layout_state) whole, in list order.
struct SnapshotHeader { char magic[4]; uint32_t version; uint64_t num_envs, payload_bytes, n_arrays, rng_key0, blob_hash; };

SnapshotHeader snapshot_header(const mp_engine* E) {
  SnapshotHeader hd{{'M', 'P', 'S', '5'}, 5u, (uint64_t)E->B, 0, 0, E->key_base, E->blob_hash};
  for (int r = 0; r < E->record.n_rows; ++r)
    if (E->record.row[r].base) { hd.payload_bytes += (uint64_t)E->B * E->record.row[r].bytes; ++hd.n_arrays; }
  return hd;
}
}  // namespace

int mp_state_size(mp_handle h, uint64_t* bytes) {
  if (!h || !bytes) return fail(MP_E_INVALID, "mp_state_size: null argument");
  *bytes = sizeof(SnapshotHeader) + snapshot_header(h).payload_bytes;
  return MP_OK;
}

int mp_state_save(mp_handle h, void* host_dst, void* stream) {
  if (!h || !host_dst) return fail(MP_E_INVALID, "mp_state_save: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const SnapshotHeader hd = snapshot_header(h);
  memcpy(host_dst, &hd, sizeof(hd));
  uint8_t* dst = static_cast<uint8_t*>(host_dst) + sizeof(hd);
  for (int r = 0; r < h->record.n_rows; ++r) {
    const RecordRow& w = h->record.row[r];
    if (!w.base) continue;
    CUDA_TRY(cudaMemcpyAsync(dst, w.base, (size_t)h->B * w.bytes, cudaMemcpyDeviceToHost, st));
    dst += (size_t)h->B * w.bytes;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return MP_OK;
}

int mp_state_load(mp_handle h, const void* host_src, uint64_t nbytes, void* stream) {
  if (!h || !host_src) return fail(MP_E_INVALID, "mp_state_load: null argument");
  if (nbytes < sizeof(SnapshotHeader)) return fail(MP_E_INVALID, "mp_state_load: %llu bytes is shorter than a snapshot header", (unsigned long long)nbytes);
  SnapshotHeader hd;
  memcpy(&hd, host_src, sizeof(hd));
  const SnapshotHeader own = snapshot_header(h);
  if (memcmp(hd.magic, own.magic, 4) != 0 || hd.version != own.version) return fail(MP_E_INVALID, "mp_state_load: not a snapshot (or one of an older engine)");
  if (hd.num_envs != own.num_envs || hd.payload_bytes != own.payload_bytes || hd.n_arrays != own.n_arrays)
    return fail(MP_E_INVALID, "mp_state_load: snapshot of %llu envs / %llu bytes does not fit this engine (%d envs / %llu bytes)",
                (unsigned long long)hd.num_envs, (unsigned long long)hd.payload_bytes, h->B, (unsigned long long)own.payload_bytes);
  if (nbytes != sizeof(SnapshotHeader) + hd.payload_bytes)
    return fail(MP_E_INVALID, "mp_state_load: buffer of %llu bytes, snapshot needs %llu (truncated?)", (unsigned long long)nbytes,
                (unsigned long long)(sizeof(SnapshotHeader) + hd.payload_bytes));
  if (hd.blob_hash != h->blob_hash) return fail(MP_E_INVALID, "mp_state_load: snapshot was taken from a different compiled substrate");
  if (hd.rng_key0 != h->key_base) return fail(MP_E_INVALID, "mp_state_load: snapshot was taken with a different seed / env_index_base (key %llu, engine %llu)",
                                              (unsigned long long)hd.rng_key0, (unsigned long long)h->key_base);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* src = static_cast<const uint8_t*>(host_src) + sizeof(hd);
  for (int r = 0; r < h->record.n_rows; ++r) {
    const RecordRow& w = h->record.row[r];
    if (!w.base) continue;
    CUDA_TRY(cudaMemcpyAsync(w.base, src, (size_t)h->B * w.bytes, cudaMemcpyHostToDevice, st));
    src += (size_t)h->B * w.bytes;
  }
  clear_last_launch(h);
  int rc = launch_render(h, st);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(st));
  return MP_OK;
}

// ---- per-env state bank (record layout: layout_state) -------------------------------------------------------------
int mp_state_record_bytes(mp_handle h, uint64_t* bytes, uint8_t tag[16]) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  if (bytes) *bytes = h->record.record_bytes;
  if (tag) memcpy(tag, &h->record.tag, 16);
  return MP_OK;
}

namespace {
// The host checks of mp_state_store / mp_state_restore / a restoring mp_run: the bank is 16-byte aligned and the index
// array 4-byte aligned. Their extents go to the front of `ext`, for check_extents: in device allocations on the engine's
// device, overlapping neither each other nor the engine's buffers nor the request's targets.
int check_bank(const void* bank, int n_slots, const int32_t* index, uint64_t index_count, uint64_t record_bytes, const char* fn,
               std::vector<DeviceExtent>& ext) {
  if ((uintptr_t)bank % 16) return fail(MP_E_INVALID, "%s: bank is not 16-byte aligned", fn);
  if ((uintptr_t)index % 4) return fail(MP_E_INVALID, "%s: index array is not 4-byte aligned", fn);
  ext.insert(ext.begin(), {{"bank", (uintptr_t)bank, (u128)n_slots * record_bytes}, {"index array", (uintptr_t)index, (u128)index_count * 4}});
  return MP_OK;
}

// The names of segment k's targets in refusals ("players segment k rgb", ...); without segments, the top-level names.
const char* segment_target_name(const mp_player_outputs* o, int k, int output) {
  static const char* const top[3] = {"players rgb", "players reward", "players scalar_obs"};
  static const std::vector<std::string> names = [] {
    std::vector<std::string> v;
    for (int s = 0; s < MP_MAX_ROW_SEGMENTS; ++s)
      for (const char* t : {"rgb", "reward", "scalar_obs"}) v.push_back("players segment " + std::to_string(s) + " " + t);
    return v;
  }();
  return o->n_segments > 0 ? names[k * 3 + output].c_str() : top[output];
}

// The checks of mp_run's `players` that need no other argument (include/mp_engine.h); its extents are appended to `ext`
// for check_extents. Row segments are checked as a table (range, order, one set of outputs), then each segment's targets
// over its own rows by the same checks as the top-level targets, which are one segment [0, n_rows) here.
int check_player_outputs(mp_engine* E, const mp_player_outputs* o, const mp_device_outputs* out, const char* fn, std::vector<DeviceExtent>& ext) {
  if (o->n_rows < 1) return fail(MP_E_INVALID, "%s: n_rows %d < 1", fn, o->n_rows);
  if (!o->row_of_player || (uintptr_t)o->row_of_player % 4) return fail(MP_E_INVALID, "%s: row_of_player is null or not 4-byte aligned", fn);
  if (E->g_world > 0 && E->S.g_world > 0)
    return fail(MP_E_UNSUPPORTED, "%s: the observation gather is enabled: its stacked slots stay dense and complete", fn);
  if (o->n_segments < 0 || o->n_segments > MP_MAX_ROW_SEGMENTS)
    return fail(MP_E_INVALID, "%s: n_segments %d outside 0..%d", fn, o->n_segments, MP_MAX_ROW_SEGMENTS);
  if (o->n_segments > 0 && (o->rgb || o->reward || o->scalar_obs))
    return fail(MP_E_INVALID, "%s: with row segments, the top-level rgb, reward and scalar_obs must be null", fn);
  for (int k = 0, end = 0; k < o->n_segments; ++k) {
    const mp_row_segment& g = o->segments[k];
    if (g.row_begin < end || g.row_end <= g.row_begin || g.row_end > o->n_rows)
      return fail(MP_E_INVALID, "%s: segment %d rows [%d, %d) are empty, unsorted, overlap segment %d or leave [0, %d)", fn, k,
                  g.row_begin, g.row_end, k - 1, o->n_rows);
    end = g.row_end;
    const mp_row_segment& g0 = o->segments[0];
    if (!g.rgb != !g0.rgb || !g.reward != !g0.reward || !g.scalar_obs != !g0.scalar_obs)
      return fail(MP_E_INVALID, "%s: segments 0 and %d carry different sets of outputs", fn, k);
  }
  const RowSegments G = row_segments(*o);
  const uint64_t n = E->T.n_scalar;
  if (G.s[0].rgb && !(E->flags & MP_FLAG_RENDER_PLAYERS)) return fail(MP_E_INVALID, "%s: rgb asked for, but the render flags switch the player images off", fn);
  if (G.s[0].rgb && out && out->rgb) return fail(MP_E_INVALID, "%s: rgb is both routed (players) and per env (out)", fn);
  if (G.s[0].scalar_obs && n == 0) return fail(MP_E_INVALID, "%s: scalar_obs asked for, but this substrate has no scalar observations", fn);
  for (int k = 0; k < G.n; ++k)
    if (G.s[k].scalar_obs && (G.s[k].scalar_obs_stride % 8 || G.s[k].scalar_obs_stride >= (1ull << 31)))
      return fail(MP_E_INVALID, "%s: %s stride is not a multiple of 8 bytes or is 2 GiB or more", fn,
                  o->n_segments ? segment_target_name(o, k, 2) : "scalar_obs");
  if (!o->world_rgb != !o->world_row_of_env) return fail(MP_E_INVALID, "%s: world_rgb and world_row_of_env go together", fn);
  if (o->world_rgb) {
    if (o->world_n_rows < 1) return fail(MP_E_INVALID, "%s: world_n_rows %d < 1", fn, o->world_n_rows);
    if ((uintptr_t)o->world_row_of_env % 4) return fail(MP_E_INVALID, "%s: world_row_of_env is not 4-byte aligned", fn);
    if (!(E->flags & MP_FLAG_RENDER_WORLD)) return fail(MP_E_INVALID, "%s: world_rgb asked for, but the render flags switch WORLD.RGB off", fn);
    if (out && out->world_rgb) return fail(MP_E_INVALID, "%s: world_rgb is both routed (players) and per env (out)", fn);
    ext.push_back({"world_row_of_env", (uintptr_t)o->world_row_of_env, (u128)E->B * 4});
  }
  ext.push_back({"row_of_player", (uintptr_t)o->row_of_player, (u128)E->B * E->T.P * 4});
  int rc;
  for (int k = 0; k < G.n; ++k) {
    const RowSegment& g = G.s[k];
    const uint64_t R = (uint64_t)(g.row_end - g.row_begin);
    if ((rc = add_strided(ext, fn, "row", segment_target_name(o, k, 0), g.rgb, g.rgb_row_stride, R, (uint64_t)E->R.player_bytes, 16, 0)) ||
        (rc = add_strided(ext, fn, "row", segment_target_name(o, k, 1), g.reward, g.reward_row_stride, R, 8, 8, 0)) ||
        (rc = add_strided(ext, fn, "row", segment_target_name(o, k, 2), g.scalar_obs, g.scalar_obs_row_stride, R, 8, 8,
                          (u128)(n - 1) * g.scalar_obs_stride)) ||
        (g.scalar_obs && (rc = check_scalar_rows(fn, "row", segment_target_name(o, k, 2), g.scalar_obs_stride, g.scalar_obs_row_stride, n, R, 8))))
      return rc;
  }
  return add_strided(ext, fn, "row", "players world_rgb", o->world_rgb, o->world_rgb_row_stride, (uint64_t)o->world_n_rows,
                     (uint64_t)E->R.world_bytes, 16, 0);
}

// The checks of mp_run's `player_actions` that need no other argument (include/mp_engine.h); its extents are appended
// to `ext` like check_player_outputs'. The row map is left out when it is `players`' own row map (both are only read).
int check_player_actions(mp_engine* E, const mp_player_actions* a, const mp_player_outputs* players, const char* fn,
                         std::vector<DeviceExtent>& ext) {
  if (a->n_rows < 1) return fail(MP_E_INVALID, "%s: actions n_rows %d < 1", fn, a->n_rows);
  if (!a->row_of_player || (uintptr_t)a->row_of_player % 4) return fail(MP_E_INVALID, "%s: actions row_of_player is null or not 4-byte aligned", fn);
  if (!a->action || (uintptr_t)a->action % 4 || a->action_row_stride % 4 || a->action_row_stride >= (1ull << 31))
    return fail(MP_E_INVALID, "%s: action is null, or its pointer or row stride is not a multiple of 4 bytes or is 2 GiB or more", fn);
  if (a->action_row_stride < 4) return fail(MP_E_INVALID, "%s: action row stride of %llu bytes is smaller than one row's 4 bytes", fn,
                                            (unsigned long long)a->action_row_stride);
  if (!players || players->row_of_player != a->row_of_player)
    ext.push_back({"actions row_of_player", (uintptr_t)a->row_of_player, (u128)E->B * E->T.P * 4});
  ext.push_back({"action", (uintptr_t)a->action, (u128)(a->n_rows - 1) * a->action_row_stride + 4});
  return MP_OK;
}

// The checks of mp_run's `draw` (include/mp_engine.h). Its row map is `players`' own, whose extent check_player_outputs
// appends (check_call requires `players` with a draw).
int check_route_draw(mp_engine* E, const mp_request& r, const char* fn) {
  const mp_route_draw* d = r.draw;
  if (d->n_rows < 1) return fail(MP_E_INVALID, "%s: draw n_rows %d < 1", fn, d->n_rows);
  if (r.players->row_of_player != d->row_of_player || r.players->n_rows != d->n_rows)
    return fail(MP_E_INVALID, "%s: players must deliver through the draw's row map and n_rows", fn);
  const mp_player_actions* a = r.player_actions;
  if (!r.reset && (!a || a->row_of_player != d->row_of_player || a->n_rows != d->n_rows))
    return fail(MP_E_INVALID, "%s: a drawn step must read player_actions through the draw's row map and n_rows", fn);
  for (int p = 0; p < E->T.P; ++p) {
    const int n = d->n_choices[p];
    if (n < 0 || n > MP_MAX_ROUTE_CHOICES)
      return fail(MP_E_INVALID, "%s: player %d has %d choices, not 0..%d", fn, p, n, MP_MAX_ROUTE_CHOICES);
    for (int j = 0; j < n; ++j) {
      const int64_t base = d->row_base[p][j], per_env = d->rows_per_env[p][j];
      if (base < 0 || per_env < 0 || base + (int64_t)(E->B - 1) * per_env >= d->n_rows)
        return fail(MP_E_INVALID, "%s: choice %d of player %d (row base %lld, %lld rows per env) leaves rows [0, %d) for %d envs",
                    fn, j, p, (long long)base, (long long)per_env, d->n_rows, E->B);
    }
  }
  return MP_OK;
}

// The restore of mp_state_restore or a restoring mp_run: slot_of_env and bank, or neither; MP_RESTORE_REKEY or no flags.
int check_restore(const int32_t* slot_of_env, const void* bank, int n_slots, uint32_t flags, const char* fn) {
  const bool restoring = slot_of_env || bank;
  if (restoring && (!slot_of_env || !bank)) return fail(MP_E_INVALID, "%s: slot_of_env and bank go together", fn);
  if (restoring && n_slots < 1) return fail(MP_E_INVALID, "%s: n_slots %d < 1", fn, n_slots);
  if (flags & ~MP_RESTORE_REKEY) return fail(MP_E_INVALID, "%s: unknown flags 0x%x", fn, flags & ~MP_RESTORE_REKEY);
  if (flags && !restoring) return fail(MP_E_INVALID, "%s: flags without a bank", fn);
  return MP_OK;
}

// Every check of `r`, in the order include/mp_engine.h lists them: the request's shape, the restore, drawn routes, row
// actions, player rows, the bank and the targets, then every extent together. A plain request does no check work.
int check_call(mp_engine* E, const mp_request& r) {
  const char* fn = "mp_run";
  if (r.reset && (r.actions || r.player_actions || r.slot_of_env || r.bank || r.restore_flags))
    return fail(MP_E_INVALID, "%s: a reset takes no actions, player_actions, slot_of_env, bank or restore_flags", fn);
  if (!r.reset && r.env_mask) return fail(MP_E_INVALID, "%s: env_mask is for a reset, not a step", fn);
  if (!r.reset && r.actions && r.player_actions) return fail(MP_E_INVALID, "%s: a step takes actions or player_actions, not both", fn);
  if (!r.reset && !r.actions && !r.player_actions) return fail(MP_E_INVALID, "%s: a step needs actions or player_actions, and has neither", fn);
  if (r.draw && !r.players) return fail(MP_E_INVALID, "%s: draw needs players", fn);
  int rc = check_restore(r.slot_of_env, r.bank, r.n_slots, r.restore_flags, fn);
  std::vector<DeviceExtent> ext;
  if (!rc && r.draw) rc = check_route_draw(E, r, fn);
  if (!rc && r.player_actions) rc = check_player_actions(E, r.player_actions, r.players, fn, ext);
  if (!rc && r.players) rc = check_player_outputs(E, r.players, r.out, fn, ext);
  if (!rc && r.bank) rc = check_bank(r.bank, r.n_slots, r.slot_of_env, (uint64_t)E->B, E->record.record_bytes, fn, ext);
  if (!rc && r.out) rc = check_device_outputs(E, r.out, fn, ext);
  if (rc) return rc;
  return ext.empty() ? MP_OK : check_extents(E, ext, fn);
}
}  // namespace

int mp_state_store(mp_handle h, const int32_t* env_of_slot, int n_slots, void* bank, void* stream) {
  if (!h || !env_of_slot || !bank) return fail(MP_E_INVALID, "mp_state_store: null argument");
  if (n_slots < 1) return fail(MP_E_INVALID, "mp_state_store: n_slots %d < 1", n_slots);
  DeviceGuard guard(h->device);
  std::vector<DeviceExtent> ext;
  int rc = check_bank(bank, n_slots, env_of_slot, (uint64_t)n_slots, h->record.record_bytes, "mp_state_store", ext);
  if (!rc) rc = check_extents(h, ext, "mp_state_store");
  if (rc) return rc;
  k_state_store<<<(n_slots + 7) / 8, 256, 0, (cudaStream_t)stream>>>(h->record, env_of_slot, n_slots, h->B, static_cast<uint8_t*>(bank));
  ++h->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

int mp_state_restore(mp_handle h, const int32_t* slot_of_env, const void* bank, int n_slots, uint32_t flags, void* stream) {
  if (!h || !slot_of_env || !bank) return fail(MP_E_INVALID, "mp_state_restore: null argument");
  if (int rc = check_restore(slot_of_env, bank, n_slots, flags, "mp_state_restore")) return rc;
  if (h->S.x_world || h->d_g_flag_ptrs)
    return fail(MP_E_UNSUPPORTED, "mp_state_restore: not available once mp_exchange_connect / mp_gather_obs_connect has run");
  DeviceGuard guard(h->device);
  std::vector<DeviceExtent> ext;
  int rc = check_bank(bank, n_slots, slot_of_env, (uint64_t)h->B, h->record.record_bytes, "mp_state_restore", ext);
  if (!rc) rc = check_extents(h, ext, "mp_state_restore");
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  k_state_restore<<<(h->B + 7) / 8, 256, 0, st>>>(h->record, slot_of_env, static_cast<const uint8_t*>(bank), n_slots, h->B,
                                                  (flags & MP_RESTORE_REKEY) ? 1 : 0, h->key_base);
  ++h->launches;
  CUDA_TRY(cudaGetLastError());
  clear_last_launch(h);
  return launch_render(h, st);
}

// Checks `r` and, when every check passes, launches it: the state transition, then the render. A refused request
// enqueues nothing. A step with neither targets nor player rows publishes its step to the exchange from a
// k_exchange_push of its own, as mp_step_state does.
int mp_run(mp_handle h, const mp_request* r, void* stream) {
  if (!h || !r) return fail(MP_E_INVALID, "mp_run: null handle or request");
  DeviceGuard guard(h->device);
  int rc = check_call(h, *r);
  if (rc) return rc;
  const StepRestore restore{h->d_record_layout, r->slot_of_env, static_cast<const uint8_t*>(r->bank), r->n_slots,
                            (r->restore_flags & MP_RESTORE_REKEY) ? 1 : 0, h->key_base};
  const mp_player_actions* a = r->player_actions;
  RowActions rows{};
  if (a) rows = {a->row_of_player, reinterpret_cast<const uint8_t*>(a->action), a->action_row_stride, a->n_rows};
  DrawnActions drawn{};
  if (r->draw) {
    const mp_route_draw& d = *r->draw;
    drawn.row_of_player = d.row_of_player; drawn.action = rows.action; drawn.stride = rows.stride;
    drawn.n_rows = d.n_rows;
    memcpy(drawn.n_choices, d.n_choices, sizeof drawn.n_choices);
    memcpy(drawn.base, d.row_base, sizeof drawn.base);
    memcpy(drawn.per_env, d.rows_per_env, sizeof drawn.per_env);
  }
  const cudaStream_t st = (cudaStream_t)stream;
  const bool render_follows = r->reset || r->out || r->players;
  if ((rc = launch_state(h, r->actions, r->env_mask, r->reset ? 1 : 0, st, render_follows, r->bank ? &restore : nullptr,
                         a ? &rows : nullptr, r->draw ? &drawn : nullptr)))
    return rc;
  return launch_render(h, st, r->out, r->players);
}

int mp_launch_count(mp_handle h, uint64_t* out) {
  if (!h || !out) return fail(MP_E_INVALID, "null argument");
  *out = h->launches;
  return MP_OK;
}

int mp_debug_render_plan(mp_handle h, int32_t out[MP_RENDER_PLAN_FIELDS]) {
  if (!h || !out) return fail(MP_E_INVALID, "mp_debug_render_plan: null argument");
  const RenderPlan& R = h->R;
  const int32_t v[MP_RENDER_PLAN_FIELDS] = {R.n_teams, R.team_threads, R.wstrip_log2, R.smem_bytes, R.n_total, R.rec_stride, R.stage_bytes,
                                            R.grid_bytes, h->lane_map_players, h->lane_map_world, h->inst_ncp, h->inst_ncw};
  memcpy(out, v, sizeof v);
  return MP_OK;
}

int mp_debug_last_launch(mp_handle h, int32_t out[MP_LAST_LAUNCH_FIELDS]) {
  if (!h || !out) return fail(MP_E_INVALID, "mp_debug_last_launch: null argument");
  memcpy(out, h->last_launch, sizeof h->last_launch);
  return MP_OK;
}

int mp_debug_render_tables(mp_handle h, int32_t* n_total, uint8_t* pair, uint8_t* flags) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  if (n_total) *n_total = h->n_total;
  if (pair) memcpy(pair, h->host_pair.data(), h->host_pair.size());
  if (flags) memcpy(flags, h->host_sflags.data(), h->host_sflags.size());
  return MP_OK;
}

int mp_debug_observations(mp_handle h, int32_t* position, int32_t* orientation, int32_t* layer, int32_t* zap_matrix, void* stream) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  DeviceGuard guard(h->device);
  k_debug_obs<<<h->B, 128, 0, (cudaStream_t)stream>>>(h->T, h->S, position, orientation, layer, zap_matrix, h->R.view_w, h->R.view_h);
  ++h->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

int mp_debug_lane_map(int n_rows, int n_cells, int pitch_slots, int iters, int scattered, uint32_t out[32]) {
  if (!out || (n_rows != 8 && n_rows != 4 && n_rows != 2) || n_cells < 1 || n_cells > 62 || iters < 1 || iters > 5) return fail(MP_E_INVALID, "mp_debug_lane_map: bad arguments");
  if (!scattered) { if (n_cells > (32 / n_rows) * iters) return fail(MP_E_INVALID, "mp_debug_lane_map: too few turns"); make_lane_map_cells(n_rows, n_cells, pitch_slots, iters, out); return MP_OK; }
  if (!make_lane_map(n_rows, n_cells, pitch_slots, iters, out)) return fail(MP_E_UNSUPPORTED, "no conflict-free dealing for %d rows x %d cells in %d turns", n_rows, n_cells, iters);
  return MP_OK;
}

int mp_algorithmic_bytes(mp_handle h, uint64_t* per_env_step, uint64_t* render_per_env_step) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  if (per_env_step) *per_env_step = h->algo_bytes;
  if (render_per_env_step) *render_per_env_step = h->render_bytes;
  return MP_OK;
}

}  // extern "C"
