// engine.cu -- host side of libmpengine.so: blob -> device tables, state allocation, launches, C ABI.
// See include/mp_engine.h for the boundary contract. No CPU implementation of the path exists in
// this library: without a CUDA device every entry point fails with MP_E_NO_DEVICE / MP_E_CUDA.
#include <cuda_runtime.h>

#include <algorithm>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <string>
#include <vector>

#include "../../include/mp_engine.h"
#include "../../include/mpb_format.h"
#include "common.cuh"
#include "render.cuh"
#include "step_clean_up.cuh"
#include "step_commons.cuh"
#include "step_territory.cuh"
#include "step_coins.cuh"
#include "step_mining.cuh"

namespace {

thread_local std::string g_error;

int fail(int code, const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  g_error = buf;
  return code;
}

#define CUDA_TRY(expr)                                                                          \
  do {                                                                                          \
    cudaError_t e_ = (expr);                                                                    \
    if (e_ != cudaSuccess) return fail(MP_E_CUDA, "%s failed: %s", #expr, cudaGetErrorString(e_)); \
  } while (0)

template <typename T>
struct Section {
  const T* data = nullptr;
  std::vector<uint32_t> shape;
  size_t count = 0;
};

template <typename T>
bool get_section(const void* blob, size_t n, const char* name, int dtype, Section<T>* out) {
  const MpbSection* s = mpb_find(blob, n, name);
  if (!s || (int)s->dtype != dtype) return false;
  out->data = static_cast<const T*>(mpb_data(blob, s));
  out->shape.assign(s->shape, s->shape + s->ndim);
  out->count = s->nbytes / sizeof(T);
  return true;
}

int round_up(int v, int m) { return (v + m - 1) / m * m; }

constexpr int kRenderSmemLimit = 227 * 1024 - 2560;  // dynamic shared memory: the 227 KB opt-in maximum less k_render's static arrays
constexpr int kMaxAtlasSprites = 96;
#define MP_MAX_DEVICES 64
#define MP_EXCHANGE_HEADER 256  // bytes reserved for the per-rank flags in front of the gathered rows  // sprites incl. pre-merged ones kept in shared memory by k_render

// Beam footprint in visiting order (policy A.8): centre ray, then for each side the lateral cells
// outwards, each followed by its forward ray of length `length - k`.
bool make_beam_geom(int length, int radius, BeamGeom* g) {
  std::vector<int> lat, fwd, parent;
  int prev = -1;
  for (int i = 1; i <= length; ++i) { lat.push_back(0); fwd.push_back(i); parent.push_back(prev); prev = (int)lat.size() - 1; }
  for (int side = 0; side < 2; ++side) {
    int sign = side == 0 ? -1 : 1;
    int prev_lat = -1;
    for (int k = 1; k <= radius; ++k) {
      lat.push_back(sign * k); fwd.push_back(0); parent.push_back(prev_lat);
      prev_lat = (int)lat.size() - 1;
      int pf = prev_lat;
      for (int i = 1; i <= length - k; ++i) { lat.push_back(sign * k); fwd.push_back(i); parent.push_back(pf); pf = (int)lat.size() - 1; }
    }
  }
  if (lat.size() > MP_MAX_BEAM_CELLS) return false;
  g->n = (int)lat.size();
  g->depth = length + radius;
  for (int i = 0; i < g->n; ++i) { g->lat[i] = (int8_t)lat[i]; g->fwd[i] = (int8_t)fwd[i]; g->parent[i] = (int8_t)parent[i]; }
  return true;
}

// A beam of `length` cells forward and `radius` to each side covers forward offsets 0..length and lateral offsets
// -radius..radius around the shooter. On a TORUS map that is smaller than the map in both directions, each footprint
// cell wraps with one conditional add (wrap_or_reject) and no two cells of a footprint land on the same map cell.
bool beam_fits_torus(const Tables& T, int length, int radius) {
  const int m = std::min(T.W, T.H);
  return T.topology != 1 || (length < m && 2 * radius + 1 <= m);
}

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

}  // namespace

struct mp_engine {
  int device = 0;
  int B = 0;
  uint32_t flags = MP_FLAG_DEFAULT;
  int family = 0;
  int n_total = 0;  // atlas sprites incl. pre-merged
  Tables T{};
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
  size_t step_smem = 0;
  void (*render_fn)(Tables, State, RenderPlan, uint32_t) = nullptr;
  void (*render_gather_fn)(Tables, State, RenderPlan, uint32_t) = nullptr;
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
  std::vector<std::pair<void*, size_t>> state_spans;  // what mp_state_save / mp_state_load copy
  uint64_t state_bytes = 0;
  int lane_map_players = 0, lane_map_world = 0;  // 0 plain, 2 scattered colouring, 1 + 16 * (extra wavefronts left) whole-cell dealing
  int inst_ncp = 0, inst_ncw = 0;                // the k_render<NCP, NCW> instantiation this engine launches
  uint64_t blob_hash = 0;  // FNV-1a of the compiled blob: a snapshot only loads into an engine built from the same blob

  template <typename T>
  int upload(const std::vector<T>& host, const T** out) {
    void* p = nullptr;
    size_t bytes = std::max<size_t>(host.size() * sizeof(T), 16);
    CUDA_TRY(cudaMalloc(&p, bytes));
    allocs.push_back(p);
    CUDA_TRY(cudaMemset(p, 0, bytes));
    if (!host.empty()) CUDA_TRY(cudaMemcpy(p, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice));
    *out = static_cast<const T*>(p);
    return MP_OK;
  }
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

int build_tables(mp_engine* E, const void* blob, size_t n) {
  Section<int32_t> meta, states, kinds, comps, objects, hits, action_table, sprite_map, scalar_obs, av_table;
  Section<double> comps_f;
  Section<uint8_t> atlas, sprite_opaque, cell_flags;
  Section<uint16_t> init_grid;
  if (!get_section(blob, n, "meta", MPB_I32, &meta) || meta.count < MPB_META_COUNT) return fail(MP_E_INVALID, "blob: missing/invalid 'meta' (not an MPB%u blob?)", MPB_VERSION);
#define NEED(sec, dt) if (!get_section(blob, n, #sec, dt, &sec)) return fail(MP_E_INVALID, "blob: missing section '%s'", #sec);
  NEED(states, MPB_I32) NEED(kinds, MPB_I32) NEED(comps, MPB_I32) NEED(comps_f, MPB_F64) NEED(objects, MPB_I32) NEED(hits, MPB_I32)
  NEED(action_table, MPB_I32) NEED(sprite_map, MPB_I32) NEED(scalar_obs, MPB_I32) NEED(av_table, MPB_I32)
  NEED(atlas, MPB_U8) NEED(sprite_opaque, MPB_U8) NEED(cell_flags, MPB_U8) NEED(init_grid, MPB_U16)
  const int32_t* m = meta.data;
  Tables& T = E->T;
  E->family = m[MPB_META_FAMILY];
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
  if (E->family != MPB_FAMILY_CLEAN_UP && E->family != MPB_FAMILY_COMMONS_HARVEST && E->family != MPB_FAMILY_TERRITORY && E->family != MPB_FAMILY_COINS && E->family != MPB_FAMILY_COOP_MINING) return fail(MP_E_UNSUPPORTED, "substrate family %d has no CUDA state-transition kernel yet", E->family);

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
  char name[64];
  auto load_group = [&](int gid, std::vector<int32_t>* out) -> int {
    snprintf(name, sizeof name, "spawn_cells_%d", gid);
    Section<int32_t> sec;
    if (!get_section(blob, n, name, MPB_I32, &sec)) return fail(MP_E_INVALID, "blob: missing section '%s'", name);
    out->assign(sec.data, sec.data + sec.count);
    return MP_OK;
  };
  std::vector<int32_t> v_spawn, v_init[2];
  int rc0;
  if ((rc0 = load_group(respawn_group, &v_spawn))) return rc0;
  T.n_spawn = (int)v_spawn.size();
  for (int k = 0; k < 2; ++k) {
    T.n_spawn_init[k] = 0;
    if (init_groups[k] < 0) continue;
    if ((rc0 = load_group(init_groups[k], &v_init[k]))) return rc0;
    T.n_spawn_init[k] = (int)v_init[k].size();
    int users = 0;
    for (int p = 0; p < T.P; ++p) users += T.avatar_init_group[p] == k;
    if (T.n_spawn_init[k] < users || T.n_spawn_init[k] > 64) return fail(MP_E_UNSUPPORTED, "%d spawn points for %d avatars (need n..64)", T.n_spawn_init[k], users);
  }
  if (T.n_spawn < 1) return fail(MP_E_INVALID, "empty respawn group");

  // ---- family tables -----------------------------------------------------------------------------
  int rc;
  std::vector<int32_t> v_apple, v_dirt, v_water;
  std::vector<std::vector<int>> hint_stacks;  // sprite stacks (bottom up) worth a pre-merged sprite before the generic enumeration
  T.nA = T.nD = T.nW = 0; T.nR = 0; T.nR_pad = 16;
  T.n_anim = 1; T.anim_frames = 1; T.clean_layer = 0;
  auto zapper = [&](const int32_t* ip) -> int {  // shared Zapper block of cu_ip / ch_ip
    T.zap_cooldown = ip[12]; T.zap_respawn = ip[15]; T.zap_remove = ip[16];
    T.zap_layer = ip[21]; T.zap_sprite = ip[22];
    T.zap_hit = 0;
    for (int h = 0; h < (int)hits.count / 2; ++h) if (hits.data[h * 2] == T.zap_layer) T.zap_hit = h;
    if (T.zap_cooldown <= 0) return fail(MP_E_UNSUPPORTED, "non-positive zap cooldown");
    if (!make_beam_geom(ip[13], ip[14], &T.zap_geom)) return fail(MP_E_UNSUPPORTED, "beam footprint larger than %d cells", MP_MAX_BEAM_CELLS);
    if (!beam_fits_torus(T, ip[13], ip[14])) return fail(MP_E_UNSUPPORTED, "zap beam (length %d, radius %d) does not fit the %dx%d TORUS map", ip[13], ip[14], T.W, T.H);
    T.end_min_frames = ip[26]; T.end_interval = ip[27];
    if (T.end_interval < 1) return fail(MP_E_INVALID, "episode interval < 1");
    return MP_OK;
  };
  if (E->family == MPB_FAMILY_CLEAN_UP) {
    Section<int32_t> cu_ip, cu_apple, cu_dirt, cu_water, cu_water_sprites;
    Section<double> cu_dp;
    NEED(cu_ip, MPB_I32) NEED(cu_dp, MPB_F64) NEED(cu_apple, MPB_I32) NEED(cu_dirt, MPB_I32) NEED(cu_water, MPB_I32) NEED(cu_water_sprites, MPB_I32)
    const int32_t* ip = cu_ip.data; const double* dp = cu_dp.data;
    T.nA = ip[0]; T.nD = ip[1]; T.nW = ip[2];
    T.apple_layer = ip[3]; T.apple_sprite = ip[4]; T.dirt_layer = ip[5]; T.dirt_sprite = ip[6];
    T.water_layer = ip[8]; T.n_anim = ip[9]; T.anim_frames = ip[10]; T.anim_random = ip[11];
    if (T.n_anim < 1 || T.n_anim > 8 || T.anim_frames < 1) return fail(MP_E_UNSUPPORTED, "animation with %d states / %d frames", T.n_anim, T.anim_frames);
    for (int i = 0; i < T.n_anim; ++i) T.water_sprite[i] = cu_water_sprites.data[i];
    if ((rc = zapper(ip))) return rc;
    T.clean_cooldown = ip[18]; T.clean_layer = ip[23]; T.clean_sprite = ip[24];
    T.clean_hit = 1;
    for (int h = 0; h < (int)hits.count / 2; ++h) if (hits.data[h * 2] == T.clean_layer) T.clean_hit = h;
    if (T.clean_cooldown < 0) return fail(MP_E_UNSUPPORTED, "negative clean cooldown");
    if (!make_beam_geom(ip[19], ip[20], &T.clean_geom)) return fail(MP_E_UNSUPPORTED, "beam footprint larger than %d cells", MP_MAX_BEAM_CELLS);
    if (!beam_fits_torus(T, ip[19], ip[20])) return fail(MP_E_UNSUPPORTED, "clean beam (length %d, radius %d) does not fit the %dx%d TORUS map", ip[19], ip[20], T.W, T.H);
    T.dirt_delay = ip[25]; T.taste_role = ip[28];
    if (T.taste_role != 0) return fail(MP_E_UNSUPPORTED, "Taste roles other than 'free'");
    T.grow_rate = dp[0]; T.grow_depletion = dp[1]; T.grow_restoration = dp[2]; T.eat_reward = dp[3];
    T.zap_penalty = dp[4]; T.zap_reward = dp[5]; T.dirt_prob = dp[6]; T.end_prob = dp[7]; T.taste_amount = dp[8];
    v_apple.assign(cu_apple.data, cu_apple.data + cu_apple.count);
    v_dirt.assign(cu_dirt.data, cu_dirt.data + cu_dirt.count);
    v_water.assign(cu_water.data, cu_water.data + cu_water.count);
    if ((rc = E->upload(v_apple, &T.apple)) || (rc = E->upload(v_dirt, &T.dirt)) || (rc = E->upload(v_water, &T.water))) return rc;
  } else if (E->family == MPB_FAMILY_COMMONS_HARVEST) {
    Section<int32_t> ch_ip, ch_apple, ch_nbr;
    Section<double> ch_dp;
    NEED(ch_ip, MPB_I32) NEED(ch_dp, MPB_F64) NEED(ch_apple, MPB_I32) NEED(ch_nbr, MPB_I32)
    const int32_t* ip = ch_ip.data; const double* dp = ch_dp.data;
    T.nA = ip[0]; T.apple_layer = ip[1]; T.apple_sprite = ip[2]; T.wait_layer = ip[3]; T.wait_sprite = ip[4];
    T.ch_n_wait = ip[5]; T.ch_n_probs = ip[6]; T.grass_layer = ip[7]; T.grass_sprite = ip[8]; T.dess_sprite = ip[9];
    if (T.ch_n_wait < 1 || T.ch_n_wait > 29 || T.ch_n_probs < 1 || T.ch_n_probs > 4) return fail(MP_E_UNSUPPORTED, "DensityRegrow with %d wait states / %d probabilities", T.ch_n_wait, T.ch_n_probs);
    if (T.nA > 2048) return fail(MP_E_UNSUPPORTED, "%d apples (max 2048)", T.nA);
    if ((rc = zapper(ip))) return rc;
    for (int i = 0; i < 4; ++i) T.ch_probs[i] = dp[i];
    T.eat_reward = dp[4]; T.zap_penalty = dp[5]; T.zap_reward = dp[6]; T.end_prob = dp[7];
    v_apple.assign(ch_apple.data, ch_apple.data + ch_apple.count);
    std::vector<int32_t> v_nbr(ch_nbr.data, ch_nbr.data + ch_nbr.count);
    if ((rc = E->upload(v_apple, &T.ch_apple)) || (rc = E->upload(v_nbr, &T.ch_nbr))) return rc;
  }
  else if (E->family == MPB_FAMILY_COINS) {
    Section<int32_t> co_ip, co_coin;
    Section<double> co_dp;
    NEED(co_ip, MPB_I32) NEED(co_dp, MPB_F64) NEED(co_coin, MPB_I32)
    const int32_t* ip = co_ip.data; const double* dp = co_dp.data;
    if (T.P != 2) return fail(MP_E_UNSUPPORTED, "coins needs exactly two players (got %d)", T.P);
    T.nA = ip[0]; T.apple_layer = ip[1]; T.coin_sprite[0] = ip[2]; T.coin_sprite[1] = ip[3];
    T.coin_terminate = ip[4]; T.coin_terminate_n = ip[5]; T.end_min_frames = ip[6]; T.end_interval = ip[7];
    T.coin_type[0] = ip[8]; T.coin_type[1] = ip[9];
    if (T.nA > 2048) return fail(MP_E_UNSUPPORTED, "%d coins (max 2048)", T.nA);
    if (T.end_interval < 1) return fail(MP_E_INVALID, "episode interval < 1");
    T.coin_rate = dp[0]; T.end_prob = dp[1];
    for (int p = 0; p < 2; ++p) for (int k = 0; k < 4; ++k) T.coin_reward[p][k] = dp[4 + p * 4 + k];
    T.zap_layer = 0; T.zap_cooldown = 1;
    v_apple.resize((size_t)T.nA * 4);
    for (int k = 0; k < T.nA; ++k) { v_apple[k * 4] = co_coin.data[k * 2]; v_apple[k * 4 + 1] = co_coin.data[k * 2 + 1]; v_apple[k * 4 + 2] = 0; v_apple[k * 4 + 3] = -1; }
    if ((rc = E->upload(v_apple, &T.ch_apple))) return rc;
  }
  else if (E->family == MPB_FAMILY_COOP_MINING) {
    Section<int32_t> cm_ip, cm_ore;
    Section<double> cm_dp;
    NEED(cm_ip, MPB_I32) NEED(cm_dp, MPB_F64) NEED(cm_ore, MPB_I32)
    const int32_t* ip = cm_ip.data; const double* dp = cm_dp.data;
    T.nA = ip[0]; T.apple_layer = ip[1];
    for (int i = 0; i < 4; ++i) T.ore_sprite[i] = ip[2 + i];
    T.mine_window = ip[6]; T.zap_cooldown = ip[7]; T.mine_length = ip[8]; T.zap_layer = ip[9]; T.zap_sprite = ip[10];
    T.end_min_frames = ip[11]; T.end_interval = ip[12]; T.zap_hit = ip[13];
    if (T.P > 8) return fail(MP_E_UNSUPPORTED, "coop_mining with %d players (max 8: miners are kept as a bit mask)", T.P);
    if (T.nA > 2048) return fail(MP_E_UNSUPPORTED, "%d ores (max 2048)", T.nA);
    if (T.zap_cooldown < 1 || T.mine_window < 1 || T.mine_window > 255 || T.mine_length < 1) return fail(MP_E_UNSUPPORTED, "MineBeam / Ore parameters out of range");
    if (T.end_interval < 1) return fail(MP_E_INVALID, "episode interval < 1");
    if (T.zap_hit < 0 || T.zap_hit > 7) return fail(MP_E_UNSUPPORTED, "mine hit id %d", T.zap_hit);
    if (!beam_fits_torus(T, T.mine_length, 0)) return fail(MP_E_UNSUPPORTED, "mine beam (length %d) does not fit the %dx%d TORUS map", T.mine_length, T.W, T.H);
    T.mine_rate[0] = dp[0]; T.mine_rate[1] = dp[1]; T.end_prob = dp[2];
    T.mine_reward[0] = dp[4]; T.mine_reward[1] = dp[5]; T.extract_reward[0] = dp[6]; T.extract_reward[1] = dp[7];
    v_apple.resize((size_t)T.nA * 4);
    for (int k = 0; k < T.nA; ++k) { v_apple[k * 4] = cm_ore.data[k * 2]; v_apple[k * 4 + 1] = cm_ore.data[k * 2 + 1]; v_apple[k * 4 + 2] = 0; v_apple[k * 4 + 3] = -1; }
    if ((rc = E->upload(v_apple, &T.ch_apple))) return rc;
  }
  else {  // MPB_FAMILY_TERRITORY
    Section<int32_t> tr_ip, tr_res, tr_player_sprites;
    Section<double> tr_dp;
    Section<uint8_t> tr_wall;
    NEED(tr_ip, MPB_I32) NEED(tr_dp, MPB_F64) NEED(tr_res, MPB_I32) NEED(tr_player_sprites, MPB_I32) NEED(tr_wall, MPB_U8)
    const int32_t* ip = tr_ip.data; const double* dp = tr_dp.data;
    T.nR = ip[0]; T.nR_pad = round_up(std::max(T.nR, 64), 16);
    T.res_layer = ip[1]; T.unclaimed_sprite = ip[2]; T.tex_layer = ip[3]; T.tex_sprite = ip[4]; T.ind_layer = ip[5];
    T.dmg_layer = ip[6]; T.dmg_sprite = ip[7]; T.mark_layer = ip[8]; T.mark_initial_level = ip[9]; T.mark_recovery = ip[10]; T.mark_n_levels = ip[11];
    if (T.res_layer != T.avatar_layer) return fail(MP_E_UNSUPPORTED, "territory: resources and avatars must share a layer");
    if (T.mark_n_levels < 1 || T.mark_n_levels > 3) return fail(MP_E_UNSUPPORTED, "%d marking levels (1..3)", T.mark_n_levels);
    if ((rc = zapper(ip))) return rc;
    if (T.zap_respawn <= T.max_frames) return fail(MP_E_UNSUPPORTED, "territory kernel assumes avatars never respawn (framesTillRespawn %d)", T.zap_respawn);
    if (!make_beam_geom(ip[18], ip[19], &T.claim_geom) || !make_beam_geom(1, 0, &T.brush_geom)) return fail(MP_E_UNSUPPORTED, "beam footprint larger than %d cells", MP_MAX_BEAM_CELLS);
    if (!beam_fits_torus(T, ip[18], ip[19])) return fail(MP_E_UNSUPPORTED, "claim beam (length %d, radius %d) does not fit the %dx%d TORUS map", ip[18], ip[19], T.W, T.H);
    T.claim_wait = ip[20]; T.brush_layer = ip[23]; T.claim_layer = ip[24];
    if (T.claim_layer != T.dmg_layer) return fail(MP_E_UNSUPPORTED, "territory: claim beam layer must be the damage indicator layer");
    T.res_health0 = ip[28]; T.res_reward_delay = ip[29]; T.res_repair_delay = ip[30]; T.tr_taste_role = ip[31];
    if (T.tr_taste_role != 0) return fail(MP_E_UNSUPPORTED, "territory Taste roles other than 'none'");
    if (T.res_health0 < 1 || T.res_health0 > 200) return fail(MP_E_UNSUPPORTED, "resource health %d", T.res_health0);
    // the resource age and frames-since-zapped counters saturate at 65535 (step_territory.cuh)
    if (T.res_reward_delay > 65535 || T.res_repair_delay > 65535)
      return fail(MP_E_UNSUPPORTED, "rewardDelay %d / delayTillSelfRepair %d (max 65535)", T.res_reward_delay, T.res_repair_delay);
    for (int l = 0; l < T.mark_n_levels; ++l) {
      T.mark_inc[l] = ip[32 + 4 * l]; T.mark_remove[l] = ip[33 + 4 * l]; T.mark_freeze[l] = ip[34 + 4 * l]; T.mark_sprite[l] = ip[35 + 4 * l];
      T.mark_src_reward[l] = dp[8 + 2 * l]; T.mark_tgt_reward[l] = dp[9 + 2 * l];
    }
    T.res_reward = dp[0]; T.res_rate = dp[1]; T.res_repair_prob = dp[2]; T.zap_penalty = dp[3]; T.zap_reward = dp[4]; T.end_prob = dp[5];
    T.tr_taste_amount = dp[6]; T.tr_taste_mult = dp[7];
    for (int p = 0; p < T.P; ++p) {
      const int32_t* ps = tr_player_sprites.data + p * 4;
      T.claimed_sprite[p] = ps[0]; T.dry_sprite[p] = ps[1]; T.brush_sprite[p] = ps[2]; T.claimbeam_sprite[p] = ps[3];
    }
    for (int p = 0; p < T.P; ++p) {  // wet paint on the resource texture, then dry paint on top: what most resource cells show
      hint_stacks.push_back({T.tex_sprite, T.claimed_sprite[p]});
      hint_stacks.push_back({T.tex_sprite, T.claimed_sprite[p], T.dry_sprite[p]});
    }
    std::vector<int32_t> v_res(tr_res.data, tr_res.data + tr_res.count);
    std::vector<int16_t> res_of(T.cells_pad, -1);
    for (int k = 0; k < T.nR; ++k) res_of[v_res[k * 3 + 1]] = (int16_t)k;
    std::vector<uint8_t> wall(T.cells_pad, 0);
    memcpy(wall.data(), tr_wall.data, std::min<size_t>(tr_wall.count, T.cells));
    if ((rc = E->upload(v_res, &T.tr_res)) || (rc = E->upload(res_of, &T.res_of_cell)) || (rc = E->upload(wall, &T.wall))) return rc;
    Section<int32_t> tr_res_cond;
    if (get_section(blob, n, "tr_res_cond", MPB_I32, &tr_res_cond)) {
      if ((int)tr_res_cond.count != T.nR * 2) return fail(MP_E_INVALID, "blob: tr_res_cond has %zu values for %d resources", tr_res_cond.count, T.nR);
      std::vector<int32_t> v(tr_res_cond.data, tr_res_cond.data + tr_res_cond.count);
      if ((rc = E->upload(v, &T.tr_res_cond))) return rc;
    }
  }
#undef NEED
  {  // 'choice' prefabs left to the engine (drawn per env and episode)
    Section<int32_t> choice_groups, obj_choice, spawn_cond;
    if (get_section(blob, n, "choice_groups", MPB_I32, &choice_groups)) {
      if (E->family != MPB_FAMILY_TERRITORY) return fail(MP_E_UNSUPPORTED, "per-env 'choice' prefabs are implemented for the territory family only (compile with a build_seed)");
      T.n_choice = (int)choice_groups.count;
      for (size_t g = 0; g < choice_groups.count; ++g) if (choice_groups.data[g] < 1 || choice_groups.data[g] > 31) return fail(MP_E_INVALID, "blob: choice group with %d options", choice_groups.data[g]);
      std::vector<int32_t> v(choice_groups.data, choice_groups.data + choice_groups.count);
      if ((rc = E->upload(v, &T.choice_n))) return rc;
      snprintf(name, sizeof name, "spawn_cond_%d", respawn_group);
      if (get_section(blob, n, name, MPB_I32, &spawn_cond)) {
        if ((int)spawn_cond.count != T.n_spawn * 2 || T.n_spawn > 64) return fail(MP_E_UNSUPPORTED, "%d conditional spawn candidates (max 64)", T.n_spawn);
        std::vector<int32_t> c(spawn_cond.data, spawn_cond.data + spawn_cond.count);
        if ((rc = E->upload(c, &T.spawn_cond))) return rc;
      }
    }
  }
  T.nA_pad = round_up(std::max(T.nA, 1), 16); T.nD_pad = round_up(std::max(std::max(T.nD, T.nA), 1), 16); T.nW_pad = round_up(std::max(T.nW, 1), 16);

  // ---- device copies -----------------------------------------------------------------------------
  std::vector<uint16_t> grid0((size_t)T.L * T.cells_pad, 0);
  for (int l = 0; l < T.L; ++l) memcpy(&grid0[(size_t)l * T.cells_pad], init_grid.data + (size_t)l * T.cells, T.cells * sizeof(uint16_t));
  if ((rc = E->upload(grid0, &T.init_grid))) return rc;
  std::vector<int32_t> act(action_table.data, action_table.data + action_table.count);
  if ((rc = E->upload(act, &T.action_table))) return rc;
  if ((rc = E->upload(v_spawn, &T.spawn_cell))) return rc;
  for (int k = 0; k < 2; ++k) {
    if (v_init[k].empty()) { T.spawn_init_cell[k] = T.spawn_cell; continue; }
    if ((rc = E->upload(v_init[k], &T.spawn_init_cell[k]))) return rc;
  }
  std::vector<uint8_t> solid(T.cells_pad, 0), flags(T.cells_pad, 0);
  for (int o = 0; o < m[MPB_META_N_OBJECTS]; ++o) {  // non-avatar pieces that start on the avatar layer
    const int32_t* od = objects.data + o * MPB_OBJ_COLS;
    const int32_t* kd = kinds.data + od[MPB_OBJ_KIND] * MPB_KIND_COLS;
    if (kd[MPB_KIND_IS_AVATAR]) continue;
    const int32_t* st = states.data + (kd[MPB_KIND_STATE0] + od[MPB_OBJ_STATE]) * MPB_STATE_COLS;
    if (st[MPB_STATE_LAYER] == T.avatar_layer) solid[od[MPB_OBJ_Y] * T.W + od[MPB_OBJ_X]] = 255;
  }
  memcpy(flags.data(), cell_flags.data, std::min<size_t>(cell_flags.count, T.cells));
  if ((rc = E->upload(solid, &T.solid)) || (rc = E->upload(flags, &T.cell_flags))) return rc;
  std::vector<int16_t> apple_of(T.cells_pad, -1), dirt_of(T.cells_pad, -1);
  T.dirt_count0 = 0;
  const int apple_cols = E->family == MPB_FAMILY_CLEAN_UP ? 3 : 4;
  for (int k = 0; k < T.nA; ++k) apple_of[v_apple[k * apple_cols + 1]] = (int16_t)k;
  for (int j = 0; j < T.nD; ++j) { dirt_of[v_dirt[j * 3 + 1]] = (int16_t)j; T.dirt_count0 += v_dirt[j * 3 + 2]; }
  if ((rc = E->upload(apple_of, &T.apple_of_cell)) || (rc = E->upload(dirt_of, &T.dirt_of_cell))) return rc;

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
    if (E->flags & MP_FLAG_DEBUG_NO_PREMERGE) return 0;  // budget zero: every stack takes the general compositing path
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
    struct Opt { std::vector<int> sprites; bool absent = false; int orient = -1; bool bad = false; };
    std::vector<Opt> opts((size_t)T.cells * T.L);
    std::vector<uint8_t> has_obj((size_t)T.cells * T.L, 0);
    for (int o = 0; o < m[MPB_META_N_OBJECTS]; ++o) {
      const int32_t* od = objects.data + o * MPB_OBJ_COLS;
      const int32_t* kd = kinds.data + od[MPB_OBJ_KIND] * MPB_KIND_COLS;
      if (kd[MPB_KIND_IS_AVATAR]) continue;
      const int cell = od[MPB_OBJ_Y] * T.W + od[MPB_OBJ_X];
      const int ns = kd[MPB_KIND_NSTATES];
      for (int si = 0; si < ns; ++si) {
        const int32_t* st = states.data + (kd[MPB_KIND_STATE0] + si) * MPB_STATE_COLS;
        const int l = st[MPB_STATE_LAYER], sp = st[MPB_STATE_SPRITE];
        if (l < 0 || sp < 0) continue;
        Opt& op = opts[(size_t)cell * T.L + l];
        if (std::find(op.sprites.begin(), op.sprites.end(), sp) == op.sprites.end()) op.sprites.push_back(sp);
        if (op.orient >= 0 && op.orient != od[MPB_OBJ_ORIENT]) op.bad = true;
        op.orient = od[MPB_OBJ_ORIENT];
        // the piece may also be somewhere else (another layer / off grid / sprite-less state)
        for (int sj = 0; sj < ns; ++sj) {
          const int32_t* s2 = states.data + (kd[MPB_KIND_STATE0] + sj) * MPB_STATE_COLS;
          if (s2[MPB_STATE_LAYER] != l || s2[MPB_STATE_SPRITE] < 0) op.absent = true;
        }
      }
    }
    for (const auto& hs : hint_stacks) {
      if (hs.empty() || !opq[hs[0]]) continue;
      int cur = hs[0];
      for (size_t q = 1; q < hs.size() && cur; ++q) { if (remapped[hs[q]] || remapped[cur]) break; cur = merged_id(cur, hs[q]); }
    }
    std::vector<int> stack_s, stack_o;
    for (int pass = 0; pass < 2; ++pass)  // pass 0: the map as it is at reset (most common stacks) gets the budget first
    for (int cell = 0; cell < T.cells; ++cell) {
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
          const int init_v = init_grid.data[(size_t)l * T.cells + cell];
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
  E->n_total = n_total;
  // atlas re-laid out as [sprite][facing][half][row][16 B] so that the 8 rows of one half are 128
  // contiguous bytes (conflict-free 128-bit shared loads).
  std::vector<uint8_t> at((size_t)n_total * 1024);
  for (int s = 0; s < n_total * 4; ++s)
    for (int row = 0; row < 8; ++row)
      for (int half = 0; half < 2; ++half)
        memcpy(&at[(size_t)s * 256 + half * 128 + row * 16], &img[(size_t)s * 256 + row * 32 + half * 16], 16);
  if ((rc = E->upload(at, &T.atlas))) return rc;
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
  E->host_pair = pair; E->host_sflags = sflags;
  E->black_sprite = -1;  // an opaque, never remapped, all-black sprite stands in for cells with nothing to draw
  for (int i = 0; i < n_total && E->black_sprite < 0; ++i) {
    if (!opq[i] || remapped[i]) continue;
    bool black = true;
    for (int px = 0; px < 256 && black; ++px) { const uint8_t* q = &img[(size_t)i * 1024 + px * 4]; black = q[0] == 0 && q[1] == 0 && q[2] == 0; }
    if (black) E->black_sprite = i;
  }
  if ((rc = E->upload(smap, &T.sprite_map)) || (rc = E->upload(sflags, &T.sprite_opaque)) || (rc = E->upload(pair, &T.sprite_pair))) return rc;
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
        // (constants fitted to measurements on the eight substrates: about three strips' worth of idle time per env and
        //  warp, 2-row WORLD.RGB strips ~15 % slower than 4-row ones, a small cost per extra team)
        const double score = teams * warps * per_warp / (per_warp + 3.0) * (wlog == 2 ? 1.0 : 0.85) * (1.0 - 0.01 * teams);
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

int raise_flags(mp_engine* E, cudaStream_t st) {
  E->x_pending_raise = false;
  k_exchange_push<<<std::min(E->sm_count, (E->B + 7) / 8), 256, 0, st>>>(E->T, E->S);
  ++E->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

// `render_follows`: the caller launches the renderer next on the same stream; it raises the exchange flags.
int launch_state(mp_engine* E, const int32_t* actions, const uint8_t* mask, int mode, cudaStream_t st, bool render_follows = true) {
  const int blocks = (E->B + 3) / 4;
  if (E->S.x_world) E->S.x_step = ++E->x_seq;
  void (*fn)(Tables, State, const int32_t*, const uint8_t*, int) =
      E->family == MPB_FAMILY_CLEAN_UP ? k_step_clean_up : E->family == MPB_FAMILY_COMMONS_HARVEST ? k_step_commons :
      E->family == MPB_FAMILY_COINS ? k_step_coins : E->family == MPB_FAMILY_COOP_MINING ? k_step_mining : k_step_territory;
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(blocks); cfg.blockDim = dim3(128); cfg.dynamicSmemBytes = E->step_smem * 4 + (E->family == MPB_FAMILY_CLEAN_UP ? clean_up_table_bytes(E->T) : E->family == MPB_FAMILY_TERRITORY ? territory_table_bytes(E->T) : 0); cfg.stream = st;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr; cfg.numAttrs = 1;
  CUDA_TRY(cudaLaunchKernelEx(&cfg, fn, E->T, E->S, actions, mask, mode));
  if (E->S.x_world) {
    E->x_pending_raise = true;
    if (!render_follows) { ++E->launches; return raise_flags(E, st); }
  }
  ++E->launches;
  CUDA_TRY(cudaGetLastError());
  return MP_OK;
}

int launch_render(mp_engine* E, cudaStream_t st) {
  if (!(E->flags & (MP_FLAG_RENDER_WORLD | MP_FLAG_RENDER_PLAYERS))) return E->x_pending_raise ? raise_flags(E, st) : MP_OK;
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
  CUDA_TRY(cudaLaunchKernelEx(&cfg, gather ? E->render_gather_fn : E->render_fn, E->T, E->S, R, E->flags));
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

}  // namespace

extern "C" {

const char* mp_last_error(void) { return g_error.c_str(); }
const char* mp_version(void) { return "meltingpot_b200 engine 0.1 (sm_90a)"; }

int mp_create(const void* blob, size_t blob_bytes, int num_envs, int device, uint64_t seed, uint64_t env_index_base, uint32_t flags, mp_handle* out) {
  if (!blob || !out || num_envs < 1) return fail(MP_E_INVALID, "mp_create: bad arguments");
  int n_dev = 0;
  cudaError_t e = cudaGetDeviceCount(&n_dev);
  if (e != cudaSuccess || n_dev == 0) return fail(MP_E_NO_DEVICE, "no CUDA device available (%s); this engine has no CPU path", cudaGetErrorString(e));
  if (device < 0 || device >= n_dev || device >= MP_MAX_DEVICES) return fail(MP_E_INVALID, "device %d out of range (0..%d)", device, n_dev - 1);
  cudaDeviceProp prop;
  CUDA_TRY(cudaGetDeviceProperties(&prop, device));
  if (prop.major != 9 || prop.minor != 0) return fail(MP_E_NO_DEVICE, "device %d is sm_%d%d; kernels are built for sm_90a only", device, prop.major, prop.minor);
  DeviceGuard guard(device);
  mp_engine* E = new mp_engine();
  E->device = device; E->B = num_envs; E->flags = flags; E->sm_count = prop.multiProcessorCount;
  {
    uint64_t hsh = 1469598103934665603ull;
    const uint8_t* bp = static_cast<const uint8_t*>(blob);
    for (size_t i = 0; i < blob_bytes; ++i) { hsh ^= bp[i]; hsh *= 1099511628211ull; }
    E->blob_hash = hsh;
  }
  int rc = build_tables(E, blob, blob_bytes);
  if (rc == MP_OK) rc = build_plan(E);
  if (rc != MP_OK) { mp_destroy(E); return rc; }
  const Tables& T = E->T;
  State& S = E->S;
  S.B = num_envs; S.seed = seed + env_index_base;
  const size_t B = num_envs, P = T.P;
  {  // Worst case of events one step can emit per env: per avatar, every cell of every beam footprint can carry a hit
     // with up to three events (zap + sanctioning + removal), plus the contact / regrowth events (<= 4) and the pair
     // events of coop_mining (<= P). Sized so that emit_event never drops a row.
    const int beam_cells = T.zap_geom.n + T.clean_geom.n + T.claim_geom.n + T.brush_geom.n;
    S.max_events = round_up(std::max(MP_MIN_EVENTS, T.P * (3 * beam_cells + 4 + T.P)), 16);
  }
  S.fam_u8_stride = std::max(16, RU_COUNT * T.nR_pad); S.fam_u16_stride = std::max(16, RS_COUNT * T.nR_pad);
  if ((rc = E->alloc(B * T.L * T.cells_pad, &S.grid)) || (rc = E->alloc(B * P * 4, &S.avatar)) || (rc = E->alloc(B * P * 4, &S.av_timer)) ||
      (rc = E->alloc(B * T.nA_pad, &S.apple)) || (rc = E->alloc(B * T.nD_pad, &S.dirt)) || (rc = E->alloc(B * T.nW_pad, &S.water)) || (rc = E->alloc(B * T.nA_pad, &S.apple_count)) || (rc = E->alloc(B * (size_t)S.fam_u8_stride, &S.fam_u8)) || (rc = E->alloc(B * (size_t)S.fam_u16_stride, &S.fam_u16)) || (rc = E->alloc(B * P * 8, &S.av_extra)) || (rc = E->alloc(B * (P + 2), &S.packed)) ||
      (rc = E->alloc(B * ENV_COLS, &S.env)) ||
      (rc = E->alloc((B * P + B + B + std::max<size_t>(1, T.n_scalar) * B * P) * 8, &E->scalar_block)) ||
      (rc = E->alloc(B * P * E->R.player_bytes, &S.rgb)) || (rc = E->alloc(B * (size_t)E->R.world_bytes, &S.world_rgb)) ||
      (rc = E->alloc(B * (size_t)S.max_events * 3, &S.events)) || (rc = E->alloc(B, &S.n_events)) ||
      (rc = E->alloc(B * P, &E->d_actions))) {
    mp_destroy(E);
    return rc;
  }
  {  // reward [B][P] | discount [B] | step_type [B] | scalar_obs [n][B][P], all 8-byte elements, one block
    E->scalar_block_bytes = (B * P + B + B + std::max<size_t>(1, T.n_scalar) * B * P) * 8;
    S.reward = reinterpret_cast<double*>(E->scalar_block);
    S.discount = S.reward + B * P;
    S.step_type = reinterpret_cast<int64_t*>(S.discount + B);
    S.scalar_obs = reinterpret_cast<double*>(S.step_type + B);
  }
  {  // everything a later step depends on, plus the current timestep scalars; the images are re-rendered on load
    const size_t ns = std::max<size_t>(1, T.n_scalar);
    auto span = [&](void* p, size_t bytes) { E->state_spans.push_back({p, bytes}); E->state_bytes += bytes; };
    span(S.grid, B * T.L * T.cells_pad * sizeof(*S.grid)); span(S.avatar, B * P * 4 * sizeof(*S.avatar));
    span(S.av_timer, B * P * 4 * sizeof(*S.av_timer)); span(S.apple, B * T.nA_pad * sizeof(*S.apple));
    span(S.dirt, B * T.nD_pad * sizeof(*S.dirt)); span(S.water, B * T.nW_pad * sizeof(*S.water));
    span(S.apple_count, B * T.nA_pad * sizeof(*S.apple_count)); span(S.fam_u8, B * (size_t)S.fam_u8_stride * sizeof(*S.fam_u8));
    span(S.fam_u16, B * (size_t)S.fam_u16_stride * sizeof(*S.fam_u16)); span(S.av_extra, B * P * 8 * sizeof(*S.av_extra));
    span(S.packed, B * (P + 2) * sizeof(*S.packed)); span(S.env, B * ENV_COLS * sizeof(*S.env));
    span(S.reward, B * P * sizeof(*S.reward)); span(S.discount, B * sizeof(*S.discount));
    span(S.step_type, B * sizeof(*S.step_type)); span(S.scalar_obs, ns * B * P * sizeof(*S.scalar_obs));
    span(S.events, B * (size_t)S.max_events * 3 * sizeof(*S.events)); span(S.n_events, B * sizeof(*S.n_events));
  }
  // episode counter starts at -1 so that the first reset plays episode 0; envs start "done".
  {
    std::vector<int32_t> env0(B * ENV_COLS, 0);
    for (size_t b = 0; b < B; ++b) { env0[b * ENV_COLS + ENV_EPISODE] = -1; env0[b * ENV_COLS + ENV_DONE] = 1; }
    cudaError_t ce = cudaMemcpy(S.env, env0.data(), env0.size() * sizeof(int32_t), cudaMemcpyHostToDevice);
    if (ce != cudaSuccess) { mp_destroy(E); return fail(MP_E_CUDA, "cudaMemcpy(env) failed: %s", cudaGetErrorString(ce)); }
  }
  E->step_smem = E->family == MPB_FAMILY_TERRITORY ? territory_scratch_bytes(T) : warp_scratch_bytes(T);
  {  // cells per lane per strip: ceil(view_w / 4) for player rows, ceil(W / 8) for world half-rows
    const int ncp = (E->R.view_w + 3) / 4, ncw = (T.W + (32 >> E->R.wstrip_log2) - 1) / (32 >> E->R.wstrip_log2);
    if (ncp <= 3 && ncw <= 3) { E->render_fn = k_render<3, 3, false>; E->render_gather_fn = k_render<3, 3, true>; E->inst_ncp = 3; E->inst_ncw = 3; }
    else if (ncp <= 3 && ncw <= 4) { E->render_fn = k_render<3, 4, false>; E->render_gather_fn = k_render<3, 4, true>; E->inst_ncp = 3; E->inst_ncw = 4; }
    else if (ncp <= 3 && ncw <= 5) { E->render_fn = k_render<3, 5, false>; E->render_gather_fn = k_render<3, 5, true>; E->inst_ncp = 3; E->inst_ncw = 5; }
    else if (ncp <= 4 && ncw <= 5) { E->render_fn = k_render<4, 5, false>; E->render_gather_fn = k_render<4, 5, true>; E->inst_ncp = 4; E->inst_ncw = 5; }
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
  cudaError_t ce = cudaFuncSetAttribute(E->render_fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kRenderSmemLimit);
  if (ce == cudaSuccess) ce = cudaFuncSetAttribute(E->render_gather_fn, cudaFuncAttributeMaxDynamicSharedMemorySize, kRenderSmemLimit);
  {
    static int step_smem_max[MP_MAX_DEVICES] = {};
    const int need = (int)(E->step_smem * 4 + (E->family == MPB_FAMILY_CLEAN_UP ? clean_up_table_bytes(T) : E->family == MPB_FAMILY_TERRITORY ? territory_table_bytes(T) : 0));
    if (ce == cudaSuccess && need > 48 * 1024 && need > step_smem_max[device]) {
      ce = cudaFuncSetAttribute(k_step_clean_up, cudaFuncAttributeMaxDynamicSharedMemorySize, need);
      if (ce == cudaSuccess) ce = cudaFuncSetAttribute(k_step_commons, cudaFuncAttributeMaxDynamicSharedMemorySize, need);
      if (ce == cudaSuccess) ce = cudaFuncSetAttribute(k_step_territory, cudaFuncAttributeMaxDynamicSharedMemorySize, need);
      if (ce == cudaSuccess) ce = cudaFuncSetAttribute(k_step_coins, cudaFuncAttributeMaxDynamicSharedMemorySize, need);
      if (ce == cudaSuccess) ce = cudaFuncSetAttribute(k_step_mining, cudaFuncAttributeMaxDynamicSharedMemorySize, need);
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

int mp_reset(mp_handle h, const uint8_t* env_mask, void* stream) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  DeviceGuard guard(h->device);
  int rc = launch_state(h, nullptr, env_mask, 1, (cudaStream_t)stream);
  return rc ? rc : launch_render(h, (cudaStream_t)stream);
}

int mp_step_state(mp_handle h, const int32_t* actions, void* stream) {
  if (!h || !actions) return fail(MP_E_INVALID, "mp_step_state: null handle or actions");
  DeviceGuard guard(h->device);
  return launch_state(h, actions, nullptr, 0, (cudaStream_t)stream, /*render_follows=*/false);
}

int mp_render(mp_handle h, void* stream) {
  if (!h) return fail(MP_E_INVALID, "null handle");
  DeviceGuard guard(h->device);
  return launch_render(h, (cudaStream_t)stream);
}

int mp_step(mp_handle h, const int32_t* actions, void* stream) {
  int rc = mp_step_state(h, actions, stream);
  return rc ? rc : mp_render(h, stream);
}

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
  DeviceGuard guard(h->device);
  int rc = async_setup(h);
  if (rc) return rc;
  cudaStream_t st = (cudaStream_t)stream;
  mp_engine::AsyncSlot& sl = h->slot[slot];
  CUDA_TRY(cudaStreamWaitEvent(st, sl.copied, 0));  // the copy-out that last used this slot's device buffers has drained
  CUDA_TRY(cudaMemcpyAsync(sl.actions, actions_host, (size_t)h->B * h->T.P * sizeof(int32_t), cudaMemcpyHostToDevice, st));
  if ((rc = launch_state(h, sl.actions, nullptr, 0, st))) return rc;
  uint8_t* rgb0 = h->S.rgb; uint8_t* world0 = h->S.world_rgb;
  h->S.rgb = sl.rgb; h->S.world_rgb = sl.world_rgb;
  rc = launch_render(h, st);
  h->S.rgb = rgb0; h->S.world_rgb = world0;
  if (rc) return rc;
  CUDA_TRY(cudaMemcpyAsync(sl.scalars, h->scalar_block, h->scalar_block_bytes, cudaMemcpyDeviceToDevice, st));
  CUDA_TRY(cudaEventRecord(sl.computed, st));
  CUDA_TRY(cudaStreamWaitEvent(h->copy_stream, sl.computed, 0));
  if (out && (out->events || out->event_count)) return fail(MP_E_INVALID, "mp_step_host_async: events are not staged per slot; read them with mp_step_host");
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
struct SnapshotHeader { char magic[4]; uint32_t version; uint64_t num_envs, payload_bytes, n_spans, rng_key0, blob_hash; };
}

int mp_state_size(mp_handle h, uint64_t* bytes) {
  if (!h || !bytes) return fail(MP_E_INVALID, "mp_state_size: null argument");
  *bytes = sizeof(SnapshotHeader) + h->state_bytes;
  return MP_OK;
}

int mp_state_save(mp_handle h, void* host_dst, void* stream) {
  if (!h || !host_dst) return fail(MP_E_INVALID, "mp_state_save: null argument");
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  SnapshotHeader hd{{'M', 'P', 'S', '3'}, 3u, (uint64_t)h->B, h->state_bytes, (uint64_t)h->state_spans.size(), h->S.seed, h->blob_hash};
  memcpy(host_dst, &hd, sizeof(hd));
  uint8_t* dst = static_cast<uint8_t*>(host_dst) + sizeof(hd);
  for (const auto& sp : h->state_spans) {
    CUDA_TRY(cudaMemcpyAsync(dst, sp.first, sp.second, cudaMemcpyDeviceToHost, st));
    dst += sp.second;
  }
  CUDA_TRY(cudaStreamSynchronize(st));
  return MP_OK;
}

int mp_state_load(mp_handle h, const void* host_src, uint64_t nbytes, void* stream) {
  if (!h || !host_src) return fail(MP_E_INVALID, "mp_state_load: null argument");
  if (nbytes < sizeof(SnapshotHeader)) return fail(MP_E_INVALID, "mp_state_load: %llu bytes is shorter than a snapshot header", (unsigned long long)nbytes);
  SnapshotHeader hd;
  memcpy(&hd, host_src, sizeof(hd));
  if (memcmp(hd.magic, "MPS3", 4) != 0 || hd.version != 3u) return fail(MP_E_INVALID, "mp_state_load: not a snapshot (or one of an older engine)");
  if (hd.num_envs != (uint64_t)h->B || hd.payload_bytes != h->state_bytes || hd.n_spans != h->state_spans.size())
    return fail(MP_E_INVALID, "mp_state_load: snapshot of %llu envs / %llu bytes does not fit this engine (%d envs / %llu bytes)",
                (unsigned long long)hd.num_envs, (unsigned long long)hd.payload_bytes, h->B, (unsigned long long)h->state_bytes);
  if (nbytes != sizeof(SnapshotHeader) + hd.payload_bytes)
    return fail(MP_E_INVALID, "mp_state_load: buffer of %llu bytes, snapshot needs %llu (truncated?)", (unsigned long long)nbytes,
                (unsigned long long)(sizeof(SnapshotHeader) + hd.payload_bytes));
  if (hd.blob_hash != h->blob_hash) return fail(MP_E_INVALID, "mp_state_load: snapshot was taken from a different compiled substrate");
  if (hd.rng_key0 != h->S.seed) return fail(MP_E_INVALID, "mp_state_load: snapshot was taken with a different seed / env_index_base (key %llu, engine %llu)",
                                            (unsigned long long)hd.rng_key0, (unsigned long long)h->S.seed);
  DeviceGuard guard(h->device);
  cudaStream_t st = (cudaStream_t)stream;
  const uint8_t* src = static_cast<const uint8_t*>(host_src) + sizeof(hd);
  for (const auto& sp : h->state_spans) {
    CUDA_TRY(cudaMemcpyAsync(sp.first, src, sp.second, cudaMemcpyHostToDevice, st));
    src += sp.second;
  }
  int rc = launch_render(h, st);
  if (rc) return rc;
  CUDA_TRY(cudaStreamSynchronize(st));
  return MP_OK;
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
