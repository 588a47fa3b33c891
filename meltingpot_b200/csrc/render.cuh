// render.cuh -- sprite compositing of {i}.RGB and WORLD.RGB for every env instance.
//
// Restates world:createView + tile.Scene:render as used by
//   Avatar:addObservations          meltingpot/lua/modules/avatar_library.lua:225-277
//   BaseSimulation:addObservations  meltingpot/lua/modules/base_simulation.lua:347-368
// (policies A.11-A.14 of the ledger: view window, sprite facing, out-of-bounds / out-of-view
// sprites, bottom-to-top alpha compositing in render order).
//
// HBM-bound by design: per env-step it reads the ~11 KB sprite grid and writes
// P*88*88*3 + H*W*192 bytes of observations. One persistent CTA per SM hosts 2-4
// independent teams of up to TEAM_THREADS threads (RenderPlan::team_threads, the most that fit in
// shared memory next to the atlas) that share one shared-memory copy of the sprite atlas
// (TMA-bulk-loaded once). Each team renders whole envs:
//   1. the env's grid arrives by TMA bulk copy behind an mbarrier (prefetched one env ahead);
//   2. a per-cell pass flattens every cell's layer stack into a short record, folding the opaque
//      bottom sprite and the map sprites stacked on it into one pre-merged opaque sprite
//      (merged on the host with exactly the compositing arithmetic, so results stay bit-exact);
//   3. warps pull "cell-row" items (8 pixel rows of one image), compose them in a warp-private
//      staging buffer (8 pixels = 24 bytes per lane-item) and hand the buffer to cp.async.bulk
//      shared->global stores, so every observation byte is written once, fully coalesced, by the
//      copy engine, with no block-wide barrier on the way. One lane per view cell resolves what the
//      cell shows to this viewer (a rotated single sprite, or a multi-sprite record) and the eight
//      lanes that draw its pixel rows fetch that by shuffle; multi-sprite cells are composited by
//      the lanes that hold them, by selection where every alpha is 0 or 255, arithmetic otherwise.
// What bounds it on H100 (tools/render_bound.py; H100 80GB HBM3 SXM at 700 W, clean_up x 4096, 3 x 10-warp layout):
// the full kernel took 0.430 ms, with the stores alone (no compositing) 0.427 ms, with the compositing alone 0.200 ms,
// and a torch fill_ of the same 1.16 GB took 0.355 ms. Compositing therefore hides under the stores, but the store
// stream itself runs ~20 % below the write ceiling. More staging slots do not close the gap: built with two or three
// slots per warp, at the layouts that then fit, the kernel was no faster, stores alone included, and a bare loop of
// one-slot 2 KB bulk stores on 8-32 warps per SM reaches the fill_ rate. What is left is the per-env skeleton (grid
// wait, per-cell pass, team barriers: 0.066 ms alone), during which a team has no stores in flight. More teams with
// fewer warps each cover those gaps better (the layout score in build_plan).
#pragma once

#include <cstdio>

#include "common.cuh"

#define RENDER_MAX_TEAMS 4   // teams per CTA (RenderPlan::n_teams, 2..4)
#define RENDER_MAX_THREADS 1024
#ifndef TEAM_THREADS
#define TEAM_THREADS 512
#endif
#ifndef RENDER_SLOTS
#define RENDER_SLOTS 1  // staging slots per warp (measured on H100: 2 or 3 bought nothing, see the header)
#endif

struct RenderPlan {  // host-computed constants of the tiling
  int view_w, view_h;        // cells
  int player_bytes;          // per-player image
  int world_bytes;
  int grid_bytes;            // L * cells_pad * 2
  int atlas_bytes;           // n_total sprites * 1024
  int n_total;               // atlas sprites including pre-merged ones
  int rec_stride;            // u16 per cell record: count + up to L entries
  uint32_t magic_view_h;     // p = (item * magic) >> 16 == item / view_h for item < 4096
  // shared memory offsets
  int off_atlas, off_pair, off_map, off_team0, team_stride;
  int toff_grid, toff_rec, toff_stage;  // within a team's region
  int wstrip_log2;                      // log2 of the pixel rows per WORLD.RGB strip (1 or 2)
  int stage_bytes;                      // warp-private staging buffer: RENDER_SLOTS slots, each one player cell-row or one WORLD.RGB strip
  int smem_bytes;
  int team_threads;                     // threads per team (multiple of 32, <= TEAM_THREADS)
  int n_teams;                          // teams per CTA (2..RENDER_MAX_TEAMS); n_teams * team_threads <= 1024
  // per-launch constants (depend on the render flags); kept here so that they are constant-bank operands, not registers
  int n_player_items, n_items;           // strips per env: player cell-rows, then WORLD.RGB strips
  int prow_bytes, wrow_bytes;            // one pixel row of a player image / of WORLD.RGB
  int pitem_bytes, witem_bytes;          // one strip
  int h_oob, h_oov;                      // fast-path headers of the OutOfBounds / OutOfView sprites
  int h_empty;                           // header of a cell with nothing visible: fast path to an opaque black sprite, or 0
  // Which cell each lane draws in each of its NCP / NCW turns on a strip (6 bits per turn, 63 = none). The lane's
  // pixel row stays lane & 7 (player strips) / lane & (rows - 1) (WORLD.RGB strips); the cells are dealt so that the
  // 16 lanes of every half-warp hit 16 different bank pairs with their 64-bit staging stores (host: make_lane_map).
  uint32_t pmap[32], wmap[32];
};

__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }

__device__ __forceinline__ void mbar_init(uint64_t* bar, int count) {
  asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
  asm volatile(
      "{\n"
      ".reg .pred p;\n"
      "WAIT_%=:\n"
      "mbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n"
      "@p bra DONE_%=;\n"
      "bra WAIT_%=;\n"
      "DONE_%=:\n"
      "}\n" ::"r"(smem_u32(bar)), "r"(parity) : "memory");
}
// TMA bulk copy global -> shared, completion signalled on an mbarrier (UBLKCP in SASS).
__device__ __forceinline__ void bulk_load(void* dst_smem, const void* src_gmem, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];" ::"r"(smem_u32(dst_smem)),
               "l"(src_gmem), "r"(bytes), "r"(smem_u32(bar))
               : "memory");
}
// TMA bulk copy shared -> global. Observations are written once and not read again by the engine,
// so they are tagged evict-first: the 47 MB of env state stays L2-resident instead.
__device__ __forceinline__ uint64_t make_evict_first_policy() {
  uint64_t policy;
  asm volatile("createpolicy.fractional.L2::evict_first.b64 %0, 1.0;" : "=l"(policy));
  return policy;
}
__device__ __forceinline__ void bulk_store(void* dst_gmem, const void* src_smem, uint32_t bytes, uint64_t policy) {
  asm volatile("cp.async.bulk.global.shared::cta.bulk_group.L2::cache_hint [%0], [%1], %2, %3;" ::"l"(dst_gmem), "r"(smem_u32(src_smem)),
               "r"(bytes), "l"(policy)
               : "memory");
  asm volatile("cp.async.bulk.commit_group;" ::: "memory");
}
template <int N>
__device__ __forceinline__ void bulk_wait_read() {
  asm volatile("cp.async.bulk.wait_group.read %0;" ::"n"(N) : "memory");
}
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
__device__ __forceinline__ void group_sync(int bar_id, int threads) { asm volatile("bar.sync %0, %1;" ::"r"(bar_id), "r"(threads) : "memory"); }

// dst, src: R | G<<8 | B<<16 (| A<<24 for src). Integer "over": (s*a + d*(255-a)) / 255, truncated.
// Branch free on purpose: a == 255 yields src and a == 0 yields dst exactly, so opaque sprites and
// empty pixels need no special case (and no divergence).
__device__ __forceinline__ uint32_t blend_px(uint32_t dst, uint32_t src) {
  const uint32_t a = src >> 24;
  const uint32_t ia = 255u - a;
  uint32_t rb = (src & 0x00FF00FFu) * a + (dst & 0x00FF00FFu) * ia;  // two 16-bit lanes, each <= 65025
  uint32_t g = ((src >> 8) & 0xFFu) * a + ((dst >> 8) & 0xFFu) * ia;
  rb += 0x00010001u; rb += (rb >> 8) & 0x00FF00FFu; rb = (rb >> 8) & 0x00FF00FFu;  // floor(t / 255) per lane
  g += 1u; g += g >> 8; g = (g >> 8) & 0xFFu;
  return rb | (g << 8);
}

// Record entry: bits 0-12 sprite * 4 + orientation, then the sprite's flag byte shifted by 13:
// bit 13 = opaque, bit 14 = remapped for some viewer (look it up in the viewer's sprite map),
// bit 15 = every alpha is 0 or 255 for every viewer (composited by selection instead of arithmetic).
// (Flag bit 3, not kept in entries: every alpha is 0 -- such sprites never reach a record.)
#define ENT_SHIFT 13
#define ENT_VALUE 0x1fff
#define ENT_OPAQUE 0x2000
#define ENT_REMAP 0x4000
#define ENT_BINARY 0x8000

__device__ __forceinline__ uint32_t select_px(uint32_t dst, uint32_t src) { return (int32_t)src < 0 ? src : dst; }  // alpha in {0, 255}

// Composites pixel row `py` of a multi-sprite record over px[8] (bottom up). Lane private: lanes of a
// warp that hold such cells run their chains side by side (the kernel is latency bound, not issue bound).
__device__ __forceinline__ void compose_row(uint32_t px[8], const uint8_t* __restrict__ s_atlas, const uint16_t* __restrict__ rec,
                                            const int16_t* __restrict__ s_map, int viewer_orient, int py) {
  const int n = rec[0];
#pragma unroll
  for (int k = 0; k < 8; ++k) px[k] = 0;
  for (int k = 1; k <= n; ++k) {
    const uint32_t e = rec[k];
    int sprite = (e & ENT_VALUE) >> 2;
    if (e & ENT_REMAP) sprite = s_map[sprite];
    const int facing = ((int)(e & 3) - viewer_orient) & 3;
    const uint8_t* t = s_atlas + (sprite * 4 + facing) * 256 + py * 16;
    const uint4 lo = *reinterpret_cast<const uint4*>(t);
    const uint4 hi = *reinterpret_cast<const uint4*>(t + 128);
    if (e & ENT_BINARY) {
      px[0] = select_px(px[0], lo.x); px[1] = select_px(px[1], lo.y); px[2] = select_px(px[2], lo.z); px[3] = select_px(px[3], lo.w);
      px[4] = select_px(px[4], hi.x); px[5] = select_px(px[5], hi.y); px[6] = select_px(px[6], hi.z); px[7] = select_px(px[7], hi.w);
    } else {
      px[0] = blend_px(px[0], lo.x); px[1] = blend_px(px[1], lo.y); px[2] = blend_px(px[2], lo.z); px[3] = blend_px(px[3], lo.w);
      px[4] = blend_px(px[4], hi.x); px[5] = blend_px(px[5], hi.y); px[6] = blend_px(px[6], hi.z); px[7] = blend_px(px[7], hi.w);
    }
  }
}

// Header of a flattened cell record: bit 15 set = the cell is a single opaque sprite and the low
// bits are sprite * 4 + orientation (fast path); otherwise the number of entries that follow.
#define REC_FAST 0x8000

// Per-cell pass of one env: flattens each cell's layer stack into a record, folding map sprites into
// pre-merged ones. LMAX >= T.L is a compile-time bound so that the layer loads are independent and
// unrolled; the layers that matter are then found with bit masks (most cells hold one sprite).
template <int LMAX>
__device__ __forceinline__ void cell_pass(const Tables& T, const RenderPlan& R, const uint16_t* __restrict__ s_grid, uint16_t* __restrict__ s_rec,
                                          const uint8_t* __restrict__ s_flags, const uint8_t* __restrict__ s_pair, int gtid, int gthreads, uint32_t dbg) {
  for (int c = gtid; c < T.cells; c += gthreads) {
    uint32_t v[LMAX];
#pragma unroll
    for (int l = 0; l < LMAX; ++l) v[l] = l < T.L ? s_grid[l * T.cells_pad + c] : 0u;
    uint32_t nz = 0, oq = 0;
#pragma unroll
    for (int l = 0; l < LMAX; ++l) {
      const uint32_t f = v[l] ? s_flags[(v[l] - 1) >> 2] : 8u;
      nz |= ((f & 8u) ? 0u : 1u) << l;  // (bit 3: every alpha is 0 -- the piece is there but draws nothing)
      oq |= (f & 1u) << l;
    }
    oq &= ~1u;
    const int lo = oq ? 31 - __clz(oq) : 0;  // the topmost opaque layer hides everything below it
    uint32_t cand = nz & (0xffffffffu << lo);
    uint16_t* r = s_rec + c * R.rec_stride;
    int n = 0;
    uint32_t cur = 0, cf = 0;
    bool merging = true;
    while (cand) {
      const int l = __ffs(cand) - 1;
      cand &= cand - 1;
      const uint32_t vl = s_grid[l * T.cells_pad + c];
      if (cur == 0) { cur = vl; cf = s_flags[(vl - 1) >> 2]; continue; }
      if (merging) {
        const uint32_t m = s_pair[((cur - 1) >> 2) * R.n_total + ((vl - 1) >> 2)];
        if (m && (((cur - 1) ^ (vl - 1)) & 3u) == 0) { cur = 1 + m * 4 + ((vl - 1) & 3u); cf = 5; continue; }  // merged sprites: opaque, binary
        merging = false;
      }
      r[1 + n++] = (uint16_t)((cur - 1) | (cf << ENT_SHIFT));
      cur = vl; cf = s_flags[(vl - 1) >> 2];
    }
    if (cur) r[1 + n++] = (uint16_t)((cur - 1) | (cf << ENT_SHIFT));
    if ((n == 1 && (cf & 1u)) || ((dbg & 256u) && cur)) r[0] = (uint16_t)(REC_FAST | (cur - 1));  // (bit 8: debug -- top sprite only)
    else r[0] = n ? (uint16_t)n : (uint16_t)R.h_empty;  // nothing to draw: the black sprite if the atlas has one, else an empty record
  }
}

// 8 RGBA pixels -> 24 packed RGB bytes at `dst` (8-byte aligned).
__device__ __forceinline__ void store_row(uint8_t* dst, const uint32_t px[8]) {
  uint2 a, b, c;
  a.x = __byte_perm(px[0], px[1], 0x4210); a.y = __byte_perm(px[1], px[2], 0x5421);
  b.x = __byte_perm(px[2], px[3], 0x6542); b.y = __byte_perm(px[4], px[5], 0x4210);
  c.x = __byte_perm(px[5], px[6], 0x5421); c.y = __byte_perm(px[6], px[7], 0x6542);
  uint2* d = reinterpret_cast<uint2*>(dst);
  d[0] = a; d[1] = b; d[2] = c;
}

// Loads pixel row `py` of the sprite variant (sprite * 4 + facing) selected by a fast-path header.
__device__ __forceinline__ void fast_row(uint32_t px[8], const uint8_t* __restrict__ s_atlas, int h, int py) {
  const uint8_t* t = s_atlas + (h & 0x7fff) * 256 + py * 16;
  const uint4 lo = *reinterpret_cast<const uint4*>(t);
  const uint4 hi = *reinterpret_cast<const uint4*>(t + 128);
  px[0] = lo.x; px[1] = lo.y; px[2] = lo.z; px[3] = lo.w; px[4] = hi.x; px[5] = hi.y; px[6] = hi.z; px[7] = hi.w;
}

struct ViewerInfo {  // per player, refreshed once per env
  int ax, ay, ao, alive, fdx, fdy, rdx, rdy;
};

// Work decomposition: an env is rendered by one team; after the per-cell pass its warps pull
// strip items from a shared counter -- one row of view cells (8 pixel rows) of a player image, or
// a half / quarter cell row (4 / 2 pixel rows) of WORLD.RGB -- compose them into a warp-private staging slot and
// hand the slot to the TMA store engine. Two team barriers per env; everything else is warp-local.
// Each lane handles NC cells per strip with the loads of all NC cells issued before any is packed.
// MODE (exclusive):
//   RENDER_GATHER: also deliver every strip into every rank's stacked observation buffer (State::g_*);
//   RENDER_ROUTED: deliver player p of env b to the row State::pr.row_of_player[b][p] of the caller's per-player
//     targets (mp_run's players), through the segment of G that holds the row. The team's first warp reads the env's
//     row map with its avatars and compacts the players whose rows lie in a segment into s_players; the env's item loop
//     then runs over those players' strips and WORLD.RGB's only, so an unrouted player is neither composited nor
//     stored. At each player strip's store, lane 0 reads the row again and resolves its segment and address. With State::pr.world_rgb set, the same warp also reads
//     the env's WORLD.RGB row (State::pr.world_row_of_env[b]): an env with a row stores its WORLD.RGB strips there,
//     an env without one has no WORLD.RGB strips.
enum { RENDER_PLAIN = 0, RENDER_GATHER = 1, RENDER_ROUTED = 2 };
template <int NCP, int NCW, int MODE>
__global__ void __launch_bounds__(RENDER_MAX_THREADS, 1) k_render(Tables T, State S, RenderPlan R, uint32_t flags,
                                                            const __grid_constant__ RowSegments G) {
  constexpr bool GATHER = MODE == RENDER_GATHER, ROUTED = MODE == RENDER_ROUTED;
  extern __shared__ __align__(128) uint8_t smem[];
  uint64_t* bar = reinterpret_cast<uint64_t*>(smem);  // [0] atlas, [1 + team] grid
  uint8_t* s_atlas = smem + R.off_atlas;
  const uint8_t* s_pair = smem + R.off_pair;                          // [n_total][n_total] merged sprite or 0
  int16_t* s_map = reinterpret_cast<int16_t*>(smem + R.off_map);      // [P+1][n_total]
  __shared__ uint8_t s_opaque[256];
  __shared__ ViewerInfo s_view_all[RENDER_MAX_TEAMS][MP_MAX_PLAYERS];
  __shared__ int s_next_item[RENDER_MAX_TEAMS];
  // RENDER_ROUTED: the env's routed players in player order, its player strips (routed players x view_h), its
  // WORLD.RGB strips and its WORLD.RGB row
  __shared__ uint8_t s_players_all[RENDER_MAX_TEAMS][MP_MAX_PLAYERS];
  __shared__ int s_route_all[RENDER_MAX_TEAMS][3];

  const int tid = threadIdx.x;
  int team = 0;
#pragma unroll
  for (int k = 1; k < RENDER_MAX_TEAMS; ++k) team += tid >= k * R.team_threads;
  // `team` feeds every shared-memory base below; pinned so that the compiler keeps it in a register instead of
  // re-deriving it from threadIdx inside the strip loop (measured: 1-2 % of the kernel)
  asm volatile("" : "+r"(team));
  const int ttid = tid - team * R.team_threads;
  const int lane = tid & 31, twarp = ttid >> 5;
  uint8_t* s_team = smem + R.off_team0 + team * R.team_stride;
  uint16_t* s_grid = reinterpret_cast<uint16_t*>(s_team + R.toff_grid);  // (these four switch to team 0's in the cooperative tail)
  uint16_t* s_rec = reinterpret_cast<uint16_t*>(s_team + R.toff_rec);
  uint8_t* s_stage = s_team + R.toff_stage + twarp * R.stage_bytes;  // warp-private
  ViewerInfo* s_view = s_view_all[team];
  uint8_t* s_players = s_players_all[team];
  int* s_route = s_route_all[team];  // [0] player strips, [1] WORLD.RGB strips, [2] WORLD.RGB row
  uint64_t* gbar = &bar[1 + team];

  // Work split. Balanced part: `rounds` = B / (teams in the grid) envs per team, rendered team by team with no
  // interaction between teams. Tail: the remaining B mod (teams in the grid) envs are dealt to the CTAs and each is
  // rendered by ALL teams of its CTA together (one cell pass into team 0's records, every warp pulling that env's
  // strips), so the kernel ends after rounds + ~1/n_teams env-times instead of rounds + 1.
  const int n_streams = gridDim.x * R.n_teams;
  const int rounds = S.B / n_streams;
  const int tail0 = rounds * n_streams;
  const int n_tail = (S.B - tail0 - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;  // >= 0: tail envs of this CTA
  const int n_iters = rounds + (n_tail > 0 ? n_tail : 0);
  const int first = blockIdx.x * R.n_teams + team;
  if (tid == 0) {
    for (int i = 0; i < 1 + R.n_teams; ++i) mbar_init(&bar[i], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  if (ttid == 0) s_next_item[team] = 0;
  asm volatile("griddepcontrol.launch_dependents;" ::: "memory");  // the next state-transition kernel may queue up behind this grid
  __syncthreads();
  if (tid == 0) {
    mbar_expect_tx(&bar[0], (uint32_t)R.atlas_bytes);
    bulk_load(s_atlas, T.atlas, (uint32_t)R.atlas_bytes, &bar[0]);
  }
  for (int i = tid; i < (T.P + 1) * R.n_total; i += (int)blockDim.x) s_map[i] = T.sprite_map[i];
  for (int i = tid; i < R.n_total; i += (int)blockDim.x) s_opaque[i] = T.sprite_opaque[i];
  for (int i = tid; i < R.n_total * R.n_total; i += (int)blockDim.x) smem[R.off_pair + i] = T.sprite_pair[i];
  // Everything above reads only static tables: with a programmatic dependent launch it overlaps the tail of the
  // state-transition kernel. The env state (grid, avatars) may be read only after this point.
  asm volatile("griddepcontrol.wait;" ::: "memory");
  if (GATHER && tid == 64 && S.g_step > 1ull) {
    // flow control of the stacked buffers: slot (g_step & 1) holds render g_step - 2; a rank is done with it once it has
    // delivered render g_step - 1 (its consumers are stream-ordered before that launch)
    for (int r = 0; r < S.g_world; ++r)
      while (*(const volatile unsigned long long*)(S.g_flags + r) + 1ull < S.g_step) __nanosleep(200);
  }
  if (ttid == 0 && rounds > 0) {
    mbar_expect_tx(gbar, (uint32_t)R.grid_bytes);
    bulk_load(s_grid, S.grid + (size_t)first * T.L * T.cells_pad, (uint32_t)R.grid_bytes, gbar);
  }
  __syncthreads();  // tables visible to every warp before the first cell pass
  mbar_wait(&bar[0], 0);

  const int wlog = R.wstrip_log2, wrows = 1 << wlog;  // pixel rows per WORLD.RGB strip (2 or 4)
  const int slot_bytes = R.stage_bytes / RENDER_SLOTS;
  const uint64_t store_policy = make_evict_first_policy();
  uint32_t pcells = R.pmap[lane], wcells = R.wmap[lane];
  // pinned: otherwise the compiler re-reads them from the parameter bank inside the strip loop, and a constant load
  // with a per-lane index is replayed 32 times through the MIO queue (measured: 2.5x on the whole kernel)
  asm volatile("" : "+r"(pcells), "+r"(wcells));
  uint32_t slot = 0;
  // the group that renders the current env: a team (balanced part) or the whole CTA (tail)
  int gtid = ttid, gthreads = R.team_threads, bar_id = 1 + team;
  int* next_ctr = &s_next_item[team];
  for (int it = 0; it < n_iters; ++it) {
    if (it == rounds) {  // switch to the cooperative tail: every team is done with its own envs
      __syncthreads();
      uint8_t* s_team0 = smem + R.off_team0;
      s_grid = reinterpret_cast<uint16_t*>(s_team0 + R.toff_grid);
      s_rec = reinterpret_cast<uint16_t*>(s_team0 + R.toff_rec);
      s_view = s_view_all[0];
      s_players = s_players_all[0]; s_route = s_route_all[0];
      gbar = &bar[1];
      next_ctr = &s_next_item[0];
      gtid = tid; gthreads = (int)blockDim.x; bar_id = 0;
      if (tid == 0) {
        mbar_expect_tx(gbar, (uint32_t)R.grid_bytes);
        bulk_load(s_grid, S.grid + (size_t)(tail0 + (int)blockIdx.x) * T.L * T.cells_pad, (uint32_t)R.grid_bytes, gbar);
      }
    }
    const int b = it < rounds ? first + it * n_streams : tail0 + (int)blockIdx.x + (it - rounds) * (int)gridDim.x;
    if (gtid < T.P) {
      const int4 a = *reinterpret_cast<const int4*>(S.avatar + ((size_t)b * T.P + gtid) * 4);
      ViewerInfo vi;
      vi.ax = a.x; vi.ay = a.y; vi.ao = a.z; vi.alive = a.w;
      vi.fdx = dir_dx(a.z); vi.fdy = dir_dy(a.z); vi.rdx = dir_dx((a.z + 1) & 3); vi.rdy = dir_dy((a.z + 1) & 3);
      s_view[gtid] = vi;
    }
    if (ROUTED && gtid < 32) {  // the group's first warp, whole: compact the routed players (all of them when the images are not routed)
      bool on = gtid < T.P;
      if (on && G.s[0].rgb) on = row_segment(G, S.pr.row_of_player[(size_t)b * T.P + gtid]) >= 0;
      const uint32_t m = __ballot_sync(MP_FULL, on);
      if (on) s_players[__popc(m & ((1u << gtid) - 1u))] = (uint8_t)gtid;
      if (gtid == 0) {
        s_route[0] = G.s[0].rgb ? __popc(m) * R.view_h : R.n_player_items;
        int wrow = 0, wn = R.n_items - R.n_player_items;
        if (S.pr.world_rgb) {
          wrow = S.pr.world_row_of_env[b];
          if ((uint32_t)wrow >= (uint32_t)S.pr.world_n_rows) wn = 0;
        }
        s_route[1] = wn; s_route[2] = wrow;
      }
    }  // (published by the group barrier after the cell pass, like s_view)
    mbar_wait(gbar, (uint32_t)(it & 1));  // (team 0's barrier has completed `rounds` phases when the tail starts, so the parity carries over)
    // ---- per-cell pass: flatten the layer stack, folding map sprites into pre-merged ones -------
    if (!(flags & 64u) || it == 0) {  // (bit 6: debug -- reuse the first env's records)
      if (T.L <= 8) cell_pass<8>(T, R, s_grid, s_rec, s_opaque, s_pair, gtid, gthreads, flags);
      else if (T.L <= 10) cell_pass<10>(T, R, s_grid, s_rec, s_opaque, s_pair, gtid, gthreads, flags);
      else if (T.L <= 12) cell_pass<12>(T, R, s_grid, s_rec, s_opaque, s_pair, gtid, gthreads, flags);
      else cell_pass<MP_MAX_LAYERS>(T, R, s_grid, s_rec, s_opaque, s_pair, gtid, gthreads, flags);
    }
    group_sync(bar_id, gthreads);  // records complete; the grid buffer is free again
    if (gtid == 0 && it + 1 < n_iters && it + 1 != rounds) {  // (the first tail env is fetched at the switch)
      const int nb = it + 1 < rounds ? b + n_streams : b + (int)gridDim.x;
      mbar_expect_tx(gbar, (uint32_t)R.grid_bytes);
      bulk_load(s_grid, S.grid + (size_t)nb * T.L * T.cells_pad, (uint32_t)R.grid_bytes, gbar);
    }

    // ---- strip items, pulled by warps -------------------------------------------------------------
    int next_item = 0;  // claimed one strip ahead so that the atomic's latency hides behind the strip being drawn
    if (lane == 0) next_item = atomicAdd(next_ctr, 1);
    // RENDER_ROUTED: this env's player and WORLD.RGB strips (the other modes read R's, as constant operands); the WORLD.RGB count is re-read at each item (held in a register, it spilled in <4, 5>)
    const int r_pitems = ROUTED ? s_route[0] : 0;
    for (;;) {
      const int item = __shfl_sync(MP_FULL, next_item, 0);
      if (ROUTED ? item - r_pitems >= s_route[1] : item >= R.n_items) break;
      if (lane == 0) next_item = atomicAdd(next_ctr, 1);
      uint8_t* buf = s_stage + (slot % RENDER_SLOTS) * slot_bytes;
      ++slot;
      if (lane == 0) bulk_wait_read<RENDER_SLOTS - 1>();  // the store that last used this slot has drained
      __syncwarp();
      if (item < (ROUTED ? r_pitems : R.n_player_items)) {
        const int k = (int)(((uint32_t)item * R.magic_view_h) >> 16), cy = item - k * R.view_h;
        const int p = ROUTED ? (int)s_players[k] : k;
        const ViewerInfo vi = s_view[p];
        const int16_t* map = s_map + p * R.n_total;
        const int py = lane & 7;
        const int df = T.view_f - cy;
        const int bx = vi.ax + vi.fdx * df - vi.rdx * T.view_l, by = vi.ay + vi.fdy * df - vi.rdy * T.view_l;
        int hdr[NCP];
        if (!(flags & 16u)) {  // (bit 4: debug / ceiling measurement -- issue the stores without composing)
        // lane cx resolves view cell cx once: a single-sprite cell becomes REC_FAST | sprite * 4 + facing as this
        // viewer sees it, anything else the cell index; the lanes that draw the cell's rows fetch it by shuffle
        int myh = R.h_oov;
        if (lane < R.view_w && vi.alive) {
          int wx = bx + vi.rdx * lane, wy = by + vi.rdy * lane;
          if (wrap_or_reject(T, wx, wy)) {
            const int cell = wy * T.W + wx, h = s_rec[cell * R.rec_stride];
            myh = (h & REC_FAST) ? ((h & ~3) | ((h - vi.ao) & 3)) : cell;
          } else {
            myh = R.h_oob;  // policy A.13
          }
        }
#pragma unroll
        for (int i = 0; i < NCP; ++i) hdr[i] = __shfl_sync(MP_FULL, myh, (pcells >> (6 * i)) & 31);
#pragma unroll
        for (int i = 0; i < NCP; ++i) {  // ... then each cell's sprite row: load (a multi-sprite cell loads a dummy), composite, pack, stage
          const int cx = (pcells >> (6 * i)) & 63;
          uint32_t q[8];
          fast_row(q, s_atlas, (hdr[i] & REC_FAST) ? hdr[i] : 0, py);
          if (!(hdr[i] & REC_FAST)) compose_row(q, s_atlas, s_rec + hdr[i] * R.rec_stride, map, vi.ao, py);
          if (cx < R.view_w) store_row(buf + py * R.prow_bytes + cx * 24, q);
        }
        }
        if (!(flags & 128u)) fence_async_smem();  // make this lane's writes visible to the async (TMA) proxy
        __syncwarp();
        if (lane == 0 && !(flags & 32u)) {
          const size_t in_env = (size_t)p * R.player_bytes + (size_t)cy * R.pitem_bytes;
          if (ROUTED && G.s[0].rgb) {
            const int row = S.pr.row_of_player[(size_t)b * T.P + p];
            const RowSegment& g = G.s[row_segment(G, row)];  // (compaction kept only players whose row lies in a segment)
            bulk_store(g.rgb + (size_t)(row - g.row_begin) * g.rgb_row_stride + (size_t)cy * R.pitem_bytes, buf, (uint32_t)R.pitem_bytes, store_policy);
          }
          else bulk_store(S.rgb + b * S.rgb_env_stride + in_env, buf, (uint32_t)R.pitem_bytes, store_policy);
          if (GATHER) {  // the stacked slots stay dense, whatever the local target's stride
            const size_t off = (size_t)b * T.P * R.player_bytes + in_env;
            for (int r = 0; r < S.g_world; ++r) bulk_store(S.g_rgb[r] + off, buf, (uint32_t)R.pitem_bytes, store_policy);
          }
        }
      } else {
        const int wi = item - (ROUTED ? r_pitems : R.n_player_items), wy = wi >> (3 - wlog);
        const int py = ((wi & ((8 >> wlog) - 1)) << wlog) | (lane & (wrows - 1));
        const int16_t* map = s_map + T.P * R.n_total;
        const uint16_t* rowrec = s_rec + wy * T.W * R.rec_stride;
        int hdr[NCW];
        if (!(flags & 16u)) {
#pragma unroll
        for (int i = 0; i < NCW; ++i) {
          const int cx = (wcells >> (6 * i)) & 63;
          hdr[i] = cx < T.W ? (int)rowrec[cx * R.rec_stride] : R.h_oov;
        }
#pragma unroll
        for (int i = 0; i < NCW; ++i) {
          const int cx = (wcells >> (6 * i)) & 63;
          uint32_t q[8];
          fast_row(q, s_atlas, (hdr[i] & REC_FAST) ? hdr[i] : 0, py);
          if (!(hdr[i] & REC_FAST)) compose_row(q, s_atlas, rowrec + min(cx, T.W - 1) * R.rec_stride, map, 0, py);
          if (cx < T.W) store_row(buf + (py & (wrows - 1)) * R.wrow_bytes + cx * 24, q);
        }
        }
        if (!(flags & 128u)) fence_async_smem();
        __syncwarp();
        if (lane == 0 && !(flags & 32u)) {
          const size_t in_env = (size_t)wi * R.witem_bytes;
          if (ROUTED && S.pr.world_rgb)
            bulk_store(S.pr.world_rgb + (size_t)s_route[2] * S.pr.world_rgb_row_stride + in_env, buf, (uint32_t)R.witem_bytes, store_policy);
          else bulk_store(S.world_rgb + b * S.world_env_stride + in_env, buf, (uint32_t)R.witem_bytes, store_policy);
          if (GATHER) {
            const size_t off = (size_t)b * R.world_bytes + in_env;
            for (int r = 0; r < S.g_world; ++r) bulk_store(S.g_wrgb[r] + off, buf, (uint32_t)R.witem_bytes, store_policy);
          }
        }
      }
    }
    // this rank's timestep rows -> every rank's gathered buffer (and the step's scalar rows -> the caller's target): by
    // each warp once it has run out of strips of its first env, so the loads and the stores overlap the other warps'
    // drawing instead of delaying the kernel's start
    if (S.x_raise && it == 0) exchange_push(T, S);
    if (S.out.on && it == 0) deliver_scalars(T, S);  // (tested here, not only inside: measured, k_render<3, 3, true> spills otherwise)
    if (ROUTED && S.pr.scalars_on && it == 0) deliver_player_scalars(T, S, G);
    group_sync(bar_id, gthreads);  // every warp is done with s_rec / s_view
    if (gtid == 0) *next_ctr = 0;
    // (the reset is ordered before the next env's item loop by the group barrier after its cell pass)
  }
  if (lane == 0) { if (GATHER) asm volatile("cp.async.bulk.wait_group 0;" ::: "memory"); else bulk_wait_read<0>(); }  // (remote stores: wait for completion, not just for the source reads)
}
