/* mp_engine.h -- C ABI of the batched Melting Pot substrate engine (libmpengine.so).
 *
 * This is the drop-in boundary for the reference's hot path. In the reference the path sits
 * behind the pybind11 module `dmlab2d` (third-party), bound at
 *   meltingpot/utils/substrates/builder.py:179-187
 *     env_raw = dmlab2d.Lab2d(_DMLAB2D_ROOT, lab2d_settings_dict)
 *     dmlab2d.Environment(env=env_raw, observation_names=..., seed=seed)
 * and is consumed through Lab2dWrapper.{reset,step,observation,...}
 *   meltingpot/utils/substrates/wrappers/base.py:26-84.
 * Each entry point below names the reference call it replaces. Plain pointers and sizes only:
 * no torch / C++ types cross this boundary. All functions return 0 on success or a negative
 * MP_E_* code; mp_last_error() describes the most recent failure on the calling thread.
 * Nothing here ever falls back to a CPU implementation.
 */
#ifndef MP_ENGINE_H_
#define MP_ENGINE_H_

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef struct mp_engine* mp_handle;

enum {
  MP_OK = 0,
  MP_E_INVALID = -1,     /* bad argument / malformed blob */
  MP_E_UNSUPPORTED = -2, /* substrate family or parameter outside what the kernels implement */
  MP_E_CUDA = -3,        /* CUDA runtime error (message in mp_last_error) */
  MP_E_NO_DEVICE = -4    /* no usable sm_90 device: the engine refuses to run */
};

/* Option flags for mp_create / mp_set_flags. */
enum {
  MP_FLAG_RENDER_WORLD = 1u << 0, /* produce WORLD.RGB (base_simulation.lua:347-362) */
  MP_FLAG_RENDER_PLAYERS = 1u << 1, /* produce {i}.RGB (avatar_library.lua:264-276) */
  MP_FLAG_DEFAULT = 3u,
  /* Diagnostics for tools/render_bound.py (the images are wrong or absent while any is set):
   * time the renderer's store path and its compositing separately. */
  MP_FLAG_DEBUG_NO_COMPOSE = 1u << 4,   /* issue the stores without drawing */
  MP_FLAG_DEBUG_NO_STORE = 1u << 5,     /* draw without storing */
  MP_FLAG_DEBUG_REUSE_RECORDS = 1u << 6, /* per-cell pass only for the first env of each team */
  MP_FLAG_DEBUG_NO_FENCE = 1u << 7,     /* skip the generic->async proxy fence */
  MP_FLAG_DEBUG_TOP_SPRITE_ONLY = 1u << 8, /* every cell drawn as its top sprite */
  MP_FLAG_DEBUG_PLAIN_LANE_MAP = 1u << 9,  /* mp_create only: deal cells to lanes in plain order (A/B) */
  MP_FLAG_DEBUG_SCATTER_LANE_MAP = 1u << 10, /* mp_create only: fully conflict-free dealing that scatters a cell's rows over turns (A/B) */
  MP_FLAG_DEBUG_NO_PREMERGE = 1u << 11,    /* mp_create only: no pre-merged sprites, every stacked cell is composited per pixel */
  /* mp_create only: forced render layout (teams per CTA 2-4, warps per team 4-16, log2 of the WORLD.RGB strip rows 1-2)
   * instead of the one the engine scores best; all three fields zero = the engine's choice. A layout whose shared memory
   * or thread count does not fit makes mp_create fail with MP_E_UNSUPPORTED. Pack with MP_RENDER_LAYOUT(). */
  MP_FLAG_LAYOUT_TEAMS_SHIFT = 16, /* 3 bits */
  MP_FLAG_LAYOUT_WARPS_SHIFT = 19, /* 5 bits */
  MP_FLAG_LAYOUT_WLOG_SHIFT = 24,  /* 2 bits */
  MP_FLAG_LAYOUT_MASK = 0x3ffu << 16
};
#define MP_RENDER_LAYOUT(teams, warps, wlog) \
  (((uint32_t)(teams) << MP_FLAG_LAYOUT_TEAMS_SHIFT) | ((uint32_t)(warps) << MP_FLAG_LAYOUT_WARPS_SHIFT) | ((uint32_t)(wlog) << MP_FLAG_LAYOUT_WLOG_SHIFT))
/* Flags that only mp_create reads; mp_set_flags keeps the values given at creation. */
#define MP_FLAGS_CREATE_ONLY (MP_FLAG_DEBUG_PLAIN_LANE_MAP | MP_FLAG_DEBUG_SCATTER_LANE_MAP | MP_FLAG_DEBUG_NO_PREMERGE | MP_FLAG_LAYOUT_MASK)

/* Device buffers owned by the engine; valid until mp_destroy. Contents are overwritten by the
 * next step or reset on the same handle (mp_run with `out` or `players`: see mp_request for the images). B = num_envs, P = players. */
typedef struct mp_buffers {
  int32_t num_envs, num_players;
  int32_t rgb_h, rgb_w;     /* per-player view in pixels (88 x 88 for clean_up) */
  int32_t world_h, world_w; /* WORLD.RGB in pixels */
  int32_t num_actions;      /* discrete actions per player */
  int32_t num_scalar_obs;   /* per-player f64 observations besides REWARD */
  uint8_t* rgb;             /* u8  [B][P][rgb_h][rgb_w][3]      "{i}.RGB" */
  uint8_t* world_rgb;       /* u8  [B][world_h][world_w][3]     "WORLD.RGB" */
  double* reward;           /* f64 [B][P]                       "{i}.REWARD" */
  double* discount;         /* f64 [B]   0.0 on FIRST/LAST, 1.0 mid-episode */
  int64_t* step_type;       /* i64 [B]   dm_env.StepType: 0 FIRST, 1 MID, 2 LAST */
  double* scalar_obs;       /* f64 [num_scalar_obs][B][P], order of blob section "scalar_obs" */
  int32_t* avatar_state;    /* i32 [B][P][4] x, y, orientation, alive (debug / parity) */
  uint16_t* grid;           /* u16 [B][L][cells_padded] sprite grid (debug / parity) */
  int32_t grid_layers, grid_cells, grid_cells_padded;
  double* timestep_packed;  /* f64 [B][P+2]: reward[0..P), discount, step type -- one buffer for the per-step all-gather */
  /* Events of the current step (SURVEY.md section 8f N3; the events:add calls of avatar_library.lua:661,1070,1088,
   * component_library.lua:996, clean_up/components.lua:152,402, territory/components.lua:133,168, coins/components.lua:133). Row = (type, a, b)
   * with 1-based player indices: 1 zap(source, target), 2 edible_consumed(player), 3 player_cleaned(player),
   * 4 claimed_resource(player), 5 destroyed_resource(player), 6 sanctioning(source, target),
   * 7 removal_due_to_sanctioning(source, target), 8 coin_consumed(player, 1 if the coin matched the player's type else 0;
   * coins/components.lua:133-137), 9 mining(player, ore type), 10 extraction(player, ore type),
   * 11 extraction_pair(player_a, player_b | ore type << 8) (coop_mining/components.lua:203-234). Rows of one step are in no particular order. max_events is the
   * family's worst case for one step (per avatar: three events per beam-footprint cell + contact events), so
   * event_count never exceeds it and no event is dropped. */
  int32_t* events;          /* i32 [B][max_events][3] */
  int32_t* event_count;     /* i32 [B] */
  int32_t max_events;
  /* reward | discount | step_type | scalar_obs above are carved, in this order, from ONE device allocation of
   * scalar_block_bytes bytes starting at scalar_block (every element is 8 bytes), so a host consumer can fetch all
   * scalar outputs of a step with a single copy (mp_host_outputs.scalar_block). */
  void* scalar_block;
  uint64_t scalar_block_bytes;
  /* After mp_exchange_create: f64 [2][gathered_world * B][P + 2], the timestep_packed rows of EVERY rank's envs in
   * global env order (rank r's envs at rows [r * B, (r + 1) * B)); slot (step & 1) holds the most recent step. */
  double* gathered;
  int32_t gathered_world;
  /* After mp_gather_obs_create: the stacked observations of EVERY rank's envs in global env order, two slots of
   * gathered_obs_slot_bytes bytes each (slot = parity of the render sequence number, mp_gather_obs_slot):
   * gathered_rgb u8 [world * B][P][rgb_h][rgb_w][3] and gathered_world_rgb u8 [world * B][world_h][world_w][3] of slot
   * 0; add gathered_obs_slot_bytes for slot 1. */
  uint8_t* gathered_rgb;
  uint8_t* gathered_world_rgb;
  uint64_t gathered_obs_slot_bytes;
} mp_buffers;

/* Replaces dmlab2d.Lab2d(...) + dmlab2d.Environment(...) (builder.py:182-187) for `num_envs`
 * independent instances on CUDA device `device`. `blob` is a compiled substrate
 * (include/mpb_format.h). Env b uses RNG key `seed + env_index_base + b`, so results do not
 * depend on how envs are sharded over GPUs. Does NOT start an episode; run a reset (mp_run). */
int mp_create(const void* blob, size_t blob_bytes, int num_envs, int device, uint64_t seed,
              uint64_t env_index_base, uint32_t flags, mp_handle* out);

/* Heterogeneous batch: one engine whose envs each run under one of `n_variants` (1..MP_MAX_VARIANTS) compiled blobs of
 * the same substrate, as separate reference builds with different `prefab_overrides` (builder.py:70-87) would. Env b
 * starts under variant env_variant_host[b] (host array of num_envs bytes; NULL = every env variant 0) and gives, byte
 * for byte, what env b of an mp_create engine built from its variant's blob with the same seed and env_index_base
 * gives. The variants must be compatible, which is checked once here; otherwise this fails with MP_E_UNSUPPORTED and
 * mp_last_error names the first section or parameter that differs:
 *   - every blob section other than the family's parameter blocks ("<fam>_ip", "<fam>_dp"), "comps", "comps_f" and
 *     "info_json" is byte-identical: the map, sprites, atlas, view, action table and 'choice' groups agree;
 *   - each variant passes every check mp_create makes;
 *   - the entity counts, the episode ending and the beam footprints agree;
 *   - the family's parameters differ only in its scalar knobs (cooldowns, rewards, probabilities, rates, delays, ...):
 *     layers, sprites, hit ids, beam shapes and whatever sizes per-env state agree.
 * Four families take map variants: blobs compiled as one set on one sprite table (compiler.compile_settings_set), such
 * as the draws of coins' config builder, commons_harvest__open, __closed and __partnership, or layouts of one territory
 * or coop_mining map. Their variants may also differ in the map: the initial grid, the object, kind and state tables,
 * the walls (BeamBlocker bits), the spawn points, the family's entity tables (coins: the coins; commons_harvest: the
 * apples and their regrowth discs; territory: the resources, walls and the resources' 'choice' conditions; coop_mining:
 * the ores), the entity count, the object, kind, state and component counts of "meta", and the sprite of each state and
 * avatar. An env
 * plays its variant's map, which changes only at an episode start. Every other "meta" field (size, layers, players,
 * view, ...), the sprite table, the other avatar columns, the hits and the episode ending still agree. commons_harvest
 * variants may also differ in the Zapper's beam footprint (its beamLength / beamRadius, such as the longer beam of
 * __closed and __partnership); the engine's event rows (max_events) are sized for the largest footprint.
 * Envs of an engine with more than one variant run a separate instantiation of the state-transition kernel that reads
 * each env's parameters from a device array; with one variant this is mp_create. */
#define MP_MAX_VARIANTS 256
int mp_create_variants(const void* const* blobs, const size_t* blob_bytes, int n_variants, const uint8_t* env_variant_host,
                       int num_envs, int device, uint64_t seed, uint64_t env_index_base, uint32_t flags, mp_handle* out);

/* Reassigns envs to variants: copies `env_variant` (DEVICE pointer to num_envs bytes) into the pending assignments on
 * `stream`. An env takes its pending variant when its next episode starts (the auto-reset after LAST, or a reset), never
 * mid-episode, as the reference's ResetWrapper rebuilds its env on every reset; reset envs with a mask to switch them
 * at once. A value >= n_variants runs as variant 0. Only for engines with more than one variant. */
int mp_set_env_variants(mp_handle h, const uint8_t* env_variant, void* stream);

/* The variant set: its size and the DEVICE arrays (u8 [B]) of the variant each env's current episode runs (`active`)
 * and its next episode will run (`pending`, writable like mp_set_env_variants). Both NULL with one variant. Snapshots
 * (mp_state_save) of a multi-variant engine include both arrays and load only into an engine built from the same
 * blobs in the same order. */
int mp_env_variants(mp_handle h, int* n_variants, uint8_t** active, uint8_t** pending);

/* Replaces Lab2dWrapper.close (wrappers/base.py:82-84). */
int mp_destroy(mp_handle h);

/* Changes the per-launch flags (render outputs, diagnostics); the MP_FLAGS_CREATE_ONLY bits keep their creation values. */
int mp_set_flags(mp_handle h, uint32_t flags);

/* Caller-owned DEVICE outputs of one step, e.g. slot t of a learner's [T, B, ...] or [B, T, ...] trajectory buffer.
 * Every pointer is optional (NULL: that output is not delivered by this call). Each output is B per-env records at a
 * byte stride between env b and b + 1; inside a record the layout is that of mp_buffers. */
typedef struct mp_device_outputs {
  uint8_t* rgb;       uint64_t rgb_env_stride;        /* [B] x (u8 [P][rgb_h][rgb_w][3], dense) */
  uint8_t* world_rgb; uint64_t world_rgb_env_stride;  /* [B] x (u8 [world_h][world_w][3], dense) */
  double*  reward;    uint64_t reward_env_stride;     /* [B] x f64 [P] */
  double*  discount;  uint64_t discount_env_stride;   /* [B] x f64 */
  int64_t* step_type; uint64_t step_type_env_stride;  /* [B] x i64 */
  double*  scalar_obs; uint64_t scalar_obs_env_stride, scalar_obs_stride; /* [n_scalar] x [B] x f64 [P] */
} mp_device_outputs;

/* State transition only / rendering only (a step request of mp_run with only `actions` == mp_step_state + mp_render). */
int mp_step_state(mp_handle h, const int32_t* actions, void* stream);
int mp_render(mp_handle h, void* stream);

/* Replaces Lab2dWrapper.observation / *_spec (wrappers/base.py:38-80): where the outputs live. */
int mp_get_buffers(mp_handle h, mp_buffers* out);

/* Host-buffer convenience used for the end-to-end metric: copies `actions_host` (int32 [B][P],
 * ideally pinned) to the device, steps, renders, copies the requested outputs into the given
 * HOST buffers (any may be NULL to skip) and synchronises `stream`. */
typedef struct mp_host_outputs {
  uint8_t* rgb;
  uint8_t* world_rgb;
  double* reward;
  double* discount;
  int64_t* step_type;
  double* scalar_obs;
  void* scalar_block; /* if non-NULL: receives mp_buffers.scalar_block (scalar_block_bytes bytes) in one transfer and the
                         four scalar pointers above are ignored */
  int32_t* events;      /* i32 [B][max_events][3], or NULL */
  int32_t* event_count; /* i32 [B], or NULL */
} mp_host_outputs;
int mp_step_host(mp_handle h, const int32_t* actions_host, const mp_host_outputs* out, void* stream);
int mp_reset_host(mp_handle h, const mp_host_outputs* out, void* stream);

/* Pipelined form of mp_step_host for host consumers that alternate two output buffer sets (the usual double-buffered
 * actor loop): enqueues H2D(actions) -> state transition -> rendering on `stream` and the device->host copies of
 * the step's outputs on an internal copy stream, then returns WITHOUT synchronising. `slot` (0 or 1) names the
 * device-side image / scalar staging set used; consecutive calls alternate slots, so step t+1's kernels run while
 * step t's observations are still crossing PCIe. mp_wait(h, slot) blocks until the outputs of the last call on
 * that slot are complete in the host buffers. `actions_host` and `out`'s buffers must stay untouched from the call
 * until mp_wait on the same slot returns. Steps are still applied in call order (one state per env). A call refused
 * with an error (e.g. `out` names events, which are not staged per slot) enqueues nothing and steps no env.
 * Slot 0 renders into the engine's own images (mp_buffers.rgb / world_rgb); every other call that renders there
 * (mp_run when neither `out` nor `players` takes a rendered image, mp_render, mp_step_host, mp_reset_host,
 * mp_state_load) first waits, on its stream, for slot 0's copy-out, so it may be issued before
 * mp_wait(h, 0). Slot 1 renders into a set of its own, as mp_run does into a dense `out`: after a slot-1 call,
 * mp_buffers holds that step's scalars and state, and the images of the last render into the engine's own set. */
int mp_step_host_async(mp_handle h, const int32_t* actions_host, const mp_host_outputs* out, int slot, void* stream);
int mp_wait(mp_handle h, int slot);

/* Stacked timestep across GPUs (SURVEY.md section 8e: the path's only exchange). Envs shard over ranks with no
 * data-path collective; what every rank needs back is ONE stacked [world * B] tensor of reward / discount / step type.
 * Instead of a collective kernel per step, the kernel that follows a state transition in the stream (the renderer,
 * in its prologue; a small delivery kernel when no render follows) writes this rank's rows straight into every
 * rank's `gathered` buffer through NVLink peer mappings (P + 2 remote stores per env and rank, hidden behind the
 * rendering), with no fence on any hot kernel. mp_exchange_wait is the collective point: every rank enqueues it after
 * its step; its one-warp kernel (which fits beside the persistent renderer) first tells the other ranks that this
 * rank's rows are complete -- true by the kernel boundary -- and then waits for theirs. Read mp_buffers.gathered after it.
 *   mp_exchange_create   allocates this rank's exchange block: 256 bytes of per-rank flags followed by `gathered`
 *                        (one allocation, so one IPC handle shares it); returns its device pointer and size;
 *   mp_ipc_export/open   turn a device pointer into a 64-byte CUDA IPC handle + offset inside the driver allocation
 *                        and back (one process per GPU: exchange handle and offset through torch.distributed);
 *   mp_enable_peer_access for ranks that live in ONE process (tests): plain cudaDeviceEnablePeerAccess;
 *   mp_exchange_connect  takes, in rank order, every rank's block as mapped into this process (its own entry = the
 *                        pointer mp_exchange_create returned); from then on every mp_run / mp_step_state
 *                        publishes. All ranks must issue the same sequence of steps and resets (the slot
 *                        is the parity of the launch sequence number);
 *   mp_exchange_wait     enqueues on `stream` (ordered after the step's kernels) the publish-and-wait of the most recent step;
 *                        every rank must call it once per step;
 *   mp_exchange_slot     which half of `gathered` the most recent step was written to (and its sequence number). */
int mp_exchange_create(mp_handle h, int rank, int world, void** block, uint64_t* block_bytes);
int mp_ipc_export(const void* device_ptr, void* handle64, uint64_t* offset);
int mp_ipc_open(int device, const void* handle64, uint64_t offset, void** device_ptr);
int mp_enable_peer_access(int device, int peer_device);
int mp_exchange_connect(mp_handle h, void* const* peer_blocks);
int mp_exchange_wait(mp_handle h, void* stream);
int mp_exchange_slot(mp_handle h, int* slot, uint64_t* step);

/* Stacked OBSERVATIONS across GPUs -- the all-gather BASELINE.json's north_star names ("an NCCL all-gather over NVLink
 * only to return a single stacked observation tensor"), fused into the renderer: with gathering on, k_render hands
 * every finished strip in its shared-memory staging buffer to one TMA bulk store per rank (cp.async.bulk over NVLink
 * peer mappings) in addition to the local one, so the pixels are composed once and travel while the next strips are
 * being drawn -- no collective kernel, no second pass over HBM. NVLink-bound by construction: every rank receives
 * (world - 1) x its own observation bytes per step. Same create / IPC / connect / wait / slot protocol as mp_exchange_*;
 * mp_gather_obs_enable switches the extra stores on and off (they start on after connect). */
int mp_gather_obs_create(mp_handle h, int rank, int world, void** block, uint64_t* block_bytes);
int mp_gather_obs_connect(mp_handle h, void* const* peer_blocks);
int mp_gather_obs_enable(mp_handle h, int on);
int mp_gather_obs_wait(mp_handle h, void* stream);
int mp_gather_obs_slot(mp_handle h, int* slot, uint64_t* step);

/* Number of kernels this engine has launched since creation (all streams). */
int mp_launch_count(mp_handle h, uint64_t* out);

/* Algorithmic bytes one env-step moves (SURVEY.md section 8d formula), for roofline reports. */
int mp_algorithmic_bytes(mp_handle h, uint64_t* per_env_step, uint64_t* render_per_env_step);

/* Snapshot / restore of every env instance (SURVEY.md section 8f, row N4). The reference has no counterpart
 * (a dmlab2d env cannot be cloned); here the state is a handful of SoA arrays and the random numbers are
 * addressed by (key, frame), where each env's Philox key is per-env state (seed + env_index_base + b at creation),
 * so a byte copy is a complete checkpoint. A snapshot is an opaque string of
 * mp_state_size() bytes in host memory, valid for an engine created from the same blob with the same num_envs,
 * seed and env_index_base: the header records the env count, payload size, RNG key and a hash of the blob, and
 * mp_state_load rejects (MP_E_INVALID) a buffer whose `nbytes` or header does not match this engine.
 * mp_state_load re-renders the observations; both calls synchronise `stream`. */
int mp_state_size(mp_handle h, uint64_t* bytes);
int mp_state_save(mp_handle h, void* host_dst, void* stream);
int mp_state_load(mp_handle h, const void* host_src, uint64_t nbytes, void* stream);

/* Per-env state bank on the device: single envs are stored into rows of a caller-owned bank and restored from them,
 * without a round trip through host memory. A record holds one env's state rows, its timestep and its RNG key, so an
 * env restored from another env's record is that env's twin (a clone: store, then restore into other envs). Every size
 * in a record follows from the blob, so a record restores into any engine built from the same blob (or the same ordered
 * variant set), whatever its num_envs, seed, env_index_base or device. Images are not stored; a restore re-renders.
 *
 * mp_state_record_bytes: bytes of one record (a multiple of 16) and the 16-byte tag every record of this engine starts
 * with (either pointer may be NULL). */
int mp_state_record_bytes(mp_handle h, uint64_t* bytes, uint8_t tag[16]);

/* Bank row k (k < n_slots) receives env env_of_slot[k] when 0 <= env_of_slot[k] < B; otherwise row k is left untouched.
 * env_of_slot: DEVICE i32 [n_slots]. bank: DEVICE, n_slots * record_bytes, 16-byte aligned, inside one allocation on the
 * engine's device and outside the engine's own buffers. Asynchronous on `stream`; one kernel. */
int mp_state_store(mp_handle h, const int32_t* env_of_slot, int n_slots, void* bank, void* stream);

/* Env b receives bank row slot_of_env[b] when 0 <= slot_of_env[b] < n_slots and that row's tag is this engine's;
 * otherwise env b is left untouched. Then the batch is re-rendered (as mp_state_load does). A restored env's timestep
 * (reward, discount, step type, scalar observations, events), images and variant are those of the stored env at store
 * time: if that step was LAST, its next step starts a new episode. The key is state, so resets keep it.
 * flags: MP_RESTORE_REKEY = restored envs take their own key (seed + env_index_base + b) instead of the record's.
 * slot_of_env: DEVICE i32 [B]. Asynchronous on `stream`; one kernel plus what mp_render launches. Refused
 * (MP_E_UNSUPPORTED) once mp_exchange_connect or mp_gather_obs_connect has run: the peers' stacked rows would go stale.
 * Both calls check their arguments before anything is enqueued; a refused call touches nothing. */
#define MP_RESTORE_REKEY 1u
int mp_state_restore(mp_handle h, const int32_t* slot_of_env, const void* bank, int n_slots, uint32_t flags, void* stream);

/* Caller-owned DEVICE rows of a step's per-player outputs: player p of env b is delivered to row row_of_player[b][p]
 * when 0 <= row < n_rows, and to no row otherwise. A learner lays rows out as it consumes them, e.g. one contiguous block
 * per policy of a population, focal players apart from background players, or unread players left out. Every target
 * pointer is optional (NULL: not delivered per player). Strides in bytes.
 * WORLD.RGB is routed per env the same way: env b's image goes to row world_row_of_env[b] of world_rgb when
 * 0 <= row < world_n_rows, and is not rendered otherwise, e.g. for the few envs of a video. A zeroed tail (world_rgb and
 * world_row_of_env NULL) leaves WORLD.RGB per env.
 * Row segments send ranges of rows to targets of their own, e.g. one [T_g, n_g, ...] trajectory buffer per group of a
 * population: with n_segments > 0 (up to MP_MAX_ROW_SEGMENTS) the top-level rgb, reward and scalar_obs stay NULL and row
 * r with segments[s].row_begin <= r < segments[s].row_end goes to segment s, at target + (r - row_begin) * row_stride
 * of each of its outputs. Segments are sorted, disjoint, non-empty and inside [0, n_rows), and each carries the same set
 * of outputs. A row in no segment is treated as a player without a row: it is neither composited nor stored and gets
 * no scalars. A zeroed tail (n_segments 0) delivers every row to the top-level targets. */
#define MP_MAX_ROW_SEGMENTS 16
typedef struct mp_row_segment {
  int32_t row_begin, row_end;                          /* rows [row_begin, row_end) of the row map */
  uint8_t* rgb;        uint64_t rgb_row_stride;        /* [row_end - row_begin] x u8 [rgb_h][rgb_w][3], dense inside a row */
  double*  reward;     uint64_t reward_row_stride;     /* [row_end - row_begin] x f64 */
  double*  scalar_obs; uint64_t scalar_obs_row_stride, scalar_obs_stride; /* [n_scalar] x [row_end - row_begin] x f64 */
} mp_row_segment;
typedef struct mp_player_outputs {
  const int32_t* row_of_player;  /* DEVICE i32 [B][P]: row of player p of env b; < 0 or >= n_rows = not delivered */
  int32_t n_rows;
  uint8_t* rgb;        uint64_t rgb_row_stride;        /* [n_rows] x u8 [rgb_h][rgb_w][3], dense inside a row */
  double*  reward;     uint64_t reward_row_stride;     /* [n_rows] x f64 */
  double*  scalar_obs; uint64_t scalar_obs_row_stride, scalar_obs_stride; /* [n_scalar] x [n_rows] x f64 */
  const int32_t* world_row_of_env;  /* DEVICE i32 [B]: row of env b's WORLD.RGB; < 0 or >= world_n_rows = not rendered */
  int32_t world_n_rows;
  uint8_t* world_rgb; uint64_t world_rgb_row_stride;  /* [world_n_rows] x u8 [world_h][world_w][3], dense inside a row */
  int32_t n_segments;                                  /* 0: rows go to rgb / reward / scalar_obs above */
  mp_row_segment segments[MP_MAX_ROW_SEGMENTS];
} mp_player_outputs;

/* Caller-owned DEVICE rows a step's actions are read from: player p of env b takes the action id in row
 * row_of_player[b][p] when 0 <= row < n_rows, and action 0 (NOOP in every shipped substrate) otherwise. A learner that
 * gets its observations in rows (mp_player_outputs) writes its actions into rows laid out the same way, and nothing is
 * scattered back into [B][P]. The row map may be the same tensor as mp_player_outputs.row_of_player. Stride in bytes. */
typedef struct mp_player_actions {
  const int32_t* row_of_player;  /* DEVICE i32 [B][P]; may be the same tensor as mp_player_outputs.row_of_player */
  int32_t n_rows;
  const int32_t* action; uint64_t action_row_stride;  /* [n_rows] x i32, stride in bytes */
} mp_player_actions;

/* Drawn routes: the row of each player is drawn again at every episode start, on the device, as a scenario's
 * background population is resampled at every reset. Player slot p lists n_choices[p] (0..MP_MAX_ROUTE_CHOICES)
 * choices, e.g. the bots that may fill it. In episode e of env b (Philox key k), slot p plays choice
 *   o = pick(philox4x32_10(counter {0, e, p, 6}, key k).x, n_choices[p])     (stream 6: RS_ROUTE; pick(w, n) = w * n >> 32)
 * that is, uniformly with replacement, independently per slot and episode. Like every other draw of the engine it is
 * addressed by (key, episode), so it does not depend on num_envs, env_index_base or sharding, a clone plays its source's
 * draw and MP_RESTORE_REKEY gives it its own. It is not Python's `random` stream. The row of (b, p) is then
 *   row_base[p][o] + b * rows_per_env[p][o],
 * and a slot without choices has no row. A group-major layout gives choice group g a block [start_g, start_g + B * n_g)
 * with n_g the number of slots that list g, and slot p the rows start_g + rank_g(p) + b * n_g, rank_g(p) being p's
 * position among those slots: row_base = start_g + rank_g(p), rows_per_env = n_g. The row map is WRITTEN by the call. */
#define MP_MAX_ROUTE_CHOICES 8
#define MP_MAX_ROUTE_PLAYERS 16
typedef struct mp_route_draw {
  int32_t* row_of_player; /* DEVICE i32 [B][P]: written by every call, row of player p of env b, -1 for none */
  int32_t n_rows;
  int32_t n_choices[MP_MAX_ROUTE_PLAYERS];  /* per player slot; entries >= P are ignored */
  int32_t row_base[MP_MAX_ROUTE_PLAYERS][MP_MAX_ROUTE_CHOICES];
  int32_t rows_per_env[MP_MAX_ROUTE_PLAYERS][MP_MAX_ROUTE_CHOICES];
} mp_route_draw;

/* One step or reset of the batch for mp_run. Every pointer is optional (NULL: not asked for) unless stated, and the
 * fields compose; what each one adds:
 *
 * reset, env_mask: reset = 1 replaces dmlab2d.Environment.reset (wrappers/base.py:30-32; api_factory.lua:85-102): every
 *   env, or only those with env_mask[b] != 0 (DEVICE u8 [B]), starts its next episode and its FIRST observation is
 *   rendered. reset = 0 is a step.
 * actions: a step replaces dmlab2d.Environment.step (wrappers/base.py:34-36; api_factory.lua:104-111) including the
 *   DiscreteActionWrapper table lookup (discrete_action_wrapper.py:97-100): DEVICE i32 [B][P] discrete action ids. Envs
 *   whose previous step was LAST ignore the action and start a new episode (FIRST). The step runs the state transition
 *   and renders all observations.
 * player_actions: a step's actions read from rows (mp_player_actions) instead of `actions`. With dense[b][p] the action
 *   the rule of mp_player_actions gives player p of env b, the request gives, byte for byte (outputs, events, state, keys,
 *   variant bytes) and launch for launch, what the same request with the dense actions those rows give does. An id out of
 *   range in a row is action 0, as in a dense step; a restored env and an env stepping after LAST ignore their actions.
 *   The row map and the rows are read on the device and never checked on the host. Without `players` the request is
 *   accepted while the observation gather is enabled (no image is routed).
 * slot_of_env, bank, n_slots, restore_flags: a step that restores at the same time: env b takes bank row slot_of_env[b]
 *   (slot_of_env: DEVICE i32 [B]) under mp_state_restore's rule (index in 0..n_slots-1, this engine's tag) instead of
 *   advancing, and ignores its action; the restore takes precedence over its auto-reset after LAST. Every other env
 *   steps as it would without them. The state transition does the restore in the same kernel, so the render that
 *   follows draws the restored envs with all the others: no second render, no extra launch. For an engine that is not
 *   connected, a request without `out` and `players` gives, byte for byte, what the same step without a restore followed
 *   by mp_state_restore(slot_of_env, bank, n_slots, restore_flags) gives: outputs, events, state, variants and keys; with
 *   `out` or `players`, the restored envs' timestep and images are delivered into them like any env's. restore_flags:
 *   MP_RESTORE_REKEY as for mp_state_restore. A restoring step is accepted after mp_exchange_connect /
 *   mp_gather_obs_connect and counts as a step in their sequence, so the restored envs' rows and images are published as
 *   a step's; every rank issues it wherever the others issue a step (an index of all -1 restores nothing).
 * out: the outputs go into caller-owned targets (mp_device_outputs, any subset):
 *   - the images named in `out` are stored by the renderer straight into `out` (no second pass over HBM) and the
 *     engine's own images are not written; an image `out` leaves NULL is rendered into the engine's own set as usual;
 *   - reward, discount, step type and scalar observations are written to the engine's scalar block as always (the
 *     exchange, the host paths and mp_buffers read them there) and also delivered into `out` by the kernel that follows
 *     the state transition, so `out` adds no launch (with rendering off and no exchange connected, the rows travel by
 *     device-to-device copies on `stream`);
 *   - afterwards mp_buffers holds that step's state and scalars, plus the images of the last render into the engine's
 *     own set (as after a slot-1 mp_step_host_async call).
 * players: the per-player outputs also go to rows (mp_player_outputs):
 *   - images: when players->rgb is set, player p of env b is drawn straight into players->rgb + row * rgb_row_stride,
 *     and the engine's own rgb is written for no player. A player without a row is neither composited nor stored, so
 *     leaving unread players out saves their share of the render. Without players->rgb the images go to `out` or the
 *     engine's own set, as without `players`;
 *   - reward and scalar observations of a routed player are written to its row as well; the engine's scalar block is
 *     still written in full, so mp_buffers, the exchange and the host paths see every player;
 *   - WORLD.RGB: when players->world_rgb is set, env b's image is drawn straight into players->world_rgb + row *
 *     world_rgb_row_stride, row = world_row_of_env[b]; an env without a row is neither composited nor stored, and the
 *     engine's own world_rgb is written for no env. Without players->world_rgb, WORLD.RGB stays per env;
 *   - discount and step type stay per env: they and any WORLD.RGB not routed go to `out` or the engine's buffers;
 *   - restored envs are routed like any other.
 *   For every routed player and every env with a world row the request gives, byte for byte, what the same request
 *   without `players` gives at (b, p) and for env b's WORLD.RGB. Two players routed to one row, or two envs to one world
 *   row, are the caller's error: the row then holds one of them, unspecified which. The row maps are read on the device
 *   and never checked on the host (that would synchronise); nothing outside [0, n_rows) or [0, world_n_rows) is written.
 *   The exchange (mp_exchange_*) works unchanged. Refused with MP_E_UNSUPPORTED while the observation gather
 *   (mp_gather_obs_*) is connected and enabled: its stacked slots stay dense and complete.
 * draw: drawn routes (mp_route_draw), with `players` and, on a step, `player_actions`. After every request,
 *   row_of_player[b][p] is the row the draw's rule gives for the episode env b is in then, for every env: one that
 *   stepped, started an episode (auto-reset, or reset), was masked out of a reset, was restored (a record's key and
 *   episode, or its own key with MP_RESTORE_REKEY) or switched variant. On a step, player p takes the action id in row
 *   row_of_player[b][p] of player_actions->action for the episode it is in before the step, action 0 without a row; envs
 *   that start an episode or are restored ignore their actions. players and player_actions must deliver and read through
 *   the draw's row map and n_rows. For every routed (b, p) the request gives, byte for byte, what the same request
 *   without `draw` gives when handed the map as a fixed input (the map before a step for its actions, the map after it
 *   for its outputs), and it launches the same kernels, as many of them.
 *
 * Launches: a reset, and a request with `out` or `players`, launch the state transition and one render, which also
 * publishes the step to a connected exchange. A step with neither launches as mp_step_state followed by mp_render: with
 * the exchange connected, k_exchange_push follows the state transition. With rendering off, `players` with reward or
 * scalar_obs rows adds one small kernel (k_exchange_push) that delivers them. A request with row segments launches
 * exactly the kernels of the same request with one target.
 *
 * Every check runs before anything is enqueued, and a refused request (MP_E_INVALID) steps no env. Refused:
 *   - the request: a NULL handle or request; a reset with actions, player_actions, slot_of_env, bank or restore_flags; a
 *     step with env_mask; a step with both actions and player_actions, or with neither; draw without players;
 *   - player_actions: n_rows < 1; a row map not 4-byte aligned or not B * P i32 inside one device allocation on the
 *     engine's device; an action pointer or stride not a multiple of 4, or of 2 GiB or more; a stride smaller than 4;
 *     action rows not inside one device allocation on the engine's device; a row map or action rows that overlap any
 *     target, the bank, the index array or the engine's buffers (the two row maps may be one tensor, both are only read);
 *   - the restore: slot_of_env without bank or the reverse; n_slots < 1; restore_flags other than MP_RESTORE_REKEY, or
 *     any without a bank; the refusals of mp_state_restore's bank and index array; a bank or index array that overlaps a
 *     target;
 *   - out: image pointers or image env strides that are not multiples of 16 (the TMA bulk store's alignment); scalar
 *     pointers or strides that are not multiples of 8, or of 2 GiB or more; an env stride smaller than one env's bytes;
 *     scalar_obs rows (n_scalar x B rows of P doubles) that overlap, or scalar_obs on a substrate without scalar
 *     observations; an image the current render flags switch off; an output whose extent does not lie in one device
 *     allocation on the engine's device; outputs whose extents overlap each other or the engine's own buffers;
 *   - players: n_rows < 1; row_of_player not 4-byte aligned or not B * P i32 inside one device allocation on the engine's
 *     device; rgb while the render flags switch player images off, or together with out->rgb; scalar_obs on a substrate
 *     without scalar observations; rgb or its row stride not a multiple of 16 bytes; reward / scalar_obs pointers or
 *     strides not multiples of 8, or of 2 GiB or more; a row stride smaller than one row; scalar_obs rows (n_scalar x
 *     n_rows) that overlap; world_rgb without world_row_of_env or the reverse, world_n_rows < 1, world_row_of_env not
 *     4-byte aligned or not B i32 inside one device allocation on the engine's device, world_rgb or its row stride not a
 *     multiple of 16 bytes, a world row stride smaller than one WORLD.RGB image, world_rgb while the render flags switch
 *     WORLD.RGB off, or together with out->world_rgb; any target or row map that overlaps another, `out`'s targets, the
 *     bank, the index array or the engine's buffers; n_segments outside 0..MP_MAX_ROW_SEGMENTS; segments together with a
 *     top-level rgb, reward or scalar_obs; segments that are empty, unsorted, overlap or leave [0, n_rows); segments
 *     that carry different sets of outputs; and every refusal above of rgb, reward and scalar_obs, applied to each
 *     segment's targets over its own rows;
 *   - draw: draw n_rows < 1; players whose map or n_rows are not the draw's; a step whose player_actions are missing or
 *     have a map or n_rows that are not the draw's; a slot with more than MP_MAX_ROUTE_CHOICES choices (or fewer than
 *     0); a choice whose rows of some env fall outside [0, n_rows). The map must not overlap any target, the action
 *     rows, the bank, the index array or the engine's buffers. */
typedef struct mp_request {
  int32_t reset;                            /* 0: a step, 1: a reset */
  const uint8_t* env_mask;                  /* reset only: DEVICE u8 [B], NULL = every env */
  const int32_t* actions;                   /* step: DEVICE i32 [B][P]; NULL when player_actions is given */
  const mp_player_actions* player_actions;  /* step only: actions read from rows */
  const mp_route_draw* draw;                /* drawn routes; needs players */
  const int32_t* slot_of_env; const void* bank; int32_t n_slots; uint32_t restore_flags;  /* step only */
  const mp_device_outputs* out;             /* optional */
  const mp_player_outputs* players;         /* optional */
} mp_request;

/* Runs request `r` on `stream` (a cudaStream_t): see mp_request. */
int mp_run(mp_handle h, const mp_request* r, void* stream);

/* Diagnostic: how the renderer was laid out for this substrate: teams per CTA, threads per team, log2 of the pixel
 * rows per WORLD.RGB strip, shared memory bytes, atlas sprites, record stride (u16), staging bytes per warp, grid bytes,
 * then the lane -> cell dealing built for player strips and for WORLD.RGB strips (0 plain, 2 scattered colouring,
 * 1 + 16 * spare wavefronts for the default whole-cell dealing) and the cells per lane of the k_render instantiation
 * (NCP for player strips, NCW for WORLD.RGB strips). */
#define MP_RENDER_PLAN_FIELDS 12
int mp_debug_render_plan(mp_handle h, int32_t out[MP_RENDER_PLAN_FIELDS]);

/* Diagnostic: which kernels the handle's last call that launched a state transition or a render launched, -1 for a
 * part it did not launch: the family (MpbFamily) and the state-transition kernel's cell (1 if the engine has more than
 * one variant, 1 if the step restores from a bank, then 0 dense actions, 1 action rows, 2 drawn routes), then the
 * render mode (0 plain, 1 observation gather, 2 player / WORLD.RGB rows), the k_render instantiation's NCP and NCW and
 * its layout (teams per CTA, warps per team, log2 of the WORLD.RGB strip rows). A call with rendering off shows -1 from
 * the render mode on; a render alone (mp_render, mp_state_restore, mp_state_load) shows -1 up to it. */
#define MP_LAST_LAUNCH_FIELDS 10
int mp_debug_last_launch(mp_handle h, int32_t out[MP_LAST_LAUNCH_FIELDS]);

/* Diagnostic: the renderer's sprite tables. *n_total = atlas sprites including the pre-merged ones;
 * pair[n_total * n_total] = pre-merged sprite for (bottom, top) or 0; flags[n_total] bit 0 opaque,
 * bit 1 remapped per viewer. Either array may be NULL (call once for n_total, then again). */
int mp_debug_render_tables(mp_handle h, int32_t* n_total, uint8_t* pair, uint8_t* flags);

/* Debug observations of the current timestep (SURVEY.md section 8f N3), written into caller-owned DEVICE buffers (any
 * may be NULL): position i32 [B][P][2] = (x, y) of each avatar, 0-based ("{i}.POSITION", LocationObserver,
 * component_library.lua:806-855; an avatar that is off the map keeps its last cell), orientation i32 [B][P] = 0 N, 1 E,
 * 2 S, 3 W ("{i}.ORIENTATION"), layer i32 [B][P][view_h][view_w][L] = the avatar's UNROTATED view window as per-layer
 * sprite ids + 1, 0 = empty, -1 = outside a BOUNDED map ("{i}.LAYER", avatar_library.lua:247-257 with orientation 'N'),
 * zap_matrix i32 [B][P][P] = how often player row zapped player column this step (from the step's 'zap' events, as
 * clean_up.py:751-784's metric does). Off by default in the reference's configs and off the hot path here. */
int mp_debug_observations(mp_handle h, int32_t* position, int32_t* orientation, int32_t* layer, int32_t* zap_matrix, void* stream);

/* Diagnostic (needs no device): the renderer's lane -> cell dealing for a strip of `n_rows` pixel rows x `n_cells` cells
 * at a row pitch of `pitch_slots` 8-byte slots, `iters` turns per lane: out[lane] holds 6 bits per turn (63 = idle).
 * Lane l draws pixel row l % n_rows. scattered = 0: the default dealing (whole cells per lane group and turn, cell order
 * chosen to minimise bank conflicts of the 64-bit staging stores); 1: the fully conflict-free colouring (A/B flag). */
int mp_debug_lane_map(int n_rows, int n_cells, int pitch_slots, int iters, int scattered, uint32_t out[32]);

const char* mp_last_error(void);
const char* mp_version(void);

#ifdef __cplusplus
}
#endif
#endif /* MP_ENGINE_H_ */
