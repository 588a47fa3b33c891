// state_bank.cuh -- per-env records of the engine state in a caller-owned device bank (mp_state_store /
// mp_state_restore, include/mp_engine.h).
//
// A record is one env's row of every state array plus its RNG key and variant bytes, at offsets engine.cu decides
// (layout_state, the one list of per-env state arrays, from which snapshots are derived too). The two kernels only
// gather: every destination (a bank row for a store, an env for a restore) is written by one warp that reads exactly one
// source, so no two threads ever write the same bytes, whatever indices the caller passes (a fan-out of one record to many envs included). Indices out of range
// and records whose tag is not this engine's are skipped in-kernel; they can neither fault nor write anything.
// The same per-warp restore (restore_env) also runs inside a step (k_step<..., kRestore>, step_common.cuh): the warp of a named
// env copies the record instead of advancing it, and the render that follows draws it with every other env.
#pragma once

#include "common.cuh"

#define MP_RECORD_MAX_ROWS 32

struct RecordRow {
  uint8_t* base;        // env b's row starts at base + b * env_stride; null: none in this engine (stored as zeros)
  uint64_t env_stride;  // bytes
  uint32_t bytes;       // row length
  uint32_t offset;      // where the row sits inside a record
};

struct RecordLayout {
  uint4 tag;              // a record's first 16 bytes
  uint64_t record_bytes;  // a multiple of 16
  int n_rows;
  int key_row;            // the row of the RNG key (mp_state_restore's MP_RESTORE_REKEY replaces it)
  RecordRow row[MP_RECORD_MAX_ROWS];
};

// One warp copies `bytes` bytes with the widest access that the two addresses and the length allow (16 B for the grid
// and the padded entity rows, 8 B for the rows of doubles, ...). src == null writes zeros.
__device__ __forceinline__ void copy_row(uint8_t* dst, const uint8_t* src, uint32_t bytes, int lane) {
  const uintptr_t a = (uintptr_t)dst | (uintptr_t)src | bytes;
  if ((a & 15) == 0) {
    for (uint32_t i = lane * 16; i < bytes; i += 32 * 16)
      *reinterpret_cast<uint4*>(dst + i) = src ? *reinterpret_cast<const uint4*>(src + i) : make_uint4(0, 0, 0, 0);
  } else if ((a & 7) == 0) {
    for (uint32_t i = lane * 8; i < bytes; i += 32 * 8)
      *reinterpret_cast<uint64_t*>(dst + i) = src ? *reinterpret_cast<const uint64_t*>(src + i) : 0ull;
  } else if ((a & 3) == 0) {
    for (uint32_t i = lane * 4; i < bytes; i += 32 * 4)
      *reinterpret_cast<uint32_t*>(dst + i) = src ? *reinterpret_cast<const uint32_t*>(src + i) : 0u;
  } else {
    for (uint32_t i = lane; i < bytes; i += 32) dst[i] = src ? src[i] : 0;
  }
}

// One warp per bank row k: row k receives env env_of_slot[k] when that is in 0..B-1.
__global__ void __launch_bounds__(256) k_state_store(const __grid_constant__ RecordLayout R, const int32_t* __restrict__ env_of_slot,
                                                     int n_slots, int B, uint8_t* __restrict__ bank) {
  const int k = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (k >= n_slots) return;
  const int e = env_of_slot[k];
  if (e < 0 || e >= B) return;
  uint8_t* rec = bank + (size_t)k * R.record_bytes;
  if (lane == 0) *reinterpret_cast<uint4*>(rec) = R.tag;
  for (int r = 0; r < R.n_rows; ++r) {
    const RecordRow& w = R.row[r];
    copy_row(rec + w.offset, w.base ? w.base + (size_t)e * w.env_stride : nullptr, w.bytes, lane);
  }
}

// Called by every lane of the warp that owns env b: env b receives bank row slot_of_env[b] when that is in
// 0..n_slots-1 and carries this engine's tag. rekey: the key row becomes key_base + b instead of the record's key.
// Returns whether the env was restored (the same on every lane).
__device__ __forceinline__ bool restore_env(const RecordLayout& R, const int32_t* __restrict__ slot_of_env, const uint8_t* __restrict__ bank,
                                            int n_slots, int b, int lane, int rekey, uint64_t key_base) {
  const int s = slot_of_env[b];
  if (s < 0 || s >= n_slots) return false;
  const uint8_t* rec = bank + (size_t)s * R.record_bytes;
  const uint4 t = *reinterpret_cast<const uint4*>(rec);
  if (t.x != R.tag.x || t.y != R.tag.y || t.z != R.tag.z || t.w != R.tag.w) return false;
  for (int r = 0; r < R.n_rows; ++r) {
    const RecordRow& w = R.row[r];
    if (!w.base) continue;
    uint8_t* dst = w.base + (size_t)b * w.env_stride;
    if (r == R.key_row && rekey) {
      if (lane == 0) *reinterpret_cast<uint64_t*>(dst) = key_base + (uint64_t)b;
      continue;
    }
    copy_row(dst, rec + w.offset, w.bytes, lane);
  }
  return true;
}

// One warp per env b (restore_env).
__global__ void __launch_bounds__(256) k_state_restore(const __grid_constant__ RecordLayout R, const int32_t* __restrict__ slot_of_env,
                                                       const uint8_t* __restrict__ bank, int n_slots, int B, int rekey, uint64_t key_base) {
  const int b = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
  if (b >= B) return;
  restore_env(R, slot_of_env, bank, n_slots, b, lane, rekey, key_base);
}

// The restore a step carries out in place of advancing the envs it names (a restoring mp_run, k_step<..., true>): the
// engine's record layout (a device copy made at mp_create, so the step's parameter space grows by one pointer, not a
// whole RecordLayout) and the call's index array, bank and rekey flag.
struct StepRestore {
  const RecordLayout* layout;
  const int32_t* slot_of_env;  // [B]
  const uint8_t* bank;
  int n_slots;
  int rekey;
  uint64_t key_base;
};
