// family_load.h -- host side: the blob access, error reporting and host tables that the decode of engine.cu
// (build_tables, load_map) and the family loaders (`load` in each step_<family>.cuh) share, and the device upload that
// create runs on those tables once the device is checked. engine.cu is the only translation unit; it includes this
// header through the family headers.
#pragma once

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

// The Zapper component (avatar_library.lua:570-850) of the clean_up, commons_harvest and territory avatars.
struct Zapper {
  int cooldown, respawn, remove, layer, sprite, hit;  // respawn: framesTillRespawn; remove: removeHitPlayer; hit: its hit id
  double penalty, reward;
  BeamGeom geom;
};

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

// A device table decoded on the host: its bytes, and the `const T*` field of a Params, Tables or MapVariant that its
// device address goes into (upload_tables in engine.cu).
struct HostTable {
  std::vector<uint8_t> bytes;
  void* field;
};

template <typename T>
void add_table(std::vector<HostTable>& tables, const T** field, const std::vector<T>& host) {
  const uint8_t* p = reinterpret_cast<const uint8_t*>(host.data());
  tables.push_back({std::vector<uint8_t>(p, p + host.size() * sizeof(T)), field});
}

// Copies `host` into a new zero-padded device allocation (at least 16 bytes), recorded in `allocs`.
template <typename T>
int upload(std::vector<void*>& allocs, const std::vector<T>& host, const T** out) {
  void* p = nullptr;
  size_t bytes = std::max<size_t>(host.size() * sizeof(T), 16);
  CUDA_TRY(cudaMalloc(&p, bytes));
  allocs.push_back(p);
  CUDA_TRY(cudaMemset(p, 0, bytes));
  if (!host.empty()) CUDA_TRY(cudaMemcpy(p, host.data(), host.size() * sizeof(T), cudaMemcpyHostToDevice));
  *out = static_cast<const T*>(p);
  return MP_OK;
}

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

// What build_tables hands a family's loader (`load(FamilyLoad&, const Tables&, Params&)`), and what the loader hands
// back besides its Params. On entry the Tables hold the geometry and the avatar tables.
struct FamilyLoad {
  const void* blob;
  size_t n;
  Section<int32_t> hits;               // [n_hits][2] layer, sprite
  // handed back: the Tables fields the family decides
  int nA = 0, nD = 0, nW = 0, nR = 0, nR_pad = 16;  // per-env entity counts (State's array sizes, Tables::nA...)
  int end_min_frames = 0, end_interval = 0;          // StochasticIntervalEpisodeEnding
  double end_prob = 0.0;
  int beam_cells = 0;                  // footprint cells of the beams State::max_events provides for
  std::vector<std::vector<int>> hint_stacks;  // sprite stacks (bottom up) worth a pre-merged sprite before the generic enumeration
  std::vector<HostTable> tables;       // the device tables of its Params

  template <typename T>
  void table(const T** field, const std::vector<T>& host) { add_table(tables, field, host); }

  template <typename T>
  int need(const char* name, int dtype, Section<T>* out) const {
    return get_section(blob, n, name, dtype, out) ? MP_OK : fail(MP_E_INVALID, "blob: missing section '%s'", name);
  }
  // The family's parameter blocks "<prefix>_ip" (int32[n_int]) and "<prefix>_dp" (f64[n_f64]), see mpb_format.h.
  int params(const char* prefix, size_t n_int, size_t n_f64, const int32_t** ip, const double** dp) const {
    char name[16];
    Section<int32_t> si;
    Section<double> sd;
    int rc;
    snprintf(name, sizeof name, "%s_ip", prefix);
    if ((rc = need(name, MPB_I32, &si))) return rc;
    if (si.count < n_int) return fail(MP_E_INVALID, "blob: section '%s' has %zu values (expected %zu)", name, si.count, n_int);
    snprintf(name, sizeof name, "%s_dp", prefix);
    if ((rc = need(name, MPB_F64, &sd))) return rc;
    if (sd.count < n_f64) return fail(MP_E_INVALID, "blob: section '%s' has %zu values (expected %zu)", name, sd.count, n_f64);
    *ip = si.data; *dp = sd.data;
    return MP_OK;
  }
};

// The cell -> entity index of the n entities of section `name`, entity k standing on cell rows.data[k * row_len + 1]:
// [cells_pad] index or -1. Refuses a section shorter than n rows or an entity off the map, so that neither this index nor
// the kernels, which read the section's first n rows, reach past what the blob holds.
int cell_index(FamilyLoad& ld, const Tables& T, const char* name, const Section<int32_t>& rows, int n, int row_len,
               const int16_t** out) {
  if (n < 0 || rows.count < (size_t)n * row_len)
    return fail(MP_E_INVALID, "blob: section '%s' has %zu values for %d entities of %d", name, rows.count, n, row_len);
  std::vector<int16_t> of(T.cells_pad, -1);
  for (int k = 0; k < n; ++k) {
    const int cell = rows.data[k * row_len + 1];
    if (cell < 0 || cell >= T.cells) return fail(MP_E_INVALID, "blob: section '%s' puts entity %d on cell %d of a %d-cell map", name, k, cell, T.cells);
    of[cell] = (int16_t)k;
  }
  ld.table(out, of);
  return MP_OK;
}

// Per-env variants (mp_create_variants): each variant runs under its own Params, and a family's same_shape(a, b) checks,
// field by field, that two Params agree on what the kernels read from params[0] (what stage() puts in shared memory) or
// what shapes per-env state. Every other field is the variant's own: its scalar knobs, and its table pointers, which
// point at the same bytes wherever the variants' tables agree. MP_SAME compares one field's bytes (Params are
// value-initialised, so padding and unused array entries are zero) and names it when they differ.
#define MP_SAME(field)                                                                                                  \
  if (memcmp(&a.field, &b.field, sizeof(a.field)) != 0)                                                               \
    return fail(MP_E_UNSUPPORTED, "Params field '%s' differs (variants may differ only in the family's scalar knobs)", #field);

#define MP_SAME_ZAPPER MP_SAME(zap.layer) MP_SAME(zap.sprite) MP_SAME(zap.hit) MP_SAME(zap.geom)

// The Zapper and episode-ending slots (MPB_FP_*) of clean_up, commons_harvest and territory. The penalty and reward sit
// in each family's own f64 slots.
int load_zapper(FamilyLoad& ld, const Tables& T, const int32_t* ip, double penalty, double reward, Zapper& z) {
  z.cooldown = ip[MPB_FP_ZAP_COOLDOWN]; z.respawn = ip[MPB_FP_ZAP_RESPAWN]; z.remove = ip[MPB_FP_ZAP_REMOVE];
  z.layer = ip[MPB_FP_ZAP_LAYER]; z.sprite = ip[MPB_FP_ZAP_SPRITE];
  z.hit = 0;
  for (int h = 0; h < (int)ld.hits.count / 2; ++h) if (ld.hits.data[h * 2] == z.layer) z.hit = h;
  z.penalty = penalty; z.reward = reward;
  const int length = ip[MPB_FP_ZAP_LENGTH], radius = ip[MPB_FP_ZAP_RADIUS];
  if (z.cooldown <= 0) return fail(MP_E_UNSUPPORTED, "non-positive zap cooldown");
  if (!make_beam_geom(length, radius, &z.geom)) return fail(MP_E_UNSUPPORTED, "beam footprint larger than %d cells", MP_MAX_BEAM_CELLS);
  if (!beam_fits_torus(T, length, radius)) return fail(MP_E_UNSUPPORTED, "zap beam (length %d, radius %d) does not fit the %dx%d TORUS map", length, radius, T.W, T.H);
  ld.end_min_frames = ip[MPB_FP_END_MIN_FRAMES]; ld.end_interval = ip[MPB_FP_END_INTERVAL];
  if (ld.end_interval < 1) return fail(MP_E_INVALID, "episode interval < 1");
  return MP_OK;
}

}  // namespace
