// dts_state.cu — snapshots of the envs' simulator state (dts_save_state / dts_load_state): the record layout that says
// where each piece of an env's state sits in its record, and the two kernels that transpose the SoA state into per-env
// records and back.
//
// A record is a list of rows, each one element of a per-env device array: a double of the dynamics, one slot of the
// delay line, one obstacle field of one map, the 128-byte RenderEp.  Element e of a row lives at base + e * size, so a
// row's elements for consecutive envs are consecutive in memory.  One CTA takes a group of kGroup envs and a chunk of
// the record (the grid's y): it stages the chunk of its envs' records in shared memory, reading each row's consecutive
// envs on one side and writing each record's consecutive words on the other, so that both sides are coalesced.
#include <algorithm>
#include <cstring>
#include <vector>

#include "dts_kernels.h"

namespace dts {

namespace {
constexpr uint64_t kLayoutVersion = 1;   // bump whenever the rows below change
constexpr int kGroup = 32;               // envs per CTA
constexpr int kChunkBytes = 1024;        // record bytes per env one CTA stages (a chunk ends at a row boundary)
constexpr int kThreads = 256;

struct Row {
  uint8_t* base;   // element of env e at base + e * size
  uint32_t off;    // byte offset in the record
  uint32_t size;   // 1, or a multiple of 4 (then off is a multiple of 4)
};
struct Chunk { int32_t row0, row1, byte0, byte1; };   // rows [row0, row1) cover record bytes [byte0, byte1)
}  // namespace

struct StateRecords {
  int n_envs = 0;
  int cap_rows = 0;
  Row* rows = nullptr;          // device [cap_rows]
  Chunk* chunks = nullptr;      // device [cap_rows]
  int n_chunks = 0;
  int stride_words = 0;         // shared-memory words per env: the largest chunk, odd
  int map_id_off = 0;           // where the record keeps its map id
  uint64_t record_bytes = 0;    // 0: no layout (its last build failed)
  uint64_t fingerprint = 0;
};

StateRecords* state_create(const dts_config& cfg) {
  StateRecords* s = new StateRecords();
  s->n_envs = cfg.num_envs;
  // RenderEp + 16 doubles + the delay line + the stream + 5 int32 + 3 uint8, and every map's obstacles at their most
  s->cap_rows = 1 + 16 + 2 * DTS_MAX_DELAY + 6 + 5 + 3 + cfg.max_maps * DTS_DYN_FIELDS * DTS_MAX_DYN;
  if (cudaMalloc(&s->rows, sizeof(Row) * s->cap_rows) != cudaSuccess ||
      cudaMalloc(&s->chunks, sizeof(Chunk) * s->cap_rows) != cudaSuccess) {
    state_destroy(s);
    return nullptr;
  }
  return s;
}

void state_destroy(StateRecords* s) {
  if (!s) return;
  if (s->rows) cudaFree(s->rows);
  if (s->chunks) cudaFree(s->chunks);
  delete s;
}

uint64_t state_record_bytes(const StateRecords& s) { return s.record_bytes; }
uint64_t state_fingerprint(const StateRecords& s) { return s.fingerprint; }

static uint64_t mix(uint64_t h, uint64_t v) {
  h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
  h = (h ^ (h >> 31)) * 0x7fb5d329728ea185ull;
  return h ^ (h >> 27);
}

std::string state_layout(StateRecords& s, const DState& S, const MapSlots& maps) {
  s.record_bytes = 0;
  const size_t n = S.n;
  std::vector<Row> rows;
  uint32_t off = 0;
  auto add = [&](void* base, uint32_t size) { rows.push_back(Row{static_cast<uint8_t*>(base), off, size}); off += size; };
  // 1. the render record first: 16-byte aligned, like its struct
  add(S.rep, sizeof(RenderEp));
  // 2. 8-byte rows: dynamics, per-step outputs, the delay line, the stream, every map's obstacles
  double* dbl[] = {S.cx, S.cy, S.ctheta, S.vu, S.vw, S.pos_x, S.pos_z, S.angle, S.speed, S.reward,
                   S.lane_dist, S.lane_dot, S.lane_angle, S.prox, S.wheel_dist, S.trim};
  for (double* p : dbl) add(p, 8);
  for (int k = 0; k < 2 * DTS_MAX_DELAY; k++) add(S.fifo + k * n, 8);
  for (int k = 0; k < 6; k++) add(S.rng + k * n, 8);
  uint64_t fp = mix(mix(mix(0, kLayoutVersion), DTS_MAX_DELAY), maps_slot_count(maps));
  for (int m = 0; m < maps_slot_count(maps); m++) {
    fp = mix(fp, maps_hash(maps, m));
    const DMap* d = maps_get(maps, m);
    if (!d || !d->n_dyn) continue;
    for (int k = 0; k < DTS_DYN_FIELDS * d->n_dyn; k++) add(d->dyn_state + k * n, 8);
  }
  // 3. 4-byte rows, then the bytes at the end, where no chunk boundary falls between them
  s.map_id_off = 0;
  int32_t* i32[] = {S.step_count, S.tile_i, S.tile_j, S.map_id, S.episode};
  for (int32_t* p : i32) {
    if (p == S.map_id) s.map_id_off = (int)off;
    add(p, 4);
  }
  uint8_t* u8[] = {S.done_code, S.in_lane, S.collided};
  for (uint8_t* p : u8) add(p, 1);
  const uint32_t bytes = (off + 15) & ~15u;
  if ((int)rows.size() > s.cap_rows) return "state layout: more rows than allocated";
  // chunks: greedy, each ends before the row that would take it past kChunkBytes, at a 4-byte boundary
  std::vector<Chunk> chunks;
  int r0 = 0;
  for (int r = 1; r <= (int)rows.size(); r++) {
    const bool end = r == (int)rows.size();
    if (!end && (rows[r].off % 4 || rows[r].off + rows[r].size - rows[r0].off <= (uint32_t)kChunkBytes)) continue;
    chunks.push_back(Chunk{r0, r, (int32_t)rows[r0].off, (int32_t)(end ? bytes : rows[r].off)});
    r0 = r;
  }
  int stride = 0;
  for (const Chunk& c : chunks) stride = std::max(stride, (c.byte1 - c.byte0) / 4);
  cudaError_t e = cudaMemcpy(s.rows, rows.data(), rows.size() * sizeof(Row), cudaMemcpyHostToDevice);
  if (e == cudaSuccess) e = cudaMemcpy(s.chunks, chunks.data(), chunks.size() * sizeof(Chunk), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return std::string("state layout upload failed: ") + cudaGetErrorString(e);
  s.n_chunks = (int)chunks.size();
  s.stride_words = stride | 1;   // odd: the envs of a group start in different banks
  s.record_bytes = bytes;
  s.fingerprint = fp;
  return "";
}

// Each warp takes one row at a time; its lanes walk the row's elements of the group's envs, consecutive in memory
__global__ void __launch_bounds__(kThreads) k_state_save(const Row* __restrict__ rows, const Chunk* __restrict__ chunks,
                                                         int n_envs, int stride, uint32_t rec_bytes, uint8_t* __restrict__ rec) {
  extern __shared__ uint32_t sm[];   // [kGroup][stride]
  const Chunk ch = chunks[blockIdx.y];
  const int e0 = blockIdx.x * kGroup;
  const int ng = min(kGroup, n_envs - e0);
  const int words = (ch.byte1 - ch.byte0) / 4;
  for (int i = threadIdx.x; i < kGroup * stride; i += kThreads) sm[i] = 0u;   // the padding and the bytes' neighbours
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = ch.row0 + warp; r < ch.row1; r += kThreads / 32) {
    const Row row = rows[r];
    const int o = (int)row.off - ch.byte0;
    if (row.size == 1) {
      if (lane < ng) reinterpret_cast<uint8_t*>(sm + lane * stride)[o] = row.base[e0 + lane];
    } else {
      const int w = (int)row.size / 4;
      const uint32_t* src = reinterpret_cast<const uint32_t*>(row.base + (size_t)e0 * row.size);
      for (int i = lane; i < ng * w; i += 32) sm[(i / w) * stride + o / 4 + i % w] = src[i];
    }
  }
  __syncthreads();
  for (int i = threadIdx.x; i < ng * words; i += kThreads) {
    const int e = i / words, w = i - e * words;
    reinterpret_cast<uint32_t*>(rec + (size_t)(e0 + e) * rec_bytes + ch.byte0)[w] = sm[e * stride + w];
  }
}

__global__ void __launch_bounds__(kThreads) k_state_load(const Row* __restrict__ rows, const Chunk* __restrict__ chunks,
                                                         int n_envs, int stride, uint32_t rec_bytes,
                                                         const uint8_t* __restrict__ rec, const uint8_t* __restrict__ mask,
                                                         const DMap* __restrict__ maps, int n_maps, int map_id_off,
                                                         int32_t* refused) {
  extern __shared__ uint32_t sm[];   // [kGroup][stride]
  __shared__ int take[kGroup];
  const Chunk ch = chunks[blockIdx.y];
  const int e0 = blockIdx.x * kGroup;
  const int ng = min(kGroup, n_envs - e0);
  const int words = (ch.byte1 - ch.byte0) / 4;
  // every CTA of the group decides alike from the record's map id, whichever chunk it holds: a record naming no
  // uploaded map is not loaded at all, so no later kernel indexes the map table with it
  if (threadIdx.x < kGroup) {
    const int e = e0 + threadIdx.x;
    int t = 0;
    if (threadIdx.x < ng && (!mask || mask[e])) {
      const int32_t mid = *reinterpret_cast<const int32_t*>(rec + (size_t)e * rec_bytes + map_id_off);
      t = mid >= 0 && mid < n_maps && maps[mid].valid;
      if (!t && blockIdx.y == 0) *reinterpret_cast<volatile int32_t*>(refused) = 1;
    }
    take[threadIdx.x] = t;
  }
  for (int i = threadIdx.x; i < ng * words; i += kThreads) {
    const int e = i / words, w = i - e * words;
    sm[e * stride + w] = reinterpret_cast<const uint32_t*>(rec + (size_t)(e0 + e) * rec_bytes + ch.byte0)[w];
  }
  __syncthreads();
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  for (int r = ch.row0 + warp; r < ch.row1; r += kThreads / 32) {
    const Row row = rows[r];
    const int o = (int)row.off - ch.byte0;
    if (row.size == 1) {
      if (lane < ng && take[lane]) row.base[e0 + lane] = reinterpret_cast<const uint8_t*>(sm + lane * stride)[o];
    } else {
      const int w = (int)row.size / 4;
      uint32_t* dst = reinterpret_cast<uint32_t*>(row.base + (size_t)e0 * row.size);
      for (int i = lane; i < ng * w; i += 32)
        if (take[i / w]) dst[i] = sm[(i / w) * stride + o / 4 + i % w];
    }
  }
}

void launch_state_save(const StateRecords& s, void* records, cudaStream_t st) {
  const dim3 grid((s.n_envs + kGroup - 1) / kGroup, s.n_chunks);
  k_state_save<<<grid, kThreads, sizeof(uint32_t) * kGroup * s.stride_words, st>>>(
      s.rows, s.chunks, s.n_envs, s.stride_words, (uint32_t)s.record_bytes, static_cast<uint8_t*>(records));
}

void launch_state_load(const StateRecords& s, const uint8_t* mask, const void* records, const DMap* maps, int n_maps,
                       int32_t* refused, cudaStream_t st) {
  const dim3 grid((s.n_envs + kGroup - 1) / kGroup, s.n_chunks);
  k_state_load<<<grid, kThreads, sizeof(uint32_t) * kGroup * s.stride_words, st>>>(
      s.rows, s.chunks, s.n_envs, s.stride_words, (uint32_t)s.record_bytes, static_cast<const uint8_t*>(records), mask,
      maps, n_maps, s.map_id_off, refused);
}

}  // namespace dts
