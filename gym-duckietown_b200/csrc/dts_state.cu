// dts_state.cu — the envs' simulator state (EnvState): the per-env device arrays of DState, the staging buffers of
// dts_reset, and snapshots of the state (dts_save_state / dts_load_state): the record layout that says where each piece
// of an env's state sits in its record, and the two kernels that transpose the SoA state into per-env records and back.
//
// kStateArrays below is the single statement of what an env's state is: it allocates the DState arrays, gives the rows
// of a record and their order, and sizes the row table.  A compile-time check holds it to DState's members, so an array
// cannot be allocated without also being saved and loaded.
//
// A record is a list of rows, each one element of a per-env device array: a double of the dynamics, one slot of the
// delay line, one obstacle field of one map, the 144-byte RenderEp.  Element e of a row lives at base + e * size, so a
// row's elements for consecutive envs are consecutive in memory.  One CTA takes a group of kGroup envs and a chunk of
// the record (the grid's y): it stages the chunk of its envs' records in shared memory, reading each row's consecutive
// envs on one side and writing each record's consecutive words on the other, so that both sides are coalesced.
#include <algorithm>
#include <cstddef>
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

// One per-env array of DState: `planes` consecutive num_envs-long planes of `size`-byte elements, one row each
struct StateArray { size_t member; uint32_t size, planes; };
#define DTS_STATE_ARRAY(m, planes) StateArray{offsetof(DState, m), (uint32_t)sizeof(*DState{}.m), planes}
// Every per-env array, in the order of its rows in a record (DESIGN.md §2): the RenderEp first, 16-byte aligned like
// its struct; the 8-byte rows, after the last of which every map's obstacles go; the 4-byte rows; the bytes at the end,
// where no chunk boundary falls between them.
constexpr StateArray kStateArrays[] = {
    DTS_STATE_ARRAY(rep, 1),
    DTS_STATE_ARRAY(cx, 1), DTS_STATE_ARRAY(cy, 1), DTS_STATE_ARRAY(ctheta, 1), DTS_STATE_ARRAY(vu, 1),
    DTS_STATE_ARRAY(vw, 1), DTS_STATE_ARRAY(pos_x, 1), DTS_STATE_ARRAY(pos_z, 1), DTS_STATE_ARRAY(angle, 1),
    DTS_STATE_ARRAY(speed, 1), DTS_STATE_ARRAY(reward, 1), DTS_STATE_ARRAY(lane_dist, 1), DTS_STATE_ARRAY(lane_dot, 1),
    DTS_STATE_ARRAY(lane_angle, 1), DTS_STATE_ARRAY(prox, 1), DTS_STATE_ARRAY(wheel_dist, 1), DTS_STATE_ARRAY(trim, 1),
    DTS_STATE_ARRAY(fifo, 2 * DTS_MAX_DELAY), DTS_STATE_ARRAY(rng, 6),
    DTS_STATE_ARRAY(step_count, 1), DTS_STATE_ARRAY(tile_i, 1), DTS_STATE_ARRAY(tile_j, 1), DTS_STATE_ARRAY(map_id, 1),
    DTS_STATE_ARRAY(episode, 1),
    DTS_STATE_ARRAY(done_code, 1), DTS_STATE_ARRAY(in_lane, 1), DTS_STATE_ARRAY(collided, 1)};
#undef DTS_STATE_ARRAY
constexpr int kNumArrays = sizeof(kStateArrays) / sizeof(kStateArrays[0]);

// DState is its int32 n followed by pointers only: the table names each pointer slot once
constexpr bool covers_dstate() {
  if (offsetof(DState, n) != 0 || kNumArrays != (int)(sizeof(DState) / sizeof(void*)) - 1) return false;
  for (int i = 0; i < kNumArrays; i++) {
    const size_t m = kStateArrays[i].member;
    if (m < sizeof(void*) || m >= sizeof(DState) || m % sizeof(void*)) return false;
    for (int j = 0; j < i; j++)
      if (kStateArrays[j].member == m) return false;
  }
  return true;
}
static_assert(covers_dstate(), "kStateArrays must list every pointer member of DState exactly once");
// Element sizes never grow down the table, so every row lands aligned to its size; the kernels move 1 or 4k bytes
constexpr bool sizes_in_order() {
  for (int i = 0; i < kNumArrays; i++) {
    const uint32_t z = kStateArrays[i].size;
    if ((z != 1 && z % 4) || (i && z > kStateArrays[i - 1].size)) return false;
  }
  return true;
}
static_assert(sizes_in_order(), "kStateArrays must run by non-increasing element size, each 1 or a multiple of 4");
constexpr int last_8byte_array() {
  int r = -1;
  for (int i = 0; i < kNumArrays; i++)
    if (kStateArrays[i].size == 8) r = i;
  return r;
}
constexpr int kObstaclesAfter = last_8byte_array();   // the obstacles' rows follow this entry's
static_assert(kObstaclesAfter >= 0, "the obstacles' 8-byte rows follow the last 8-byte array");
constexpr int state_rows() {
  int r = 0;
  for (const StateArray& a : kStateArrays) r += a.planes;
  return r;
}

// One member of dts_episode_params: its element size and elements per env, which size its staging buffer
struct EpisodeField { size_t member; uint32_t size, width; };
#define DTS_EPISODE_FIELD(m, width) \
  EpisodeField{offsetof(dts_episode_params, m), (uint32_t)sizeof(*dts_episode_params{}.m), width}
constexpr EpisodeField kEpisodeFields[] = {
    DTS_EPISODE_FIELD(map_id, 1), DTS_EPISODE_FIELD(pos_x, 1), DTS_EPISODE_FIELD(pos_z, 1), DTS_EPISODE_FIELD(angle, 1),
    DTS_EPISODE_FIELD(wheel_dist, 1), DTS_EPISODE_FIELD(trim, 1), DTS_EPISODE_FIELD(cam_height, 1),
    DTS_EPISODE_FIELD(cam_angle_deg, 1), DTS_EPISODE_FIELD(cam_fov_y_deg, 1), DTS_EPISODE_FIELD(cam_noise, 3),
    DTS_EPISODE_FIELD(horizon_color, 3), DTS_EPISODE_FIELD(light_ambient, 3), DTS_EPISODE_FIELD(light_diffuse, 3),
    DTS_EPISODE_FIELD(light_pos, 4), DTS_EPISODE_FIELD(light_stale, 1), DTS_EPISODE_FIELD(ground_color, 3),
    DTS_EPISODE_FIELD(obj_hidden, 8)};
#undef DTS_EPISODE_FIELD
constexpr int kNumEpisodeFields = sizeof(kEpisodeFields) / sizeof(kEpisodeFields[0]);
constexpr bool covers_episode_params() {
  if (kNumEpisodeFields * sizeof(void*) != sizeof(dts_episode_params)) return false;
  for (int i = 0; i < kNumEpisodeFields; i++)
    if (kEpisodeFields[i].member != i * sizeof(void*)) return false;
  return true;
}
static_assert(covers_episode_params(), "kEpisodeFields must list every member of dts_episode_params, in its order");

// The pointer member at byte offset `member` of a struct of pointers (DState, dts_episode_params)
template <typename T> void* get_member(const T& t, size_t member) {
  void* p;
  memcpy(&p, reinterpret_cast<const char*>(&t) + member, sizeof p);
  return p;
}
template <typename T> void set_member(T& t, size_t member, const void* p) {
  memcpy(reinterpret_cast<char*>(&t) + member, &p, sizeof p);
}
}  // namespace

struct EnvState {
  DState S{};
  std::vector<void*> allocs;                 // the arrays of S and the staging buffers
  void* stage[kNumEpisodeFields] = {};       // dts_reset's device copies of the episode parameters
  bool seeded = false;
  // the snapshot record layout
  int cap_rows = 0;
  Row* rows = nullptr;          // device [cap_rows]
  Chunk* chunks = nullptr;      // device [cap_rows]
  int n_chunks = 0;
  int stride_words = 0;         // shared-memory words per env: the largest chunk, odd
  int map_id_off = 0;           // where the record keeps its map id
  uint64_t record_bytes = 0;    // 0: no layout (its last build failed)
  uint64_t fingerprint = 0;
};

// `bytes` of zeroed device memory, and 16 more past them, owned by `s`
static std::string alloc_zeroed(EnvState& s, void** p, size_t bytes) {
  const cudaError_t e = cudaMalloc(p, bytes + 16);
  if (e != cudaSuccess) return "cudaMalloc(" + std::to_string(bytes) + " B) failed: " + cudaGetErrorString(e);
  cudaMemset(*p, 0, bytes + 16);
  s.allocs.push_back(*p);
  return "";
}

EnvState* state_create(const dts_config& cfg, const MapSlots& maps, std::string& err) {
  EnvState* s = new EnvState();
  const size_t n = cfg.num_envs;
  s->S.n = cfg.num_envs;
  err.clear();
  for (int k = 0; k < kNumArrays && err.empty(); k++) {
    const StateArray& a = kStateArrays[k];
    void* p = nullptr;
    err = alloc_zeroed(*s, &p, a.planes * a.size * n);
    set_member(s->S, a.member, p);
  }
  for (int k = 0; k < kNumEpisodeFields && err.empty(); k++)
    err = alloc_zeroed(*s, &s->stage[k], kEpisodeFields[k].width * kEpisodeFields[k].size * n);
  // the per-env arrays' rows, and every map's obstacles at their most
  s->cap_rows = state_rows() + cfg.max_maps * DTS_DYN_FIELDS * DTS_MAX_DYN;
  if (err.empty() && (cudaMalloc(&s->rows, sizeof(Row) * s->cap_rows) != cudaSuccess ||
                      cudaMalloc(&s->chunks, sizeof(Chunk) * s->cap_rows) != cudaSuccess))
    err = "cudaMalloc(state record layout) failed";
  if (err.empty()) err = state_layout(*s, maps);
  if (!err.empty()) {
    state_destroy(s);
    return nullptr;
  }
  return s;
}

void state_destroy(EnvState* s) {
  if (!s) return;
  for (void* p : s->allocs) cudaFree(p);
  if (s->rows) cudaFree(s->rows);
  if (s->chunks) cudaFree(s->chunks);
  delete s;
}

const DState& state_arrays(const EnvState& s) { return s.S; }

dts_state_view state_view(const EnvState& s) {
  const DState& S = s.S;
  return dts_state_view{S.pos_x, S.pos_z, S.angle, S.speed, S.reward, S.lane_dist, S.lane_dot, S.lane_angle, S.prox,
                        S.wheel_dist, S.step_count, S.tile_i, S.tile_j, S.map_id, S.episode, S.done_code, S.in_lane,
                        S.collided};
}

bool state_seeded(const EnvState& s) { return s.seeded; }

std::string state_seed_streams(EnvState& s, const uint8_t* mask_host, const uint64_t* streams) {
  const size_t n = s.S.n;
  std::vector<uint64_t> soa(6 * n);   // the device's [6][N]: the masked-out envs keep theirs
  cudaError_t e = cudaMemcpy(soa.data(), s.S.rng, 6 * n * sizeof(uint64_t), cudaMemcpyDeviceToHost);
  for (size_t i = 0; i < n; i++) {
    if (mask_host && !mask_host[i]) continue;
    for (int k = 0; k < 6; k++) soa[k * n + i] = streams[6 * i + k];
  }
  if (e == cudaSuccess) e = cudaMemcpy(s.S.rng, soa.data(), 6 * n * sizeof(uint64_t), cudaMemcpyHostToDevice);
  if (e != cudaSuccess) return std::string("stream upload failed: ") + cudaGetErrorString(e);
  s.seeded = true;
  return "";
}

std::string state_read_streams(const EnvState& s, uint64_t* out) {
  const size_t n = s.S.n;
  std::vector<uint64_t> soa(6 * n);
  const cudaError_t e = cudaMemcpy(soa.data(), s.S.rng, 6 * n * sizeof(uint64_t), cudaMemcpyDeviceToHost);
  if (e != cudaSuccess) return std::string("stream download failed: ") + cudaGetErrorString(e);
  for (size_t i = 0; i < n; i++)
    for (int k = 0; k < 6; k++) out[6 * i + k] = soa[k * n + i];
  return "";
}

std::string state_stage(EnvState& s, const dts_episode_params& host, dts_episode_params& dev, cudaStream_t st) {
  dev = dts_episode_params{};
  for (int k = 0; k < kNumEpisodeFields; k++) {
    const EpisodeField& f = kEpisodeFields[k];
    const void* src = get_member(host, f.member);
    if (!src) continue;
    const size_t bytes = (size_t)f.width * f.size * s.S.n;
    const cudaError_t e = cudaMemcpyAsync(s.stage[k], src, bytes, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) return std::string("episode parameter staging failed: ") + cudaGetErrorString(e);
    set_member(dev, f.member, s.stage[k]);
  }
  return "";
}

uint64_t state_record_bytes(const EnvState& s) { return s.record_bytes; }
uint64_t state_fingerprint(const EnvState& s) { return s.fingerprint; }

static uint64_t mix(uint64_t h, uint64_t v) {
  h ^= v + 0x9e3779b97f4a7c15ull + (h << 6) + (h >> 2);
  h = (h ^ (h >> 31)) * 0x7fb5d329728ea185ull;
  return h ^ (h >> 27);
}

std::string state_layout(EnvState& s, const MapSlots& maps) {
  s.record_bytes = 0;
  const size_t n = s.S.n;
  uint64_t fp = mix(mix(mix(0, kLayoutVersion), DTS_MAX_DELAY), maps_slot_count(maps));
  for (int m = 0; m < maps_slot_count(maps); m++) fp = mix(fp, maps_hash(maps, m));
  std::vector<Row> rows;
  uint32_t off = 0;
  auto add = [&](void* base, uint32_t size) { rows.push_back(Row{static_cast<uint8_t*>(base), off, size}); off += size; };
  for (int k = 0; k < kNumArrays; k++) {
    const StateArray& a = kStateArrays[k];
    uint8_t* base = static_cast<uint8_t*>(get_member(s.S, a.member));
    if (a.member == offsetof(DState, map_id)) s.map_id_off = (int)off;
    for (uint32_t p = 0; p < a.planes; p++) add(base + p * a.size * n, a.size);
    if (k != kObstaclesAfter) continue;
    for (int m = 0; m < maps_slot_count(maps); m++) {   // every map's obstacles: f64[DTS_DYN_FIELDS][n_dyn][n]
      const DMap* d = maps_get(maps, m);
      if (!d || !d->n_dyn) continue;
      for (int r = 0; r < DTS_DYN_FIELDS * d->n_dyn; r++) add(d->dyn_state + r * n, 8);
    }
  }
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

void launch_state_save(const EnvState& s, void* records, cudaStream_t st) {
  const dim3 grid((s.S.n + kGroup - 1) / kGroup, s.n_chunks);
  k_state_save<<<grid, kThreads, sizeof(uint32_t) * kGroup * s.stride_words, st>>>(
      s.rows, s.chunks, s.S.n, s.stride_words, (uint32_t)s.record_bytes, static_cast<uint8_t*>(records));
}

void launch_state_load(EnvState& s, const uint8_t* mask, const void* records, const DMap* maps, int n_maps,
                       int32_t* refused, cudaStream_t st) {
  const dim3 grid((s.S.n + kGroup - 1) / kGroup, s.n_chunks);
  k_state_load<<<grid, kThreads, sizeof(uint32_t) * kGroup * s.stride_words, st>>>(
      s.rows, s.chunks, s.S.n, s.stride_words, (uint32_t)s.record_bytes, static_cast<const uint8_t*>(records), mask,
      maps, n_maps, s.map_id_off, refused);
  s.seeded = true;   // the envs' streams came with their records
}

}  // namespace dts
