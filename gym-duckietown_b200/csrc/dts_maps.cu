// dts_maps.cu — the map slots of one handle (dts_upload_map): a dts_map_blob checked, built into a DMap on the host and
// copied to the device, and the device table of every slot's DMap that the kernels index by S.map_id.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <type_traits>
#include <utility>
#include <vector>

#include "dts_kernels.h"

namespace dts {

struct MapSlot {
  DMap rec{};                   // host copy of the device table's entry (valid = 0: empty)
  const float2* extent = nullptr;   // host copy of the extent table's entry (maps_extent_table)
  std::vector<void*> allocs;    // the device memory behind it
  uint64_t hash = 0;            // content hash of the blob it was built from (0: empty)
};

struct MapSlots {
  int n_envs;
  DMap* table = nullptr;          // device [max_maps]
  const float2** extent = nullptr;   // device [max_maps]: each slot's object extents (maps_extent_table)
  std::vector<MapSlot> slots;     // [max_maps]
  std::vector<MapCounts> counts;  // [max_maps]
};

MapSlots* maps_create(const dts_config& cfg) {
  const size_t bytes = sizeof(DMap) * cfg.max_maps, ext_bytes = sizeof(float2*) * cfg.max_maps;
  void *t = nullptr, *x = nullptr;
  if (cudaMalloc(&t, bytes) != cudaSuccess) return nullptr;
  if (cudaMalloc(&x, ext_bytes) != cudaSuccess) { cudaFree(t); return nullptr; }
  cudaMemset(t, 0, bytes);
  cudaMemset(x, 0, ext_bytes);
  return new MapSlots{cfg.num_envs, static_cast<DMap*>(t), static_cast<const float2**>(x),
                      std::vector<MapSlot>(cfg.max_maps), std::vector<MapCounts>(cfg.max_maps)};
}

void maps_destroy(MapSlots* m) {
  if (!m) return;
  for (const MapSlot& s : m->slots)
    for (void* p : s.allocs) cudaFree(p);
  cudaFree(m->table);
  cudaFree(m->extent);
  delete m;
}

const DMap* maps_table(const MapSlots& m) { return m.table; }

const float2* const* maps_extent_table(const MapSlots& m) { return m.extent; }

const DMap* maps_get(const MapSlots& m, int slot) {
  return slot >= 0 && slot < (int)m.slots.size() && m.slots[slot].rec.valid ? &m.slots[slot].rec : nullptr;
}

const std::vector<MapCounts>& maps_counts(const MapSlots& m) { return m.counts; }

int maps_slot_count(const MapSlots& m) { return (int)m.slots.size(); }

uint64_t maps_hash(const MapSlots& m, int slot) { return maps_get(m, slot) ? m.slots[slot].hash : 0; }

// 64-bit FNV-1a over 8-byte words (the tail byte by byte), with a final avalanche
namespace {
struct Hasher {
  uint64_t h = 0xcbf29ce484222325ull;
  void bytes(const void* p, size_t n) {
    const uint8_t* b = static_cast<const uint8_t*>(p);
    size_t i = 0;
    for (; i + 8 <= n; i += 8) {
      uint64_t w;
      memcpy(&w, b + i, 8);
      h = (h ^ w) * 0x100000001b3ull;
    }
    for (; i < n; i++) h = (h ^ b[i]) * 0x100000001b3ull;
  }
  template <typename T> void arr(const T* p, size_t count) {   // the element count, then the contents
    const uint64_t c = p ? count : 0;
    bytes(&c, sizeof c);
    if (p && count) bytes(p, count * sizeof(T));
  }
  template <typename T> void val(const T& v) { bytes(&v, sizeof v); }
  uint64_t done() const {
    uint64_t z = h;
    z = (z ^ (z >> 30)) * 0xbf58476d1ce4e5b9ull;
    z = (z ^ (z >> 27)) * 0x94d049bb133111ebull;
    z ^= z >> 31;
    return z ? z : 1;   // 0 stands for an empty slot
  }
};
}  // namespace

// Everything a blob says, pointers aside: two uploads of the same map hash alike, in any process
static uint64_t blob_hash(const dts_map_blob& b) {
  Hasher H;
  const size_t T = (size_t)b.grid_w * b.grid_h;
  H.val(b.tile_size); H.val(b.grid_w); H.val(b.grid_h);
  H.arr(b.tile_kind, T); H.arr(b.tile_angle, T); H.arr(b.tile_drivable, T); H.arr(b.tile_tex, T);
  H.arr(b.tile_curve_off, T); H.arr(b.tile_curve_cnt, T);
  H.arr(b.curves, (size_t)b.n_curves * 12);
  H.arr(b.coll_corners, (size_t)b.n_coll * 8); H.arr(b.coll_norms, (size_t)b.n_coll * 4);
  H.arr(b.coll_centers, (size_t)b.n_coll * 3); H.arr(b.coll_radii, (size_t)b.n_coll);
  H.val(b.n_objects);
  for (int o = 0; o < b.n_objects; o++) { dts_object s = b.objects[o]; s.reserved = 0; H.val(s); }
  H.val(b.n_meshes);
  for (int i = 0; i < b.n_meshes; i++) { dts_mesh s = b.meshes[i]; s.reserved = 0; H.val(s); }
  H.arr(b.tri_pos, (size_t)b.n_tris * 9); H.arr(b.tri_nrm, (size_t)b.n_tris * 9); H.arr(b.tri_uv, (size_t)b.n_tris * 6);
  H.arr(b.tri_col, (size_t)b.n_tris * 9); H.arr(b.tri_tex, (size_t)b.n_tris);
  H.val(b.n_textures);
  for (int t = 0; t < b.n_textures; t++) {
    const dts_texture& s = b.textures[t];
    H.val(s.width); H.val(s.height);
    H.arr(s.rgba, (size_t)s.width * s.height * 4);
  }
  H.arr(b.tex_segment, b.tex_segment ? (size_t)b.n_textures : 0);
  if (b.tex_class) {   // (a blob without classes hashes as before they existed)
    size_t texels = 0;
    for (int t = 0; t < b.n_textures; t++) texels += (size_t)b.textures[t].width * b.textures[t].height;
    H.arr(b.tex_class, texels);
  }
  if (b.obj_corners) H.arr(b.obj_corners, (size_t)b.n_objects * 8);   // (likewise for footprints)
  H.val(b.start_tile[0]); H.val(b.start_tile[1]); H.val(b.has_start_pose);
  for (int k = 0; k < 3; k++) H.val(b.start_pose[k]);
  H.val(b.agent_mesh);
  H.val(b.n_dyn);
  for (int s = 0; s < b.n_dyn; s++) { dts_dyn_object q = b.dyn[s]; q.reserved = 0; H.val(q); }
  return H.done();
}

static std::string format(const char* fmt, ...) {
  char buf[512];
  va_list ap;
  va_start(ap, fmt);
  vsnprintf(buf, sizeof buf, fmt, ap);
  va_end(ap);
  return buf;
}

// bytes a texture takes in its map's pool: each starts 256-byte aligned
static size_t pool_bytes(const dts_texture& s) { return ((size_t)s.width * s.height * 4 + 255) & ~size_t(255); }

// Every refusal of a blob, before anything is built from it
static std::string validate(const dts_map_blob* b, int slot, int n_slots) {
  if (!b || slot < 0 || slot >= n_slots) return format("bad map_id %d", slot);
  if (b->n_objects > DTS_MAX_OBJECTS) return format("map has %d objects, limit %d", b->n_objects, DTS_MAX_OBJECTS);
  if (b->grid_w <= 0 || b->grid_h <= 0 || !(b->tile_size > 0)) return "invalid tile grid";
  if (b->n_dyn < 0 || b->n_dyn > DTS_MAX_DYN) return format("map has %d dynamic obstacles, limit %d", b->n_dyn, DTS_MAX_DYN);
  for (int o = 0; o < b->n_objects; o++) {
    const dts_object& s = b->objects[o];
    if (s.mesh_id < 0 || s.mesh_id >= b->n_meshes) return format("object %d: bad mesh_id", o);
    if (s.alt_tex_to >= b->n_textures || s.alt_tex_from >= b->n_textures) return format("object %d: alt texture out of range", o);
    if (s.dyn_slot >= b->n_dyn) return format("object %d: dyn_slot %d out of range", o, s.dyn_slot);
    for (int k = 0; b->obj_corners && k < 8; k++)
      if (!std::isfinite(b->obj_corners[(size_t)o * 8 + k])) return format("object %d: footprint corner is not finite", o);
  }
  // the bounding spheres are computed from tri_pos on the host
  for (int i = 0; i < b->n_meshes; i++) {
    const dts_mesh& me = b->meshes[i];
    if (me.tri_offset < 0 || me.tri_count < 0 || (int64_t)me.tri_offset + me.tri_count > b->n_tris)
      return format("mesh %d: triangles %d .. %d past n_tris %d", i, me.tri_offset, me.tri_offset + me.tri_count, b->n_tris);
  }
  size_t pool = 0;
  for (int t = 0; t < b->n_textures; t++) {
    const dts_texture& s = b->textures[t];
    if (s.width <= 0 || s.height <= 0 || (s.width & (s.width - 1)) || (s.height & (s.height - 1)))
      return format("texture %d: %dx%d is not a power of two", t, s.width, s.height);
    // DTexture::info holds log2 of each side in 4 bits and the pool offset >> 8 in 24
    if (s.width > (1 << 15) || s.height > (1 << 15)) return format("texture %d: %dx%d too large", t, s.width, s.height);
    pool += pool_bytes(s);
  }
  if (pool >= (size_t(1) << 32)) return "textures exceed 4 GB";
  for (int s = 0; s < b->n_dyn; s++) {
    const dts_dyn_object& q = b->dyn[s];
    if (q.kind != DTS_DYN_DUCKIE && q.kind != DTS_DYN_DUCKIEBOT && q.kind != DTS_DYN_TRAFFICLIGHT) return format("dyn %d: bad kind %d", s, q.kind);
    if (q.object_index < 0 || q.object_index >= b->n_objects || b->objects[q.object_index].dyn_slot != s)
      return format("dyn %d: object_index %d does not point back to this slot", s, q.object_index);
  }
  return "";
}

// A DObject drawing mesh `mesh_id`: its triangles, segment texture and object-space bounding sphere.  `top` = the
// largest coordinate of its bounding box, for the spawn radius; `y_extent` = its least and largest y, ObjMesh's
// min_coords[1] / max_coords[1] (objmesh.py:228-232).
static DObject mesh_object(const dts_map_blob& b, int mesh_id, float& top, float2& y_extent) {
  const dts_mesh& me = b.meshes[mesh_id];
  DObject d{};
  d.mesh_id = mesh_id; d.tri_offset = me.tri_offset; d.tri_count = me.tri_count;
  d.seg_tex = (me.seg_flat_tex >= 0 && me.seg_flat_tex < b.n_textures) ? me.seg_flat_tex : -1;
  float lo[3] = {1e30f, 1e30f, 1e30f}, hi[3] = {-1e30f, -1e30f, -1e30f};
  for (int t = 0; t < me.tri_count * 3; t++)
    for (int k = 0; k < 3; k++) {
      const float v = b.tri_pos[((size_t)me.tri_offset * 3 + t) * 3 + k];
      lo[k] = v < lo[k] ? v : lo[k];
      hi[k] = v > hi[k] ? v : hi[k];
    }
  top = hi[0] > hi[1] ? hi[0] : hi[1];
  top = top > hi[2] ? top : hi[2];
  y_extent = make_float2(lo[1], hi[1]);
  float r2 = 0.f;
  for (int k = 0; k < 3; k++) { d.centre[k] = 0.5f * (lo[k] + hi[k]); const float h = 0.5f * (hi[k] - lo[k]); r2 += h * h; }
  d.bound_rad = sqrtf(r2);
  return d;
}

// src[0 .. count) -> a new device allocation at dst, listed in `owned`: zeroed, at least one element, and 16 bytes of
// slack past the end
template <typename T>
static std::string upload(T*& dst, const std::remove_const_t<T>* src, size_t count, std::vector<void*>& owned) {
  const size_t bytes = (count ? count : 1) * sizeof(T);
  void* d = nullptr;
  cudaError_t e = cudaMalloc(&d, bytes + 16);
  if (e != cudaSuccess) return format("cudaMalloc(%zu B) failed: %s", bytes, cudaGetErrorString(e));
  owned.push_back(d);
  cudaMemset(d, 0, bytes + 16);
  if (count && src && (e = cudaMemcpy(d, src, count * sizeof(T), cudaMemcpyHostToDevice)) != cudaSuccess)
    return format("cudaMemcpy H2D failed: %s", cudaGetErrorString(e));
  dst = static_cast<T*>(d);
  return "";
}

std::string maps_upload(MapSlots& ms, int slot, const dts_map_blob* blob) {
  std::string err = validate(blob, slot, (int)ms.slots.size());
  if (!err.empty()) return err;
  const dts_map_blob& b = *blob;
  // 1. the host-side arrays
  DMap m{};
  const size_t T = (size_t)b.grid_w * b.grid_h;
  m.tile_size = b.tile_size; m.grid_w = b.grid_w; m.grid_h = b.grid_h; m.n_tiles = (int)T;
  m.n_coll = b.n_coll;
  std::vector<int32_t> drv;
  for (int j = 0; j < b.grid_h; j++)       // reference scan order S:810-860
    for (int i = 0; i < b.grid_w; i++)
      if (b.tile_kind[j * b.grid_w + i] >= 0 && b.tile_drivable[j * b.grid_w + i]) { drv.push_back(i); drv.push_back(j); }
  m.start_i = b.start_tile[0]; m.start_j = b.start_tile[1];
  if (m.start_i < 0 || m.start_j < 0 || m.start_i >= b.grid_w || m.start_j >= b.grid_h) { m.start_i = -1; m.start_j = -1; }
  m.has_start_pose = b.has_start_pose != 0;
  for (int k = 0; k < 3; k++) m.start_pose[k] = b.start_pose[k];
  m.n_drivable = (int)drv.size() / 2;
  // objects: add spawn radius (S:1467) and a bounding sphere per placed mesh
  MapCounts counts{m.n_tiles, b.n_objects, 0};
  std::vector<DObject> objs(b.n_objects);
  std::vector<float2> y_extent(b.n_objects);
  for (int o = 0; o < b.n_objects; o++) {
    const dts_object& s = b.objects[o];
    float top;
    DObject& d = objs[o] = mesh_object(b, s.mesh_id, top, y_extent[o]);
    d.tri_base = (int32_t)counts.n_tris;   // (the objects' triangles so far: the agent's are added after the loop)
    for (int k = 0; k < 3; k++) { d.pos[k] = (float)s.pos[k]; d.dpos[k] = s.pos[k]; }   // glTranslatef takes floats
    d.dyn_slot = s.dyn_slot;
    d.alt_from = s.alt_tex_from; d.alt_to = s.alt_tex_to;
    d.scale = s.scale; d.y_rot_deg = s.y_rot_deg; d.optional = s.optional;
    d.spawn_rad = top * 0.5f * s.scale + 0.25f;     // MIN_SPAWN_OBJ_DIST S:156
    counts.n_tris += d.tri_count;
  }
  m.n_objects = b.n_objects;
  m.n_tris = b.n_tris;
  if (b.agent_mesh >= 0 && b.agent_mesh < b.n_meshes) {   // self.mesh, drawn by top-down views at cur_pos (S:1923-1929)
    float top;
    float2 y_extent_agent;
    m.agent = mesh_object(b, b.agent_mesh, top, y_extent_agent);
    m.agent.scale = 1.0f; m.agent.dyn_slot = -1; m.agent.alt_from = m.agent.alt_to = -1;
  }
  m.agent.tri_base = (int32_t)counts.n_tris;   // the agent's draw ids follow every object's
  counts.n_tris += m.agent.tri_count;
  std::vector<DTexture> tex(b.n_textures);
  std::vector<size_t> off(b.n_textures);
  size_t pool_size = 0;
  for (int t = 0; t < b.n_textures; t++) {
    off[t] = pool_size;
    pool_size += pool_bytes(b.textures[t]);
  }
  // the texel classes follow the texels in the same allocation, a byte per texel at the texture's texel offset (off / 4),
  // so that a prim's texture word finds both and a refused upload leaves the slot's classes with its texels
  const size_t class_off = pool_size ? pool_size : 256;
  std::vector<uint8_t> pool(class_off + class_off / 4, 0);
  size_t class_src = 0;
  for (int t = 0; t < b.n_textures; t++) {
    const dts_texture& s = b.textures[t];
    memcpy(pool.data() + off[t], s.rgba, (size_t)s.width * s.height * 4);
    if (b.tex_class) memcpy(pool.data() + class_off + off[t] / 4, b.tex_class + class_src, (size_t)s.width * s.height);
    class_src += (size_t)s.width * s.height;
    int lw = 0, lh = 0;
    while ((1 << lw) < s.width) lw++;
    while ((1 << lh) < s.height) lh++;
    tex[t].w = s.width; tex[t].h = s.height;   // (rgba once the pool is on the device)
    tex[t].info = (uint32_t)(off[t] >> 8) | ((uint32_t)lw << 24) | ((uint32_t)lh << 28);
    tex[t].pad = 0;
  }
  m.n_textures = b.n_textures;
  m.tex_class_off = (uint32_t)class_off;   // (validate() keeps the pool below 4 GB)
  std::vector<int16_t> seg(b.n_textures > 0 ? b.n_textures : 1);
  for (int t = 0; t < b.n_textures; t++) {
    const int v = b.tex_segment ? b.tex_segment[t] : -1;
    seg[t] = (int16_t)((v >= 0 && v < b.n_textures) ? v : t);
  }
  // dynamic obstacles: constants + every env's copy of the load-time state ([field][slot][env])
  m.n_dyn = b.n_dyn;
  const size_t N = ms.n_envs, D = b.n_dyn;
  std::vector<DDyn> par(D);
  std::vector<double> st((size_t)DTS_DYN_FIELDS * D * N);
  for (size_t s = 0; s < D; s++) {
    const dts_dyn_object& q = b.dyn[s];
    DDyn& p = par[s];
    p.kind = q.kind; p.object_index = q.object_index; p.pos_y = q.pos[1];
    for (int k = 0; k < 4; k++) p.norms[k] = q.norms[k / 2][k % 2];
    p.safety_radius = q.safety_radius; p.walk_distance = q.walk_distance; p.wiggle = q.wiggle; p.angle0 = q.angle;
    p.follow_dist = q.follow_dist; p.velocity = q.velocity; p.gain = q.gain; p.trim = q.trim; p.radius = q.radius;
    p.k = q.k; p.limit = q.limit; p.wheel_dist = q.wheel_dist; p.robot_width = q.robot_width; p.robot_length = q.robot_length;
    double f[DTS_DYN_FIELDS] = {};
    f[DTS_DYN_PX] = q.pos[0]; f[DTS_DYN_PZ] = q.pos[2]; f[DTS_DYN_ANGLE] = q.angle;
    f[DTS_DYN_YROT] = q.angle * (180.0 / 3.14159265358979323846);       // np.rad2deg O:57
    for (int k = 0; k < 4; k++) { f[DTS_DYN_CORNERS + 2 * k] = q.corners[k][0]; f[DTS_DYN_CORNERS + 2 * k + 1] = q.corners[k][1]; }
    f[DTS_DYN_START_X] = q.pos[0]; f[DTS_DYN_START_Z] = q.pos[2];
    f[DTS_DYN_WAIT] = q.wait_time; f[DTS_DYN_VEL] = q.vel; f[DTS_DYN_TIME] = 0.0; f[DTS_DYN_ACTIVE] = 0.0;
    p.freq = q.freq; p.tl_first = -1; p.pad = 0;
    if (q.kind == DTS_DYN_TRAFFICLIGHT) f[DTS_DYN_PATTERN] = q.pattern ? 1.0 : 0.0;
    for (int k = 0; k < DTS_DYN_FIELDS; k++)
      for (size_t e = 0; e < N; e++) st[((size_t)k * D + s) * N + e] = f[k];
  }
  int tl_first = -1, tl_last = -1;
  for (size_t s = 0; s < D; s++)
    if (par[s].kind == DTS_DYN_TRAFFICLIGHT) { if (tl_first < 0) tl_first = (int)s; tl_last = (int)s; }
  for (size_t s = 0; s < D; s++) par[s].tl_first = tl_first;
  if (tl_first >= 0)   // every constructor assigns the shared mesh's card (O:453): the last light's pattern shows
    for (size_t e = 0; e < N; e++) st[((size_t)DTS_DYN_SHOWN * D + tl_first) * N + e] = b.dyn[tl_last].pattern ? 1.0 : 0.0;
  std::vector<double> init((size_t)DTS_DYN_FIELDS * D);
  for (int k = 0; k < DTS_DYN_FIELDS; k++)
    for (size_t s = 0; s < D; s++) init[(size_t)k * D + s] = N ? st[((size_t)k * D + s) * N] : 0.0;
  // 2. the new map's device memory, built beside the slot, which keeps its map until this one is complete
  MapSlot fresh;
  auto put = [&](auto*& dst, const auto* src, size_t count) { if (err.empty()) err = upload(dst, src, count, fresh.allocs); };
  put(m.tile_kind, b.tile_kind, T);
  put(m.tile_angle, b.tile_angle, T);
  put(m.tile_drivable, b.tile_drivable, T);
  put(m.tile_tex, b.tile_tex, T);
  put(m.tile_curve_off, b.tile_curve_off, T);
  put(m.tile_curve_cnt, b.tile_curve_cnt, T);
  put(m.curves, b.curves, (size_t)b.n_curves * 12);
  put(m.coll_corners, b.coll_corners, (size_t)b.n_coll * 8);
  put(m.coll_norms, b.coll_norms, (size_t)b.n_coll * 4);
  put(m.coll_centers, b.coll_centers, (size_t)b.n_coll * 3);
  put(m.coll_radii, b.coll_radii, (size_t)b.n_coll);
  put(m.drivable_ij, drv.data(), drv.size());
  put(m.objects, objs.data(), objs.size());
  put(m.tri_pos, b.tri_pos, (size_t)b.n_tris * 9);
  put(m.tri_nrm, b.tri_nrm, (size_t)b.n_tris * 9);
  put(m.tri_uv, b.tri_uv, (size_t)b.n_tris * 6);
  put(m.tri_col, b.tri_col, (size_t)b.n_tris * 9);
  put(m.tri_tex, b.tri_tex, (size_t)b.n_tris);
  put(m.tex_pool, pool.data(), pool.size());
  for (int t = 0; t < b.n_textures && err.empty(); t++) tex[t].rgba = m.tex_pool + off[t];
  put(m.textures, tex.data(), tex.size());
  put(m.tex_segment, seg.data(), seg.size());
  put(m.dyn, par.data(), par.size());
  put(m.dyn_state, st.data(), st.size());
  put(m.dyn_init, init.data(), init.size());
  if (b.obj_corners) put(m.obj_corners, b.obj_corners, (size_t)b.n_objects * 8);
  const float2* extent = nullptr;
  put(extent, y_extent.data(), y_extent.size());
  m.valid = 1;
  // 3. once no kernel still reads the slot's old map: the table entry, the host record, and the old map's memory
  if (err.empty()) {
    cudaError_t e = cudaDeviceSynchronize();
    // the extent entry first, and back to the old one if the map entry cannot follow: either both entries name the
    // new map or both the old one
    if (e == cudaSuccess) e = cudaMemcpy(ms.extent + slot, &extent, sizeof(extent), cudaMemcpyHostToDevice);
    if (e == cudaSuccess) {
      e = cudaMemcpy(ms.table + slot, &m, sizeof(DMap), cudaMemcpyHostToDevice);
      if (e != cudaSuccess)
        cudaMemcpy(ms.extent + slot, &ms.slots[slot].extent, sizeof(extent), cudaMemcpyHostToDevice);
    }
    if (e != cudaSuccess) err = format("map table update failed: %s", cudaGetErrorString(e));
  }
  if (err.empty()) {
    fresh.rec = m;
    fresh.extent = extent;
    fresh.hash = blob_hash(b);
    std::swap(ms.slots[slot], fresh);   // fresh: what to release, the old map or the new one that failed
    ms.counts[slot] = counts;
  }
  for (void* p : fresh.allocs) cudaFree(p);
  return err;
}

}  // namespace dts
