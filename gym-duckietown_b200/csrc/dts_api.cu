// dts_api.cu — the C ABI of libdtsim.so (include/dtsim.h): handle management, host->device
// staging of episode parameters, and stream-ordered launches of the kernels.
#include <cmath>
#include <cstdarg>
#include <cstdio>
#include <cstring>
#include <dlfcn.h>
#include <string>
#include <vector>

#include "dts_kernels.h"

using namespace dts;

namespace {
thread_local std::string g_create_error;

#define DTS_CUDA(expr)                                                                          \
  do {                                                                                          \
    cudaError_t _e = (expr);                                                                    \
    if (_e != cudaSuccess) return sim->fail("%s failed: %s", #expr, cudaGetErrorString(_e));     \
  } while (0)
}  // namespace

struct dts_sim {
  dts_config cfg;
  StepCfg step_cfg;
  std::vector<void*> allocs;           // freed in dts_destroy
  EnvState* state = nullptr;            // the envs' simulator state, its reset staging and snapshot records
  MapSlots* maps = nullptr;             // the uploaded maps (dts_upload_map)
  Renderer* render = nullptr;           // frame memory and fisheye tables
  Resizer* resize = nullptr;            // the post-render ResizeWrapper (dts_set_resize_filter)
  int32_t* d_err = nullptr;
  int32_t* h_status = nullptr;          // mapped pinned host words: [0] a frame overflowed its frame memory,
                                        // [1] dts_load_state met a record naming no uploaded map
  int32_t* d_status = nullptr;          // its device address
  int32_t* ended = nullptr;             // dts_step_terminal: [N] the envs whose episode ended this step, *n_ended of them
  int32_t* n_ended = nullptr;
  // fused end-of-rollout gather over peer memory (dts_gather_*)
  uint8_t* gather_buf = nullptr;        // [world][bytes_per_rank], this rank's copy of everybody's observations
  uint64_t gather_bytes = 0;
  int gather_world = 0, gather_rank = 0;
  void* gather_peer[DTS_MAX_PEERS] = {};   // peers' buffers opened with cudaIpcOpenMemHandle (own entry = gather_buf)
  bool gather_next = false;
  int render_mode = 0;                  // dts_set_render_mode             // the next dts_render also stores into the gather buffers
  AuxTargets aux{};                     // dts_set_{depth,label,marking}_target: caller-owned images, or null
  BevTarget bev{};                      // dts_set_bev_target: caller-owned grids, both null = off
  ScanTarget scan{};                    // dts_set_scan_target: caller-owned range and hit, both null = off
  FlowTarget flow{};                    // dts_set_flow_target: caller-owned image and the record it owns, null = off
  OcclusionTarget occ{};                // dts_set_occlusion_target: caller-owned mask and the slots it owns, null = off
  BevViewTarget bev_view{};             // dts_set_bev_visibility_target: caller-owned outputs, both null = off
  ObjectTarget objects{};               // dts_set_object_target: caller-owned outputs, max_objects 0 = off
  LanePathTarget lane_path{};           // dts_set_lane_path_target: caller-owned outputs, n_points 0 = off
  bool drawn = false;                   // frame memory holds a frame of every env (dts_get_frame_cameras)
  // per-kernel timing (dts_profile_*): event pairs recorded around the render launches
  int profiling = 0;                    // 0 off, 1 events around k_raster only, 2 around every render kernel
  std::vector<cudaEvent_t> prof_events; // kProfMarks events per profiled frame
  int64_t prof_frames = 0;
  // query scratch
  double* q_in = nullptr; double* q_outd = nullptr; int32_t* q_outi = nullptr; uint32_t* q_hidden = nullptr; int q_cap = 0;
  // nccl (dlopen'ed)
  void* nccl_lib = nullptr; void* nccl_comm = nullptr;
  uint64_t launches = 0;
  dts_output_format fmt{DTS_OBS_HWC, DTS_OBS_U8, DTS_REWARD_RAW, DTS_ACTIONS_CONTINUOUS, 1.0};
  std::string err;

  int fail(const char* fmt, ...) {
    char buf[512];
    va_list ap;
    va_start(ap, fmt);
    vsnprintf(buf, sizeof buf, fmt, ap);
    va_end(ap);
    err = buf;
    return 1;
  }
  template <typename T> int dalloc(T** p, size_t count) {
    void* q = nullptr;
    cudaError_t e = cudaMalloc(&q, count * sizeof(T) + 16);
    if (e != cudaSuccess) return fail("cudaMalloc(%zu B) failed: %s", count * sizeof(T), cudaGetErrorString(e));
    cudaMemset(q, 0, count * sizeof(T) + 16);
    allocs.push_back(q);
    *p = (T*)q;
    return 0;
  }
};

extern "C" {

const char* dts_last_error(dts_sim* sim) { return sim ? sim->err.c_str() : g_create_error.c_str(); }

int dts_create(const dts_config* cfg, dts_sim** out) {
  if (!cfg || !out) { g_create_error = "null argument"; return 1; }
  if (cfg->abi_version != DTS_ABI_VERSION) { g_create_error = "dts_config.abi_version mismatch"; return 1; }
  if (cfg->num_envs <= 0 || cfg->cam_width <= 0 || cfg->cam_height <= 0 || cfg->max_maps <= 0) {
    g_create_error = "num_envs, cam_width, cam_height and max_maps must be positive";
    return 1;
  }
  if (cfg->cam_width > 800 || cfg->cam_height > 800) {  // guard band of the rasteriser: 2.5*size*64 < 2^17
    g_create_error = "camera larger than 800x800 is not supported by the rasteriser's fixed-point range";
    return 1;
  }
  cudaError_t e = cudaSetDevice(cfg->device);
  if (e != cudaSuccess) { g_create_error = std::string("cudaSetDevice failed: ") + cudaGetErrorString(e); return 1; }
  dts_sim* sim = new dts_sim();
  sim->cfg = *cfg;
  const int n = cfg->num_envs;
  StepCfg& c = sim->step_cfg;
  c.dt = 1.0 / cfg->frame_rate;                       // S:300
  c.robot_speed = cfg->robot_speed;
  c.accept_angle_deg = cfg->accept_start_angle_deg;
  c.gain = cfg->gain; c.trim = cfg->trim; c.radius = cfg->radius; c.k = cfg->k; c.limit = cfg->limit;
  c.dyn = DynParams{cfg->dyn_u1, cfg->dyn_u2, cfg->dyn_u3, cfg->dyn_w1, cfg->dyn_w2, cfg->dyn_w3,
                    cfg->dyn_uar, cfg->dyn_ual, cfg->dyn_war, cfg->dyn_wal, 0};
  // a command issued at t acts on integration intervals starting at or after t + delay
  int d = 0;
  while (d * c.dt < cfg->dyn_delay - 1e-12) d++;
  if (d > DTS_MAX_DELAY) { g_create_error = "dyn_delay exceeds DTS_MAX_DELAY steps"; delete sim; return 1; }
  c.dyn.delay_steps = d;
  c.frame_skip = cfg->frame_skip; c.max_steps = cfg->max_steps; c.action_mode = cfg->action_mode; c.flags = cfg->flags;
  c.seed = cfg->seed; c.env_id_offset = cfg->env_id_offset;
  c.random_maps = cfg->random_maps;
  c.reward_mode = DTS_REWARD_RAW; c.action_map = DTS_ACTIONS_CONTINUOUS; c.action_vel_scale = 1.0;
  if (cfg->num_tris_distractors < 0 || cfg->n_dr_ops < 0 || cfg->n_dr_ops > DTS_MAX_DR_OPS) {
    g_create_error = "num_tris_distractors / n_dr_ops out of range"; delete sim; return 1;
  }
  c.num_tris_distractors = cfg->num_tris_distractors;
  for (int k = 0; k < 3; k++) { c.color_sky[k] = cfg->color_sky[k]; c.color_ground[k] = cfg->color_ground[k]; }
  if (cfg->n_dr_ops > 0) {
    c.n_dr_ops = cfg->n_dr_ops;
    for (int k = 0; k < cfg->n_dr_ops; k++) {
      c.dr_ops[k] = cfg->dr_ops[k];
      const dts_dr_op& op = cfg->dr_ops[k];
      if (op.type < DTS_DR_INT || op.type > DTS_DR_NORMAL || op.size < 0 || op.target < DTS_DR_NONE || op.target > DTS_DR_TRIM) {
        g_create_error = "bad dts_dr_op"; delete sim; return 1;
      }
      // Generator.integers raises ValueError("low >= high") on an empty range; the device would draw garbage.  The
      // device takes int64 bounds, so a high of 2^63 or more is refused too.
      for (int j = 0; op.type == DTS_DR_INT && j < (op.size < 3 ? op.size : 3); j++) {
        if (!(op.a[j] < op.b[j]) || !(op.a[j] >= -9223372036854775808.0) || !(op.b[j] < 9223372036854775808.0)) {
          char buf[160];
          snprintf(buf, sizeof buf, "dts_dr_op %d: int draw needs low < high within int64, got low %.17g high %.17g",
                   k, op.a[j], op.b[j]);
          g_create_error = buf; delete sim; return 1;
        }
      }
    }
  } else {   // randomization/config/default_dr.json, keys sorted (randomizer.py:33)
    const dts_dr_op def[7] = {
        {DTS_DR_UNIFORM, 1, DTS_DR_CAMERA_ANGLE, 0, {0.8, 0, 0}, {1.2, 0, 0}},
        {DTS_DR_UNIFORM, 1, DTS_DR_CAMERA_FOV_Y, 0, {0.8, 0, 0}, {1.2, 0, 0}},
        {DTS_DR_UNIFORM, 1, DTS_DR_CAMERA_HEIGHT, 0, {0.92, 0, 0}, {1.08, 0, 0}},
        {DTS_DR_UNIFORM, 3, DTS_DR_CAMERA_NOISE, 0, {-0.005, -0.005, -0.005}, {0.005, 0.005, 0.005}},
        {DTS_DR_INT, 1, DTS_DR_HORZ_MODE, 0, {0, 0, 0}, {4, 0, 0}},
        {DTS_DR_UNIFORM, 3, DTS_DR_LIGHT_POS, 0, {-150, 170, -150}, {150, 220, 150}},
        {DTS_DR_NORMAL, 1, DTS_DR_TRIM, 0, {0, 0, 0}, {0.02, 0, 0}}};
    c.n_dr_ops = 7;
    for (int k = 0; k < 7; k++) c.dr_ops[k] = def[k];
  }
  int bad = 0;
  std::string se;
  if (!(sim->maps = maps_create(*cfg))) bad |= sim->fail("cudaMalloc(map table of %d slots) failed", cfg->max_maps);
  else if (!(sim->state = state_create(*cfg, *sim->maps, se))) bad |= sim->fail("%s", se.c_str());
  bad |= sim->dalloc(&sim->d_err, 32);
  bad |= sim->dalloc(&sim->ended, n);
  bad |= sim->dalloc(&sim->n_ended, 1);
  if (cudaHostAlloc((void**)&sim->h_status, 64, cudaHostAllocMapped) != cudaSuccess ||
      cudaHostGetDevicePointer((void**)&sim->d_status, sim->h_status, 0) != cudaSuccess) {
    sim->fail("cudaHostAlloc(mapped status word) failed"); bad = 1;
  } else {
    memset(sim->h_status, 0, 64);
  }
  sim->render = renderer_create(*cfg);
  sim->resize = resizer_create(*cfg);
  if (bad) { g_create_error = sim->err; dts_destroy(sim); return 1; }
  *out = sim;
  return 0;
}

void dts_destroy(dts_sim* sim) {
  if (!sim) return;
  cudaSetDevice(sim->cfg.device);
  cudaDeviceSynchronize();
  for (void* p : sim->allocs) cudaFree(p);
  maps_destroy(sim->maps);
  renderer_destroy(sim->render);
  resizer_destroy(sim->resize);
  state_destroy(sim->state);
  flow_record_free(sim->flow.rec);
  occlusion_free(sim->occ);
  void* extra[] = {sim->q_in, sim->q_outd, sim->q_outi, sim->q_hidden};
  for (void* p : extra) if (p) cudaFree(p);
  for (int p = 0; p < sim->gather_world; p++)
    if (sim->gather_peer[p] && sim->gather_peer[p] != sim->gather_buf) cudaIpcCloseMemHandle(sim->gather_peer[p]);
  if (sim->gather_buf) cudaFree(sim->gather_buf);
  if (sim->h_status) cudaFreeHost(sim->h_status);
  for (cudaEvent_t e : sim->prof_events) cudaEventDestroy(e);
  delete sim;
}

// The largest label (render spec item 10) of a map of these sizes: the agent's mesh, after the ground, cells and objects
static long long largest_label(long long n_cells, long long n_objects) { return 2 + n_cells + n_objects; }

// The most dynamic slots any uploaded map has (the flow record's size)
static int largest_n_dyn(dts_sim* sim) {
  int n = 0;
  for (int s = 0; s < maps_slot_count(*sim->maps); s++)
    if (const DMap* m = maps_get(*sim->maps, s)) n = m->n_dyn > n ? m->n_dyn : n;
  return n;
}

int dts_upload_map(dts_sim* sim, int map_id, const dts_map_blob* b) {
  if (!sim) return 1;
  if ((sim->aux.labels || sim->bev.labels || sim->scan.hit) && b && largest_label((long long)b->grid_w * b->grid_h, b->n_objects) > INT16_MAX)
    return sim->fail("a label target is set and this map's largest label, %lld, does not fit in int16",
                     largest_label((long long)b->grid_w * b->grid_h, b->n_objects));
  if (sim->objects.max_objects && b && b->n_objects > sim->objects.max_objects)
    return sim->fail("an object target of %d objects is set and this map has %d", sim->objects.max_objects, b->n_objects);
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  const std::string e = maps_upload(*sim->maps, map_id, b);
  if (!e.empty()) return sim->fail("%s", e.c_str());
  renderer_release_frame(*sim->render);
  sim->drawn = false;
  // the records now cover this map's obstacles, and the fingerprint its content: older records no longer load
  const std::string ls = state_layout(*sim->state, *sim->maps);
  if (!ls.empty()) return sim->fail("%s", ls.c_str());
  // the flow record, sized for the maps now uploaded: every env's previous frame is forgotten
  if (sim->flow.out) {
    FlowRecord rec;
    const std::string fe = flow_record_alloc(rec, sim->cfg.num_envs, largest_n_dyn(sim));
    if (!fe.empty()) {   // (the map is in: flow goes off rather than run against a record too small for it)
      flow_record_free(sim->flow.rec);
      sim->flow = FlowTarget{};
      occlusion_free(sim->occ);
      return sim->fail("%s; the flow and occlusion targets are cleared", fe.c_str());
    }
    flow_record_free(sim->flow.rec);
    sim->flow.rec = rec;
  }
  if (sim->occ.out) {   // the slots' frames were drawn from the old map
    const std::string oe = occlusion_empty(sim->occ, sim->cfg.num_envs);
    if (!oe.empty()) return sim->fail("%s", oe.c_str());
  }
  return 0;
}

int dts_set_fisheye_lut(dts_sim* sim, const float* rmapx, const float* rmapy, int width, int height) {
  if (!sim) return 1;
  if (!rmapx || !rmapy) return sim->fail("fisheye LUT is NULL");
  if (width != sim->cfg.cam_width || height != sim->cfg.cam_height)
    return sim->fail("fisheye LUT is %dx%d but the camera is %dx%d", width, height, sim->cfg.cam_width, sim->cfg.cam_height);
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  DTS_CUDA(cudaDeviceSynchronize());
  const std::string e = renderer_set_lut(*sim->render, false, 1, rmapx, rmapy, nullptr);
  return e.empty() ? 0 : sim->fail("%s", e.c_str());
}

int dts_set_fisheye_luts(dts_sim* sim, int count, const float* rmapx, const float* rmapy, int width, int height,
                         const int32_t* lut_of_env) {
  if (!sim) return 1;
  if (!(sim->cfg.flags & DTS_FLAG_DISTORTION)) return sim->fail("fisheye LUT pool on a handle created without DTS_FLAG_DISTORTION");
  if (count < 1 || count > 65536) return sim->fail("fisheye LUT pool of %d tables: 1 to 65536 are accepted", count);
  if (!rmapx || !rmapy || !lut_of_env) return sim->fail("fisheye LUT pool: rmapx, rmapy and lut_of_env must not be NULL");
  if (width != sim->cfg.cam_width || height != sim->cfg.cam_height)
    return sim->fail("fisheye LUTs are %dx%d but the camera is %dx%d", width, height, sim->cfg.cam_width, sim->cfg.cam_height);
  for (int e = 0; e < sim->cfg.num_envs; e++)
    if (lut_of_env[e] < 0 || lut_of_env[e] >= count)
      return sim->fail("lut_of_env[%d] = %d is not a table of the pool (0 to %d)", e, lut_of_env[e], count - 1);
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  DTS_CUDA(cudaDeviceSynchronize());
  const std::string e = renderer_set_lut(*sim->render, false, count, rmapx, rmapy, lut_of_env);
  return e.empty() ? 0 : sim->fail("%s", e.c_str());
}

int dts_set_rectify_lut(dts_sim* sim, const float* mapx, const float* mapy, int width, int height) {
  if (!sim) return 1;
  // a gather's bins are overlapping source boxes: only a DTS_FLAG_DISTORTION handle sizes its pair pool for them
  if (!(sim->cfg.flags & DTS_FLAG_DISTORTION)) return sim->fail("rectification LUT on a handle created without DTS_FLAG_DISTORTION");
  if (!mapx != !mapy) return sim->fail("rectification LUT: one of mapx / mapy is NULL");
  if (mapx && (width != sim->cfg.cam_width || height != sim->cfg.cam_height))
    return sim->fail("rectification LUT is %dx%d but the camera is %dx%d", width, height, sim->cfg.cam_width, sim->cfg.cam_height);
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  DTS_CUDA(cudaDeviceSynchronize());
  const std::string e = renderer_set_lut(*sim->render, true, 1, mapx, mapy, nullptr);
  return e.empty() ? 0 : sim->fail("%s", e.c_str());
}

// > 0: round-robin over that many slots; < 0: uniform draw over -n slots; 0: the env keeps its map
static int map_select(const dts_sim* sim) { return sim->cfg.random_maps > 0 ? -sim->cfg.random_maps : sim->cfg.cycle_maps; }

// status bit 1: a dts_load_state was handed a record naming no uploaded map (that env kept its state)
static int check_loaded(dts_sim* sim) {
  if (((volatile int32_t*)sim->h_status)[1])
    return sim->fail("an earlier dts_load_state met a record whose map_id names no uploaded map; that env was not loaded");
  return 0;
}

static int check_maps(dts_sim* sim) {
  if (!maps_get(*sim->maps, 0)) return sim->fail("no map uploaded in slot 0");
  const int cyc = sim->cfg.cycle_maps > sim->cfg.random_maps ? sim->cfg.cycle_maps : sim->cfg.random_maps;
  for (int k = 0; k < cyc; k++)
    if (!maps_get(*sim->maps, k)) return sim->fail("cycle_maps / random_maps = %d but slot %d is empty", cyc, k);
  return 0;
}

int dts_reset(dts_sim* sim, const uint8_t* mask_dev, const dts_episode_params* p, void* stream) {
  if (!sim) return 1;
  if (check_maps(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  const size_t n = sim->cfg.num_envs;
  dts_episode_params z{}, dev;
  if (!p) p = &z;
  if (p->map_id) {
    for (size_t e = 0; e < n; e++)
      if (!maps_get(*sim->maps, p->map_id[e]))
        return sim->fail("episode map_id[%zu]=%d has no uploaded map", e, p->map_id[e]);
  }
  const std::string e = state_stage(*sim->state, *p, dev, st);
  if (!e.empty()) return sim->fail("%s", e.c_str());
  launch_reset_params(state_arrays(*sim->state), maps_table(*sim->maps), sim->step_cfg, mask_dev, dev, st);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  // the staging buffers are pageable-host copies: make them safe to reuse before returning
  DTS_CUDA(cudaStreamSynchronize(st));
  return 0;
}

int dts_seed_streams(dts_sim* sim, const uint8_t* mask_host, const uint64_t* streams) {
  if (!sim) return 1;
  if (!streams) return sim->fail("streams is NULL");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  const std::string e = state_seed_streams(*sim->state, mask_host, streams);
  return e.empty() ? 0 : sim->fail("%s", e.c_str());
}

int dts_reset_random(dts_sim* sim, const uint8_t* mask_dev, void* stream) {
  if (!sim) return 1;
  if (check_maps(sim)) return 1;
  if (!state_seeded(*sim->state)) return sim->fail("dts_seed_streams must be called before a device-side reset");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_reset_random(state_arrays(*sim->state), maps_table(*sim->maps), sim->step_cfg, map_select(sim), mask_dev,
                      (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

// The bytes an armed gather writes into slot `rank` of every rank's buffer: the whole batch at the camera size, in the
// selected dtype
static uint64_t gather_batch_bytes(const dts_sim* sim) {
  const uint64_t elem = sim->fmt.obs_dtype == DTS_OBS_F32_UNIT ? 4 : 1;
  return (uint64_t)sim->cfg.num_envs * sim->cfg.cam_height * sim->cfg.cam_width * 3 * elem;
}
static int check_gather_fits(dts_sim* sim) {
  const uint64_t need = gather_batch_bytes(sim);
  if (need > sim->gather_bytes)
    return sim->fail("the fused gather holds %llu bytes per rank (dts_gather_alloc) but the observation batch is %llu bytes "
                     "in the current output format", (unsigned long long)sim->gather_bytes, (unsigned long long)need);
  return 0;
}
// An armed gather is checked before a step or render launches anything: a refused call leaves the state, every buffer
// and the armed gather as they were
static int check_gather(dts_sim* sim) {
  if (!sim->gather_next) return 0;
  if (resizer_target(*sim->resize).ow)
    return sim->fail("the fused gather writes the rasteriser's own output: not combined with dts_set_resize");
  return check_gather_fits(sim);
}

// dts_render of every env, or of the envs on a device list (dts_step_terminal's second pass; not profiled)
// Whether a target reads the fisheye tables' forward maps: flow, the bird's-eye visibility, the object boxes and the lane
// path.  They share one set; clearing one target frees it only when no other still reads it.
static bool reads_forward_maps(const dts_sim* sim) {
  return sim->flow.out || sim->bev_view.vis || sim->bev_view.pix || sim->objects.max_objects || sim->lane_path.n_points;
}

static int render_pass(dts_sim* sim, void* obs_dev, void* stream, const int32_t* env_list, const int32_t* env_count) {
  if (!obs_dev) return sim->fail("obs_dev is NULL");
  if (check_gather(sim)) return 1;
  if (check_maps(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  const std::string e = renderer_prepare(*sim->render, maps_counts(*sim->maps), sim->render_mode, reads_forward_maps(sim));
  if (!e.empty()) return sim->fail("%s", e.c_str());
  RenderCfg rc{sim->cfg.cam_width, sim->cfg.cam_height, sim->cfg.flags, sim->cfg.num_envs,
               (sim->cfg.flags & DTS_FLAG_TESSELLATE) ? 1 : 0, sim->render_mode, 0, env_list, env_count};
  if (*(volatile int32_t*)sim->h_status & 1)
    return sim->fail("an earlier frame overflowed its render frame memory (prim slab / bin lists) and was left incomplete");
  if (check_loaded(sim)) return 1;
  cudaEvent_t* marks = nullptr;
  if (sim->profiling && !env_list) {
    const size_t base = sim->prof_events.size();
    sim->prof_events.resize(base + kProfMarks);
    for (int k = 0; k < kProfMarks; k++) DTS_CUDA(cudaEventCreate(&sim->prof_events[base + k]));
    marks = sim->prof_events.data() + base;
    sim->prof_frames++;
  }
  const int mark_level = marks ? sim->profiling : 0;
  GatherTab gt{};
  if (sim->gather_next) {   // (check_gather: no resize target, and the batch fits the slot)
    gt.n = sim->gather_world;
    for (int p = 0; p < sim->gather_world; p++)
      gt.base[p] = reinterpret_cast<uint8_t*>(sim->gather_peer[p]) + (uint64_t)sim->gather_rank * sim->gather_bytes;
    sim->gather_next = false;
  }
  // the rasterisers draw packed u8 HWC at the camera size: into obs, or into the staging frame, from which the resize or
  // the format pass writes obs (and the gather's slots)
  const ResizeTarget rz = resizer_target(*sim->resize);
  const GatherTab raster_gt = rz.staging ? GatherTab{} : gt;
  rc.all_rows = raster_gt.n > 0;
  int k = launch_render(*sim->render, state_arrays(*sim->state), maps_table(*sim->maps), rc, sim->aux, sim->flow, sim->occ,
                        rz.staging ? rz.staging : obs_dev, raster_gt, sim->d_err, sim->d_status, marks, mark_level,
                        (cudaStream_t)stream);
  if (rz.ow) {
    launch_resize(*sim->resize, rz.staging, obs_dev, sim->fmt.obs_layout, sim->fmt.obs_dtype, env_list, env_count,
                  (cudaStream_t)stream);
    k++;
  } else if (rz.staging) {
    launch_format(*sim->resize, obs_dev, gt, env_list, env_count, (cudaStream_t)stream);
    k++;
  }
  if (marks && mark_level >= 2) cudaEventRecord(marks[kProfMarks - 1], (cudaStream_t)stream);   // closes the "post" interval
  sim->launches += k;
  DTS_CUDA(cudaGetLastError());
  sim->drawn = sim->drawn || !env_list;
  return 0;
}

// The bird's-eye grids of every env's current state, where a target is set (dts_set_bev_target)
static int bev_pass(dts_sim* sim, void* stream) {
  if (!sim->bev.labels && !sim->bev.marks) return 0;
  if (check_maps(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_bev(state_arrays(*sim->state), maps_table(*sim->maps), sim->bev, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

// The range scan of every env's current state, where a target is set (dts_set_scan_target)
static int scan_pass(dts_sim* sim, void* stream) {
  if (!sim->scan.range && !sim->scan.hit) return 0;
  if (check_maps(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  int max_objects = 0;
  for (const MapCounts& c : maps_counts(*sim->maps)) max_objects = c.n_objects > max_objects ? c.n_objects : max_objects;
  launch_scan(state_arrays(*sim->state), maps_table(*sim->maps), sim->scan, max_objects, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

// The outputs sampled from the map rather than rendered, in their order: the bird's-eye grids, then the range scan
static int map_pass(dts_sim* sim, void* stream) {
  if (bev_pass(sim, stream)) return 1;
  return scan_pass(sim, stream);
}

// The camera visibility of the grids bev_pass wrote, where a target is set (dts_set_bev_visibility_target): launched
// last in the call, against the frame the call drew (its camera, labels and remap), or with none every cell UNKNOWN
static int bev_view_pass(dts_sim* sim, void* stream, bool drew_frame) {
  if (!sim->bev_view.vis && !sim->bev_view.pix) return 0;
  launch_bev_view(state_arrays(*sim->state), maps_table(*sim->maps), sim->bev, sim->bev_view,
                  drew_frame ? renderer_frame_ctx(*sim->render) : nullptr, sim->aux.labels, sim->cfg.cam_width,
                  sim->cfg.cam_height, renderer_remap(*sim->render, sim->render_mode), drew_frame, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

// The object boxes of every env's current state, where a target is set (dts_set_object_target), and where they land in
// the frame the call drew (none: every corner NaN)
static int objects_pass(dts_sim* sim, void* stream, bool drew_frame) {
  if (!sim->objects.max_objects) return 0;
  if (check_maps(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_objects(state_arrays(*sim->state), maps_table(*sim->maps), maps_extent_table(*sim->maps), sim->objects,
                 drew_frame ? renderer_frame_ctx(*sim->render) : nullptr, sim->cfg.cam_width, sim->cfg.cam_height,
                 renderer_remap(*sim->render, sim->render_mode), drew_frame, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

// The lane path of every env's current state, where a target is set (dts_set_lane_path_target), and where its points
// land in the frame the call drew (none: every pixel NaN)
static int lane_path_pass(dts_sim* sim, void* stream, bool drew_frame) {
  if (!sim->lane_path.n_points) return 0;
  if (check_maps(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_lane_path(state_arrays(*sim->state), maps_table(*sim->maps), sim->lane_path,
                   drew_frame ? renderer_frame_ctx(*sim->render) : nullptr, sim->cfg.cam_width, sim->cfg.cam_height,
                   renderer_remap(*sim->render, sim->render_mode), drew_frame, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

// The passes that read the frame the call drew, last in the call and in this order: the grids' visibility, the object
// boxes, then the lane path
static int view_passes(dts_sim* sim, void* stream, bool drew_frame) {
  if (bev_view_pass(sim, stream, drew_frame)) return 1;
  if (objects_pass(sim, stream, drew_frame)) return 1;
  return lane_path_pass(sim, stream, drew_frame);
}

int dts_render(dts_sim* sim, void* obs_dev, void* stream) {
  if (!sim) return 1;
  if (render_pass(sim, obs_dev, stream, nullptr, nullptr)) return 1;
  if (map_pass(sim, stream)) return 1;
  return view_passes(sim, stream, true);
}

int dts_render_bev(dts_sim* sim, void* stream) {
  if (!sim) return 1;
  if (!sim->bev.labels && !sim->bev.marks) return sim->fail("no bird's-eye target is set (dts_set_bev_target)");
  if (bev_pass(sim, stream)) return 1;
  return bev_view_pass(sim, stream, false);
}

int dts_render_scan(dts_sim* sim, void* stream) {
  if (!sim) return 1;
  if (!sim->scan.range && !sim->scan.hit) return sim->fail("no range scan target is set (dts_set_scan_target)");
  return scan_pass(sim, stream);
}

int dts_render_objects(dts_sim* sim, void* stream) {
  if (!sim) return 1;
  if (!sim->objects.max_objects) return sim->fail("no object target is set (dts_set_object_target)");
  return objects_pass(sim, stream, false);
}

int dts_render_lane_path(dts_sim* sim, void* stream) {
  if (!sim) return 1;
  if (!sim->lane_path.n_points) return sim->fail("no lane path target is set (dts_set_lane_path_target)");
  return lane_path_pass(sim, stream, false);
}

int dts_object_pixels(dts_sim* sim, const int16_t* labels_dev, int32_t* pixels_dev, int32_t* boxes_dev, int max_objects,
                      void* stream) {
  if (!sim) return 1;
  if (max_objects < 1 || max_objects > DTS_MAX_OBJECTS)
    return sim->fail("object pixels for %d objects: 1 to %d are accepted", max_objects, DTS_MAX_OBJECTS);
  if (!labels_dev || !pixels_dev || !boxes_dev) return sim->fail("labels_dev, pixels_dev and boxes_dev must not be NULL");
  if (reinterpret_cast<uintptr_t>(labels_dev) & 1) return sim->fail("labels_dev is not aligned to 2 bytes");
  if ((reinterpret_cast<uintptr_t>(pixels_dev) | reinterpret_cast<uintptr_t>(boxes_dev)) & 3)
    return sim->fail("pixels_dev and boxes_dev must be aligned to 4 bytes");
  if (check_maps(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_object_pixels(state_arrays(*sim->state), maps_table(*sim->maps), labels_dev, sim->cfg.cam_width,
                       sim->cfg.cam_height, pixels_dev, boxes_dev, max_objects, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

// With a flow target: every env's camera and obstacles before the step, the previous frame of the next render's flow
static int flow_record(dts_sim* sim, cudaStream_t st) {
  if (!sim->flow.out) return 0;
  launch_flow_record(state_arrays(*sim->state), maps_table(*sim->maps), sim->flow.rec, st);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

int dts_step_terminal(dts_sim* sim, const float* actions_dev, void* obs_dev, void* terminal_obs_dev, float* reward_dev,
                      uint8_t* done_dev, void* stream) {
  if (!sim) return 1;
  if (!actions_dev) return sim->fail("actions_dev is NULL");
  if (!(sim->cfg.flags & DTS_FLAG_AUTO_RESET)) return sim->fail("dts_step_terminal needs a handle created with DTS_FLAG_AUTO_RESET");
  if (obs_dev && !terminal_obs_dev) return sim->fail("terminal_obs_dev is NULL");
  if (obs_dev && terminal_obs_dev == obs_dev) return sim->fail("terminal_obs_dev must be a buffer of its own, not obs_dev");
  if (sim->gather_next) return sim->fail("a fused gather is armed (dts_gather_next): dts_step_terminal does not write it");
  if (check_maps(sim) || check_loaded(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if (!state_seeded(*sim->state)) return sim->fail("auto-reset needs seeded streams: call dts_seed_streams first");
  cudaStream_t st = (cudaStream_t)stream;
  // 1. the step with the respawn held back: k_step_logic's only use of DTS_FLAG_AUTO_RESET is that respawn
  StepCfg deferred = sim->step_cfg;
  deferred.flags &= ~DTS_FLAG_AUTO_RESET;
  if (flow_record(sim, st)) return 1;
  launch_step_logic(state_arrays(*sim->state), maps_table(*sim->maps), deferred, map_select(sim), actions_dev, reward_dev,
                    done_dev, st);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  // 2. every env's frame of the state the step left: the terminal frame where the episode ended
  if (obs_dev && render_pass(sim, obs_dev, stream, nullptr, nullptr)) return 1;
  // 3. the ended envs respawn, in the same order of draws as inside k_step_logic, and are listed
  DTS_CUDA(cudaMemsetAsync(sim->n_ended, 0, sizeof(int32_t), st));
  launch_respawn_ended(state_arrays(*sim->state), maps_table(*sim->maps), sim->step_cfg, map_select(sim), sim->ended,
                       sim->n_ended, st);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  // the grids and scans of the state obs_dev will show: the ended envs' first states (every env's row, as the others did
  // not move)
  if (map_pass(sim, stream)) return 1;
  if (!obs_dev) return view_passes(sim, stream, false);
  // 4. their terminal frames -> terminal_obs_dev; 5. their first frames -> obs_dev
  const ResizeTarget rz = resizer_target(*sim->resize);
  const size_t px = rz.ow ? (size_t)rz.ow * rz.oh : (size_t)sim->cfg.cam_width * sim->cfg.cam_height;
  const size_t row_bytes = px * 3 * (sim->fmt.obs_dtype == DTS_OBS_F32_UNIT ? 4 : 1);
  launch_copy_rows(obs_dev, terminal_obs_dev, row_bytes, sim->ended, sim->n_ended, sim->cfg.num_envs, st);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  if (render_pass(sim, obs_dev, stream, sim->ended, sim->n_ended)) return 1;
  return view_passes(sim, stream, true);   // every row against the frame obs_dev shows
}

int dts_step(dts_sim* sim, const float* actions_dev, void* obs_dev, float* reward_dev, uint8_t* done_dev,
             void* stream) {
  if (!sim) return 1;
  if (!actions_dev) return sim->fail("actions_dev is NULL");
  if (check_maps(sim) || check_loaded(sim) || check_gather(sim)) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if ((sim->cfg.flags & DTS_FLAG_AUTO_RESET) && !state_seeded(*sim->state))
    return sim->fail("auto-reset needs seeded streams: call dts_seed_streams first");
  if (flow_record(sim, (cudaStream_t)stream)) return 1;
  launch_step_logic(state_arrays(*sim->state), maps_table(*sim->maps), sim->step_cfg, map_select(sim), actions_dev, reward_dev, done_dev,
                    (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  if (map_pass(sim, stream)) return 1;
  if (obs_dev && render_pass(sim, obs_dev, stream, nullptr, nullptr)) return 1;
  return view_passes(sim, stream, obs_dev != nullptr);
}

int dts_get_state(dts_sim* sim, dts_state_view* v) {
  if (!sim || !v) return 1;
  *v = state_view(*sim->state);
  return 0;
}

int dts_query_poses(dts_sim* sim, int map_id, int dyn_env, int n, const double* query, const uint32_t* hidden,
                    double* out_f64, int32_t* out_i32, void* stream) {
  cudaStream_t qs = (cudaStream_t)stream;   // ordered after the caller's in-flight steps (they move the dynamic obstacles)
  if (!sim) return 1;
  if (!maps_get(*sim->maps, map_id)) return sim->fail("bad map_id %d", map_id);
  if (dyn_env >= sim->cfg.num_envs) return sim->fail("dyn_env %d out of range", dyn_env);
  if (n <= 0) return 0;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if (n > sim->q_cap) {
    void* old[] = {sim->q_in, sim->q_outd, sim->q_outi, sim->q_hidden};
    for (void* p : old) if (p) cudaFree(p);
    sim->q_cap = n;
    DTS_CUDA(cudaMalloc(&sim->q_in, (size_t)n * 32));
    DTS_CUDA(cudaMalloc(&sim->q_outd, (size_t)n * 32));
    DTS_CUDA(cudaMalloc(&sim->q_outi, (size_t)n * 32));
    DTS_CUDA(cudaMalloc(&sim->q_hidden, (size_t)n * 32));
  }
  DTS_CUDA(cudaMemcpyAsync(sim->q_in, query, (size_t)n * 32, cudaMemcpyHostToDevice, qs));
  if (hidden) DTS_CUDA(cudaMemcpyAsync(sim->q_hidden, hidden, (size_t)n * 32, cudaMemcpyHostToDevice, qs));
  launch_query(maps_table(*sim->maps), map_id, dyn_env < 0 ? -1 : dyn_env, sim->cfg.num_envs, n, sim->q_in, hidden ? sim->q_hidden : nullptr, sim->q_outd, sim->q_outi, qs);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  DTS_CUDA(cudaMemcpyAsync(out_f64, sim->q_outd, (size_t)n * 32, cudaMemcpyDeviceToHost, qs));
  DTS_CUDA(cudaMemcpyAsync(out_i32, sim->q_outi, (size_t)n * 32, cudaMemcpyDeviceToHost, qs));
  DTS_CUDA(cudaStreamSynchronize(qs));
  return 0;
}

int dts_assign_maps(dts_sim* sim, const uint8_t* mask_dev, const int32_t* map_id_host, void* stream) {
  if (!sim) return 1;
  if (!map_id_host) return sim->fail("map_id_host is NULL");
  const size_t n = sim->cfg.num_envs;
  for (size_t e = 0; e < n; e++)
    if (!maps_get(*sim->maps, map_id_host[e]))
      return sim->fail("dts_assign_maps: map_id[%zu]=%d has no uploaded map", e, map_id_host[e]);
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  dts_episode_params host{}, dev;
  host.map_id = map_id_host;
  const std::string e = state_stage(*sim->state, host, dev, st);
  if (!e.empty()) return sim->fail("%s", e.c_str());
  launch_assign_maps(state_arrays(*sim->state), maps_table(*sim->maps), mask_dev, dev.map_id, st);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  DTS_CUDA(cudaStreamSynchronize(st));   // pageable host source
  return 0;
}

int dts_set_resize(dts_sim* sim, int out_w, int out_h) { return dts_set_resize_filter(sim, out_w, out_h, DTS_RESIZE_CV2_CUBIC); }

int dts_set_resize_filter(dts_sim* sim, int out_w, int out_h, int filter) {
  if (!sim) return 1;
  if (filter != DTS_RESIZE_CV2_CUBIC && filter != DTS_RESIZE_PIL_BILINEAR) return sim->fail("bad resize filter %d", filter);
  if (out_w < 0 || out_h < 0 || (out_w == 0) != (out_h == 0)) return sim->fail("bad resize target %dx%d", out_w, out_h);
  if (out_w > 4096 || out_h > 4096) return sim->fail("resize target %dx%d too large", out_w, out_h);
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  DTS_CUDA(cudaDeviceSynchronize());
  const std::string e = resizer_set(*sim->resize, filter, out_w, out_h);
  return e.empty() ? 0 : sim->fail("%s", e.c_str());
}

// ---- fused end-of-rollout gather: peer buffers over cudaIpc, written by the rasteriser itself --------------------
int dts_gather_alloc(dts_sim* sim, uint64_t bytes_per_rank, int rank, int world, uint8_t handle_out[64], void** buf_out) {
  if (!sim) return 1;
  if (world < 1 || world > DTS_MAX_PEERS || rank < 0 || rank >= world) return sim->fail("bad rank %d / world %d (max %d)", rank, world, DTS_MAX_PEERS);
  static_assert(sizeof(cudaIpcMemHandle_t) == 64, "cudaIpcMemHandle_t is 64 bytes");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if (sim->gather_buf) return sim->fail("gather buffer already allocated");
  DTS_CUDA(cudaMalloc(&sim->gather_buf, bytes_per_rank * (uint64_t)world));
  DTS_CUDA(cudaMemset(sim->gather_buf, 0, bytes_per_rank * (uint64_t)world));
  sim->gather_bytes = bytes_per_rank; sim->gather_rank = rank; sim->gather_world = world;
  for (int p = 0; p < DTS_MAX_PEERS; p++) sim->gather_peer[p] = nullptr;
  sim->gather_peer[rank] = sim->gather_buf;
  cudaIpcMemHandle_t h;
  DTS_CUDA(cudaIpcGetMemHandle(&h, sim->gather_buf));
  memcpy(handle_out, &h, 64);
  if (buf_out) *buf_out = sim->gather_buf;
  return 0;
}

int dts_gather_open(dts_sim* sim, const uint8_t* handles /*[world][64]*/) {
  if (!sim || !sim->gather_buf) return sim ? sim->fail("dts_gather_alloc first") : 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  for (int p = 0; p < sim->gather_world; p++) {
    if (p == sim->gather_rank) continue;
    cudaIpcMemHandle_t h;
    memcpy(&h, handles + 64 * p, 64);
    cudaError_t e = cudaIpcOpenMemHandle(&sim->gather_peer[p], h, cudaIpcMemLazyEnablePeerAccess);
    if (e != cudaSuccess) return sim->fail("cudaIpcOpenMemHandle(rank %d) failed: %s", p, cudaGetErrorString(e));
  }
  return 0;
}

int dts_gather_next(dts_sim* sim) {
  if (!sim || !sim->gather_buf) return sim ? sim->fail("dts_gather_alloc first") : 1;
  for (int p = 0; p < sim->gather_world; p++)
    if (!sim->gather_peer[p]) return sim->fail("dts_gather_open first (rank %d not mapped)", p);
  if (check_gather_fits(sim)) return 1;
  sim->gather_next = true;
  return 0;
}

int dts_blend4(dts_sim* sim, const uint8_t* const frames_dev[4], const double weights[4], double* out_dev, uint64_t n, void* stream) {
  if (!sim) return 1;
  if (!frames_dev || !weights || !out_dev) return sim->fail("NULL argument");
  for (int k = 0; k < 4; k++) if (!frames_dev[k]) return sim->fail("frame %d is NULL", k);
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_blend4(frames_dev, weights, out_dev, (size_t)n, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

int dts_set_timing(dts_sim* sim, double delta_time, int frame_skip, int action_mode) {
  if (!sim) return 1;
  if (!(delta_time > 0) || frame_skip < 1) return sim->fail("bad delta_time / frame_skip");
  if (action_mode != DTS_ACTION_PWM && action_mode != DTS_ACTION_VEL_STEER) return sim->fail("bad action_mode");
  int d = 0;
  while (d * delta_time < sim->cfg.dyn_delay - 1e-12) d++;
  if (d > DTS_MAX_DELAY) return sim->fail("dyn_delay / delta_time exceeds DTS_MAX_DELAY steps");
  sim->step_cfg.dt = delta_time; sim->step_cfg.frame_skip = frame_skip; sim->step_cfg.action_mode = action_mode;
  sim->step_cfg.dyn.delay_steps = d;
  sim->cfg.frame_skip = frame_skip; sim->cfg.action_mode = action_mode; sim->cfg.frame_rate = 1.0 / delta_time;
  return 0;
}

int dts_set_render_mode(dts_sim* sim, int mode) {
  if (!sim) return 1;
  if (mode & ~(DTS_RENDER_SEGMENT | DTS_RENDER_TOP_DOWN | DTS_RENDER_PINHOLE | DTS_RENDER_RECTIFY))
    return sim->fail("bad render mode %d", mode);
  sim->render_mode = mode;
  return 0;
}

int dts_set_depth_target(dts_sim* sim, float* depth_dev) {
  if (!sim) return 1;
  if (!depth_dev && sim->flow.out) return sim->fail("the flow target reads the depth image: clear it (dts_set_flow_target) first");
  if (reinterpret_cast<uintptr_t>(depth_dev) & 3) return sim->fail("depth target is not aligned to 4 bytes");
  sim->aux.depth = depth_dev;
  return 0;
}

// Every uploaded map's labels fit in int16, as a label target needs
static int check_labels_fit(dts_sim* sim) {
  const std::vector<MapCounts>& counts = maps_counts(*sim->maps);
  for (size_t s = 0; s < counts.size(); s++)
    if (counts[s].n_tiles && largest_label(counts[s].n_tiles, counts[s].n_objects) > INT16_MAX)
      return sim->fail("map slot %zu's largest label, %lld, does not fit in int16", s,
                       largest_label(counts[s].n_tiles, counts[s].n_objects));
  return 0;
}

int dts_set_label_target(dts_sim* sim, int16_t* labels_dev) {
  if (!sim) return 1;
  if (reinterpret_cast<uintptr_t>(labels_dev) & 1) return sim->fail("label target is not aligned to 2 bytes");
  if (!labels_dev && sim->flow.out) return sim->fail("the flow target reads the label image: clear it (dts_set_flow_target) first");
  if (!labels_dev && (sim->bev_view.vis || sim->bev_view.pix))
    return sim->fail("the bird's-eye visibility reads the label image: clear it (dts_set_bev_visibility_target) first");
  if (labels_dev && check_labels_fit(sim)) return 1;
  sim->aux.labels = labels_dev;
  return 0;
}

int dts_set_bev_target(dts_sim* sim, const dts_bev_config* cfg, int16_t* labels_dev, uint8_t* markings_dev) {
  if (!sim) return 1;
  if (sim->bev_view.vis || sim->bev_view.pix) {   // its outputs are sized for this grid, and it reads its labels
    if (!cfg || !labels_dev)
      return sim->fail("the bird's-eye visibility reads the grid's labels: clear it (dts_set_bev_visibility_target) first");
    if (cfg->width != sim->bev.cfg.width || cfg->height != sim->bev.cfg.height)
      return sim->fail("the bird's-eye visibility target is sized for the %d x %d grid: clear it "
                       "(dts_set_bev_visibility_target) before reshaping the grid", sim->bev.cfg.width, sim->bev.cfg.height);
  }
  if (!cfg || (!labels_dev && !markings_dev)) {
    sim->bev = BevTarget{};
    return 0;
  }
  if (cfg->width < 1 || cfg->width > 2048 || cfg->height < 1 || cfg->height > 2048)
    return sim->fail("bird's-eye grid of %d x %d cells: 1 to 2048 per side are accepted", cfg->width, cfg->height);
  if (!std::isfinite(cfg->cell) || !(cfg->cell > 0))
    return sim->fail("bird's-eye cell size %g: a finite size > 0 is needed", cfg->cell);
  if (!std::isfinite(cfg->origin_x) || !std::isfinite(cfg->origin_y))
    return sim->fail("bird's-eye origin (%g, %g) is not finite", cfg->origin_x, cfg->origin_y);
  if (reinterpret_cast<uintptr_t>(labels_dev) & 1) return sim->fail("bird's-eye label target is not aligned to 2 bytes");
  if (labels_dev && check_labels_fit(sim)) return 1;
  sim->bev = BevTarget{*cfg, labels_dev, markings_dev};
  return 0;
}

int dts_set_scan_target(dts_sim* sim, const dts_scan_config* cfg, float* range_dev, int16_t* hit_dev) {
  if (!sim) return 1;
  if (!cfg || (!range_dev && !hit_dev)) {
    sim->scan = ScanTarget{};
    return 0;
  }
  if (cfg->n_rays < 1 || cfg->n_rays > 4096) return sim->fail("range scan of %d rays: 1 to 4096 are accepted", cfg->n_rays);
  if (!(cfg->fov > 0 && cfg->fov <= 2 * M_PI)) return sim->fail("range scan field of view %g: (0, 2 pi] is accepted", cfg->fov);
  if (!std::isfinite(cfg->max_range) || !(cfg->max_range > 0))
    return sim->fail("range scan max_range %g: a finite range > 0 is needed", cfg->max_range);
  if (!std::isfinite(cfg->origin_forward) || !std::isfinite(cfg->origin_right))
    return sim->fail("range scan origin (%g, %g) is not finite", cfg->origin_forward, cfg->origin_right);
  if (reinterpret_cast<uintptr_t>(range_dev) & 3) return sim->fail("range scan range target is not aligned to 4 bytes");
  if (reinterpret_cast<uintptr_t>(hit_dev) & 1) return sim->fail("range scan hit target is not aligned to 2 bytes");
  if (hit_dev && check_labels_fit(sim)) return 1;
  sim->scan = ScanTarget{*cfg, range_dev, hit_dev};
  return 0;
}

// The forward maps a flow, bird's-eye visibility, object or lane path target takes: one per fisheye table on a
// DTS_FLAG_DISTORTION handle, none without
static int check_forward_maps(dts_sim* sim, const float* fwd_x, const float* fwd_y, int n_tables) {
  const bool fish = (sim->cfg.flags & DTS_FLAG_DISTORTION) != 0;
  if (fish && (!fwd_x || !fwd_y || n_tables < 1))
    return sim->fail("a DTS_FLAG_DISTORTION handle needs the forward map of every fisheye table (fwd_x, fwd_y, n_tables)");
  if (!fish && (fwd_x || fwd_y || n_tables))
    return sim->fail("forward maps on a handle without DTS_FLAG_DISTORTION: pass NULL, NULL, 0");
  return 0;
}

int dts_set_flow_target(dts_sim* sim, float* flow_dev, const float* fwd_x, const float* fwd_y, int n_tables) {
  if (!sim) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if (!flow_dev && sim->occ.out)
    return sim->fail("the occlusion mask is taken with the flow image: clear it (dts_set_occlusion_target) first");
  if (!flow_dev) {
    DTS_CUDA(cudaDeviceSynchronize());   // no step or render in flight still writes the record or reads the maps
    flow_record_free(sim->flow.rec);
    sim->flow = FlowTarget{};
    if (!reads_forward_maps(sim)) renderer_set_flow_maps(*sim->render, 0, nullptr, nullptr);
    return 0;
  }
  if (reinterpret_cast<uintptr_t>(flow_dev) & 7) return sim->fail("flow target is not aligned to 8 bytes");
  if (!sim->aux.depth || !sim->aux.labels)
    return sim->fail("the flow image is taken from the depth and label images: set both targets first");
  if (check_forward_maps(sim, fwd_x, fwd_y, n_tables)) return 1;
  const bool fish = (sim->cfg.flags & DTS_FLAG_DISTORTION) != 0;
  DTS_CUDA(cudaDeviceSynchronize());
  FlowRecord rec;
  std::string e = flow_record_alloc(rec, sim->cfg.num_envs, largest_n_dyn(sim));
  if (e.empty() && fish) {
    e = renderer_set_flow_maps(*sim->render, n_tables, fwd_x, fwd_y);
    if (!e.empty()) flow_record_free(rec);
  }
  if (!e.empty()) return sim->fail("%s", e.c_str());
  flow_record_free(sim->flow.rec);
  sim->flow = FlowTarget{flow_dev, rec};
  if (sim->occ.out) {   // the new record, and perhaps new forward maps and fisheye tables, start from no frame
    e = occlusion_empty(sim->occ, sim->cfg.num_envs);
    if (!e.empty()) return sim->fail("%s", e.c_str());
  }
  return 0;
}

int dts_set_occlusion_target(dts_sim* sim, uint8_t* occ_dev) {
  if (!sim) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if (occ_dev && !sim->flow.out)
    return sim->fail("the occlusion mask is taken with the flow image: set the flow target (dts_set_flow_target) first");
  DTS_CUDA(cudaDeviceSynchronize());   // no render in flight still reads or writes the slots
  OcclusionTarget occ{};
  if (occ_dev) {
    const std::string e = occlusion_alloc(occ, occ_dev, sim->cfg.num_envs, sim->cfg.cam_width, sim->cfg.cam_height);
    if (!e.empty()) return sim->fail("%s", e.c_str());
  }
  occlusion_free(sim->occ);
  sim->occ = occ;
  return 0;
}

int dts_set_bev_visibility_target(dts_sim* sim, uint8_t* vis_dev, float* pix_dev, const float* fwd_x, const float* fwd_y,
                                  int n_tables) {
  if (!sim) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if (!vis_dev && !pix_dev) {
    DTS_CUDA(cudaDeviceSynchronize());   // no call in flight still reads the forward maps
    sim->bev_view = BevViewTarget{};
    if (!reads_forward_maps(sim)) renderer_set_flow_maps(*sim->render, 0, nullptr, nullptr);
    return 0;
  }
  if (reinterpret_cast<uintptr_t>(pix_dev) & 7) return sim->fail("bird's-eye pixel target is not aligned to 8 bytes");
  if (!sim->bev.labels || !sim->aux.labels)
    return sim->fail("the bird's-eye visibility compares the grid's labels with the frame's: set the bird's-eye label "
                     "target (dts_set_bev_target) and the label target (dts_set_label_target) first");
  if (check_forward_maps(sim, fwd_x, fwd_y, n_tables)) return 1;
  DTS_CUDA(cudaDeviceSynchronize());
  if (sim->cfg.flags & DTS_FLAG_DISTORTION) {
    const std::string e = renderer_set_flow_maps(*sim->render, n_tables, fwd_x, fwd_y);
    if (!e.empty()) return sim->fail("%s", e.c_str());
  }
  sim->bev_view = BevViewTarget{vis_dev, reinterpret_cast<float2*>(pix_dev)};
  return 0;
}

int dts_set_object_target(dts_sim* sim, int max_objects, float* boxes_dev, uint8_t* state_dev, float* corners_dev,
                          const float* fwd_x, const float* fwd_y, int n_tables) {
  if (!sim) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if (!boxes_dev && !state_dev && !corners_dev) {
    DTS_CUDA(cudaDeviceSynchronize());   // no call in flight still reads the forward maps
    sim->objects = ObjectTarget{};
    if (!reads_forward_maps(sim)) renderer_set_flow_maps(*sim->render, 0, nullptr, nullptr);
    return 0;
  }
  if (max_objects < 1 || max_objects > DTS_MAX_OBJECTS)
    return sim->fail("object target of %d objects: 1 to %d are accepted", max_objects, DTS_MAX_OBJECTS);
  const std::vector<MapCounts>& counts = maps_counts(*sim->maps);
  for (size_t s = 0; s < counts.size(); s++)
    if (counts[s].n_objects > max_objects)
      return sim->fail("map slot %zu has %d objects, more than the object target's %d", s, counts[s].n_objects, max_objects);
  if ((reinterpret_cast<uintptr_t>(boxes_dev) | reinterpret_cast<uintptr_t>(corners_dev)) & 3)
    return sim->fail("object box and corner targets must be aligned to 4 bytes");
  if (check_forward_maps(sim, fwd_x, fwd_y, n_tables)) return 1;
  DTS_CUDA(cudaDeviceSynchronize());
  if (sim->cfg.flags & DTS_FLAG_DISTORTION) {
    const std::string e = renderer_set_flow_maps(*sim->render, n_tables, fwd_x, fwd_y);
    if (!e.empty()) return sim->fail("%s", e.c_str());
  }
  sim->objects = ObjectTarget{max_objects, boxes_dev, state_dev, reinterpret_cast<float2*>(corners_dev)};
  return 0;
}

int dts_set_lane_path_target(dts_sim* sim, int n_points, double spacing, float* points_dev, int16_t* count_dev,
                             float* px_dev, const float* fwd_x, const float* fwd_y, int n_tables) {
  if (!sim) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  if (!points_dev && !count_dev && !px_dev) {
    DTS_CUDA(cudaDeviceSynchronize());   // no call in flight still reads the forward maps
    sim->lane_path = LanePathTarget{};
    if (!reads_forward_maps(sim)) renderer_set_flow_maps(*sim->render, 0, nullptr, nullptr);
    return 0;
  }
  if (n_points < 1 || n_points > DTS_LANE_PATH_MAX_POINTS)
    return sim->fail("lane path of %d points: 1 to %d are accepted", n_points, DTS_LANE_PATH_MAX_POINTS);
  if (!(spacing > 0.0 && spacing <= 1.0)) return sim->fail("lane path spacing %g: 0 < spacing <= 1 m is accepted", spacing);
  if ((reinterpret_cast<uintptr_t>(points_dev) | reinterpret_cast<uintptr_t>(px_dev)) & 3)
    return sim->fail("lane path point and pixel targets must be aligned to 4 bytes");
  if (reinterpret_cast<uintptr_t>(count_dev) & 1) return sim->fail("lane path count target is not aligned to 2 bytes");
  if (check_forward_maps(sim, fwd_x, fwd_y, n_tables)) return 1;
  DTS_CUDA(cudaDeviceSynchronize());
  if (sim->cfg.flags & DTS_FLAG_DISTORTION) {
    const std::string e = renderer_set_flow_maps(*sim->render, n_tables, fwd_x, fwd_y);
    if (!e.empty()) return sim->fail("%s", e.c_str());
  }
  sim->lane_path = LanePathTarget{n_points, spacing, points_dev, count_dev, px_dev};
  return 0;
}

int dts_get_frame_cameras(dts_sim* sim, double* V_dev, float* P_dev, void* stream) {
  if (!sim) return 1;
  if (!V_dev || !P_dev) return sim->fail("V_dev and P_dev must not be NULL");
  if (!sim->drawn) return sim->fail("no frame drawn since the handle was created or a map was uploaded");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_frame_cameras(renderer_frame_ctx(*sim->render), sim->cfg.num_envs, V_dev, P_dev, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

int dts_set_marking_target(dts_sim* sim, uint8_t* markings_dev) {
  if (!sim) return 1;
  sim->aux.marks = markings_dev;
  return 0;
}

int dts_resize_frames(dts_sim* sim, const uint8_t* src_dev, void* dst_dev, void* stream) {
  if (!sim) return 1;
  if (!resizer_target(*sim->resize).ow) return sim->fail("dts_set_resize first");
  if (!src_dev || !dst_dev) return sim->fail("NULL frame pointer");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_resize(*sim->resize, src_dev, dst_dev, sim->fmt.obs_layout, sim->fmt.obs_dtype, nullptr, nullptr, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

int dts_status(dts_sim* sim) {
  if (!sim || !sim->h_status) return 0;
  const volatile int32_t* w = sim->h_status;
  return (w[0] ? 1 : 0) | (w[1] ? 2 : 0);
}

// ---- snapshots: every env's state as one record, out of and back into the library's arrays (dts_state.cu) --------
int dts_state_info(dts_sim* sim, uint64_t* record_bytes, uint64_t* fingerprint) {
  if (!sim) return 1;
  if (!state_record_bytes(*sim->state)) return sim->fail("no state record layout: the last map upload could not build it");
  if (record_bytes) *record_bytes = state_record_bytes(*sim->state);
  if (fingerprint) *fingerprint = state_fingerprint(*sim->state);
  return 0;
}

int dts_save_state(dts_sim* sim, void* records_dev, void* stream) {
  if (!sim) return 1;
  if (!records_dev) return sim->fail("records_dev is NULL");
  if (!state_record_bytes(*sim->state)) return sim->fail("no state record layout: the last map upload could not build it");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_state_save(*sim->state, records_dev, (cudaStream_t)stream);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  return 0;
}

int dts_load_state(dts_sim* sim, const uint8_t* mask_dev, const void* records_dev, uint64_t fingerprint, void* stream) {
  if (!sim) return 1;
  if (!records_dev) return sim->fail("records_dev is NULL");
  if (!state_record_bytes(*sim->state)) return sim->fail("no state record layout: the last map upload could not build it");
  const uint64_t mine = state_fingerprint(*sim->state);
  if (fingerprint != mine)
    return sim->fail("record fingerprint %016llx is not this handle's %016llx: the records were saved with other maps "
                     "(or before a map upload) or another record layout", (unsigned long long)fingerprint,
                     (unsigned long long)mine);
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  launch_state_load(*sim->state, mask_dev, records_dev, maps_table(*sim->maps), maps_slot_count(*sim->maps),
                    sim->d_status + 1, (cudaStream_t)stream);
  sim->launches++;
  if (sim->flow.out) {   // a loaded env's flow record would pair its episode number with another state's pose
    launch_flow_forget(sim->flow.rec, sim->occ, mask_dev, sim->cfg.num_envs, (cudaStream_t)stream);
    sim->launches++;
  }
  DTS_CUDA(cudaGetLastError());
  return 0;
}

int dts_profile_enable(dts_sim* sim, int on) {
  if (!sim) return 1;
  sim->profiling = on < 0 ? 0 : (on > 2 ? 2 : on);
  return 0;
}

int dts_profile_read(dts_sim* sim, double ms_out[8], int64_t* frames) {
  if (!sim || !ms_out) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  for (int k = 0; k < 8; k++) ms_out[k] = 0.0;
  const size_t per = kProfMarks;
  DTS_CUDA(cudaDeviceSynchronize());
  for (size_t f = 0; f + per <= sim->prof_events.size(); f += per) {
    for (size_t k = 0; k + 1 < per; k++) {
      float ms = 0.f;   // an interval whose events were not recorded (level 1 marks only k_raster) reports an error: skipped
      if (cudaEventElapsedTime(&ms, sim->prof_events[f + k], sim->prof_events[f + k + 1]) == cudaSuccess) ms_out[k] += ms;
    }
  }
  cudaGetLastError();
  if (frames) *frames = sim->prof_frames;
  for (cudaEvent_t e : sim->prof_events) cudaEventDestroy(e);
  sim->prof_events.clear();
  sim->prof_frames = 0;
  return 0;
}

int dts_set_output_format(dts_sim* sim, const dts_output_format* f) {
  if (!sim) return 1;
  if (!f) return sim->fail("format is NULL");
  if (f->obs_layout < DTS_OBS_HWC || f->obs_layout > DTS_OBS_CWH) return sim->fail("bad obs_layout %d", f->obs_layout);
  if (f->obs_dtype != DTS_OBS_U8 && f->obs_dtype != DTS_OBS_F32_UNIT) return sim->fail("bad obs_dtype %d", f->obs_dtype);
  if (f->reward_mode != DTS_REWARD_RAW && f->reward_mode != DTS_REWARD_DT) return sim->fail("bad reward_mode %d", f->reward_mode);
  if (f->action_map != DTS_ACTIONS_CONTINUOUS && f->action_map != DTS_ACTIONS_DISCRETE3) return sim->fail("bad action_map %d", f->action_map);
  if (f->action_map == DTS_ACTIONS_DISCRETE3 && sim->cfg.action_mode != DTS_ACTION_VEL_STEER)
    return sim->fail("discrete actions are [vel, steering] pairs (DiscreteWrapper wraps DuckietownEnv): action_mode must be VEL_STEER");
  if (f->obs_layout != sim->fmt.obs_layout || f->obs_dtype != sim->fmt.obs_dtype) {
    // the staging frame may be allocated or freed: no render may be using it
    DTS_CUDA(cudaSetDevice(sim->cfg.device));
    DTS_CUDA(cudaDeviceSynchronize());
    const std::string e = resizer_set_format(*sim->resize, f->obs_layout, f->obs_dtype);
    if (!e.empty()) return sim->fail("%s", e.c_str());
  }
  sim->fmt = *f;
  sim->step_cfg.reward_mode = f->reward_mode; sim->step_cfg.action_map = f->action_map;
  sim->step_cfg.action_vel_scale = f->action_vel_scale;
  return 0;
}

int dts_get_dyn_state(dts_sim* sim, int map_id, double** state_dev, int32_t* n_dyn) {
  if (!sim) return 1;
  const DMap* m = maps_get(*sim->maps, map_id);
  if (!m) return sim->fail("bad map_id %d", map_id);
  if (state_dev) *state_dev = m->n_dyn ? m->dyn_state : nullptr;
  if (n_dyn) *n_dyn = m->n_dyn;
  return 0;
}

uint64_t dts_launch_count(dts_sim* sim) { return sim ? sim->launches : 0; }

int dts_debug_episode(dts_sim* sim, int env, void* out144) {
  if (!sim) return 1;
  if (env < 0 || env >= sim->cfg.num_envs) return sim->fail("env out of range");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  DTS_CUDA(cudaMemcpy(out144, state_arrays(*sim->state).rep + env, sizeof(RenderEp), cudaMemcpyDeviceToHost));
  return 0;
}

/* debug: frame setup of `env` in the last dts_render (synchronises) */
int dts_debug_frame(dts_sim* sim, int env, double V[12], float P[4], int32_t counts[4], float* lattice_by_cell, int n_cells) {
  if (!sim) return 1;
  if (env < 0 || env >= sim->cfg.num_envs) return sim->fail("env out of range");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  DTS_CUDA(cudaDeviceSynchronize());
  const std::string e = debug_frame_copy(*sim->render, env, V, P, counts, lattice_by_cell, n_cells);
  return e.empty() ? 0 : sim->fail("%s", e.c_str());
}

/* debug: copy the 32 int32 diagnostic counters (word 0 = overflow flag; 8.. = DTS_STATS counters) */
int dts_debug_counters(dts_sim* sim, int32_t out[32]) {
  if (!sim) return 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  DTS_CUDA(cudaMemcpy(out, sim->d_err, 32 * sizeof(int32_t), cudaMemcpyDeviceToHost));
  return 0;
}

/* debug: every env's stream as [N][6] (dts_seed_streams' layout); synchronises */
int dts_debug_streams(dts_sim* sim, uint64_t* out_host) {
  if (!sim) return 1;
  if (!out_host) return sim->fail("out_host is NULL");
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  DTS_CUDA(cudaDeviceSynchronize());
  const std::string e = state_read_streams(*sim->state, out_host);
  return e.empty() ? 0 : sim->fail("%s", e.c_str());
}

/* debug: a program of NpStream draws from every env's stream (see dtsim.h) */
int dts_debug_draw(dts_sim* sim, const dts_draw_op* ops, int n_ops, uint64_t* out_dev, void* stream) {
  if (!sim) return 1;
  if (!ops || !out_dev || n_ops <= 0) return sim->fail("dts_debug_draw needs ops, n_ops > 0 and out_dev");
  int64_t total = 0;
  for (int k = 0; k < n_ops; k++) {
    const dts_draw_op& op = ops[k];
    if (op.kind < DTS_DRAW_NEXT64 || op.kind > DTS_DRAW_NORMAL || op.count < 0) return sim->fail("bad dts_draw_op %d", k);
    if (op.kind == DTS_DRAW_INTEGERS && !(op.lo < op.hi)) return sim->fail("dts_draw_op %d: integers needs lo < hi", k);
    total += op.count;
  }
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  cudaStream_t st = (cudaStream_t)stream;
  dts_draw_op* d_ops = nullptr;
  DTS_CUDA(cudaMallocAsync((void**)&d_ops, n_ops * sizeof(dts_draw_op), st));
  DTS_CUDA(cudaMemcpyAsync(d_ops, ops, n_ops * sizeof(dts_draw_op), cudaMemcpyHostToDevice, st));
  launch_debug_draw(state_arrays(*sim->state), d_ops, n_ops, total, out_dev, st);
  sim->launches++;
  DTS_CUDA(cudaGetLastError());
  DTS_CUDA(cudaFreeAsync(d_ops, st));
  return 0;
}

// ---- multi-GPU: one NCCL all-gather of the end-of-rollout observation batch (SURVEY 8e) ----------
// libnccl is dlopen'ed (the torch-bundled copy); the communicator is created from a unique id that
// the Python side broadcasts with torch.distributed.

int dts_comm_load(dts_sim* sim, const char* libnccl_path) {
  if (!sim) return 1;
  if (sim->nccl_lib) return 0;
  sim->nccl_lib = dlopen(libnccl_path, RTLD_NOW | RTLD_GLOBAL);
  if (!sim->nccl_lib) return sim->fail("dlopen(%s) failed: %s", libnccl_path, dlerror());
  return 0;
}

int dts_comm_unique_id(dts_sim* sim, uint8_t out[128]) {
  if (!sim || !sim->nccl_lib) return sim ? sim->fail("dts_comm_load first") : 1;
  auto f = (int (*)(void*))dlsym(sim->nccl_lib, "ncclGetUniqueId");
  if (!f) return sim->fail("ncclGetUniqueId not found");
  const int r = f(out);
  return r ? sim->fail("ncclGetUniqueId -> %d", r) : 0;
}

struct nccl_uid { char b[128]; };

int dts_comm_init(dts_sim* sim, const uint8_t id[128], int rank, int world) {
  if (!sim || !sim->nccl_lib) return sim ? sim->fail("dts_comm_load first") : 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  auto f = (int (*)(void**, int, nccl_uid, int))dlsym(sim->nccl_lib, "ncclCommInitRank");
  if (!f) return sim->fail("ncclCommInitRank not found");
  nccl_uid u;
  memcpy(u.b, id, 128);
  const int r = f(&sim->nccl_comm, world, u, rank);
  return r ? sim->fail("ncclCommInitRank -> %d", r) : 0;
}

int dts_allgather_obs(dts_sim* sim, const void* send_dev, void* recv_dev, uint64_t bytes_per_rank, void* stream) {
  if (!sim || !sim->nccl_comm) return sim ? sim->fail("dts_comm_init first") : 1;
  DTS_CUDA(cudaSetDevice(sim->cfg.device));
  auto f = (int (*)(const void*, void*, size_t, int, void*, cudaStream_t))dlsym(sim->nccl_lib, "ncclAllGather");
  if (!f) return sim->fail("ncclAllGather not found");
  const int r = f(send_dev, recv_dev, (size_t)bytes_per_rank, /*ncclUint8*/ 1, sim->nccl_comm, (cudaStream_t)stream);
  return r ? sim->fail("ncclAllGather -> %d", r) : 0;
}

}  // extern "C"
