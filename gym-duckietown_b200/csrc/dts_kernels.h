// dts_kernels.h — host-callable launchers of the dtsim kernels.
#pragma once
#include <string>
#include <vector>

#include "dts_common.cuh"

namespace dts {

struct RenderCfg {
  int32_t width, height;      // output obs size
  int32_t flags;
  int32_t n_envs;
  int32_t tessellate;         // 1: literal 98 triangles per road tile (spec tile mode 0)
  int32_t mode;               // DTS_RENDER_* (dts_set_render_mode)
  int32_t all_rows;           // 1: k_bin puts every row on k_raster's list (a gathering step, which ships every row)
  // Optional device list of the envs to draw: env_list[0 .. *env_count).  NULL: all n_envs.  The host never reads the
  // count: grids stay sized for n_envs and slots at or past the count exit.  Frame memory stays indexed by env id, so
  // the envs left out keep what the previous pass put there.  (n_envs stays the SoA stride of the per-env state.)
  const int32_t* env_list;
  const int32_t* env_count;
};

// The per-pixel images the rasterisers write beside obs, for the listed envs only where there is a list; NULL: that
// image is not computed.  Each is [n_envs][height][width]: eye-space depth (dts_set_depth_target), the label
// (dts_set_label_target) and the lane marking (dts_set_marking_target).  Not RenderCfg members: RenderCfg is every render
// kernel's parameter block, and only the rasterisers read these.
struct AuxTargets {
  float* depth;
  int16_t* labels;
  uint8_t* marks;
};

// The camera of one env's frame, per env in frame memory: written by k_frame_setup, read by the render kernels and the
// flow pass (dts_flow.cu)
struct __align__(16) FrameCtx {
  double V[12];                  // agent camera modelview (S:1780-1803)
  float P00, P11, P22, P23;      // gluPerspective (S:1761)
  int32_t n_prims, n_lat, overflow, pad;
};

// The previous frame of the flow image (dts_set_flow_target, dts_flow.cu): what every env's camera and obstacles were at
// the start of its last step, recorded by k_flow_record just before k_step_logic.  `episode` null: no record.
struct FlowRecord {
  double* pose;        // [3][n_envs] pos_x, pos_z, angle
  double* dyn;         // [3][max_dyn][n_envs] DTS_DYN_PX, DTS_DYN_PZ, DTS_DYN_YROT of every dynamic slot of the env's map
  int32_t* episode;    // [2][n_envs] the episode the record belongs to (DState::episode; -1: none), then its step_count
  int32_t max_dyn;     // the largest n_dyn over the uploaded maps
};

void launch_step_logic(const DState& S, const DMap* maps, const StepCfg& c, int n_maps_cycle, const float* actions,
                       float* reward, uint8_t* done, cudaStream_t st);
void launch_reset_random(const DState& S, const DMap* maps, const StepCfg& c, int n_maps_cycle, const uint8_t* mask,
                         cudaStream_t st);
// `p` holds DEVICE copies of the host's episode parameters (state_stage); NULL members keep the defaults
void launch_reset_params(const DState& S, const DMap* maps, const StepCfg& c, const uint8_t* mask,
                         const dts_episode_params& p, cudaStream_t st);
// dts_set_goals: goals int16 [n][2] (device) -> the goal tiles of the envs with mask[e] (null: all); an entry that is not
// a drivable tile of the env's map is not taken and sets *refused (device address of a status word) to 1
void launch_set_goals(const DState& S, const DMap* maps, const uint8_t* mask, const int16_t* goals, int32_t* refused,
                      cudaStream_t st);
void launch_assign_maps(const DState& S, const DMap* maps, const uint8_t* mask, const int32_t* map_id, cudaStream_t st);
// The auto-reset k_step_logic does in place, deferred (dts_step_terminal): every env whose episode ended re-spawns, and
// is appended to ended[0 .. *n_ended), which the caller zeroes first.  The list's order is not deterministic.
void launch_respawn_ended(const DState& S, const DMap* maps, const StepCfg& c, int n_maps_cycle, int32_t* ended,
                          int32_t* n_ended, cudaStream_t st);
void launch_query(const DMap* maps, int map_id, int dyn_env, int n_envs, int n, const double* q, const uint32_t* hidden,
                  double* outd, int32_t* outi, cudaStream_t st);
// dts_debug_draw: every env runs ops[0 .. n_ops) (device copy) from its stream; out[env][0 .. total)
void launch_debug_draw(const DState& S, const dts_draw_op* ops, int n_ops, int64_t total, uint64_t* out, cudaStream_t st);

// Fused end-of-rollout observation gather (SURVEY 8e): on the rollout's last step every frame is stored, besides the
// caller's tensor, straight into the gather buffers of all GPUs of the box — peer memory mapped with cudaIpc, written
// over NVLink — instead of a separate all-gather pass afterwards: by k_raster as it finishes each row of a packed u8 HWC
// frame, or by the format pass (launch_format) for the other layouts and dtypes.
// base[p] = (rank p's gather buffer) + my_rank * bytes_per_rank.
#define DTS_MAX_PEERS 8
struct GatherTab {
  int32_t n, pad;                 // 0: off
  uint8_t* base[DTS_MAX_PEERS];
};

// maps (dts_maps.cu).  The map slots of one handle (dts_upload_map): each slot's DMap, on the host and in the device
// table the kernels index by S.map_id, and the device memory behind it.
struct MapSlots;
// What frame memory is sized from: road tiles, placed objects, and the triangles of the placed meshes and the agent's
// mesh (all zero: an empty slot)
struct MapCounts { int n_tiles, n_objects; long long n_tris; };
MapSlots* maps_create(const dts_config& cfg);   // cfg.max_maps empty slots on the current device; null if out of memory
void maps_destroy(MapSlots* m);
// The blob `b` into `slot`, synchronising the device.  Returns the error text, empty on success.  The whole blob is
// checked and the new map's device memory filled before the slot changes: a refusal or a failed allocation leaves the
// slot, on the host and on the device, as it was.
std::string maps_upload(MapSlots& m, int slot, const dts_map_blob* b);
const DMap* maps_table(const MapSlots& m);           // device [max_maps]
// device [max_maps]: each slot's objects' (least, largest) object-space mesh y, [n_objects] (null: an empty slot)
const float2* const* maps_extent_table(const MapSlots& m);
const DMap* maps_get(const MapSlots& m, int slot);   // the slot's host record; null if out of range or empty
const std::vector<MapCounts>& maps_counts(const MapSlots& m);   // [max_maps]
int maps_slot_count(const MapSlots& m);                           // max_maps
// Content hash of the blob the slot's map was built from (never 0); 0 for an empty slot
uint64_t maps_hash(const MapSlots& m, int slot);

// per-env state (dts_state.cu).  The envs' simulator state of one handle: the DState arrays, the staging buffers of
// dts_reset, the snapshot record layout with its fingerprint, and whether the envs' streams are seeded.  One table,
// kStateArrays, is the single statement of the per-env state: it allocates the arrays and lays out the records.
// Functions that can fail return the error text, empty on success.
struct EnvState;
// On the current device, the records laid out for the maps now in `maps`; null (and `err`) if out of memory
EnvState* state_create(const dts_config& cfg, const MapSlots& maps, std::string& err);
void state_destroy(EnvState* s);
const DState& state_arrays(const EnvState& s);   // what the launchers take
dts_state_view state_view(const EnvState& s);
bool state_seeded(const EnvState& s);   // dts_seed_streams or dts_load_state has given the envs their streams
// streams[N][6] (dts_seed_streams' layout, HOST) -> the streams of the envs with mask_host[e] (null: all); synchronous
std::string state_seed_streams(EnvState& s, const uint8_t* mask_host, const uint64_t* streams);
// every env's stream -> out[N][6] (HOST); synchronous on the legacy stream
std::string state_read_streams(const EnvState& s, uint64_t* out);
// The host arrays of `host` -> the staging buffers, on `st`; `dev` gets their device addresses, null where `host` has
// none.  The host arrays must stay unchanged until `st` has passed the copies.
std::string state_stage(EnvState& s, const dts_episode_params& host, dts_episode_params& dev, cudaStream_t st);
// Re-lay the records out for the maps now in `maps` (after every map upload).  Synchronous; no save or load may be in
// flight.
std::string state_layout(EnvState& s, const MapSlots& maps);
uint64_t state_record_bytes(const EnvState& s);   // one env's record, a multiple of 16; 0: the last layout failed
uint64_t state_fingerprint(const EnvState& s);
// records u8[n_envs][record_bytes] <- every env's state
void launch_state_save(const EnvState& s, void* records, cudaStream_t st);
// every env e with mask[e] (null: all) whose record names an uploaded map in `maps[0 .. n_maps)` <- record e; an env
// whose record names none keeps its state, and `refused` (device address of a status word) is set to 1.  The envs'
// streams count as seeded from then on.
void launch_state_load(EnvState& s, const uint8_t* mask, const void* records, const DMap* maps, int n_maps,
                       int32_t* refused, cudaStream_t st);

// render (dts_render.cu).  The renderer of one handle: the launch sizes, the frame memory, sized from the uploaded maps,
// and the fisheye tables.  Functions that can fail return the error text, empty on success.
struct Renderer;
Renderer* renderer_create(const dts_config& cfg);   // on cfg.device, which must be current
void renderer_destroy(Renderer* r);
void renderer_release_frame(Renderer& r);   // the maps changed: the next render re-sizes frame memory for them
// Before every render: reserves frame memory for the maps of `counts` unless it is reserved, and checks that a fisheye
// LUT is set if the camera needs one, a rectification LUT if render `mode` asks for it, and (`forward`: a flow, bird's-eye
// visibility, object or lane path target is set) the fisheye tables' forward maps if the frame goes through them.
std::string renderer_prepare(Renderer& r, const std::vector<MapCounts>& counts, int mode, bool forward);
// The rasteriser's remap table for a LUT of the camera's size (obs[y, x] = frame[rint(rmapy), rint(rmapx)]), in the
// fisheye slot or (`rectify`) the rectification slot; it replaces that slot's previous one, so no render may be in
// flight.  A LUT the rasteriser cannot take leaves the previous table; NULL maps free the slot.  A fisheye pool: `count`
// LUTs back to back in rmapx / rmapy, env e remapped through LUT lut_of_env[e] (HOST, [n_envs], checked by the caller;
// read only when count > 1, and then kept in the table).  The rectification slot takes one LUT.
std::string renderer_set_lut(Renderer& r, bool rectify, int count, const float* rmapx, const float* rmapy,
                             const int32_t* lut_of_env);
// The forward maps of the fisheye tables (F of the flow image and the bird's-eye visibility): `count` float32 [H][W] tables of x
// and of y back to back, one per table of the fisheye pool and in its order; they replace the previous ones.  Refused
// (error text, previous maps kept) unless the fisheye slot holds exactly `count` tables.  NULL maps free them.  A new
// fisheye LUT (renderer_set_lut) drops them with the tables they belong to.
std::string renderer_set_flow_maps(Renderer& r, int count, const float* fwd_x, const float* fwd_y);
// `marks`: NULL or kProfMarks events recorded on `st` before k_frame_setup and after each of k_frame_setup, k_geometry,
// k_bin, k_raster and the post passes (dts_profile_*).  `status_dev`: device address of the mapped host status word.
// `flow`: the flow image's target (dts_flow.cu), launched after the rasterisers over the same envs; null `out`: none.
// `occ`: its occlusion mask; null `out`: none.
struct FlowTarget;
struct OcclusionTarget;
constexpr int kProfMarks = 6;
int launch_render(const Renderer& r, const DState& S, const DMap* maps, const RenderCfg& rc, const AuxTargets& aux,
                  const FlowTarget& flow, const OcclusionTarget& occ, void* obs, const GatherTab& gather, int32_t* err_flag, int32_t* status_dev,
                  cudaEvent_t* marks, int mark_level, cudaStream_t st);
// Every env's camera of the last render (k_frame_setup's), device [n_envs]; null while no frame memory is reserved
const FrameCtx* renderer_frame_ctx(const Renderer& r);
struct FlowRemap;
// The remap a render in `mode` goes through, as the passes after it read it (flow, bird's-eye visibility)
FlowRemap renderer_remap(const Renderer& r, int mode);
// What the last render left in frame memory for one env (dts_debug_frame), after the device has synchronised
std::string debug_frame_copy(const Renderer& r, int env, double* V, float* P, int32_t* counts, float* lattice_by_cell,
                             int n_cells);

// post passes (dts_post.cu).  The rasterisers draw packed u8 HWC at the camera size.  Where the caller's obs is anything
// else, they draw into a staging frame and a post pass writes obs: the ResizeWrapper (dts_set_resize_filter) or the
// format pass (dts_set_output_format).  A Resizer is the one handle's setting of both, their tables and the staging frame.
struct Resizer;
Resizer* resizer_create(const dts_config& cfg);   // no resize, packed u8 HWC
void resizer_destroy(Resizer* z);
// `filter` (DTS_RESIZE_*) from the camera to ow x oh, 0 x 0: off; on the handle's device, with no render in flight.  A
// target the filter refuses (Pillow: less than 1/32 of the camera size) or a failed allocation returns the error text
// and leaves the previous setting.
std::string resizer_set(Resizer& z, int filter, int ow, int oh);
// The caller's obs layout and dtype (DTS_OBS_*), with no render in flight.  A failed allocation of the staging frame
// returns the error text and leaves the previous setting.
std::string resizer_set_format(Resizer& z, int layout, int dtype);
// 0 x 0: no resize.  staging: u8[N][H][W][3], the full-size frames; null while the rasterisers write obs themselves.
struct ResizeTarget { int ow, oh; uint8_t* staging; };
ResizeTarget resizer_target(const Resizer& z);
// src u8[N][H][W][3] -> dst [N] x (ow x oh) in `layout` / `dtype`, over an optional device env list like RenderCfg's
void launch_resize(const Resizer& z, const uint8_t* src, void* dst, int layout, int dtype, const int32_t* env_list,
                   const int32_t* env_count, cudaStream_t st);
// The staging frames -> dst at the camera size in z's layout / dtype (no resize target), and on a gathering step
// (gt.n > 0) into every peer's gather slot as well, over an optional device env list like RenderCfg's
void launch_format(const Resizer& z, void* dst, const GatherTab& gt, const int32_t* env_list, const int32_t* env_count,
                   cudaStream_t st);
// dst row e = src row e (row_bytes each) for every env e of list[0 .. *count), count <= n_envs
void launch_copy_rows(const void* src, void* dst, size_t row_bytes, const int32_t* list, const int32_t* count, int n_envs,
                      cudaStream_t st);
void launch_blend4(const uint8_t* const f[4], const double w[4], double* out, size_t n, cudaStream_t st);

// bird's-eye map (dts_bev.cu): the grid of dts_set_bev_target and its outputs, each [n_envs][height][width] or null
struct BevTarget {
  dts_bev_config cfg;
  int16_t* labels;
  uint8_t* marks;
};
// every env's grid of its current state, one launch
void launch_bev(const DState& S, const DMap* maps, const BevTarget& b, cudaStream_t st);
// The camera visibility of the grid (dts_set_bev_visibility_target, DESIGN.md section 5 item 15): uint8 [n_envs][height]
// [width] and the pixel of every cell, float32 x, y; either null.  Both null: off.
struct BevViewTarget {
  uint8_t* vis;
  float2* pix;
};
// The range scan of dts_set_scan_target (DESIGN.md section 5 item 16): float32 range and int16 hit, each
// [n_envs][n_rays] or null
struct ScanTarget {
  dts_scan_config cfg;
  float* range;
  int16_t* hit;
};
// every env's scan of its current state, one launch; max_objects: the most objects of an uploaded map
void launch_scan(const DState& S, const DMap* maps, const ScanTarget& sc, int max_objects, cudaStream_t st);
// every env's cameras V [n_envs][12] and P [n_envs][4] from `ctx` (dts_get_frame_cameras), one launch
void launch_frame_cameras(const FrameCtx* ctx, int n_envs, double* V, float* P, cudaStream_t st);

// motion flow (dts_flow.cu): the image of dts_set_flow_target, float32 [n_envs][H][W][2], and the record it is taken
// against.  Null `out`: off, and then the record is unallocated.
struct FlowTarget {
  float* out;
  FlowRecord rec;
};
// The occlusion mask of dts_set_occlusion_target (DESIGN.md section 5 item 14), uint8 [n_envs][H][W], and the two
// slots per env holding the frames it is taken against.  Null `out`: off, and then nothing is allocated.
struct OcclusionTarget {
  uint8_t* out;
  float* depth;        // [2][n_envs][H][W] each slot's depth image
  int16_t* labels;     // [2][n_envs][H][W] each slot's label image
  int32_t* tag;        // [2][3][n_envs] each slot's frame: its episode (-1: empty), step_count and view (occ_view)
  uint8_t* newest;     // [n_envs] the slot written last
};
// What the flow pass reads of the frame's remap: nothing (src_xy null: the pinhole frame), the fisheye table or pool
// with its forward maps (fwd: [tables][H][W], the env's table named by table_of_env where that is not null), or the
// rectification, whose forward map does not exist: every pixel NaN.
struct FlowRemap {
  const int32_t* src_xy;
  const uint16_t* table_of_env;
  const float2* fwd;
  bool rectify;
};
// Every env's visibility of the grid `b` (its labels, written by k_bev earlier in the call) in the frame the call drew:
// its camera in `ctx`, its label image `labels` [n_envs][H][W] and remap `rm`; drew_frame false (ctx and labels unread):
// every cell UNKNOWN.  One launch.
void launch_bev_view(const DState& S, const DMap* maps, const BevTarget& b, const BevViewTarget& v, const FrameCtx* ctx,
                     const int16_t* labels, int W, int H, const FlowRemap& rm, bool drew_frame, cudaStream_t st);
// objects (dts_objects.cu).  The object boxes of dts_set_object_target (DESIGN.md section 5 item 17), each
// [n_envs][max_objects][...] or null: float32 boxes [7], uint8 state, float32 corner pixels [9][2].  All null: off.
struct ObjectTarget {
  int32_t max_objects;
  float* boxes;
  uint8_t* state;
  float2* corners;
};
// Every env's object boxes of its current state and, where drew_frame (ctx read), where their corners land in the frame
// the call drew: its camera in `ctx` and remap `rm` at W x H; else every corner NaN.  `extent`: maps_extent_table.
// One launch.
void launch_objects(const DState& S, const DMap* maps, const float2* const* extent, const ObjectTarget& t,
                    const FrameCtx* ctx, int W, int H, const FlowRemap& rm, bool drew_frame, cudaStream_t st);
// Every env's object pixel statistics (dts_object_pixels) from its label image labels [n_envs][H][W]: pixels int32
// [n_envs][max_objects] and boxes int32 [n_envs][max_objects][4].  One launch.
void launch_object_pixels(const DState& S, const DMap* maps, const int16_t* labels, int W, int H, int32_t* pixels,
                          int32_t* boxes, int max_objects, cudaStream_t st);
// lane path (dts_path.cu).  The lane path of dts_set_lane_path_target (DESIGN.md section 5 item 18), each
// [n_envs][n_points][...] or null: float32 points [3], int16 count [n_envs], float32 pixels [2].  All null: off.
struct LanePathTarget {
  int32_t n_points;
  double spacing;
  float* points;
  int16_t* count;
  float* px;
};
// Every env's lane path from its current state and, where drew_frame (ctx read), where its points land in the frame the
// call drew: its camera in `ctx` and remap `rm` at W x H; else every pixel NaN.  One launch.
void launch_lane_path(const DState& S, const DMap* maps, const LanePathTarget& t, const FrameCtx* ctx, int W, int H,
                      const FlowRemap& rm, bool drew_frame, cudaStream_t st);
// A record for n_envs envs and max_dyn dynamic slots, every env's record invalid (episode -1); synchronous.  On failure
// (error text) `rec` is untouched.
std::string flow_record_alloc(FlowRecord& rec, int n_envs, int max_dyn);
void flow_record_free(FlowRecord& rec);
// every env's camera and obstacles now, as the previous frame of its next render: launched just before k_step_logic
void launch_flow_record(const DState& S, const DMap* maps, const FlowRecord& rec, cudaStream_t st);
// every env e with mask[e] (null: all) forgets its previous frame (episode -1) and, where `occ` is set, empties its
// occlusion slots; stream-ordered
void launch_flow_forget(const FlowRecord& rec, const OcclusionTarget& occ, const uint8_t* mask, int n_envs,
                        cudaStream_t st);
// Slots for n_envs frames of width x height, all empty, and the mask at `out`; synchronous.  On failure (error text)
// `occ` is untouched.
std::string occlusion_alloc(OcclusionTarget& occ, uint8_t* out, int n_envs, int width, int height);
std::string occlusion_empty(const OcclusionTarget& occ, int n_envs);   // every slot; synchronous
void occlusion_free(OcclusionTarget& occ);
// The flow image of the listed envs (rc.env_list, or all) from the depth and label images the render just wrote and
// the frames' cameras in `ctx`; with `occ.out`, also the occlusion mask, then the slots' tags.  Returns the launches.
int launch_flow(const DState& S, const DMap* maps, const RenderCfg& rc, const FrameCtx* ctx, const AuxTargets& aux,
                const FlowTarget& f, const FlowRemap& rm, const OcclusionTarget& occ, cudaStream_t st);

}  // namespace dts
