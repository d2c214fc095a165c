// sdv_ctx.cuh — the context object behind the opaque sdv_ctx handle (host bookkeeping only).
#pragma once
#include <vector>
#include <unordered_map>
#include <mutex>
#include <atomic>
#include "sdv_kernels.cuh"
#include "sdv_core_common.cuh"
#include "../../include/sdv_b200.h"

namespace sdv {

// pinned host twin of Scratch: taken in the same order as its device instance, a staged layout moves in one copy (or one launch_h2d_words)
struct PinnedMem { static cudaError_t alloc(void** p, size_t n) { return cudaMallocHost(p, n); } static void dealloc(void* p) { cudaFreeHost(p); } };
using PinnedScratch = ScratchOf<PinnedMem>;

struct FrameDev {                         // one FrameHessian's images on the device
  uint64_t id; float exposure; bool used;
  float* I0; float* I0_own; bool adopted;  // level-0 intensity plane (own storage, or an adopted caller buffer)
  float* pyr;                             // planar intensity of levels >= 1, level l at the offsets of the frame's own size (frame_layout)
  const float* img[kLevels];              // planar intensity of every level: img[0] = I0, img[l] = pyr + offset of level l
  // packed {I,dx,dy,|grad|^2} texels: a cache built on demand from the planes (ensure_texels) for the keyframe-rate consumers, dropped by a re-ingest.
  // lvl[0] is an image of its pool's keyframe level-0 images (lvl0_slot, -1 if not built); levels >= 1 live in `base` at the offsets of img[l] and are
  // valid while hi_tex is set.
  float4* base; float4* lvl[kLevels]; int lvl0_slot; bool hi_tex;
  long long ingest_seq;                   // ingest call that (re)built this frame's pyramid
  int cam;                                // camera it was ingested for: its size is sdv_ctx::cam_w/cam_h[cam]
  int pool;                               // the FramePool its storage belongs to: 0 (the context's) or a camera with its own (sdv_set_camera_storage)
  bool trk_async;                         // read by tracker-stream work that may still be pending (sdv_ctx::ev_trk_async marks its end)
};

// Storage of frames and keyframe level-0 images of one size.  pools[0] is the context's (sdv_create: max_frames frames and max_kf_images images at the
// context size); pools[k], k >= 1, is camera k's own (sdv_set_camera_storage, at its rectified size), active while n_frames > 0.  The frames themselves
// sit in sdv_ctx::frames, each naming its pool; a frame of a camera with a pool is always claimed from that pool, every other frame from pools[0].
struct FramePool { int w = 0, h = 0, n_frames = 0; std::vector<float4*> lvl0; std::vector<int> lvl0_free; };

struct TrackerSlot {                      // one CoarseTracker instance (reference keeps two: FullSystem.h coarseTracker / coarseTracker_forNewKF)
  float4* pts[kLevels]; int npts[kLevels]; int cap[kLevels];
  uint64_t ref_frame; float refExposure; double ref_a, ref_b;   // lastRef, lastRef_aff_g2l
  double totals[kNAcc]; bool has_totals;                        // reduced sums of the last calc_res (what calcGSSSE reads from buf_warped_*)
  int geom_row;                                                 // row of sdv_ctx::geom this instance's makeK wrote (1 + slot), or 0: the context calibration
  int cam;                                                      // camera of this tracker slot and the map slot of the same index (sdv_set_calib_slots_cams)
};

struct BAState;                           // sdv_ba.cuh
struct RpState;                           // sdv_reproject.cu

} // namespace sdv

struct sdv_ctx {
  // Two call domains, as in the reference (FullSystem::trackMutex / mapMutex): tracker-slot, frame, map and policy entries run under mu_trk on stream `st`;
  // back-end (sdv_ba_*) entries run under mu_ba on stream `st_ba`.  A tracking thread and a mapping thread may therefore use ONE context concurrently.
  // Back-end entries that touch the frame table (set_window, marginalize_frame, clear) take mu_trk as well, always after mu_ba (tracker entries never take mu_ba).
  std::recursive_mutex mu_trk, mu_ba; std::mutex mu_err;
  int device; cudaStream_t st, st_in, st_cp, st_ba; cudaEvent_t ev0, ev1, ev_in, ba_ev0, ba_ev1, ev_xdom; bool ingest_pending; std::atomic<long long> launches;
  float ba_last_ms = 0.f;
  // ingest pipeline: H2D copies on st_cp, pyramids on st_in, one completion event per ingest call (ring); a frame remembers the ingest that built it
  static constexpr int kIngRing = 8; cudaEvent_t ev_ing[kIngRing], ev_cp[2]; long long ingest_seq = 0, seq_waited = 0;
  int w, h, levels; sdv_settings set;
  int cam_w[SDV_MAX_CAMERAS], cam_h[SDV_MAX_CAMERAS];                  // rectified size per camera (sdv_set_camera_size); camera 0 is always w x h
  int cam_levels[SDV_MAX_CAMERAS];                                     // pyramid depth per camera (sdv_set_camera_levels), 1..levels: what its slots and jobs use; frames are stored at `levels`
  sdv::FramePool pools[SDV_MAX_CAMERAS];                               // frame storage: the context's (0) and the cameras' own (sdv_set_camera_storage)
  sdv::TrackConst tc; sdv::TrackConst* tc_dev;
  // geometry table (CoarseTracker::makeK per K): row 0 = the context calibration (sdv_set_calib), row 1 + s = tracker slot s's own K (sdv_set_calib_slots).
  // Host mirror + device copy; every consumer indexes it with TrackerSlot::geom_row, none derives the geometry from K itself.
  std::vector<sdv::GeomRow> geom; sdv::GeomRow* geom_dev;
  std::vector<sdv::FrameDev> frames; std::unordered_map<uint64_t,int> frame_index;
  // frames whose device images are referenced by a resident BA window (BAHeader::frames[].img0) or map slot (MapDev::hostI0): refcount per handle.
  // A pinned frame can be neither released nor re-uploaded (SDV_ERR_STATE) — its pool storage would be handed to another frame under the reader.
  std::unordered_map<uint64_t,int> pins;
  // ingest staging, double-buffered by ingest parity (serves st_in): pyramid descriptors, then the contiguous mono8 images (adjacent host images coalesce into one copy)
  sdv::Scratch ing_dev[2]; sdv::PinnedScratch ing_host[2];
  sdv::UndistortCams und = {}; float* und_buf[SDV_MAX_CAMERAS] = {};                 // sdv_set_undistort_cam: per camera, remap tables (+ response / vignette) of the raw-image ingest
                                                                                    // in one allocation und_buf[k]; a camera is set iff und.cam[k].remapX != nullptr
  // sdv_set_gamma_cam: per camera, the 256 factors gamma_w2 reads (FullSystem::setGammaFunction's B as makeImages weighs |grad|^2 with it), in one allocation
  // of SDV_MAX_CAMERAS rows; a camera without gamma (B[i] = i) passes nullptr to the kernels
  float* gw2_dev = nullptr; bool gamma_set[SDV_MAX_CAMERAS] = {};
  std::vector<void*> cp_dst, cp_src; std::vector<size_t> cp_sz; bool no_batch_copy = false;
  std::vector<sdv::TrackerSlot> slots;
  double* partials; unsigned int* ticket; double* totals_dev; double* totals_host;
  float last_ms;
  // per-call scratch of the tracker stream st (splats, tracker jobs, refine, Reprojector, immature points); valid until the next call that takes from it
  sdv::Scratch scr; sdv::PinnedScratch scr_host;
  cudaEvent_t ev_trk_async = nullptr;           // recorded on st after the last call that returned with a kernel still reading frames (FrameDev::trk_async)
  void* imm_store = nullptr;                    // sdv::ImmStore: device-resident immature points, one block per host keyframe (sdv_trace.cu)
  void* lidar = nullptr;                        // sdv::LidarState: engine of the LiDAR front-end (sdv_lidar.cu)
  void* lidar_rows = nullptr;                   // sdv::RowStore: LiDAR pixel rows per frame handle, FullSystem::qCloudPixel on the device (sdv_lidar.cu)
  void* sel = nullptr;                          // sdv::SelState: PixelSelector slots + engine of the candidate management (sdv_select.cu)
  sdv::RpState* rp = nullptr;                   // map slots + scratch of the Reprojector path (sdv_reproject.cu)
  sdv::BAState* ba = nullptr;                   // selected back-end window
  // ba_wins_dev serves st_ba and holds only the window descriptors, at offset 0: its address keys ba_graph
  std::vector<sdv::BAState*> ba_windows; sdv::Scratch ba_wins_dev; sdv::PinnedScratch ba_wins_host;
  // staging of the batched install and hand-over entries (serves st_ba): a leading part taken alike from both moves in one copy, rows follow on the device
  sdv::Scratch ba_scr; sdv::PinnedScratch ba_scr_host;
  long long ba_waits = 0;                       // host waits on st_ba (sdv_ba_host_wait_count), under mu_ba
  // the fixed Gauss-Newton launch schedule of sdv_ba_optimize_batch as a CUDA graph, keyed by what the launches depend on
  cudaGraphExec_t ba_graph = nullptr; const void* bag_wins = nullptr; int bag_n = 0, bag_maxP = 0, bag_maxR = 0, bag_its = 0;
  char err[512];
};

namespace sdv {
void rp_destroy(sdv_ctx* c);
void sel_destroy(sdv_ctx* c);
void lidar_destroy(sdv_ctx* c);
void imm_store_destroy(sdv_ctx* c);
void lidar_rows_destroy(sdv_ctx* c);
// the header of a frame's LiDAR row set as the handler left it (sdv_lidar_handler_rows_batch)
struct LidarRowsInfo { int rows, overflow, lrud[4], addFeaturePoint, numGround, n_segmented, room; };   // rows: true count; room: rows the set can hold
// row sets of frames[j]: their device rows and headers (one copy back, waits for the tracker stream); SDV_ERR_NOFRAME for a frame without a set
int  lidar_rows_fetch(sdv_ctx* c, int n, const uint64_t* frames, const double** rows_dev, LidarRowsInfo* info, const char* who);
int  sel_n_slots(const sdv_ctx* c);                                                      // selector slots (sdv_selector_init), -1 without a selector
// selector slot `slot` (in range): its camera and its running LiDAR pixel box FullSystem::left/right/up/down (4 ints on the device)
void sel_slot_box(const sdv_ctx* c, int slot, int* cam, int** box_dev);
// makeNewTraces into the store: job j's n[j] records (sel::NewTrace / sel::ImmPt device arrays, stream-ordered on c->st) replace the block of hosts[j]
int  imm_store_deposit(sdv_ctx* c, int nj, const uint64_t* hosts, const int* n, const void* const* new_trace_dev, const void* const* imm_dev);
// one job of the initialiser's point construction (launch_init_points, sdv_trace.cu): n cloud rows {Ku, Kv, depth} with their level-0 status bytes, the job's
// rand() draws, its keyframe's level-0 plane (w x h); out, up to n points each: records, idepth, splat rows {u, v, idepth, HdiF} + round_half, map rows; counts[2] =
// {numPoints[0], points kept}.  All device pointers.
struct InitPointsJob { const double* cloud; const unsigned char* map; const int32_t* draws; const float* I0; int n, w, h; float desired;
                       sdv_immature_pt* pts; sdv_immature_meta* meta; float* idepth; float* splat4; int* round; sdv_map_pt* mp; int* counts; };
int  launch_init_points(sdv_ctx* c, int nj, const InitPointsJob* jobs_dev);
// sdv_tracker_set_ref_batch after its checks (sdv_coarse_depth.cu): makeCoarseDepthL0 of nj jobs and the install with the capacity rule.  Job j is slot
// slots[j] (distinct, in range) with reference frame F[j] = ref_frames[j] (checked against the slot) and the splat rows pt_begin[j] .. pt_begin[j+1] of
// pts4 / round_half, in memory of kind `kind` (cudaMemcpyHostToDevice: host rows inside their slot camera's image, cudaMemcpyDeviceToDevice: device rows).
// ref_ab (2 nj) and npts_out (nj x SDV_PYR_LEVELS) may be NULL.  Waits for the device once; *launches (may be NULL) grows by the kernels it ran.
int  set_ref_build(sdv_ctx* c, int nj, const int32_t* slots, FrameDev* const* F, const uint64_t* ref_frames, const int32_t* pt_begin, const float* pts4,
                   const int32_t* round_half, cudaMemcpyKind kind, const double* ref_ab, int32_t* npts_out, int* launches);
// sdv_map_set_batch with its points already in memory of kind `kind` (cudaMemcpyHostToDevice: host rows, cudaMemcpyDeviceToDevice: device rows)
int  map_set_impl(sdv_ctx* c, int n, const int32_t* slots, const int32_t* host_begin, const uint64_t* host_frames, const double* host_T7, const double* host_ab,
                  const int32_t* pt_begin, const sdv_map_pt* pts, cudaMemcpyKind kind);
int  sel_activate_select(sdv_ctx* c, int n, const int32_t* host_begin, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* uvid,
                         const int32_t* cand_host_begin, const int32_t* cand_begin, const float* cKRKi9, const float* cKt3, const float* cand4, const float* cand4_dev,
                         const float* min_act_dist, const int32_t* cams, int32_t* decision_out, float* dist_map_out);
// frames read by a tracker-stream call that returned before its kernel ran (sdv_immature_trace_store_batch without counts) carry FrameDev::trk_async; frame_fence
// makes an ingest that overwrites such a frame wait for that work on the device, and waits on the host before an adopted buffer is handed back
int  frame_fence(sdv_ctx* c, FrameDev& f, cudaStream_t a, cudaStream_t b, bool host_wait);
int ctx_fail(sdv_ctx* c, int code, const char* fmt, ...);
void ba_destroy(sdv_ctx* c);
int  ensure_lvl0(sdv_ctx* c, FrameDev& f);     // build the packed level-0 texels of a frame on demand (keyframes / read-back)
int  ensure_texels(sdv_ctx* c, FrameDev& f, int lvl);   // f.lvl[lvl] holds the packed texels of that level afterwards (levels >= 1 are built together)
inline void frame_pin(sdv_ctx* c, uint64_t id) { c->pins[id]++; }
inline void frame_unpin(sdv_ctx* c, uint64_t id) { auto it = c->pins.find(id); if (it != c->pins.end() && --it->second <= 0) c->pins.erase(it); }
inline bool frame_pinned(const sdv_ctx* c, uint64_t id) { return c->pins.find(id) != c->pins.end(); }
int  join_ingest(sdv_ctx* c);                  // compute stream waits for every ingest enqueued so far
int  join_ingest_upto(sdv_ctx* c, long long seq);   // ... for ingest calls <= seq only (frames carry their ingest_seq)
inline const GeomRow& slot_geom(const sdv_ctx* c, int slot) { return c->geom[c->slots[slot].geom_row]; }   // the K a tracker / map slot uses, at every level
// the pool a frame of camera cam is claimed from: the camera's own, or the context's
inline int frame_pool_of(const sdv_ctx* c, int cam) { return cam > 0 && c->pools[cam].n_frames > 0 ? cam : 0; }
// frames are depth-agnostic (stored at the context's depth): a frame fits a camera of the same size.  A tracker / map slot holds clouds built at its camera's
// depth as well: it may only keep them on a camera of the same size and depth.
inline const float* cam_gw2(const sdv_ctx* c, int cam) { return c->gamma_set[cam] ? c->gw2_dev + 256*(size_t)cam : nullptr; }   // gamma weights of camera cam, or nullptr
inline bool same_size(const sdv_ctx* c, int cam_a, int cam_b) { return c->cam_w[cam_a] == c->cam_w[cam_b] && c->cam_h[cam_a] == c->cam_h[cam_b]; }
inline bool same_size_depth(const sdv_ctx* c, int cam_a, int cam_b) { return same_size(c, cam_a, cam_b) && c->cam_levels[cam_a] == c->cam_levels[cam_b]; }
inline int slot_levels(const sdv_ctx* c, int slot) { return c->cam_levels[c->slots[slot].cam]; }   // pyrLevelsUsed of a tracker / map slot
int  check_frame_slot(sdv_ctx* c, const FrameDev& f, int slot, const char* who);   // SDV_ERR_ARG (with a message) when frame f's size differs from slot's
int  check_frame_cam(sdv_ctx* c, const FrameDev& f, int cam, const char* who);     // ... from camera cam's (keyframe-rate stages: the job names its camera)
inline FrameDev* find_frame(sdv_ctx* c, uint64_t id) { auto it = c->frame_index.find(id); return it == c->frame_index.end() ? nullptr : &c->frames[it->second]; }
// *out = the frame entry k of `who` names: SDV_ERR_NOFRAME for an unknown handle, SDV_ERR_ARG when its size is not that of tracker / map slot `slot` (slot >= 0) or
// of camera cam (cam >= 0; neither: any size).  *need_seq (if given) rises to the ingest that built it: join_ingest_upto(need_seq) once after the caller's loop.
int  job_frame(sdv_ctx* c, const char* who, int k, uint64_t id, int cam, int slot, long long* need_seq, FrameDev** out);
// SDV_ERR_ARG (with a message) unless every cams[k] of the n is a camera; cams == NULL: every entry is camera 0
int  check_cams(sdv_ctx* c, int n, const int32_t* cams, const char* who, const char* what);
// the argument checks of the batched entries, each SDV_ERR_ARG (with a message) when it fails: the CSR offsets off[0..n] (named `what`) start at 0 and never
// decrease; each of the n ids (slots or windows) is in [0, limit) and none repeats; none of the n frame / host handles repeats
int  check_offsets(sdv_ctx* c, int n, const int32_t* off, const char* who, const char* what);
int  check_ids(sdv_ctx* c, int n, const int32_t* ids, int limit, const char* who, const char* what);
int  check_distinct(sdv_ctx* c, int n, const uint64_t* ids, const char* who, const char* what);
bool sel_cam_bound(const sdv_ctx* c, int cam, int* slot);                          // a selector slot (*slot) is bound to camera cam (sdv_selector_set_slot_cams)
bool rp_slot_set(const sdv_ctx* c, int slot);                                     // map slot `slot` holds a resident map (sdv_map_set, not cleared)
}
// entry-point guards (a NULL context falls through to the entry's own argument check)
#define SDV_GUARD_TRK(c) std::unique_lock<std::recursive_mutex> lk_trk_; if (c) lk_trk_ = std::unique_lock<std::recursive_mutex>((c)->mu_trk)
#define SDV_GUARD_BA(c)  std::unique_lock<std::recursive_mutex> lk_ba_;  if (c) lk_ba_  = std::unique_lock<std::recursive_mutex>((c)->mu_ba)
// a failed CUDA call returns SDV_ERR_CUDA from the enclosing function, with the call and the place in the context's message (needs `c` in scope)
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return sdv::ctx_fail(c, SDV_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } while (0)
