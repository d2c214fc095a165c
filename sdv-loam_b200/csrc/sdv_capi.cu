// sdv_capi.cu — context + extern "C" boundary (include/sdv_b200.h).  Host logic only; all numerics run in the kernels of
// sdv_kernels.cu / sdv_ba_kernels.cu.  There is deliberately NO CPU fallback: every entry point fails with SDV_ERR_CUDA when
// the device path is unavailable.
#include "../../include/sdv_b200.h"
#include "sdv_ctx.cuh"
#include "sdv_refine.cuh"
#include <cstdio>
#include <cstring>
#include <cstdarg>
#include <cmath>
#include <algorithm>

using namespace sdv;

namespace sdv {
int ctx_fail(sdv_ctx* c, int code, const char* fmt, ...) {
  if (c) { std::lock_guard<std::mutex> lk(c->mu_err); va_list ap; va_start(ap, fmt); vsnprintf(c->err, sizeof(c->err), fmt, ap); va_end(ap); }
  return code;
}
}

extern "C" {

void sdv_default_settings(sdv_settings* s) {
  s->huberTH = 6; s->coarseCutoffTH = 20; s->affineOptModeA = 0; s->affineOptModeB = 0;
  s->outlierTH = 12*12; s->outlierTHSumComponent = 50*50; s->idepthFixPrior = 50*50;
  s->max_ref_points = 0; s->n_tracker_slots = 2; s->max_frames = 16; s->cluster_size = 1; s->track_threads = 128; s->max_kf_images = 0;
}

int sdv_pyr_levels(int w, int h) {               // util/globalCalib.cpp:22-30
  int wl = w, hl = h, used = 1;
  while (wl%2==0 && hl%2==0 && wl*hl > 5000 && used < SDV_PYR_LEVELS) { wl/=2; hl/=2; used++; }
  return used;
}

static thread_local char g_create_err[512] = "null context";   // message of the last failed sdv_create on this thread (there is no context to hold it)
const char* sdv_last_error(sdv_ctx* c) { return c ? c->err : g_create_err; }

// CoarseTracker::makeK (CoarseTracker.cpp:77-106) into one row of the geometry table, at camera cam's rectified size
static void make_geom(sdv_ctx* c, const sdv_calib* K, int row, int cam) {
  float fx[SDV_PYR_LEVELS], fy[SDV_PYR_LEVELS], cx[SDV_PYR_LEVELS], cy[SDV_PYR_LEVELS];
  fx[0]=K->fx; fy[0]=K->fy; cx[0]=K->cx; cy[0]=K->cy;
  for (int l=1;l<c->levels;l++) {
    fx[l] = fx[l-1]*0.5; fy[l] = fy[l-1]*0.5;
    cx[l] = (cx[0]+0.5)/((int)1<<l) - 0.5; cy[l] = (cy[0]+0.5)/((int)1<<l) - 0.5;
  }
  for (int l=0;l<c->levels;l++) {
    LevelGeom& g = c->geom[row].g[l]; g.w = c->cam_w[cam]>>l; g.h = c->cam_h[cam]>>l; g.fx=fx[l]; g.fy=fy[l]; g.cx=cx[l]; g.cy=cy[l];
    float Km[9] = {fx[l],0,cx[l], 0,fy[l],cy[l], 0,0,1}; inv3f(Km, g.Ki);
  }
}

// rows [lo, hi] of the host mirror to the device, stream-ordered after the work already enqueued on the compute stream (pageable source: staged before the call returns)
static int upload_geom(sdv_ctx* c, int lo, int hi) {
  CK(cudaMemcpyAsync(c->geom_dev + lo, &c->geom[lo], (size_t)(hi - lo + 1)*sizeof(GeomRow), cudaMemcpyHostToDevice, c->st));
  return SDV_OK;
}

// CoarseTracker::makeK(HCalib) / the CalibHessian the Reprojector reads (FullSystem::optimize moves the intrinsics at every keyframe): the context calibration,
// used by every later call on a slot without a K of its own.
int sdv_set_calib(sdv_ctx* c, const sdv_calib* K) { SDV_GUARD_TRK(c);
  if (!c || !K) return SDV_ERR_ARG;
  if (!(K->fx > 0 && K->fy > 0)) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_calib: focal lengths must be positive");
  CK(cudaSetDevice(c->device));
  make_geom(c, K, 0, 0);
  return upload_geom(c, 0, 0);
}

// CoarseTracker::makeK per tracker instance: slot slots[i] uses K[i] (its own row 1 + slot, built at camera cams[i]'s size), or the context calibration
// again when K is NULL (camera 0 only: row 0 has the context size).  Everything is checked before anything changes.
int sdv_set_calib_slots_cams(sdv_ctx* c, int n, const int32_t* slots, const sdv_calib* K, const int32_t* cams) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n > 0 && !slots)) return SDV_ERR_ARG;
  { int rc = check_cams(c, n, cams, "sdv_set_calib_slots", "entry"); if (rc) return rc; }
  for (int i=0;i<n;i++) {
    if (slots[i] < 0 || slots[i] >= (int)c->slots.size()) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_calib_slots: entry %d names slot %d of %d", i, slots[i], (int)c->slots.size());
    if (K && !(K[i].fx > 0 && K[i].fy > 0 && std::isfinite(K[i].fx) && std::isfinite(K[i].fy) && std::isfinite(K[i].cx) && std::isfinite(K[i].cy)))
      return ctx_fail(c, SDV_ERR_ARG, "sdv_set_calib_slots: entry %d (slot %d): fx, fy must be positive and finite, cx, cy finite", i, slots[i]);
    const int cam = cams ? cams[i] : 0;
    if (!K && cam != 0) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_calib_slots: entry %d binds camera %d without a K (the context calibration is camera 0's)", i, cam);
  }
  for (int i=0;i<n;i++) {                                                // a slot's reference cloud and resident map hold frames of its current size, built at its current depth
    const TrackerSlot& t = c->slots[slots[i]]; const int cam = cams ? cams[i] : 0;
    if (!same_size_depth(c, t.cam, cam) && (t.ref_frame != ~0ull || rp_slot_set(c, slots[i])))
      return ctx_fail(c, SDV_ERR_STATE, "sdv_set_calib_slots: entry %d would move slot %d from camera %d (%dx%d, %d levels) to camera %d (%dx%d, %d levels) while its %s holds frames of the old camera",
                      i, slots[i], t.cam, c->cam_w[t.cam], c->cam_h[t.cam], c->cam_levels[t.cam], cam, c->cam_w[cam], c->cam_h[cam], c->cam_levels[cam],
                      t.ref_frame != ~0ull ? "tracker reference" : "map");
  }
  CK(cudaSetDevice(c->device));
  int lo = (int)c->geom.size(), hi = -1;
  for (int i=0;i<n;i++) {
    TrackerSlot& t = c->slots[slots[i]]; t.cam = cams ? cams[i] : 0;
    if (!K) { t.geom_row = 0; continue; }
    t.geom_row = 1 + slots[i]; make_geom(c, &K[i], t.geom_row, t.cam); lo = std::min(lo, t.geom_row); hi = std::max(hi, t.geom_row);
  }
  return hi >= lo ? upload_geom(c, lo, hi) : SDV_OK;
}
int sdv_set_calib_slots(sdv_ctx* c, int n, const int32_t* slots, const sdv_calib* K) { return sdv_set_calib_slots_cams(c, n, slots, K, nullptr); }

// A camera's rectified size: at most the context size, with the context's pyramid depth.  Refused while anything depends on the old size, its own
// frame pool included (sized for the old size).
int sdv_set_camera_size(sdv_ctx* c, int cam, int w, int h) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG;
  if (cam == 0) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_camera_size: camera 0 always has the context size %dx%d", c->w, c->h);
  if (cam < 1 || cam >= SDV_MAX_CAMERAS) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_camera_size: camera %d outside 1..%d", cam, SDV_MAX_CAMERAS - 1);
  if (w < 1 || h < 1 || w > c->w || h > c->h) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_camera_size: %dx%d does not fit the context size %dx%d", w, h, c->w, c->h);
  if (c->levels > 1 && ((w | h) & 1)) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_camera_size: %dx%d: the pyramid needs even image sizes", w, h);
  if ((w >> (c->levels - 1)) < 1 || (h >> (c->levels - 1)) < 1) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_camera_size: %dx%d has an empty level at the context's %d levels", w, h, c->levels);
  if (w == c->cam_w[cam] && h == c->cam_h[cam]) return SDV_OK;
  if (c->und.cam[cam].remapX) return ctx_fail(c, SDV_ERR_STATE, "sdv_set_camera_size: camera %d has Undistort tables of its current size", cam);
  if (c->pools[cam].n_frames > 0) return ctx_fail(c, SDV_ERR_STATE, "sdv_set_camera_size: camera %d has a frame pool of its current size (sdv_set_camera_storage)", cam);
  for (const FrameDev& f : c->frames) if (f.used && f.cam == cam) return ctx_fail(c, SDV_ERR_STATE, "sdv_set_camera_size: camera %d has resident frame %llu", cam, (unsigned long long)f.id);
  for (size_t s=0;s<c->slots.size();s++) if (c->slots[s].cam == cam) return ctx_fail(c, SDV_ERR_STATE, "sdv_set_camera_size: slot %d is bound to camera %d", (int)s, cam);
  { int s; if (sel_cam_bound(c, cam, &s)) return ctx_fail(c, SDV_ERR_STATE, "sdv_set_camera_size: selector slot %d is bound to camera %d", s, cam); }
  c->cam_w[cam] = w; c->cam_h[cam] = h;
  return SDV_OK;
}

// A camera's pyramid depth (pyrLevelsUsed): what its tracker / map slots and jobs use, at most the context's storage depth.  Refused while a slot of the
// camera holds clouds or a map built at the old depth, and below the selector's 3 levels while a selector slot is bound to it.
int sdv_set_camera_levels(sdv_ctx* c, int cam, int levels) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG;
  { int rc = check_cams(c, 1, &cam, "sdv_set_camera_levels", nullptr); if (rc) return rc; }
  if (levels < 1 || levels > c->levels) return ctx_fail(c, SDV_ERR_ARG, "sdv_set_camera_levels: %d levels outside 1..%d (the context's storage depth)", levels, c->levels);
  if (levels == c->cam_levels[cam]) return SDV_OK;
  for (size_t s=0;s<c->slots.size();s++) if (c->slots[s].cam == cam && (c->slots[s].ref_frame != ~0ull || rp_slot_set(c, (int)s)))
    return ctx_fail(c, SDV_ERR_STATE, "sdv_set_camera_levels: slot %d of camera %d holds a %s built at %d levels", (int)s, cam,
                    c->slots[s].ref_frame != ~0ull ? "tracker reference" : "map", c->cam_levels[cam]);
  { int s; if (levels < 3 && sel_cam_bound(c, cam, &s)) return ctx_fail(c, SDV_ERR_STATE, "sdv_set_camera_levels: selector slot %d is bound to camera %d and reads levels 0..2", s, cam); }
  c->cam_levels[cam] = levels;
  return SDV_OK;
}

// ------------------------------------------------------------------------------------------------ frame storage
// One frame of a pool of w x h: planar intensity of every level (level 0, plus one allocation for levels >= 1) and the storage of the packed-texel cache
// of levels >= 1, both at the offsets of the frame's own size (frame_layout); packed level-0 texels come from the pool's keyframe level-0 images.
static size_t pyr_texels(int w, int h, int levels) { size_t n = 0; for (int l=1;l<levels;l++) n += (size_t)(w>>l)*(h>>l); return n; }
static uint64_t frame_bytes(int w, int h, int levels) { return (uint64_t)w*h*sizeof(float) + pyr_texels(w, h, levels)*(sizeof(float) + sizeof(float4)); }
static uint64_t kf_image_bytes(int w, int h) { return (uint64_t)w*h*sizeof(float4); }
static int kf_count(int max_kf_images, int max_frames) { const int n = max_kf_images > 0 ? max_kf_images : SDV_MAX_FRAMES_WINDOW + 4; return n > max_frames ? max_frames : n; }
// every field set before the first allocation, so frame_free is safe on a frame whose allocation failed half way
static cudaError_t frame_alloc(FrameDev& f, int pool, int w, int h, int levels) {
  f = FrameDev{}; f.lvl0_slot = -1; f.pool = pool;
  const size_t texels = pyr_texels(w, h, levels);
  cudaError_t e = cudaMalloc(&f.I0_own, (size_t)w*h*sizeof(float)); f.I0 = f.I0_own; f.img[0] = f.I0;
  if (e == cudaSuccess && texels) e = cudaMalloc(&f.pyr, texels*sizeof(float));
  if (e == cudaSuccess && texels) e = cudaMalloc(&f.base, texels*sizeof(float4));
  return e;
}
static void frame_free(FrameDev& f) { cudaFree(f.base); cudaFree(f.pyr); cudaFree(f.I0_own); f.base = nullptr; f.pyr = nullptr; f.I0_own = nullptr; }
static cudaError_t kf_alloc(FramePool& P, int n, int w, int h) {
  P.lvl0.assign(n, nullptr); P.lvl0_free.clear();
  for (int i=0;i<n;i++) { cudaError_t e = cudaMalloc(&P.lvl0[i], kf_image_bytes(w, h)); if (e != cudaSuccess) return e; P.lvl0_free.push_back(n-1-i); }
  return cudaSuccess;
}
static void kf_free(FramePool& P) { for (float4* p : P.lvl0) cudaFree(p); P.lvl0.clear(); P.lvl0_free.clear(); }
// where the levels >= 1 of a frame of camera f.cam sit in its storage: level l at the sum of the sizes of levels 1..l-1 of the camera's own size, in every
// pool (pyr_fused_kernel writes them there); set whenever the frame is claimed for a camera
static void frame_layout(const sdv_ctx* c, FrameDev& f) {
  const int w = c->cam_w[f.cam], h = c->cam_h[f.cam]; size_t off = 0;
  for (int l=1;l<c->levels;l++) { f.img[l] = f.pyr + off; f.lvl[l] = f.base + off; off += (size_t)(w>>l)*(h>>l); }
}

// Camera cam's own frame pool: max_frames frames and max_kf_images keyframe level-0 images (0: the default, at most max_frames) at its rectified size, or,
// with max_frames == 0, none (its frames come from the context pool again).  Refused while a frame of the pool is resident or one of its keyframe images is
// taken.  All-or-nothing: the new pool is allocated before the old one is freed.
int sdv_set_camera_storage(sdv_ctx* c, int cam, int max_frames, int max_kf_images) { SDV_GUARD_TRK(c);
  const char* who = "sdv_set_camera_storage";
  if (!c) return SDV_ERR_ARG;
  if (cam < 1 || cam >= SDV_MAX_CAMERAS) return ctx_fail(c, SDV_ERR_ARG, "%s: camera %d outside 1..%d (camera 0 uses the context pool)", who, cam, SDV_MAX_CAMERAS - 1);
  if (max_frames < 0 || max_kf_images < 0) return ctx_fail(c, SDV_ERR_ARG, "%s: negative count (max_frames %d, max_kf_images %d)", who, max_frames, max_kf_images);
  FramePool& P = c->pools[cam];
  for (const FrameDev& f : c->frames) if (f.used && f.pool == cam)
    return ctx_fail(c, SDV_ERR_STATE, "%s: frame %llu of camera %d's pool is resident: release it first", who, (unsigned long long)f.id, cam);
  if (P.lvl0_free.size() != P.lvl0.size()) return ctx_fail(c, SDV_ERR_STATE, "%s: a keyframe image of camera %d's pool is taken", who, cam);
  if (max_frames == 0 && P.n_frames == 0) return SDV_OK;
  CK(cudaSetDevice(c->device));
  CK(cudaStreamSynchronize(c->st_cp)); CK(cudaStreamSynchronize(c->st_in)); CK(cudaStreamSynchronize(c->st)); CK(cudaStreamSynchronize(c->st_ba));   // work enqueued before may still read the old pool's released frames
  const int w = c->cam_w[cam], h = c->cam_h[cam];
  std::vector<FrameDev> nf(max_frames); FramePool np; np.w = w; np.h = h; np.n_frames = max_frames;
  cudaError_t e = cudaSuccess;
  for (auto& f : nf) if ((e = frame_alloc(f, cam, w, h, c->levels)) != cudaSuccess) break;
  if (e == cudaSuccess && max_frames > 0) e = kf_alloc(np, kf_count(max_kf_images, max_frames), w, h);
  if (e != cudaSuccess) {
    cudaGetLastError(); for (auto& f : nf) frame_free(f); kf_free(np);
    return ctx_fail(c, SDV_ERR_CUDA, "%s: camera %d: %d frames and their keyframe images of %dx%d -> %s (the old pool is kept)", who, cam, max_frames, w, h, cudaGetErrorString(e));
  }
  std::vector<FrameDev> keep; keep.reserve(c->frames.size() + nf.size());
  for (FrameDev& f : c->frames) { if (f.pool == cam) frame_free(f); else keep.push_back(f); }
  kf_free(P);
  for (const FrameDev& f : nf) keep.push_back(f);
  c->frames.swap(keep); P = np;
  c->frame_index.clear();                                                // indices moved: every resident handle is found again
  for (size_t i=0;i<c->frames.size();i++) if (c->frames[i].used) c->frame_index[c->frames[i].id] = (int)i;
  return SDV_OK;
}
// device bytes of one frame and one keyframe level-0 image of camera cam as its frames are stored now: in its own pool, or at the context size
int sdv_camera_storage_bytes(sdv_ctx* c, int cam, uint64_t* frame_bytes_out, uint64_t* kf_image_bytes_out) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG;
  { int rc = check_cams(c, 1, &cam, "sdv_camera_storage_bytes", nullptr); if (rc) return rc; }
  const FramePool& P = c->pools[frame_pool_of(c, cam)];
  if (frame_bytes_out) *frame_bytes_out = frame_bytes(P.w, P.h, c->levels);
  if (kf_image_bytes_out) *kf_image_bytes_out = kf_image_bytes(P.w, P.h);
  return SDV_OK;
}

static int create_impl(sdv_ctx* c, const sdv_calib* K, int w, int h, int levels, const sdv_settings* s_in, int device);
int sdv_create(const sdv_calib* K, int w, int h, int levels, const sdv_settings* s_in, int device, sdv_ctx** out) {
  if (out) *out = nullptr;
  if (!K || !out || w <= 0 || h <= 0 || levels < 1 || levels > SDV_PYR_LEVELS || device < 0) { snprintf(g_create_err, sizeof g_create_err, "sdv_create: bad argument"); return SDV_ERR_ARG; }
  int ndev = 0; if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev <= device) { snprintf(g_create_err, sizeof g_create_err, "sdv_create: no CUDA device %d (this library has no CPU fallback)", device); return SDV_ERR_CUDA; }
  sdv_ctx* c = new sdv_ctx();                              // value-initialised: every pointer/handle member starts null, so sdv_destroy is safe on a partially built context
  c->err[0] = 0;
  int rc = create_impl(c, K, w, h, levels, s_in, device);
  if (rc != SDV_OK) { snprintf(g_create_err, sizeof g_create_err, "%s", c->err[0] ? c->err : "sdv_create failed"); sdv_destroy(c); return rc; }
  *out = c; return SDV_OK;
}
static int create_impl(sdv_ctx* c, const sdv_calib* K, int w, int h, int levels, const sdv_settings* s_in, int device) {
  sdv_settings s; if (s_in) s = *s_in; else sdv_default_settings(&s);
  if (s.n_tracker_slots < 1) s.n_tracker_slots = 2;
  if (s.max_frames < 2) s.max_frames = 2;
  if (s.cluster_size <= 0) s.cluster_size = 1;
  if (s.track_threads != 64 && s.track_threads != 256) s.track_threads = 128;
  if (s.cluster_size > 16) s.cluster_size = 16;
  c->set = s; c->device = device; c->w = w; c->h = h; c->levels = levels;
  for (int k=0;k<SDV_MAX_CAMERAS;k++) { c->cam_w[k] = w; c->cam_h[k] = h; c->cam_levels[k] = levels; }
  CK(cudaSetDevice(device));
  CK(kernels_init_device()); CK(refine_init_device());      // per-device function attributes (opt-in shared memory, cluster sizes)
  CK(cudaStreamCreateWithFlags(&c->st, cudaStreamNonBlocking)); CK(cudaStreamCreateWithFlags(&c->st_ba, cudaStreamNonBlocking));
  CK(cudaStreamCreateWithFlags(&c->st_in, cudaStreamNonBlocking)); CK(cudaStreamCreateWithFlags(&c->st_cp, cudaStreamNonBlocking));
  for (int i=0;i<sdv_ctx::kIngRing;i++) CK(cudaEventCreateWithFlags(&c->ev_ing[i], cudaEventDisableTiming)); for (int i=0;i<2;i++) CK(cudaEventCreateWithFlags(&c->ev_cp[i], cudaEventDisableTiming));
  CK(cudaEventCreateWithFlags(&c->ev_in, cudaEventDisableTiming)); c->ingest_pending = false; c->launches = 0;
  CK(cudaEventCreate(&c->ev0)); CK(cudaEventCreate(&c->ev1)); CK(cudaEventCreate(&c->ba_ev0)); CK(cudaEventCreate(&c->ba_ev1)); CK(cudaEventCreateWithFlags(&c->ev_xdom, cudaEventDisableTiming));
  memset(&c->tc, 0, sizeof(c->tc));
  c->tc.levels = levels; c->tc.huberTH = s.huberTH; c->tc.coarseCutoffTH = s.coarseCutoffTH;
  c->tc.affineOptModeA = s.affineOptModeA; c->tc.affineOptModeB = s.affineOptModeB;
  CK(cudaMalloc(&c->tc_dev, sizeof(TrackConst)));
  CK(cudaMemcpy(c->tc_dev, &c->tc, sizeof(TrackConst), cudaMemcpyHostToDevice));
  c->geom.assign(s.n_tracker_slots + 1, GeomRow{});                // slot rows are written by sdv_set_calib_slots before a slot points at them
  make_geom(c, K, 0, 0);
  CK(cudaMalloc(&c->geom_dev, c->geom.size()*sizeof(GeomRow)));
  CK(cudaMemcpy(c->geom_dev, c->geom.data(), c->geom.size()*sizeof(GeomRow), cudaMemcpyHostToDevice));
  // the context's frame pool: max_frames frames and the keyframe level-0 images, at the context size
  c->frames.resize(s.max_frames);
  for (auto& f : c->frames) CK(frame_alloc(f, 0, w, h, levels));
  c->pools[0].w = w; c->pools[0].h = h; c->pools[0].n_frames = s.max_frames;
  CK(kf_alloc(c->pools[0], kf_count(s.max_kf_images, s.max_frames), w, h));
  // tracker slots
  c->slots.resize(s.n_tracker_slots);
  for (auto& t : c->slots) {
    for (int l=0;l<levels;l++) {
      size_t cap = (size_t)(w>>l)*(h>>l); if (s.max_ref_points > 0 && (size_t)s.max_ref_points < cap) cap = s.max_ref_points;
      t.cap[l] = (int)cap; t.npts[l] = 0; CK(cudaMalloc(&t.pts[l], cap*sizeof(float4)));
    }
    t.ref_frame = ~0ull; t.has_totals = false; t.geom_row = 0; t.cam = 0;
  }
  // step-kernel reduction buffers
  CK(cudaMalloc(&c->partials, (size_t)step_kernel_max_grid()*kNAcc*sizeof(double)));
  CK(cudaMalloc(&c->ticket, sizeof(unsigned int))); CK(cudaMemset(c->ticket, 0, sizeof(unsigned int)));
  CK(cudaMalloc(&c->totals_dev, kNAcc*sizeof(double)));
  CK(cudaMallocHost(&c->totals_host, kNAcc*sizeof(double)));
  c->last_ms = 0;
  return SDV_OK;
}

void sdv_destroy(sdv_ctx* c) {
  if (!c) return;
  cudaSetDevice(c->device);
  if (c->st_cp) cudaStreamSynchronize(c->st_cp); if (c->st_in) cudaStreamSynchronize(c->st_in); if (c->st) cudaStreamSynchronize(c->st);
  for (auto& f : c->frames) frame_free(f);
  for (auto& P : c->pools) kf_free(P);
  for (auto& t : c->slots) for (int l=0;l<c->levels;l++) cudaFree(t.pts[l]);
  for (int i=0;i<2;i++) { c->ing_dev[i].release(); c->ing_host[i].release(); } cudaFree(c->partials); cudaFree(c->ticket); cudaFree(c->totals_dev); cudaFreeHost(c->totals_host);
  cudaFree(c->tc_dev); cudaFree(c->geom_dev); c->scr.release(); c->scr_host.release();
  for (float* u : c->und_buf) cudaFree(u);
  cudaFree(c->gw2_dev);
  for (int i=0;i<sdv_ctx::kIngRing;i++) if (c->ev_ing[i]) cudaEventDestroy(c->ev_ing[i]); for (int i=0;i<2;i++) if (c->ev_cp[i]) cudaEventDestroy(c->ev_cp[i]); if (c->st_cp) cudaStreamDestroy(c->st_cp);
  rp_destroy(c);
  sel_destroy(c);
  lidar_destroy(c);
  lidar_rows_destroy(c);
  imm_store_destroy(c);
  ba_destroy(c);
  if (c->ba_ev0) cudaEventDestroy(c->ba_ev0); if (c->ba_ev1) cudaEventDestroy(c->ba_ev1); if (c->ev_xdom) cudaEventDestroy(c->ev_xdom); if (c->st_ba) cudaStreamDestroy(c->st_ba);
  if (c->ev_trk_async) cudaEventDestroy(c->ev_trk_async);
  if (c->ev0) cudaEventDestroy(c->ev0); if (c->ev1) cudaEventDestroy(c->ev1); if (c->ev_in) cudaEventDestroy(c->ev_in); if (c->st) cudaStreamDestroy(c->st); if (c->st_in) cudaStreamDestroy(c->st_in);
  cudaGetLastError();                                      // a partially built context may have produced benign errors above: do not leave them sticky
  delete c;
}

int sdv_sync(sdv_ctx* c) { SDV_GUARD_TRK(c); if (!c) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); CK(cudaStreamSynchronize(c->st_cp)); CK(cudaStreamSynchronize(c->st_in)); CK(cudaStreamSynchronize(c->st)); CK(cudaStreamSynchronize(c->st_ba)); return SDV_OK; }
long long sdv_launch_count(sdv_ctx* c) { return c ? c->launches.load() : 0LL; }
int sdv_track_job_bytes(void) { return (int)sizeof(TrackJob); }
int sdv_debug_gs_entry_rc(int k) { int r, c; if (k < 0 || k >= kNH) return -1; gs_entry_rc(k, r, c); return r*16 + c; }   // test hook (host evaluation of the device index walk)
float sdv_last_kernel_ms(sdv_ctx* c) { return c ? c->last_ms : 0.f; }

// ------------------------------------------------------------------------------------------------ frames
static void frame_drop_texels(sdv_ctx* c, FrameDev& f) { if (f.lvl0_slot >= 0) { c->pools[f.pool].lvl0_free.push_back(f.lvl0_slot); f.lvl0_slot = -1; } f.lvl[0] = nullptr; f.hi_tex = false; }
// hands frame entry idx back to its pool (sdv_frame_release): the caller may reuse an adopted buffer at once, its keyframe image goes back to the pool
static int frame_release_idx(sdv_ctx* c, int idx) {
  FrameDev& f = c->frames[idx];
  { int rcf = frame_fence(c, f, nullptr, nullptr, f.adopted); if (rcf) return rcf; }
  f.used = false; frame_drop_texels(c, f); f.adopted = false; f.I0 = f.I0_own; f.img[0] = f.I0; c->frame_index.erase(f.id);
  return SDV_OK;
}

// kind bit0: mono8 input, bit1: input already in device memory, bit2: adopt the (device, float) buffer as the frame's level-0 plane,
// bit3: RAW mono8 input of the camera's native size, rectified through the tables of sdv_set_undistort_cam inside the level-0 kernel.
// Image k is camera cams[k] (cams == NULL: camera 0) and becomes a frame of that camera's rectified size, so the byte size, the staging offset and the
// coalesced copies are per frame.  Its storage comes from the camera's pool (frame_pool_of); a handle resident in another pool moves: every image's frame
// is claimed first (a pinned handle or a full pool refuses the batch and leaves every handle as it was), then the moved handles' old frames are released.
// Everything is enqueued on the ingest stream; the compute stream picks it up through ev_in at the next tracker / BA call, so an
// upload overlaps the tracking of the previous batch.  Every level is a planar intensity image: a pinned-host float upload lands directly in
// frame storage, levels >= 1 are built by one fused launch, and the consumers form gradients on the fly.
static int frame_ingest(sdv_ctx* c, int n, const uint64_t* frames, const void* const* imgs, const float* exposures, int kind, const int32_t* cams = nullptr) {
  if (!c || n < 0 || !frames || !imgs) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK;
  const bool raw = (kind & 8), u8 = (kind & 1) || raw, dev = (kind & 2), adopt = (kind & 4) && dev && !u8;
  { int rc = check_cams(c, n, cams, "frame upload", "image"); if (rc) return rc; }   // before any frame handle is claimed or anything is enqueued: a refused call changes no frame
  auto cam_of = [&](int k) { return cams ? cams[k] : 0; };
  if (raw) for (int k=0;k<n;k++)
    if (!c->und.cam[cam_of(k)].remapX) return ctx_fail(c, SDV_ERR_STATE, "raw upload before sdv_set_undistort (camera %d has no tables)", cam_of(k));
  CK(cudaSetDevice(c->device));
  const long long seq = c->ingest_seq + 1; const int par = (int)(seq & 1);
  // staging buffers + descriptors of this parity were last used by ingest seq-2: it must have drained before the host rewrites the pinned
  // descriptors (the device-side order copy(seq) after pyramid(seq-2) is enforced on the copy stream below)
  if (seq > 2) CK(cudaEventSynchronize(c->ev_ing[(seq-2) % sdv_ctx::kIngRing]));
  auto px = [&](int k) { return (size_t)c->cam_w[cam_of(k)]*c->cam_h[cam_of(k)]; };                  // rectified pixels of frame k
  auto px_in = [&](int k) { const sdv::UndistortDev& u = c->und.cam[cam_of(k)]; return raw ? (size_t)u.wOrg*u.hOrg : px(k); };   // bytes of mono8 input image k
  size_t stage = 0; if (u8 && !dev) for (int k=0;k<n;k++) stage += px_in(k);
  Scratch& sd = c->ing_dev[par]; PinnedScratch& sh = c->ing_host[par];      // need() leaves the descriptors the 16 B of slack launch_h2d_words reads past them
  if (sd.reserve(Scratch::need(n, sizeof(PyrBatchHost)) + Scratch::need(stage, 1), c->st_in) || sh.reserve(Scratch::need(n, sizeof(PyrBatchHost)), c->st_in))
    return ctx_fail(c, SDV_ERR_CUDA, "frame upload: staging of %d images", n);
  sd.reset(); sh.reset(); PyrBatchHost* desc_dev = sd.take<PyrBatchHost>(n); PyrBatchHost* desc = sh.take<PyrBatchHost>(n); unsigned char* stage_u8 = sd.take<unsigned char>(stage);
  c->cp_dst.clear(); c->cp_src.clear(); c->cp_sz.clear();
  if (c->levels > 1 && ((c->w | c->h) & 1)) return ctx_fail(c, SDV_ERR_ARG, "pyramid needs even image sizes");
  // every image's frame is planned before any frame changes: a refused batch (a pinned handle, a full pool) leaves every handle as it was
  std::vector<int> idx_of(n), old_of(n, -1); std::vector<char> taken(c->frames.size(), 0); std::unordered_map<uint64_t, int> planned;
  for (int k=0;k<n;k++) {
    const int p = frame_pool_of(c, cam_of(k));
    auto pl = planned.find(frames[k]);
    if (pl != planned.end()) {                                            // the same handle twice in one batch: one frame for both, as before
      if (c->frames[idx_of[pl->second]].pool != p)
        return ctx_fail(c, SDV_ERR_ARG, "frame %llu appears twice in one upload with cameras of different frame pools", (unsigned long long)frames[k]);
      idx_of[k] = idx_of[pl->second]; continue;
    }
    planned[frames[k]] = k; int idx = -1;
    auto it = c->frame_index.find(frames[k]);
    if (it != c->frame_index.end()) {
      if (frame_pinned(c, frames[k])) return ctx_fail(c, SDV_ERR_STATE, "frame %llu is referenced by a resident BA window / map slot and cannot be re-uploaded", (unsigned long long)frames[k]);
      if (c->frames[it->second].pool == p) idx = it->second; else old_of[k] = it->second;   // storage in another pool: the handle moves to pool p
    }
    if (idx < 0) for (size_t i=0;i<c->frames.size();i++) if (!c->frames[i].used && !taken[i] && c->frames[i].pool == p) { idx = (int)i; break; }
    if (idx < 0) return p == 0 ? ctx_fail(c, SDV_ERR_CAPACITY, "frame pool exhausted (max_frames=%d)", c->pools[0].n_frames)
                               : ctx_fail(c, SDV_ERR_CAPACITY, "frame pool of camera %d exhausted (max_frames=%d)", p, c->pools[p].n_frames);
    taken[idx] = 1; idx_of[k] = idx;
  }
  bool vec = true; size_t stage_off = 0; int max_w = 0, max_h = 0;
  for (int k=0;k<n;k++) {
    const int idx = idx_of[k];
    if (old_of[k] >= 0) { int rco = frame_release_idx(c, old_of[k]); if (rco) return rco; }   // the moved handle's old frame, once its new one is certain
    { int rcf = frame_fence(c, c->frames[idx], c->st_cp, c->st_in, c->frames[idx].adopted); if (rcf) return rcf; }   // an earlier trace may still read its storage
    FrameDev& f = c->frames[idx]; f.used = true; f.id = frames[k]; f.exposure = exposures ? exposures[k] : 1.0f; c->frame_index[frames[k]] = idx;
    frame_drop_texels(c, f); f.ingest_seq = seq; f.cam = cam_of(k); frame_layout(c, f);
    f.adopted = adopt; f.I0 = adopt ? const_cast<float*>(reinterpret_cast<const float*>(imgs[k])) : f.I0_own; f.img[0] = f.I0;
    PyrBatchHost& b = desc[k];
    b.pyr = f.pyr; b.I0 = f.I0; b.flags = (f.exposure > 0.f) ? 1 : 0; b.cam = f.cam; b.w = c->cam_w[f.cam]; b.h = c->cam_h[f.cam];
    max_w = std::max(max_w, b.w); max_h = std::max(max_h, b.h);
    if (dev) b.src = imgs[k];
    else if (u8) { const size_t sz = px_in(k); unsigned char* d8 = stage_u8 + stage_off; stage_off += sz; b.src = d8;
      if (!c->cp_dst.empty() && (unsigned char*)c->cp_src.back() + c->cp_sz.back() == (const unsigned char*)imgs[k] && (unsigned char*)c->cp_dst.back() + c->cp_sz.back() == d8) c->cp_sz.back() += sz;   // adjacent in host memory: one copy, whatever the cameras
      else { c->cp_dst.push_back(d8); c->cp_src.push_back(const_cast<void*>(imgs[k])); c->cp_sz.push_back(sz); } }
    else { b.src = f.I0; c->cp_dst.push_back(f.I0); c->cp_src.push_back(const_cast<void*>(imgs[k])); c->cp_sz.push_back(px(k)*sizeof(float)); }
    vec = vec && ((uintptr_t)b.src % (u8 ? 4 : 16)) == 0 && ((uintptr_t)b.I0 % 16) == 0 && b.w % 4 == 0;   // 4-pixel vector loads / stores of the pyramid kernel
  }
  if (!c->cp_dst.empty()) {                                               // all H2D copies of the batch in ONE runtime call, on the copy stream: PCIe stays busy while the
    if (seq > 2) CK(cudaStreamWaitEvent(c->st_cp, c->ev_ing[(seq-2) % sdv_ctx::kIngRing], 0));   // previous batch's pyramid runs on st_in
    bool done = false;
    if (c->cp_dst.size() > 1 && !c->no_batch_copy) {
      cudaMemcpyAttributes at; memset(&at, 0, sizeof(at)); at.srcAccessOrder = cudaMemcpySrcAccessOrderStream;
      size_t aidx = 0, fail = 0;
      cudaError_t e = cudaMemcpyBatchAsync(c->cp_dst.data(), c->cp_src.data(), c->cp_sz.data(), c->cp_dst.size(), &at, &aidx, 1, &fail, c->st_cp);
      if (e == cudaSuccess) done = true; else { cudaGetLastError(); c->no_batch_copy = true; }
    }
    if (!done) for (size_t i=0;i<c->cp_dst.size();i++) CK(cudaMemcpyAsync(c->cp_dst[i], c->cp_src[i], c->cp_sz[i], cudaMemcpyHostToDevice, c->st_cp));
    c->cp_dst.clear(); c->cp_src.clear(); c->cp_sz.clear();
    CK(cudaEventRecord(c->ev_cp[par], c->st_cp)); CK(cudaStreamWaitEvent(c->st_in, c->ev_cp[par], 0));
  }
  launch_h2d_words(desc_dev, desc, (size_t)n*sizeof(PyrBatchHost), c->st_in);   // kernel copy: a cudaMemcpyAsync here becomes ready only after this batch's bulk copy and
  c->launches += 1;                                                                              // would queue behind the NEXT batch's bulk copy on the H2D engine
  const UndistortCams* und = raw ? &c->und : nullptr;
  if (c->levels > 1) { launch_pyramid_batch(desc_dev, n, u8, vec, max_w, max_h, c->levels, c->st_in, und); c->launches += 1; }
  else if (u8 || (dev && !adopt)) { launch_pyramid_copy0(desc_dev, n, u8, max_w, max_h, c->st_in, und); c->launches += 1; }
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev_ing[seq % sdv_ctx::kIngRing], c->st_in)); c->ingest_seq = seq; c->ingest_pending = true;
  return SDV_OK;
}
}  // extern "C"
namespace sdv {
int frame_fence(sdv_ctx* c, FrameDev& f, cudaStream_t a, cudaStream_t b, bool host_wait) {
  if (!f.trk_async || !c->ev_trk_async) return SDV_OK;
  if (host_wait) { CK(cudaEventSynchronize(c->ev_trk_async)); f.trk_async = false; return SDV_OK; }
  if (a) CK(cudaStreamWaitEvent(a, c->ev_trk_async, 0));
  if (b) CK(cudaStreamWaitEvent(b, c->ev_trk_async, 0));
  if (a || b) f.trk_async = false;                                       // the writers of the new contents are ordered after the readers
  return SDV_OK;
}
int join_ingest_upto(sdv_ctx* c, long long seq) {  // the compute stream waits for ingest calls <= seq (st_in is in order, so one event covers all earlier ones)
  if (seq > c->ingest_seq) seq = c->ingest_seq;
  if (seq <= c->seq_waited) return SDV_OK;
  if (seq > c->ingest_seq - sdv_ctx::kIngRing) CK(cudaStreamWaitEvent(c->st, c->ev_ing[seq % sdv_ctx::kIngRing], 0));   // older ones have drained (frame_ingest syncs on seq-2)
  c->seq_waited = seq;
  return SDV_OK;
}
int join_ingest(sdv_ctx* c) { c->ingest_pending = false; return join_ingest_upto(c, c->ingest_seq); }
int ensure_lvl0(sdv_ctx* c, FrameDev& f) {        // FrameHessian::dI of a keyframe: packed level-0 texels, built once on demand
  if (f.lvl[0]) return SDV_OK;
  FramePool& P = c->pools[f.pool];                                       // the pool of the frame's storage: no fallback to another pool
  if (P.lvl0_free.empty()) return f.pool == 0 ? ctx_fail(c, SDV_ERR_CAPACITY, "keyframe level-0 image pool exhausted (max_kf_images=%d)", (int)P.lvl0.size())
                                              : ctx_fail(c, SDV_ERR_CAPACITY, "keyframe level-0 image pool of camera %d exhausted (max_kf_images=%d)", f.pool, (int)P.lvl0.size());
  int rc = join_ingest(c); if (rc) return rc;
  f.lvl0_slot = P.lvl0_free.back(); P.lvl0_free.pop_back(); f.lvl[0] = P.lvl0[f.lvl0_slot];
  launch_grad_texels(f.I0, f.lvl[0], c->cam_w[f.cam], c->cam_h[f.cam], cam_gw2(c, f.cam), c->st); c->launches += 1;
  CK(cudaGetLastError());
  return SDV_OK;
}
int ensure_texels(sdv_ctx* c, FrameDev& f, int lvl) {   // FrameHessian::dIp / absSquaredGrad of levels >= 1 for the selector and read-back, built once per ingest
  if (lvl == 0) return ensure_lvl0(c, f);
  if (f.hi_tex) return SDV_OK;
  int rc = join_ingest_upto(c, f.ingest_seq); if (rc) return rc;        // only the ingest that built this frame: a later batch keeps streaming
  for (int l=1;l<c->levels;l++) launch_grad_texels(f.img[l], f.lvl[l], c->cam_w[f.cam]>>l, c->cam_h[f.cam]>>l, cam_gw2(c, f.cam), c->st);
  c->launches += c->levels - 1;
  CK(cudaGetLastError());
  f.hi_tex = true;
  return SDV_OK;
}
int check_frame_slot(sdv_ctx* c, const FrameDev& f, int slot, const char* who) {
  const int fc = f.cam, sc = c->slots[slot].cam;
  if (same_size(c, fc, sc)) return SDV_OK;
  return ctx_fail(c, SDV_ERR_ARG, "%s: frame %llu is %dx%d (camera %d) but slot %d is bound to camera %d, %dx%d", who, (unsigned long long)f.id,
                  c->cam_w[fc], c->cam_h[fc], fc, slot, sc, c->cam_w[sc], c->cam_h[sc]);
}
int check_frame_cam(sdv_ctx* c, const FrameDev& f, int cam, const char* who) {
  if (same_size(c, f.cam, cam)) return SDV_OK;
  return ctx_fail(c, SDV_ERR_ARG, "%s: frame %llu is %dx%d (camera %d) but the job names camera %d, %dx%d", who, (unsigned long long)f.id,
                  c->cam_w[f.cam], c->cam_h[f.cam], f.cam, cam, c->cam_w[cam], c->cam_h[cam]);
}
int job_frame(sdv_ctx* c, const char* who, int k, uint64_t id, int cam, int slot, long long* need_seq, FrameDev** out) {
  FrameDev* f = find_frame(c, id); if (!f) return ctx_fail(c, SDV_ERR_NOFRAME, "%s: entry %d names unknown frame %llu", who, k, (unsigned long long)id);
  const int rc = slot >= 0 ? check_frame_slot(c, *f, slot, who) : cam >= 0 ? check_frame_cam(c, *f, cam, who) : SDV_OK; if (rc) return rc;
  if (need_seq && f->ingest_seq > *need_seq) *need_seq = f->ingest_seq;
  *out = f; return SDV_OK;
}
int check_cams(sdv_ctx* c, int n, const int32_t* cams, const char* who, const char* what) {
  if (cams) for (int k=0;k<n;k++) if (cams[k] < 0 || cams[k] >= SDV_MAX_CAMERAS) {
    if (!what) return ctx_fail(c, SDV_ERR_ARG, "%s: camera %d outside 0..%d", who, cams[k], SDV_MAX_CAMERAS - 1);
    return ctx_fail(c, SDV_ERR_ARG, "%s: %s %d names camera %d (valid: 0..%d)", who, what, k, cams[k], SDV_MAX_CAMERAS - 1);
  }
  return SDV_OK;
}
int check_offsets(sdv_ctx* c, int n, const int32_t* off, const char* who, const char* what) {
  if (off[0] != 0) return ctx_fail(c, SDV_ERR_ARG, "%s: %s[0] = %d (must be 0)", who, what, off[0]);
  for (int k=0;k<n;k++) if (off[k+1] < off[k]) return ctx_fail(c, SDV_ERR_ARG, "%s: %s decreases at entry %d", who, what, k);
  return SDV_OK;
}
template <class T> static bool find_repeat(int n, const T* v, T* rep) {
  std::vector<T> s(v, v + n); std::sort(s.begin(), s.end());
  const auto it = std::adjacent_find(s.begin(), s.end()); if (it == s.end()) return false;
  *rep = *it; return true;
}
int check_ids(sdv_ctx* c, int n, const int32_t* ids, int limit, const char* who, const char* what) {
  for (int k=0;k<n;k++) if (ids[k] < 0 || ids[k] >= limit) return ctx_fail(c, SDV_ERR_ARG, "%s: entry %d names %s %d (valid: 0..%d)", who, k, what, ids[k], limit - 1);
  int32_t r; if (find_repeat(n, ids, &r)) return ctx_fail(c, SDV_ERR_ARG, "%s: %s %d appears twice in one call", who, what, r);
  return SDV_OK;
}
int check_distinct(sdv_ctx* c, int n, const uint64_t* ids, const char* who, const char* what) {
  uint64_t r; if (find_repeat(n, ids, &r)) return ctx_fail(c, SDV_ERR_ARG, "%s: %s %llu appears twice in one call", who, what, (unsigned long long)r);
  return SDV_OK;
}
}
extern "C" {

int sdv_frame_upload_batch(sdv_ctx* c, int n, const uint64_t* frames, const float* const* imgs, const float* exposures) { SDV_GUARD_TRK(c);
  return frame_ingest(c, n, frames, reinterpret_cast<const void* const*>(imgs), exposures, 0);
}
int sdv_frame_upload_batch_u8(sdv_ctx* c, int n, const uint64_t* frames, const uint8_t* const* imgs, const float* exposures) { SDV_GUARD_TRK(c);
  return frame_ingest(c, n, frames, reinterpret_cast<const void* const*>(imgs), exposures, 1);
}
// Undistort (util/Undistort.cpp) as data: the tables the reference builds once per calibration file, kept on the device for the raw-image ingest, one entry per camera
int sdv_set_undistort_cam(sdv_ctx* c, int cam, int w_org, int h_org, const float* remapX, const float* remapY, float factor, const float* G256, const float* vignette_inv) { SDV_GUARD_TRK(c);
  if (!c || w_org < 2 || h_org < 2 || !remapX || !remapY) return SDV_ERR_ARG;
  { int rc = check_cams(c, 1, &cam, "sdv_set_undistort_cam", nullptr); if (rc) return rc; }
  if (vignette_inv && !G256) return ctx_fail(c, SDV_ERR_ARG, "a vignette map needs a response function (PhotometricUndistorter::processFrame applies it to G[v] only)");
  CK(cudaSetDevice(c->device));
  const size_t px = (size_t)c->cam_w[cam]*c->cam_h[cam], po = (size_t)w_org*h_org;   // tables of the camera's rectified size
  for (size_t i=0;i<px;i++) {                                              // Undistort.cpp:871 tests iy against wOrg-1: a table built that way may read below the raw image
    const float x = remapX[i], y = remapY[i];
    if (x < 0) continue;
    if (!(x > 0 && y > 0 && x < w_org-1 && y < h_org-1)) return ctx_fail(c, SDV_ERR_ARG, "remap table entry %zu (%g,%g) reads outside the %dx%d raw image", i, x, y, w_org, h_org);
  }
  CK(cudaStreamSynchronize(c->st_in));                                     // an ingest in flight may still read the previous tables of this camera
  sdv::UndistortDev& u = c->und.cam[cam];
  cudaFree(c->und_buf[cam]); c->und_buf[cam] = nullptr; u = {};
  const size_t nfl = 2*px + (G256 ? 256 : 0) + (vignette_inv ? po : 0);
  float* p = nullptr; CK(cudaMalloc(&p, nfl*sizeof(float))); c->und_buf[cam] = p;
  sdv::UndistortDev d = {};
  CK(cudaMemcpy(p, remapX, px*sizeof(float), cudaMemcpyHostToDevice)); d.remapX = p; p += px;
  CK(cudaMemcpy(p, remapY, px*sizeof(float), cudaMemcpyHostToDevice)); d.remapY = p; p += px;
  if (G256) { CK(cudaMemcpy(p, G256, 256*sizeof(float), cudaMemcpyHostToDevice)); d.G = p; p += 256; }
  if (vignette_inv) { CK(cudaMemcpy(p, vignette_inv, po*sizeof(float), cudaMemcpyHostToDevice)); d.vignette = p; p += po; }
  d.wOrg = w_org; d.hOrg = h_org; d.factor = factor; u = d;                // set only once every table is on the device
  return SDV_OK;
}
// FullSystem::setGammaFunction (FullSystem.cpp:225-249) for one camera: B inverts BInv on the host in the reference's float arithmetic, the device keeps
// gw2[c] = (B[c+1]-B[c])*(B[c+1]-B[c]), the factor FrameHessian::makeImages applies to absSquaredGrad (HessianBlocks.cpp:158-164)
int sdv_set_gamma_cam(sdv_ctx* c, int cam, const float* BInv256) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG;
  { int rc = check_cams(c, 1, &cam, "sdv_set_gamma_cam", nullptr); if (rc) return rc; }
  for (const auto& kv : c->frame_index) if (c->frames[kv.second].cam == cam)       // texels and level-0 pool entries were weighed with the camera's current table
    return ctx_fail(c, SDV_ERR_STATE, "sdv_set_gamma_cam: frame %llu of camera %d is resident: set the gamma before the camera's first frame", (unsigned long long)kv.first, cam);
  if (!BInv256) { c->gamma_set[cam] = false; return SDV_OK; }
  float B[256];
  for (int i=0;i<256;i++) B[i] = (float)i;                                  // CalibHessian(): B[i] = i (HessianBlocks.h:293); an i no bracket finds keeps it
  for (int i=1;i<255;i++)
    for (int s=1;s<255;s++)
      if (BInv256[s] <= i && BInv256[s+1] >= i) { B[i] = s+(i - BInv256[s]) / (BInv256[s+1]-BInv256[s]); break; }
  B[0] = 0; B[255] = 255;
  float gw2[256];
  for (int k=0;k<255;k++) { const float gw = B[k+1]-B[k]; gw2[k] = gw*gw; }
  gw2[255] = 1.0f;                                                          // never read: gamma_w2 clamps c to [5, 250]
  CK(cudaSetDevice(c->device));
  if (!c->gw2_dev) CK(cudaMalloc(&c->gw2_dev, (size_t)SDV_MAX_CAMERAS*256*sizeof(float)));
  CK(cudaMemcpy(c->gw2_dev + 256*(size_t)cam, gw2, sizeof(gw2), cudaMemcpyHostToDevice));   // no resident frame of this camera: no pending kernel reads the row
  c->gamma_set[cam] = true;
  return SDV_OK;
}
int sdv_set_undistort(sdv_ctx* c, int w_org, int h_org, const float* remapX, const float* remapY, float factor, const float* G256, const float* vignette_inv) {
  return sdv_set_undistort_cam(c, 0, w_org, h_org, remapX, remapY, factor, G256, vignette_inv);
}
int sdv_frame_upload_batch_raw_u8_cams(sdv_ctx* c, int n, const uint64_t* frames, const uint8_t* const* raw_imgs, const int32_t* cams, const float* exposures) { SDV_GUARD_TRK(c);
  return frame_ingest(c, n, frames, reinterpret_cast<const void* const*>(raw_imgs), exposures, 8, cams);
}
int sdv_frame_upload_batch_raw_u8(sdv_ctx* c, int n, const uint64_t* frames, const uint8_t* const* raw_imgs, const float* exposures) {
  return sdv_frame_upload_batch_raw_u8_cams(c, n, frames, raw_imgs, nullptr, exposures);
}
int sdv_frame_build_batch_dev_cams(sdv_ctx* c, int n, const uint64_t* frames, const void* const* imgs_dev, const int32_t* cams, int fmt, const float* exposures) { SDV_GUARD_TRK(c);
  if (fmt < 0 || fmt > 2) return SDV_ERR_ARG;
  return frame_ingest(c, n, frames, imgs_dev, exposures, 2 | (fmt == 1 ? 1 : 0) | (fmt == 2 ? 4 : 0), cams);
}
int sdv_frame_build_batch_dev(sdv_ctx* c, int n, const uint64_t* frames, const void* const* imgs_dev, int fmt, const float* exposures) {
  return sdv_frame_build_batch_dev_cams(c, n, frames, imgs_dev, nullptr, fmt, exposures);
}
int sdv_frame_upload_batch_cams(sdv_ctx* c, int n, const uint64_t* frames, const void* const* imgs, const int32_t* cams, int fmt, const float* exposures) { SDV_GUARD_TRK(c);
  if (fmt < 0 || fmt > 1) return SDV_ERR_ARG;
  return frame_ingest(c, n, frames, imgs, exposures, fmt, cams);
}
int sdv_frame_upload(sdv_ctx* c, uint64_t frame, const float* img, float exposure) { SDV_GUARD_TRK(c);
  const float* imgs[1] = {img}; return sdv_frame_upload_batch(c, 1, &frame, imgs, &exposure);
}
int sdv_frame_release(sdv_ctx* c, uint64_t frame) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG;
  auto it = c->frame_index.find(frame); if (it == c->frame_index.end()) return ctx_fail(c, SDV_ERR_NOFRAME, "unknown frame %llu", (unsigned long long)frame);
  if (frame_pinned(c, frame)) return ctx_fail(c, SDV_ERR_STATE, "frame %llu is referenced by a resident BA window / map slot: replace or clear that window / map first", (unsigned long long)frame);
  return frame_release_idx(c, it->second);
}
int sdv_frame_download(sdv_ctx* c, uint64_t frame, int lvl, float* dI3_out, float* abs_out) { SDV_GUARD_TRK(c);
  if (!c || lvl < 0 || lvl >= c->levels) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  FrameDev* f; { int rc = job_frame(c, "sdv_frame_download", 0, frame, -1, -1, nullptr, &f); if (rc) return rc; }
  if (lvl >= c->cam_levels[f->cam]) return ctx_fail(c, SDV_ERR_ARG, "sdv_frame_download: level %d of frame %llu, whose camera %d has %d levels", lvl, (unsigned long long)frame, f->cam, c->cam_levels[f->cam]);
  { int rcj = join_ingest(c); if (rcj) return rcj; }
  { int rct = ensure_texels(c, *f, lvl); if (rct) return rct; }
  int n = (c->cam_w[f->cam]>>lvl)*(c->cam_h[f->cam]>>lvl); float *d3 = nullptr, *da = nullptr;   // the frame's own size
  if (dI3_out) CK(cudaMalloc(&d3, (size_t)3*n*sizeof(float)));
  if (abs_out) CK(cudaMalloc(&da, (size_t)n*sizeof(float)));
  launch_unpack_level(f->lvl[lvl], d3, da, n, c->st);
  if (d3) CK(cudaMemcpyAsync(dI3_out, d3, (size_t)3*n*sizeof(float), cudaMemcpyDeviceToHost, c->st));
  if (da) CK(cudaMemcpyAsync(abs_out, da, (size_t)n*sizeof(float), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  cudaFree(d3); cudaFree(da);
  return SDV_OK;
}

// ------------------------------------------------------------------------------------------------ tracker reference
int sdv_tracker_set_cloud(sdv_ctx* c, int slot, uint64_t ref_frame, int lvl, int n, const float* u, const float* v,
                          const float* idepth, const float* color, double ref_a, double ref_b) { SDV_GUARD_TRK(c);
  if (!c || slot < 0 || slot >= (int)c->slots.size() || lvl < 0 || lvl >= c->levels || n < 0) return SDV_ERR_ARG;
  if (lvl >= slot_levels(c, slot)) return ctx_fail(c, SDV_ERR_ARG, "sdv_tracker_set_cloud: level %d, but slot %d's camera has %d levels", lvl, slot, slot_levels(c, slot));
  CK(cudaSetDevice(c->device));
  TrackerSlot& t = c->slots[slot];
  if (n > t.cap[lvl]) return ctx_fail(c, SDV_ERR_CAPACITY, "cloud of %d points exceeds capacity %d", n, t.cap[lvl]);
  FrameDev* f; { int rc = job_frame(c, "sdv_tracker_set_cloud", 0, ref_frame, -1, slot, nullptr, &f); if (rc) return rc; }
  { int rcj = join_ingest(c); if (rcj) return rcj; }
  float* tmp = nullptr; CK(cudaMalloc(&tmp, (size_t)4*(n+1)*sizeof(float)));
  const float* src[4] = {u, v, idepth, color};
  for (int k=0;k<4;k++) CK(cudaMemcpyAsync(tmp + (size_t)k*n, src[k], (size_t)n*sizeof(float), cudaMemcpyHostToDevice, c->st));
  launch_pack_cloud(tmp, tmp+n, tmp+2*(size_t)n, tmp+3*(size_t)n, n, t.pts[lvl], c->st);
  CK(cudaStreamSynchronize(c->st)); cudaFree(tmp);
  t.npts[lvl] = n; t.ref_frame = ref_frame; t.ref_a = ref_a; t.ref_b = ref_b; t.refExposure = f->exposure; t.has_totals = false;
  return SDV_OK;
}

int sdv_tracker_get_cloud(sdv_ctx* c, int slot, int lvl, int* n_out, float* u, float* v, float* idepth, float* color) { SDV_GUARD_TRK(c);
  if (!c || slot < 0 || slot >= (int)c->slots.size() || lvl < 0 || lvl >= c->levels || !n_out) return SDV_ERR_ARG;
  if (lvl >= slot_levels(c, slot)) return ctx_fail(c, SDV_ERR_ARG, "sdv_tracker_get_cloud: level %d, but slot %d's camera has %d levels", lvl, slot, slot_levels(c, slot));
  CK(cudaSetDevice(c->device));
  TrackerSlot& t = c->slots[slot]; int n = t.npts[lvl]; *n_out = n;
  if (!u || n == 0) return SDV_OK;
  std::vector<float4> h(n);
  CK(cudaMemcpyAsync(h.data(), t.pts[lvl], (size_t)n*sizeof(float4), cudaMemcpyDeviceToHost, c->st)); CK(cudaStreamSynchronize(c->st));
  for (int i=0;i<n;i++) { u[i]=h[i].x; v[i]=h[i].y; idepth[i]=h[i].z; color[i]=h[i].w; }
  return SDV_OK;
}

// CoarseTracker::setCoarseTrackingRef for n slots: every check runs before anything is enqueued, then one build (set_ref_build) serves all jobs
int sdv_tracker_set_ref_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* ref_frames, const int32_t* pt_begin, const float* pts4, const int32_t* round_half,
                              const double* ref_ab, int32_t* npts_out) { SDV_GUARD_TRK(c);
  const char* who = "sdv_tracker_set_ref_batch";
  if (!c || n < 0 || (n > 0 && (!slots || !ref_frames || !pt_begin))) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK;
  { int rc = check_offsets(c, n, pt_begin, who, "pt_begin"); if (rc) return rc; }
  if (pt_begin[n] > 0 && (!pts4 || !round_half)) return SDV_ERR_ARG;
  { int rc = check_ids(c, n, slots, (int)c->slots.size(), who, "slot"); if (rc) return rc; }
  std::vector<FrameDev*> F(n);
  for (int j = 0; j < n; j++) {
    { int rc = job_frame(c, who, j, ref_frames[j], -1, slots[j], nullptr, &F[j]); if (rc) return rc; }
    const int cam = c->slots[slots[j]].cam, w = c->cam_w[cam], h = c->cam_h[cam];        // makeCoarseDepthL0 at the slot's size
    for (int i = pt_begin[j]; i < pt_begin[j+1]; i++) {                                   // the reference would write out of bounds here; we refuse instead
      const int u = round_half[i] ? (int)(pts4[4*i]+0.5f) : (int)pts4[4*i], v = round_half[i] ? (int)(pts4[4*i+1]+0.5f) : (int)pts4[4*i+1];
      if (u < 0 || v < 0 || u >= w || v >= h) return ctx_fail(c, SDV_ERR_ARG, "%s: job %d, row %d: splat (%d,%d) outside the %dx%d image", who, j, i - pt_begin[j], u, v, w, h);
    }
  }
  CK(cudaSetDevice(c->device));
  int launches = 0;
  CK(cudaEventRecord(c->ev0, c->st));
  const int rc = set_ref_build(c, n, slots, F.data(), ref_frames, pt_begin, pts4, round_half, cudaMemcpyHostToDevice, ref_ab, npts_out, &launches);
  c->launches += launches;
  if (rc && rc != SDV_ERR_CAPACITY) return rc;
  CK(cudaEventRecord(c->ev1, c->st)); CK(cudaEventSynchronize(c->ev1)); CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  return rc;
}
int sdv_tracker_set_ref(sdv_ctx* c, int slot, uint64_t ref_frame, int n, const float* pts4, const int32_t* round_half,
                        float /*unused*/, double ref_a, double ref_b) {
  if (!c || n < 0 || (n > 0 && (!pts4 || !round_half))) return SDV_ERR_ARG;
  const int32_t s = slot, pb[2] = {0, n}; const double ab[2] = {ref_a, ref_b};
  return sdv_tracker_set_ref_batch(c, 1, &s, &ref_frame, pb, pts4, round_half, ab, nullptr);
}
}  // extern "C"
extern "C" {

// ------------------------------------------------------------------------------------------------ calcRes / calcGSSSE
int sdv_tracker_calc_res(sdv_ctx* c, int slot, uint64_t new_frame, int lvl, const double T[7], double a, double b, float cutoffTH, double rs_out[6]) { SDV_GUARD_TRK(c);
  if (!c || slot < 0 || slot >= (int)c->slots.size() || lvl < 0 || lvl >= c->levels || !T || !rs_out) return SDV_ERR_ARG;
  if (lvl >= slot_levels(c, slot)) return ctx_fail(c, SDV_ERR_ARG, "sdv_tracker_calc_res: level %d, but slot %d's camera has %d levels", lvl, slot, slot_levels(c, slot));
  CK(cudaSetDevice(c->device));
  TrackerSlot& t = c->slots[slot];
  FrameDev* f; { int rc = job_frame(c, "sdv_tracker_calc_res", 0, new_frame, -1, -1, nullptr, &f); if (rc) return rc; }
  if (t.ref_frame == ~0ull) return ctx_fail(c, SDV_ERR_STATE, "tracker slot %d has no reference", slot);
  { int rcs = check_frame_slot(c, *f, slot, "sdv_tracker_calc_res"); if (rcs) return rcs; }
  const LevelGeom& g = slot_geom(c, slot).g[lvl];
  EvalParams ep; make_eval_params(se3_from7(T), a, b, t.refExposure, f->exposure, t.ref_a, t.ref_b, g, lvl, cutoffTH, c->tc.huberTH, ep);
  { int rcj = join_ingest(c); if (rcj) return rcj; }
  CK(cudaEventRecord(c->ev0, c->st));
  c->launches += 1;
  launch_coarse_res_gs(t.pts[lvl], t.npts[lvl], f->img[lvl], g, ep, c->partials, c->ticket, c->totals_dev, c->st);
  CK(cudaEventRecord(c->ev1, c->st));
  CK(cudaMemcpyAsync(c->totals_host, c->totals_dev, kNAcc*sizeof(double), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st)); CK(cudaGetLastError());
  CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  memcpy(t.totals, c->totals_host, sizeof(t.totals)); t.has_totals = true;
  finalize_res(t.totals, rs_out);
  return SDV_OK;
}
int sdv_tracker_calc_gs(sdv_ctx* c, int slot, int /*lvl*/, double H[64], double b[8]) { SDV_GUARD_TRK(c);
  if (!c || slot < 0 || slot >= (int)c->slots.size() || !H || !b) return SDV_ERR_ARG;
  TrackerSlot& t = c->slots[slot];
  if (!t.has_totals) return ctx_fail(c, SDV_ERR_STATE, "calc_gs before calc_res on slot %d", slot);
  finalize_gs(t.totals, H, b);
  return SDV_OK;
}

// ------------------------------------------------------------------------------------------------ trackNewestCoarse
// coarsest: job k starts its LM at coarsest[k]; NULL: at its slot camera's depth - 1 (FullSystem.cpp:421, coarseTracker->trackNewestCoarse(.., pyrLevelsUsed-1, ..)).
// all_coarsest >= 0 (sdv_tracker_track_batch): that level for every job.  Every level is checked against its job's depth before anything is enqueued.
static int track_batch_impl(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* new_frames, double* T_io, double* ab_io, const int32_t* coarsest, int all_coarsest,
                            const double* minRes, double* lastRes, double* flow, int32_t* good, sdv_track_stats* stats) {
  if (!c || n <= 0 || !slots || !new_frames || !T_io || !ab_io) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  const size_t bytes = Scratch::need(n, sizeof(TrackJob));                // need(): the 16 B of slack launch_h2d_words reads past the jobs
  if (c->scr.reserve(bytes, c->st) || c->scr_host.reserve(bytes, c->st)) return ctx_fail(c, SDV_ERR_CUDA, "sdv_tracker_track_batch: staging of %d jobs", n);
  c->scr.reset(); c->scr_host.reset(); TrackJob* jobs_dev = c->scr.take<TrackJob>(n); TrackJob* jobs_host = c->scr_host.take<TrackJob>(n);
  long long need_seq = 0;
  for (int k=0;k<n;k++) {
    if (slots[k] < 0 || slots[k] >= (int)c->slots.size()) return SDV_ERR_ARG;
    TrackerSlot& t = c->slots[slots[k]];
    FrameDev* f; { int rc = job_frame(c, "sdv_tracker_track_batch", k, new_frames[k], -1, -1, &need_seq, &f); if (rc) return rc; }
    if (t.ref_frame == ~0ull) return ctx_fail(c, SDV_ERR_STATE, "tracker slot %d has no reference", slots[k]);
    { int rcs = check_frame_slot(c, *f, slots[k], "sdv_tracker_track_batch"); if (rcs) return rcs; }
    const int L = slot_levels(c, slots[k]), co = all_coarsest >= 0 ? all_coarsest : (coarsest ? coarsest[k] : L - 1);
    if (co < 0 || co >= L || co >= 5)                                   // CoarseTracker.cpp:672: assert(coarsestLvl < 5 && coarsestLvl < pyrLevelsUsed)
      return ctx_fail(c, SDV_ERR_ARG, "sdv_tracker_track_batch: job %d starts at level %d, but slot %d's camera has %d levels (and the tracker at most 5)", k, co, slots[k], L);
    TrackJob& J = jobs_host[k]; memset(&J, 0, sizeof(J));
    for (int l=0;l<c->levels;l++) { J.img[l] = f->img[l]; J.pts[l] = t.pts[l]; J.npts[l] = t.npts[l]; }
    J.refExposure = t.refExposure; J.newExposure = f->exposure; J.ref_a = t.ref_a; J.ref_b = t.ref_b;
    for (int i=0;i<7;i++) J.T[i] = T_io[7*k+i];
    J.ab[0] = ab_io[2*k]; J.ab[1] = ab_io[2*k+1];
    for (int i=0;i<5;i++) J.minRes[i] = minRes ? minRes[5*k+i] : nan("");
    J.coarsest = co; J.geom_row = t.geom_row;
  }
  { int rcj = join_ingest_upto(c, need_seq); if (rcj) return rcj; }     // only the uploads that built THESE frames: batch k+1's upload keeps streaming
  c->launches += 2;                                                    // descriptor copy kernel + track_cluster_kernel
  launch_h2d_words(jobs_dev, jobs_host, (size_t)n*sizeof(TrackJob), c->st);      // kernel copy: not queued behind the next batch's image upload
  CK(cudaEventRecord(c->ev0, c->st));
  CK(launch_track_cluster(jobs_dev, n, c->tc_dev, c->geom_dev, c->set.cluster_size, c->set.track_threads, c->st));
  CK(cudaEventRecord(c->ev1, c->st));
  CK(cudaMemcpyAsync(jobs_host, jobs_dev, (size_t)n*sizeof(TrackJob), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st)); CK(cudaGetLastError());
  CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  for (int k=0;k<n;k++) {
    const TrackJob& J = jobs_host[k];
    for (int i=0;i<7;i++) T_io[7*k+i] = J.T[i];
    ab_io[2*k] = J.ab[0]; ab_io[2*k+1] = J.ab[1];
    if (lastRes) for (int i=0;i<5;i++) lastRes[5*k+i] = J.lastRes[i];
    if (flow) for (int i=0;i<3;i++) flow[3*k+i] = J.flow[i];
    if (good) good[k] = J.good;
    if (stats) for (int l=0;l<SDV_PYR_LEVELS;l++) { stats[k].point_evals[l] = J.point_evals[l]; stats[k].iterations[l] = J.iterations[l]; stats[k].accepts[l] = J.accepts[l]; }
  }
  return SDV_OK;
}
int sdv_tracker_track_batch_levels(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* new_frames, double* T_io, double* ab_io, const int32_t* coarsest,
                                   const double* minRes, double* lastRes, double* flow, int32_t* good, sdv_track_stats* stats) { SDV_GUARD_TRK(c);
  return track_batch_impl(c, n, slots, new_frames, T_io, ab_io, coarsest, -1, minRes, lastRes, flow, good, stats);
}
int sdv_tracker_track_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* new_frames, double* T_io, double* ab_io, int coarsest,
                            const double* minRes, double* lastRes, double* flow, int32_t* good, sdv_track_stats* stats) { SDV_GUARD_TRK(c);
  if (!c || coarsest < 0 || coarsest >= c->levels || coarsest >= 5) return SDV_ERR_ARG;
  return track_batch_impl(c, n, slots, new_frames, T_io, ab_io, nullptr, coarsest, minRes, lastRes, flow, good, stats);
}
int sdv_tracker_track(sdv_ctx* c, int slot, uint64_t new_frame, double T_io[7], double ab_io[2], int coarsest, const double minRes[5],
                      double lastRes[5], double flow[3], int* good, sdv_track_stats* stats) { SDV_GUARD_TRK(c);
  int32_t s = slot, g = 0;
  int rc = sdv_tracker_track_batch(c, 1, &s, &new_frame, T_io, ab_io, coarsest, minRes, lastRes, flow, &g, stats);
  if (good) *good = g; return rc;
}

} // extern "C"
