// sdv_select.cu — C-ABI of the candidate management at keyframe rate (SURVEY.md §8f rank 4 + the caller half of rank 2): binds the engine of sdv_select_core.cuh
// (kernels + host orchestration; see the header for the reference map and the design) to the context's resident frames and tracker-domain stream.
//   sdv_selector_init / _potential / _get_map   PixelSelector::PixelSelector, currentPotential, FullSystem::selectionMap      PixelSelector2.cpp:11-26, FullSystem.cpp:180-186
//   sdv_selector_make_hists(_cam)               PixelSelector::makeHists                                                     PixelSelector2.cpp:47-106
//   sdv_selector_make_maps_batch                PixelSelector::makeMapsFromLidar / makeMaps                                  PixelSelector2.cpp:354-449 / :108-200
//   sdv_make_new_traces_batch                   FullSystem::makeNewTraces (+ shiTomasiScore, setMask, ImmaturePoint ctor)    FullSystem.cpp:1261-1356, 1540-1583
//   sdv_activate_select_batch(_cams)            CoarseDistanceMap::makeDistanceMap + the candidate walk of activatePointsMT  CoarseTracker.cpp:1139-1282, FullSystem.cpp:600-671
// A selector slot is bound to a camera (sdv_selector_set_slot_cams; camera 0 after init) and works at that camera's size: its frames, its persistent map.
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include <stdlib.h>
#include "sdv_ctx.cuh"
#include "sdv_select_core.cuh"

using namespace sdv;
static_assert(sizeof(sel::NewTrace) == sizeof(sdv_new_trace) && sizeof(sel::ImmPt) == sizeof(sdv_immature_pt), "engine records mirror the C-ABI structs");

namespace sdv {
struct SelState { sel::SelEngine eng; std::vector<sel::SelectorSlot> slots; std::vector<int> cam;   // cam[s]: camera of slot s
                  int* boxD = nullptr; };                                                // FullSystem::left/right/up/down of every slot (4 ints each, device), FullSystem.h:191-194
static const int32_t kBox0[4] = {10000, -1, 10000, -1};                                   // their initial values
void sel_destroy(sdv_ctx* c) {
  SelState* s = (SelState*)c->sel; if (!s) return;
  for (auto& sl : s->slots) if (sl.mapD) cudaFree(sl.mapD);
  cudaFree(s->boxD);
  s->eng.io.release(); s->eng.destroy(); delete s; c->sel = nullptr;
}
bool sel_cam_bound(const sdv_ctx* c, int cam, int* slot) {
  const SelState* s = (const SelState*)c->sel; if (!s) return false;
  for (size_t k = 0; k < s->cam.size(); k++) if (s->cam[k] == cam) { *slot = (int)k; return true; }
  return false;
}
static int sel_frame(sdv_ctx* c, int k, uint64_t id, int cam, sel::FrameImg& F, const float*& gw2, long long& need_seq, const char* who, bool texels = true) {
  FrameDev* f; { int rc = job_frame(c, who, k, id, cam, -1, &need_seq, &f); if (rc) return rc; }
  F.I0 = f->I0; F.L1 = nullptr; F.L2 = nullptr; gw2 = cam_gw2(c, f->cam);           // the frame's camera weighed its texels: its table serves level 0 too
  if (texels) { int rc = ensure_texels(c, *f, 1); if (rc) return rc; F.L1 = f->lvl[1]; F.L2 = f->lvl[2]; }   // |grad|^2 of levels 1 and 2 (makeMaps / makeNewTraces read the packed texels)
  return SDV_OK;
}
int sel_n_slots(const sdv_ctx* c) { const SelState* s = (const SelState*)c->sel; return s ? (int)s->slots.size() : -1; }
void sel_slot_box(const sdv_ctx* c, int slot, int* cam, int** box_dev) { const SelState* s = (const SelState*)c->sel; *cam = s->cam[slot]; *box_dev = s->boxD + 4*(size_t)slot; }
static int sel_fail(sdv_ctx* c, SelState* s, int rc, const char* who) { return ctx_fail(c, rc == -2 ? SDV_ERR_CAPACITY : SDV_ERR_CUDA, "%s: %s", who, s->eng.err.c_str()); }
}  // namespace sdv
#define SEL_STATE(who) SelState* s = (SelState*)c->sel; if (!s) return ctx_fail(c, SDV_ERR_STATE, who ": sdv_selector_init has not been called")

extern "C" {

int sdv_selector_init(sdv_ctx* c, const uint8_t* random_pattern, int n_slots) { SDV_GUARD_TRK(c);
  if (!c || !random_pattern || n_slots < 1) return SDV_ERR_ARG;
  if (c->levels < 3) return ctx_fail(c, SDV_ERR_ARG, "selector_init: the selector reads pyramid levels 0..2 (context has %d levels)", c->levels);
  if (c->cam_levels[0] < 3) return ctx_fail(c, SDV_ERR_ARG, "selector_init: the selector reads pyramid levels 0..2 and binds every slot to camera 0, which has %d levels", c->cam_levels[0]);
  CK(cudaSetDevice(c->device));
  sel_destroy(c);
  SelState* s = new SelState(); c->sel = s;
  sel::SelSet S; S.minGradHistCut = 0.5f; S.minGradHistAdd = 3; S.gradDownweightPerLevel = 0.75f; S.selectDirectionDistribution = 1;            // util/settings.cpp:119-122
  S.outlierTH = c->set.outlierTH; S.outlierTHSumComponent = c->set.outlierTHSumComponent; S.overallEnergyTHWeight = 1;
  if (s->eng.init(c->w, c->h, S, random_pattern, c->st)) { int rc = sel_fail(c, s, -1, "selector_init"); sel_destroy(c); return rc; }
  s->slots.resize(n_slots); s->cam.assign(n_slots, 0);
  { std::vector<int32_t> b0((size_t)4*n_slots); for (size_t k = 0; k < b0.size(); k++) b0[k] = kBox0[k & 3];
    if (cudaMalloc((void**)&s->boxD, b0.size()*sizeof(int32_t)) != cudaSuccess || cudaMemcpy(s->boxD, b0.data(), b0.size()*sizeof(int32_t), cudaMemcpyHostToDevice) != cudaSuccess) {
      cudaGetLastError(); sel_destroy(c); return ctx_fail(c, SDV_ERR_CUDA, "selector_init: pixel boxes of %d slots", n_slots); } }
  if (const char* e = getenv("SDV_WALK_THREADS")) { const int t = atoi(e); if (t == 32 || t == 64 || t == 128 || t == 256) s->eng.walk_threads = t; }   // tuning knobs
  if (const char* e = getenv("SDV_FUSE_MAP")) s->eng.fuse_map = atoi(e) != 0;
  return SDV_OK;
}
// Rebinding a slot to a camera of another size starts it afresh (map dropped, currentPotential 3, LiDAR pixel box at its initial value: a new PixelSelector /
// selectionMap / sequence); the same size keeps its state.
int sdv_selector_set_slot_cams(sdv_ctx* c, int n, const int32_t* slots, const int32_t* cams) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!slots || !cams))) return SDV_ERR_ARG; SEL_STATE("selector_set_slot_cams");
  { int rc = check_cams(c, n, cams, "selector_set_slot_cams", "entry"); if (rc) return rc; }
  for (int i = 0; i < n; i++) {
    if (slots[i] < 0 || slots[i] >= (int)s->slots.size()) return ctx_fail(c, SDV_ERR_ARG, "selector_set_slot_cams: entry %d names slot %d of %d", i, slots[i], (int)s->slots.size());
    if (c->cam_levels[cams[i]] < 3) return ctx_fail(c, SDV_ERR_ARG, "selector_set_slot_cams: entry %d names camera %d of %d levels (the selector reads levels 0..2)", i, cams[i], c->cam_levels[cams[i]]);
  }
  CK(cudaSetDevice(c->device));
  for (int i = 0; i < n; i++) { const int sl = slots[i];
    if (!same_size(c, s->cam[sl], cams[i])) { sel::SelectorSlot& S = s->slots[sl]; if (S.mapD) { CK(cudaStreamSynchronize(c->st)); CK(cudaFree(S.mapD)); } S = sel::SelectorSlot();
      CK(cudaMemcpyAsync(s->boxD + 4*(size_t)sl, kBox0, sizeof(kBox0), cudaMemcpyHostToDevice, c->st)); }
    s->cam[sl] = cams[i]; }
  return SDV_OK;
}
int sdv_selector_potential(sdv_ctx* c, int slot, int set_to, int* out) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG; SEL_STATE("selector_potential");
  if (slot < 0 || slot >= (int)s->slots.size()) return ctx_fail(c, SDV_ERR_ARG, "selector_potential: slot %d of %d", slot, (int)s->slots.size());
  if (set_to > 0) s->slots[slot].currentPotential = set_to;
  if (out) *out = s->slots[slot].currentPotential;
  return SDV_OK;
}
int sdv_selector_lidar_box(sdv_ctx* c, int slot, const int32_t* set_to, int32_t* lrud_out) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG; SEL_STATE("selector_lidar_box");
  if (slot < 0 || slot >= (int)s->slots.size()) return ctx_fail(c, SDV_ERR_ARG, "selector_lidar_box: slot %d of %d", slot, (int)s->slots.size());
  CK(cudaSetDevice(c->device));
  if (set_to) CK(cudaMemcpyAsync(s->boxD + 4*(size_t)slot, set_to, 4*sizeof(int32_t), cudaMemcpyHostToDevice, c->st));   // stream-ordered: after the handlers enqueued so far
  if (lrud_out) { CK(cudaMemcpyAsync(lrud_out, s->boxD + 4*(size_t)slot, 4*sizeof(int32_t), cudaMemcpyDeviceToHost, c->st)); CK(cudaStreamSynchronize(c->st)); }
  return SDV_OK;
}
int sdv_selector_get_map(sdv_ctx* c, int slot, uint8_t* out) { SDV_GUARD_TRK(c);
  if (!c || !out) return SDV_ERR_ARG; SEL_STATE("selector_get_map");
  if (slot < 0 || slot >= (int)s->slots.size()) return ctx_fail(c, SDV_ERR_ARG, "selector_get_map: slot %d of %d", slot, (int)s->slots.size());
  CK(cudaSetDevice(c->device));
  const int cam = s->cam[slot]; const size_t wh = (size_t)c->cam_w[cam]*c->cam_h[cam];
  if (!s->slots[slot].mapD) { memset(out, 0, wh); return SDV_OK; }
  CK(cudaMemcpyAsync(out, s->slots[slot].mapD, wh, cudaMemcpyDeviceToHost, c->st)); CK(cudaStreamSynchronize(c->st));
  return SDV_OK;
}
int sdv_selector_make_hists_cam(sdv_ctx* c, int cam, uint64_t frame, float* ths_out, float* thsSmoothed_out) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG; SEL_STATE("selector_make_hists");
  { int rc = check_cams(c, 1, &cam, "selector_make_hists", nullptr); if (rc) return rc; }
  CK(cudaSetDevice(c->device));
  sel::FrameImg F; const float* gw2; long long need = 0; { int rc = sel_frame(c, 0, frame, cam, F, gw2, need, "selector_make_hists", false); if (rc) return rc; }
  { int rc = join_ingest_upto(c, need); if (rc) return rc; }
  const int w = c->cam_w[cam], h = c->cam_h[cam];
  const size_t tf = sel::SelEngine::ths_floats(w, h); if (c->scr.reserve(2*Scratch::need(tf, 4), c->st)) return ctx_fail(c, SDV_ERR_CUDA, "selector_make_hists: scratch");
  c->scr.reset(); float* a = c->scr.take<float>(tf); float* b = c->scr.take<float>(tf);
  CK(cudaMemsetAsync(a, 0, tf*4, c->st)); CK(cudaMemsetAsync(b, 0, tf*4, c->st));
  sel::HistJob J{F.I0, a, b, w, h, gw2}; const long long l0 = s->eng.launches;
  if (s->eng.make_hists(1, &J)) return sel_fail(c, s, -1, "selector_make_hists");
  c->launches += s->eng.launches - l0;
  const int n = (w/32)*(h/32);
  if (ths_out) CK(cudaMemcpyAsync(ths_out, a, n*4, cudaMemcpyDeviceToHost, c->st));
  if (thsSmoothed_out) CK(cudaMemcpyAsync(thsSmoothed_out, b, n*4, cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  return SDV_OK;
}
int sdv_selector_make_hists(sdv_ctx* c, uint64_t frame, float* ths_out, float* thsSmoothed_out) { return sdv_selector_make_hists_cam(c, 0, frame, ths_out, thsSmoothed_out); }

int sdv_selector_make_maps_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const float* density,
                                 const int32_t* recursions_left, const float* th_factor, uint8_t* maps_out, int32_t* num_have_out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!slots || !frames || !density || !recursions_left || !th_factor || !maps_out))) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK; SEL_STATE("selector_make_maps");
  const bool lidar = cloud_begin != nullptr; if (lidar && !cloud3) return SDV_ERR_ARG;
  if (lidar) { int rc = check_offsets(c, n, cloud_begin, "selector_make_maps", "cloud_begin"); if (rc) return rc; }
  { int rc = check_ids(c, n, slots, (int)s->slots.size(), "selector_make_maps", "slot"); if (rc) return rc; }
  CK(cudaSetDevice(c->device));
  long long need = 0; std::vector<int> jw(n), jh(n);                                   // job j works at its slot's camera size
  for (int j = 0; j < n; j++) { const int cam = s->cam[slots[j]]; jw[j] = c->cam_w[cam]; jh[j] = c->cam_h[cam]; }
  std::vector<sel::FrameImg> F(n); std::vector<const float*> G(n);
  for (int j = 0; j < n; j++) { int rc = sel_frame(c, j, frames[j], s->cam[slots[j]], F[j], G[j], need, "selector_make_maps"); if (rc) return rc; }
  { int rc = join_ingest_upto(c, need); if (rc) return rc; }
  size_t bytes = 1024; for (int j = 0; j < n; j++) { const int m = lidar ? cloud_begin[j+1] - cloud_begin[j] : 0;
    bytes += 2*Scratch::need(sel::SelEngine::ths_floats(jw[j], jh[j]), 4) + Scratch::need(3*(size_t)m, 8) + Scratch::need(lidar ? (size_t)std::max(m, 1) : (size_t)jw[j]*jh[j], 1); }
  if (c->scr.reserve(bytes, c->st)) return ctx_fail(c, SDV_ERR_CUDA, "selector_make_maps: scratch");
  c->scr.reset(); std::vector<sel::MapsJobHost> M(n); std::vector<sel::HistJob> Hj(n);
  for (int j = 0; j < n; j++) { const int m = lidar ? cloud_begin[j+1] - cloud_begin[j] : 0; const size_t wh = (size_t)jw[j]*jh[j], tf = sel::SelEngine::ths_floats(jw[j], jh[j]);
    float* a = c->scr.take<float>(tf); float* b = c->scr.take<float>(tf); CK(cudaMemsetAsync(a, 0, tf*4, c->st)); CK(cudaMemsetAsync(b, 0, tf*4, c->st));
    double* cl = nullptr; if (lidar) { cl = c->scr.take<double>(3*(size_t)std::max(m, 1)); if (m) CK(cudaMemcpyAsync(cl, cloud3 + 3*(size_t)cloud_begin[j], 3*(size_t)m*sizeof(double), cudaMemcpyHostToDevice, c->st)); }
    sel::SelectorSlot& sl = s->slots[slots[j]];
    if (!lidar && !sl.mapD) { CK(cudaMalloc((void**)&sl.mapD, wh)); CK(cudaMemsetAsync(sl.mapD, 0, wh, c->st)); }
    Hj[j] = sel::HistJob{F[j].I0, a, b, jw[j], jh[j], G[j]};
    M[j].img = F[j]; M[j].w = jw[j]; M[j].h = jh[j]; M[j].thsSm = b; M[j].cloud_dev = cl; M[j].n = m; M[j].map = lidar ? c->scr.take<unsigned char>(std::max(m, 1)) : sl.mapD; M[j].density = density[j];
    M[j].recursionsLeft = recursions_left[j]; M[j].thFactor = th_factor[j]; M[j].currentPotential = &sl.currentPotential; M[j].numHaveSub = 0; M[j].passes = 0; M[j].gw2 = G[j]; }
  const long long l0 = s->eng.launches;
  if (s->eng.make_hists(n, Hj.data())) return sel_fail(c, s, -1, "selector_make_maps");
  if (s->eng.make_maps(M, lidar)) return sel_fail(c, s, -1, "selector_make_maps");
  c->launches += s->eng.launches - l0;
  size_t o = 0;
  for (int j = 0; j < n; j++) { const size_t sz = lidar ? (size_t)(cloud_begin[j+1] - cloud_begin[j]) : (size_t)jw[j]*jh[j];
    if (sz) CK(cudaMemcpyAsync(maps_out + o, M[j].map, sz, cudaMemcpyDeviceToHost, c->st)); o += sz; if (num_have_out) num_have_out[j] = M[j].numHaveSub; }
  CK(cudaStreamSynchronize(c->st));
  return SDV_OK;
}

}  // extern "C"
// makeNewTraces for n jobs; out == nullptr: the records go into the immature-point store (block of frames[j]) instead of to the caller
static int make_new_traces(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const float* density_lidar,
                           const float* density_dense, const int32_t* add_feature_point, int cap, sdv_new_trace* out, sdv_immature_pt* imm_out, int32_t* n_out, int32_t* num_points2,
                           const double* const* cloud_dev = nullptr /* job j's rows on the device (row sets), instead of cloud3 */) {
  if (n == 0) return SDV_OK; SEL_STATE("make_new_traces");
  { int rc = check_offsets(c, n, cloud_begin, "make_new_traces", "cloud_begin"); if (rc) return rc; }
  if (cloud_begin[n] > 0 && !cloud3 && !cloud_dev) return SDV_ERR_ARG;
  { int rc = check_ids(c, n, slots, (int)s->slots.size(), "make_new_traces", "slot"); if (rc) return rc; }
  if (!out) { int rc = check_distinct(c, n, frames, "make_new_traces_store", "frame"); if (rc) return rc; }
  CK(cudaSetDevice(c->device));
  long long need = 0; std::vector<sel::SelEngine::NewTracesJob> J(n);
  for (int j = 0; j < n; j++) { const int cam = s->cam[slots[j]]; int rc = sel_frame(c, j, frames[j], cam, J[j].img, J[j].gw2, need, "make_new_traces"); if (rc) return rc; J[j].w = c->cam_w[cam]; J[j].h = c->cam_h[cam];
    J[j].cloud_host = cloud3 ? cloud3 + 3*(size_t)cloud_begin[j] : nullptr; J[j].cloud_dev = cloud_dev ? cloud_dev[j] : nullptr; J[j].n = cloud_begin[j+1] - cloud_begin[j]; J[j].slot = &s->slots[slots[j]]; J[j].densityLidar = density_lidar[j];
    J[j].densityDense = density_dense[j]; J[j].addFeaturePoint = add_feature_point[j]; J[j].out_host = out ? (sel::NewTrace*)out + (size_t)j*cap : nullptr;
    J[j].imm_host = (out && imm_out) ? (sel::ImmPt*)imm_out + (size_t)j*cap : nullptr; J[j].cap = cap; }
  { int rc = join_ingest_upto(c, need); if (rc) return rc; }
  const long long l0 = s->eng.launches;
  CK(cudaEventRecord(c->ev0, c->st));
  { int rc = s->eng.make_new_traces(J); if (rc) return sel_fail(c, s, rc, "make_new_traces"); }
  if (!out) {                                                                            // device-output path: the records go from the engine's scratch into the store
    std::vector<int> cnt(n); std::vector<const void*> nt(n), im(n);
    for (int j = 0; j < n; j++) { cnt[j] = J[j].n_out; nt[j] = J[j].out_dev; im[j] = J[j].imm_dev; }
    int rc = imm_store_deposit(c, n, frames, cnt.data(), nt.data(), im.data()); if (rc) return rc;
  }
  CK(cudaEventRecord(c->ev1, c->st)); CK(cudaStreamSynchronize(c->st)); CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  c->launches += s->eng.launches - l0;
  for (int j = 0; j < n; j++) { n_out[j] = J[j].n_out; if (num_points2) { num_points2[2*j] = J[j].numPoints[0]; num_points2[2*j+1] = J[j].numPoints[1]; } }
  return SDV_OK;
}
extern "C" {
int sdv_make_new_traces_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const float* density_lidar,
                              const float* density_dense, const int32_t* add_feature_point, int cap, sdv_new_trace* out, sdv_immature_pt* imm_out, int32_t* n_out, int32_t* num_points2) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!slots || !frames || !cloud_begin || !density_lidar || !density_dense || !add_feature_point || !out || !n_out || cap < 1))) return SDV_ERR_ARG;
  return make_new_traces(c, n, slots, frames, cloud_begin, cloud3, density_lidar, density_dense, add_feature_point, cap, out, imm_out, n_out, num_points2);
}
int sdv_make_new_traces_store_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const float* density_lidar,
                                    const float* density_dense, const int32_t* add_feature_point, int cap, int32_t* n_out, int32_t* num_points2) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!slots || !frames || !cloud_begin || !density_lidar || !density_dense || !add_feature_point || !n_out || cap < 1))) return SDV_ERR_ARG;
  return make_new_traces(c, n, slots, frames, cloud_begin, cloud3, density_lidar, density_dense, add_feature_point, cap, nullptr, nullptr, n_out, num_points2);
}
// The same fed from the LiDAR row sets of frames[j] (sdv_lidar_handler_rows_batch): rows, box and addFeaturePoint as the handler left them for that frame.
int sdv_make_new_traces_rows_store_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const float* desired_density, int cap, int32_t* n_out,
                                         int32_t* num_points2) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!slots || !frames || !desired_density || !n_out || cap < 1))) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK; SEL_STATE("make_new_traces_rows");
  { int rc = check_ids(c, n, slots, (int)s->slots.size(), "make_new_traces_rows", "slot"); if (rc) return rc; }
  CK(cudaSetDevice(c->device));
  std::vector<const double*> rows(n); std::vector<LidarRowsInfo> I(n);                   // all headers in one copy: the row counts size the engine's scratch and grids
  { int rc = lidar_rows_fetch(c, n, frames, rows.data(), I.data(), "make_new_traces_rows"); if (rc) return rc; }
  std::vector<int32_t> cb(n + 1, 0), add(n); std::vector<float> dl(n);
  for (int j = 0; j < n; j++) { const LidarRowsInfo& q = I[j]; const int cam = s->cam[slots[j]];
    if (q.overflow) return ctx_fail(c, SDV_ERR_CAPACITY, "make_new_traces_rows: the sweep of frame %llu left %d pixel rows, its row set holds %d", (unsigned long long)frames[j], q.rows, q.room);
    dl[j] = ((float)((q.lrud[1] - q.lrud[0])*(q.lrud[3] - q.lrud[2])) / (float)(c->cam_w[cam]*c->cam_h[cam])) * desired_density[j];   // FullSystem.cpp:1287-1290
    add[j] = q.addFeaturePoint; cb[j+1] = cb[j] + q.rows; }
  return make_new_traces(c, n, slots, frames, cb.data(), nullptr, dl.data(), desired_density, add.data(), cap, nullptr, nullptr, n_out, num_points2, rows.data());
}

}  // extern "C"
// The start of a sequence for n jobs: CoarseInitializer::setFirstFromLidar at level 0 (CoarseInitializer.cpp:766-888), the point loop of
// FullSystem::initializeFromInitializer (FullSystem.cpp:1176-1225) and CoarseTracker::setCTRefForFirstFrame (CoarseTracker.cpp:636-647, :108-256).  Job j's rows are
// cloud3 + 3*cloud_begin[j] (host) or cloud_dev[j] (a row set), its box lrud[4j..].  Every check runs before anything is enqueued; the tracker and map slots
// are written only once every job's points are known to fit `cap`.
static int init_from_lidar(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const double* const* cloud_dev,
                           const int32_t* lrud, const float* desired, const int32_t* draw_begin, const int32_t* rand_draws, int cap, int32_t* n_out, int32_t* n_sel_out,
                           sdv_immature_pt* pts_out, sdv_immature_meta* meta_out, float* idepth_out) {
  const char* who = "init_from_lidar";
  if (n == 0) return SDV_OK; SEL_STATE("init_from_lidar");
  { int rc = check_offsets(c, n, cloud_begin, who, "cloud_begin"); if (rc) return rc; }
  if (draw_begin[0] < 0) return ctx_fail(c, SDV_ERR_ARG, "%s: draw_begin[0] = %d (must be >= 0)", who, draw_begin[0]);
  if (cloud_begin[n] > 0 && !cloud3 && !cloud_dev) return SDV_ERR_ARG;
  for (int j = 0; j < n; j++) { const int m = cloud_begin[j+1] - cloud_begin[j];
    if (draw_begin[j+1] - draw_begin[j] < m) return ctx_fail(c, SDV_ERR_ARG, "%s: job %d has %d rows and %d rand() draws", who, j, m, draw_begin[j+1] - draw_begin[j]); }
  { int rc = check_ids(c, n, slots, (int)c->slots.size(), who, "slot"); if (rc) return rc; }
  { int rc = check_distinct(c, n, frames, who, "frame"); if (rc) return rc; }
  CK(cudaSetDevice(c->device));
  long long need = 0; std::vector<FrameDev*> F(n); std::vector<int> cam(n);
  for (int j = 0; j < n; j++) { cam[j] = c->slots[slots[j]].cam;
    if (c->cam_levels[cam[j]] < 3) return ctx_fail(c, SDV_ERR_ARG, "%s: slot %d's camera has %d levels (the selector reads levels 0..2)", who, slots[j], c->cam_levels[cam[j]]);
    int rc = job_frame(c, who, j, frames[j], -1, slots[j], &need, &F[j]); if (rc) return rc; }
  std::vector<sel::FrameImg> img(n);
  for (int j = 0; j < n; j++) { int rc = ensure_texels(c, *F[j], 1); if (rc) return rc; img[j] = sel::FrameImg{F[j]->I0, F[j]->lvl[1], F[j]->lvl[2]}; }
  { int rc = join_ingest_upto(c, need); if (rc) return rc; }
  // every device array of the call in the engine's io scratch: the selection uses scr / scr2, the tracker reference c->scr
  const size_t nrows = (size_t)cloud_begin[n], ndraw = (size_t)(draw_begin[n] - draw_begin[0]);
  size_t bytes = Scratch::need(n, sizeof(InitPointsJob)) + Scratch::need(2*(size_t)n, 4) + Scratch::need(std::max(ndraw, (size_t)1), 4) + Scratch::need(cloud3 ? 3*std::max(nrows, (size_t)1) : 1, 8);
  for (int j = 0; j < n; j++) { const size_t m = std::max(cloud_begin[j+1] - cloud_begin[j], 1);
    bytes += 2*Scratch::need(sel::SelEngine::ths_floats(c->cam_w[cam[j]], c->cam_h[cam[j]]), 4) + Scratch::need(m, 1) + Scratch::need(m, sizeof(sdv_immature_pt)) + Scratch::need(m, sizeof(sdv_immature_meta))
           + Scratch::need(m, 4) + Scratch::need(4*m, 4) + Scratch::need(m, 4) + Scratch::need(m, sizeof(sdv_map_pt)); }
  Scratch& io = s->eng.io;
  if (io.reserve(bytes, c->st)) return ctx_fail(c, SDV_ERR_CUDA, "%s: scratch of %zu bytes", who, bytes);
  const long long l0 = s->eng.launches; int cd_launches = 0;
  CK(cudaEventRecord(c->ev0, c->st));
  io.reset(); InitPointsJob* dJ = io.take<InitPointsJob>(n); int* counts = io.take<int>(2*(size_t)n); int32_t* draws = io.take<int32_t>(std::max(ndraw, (size_t)1));
  double* cl = cloud3 ? io.take<double>(3*std::max(nrows, (size_t)1)) : nullptr;
  if (ndraw) CK(cudaMemcpyAsync(draws, rand_draws + draw_begin[0], ndraw*sizeof(int32_t), cudaMemcpyHostToDevice, c->st));
  if (cloud3 && nrows) CK(cudaMemcpyAsync(cl, cloud3, 3*nrows*sizeof(double), cudaMemcpyHostToDevice, c->st));
  std::vector<int> pot(n, 3); std::vector<sel::HistJob> Hj(n); std::vector<sel::MapsJobHost> M(n); std::vector<InitPointsJob> J(n);
  for (int j = 0; j < n; j++) { const int m = cloud_begin[j+1] - cloud_begin[j], w = c->cam_w[cam[j]], h = c->cam_h[cam[j]]; const size_t tf = sel::SelEngine::ths_floats(w, h), mm = std::max(m, 1);
    float* a = io.take<float>(tf); float* b = io.take<float>(tf); CK(cudaMemsetAsync(a, 0, tf*4, c->st)); CK(cudaMemsetAsync(b, 0, tf*4, c->st));
    const double* rows = cloud3 ? cl + 3*(size_t)cloud_begin[j] : cloud_dev[j];
    const int area = (lrud[4*j+1] - lrud[4*j])*(lrud[4*j+3] - lrud[4*j+2]);                      // lidarArea of the FullSystem box
    const float* gw2 = cam_gw2(c, F[j]->cam);
    Hj[j] = sel::HistJob{F[j]->I0, a, b, w, h, gw2};                                                  // a fresh PixelSelector: makeHists runs
    sel::MapsJobHost& q = M[j]; q.img = img[j]; q.w = w; q.h = h; q.thsSm = b; q.cloud_dev = rows; q.n = m; q.map = io.take<unsigned char>(mm);
    q.density = 0.03f*area; q.recursionsLeft = 1; q.thFactor = 2; q.currentPotential = &pot[j]; q.numHaveSub = 0; q.passes = 0; q.gw2 = gw2;   // makeMapsFromLidar(.., 0.03*lidarArea, 1, false, 2, ..)
    InitPointsJob& P = J[j]; P.cloud = rows; P.map = q.map; P.draws = draws + (draw_begin[j] - draw_begin[0]); P.I0 = F[j]->I0; P.n = m; P.w = w; P.h = h; P.desired = desired[j];
    P.pts = io.take<sdv_immature_pt>(mm); P.meta = io.take<sdv_immature_meta>(mm); P.idepth = io.take<float>(mm); P.splat4 = io.take<float>(4*mm); P.round = io.take<int>(mm);
    P.mp = io.take<sdv_map_pt>(mm); P.counts = counts + 2*j; }
  if (s->eng.make_hists(n, Hj.data())) return sel_fail(c, s, -1, who);
  if (s->eng.make_maps(M, true)) return sel_fail(c, s, -1, who);
  CK(cudaMemcpyAsync(dJ, J.data(), n*sizeof(InitPointsJob), cudaMemcpyHostToDevice, c->st));
  { int rc = launch_init_points(c, n, dJ); if (rc) return rc; }
  std::vector<int> cnt(2*(size_t)n);
  CK(cudaMemcpyAsync(cnt.data(), counts, cnt.size()*sizeof(int), cudaMemcpyDeviceToHost, c->st)); CK(cudaStreamSynchronize(c->st));
  int over = -1;
  for (int j = 0; j < n; j++) { n_sel_out[j] = cnt[2*j]; n_out[j] = cnt[2*j+1]; if (cnt[2*j+1] > cap && over < 0) over = j; }
  c->launches += s->eng.launches - l0;
  if (over >= 0) return ctx_fail(c, SDV_ERR_CAPACITY, "%s: job %d keeps %d points, cap is %d", who, over, n_out[over], cap);
  for (int j = 0; j < n; j++) { const size_t k = (size_t)n_out[j]; if (!k) continue;
    if (pts_out) CK(cudaMemcpyAsync(pts_out + (size_t)j*cap, J[j].pts, k*sizeof(sdv_immature_pt), cudaMemcpyDeviceToHost, c->st));
    if (meta_out) CK(cudaMemcpyAsync(meta_out + (size_t)j*cap, J[j].meta, k*sizeof(sdv_immature_meta), cudaMemcpyDeviceToHost, c->st));
    if (idepth_out) CK(cudaMemcpyAsync(idepth_out + (size_t)j*cap, J[j].idepth, k*sizeof(float), cudaMemcpyDeviceToHost, c->st)); }
  // install: setCTRefForFirstFrame from the splat rows (round_half 1, HdiF 0, lastRef_aff_g2l = (0,0)), and the map of one keyframe at camToWorld = SE3(), aff_g2l = (0,0)
  // one job per build: a job over max_ref_points stops the loop with the jobs before it installed
  static const double kT0[7] = {1, 0, 0, 0, 0, 0, 0}, kAb0[2] = {0, 0};
  for (int j = 0; j < n; j++) {
    const int32_t pb[2] = {0, n_out[j]}, hb[2] = {0, 1};
    { int rc = set_ref_build(c, 1, &slots[j], &F[j], &frames[j], pb, J[j].splat4, J[j].round, cudaMemcpyDeviceToDevice, nullptr, nullptr, &cd_launches); if (rc) return rc; }
    { int rc = map_set_impl(c, 1, &slots[j], hb, &frames[j], kT0, kAb0, pb, J[j].mp, cudaMemcpyDeviceToDevice); if (rc) return rc; }
  }
  CK(cudaEventRecord(c->ev1, c->st)); CK(cudaStreamSynchronize(c->st)); CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  c->launches += cd_launches;
  return SDV_OK;
}
extern "C" {
int sdv_init_from_lidar_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* cloud_begin, const double* cloud3, const int32_t* lrud,
                              const float* desired_point_density, const int32_t* draw_begin, const int32_t* rand_draws, int cap, int32_t* n_out, int32_t* n_selected_out,
                              sdv_immature_pt* pts_out, sdv_immature_meta* meta_out, float* idepth_out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!slots || !frames || !cloud_begin || !lrud || !desired_point_density || !draw_begin || !rand_draws || !n_out || !n_selected_out || cap < 0))) return SDV_ERR_ARG;
  return init_from_lidar(c, n, slots, frames, cloud_begin, cloud3, nullptr, lrud, desired_point_density, draw_begin, rand_draws, cap, n_out, n_selected_out, pts_out, meta_out, idepth_out);
}
// The same fed from the LiDAR row sets of frames[j]: rows and box as the handler left them for that frame (sdv_make_new_traces_rows_store_batch reads them the same way).
int sdv_init_from_lidar_rows_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const float* desired_point_density, const int32_t* draw_begin,
                                   const int32_t* rand_draws, int cap, int32_t* n_out, int32_t* n_selected_out, sdv_immature_pt* pts_out, sdv_immature_meta* meta_out,
                                   float* idepth_out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!slots || !frames || !desired_point_density || !draw_begin || !rand_draws || !n_out || !n_selected_out || cap < 0))) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK; SEL_STATE("init_from_lidar_rows");
  CK(cudaSetDevice(c->device));
  std::vector<const double*> rows(n); std::vector<LidarRowsInfo> I(n);                   // all headers in one copy
  { int rc = lidar_rows_fetch(c, n, frames, rows.data(), I.data(), "init_from_lidar_rows"); if (rc) return rc; }
  std::vector<int32_t> cb(n + 1, 0), box(4*(size_t)n);
  for (int j = 0; j < n; j++) { const LidarRowsInfo& q = I[j];
    if (q.overflow) return ctx_fail(c, SDV_ERR_CAPACITY, "init_from_lidar_rows: the sweep of frame %llu left %d pixel rows, its row set holds %d", (unsigned long long)frames[j], q.rows, q.room);
    for (int k = 0; k < 4; k++) box[4*j+k] = q.lrud[k];
    cb[j+1] = cb[j] + q.rows; }
  return init_from_lidar(c, n, slots, frames, cb.data(), nullptr, rows.data(), box.data(), desired_point_density, draw_begin, rand_draws, cap, n_out, n_selected_out, pts_out, meta_out, idepth_out);
}
}  // extern "C"
namespace sdv {
// makeDistanceMap + the candidate walk; cand4_dev != nullptr: the cand4 rows are device memory (the activation on the immature-point store)
int sel_activate_select(sdv_ctx* c, int n, const int32_t* host_begin, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* uvid,
                        const int32_t* cand_host_begin, const int32_t* cand_begin, const float* cKRKi9, const float* cKt3, const float* cand4, const float* cand4_dev,
                        const float* min_act_dist, const int32_t* cams, int32_t* decision_out, float* dist_map_out) {
  if (!c || n < 0 || (n && (!host_begin || !pt_begin || !cand_host_begin || !cand_begin || !min_act_dist))) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK; SEL_STATE("activate_select");
  { int rc = check_offsets(c, n, host_begin, "activate_select", "host_begin"); if (rc) return rc; }
  { int rc = check_offsets(c, n, cand_host_begin, "activate_select", "cand_host_begin"); if (rc) return rc; }
  { int rc = check_cams(c, n, cams, "activate_select", "sequence"); if (rc) return rc; }
  // the engine wants, per sequence, CSR offsets that start at 0: rebase the global ones
  std::vector<std::vector<int>> pb(n), cb(n); std::vector<sel::SelEngine::ActJob> J(n); size_t map_off = 0;     // distance maps back to back, each at its camera's level-1 size
  for (int j = 0; j < n; j++) {
    const int h0 = host_begin[j], h1 = host_begin[j+1], g0 = cand_host_begin[j], g1 = cand_host_begin[j+1];
    if (h1 - h0 > 16 || g1 - g0 > 16) return ctx_fail(c, SDV_ERR_ARG, "activate_select: sequence %d has %d source / %d candidate keyframes (0..16)", j, h1 - h0, g1 - g0);
    for (int k = h0; k <= h1; k++) { if (k > h0 && pt_begin[k] < pt_begin[k-1]) return ctx_fail(c, SDV_ERR_ARG, "activate_select: pt_begin is not ascending"); pb[j].push_back(pt_begin[k] - pt_begin[h0]); }
    for (int k = g0; k <= g1; k++) { if (k > g0 && cand_begin[k] < cand_begin[k-1]) return ctx_fail(c, SDV_ERR_ARG, "activate_select: cand_begin is not ascending"); cb[j].push_back(cand_begin[k] - cand_begin[g0]); }
    const int np = pb[j].back(), nc = cb[j].back();
    if ((np && (!KRKi9 || !Kt3 || !uvid)) || (nc && (!cKRKi9 || !cKt3 || (!cand4 && !cand4_dev) || !decision_out))) return SDV_ERR_ARG;
    sel::SelEngine::ActJob& a = J[j]; a.nHosts = h1 - h0; a.pt_begin = pb[j].data(); a.KRKi = KRKi9 ? KRKi9 + 9*(size_t)h0 : nullptr; a.Kt = Kt3 ? Kt3 + 3*(size_t)h0 : nullptr;
    a.uvid = uvid ? uvid + 3*(size_t)pt_begin[h0] : nullptr; a.nCandHosts = g1 - g0; a.cand_begin = cb[j].data(); a.cKRKi = cKRKi9 ? cKRKi9 + 9*(size_t)g0 : nullptr; a.cKt = cKt3 ? cKt3 + 3*(size_t)g0 : nullptr;
    a.cand4 = cand4 ? cand4 + 4*(size_t)cand_begin[g0] : nullptr; a.cand4_dev = cand4_dev ? cand4_dev + 4*(size_t)cand_begin[g0] : nullptr; a.minActDist = min_act_dist[j]; a.decision_host = decision_out ? decision_out + cand_begin[g0] : nullptr;
    const int cam = cams ? cams[j] : 0; a.w1 = c->cam_w[cam] >> 1; a.h1 = c->cam_h[cam] >> 1;
    a.map_host = dist_map_out ? dist_map_out + map_off : nullptr; map_off += (size_t)a.w1*a.h1;
  }
  CK(cudaSetDevice(c->device));
  const long long l0 = s->eng.launches;
  CK(cudaEventRecord(c->ev0, c->st));
  { int rc = s->eng.activate(J); if (rc) return sel_fail(c, s, rc, "activate_select"); }
  CK(cudaEventRecord(c->ev1, c->st)); CK(cudaStreamSynchronize(c->st)); CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  if (s->eng.have_ev) c->last_ms = s->eng.last_kernel_ms;                                  // the 43 launches, copies excluded
  c->launches += s->eng.launches - l0;
  return SDV_OK;
}
}  // namespace sdv
extern "C" {
int sdv_activate_select_batch_cams(sdv_ctx* c, int n, const int32_t* host_begin, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* uvid,
                                   const int32_t* cand_host_begin, const int32_t* cand_begin, const float* cKRKi9, const float* cKt3, const float* cand4, const float* min_act_dist,
                                   const int32_t* cams, int32_t* decision_out, float* dist_map_out) { SDV_GUARD_TRK(c);
  return sel_activate_select(c, n, host_begin, pt_begin, KRKi9, Kt3, uvid, cand_host_begin, cand_begin, cKRKi9, cKt3, cand4, nullptr, min_act_dist, cams, decision_out, dist_map_out);
}
int sdv_activate_select_batch(sdv_ctx* c, int n, const int32_t* host_begin, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* uvid,
                              const int32_t* cand_host_begin, const int32_t* cand_begin, const float* cKRKi9, const float* cKt3, const float* cand4, const float* min_act_dist,
                              int32_t* decision_out, float* dist_map_out) {
  return sdv_activate_select_batch_cams(c, n, host_begin, pt_begin, KRKi9, Kt3, uvid, cand_host_begin, cand_begin, cKRKi9, cKt3, cand4, min_act_dist, nullptr, decision_out, dist_map_out);
}

}  // extern "C"
