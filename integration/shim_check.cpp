// integration/shim_check.cpp — the shims of INTEGRATION.md as a COMPILED translation unit.
//
// The reference has no plugin layer: libsdv_b200.so is dropped in by swapping the bodies of a few member functions (INTEGRATION.md §3).  The reference's own
// headers cannot be compiled in this image (Eigen3/Boost/ROS absent), so this file declares minimal stand-ins with the SAME member names and types the shims
// touch (FrameShell::id, PointHessian::{u,v,idepth,...}, SE3, AffLight, Vec5, ...) and then contains the shim bodies verbatim.  tests/test_abi.py compiles it
// (g++ -std=c++14 -Wall -Werror -fsyntax-only) and links it against libsdv_b200.so with --no-undefined: every call in INTEGRATION.md is type-checked against
// include/sdv_b200.h and resolves to an exported C symbol.  It is never executed.
#include <cstddef>
#include <cstdint>
#include <utility>
#include <vector>
#include <cstdlib>
#include "sdv_b200.h"

// ------------------------------------------------------------------------------------------------ stand-ins for the reference's types (names as in the reference)
struct Quat { double w_, x_, y_, z_; double w() const { return w_; } double x() const { return x_; } double y() const { return y_; } double z() const { return z_; } };
struct Vec3 { double v[3]; double operator[](int i) const { return v[i]; } };
struct SE3 {                                                                   // Sophus::SE3d: unit_quaternion(), translation()
  Quat q; Vec3 t;
  SE3() : q{1, 0, 0, 0}, t{{0, 0, 0}} {}
  SE3(const Quat& q_, const Vec3& t_) : q(q_), t(t_) {}
  const Quat& unit_quaternion() const { return q; } const Vec3& translation() const { return t; }
};
struct AffLight { double a, b; AffLight(double a_ = 0, double b_ = 0) : a(a_), b(b_) {} };   // util/NumType.h:129-175
struct Vec5 { double v[5]; const double* data() const { return v; } double& operator[](int i) { return v[i]; } };
struct Vec4 { double v[4]; };
struct Vec10 { double v[10]; const double* data() const { return v; } };
struct VecC { double v[4]; const double* data() const { return v; } };
enum class ResState { IN = 0, OOB, OUTLIER };
struct FrameHessian; struct PointHessian;
struct FrameShell { int id; SE3 camToWorld, camToTrackingRef; AffLight aff_g2l; bool poseValid; FrameShell* trackingRef; };   // util/FrameShell.h
struct EFPoint { float HdiF; };
struct Vec3f { float v[3]; float operator[](int i) const { return v[i]; } };
struct PointFrameResidual { Vec3f centerProjectedTo; ResState state_state; FrameHessian* host; FrameHessian* target; bool hasMatcher; float matcher[2]; bool isNew; };
struct PointHessian {                                                          // FullSystem/HessianBlocks.h:361-465
  float u, v, idepth, idepth_zero, color[8], weights[8]; bool hasDepthPrior, isFromSensor; int type; enum { EDGELET = 1 };
  FrameHessian* host; EFPoint* efPoint; std::vector<PointFrameResidual*> residuals; std::pair<PointFrameResidual*, ResState> lastResiduals[2];
};
struct FrameHessian {                                                          // FullSystem/HessianBlocks.h:104-258
  FrameShell* shell; float ab_exposure; int idx, frameID; float frameEnergyTH; bool flaggedForMarginalization;
  std::vector<PointHessian*> pointHessians; SE3 worldToCam_evalPT; Vec10 state, state_zero;
  AffLight aff_g2l() const { return shell->aff_g2l; }
  void makeImages(float* color, struct CalibHessian* HCalib);
};
struct CalibHessian { VecC value_scaled, value_zero; float fxl() const { return (float)value_scaled.v[0]; } float fyl() const { return (float)value_scaled.v[1]; }
                      float cxl() const { return (float)value_scaled.v[2]; } float cyl() const { return (float)value_scaled.v[3]; } };
struct Undistort { int wOrg, hOrg; float* remapX; float* remapY; };           // util/Undistort.h (remapX/remapY: protected there — one friend declaration or two getters)
namespace IOWrap { struct Output3DWrapper; }
static sdv_ctx* gpu = nullptr;                                                 // FullSystem member in the real integration (INTEGRATION.md §2)
extern float setting_huberTH, setting_coarseCutoffTH, setting_affineOptModeA, setting_affineOptModeB, setting_outlierTHSumComponent, setting_idepthFixPrior, setting_desiredImmatureDensity;
extern int setting_maxFrames, pyrLevelsUsed, wG[8], hG[8];

static void se3_to7(const SE3& T, double o[7]) {
  o[0] = T.unit_quaternion().w(); o[1] = T.unit_quaternion().x(); o[2] = T.unit_quaternion().y(); o[3] = T.unit_quaternion().z();
  o[4] = T.translation()[0]; o[5] = T.translation()[1]; o[6] = T.translation()[2];
}
static SE3 se3_from7(const double* v) { return SE3(Quat{v[0], v[1], v[2], v[3]}, Vec3{{v[4], v[5], v[6]}}); }

// ------------------------------------------------------------------------------------------------ §2 one context per FullSystem (FullSystem.cpp:119)
int shim_create(CalibHessian& Hcalib) {
  sdv_settings s; sdv_default_settings(&s);
  s.huberTH = setting_huberTH; s.coarseCutoffTH = setting_coarseCutoffTH; s.affineOptModeA = setting_affineOptModeA; s.affineOptModeB = setting_affineOptModeB;
  s.outlierTHSumComponent = setting_outlierTHSumComponent; s.idepthFixPrior = setting_idepthFixPrior;
  s.n_tracker_slots = 2; s.max_frames = setting_maxFrames + 3; s.cluster_size = 8; s.track_threads = 256;
  sdv_calib K{Hcalib.fxl(), Hcalib.fyl(), Hcalib.cxl(), Hcalib.cyl()};
  return sdv_create(&K, wG[0], hG[0], pyrLevelsUsed, &s, /*device*/0, &gpu);
}

// ------------------------------------------------------------------------------------------------ §3 FrameHessian::makeImages (HessianBlocks.cpp:107-167)
void FrameHessian::makeImages(float* color, CalibHessian*) { sdv_frame_upload(gpu, (uint64_t)shell->id, color, ab_exposure); }
void shim_frame_destructor(FrameHessian* fh) { sdv_frame_release(gpu, (uint64_t)fh->shell->id); }

// §3b ingest: Undistort tables once, raw mono8 per frame (util/DatasetReader.h:223-230, Undistort.cpp:341-435)
int shim_set_undistort(const Undistort* u, const float* G256_or_null, const float* vignetteInv_or_null) {
  return sdv_set_undistort(gpu, u->wOrg, u->hOrg, u->remapX, u->remapY, 1.0f, G256_or_null, vignetteInv_or_null);
}
int shim_ingest_raw(FrameShell* shell, const uint8_t* raw_mono8, float exposure) {
  uint64_t id = (uint64_t)shell->id; return sdv_frame_upload_batch_raw_u8(gpu, 1, &id, &raw_mono8, &exposure);
}
// §4 batched mode, one context for several cameras: tables per camera, each raw image names its camera
int shim_set_undistort_cam(int cam, const Undistort* u) {
  return sdv_set_undistort_cam(gpu, cam, u->wOrg, u->hOrg, u->remapX, u->remapY, 1.0f, nullptr, nullptr);
}
// §4 one FullSystem::setGammaFunction per camera: G of that camera's PhotometricUndistorter (NULL: no calibration), before any frame of the camera is resident
int shim_set_gamma_cam(int cam, float* G_or_null) { return sdv_set_gamma_cam(gpu, cam, G_or_null); }
int shim_ingest_raw_cams(int n, const uint64_t* ids, const uint8_t* const* raw_mono8, const int32_t* cams, const float* exposures) {
  return sdv_frame_upload_batch_raw_u8_cams(gpu, n, ids, raw_mono8, cams, exposures);
}
// §4 cameras of different rectified sizes in one context (created at the largest, KITTI-360's 1400x360): KITTI's 1200x360 on camera 1, its
// sequences' slots bound to that camera, rectified or device-resident frames of each camera's size
// §4 the per-keyframe makeK of a slot bound to camera `cam`: the K moves, the camera stays
int shim_makeK_cam(int slot, int cam, const sdv_calib* K_after_ba) { const int32_t s = slot, c = cam; return sdv_set_calib_slots_cams(gpu, 1, &s, K_after_ba, &c); }
int shim_kitti_camera(int cam, const Undistort* u, int w, int h /*Undistort::getSize()*/, int n, const int32_t* slots, const sdv_calib* K) {
  int rc = sdv_set_camera_size(gpu, cam, w, h); if (rc) return rc;
  rc = shim_set_undistort_cam(cam, u); if (rc) return rc;
  std::vector<int32_t> cams(n, cam);
  return sdv_set_calib_slots_cams(gpu, n, slots, K, cams.data());
}
int shim_ingest_cams(int n, const uint64_t* ids, const uint8_t* const* mono8, const void* const* dev_float, const int32_t* cams, const float* exposures) {
  return sdv_frame_upload_batch_cams(gpu, n, ids, reinterpret_cast<const void* const*>(mono8), cams, /*fmt mono8*/1, exposures)
       | sdv_frame_build_batch_dev_cams(gpu, n, ids, dev_float, cams, /*fmt float*/0, exposures);
}
// §4 the keyframe path of a KITTI sequence on camera 1 in a KITTI-360 context: its selector slot bound to camera 1, then every keyframe-rate stage names camera 1
struct KittiKeyframe { int32_t slot, cam; uint64_t kf, next; std::vector<float> xyzi; double Rlc9[9], tlc3[3]; float K4[4]; int32_t lrud[4]; };
int shim_kitti_keyframe(KittiKeyframe& k, float density, std::vector<sdv_new_trace>& tr, std::vector<sdv_immature_pt>& imm, std::vector<int32_t>& decision) {
  int rc = sdv_selector_set_slot_cams(gpu, 1, &k.slot, &k.cam);                               // once per sequence: its PixelSelector works at 1200x360
  const int32_t sweep_begin[2] = {0, (int32_t)(k.xyzi.size() / 4)}; const int cap = 64 * 1800; std::vector<double> px(3 * (size_t)cap); int32_t n_px = 0, add = 0;
  rc |= sdv_lidar_handler_batch_cams(gpu, 1, sweep_begin, k.xyzi.data(), k.Rlc9, k.tlc3, k.K4, &k.cam, k.lrud, cap, px.data(), &n_px, &add, nullptr);   // box bounded by 1200x360
  const int32_t cloud_begin[2] = {0, n_px}; const float dl = density * (float)((k.lrud[1] - k.lrud[0]) * (k.lrud[3] - k.lrud[2])) / (1200.f * 360.f);
  tr.resize(1 << 15); imm.resize(1 << 15); int32_t n_out = 0, num[2];
  rc |= sdv_make_new_traces_batch(gpu, 1, &k.slot, &k.kf, cloud_begin, px.data(), &dl, &density, &add, 1 << 15, tr.data(), imm.data(), &n_out, num);   // the slot's camera
  tr.resize(n_out); imm.resize(n_out);
  const int32_t pt_begin[2] = {0, n_out}; const float I9[9] = {1, 0, 0, 0, 1, 0, 0, 0, 1}, z3[3] = {0, 0, 0}, aff[2] = {1, 0};
  rc |= sdv_immature_trace_batch_cams(gpu, 1, &k.next, &k.cam, pt_begin, I9, z3, aff, imm.data(), nullptr);                    // traceNewCoarse at 1200x360
  std::vector<float> cand4; for (int i = 0; i < n_out; i++) cand4.insert(cand4.end(), {imm[i].u, imm[i].v, 0.5f * (imm[i].idepth_max + imm[i].idepth_min), tr[i].my_type});
  const int32_t host_begin[2] = {0, 0}, pt0[1] = {0}, cand_host_begin[2] = {0, 1}, cand_begin[2] = {0, n_out}; const float md = 2.f; decision.resize(n_out);
  return rc | sdv_activate_select_batch_cams(gpu, 1, host_begin, pt0, nullptr, nullptr, nullptr, cand_host_begin, cand_begin, I9, z3, cand4.data(), &md, &k.cam,
                                             decision.data(), nullptr);                            // distance map and walk at 600x180
}
// §4 cameras of different pyramid depths (KITTI-CARLA 1392x1024 at 5 levels next to KITTI at 4, in a 1400x1024 context at 5): each camera at pyrLevelsUsed
int shim_camera_depths(int n_cams, const int* w, const int* h) {
  int rc = 0;
  for (int cam = 0; cam < n_cams; cam++) rc |= sdv_set_camera_levels(gpu, cam, sdv_pyr_levels(w[cam], h[cam]));
  return rc;
}
// §4 frame storage per camera: each camera's pool at its own size (before its first frame), and the bytes one frame and one keyframe image take there
int shim_camera_storage(int n_cams, const int* max_frames, const int* max_kf_images, uint64_t* frame_bytes, uint64_t* kf_bytes) {
  int rc = 0;
  for (int cam = 1; cam < n_cams; cam++) rc |= sdv_set_camera_storage(gpu, cam, max_frames[cam], max_kf_images[cam]);
  for (int cam = 0; cam < n_cams; cam++) rc |= sdv_camera_storage_bytes(gpu, cam, &frame_bytes[cam], &kf_bytes[cam]);
  return rc;
}
int shim_track_own_depths(int n, const int32_t* slots, const uint64_t* frames, double* T, double* ab, double* lastRes, double* flow, int32_t* good) {
  return sdv_tracker_track_batch_levels(gpu, n, slots, frames, T, ab, /*each job at its camera's depth - 1*/nullptr, nullptr, lastRes, flow, good, nullptr);
}
// §3c CoarseTracker::makeK (CoarseTracker.cpp:77-106): a member of each tracker instance, so it sets the K of that instance's slot only
int shim_makeK(int slot, CalibHessian* HCalib) { sdv_calib K{HCalib->fxl(), HCalib->fyl(), HCalib->cxl(), HCalib->cyl()}; const int32_t s = slot; return sdv_set_calib_slots(gpu, 1, &s, &K); }

// ------------------------------------------------------------------------------------------------ CoarseTracker (CoarseTracker.cpp:649-660, 662-838)
struct CoarseTracker {
  int slot; FrameHessian* lastRef; int refFrameID; AffLight lastRef_aff_g2l; double firstCoarseRMSE; Vec5 lastResiduals; double lastFlowIndicators[3];
  // the graph walk of makeCoarseDepthL0 :264-294 stays on the host: one row per splat, appended to pts / round_half
  static void splat_rows(const std::vector<FrameHessian*>& frameHessians, std::vector<float>& pts, std::vector<int32_t>& round_half) {
    for (FrameHessian* fh : frameHessians) for (PointHessian* ph : fh->pointHessians) {
      if (fh == frameHessians.back() && ph->isFromSensor) {
        pts.insert(pts.end(), {ph->u, ph->v, ph->idepth, ph->efPoint->HdiF}); round_half.push_back(0);
      } else if (ph->lastResiduals[0].first && ph->lastResiduals[0].second == ResState::IN && fh != frameHessians.back() && ph->isFromSensor) {
        PointFrameResidual* r = ph->lastResiduals[0].first;
        pts.insert(pts.end(), {r->centerProjectedTo[0], r->centerProjectedTo[1], r->centerProjectedTo[2], ph->efPoint->HdiF}); round_half.push_back(1);
      }
    }
  }
  void setCoarseTrackingRef(std::vector<FrameHessian*> frameHessians) {
    lastRef = frameHessians.back();
    std::vector<float> pts; std::vector<int32_t> round_half; splat_rows(frameHessians, pts, round_half);
    sdv_tracker_set_ref(gpu, slot, (uint64_t)lastRef->shell->id, (int)round_half.size(), pts.data(), round_half.data(), 0.f, lastRef->aff_g2l().a, lastRef->aff_g2l().b);
    refFrameID = lastRef->shell->id; lastRef_aff_g2l = lastRef->aff_g2l(); firstCoarseRMSE = -1;
  }
  bool trackNewestCoarse(FrameHessian* fh, SE3& lastToNew_out, AffLight& aff_g2l_out, int coarsestLvl, Vec5 minResForAbort, IOWrap::Output3DWrapper*) {
    double T[7]; se3_to7(lastToNew_out, T);
    double ab[2] = {aff_g2l_out.a, aff_g2l_out.b}, res[5], flow[3]; int good = 0;
    sdv_tracker_track(gpu, slot, (uint64_t)fh->shell->id, T, ab, coarsestLvl, minResForAbort.data(), res, flow, &good, nullptr);
    lastToNew_out = se3_from7(T); aff_g2l_out = AffLight(ab[0], ab[1]);
    for (int i = 0; i < 5; i++) lastResiduals[i] = res[i];
    for (int i = 0; i < 3; i++) lastFlowIndicators[i] = flow[i];
    return good != 0;
  }
};

// ------------------------------------------------------------------------------------------------ FullSystem members
struct FullSystem {
  std::vector<FrameHessian*> frameHessians; std::vector<FrameShell*> allFrameHistory; CalibHessian Hcalib; CoarseTracker* coarseTracker; Vec5 lastCoarseRMSE;
  std::vector<double> HM, bM;                                                   // ef->HM / ef->bM, row-major copies
  std::vector<int32_t> cell_order;                                              // Reprojector grid_.cell_order (Reprojector.cpp:107)

  // FullSystem::setGammaFunction (FullSystem.cpp:225-249), called by main.cpp with getPhotometricGamma() before the first frame: the body stays (Hcalib.B) and
  // the same BInv goes to the library, which inverts it alike and weighs every absSquaredGrad of this context's camera with it.  A NULL BInv returns at once in
  // the reference; the library takes it as the identity, which is what a fresh FullSystem has.
  void setGammaFunction(float* BInv) { if (BInv == 0) return; sdv_set_gamma_cam(gpu, 0, BInv); }

  // a window flattened in ef->frames / allPoints / residualsAll order (EnergyFunctional::makeIDX, EnergyFunctional.cpp:761-782); append() adds one window to the
  // concatenated arrays of a batched install (res_begin block of nP + 1 window-local entries, per-window begins)
  struct WindowRows {
    std::vector<uint64_t> ids; std::vector<double> T_eval, state, state_zero, calib, calib_zero, HM, bM; std::vector<float> exposure, energyTH; std::vector<int32_t> frameID;
    std::vector<float> uv, idepth, idepth_zero, color, weights, r_matcher; std::vector<int32_t> host, hasPrior, fromSensor, res_begin, r_point, r_host, r_target, r_hasM, r_isNew;
    std::vector<int32_t> f_begin{0}, p_begin{0}, r_begin{0};
  };
  void append(WindowRows& w) const {
    const int nF = (int)frameHessians.size(), p0 = (int)w.host.size(), r0 = (int)w.r_point.size();
    for (int i = 0; i < nF; i++) { FrameHessian* fh = frameHessians[i]; double T[7]; se3_to7(fh->worldToCam_evalPT, T);
      w.ids.push_back((uint64_t)fh->shell->id); w.T_eval.insert(w.T_eval.end(), T, T + 7); w.exposure.push_back(fh->ab_exposure); w.frameID.push_back(fh->frameID); w.energyTH.push_back(fh->frameEnergyTH);
      for (int k = 0; k < 10; k++) { w.state.push_back(fh->state.data()[k]); w.state_zero.push_back(fh->state_zero.data()[k]); } }
    w.calib.insert(w.calib.end(), Hcalib.value_scaled.data(), Hcalib.value_scaled.data() + 4); w.calib_zero.insert(w.calib_zero.end(), Hcalib.value_zero.data(), Hcalib.value_zero.data() + 4);
    w.HM.insert(w.HM.end(), HM.begin(), HM.begin() + (size_t)(4 + 6*nF)*(4 + 6*nF)); w.bM.insert(w.bM.end(), bM.begin(), bM.begin() + 4 + 6*nF);
    w.res_begin.push_back(0);
    for (FrameHessian* fh : frameHessians) for (PointHessian* ph : fh->pointHessians) {
      const int p = (int)w.host.size() - p0;
      w.uv.push_back(ph->u); w.uv.push_back(ph->v); w.idepth.push_back(ph->idepth); w.idepth_zero.push_back(ph->idepth_zero);
      w.color.insert(w.color.end(), ph->color, ph->color + 8); w.weights.insert(w.weights.end(), ph->weights, ph->weights + 8);
      w.host.push_back(fh->idx); w.hasPrior.push_back(ph->hasDepthPrior); w.fromSensor.push_back(ph->isFromSensor);
      for (PointFrameResidual* r : ph->residuals) { w.r_point.push_back(p); w.r_host.push_back(r->host->idx); w.r_target.push_back(r->target->idx); w.r_hasM.push_back(r->hasMatcher);
        w.r_matcher.push_back(r->matcher[0]); w.r_matcher.push_back(r->matcher[1]); w.r_isNew.push_back(r->isNew); }
      w.res_begin.push_back((int32_t)w.r_point.size() - r0);
    }
    w.f_begin.push_back((int32_t)w.ids.size()); w.p_begin.push_back((int32_t)w.host.size()); w.r_begin.push_back((int32_t)w.r_point.size());
  }

  // FullSystem::optimize (FullSystemOptimize.cpp:344-502) on this system's window alone
  float optimize(int mnumOptIts) {
    const int nF = (int)frameHessians.size(); WindowRows w; append(w);
    const std::vector<int32_t>& host = w.host;
    int rc = sdv_ba_set_window(gpu, nF, w.ids.data(), w.T_eval.data(), w.state.data(), w.state_zero.data(), w.exposure.data(), w.frameID.data(), w.energyTH.data(), Hcalib.value_scaled.data(), HM.data(), bM.data());
    if (rc == SDV_OK) rc = sdv_ba_set_calib_zero(gpu, Hcalib.value_zero.data());                   // the linearisation point of the intrinsics stays at the initial K (HessianBlocks.h:287)
    if (rc == SDV_OK) rc = sdv_ba_set_points(gpu, (int)host.size(), w.uv.data(), w.idepth.data(), w.idepth_zero.data(), w.color.data(), w.weights.data(), host.data(), w.hasPrior.data(), w.fromSensor.data(),
                                             w.res_begin.data(), (int)w.r_point.size(), w.r_point.data(), w.r_host.data(), w.r_target.data(), w.r_hasM.data(), w.r_matcher.data(), w.r_isNew.data());
    float rmse = 0; int32_t its = 0, acc = 0;
    if (rc == SDV_OK) rc = sdv_ba_optimize(gpu, mnumOptIts, &rmse, &its, &acc);
    std::vector<double> Tn(7*nF), st(10*nF), step(10*nF), pre(7*nF); std::vector<float> th(nF); double cv[4], cs[4];
    if (rc == SDV_OK) sdv_ba_get_frames(gpu, Tn.data(), st.data(), step.data(), th.data(), pre.data(), cv, cs);        // -> FrameHessian::setEvalPT / setState, Hcalib.setValue
    std::vector<float> idn(host.size()), stp(host.size()), hdi(host.size()), bds(host.size()), mrb(host.size()), idh(host.size()); std::vector<int32_t> ngood(host.size());
    if (rc == SDV_OK) sdv_ba_get_points(gpu, idn.data(), stp.data(), hdi.data(), bds.data(), mrb.data(), ngood.data(), idh.data());   // -> PointHessian::setIdepth, idepth_hessian, maxRelBaseline, numGoodResiduals
    return rmse;
  }

  // FullSystem::makeKeyFrame: keep the map resident for the Reprojector (Reprojector.cpp:117-156) ...
  void map_rows(std::vector<uint64_t>& ids, std::vector<double>& c2w, std::vector<double>& ab, std::vector<sdv_map_pt>& pts) const {   // appended, host index job-local
    for (FrameHessian* fh : frameHessians) {
      ids.push_back((uint64_t)fh->shell->id); double T[7]; se3_to7(fh->shell->camToWorld, T); c2w.insert(c2w.end(), T, T + 7); ab.push_back(fh->aff_g2l().a); ab.push_back(fh->aff_g2l().b);
      for (PointHessian* ph : fh->pointHessians) pts.push_back(sdv_map_pt{ph->u, ph->v, ph->idepth, fh->idx, ph->type == PointHessian::EDGELET});
    }
  }
  int set_map(int slot) {
    std::vector<sdv_map_pt> pts; std::vector<uint64_t> ids; std::vector<double> c2w, ab; map_rows(ids, c2w, ab, pts);
    return sdv_map_set(gpu, slot, (int)ids.size(), ids.data(), c2w.data(), ab.data(), (int)pts.size(), pts.data());
  }
  // ... and the hand-over after optimize(): flagPointsForRemoval / marginalizePointsF / marginalizeFrame (FullSystem.cpp:1152-1171)
  int handover(const std::vector<int32_t>& selected, std::vector<int32_t>& status) {
    status.resize(selected.size());
    int rc = sdv_ba_flag_points(gpu, selected.data(), status.data());
    if (rc == SDV_OK) rc = sdv_ba_marginalize_points(gpu, nullptr);
    for (FrameHessian* fh : frameHessians) if (rc == SDV_OK && fh->flaggedForMarginalization) rc = sdv_ba_marginalize_frame(gpu, fh->idx);
    int dim = 0; HM.resize(68*68); bM.resize(68); if (rc == SDV_OK) rc = sdv_ba_get_prior(gpu, &dim, HM.data(), bM.data());
    return rc;
  }

  // Vec4 FullSystem::trackNewCoarse(FrameHessian* fh) for a running system (FullSystem.cpp:283-500)
  Vec4 trackNewCoarse(FrameHessian* fh) {
    FrameShell* slast = allFrameHistory[allFrameHistory.size() - 2]; FrameShell* sprelast = allFrameHistory[allFrameHistory.size() - 3]; FrameHessian* lastF = coarseTracker->lastRef;
    sdv_track_new_coarse_io io{}; io.slot = coarseTracker->slot; io.frame = (uint64_t)fh->shell->id;
    io.poses_valid = slast->poseValid && sprelast->poseValid && lastF->shell->poseValid;
    se3_to7(sprelast->camToWorld, io.sprelast_c2w); se3_to7(slast->camToWorld, io.slast_c2w); se3_to7(lastF->shell->camToWorld, io.lastF_c2w);
    io.aff_last[0] = slast->aff_g2l.a; io.aff_last[1] = slast->aff_g2l.b;
    for (int i = 0; i < 5; i++) io.lastCoarseRMSE[i] = lastCoarseRMSE[i];
    sdv_track_new_coarse_batch(gpu, 1, &io, cell_order.data(), (int)(0.8f*setting_desiredImmatureDensity));
    fh->shell->camToWorld = se3_from7(io.camToWorld); fh->shell->camToTrackingRef = se3_from7(io.camToTrackingRef); fh->shell->trackingRef = lastF->shell;
    fh->shell->aff_g2l = AffLight(io.aff_g2l[0], io.aff_g2l[1]);
    for (int i = 0; i < 5; i++) lastCoarseRMSE[i] = io.lastCoarseRMSE[i];
    return Vec4{{io.lastCoarseRMSE[0], io.flow[0], io.flow[1], io.flow[2]}};
  }
  // the two members of the tail separately (overlap_pts wanted by the caller): Reprojector::reprojectMap + CoarseTracker::structPoseEstimation
  int refine_only(FrameHessian* fh) {
    double T[7]; se3_to7(fh->shell->camToWorld, T); double ab[2] = {fh->aff_g2l().a, fh->aff_g2l().b}; int32_t s = coarseTracker->slot, nm = 0; uint64_t id = (uint64_t)fh->shell->id;
    int rc = sdv_tracker_refine_batch(gpu, 1, &s, &id, T, ab, cell_order.data(), (int)(0.8f*setting_desiredImmatureDensity), &nm, nullptr, nullptr, nullptr);
    fh->shell->camToWorld = se3_from7(T); return rc;
  }
};

// ------------------------------------------------------------------------------------------------ immature points: FullSystem::traceNewCoarse (FullSystem.cpp:519-552)
struct Mat33f { float m[9]; }; struct Vec2f { float v[2]; };
struct ImmaturePoint { sdv_immature_pt rec; FrameHessian* host; };            // the reference's members u,v,idepth_min/max,color,weights,gradH,energyTH,quality,lastTrace* in one record
struct HostImmatures { FrameHessian* host; std::vector<ImmaturePoint*> immaturePoints; Mat33f KRKi; Vec3f Kt; Vec2f aff; };   // per host: what :532-538 computes
int shim_makeNewTraces(FrameHessian* newFrame, const std::vector<int32_t>& uv /*2 per selected pixel (PixelSelector)*/, std::vector<ImmaturePoint*>& out) {
  std::vector<sdv_immature_pt> rec(uv.size()/2);
  int rc = sdv_immature_init(gpu, (uint64_t)newFrame->shell->id, (int)rec.size(), uv.data(), rec.data());   // ImmaturePoint::ImmaturePoint for every candidate (FullSystem.cpp:1273-1356)
  for (std::size_t i = 0; i < rec.size() && rc == SDV_OK; i++) out.push_back(new ImmaturePoint{rec[i], newFrame});
  return rc;
}
int shim_traceNewCoarse(FrameHessian* fh, std::vector<HostImmatures>& hosts) {
  std::vector<uint64_t> frames; std::vector<int32_t> pt_begin{0}; std::vector<float> KRKi, Kt, aff; std::vector<sdv_immature_pt> pts;
  for (HostImmatures& h : hosts) {
    frames.push_back((uint64_t)fh->shell->id); KRKi.insert(KRKi.end(), h.KRKi.m, h.KRKi.m + 9); for (int i = 0; i < 3; i++) Kt.push_back((float)h.Kt[i]); aff.push_back(h.aff.v[0]); aff.push_back(h.aff.v[1]);
    for (ImmaturePoint* ph : h.immaturePoints) pts.push_back(ph->rec);
    pt_begin.push_back((int32_t)pts.size());
  }
  int rc = sdv_immature_trace_batch(gpu, (int)hosts.size(), frames.data(), pt_begin.data(), KRKi.data(), Kt.data(), aff.data(), pts.data(), nullptr);
  std::size_t k = 0; for (HostImmatures& h : hosts) for (ImmaturePoint* ph : h.immaturePoints) ph->rec = pts[k++];       // lastTraceStatus etc. back into the graph
  return rc;
}

// FullSystem::activatePointsMT -> optimizeImmaturePoint (FullSystem.cpp:569-723, FullSystemOptPoint.cpp:18-183): all candidates picked for activation, grouped by host
struct ActivationGroup { FrameHessian* host; std::vector<ImmaturePoint*> toOptimize; std::vector<uint8_t> isFromSensor; std::vector<FrameHessian*> targets; std::vector<float> pre14; float calib6[6]; };
int shim_activatePoints(std::vector<ActivationGroup>& groups, std::vector<int32_t>& status, std::vector<float>& idepth, std::vector<int32_t>& res_state, int res_stride) {
  std::vector<int32_t> pt_begin{0}, tgt_begin{0}; std::vector<uint64_t> tf; std::vector<float> pre, cal; std::vector<sdv_immature_pt> pts; std::vector<uint8_t> fs;
  for (ActivationGroup& g : groups) {
    for (ImmaturePoint* ph : g.toOptimize) pts.push_back(ph->rec);
    fs.insert(fs.end(), g.isFromSensor.begin(), g.isFromSensor.end());
    for (FrameHessian* t : g.targets) tf.push_back((uint64_t)t->shell->id);
    pre.insert(pre.end(), g.pre14.begin(), g.pre14.end()); cal.insert(cal.end(), g.calib6, g.calib6 + 6);
    pt_begin.push_back((int32_t)pts.size()); tgt_begin.push_back((int32_t)tf.size());
  }
  status.resize(pts.size()); idepth.resize(pts.size()); res_state.resize(pts.size()*(std::size_t)res_stride);
  return sdv_immature_optimize_batch(gpu, (int)groups.size(), pt_begin.data(), tgt_begin.data(), tf.data(), pre.data(), cal.data(), /*minObs*/1, pts.data(), fs.data(), res_stride,
                                     status.data(), idepth.data(), res_state.data());     // status 1 -> new PointHessian(point) + PointFrameResidual per IN state, -1 -> delete, 0 -> keep immature
}

// ------------------------------------------------------------------------------------------------ §3e keyframe-rate candidate management (SURVEY §8f ranks 3b / 4 / 2)
// PixelSelector::PixelSelector (PixelSelector2.cpp:11-26): the selector's random pattern is generated where the reference generates it and handed to the library once
struct PixelSelector { unsigned char* randomPattern; int currentPotential; };
int shim_selector_ctor(PixelSelector& ps) {
  ps.randomPattern = new unsigned char[(std::size_t)wG[0]*hG[0]]; std::srand(3141592); for (int i = 0; i < wG[0]*hG[0]; i++) ps.randomPattern[i] = std::rand() & 0xFF;   // :14-16
  ps.currentPotential = 3; return sdv_selector_init(gpu, ps.randomPattern, /*slots: one per FullSystem*/1);
}
// void lidarCloudHandler(const sensor_msgs::PointCloud2ConstPtr&)  main.cpp:785-858: the decoded XYZI rows of one sweep in, vCloudPixel + addFeaturePoint out
struct LidarRig { double Rlc[9], tlc[3]; float fx, fy, cx, cy; int left, right, up, down; bool addFeaturePoint; };           // the FullSystem members main.cpp:368-377, :834-854 touches
int shim_lidarCloudHandler(LidarRig& fsys, const float* xyzi, int n, std::vector<double>& vCloudPixel3) {
  static bool once = false; if (!once) { int rc = sdv_lidar_init(gpu, /*N_SCAN*/64, /*Horizon_SCAN*/1800, 0.2f, 0.427f, 24.9f, /*groundScanInd*/50); if (rc) return rc; once = true; }   // main.cpp:103-108
  const int32_t sweep_begin[2] = {0, n}; const float K4[4] = {fsys.fx, fsys.fy, fsys.cx, fsys.cy}; int32_t lrud[4] = {fsys.left, fsys.right, fsys.up, fsys.down}, n_out = 0, add = 0;
  const int cap = 64*1800; vCloudPixel3.resize(3*(std::size_t)cap);
  int rc = sdv_lidar_handler_batch(gpu, 1, sweep_begin, xyzi, fsys.Rlc, fsys.tlc, K4, lrud, cap, vCloudPixel3.data(), &n_out, &add, nullptr);
  fsys.left = lrud[0]; fsys.right = lrud[1]; fsys.up = lrud[2]; fsys.down = lrud[3]; fsys.addFeaturePoint = add != 0; vCloudPixel3.resize(3*(std::size_t)n_out);           // -> fullSystem->qCloudPixel.push(vCloudPixel)
  return rc;
}
// void FullSystem::makeNewTraces(FrameHessian* newFrame, float*)  FullSystem.cpp:1273-1356, whole: selection, Shi-Tomasi typing, occupancy mask, ImmaturePoint construction
int shim_makeNewTraces_whole(FrameHessian* newFrame, const LidarRig& fsys, const std::vector<double>& vCloudPixel3, std::vector<sdv_new_trace>& traces, std::vector<sdv_immature_pt>& recs) {
  const int32_t slot = 0, cloud_begin[2] = {0, (int32_t)(vCloudPixel3.size()/3)}, add = fsys.addFeaturePoint ? 1 : 0; const uint64_t id = (uint64_t)newFrame->shell->id;
  const int lidarArea = (fsys.right - fsys.left)*(fsys.down - fsys.up), imageArea = wG[0]*hG[0];
  const float dl = ((float)lidarArea/(float)imageArea) * setting_desiredImmatureDensity, dd = setting_desiredImmatureDensity;                                                   // :1287-1293
  const int cap = 1 << 14; traces.resize(cap); recs.resize(cap); int32_t n_out = 0, num[2];
  int rc = sdv_make_new_traces_batch(gpu, 1, &slot, &id, cloud_begin, vCloudPixel3.data(), &dl, &dd, &add, cap, traces.data(), recs.data(), &n_out, num);
  traces.resize(n_out); recs.resize(n_out);   // per row: new ImmaturePoint{rec}, my_type, score, type, isFromSensor, idepth_fromSensor (:1307-1325, :1343-1352) -> newFrame->immaturePoints
  return rc;
}
// the selection half of void FullSystem::activatePointsMT()  FullSystem.cpp:600-671 (makeDistanceMap + candidate walk); the survivors go to shim_activatePoints
struct ActivationInputs { std::vector<int32_t> pt_begin, cand_begin; std::vector<float> KRKi9, Kt3, uvid, cKRKi9, cKt3, cand4; float currentMinActDist; };   // per keyframe: K[1] R K[0]^-1, K[1] t (:606-608)
int shim_activateSelect(const ActivationInputs& in, std::vector<int32_t>& decision) {
  const int32_t host_begin[2] = {0, (int32_t)in.pt_begin.size() - 1}, cand_host_begin[2] = {0, (int32_t)in.cand_begin.size() - 1};
  decision.resize(in.cand_begin.back());
  return sdv_activate_select_batch(gpu, 1, host_begin, in.pt_begin.data(), in.KRKi9.data(), in.Kt3.data(), in.uvid.data(), cand_host_begin, in.cand_begin.data(), in.cKRKi9.data(), in.cKt3.data(),
                                   in.cand4.data(), &in.currentMinActDist, decision.data(), nullptr);   // 1 -> toOptimize.push_back(ph), 0 -> skipped, -1 -> delete ph (:653-669)
}

// ------------------------------------------------------------------------------------------------ device-resident immature points (sdv_immature_store_*)
// host->immaturePoints keeps only a count; the records live in the context's store block of the host, keyed by its frame id.
struct StoreHost { FrameHessian* host; int32_t cam; int32_t nImmature; Mat33f KRKi; Vec3f Kt; Vec2f aff; };    // per host: what :532-538 computes
// makeKeyFrame -> makeNewTraces (FullSystem.cpp:1273-1356) + the SKIPPED loop (:1080-1084): the new keyframe's points go straight into its block
int shim_makeNewTraces_store(FrameHessian* newFrame, const LidarRig& fsys, int32_t slot, const std::vector<double>& vCloudPixel3, int32_t& nImmature) {
  const int32_t cloud_begin[2] = {0, (int32_t)(vCloudPixel3.size()/3)}, add = fsys.addFeaturePoint ? 1 : 0; const uint64_t id = (uint64_t)newFrame->shell->id;
  const int lidarArea = (fsys.right - fsys.left)*(fsys.down - fsys.up), imageArea = wG[0]*hG[0];
  const float dl = ((float)lidarArea/(float)imageArea) * setting_desiredImmatureDensity, dd = setting_desiredImmatureDensity; int32_t num[2];
  return sdv_make_new_traces_store_batch(gpu, 1, &slot, &id, cloud_begin, vCloudPixel3.data(), &dl, &dd, &add, 1 << 14, &nImmature, num);
}
// FullSystem::traceNewCoarse (FullSystem.cpp:519-552): every host of the window in one launch, nothing copied; counts only when the caller logs them (:543-548)
int shim_traceNewCoarse_store(FrameHessian* fh, const std::vector<StoreHost>& hosts, std::vector<int32_t>* counts6) {
  std::vector<uint64_t> hid, frames; std::vector<int32_t> cams; std::vector<float> KRKi, Kt, aff;
  for (const StoreHost& h : hosts) {
    hid.push_back((uint64_t)h.host->shell->id); frames.push_back((uint64_t)fh->shell->id); cams.push_back(h.cam);
    KRKi.insert(KRKi.end(), h.KRKi.m, h.KRKi.m + 9); for (int i = 0; i < 3; i++) Kt.push_back((float)h.Kt[i]); aff.push_back(h.aff.v[0]); aff.push_back(h.aff.v[1]);
  }
  if (counts6) counts6->resize(6*hosts.size());
  return sdv_immature_trace_store_batch(gpu, (int)hosts.size(), hid.data(), frames.data(), cams.data(), KRKi.data(), Kt.data(), aff.data(), counts6 ? counts6->data() : nullptr);
}
// FullSystem::marginalizeFrame -> FrameHessian::release (HessianBlocks.cpp:90-105): the keyframe's immature points go with it
int shim_drop_immatures(FrameHessian* fh) { const uint64_t id = (uint64_t)fh->shell->id; return sdv_immature_store_drop(gpu, 1, &id); }
// read-back of a block (debugging, plotting): the records in host->immaturePoints order
int shim_read_immatures(FrameHessian* host, std::vector<sdv_immature_pt>& pts, std::vector<sdv_immature_meta>& meta) {
  const uint64_t id = (uint64_t)host->shell->id; int32_t n = 0; int rc = sdv_immature_store_count(gpu, 1, &id, &n); if (rc) return rc;
  pts.resize(n); meta.resize(n); return sdv_immature_store_get(gpu, id, n, pts.data(), meta.data(), &n);
}
// activatePointsMT (FullSystem.cpp:598-720) on the store for one window; the caller builds PointHessians from the activated records
int shim_activatePoints_store(const std::vector<uint64_t>& window, const std::vector<int32_t>& flagged, const ActivationInputs& in, const std::vector<float>& pre14, const float calib6[6],
                              std::vector<sdv_immature_pt>& act, std::vector<float>& idepth, std::vector<int32_t>& res_state, std::vector<int32_t>& counts) {
  const int32_t host_begin[2] = {0, (int32_t)window.size()}, src_host_begin[2] = {0, (int32_t)in.pt_begin.size() - 1}; const int cap = 4096; int32_t n_act = 0;
  std::vector<int32_t> ah(cap), ai(cap); std::vector<sdv_immature_meta> am(cap); act.resize(cap); idepth.resize(cap); res_state.resize((size_t)cap*SDV_MAX_FRAMES_WINDOW); counts.resize(window.size());
  int rc = sdv_activate_points_store_batch(gpu, 1, host_begin, window.data(), flagged.data(), in.cKRKi9.data(), in.cKt3.data(), src_host_begin, in.pt_begin.data(), in.KRKi9.data(), in.Kt3.data(),
                                           in.uvid.data(), &in.currentMinActDist, pre14.data(), calib6, nullptr, cap, &n_act, ah.data(), ai.data(), act.data(), am.data(), idepth.data(),
                                           res_state.data(), counts.data());
  act.resize(n_act); idepth.resize(n_act); return rc;
}
int shim_set_immatures(FrameHessian* host, const std::vector<sdv_immature_pt>& pts, const std::vector<sdv_immature_meta>& meta) {
  return sdv_immature_store_set(gpu, (uint64_t)host->shell->id, (int)pts.size(), pts.data(), meta.empty() ? nullptr : meta.data());
}

// ------------------------------------------------------------------------------------------------ LiDAR row sets (sdv_lidar_handler_rows_batch, sdv_lidar_rows_*)
// FullSystem::qCloudPixel holds frame handles; the rows, the box FullSystem::left/right/up/down (FullSystem.h:191-194) and addFeaturePoint stay on the device
struct RowsQueue { std::vector<uint64_t> qCloudPixel; int32_t slot; };
// void lidarCloudHandler(const sensor_msgs::PointCloud2ConstPtr&)  main.cpp:785-858: the sweep is deposited under the id its paired image will get; nothing waits
int shim_lidarCloudHandler_rows(RowsQueue& fsys, const LidarRig& rig, uint64_t next_frame_id, const float* xyzi, int n) {
  const int32_t sweep_begin[2] = {0, n}; const float K4[4] = {rig.fx, rig.fy, rig.cx, rig.cy};
  int rc = sdv_lidar_handler_rows_batch(gpu, 1, &fsys.slot, &next_frame_id, sweep_begin, xyzi, rig.Rlc, rig.tlc, K4, /*cap*/64*1800, nullptr);
  if (!rc) fsys.qCloudPixel.push_back(next_frame_id);                                     // -> fullSystem->qCloudPixel.push(vCloudPixel)
  return rc;
}
// void FullSystem::makeNewTraces(FrameHessian* newFrame, float*)  FullSystem.cpp:1273-1356: rows, box and addFeaturePoint of newFrame's set; points into its store block
int shim_makeNewTraces_rows(FrameHessian* newFrame, const RowsQueue& fsys, int32_t& nImmature) {
  const uint64_t id = (uint64_t)newFrame->shell->id; const float dens = setting_desiredImmatureDensity; int32_t num[2];
  return sdv_make_new_traces_rows_store_batch(gpu, 1, &fsys.slot, &id, &dens, 1 << 14, &nImmature, num);
}
// process() (main.cpp:470-508): after addActiveFrame, qCloudPixel.pop() with the image
int shim_process_pop(RowsQueue& fsys) {
  if (fsys.qCloudPixel.empty()) return SDV_OK;
  const uint64_t id = fsys.qCloudPixel.front(); fsys.qCloudPixel.erase(fsys.qCloudPixel.begin()); return sdv_lidar_rows_drop(gpu, 1, &id);
}

// ------------------------------------------------------------------------------------------------ the initializer branch (FullSystem.cpp:842-850, :299-338)
// Frame 0 (coarseInitializer->setFirstFromLidar): nothing runs on the host; the frame's handle keys its row set, where frame 1 finds the rows and the box.
// Frame 1 (trackNewCoarse with allFrameHistory.size() == 2): initializeFromInitializer + setCTRefForFirstFrame in one call, the PointHessians from its records,
// then the 53-hypothesis track of frame 1.
extern float setting_desiredPointDensity;
struct InitBranch { FrameHessian* firstFrame; int32_t slot; };
void shim_setFirstFromLidar(InitBranch& ib, FrameHessian* fh) { ib.firstFrame = fh; }
Vec4 shim_initializer_frame1(FullSystem& fs, InitBranch& ib, FrameHessian* newFrame, int& rc) {
  const uint64_t id0 = (uint64_t)ib.firstFrame->shell->id; int32_t rows = 0;
  rc = sdv_lidar_rows_get(gpu, id0, 0, nullptr, &rows, nullptr, nullptr); if (rc) return Vec4{};
  // the C library's stream here is srand(3141592) and w*h draws by frame 0's PixelSelector (PixelSelector2.cpp:14-16); nothing else draws in between
  const long skip = (long)wG[0]*hG[0];
  srand(3141592); for (long k = 0; k < skip; k++) rand();
  std::vector<int32_t> draws(rows > 0 ? rows : 1); for (int k = 0; k < rows; k++) draws[k] = rand();
  const int32_t draw_begin[2] = {0, rows}; const float dens = setting_desiredPointDensity; const int cap = 1 << 14; int32_t n = 0, n_sel = 0;
  std::vector<sdv_immature_pt> pts(cap); std::vector<sdv_immature_meta> meta(cap); std::vector<float> idepth(cap);
  rc = sdv_init_from_lidar_rows_batch(gpu, 1, &ib.slot, &id0, &dens, draw_begin, draws.data(), cap, &n, &n_sel, pts.data(), meta.data(), idepth.data());
  if (rc) return Vec4{};
  srand(3141592); for (long k = 0; k < skip + n_sel; k++) rand();        // the stream as initializeFromInitializer leaves it (:1203): numPoints[0] draws on
  for (int i = 0; i < n; i++) {                                           // :1205-1231: PointHessian(pt), setIdepthScaled / setIdepthZero(midepth), prior, ACTIVE
    PointHessian* ph = new PointHessian(); ph->u = pts[i].u; ph->v = pts[i].v; ph->idepth = ph->idepth_zero = idepth[i];
    for (int k = 0; k < 8; k++) { ph->color[k] = pts[i].color[k]; ph->weights[k] = pts[i].weights[k]; }
    ph->hasDepthPrior = true; ph->isFromSensor = meta[i].isFromSensor != 0; ph->type = meta[i].type; ph->host = ib.firstFrame; ph->efPoint = nullptr;
    ib.firstFrame->pointHessians.push_back(ph);                           // + ef->insertPoint(ph), as in the reference
  }
  ib.firstFrame->shell->camToWorld = SE3(); ib.firstFrame->shell->aff_g2l = AffLight(0, 0);   // :1235-1256
  // the tracker slot holds setCTRefForFirstFrame's reference and the map slot the first keyframe: frame 1 is tracked with the 53 hypotheses of :299-331
  // (the Reprojector behind fs.cell_order shuffles with the stream as it stands now)
  sdv_track_new_coarse_io io{}; io.slot = ib.slot; io.frame = (uint64_t)newFrame->shell->id; io.poses_valid = 2;
  se3_to7(SE3(), io.sprelast_c2w); se3_to7(SE3(), io.slast_c2w); se3_to7(SE3(), io.lastF_c2w);
  for (int i = 0; i < 5; i++) io.lastCoarseRMSE[i] = fs.lastCoarseRMSE[i];
  rc = sdv_track_new_coarse_batch(gpu, 1, &io, fs.cell_order.data(), (int)(0.8f*setting_desiredImmatureDensity));
  newFrame->shell->camToWorld = se3_from7(io.camToWorld); newFrame->shell->camToTrackingRef = se3_from7(io.camToTrackingRef); newFrame->shell->trackingRef = ib.firstFrame->shell;
  newFrame->shell->aff_g2l = AffLight(io.aff_g2l[0], io.aff_g2l[1]);
  for (int i = 0; i < 5; i++) fs.lastCoarseRMSE[i] = io.lastCoarseRMSE[i];
  return Vec4{{io.lastCoarseRMSE[0], io.flow[0], io.flow[1], io.flow[2]}};
}

// ------------------------------------------------------------------------------------------------ batched makeKeyFrame (INTEGRATION.md §4)
// one context serving many FullSystems: each sequence that made a keyframe walks its own graph, then ONE call installs every tracker reference
// (setCoarseTrackingRef of coarseTracker_forNewKF, slot ref_slot[i]) and ONE call every resident map (slot map_slot[i])
int shim_makeKeyFrame_batch(const std::vector<FullSystem*>& fss, const std::vector<int32_t>& ref_slot, const std::vector<int32_t>& map_slot, std::vector<int32_t>& npts) {
  const int n = (int)fss.size();
  std::vector<float> pts; std::vector<int32_t> rh, pb{0}, hb{0}, mb{0}; std::vector<uint64_t> ref_ids, ids; std::vector<double> ref_ab, c2w, ab; std::vector<sdv_map_pt> mp;
  for (FullSystem* fs : fss) {
    CoarseTracker::splat_rows(fs->frameHessians, pts, rh); pb.push_back((int32_t)rh.size());
    FrameHessian* ref = fs->frameHessians.back(); ref_ids.push_back((uint64_t)ref->shell->id); ref_ab.push_back(ref->aff_g2l().a); ref_ab.push_back(ref->aff_g2l().b);
    fs->map_rows(ids, c2w, ab, mp); hb.push_back((int32_t)ids.size()); mb.push_back((int32_t)mp.size());
  }
  npts.assign((size_t)n*SDV_PYR_LEVELS, 0);
  int rc = sdv_tracker_set_ref_batch(gpu, n, ref_slot.data(), ref_ids.data(), pb.data(), pts.data(), rh.data(), ref_ab.data(), npts.data());
  if (rc == SDV_OK) rc = sdv_map_set_batch(gpu, n, map_slot.data(), hb.data(), ids.data(), c2w.data(), ab.data(), mb.data(), mp.data());
  for (FullSystem* fs : fss) { FrameHessian* ref = fs->frameHessians.back(); CoarseTracker* t = fs->coarseTracker; t->lastRef = ref; t->refFrameID = ref->shell->id; t->lastRef_aff_g2l = ref->aff_g2l(); t->firstCoarseRMSE = -1; }
  return rc;
}

// ------------------------------------------------------------------------------------------------ batched back-end makeKeyFrame (INTEGRATION.md §4)
// the back-end part of makeKeyFrame for every sequence that made a keyframe: each flattens its own window (window[i] of the context), then one call per step
// serves them all: install, optimize, flagPointsForRemoval, marginalizePointsF, marginalizeFrame (frames flagged for marginalisation, in the reference's
// restart order) with the priors back into ef->HM / ef->bM
int shim_backend_keyframe_batch(const std::vector<FullSystem*>& fss, const std::vector<int32_t>& windows, const std::vector<std::vector<int32_t>>& selected,
                                std::vector<float>& rmse) {
  const int n = (int)fss.size(); FullSystem::WindowRows w;
  for (FullSystem* fs : fss) fs->append(w);
  int rc = sdv_ba_set_window_batch(gpu, n, windows.data(), w.f_begin.data(), w.ids.data(), w.T_eval.data(), w.state.data(), w.state_zero.data(), w.exposure.data(),
                                   w.frameID.data(), w.energyTH.data(), w.calib.data(), w.calib_zero.data(), w.HM.data(), w.bM.data());
  if (rc == SDV_OK) rc = sdv_ba_set_points_batch(gpu, n, windows.data(), w.p_begin.data(), w.r_begin.data(), w.uv.data(), w.idepth.data(), w.idepth_zero.data(), w.color.data(),
                                                 w.weights.data(), w.host.data(), w.hasPrior.data(), w.fromSensor.data(), w.res_begin.data(), w.r_point.data(), w.r_host.data(),
                                                 w.r_target.data(), w.r_hasM.data(), w.r_matcher.data(), w.r_isNew.data());
  rmse.assign(n, 0.f); std::vector<int32_t> its(n), acc(n);
  if (rc == SDV_OK) rc = sdv_ba_optimize_batch(gpu, n, windows.data(), 6, rmse.data(), its.data(), acc.data());
  std::vector<int32_t> sel, status, kb{0}, idx;
  for (const std::vector<int32_t>& s : selected) sel.insert(sel.end(), s.begin(), s.end());
  status.resize(sel.size());
  if (rc == SDV_OK) rc = sdv_ba_flag_points_batch(gpu, n, windows.data(), sel.data(), status.data());
  if (rc == SDV_OK) rc = sdv_ba_marginalize_points_batch(gpu, n, windows.data(), nullptr);
  for (FullSystem* fs : fss) {                                                   // for (i ...) if (flaggedForMarginalization) { marginalizeFrame; i = 0; }
    int removed = 0;
    for (FrameHessian* fh : fs->frameHessians) if (fh->flaggedForMarginalization) idx.push_back(fh->idx - removed++);
    kb.push_back((int32_t)idx.size());
  }
  std::vector<double> HM, bM;
  for (int i = 0; i < n; i++) { const int nF = (int)fss[i]->frameHessians.size() - (kb[i+1] - kb[i]), N = 4 + 6*nF; HM.resize(HM.size() + (size_t)N*N); bM.resize(bM.size() + N); }
  if (rc == SDV_OK) rc = sdv_ba_marginalize_frames_batch(gpu, n, windows.data(), kb.data(), idx.data(), HM.data(), bM.data());
  size_t h = 0, b = 0;
  for (int i = 0; i < n && rc == SDV_OK; i++) { FullSystem* fs = fss[i]; const int N = 4 + 6*((int)fs->frameHessians.size() - (kb[i+1] - kb[i]));
    fs->HM.assign(HM.begin() + h, HM.begin() + h + (size_t)N*N); fs->bM.assign(bM.begin() + b, bM.begin() + b + N); h += (size_t)N*N; b += N; }
  return rc;
}

// referenced so that -Wunused does not hide a missing call path
int shim_check_anchor(FullSystem& fs, FrameHessian* fh, CalibHessian& hc, const Undistort* u, const uint8_t* raw) {
  std::vector<int32_t> sel, st; Vec5 mr{}; SE3 T; AffLight a;
  int rc = shim_create(hc) | shim_set_undistort(u, nullptr, nullptr) | shim_ingest_raw(fh->shell, raw, 1.0f) | shim_makeK(fs.coarseTracker->slot, &hc);
  { const uint64_t id = (uint64_t)fh->shell->id; const int32_t cam = 1; const float ex = 1.0f; rc |= shim_set_undistort_cam(cam, u) | shim_ingest_raw_cams(1, &id, &raw, &cam, &ex); }
  { const uint64_t id = (uint64_t)fh->shell->id; const int32_t cam = 2, slot = 3; const float ex = 1.0f; const void* dev = nullptr; const sdv_calib K{hc.fxl(), hc.fyl(), hc.cxl(), hc.cyl()};
    rc |= shim_kitti_camera(cam, u, 1200, 360, 1, &slot, &K) | shim_ingest_cams(1, &id, &raw, &dev, &cam, &ex) | shim_makeK_cam(slot, cam, &K); }
  fs.coarseTracker->setCoarseTrackingRef(fs.frameHessians); fs.coarseTracker->trackNewestCoarse(fh, T, a, 3, mr, nullptr);
  std::vector<ImmaturePoint*> imm; std::vector<HostImmatures> hi; rc |= shim_makeNewTraces(fh, sel, imm) | shim_traceNewCoarse(fh, hi);
  std::vector<ActivationGroup> ag; std::vector<float> idp; rc |= shim_activatePoints(ag, st, idp, sel, 7);
  PixelSelector ps; LidarRig rig{}; std::vector<double> px; std::vector<sdv_new_trace> tr; std::vector<sdv_immature_pt> rc2; ActivationInputs ai; ai.pt_begin = {0}; ai.cand_begin = {0}; ai.currentMinActDist = 2;
  rc |= shim_selector_ctor(ps) | shim_lidarCloudHandler(rig, nullptr, 0, px) | shim_makeNewTraces_whole(fh, rig, px, tr, rc2) | shim_activateSelect(ai, st);
  { KittiKeyframe k{}; k.slot = 1; k.cam = 1; rc |= shim_kitti_keyframe(k, 1500.f, tr, rc2, st); }
  { std::vector<StoreHost> sh; std::vector<sdv_immature_meta> me; int32_t ni = 0;
    rc |= shim_makeNewTraces_store(fh, rig, 0, px, ni) | shim_traceNewCoarse_store(fh, sh, &st) | shim_read_immatures(fh, rc2, me) | shim_set_immatures(fh, rc2, me) | shim_drop_immatures(fh);
    std::vector<float> idp2; std::vector<int32_t> rs2, cn2; const float cal6[6] = {1, 1, 0, 0, 1, 1};
    rc |= shim_activatePoints_store({(uint64_t)fh->shell->id}, {0}, ai, {}, cal6, rc2, idp2, rs2, cn2); }
  { RowsQueue q{{}, 0}; int32_t ni = 0; rc |= shim_lidarCloudHandler_rows(q, rig, (uint64_t)fh->shell->id, nullptr, 0) | shim_makeNewTraces_rows(fh, q, ni) | shim_process_pop(q); }
  { InitBranch ib{nullptr, 0}; int rci = 0; shim_setFirstFromLidar(ib, fh); shim_initializer_frame1(fs, ib, fh, rci); rc |= rci; }
  { std::vector<FullSystem*> fss{&fs}; std::vector<int32_t> np; rc |= shim_makeKeyFrame_batch(fss, {0}, {0}, np); }
  { std::vector<FullSystem*> fss{&fs}; std::vector<float> rm; rc |= shim_backend_keyframe_batch(fss, {0}, {sel}, rm); }
  fs.optimize(6); fs.set_map(0); fs.handover(sel, st); fs.trackNewCoarse(fh); fs.refine_only(fh); shim_frame_destructor(fh);
  return rc;
}
