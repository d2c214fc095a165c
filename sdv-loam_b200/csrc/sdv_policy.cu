// sdv_policy.cu — FullSystem::trackNewCoarse as a batched host policy over the device kernels (SURVEY.md §8 row a4).
//
// Restates /root/reference/src/FullSystem/FullSystem.cpp:283-500: the branch for a running system (:334-395: allFrameHistory.size() > 2) and the hypothesis set of the
// second frame (:299-331: identity + 2 x 26 small rotations; poses_valid == 2 — its initializeFromInitializer / setCTRefForFirstFrame bookkeeping stays with the caller):
//   motion hypotheses lastF_2_fh_tries (constant / double / half / zero motion, zero from KF, 26 small rotations — the rotDelta loop of :357
//   increments by 1.0, so it runs once), the re-track loop with the per-level "at least as good as the best try" abort vector (:410-462),
//   the fallback when every try fails (:464-470), pose composition (:474-479), reprojectMap + structPoseEstimation (:481-488).
// Batched form: try i is ONE sdv_tracker_track_batch launch over the sequences that have not met the immediate-accept rule (:460) yet —
// with healthy tracking every sequence stops after try 0, stragglers continue in smaller launches.  The refinement of all sequences is one
// sdv_tracker_refine_batch call.  Host code only; all numerics happen in the kernels the two entries launch.
#include <vector>
#include <math.h>
#include <string.h>
#include "sdv_ctx.cuh"

using namespace sdv;

static SE3d quatT(double w, double x, double y, double z) { SE3d s; s.q = qnormalize(Quat{w, x, y, z}); s.t[0] = s.t[1] = s.t[2] = 0; return s; }   // SE3(Quaterniond, Vec3) normalises

// Hypothesis i of FullSystem.cpp:346-388, generated on demand (healthy tracking only ever needs i = 0; building all 31 for every sequence of a batch
// would cost more host time than the launch they feed).
struct TryGen { bool valid; bool second_frame; SE3d inv, lastF_2_slast, cm, fh_2_slast; };
static TryGen try_gen(const sdv_track_new_coarse_io& io) {
  TryGen g; g.valid = io.poses_valid != 0; g.second_frame = io.poses_valid == 2; if (!g.valid || g.second_frame) return g;   // :390-394 -> {SE3()}; :299-331 needs no history
  const SE3d sprelast = se3_from7(io.sprelast_c2w), slast = se3_from7(io.slast_c2w), lastF = se3_from7(io.lastF_c2w);
  g.fh_2_slast = se3_mul(se3_inv(sprelast), slast);                                      // slast_2_sprelast, assumed equal to fh_2_slast (:343,347)
  g.lastF_2_slast = se3_mul(se3_inv(slast), lastF);                                      // :344
  g.inv = se3_inv(g.fh_2_slast); g.cm = se3_mul(g.inv, g.lastF_2_slast);
  return g;
}
static const int kRotPattern[26][3] = {{1,0,0},{0,1,0},{0,0,1},{-1,0,0},{0,-1,0},{0,0,-1},{1,1,0},{0,1,1},{1,0,1},{-1,1,0},{0,-1,1},{-1,0,1},{1,-1,0},{0,1,-1},{1,0,-1},
                                       {-1,-1,0},{0,-1,-1},{-1,0,-1},{-1,-1,-1},{-1,-1,1},{-1,1,-1},{-1,1,1},{1,-1,-1},{1,-1,1},{1,1,-1},{1,1,1}};
static int n_tries(const TryGen& g) { return !g.valid ? 1 : (g.second_frame ? 53 : 31); }
static SE3d make_try(const TryGen& g, int i) {
  if (!g.valid) return se3_identity();
  if (g.second_frame) {                                                                  // allFrameHistory.size() == 2 (:299-331): identity, then 26 pure rotations for
    if (i == 0) return se3_identity();                                                   // rotDelta = 0.02f and 0.04f (float loop `rotDelta = rotDelta + 0.02` while < 0.05)
    const float rd = (i - 1 < 26) ? 0.02f : (0.02f + 0.02f); const double r = (double)rd; const int k = (i - 1) % 26;
    return quatT(1, kRotPattern[k][0]*r, kRotPattern[k][1]*r, kRotPattern[k][2]*r);
  }
  switch (i) {
    case 0: return g.cm;                                                                 // constant motion
    case 1: return se3_mul(se3_mul(g.inv, g.inv), g.lastF_2_slast);                      // double motion (left-associated like the expression :351)
    case 2: { double lg[6]; se3_log(g.fh_2_slast, lg); for (int k=0;k<6;k++) lg[k] = lg[k]*0.5; return se3_mul(se3_inv(se3_exp(lg)), g.lastF_2_slast); }   // half motion
    case 3: return g.lastF_2_slast;                                                      // zero motion
    case 4: return se3_identity();                                                       // zero motion from KF
    default: break;
  }
  const double r = (double)0.02f;                                                        // float rotDelta promoted to double in the Quaterniond ctor; the loop of :357 runs once
  const int k = i - 5;
  return se3_mul(g.cm, quatT(1, kRotPattern[k][0]*r, kRotPattern[k][1]*r, kRotPattern[k][2]*r));                       // (fh_2_slast^-1 * lastF_2_slast) * dR, left-associated
}

// Host-only helper (no device work): hypothesis i of the re-track loop for one job, so the generation can be checked without a GPU.
extern "C" int sdv_track_hypothesis(const sdv_track_new_coarse_io* io, int i, double T7_out[7], int* n_tries_out) {
  if (!io || !T7_out) return SDV_ERR_ARG;
  const TryGen g = try_gen(*io); const int n = n_tries(g);
  if (n_tries_out) *n_tries_out = n;
  if (i < 0 || i >= n) return SDV_ERR_ARG;
  se3_to7(make_try(g, i), T7_out); return SDV_OK;
}

extern "C" int sdv_track_new_coarse_batch(sdv_ctx* c, int n, sdv_track_new_coarse_io* io, const int32_t* cell_order, int max_matches) {
  if (!c || n <= 0 || !io) return SDV_ERR_ARG;
  const float setting_reTrackThreshold = 1.5f;                                           // settings.cpp:130
  struct St { TryGen gen; int ntries; SE3d try0; double achieved[5]; bool haveOneGood, done; SE3d lastF_2_fh; double aff[2]; double flow[3]; int tryIterations; };
  std::vector<St> st(n);
  size_t maxTries = 0;
  for (int k=0;k<n;k++) { St& s = st[k]; s.gen = try_gen(io[k]); s.ntries = n_tries(s.gen); s.try0 = make_try(s.gen, 0); maxTries = std::max(maxTries, (size_t)s.ntries);
    for (int i=0;i<5;i++) s.achieved[i] = nan(""); s.haveOneGood = false; s.done = false; s.lastF_2_fh = se3_identity(); s.aff[0] = s.aff[1] = 0; s.flow[0] = s.flow[1] = s.flow[2] = 100; s.tryIterations = 0; }
  std::vector<int> act; std::vector<int32_t> slots, good; std::vector<uint64_t> frames; std::vector<double> T, ab, minRes, lastRes, flow;
  for (size_t i = 0; i < maxTries; i++) {
    act.clear(); for (int k=0;k<n;k++) if (!st[k].done && (int)i < st[k].ntries) act.push_back(k);
    if (act.empty()) break;
    const int m = (int)act.size();
    slots.resize(m); frames.resize(m); good.resize(m); T.resize(7*m); ab.resize(2*m); minRes.resize(5*m); lastRes.resize(5*m); flow.resize(3*m);
    for (int a=0;a<m;a++) { const int k = act[a]; slots[a] = io[k].slot; frames[a] = io[k].frame; se3_to7(i == 0 ? st[k].try0 : make_try(st[k].gen, (int)i), &T[7*a]);
      ab[2*a] = io[k].aff_last[0]; ab[2*a+1] = io[k].aff_last[1]; for (int l=0;l<5;l++) minRes[5*a+l] = st[k].achieved[l]; }
    // every sequence starts at its own slot camera's pyrLevelsUsed-1 (:421, :429)
    int rc = sdv_tracker_track_batch_levels(c, m, slots.data(), frames.data(), T.data(), ab.data(), nullptr, minRes.data(), lastRes.data(), flow.data(), good.data(), nullptr);
    if (rc) return rc;
    for (int a=0;a<m;a++) { const int k = act[a]; St& s = st[k]; s.tryIterations++;
      const double* lr = &lastRes[5*a];
      if (good[a] && isfinite((float)lr[0]) && !(lr[0] >= s.achieved[0])) {             // :444-450 "do we have a new winner?"
        for (int l=0;l<3;l++) s.flow[l] = flow[3*a+l]; s.aff[0] = ab[2*a]; s.aff[1] = ab[2*a+1]; s.lastF_2_fh = se3_from7(&T[7*a]); s.haveOneGood = true; }
      if (s.haveOneGood) for (int l=0;l<5;l++) if (!isfinite((float)s.achieved[l]) || s.achieved[l] > lr[l]) s.achieved[l] = lr[l];   // :453-459
      if (s.haveOneGood && s.achieved[0] < io[k].lastCoarseRMSE[0]*setting_reTrackThreshold) s.done = true;                           // :461-462
    }
  }
  std::vector<double> c2w(7*n), cab(2*n);
  slots.resize(n); frames.resize(n);
  for (int k=0;k<n;k++) { St& s = st[k]; sdv_track_new_coarse_io& o = io[k];
    if (!s.haveOneGood) { s.flow[0] = s.flow[1] = s.flow[2] = 0; s.aff[0] = o.aff_last[0]; s.aff[1] = o.aff_last[1]; s.lastF_2_fh = s.try0; }   // :464-470
    for (int l=0;l<5;l++) o.lastCoarseRMSE[l] = s.achieved[l];                           // :472
    const SE3d camToTrackingRef = se3_inv(s.lastF_2_fh); const SE3d camToWorld = se3_mul(se3_from7(o.lastF_c2w), camToTrackingRef);   // :475-479
    se3_to7(camToWorld, &c2w[7*k]); cab[2*k] = s.aff[0]; cab[2*k+1] = s.aff[1]; slots[k] = o.slot; frames[k] = o.frame;
    o.aff_g2l[0] = s.aff[0]; o.aff_g2l[1] = s.aff[1]; for (int l=0;l<3;l++) o.flow[l] = s.flow[l]; o.have_one_good = s.haveOneGood ? 1 : 0; o.tries = s.tryIterations; }
  std::vector<int32_t> nm(n), its(n), acc(n); std::vector<float> res(n);
  int rc = sdv_tracker_refine_batch(c, n, slots.data(), frames.data(), c2w.data(), cab.data(), cell_order, max_matches, nm.data(), res.data(), its.data(), acc.data());   // :481-488
  if (rc) return rc;
  for (int k=0;k<n;k++) { sdv_track_new_coarse_io& o = io[k];
    for (int i=0;i<7;i++) o.camToWorld[i] = c2w[7*k+i];
    const SE3d rel = se3_mul(se3_inv(se3_from7(o.lastF_c2w)), se3_from7(o.camToWorld)); se3_to7(rel, o.camToTrackingRef);              // :490-491
    o.n_matches = nm[k]; o.refine_res = res[k]; o.refine_iterations = its[k]; o.refine_accepts = acc[k]; }
  return SDV_OK;
}
