// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).  Pinned on oracle/_ref (the reference's own CoarseInitializer.cpp / FullSystem.cpp /
// CoarseTracker.cpp, compiled unmodified): tests/test_ref_pin_init.py.
//
// orc_init.cpp — restatement of the start of a sequence on the LiDAR path (FullSystem::addActiveFrame, frames 0 and 1: FullSystem.cpp:842-850, :299-338):
//   CoarseInitializer::setFirstFromLidar, level 0 only   FullSystem/CoarseInitializer.cpp:766-888   a fresh PixelSelector, makeMapsFromLidar(.., 0.03*lidarArea, 1, false, 2, ..),
//                                                                                                   the Pnt list of the selected rows with depth > 0
//   FullSystem::initializeFromInitializer, point loop    FullSystem/FullSystem.cpp:1176-1225         one rand() per Pnt, keep test, ImmaturePoint at (int)(u+0.5f), PointHessian
//   CoarseTracker::makeCoarseDepthForFirstFrame          FullSystem/CoarseTracker.cpp:108-256         = setCoarseTrackingRef with round_half 1 and HdiF 0
// It is built from the oracle's own pieces (orc_select.cpp, orc_trace.cpp, orc_tracker.cpp) through their C entries.  The levels >= 1 of setFirstFromLidar, makeNN and
// the sumGrad2 loop feed nothing that is read later (CoarseInitializer::trackFrame has no caller) and are not restated.
// Reference behaviour restated: EFPoint::HdiF is uninitialised when setCTRefForFirstFrame reads it (0 here, a zeroed block); a point whose 8-pattern reads outside the
// image plane is not kept (the reference reads past its buffer there).
#include <cmath>
#include <cstdint>
#include <vector>

extern "C" {
void* orc_selector_create(int w, int h, const uint8_t* randomPattern);
void  orc_selector_destroy(void* s);
int   orc_selector_make_maps(void* s, void* frame, float* map_out, float density, int recursionsLeft, float thFactor, const double* cloud3, int n);
void  orc_immature_init(void* host_frame, int n, const int32_t* uv, void* pts_out);
void  orc_tracker_set_ref(void* t, void* ref_frame, const float* pts, const int* round_half, int n, double ref_a, double ref_b);
}

namespace {
struct ImmPt { float u, v, idepth_min, idepth_max, color[8], weights[8], gradH[4], energyTH, quality, lastTraceUV[2], lastTracePixelInterval; int32_t lastTraceStatus; };   // orc_trace.cpp
}

extern "C" {
// One sequence's bootstrap on `frame` (an orc Frame of w x h; rp: the first w*h bytes of the PixelSelector random pattern).  cloud3: n rows {Ku, Kv, depth}; lrud: the
// FullSystem box; draws: at least n rand() values.  Out: *n_sel = numPoints[0]; pnt5[5k..] = {u, v, my_type, mdepth, isFromSensor} of Pnt k and keep[k] (numPoints[0]
// entries, n is enough); for the kept points, in order: the ImmaturePoint record pts[i], meta4[4i..] = {my_type, type 0, isFromSensor 1, idepth_fromSensor} and idepth[i] =
// the PointHessian's idepth / idepth_zero.  tracker (may be NULL): an orc CoarseTracker that gets setCTRefForFirstFrame.  Returns the number kept.
int orc_init_from_lidar(void* frame, int w, int h, const uint8_t* rp, const double* cloud3, int n, const int32_t lrud[4], float desiredPointDensity, const int32_t* draws,
                        void* tracker, int32_t* n_sel, float* pnt5, int32_t* keep, void* pts, float* meta4, float* idepth) {
  const int lidarArea = (lrud[1] - lrud[0]) * (lrud[3] - lrud[2]);
  std::vector<float> statusMap(n > 0 ? n : 1, 0.f);
  void* sel = orc_selector_create(w, h, rp);                                              // PixelSelector sel(w[0], h[0]); currentPotential = 3
  const float densities0 = 0.03f;
  const double no_rows[3] = {0, 0, 0};                                                     // a null cloud would select over all pixels (makeMaps)
  orc_selector_make_maps(sel, frame, statusMap.data(), densities0*lidarArea, 1, 2, cloud3 ? cloud3 : no_rows, n);
  orc_selector_destroy(sel);
  int nl = 0;
  for (int i = 0; i < n; i++) {
    if (statusMap[i] == 0) continue;
    const float mdepth = (float)cloud3[3*i+2];
    if (!(mdepth > 0)) continue;                                                          // isFromSensor = false; continue (before nl++)
    float* P = pnt5 + 5*(size_t)nl; P[0] = (float)cloud3[3*i]; P[1] = (float)cloud3[3*i+1]; P[2] = statusMap[i]; P[3] = mdepth; P[4] = 1.f;
    nl++;
  }
  *n_sel = nl;
  const float keepPercentage = desiredPointDensity / nl;
  ImmPt* out = (ImmPt*)pts; std::vector<float> splat; std::vector<int> rh; int m = 0;
  for (int k = 0; k < nl; k++) {
    keep[k] = 0;
    if (draws[k]/(float)2147483647 > keepPercentage) continue;                            // rand()/(float)RAND_MAX, glibc
    const float* P = pnt5 + 5*(size_t)k;
    const int u = (int)(P[0] + 0.5f), v = (int)(P[1] + 0.5f);                              // ImmaturePoint(int u_, int v_, ...)
    if (u < 0 || u >= w || v < 0 || v >= h || u + (v-2)*w < 0 || u + 1 + (v+3)*w >= w*h) continue;
    ImmPt p; const int32_t uv[2] = {u, v}; orc_immature_init(frame, 1, uv, &p);
    const float midepth = 1 / P[3];
    p.idepth_min = midepth; p.idepth_max = midepth;
    if (!std::isfinite(p.energyTH)) continue;
    keep[k] = 1; out[m] = p;
    meta4[4*m] = P[2]; ((int32_t*)meta4)[4*m+1] = 0; ((int32_t*)meta4)[4*m+2] = 1; meta4[4*m+3] = midepth;
    idepth[m] = midepth;
    splat.insert(splat.end(), {(float)u, (float)v, midepth, 0.f}); rh.push_back(1);         // makeCoarseDepthForFirstFrame: int(ph->u + 0.5f), ph->idepth, HdiF 0
    m++;
  }
  if (tracker) orc_tracker_set_ref(tracker, frame, splat.data(), rh.data(), m, 0.0, 0.0);
  return m;
}
}  // extern "C"
