// ref_init_shim.cpp — C entry points over the UNMODIFIED reference sources for the start of a sequence.  TEST INFRASTRUCTURE ONLY.
//
// Built by oracle/init.mk into oracle/_ref/libsdvref_init.so, linked against oracle/_ref/libsdvref.so (the reference's own translation units, oracle/Makefile
// `ref`), with the same flags and stand-in headers.  It calls the reference's own members one at a time on the objects ref_shim.cpp creates: a RefSys
// (ref_sys_create) and RefFrames (ref_frame_create), whose FIRST members are the FullSystem* and the FrameHessian* (ref_shim.cpp) — the only layout this file
// relies on.  Only needed where the reference is built: what it returns is stored in tests/golden/ref_pin_init.npz / seq_init_ref.npz.
#include <vector>
#include <queue>
#include <deque>
#include <mutex>
#include <thread>
#include <condition_variable>
#include <functional>
#include <memory>
#include <cstdlib>
#include "Eigen/Core"
#include "sophus/se3.hpp"
#include "boost/thread.hpp"
#define private public                                     // the members read back (points, numPoints, efPoint->HdiF) are not all public
#define protected public
#include "FullSystem/FullSystem.h"
#include "FullSystem/CoarseTracker.h"
#include "FullSystem/CoarseInitializer.h"
#include "FullSystem/ImmaturePoint.h"
#include "OptimizationBackend/EnergyFunctionalStructs.h"
#include "util/settings.h"
#include "util/FrameShell.h"
#undef private
#undef protected

using namespace sdv_loam;

namespace {
struct SysView { FullSystem* fs; };                       // ref_shim.cpp's RefSys starts with its FullSystem*
struct FrameView { FrameHessian* fh; };                   // ref_shim.cpp's RefFrame starts with its FrameHessian*
}

extern "C" {
// CoarseInitializer::setFirstFromLidar (CoarseInitializer.cpp:766-888) on `frame`, with qCloudPixel.front() = the n rows and the FullSystem box lrud; reads back
// numPoints[0] and points[0][k] as {u, v, my_type, mdepth, isFromSensor}.
int ref_init_first(void* sys, void* frame, const double* cloud_px, int n, const int* lrud, float* pnt5) {
  FullSystem* fs = ((SysView*)sys)->fs;
  std::vector<Eigen::Vector3d, Eigen::aligned_allocator<Eigen::Vector3d> > v(n); for (int i = 0; i < n; i++) v[i] = Eigen::Vector3d(cloud_px[3*i], cloud_px[3*i+1], cloud_px[3*i+2]);
  while (!fs->qCloudPixel.empty()) fs->qCloudPixel.pop();
  fs->qCloudPixel.push(v); fs->left = lrud[0]; fs->right = lrud[1]; fs->up = lrud[2]; fs->down = lrud[3];
  fs->coarseInitializer->setFirstFromLidar(&fs->Hcalib, ((FrameView*)frame)->fh, fs);
  fs->qCloudPixel.pop();
  CoarseInitializer* ci = fs->coarseInitializer; const int m = ci->numPoints[0];
  for (int k = 0; k < m; k++) { const Pnt& q = ci->points[0][k]; float* o = pnt5 + 5*(size_t)k; o[0] = q.u; o[1] = q.v; o[2] = q.my_type; o[3] = q.mdepth; o[4] = q.isFromSensor ? 1.f : 0.f; }
  return m;
}
// setting_desiredPointDensity = density; srand(seed); FullSystem::initializeFromInitializer(new_frame) (FullSystem.cpp:1176-1259); then efPoint->HdiF = 0 on the new
// points (the value of a fresh zeroed block: nothing has written it before setCTRefForFirstFrame reads it).  Reads back every PointHessian of the first frame, 26
// floats each: {u, v, idepth, idepth_zero, idepth_scaled, my_type, energyTH, hasDepthPrior, isFromSensor, status, color[8], weights[8]}.
int ref_init_from_initializer(void* sys, void* new_frame, unsigned seed, float density, float* ph26, int cap) {
  FullSystem* fs = ((SysView*)sys)->fs;
  const float keep_density = setting_desiredPointDensity; setting_desiredPointDensity = density;
  srand(seed);
  fs->initializeFromInitializer(((FrameView*)new_frame)->fh);
  setting_desiredPointDensity = keep_density;
  FrameHessian* first = fs->coarseInitializer->firstFrame; int m = (int)first->pointHessians.size();
  for (int i = 0; i < m && i < cap; i++) { PointHessian* ph = first->pointHessians[i]; ph->efPoint->HdiF = 0; float* o = ph26 + 26*(size_t)i;
    o[0] = ph->u; o[1] = ph->v; o[2] = ph->idepth; o[3] = ph->idepth_zero; o[4] = ph->idepth_scaled; o[5] = ph->my_type; o[6] = ph->energyTH;
    o[7] = ph->hasDepthPrior ? 1.f : 0.f; o[8] = ph->isFromSensor ? 1.f : 0.f; o[9] = (float)ph->status;
    for (int k = 0; k < 8; k++) { o[10+k] = ph->color[k]; o[18+k] = ph->weights[k]; } }
  return m;
}
// CoarseInitializer::numPoints[0] of the running system (its last setFirstFromLidar)
int ref_init_num_points(void* sys) { return ((SysView*)sys)->fs->coarseInitializer->numPoints[0]; }
// CoarseTracker::setCTRefForFirstFrame(frameHessians) (CoarseTracker.cpp:636-647) on a tracker of ref_tracker_create; its clouds are read with ref_tracker_get_cloud
void ref_init_tracker_set_first(void* sys, void* tracker) { ((CoarseTracker*)tracker)->setCTRefForFirstFrame(((SysView*)sys)->fs->frameHessians); }
}  // extern "C"
