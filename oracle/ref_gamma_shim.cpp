// ref_gamma_shim.cpp — C entry points over the UNMODIFIED reference sources for a photometrically calibrated camera.  TEST INFRASTRUCTURE ONLY.
//
// Built by oracle/gamma.mk into oracle/_ref/libsdvref_gamma.so, linked against oracle/_ref/libsdvref.so (oracle/Makefile `ref`), with the same flags and
// stand-in headers.  Like ref_init_shim.cpp it works on the objects ref_shim.cpp creates — a RefSys (ref_sys_create) and RefFrames (ref_frame_create) —
// relying only on their FIRST members, the FullSystem* and the FrameHessian*.  What it returns is stored in tests/golden/ref_pin_gamma.npz.
#include <vector>
#include <cstring>
#include "Eigen/Core"
#include "sophus/se3.hpp"
#include "boost/thread.hpp"
#include "FullSystem/FullSystem.h"
#include "FullSystem/HessianBlocks.h"
#include "util/globalCalib.h"

using namespace sdv_loam;

namespace {
struct SysView { FullSystem* fs; };                       // ref_shim.cpp's RefSys starts with its FullSystem*
struct FrameView { FrameHessian* fh; };                   // ref_shim.cpp's RefFrame starts with its FrameHessian*
}

extern "C" {
// FullSystem::setGammaFunction(G) (FullSystem.cpp:225-249) on the system's CalibHessian (G == NULL: the call returns at once) -> Hcalib.B
void ref_gamma_set(void* sys, const float* G, float* B_out) {
  FullSystem* fs = ((SysView*)sys)->fs;
  fs->setGammaFunction(const_cast<float*>(G));
  memcpy(B_out, fs->Hcalib.B, sizeof(float)*256);
}
// FrameHessian::makeImages(color, &fs->Hcalib) (HessianBlocks.cpp:107-167) again on a frame of ref_frame_create, now with the system's CalibHessian (its B weighs
// absSquaredGrad); the rows makeImages leaves unwritten are zeroed as ref_frame_create zeroes them
void ref_gamma_make_images(void* sys, void* frame, const float* color) {
  FullSystem* fs = ((SysView*)sys)->fs; FrameHessian* fh = ((FrameView*)frame)->fh;
  for (int i = 0; i < pyrLevelsUsed; i++) { delete[] fh->dIp[i]; delete[] fh->absSquaredGrad[i]; }
  std::vector<float> c(color, color + (size_t)wG[0]*hG[0]);
  fh->makeImages(c.data(), &fs->Hcalib);
  for (int l = 0; l < pyrLevelsUsed; l++) { int wl = wG[l], hl = hG[l]; float* a = fh->absSquaredGrad[l]; Eigen::Vector3f* d = fh->dIp[l];
    for (int x = 0; x < wl; x++) { a[x] = 0; a[(size_t)wl*(hl-1)+x] = 0; d[x][1] = d[x][2] = 0; d[(size_t)wl*(hl-1)+x][1] = d[(size_t)wl*(hl-1)+x][2] = 0; } }
}
}
