// ORACLE — TEST INFRASTRUCTURE ONLY (see orc_math.hpp header).  Pinned on oracle/_ref (the reference's own FullSystem::setGammaFunction and
// FrameHessian::makeImages with that CalibHessian, oracle/ref_gamma_shim.cpp): tests/test_ref_pin_gamma.py.
//
// orc_gamma.cpp — a frame of a photometrically calibrated camera.  FrameHessian::makeImages (HessianBlocks.cpp:107-167) writes absSquaredGrad[lvl][idx] = dx*dx+dy*dy
// and, with setting_gammaWeightsPixelSelect == 1 and a CalibHessian, then multiplies it by gw*gw, gw = CalibHessian::getBGradOnly(dI_l[idx][0]) (HessianBlocks.h:343-349).
// The oracle's makeImages (orc_tracker.cpp) is the first step, for the identity B; this file adds the second, the same float multiplication on the stored value, over
// the same index range [wl, wl*(hl-1)).  Built from the oracle's C entries (oracle/gamma.mk `orc`, over liborc.so), so the frames are liborc's and every oracle
// entry takes them.
#include <climits>

extern "C" {
void*        orc_frame_create(const float* color, int w, int h, int levels, float exposure);
const float* orc_frame_dI(void* f, int lvl);
const float* orc_frame_abs(void* f, int lvl);

// (int)(color+0.5f) clamped to [5, 250]: the reference's x86 build converts NaN and values outside the int range to INT_MIN (cvttss2si), hence 5
static int gamma_index(float color) {
  const float t = color + 0.5f;
  int c = (t >= -2147483648.0f && t < 2147483648.0f) ? (int)t : INT_MIN;
  if (c < 5) c = 5;
  if (c > 250) c = 250;
  return c;
}

// makeImages of a w x h frame with CalibHessian::B = B (256 floats)
void* orc_frame_create_gamma(const float* color, int w, int h, int levels, float exposure, const float* B) {
  void* f = orc_frame_create(color, w, h, levels, exposure);
  for (int lvl = 0; lvl < levels; lvl++) {
    const int wl = w >> lvl, hl = h >> lvl; const float* dI = orc_frame_dI(f, lvl); float* dabs = const_cast<float*>(orc_frame_abs(f, lvl));
    for (int idx = wl; idx < wl*(hl-1); idx++) {
      const int c = gamma_index(dI[3*idx]);
      const float gw = B[c+1] - B[c];
      dabs[idx] *= gw*gw;
    }
  }
  return f;
}
}
