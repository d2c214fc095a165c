// sdv_device.cuh — device-side data layout and per-point evaluation shared by the tracker kernels.
//
// HBM layout (DESIGN.md §3):
//   image pyramid level : planar float intensity (reference: AoS Vector3f dIp[lvl] + float absSquaredGrad[lvl], HessianBlocks.h:190-204); the consumers
//                         form the central differences of a bilinear footprint from its 12 planar taps, bit-identically to makeImages.  Packed float4
//                         {I, dx, dy, absSquaredGrad} texels are a per-frame cache built only for keyframe-rate consumers (selector, BA, read-back).
//   reference cloud     : float4 point {u, v, idepth, color}         (reference: 4 SoA arrays pc_u/pc_v/pc_idepth/pc_color,
//                         CoarseTracker.h) -> one coalesced 16-byte LDG per point
#pragma once
#include <cuda_runtime.h>
#include <stdint.h>
#include "sdv_math.cuh"
#include "sdv_core_common.cuh"

namespace sdv {

constexpr int kLevels = 6;
constexpr int kNH = 45;                  // upper triangle of the 9x9 Accumulator9 system
constexpr int kIdxE = 45, kIdxNE = 46, kIdxNSat = 47, kIdxFlowT = 48, kIdxFlowRT = 49, kIdxFlowN = 50;
constexpr int kNAcc = 51;

struct LevelGeom { int w, h; float fx, fy, cx, cy; float Ki[9]; };

struct EvalParams {                       // everything calcRes/calcGSSSE derive from (refToNew, aff_g2l, cutoffTH) at one level
  float RKi[9]; float t[3];
  float aLL, bLL;                         // AffLight::fromToVecExposure(...).cast<float>()   CoarseTracker.cpp:504
  float cutoff, maxEnergy, huber;
  float b0;                               // (float) lastRef_aff_g2l.b                          CoarseTracker.cpp:433
  int lvl;
};

SDV_HD void make_eval_params(const SE3d& refToNew, double a, double b, float refExposure, float newExposure, double ref_a, double ref_b,
                             const LevelGeom& g, int lvl, float cutoffTH, float huberTH, EvalParams& ep) {
  double R[9]; qmat(refToNew.q, R);
  float Rf[9]; for (int i=0;i<9;i++) Rf[i] = (float)R[i];
  for (int i=0;i<3;i++) for (int j=0;j<3;j++) ep.RKi[i*3+j] = (Rf[i*3]*g.Ki[j] + Rf[i*3+1]*g.Ki[3+j]) + Rf[i*3+2]*g.Ki[6+j];
  for (int i=0;i<3;i++) ep.t[i] = (float)refToNew.t[i];
  double aff[2]; aff_from_to(refExposure, newExposure, ref_a, ref_b, a, b, aff);
  ep.aLL = (float)aff[0]; ep.bLL = (float)aff[1];
  ep.cutoff = cutoffTH; ep.huber = huberTH;
  ep.maxEnergy = 2*huberTH*cutoffTH - huberTH*huberTH;
  ep.b0 = (float)ref_b; ep.lvl = lvl;
}

// Finalisation of the reduced sums into the reference's return values.
//   rs[6]            : Vec6 of calcRes            CoarseTracker.cpp:625-633
//   H (8x8), b (8)   : calcGSSSE outputs          CoarseTracker.cpp:468-483 (divide by PADDED n, then SCALE_* rows/cols)
SDV_HD void finalize_res(const double* tot, double* rs) {
  float E = (float)tot[kIdxE]; float nE = (float)tot[kIdxNE]; float nSat = (float)tot[kIdxNSat];
  float fT = (float)tot[kIdxFlowT], fRT = (float)tot[kIdxFlowRT], fN = (float)tot[kIdxFlowN];
  rs[0] = E; rs[1] = nE; rs[2] = fT/(fN+0.1); rs[3] = 0; rs[4] = fRT/(fN+0.1); rs[5] = nSat/nE;
}
SDV_HD void finalize_gs(const double* tot, double* H /*64*/, double* b /*8*/) {
  int nW = (int)(tot[kIdxNE] - tot[kIdxNSat]);
  int npad = (nW + 3) & ~3;
  float invn = 1.0f/npad;
  const float sc[8] = {1.0f,1.0f,1.0f,0.5f,0.5f,0.5f,10.0f,1000.0f};   // SCALE_XI_ROT x3, SCALE_XI_TRANS x3, SCALE_A, SCALE_B (HessianBlocks.h:33-40)
  int k = 0;
  for (int r=0;r<9;r++) for (int c=r;c<9;c++) {
    float hv = (float)tot[k++];
    if (r < 8 && c < 8) { double v = (double)hv * invn; v *= sc[c]; v *= sc[r]; H[r*8+c] = v; H[c*8+r] = v; }
    else if (r < 8 && c == 8) { double v = (double)hv * invn; v *= sc[r]; b[r] = v; }
  }
}

// (r,c) of the k-th entry of the row-major upper triangle of the 9x9 system (k = 0..44).  Host+device: tests/test_abi.py walks all 45 on the CPU (a wrong walk here
// silently mixes H entries; it once did, and only the GPU LM tests noticed).
SDV_HD void gs_entry_rc(int k, int& r, int& c) {
  r = 0; int base = 0; bool walking = true;
  for (int rr = 0; rr < 8; rr++) { const int next = base + (9 - rr); if (walking && k >= next) { r = rr + 1; base = next; } else walking = false; }
  c = r + (k - base);
}

#if defined(__CUDACC__)
// finalize_gs spread over the 32 lanes of a warp: lane handles upper-triangle entries k = lane and lane + 32 (45 entries), same arithmetic per entry as finalize_gs
// (CoarseTracker.cpp:468-483).  45 dependent read-convert-scale-store chains on one lane cost ~9k cycles per LM evaluation; this is ~0.5k.
__device__ __forceinline__ void finalize_gs_warp(const double* tot, double* H /*64*/, double* b /*8*/, int lane) {
  const int nW = (int)(tot[kIdxNE] - tot[kIdxNSat]);
  const int npad = (nW + 3) & ~3;
  const float invn = 1.0f/npad;
#pragma unroll
  for (int rep = 0; rep < 2; rep++) {
    const int k = lane + 32*rep;
    if (k < kNH) {
      // (r,c) of the k-th entry of the row-major upper triangle of the 9x9 system
      int r, c; gs_entry_rc(k, r, c);
      const float scr = (r < 3) ? 1.0f : ((r < 6) ? 0.5f : ((r == 6) ? 10.0f : 1000.0f));   // SCALE_XI_ROT x3, SCALE_XI_TRANS x3, SCALE_A, SCALE_B
      const float scc = (c < 3) ? 1.0f : ((c < 6) ? 0.5f : ((c == 6) ? 10.0f : 1000.0f));
      const float hv = (float)tot[k];
      if (r < 8 && c < 8) { double v = (double)hv * invn; v *= scc; v *= scr; H[r*8+c] = v; H[c*8+r] = v; }
      else if (r < 8 && c == 8) { double v = (double)hv * invn; v *= scr; b[r] = v; }
    }
  }
}
#endif

#if defined(__CUDACC__)
// One reference point through calcRes (CoarseTracker.cpp:525-601) and, if it lands in buf_warped_*, through the
// Jacobian/outer-product of calcGSSSE + Accumulator9::updateSSE_eighted (CoarseTracker.cpp:442-466, MatrixAccumulators.h:1040-1115), in pieces that
// both tracker kernels compose: eval_point (coarse_res_gs_kernel) and stage_project / stage_accumulate (track_cluster_kernel, which gathers the taps
// asynchronously between the two).  Arithmetic order follows the reference expression trees; the TU is compiled with --fmad=false so only the explicit
// fmaf() of the accumulation contracts.
struct ProjPt { float u, v, Ku, Kv, nid; };               // normalised and pixel coordinates, new inverse depth
__device__ __forceinline__ ProjPt project_point(const float4 p, const LevelGeom& g, const EvalParams& ep) {
  const float x = p.x, y = p.y, id = p.z;
  float pt0 = ((ep.RKi[0]*x + ep.RKi[1]*y) + ep.RKi[2]*1.0f) + ep.t[0]*id;
  float pt1 = ((ep.RKi[3]*x + ep.RKi[4]*y) + ep.RKi[5]*1.0f) + ep.t[1]*id;
  float pt2 = ((ep.RKi[6]*x + ep.RKi[7]*y) + ep.RKi[8]*1.0f) + ep.t[2]*id;
  ProjPt q;
  q.u = pt0 / pt2; q.v = pt1 / pt2;
  q.Ku = g.fx*q.u + g.cx; q.Kv = g.fy*q.v + g.cy;
  q.nid = id / pt2;
  return q;
}
__device__ __forceinline__ bool proj_inside(const ProjPt& q, const LevelGeom& g) {
  return q.Ku > 2 && q.Kv > 2 && q.Ku < (float)(g.w-3) && q.Kv < (float)(g.h-3) && q.nid > 0;
}

// flow indicators of one level-0 point with index % 32 == 0 (CoarseTracker.cpp:538-566)
__device__ __forceinline__ void flow_point(const float4 p, const LevelGeom& g, const EvalParams& ep, float (&acc)[kNAcc]) {
  const float x = p.x, y = p.y, id = p.z;
  const ProjPt q = project_point(p, g, ep);
  float k0 = (g.Ki[0]*x + g.Ki[1]*y) + g.Ki[2]*1.0f, k1 = (g.Ki[3]*x + g.Ki[4]*y) + g.Ki[5]*1.0f, k2 = (g.Ki[6]*x + g.Ki[7]*y) + g.Ki[8]*1.0f;
  float r0 = (ep.RKi[0]*x + ep.RKi[1]*y) + ep.RKi[2]*1.0f, r1 = (ep.RKi[3]*x + ep.RKi[4]*y) + ep.RKi[5]*1.0f, r2 = (ep.RKi[6]*x + ep.RKi[7]*y) + ep.RKi[8]*1.0f;
  float a0 = k0 + ep.t[0]*id, a1 = k1 + ep.t[1]*id, a2 = k2 + ep.t[2]*id;
  float KuT = g.fx*(a0/a2) + g.cx, KvT = g.fy*(a1/a2) + g.cy;
  float b0_ = k0 - ep.t[0]*id, b1_ = k1 - ep.t[1]*id, b2_ = k2 - ep.t[2]*id;
  float KuT2 = g.fx*(b0_/b2_) + g.cx, KvT2 = g.fy*(b1_/b2_) + g.cy;
  float c0 = r0 - ep.t[0]*id, c1 = r1 - ep.t[1]*id, c2 = r2 - ep.t[2]*id;
  float Ku3 = g.fx*(c0/c2) + g.cx, Kv3 = g.fy*(c1/c2) + g.cy;
  acc[kIdxFlowT]  += (KuT-x)*(KuT-x) + (KvT-y)*(KvT-y);
  acc[kIdxFlowT]  += (KuT2-x)*(KuT2-x) + (KvT2-y)*(KvT2-y);
  acc[kIdxFlowRT] += (q.Ku-x)*(q.Ku-x) + (q.Kv-y)*(q.Kv-y);
  acc[kIdxFlowRT] += (Ku3-x)*(Ku3-x) + (Kv3-y)*(Kv3-y);
  acc[kIdxFlowN]  += 2.0f;
}

// getInterpolatedElement33 (util/globalFuncs.h:51-65) at fractional offset (dx, dy) of the inside point q, residual, Huber weight and outer product.
// tap(k), k = 0..11: the 12-tap planar footprint rows -1..2 around the integer pixel — row -1: 0,1; row 0: -1..2; row 1: -1..2; row 2: 0,1 — from which the
// gradients are formed exactly like makeImages does (HessianBlocks.cpp:147-156; the taps never touch rows 0 / h-1).
template <class Tap>
__device__ __forceinline__ void accumulate_point(const Tap& tap, float dx, float dy, const ProjPt& q, float refColor, const LevelGeom& g, const EvalParams& ep,
                                                 float (&acc)[kNAcc]) {
  float4 p00, p10, p01, p11;
  float a_m1_0 = tap(0), a_m1_1 = tap(1);
  float a_0_m1 = tap(2), a_0_0 = tap(3), a_0_1 = tap(4), a_0_2 = tap(5);
  float a_1_m1 = tap(6), a_1_0 = tap(7), a_1_1 = tap(8), a_1_2 = tap(9);
  float a_2_0 = tap(10), a_2_1 = tap(11);
  p00.x = a_0_0; p00.y = grad_guard(0.5f*(a_0_1 - a_0_m1)); p00.z = grad_guard(0.5f*(a_1_0 - a_m1_0));
  p10.x = a_0_1; p10.y = grad_guard(0.5f*(a_0_2 - a_0_0));  p10.z = grad_guard(0.5f*(a_1_1 - a_m1_1));
  p01.x = a_1_0; p01.y = grad_guard(0.5f*(a_1_1 - a_1_m1)); p01.z = grad_guard(0.5f*(a_2_0 - a_0_0));
  p11.x = a_1_1; p11.y = grad_guard(0.5f*(a_1_2 - a_1_0));  p11.z = grad_guard(0.5f*(a_2_1 - a_0_1));
  const float dxdy = dx*dy, u = q.u, v = q.v, new_idepth = q.nid;
  float w11 = dxdy, w01 = dy-dxdy, w10 = dx-dxdy, w00 = 1-dx-dy+dxdy;
  float hit0 = ((w11*p11.x + w01*p01.x) + w10*p10.x) + w00*p00.x;
  float hit1 = ((w11*p11.y + w01*p01.y) + w10*p10.y) + w00*p00.y;
  float hit2 = ((w11*p11.z + w01*p01.z) + w10*p10.z) + w00*p00.z;
  if (!isfinite(hit0)) return;

  float residual = hit0 - (ep.aLL*refColor + ep.bLL);
  float ar = fabsf(residual);
  float hw = ar < ep.huber ? 1.0f : ep.huber / ar;
  acc[kIdxNE] += 1.0f;
  if (ar > ep.cutoff) { acc[kIdxE] += ep.maxEnergy; acc[kIdxNSat] += 1.0f; return; }
  acc[kIdxE] += hw*residual*residual*(2-hw);

  float dxf = hit1*g.fx, dyf = hit2*g.fy;
  float J[9];
  J[0] = new_idepth*dxf;
  J[1] = new_idepth*dyf;
  J[2] = 0.0f - new_idepth*(u*dxf + v*dyf);
  J[3] = 0.0f - ((u*v)*dxf + dyf*(1.0f + v*v));
  J[4] = (u*v)*dyf + dxf*(1.0f + u*u);
  J[5] = u*dyf - v*dxf;
  J[6] = ep.aLL*(ep.b0 - refColor);
  J[7] = -1.0f;
  J[8] = residual;
  int k = 0;
#pragma unroll
  for (int r = 0; r < 9; r++) {
    float Jw = J[r]*hw;
#pragma unroll
    for (int c = r; c < 9; c++) { acc[k] = fmaf(Jw, J[c], acc[k]); k++; }
  }
}

// point i of the reference cloud, taps read straight from the planar level I
__device__ __forceinline__ void eval_point(const float4 p, int i, const LevelGeom& g, const EvalParams& ep,
                                           const float* __restrict__ I, float (&acc)[kNAcc]) {
  const ProjPt q = project_point(p, g, ep);
  if (ep.lvl == 0 && (i & 31) == 0) flow_point(p, g, ep, acc);
  if (!proj_inside(q, g)) return;
  const int ix = (int)q.Ku, iy = (int)q.Kv, w = g.w;
  const float* b = I + ix + iy*w;
  const auto tap = [&](int k) {
    const float* r = k < 2 ? b - w : (k < 6 ? b : (k < 10 ? b + w : b + 2*w));
    return __ldg(r + (k < 2 ? k : (k < 6 ? k - 3 : (k < 10 ? k - 7 : k - 10))));
  };
  accumulate_point(tap, q.Ku - ix, q.Kv - iy, q, p.w, g, ep, acc);
}
#endif

// -------------------------------------------------------------------------------------------- job descriptors
struct TrackerRef {                       // one CoarseTracker instance's reference state (device pointers)
  const float4* pts[kLevels]; int npts[kLevels];
  uint64_t ref_frame; float refExposure; double ref_a, ref_b;
};

struct TrackJob {                         // one trackNewestCoarse call
  const float* img[kLevels];              // newFrame planar intensity of every level (gradients formed on the fly)
  const float4* pts[kLevels]; int npts[kLevels];
  float refExposure, newExposure; double ref_a, ref_b;
  double T[7]; double ab[2];              // in: lastToNew_out / aff_g2l_out initial ; out: result (if not aborted)
  double minRes[5]; int coarsest;
  int geom_row;                           // row of the geometry table (sdv_ctx::geom_dev) this job's tracker slot uses
  double lastRes[5]; double flow[3]; int good;
  long long point_evals[kLevels]; int iterations[kLevels]; int accepts[kLevels];
};
static_assert(sizeof(TrackJob) == 432, "geom_row lives in the padding after coarsest: the job descriptor (sdv_track_job_bytes) keeps its size");

// One row of the geometry table: CoarseTracker::makeK (CoarseTracker.cpp:77-106) of one K at every level.  The table holds one row for the context
// calibration (row 0) and one per tracker slot (row 1 + slot); a slot without its own K points at row 0.
struct GeomRow { LevelGeom g[kLevels]; };

struct TrackConst {                       // per-context scalar settings
  int levels;
  float huberTH, coarseCutoffTH, affineOptModeA, affineOptModeB;
};

} // namespace sdv
