// sdv_trace.cu — immature-point path (SURVEY.md §8f rank 2): candidate construction and epipolar tracing on the device.
//
//   ImmaturePoint::ImmaturePoint   /root/reference/src/FullSystem/ImmaturePoint.cpp:8-36    -> imm_init_kernel
//   ImmaturePoint::traceOn         /root/reference/src/FullSystem/ImmaturePoint.cpp:50-352  -> imm_trace_kernel
//   the per-host loop of FullSystem::traceNewCoarse (FullSystem.cpp:519-552) is the "group" dimension of sdv_immature_trace_batch
//
// One thread per candidate: the function is a sequential state machine per point (<= 99 discrete steps of an 8-pixel pattern along the epipolar segment, <= 3
// Gauss-Newton steps along the line, interval update), the ~500 x nF candidates of a frame — times the resident sequences in batched mode — are the parallelism.
// It reads the level-0 image of the traced frame only: intensities for the discrete search (planar plane, 4 taps per sample), {I,dx,dy} for the refinement, with
// the gradients formed from the planar plane exactly as FrameHessian::makeImages forms them (HessianBlocks.cpp:147-156), so no packed level-0 image is needed.
// float arithmetic in the reference's operation order, compiled with --fmad=false like the rest of the library: results are bit-identical to the CPU code
// (tests/test_gpu_trace.py against the oracle, which tests/test_ref_pin_trace.py pins on the reference's own compiled ImmaturePoint.cpp).
#include <cuda_runtime.h>
#include <stdint.h>
#include <math.h>
#include <string.h>
#include <vector>
#include <algorithm>
#include "sdv_ctx.cuh"
#include "sdv_pool.cuh"

using namespace sdv;

namespace sdv {


struct TraceGroupDev { const float* I0; float KRKi[9], Kt[3], aff[2]; int pt_begin, pt_end; int w, h; };   // one (host keyframe, traced frame) pair; w, h: its camera's size
struct TraceSet { float outlierTH, outlierTHSumComponent, overallEnergyTHWeight, huberTH, maxPixSearch; int minTraceTestRadius; float stepsize; int GNIterations;
                  float GNThreshold, extraSlackOnTH, slackInterval, minImprovementFactor; };

// dIp[0][idx] = {I, dx, dy} from the planar level-0 plane
__device__ __forceinline__ void texel0(const float* __restrict__ I, int idx, int w, int h, float& c, float& dx, float& dy) {
  c = __ldg(I + idx); planar_grad(I, idx, w, h, dx, dy);
}
__device__ __forceinline__ void interp33(const float* __restrict__ I, float x, float y, int w, int h, float out[3]) {   // getInterpolatedElement33, :51-65
  const int ix = (int)x, iy = (int)y; const float dx = x - ix, dy = y - iy, dxdy = dx*dy; const int b = ix + iy*w;
  float c11[3], c01[3], c10[3], c00[3];
  texel0(I, b+1+w, w, h, c11[0], c11[1], c11[2]); texel0(I, b+w, w, h, c01[0], c01[1], c01[2]); texel0(I, b+1, w, h, c10[0], c10[1], c10[2]); texel0(I, b, w, h, c00[0], c00[1], c00[2]);
  const float w11 = dxdy, w01 = dy-dxdy, w10 = dx-dxdy, w00 = 1-dx-dy+dxdy;
#pragma unroll
  for (int k = 0; k < 3; k++) out[k] = w11*c11[k] + w01*c01[k] + w10*c10[k] + w00*c00[k];
}

// one thread per candidate
__global__ void __launch_bounds__(128) imm_init_kernel(const float* __restrict__ I0, int w, int h, int n, const int* __restrict__ uv, sdv_immature_pt* __restrict__ out, TraceSet S) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= n) return;
  sdv_immature_pt p; imm_construct(I0, w, uv[2*i], uv[2*i+1], S, p);
  out[i] = p;
}

// ---- ImmaturePoint::traceOn (ImmaturePoint.cpp:50-352)
__device__ int trace_on(sdv_immature_pt& p, const float* __restrict__ I, int wG0, int hG0, const float* KRKi, const float* Kt, const float* aff, const TraceSet& S) {
  if (p.lastTraceStatus == IPS_OOB) return p.lastTraceStatus;
  const float maxPixSearch = (wG0+hG0)*S.maxPixSearch;
  float pr[3];
#pragma unroll
  for (int i = 0; i < 3; i++) pr[i] = (KRKi[i*3]*p.u + KRKi[i*3+1]*p.v) + KRKi[i*3+2]*1.0f;
  float ptpMin[3];
#pragma unroll
  for (int i = 0; i < 3; i++) ptpMin[i] = pr[i] + Kt[i]*p.idepth_min;
  const float uMin = ptpMin[0]/ptpMin[2], vMin = ptpMin[1]/ptpMin[2];
#define TRACE_OOB() do { p.lastTraceUV[0] = -1; p.lastTraceUV[1] = -1; p.lastTracePixelInterval = 0; return p.lastTraceStatus = IPS_OOB; } while (0)
  if (!(uMin > 4 && vMin > 4 && uMin < wG0-5 && vMin < hG0-5)) TRACE_OOB();
  float dist, uMax, vMax, ptpMax[3];
  if (isfinite(p.idepth_max)) {
#pragma unroll
    for (int i = 0; i < 3; i++) ptpMax[i] = pr[i] + Kt[i]*p.idepth_max;
    uMax = ptpMax[0]/ptpMax[2]; vMax = ptpMax[1]/ptpMax[2];
    if (!(uMax > 4 && vMax > 4 && uMax < wG0-5 && vMax < hG0-5)) TRACE_OOB();
    dist = (uMin-uMax)*(uMin-uMax) + (vMin-vMax)*(vMin-vMax);
    dist = sqrtf(dist);
    if (dist < S.slackInterval) {
      p.lastTraceUV[0] = (uMax+uMin)*0.5f; p.lastTraceUV[1] = (vMax+vMin)*0.5f; p.lastTracePixelInterval = dist;
      return p.lastTraceStatus = IPS_SKIPPED;
    }
  } else {
    dist = maxPixSearch;
#pragma unroll
    for (int i = 0; i < 3; i++) ptpMax[i] = pr[i] + Kt[i]*0.01f;
    uMax = ptpMax[0]/ptpMax[2]; vMax = ptpMax[1]/ptpMax[2];
    const float ddx = uMax-uMin, ddy = vMax-vMin;
    const float d = 1.0f / sqrtf(ddx*ddx+ddy*ddy);
    uMax = uMin + dist*ddx*d; vMax = vMin + dist*ddy*d;
    if (!(uMax > 4 && vMax > 4 && uMax < wG0-5 && vMax < hG0-5)) TRACE_OOB();
  }
  if (!(p.idepth_min < 0 || (ptpMin[2] > 0.75f && ptpMin[2] < 1.5f))) TRACE_OOB();
  float dx = S.stepsize*(uMax-uMin), dy = S.stepsize*(vMax-vMin);
  const float* g = p.gradH;
  const float a = (dx*g[0] + dy*g[2])*dx + (dx*g[1] + dy*g[3])*dy;
  const float ndx = -dx;
  const float b = (dy*g[0] + ndx*g[2])*dy + (dy*g[1] + ndx*g[3])*ndx;
  float errorInPixel = 0.2f + 0.2f*(a+b)/a;
  if (errorInPixel*S.minImprovementFactor > dist && isfinite(p.idepth_max)) {
    p.lastTraceUV[0] = (uMax+uMin)*0.5f; p.lastTraceUV[1] = (vMax+vMin)*0.5f; p.lastTracePixelInterval = dist;
    return p.lastTraceStatus = IPS_BADCONDITION;
  }
  if (errorInPixel > 10) errorInPixel = 10;
  dx /= dist; dy /= dist;
  if (dist > maxPixSearch) { uMax = uMin + maxPixSearch*dx; vMax = vMin + maxPixSearch*dy; dist = maxPixSearch; }
  int numSteps = (int)(1.9999f + dist / S.stepsize);
  const float R00 = KRKi[0], R01 = KRKi[1], R10 = KRKi[3], R11 = KRKi[4];
  const float randShift = uMin*1000-floorf(uMin*1000);
  float ptx = uMin-randShift*dx, pty = vMin-randShift*dy;
  float rpx[8], rpy[8];
#pragma unroll
  for (int idx = 0; idx < 8; idx++) { const float px = (float)staticPattern[idx][0], py = (float)staticPattern[idx][1]; rpx[idx] = R00*px + R01*py; rpy[idx] = R10*px + R11*py; }
  if (!isfinite(dx) || !isfinite(dy)) { p.lastTracePixelInterval = 0; p.lastTraceUV[0] = -1; p.lastTraceUV[1] = -1; return p.lastTraceStatus = IPS_OOB; }
  float errors[100]; float bestU = 0, bestV = 0, bestEnergy = 1e10f; int bestIdx = -1;
  if (numSteps >= 100) numSteps = 99;
  float affc[8];
#pragma unroll
  for (int idx = 0; idx < 8; idx++) affc[idx] = (float)(aff[0]*p.color[idx] + aff[1]);
  for (int i = 0; i < numSteps; i++) {
    float energy = 0;
#pragma unroll
    for (int idx = 0; idx < 8; idx++) {
      const float hitColor = interp31(I, (float)(ptx+rpx[idx]), (float)(pty+rpy[idx]), wG0);
      if (!isfinite(hitColor)) { energy += 1e5f; continue; }
      const float residual = hitColor - affc[idx];
      const float hw = fabsf(residual) < S.huberTH ? 1 : S.huberTH / fabsf(residual);
      energy += hw*residual*residual*(2-hw);
    }
    errors[i] = energy;
    if (energy < bestEnergy) { bestU = ptx; bestV = pty; bestEnergy = energy; bestIdx = i; }
    ptx += dx; pty += dy;
  }
  float secondBest = 1e10f;
  for (int i = 0; i < numSteps; i++)
    if ((i < bestIdx-S.minTraceTestRadius || i > bestIdx+S.minTraceTestRadius) && errors[i] < secondBest) secondBest = errors[i];
  const float newQuality = secondBest / bestEnergy;
  if (newQuality < p.quality || numSteps > 10) p.quality = newQuality;
  float uBak = bestU, vBak = bestV, stepBack = 0; const float gnstepsize = 1;
  if (S.GNIterations > 0) bestEnergy = 1e5f;
  for (int it = 0; it < S.GNIterations; it++) {
    float H = 1, bb = 0, energy = 0;
    for (int idx = 0; idx < 8; idx++) {
      float hc[3]; interp33(I, (float)(bestU+rpx[idx]), (float)(bestV+rpy[idx]), wG0, hG0, hc);
      if (!isfinite(hc[0])) { energy += 1e5f; continue; }
      const float residual = hc[0] - (aff[0]*p.color[idx] + aff[1]);
      const float dResdDist = dx*hc[1] + dy*hc[2];
      const float hw = fabsf(residual) < S.huberTH ? 1 : S.huberTH / fabsf(residual);
      H += hw*dResdDist*dResdDist;
      bb += hw*residual*dResdDist;
      energy += p.weights[idx]*p.weights[idx]*hw*residual*residual*(2-hw);
    }
    if (energy > bestEnergy) {
      stepBack *= 0.5f;
      bestU = uBak + stepBack*dx; bestV = vBak + stepBack*dy;
    } else {
      float step = -gnstepsize*bb/H;
      if (step < -0.5f) step = -0.5f; else if (step > 0.5f) step = 0.5f;
      if (!isfinite(step)) step = 0;
      uBak = bestU; vBak = bestV; stepBack = step;
      bestU += step*dx; bestV += step*dy; bestEnergy = energy;
    }
    if (fabsf(stepBack) < S.GNThreshold) break;
  }
  if (!(bestEnergy < p.energyTH*S.extraSlackOnTH)) {
    p.lastTracePixelInterval = 0; p.lastTraceUV[0] = -1; p.lastTraceUV[1] = -1;
    if (p.lastTraceStatus == IPS_OUTLIER) return p.lastTraceStatus = IPS_OOB;
    return p.lastTraceStatus = IPS_OUTLIER;
  }
  if (dx*dx > dy*dy) {
    p.idepth_min = (pr[2]*(bestU-errorInPixel*dx) - pr[0]) / (Kt[0] - Kt[2]*(bestU-errorInPixel*dx));
    p.idepth_max = (pr[2]*(bestU+errorInPixel*dx) - pr[0]) / (Kt[0] - Kt[2]*(bestU+errorInPixel*dx));
  } else {
    p.idepth_min = (pr[2]*(bestV-errorInPixel*dy) - pr[1]) / (Kt[1] - Kt[2]*(bestV-errorInPixel*dy));
    p.idepth_max = (pr[2]*(bestV+errorInPixel*dy) - pr[1]) / (Kt[1] - Kt[2]*(bestV+errorInPixel*dy));
  }
  if (p.idepth_min > p.idepth_max) { const float t = p.idepth_min; p.idepth_min = p.idepth_max; p.idepth_max = t; }
  if (!isfinite(p.idepth_min) || !isfinite(p.idepth_max) || (p.idepth_max < 0)) {
    p.lastTracePixelInterval = 0; p.lastTraceUV[0] = -1; p.lastTraceUV[1] = -1;
    return p.lastTraceStatus = IPS_OUTLIER;
  }
  p.lastTracePixelInterval = 2*errorInPixel;
  p.lastTraceUV[0] = bestU; p.lastTraceUV[1] = bestV;
  return p.lastTraceStatus = IPS_GOOD;
#undef TRACE_OOB
}

__global__ void __launch_bounds__(128) imm_trace_kernel(const TraceGroupDev* __restrict__ groups, const int* __restrict__ group_of, int n, sdv_immature_pt* __restrict__ pts, int* __restrict__ status,
                                                        TraceSet S) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= n) return;
  const TraceGroupDev& G = groups[group_of[i]];
  sdv_immature_pt p = pts[i];
  const int st = trace_on(p, G.I0, G.w, G.h, G.KRKi, G.Kt, G.aff, S);
  pts[i] = p; status[i] = st;
}

// ---- activation: FullSystem::optimizeImmaturePoint (FullSystemOptPoint.cpp:18-183) over ImmaturePoint::linearizeResidual (ImmaturePoint.cpp:410-476)
struct OptTargetDev { const float* I0; float R[9], t[3], aff[2]; };          // target image + FrameFramePrecalc {PRE_RTll, PRE_tTll, PRE_aff_mode} of (host,target)
struct OptGroupDev { int tgt_begin, nres; float fxl, fyl, cxl, cyl, fxli, fyli; int w, h; };    // w, h: the size of the group's camera (every target's)
enum { RS_IN = 0, RS_OOB, RS_OUTLIER };
struct TmpResDev { int state_state; double state_energy; int state_NewState; double state_NewEnergy; };

__device__ double linearize_residual(const sdv_immature_pt& p, const OptTargetDev& T, const OptGroupDev& C, int wG0, int hG0, float outlierTHSlack, TmpResDev& r, float& Hdd, float& bd,
                                     float idepth, float huberTH) {
  if (r.state_state == RS_OOB) { r.state_NewState = RS_OOB; return r.state_energy; }
  float energyLeft = 0; const float wM3G = (float)(wG0-3), hM3G = (float)(hG0-3);
  for (int idx = 0; idx < 8; idx++) {
    const int dx = staticPattern[idx][0], dy = staticPattern[idx][1];
    const float K0 = (p.u+dx-C.cxl)*C.fxli, K1 = (p.v+dy-C.cyl)*C.fyli, K2 = 1;
    float ptp[3];
#pragma unroll
    for (int i = 0; i < 3; i++) ptp[i] = ((T.R[i*3]*K0 + T.R[i*3+1]*K1) + T.R[i*3+2]*K2) + T.t[i]*idepth;
    const float drescale = 1.0f/ptp[2];
    if (!(drescale > 0)) { r.state_NewState = RS_OOB; return r.state_energy; }
    const float u = ptp[0]*drescale, v = ptp[1]*drescale;
    const float Ku = u*C.fxl + C.cxl, Kv = v*C.fyl + C.cyl;
    if (!(Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G)) { r.state_NewState = RS_OOB; return r.state_energy; }
    float hc[3]; interp33(T.I0, Ku, Kv, wG0, hG0, hc);
    if (!isfinite(hc[0])) { r.state_NewState = RS_OOB; return r.state_energy; }
    const float residual = hc[0] - (T.aff[0]*p.color[idx] + T.aff[1]);
    float hw = fabsf(residual) < huberTH ? 1 : huberTH / fabsf(residual);
    energyLeft += p.weights[idx]*p.weights[idx]*hw*residual*residual*(2-hw);
    const float dxInterp = hc[1]*C.fxl, dyInterp = hc[2]*C.fyl;
    const float d_idepth = (dxInterp*drescale*(T.t[0]-T.t[2]*u) + dyInterp*drescale*(T.t[1]-T.t[2]*v))*1.0f;
    hw *= p.weights[idx]*p.weights[idx];
    Hdd += (hw*d_idepth)*d_idepth;
    bd += (hw*residual)*d_idepth;
  }
  if (energyLeft > p.energyTH*outlierTHSlack) { energyLeft = p.energyTH*outlierTHSlack; r.state_NewState = RS_OUTLIER; }
  else r.state_NewState = RS_IN;
  r.state_NewEnergy = energyLeft;
  return energyLeft;
}

constexpr int kOptMaxRes = SDV_MAX_FRAMES_WINDOW;
__global__ void __launch_bounds__(64) imm_optimize_kernel(const OptGroupDev* __restrict__ groups, const OptTargetDev* __restrict__ targets, const int* __restrict__ group_of, int n,
                                                           const sdv_immature_pt* __restrict__ pts, const unsigned char* __restrict__ from_sensor, int min_obs, int res_stride,
                                                           int* __restrict__ status, float* __restrict__ idepth_out, int* __restrict__ res_state, float huberTH) {
  const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= n) return;
  const OptGroupDev G = groups[group_of[k]]; const OptTargetDev* T = targets + G.tgt_begin; const int nres = G.nres, w = G.w, h = G.h;
  const sdv_immature_pt p = pts[k]; const bool isFromSensor = from_sensor && from_sensor[k];
  const float minIdepthH_act = 100; const int GNIts = 3;                      // util/settings.cpp:41,133
  TmpResDev res[kOptMaxRes];
  for (int i = 0; i < nres; i++) { res[i].state_NewEnergy = res[i].state_energy = 0; res[i].state_NewState = RS_OUTLIER; res[i].state_state = RS_IN; }
  for (int i = 0; i < res_stride; i++) res_state[(size_t)k*res_stride + i] = -1;
  idepth_out[k] = 0;
  float lastEnergy = 0, lastHdd = 0, lastbd = 0;
  float currentIdepth = (p.idepth_max+p.idepth_min)*0.5f;
  const float trueDepth = currentIdepth;
  if (!isFromSensor) {
    for (int i = 0; i < nres; i++) {
      lastEnergy = (float)((double)lastEnergy + linearize_residual(p, T[i], G, w, h, 1000, res[i], lastHdd, lastbd, currentIdepth, huberTH));
      res[i].state_state = res[i].state_NewState; res[i].state_energy = res[i].state_NewEnergy;
    }
    if (!isfinite(lastEnergy) || lastHdd < minIdepthH_act) { status[k] = 0; return; }
    float lambda = 0.1f;
    for (int iteration = 0; iteration < GNIts; iteration++) {
      float H = lastHdd; H *= 1+lambda;
      const float step = (float)((1.0/(double)H) * (double)lastbd);
      const float newIdepth = currentIdepth - step;
      float newHdd = 0, newbd = 0, newEnergy = 0;
      for (int i = 0; i < nres; i++) newEnergy = (float)((double)newEnergy + linearize_residual(p, T[i], G, w, h, 1, res[i], newHdd, newbd, newIdepth, huberTH));
      if (!isfinite(lastEnergy) || newHdd < minIdepthH_act) { status[k] = 0; return; }
      if (newEnergy < lastEnergy) {
        currentIdepth = newIdepth; lastHdd = newHdd; lastbd = newbd; lastEnergy = newEnergy;
        for (int i = 0; i < nres; i++) { res[i].state_state = res[i].state_NewState; res[i].state_energy = res[i].state_NewEnergy; }
        lambda = (float)((double)lambda*0.5);
      } else lambda = (float)((double)lambda*5.0);
      if ((double)fabsf(step) < 0.0001*(double)currentIdepth) break;
    }
  }
  if (!isfinite(currentIdepth)) { status[k] = -1; return; }
  int numGoodRes = 0; for (int i = 0; i < nres; i++) if (res[i].state_state == RS_IN) numGoodRes++;
  if (numGoodRes < min_obs || !isfinite(p.energyTH)) { status[k] = -1; return; }
  idepth_out[k] = isFromSensor ? trueDepth : currentIdepth;
  for (int i = 0; i < nres; i++) res_state[(size_t)k*res_stride + i] = res[i].state_state;
  status[k] = 1;
}

static TraceSet trace_settings(const sdv_ctx* c) {
  TraceSet S; S.outlierTH = c->set.outlierTH; S.outlierTHSumComponent = c->set.outlierTHSumComponent; S.overallEnergyTHWeight = 1; S.huberTH = c->set.huberTH;
  S.maxPixSearch = 0.027f; S.minTraceTestRadius = 2; S.stepsize = 1.0f; S.GNIterations = 3; S.GNThreshold = 0.1f; S.extraSlackOnTH = 1.2f; S.slackInterval = 1.5f;
  S.minImprovementFactor = 2;                                                                   // util/settings.cpp:111,130-139
  return S;
}
// The immature-point calls carve their device arrays from the tracker-stream scratch c->scr and upload from pageable vectors, whose copies are staged before
// the call returns.  Not from pinned memory: sdv_immature_trace_store_batch without counts returns with its kernel still queued, and the next call rewrites c->scr_host.
#define TRACE_SCRATCH(bytes, who) do { if (c->scr.reserve(bytes, c->st)) return ctx_fail(c, SDV_ERR_CUDA, "%s: scratch of %zu bytes", who, (size_t)(bytes)); c->scr.reset(); } while (0)

// ---- the immature-point store: host->immaturePoints of every keyframe kept on the device (sdv_immature_store_*, sdv_immature_trace_store_batch)
// A block keeps each record in two arrays split by what traceOn does with the fields: ImmRO (92 B) it only reads, ImmRW (28 B) it writes.  A per-frame trace
// therefore writes 28 B per point instead of 120, and a point that is already OOB (traceOn returns at once) costs one 4-byte status read.
struct ImmRO { float u, v, color[8], weights[8], gradH[4], energyTH; };
struct ImmRW { float idepth_min, idepth_max, quality, lastTraceUV[2], lastTracePixelInterval; int32_t status; };
static_assert(sizeof(ImmRO) + sizeof(ImmRW) == sizeof(sdv_immature_pt) && sizeof(sdv_immature_meta) == 16, "store layout");
__host__ __device__ __forceinline__ void imm_split(const sdv_immature_pt& p, ImmRO& a, ImmRW& b) {
  a.u = p.u; a.v = p.v; for (int k = 0; k < 8; k++) { a.color[k] = p.color[k]; a.weights[k] = p.weights[k]; } for (int k = 0; k < 4; k++) a.gradH[k] = p.gradH[k]; a.energyTH = p.energyTH;
  b.idepth_min = p.idepth_min; b.idepth_max = p.idepth_max; b.quality = p.quality; b.lastTraceUV[0] = p.lastTraceUV[0]; b.lastTraceUV[1] = p.lastTraceUV[1];
  b.lastTracePixelInterval = p.lastTracePixelInterval; b.status = p.lastTraceStatus;
}
__host__ __device__ __forceinline__ void imm_join(const ImmRO& a, const ImmRW& b, sdv_immature_pt& p) {
  p.u = a.u; p.v = a.v; for (int k = 0; k < 8; k++) { p.color[k] = a.color[k]; p.weights[k] = a.weights[k]; } for (int k = 0; k < 4; k++) p.gradH[k] = a.gradH[k]; p.energyTH = a.energyTH;
  p.idepth_min = b.idepth_min; p.idepth_max = b.idepth_max; p.quality = b.quality; p.lastTraceUV[0] = b.lastTraceUV[0]; p.lastTraceUV[1] = b.lastTraceUV[1];
  p.lastTracePixelInterval = b.lastTracePixelInterval; p.lastTraceStatus = b.status;
}
static size_t al16(size_t b) { return (b + 15) & ~(size_t)15; }
struct ImmBlock {                                                                          // one allocation: ro | rw | meta, cap points each
  ImmRO* ro = nullptr; ImmRW* rw = nullptr; sdv_immature_meta* meta = nullptr; int n = 0, cap = 0;
  char* base() const { return (char*)ro; }
  static size_t bytes(int cap) { return al16((size_t)cap*sizeof(ImmRO)) + al16((size_t)cap*sizeof(ImmRW)) + (size_t)cap*sizeof(sdv_immature_meta); }
  static ImmBlock layout(char* p, int cap) {
    ImmBlock nb; const size_t o_rw = al16((size_t)cap*sizeof(ImmRO)), o_m = o_rw + al16((size_t)cap*sizeof(ImmRW));
    nb.ro = (ImmRO*)p; nb.rw = (ImmRW*)(p + o_rw); nb.meta = (sdv_immature_meta*)(p + o_m); nb.cap = cap; return nb;
  }
};
struct ImmStore : BlockPool<ImmBlock> {};                                                 // one block per host keyframe (sdv_pool.cuh: plan / commit / abandon)
using ImmPlan = ImmStore::Plan;
void imm_store_destroy(sdv_ctx* c) {
  ImmStore* S = (ImmStore*)c->imm_store; if (!S) return;
  S->release(); delete S; c->imm_store = nullptr;
}
static ImmStore* imm_store(sdv_ctx* c) { if (!c->imm_store) c->imm_store = new ImmStore(); return (ImmStore*)c->imm_store; }
static int imm_store_plan(sdv_ctx* c, ImmStore* S, int nh, const uint64_t* hosts, const int* n, std::vector<ImmPlan>& P) { return S->plan(c, nh, hosts, n, P, "immature store", "points"); }
static void imm_store_commit(ImmStore* S, std::vector<ImmPlan>& P) { S->commit(P); }
static void imm_store_abandon(ImmStore* S, std::vector<ImmPlan>& P) { S->abandon(P); }

// makeNewTraces into the store: the records of the selector engine (sdv_new_trace + sdv_immature_pt) with FullSystem.cpp:1313-1317 and :1080-1084 applied
struct DepositJob { const sdv_new_trace* t; const sdv_immature_pt* p; ImmRO* ro; ImmRW* rw; sdv_immature_meta* meta; int n; };
__global__ void __launch_bounds__(128) imm_deposit_kernel(const DepositJob* __restrict__ jobs) {
  const DepositJob J = jobs[blockIdx.y]; const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= J.n) return;
  const sdv_new_trace t = J.t[i]; sdv_immature_pt p = J.p[i];
  if (t.isFromSensor) { p.idepth_min = p.idepth_max = t.idepth_fromSensor; p.lastTraceStatus = IPS_SKIPPED; }   // idepth_max = idepth_fromSensor*1.0: the float survives the double product
  ImmRO a; ImmRW b; imm_split(p, a, b); J.ro[i] = a; J.rw[i] = b;
  sdv_immature_meta m; m.my_type = t.my_type; m.type = t.type; m.isFromSensor = t.isFromSensor; m.idepth_fromSensor = t.idepth_fromSensor; J.meta[i] = m;
}
int imm_store_deposit(sdv_ctx* c, int nj, const uint64_t* hosts, const int* n, const void* const* nt_dev, const void* const* imm_dev) {
  ImmStore* S = imm_store(c); std::vector<ImmPlan> P; { int rc = imm_store_plan(c, S, nj, hosts, n, P); if (rc) return rc; }
  std::vector<DepositJob> D(nj); int maxN = 0;
  for (int j = 0; j < nj; j++) { D[j] = DepositJob{(const sdv_new_trace*)nt_dev[j], (const sdv_immature_pt*)imm_dev[j], P[j].b.ro, P[j].b.rw, P[j].b.meta, n[j]}; maxN = std::max(maxN, n[j]); }
  if (maxN > 0) {
    if (c->scr.reserve(Scratch::need(nj, sizeof(DepositJob)), c->st)) { imm_store_abandon(S, P); return ctx_fail(c, SDV_ERR_CUDA, "immature store: deposit scratch"); }
    c->scr.reset(); DepositJob* dD = c->scr.take<DepositJob>(nj);
    if (cudaMemcpyAsync(dD, D.data(), nj*sizeof(DepositJob), cudaMemcpyHostToDevice, c->st) != cudaSuccess) { imm_store_abandon(S, P); CK(cudaGetLastError()); }
    imm_deposit_kernel<<<dim3((maxN + 127)/128, nj), 128, 0, c->st>>>(dD); c->launches += 1;
    if (cudaGetLastError() != cudaSuccess) { imm_store_abandon(S, P); return ctx_fail(c, SDV_ERR_CUDA, "immature store: deposit launch"); }
  }
  imm_store_commit(S, P);
  return SDV_OK;
}

// traceNewCoarse on the store: thread per point of all groups; the group is found by binary search over the groups' starts.  Calls trace_on, as imm_trace_kernel does.
struct TraceStoreGroupDev { const float* I0; float KRKi[9], Kt[3], aff[2]; int w, h; const ImmRO* ro; ImmRW* rw; };
__global__ void __launch_bounds__(128) imm_trace_store_kernel(const TraceStoreGroupDev* __restrict__ groups, const int* __restrict__ gbeg, int n_groups, int n, TraceSet S,
                                                              int* __restrict__ counts) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= n) return;
  int lo = 0, hi = n_groups - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (__ldg(gbeg + mid) <= i) lo = mid; else hi = mid - 1; }   // the last group starting at or before i: empty groups drop out
  const TraceStoreGroupDev& G = groups[lo]; const int k = i - __ldg(gbeg + lo);
  int st = G.rw[k].status;
  if (st != IPS_OOB) {                                                                   // traceOn returns an OOB point unchanged (ImmaturePoint.cpp:52)
    sdv_immature_pt p; imm_join(G.ro[k], G.rw[k], p);
    st = trace_on(p, G.I0, G.w, G.h, G.KRKi, G.Kt, G.aff, S);
    ImmRO a; ImmRW b; imm_split(p, a, b); G.rw[k] = b;
  }
  if (counts && (unsigned)st < 6u) atomicAdd(counts + 6*lo + st, 1);
}

// ---- activatePointsMT on the store (FullSystem.cpp:598-720), device side: the filter of :612-645, gathers, the post pass's compaction
struct ActHostDev { const ImmRO* ro; const ImmRW* rw; const sdv_immature_meta* meta; int newest, flagged; };
enum { ACT_KEEP = 0, ACT_DELETE = 1, ACT_CAND = 2 };
__device__ __forceinline__ int group_of_point(const int* __restrict__ gbeg, int n_groups, int i) {
  int lo = 0, hi = n_groups - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (__ldg(gbeg + mid) <= i) lo = mid; else hi = mid - 1; }
  return lo;
}
// per point: code = class | lastTraceStatus << 4, and for a candidate its cand4 row {u, v, 0.5f*(idepth_max+idepth_min), my_type}
__global__ void __launch_bounds__(128) imm_act_filter_kernel(const ActHostDev* __restrict__ hosts, const int* __restrict__ gbeg, int n_hosts, int n, float minTraceQuality,
                                                             int* __restrict__ code, float4* __restrict__ rows) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= n) return;
  const int g = group_of_point(gbeg, n_hosts, i); const ActHostDev& H = hosts[g]; const int k = i - __ldg(gbeg + g);
  const ImmRW b = H.rw[k]; const sdv_immature_meta m = H.meta[k]; int cls = ACT_KEEP;
  if (!(m.isFromSensor == 0 && H.newest)) {                                                  // :617 non-sensor points of the newest keyframe are skipped
    if (!isfinite(b.idepth_max) || b.status == IPS_OUTLIER) cls = ACT_DELETE;              // :621
    else {
      const bool canActivate = (b.status == IPS_GOOD || b.status == IPS_SKIPPED || b.status == IPS_BADCONDITION || b.status == IPS_OOB)
                               && b.lastTracePixelInterval < 8 && b.quality > minTraceQuality && (b.idepth_max+b.idepth_min) > 0;     // :630-636
      if (!canActivate) cls = (H.flagged || b.status == IPS_OOB) ? ACT_DELETE : ACT_KEEP;  // :641
      else { cls = ACT_CAND; const ImmRO a = H.ro[k]; rows[i] = make_float4(a.u, a.v, 0.5f*(b.idepth_max+b.idepth_min), m.my_type); }
    }
  }
  code[i] = cls | (b.status << 4);
}
__global__ void __launch_bounds__(128) imm_act_rows_kernel(const float4* __restrict__ rows, const int* __restrict__ idx, int n, float4* __restrict__ out) {
  const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k < n) out[k] = rows[idx[k]];
}
// toOptimize k = point idx[k] of the call's point numbering: its full record, meta and isFromSensor byte
__global__ void __launch_bounds__(128) imm_act_gather_kernel(const ActHostDev* __restrict__ hosts, const int* __restrict__ gbeg, int n_hosts, const int* __restrict__ idx, int n,
                                                             sdv_immature_pt* __restrict__ pts, sdv_immature_meta* __restrict__ meta, unsigned char* __restrict__ fs) {
  const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= n) return;
  const int i = idx[k], g = group_of_point(gbeg, n_hosts, i); const ActHostDev& H = hosts[g]; const int j = i - __ldg(gbeg + g);
  sdv_immature_pt p; imm_join(H.ro[j], H.rw[j], p); pts[k] = p; const sdv_immature_meta m = H.meta[j]; meta[k] = m; fs[k] = m.isFromSensor ? 1 : 0;
}
// compaction: the new block of host g is its old entries perm[nbeg[g] ..] in that order; pass 0 gathers into scratch, pass 1 writes back in place
struct ActBlockDev { ImmRO* ro; ImmRW* rw; sdv_immature_meta* meta; };
__global__ void __launch_bounds__(128) imm_act_permute_kernel(const ActBlockDev* __restrict__ blocks, const int* __restrict__ nbeg, int n_hosts, const int* __restrict__ perm, int n,
                                                              ImmRO* __restrict__ sro, ImmRW* __restrict__ srw, sdv_immature_meta* __restrict__ smeta, int pass) {
  const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= n) return;
  const int g = group_of_point(nbeg, n_hosts, k); const ActBlockDev& B = blocks[g]; const int j = k - __ldg(nbeg + g);
  if (pass == 0) { const int o = perm[k]; sro[k] = B.ro[o]; srw[k] = B.rw[o]; smeta[k] = B.meta[o]; }
  else { B.ro[j] = sro[k]; B.rw[j] = srw[k]; B.meta[j] = smeta[k]; }
}

// ---- the point loop of FullSystem::initializeFromInitializer (FullSystem.cpp:1176-1225) over the level-0 Pnt list of CoarseInitializer::setFirstFromLidar
// (CoarseInitializer.cpp:766-888): one CTA per job, the rows in chunks of blockDim in cloud order.  A Pnt is a row with status != 0 and (float)depth > 0 (the
// first block scan numbers them: draw k belongs to Pnt k); it is kept unless rand()/(float)RAND_MAX > keepPercentage, and if its ImmaturePoint at
// (int)(u+0.5f), (int)(v+0.5f) has a finite energyTH (the second scan numbers the kept points).  A point whose 8-pattern would read outside the frame's
// plane is not kept: the reference reads past its image there.
__device__ __forceinline__ int block_excl_scan(bool pred, int* wt /* 33 ints of shared memory */, int& total) {
  const unsigned b = __ballot_sync(0xffffffffu, pred); const int lane = threadIdx.x & 31, wid = threadIdx.x >> 5;
  if (lane == 0) wt[wid] = __popc(b);
  __syncthreads();
  if (threadIdx.x == 0) { int a = 0; for (int k = 0; k < (int)(blockDim.x >> 5); k++) { const int t = wt[k]; wt[k] = a; a += t; } wt[32] = a; }
  __syncthreads();
  const int r = wt[wid] + __popc(b & ((1u << lane) - 1u)); total = wt[32];
  __syncthreads();
  return r;
}
__global__ void __launch_bounds__(256) init_points_kernel(const InitPointsJob* __restrict__ jobs, TraceSet S) {
  const InitPointsJob& J = jobs[blockIdx.x]; __shared__ int wt[33];
  const int n = J.n, w = J.w, h = J.h;
  int nsel = 0;
  for (int base = 0; base < n; base += blockDim.x) { const int i = base + threadIdx.x;
    nsel += __syncthreads_count(i < n && J.map[i] != 0 && (float)J.cloud[3*i+2] > 0.f); }
  const float keepPercentage = J.desired / nsel;                                                  // setting_desiredPointDensity / numPoints[0]
  int kbase = 0, obase = 0;
  for (int base = 0; base < n; base += blockDim.x) { const int i = base + threadIdx.x;
    const bool sel = i < n && J.map[i] != 0 && (float)J.cloud[3*i+2] > 0.f;
    int tot; const int k = kbase + block_excl_scan(sel, wt, tot); kbase += tot;
    bool keep = false; sdv_immature_pt p; int pu = 0, pv = 0;
    if (sel && !((float)J.draws[k] / (float)2147483647 > keepPercentage)) {                      // glibc RAND_MAX
      pu = (int)((float)J.cloud[3*i] + 0.5f); pv = (int)((float)J.cloud[3*i+1] + 0.5f);
      keep = pu >= 0 && pu < w && pv >= 0 && pv < h && pu + (pv-2)*w >= 0 && pu + 1 + (pv+3)*w < w*h;
      if (keep) { imm_construct(J.I0, w, pu, pv, S, p); keep = isfinite(p.energyTH); }
    }
    const int o = obase + block_excl_scan(keep, wt, tot); obase += tot;
    if (keep) {
      const float mdepth = (float)J.cloud[3*i+2], midepth = 1 / mdepth;
      p.idepth_min = p.idepth_max = midepth; J.pts[o] = p;
      sdv_immature_meta m; m.my_type = (float)J.map[i]; m.type = 0; m.isFromSensor = 1; m.idepth_fromSensor = midepth; J.meta[o] = m;
      J.idepth[o] = midepth;
      J.splat4[4*o] = (float)pu; J.splat4[4*o+1] = (float)pv; J.splat4[4*o+2] = midepth; J.splat4[4*o+3] = 0.f; J.round[o] = 1;   // HdiF = 0, int(u + 0.5f)
      sdv_map_pt q; q.u = (float)pu; q.v = (float)pv; q.idepth = midepth; q.host = 0; q.type = 0; J.mp[o] = q;
    }
  }
  if (threadIdx.x == 0) { J.counts[0] = nsel; J.counts[1] = obase; }
}
int launch_init_points(sdv_ctx* c, int nj, const InitPointsJob* jobs_dev) {
  init_points_kernel<<<nj, 256, 0, c->st>>>(jobs_dev, trace_settings(c)); c->launches += 1;
  CK(cudaGetLastError()); return SDV_OK;
}
}  // namespace sdv

extern "C" {

int sdv_immature_init_cam(sdv_ctx* c, int cam, uint64_t host_frame, int n, const int32_t* uv, sdv_immature_pt* out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!uv || !out))) return SDV_ERR_ARG;
  { int rc = check_cams(c, 1, &cam, "immature_init", nullptr); if (rc) return rc; }
  if (n == 0) return SDV_OK;
  CK(cudaSetDevice(c->device));
  long long need_seq = 0; FrameDev* f; { int rc = job_frame(c, "immature_init", 0, host_frame, cam, -1, &need_seq, &f); if (rc) return rc; }
  const int w = c->cam_w[cam], h = c->cam_h[cam];
  for (int i = 0; i < n; i++) if (uv[2*i] < 2 || uv[2*i+1] < 2 || uv[2*i] >= w-3 || uv[2*i+1] >= h-3)     // the 8-pattern (+-2) and the +1 bilinear neighbour must stay inside the image
    return ctx_fail(c, SDV_ERR_ARG, "immature_init: candidate %d at (%d,%d) is closer than 3 px to the border", i, uv[2*i], uv[2*i+1]);
  { int rc = join_ingest_upto(c, need_seq); if (rc) return rc; }
  TRACE_SCRATCH(Scratch::need(2*(size_t)n, sizeof(int)) + Scratch::need(n, sizeof(sdv_immature_pt)), "immature_init");
  int* d_uv = c->scr.take<int>(2*(size_t)n); sdv_immature_pt* d_pts = c->scr.take<sdv_immature_pt>(n);
  CK(cudaMemcpyAsync(d_uv, uv, (size_t)n*2*sizeof(int), cudaMemcpyHostToDevice, c->st));
  imm_init_kernel<<<(n + 127)/128, 128, 0, c->st>>>(f->I0, w, h, n, d_uv, d_pts, trace_settings(c)); c->launches += 1;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, d_pts, (size_t)n*sizeof(sdv_immature_pt), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  return SDV_OK;
}
int sdv_immature_init(sdv_ctx* c, uint64_t host_frame, int n, const int32_t* uv, sdv_immature_pt* out) { return sdv_immature_init_cam(c, 0, host_frame, n, uv, out); }

int sdv_immature_trace_batch_cams(sdv_ctx* c, int n_groups, const uint64_t* frames, const int32_t* cams, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* aff2,
                                  sdv_immature_pt* pts_io, int32_t* status_out) { SDV_GUARD_TRK(c);
  if (!c || n_groups < 0 || (n_groups && (!frames || !pt_begin || !KRKi9 || !Kt3 || !aff2))) return SDV_ERR_ARG;
  if (n_groups == 0) return SDV_OK;
  { int rc = check_cams(c, n_groups, cams, "immature_trace", "group"); if (rc) return rc; }
  { int rc = check_offsets(c, n_groups, pt_begin, "immature_trace", "pt_begin"); if (rc) return rc; }
  const int n = pt_begin[n_groups];
  if (n == 0) return SDV_OK;
  if (!pts_io) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  std::vector<TraceGroupDev> G(n_groups); std::vector<int> gof(n); long long need_seq = 0;
  for (int g = 0; g < n_groups; g++) {
    const int cam = cams ? cams[g] : 0; FrameDev* f; { int rc = job_frame(c, "immature_trace", g, frames[g], cam, -1, &need_seq, &f); if (rc) return rc; }
    G[g].w = c->cam_w[cam]; G[g].h = c->cam_h[cam]; G[g].I0 = f->I0; for (int k = 0; k < 9; k++) G[g].KRKi[k] = KRKi9[9*g+k]; for (int k = 0; k < 3; k++) G[g].Kt[k] = Kt3[3*g+k]; G[g].aff[0] = aff2[2*g]; G[g].aff[1] = aff2[2*g+1];
    G[g].pt_begin = pt_begin[g]; G[g].pt_end = pt_begin[g+1];
    for (int i = pt_begin[g]; i < pt_begin[g+1]; i++) gof[i] = g;
  }
  { int rc = join_ingest_upto(c, need_seq); if (rc) return rc; }
  TRACE_SCRATCH(Scratch::need(n_groups, sizeof(TraceGroupDev)) + 2*Scratch::need(n, sizeof(int)) + Scratch::need(n, sizeof(sdv_immature_pt)), "immature_trace");
  TraceGroupDev* dG = c->scr.take<TraceGroupDev>(n_groups); int* dof = c->scr.take<int>(n); int* dst = c->scr.take<int>(n); sdv_immature_pt* dpts = c->scr.take<sdv_immature_pt>(n);
  CK(cudaMemcpyAsync(dG, G.data(), n_groups*sizeof(TraceGroupDev), cudaMemcpyHostToDevice, c->st));       // pageable sources: staged before the calls return
  CK(cudaMemcpyAsync(dof, gof.data(), (size_t)n*sizeof(int), cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(dpts, pts_io, (size_t)n*sizeof(sdv_immature_pt), cudaMemcpyHostToDevice, c->st));
  CK(cudaEventRecord(c->ev0, c->st));
  imm_trace_kernel<<<(n + 127)/128, 128, 0, c->st>>>(dG, dof, n, dpts, dst, trace_settings(c));
  c->launches += 1;
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev1, c->st));
  CK(cudaMemcpyAsync(pts_io, dpts, (size_t)n*sizeof(sdv_immature_pt), cudaMemcpyDeviceToHost, c->st));
  if (status_out) CK(cudaMemcpyAsync(status_out, dst, (size_t)n*sizeof(int), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  return SDV_OK;
}
int sdv_immature_trace_batch(sdv_ctx* c, int n_groups, const uint64_t* frames, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* aff2,
                             sdv_immature_pt* pts_io, int32_t* status_out) { return sdv_immature_trace_batch_cams(c, n_groups, frames, nullptr, pt_begin, KRKi9, Kt3, aff2, pts_io, status_out); }

int sdv_immature_optimize_batch_cams(sdv_ctx* c, int n_groups, const int32_t* pt_begin, const int32_t* tgt_begin, const uint64_t* target_frames, const float* pre14, const float* calib6,
                                     const int32_t* cams, int min_obs, const sdv_immature_pt* pts, const uint8_t* is_from_sensor, int res_stride, int32_t* status_out, float* idepth_out,
                                     int32_t* res_state_out) { SDV_GUARD_TRK(c);
  if (!c || n_groups < 0 || (n_groups && (!pt_begin || !tgt_begin || !target_frames || !pre14 || !calib6))) return SDV_ERR_ARG;
  if (n_groups == 0) return SDV_OK;
  { int rc = check_cams(c, n_groups, cams, "immature_optimize", "group"); if (rc) return rc; }
  { int rc = check_offsets(c, n_groups, pt_begin, "immature_optimize", "pt_begin"); if (rc) return rc; }
  { int rc = check_offsets(c, n_groups, tgt_begin, "immature_optimize", "tgt_begin"); if (rc) return rc; }
  for (int g = 0; g < n_groups; g++) { const int nres = tgt_begin[g+1] - tgt_begin[g]; if (nres > kOptMaxRes || nres > res_stride) return ctx_fail(c, SDV_ERR_ARG, "immature_optimize: group %d has %d targets (max %d, res_stride %d)", g, nres, kOptMaxRes, res_stride); }
  const int n = pt_begin[n_groups], nt = tgt_begin[n_groups];
  if (n == 0) return SDV_OK;
  if (!pts || !status_out || !idepth_out || !res_state_out || res_stride < 1) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  std::vector<OptGroupDev> G(n_groups); std::vector<OptTargetDev> T(nt); std::vector<int> gof(n); long long need_seq = 0;
  std::vector<int> cam_of(nt, 0); if (cams) for (int g = 0; g < n_groups; g++) for (int t = tgt_begin[g]; t < tgt_begin[g+1]; t++) cam_of[t] = cams[g];
  for (int t = 0; t < nt; t++) {
    FrameDev* f; { int rc = job_frame(c, "immature_optimize", t, target_frames[t], cam_of[t], -1, &need_seq, &f); if (rc) return rc; }
    T[t].I0 = f->I0; for (int k = 0; k < 9; k++) T[t].R[k] = pre14[14*t+k]; for (int k = 0; k < 3; k++) T[t].t[k] = pre14[14*t+9+k]; T[t].aff[0] = pre14[14*t+12]; T[t].aff[1] = pre14[14*t+13];
  }
  for (int g = 0; g < n_groups; g++) { G[g].tgt_begin = tgt_begin[g]; G[g].nres = tgt_begin[g+1] - tgt_begin[g]; const float* q = calib6 + 6*g;
    G[g].fxl = q[0]; G[g].fyl = q[1]; G[g].cxl = q[2]; G[g].cyl = q[3]; G[g].fxli = q[4]; G[g].fyli = q[5]; const int cam = cams ? cams[g] : 0; G[g].w = c->cam_w[cam]; G[g].h = c->cam_h[cam];
    for (int i = pt_begin[g]; i < pt_begin[g+1]; i++) gof[i] = g; }
  { int rc = join_ingest_upto(c, need_seq); if (rc) return rc; }
  TRACE_SCRATCH(Scratch::need(n_groups, sizeof(OptGroupDev)) + Scratch::need(nt, sizeof(OptTargetDev)) + 3*Scratch::need(n, sizeof(int)) + Scratch::need(n, 1)
                + Scratch::need((size_t)n*res_stride, sizeof(int)) + Scratch::need(n, sizeof(sdv_immature_pt)), "immature_optimize");
  OptGroupDev* dG = c->scr.take<OptGroupDev>(n_groups); OptTargetDev* dT = c->scr.take<OptTargetDev>(nt); int* dof = c->scr.take<int>(n); unsigned char* dfs = c->scr.take<unsigned char>(n);
  int* dst = c->scr.take<int>(n); float* did = c->scr.take<float>(n); int* drs = c->scr.take<int>((size_t)n*res_stride); sdv_immature_pt* dpts = c->scr.take<sdv_immature_pt>(n);
  CK(cudaMemcpyAsync(dG, G.data(), n_groups*sizeof(OptGroupDev), cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(dT, T.data(), nt*sizeof(OptTargetDev), cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(dof, gof.data(), (size_t)n*sizeof(int), cudaMemcpyHostToDevice, c->st));
  if (is_from_sensor) CK(cudaMemcpyAsync(dfs, is_from_sensor, (size_t)n, cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(dpts, pts, (size_t)n*sizeof(sdv_immature_pt), cudaMemcpyHostToDevice, c->st));
  CK(cudaEventRecord(c->ev0, c->st));
  imm_optimize_kernel<<<(n + 63)/64, 64, 0, c->st>>>(dG, dT, dof, n, dpts, is_from_sensor ? dfs : nullptr, min_obs, res_stride, dst, did, drs, c->set.huberTH);
  c->launches += 1;
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev1, c->st));
  CK(cudaMemcpyAsync(status_out, dst, (size_t)n*sizeof(int), cudaMemcpyDeviceToHost, c->st));
  CK(cudaMemcpyAsync(idepth_out, did, (size_t)n*sizeof(float), cudaMemcpyDeviceToHost, c->st));
  CK(cudaMemcpyAsync(res_state_out, drs, (size_t)n*res_stride*sizeof(int), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  return SDV_OK;
}
int sdv_immature_optimize_batch(sdv_ctx* c, int n_groups, const int32_t* pt_begin, const int32_t* tgt_begin, const uint64_t* target_frames, const float* pre14, const float* calib6,
                                int min_obs, const sdv_immature_pt* pts, const uint8_t* is_from_sensor, int res_stride, int32_t* status_out, float* idepth_out, int32_t* res_state_out) {
  return sdv_immature_optimize_batch_cams(c, n_groups, pt_begin, tgt_begin, target_frames, pre14, calib6, nullptr, min_obs, pts, is_from_sensor, res_stride, status_out, idepth_out, res_state_out);
}

// ---- the immature-point store
int sdv_immature_store_set(sdv_ctx* c, uint64_t host_frame, int n, const sdv_immature_pt* pts, const sdv_immature_meta* meta) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && !pts)) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  std::vector<ImmRO> a(n); std::vector<ImmRW> b(n); std::vector<sdv_immature_meta> m(n);
  for (int i = 0; i < n; i++) { imm_split(pts[i], a[i], b[i]); m[i] = meta ? meta[i] : sdv_immature_meta{1.f, -1, 0, 0.f}; }
  ImmStore* S = imm_store(c); std::vector<ImmPlan> P; { int rc = imm_store_plan(c, S, 1, &host_frame, &n, P); if (rc) return rc; }
  if (n) {                                                                               // pageable sources: staged before the copies return
    const ImmBlock& blk = P[0].b;
    if (cudaMemcpyAsync(blk.ro, a.data(), (size_t)n*sizeof(ImmRO), cudaMemcpyHostToDevice, c->st) != cudaSuccess ||
        cudaMemcpyAsync(blk.rw, b.data(), (size_t)n*sizeof(ImmRW), cudaMemcpyHostToDevice, c->st) != cudaSuccess ||
        cudaMemcpyAsync(blk.meta, m.data(), (size_t)n*sizeof(sdv_immature_meta), cudaMemcpyHostToDevice, c->st) != cudaSuccess) {
      imm_store_abandon(S, P); cudaGetLastError(); return ctx_fail(c, SDV_ERR_CUDA, "immature_store_set: copies");
    }
  }
  imm_store_commit(S, P);
  return SDV_OK;
}
int sdv_immature_store_count(sdv_ctx* c, int n, const uint64_t* hosts, int32_t* counts_out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!hosts || !counts_out))) return SDV_ERR_ARG;
  const ImmStore* S = (const ImmStore*)c->imm_store;
  for (int i = 0; i < n; i++) if (!S || !S->blocks.count(hosts[i])) return ctx_fail(c, SDV_ERR_NOFRAME, "immature_store_count: host %llu has no block", (unsigned long long)hosts[i]);
  for (int i = 0; i < n; i++) counts_out[i] = S->blocks.at(hosts[i]).n;
  return SDV_OK;
}
int sdv_immature_store_get(sdv_ctx* c, uint64_t host_frame, int cap, sdv_immature_pt* pts_out, sdv_immature_meta* meta_out, int32_t* n_out) { SDV_GUARD_TRK(c);
  if (!c || !n_out || cap < 0) return SDV_ERR_ARG;
  const ImmStore* S = (const ImmStore*)c->imm_store; auto it = S ? S->blocks.find(host_frame) : decltype(S->blocks.end())();
  if (!S || it == S->blocks.end()) return ctx_fail(c, SDV_ERR_NOFRAME, "immature_store_get: host %llu has no block", (unsigned long long)host_frame);
  const ImmBlock& blk = it->second; const int n = blk.n; *n_out = n;
  if (cap < n) return ctx_fail(c, SDV_ERR_CAPACITY, "immature_store_get: host %llu holds %d points, room for %d", (unsigned long long)host_frame, n, cap);
  if (n == 0 || (!pts_out && !meta_out)) return SDV_OK;
  CK(cudaSetDevice(c->device));
  std::vector<ImmRO> a(pts_out ? n : 0); std::vector<ImmRW> b(pts_out ? n : 0);
  if (pts_out) { CK(cudaMemcpyAsync(a.data(), blk.ro, (size_t)n*sizeof(ImmRO), cudaMemcpyDeviceToHost, c->st)); CK(cudaMemcpyAsync(b.data(), blk.rw, (size_t)n*sizeof(ImmRW), cudaMemcpyDeviceToHost, c->st)); }
  if (meta_out) CK(cudaMemcpyAsync(meta_out, blk.meta, (size_t)n*sizeof(sdv_immature_meta), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  if (pts_out) for (int i = 0; i < n; i++) imm_join(a[i], b[i], pts_out[i]);
  return SDV_OK;
}
int sdv_immature_store_drop(sdv_ctx* c, int n, const uint64_t* hosts) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && !hosts)) return SDV_ERR_ARG;
  ImmStore* S = (ImmStore*)c->imm_store;
  for (int i = 0; i < n; i++) if (!S || !S->blocks.count(hosts[i])) return ctx_fail(c, SDV_ERR_NOFRAME, "immature_store_drop: host %llu has no block", (unsigned long long)hosts[i]);
  for (int i = 0; i < n; i++) S->drop(hosts[i]);                                          // a host named twice is dropped once
  return SDV_OK;
}

int sdv_immature_trace_store_batch(sdv_ctx* c, int n_groups, const uint64_t* hosts, const uint64_t* frames, const int32_t* cams, const float* KRKi9, const float* Kt3,
                                   const float* aff2, int32_t* counts_out) { SDV_GUARD_TRK(c);
  if (!c || n_groups < 0 || (n_groups && (!hosts || !frames || !KRKi9 || !Kt3 || !aff2))) return SDV_ERR_ARG;
  if (n_groups == 0) return SDV_OK;
  { int rc = check_cams(c, n_groups, cams, "immature_trace_store", "group"); if (rc) return rc; }
  { int rc = check_distinct(c, n_groups, hosts, "immature_trace_store", "host"); if (rc) return rc; }
  const ImmStore* S = (const ImmStore*)c->imm_store;
  std::vector<TraceStoreGroupDev> G(n_groups); std::vector<int> gbeg(n_groups + 1, 0); std::vector<FrameDev*> F(n_groups); long long need_seq = 0;
  for (int g = 0; g < n_groups; g++) {
    auto bt = S ? S->blocks.find(hosts[g]) : decltype(S->blocks.end())();
    if (!S || bt == S->blocks.end()) return ctx_fail(c, SDV_ERR_NOFRAME, "immature_trace_store: host %llu has no block (group %d)", (unsigned long long)hosts[g], g);
    const int cam = cams ? cams[g] : 0; { int rc = job_frame(c, "immature_trace_store", g, frames[g], cam, -1, &need_seq, &F[g]); if (rc) return rc; }
    const ImmBlock& blk = bt->second; TraceStoreGroupDev& D = G[g];
    D.I0 = F[g]->I0; D.w = c->cam_w[cam]; D.h = c->cam_h[cam]; D.ro = blk.ro; D.rw = blk.rw;
    for (int k = 0; k < 9; k++) D.KRKi[k] = KRKi9[9*g+k]; for (int k = 0; k < 3; k++) D.Kt[k] = Kt3[3*g+k]; D.aff[0] = aff2[2*g]; D.aff[1] = aff2[2*g+1];
    gbeg[g+1] = gbeg[g] + blk.n;
  }
  const int n = gbeg[n_groups];
  if (n == 0) { if (counts_out) memset(counts_out, 0, (size_t)6*n_groups*sizeof(int32_t)); return SDV_OK; }
  CK(cudaSetDevice(c->device));
  { int rc = join_ingest_upto(c, need_seq); if (rc) return rc; }
  TRACE_SCRATCH(Scratch::need(n_groups, sizeof(TraceStoreGroupDev)) + Scratch::need(n_groups + 1, sizeof(int)) + Scratch::need((size_t)6*n_groups, sizeof(int)), "immature_trace_store");
  TraceStoreGroupDev* dG = c->scr.take<TraceStoreGroupDev>(n_groups); int* dgb = c->scr.take<int>(n_groups + 1); int* dcnt = c->scr.take<int>((size_t)6*n_groups);
  CK(cudaMemcpyAsync(dG, G.data(), n_groups*sizeof(TraceStoreGroupDev), cudaMemcpyHostToDevice, c->st));       // pageable sources: staged before the calls return
  CK(cudaMemcpyAsync(dgb, gbeg.data(), (n_groups + 1)*sizeof(int), cudaMemcpyHostToDevice, c->st));
  if (counts_out) CK(cudaMemsetAsync(dcnt, 0, (size_t)6*n_groups*sizeof(int), c->st));
  CK(cudaEventRecord(c->ev0, c->st));
  imm_trace_store_kernel<<<(n + 127)/128, 128, 0, c->st>>>(dG, dgb, n_groups, n, trace_settings(c), counts_out ? dcnt : nullptr);
  c->launches += 1;
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev1, c->st));
  if (counts_out) {
    CK(cudaMemcpyAsync(counts_out, dcnt, (size_t)6*n_groups*sizeof(int), cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st)); CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  } else {                                                                               // returns with the kernel pending: a re-ingest or release of a traced frame waits for it
    if (!c->ev_trk_async) CK(cudaEventCreateWithFlags(&c->ev_trk_async, cudaEventDisableTiming));
    CK(cudaEventRecord(c->ev_trk_async, c->st));
    for (FrameDev* f : F) f->trk_async = true;
  }
  return SDV_OK;
}

}  // extern "C"

extern "C" {
int sdv_activate_points_store_batch(sdv_ctx* c, int n, const int32_t* host_begin, const uint64_t* hosts, const int32_t* flagged, const float* cKRKi9, const float* cKt3,
                                    const int32_t* src_host_begin, const int32_t* src_pt_begin, const float* KRKi9, const float* Kt3, const float* uvid, const float* min_act_dist,
                                    const float* pre14, const float* calib6, const int32_t* cams, int cap, int32_t* n_act_out, int32_t* act_host, int32_t* act_idx,
                                    sdv_immature_pt* act_pts, sdv_immature_meta* act_meta, float* act_idepth, int32_t* act_res_state, int32_t* counts_out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || cap < 0 || (n && (!host_begin || !hosts || !flagged || !cKRKi9 || !cKt3 || !src_host_begin || !src_pt_begin || !min_act_dist || !pre14 || !calib6 || !n_act_out)))
    return SDV_ERR_ARG;
  if (n == 0) return SDV_OK;
  if (cap > 0 && (!act_host || !act_idx || !act_pts || !act_meta || !act_idepth || !act_res_state)) return SDV_ERR_ARG;
  if (!c->sel) return ctx_fail(c, SDV_ERR_STATE, "activate_points_store: sdv_selector_init has not been called");
  { int rc = check_cams(c, n, cams, "activate_points_store", "sequence"); if (rc) return rc; }
  { int rc = check_offsets(c, n, host_begin, "activate_points_store", "host_begin"); if (rc) return rc; }
  for (int j = 0; j < n; j++) { const int nH = host_begin[j+1] - host_begin[j];
    if (nH < 1 || nH > 16 || nH - 1 > SDV_MAX_FRAMES_WINDOW) return ctx_fail(c, SDV_ERR_ARG, "activate_points_store: sequence %d has %d keyframes (1..16, at most %d targets)", j, nH, SDV_MAX_FRAMES_WINDOW); }
  const int NH = host_begin[n]; const ImmStore* S = (const ImmStore*)c->imm_store;
  { int rc = check_distinct(c, NH, hosts, "activate_points_store", "host"); if (rc) return rc; }
  std::vector<int> seq_of(NH), gbeg(NH + 1, 0), pre_begin(n + 1, 0); std::vector<FrameDev*> F(NH); std::vector<ActHostDev> HD(NH); long long need_seq = 0;
  for (int j = 0; j < n; j++) { const int nH = host_begin[j+1] - host_begin[j]; pre_begin[j+1] = pre_begin[j] + nH*(nH - 1);
    for (int g = host_begin[j]; g < host_begin[j+1]; g++) { seq_of[g] = j;
      auto bt = S ? S->blocks.find(hosts[g]) : decltype(S->blocks.end())();
      if (!S || bt == S->blocks.end()) return ctx_fail(c, SDV_ERR_NOFRAME, "activate_points_store: host %llu has no block", (unsigned long long)hosts[g]);
      { int rc = job_frame(c, "activate_points_store", g, hosts[g], cams ? cams[j] : 0, -1, &need_seq, &F[g]); if (rc) return rc; }
      const ImmBlock& blk = bt->second; HD[g] = ActHostDev{blk.ro, blk.rw, blk.meta, g == host_begin[j+1] - 1 ? 1 : 0, flagged[g] ? 1 : 0}; gbeg[g+1] = gbeg[g] + blk.n; } }
  const int N = gbeg[NH];
  CK(cudaSetDevice(c->device));
  { int rc = join_ingest_upto(c, need_seq); if (rc) return rc; }
  // scratch, sized once for every phase
  const size_t nN = (size_t)std::max(N, 1), R = SDV_MAX_FRAMES_WINDOW;
  TRACE_SCRATCH(Scratch::need(NH, sizeof(ActHostDev)) + 2*Scratch::need(NH + 1, sizeof(int)) + 6*Scratch::need(nN, sizeof(int)) + 2*Scratch::need(nN, sizeof(float4))
                + Scratch::need(NH, sizeof(OptGroupDev)) + Scratch::need(pre_begin[n], sizeof(OptTargetDev)) + Scratch::need(nN, sizeof(sdv_immature_pt)) + 2*Scratch::need(nN, sizeof(sdv_immature_meta))
                + Scratch::need(nN, 1) + Scratch::need(nN*R, sizeof(int)) + Scratch::need(NH, sizeof(ActBlockDev)) + Scratch::need(nN, sizeof(ImmRO)) + Scratch::need(nN, sizeof(ImmRW)), "activate_points_store");
  Scratch& D = c->scr;
  ActHostDev* dHD = D.take<ActHostDev>(NH); int* dGB = D.take<int>(NH + 1); int* dcode = D.take<int>(nN); float4* drows = D.take<float4>(nN); float4* dc4 = D.take<float4>(nN);
  int* didx = D.take<int>(nN); OptGroupDev* dOG = D.take<OptGroupDev>(NH); OptTargetDev* dOT = D.take<OptTargetDev>(pre_begin[n]); int* dgof = D.take<int>(nN);
  sdv_immature_pt* dpts = D.take<sdv_immature_pt>(nN); sdv_immature_meta* dmeta = D.take<sdv_immature_meta>(nN); unsigned char* dfs = D.take<unsigned char>(nN); int* dst = D.take<int>(nN);
  float* did = D.take<float>(nN); int* drs = D.take<int>(nN*R); int* dperm = D.take<int>(nN); int* dnb = D.take<int>(NH + 1); ActBlockDev* dBD = D.take<ActBlockDev>(NH);
  ImmRO* dsro = D.take<ImmRO>(nN); ImmRW* dsrw = D.take<ImmRW>(nN); sdv_immature_meta* dsme = D.take<sdv_immature_meta>(nN);
  // (1) the filter of :612-645 on the device; the host reads one code per point back (class and status, 4 bytes), no record
  std::vector<int> code(nN, 0);
  CK(cudaMemcpyAsync(dHD, HD.data(), NH*sizeof(ActHostDev), cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(dGB, gbeg.data(), (NH + 1)*sizeof(int), cudaMemcpyHostToDevice, c->st));
  if (N) { imm_act_filter_kernel<<<(N + 127)/128, 128, 0, c->st>>>(dHD, dGB, NH, N, 3.0f /* setting_minTraceQuality, settings.cpp:131 */, dcode, drows);
           c->launches += 1; CK(cudaGetLastError());
           CK(cudaMemcpyAsync(code.data(), dcode, (size_t)N*4, cudaMemcpyDeviceToHost, c->st)); }
  CK(cudaStreamSynchronize(c->st));
  // (2) makeDistanceMap + the walk (:597-671) over the candidates, rows gathered on the device in host-then-point order
  std::vector<int> cidx, cand_begin(NH + 1, 0);
  for (int g = 0; g < NH; g++) { for (int i = gbeg[g]; i < gbeg[g+1]; i++) if ((code[i] & 3) == ACT_CAND) cidx.push_back(i); cand_begin[g+1] = (int)cidx.size(); }
  const int NC = (int)cidx.size(); std::vector<int32_t> decision(std::max(NC, 1), 0);
  if (NC) { CK(cudaMemcpyAsync(didx, cidx.data(), (size_t)NC*4, cudaMemcpyHostToDevice, c->st));
            imm_act_rows_kernel<<<(NC + 127)/128, 128, 0, c->st>>>(drows, didx, NC, dc4); c->launches += 1; CK(cudaGetLastError()); }
  { int rc = sel_activate_select(c, n, src_host_begin, src_pt_begin, KRKi9, Kt3, uvid, host_begin, cand_begin.data(), cKRKi9, cKt3, nullptr, (const float*)dc4, min_act_dist, cams,
                                 decision.data(), nullptr); if (rc) return rc; }
  // (3) optimizeImmaturePoint (min_obs 1) on the accepted candidates, toOptimize order, read from the store
  std::vector<int> oidx, ohost; std::vector<int> opt_of(NC, -1);
  for (int k = 0; k < NC; k++) if (decision[k] == 1) { opt_of[k] = (int)oidx.size(); oidx.push_back(cidx[k]); }
  const int NO = (int)oidx.size(); std::vector<int> gof(std::max(NO, 1)); std::vector<OptGroupDev> OG(NH); std::vector<OptTargetDev> OT(pre_begin[n]);
  { int k = 0; for (int g = 0; g < NH; g++) while (k < NO && oidx[k] < gbeg[g+1]) gof[k++] = g; }
  for (int g = 0; g < NH; g++) { const int j = seq_of[g], h0 = host_begin[j], nH = host_begin[j+1] - h0, h = g - h0, cam = cams ? cams[j] : 0; const float* q = calib6 + 6*j;
    OptGroupDev& G = OG[g]; G.tgt_begin = pre_begin[j] + h*(nH - 1); G.nres = nH - 1; G.fxl = q[0]; G.fyl = q[1]; G.cxl = q[2]; G.cyl = q[3]; G.fxli = q[4]; G.fyli = q[5]; G.w = c->cam_w[cam]; G.h = c->cam_h[cam];
    int t = 0; for (int tg = h0; tg < h0 + nH; tg++) { if (tg == g) continue; OptTargetDev& T = OT[G.tgt_begin + t]; const float* r = pre14 + 14*(size_t)(G.tgt_begin + t); t++;
      T.I0 = F[tg]->I0; for (int e = 0; e < 9; e++) T.R[e] = r[e]; for (int e = 0; e < 3; e++) T.t[e] = r[9+e]; T.aff[0] = r[12]; T.aff[1] = r[13]; } }
  std::vector<sdv_immature_pt> opts(NO); std::vector<sdv_immature_meta> ometa(NO); std::vector<int> ost(NO); std::vector<float> oid(NO); std::vector<int> ors((size_t)NO*R);
  if (NO) {
    CK(cudaMemcpyAsync(didx, oidx.data(), (size_t)NO*4, cudaMemcpyHostToDevice, c->st));
    CK(cudaMemcpyAsync(dOG, OG.data(), NH*sizeof(OptGroupDev), cudaMemcpyHostToDevice, c->st));
    if (!OT.empty()) CK(cudaMemcpyAsync(dOT, OT.data(), OT.size()*sizeof(OptTargetDev), cudaMemcpyHostToDevice, c->st));
    CK(cudaMemcpyAsync(dgof, gof.data(), (size_t)NO*4, cudaMemcpyHostToDevice, c->st));
    imm_act_gather_kernel<<<(NO + 127)/128, 128, 0, c->st>>>(dHD, dGB, NH, didx, NO, dpts, dmeta, dfs);
    imm_optimize_kernel<<<(NO + 63)/64, 64, 0, c->st>>>(dOG, dOT, dgof, NO, dpts, dfs, 1, (int)R, dst, did, drs, c->set.huberTH);
    c->launches += 2; CK(cudaGetLastError());
    CK(cudaMemcpyAsync(ost.data(), dst, (size_t)NO*4, cudaMemcpyDeviceToHost, c->st)); CK(cudaMemcpyAsync(oid.data(), did, (size_t)NO*4, cudaMemcpyDeviceToHost, c->st));
    CK(cudaMemcpyAsync(ors.data(), drs, (size_t)NO*R*4, cudaMemcpyDeviceToHost, c->st));
    CK(cudaMemcpyAsync(opts.data(), dpts, (size_t)NO*sizeof(sdv_immature_pt), cudaMemcpyDeviceToHost, c->st));
    CK(cudaMemcpyAsync(ometa.data(), dmeta, (size_t)NO*16, cudaMemcpyDeviceToHost, c->st));
    CK(cudaStreamSynchronize(c->st));
  }
  std::vector<int> nact(n, 0); int total = 0; for (int k = 0; k < NO; k++) if (ost[k] == 1) { nact[seq_of[gof[k]]]++; total++; }
  if (total > cap) return ctx_fail(c, SDV_ERR_CAPACITY, "activate_points_store: %d points activated, room for %d", total, cap);    // nothing has changed yet
  // (4) the post pass (:683-707) and the swap-with-back compaction of every host's vector (:709-720)
  std::vector<char> dead(nN, 0);
  for (int i = 0; i < N; i++) if ((code[i] & 3) == ACT_DELETE) dead[i] = 1;
  for (int k = 0; k < NC; k++) if (decision[k] == -1) dead[cidx[k]] = 1;
  for (int k = 0; k < NO; k++) if (ost[k] == 1 || ost[k] == -1 || (code[oidx[k]] >> 4) == IPS_OOB) dead[oidx[k]] = 1;
  std::vector<int> perm, nbeg(NH + 1, 0); std::vector<ActBlockDev> BD(NH);
  for (int g = 0; g < NH; g++) { std::vector<int> v(gbeg[g+1] - gbeg[g]); for (size_t i = 0; i < v.size(); i++) v[i] = (int)i;
    for (int i = 0; i < (int)v.size(); i++) if (dead[gbeg[g] + v[i]]) { v[i] = v.back(); v.pop_back(); i--; }
    perm.insert(perm.end(), v.begin(), v.end()); nbeg[g+1] = (int)perm.size(); BD[g] = ActBlockDev{const_cast<ImmRO*>(HD[g].ro), const_cast<ImmRW*>(HD[g].rw), const_cast<sdv_immature_meta*>(HD[g].meta)}; }
  const int NP = (int)perm.size();
  if (NP) {
    CK(cudaMemcpyAsync(dperm, perm.data(), (size_t)NP*4, cudaMemcpyHostToDevice, c->st)); CK(cudaMemcpyAsync(dnb, nbeg.data(), (NH + 1)*sizeof(int), cudaMemcpyHostToDevice, c->st));
    CK(cudaMemcpyAsync(dBD, BD.data(), NH*sizeof(ActBlockDev), cudaMemcpyHostToDevice, c->st));
    for (int pass = 0; pass < 2; pass++)
      imm_act_permute_kernel<<<(NP + 127)/128, 128, 0, c->st>>>(dBD, dnb, NH, dperm, NP, dsro, dsrw, dsme, pass);
    c->launches += 2; CK(cudaGetLastError());
  }
  ImmStore* SW = (ImmStore*)c->imm_store;
  for (int g = 0; g < NH; g++) { SW->blocks[hosts[g]].n = nbeg[g+1] - nbeg[g]; if (counts_out) counts_out[g] = nbeg[g+1] - nbeg[g]; }
  // activated points, toOptimize order: what new PointHessian(ph) copies, its idepth and the residual states of FullSystemOptPoint.cpp:157-177
  int o = 0;
  for (int k = 0; k < NO; k++) if (ost[k] == 1) { const int g = gof[k];
    act_host[o] = g; act_idx[o] = oidx[k] - gbeg[g]; act_pts[o] = opts[k]; act_meta[o] = ometa[k]; act_idepth[o] = oid[k];
    for (size_t r = 0; r < R; r++) act_res_state[(size_t)o*R + r] = ors[(size_t)k*R + r];
    o++; }
  for (int j = 0; j < n; j++) n_act_out[j] = nact[j];
  CK(cudaStreamSynchronize(c->st));
  return SDV_OK;
}
}  // extern "C"
