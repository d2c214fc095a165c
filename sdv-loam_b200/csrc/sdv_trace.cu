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
#include <vector>
#include "sdv_ctx.cuh"

using namespace sdv;
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return ctx_fail(c, SDV_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } while (0)

namespace sdv {

__constant__ int kTracePat[8][2] = {{0,-2},{-1,-1},{1,-1},{-2,0},{0,0},{2,0},{-1,1},{0,2}};   // staticPattern[8], util/settings.cpp:250
enum { IPS_GOOD = 0, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED };

struct TraceGroupDev { const float* I0; float KRKi[9], Kt[3], aff[2]; int pt_begin, pt_end; int w, h; };   // one (host keyframe, traced frame) pair; w, h: its camera's size
struct TraceSet { float outlierTH, outlierTHSumComponent, overallEnergyTHWeight, huberTH, maxPixSearch; int minTraceTestRadius; float stepsize; int GNIterations;
                  float GNThreshold, extraSlackOnTH, slackInterval, minImprovementFactor; };

// dIp[0][idx] = {I, dx, dy} from the planar level-0 plane: central differences, zero on the first / last image row (flat-index rule), non-finite -> 0
__device__ __forceinline__ void texel0(const float* __restrict__ I, int idx, int w, int h, float& c, float& dx, float& dy) {
  c = __ldg(I + idx); dx = 0.f; dy = 0.f;
  if (idx >= w && idx < w*(h-1)) {
    dx = 0.5f*(__ldg(I + idx+1) - __ldg(I + idx-1));
    dy = 0.5f*(__ldg(I + idx+w) - __ldg(I + idx-w));
    if (!isfinite(dx)) dx = 0;
    if (!isfinite(dy)) dy = 0;
  }
}
__device__ __forceinline__ float interp31(const float* __restrict__ I, float x, float y, int w) {   // getInterpolatedElement31, util/globalFuncs.h:102-116
  const int ix = (int)x, iy = (int)y; const float dx = x - ix, dy = y - iy, dxdy = dx*dy; const float* bp = I + ix + iy*w;
  return dxdy*__ldg(bp+1+w) + (dy-dxdy)*__ldg(bp+w) + (dx-dxdy)*__ldg(bp+1) + (1-dx-dy+dxdy)*__ldg(bp);
}
__device__ __forceinline__ void interp33(const float* __restrict__ I, float x, float y, int w, int h, float out[3]) {   // getInterpolatedElement33, :51-65
  const int ix = (int)x, iy = (int)y; const float dx = x - ix, dy = y - iy, dxdy = dx*dy; const int b = ix + iy*w;
  float c11[3], c01[3], c10[3], c00[3];
  texel0(I, b+1+w, w, h, c11[0], c11[1], c11[2]); texel0(I, b+w, w, h, c01[0], c01[1], c01[2]); texel0(I, b+1, w, h, c10[0], c10[1], c10[2]); texel0(I, b, w, h, c00[0], c00[1], c00[2]);
  const float w11 = dxdy, w01 = dy-dxdy, w10 = dx-dxdy, w00 = 1-dx-dy+dxdy;
#pragma unroll
  for (int k = 0; k < 3; k++) out[k] = w11*c11[k] + w01*c01[k] + w10*c10[k] + w00*c00[k];
}

// ---- ImmaturePoint::ImmaturePoint (ImmaturePoint.cpp:8-36): one thread per candidate
__global__ void __launch_bounds__(128) imm_init_kernel(const float* __restrict__ I0, int w, int h, int n, const int* __restrict__ uv, sdv_immature_pt* __restrict__ out, TraceSet S) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= n) return;
  sdv_immature_pt p;
  p.u = (float)uv[2*i]; p.v = (float)uv[2*i+1]; p.idepth_min = 0; p.idepth_max = NAN; p.lastTraceStatus = IPS_UNINITIALIZED;
  for (int k = 0; k < 4; k++) p.gradH[k] = 0;
  p.lastTraceUV[0] = p.lastTraceUV[1] = 0; p.quality = 10000; p.lastTracePixelInterval = 0; p.energyTH = NAN;
  for (int k = 0; k < 8; k++) { p.color[k] = 0; p.weights[k] = 0; }
  bool finite = true;
  for (int idx = 0; idx < 8 && finite; idx++) {
    const float x = p.u + kTracePat[idx][0], y = p.v + kTracePat[idx][1];
    const int ix = (int)x, iy = (int)y; const float* bp = I0 + ix + iy*w;                       // getInterpolatedElement33BiLin, util/globalFuncs.h:142-164
    const float tl = __ldg(bp), tr = __ldg(bp+1), bl = __ldg(bp+w), br = __ldg(bp+w+1);
    const float dx = x - ix, dy = y - iy;
    const float topInt = dx*tr + (1-dx)*tl, botInt = dx*br + (1-dx)*bl, leftInt = dy*bl + (1-dy)*tl, rightInt = dy*br + (1-dy)*tr;
    const float c0 = dx*rightInt + (1-dx)*leftInt, gx = rightInt-leftInt, gy = botInt-topInt;
    p.color[idx] = c0;
    if (!isfinite(c0)) { finite = false; break; }
    p.gradH[0] += gx*gx; p.gradH[1] += gx*gy; p.gradH[2] += gy*gx; p.gradH[3] += gy*gy;
    p.weights[idx] = sqrtf(S.outlierTHSumComponent / (S.outlierTHSumComponent + (gx*gx + gy*gy)));
  }
  if (finite) { p.energyTH = 8*S.outlierTH; p.energyTH *= S.overallEnergyTHWeight*S.overallEnergyTHWeight; }
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
  for (int idx = 0; idx < 8; idx++) { const float px = (float)kTracePat[idx][0], py = (float)kTracePat[idx][1]; rpx[idx] = R00*px + R01*py; rpy[idx] = R10*px + R11*py; }
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
    const int dx = kTracePat[idx][0], dy = kTracePat[idx][1];
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
static int trace_scratch(sdv_ctx* c, size_t bytes) {
  if (bytes <= c->trace_cap) return SDV_OK;
  CK(cudaStreamSynchronize(c->st)); cudaFree(c->trace_dev); c->trace_dev = nullptr; c->trace_cap = 0;
  CK(cudaMalloc(&c->trace_dev, bytes + bytes/2)); c->trace_cap = bytes + bytes/2; return SDV_OK;
}
}  // namespace sdv

extern "C" {

int sdv_immature_init_cam(sdv_ctx* c, int cam, uint64_t host_frame, int n, const int32_t* uv, sdv_immature_pt* out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!uv || !out))) return SDV_ERR_ARG;
  if (cam < 0 || cam >= SDV_MAX_CAMERAS) return ctx_fail(c, SDV_ERR_ARG, "immature_init: camera %d (valid: 0..%d)", cam, SDV_MAX_CAMERAS - 1);
  if (n == 0) return SDV_OK;
  CK(cudaSetDevice(c->device));
  auto it = c->frame_index.find(host_frame); if (it == c->frame_index.end()) return ctx_fail(c, SDV_ERR_NOFRAME, "immature_init: unknown host frame %llu", (unsigned long long)host_frame);
  { int rcs = check_frame_cam(c, c->frames[it->second], cam, "immature_init"); if (rcs) return rcs; }
  const int w = c->cam_w[cam], h = c->cam_h[cam];
  for (int i = 0; i < n; i++) if (uv[2*i] < 2 || uv[2*i+1] < 2 || uv[2*i] >= w-3 || uv[2*i+1] >= h-3)     // the 8-pattern (+-2) and the +1 bilinear neighbour must stay inside the image
    return ctx_fail(c, SDV_ERR_ARG, "immature_init: candidate %d at (%d,%d) is closer than 3 px to the border", i, uv[2*i], uv[2*i+1]);
  FrameDev& f = c->frames[it->second];
  { int rc = join_ingest_upto(c, f.ingest_seq); if (rc) return rc; }
  const size_t o_pts = (size_t)n*2*sizeof(int), bytes = o_pts + (size_t)n*sizeof(sdv_immature_pt);
  { int rc = trace_scratch(c, bytes); if (rc) return rc; }
  char* d = (char*)c->trace_dev;
  CK(cudaMemcpyAsync(d, uv, o_pts, cudaMemcpyHostToDevice, c->st));
  imm_init_kernel<<<(n + 127)/128, 128, 0, c->st>>>(f.I0, w, h, n, (const int*)d, (sdv_immature_pt*)(d + o_pts), trace_settings(c)); c->launches += 1;
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(out, d + o_pts, (size_t)n*sizeof(sdv_immature_pt), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  return SDV_OK;
}
int sdv_immature_init(sdv_ctx* c, uint64_t host_frame, int n, const int32_t* uv, sdv_immature_pt* out) { return sdv_immature_init_cam(c, 0, host_frame, n, uv, out); }

int sdv_immature_trace_batch_cams(sdv_ctx* c, int n_groups, const uint64_t* frames, const int32_t* cams, const int32_t* pt_begin, const float* KRKi9, const float* Kt3, const float* aff2,
                                  sdv_immature_pt* pts_io, int32_t* status_out) { SDV_GUARD_TRK(c);
  if (!c || n_groups < 0 || (n_groups && (!frames || !pt_begin || !KRKi9 || !Kt3 || !aff2))) return SDV_ERR_ARG;
  if (n_groups == 0) return SDV_OK;
  if (cams) for (int g = 0; g < n_groups; g++) if (cams[g] < 0 || cams[g] >= SDV_MAX_CAMERAS) return ctx_fail(c, SDV_ERR_ARG, "immature_trace: group %d names camera %d (valid: 0..%d)", g, cams[g], SDV_MAX_CAMERAS - 1);
  if (pt_begin[0] != 0) return ctx_fail(c, SDV_ERR_ARG, "immature_trace: pt_begin[0] must be 0");
  for (int g = 0; g < n_groups; g++) if (pt_begin[g+1] < pt_begin[g]) return ctx_fail(c, SDV_ERR_ARG, "immature_trace: pt_begin is not ascending at group %d", g);
  const int n = pt_begin[n_groups];
  if (n == 0) return SDV_OK;
  if (!pts_io) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  std::vector<TraceGroupDev> G(n_groups); std::vector<int> gof(n); long long need_seq = 0;
  for (int g = 0; g < n_groups; g++) {
    auto it = c->frame_index.find(frames[g]); if (it == c->frame_index.end()) return ctx_fail(c, SDV_ERR_NOFRAME, "immature_trace: unknown frame %llu (group %d)", (unsigned long long)frames[g], g);
    const int cam = cams ? cams[g] : 0; const FrameDev& f = c->frames[it->second]; { int rcs = check_frame_cam(c, f, cam, "immature_trace"); if (rcs) return rcs; }
    if (f.ingest_seq > need_seq) need_seq = f.ingest_seq;
    G[g].w = c->cam_w[cam]; G[g].h = c->cam_h[cam]; G[g].I0 = f.I0; for (int k = 0; k < 9; k++) G[g].KRKi[k] = KRKi9[9*g+k]; for (int k = 0; k < 3; k++) G[g].Kt[k] = Kt3[3*g+k]; G[g].aff[0] = aff2[2*g]; G[g].aff[1] = aff2[2*g+1];
    G[g].pt_begin = pt_begin[g]; G[g].pt_end = pt_begin[g+1];
    for (int i = pt_begin[g]; i < pt_begin[g+1]; i++) gof[i] = g;
  }
  { int rc = join_ingest_upto(c, need_seq); if (rc) return rc; }
  const size_t o_g = 0, o_of = (n_groups*sizeof(TraceGroupDev) + 15) & ~(size_t)15, o_st = o_of + (((size_t)n*sizeof(int) + 15) & ~(size_t)15),
               o_pts = o_st + (((size_t)n*sizeof(int) + 15) & ~(size_t)15), bytes = o_pts + (size_t)n*sizeof(sdv_immature_pt);
  { int rc = trace_scratch(c, bytes); if (rc) return rc; }
  char* d = (char*)c->trace_dev;
  CK(cudaMemcpyAsync(d + o_g, G.data(), n_groups*sizeof(TraceGroupDev), cudaMemcpyHostToDevice, c->st));       // pageable sources: staged before the calls return
  CK(cudaMemcpyAsync(d + o_of, gof.data(), (size_t)n*sizeof(int), cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(d + o_pts, pts_io, (size_t)n*sizeof(sdv_immature_pt), cudaMemcpyHostToDevice, c->st));
  CK(cudaEventRecord(c->ev0, c->st));
  imm_trace_kernel<<<(n + 127)/128, 128, 0, c->st>>>((const TraceGroupDev*)(d + o_g), (const int*)(d + o_of), n, (sdv_immature_pt*)(d + o_pts), (int*)(d + o_st), trace_settings(c));
  c->launches += 1;
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev1, c->st));
  CK(cudaMemcpyAsync(pts_io, d + o_pts, (size_t)n*sizeof(sdv_immature_pt), cudaMemcpyDeviceToHost, c->st));
  if (status_out) CK(cudaMemcpyAsync(status_out, d + o_st, (size_t)n*sizeof(int), cudaMemcpyDeviceToHost, c->st));
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
  if (cams) for (int g = 0; g < n_groups; g++) if (cams[g] < 0 || cams[g] >= SDV_MAX_CAMERAS) return ctx_fail(c, SDV_ERR_ARG, "immature_optimize: group %d names camera %d (valid: 0..%d)", g, cams[g], SDV_MAX_CAMERAS - 1);
  if (pt_begin[0] != 0 || tgt_begin[0] != 0) return ctx_fail(c, SDV_ERR_ARG, "immature_optimize: pt_begin[0] and tgt_begin[0] must be 0");
  for (int g = 0; g < n_groups; g++) { if (pt_begin[g+1] < pt_begin[g] || tgt_begin[g+1] < tgt_begin[g]) return ctx_fail(c, SDV_ERR_ARG, "immature_optimize: offsets not ascending at group %d", g);
    const int nres = tgt_begin[g+1] - tgt_begin[g]; if (nres > kOptMaxRes || nres > res_stride) return ctx_fail(c, SDV_ERR_ARG, "immature_optimize: group %d has %d targets (max %d, res_stride %d)", g, nres, kOptMaxRes, res_stride); }
  const int n = pt_begin[n_groups], nt = tgt_begin[n_groups];
  if (n == 0) return SDV_OK;
  if (!pts || !status_out || !idepth_out || !res_state_out || res_stride < 1) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  std::vector<OptGroupDev> G(n_groups); std::vector<OptTargetDev> T(nt); std::vector<int> gof(n); long long need_seq = 0;
  std::vector<int> cam_of(nt, 0); if (cams) for (int g = 0; g < n_groups; g++) for (int t = tgt_begin[g]; t < tgt_begin[g+1]; t++) cam_of[t] = cams[g];
  for (int t = 0; t < nt; t++) {
    auto it = c->frame_index.find(target_frames[t]); if (it == c->frame_index.end()) return ctx_fail(c, SDV_ERR_NOFRAME, "immature_optimize: unknown target frame %llu", (unsigned long long)target_frames[t]);
    const FrameDev& f = c->frames[it->second]; { int rcs = check_frame_cam(c, f, cam_of[t], "immature_optimize"); if (rcs) return rcs; }
    if (f.ingest_seq > need_seq) need_seq = f.ingest_seq;
    T[t].I0 = f.I0; for (int k = 0; k < 9; k++) T[t].R[k] = pre14[14*t+k]; for (int k = 0; k < 3; k++) T[t].t[k] = pre14[14*t+9+k]; T[t].aff[0] = pre14[14*t+12]; T[t].aff[1] = pre14[14*t+13];
  }
  for (int g = 0; g < n_groups; g++) { G[g].tgt_begin = tgt_begin[g]; G[g].nres = tgt_begin[g+1] - tgt_begin[g]; const float* q = calib6 + 6*g;
    G[g].fxl = q[0]; G[g].fyl = q[1]; G[g].cxl = q[2]; G[g].cyl = q[3]; G[g].fxli = q[4]; G[g].fyli = q[5]; const int cam = cams ? cams[g] : 0; G[g].w = c->cam_w[cam]; G[g].h = c->cam_h[cam];
    for (int i = pt_begin[g]; i < pt_begin[g+1]; i++) gof[i] = g; }
  { int rc = join_ingest_upto(c, need_seq); if (rc) return rc; }
  auto al = [](size_t b) { return (b + 15) & ~(size_t)15; };
  const size_t o_g = 0, o_t = al(n_groups*sizeof(OptGroupDev)), o_of = o_t + al(nt*sizeof(OptTargetDev)), o_fs = o_of + al((size_t)n*sizeof(int)), o_st = o_fs + al((size_t)n),
               o_id = o_st + al((size_t)n*sizeof(int)), o_rs = o_id + al((size_t)n*sizeof(float)), o_pts = o_rs + al((size_t)n*res_stride*sizeof(int)), bytes = o_pts + (size_t)n*sizeof(sdv_immature_pt);
  { int rc = trace_scratch(c, bytes); if (rc) return rc; }
  char* d = (char*)c->trace_dev;
  CK(cudaMemcpyAsync(d + o_g, G.data(), n_groups*sizeof(OptGroupDev), cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(d + o_t, T.data(), nt*sizeof(OptTargetDev), cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(d + o_of, gof.data(), (size_t)n*sizeof(int), cudaMemcpyHostToDevice, c->st));
  if (is_from_sensor) CK(cudaMemcpyAsync(d + o_fs, is_from_sensor, (size_t)n, cudaMemcpyHostToDevice, c->st));
  CK(cudaMemcpyAsync(d + o_pts, pts, (size_t)n*sizeof(sdv_immature_pt), cudaMemcpyHostToDevice, c->st));
  CK(cudaEventRecord(c->ev0, c->st));
  imm_optimize_kernel<<<(n + 63)/64, 64, 0, c->st>>>((const OptGroupDev*)(d + o_g), (const OptTargetDev*)(d + o_t), (const int*)(d + o_of), n, (const sdv_immature_pt*)(d + o_pts),
      is_from_sensor ? (const unsigned char*)(d + o_fs) : nullptr, min_obs, res_stride, (int*)(d + o_st), (float*)(d + o_id), (int*)(d + o_rs), c->set.huberTH);
  c->launches += 1;
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev1, c->st));
  CK(cudaMemcpyAsync(status_out, d + o_st, (size_t)n*sizeof(int), cudaMemcpyDeviceToHost, c->st));
  CK(cudaMemcpyAsync(idepth_out, d + o_id, (size_t)n*sizeof(float), cudaMemcpyDeviceToHost, c->st));
  CK(cudaMemcpyAsync(res_state_out, d + o_rs, (size_t)n*res_stride*sizeof(int), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  return SDV_OK;
}
int sdv_immature_optimize_batch(sdv_ctx* c, int n_groups, const int32_t* pt_begin, const int32_t* tgt_begin, const uint64_t* target_frames, const float* pre14, const float* calib6,
                                int min_obs, const sdv_immature_pt* pts, const uint8_t* is_from_sensor, int res_stride, int32_t* status_out, float* idepth_out, int32_t* res_state_out) {
  return sdv_immature_optimize_batch_cams(c, n_groups, pt_begin, tgt_begin, target_frames, pre14, calib6, nullptr, min_obs, pts, is_from_sensor, res_stride, status_out, idepth_out, res_state_out);
}

}  // extern "C"
