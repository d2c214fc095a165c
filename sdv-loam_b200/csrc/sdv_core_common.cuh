// sdv_core_common.cuh — what the self-contained device cores (sdv_select_core.cuh, sdv_lidar_core.cuh) share: launch macros (CUDA, or the host emulation of tests/emu),
// a block-wide exclusive scan, a grow-only scratch allocator, makeImages' gradient of a planar plane, and the reference rules that more than one kernel restates:
// staticPattern, getInterpolatedElement31 on a planar plane, the ImmaturePoint constructor and its status codes.  Depends on nothing but the CUDA runtime.
#pragma once
#include <stdint.h>
#include <math.h>
#include <vector>
#include <algorithm>
#include <string>
#include <limits.h>
#include <string.h>
#ifndef SDV_EMU
#include <cuda_runtime.h>
#define SDV_LAUNCH(kern, grid, block, st, ...)      kern<<<grid, block, 0, st>>>(__VA_ARGS__)
#define SDV_LAUNCH_SYNC(kern, grid, block, st, ...) kern<<<grid, block, 0, st>>>(__VA_ARGS__)
#define SDV_DEVCONST static __constant__
#define SDV_DYN_SMEM(T, name) extern __shared__ __align__(16) unsigned char name##_raw_[]; T* name = reinterpret_cast<T*>(name##_raw_)
#define SDV_SET_SMEM(kern, bytes) cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)(bytes))
#define SDV_LAUNCH_SYNC_SMEM(kern, grid, block, smem, st, ...) kern<<<grid, block, smem, st>>>(__VA_ARGS__)
#endif

namespace sdv {

__device__ __forceinline__ float grad_guard(float d) { return isfinite(d) ? d : 0.0f; }     // if(!std::isfinite(dx)) dx=0;
// gradient of texel idx of a planar intensity plane as FrameHessian::makeImages forms it (HessianBlocks.cpp:147-156): central differences of flat-index
// neighbours (at x = 0 / x = w-1 the reference reads across the row boundary, and so does this), zero on the first and last row
// (returns false there), non-finite -> 0.
__device__ __forceinline__ bool planar_grad(const float* __restrict__ I, int idx, int w, int h, float& dx, float& dy) {
  dx = 0.f; dy = 0.f;
  if (idx >= w && idx < w*(h-1)) {
    dx = 0.5f*(__ldg(I + idx+1) - __ldg(I + idx-1));
    dy = 0.5f*(__ldg(I + idx+w) - __ldg(I + idx-w));
    if (!isfinite(dx)) dx = 0;
    if (!isfinite(dy)) dy = 0;
    return true;
  }
  return false;
}
// the factor makeImages applies to |grad|^2 of a texel of intensity I (HessianBlocks.cpp:158-164): gw*gw with gw = CalibHessian::getBGradOnly(I) = B[c+1]-B[c],
// c = (int)(I+0.5f) clamped to [5, 250] (HessianBlocks.h:343-349).  gw2[c] holds that product per camera (sdv_set_gamma_cam); nullptr is the identity B[i] = i (gw = 1).
// (int) of a NaN or of a value outside the int range is undefined in C++; the reference's x86 build converts with cvttss2si, which gives INT_MIN there, so c = 5.
// The device conversion saturates instead, so that case is restated explicitly (DESIGN §0).
__host__ __device__ __forceinline__ float gamma_w2(float I, const float* __restrict__ gw2) {
  if (!gw2) return 1.0f;
  const float t = I + 0.5f;
  int c = 5;
  if (t >= 6.0f && t < 2147483648.0f) c = t >= 250.0f ? 250 : (int)t;
  return gw2[c];
}

SDV_DEVCONST int staticPattern[8][2] = {{0,-2},{-1,-1},{1,-1},{-2,0},{0,0},{2,0},{-1,1},{0,2}};   // util/settings.cpp:250
enum { IPS_GOOD = 0, IPS_OOB, IPS_OUTLIER, IPS_SKIPPED, IPS_BADCONDITION, IPS_UNINITIALIZED };      // ImmaturePointStatus (ImmaturePoint.h)

// getInterpolatedElement31 (util/globalFuncs.h:102-116) on a planar plane of row stride w; the sum is ((a + b) + c) + d as in the reference
__device__ __forceinline__ float interp31(const float* __restrict__ I, float x, float y, int w) {
  const int ix = (int)x, iy = (int)y; const float dx = x - ix, dy = y - iy, dxdy = dx*dy; const float* bp = I + ix + iy*w;
  return dxdy*__ldg(bp+1+w) + (dy-dxdy)*__ldg(bp+w) + (dx-dxdy)*__ldg(bp+1) + (1-dx-dy+dxdy)*__ldg(bp);
}

// ImmaturePoint::ImmaturePoint (ImmaturePoint.cpp:8-36) at integer pixel (u, v) of the level-0 plane I0 (row stride w); returns whether energyTH is finite.
// Pt: sdv_immature_pt or its layout twin sel::ImmPt; Set: a settings struct with outlierTH, outlierTHSumComponent and overallEnergyTHWeight.
template <class Pt, class Set>
__device__ __forceinline__ bool imm_construct(const float* __restrict__ I0, int w, int u, int v, const Set& S, Pt& p) {
  p.u = (float)u; p.v = (float)v; p.idepth_min = 0; p.idepth_max = NAN; p.lastTraceStatus = IPS_UNINITIALIZED;
  for (int k = 0; k < 4; k++) p.gradH[k] = 0;
  p.lastTraceUV[0] = p.lastTraceUV[1] = 0; p.quality = 10000; p.lastTracePixelInterval = 0; p.energyTH = NAN;
  for (int k = 0; k < 8; k++) { p.color[k] = 0; p.weights[k] = 0; }
  for (int idx = 0; idx < 8; idx++) {
    const float x = p.u + staticPattern[idx][0], y = p.v + staticPattern[idx][1];
    const int ix = (int)x, iy = (int)y; const float* bp = I0 + ix + iy*w;                         // getInterpolatedElement33BiLin, util/globalFuncs.h:142-164
    const float tl = __ldg(bp), tr = __ldg(bp+1), bl = __ldg(bp+w), br = __ldg(bp+w+1);
    const float dx = x - ix, dy = y - iy;
    const float topInt = dx*tr + (1-dx)*tl, botInt = dx*br + (1-dx)*bl, leftInt = dy*bl + (1-dy)*tl, rightInt = dy*br + (1-dy)*tr;
    const float c0 = dx*rightInt + (1-dx)*leftInt, gx = rightInt-leftInt, gy = botInt-topInt;
    p.color[idx] = c0;
    if (!isfinite(c0)) return false;
    p.gradH[0] += gx*gx; p.gradH[1] += gx*gy; p.gradH[2] += gy*gx; p.gradH[3] += gy*gy;
    p.weights[idx] = sqrtf(S.outlierTHSumComponent / (S.outlierTHSumComponent + (gx*gx + gy*gy)));
  }
  p.energyTH = 8*S.outlierTH; p.energyTH *= S.overallEnergyTHWeight*S.overallEnergyTHWeight;
  return true;
}

namespace sel {

__device__ __forceinline__ int imin_(int a, int b) { return a < b ? a : b; }
// exclusive prefix sum of a block's values through shared memory (Hillis-Steele); every thread of the CTA must call it
__device__ __forceinline__ int block_excl_scan(int v, int* sm /* 2*blockDim */, int& total) {
  const int t = threadIdx.x, n = blockDim.x; int cur = 0;
  sm[t] = v; __syncthreads();
  for (int d = 1; d < n; d <<= 1) { const int x = sm[cur*n + t] + (t >= d ? sm[cur*n + t - d] : 0); sm[(cur^1)*n + t] = x; cur ^= 1; __syncthreads(); }
  const int incl = sm[cur*n + t]; total = sm[cur*n + n-1]; __syncthreads();
  return incl - v;
}

#define SEL_CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) { err = std::string(#call) + " -> " + cudaGetErrorString(e_); return -1; } } while (0)

}  // namespace sel

// Grow-only buffer carved into 256-byte aligned pieces: reserve(sum of need()), reset, then take the pieces in order.  One instance serves one stream:
// reserve waits for that stream before it frees a buffer that is too small, and keeps 25 % headroom, so the steady state allocates nothing.
// need() includes 256 bytes of slack past the piece.  Mem: alloc / dealloc of the memory kind (DeviceMem here; sdv_ctx.cuh adds pinned host memory).
template <class Mem> struct ScratchOf {
  char* p = nullptr; size_t cap = 0, used = 0;
  int reserve(size_t bytes, cudaStream_t st) { if (bytes <= cap) return 0; cudaStreamSynchronize(st); release(); if (Mem::alloc((void**)&p, bytes + bytes/4) != cudaSuccess) { p = nullptr; return -1; } cap = bytes + bytes/4; return 0; }
  void reset() { used = 0; }
  template <class T> T* take(size_t n) { used = (used + 255) & ~(size_t)255; T* r = (T*)(p + used); used += n*sizeof(T); return r; }
  static size_t need(size_t n, size_t sz) { return ((n*sz + 255) & ~(size_t)255) + 256; }
  void release() { if (p) Mem::dealloc(p); p = nullptr; cap = 0; }
};
struct DeviceMem { static cudaError_t alloc(void** p, size_t n) { return cudaMalloc(p, n); } static void dealloc(void* p) { cudaFree(p); } };
using Scratch = ScratchOf<DeviceMem>;

}  // namespace sdv
