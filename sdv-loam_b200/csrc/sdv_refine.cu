// sdv_refine.cu — semi-direct pose refinement on matched map points (SURVEY.md §8 row a11, D4).
//
// Replaces CoarseTracker::structPoseEstimation + calculateRes + calculateWeight + calcHandb
// (/root/reference/src/FullSystem/CoarseTracker.cpp:840-1007).  One CTA per frame ("job"), the whole damped Gauss-Newton loop is
// device resident: one launch refines the poses of all sequences of a batch.
//
// Numerics contract (what keeps accept/reject decisions identical to the host code):
//   * the energy is a float sum in point order ((e + r0*r0) + r1*r1), CoarseTracker.cpp:865 -> the per-point squares are computed by all
//     threads into shared memory, one thread then adds them in order;
//   * H (6x6) and b are double sums in point order of (Jx_i*Jx_j + Jy_i*Jy_j)*w, (Jx_i*r0 + Jy_i*r1)*w (:943-944) -> 27 threads (21 upper
//     entries + 6), each walking the staged points in order;
//   * the damping is applied to H in place, so it compounds over rejected steps (:966), and after an accepted step H,b are re-linearised at
//     the pose BEFORE the step (:989 precedes :990).  Both are load-bearing and kept.
// Compiled with --fmad=false like the rest of the library.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include "sdv_ctx.cuh"
#include "sdv_refine.cuh"
#include "sdv_warp_solve.cuh"

namespace sdv {

constexpr int kRefThreads = 128;
constexpr int kRefChunk = 256;           // points staged per pass
constexpr int kRefMaxHosts = 16;


struct RefShared {
  float hostR[kRefMaxHosts][9], hostT[kRefMaxHosts][3];
  float R[9], t[3];
  float J[12][kRefChunk]; float r0[kRefChunk], r1[kRefChunk]; float wgt[kRefChunk]; int ok[kRefChunk];
  double H[36], b[6]; double H0[36], b0[6];   // H0,b0: undamped system of the last calcHandb evaluation (restored instead of re-evaluating the same pose)
  double inc[6];
  float energy; int num; int done;
};

__device__ __forceinline__ bool ref_project(const sdv_overlap_pt& p, const RefShared& S, const LevelGeom& g, float fxi, float fyi, float* pf, float& Ku, float& Kv) {
  float k0 = (p.u + 0 - g.cx)*fxi, k1 = (p.v + 0 - g.cy)*fyi, k2 = 1.f;                 // point2world, ResidualProjections.h:61-77
  float a0 = k0/p.idepth, a1 = k1/p.idepth, a2 = k2/p.idepth;
  const float* Rh = S.hostR[p.host]; const float* th = S.hostT[p.host];
  float w0 = ((Rh[0]*a0 + Rh[1]*a1) + Rh[2]*a2) + th[0];
  float w1 = ((Rh[3]*a0 + Rh[4]*a1) + Rh[5]*a2) + th[1];
  float w2 = ((Rh[6]*a0 + Rh[7]*a1) + Rh[8]*a2) + th[2];
  pf[0] = ((S.R[0]*w0 + S.R[1]*w1) + S.R[2]*w2) + S.t[0];                                 // world2frame :79-94
  pf[1] = ((S.R[3]*w0 + S.R[4]*w1) + S.R[5]*w2) + S.t[1];
  pf[2] = ((S.R[6]*w0 + S.R[7]*w1) + S.R[8]*w2) + S.t[2];
  float u0 = pf[0]/pf[2], u1 = pf[1]/pf[2];
  Ku = u0*g.fx + g.cx; Kv = u1*g.fy + g.cy;
  return Ku > 1.1f && Kv > 1.1f && Ku < (float)(g.w-3) && Kv < (float)(g.h-3);
}

__device__ void ref_set_pose(RefShared& S, const SE3d& w2c) {      // thread 0
  double R[9]; qmat(w2c.q, R);
  for (int i=0;i<9;i++) S.R[i] = (float)R[i];
  for (int i=0;i<3;i++) S.t[i] = (float)w2c.t[i];
}

// float energy of the pose staged in S.R/S.t ; result in S.energy / S.num (all threads call)
__device__ void ref_energy(RefShared& S, const int pt_begin, const int pt_end, const sdv_overlap_pt* __restrict__ pts, const LevelGeom& g, float fxi, float fyi) {
  if (threadIdx.x == 0) { S.energy = 0.f; S.num = 0; }
  for (int base = pt_begin; base < pt_end; base += kRefChunk) {
    int cnt = min(kRefChunk, pt_end - base);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      sdv_overlap_pt p = pts[base+i]; float pf[3], Ku, Kv;
      bool ok = ref_project(p, S, g, fxi, fyi, pf, Ku, Kv);
      float a = Ku - p.obs_x, b = Kv - p.obs_y;
      S.r0[i] = ok ? a*a : 0.f; S.r1[i] = ok ? b*b : 0.f; S.ok[i] = ok;        // skipped points add exact zeros: the chain below is branch-free
    }
    __syncthreads();
    if (threadIdx.x == 0) { float e = S.energy; int n = S.num;
#pragma unroll 8
      for (int i=0;i<cnt;i++) { e = e + S.r0[i] + S.r1[i]; n += S.ok[i]; }
      S.energy = e; S.num = n; }
  }
  __syncthreads();
}

// H,b at the pose staged in S.R/S.t, accumulated onto S.H/S.b (all threads call)
__device__ void ref_hb(RefShared& S, const int pt_begin, const int pt_end, const sdv_overlap_pt* __restrict__ pts, const LevelGeom& g, float fxi, float fyi) {
  int role = threadIdx.x, ri = 0, rj = 0;            // 0..20 upper H entries (row-major over i<=j), 21..26 b
  if (role < 21) { int r = role; for (ri = 0; r >= 6-ri; ri++) r -= 6-ri; rj = ri + r; }
  double acc = 0.0;
  if (role < 21) acc = S.H[ri*6+rj]; else if (role < 27) acc = S.b[role-21];
  for (int base = pt_begin; base < pt_end; base += kRefChunk) {
    int cnt = min(kRefChunk, pt_end - base);
    __syncthreads();
    for (int i = threadIdx.x; i < cnt; i += blockDim.x) {
      sdv_overlap_pt p = pts[base+i]; float pf[3], Ku, Kv;
      bool ok = ref_project(p, S, g, fxi, fyi, pf, Ku, Kv);
      float dx[6], dy[6];
      dx[0] = 1.f / pf[2]; dx[1] = 0.f; dx[2] = - pf[0] / (pf[2]*pf[2]); dx[3] = dx[2]*pf[1]; dx[4] = 1 + pf[0]*dx[2]; dx[5] = - pf[1]/pf[2];
      dy[0] = 0.f; dy[1] = 1.f / pf[2]; dy[2] = - pf[1] / (pf[2]*pf[2]); dy[3] = - (1 + pf[1]*dy[2]); dy[4] = - dx[3]; dy[5] = pf[0]/pf[2];
      float up = (Ku - g.cx)*fxi, vp = (Kv - g.cy)*fyi, uo = (p.obs_x - g.cx)*fxi, vo = (p.obs_y - g.cy)*fyi;       // pixel2unit :96-102
      float r0 = up - uo, r1 = vp - vo;
      float x = sqrtf(r0*r0 + r1*r1);
      const float tb = 4.6851f; float b2 = tb*tb, x2 = x*x, wv = 0.f;                                                   // Tukey :873-887
      if (x2 <= b2) { float tmp = 1.0f - x2/b2; wv = tmp*tmp; }
      for (int k=0;k<6;k++) { S.J[k][i] = ok ? dx[k] : 0.f; S.J[6+k][i] = ok ? dy[k] : 0.f; }   // skipped points contribute exact zeros (no NaN*0)
      S.r0[i] = ok ? r0 : 0.f; S.r1[i] = ok ? r1 : 0.f; S.wgt[i] = ok ? wv : 0.f; S.ok[i] = ok;
    }
    __syncthreads();
    if (role < 21) {
      const float* __restrict__ a0 = S.J[ri]; const float* __restrict__ a1 = S.J[rj]; const float* __restrict__ c0 = S.J[6+ri]; const float* __restrict__ c1 = S.J[6+rj];
#pragma unroll 4
      for (int i=0;i<cnt;i++) acc += ((double)a0[i]*(double)a1[i] + (double)c0[i]*(double)c1[i])*(double)S.wgt[i];
    } else if (role < 27) { const int k = role-21; const float* __restrict__ a0 = S.J[k]; const float* __restrict__ c0 = S.J[6+k];
#pragma unroll 4
      for (int i=0;i<cnt;i++) acc += ((double)a0[i]*(double)S.r0[i] + (double)c0[i]*(double)S.r1[i])*(double)S.wgt[i];
    }
  }
  __syncthreads();
  if (role < 21) { S.H[ri*6+rj] = acc; S.H[rj*6+ri] = acc; } else if (role < 27) S.b[role-21] = acc;
  __syncthreads();
}

__global__ void __launch_bounds__(kRefThreads) struct_pose_kernel(RefineJob* jobs, const sdv_overlap_pt* pts, const double* hostT7, const GeomRow* geom_tab) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  RefShared& S = *reinterpret_cast<RefShared*>(smem_raw);
  __shared__ SE3d cur, cand;             // worldToCur_current / worldToCur_new
  __shared__ float s_lambda, s_resOld;
  RefineJob& jb = jobs[blockIdx.x];
  const int pt_begin = jb.pt_begin, pt_end = jb.pt_end, nH = jb.nH, host_begin = jb.host_begin; const double* __restrict__ hostT = jb.hostT;   // read once: jb is written below, so the
                                                                        // compiler would otherwise re-load these from global memory inside every loop
  const LevelGeom g = geom_tab[jb.geom_row].g[0];
  const float fxi = g.Ki[0], fyi = g.Ki[4];
  for (int k = threadIdx.x; k < nH; k += blockDim.x) {
    SE3d h = se3_from7(hostT ? hostT + 7*k : hostT7 + 7*(size_t)(host_begin + k)); double R[9]; qmat(h.q, R);
    for (int i=0;i<9;i++) S.hostR[k][i] = (float)R[i];
    for (int i=0;i<3;i++) S.hostT[k][i] = (float)h.t[i];
  }
  if (threadIdx.x < 36) S.H[threadIdx.x] = 0.0; if (threadIdx.x < 6) S.b[threadIdx.x] = 0.0;
  if (threadIdx.x == 0) { cur = se3_inv(se3_from7(jb.T)); ref_set_pose(S, cur); s_lambda = 0.01f; S.done = 0; jb.iterations = 0; jb.accepts = 0; }
  __syncthreads();
  ref_energy(S, pt_begin, pt_end, pts, g, fxi, fyi);
  if (threadIdx.x == 0) s_resOld = S.energy / S.num;
  ref_hb(S, pt_begin, pt_end, pts, g, fxi, fyi);
  const float lambdaExtrapolationLimit = 0.001f;
  // undamped copy of the system at the current pose: structPoseEstimation re-linearises at the pose BEFORE an accepted step (:989), i.e. for the
  // first accepted step at the very pose the loop started from — identical values, so they are restored rather than recomputed
  __shared__ int cur_id, hb_id;
  if (threadIdx.x < 36) S.H0[threadIdx.x] = S.H[threadIdx.x]; if (threadIdx.x < 6) S.b0[threadIdx.x] = S.b[threadIdx.x];
  if (threadIdx.x == 0) { cur_id = 0; hb_id = 0; }
  __syncthreads();
  for (int iteration = 0; iteration < 10; iteration++) {
    __shared__ double s_incn;
    if (threadIdx.x < 32) {                                              // warp 0: damp, solve (6x6 padded to the 8x8 warp LDLT), propose
      const int r = threadIdx.x & 7; const float lambda = s_lambda;
      if (threadIdx.x < 6) S.H[threadIdx.x*6+threadIdx.x] *= (1 + lambda);
      __syncwarp();
      double a[8];
#pragma unroll
      for (int j = 0; j < 8; j++) a[j] = (r < 6 && j < 6) ? S.H[r*6+j] : ((r == j) ? 1.0 : 0.0);
      const double rhs = (r < 6) ? -S.b[r] : 0.0;
      const double x = warp_ldlt_solve8(a, rhs);
      float extrapFac = 1;
      if (lambda < lambdaExtrapolationLimit) extrapFac = sqrtf(sqrtf(lambdaExtrapolationLimit / lambda));
      if (threadIdx.x < 6) S.inc[threadIdx.x] = x*extrapFac;
      __syncwarp();
      if (threadIdx.x == 0) {
        jb.iterations++;
        double inc[6]; for (int i=0;i<6;i++) inc[i] = S.inc[i];
        cand = se3_mul(se3_exp(inc), cur);
        ref_set_pose(S, cand);
        double n2 = 0; for (int i=0;i<6;i++) n2 += inc[i]*inc[i]; s_incn = sqrt(n2);
      }
    }
    __syncthreads();
    ref_energy(S, pt_begin, pt_end, pts, g, fxi, fyi);
    __shared__ int s_accept, s_recompute;
    if (threadIdx.x == 0) {
      float resNew = (S.num == 0) ? 1000000.0f : S.energy / S.num;
      s_accept = (resNew < s_resOld); s_recompute = 0;
      if (s_accept) { s_resOld = resNew; jb.accepts++; s_recompute = (hb_id != cur_id); if (s_recompute) ref_set_pose(S, cur); }
    }
    __syncthreads();
    if (s_accept) {
      if (s_recompute) {
        if (threadIdx.x < 36) S.H[threadIdx.x] = 0.0; if (threadIdx.x < 6) S.b[threadIdx.x] = 0.0;
        __syncthreads();
        ref_hb(S, pt_begin, pt_end, pts, g, fxi, fyi);                                 // (sic) at the pose before the accepted step
        if (threadIdx.x < 36) S.H0[threadIdx.x] = S.H[threadIdx.x]; if (threadIdx.x < 6) S.b0[threadIdx.x] = S.b[threadIdx.x];
        if (threadIdx.x == 0) hb_id = cur_id;
      } else {
        if (threadIdx.x < 36) S.H[threadIdx.x] = S.H0[threadIdx.x]; if (threadIdx.x < 6) S.b[threadIdx.x] = S.b0[threadIdx.x];
      }
      if (threadIdx.x == 0) { cur = cand; cur_id++; SE3d c2w = se3_inv(cand); se3_to7(c2w, jb.T); s_lambda *= 0.5f; }
    } else if (threadIdx.x == 0) { float l = s_lambda*4; if (l < lambdaExtrapolationLimit) l = lambdaExtrapolationLimit; s_lambda = l; }
    __syncthreads();
    const bool small = !(s_incn > 1e-5);
    __syncthreads();                                                     // s_incn is rewritten by warp 0 at the top of the next iteration
    if (small) break;
  }
  if (threadIdx.x == 0) { jb.res = s_resOld; jb.num = S.num; }
}

cudaError_t refine_init_device() {         // per-device opt-in shared memory size (called by sdv_create after cudaSetDevice)
  return cudaFuncSetAttribute(struct_pose_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sizeof(RefShared));
}
void launch_struct_pose(RefineJob* jobs, int n_jobs, const sdv_overlap_pt* pts, const double* hostT7, const GeomRow* geom_tab, cudaStream_t st) {
  struct_pose_kernel<<<n_jobs, kRefThreads, sizeof(RefShared), st>>>(jobs, pts, hostT7, geom_tab);
}

} // namespace sdv

using namespace sdv;

extern "C" {

// slots == NULL: every job uses the context calibration (row 0 of the geometry table)
int sdv_tracker_struct_pose_batch_slots(sdv_ctx* c, int n_jobs, const int32_t* slots, const int32_t* pt_begin, const sdv_overlap_pt* pts, const int32_t* host_begin,
                                        const double* host_T7, double* curToWorld_io, float* res_out, int32_t* iterations, int32_t* accepts) { SDV_GUARD_TRK(c);
  if (!c || n_jobs <= 0 || !pt_begin || !host_begin || !host_T7 || !curToWorld_io) return SDV_ERR_ARG;
  if (slots) for (int k=0;k<n_jobs;k++) if (slots[k] < 0 || slots[k] >= (int)c->slots.size()) return ctx_fail(c, SDV_ERR_ARG, "struct_pose job %d: slot %d of %d", k, slots[k], (int)c->slots.size());
  { int rc = check_offsets(c, n_jobs, pt_begin, "struct_pose", "pt_begin"); if (rc) return rc; }
  { int rc = check_offsets(c, n_jobs, host_begin, "struct_pose", "host_begin"); if (rc) return rc; }
  const int nP = pt_begin[n_jobs], nH = host_begin[n_jobs];
  if (nH <= 0 || (nP > 0 && !pts)) return SDV_ERR_ARG;
  for (int k=0;k<n_jobs;k++) {
    int hs = host_begin[k+1]-host_begin[k];
    if (hs > kRefMaxHosts) return ctx_fail(c, SDV_ERR_ARG, "struct_pose job %d: bad ranges (hosts %d, max %d)", k, hs, kRefMaxHosts);
    for (int i=pt_begin[k]; i<pt_begin[k+1]; i++) if (pts[i].host < 0 || pts[i].host >= hs) return ctx_fail(c, SDV_ERR_ARG, "struct_pose job %d: point %d names host %d of %d", k, i, pts[i].host, hs);
  }
  CK(cudaSetDevice(c->device));
  Scratch& D = c->scr; PinnedScratch& Hs = c->scr_host;                  // the same layout on both sides: one copy stages jobs, points and host poses
  const size_t bytes = Scratch::need(n_jobs, sizeof(RefineJob)) + Scratch::need(nP, sizeof(sdv_overlap_pt)) + Scratch::need((size_t)nH*7, sizeof(double));
  if (D.reserve(bytes, c->st) || Hs.reserve(bytes, c->st)) return ctx_fail(c, SDV_ERR_CUDA, "struct_pose: staging of %d jobs", n_jobs);
  D.reset(); Hs.reset();
  RefineJob* J = Hs.take<RefineJob>(n_jobs); sdv_overlap_pt* hpts = Hs.take<sdv_overlap_pt>(nP); double* hT = Hs.take<double>((size_t)nH*7);
  RefineJob* dJ = D.take<RefineJob>(n_jobs); const sdv_overlap_pt* dpts = D.take<sdv_overlap_pt>(nP); const double* dT = D.take<double>((size_t)nH*7);
  for (int k=0;k<n_jobs;k++) { memset(&J[k], 0, sizeof(RefineJob)); for (int i=0;i<7;i++) J[k].T[i] = curToWorld_io[7*k+i];
    J[k].pt_begin = pt_begin[k]; J[k].pt_end = pt_begin[k+1]; J[k].host_begin = host_begin[k]; J[k].nH = host_begin[k+1]-host_begin[k];
    J[k].geom_row = slots ? c->slots[slots[k]].geom_row : 0; }
  if (nP) memcpy(hpts, pts, (size_t)nP*sizeof(sdv_overlap_pt));
  memcpy(hT, host_T7, (size_t)nH*7*sizeof(double));
  c->launches += 1;
  CK(cudaMemcpyAsync(D.p, Hs.p, Hs.used, cudaMemcpyHostToDevice, c->st));
  CK(cudaEventRecord(c->ev0, c->st));
  launch_struct_pose(dJ, n_jobs, dpts, dT, c->geom_dev, c->st);
  CK(cudaGetLastError());
  CK(cudaEventRecord(c->ev1, c->st));
  CK(cudaMemcpyAsync(J, dJ, (size_t)n_jobs*sizeof(RefineJob), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  for (int k=0;k<n_jobs;k++) { for (int i=0;i<7;i++) curToWorld_io[7*k+i] = J[k].T[i];
    if (res_out) res_out[k] = J[k].res; if (iterations) iterations[k] = J[k].iterations; if (accepts) accepts[k] = J[k].accepts; }
  return SDV_OK;
}

int sdv_tracker_struct_pose_batch(sdv_ctx* c, int n_jobs, const int32_t* pt_begin, const sdv_overlap_pt* pts, const int32_t* host_begin, const double* host_T7,
                                  double* curToWorld_io, float* res_out, int32_t* iterations, int32_t* accepts) {
  return sdv_tracker_struct_pose_batch_slots(c, n_jobs, nullptr, pt_begin, pts, host_begin, host_T7, curToWorld_io, res_out, iterations, accepts);
}

int sdv_tracker_struct_pose(sdv_ctx* c, int n, const sdv_overlap_pt* pts, int nH, const double* host_T7, double curToWorld_io[7], float* res_out, int* iterations, int* accepts) { SDV_GUARD_TRK(c);
  int32_t pb[2] = {0, n}, hbeg[2] = {0, nH}, it = 0, ac = 0;
  int rc = sdv_tracker_struct_pose_batch(c, 1, pb, pts, hbeg, host_T7, curToWorld_io, res_out, &it, &ac);
  if (iterations) *iterations = it; if (accepts) *accepts = ac; return rc;
}

} // extern "C"
