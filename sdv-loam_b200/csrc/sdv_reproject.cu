// sdv_reproject.cu — map reprojection + direct feature alignment (SURVEY.md §8 row a10, D4).
//
// Replaces Reprojector::reprojectMap / backprojectMap / reprojectCell / findMatchDirect / getWarpMatrixAffine / getBestSearchLevel /
// warpAffine / align1D / align2D / reprojectPoint (/root/reference/src/FullSystem/Reprojector.cpp:14-616), batched over frames:
//   rp_project_kernel   one thread per map point: world point, projection into the target frame (fp64, reference operation order), grid cell,
//                       sort key (host gradient magnitude)                                                     reprojectPoint :600-616
//   rp_scan / rp_scatter  counting sort of the candidates into their 25 px grid cells                           Grid :100-112
//   rp_match_kernel     one WARP per (frame, cell): candidates are tried in the order of the reference's stable list sort — (gradient key,
//                       insertion rank) ascending, selected lazily — until one aligns                          reprojectCell :198-233
// Numerics contract: all geometry in fp64 with the reference's expression order (--fmad=false); patch warp, Jacobians and the Gauss-Newton
// alignment in float; the three Jres sums of an iteration are accumulated in PIXEL ORDER by one lane each (the host code's order), the
// patch Hessian of align2D is an exact sum (multiples of 1/4 below 2^22) so a butterfly reduction is bit-identical.
// The grid's cell visiting order is an input (std::random_shuffle(rand()) in the reference, :111); the per-cell result does not depend on it.
#include <cuda_runtime.h>
#include <stdint.h>
#include <string.h>
#include <vector>
#include <algorithm>
#include "sdv_ctx.cuh"
#include "sdv_refine.cuh"

namespace sdv {

constexpr int kRpMaxHosts = 16;
constexpr int kRpCell = 25;

struct MapDev {                           // device-resident map of one sequence (set per keyframe)
  int nH, nP; double hostT[kRpMaxHosts][7]; const float* hostI0[kRpMaxHosts]; const sdv_map_pt* pts;
};
struct RpJob {
  const MapDev* map; const float* cur[kLevels]; double curT[7], curTinv[7];
  double K[9], Ki[9];                     // the map slot's K (its tracker slot's row of the geometry table at level 0) and K^-1, built on the host (rp_launch)
  float affLL[kRpMaxHosts][2]; int frame_rank[kRpMaxHosts];
  int cur_kf_index, backup, nH, nP; long long pt_off;
  unsigned char error;                    // set by rp_project_kernel: a map point names a host outside [0, nH)
  unsigned char cam;                      // camera of the map slot: its level-0 size is RpConst::cam_w/cam_h[cam]
  int geom_row;                           // handed to the structPoseEstimation job of the fused refinement (rp_emit_kernel)
};
static_assert(sizeof(RpJob) == 536, "RpJob keeps its size: the camera byte sits beside the one-byte error flag");
// K, Ki: the context calibration (geometry row 0), as launch constants.  cam_w/cam_h: level-0 size per camera (the job's grid is ceil(w/25) x ceil(h/25));
// cam_levels: pyramid depth per camera (getBestSearchLevel's cap is the job camera's depth - 1); ncols, ncells: the context grid, which strides the per-job
// outputs and numbers cell_order.
struct RpConst { double K[9], Ki[9]; int cam_w[SDV_MAX_CAMERAS], cam_h[SDV_MAX_CAMERAS], cam_levels[SDV_MAX_CAMERAS]; int ncols, ncells; };
struct RpScratch { double2* cand_px; float* cand_key; int* cand_cell; unsigned long long* list;   // list: per cell, (key bits << 32) | (frame rank << 27) | point index
                   int* count; int* begin; int* cursor; int* out_pt; double2* out_px;
                   double* xf; };   // xf[job][host][14]: camToWorld_host^-1 and T_cur_ref = camToWorld_cur^-1 * camToWorld_host (7 doubles each), built by rp_project_kernel

__device__ __forceinline__ void mv3(const double* M, double x, double y, double z, double* o) {
  o[0] = (M[0]*x + M[1]*y) + M[2]*z; o[1] = (M[3]*x + M[4]*y) + M[5]*z; o[2] = (M[6]*x + M[7]*y) + M[8]*z;
}
__device__ __forceinline__ void xform(const SE3d& T, const double* p, double* o) { double r[3]; qrot(T.q, p, r); o[0] = r[0]+T.t[0]; o[1] = r[1]+T.t[1]; o[2] = r[2]+T.t[2]; }
__device__ __forceinline__ void point_world(const double* Ki, const MapDev* __restrict__ m, const sdv_map_pt& p, double* pw) {   // pixelFrame2PointWorld :570-577
  double k[3]; mv3(Ki, (double)p.u, (double)p.v, 1.0, k);
  const double s = (double)(1/p.idepth);
  double r[3] = {k[0]*s, k[1]*s, k[2]*s};
  SE3d c2w = se3_from7(m->hostT[p.host]); xform(c2w, r, pw);
}
__device__ __forceinline__ void pixel_from_cam(const double* K, double* c, double* px) {                                          // :579-586 / :603-610
  c[0] = c[0]/c[2]; c[1] = c[1]/c[2]; c[2] = c[2]/c[2];
  double o[3]; mv3(K, c[0], c[1], c[2], o); px[0] = o[0]; px[1] = o[1];
}
__device__ __forceinline__ bool in_frame(int w, int h, double x, double y, int boundary) {
  if (!isfinite(x) || !isfinite(y) || fabs(x) > 1e9 || fabs(y) > 1e9) return false;
  const int ox = (int)x, oy = (int)y;
  return ox >= boundary && ox < w-boundary && oy >= boundary && oy < h-boundary;
}
template <bool OWN_K>                                                          // OWN_K: as in find_match_direct
__device__ __forceinline__ void project_point(const RpJob& jb, const RpConst& C, const MapDev* __restrict__ m, const sdv_map_pt& p, double* px) {
  double pw[3], c[3]; point_world(OWN_K ? jb.Ki : C.Ki, m, p, pw);
  SE3d w2c = se3_from7(jb.curTinv); xform(w2c, pw, c); pixel_from_cam(OWN_K ? jb.K : C.K, c, px);
}

__global__ void __launch_bounds__(256) rp_project_kernel(RpJob* __restrict__ jobs, RpConst C, RpScratch S) {
  RpJob& jb = jobs[blockIdx.y]; const MapDev* __restrict__ m = jb.map;
  if (blockIdx.x == 0 && threadIdx.x < jb.nH) {                              // per (frame, keyframe) transforms used by every findMatchDirect attempt (:262)
    const SE3d refPose = se3_from7(m->hostT[threadIdx.x]); double* o = S.xf + ((size_t)blockIdx.y*kRpMaxHosts + threadIdx.x)*14;
    se3_to7(se3_inv(refPose), o); se3_to7(se3_mul(se3_from7(jb.curTinv), refPose), o + 7);
  }
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= jb.nP) return;
  const long long gi = jb.pt_off + i; S.cand_cell[gi] = -1;
  const sdv_map_pt p = m->pts[i];
  if (p.host < 0 || p.host >= jb.nH) { jb.error = 1; return; }
  if (jb.frame_rank[p.host] < 0) return;
  double px[2];
  if (jb.geom_row) project_point<true>(jb, C, m, p, px); else project_point<false>(jb, C, m, p, px);
  const int w = C.cam_w[jb.cam], h = C.cam_h[jb.cam];
  if (!in_frame(w, h, px[0], px[1], 8)) return;
  const int k = (int)(px[1]/kRpCell)*((w + kRpCell - 1)/kRpCell) + (int)(px[0]/kRpCell);      // the job's own grid
  const float* __restrict__ I = m->hostI0[p.host]; const int idx = (int)(p.v*w + p.u);
  float gx, gy, key = 0.f;
  if (planar_grad(I, idx, w, h, gx, gy)) key = sqrtf(gx*gx + gy*gy);
  S.cand_px[gi] = make_double2(px[0], px[1]); S.cand_key[gi] = key; S.cand_cell[gi] = k;
  atomicAdd(&S.count[(long long)blockIdx.y*C.ncells + k], 1);
}

__global__ void __launch_bounds__(1024) rp_scan_kernel(RpConst C, RpScratch S) {
  const long long base = (long long)blockIdx.x*C.ncells; const int per = (C.ncells + 1023)/1024;
  __shared__ int part[1024];
  int s = 0; for (int k = 0; k < per; k++) { int c = threadIdx.x*per + k; if (c < C.ncells) s += S.count[base+c]; }
  part[threadIdx.x] = s; __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) { int v = (threadIdx.x >= o) ? part[threadIdx.x-o] : 0; __syncthreads(); part[threadIdx.x] += v; __syncthreads(); }
  int run = part[threadIdx.x] - s;
  for (int k = 0; k < per; k++) { int c = threadIdx.x*per + k; if (c < C.ncells) { S.begin[base+c] = run; run += S.count[base+c]; S.cursor[base+c] = 0; } }
}

__global__ void __launch_bounds__(256) rp_scatter_kernel(const RpJob* __restrict__ jobs, RpConst C, RpScratch S) {
  const RpJob& jb = jobs[blockIdx.y]; const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= jb.nP) return;
  const int k = S.cand_cell[jb.pt_off + i]; if (k < 0) return;
  const long long cb = (long long)blockIdx.y*C.ncells + k;
  const int pos = atomicAdd(&S.cursor[cb], 1);
  // sort key of reprojectCell's stable list sort: gradient magnitude (non-negative float: its bit pattern orders like the value), then insertion order
  // = (close_kfs rank of the host keyframe, index within the map)
  const unsigned long long key = ((unsigned long long)__float_as_uint(S.cand_key[jb.pt_off + i]) << 32) | ((unsigned long long)jb.frame_rank[jb.map->pts[i].host] << 27) | (unsigned int)i;
  S.list[jb.pt_off + S.begin[cb] + pos] = key;
}

// ---------------------------------------------------------------------------------------------------------------- findMatchDirect (one warp)
struct __align__(16) RpWarpSmem { float a0[64], a1[64], a2[64]; float jx[64], jy[64]; float pwb[100]; };
// J = ((0 - a[0]) - a[1]) - ... - a[63]: the host loop's order, 16 vector loads feeding one dependent FADD chain
__device__ __forceinline__ float chain_sub64(const float* a) {
  const float4* a4 = reinterpret_cast<const float4*>(a); float J = 0;
#pragma unroll
  for (int q = 0; q < 16; q++) { const float4 t = a4[q]; J -= t.x; J -= t.y; J -= t.z; J -= t.w; }
  return J;
}
constexpr int kRpWarps = 4;
#ifndef RP_MATCH_MINB
#define RP_MATCH_MINB 6
#endif

__device__ __forceinline__ float cur_pixel(const RpJob& jb, int level, int idx) { return __ldg(jb.cur[level] + idx); }

// OWN_K: the job's slot has a K of its own (RpJob::K, Ki in global memory); otherwise the context calibration is read from the launch constants, which the
// compiler folds into the fp64 instructions as constant-bank operands (reading every job's K from its descriptor cost the fused refinement 4.5 % on an H100)
template <bool OWN_K>
__device__ bool find_match_direct(const RpJob& jb, const RpConst& C, const sdv_map_pt& pt, double2& px_io, RpWarpSmem& sm, const int lane, const double* __restrict__ xf) {
  const double* __restrict__ K = OWN_K ? jb.K : C.K; const double* __restrict__ Ki = OWN_K ? jb.Ki : C.Ki;
  const MapDev* __restrict__ m = jb.map;
  // the job's level-0 size and getBestSearchLevel's cap (read here: passing them in from the kernel, or reading the depth where it is used, adds spills)
  const int w0 = C.cam_w[jb.cam], h0 = C.cam_h[jb.cam], max_level = C.cam_levels[jb.cam] - 1;
  int ref;
  if (jb.nH <= 2) { if (!jb.backup) ref = 0; else if (jb.cur_kf_index == 0) ref = 1; else if (jb.cur_kf_index == 1) ref = 0; else return false; }
  else ref = pt.host;
  const float aLL0 = jb.affLL[ref][0], aLL1 = jb.affLL[ref][1];
  double pw[3]; point_world(Ki, m, pt, pw);
  const SE3d refInv = se3_from7(xf + ref*14);
  double ptRef[3]; xform(refInv, pw, ptRef);
  double cR[3] = {ptRef[0], ptRef[1], ptRef[2]}, px[2]; pixel_from_cam(K, cR, px);
  if (!in_frame(w0, h0, px[0], px[1], 4+2)) return false;
  // getWarpMatrixAffine :14-37
  double A[4];
  { const int hp = 5; double du[3], dv[3]; mv3(Ki, px[0]+hp, px[1]+0, 1.0, du); mv3(Ki, px[0]+0, px[1]+hp, 1.0, dv);
    const double su = ptRef[2]/du[2], sv = ptRef[2]/dv[2];
    for (int i=0;i<3;i++) { du[i] *= su; dv[i] *= sv; }
    const SE3d Tcr = se3_from7(xf + ref*14 + 7);
    double c0[3], c1[3], c2[3], pc[2], pu[2], pv[2];
    xform(Tcr, ptRef, c0); pixel_from_cam(K, c0, pc); xform(Tcr, du, c1); pixel_from_cam(K, c1, pu); xform(Tcr, dv, c2); pixel_from_cam(K, c2, pv);
    A[0] = (pu[0]-pc[0])/hp; A[2] = (pu[1]-pc[1])/hp; A[1] = (pv[0]-pc[0])/hp; A[3] = (pv[1]-pc[1])/hp; }
  int level = 0; { double D = A[0]*A[3] - A[2]*A[1]; while (D > 3.0 && level < max_level) { level += 1; D *= 0.25; } }   // getBestSearchLevel :39-51, :268
  // warpAffine :53-86 (halfpatch 5 -> 10x10 patch with border), values truncated to uint8
  { const double det = A[0]*A[3] - A[2]*A[1], invdet = 1.0/det;
    const float a00 = (float)(A[3]*invdet), a10 = (float)(-A[2]*invdet), a01 = (float)(-A[1]*invdet), a11 = (float)(A[0]*invdet);
    __syncwarp();
    if (!isnan(a00)) {
      const float prx = (float)px[0], pry = (float)px[1]; const float* __restrict__ I = m->hostI0[ref];
      for (int q = lane; q < 100; q += 32) { const int y = q/10, x = q - y*10;
        float p0 = (float)(x-5), p1 = (float)(y-5); p0 *= (1<<level); p1 *= (1<<level);
        const float qx = (a00*p0 + a01*p1) + prx, qy = (a10*p0 + a11*p1) + pry;
        float v = 0.f;
        if (!(qx < 0 || qy < 0 || qx >= w0-1 || qy >= h0-1)) v = (float)(unsigned char)(interp31(I, qx, qy, w0));
        sm.pwb[q] = v; } }
    __syncwarp(); }
  double pxs[2] = {px_io.x/(1<<level), px_io.y/(1<<level)};
  const int wl = w0 >> level, hl = h0 >> level;
  const float min_update_squared = (float)(0.03*0.03);
  bool converged = false;
  float u = (float)pxs[0], v = (float)pxs[1], mean_diff = 0;
  const int q0 = lane, q1 = lane + 32;                                        // the two patch pixels of this lane (row-major 8x8)
  const int y0 = q0 >> 3, x0 = q0 & 7, y1 = q1 >> 3, x1 = q1 & 7;
  const float ref0 = sm.pwb[(y0+1)*10 + 1 + x0], ref1 = sm.pwb[(y1+1)*10 + 1 + x1];       // createPatchFromPatchWithBorder :334-344
  bool early_false = false;
  if (pt.type == 1) {                                                          // EDGELET: align1D :346-455
    const float* __restrict__ I = m->hostI0[ref]; const int idx = (int)(px[0] + px[1]*w0);
    double g0 = (double)grad_guard(0.5f*(__ldg(I+idx+1) - __ldg(I+idx-1))), g1 = (double)grad_guard(0.5f*(__ldg(I+idx+w0) - __ldg(I+idx-w0)));
    { const double n = sqrt(g0*g0 + g1*g1); g0 /= n; g1 /= n; }
    double d0 = A[0]*g0 + A[1]*g1, d1 = A[2]*g0 + A[3]*g1; { const double n2 = sqrt(d0*d0 + d1*d1); d0 /= n2; d1 /= n2; }
    const float dir0 = (float)d0, dir1 = (float)d1;
    { const int c0 = (y0+1)*10 + 1 + x0, c1 = (y1+1)*10 + 1 + x1;
      sm.jx[q0] = (float)(0.5*(double)(dir0*(sm.pwb[c0+1] - sm.pwb[c0-1]) + dir1*(sm.pwb[c0+10] - sm.pwb[c0-10])));
      sm.jx[q1] = (float)(0.5*(double)(dir0*(sm.pwb[c1+1] - sm.pwb[c1-1]) + dir1*(sm.pwb[c1+10] - sm.pwb[c1-10]))); }
    __syncwarp();
    float H00 = 0, H01 = 0;
    if (lane == 0) { for (int q = 0; q < 64; q++) H00 += sm.jx[q]*sm.jx[q]; }
    if (lane == 1) { for (int q = 0; q < 64; q++) H01 += sm.jx[q]*1.0f; }
    H00 = __shfl_sync(0xffffffffu, H00, 0); H01 = __shfl_sync(0xffffffffu, H01, 1);
    const float H10 = H01, H11 = 64.0f;
    const float det = H00*H11 - H10*H01, invdet = 1.0f/det;
    const float Hi00 = H11*invdet, Hi10 = -H10*invdet, Hi01 = -H01*invdet, Hi11 = H00*invdet;
    const float jv0 = sm.jx[q0], jv1 = sm.jx[q1];
    for (int iter = 0; iter < 10; ++iter) {
      const int u_r = (int)floorf(u), v_r = (int)floorf(v);
      if (u_r < 4 || v_r < 4 || u_r >= wl-4 || v_r >= hl-4) break;
      if (isnan(u) || isnan(v)) { early_false = true; break; }
      const float sx = u-u_r, sy = v-v_r;
      const float wTL = (float)((1.0-(double)sx)*(1.0-(double)sy)), wTR = (float)((double)sx*(1.0-(double)sy)), wBL = (float)((1.0-(double)sx)*(double)sy), wBR = sx*sy;
      { const int b0 = (v_r+y0-4)*wl + u_r-4 + x0, b1 = (v_r+y1-4)*wl + u_r-4 + x1;
        const float s0 = ((wTL*cur_pixel(jb, level, b0) + wTR*cur_pixel(jb, level, b0+1)) + wBL*cur_pixel(jb, level, b0+wl)) + wBR*cur_pixel(jb, level, b0+wl+1);
        const float s1 = ((wTL*cur_pixel(jb, level, b1) + wTR*cur_pixel(jb, level, b1+1)) + wBL*cur_pixel(jb, level, b1+wl)) + wBR*cur_pixel(jb, level, b1+wl+1);
        const float r0 = s0 - (float)(aLL0*ref0 + aLL1) + mean_diff, r1 = s1 - (float)(aLL0*ref1 + aLL1) + mean_diff;
        __syncwarp();
        sm.a0[q0] = r0*jv0; sm.a0[q1] = r1*jv1; sm.a2[q0] = r0; sm.a2[q1] = r1; }
      __syncwarp();
      float J = 0;
      if (lane < 2) J = chain_sub64(lane == 0 ? sm.a0 : sm.a2);
      const float Jres0 = __shfl_sync(0xffffffffu, J, 0), Jres1 = __shfl_sync(0xffffffffu, J, 1);
      const float up0 = Hi00*Jres0 + Hi01*Jres1, up1 = Hi10*Jres0 + Hi11*Jres1;
      u += up0*dir0; v += up0*dir1; mean_diff += up1;
      if (up0*up0 + up1*up1 < min_update_squared) { converged = true; break; }
    }
  } else {                                                                     // CORNER: align2D :457-560
    const int c0 = (y0+1)*10 + 1 + x0, c1 = (y1+1)*10 + 1 + x1;
    const float dx0 = (float)(0.5*(double)(sm.pwb[c0+1] - sm.pwb[c0-1])), dy0 = (float)(0.5*(double)(sm.pwb[c0+10] - sm.pwb[c0-10]));
    const float dx1 = (float)(0.5*(double)(sm.pwb[c1+1] - sm.pwb[c1-1])), dy1 = (float)(0.5*(double)(sm.pwb[c1+10] - sm.pwb[c1-10]));
    float h[5] = {dx0*dx0 + dx1*dx1, dx0*dy0 + dx1*dy1, dx0 + dx1, dy0*dy0 + dy1*dy1, dy0 + dy1};     // exact sums (multiples of 1/4, < 2^22)
#pragma unroll
    for (int k = 0; k < 5; k++) for (int o = 16; o > 0; o >>= 1) h[k] += __shfl_xor_sync(0xffffffffu, h[k], o);
    const float Hm[9] = {h[0], h[1], h[2], h[1], h[3], h[4], h[2], h[4], 64.0f}; float Hi[9]; inv3f(Hm, Hi);
    for (int iter = 0; iter < 10; ++iter) {
      const int u_r = (int)floorf(u), v_r = (int)floorf(v);
      if (u_r < 4 || v_r < 4 || u_r >= wl-4 || v_r >= hl-4) break;
      if (isnan(u) || isnan(v)) { early_false = true; break; }
      const float sx = u-u_r, sy = v-v_r;
      const float wTL = (float)((1.0-(double)sx)*(1.0-(double)sy)), wTR = (float)((double)sx*(1.0-(double)sy)), wBL = (float)((1.0-(double)sx)*(double)sy), wBR = sx*sy;
      { const int b0 = (v_r+y0-4)*wl + u_r-4 + x0, b1 = (v_r+y1-4)*wl + u_r-4 + x1;
        const float s0 = ((wTL*cur_pixel(jb, level, b0) + wTR*cur_pixel(jb, level, b0+1)) + wBL*cur_pixel(jb, level, b0+wl)) + wBR*cur_pixel(jb, level, b0+wl+1);
        const float s1 = ((wTL*cur_pixel(jb, level, b1) + wTR*cur_pixel(jb, level, b1+1)) + wBL*cur_pixel(jb, level, b1+wl)) + wBR*cur_pixel(jb, level, b1+wl+1);
        const float r0 = s0 - (float)(aLL0*ref0 + aLL1) + mean_diff, r1 = s1 - (float)(aLL0*ref1 + aLL1) + mean_diff;
        __syncwarp();
        sm.a0[q0] = r0*dx0; sm.a0[q1] = r1*dx1; sm.a1[q0] = r0*dy0; sm.a1[q1] = r1*dy1; sm.a2[q0] = r0; sm.a2[q1] = r1; }
      __syncwarp();
      float J = 0;
      if (lane < 3) J = chain_sub64(lane == 0 ? sm.a0 : (lane == 1 ? sm.a1 : sm.a2));
      const float J0 = __shfl_sync(0xffffffffu, J, 0), J1 = __shfl_sync(0xffffffffu, J, 1), J2 = __shfl_sync(0xffffffffu, J, 2);
      const float up0 = (Hi[0]*J0 + Hi[1]*J1) + Hi[2]*J2, up1 = (Hi[3]*J0 + Hi[4]*J1) + Hi[5]*J2, up2 = (Hi[6]*J0 + Hi[7]*J1) + Hi[8]*J2;
      u += up0; v += up1; mean_diff += up2;
      if (up0*up0 + up1*up1 < min_update_squared) { converged = true; break; }
    }
  }
  if (!early_false) { pxs[0] = (double)u; pxs[1] = (double)v; }
  px_io.x = pxs[0]*(1<<level); px_io.y = pxs[1]*(1<<level);
  return converged && !early_false;
}

__global__ void __launch_bounds__(32*kRpWarps, RP_MATCH_MINB) rp_match_kernel(const RpJob* __restrict__ jobs, RpConst C, RpScratch S) {
  __shared__ RpWarpSmem smem[kRpWarps];
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const int cell = blockIdx.x*kRpWarps + warp; if (cell >= C.ncells) return;
  const RpJob& jb = jobs[blockIdx.y]; const MapDev* __restrict__ m = jb.map;
  const long long cb = (long long)blockIdx.y*C.ncells + cell;
  const int n = S.count[cb]; const unsigned long long* __restrict__ lst = S.list + jb.pt_off + S.begin[cb];
  int found = -1; double2 fpx = make_double2(0, 0);
  unsigned long long last = 0; bool first = true;
  for (int tries = 0; tries < n; tries++) {
    // next candidate in (key, insertion rank) order = what the stable list sort of reprojectCell :200 visits: smallest packed key above the last one tried
    unsigned long long best = ~0ull;
    for (int j = lane; j < n; j += 32) { const unsigned long long k = lst[j]; if ((first || k > last) && k < best) best = k; }
    for (int o = 16; o > 0; o >>= 1) { const unsigned long long ob = __shfl_xor_sync(0xffffffffu, best, o); best = ob < best ? ob : best; }
    if (best == ~0ull) break;
    last = best; first = false;
    const int bi = (int)(best & 0x7ffffffull);
    double2 px = S.cand_px[jb.pt_off + bi];
    const double* xf = S.xf + (size_t)blockIdx.y*kRpMaxHosts*14;
    if (jb.geom_row ? find_match_direct<true>(jb, C, m->pts[bi], px, smem[warp], lane, xf) : find_match_direct<false>(jb, C, m->pts[bi], px, smem[warp], lane, xf)) { found = bi; fpx = px; break; }
  }
  if (lane == 0) { S.out_pt[cb] = found; S.out_px[cb] = fpx; }
}

// cell `cell` of the context grid (ncols columns) as a cell of a job's grid of jcols x jrows, or -1 when the job's grid does not have it: a job on a smaller
// camera walks the context's cell_order and skips the cells outside its grid (sdv_b200.h, sdv_reproject_map_batch); on the context grid this is the identity
__host__ __device__ __forceinline__ int job_cell(int cell, int ncols, int jcols, int jrows) {
  const int r = cell / ncols, col = cell - r*ncols;
  return (col < jcols && r < jrows) ? r*jcols + col : -1;
}
__host__ __device__ __forceinline__ int grid_dim(int px) { return (px + kRpCell - 1)/kRpCell; }

// Ordered emission of the per-cell results (reprojectMap :147-155): cells are visited in cell_order, every cell with a match contributes one
// overlap point, the walk stops once more than max_matches were produced.  One CTA per frame; also fills the structPoseEstimation job.
__global__ void __launch_bounds__(1024) rp_emit_kernel(const RpJob* __restrict__ jobs, RpConst C, RpScratch S, const int* __restrict__ cell_order, int max_matches,
                                                       sdv_overlap_pt* __restrict__ ov, RefineJob* __restrict__ rj, int* __restrict__ n_out) {
  const RpJob& jb = jobs[blockIdx.x]; const MapDev* __restrict__ m = jb.map;
  const long long base = (long long)blockIdx.x*C.ncells; const int per = (C.ncells + 1023)/1024;
  const int jcols = grid_dim(C.cam_w[jb.cam]), jrows = grid_dim(C.cam_h[jb.cam]);
  __shared__ int part[1024];
  int s = 0; for (int k = 0; k < per; k++) { const int i = threadIdx.x*per + k; if (i < C.ncells) { const int cell = job_cell(cell_order ? cell_order[i] : i, C.ncols, jcols, jrows); s += (cell >= 0 && S.out_pt[base+cell] >= 0) ? 1 : 0; } }
  part[threadIdx.x] = s; __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) { int v = (threadIdx.x >= o) ? part[threadIdx.x-o] : 0; __syncthreads(); part[threadIdx.x] += v; __syncthreads(); }
  int run = part[threadIdx.x] - s;
  const int total = min(part[1023], max_matches + 1);
  for (int k = 0; k < per; k++) { const int i = threadIdx.x*per + k; if (i >= C.ncells) break; const int cell = job_cell(cell_order ? cell_order[i] : i, C.ncols, jcols, jrows);
    if (cell < 0) continue;
    const int pi = S.out_pt[base+cell]; if (pi < 0) continue;
    if (run < total) { const sdv_map_pt p = m->pts[pi]; const double2 px = S.out_px[base+cell];
      sdv_overlap_pt o; o.u = p.u; o.v = p.v; o.idepth = p.idepth; o.host = p.host; o.obs_x = (float)px.x; o.obs_y = (float)px.y; ov[base + run] = o; }
    run++; }
  if (threadIdx.x == 0) { RefineJob& r = rj[blockIdx.x]; for (int i=0;i<7;i++) r.T[i] = jb.curT[i]; r.hostT = &m->hostT[0][0]; r.pt_begin = (int)base; r.pt_end = (int)base + total;
    r.host_begin = 0; r.nH = jb.nH; r.geom_row = jb.geom_row; r.res = 0; r.iterations = 0; r.accepts = 0; r.num = 0; n_out[blockIdx.x] = total; }
}

} // namespace sdv

using namespace sdv;

namespace sdv {
struct MapSlot { long long ingest_seq = 0; MapDev host_copy; MapDev* dev = nullptr; sdv_map_pt* pts = nullptr; int cap = 0; int nH = 0, nP = 0; uint64_t host_ids[kRpMaxHosts]; double host_ab[kRpMaxHosts][2]; float host_exposure[kRpMaxHosts]; bool set = false; };
struct RpState { std::vector<MapSlot> maps; RpConst C; };
static void rp_job_K(const LevelGeom& g, double* K, double* Ki);
static RpState* rp_state(sdv_ctx* c) {
  if (!c->rp) { c->rp = new RpState(); c->rp->maps.resize(c->slots.size()); RpConst& C = c->rp->C;
    C.ncols = grid_dim(c->w); C.ncells = C.ncols*grid_dim(c->h); }
  return c->rp;
}
bool rp_slot_set(const sdv_ctx* c, int slot) { return c->rp && slot < (int)c->rp->maps.size() && c->rp->maps[slot].set; }
void rp_destroy(sdv_ctx* c) { if (!c->rp) return; for (auto& m : c->rp->maps) { if (m.set) for (int k=0;k<m.nH;k++) frame_unpin(c, m.host_ids[k]); cudaFree(m.dev); cudaFree(m.pts); } delete c->rp; c->rp = nullptr; }
static void rp_job_K(const LevelGeom& g, double* K, double* Ki) {        // the Reprojector's K_ and K_.inverse() (Reprojector.cpp:565) from level 0 of a geometry row
  for (int i=0;i<9;i++) K[i] = 0; K[0] = (double)g.fx; K[2] = (double)g.cx; K[4] = (double)g.fy; K[5] = (double)g.cy; K[8] = 1.0;
  { const double* A = K; double* R = Ki;                                       // Eigen fixed 3x3 inverse: cofactors / determinant
#define COF(i,j) (A[((i+1)%3)*3+((j+1)%3)]*A[((i+2)%3)*3+((j+2)%3)] - A[((i+1)%3)*3+((j+2)%3)]*A[((i+2)%3)*3+((j+1)%3)])
    const double c00 = COF(0,0), c10 = COF(1,0), c20 = COF(2,0); const double det = (c00*A[0] + c10*A[3]) + c20*A[6], invdet = 1.0/det;
    R[0]=c00*invdet; R[1]=c10*invdet; R[2]=c20*invdet; R[3]=COF(0,1)*invdet; R[4]=COF(1,1)*invdet; R[5]=COF(2,1)*invdet; R[6]=COF(0,2)*invdet; R[7]=COF(1,2)*invdet; R[8]=COF(2,2)*invdet;
#undef COF
  }
}
}

extern "C" {

int sdv_reproject_grid(sdv_ctx* c, int* n_cols, int* n_rows) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG; if (n_cols) *n_cols = grid_dim(c->w); if (n_rows) *n_rows = grid_dim(c->h); return SDV_OK;
}

int sdv_map_set(sdv_ctx* c, int slot, int nH, const uint64_t* host_frames, const double* host_T7, const double* host_ab, int nP, const sdv_map_pt* pts) { SDV_GUARD_TRK(c);
  if (nH < 0 || nP < 0) return SDV_ERR_ARG;
  const int32_t hb[2] = {0, nH}, pb[2] = {0, nP};
  return map_set_impl(c, 1, &slot, hb, host_frames, host_T7, host_ab, pb, pts, cudaMemcpyHostToDevice);
}
int sdv_map_set_batch(sdv_ctx* c, int n, const int32_t* slots, const int32_t* host_begin, const uint64_t* host_frames, const double* host_T7,
                      const double* host_ab, const int32_t* pt_begin, const sdv_map_pt* pts) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n > 0 && (!slots || !host_begin || !pt_begin))) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK;
  return map_set_impl(c, n, slots, host_begin, host_frames, host_T7, host_ab, pt_begin, pts, cudaMemcpyHostToDevice);
}
}  // extern "C"
namespace sdv {
// the single staged upload of sdv_map_set_batch: segment k copies words[k] 4-byte words from src[k] to dst[k]; blockIdx.y strides over the segments
struct MapCopySeg { const uint32_t* src; uint32_t* dst; size_t words; };
__global__ void map_copy_kernel(const MapCopySeg* __restrict__ seg, int nseg) {
  for (int k = blockIdx.y; k < nseg; k += gridDim.y) { const MapCopySeg q = seg[k];
    for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < q.words; i += (size_t)gridDim.x*blockDim.x) q.dst[i] = q.src[i]; }
}
}
int sdv::map_set_impl(sdv_ctx* c, int n, const int32_t* slots, const int32_t* host_begin, const uint64_t* host_frames, const double* host_T7, const double* host_ab,
                      const int32_t* pt_begin, const sdv_map_pt* pts, cudaMemcpyKind kind) {
  if (!c) return SDV_ERR_ARG;
  // every check of every job before any slot, pin or buffer changes
  { int rc = check_offsets(c, n, host_begin, "sdv_map_set_batch", "host_begin"); if (rc) return rc; }
  { int rc = check_offsets(c, n, pt_begin, "sdv_map_set_batch", "pt_begin"); if (rc) return rc; }
  CK(cudaSetDevice(c->device)); RpState* st = rp_state(c);
  { int rc = check_ids(c, n, slots, (int)st->maps.size(), "sdv_map_set_batch", "slot"); if (rc) return rc; }
  std::vector<FrameDev*> F((size_t)host_begin[n]); long long need_seq = 0; size_t maxP = 0, totP = 0;
  for (int j = 0; j < n; j++) {
    const int nH = host_begin[j+1] - host_begin[j], nP = pt_begin[j+1] - pt_begin[j];
    if (nH < 1 || nH > kRpMaxHosts || !host_frames || !host_T7 || nP >= (1 << 27) || (nP > 0 && !pts)) return SDV_ERR_ARG;   // point index packs into 27 bits of the sort key
    for (int k = host_begin[j]; k < host_begin[j+1]; k++) { int rcs = job_frame(c, "sdv_map_set", k - host_begin[j], host_frames[k], -1, slots[j], &need_seq, &F[k]); if (rcs) return rcs; }
    maxP = std::max(maxP, (size_t)nP); totP += nP;
  }
  { int rcj = join_ingest(c); if (rcj) return rcj; }
  CK(cudaStreamSynchronize(c->st));                                            // host wait 1: a previous launch may still read the slots
  const bool staged = kind == cudaMemcpyHostToDevice;
  const size_t seg_bytes = Scratch::need(2*(size_t)n, sizeof(MapCopySeg)), dev_bytes = Scratch::need(n, sizeof(MapDev)) + (staged ? Scratch::need(totP, sizeof(sdv_map_pt)) : 0);
  if (c->scr.reserve(seg_bytes + dev_bytes, c->st) || c->scr_host.reserve(seg_bytes + dev_bytes, c->st)) return ctx_fail(c, SDV_ERR_CUDA, "sdv_map_set_batch: staging of %d maps", n);
  for (int j = 0; j < n; j++) {                                                  // room for the points (not visible until the slot is rewritten below)
    MapSlot& m = st->maps[slots[j]]; const int nP = pt_begin[j+1] - pt_begin[j];
    if (!m.dev) CK(cudaMalloc(&m.dev, sizeof(MapDev)));
    if (nP > m.cap) { cudaFree(m.pts); m.pts = nullptr; m.cap = nP + nP/4 + 256; CK(cudaMalloc(&m.pts, (size_t)m.cap*sizeof(sdv_map_pt))); }
  }
  // one pinned image of the upload, laid out as its device twin: segment table, the MapDev of every job, the points of every job
  c->scr.reset(); c->scr_host.reset();
  MapCopySeg* seg_d = c->scr.take<MapCopySeg>(2*(size_t)n); MapDev* md_d = c->scr.take<MapDev>(n); sdv_map_pt* pts_d = staged ? c->scr.take<sdv_map_pt>(totP) : nullptr;
  MapCopySeg* seg = c->scr_host.take<MapCopySeg>(2*(size_t)n); MapDev* md = c->scr_host.take<MapDev>(n); sdv_map_pt* pts_h = staged ? c->scr_host.take<sdv_map_pt>(totP) : nullptr;
  const size_t up_bytes = staged ? (size_t)((char*)(pts_h + totP) - (char*)seg) : (size_t)((char*)(md + n) - (char*)seg);
  int nseg = 0;
  for (int j = 0; j < n; j++) {
    MapSlot& m = st->maps[slots[j]]; const int h0 = host_begin[j], nH = host_begin[j+1] - h0, nP = pt_begin[j+1] - pt_begin[j];
    if (m.set) for (int k=0;k<m.nH;k++) frame_unpin(c, m.host_ids[k]);       // the slot's previous keyframes are no longer referenced by it
    for (int k=0;k<nH;k++) frame_pin(c, host_frames[h0+k]);
    MapDev& h = m.host_copy; memset(&h, 0, sizeof(h)); h.nH = nH; h.nP = nP; h.pts = m.pts; m.ingest_seq = need_seq;
    for (int k=0;k<nH;k++) {
      const FrameDev& f = *F[h0+k]; h.hostI0[k] = f.I0; m.host_exposure[k] = f.exposure; m.host_ids[k] = host_frames[h0+k];
      for (int i=0;i<7;i++) h.hostT[k][i] = host_T7[7*(h0+k)+i]; m.host_ab[k][0] = host_ab ? host_ab[2*(h0+k)] : 0.0; m.host_ab[k][1] = host_ab ? host_ab[2*(h0+k)+1] : 0.0; }
    m.nH = nH; m.nP = nP; m.set = true;
    md[j] = h; seg[nseg++] = MapCopySeg{(const uint32_t*)(md_d + j), (uint32_t*)m.dev, sizeof(MapDev)/4};
    if (nP) {
      const sdv_map_pt* src = pts + pt_begin[j];
      if (staged) { memcpy(pts_h + pt_begin[j], src, (size_t)nP*sizeof(sdv_map_pt)); src = pts_d + pt_begin[j]; }
      seg[nseg++] = MapCopySeg{(const uint32_t*)src, (uint32_t*)m.pts, (size_t)nP*sizeof(sdv_map_pt)/4};
    }
  }
  CK(cudaMemcpyAsync(seg_d, seg, up_bytes, cudaMemcpyHostToDevice, c->st));
  map_copy_kernel<<<dim3((unsigned)std::min<size_t>((maxP*sizeof(sdv_map_pt)/4 + 255)/256 + 1, 64), (unsigned)std::min(nseg, 65535)), 256, 0, c->st>>>(seg_d, nseg);
  c->launches += 1;
  CK(cudaGetLastError());
  CK(cudaStreamSynchronize(c->st));                                            // host wait 2: the upload has landed (the caller may reuse its rows)
  return SDV_OK;
}
extern "C" {

int sdv_map_clear(sdv_ctx* c, int slot) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); RpState* st = rp_state(c);
  if (slot < 0 || slot >= (int)st->maps.size()) return SDV_ERR_ARG;
  MapSlot& m = st->maps[slot]; if (!m.set) return SDV_OK;
  CK(cudaStreamSynchronize(c->st));                                            // a launch may still read the slot
  for (int k=0;k<m.nH;k++) frame_unpin(c, m.host_ids[k]); m.set = false; m.nH = 0; m.nP = 0; return SDV_OK;
}

// shared front half: builds the jobs, sizes the scratch and launches project / scan / scatter / match.  Results stay on the device.
struct RpRun { RpScratch S; RpJob* jobs_dev; RpJob* jobs_host; int32_t* h_opt; double2* h_opx; sdv_overlap_pt* ov; RefineJob* rj; RefineJob* rj_host; int* n_out_dev; int* n_out_host; int* cell_order_dev; long long nc; };
static int rp_launch(sdv_ctx* c, int n_jobs, const int32_t* slots, const uint64_t* cur_frames, const double* cur_T7, const double* cur_ab,
                     const int32_t* cur_kf_index, const int32_t* only_host, const int32_t* backup, RpRun& R) {
  RpState* st = rp_state(c); rp_job_K(c->geom[0].g[0], st->C.K, st->C.Ki);
  for (int k=0;k<SDV_MAX_CAMERAS;k++) { st->C.cam_w[k] = c->cam_w[k]; st->C.cam_h[k] = c->cam_h[k]; st->C.cam_levels[k] = c->cam_levels[k]; }
  const RpConst& C = st->C;
  long long totalP = 0; int maxP = 1;
  for (int k=0;k<n_jobs;k++) { if (slots[k] < 0 || slots[k] >= (int)st->maps.size() || !st->maps[slots[k]].set) return ctx_fail(c, SDV_ERR_STATE, "reproject job %d: map slot %d not set", k, slots[k]);
    totalP += st->maps[slots[k]].nP; maxP = std::max(maxP, st->maps[slots[k]].nP); }
  const long long nc = (long long)n_jobs*C.ncells; R.nc = nc;
  Scratch& D = c->scr; PinnedScratch& H = c->scr_host;
  const size_t d_bytes = Scratch::need(n_jobs, sizeof(RpJob)) + Scratch::need(totalP, sizeof(double2)) + 2*Scratch::need(totalP, 4) + Scratch::need(totalP, 8) + 4*Scratch::need(nc, 4)
                       + Scratch::need(nc, sizeof(double2)) + Scratch::need((size_t)n_jobs*kRpMaxHosts*14, sizeof(double)) + Scratch::need(nc, sizeof(sdv_overlap_pt))
                       + Scratch::need(n_jobs, sizeof(RefineJob)) + Scratch::need(n_jobs, 4) + Scratch::need(C.ncells, 4),
               h_bytes = Scratch::need(n_jobs, sizeof(RpJob)) + Scratch::need(nc, 4) + Scratch::need(nc, sizeof(double2)) + Scratch::need(n_jobs, sizeof(RefineJob)) + Scratch::need(n_jobs, 4);
  if (D.reserve(d_bytes, c->st) || H.reserve(h_bytes, c->st)) return ctx_fail(c, SDV_ERR_CUDA, "reproject / refine: scratch of %d jobs", n_jobs);
  D.reset(); H.reset();
  RpJob* J = H.take<RpJob>(n_jobs); R.jobs_host = J; R.h_opt = H.take<int32_t>(nc); R.h_opx = H.take<double2>(nc); R.rj_host = H.take<RefineJob>(n_jobs); R.n_out_host = H.take<int>(n_jobs);
  long long need_seq = 0; std::vector<FrameDev*> F(n_jobs);
  for (int k=0;k<n_jobs;k++) { int rcs = job_frame(c, "reproject / refine", k, cur_frames[k], -1, slots[k], &need_seq, &F[k]); if (rcs) return rcs;
    need_seq = std::max(need_seq, st->maps[slots[k]].ingest_seq); }
  { int rcj = join_ingest_upto(c, need_seq); if (rcj) return rcj; }     // only the uploads these frames came from (a later batch may still be streaming in)
  long long off = 0;
  for (int k=0;k<n_jobs;k++) {
    const MapSlot& m = st->maps[slots[k]]; RpJob& j = J[k]; memset(&j, 0, sizeof(j));
    const FrameDev& f = *F[k];
    j.map = m.dev; for (int l=0;l<c->levels;l++) j.cur[l] = f.img[l];
    rp_job_K(slot_geom(c, slots[k]).g[0], j.K, j.Ki); j.geom_row = c->slots[slots[k]].geom_row; j.cam = (unsigned char)c->slots[slots[k]].cam;
    for (int i=0;i<7;i++) j.curT[i] = cur_T7[7*k+i];
    const SE3d cur = se3_from7(j.curT); se3_to7(se3_inv(cur), j.curTinv);
    j.cur_kf_index = cur_kf_index ? cur_kf_index[k] : -1; j.backup = backup ? backup[k] : 0; j.nH = m.nH; j.nP = m.nP; j.pt_off = off; off += m.nP;
    const int oh = only_host ? only_host[k] : -1;
    // close_kfs (:123-131): keyframes in reverse index order, stable sort by distance to the target frame; the target itself is skipped (:138-139)
    std::pair<int,double> ck[kRpMaxHosts]; int nk = 0;
    for (int i = m.nH-1; i >= 0; i--) { const double d0 = cur.t[0]-m.host_copy.hostT[i][4], d1 = cur.t[1]-m.host_copy.hostT[i][5], d2 = cur.t[2]-m.host_copy.hostT[i][6]; ck[nk++] = {i, sqrt(d0*d0 + d1*d1 + d2*d2)}; }
    std::stable_sort(ck, ck + nk, [](const std::pair<int,double>& a, const std::pair<int,double>& b) { return a.second < b.second; });
    for (int i=0;i<kRpMaxHosts;i++) j.frame_rank[i] = -1;
    if (oh >= 0) { if (oh >= m.nH) return ctx_fail(c, SDV_ERR_ARG, "reproject job %d: only_host %d of %d", k, oh, m.nH); j.frame_rank[oh] = 0; }
    else { int r = 0; for (int e = 0; e < nk; e++) if (ck[e].first != j.cur_kf_index) j.frame_rank[ck[e].first] = r++; }
    const double ca = cur_ab ? cur_ab[2*k] : 0.0, cbb = cur_ab ? cur_ab[2*k+1] : 0.0;
    for (int i=0;i<m.nH;i++) { double o2[2]; aff_from_to(m.host_exposure[i], f.exposure, m.host_ab[i][0], m.host_ab[i][1], ca, cbb, o2); j.affLL[i][0] = (float)o2[0]; j.affLL[i][1] = (float)o2[1]; }
  }
  RpJob* jd = D.take<RpJob>(n_jobs); R.jobs_dev = jd;
  RpScratch& S = R.S; S.cand_px = D.take<double2>(totalP); S.cand_key = D.take<float>(totalP); S.cand_cell = D.take<int>(totalP); S.list = D.take<unsigned long long>(totalP);
  S.count = D.take<int>(nc); S.begin = D.take<int>(nc); S.cursor = D.take<int>(nc); S.out_pt = D.take<int>(nc); S.out_px = D.take<double2>(nc); S.xf = D.take<double>((size_t)n_jobs*kRpMaxHosts*14);
  R.ov = D.take<sdv_overlap_pt>(nc); R.rj = D.take<RefineJob>(n_jobs); R.n_out_dev = D.take<int>(n_jobs); R.cell_order_dev = D.take<int>(C.ncells);
  cudaStream_t s = c->st;
  launch_h2d_words(jd, J, (size_t)n_jobs*sizeof(RpJob), s);                      // kernel copy (see launch_h2d_words); need() leaves it its 16 B of slack
  CK(cudaMemsetAsync(S.count, 0, (size_t)nc*4, s));
  CK(cudaEventRecord(c->ev0, s));
  rp_project_kernel<<<dim3((maxP + 255)/256, n_jobs), 256, 0, s>>>(jd, C, S);
  rp_scan_kernel<<<n_jobs, 1024, 0, s>>>(C, S);
  rp_scatter_kernel<<<dim3((maxP + 255)/256, n_jobs), 256, 0, s>>>(jd, C, S);
  rp_match_kernel<<<dim3((C.ncells + kRpWarps - 1)/kRpWarps, n_jobs), 32*kRpWarps, 0, s>>>(jd, C, S);
  CK(cudaGetLastError()); c->launches += 5;
  return SDV_OK;
}

int sdv_reproject_map_batch(sdv_ctx* c, int n_jobs, const int32_t* slots, const uint64_t* cur_frames, const double* cur_T7, const double* cur_ab,
                            const int32_t* cur_kf_index, const int32_t* only_host, const int32_t* backup, const int32_t* cell_order, int max_matches,
                            int32_t* n_out, int32_t* out_pt, double* out_px) { SDV_GUARD_TRK(c);
  if (!c || n_jobs <= 0 || !slots || !cur_frames || !cur_T7 || !n_out || !out_pt || !out_px) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device)); RpRun R; { int rc = rp_launch(c, n_jobs, slots, cur_frames, cur_T7, cur_ab, cur_kf_index, only_host, backup, R); if (rc) return rc; }
  const RpConst& C = c->rp->C; cudaStream_t s = c->st; const long long nc = R.nc;
  CK(cudaEventRecord(c->ev1, s));
  CK(cudaMemcpyAsync(R.h_opt, R.S.out_pt, (size_t)nc*4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(R.h_opx, R.S.out_px, (size_t)nc*sizeof(double2), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(R.jobs_host, R.jobs_dev, (size_t)n_jobs*sizeof(RpJob), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s)); CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  for (int k=0;k<n_jobs;k++) {
    if (R.jobs_host[k].error) return ctx_fail(c, SDV_ERR_ARG, "reproject job %d: a map point names a host outside [0,%d)", k, R.jobs_host[k].nH);
    int n = 0, matches = 0; int32_t* op = out_pt + (size_t)k*C.ncells; double* ox = out_px + (size_t)k*C.ncells*2;
    const int jcols = grid_dim(C.cam_w[R.jobs_host[k].cam]), jrows = grid_dim(C.cam_h[R.jobs_host[k].cam]);
    for (int i=0;i<C.ncells;i++) { int cell = cell_order ? cell_order[i] : i; if (cell < 0 || cell >= C.ncells) return ctx_fail(c, SDV_ERR_ARG, "cell_order[%d] = %d", i, cell);
      cell = job_cell(cell, C.ncols, jcols, jrows); if (cell < 0) continue;
      const long long cb = (long long)k*C.ncells + cell;
      if (R.h_opt[cb] >= 0) { op[n] = R.h_opt[cb]; ox[2*n] = R.h_opx[cb].x; ox[2*n+1] = R.h_opx[cb].y; n++; matches++; }
      if (matches > max_matches) break; }                                      // Reprojector.cpp:151-153
    n_out[k] = n;
  }
  return SDV_OK;
}

int sdv_tracker_refine_batch(sdv_ctx* c, int n_jobs, const int32_t* slots, const uint64_t* cur_frames, double* curToWorld_io, const double* cur_ab,
                             const int32_t* cell_order, int max_matches, int32_t* n_matches, float* res, int32_t* iterations, int32_t* accepts) { SDV_GUARD_TRK(c);
  if (!c || n_jobs <= 0 || !slots || !cur_frames || !curToWorld_io) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device)); RpRun R; { int rc = rp_launch(c, n_jobs, slots, cur_frames, curToWorld_io, cur_ab, nullptr, nullptr, nullptr, R); if (rc) return rc; }
  const RpConst& C = c->rp->C; cudaStream_t s = c->st;
  if (cell_order) { for (int i=0;i<C.ncells;i++) if (cell_order[i] < 0 || cell_order[i] >= C.ncells) return ctx_fail(c, SDV_ERR_ARG, "cell_order[%d] = %d", i, cell_order[i]);
    CK(cudaMemcpyAsync(R.cell_order_dev, cell_order, (size_t)C.ncells*4, cudaMemcpyHostToDevice, s)); }
  rp_emit_kernel<<<n_jobs, 1024, 0, s>>>(R.jobs_dev, C, R.S, cell_order ? R.cell_order_dev : nullptr, max_matches, R.ov, R.rj, R.n_out_dev);
  launch_struct_pose(R.rj, n_jobs, R.ov, nullptr, c->geom_dev, s);
  CK(cudaGetLastError()); c->launches += 2;
  CK(cudaEventRecord(c->ev1, s));
  CK(cudaMemcpyAsync(R.rj_host, R.rj, (size_t)n_jobs*sizeof(RefineJob), cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(R.n_out_host, R.n_out_dev, (size_t)n_jobs*4, cudaMemcpyDeviceToHost, s));
  CK(cudaMemcpyAsync(R.jobs_host, R.jobs_dev, (size_t)n_jobs*sizeof(RpJob), cudaMemcpyDeviceToHost, s));
  CK(cudaStreamSynchronize(s)); CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  for (int k=0;k<n_jobs;k++) {
    if (R.jobs_host[k].error) return ctx_fail(c, SDV_ERR_ARG, "refine job %d: a map point names a host outside [0,%d)", k, R.jobs_host[k].nH);
    for (int i=0;i<7;i++) curToWorld_io[7*k+i] = R.rj_host[k].T[i];
    if (n_matches) n_matches[k] = R.n_out_host[k]; if (res) res[k] = R.rj_host[k].res; if (iterations) iterations[k] = R.rj_host[k].iterations; if (accepts) accepts[k] = R.rj_host[k].accepts;
  }
  return SDV_OK;
}

} // extern "C"
