// sdv_lidar_core.cuh — LiDAR front-end of the node on the device (SURVEY.md §8f rank 3, second half), all file:line in /root/reference/src/main.cpp:
//
//   projectPointCloud   :563-607   -> lf_project_kernel (thread per return: ring / azimuth cell, the LAST return written to a cell wins = atomicMax of the input index)
//                                     lf_gather_kernel  (thread per cell: range image + organised cloud; an empty cell holds the point (0,0,0), intensity 0 — `nanPoint` is never
//                                     initialised in the reference, main.cpp:84, so PCL's default point takes part in the ground test)
//   groundRemoval       :609-655   -> lf_ground_kernel (thread per azimuth column, the 50 vertical pairs in order)
//   labelComponents / cloudSegmentation :657-783 -> the BFS of the reference grows connected components of a symmetric relation (range-difference angle > 60 deg over
//                                     the 4-neighbourhood, columns wrap), so the segmentation is a connected-component labelling: lock-free union-find (lf_union_kernel, roots =
//                                     smallest raster index = the BFS seed), component size and row set by atomics (lf_stats_kernel; the seed itself does not count towards
//                                     the row set, like lineCountFlag), feasibility = size >= 30 or (size >= 5 and >= 3 rows)
//   lidarCloudHandler   :785-858   -> lf_keep_kernel (Rlc p + tlc in fp64, pinhole projection in float, image bounds), lf_scan_kernel (raster-order compaction),
//                                     lf_emit_kernel (rows {Ku, Kv, depth}, running pixel box by atomicMin/Max, ground count -> addFeaturePoint)
// Two host paths share the nine launches: handle() copies the rows and the box back and waits; handle_rows() (the row sets of sdv_lidar.cu) writes the rows into a
// caller-owned device block, seeds the box from device memory (lf_rows_seed_kernel), writes a header and the box back (lf_rows_finalize_kernel) and need not wait.
// Float math: the reference's build resolves atan2 / sqrt / sin / cos of floats to the float overloads (FullSystem.h:19 includes <math.h>).  sqrtf and the divisions are IEEE
// on both sides; atan2f is NOT specified by IEEE, so the device carries a restatement of the C library's algorithm (fdlibm e_atan2f.c / s_atanf.c — float operations
// only, bit-identical to glibc 2.39's atan2f on 2e7 random arguments, tests/test_select_emu_cpu.py::test_atan2f_matches_libm); sinf / cosf are only ever taken of the two
// angular resolutions and come from the host's libm through the settings.  Results are bit-identical to the CPU code.
#pragma once
#include "sdv_core_common.cuh"
#include <float.h>

namespace sdv { namespace lidar {

struct LidarSet { int N, H; float ang_res_x, ang_res_y, ang_bottom; int groundScanInd; float sensorMountAngle, segmentTheta, sinX, cosX, sinY, cosY; int validPointNum, validLineNum; };
struct LidarJob {
  const float4* pts; int n;                                  // one raw sweep, XYZI rows
  int* cellIdx; float* range; float4* cloud; signed char* ground; int* parent; int* csize; unsigned long long* rowmask;   // per cell (rowmask: 2 words per cell, N <= 128)
  unsigned char* flag; int* pos; float* kuv;                 // per cell: survives the projection, its output row, {Ku, Kv}
  double R[9], t[3]; float fx, fy, cx, cy; int w, h;
  double* out3; int cap; int* counters;                      // counters: [0] rows out [1] numGround [2] left [3] right [4] up [5] down [6] size of segmentedCloud
};

__device__ __forceinline__ int f2i_(float x) { return __float_as_int(x); }
__device__ __forceinline__ float i2f_(int i) { return __int_as_float(i); }
// ---- atanf / atan2f of the C library (fdlibm s_atanf.c, e_atan2f.c), float operations in the library's order
__device__ float lib_atanf(float x) {
  const float atanhi[4] = {4.6364760399e-01f, 7.8539812565e-01f, 9.8279368877e-01f, 1.5707962513e+00f};
  const float atanlo[4] = {5.0121582440e-09f, 3.7748947079e-08f, 3.4473217170e-08f, 7.5497894159e-08f};
  const float aT[11] = {3.3333334327e-01f, -2.0000000298e-01f, 1.4285714924e-01f, -1.1111110449e-01f, 9.0908870101e-02f, -7.6918758452e-02f, 6.6610731184e-02f, -5.8335702866e-02f,
                        4.9768779427e-02f, -3.6531571299e-02f, 1.6285819933e-02f};
  const float one = 1.0f, huge = 1.0e30f;
  float w, s1, s2, z; int ix, hx, id; hx = f2i_(x); ix = hx & 0x7fffffff;
  if (ix >= 0x4c000000) { if (ix > 0x7f800000) return x + x; if (hx > 0) return atanhi[3] + atanlo[3]; else return -atanhi[3] - atanlo[3]; }
  if (ix < 0x3ee00000) { if (ix < 0x31000000) { if (huge + x > one) return x; } id = -1; }
  else { x = fabsf(x);
    if (ix < 0x3f980000) { if (ix < 0x3f300000) { id = 0; x = (2.0f*x - one)/(2.0f + x); } else { id = 1; x = (x - one)/(x + one); } }
    else { if (ix < 0x401c0000) { id = 2; x = (x - 1.5f)/(one + 1.5f*x); } else { id = 3; x = -1.0f/x; } } }
  z = x*x; w = z*z;
  s1 = z*(aT[0] + w*(aT[2] + w*(aT[4] + w*(aT[6] + w*(aT[8] + w*aT[10])))));
  s2 = w*(aT[1] + w*(aT[3] + w*(aT[5] + w*(aT[7] + w*aT[9]))));
  if (id < 0) return x - x*(s1 + s2);
  z = atanhi[id] - ((x*(s1 + s2) - atanlo[id]) - x); return (hx < 0) ? -z : z;
}
__device__ float lib_atan2f(float y, float x) {
  const float tiny = 1.0e-30f, pi_o_4 = 7.8539818525e-01f, pi_o_2 = 1.5707963705e+00f, pi = 3.1415927410e+00f, pi_lo = -8.7422776573e-08f;
  float z; int k, m, hx, hy, ix, iy; hx = f2i_(x); ix = hx & 0x7fffffff; hy = f2i_(y); iy = hy & 0x7fffffff;
  if ((ix > 0x7f800000) || (iy > 0x7f800000)) return x + y;
  if (hx == 0x3f800000) return lib_atanf(y);
  m = ((hy >> 31) & 1) | ((hx >> 30) & 2);
  if (iy == 0) { if (m < 2) return y; return (m == 2) ? pi + tiny : -pi - tiny; }
  if (ix == 0) return (hy < 0) ? -pi_o_2 - tiny : pi_o_2 + tiny;
  if (ix == 0x7f800000) {
    if (iy == 0x7f800000) return (m == 0) ? pi_o_4 + tiny : (m == 1) ? -pi_o_4 - tiny : (m == 2) ? 3.0f*pi_o_4 + tiny : -3.0f*pi_o_4 - tiny;
    return (m == 0) ? 0.0f : (m == 1) ? -0.0f : (m == 2) ? pi + tiny : -pi - tiny; }
  if (iy == 0x7f800000) return (hy < 0) ? -pi_o_2 - tiny : pi_o_2 + tiny;
  k = (iy - ix) >> 23;
  if (k > 60) z = pi_o_2 + 0.5f*pi_lo; else if (hx < 0 && k < -60) z = 0.0f; else z = lib_atanf(fabsf(y/x));
  if (m == 0) return z;
  if (m == 1) return i2f_(f2i_(z) ^ (int)0x80000000);
  if (m == 2) return pi - (z - pi_lo);
  return (z - pi_lo) - pi;
}
#ifdef SDV_EMU
static inline float emu_lib_atan2f(float y, float x) { return lib_atan2f(y, x); }
#endif

__global__ void __launch_bounds__(128) lf_project_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {       // thread per return (main.cpp:563-607; NaN rows dropped like :792)
  const LidarJob J = jobs[blockIdx.y]; const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= J.n) return;
  const float4 p = J.pts[i]; const float x = p.x, y = p.y, z = p.z;
  if (!isfinite(x) || !isfinite(y) || !isfinite(z)) return;
  const float verticalAngle = (float)((double)(lib_atan2f(z, sqrtf(x*x + y*y)) * 180) / M_PI);
  const float rowf = (verticalAngle + S.ang_bottom) / S.ang_res_y;
  if (!(rowf > -1.0f)) return;                                                            // size_t rowIdn: anything <= -1 is a huge index
  const long long row = (long long)rowf; if (row >= S.N) return;
  const float horizonAngle = (float)((double)(lib_atan2f(x, y) * 180) / M_PI);
  const double cold = -round(((double)horizonAngle - 90.0) / (double)S.ang_res_x) + (double)(S.H/2);
  if (!(cold > -1.0)) return;
  long long col = (long long)cold; if (col >= S.H) col -= S.H;
  if (col >= S.H) return;
  const float rng = sqrtf(x*x + y*y + z*z);
  if ((double)rng < 0.1) return;
  atomicMax(&J.cellIdx[(int)col + (int)row*S.H], i);
}
__global__ void __launch_bounds__(128) lf_gather_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {        // thread per cell
  const LidarJob J = jobs[blockIdx.y]; const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= S.N*S.H) return;
  const int i = J.cellIdx[k]; float rng = FLT_MAX; float4 c = make_float4(0.f, 0.f, 0.f, 0.f);
  if (i >= 0) { const float4 p = J.pts[i]; const int row = k / S.H, col = k - row*S.H; rng = sqrtf(p.x*p.x + p.y*p.y + p.z*p.z);
    c = make_float4(p.x, p.y, p.z, (float)((double)(float)row + (double)(float)col / 10000.0)); }
  J.range[k] = rng; J.cloud[k] = c; J.ground[k] = 0;
}
__global__ void __launch_bounds__(128) lf_ground_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {        // thread per column (:617-640)
  const LidarJob J = jobs[blockIdx.y]; const int j = blockIdx.x*blockDim.x + threadIdx.x; if (j >= S.H) return;
  float4 lo = J.cloud[j];
  for (int i = 0; i < S.groundScanInd; i++) {
    const float4 up = J.cloud[j + (i+1)*S.H];
    if (lo.w == -1 || up.w == -1) { J.ground[j + i*S.H] = -1; lo = up; continue; }
    const float dX = up.x - lo.x, dY = up.y - lo.y, dZ = up.z - lo.z;
    const float angle = (float)((double)(lib_atan2f(dZ, sqrtf(dX*dX + dY*dY)) * 180) / M_PI);
    if (fabsf(angle - S.sensorMountAngle) <= 10) { J.ground[j + i*S.H] = 1; J.ground[j + (i+1)*S.H] = 1; }
    lo = up;
  }
}
__device__ __forceinline__ bool lf_valid(const LidarJob& J, int k) { return !(J.ground[k] == 1 || J.range[k] == FLT_MAX); }      // labelMat == 0 after groundRemoval (:642-648)
__global__ void __launch_bounds__(128) lf_cc_init_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {
  const LidarJob J = jobs[blockIdx.y]; const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= S.N*S.H) return;
  J.parent[k] = lf_valid(J, k) ? k : -1; J.csize[k] = 0; J.rowmask[2*k] = 0ull; J.rowmask[2*k+1] = 0ull;
}
__device__ __forceinline__ int lf_find(volatile int* parent, int x) { int p; while ((p = parent[x]) != x) x = p; return x; }
__device__ __forceinline__ void lf_union(int* parent, int a, int b) {                     // the larger root is hooked under the smaller: the root of a component is its smallest raster index
  for (;;) { a = lf_find(parent, a); b = lf_find(parent, b); if (a == b) return; if (a < b) { const int t = a; a = b; b = t; }
    const int old = atomicMin(&parent[a], b); if (old == a) return; a = old; }
}
__device__ __forceinline__ bool lf_connected(const LidarJob& J, const LidarSet& S, int k0, int k1, bool horizontal) {   // :702-713
  const float r0 = J.range[k0], r1 = J.range[k1], d1 = fmaxf(r0, r1), d2 = fminf(r0, r1);
  const float sa = horizontal ? S.sinX : S.sinY, ca = horizontal ? S.cosX : S.cosY;
  return lib_atan2f(d2*sa, (d1 - d2*ca)) > S.segmentTheta;
}
__global__ void __launch_bounds__(128) lf_union_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {         // thread per cell: its right (wrapping) and lower neighbour
  const LidarJob J = jobs[blockIdx.y]; const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= S.N*S.H) return;
  if (J.parent[k] < 0) return;
  const int row = k / S.H, col = k - row*S.H;
  const int kr = row*S.H + ((col + 1 >= S.H) ? 0 : col + 1);
  if (S.H > 1 && kr != k && J.parent[kr] >= 0 && lf_connected(J, S, k, kr, true)) lf_union(J.parent, k, kr);
  if (row + 1 < S.N) { const int kd = k + S.H; if (J.parent[kd] >= 0 && lf_connected(J, S, k, kd, false)) lf_union(J.parent, k, kd); }
}
__global__ void __launch_bounds__(128) lf_stats_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {         // thread per cell
  const LidarJob J = jobs[blockIdx.y]; const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= S.N*S.H) return;
  if (J.parent[k] < 0) return;
  const int root = lf_find(J.parent, k), row = k / S.H;
  atomicAdd(&J.csize[root], 1);
  if (k != root) atomicOr(&J.rowmask[2*root + (row >> 6)], 1ull << (row & 63));                                   // lineCountFlag is set for pushed neighbours only (:723)
  J.pos[k] = root;                                                                                                // remembered for lf_keep_kernel (parent[] keeps changing under path walks? no: read-only from here)
}
__global__ void __launch_bounds__(128) lf_keep_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {          // thread per cell (:754-783, :806-849)
  const LidarJob J = jobs[blockIdx.y]; const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= S.N*S.H) return;
  const bool ground = J.ground[k] == 1; bool keep = ground;
  if (!keep && J.parent[k] >= 0) { const int root = J.pos[k], sz = J.csize[root];
    keep = sz >= 30 || (sz >= S.validPointNum && (__popcll(J.rowmask[2*root]) + __popcll(J.rowmask[2*root+1])) >= S.validLineNum); }
  unsigned char f = 0;
  if (keep) {
    atomicAdd(&J.counters[6], 1);
    const float4 c = J.cloud[k]; const double p0 = c.x, p1 = c.y, p2 = c.z; double tmp[3];
#pragma unroll
    for (int r = 0; r < 3; r++) tmp[r] = ((J.R[3*r]*p0 + J.R[3*r+1]*p1) + J.R[3*r+2]*p2) + J.t[r];
    if (!(tmp[2] < 0.2)) {
      const float u = (float)(tmp[0] / tmp[2]), v = (float)(tmp[1] / tmp[2]); const float Ku = u*J.fx + J.cx, Kv = v*J.fy + J.cy;
      if (!((int)Ku < 4 || (int)Ku >= J.w-5 || (int)Kv < 4 || (int)Kv > J.h-4)) { f = ground ? 2 : 1; J.kuv[2*k] = Ku; J.kuv[2*k+1] = Kv; }
    }
  }
  J.flag[k] = f;
}
__global__ void __launch_bounds__(256) lf_scan_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {          // CTA per job: raster-order output rows
  const LidarJob J = jobs[blockIdx.x]; const int n = S.N*S.H;
  __shared__ int sm[512]; __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int s0 = 0; s0 < n; s0 += blockDim.x*8) {
    const int s = s0 + threadIdx.x*8; int loc[8], sum = 0;
    for (int k = 0; k < 8; k++) { loc[k] = (s+k < n && J.flag[s+k]) ? 1 : 0; sum += loc[k]; }
    int total; int ex = sel::block_excl_scan(sum, sm, total) + base;
    for (int k = 0; k < 8; k++) { if (s+k < n) J.pos[s+k] = ex; ex += loc[k]; }
    __syncthreads();
    if (threadIdx.x == 0) base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) J.counters[0] = base;
}
__global__ void __launch_bounds__(128) lf_emit_kernel(const LidarJob* __restrict__ jobs, LidarSet S) {          // thread per cell
  const LidarJob J = jobs[blockIdx.y]; const int k = blockIdx.x*blockDim.x + threadIdx.x; if (k >= S.N*S.H) return;
  const unsigned char f = J.flag[k]; if (!f) return;
  const float Ku = J.kuv[2*k], Kv = J.kuv[2*k+1]; const int m = J.pos[k];
  if (m < J.cap) { const float4 c = J.cloud[k]; const double depth = ((J.R[6]*(double)c.x + J.R[7]*(double)c.y) + J.R[8]*(double)c.z) + J.t[2];
    J.out3[3*m] = (double)Ku; J.out3[3*m+1] = (double)Kv; J.out3[3*m+2] = depth; }
  atomicMin(&J.counters[2], (int)Ku); atomicMax(&J.counters[3], (int)Ku); atomicMin(&J.counters[4], (int)Kv); atomicMax(&J.counters[5], (int)Kv);   // :834-837 in closed form (Ku, Kv >= 4)
  if (f == 2) atomicAdd(&J.counters[1], 1);
}

// ---- device-output path (sdv_lidar_handler_rows_batch): the rows go straight into a row set's block, the running pixel box is read from and written back to
// device memory (the selector slot's), and nothing waits for the device
struct RowsHdr { int rows, overflow, left, right, up, down, addFeaturePoint, numGround, n_segmented, pad_[7]; };   // 64 B ahead of the block's rows; rows: the true count
struct RowsJob { int* counters; int* box; RowsHdr* hdr; int cap; };
__global__ void __launch_bounds__(128) lf_rows_seed_kernel(const RowsJob* __restrict__ jobs, int nj) {            // thread per sweep: the box as the previous sweep left it
  const int j = blockIdx.x*blockDim.x + threadIdx.x; if (j >= nj) return;
  const RowsJob R = jobs[j];
  for (int k = 0; k < 4; k++) R.counters[2+k] = R.box[k];
}
__global__ void __launch_bounds__(128) lf_rows_finalize_kernel(const RowsJob* __restrict__ jobs, int nj) {        // thread per sweep: header + the slot's new box
  const int j = blockIdx.x*blockDim.x + threadIdx.x; if (j >= nj) return;
  const RowsJob R = jobs[j]; const int* c = R.counters; RowsHdr h;
  h.rows = c[0]; h.overflow = c[0] > R.cap ? 1 : 0; h.left = c[2]; h.right = c[3]; h.up = c[4]; h.down = c[5]; h.numGround = c[1]; h.n_segmented = c[6];
  h.addFeaturePoint = ((float)c[1] / (float)c[0] > 0.8) ? 1 : 0;                                                     // :851-854, the host path's expression (0/0: NaN, 0)
  for (int k = 0; k < 7; k++) h.pad_[k] = 0;
  *R.hdr = h;
  for (int k = 0; k < 4; k++) R.box[k] = c[2+k];
}
#ifdef SDV_EMU
static inline cudaError_t cudaStreamWaitEvent(cudaStream_t, cudaEvent_t, unsigned) { return 0; }                   // one host thread: every copy and launch is in order already
#endif

// ================================================================================================ host engine
struct LidarEngine {
  LidarSet S; cudaStream_t st = nullptr; std::string err; Scratch io; long long launches = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr; bool have_ev = false; float last_kernel_ms = 0.f;   // device time of the nine launches of the last handle() (copies excluded)
  cudaStream_t st_up = nullptr;                                                                 // copy stream of the device-output path's sweep uploads (nullptr: st)
  cudaEvent_t ev_up = nullptr, ev_done = nullptr; bool have_sync_ev = false;                    // uploads done / the kernels of the last call done (they read the staging)
  // sinf / cosf of the two angular resolutions come from the host's libm (only these four values are ever needed)
  void init(int n_scan, int horizon, float ang_res_x, float ang_res_y, float ang_bottom, int groundScanInd, cudaStream_t st_) {
    if (!have_ev) { have_ev = (cudaEventCreate(&ev0) == cudaSuccess && cudaEventCreate(&ev1) == cudaSuccess); }
    if (!have_sync_ev) { have_sync_ev = (cudaEventCreate(&ev_up) == cudaSuccess && cudaEventCreate(&ev_done) == cudaSuccess); }
    st = st_; S.N = n_scan; S.H = horizon; S.ang_res_x = ang_res_x; S.ang_res_y = ang_res_y; S.ang_bottom = ang_bottom; S.groundScanInd = groundScanInd; S.sensorMountAngle = 0.0f;
    S.segmentTheta = (float)(60.0/180.0*M_PI); const float ax = (float)(ang_res_x / 180.0 * M_PI), ay = (float)(ang_res_y / 180.0 * M_PI);           // main.cpp:118-122
    S.sinX = sinf(ax); S.cosX = cosf(ax); S.sinY = sinf(ay); S.cosY = cosf(ay); S.validPointNum = 5; S.validLineNum = 3;
  }
  void destroy() { io.release(); if (have_ev) { cudaEventDestroy(ev0); cudaEventDestroy(ev1); have_ev = false; }
                   if (have_sync_ev) { cudaEventDestroy(ev_up); cudaEventDestroy(ev_done); have_sync_ev = false; } }
  struct Sweep { const float* xyzi_host; int n; double R[9], t[3]; float K[4]; int w, h; int lrud[4];      // in (lrud: FullSystem::left/right/up/down, updated)
                 double* out3_host; int cap; int n_out, numGround, n_segmented, addFeaturePoint;          // out
                 int* box_dev = nullptr; RowsHdr* hdr_dev = nullptr; double* out3_dev = nullptr; };      // device-output path: the slot's box, the row set's header and rows
  // host path: waits, copies the rows to out3_host and the box to lrud
  int handle(std::vector<Sweep>& sw) {
    const int nj = (int)sw.size(); if (!nj) return 0;
    std::vector<LidarJob> J; int* counters_all = nullptr;
    if (enqueue(sw, false, st, J, counters_all)) return -1;
    std::vector<int> cnt((size_t)nj*8);
    SEL_CK(cudaMemcpyAsync(cnt.data(), counters_all, cnt.size()*sizeof(int), cudaMemcpyDeviceToHost, st));
    SEL_CK(cudaStreamSynchronize(st));
    if (have_ev) cudaEventElapsedTime(&last_kernel_ms, ev0, ev1);
    for (int j = 0; j < nj; j++) { Sweep& s = sw[j]; const int* c = &cnt[8*j]; s.n_out = c[0]; s.numGround = c[1]; for (int k = 0; k < 4; k++) s.lrud[k] = c[2+k]; s.n_segmented = c[6];
      s.addFeaturePoint = ((float)s.numGround / (float)s.n_out > 0.8) ? 1 : 0;                                 // :851-854
      if (s.n_out > s.cap) { err = "lidar: output capacity too small"; return -2; }
      if (s.n_out) SEL_CK(cudaMemcpyAsync(s.out3_host, J[j].out3, 3*(size_t)s.n_out*sizeof(double), cudaMemcpyDeviceToHost, st)); }
    SEL_CK(cudaStreamSynchronize(st));
    return 0;
  }
  // device-output path: sweep j's rows go to sw[j].out3_dev (at most cap), its header to hdr_dev, the box is read from and written back to box_dev (4 ints).
  // stats5 == nullptr: enqueue and return; else wait and fill {rows, numGround, n_segmented, addFeaturePoint, overflow} per sweep
  int handle_rows(std::vector<Sweep>& sw, int* stats5) {
    const int nj = (int)sw.size(); if (!nj) return 0;
    std::vector<LidarJob> J; int* counters_all = nullptr;
    if (enqueue(sw, true, st_up ? st_up : st, J, counters_all)) return -1;
    if (!stats5) return 0;
    std::vector<int> cnt((size_t)nj*8);
    SEL_CK(cudaMemcpyAsync(cnt.data(), counters_all, cnt.size()*sizeof(int), cudaMemcpyDeviceToHost, st));
    SEL_CK(cudaStreamSynchronize(st));
    if (have_ev) cudaEventElapsedTime(&last_kernel_ms, ev0, ev1);
    for (int j = 0; j < nj; j++) { const int* c = &cnt[8*j]; int* o = stats5 + 5*j;
      o[0] = c[0]; o[1] = c[1]; o[2] = c[6]; o[3] = ((float)c[1] / (float)c[0] > 0.8) ? 1 : 0; o[4] = c[0] > sw[j].cap ? 1 : 0; }
    return 0;
  }
  // scratch, job table, sweep uploads (on `up`; the kernels wait for them by event when up != st) and the nine launches of one call; rows: the device-output
  // path (rows into out3_dev, box seeded from and written back to box_dev, header)
  int enqueue(std::vector<Sweep>& sw, bool rows, cudaStream_t up, std::vector<LidarJob>& J, int*& counters_all) {
    const int nj = (int)sw.size();
    if (S.N > 128 || S.groundScanInd >= S.N) { err = "lidar: at most 128 rings, groundScanInd < rings"; return -1; }
    const size_t m = (size_t)S.N*S.H; size_t bytes = Scratch::need(nj, sizeof(LidarJob)) + Scratch::need(nj, sizeof(RowsJob)) + 1024;
    for (auto& s : sw) bytes += Scratch::need(std::max(s.n, 1), 16) + 5*Scratch::need(m, 4) + Scratch::need(m, 16) + 2*Scratch::need(m, 1) + Scratch::need(2*m, 8) + Scratch::need(2*m, 4)
                              + (rows ? 0 : Scratch::need(3*(size_t)s.cap, 8)) + Scratch::need(8, 4) + 1024;
    if (io.reserve(bytes, st)) { err = "scratch"; return -1; }
    io.reset(); J.assign(nj, LidarJob()); LidarJob* dJ = io.take<LidarJob>(nj); RowsJob* dR = io.take<RowsJob>(nj); int maxN = 0;
    // per-type arrays of all sweeps back to back: one memset / one counter upload / one counter read-back per call instead of one per sweep
    int* cellIdx_all = io.take<int>(m*nj); counters_all = io.take<int>((size_t)8*nj); std::vector<int> c0((size_t)8*nj, 0); std::vector<RowsJob> R(rows ? nj : 0);
    size_t tot_pts = 0; for (auto& s : sw) tot_pts += (size_t)std::max(s.n, 0);
    float4* pts_all = io.take<float4>(std::max(tot_pts, (size_t)1)); size_t off = 0;
    if (up != st && have_sync_ev) SEL_CK(cudaStreamWaitEvent(up, ev_done, 0));            // the staging is rewritten only after the last call's kernels have read it
    for (int j = 0; j < nj; j++) { Sweep& s = sw[j]; LidarJob& L = J[j];
      float4* pts = pts_all + off;
      if (s.n) {                                              // sweeps that follow each other in host memory (the C-ABI's layout) travel in ONE copy
        int j2 = j; size_t run = (size_t)s.n;
        const bool starts_run = (j == 0) || !(sw[j-1].n > 0 && sw[j-1].xyzi_host + 4*(size_t)sw[j-1].n == s.xyzi_host);
        if (starts_run) { while (j2 + 1 < nj && sw[j2+1].n > 0 && sw[j2].xyzi_host + 4*(size_t)sw[j2].n == sw[j2+1].xyzi_host) { j2++; run += (size_t)sw[j2].n; }
          SEL_CK(cudaMemcpyAsync(pts, s.xyzi_host, run*16, cudaMemcpyHostToDevice, up)); }
      }
      off += (size_t)std::max(s.n, 0);
      L.pts = pts; L.n = s.n; L.cellIdx = cellIdx_all + (size_t)j*m; L.range = io.take<float>(m); L.cloud = io.take<float4>(m); L.ground = io.take<signed char>(m); L.parent = io.take<int>(m); L.csize = io.take<int>(m);
      L.rowmask = io.take<unsigned long long>(2*m); L.flag = io.take<unsigned char>(m); L.pos = io.take<int>(m); L.kuv = io.take<float>(2*m);
      for (int k = 0; k < 9; k++) L.R[k] = s.R[k]; for (int k = 0; k < 3; k++) L.t[k] = s.t[k]; L.fx = s.K[0]; L.fy = s.K[1]; L.cx = s.K[2]; L.cy = s.K[3]; L.w = s.w; L.h = s.h;
      L.out3 = rows ? s.out3_dev : io.take<double>(3*(size_t)std::max(s.cap, 1)); L.cap = s.cap; L.counters = counters_all + 8*j;
      if (rows) R[j] = RowsJob{L.counters, s.box_dev, s.hdr_dev, s.cap};
      else for (int k = 0; k < 4; k++) c0[8*j+2+k] = s.lrud[k];
      maxN = std::max(maxN, s.n); }
    if (up != st) { SEL_CK(cudaEventRecord(ev_up, up)); SEL_CK(cudaStreamWaitEvent(st, ev_up, 0)); }
    SEL_CK(cudaMemcpyAsync(counters_all, c0.data(), c0.size()*sizeof(int), cudaMemcpyHostToDevice, st)); SEL_CK(cudaMemsetAsync(cellIdx_all, 0xFF, m*nj*sizeof(int), st));
    SEL_CK(cudaMemcpyAsync(dJ, J.data(), nj*sizeof(LidarJob), cudaMemcpyHostToDevice, st));
    if (rows) { SEL_CK(cudaMemcpyAsync(dR, R.data(), nj*sizeof(RowsJob), cudaMemcpyHostToDevice, st));
                SDV_LAUNCH(lf_rows_seed_kernel, dim3((nj + 127)/128), dim3(128), st, dR, nj); launches += 1; }
    const dim3 gc((unsigned)((m + 127)/128), nj), b128(128);
    if (have_ev) cudaEventRecord(ev0, st);
    if (maxN > 0) SDV_LAUNCH(lf_project_kernel, dim3((maxN + 127)/128, nj), b128, st, dJ, S);
    SDV_LAUNCH(lf_gather_kernel, gc, b128, st, dJ, S);
    SDV_LAUNCH(lf_ground_kernel, dim3((S.H + 127)/128, nj), b128, st, dJ, S);
    SDV_LAUNCH(lf_cc_init_kernel, gc, b128, st, dJ, S);
    SDV_LAUNCH(lf_union_kernel, gc, b128, st, dJ, S);
    SDV_LAUNCH(lf_stats_kernel, gc, b128, st, dJ, S);
    SDV_LAUNCH(lf_keep_kernel, gc, b128, st, dJ, S);
    SDV_LAUNCH_SYNC(lf_scan_kernel, dim3(nj), dim3(256), st, dJ, S);
    SDV_LAUNCH(lf_emit_kernel, gc, b128, st, dJ, S);
    if (have_ev) cudaEventRecord(ev1, st);
    launches += 9;
    if (rows) { SDV_LAUNCH(lf_rows_finalize_kernel, dim3((nj + 127)/128), dim3(128), st, dR, nj); launches += 1; }
    if (have_sync_ev) SEL_CK(cudaEventRecord(ev_done, st));
    SEL_CK(cudaGetLastError());
    return 0;
  }
  // debugging / test read-back of the images of job 0 of the last call is not kept: tests compare the pixel rows, the box, the counts
};

}}  // namespace sdv::lidar
