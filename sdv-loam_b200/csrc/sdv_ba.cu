// sdv_ba.cu — host side of the sliding-window back-end: window upload (the makeIDX mirror), the Gauss-Newton loop of
// FullSystem::optimize (FullSystemOptimize.cpp:344-502) driven over the kernels of sdv_ba_kernels.cu, and the C-ABI.
// Only control flow lives here (accept/reject, lambda schedule, break test); every number is produced on the device.
#include "../../include/sdv_b200.h"
#include "sdv_ctx.cuh"
#include "sdv_ba.cuh"
#include <stdlib.h>
#include <cstring>
#include <cstddef>
#include <vector>
#include <algorithm>
#include <cmath>

using namespace sdv;

namespace sdv {
void ba_destroy(sdv_ctx* c) {
  if (!c) return;
  for (BAState* b : c->ba_windows) { if (!b) continue;
    for (int i=0;i<b->n_pinned;i++) frame_unpin(c, b->pinned[i]);
    cudaFree(b->hdr); cudaFreeHost(b->hdr_host); cudaFree(b->pool); cudaFree(b->partials); cudaFree(b->thbuf); cudaFree(b->thcount); delete b; }
  c->ba_windows.clear(); c->ba = nullptr;
  c->ba_wins_dev.release(); c->ba_wins_host.release(); c->ba_scr.release(); c->ba_scr_host.release();
  if (c->ba_graph) { cudaGraphExecDestroy(c->ba_graph); c->ba_graph = nullptr; }
}
}

constexpr int kMaxWindows = (1<<20) + 1;                                     // window indices 0 .. 1<<20
// the state of window `window` (sdv_ba_select numbering), created on first use
static int ba_window(sdv_ctx* c, int window, BAState** out) {
  if (window < 0 || window >= kMaxWindows) return SDV_ERR_ARG;
  if ((int)c->ba_windows.size() <= window) c->ba_windows.resize(window+1, nullptr);
  if (!c->ba_windows[window]) {
    BAState* b = new BAState(); memset(b, 0, sizeof(*b)); c->ba_windows[window] = b;
    CK(cudaMalloc(&b->hdr, sizeof(BAHeader))); CK(cudaMemset(b->hdr, 0, sizeof(BAHeader)));
    CK(cudaMallocHost(&b->hdr_host, sizeof(BAHeader))); memset(b->hdr_host, 0, sizeof(BAHeader));
    CK(cudaMalloc(&b->thcount, sizeof(int))); CK(cudaMemset(b->thcount, 0, sizeof(int)));
  }
  *out = c->ba_windows[window]; return SDV_OK;
}
static void ba_window_drop(sdv_ctx* c, int window) {                       // a window created by a call that then failed: it holds no pins or pool
  BAState* b = c->ba_windows[window]; cudaFree(b->hdr); cudaFreeHost(b->hdr_host); cudaFree(b->thcount); delete b; c->ba_windows[window] = nullptr;
}
static int ba_select(sdv_ctx* c, int window) { BAState* b; int rc = ba_window(c, window, &b); if (rc) return rc; c->ba = b; return SDV_OK; }
static int ba_get(sdv_ctx* c, BAState** out) {
  if (!c->ba) { int rc = ba_select(c, 0); if (rc) return rc; }
  *out = c->ba; return SDV_OK;
}
static int32_t ba_index(const sdv_ctx* c, const BAState* b) { for (size_t i=0;i<c->ba_windows.size();i++) if (c->ba_windows[i] == b) return (int32_t)i; return -1; }
// a batched entry's window list: n distinct indices in range, each naming a window that has been set (*bs gets them)
static int ba_list(sdv_ctx* c, const char* who, int n, const int32_t* windows, std::vector<BAState*>* bs) {
  { int rc = check_ids(c, n, windows, kMaxWindows, who, "window"); if (rc) return rc; }
  bs->resize(n);
  for (int i=0;i<n;i++) {
    if (windows[i] >= (int)c->ba_windows.size() || !c->ba_windows[windows[i]]) return ctx_fail(c, SDV_ERR_ARG, "%s: BA window %d not set", who, windows[i]);
    (*bs)[i] = c->ba_windows[windows[i]];
  }
  return SDV_OK;
}

static int ba_wait(sdv_ctx* c) { c->ba_waits++; CK(cudaStreamSynchronize(c->st_ba)); return SDV_OK; }   // every host wait on the back-end stream
#define BA_WAIT() do { int rcw_ = ba_wait(c); if (rcw_) return rcw_; } while (0)

template <typename T> static T* bump(char*& p, size_t n) { T* r = reinterpret_cast<T*>(p); p += ((n*sizeof(T) + 255)/256)*256; return r; }

static size_t ba_layout(BAPointsDev& P, BAResDev& R, char* base, int cp, int cr) {
  char* p = base;
  P.uv = bump<float2>(p, cp); P.idepth = bump<float>(p, cp); P.idepth_zero = bump<float>(p, cp); P.idepth_backup = bump<float>(p, cp); P.step = bump<float>(p, cp);
  P.color = bump<float>(p, (size_t)cp*8); P.weights = bump<float>(p, (size_t)cp*8);
  P.host = bump<int>(p, cp); P.hasDepthPrior = bump<int>(p, cp); P.isFromSensor = bump<int>(p, cp); P.res_begin = bump<int>(p, cp+1);
  P.priorF = bump<float>(p, cp); P.deltaF = bump<float>(p, cp); P.HdiF = bump<float>(p, cp); P.bdSumF = bump<float>(p, cp);
  P.Hdd_accAF = bump<float>(p, cp); P.bd_accAF = bump<float>(p, cp); P.Hcd_accAF = bump<float>(p, (size_t)cp*4);
  P.idepth_hessian = bump<float>(p, cp); P.maxRelBaseline = bump<float>(p, cp); P.numGoodResiduals = bump<int>(p, cp); P.ngood = bump<int>(p, cp);
  P.res_of_target = bump<int>(p, (size_t)cp*kMaxF); P.marg_status = bump<int>(p, cp);
  R.point = bump<int>(p, cr); R.host = bump<int>(p, cr); R.target = bump<int>(p, cr); R.hasMatcher = bump<int>(p, cr); R.matcher = bump<float2>(p, cr); R.isNew = bump<int>(p, cr);
  R.state_state = bump<int>(p, cr); R.state_NewState = bump<int>(p, cr); R.state_energy = bump<float>(p, cr); R.state_NewEnergy = bump<float>(p, cr); R.state_NewEnergyWithOutlier = bump<float>(p, cr);
  R.isActive = bump<int>(p, cr); R.toRemove = bump<int>(p, cr);
  R.J = bump<float>(p, (size_t)cr*24); R.efJ = bump<float>(p, (size_t)cr*24); R.JpJdF = bump<float>(p, (size_t)cr*8); R.center = bump<float>(p, (size_t)cr*3);
  R.res_toZero = bump<float2>(p, cr); R.isLinearized = bump<int>(p, cr);
  R.pair_begin = bump<int>(p, kMaxF*kMaxF+1); R.pair_res = bump<int>(p, cr); R.host_begin = bump<int>(p, kMaxF+1);
  return (size_t)(p - base);
}
// a window's point / residual storage: one pool carved by ba_layout, plus the reduction buffers sized by the residual capacity
struct BAPool { void* pool; size_t bytes; BAPointsDev P; BAResDev R; double* partials; float* thbuf; int capP, capR; };
static void ba_pool_free(BAPool& q) { cudaFree(q.pool); cudaFree(q.partials); cudaFree(q.thbuf); q = BAPool{}; }
static int ba_pool_new(sdv_ctx* c, int nP, int nR, BAPool& q) {
  q = BAPool{}; const int cp = nP + nP/4 + 256, cr = nR + nR/4 + 1024;
  const size_t bytes = ba_layout(q.P, q.R, nullptr, cp, cr);
  cudaError_t e = cudaMalloc(&q.pool, bytes);
  if (e == cudaSuccess) e = cudaMemset(q.pool, 0, bytes);
  if (e == cudaSuccess) e = cudaMalloc(&q.partials, (size_t)((cr + 127)/128 + 1)*sizeof(double));
  if (e == cudaSuccess) e = cudaMalloc(&q.thbuf, (size_t)cr*sizeof(float));
  if (e != cudaSuccess) { ba_pool_free(q); return ctx_fail(c, SDV_ERR_CUDA, "BA: pool of %d points, %d residuals: %s", cp, cr, cudaGetErrorString(e)); }
  ba_layout(q.P, q.R, (char*)q.pool, cp, cr); q.bytes = bytes; q.capP = cp; q.capR = cr;
  return SDV_OK;
}
static void ba_pool_swap(BAState* b, BAPool& q) {                           // the window's old pool is freed; q is the window's now
  cudaFree(b->pool); cudaFree(b->partials); cudaFree(b->thbuf);
  b->pool = q.pool; b->pool_bytes = q.bytes; b->P = q.P; b->R = q.R; b->partials = q.partials; b->thbuf = q.thbuf; b->capP = q.capP; b->capR = q.capR; q = BAPool{};
}

static BAWinDev win_of(const BAState* b) { BAWinDev w; w.hdr = b->hdr; w.P = b->P; w.R = b->R; w.partials = b->partials; w.thbuf = b->thbuf; w.thcount = b->thcount; return w; }
// device array of window descriptors for one (batched) launch sequence; maxP/maxR size the grids
static int ba_wins(sdv_ctx* c, int n, BAState* const* bs, const BAWinDev** out, int* maxP, int* maxR) {
  const size_t bytes = Scratch::need(n, sizeof(BAWinDev));
  if (bytes > c->ba_wins_dev.cap || bytes > c->ba_wins_host.cap) c->ba_waits++;                // a growing scratch waits for the stream before it frees
  if (c->ba_wins_dev.reserve(bytes, c->st_ba) || c->ba_wins_host.reserve(bytes, c->st_ba)) return ctx_fail(c, SDV_ERR_CUDA, "BA: descriptors of %d windows", n);
  c->ba_wins_dev.reset(); c->ba_wins_host.reset(); BAWinDev* d = c->ba_wins_dev.take<BAWinDev>(n); BAWinDev* h = c->ba_wins_host.take<BAWinDev>(n); int mp = 1, mr = 1;
  BA_WAIT();                                          // the pinned staging array may still feed a previous launch sequence
  for (int i=0;i<n;i++) { h[i] = win_of(bs[i]); if (bs[i]->nP > mp) mp = bs[i]->nP; if (bs[i]->nR > mr) mr = bs[i]->nR; }
  CK(cudaMemcpyAsync(d, h, (size_t)n*sizeof(BAWinDev), cudaMemcpyHostToDevice, c->st_ba));
  *out = d; if (maxP) *maxP = mp; if (maxR) *maxR = mr;
  return SDV_OK;
}
#define WIN1() const BAWinDev* wins; int maxP, maxR; { int rcw = ba_wins(c, 1, &b, &wins, &maxP, &maxR); if (rcw) return rcw; }

// staging of one batched call in c->ba_scr / ba_scr_host: reserve, then take the leading pieces from both alike (stage2), copy that part in one
// cudaMemcpyAsync (stage_up), then take the device-only pieces.  Every batched entry ends in a wait on st_ba, so the pinned half is free at the next call.
static int stage_reserve(sdv_ctx* c, size_t both, size_t dev_only, size_t host_only, const char* who) {
  if (both + dev_only > c->ba_scr.cap || both + host_only > c->ba_scr_host.cap) c->ba_waits++;   // a growing scratch waits for the stream before it frees
  if (c->ba_scr.reserve(both + dev_only, c->st_ba) || c->ba_scr_host.reserve(both + host_only, c->st_ba)) return ctx_fail(c, SDV_ERR_CUDA, "%s: staging of %zu bytes", who, both + dev_only);
  c->ba_scr.reset(); c->ba_scr_host.reset(); return SDV_OK;
}
template <class T> static void stage2(sdv_ctx* c, size_t n, T** h, T** d) { *h = c->ba_scr_host.take<T>(n); *d = c->ba_scr.take<T>(n); }
static int stage_up(sdv_ctx* c) { CK(cudaMemcpyAsync(c->ba_scr.p, c->ba_scr_host.p, c->ba_scr_host.used, cudaMemcpyHostToDevice, c->st_ba)); return SDV_OK; }
static size_t need(size_t n, size_t sz) { return Scratch::need(n, sz); }
// device staging above this is freed when the call that needed it returns (rows of ~250 bench windows), so that one large install does not keep its
// scratch for the life of the context
constexpr size_t kBaStageKeep = size_t(256) << 20;
struct StageTrim { sdv_ctx* c; ~StageTrim() { if (c->ba_scr.cap > kBaStageKeep) c->ba_scr.release(); } };

static int ba_pull_scalars(sdv_ctx* c, BAState* b) {                        // energyP .. end of header
  const size_t off = offsetof(BAHeader, energyP), len = sizeof(BAHeader) - off;
  CK(cudaMemcpyAsync((char*)b->hdr_host + off, (char*)b->hdr + off, len, cudaMemcpyDeviceToHost, c->st_ba));
  BA_WAIT(); CK(cudaGetLastError());
  return SDV_OK;
}

extern "C" {

/* insertFrame + setAdjointsF + the HM/bM carry-over (+ CalibHessian::value_zero) for n windows.  Every check runs before any window changes;
 * the headers are written on the device: the host-set prefix and HM / bM are copied, the rest is zeroed by the install kernel. */
int sdv_ba_set_window_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* f_begin, const uint64_t* frame_ids, const double* T_evalPT7,
                            const double* state10, const double* state_zero10, const float* ab_exposure, const int32_t* frameID, const float* frameEnergyTH,
                            const double* calib_value_scaled, const double* calib_value_zero, const double* HM, const double* bM) { SDV_GUARD_BA(c);
  const char* who = "sdv_ba_set_window_batch";
  if (!c || n < 1 || !windows || !f_begin || !frame_ids || !T_evalPT7 || !state10 || !state_zero10 || !calib_value_scaled) return SDV_ERR_ARG;
  SDV_GUARD_TRK(c);                                                           // frame table, pins, level-0 texel pool and the ingest join belong to the tracker domain
  CK(cudaSetDevice(c->device));
  { int rc = check_ids(c, n, windows, kMaxWindows, who, "window"); if (rc) return rc; }
  { int rc = check_offsets(c, n, f_begin, who, "f_begin"); if (rc) return rc; }
  for (int i=0;i<n;i++) { const int nF = f_begin[i+1] - f_begin[i];
    if (nF < 1 || nF > SDV_MAX_FRAMES_WINDOW) return ctx_fail(c, SDV_ERR_ARG, "%s: window %d has %d frames (1 .. %d)", who, windows[i], nF, SDV_MAX_FRAMES_WINDOW); }
  std::vector<FrameDev*> Fr(f_begin[n]); std::vector<int> cam0(n);
  for (int i=0;i<n;i++) { cam0[i] = -1;                                      // one size per window: BAHeader::w/h are the window's frames' size
    for (int f=f_begin[i]; f<f_begin[i+1]; f++) { int rcf = job_frame(c, who, f, frame_ids[f], -1, -1, nullptr, &Fr[f]); if (rcf) return rcf;
      const int cam = Fr[f]->cam; if (cam0[i] < 0) cam0[i] = cam;
      if (!same_size(c, cam, cam0[i])) return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: BA frame %d is %dx%d but frame 0 is %dx%d: one window holds frames of one size", who, windows[i],
                                                   f - f_begin[i], c->cam_w[cam], c->cam_h[cam], c->cam_w[cam0[i]], c->cam_h[cam0[i]]); } }
  for (int f=0; f<f_begin[n]; f++) { int rc0 = ensure_lvl0(c, *Fr[f]); if (rc0) return rc0; }
  // staged headers: window i's prefix at src[i], then its HM and bM (dim = 4 + 6 nF_i each)
  std::vector<long long> src(n); long long bytes = 0;
  for (int i=0;i<n;i++) { const int N = kCP + 6*(f_begin[i+1] - f_begin[i]); src[i] = bytes; bytes += kHdrPrefix + 8ll*((HM ? N*N : 0) + (bM ? N : 0)); }
  { int rc = stage_reserve(c, need(n, sizeof(BAHdrInstall)) + need(bytes, 1), 0, 0, who); if (rc) return rc; }
  BAHdrInstall *Dh, *Dd; char *Sh, *Sd; stage2(c, n, &Dh, &Dd); stage2(c, bytes, &Sh, &Sd);
  long long hm_off = 0, bm_off = 0;
  for (int i=0;i<n;i++) {
    const int f0 = f_begin[i], nF = f_begin[i+1] - f0, N = kCP + 6*nF;
    BAHeader* H = reinterpret_cast<BAHeader*>(Sh + src[i]); memset(H, 0, kHdrPrefix);   // the fields before precalc only
    H->nF = nF; H->w = c->cam_w[cam0[i]]; H->h = c->cam_h[cam0[i]]; H->dim = N;
    BASettingsDev& s = H->set;
    s.huberTH = c->set.huberTH; s.outlierTHSumComponent = c->set.outlierTHSumComponent; s.idepthFixPrior = c->set.idepthFixPrior;
    s.initialRotPrior = 1e11f; s.initialTransPrior = 1e10f; s.initialCalibHessian = 5e9f;            // settings.cpp:23-27
    s.frameEnergyTHConstWeight = 0.5f; s.frameEnergyTHN = 0.7f; s.frameEnergyTHFacMedian = 1.5f; s.overallEnergyTHWeight = 1;   // :108-111
    s.thOptIterations = 1.2f; s.minOptIterations = 1; s.solverModeDelta = 0.00001;                  // :56-57, :35
    BACalibDev& cal = H->calib;                                                                       // CalibHessian ctor: setValueScaled + value_zero = value
    const double* vs = calib_value_scaled + 4*i; const float SFI = 1.0f/50.0f;
    for (int k=0;k<4;k++) { cal.value_scaled[k] = vs[k]; cal.sf[k] = (float)vs[k]; cal.value[k] = SFI*vs[k];
      cal.value_zero[k] = cal.value[k]; cal.vmvz[k] = 0; cal.step[k] = 0; cal.value_backup[k] = cal.value[k]; }
    cal.si[0] = 1.0f/cal.sf[0]; cal.si[1] = 1.0f/cal.sf[1]; cal.si[2] = -cal.sf[2]/cal.sf[0]; cal.si[3] = -cal.sf[3]/cal.sf[1];
    if (calib_value_zero) for (int k=0;k<4;k++) { cal.value_zero[k] = calib_value_zero[4*i+k]; cal.vmvz[k] = cal.value[k] - calib_value_zero[4*i+k]; }   // a live CalibHessian
    for (int f=0; f<nF; f++) { const int g = f0 + f;
      BAFrameDev& F = H->frames[f];
      F.evalPT = se3_from7(T_evalPT7 + 7*g);
      for (int k=0;k<10;k++) { F.state[k] = state10[10*g+k]; F.state_zero[k] = state_zero10[10*g+k]; F.state_backup[k] = F.state[k]; F.step[k] = 0; }
      F.ab_exposure = ab_exposure ? ab_exposure[g] : 1.0f; F.frameID = frameID ? frameID[g] : f; F.frameEnergyTH = frameEnergyTH ? frameEnergyTH[g] : 8*8*8;
      F.img0 = Fr[g]->lvl[0];
    }
    double* tail = reinterpret_cast<double*>(Sh + src[i] + kHdrPrefix);
    if (HM) { memcpy(tail, HM + hm_off, (size_t)N*N*sizeof(double)); tail += (size_t)N*N; hm_off += (long long)N*N; }
    if (bM) { memcpy(tail, bM + bm_off, (size_t)N*sizeof(double)); bm_off += N; }
    Dh[i].src = src[i]; Dh[i].hm_n = HM ? N*N : 0; Dh[i].bm_n = bM ? N : 0;
  }
  // the listed windows exist before anything is committed; if one cannot be created, the ones this call created are removed again
  { std::vector<int32_t> made;
    for (int i=0;i<n;i++) {
      const bool had = windows[i] < (int)c->ba_windows.size() && c->ba_windows[windows[i]];
      BAState* b; int rc = ba_window(c, windows[i], &b);
      if (!had && c->ba_windows.size() > (size_t)windows[i] && c->ba_windows[windows[i]]) made.push_back(windows[i]);
      if (rc) { for (int32_t w : made) ba_window_drop(c, w); return rc; } } }
  // commit: the windows take their frames (the references of the ones they held are dropped) and their headers
  for (int i=0;i<n;i++) {
    BAState* b = c->ba_windows[windows[i]];
    const int f0 = f_begin[i], nF = f_begin[i+1] - f0;
    for (int k=0;k<b->n_pinned;k++) frame_unpin(c, b->pinned[k]);
    b->n_pinned = nF; for (int f=0; f<nF; f++) { b->pinned[f] = frame_ids[f0+f]; frame_pin(c, frame_ids[f0+f]); }
    memcpy(b->hdr_host, Sh + src[i], kHdrPrefix); b->nF = nF;
    Dh[i].hdr = b->hdr;
  }
  { int rcj = join_ingest(c); if (rcj) return rcj; }                          // the keyframes' pyramids (ingest stream) and level-0 texels (tracker stream) are complete
  CK(cudaEventRecord(c->ev_xdom, c->st)); CK(cudaStreamWaitEvent(c->st_ba, c->ev_xdom, 0));   // before the back-end stream reads them; pinned frames cannot change afterwards
  { int rc = stage_up(c); if (rc) return rc; }
  launch_ba_hdr_install(Dd, n, Sd, c->st_ba); c->launches += 1;
  BA_WAIT(); CK(cudaGetLastError());
  return SDV_OK;
}

int sdv_ba_set_window(sdv_ctx* c, int nF, const uint64_t* frame_ids, const double* T_evalPT7, const double* state10, const double* state_zero10,
                      const float* ab_exposure, const int32_t* frameID, const float* frameEnergyTH, const double calib_value_scaled[4],
                      const double* HM, const double* bM) { SDV_GUARD_BA(c);
  if (!c || nF < 1 || nF > SDV_MAX_FRAMES_WINDOW || !frame_ids || !T_evalPT7 || !state10 || !state_zero10 || !calib_value_scaled) return SDV_ERR_ARG;
  BAState* b; int rc = ba_get(c, &b); if (rc) return rc;
  const int32_t w = ba_index(c, b), fb[2] = {0, nF};
  return sdv_ba_set_window_batch(c, 1, &w, fb, frame_ids, T_evalPT7, state10, state_zero10, ab_exposure, frameID, frameEnergyTH, calib_value_scaled, nullptr, HM, bM);
}

/* the makeIDX mirror (EnergyFunctional.cpp:761-782) and setPrecalcValues (FullSystem.cpp:1358-1368) for n windows.  Plan first, commit last: the rows are
 * staged and checked on the device and one refusal word per window is read back (wait 1) before any window changes; a window whose pool must grow gets
 * its new pool aside, swapped in at commit and freed on refusal.  Then the pair lists, the scatter into the pools and the setup run for all windows (wait 2). */
int sdv_ba_set_points_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* p_begin, const int32_t* r_begin, const float* uv, const float* idepth,
                            const float* idepth_zero, const float* color8, const float* weights8, const int32_t* host, const int32_t* hasDepthPrior,
                            const int32_t* isFromSensor, const int32_t* res_begin, const int32_t* r_point, const int32_t* r_host, const int32_t* r_target,
                            const int32_t* r_hasMatcher, const float* r_matcher, const int32_t* r_isNew) { SDV_GUARD_BA(c);
  const char* who = "sdv_ba_set_points_batch";
  if (!c || n < 1 || !windows || !p_begin || !r_begin || !res_begin) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device)); cudaStream_t st = c->st_ba;
  std::vector<BAState*> bs; { int rc = ba_list(c, who, n, windows, &bs); if (rc) return rc; }
  { int rc = check_offsets(c, n, p_begin, who, "p_begin"); if (rc) return rc; }
  { int rc = check_offsets(c, n, r_begin, who, "r_begin"); if (rc) return rc; }
  int maxP = 1, maxR = 1;
  for (int i=0;i<n;i++) { const int nP = p_begin[i+1] - p_begin[i], nR = r_begin[i+1] - r_begin[i];
    if (nP > kMaxPtsWin || nR > kMaxResWin) return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: %d points, %d residuals", who, windows[i], nP, nR);
    if (nP == 0 && nR != 0) return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: residuals without points", who, windows[i]);
    maxP = std::max(maxP, nP); maxR = std::max(maxR, nR); }
  const int totP = p_begin[n], totR = r_begin[n];
  if (totP > 0 && (!uv || !idepth || !idepth_zero || !color8 || !weights8 || !host || !hasDepthPrior || !isFromSensor)) return SDV_ERR_ARG;
  if (totR > 0 && (!r_point || !r_host || !r_target || !r_hasMatcher || !r_matcher || !r_isNew)) return SDV_ERR_ARG;
  const size_t P = std::max(totP, 1), R = std::max(totR, 1), sort_bytes = std::max(ba_pts_sort_bytes(n, totR), (size_t)1);
  const size_t both = need(n, sizeof(BAPtsInstall)) + need(n, sizeof(BAWinDev)) + need(n, 8);
  const size_t dev = need(P, 8) + 4*need(P, 4) + 2*need(P*8, 4) + 3*need(P, 4) + need(P + n, 4) + need(P*kMaxF, 4) + need((size_t)n*kPairCnt, 4)
                   + 6*need(R, 4) + need(R, 8) + 4*need(R, 4) + need(sort_bytes, 1);
  { int rc = stage_reserve(c, both, dev, 0, who); if (rc) return rc; }
  StageTrim trim{c};
  BAPtsInstall *Dh, *Dd; BAWinDev *Wh, *Wd; unsigned long long *Eh, *Ed;
  stage2(c, n, &Dh, &Dd); stage2(c, n, &Wh, &Wd); stage2(c, n, &Eh, &Ed);
  Scratch& S = c->ba_scr; BAPtsStage G;
  float2* d_uv = S.take<float2>(P); float* d_id = S.take<float>(P); float* d_idz = S.take<float>(P); float* d_col = S.take<float>(P*8); float* d_wt = S.take<float>(P*8);
  int* d_host = S.take<int>(P); int* d_hdp = S.take<int>(P); int* d_ifs = S.take<int>(P); int* d_rb = S.take<int>(P + n);
  int* d_rp = S.take<int>(R); int* d_rh = S.take<int>(R); int* d_rt = S.take<int>(R); int* d_rm = S.take<int>(R); float2* d_rmat = S.take<float2>(R); int* d_rn = S.take<int>(R);
  G.uv = d_uv; G.idepth = d_id; G.idepth_zero = d_idz; G.color = d_col; G.weights = d_wt; G.host = d_host; G.hasDepthPrior = d_hdp; G.isFromSensor = d_ifs; G.res_begin = d_rb;
  G.r_point = d_rp; G.r_host = d_rh; G.r_target = d_rt; G.r_hasMatcher = d_rm; G.r_matcher = d_rmat; G.r_isNew = d_rn;
  G.rot = S.take<int>(P*kMaxF); G.cnt = S.take<int>((size_t)n*kPairCnt);
  G.key_in = S.take<unsigned>(R); G.key = S.take<unsigned>(R); G.val_in = S.take<int>(R); G.pair_res = S.take<int>(R); void* sort_tmp = S.take<char>(sort_bytes);
  // pools that must grow, allocated aside
  std::vector<BAPool> fresh(n, BAPool{});
  auto drop = [&]() { for (BAPool& q : fresh) if (q.pool) ba_pool_free(q); };
  for (int i=0;i<n;i++) { const int nP = p_begin[i+1] - p_begin[i], nR = r_begin[i+1] - r_begin[i]; BAState* b = bs[i];
    Dh[i] = BAPtsInstall{p_begin[i], r_begin[i], nP, nR, b->nF}; Eh[i] = ~0ull;
    Wh[i] = win_of(b);
    if (!b->pool || nP > b->capP || nR > b->capR) { int rc = ba_pool_new(c, nP, nR, fresh[i]); if (rc) { drop(); return rc; }   // a window's first points, or growth
      Wh[i].P = fresh[i].P; Wh[i].R = fresh[i].R; Wh[i].partials = fresh[i].partials; Wh[i].thbuf = fresh[i].thbuf; } }
#define UP(dst, src, cnt, T) do { if ((cnt) > 0) { cudaError_t e_ = cudaMemcpyAsync(dst, src, (size_t)(cnt)*sizeof(T), cudaMemcpyHostToDevice, st); \
                                    if (e_ != cudaSuccess) { drop(); return ctx_fail(c, SDV_ERR_CUDA, "%s: staging: %s", who, cudaGetErrorString(e_)); } } } while (0)
  UP(c->ba_scr.p, c->ba_scr_host.p, c->ba_scr_host.used, char);
  UP(d_uv, uv, (size_t)totP*2, float); UP(d_id, idepth, totP, float); UP(d_idz, idepth_zero, totP, float); UP(d_col, color8, (size_t)totP*8, float); UP(d_wt, weights8, (size_t)totP*8, float);
  UP(d_host, host, totP, int); UP(d_hdp, hasDepthPrior, totP, int); UP(d_ifs, isFromSensor, totP, int); UP(d_rb, res_begin, totP + n, int);
  UP(d_rp, r_point, totR, int); UP(d_rh, r_host, totR, int); UP(d_rt, r_target, totR, int); UP(d_rm, r_hasMatcher, totR, int); UP(d_rmat, r_matcher, (size_t)totR*2, float); UP(d_rn, r_isNew, totR, int);
#undef UP
  cudaMemsetAsync(G.rot, 0xff, (size_t)totP*kMaxF*sizeof(int), st); cudaMemsetAsync(G.cnt, 0, (size_t)n*kPairCnt*sizeof(int), st);
  launch_ba_pts_check(Dd, n, totP, G, Ed, st);
  cudaMemcpyAsync(Eh, Ed, (size_t)n*8, cudaMemcpyDeviceToHost, st);
  { c->ba_waits++; cudaError_t e = cudaStreamSynchronize(st); if (e == cudaSuccess) e = cudaGetLastError();
    if (e != cudaSuccess) { drop(); return ctx_fail(c, SDV_ERR_CUDA, "%s: check: %s", who, cudaGetErrorString(e)); } }
  int nl = totP > 0 ? 1 : 0;
  for (int i=0;i<n;i++) { const unsigned long long e = Eh[i]; if (e == ~0ull) continue;
    drop(); c->launches += nl;
    const int w = windows[i], p = ba_err_point(e), r = ba_err_res(e); const int32_t* rb = res_begin + p_begin[i] + i;
    switch (ba_err_code(e)) {
      case BA_ERR_SPAN: return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: res_begin must span all residuals (res_begin[0]=%d, res_begin[nP]=%d, nR=%d)", who, w, rb[0], rb[Dh[i].nP], Dh[i].nR);
      case BA_ERR_MONO: return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: res_begin not monotone at point %d", who, w, p);
      case BA_ERR_HOST: return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: point %d: points must be grouped by host frame in frame order (ef->allPoints order)", who, w, p);
      case BA_ERR_RES:  return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: residual %d inconsistent with its point %d", who, w, r, p);
      default:          return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: two residuals of point %d share a target (residual %d)", who, w, p, r);
    }
  }
  // commit: the pair sort is enqueued before anything writes a window, so its failure still changes none; then the pools, the setup, the host state
  const int li = launch_ba_pts_install(Wd, Dd, n, totR, maxP, maxR, G, sort_tmp, sort_bytes, st);
  if (li < 0) { drop(); return ctx_fail(c, SDV_ERR_CUDA, "%s: pair sort", who); }
  launch_ba_setup(Wd, n, maxP, st); launch_ba_reset_oob(Wd, n, maxR, st);
  for (int i=0;i<n;i++) { BAState* b = bs[i]; if (fresh[i].pool) ba_pool_swap(b, fresh[i]);
    b->nP = Dh[i].nP; b->nR = Dh[i].nR; b->hdr_host->nP = b->nP; b->hdr_host->nR = b->nR; }
  c->launches += nl + li + 3;
  BA_WAIT(); CK(cudaGetLastError());
  return SDV_OK;
}

int sdv_ba_set_points(sdv_ctx* c, int nP, const float* uv, const float* idepth, const float* idepth_zero, const float* color8, const float* weights8,
                      const int32_t* host, const int32_t* hasDepthPrior, const int32_t* isFromSensor, const int32_t* res_begin,
                      int nR, const int32_t* r_point, const int32_t* r_host, const int32_t* r_target, const int32_t* r_hasMatcher,
                      const float* r_matcher, const int32_t* r_isNew) { SDV_GUARD_BA(c);
  if (!c || !c->ba || nP < 0 || nR < 0) return SDV_ERR_ARG;
  const int32_t w = ba_index(c, c->ba), pb[2] = {0, nP}, rb[2] = {0, nR};
  return sdv_ba_set_points_batch(c, 1, &w, pb, rb, uv, idepth, idepth_zero, color8, weights8, host, hasDepthPrior, isFromSensor, res_begin,
                                 r_point, r_host, r_target, r_hasMatcher, r_matcher, r_isNew);
}

int sdv_ba_clear(sdv_ctx* c) { SDV_GUARD_BA(c);               // empties the selected window and drops its references to frame images
  if (!c) return SDV_ERR_ARG; if (!c->ba) return SDV_OK; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  BA_WAIT();
  { SDV_GUARD_TRK(c); for (int i=0;i<b->n_pinned;i++) frame_unpin(c, b->pinned[i]); }
  b->n_pinned = 0; b->nF = 0; b->nP = 0; b->nR = 0; return SDV_OK;
}
int sdv_ba_select(sdv_ctx* c, int window) { SDV_GUARD_BA(c); if (!c) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); return ba_select(c, window); }

// CalibHessian::value_zero of a LIVE system: the linearisation point of the intrinsics stays where the CalibHessian was constructed (HessianBlocks.h:287) while value moves with
// every bundle adjustment; sdv_ba_set_window assumes value_zero == value (a fresh CalibHessian).  Call this between sdv_ba_set_window and sdv_ba_set_points when they differ:
// value_minus_value_zero (-> cDeltaF, EnergyFunctional.cpp:144) is what the marginalisation prior HM / bM acts on.  value_zero in CalibHessian::value units (value_scaled / SCALE).
int sdv_ba_set_calib_zero(sdv_ctx* c, const double value_zero[4]) { SDV_GUARD_BA(c);
  if (!c || !c->ba || !value_zero) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; BACalibDev& cal = b->hdr_host->calib;
  for (int i=0;i<4;i++) { cal.value_zero[i] = value_zero[i]; cal.vmvz[i] = cal.value[i] - value_zero[i]; }
  CK(cudaMemcpyAsync(&b->hdr->calib, &cal, sizeof(BACalibDev), cudaMemcpyHostToDevice, c->st_ba)); BA_WAIT();
  return SDV_OK;
}

int sdv_ba_reset_oob(sdv_ctx* c) { SDV_GUARD_BA(c); if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; WIN1(); launch_ba_reset_oob(wins, 1, maxR, c->st_ba); c->launches++; return SDV_OK; }

int sdv_ba_linearize(sdv_ctx* c, int fix, double* energy) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; WIN1();
  launch_ba_linearize(wins, 1, maxR, fix, GATE_ALWAYS, c->st_ba); c->launches += 2;
  int rc = ba_pull_scalars(c, b); if (rc) return rc;
  if (energy) *energy = b->hdr_host->energyP;
  return SDV_OK;
}
int sdv_ba_apply_res(sdv_ctx* c) { SDV_GUARD_BA(c); if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; WIN1(); launch_ba_apply(wins, 1, maxR, GATE_ALWAYS, c->st_ba); c->launches++; BA_WAIT(); return SDV_OK; }
int sdv_ba_energy(sdv_ctx* c, double* EL, double* EM) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; WIN1();
  launch_ba_energies(wins, 1, GATE_ALWAYS, c->st_ba); c->launches++;
  int rc = ba_pull_scalars(c, b); if (rc) return rc;
  if (EL) *EL = b->hdr_host->energyL; if (EM) *EM = b->hdr_host->energyM;
  return SDV_OK;
}
int sdv_ba_solve(sdv_ctx* c, int iteration, double lambda, double* x_out) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; WIN1();
  launch_ba_accumulate(wins, 1, maxP, GATE_ALWAYS, c->st_ba);
  launch_ba_solve(wins, 1, maxP, iteration, lambda, 0, GATE_ALWAYS, c->st_ba); c->launches += 5;
  if (x_out) { CK(cudaMemcpyAsync(x_out, b->hdr->lastX, (size_t)(kCP+6*b->nF)*sizeof(double), cudaMemcpyDeviceToHost, c->st_ba)); }
  BA_WAIT(); CK(cudaGetLastError());
  return SDV_OK;
}
int sdv_ba_backup(sdv_ctx* c) { SDV_GUARD_BA(c); if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; WIN1(); launch_ba_backup(wins, 1, maxP, GATE_ALWAYS, c->st_ba); c->launches++; return SDV_OK; }
int sdv_ba_step(sdv_ctx* c, float stepfac, int load_backup, int* canbreak) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; WIN1();
  launch_ba_step(wins, 1, stepfac, load_backup, GATE_ALWAYS, c->st_ba); c->launches += 2;
  int rc = ba_pull_scalars(c, b); if (rc) return rc;
  if (canbreak) *canbreak = b->hdr_host->canbreak;
  return SDV_OK;
}

/* float FullSystem::optimize(int mnumOptIts)   FullSystemOptimize.cpp:344-502, for n windows at once.
 * The Gauss-Newton loop is DEVICE-RESIDENT: every kernel is launched for all windows (grid.y = window) on a fixed schedule and
 * gated by per-window flags that ba_decide_kernel sets (accept -> APPLY, reject -> RELOAD, converged -> not ACTIVE); the host
 * never reads a decision back.  One D2H of the per-window tail at the end. */
int sdv_ba_optimize_batch(sdv_ctx* c, int n, const int32_t* windows, int mnumOptIts, float* rmse_out, int32_t* iterations_out, int32_t* accepts_out) { SDV_GUARD_BA(c);
  if (!c || n < 1 || !windows) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device)); cudaStream_t st = c->st_ba;
  std::vector<BAState*> bs(n); int maxIts = 0;
  for (int i=0;i<n;i++) {
    if (windows[i] < 0 || windows[i] >= (int)c->ba_windows.size() || !c->ba_windows[windows[i]]) return ctx_fail(c, SDV_ERR_ARG, "BA window %d not set", windows[i]);
    bs[i] = c->ba_windows[windows[i]];
    int m = mnumOptIts; if (bs[i]->nF < 3) m = 100; if (bs[i]->nF < 4) m = 75; if (bs[i]->nF < 2) m = 0; if (m > maxIts) maxIts = m;
    bs[i]->hdr_host->mnumOptIts = mnumOptIts;
    CK(cudaMemcpyAsync(&bs[i]->hdr->mnumOptIts, &bs[i]->hdr_host->mnumOptIts, sizeof(int), cudaMemcpyHostToDevice, st));
  }
  const BAWinDev* wins; int maxP, maxR; { int rcw = ba_wins(c, n, bs.data(), &wins, &maxP, &maxR); if (rcw) return rcw; }
  // The schedule is fixed (decisions are taken on the device and gate the launches), so for the usual short schedules it is captured once into a CUDA graph and
  // replayed: one graph launch instead of 6 + 19 per iteration + 5 kernel launches — what a single window (launch-latency bound) pays for.
  auto schedule = [&](cudaStream_t st, bool poll) -> int {
    launch_ba_reset_oob(wins, n, maxR, st);
    launch_ba_linearize(wins, n, maxR, 0, GATE_ALWAYS, st);
    launch_ba_energies(wins, n, GATE_ALWAYS, st);
    launch_ba_decide(wins, n, 0, st);
    launch_ba_apply(wins, n, maxR, GATE_ALWAYS, st);
    for (int iteration = 0; iteration < maxIts; iteration++) {
      launch_ba_backup(wins, n, maxP, GATE_ACTIVE, st);
      launch_ba_accumulate(wins, n, maxP, GATE_ACTIVE, st);
      launch_ba_solve(wins, n, maxP, 0, 0.0, 1, GATE_ACTIVE, st);
      launch_ba_step(wins, n, 1.0f, 0, GATE_ACTIVE, st);
      launch_ba_linearize(wins, n, maxR, 0, GATE_ACTIVE, st);
      launch_ba_energies(wins, n, GATE_ACTIVE, st);
      launch_ba_decide(wins, n, 1, st);
      launch_ba_apply(wins, n, maxR, GATE_ACTIVE | GATE_APPLY, st);
      launch_ba_step(wins, n, 1.0f, 1, GATE_ACTIVE | GATE_RELOAD, st);          // loadSateBackup
      launch_ba_linearize(wins, n, maxR, 0, GATE_ACTIVE | GATE_RELOAD, st);
      launch_ba_energies(wins, n, GATE_ACTIVE | GATE_RELOAD, st);
      launch_ba_decide(wins, n, 2, st);
      if (poll && maxIts > 8 && iteration >= 5 && (iteration % 4) == 1) {        // long schedules (tiny windows at start-up): poll for early exit
        bool any = false;
        for (int i=0;i<n;i++) { CK(cudaMemcpyAsync(&bs[i]->hdr_host->flags, &bs[i]->hdr->flags, sizeof(int), cudaMemcpyDeviceToHost, st)); }
        BA_WAIT();
        for (int i=0;i<n;i++) any = any || (bs[i]->hdr_host->flags & BA_ACTIVE);
        if (!any) break;
      }
    }
    launch_ba_reanchor(wins, n, maxP, st);
    launch_ba_linearize(wins, n, maxR, 1, GATE_ALWAYS, st);
    launch_ba_decide(wins, n, 3, st);
    return SDV_OK;
  };
  c->launches += 6 + 19*(long long)maxIts + 5;
  if (maxIts <= 8 && !getenv("SDV_BA_NO_GRAPH")) {
    if (!c->ba_graph || c->bag_wins != (const void*)wins || c->bag_n != n || c->bag_maxP != maxP || c->bag_maxR != maxR || c->bag_its != maxIts) {
      if (c->ba_graph) { cudaGraphExecDestroy(c->ba_graph); c->ba_graph = nullptr; }
      cudaGraph_t g = nullptr;
      CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      schedule(st, false);
      CK(cudaStreamEndCapture(st, &g));
      CK(cudaGraphInstantiate(&c->ba_graph, g, 0)); cudaGraphDestroy(g);
      c->bag_wins = wins; c->bag_n = n; c->bag_maxP = maxP; c->bag_maxR = maxR; c->bag_its = maxIts;
    }
    CK(cudaEventRecord(c->ba_ev0, st));
    CK(cudaGraphLaunch(c->ba_graph, st));
  } else {
    CK(cudaEventRecord(c->ba_ev0, st));
    { int rcs = schedule(st, true); if (rcs) return rcs; }
  }
  CK(cudaEventRecord(c->ba_ev1, st));
  for (int i=0;i<n;i++) { const size_t off = offsetof(BAHeader, energyP), len = sizeof(BAHeader) - off;
    CK(cudaMemcpyAsync((char*)bs[i]->hdr_host + off, (char*)bs[i]->hdr + off, len, cudaMemcpyDeviceToHost, st)); }
  BA_WAIT(); CK(cudaGetLastError());
  CK(cudaEventElapsedTime(&c->ba_last_ms, c->ba_ev0, c->ba_ev1));
  for (int i=0;i<n;i++) { const BAHeader* H = bs[i]->hdr_host;
    if (rmse_out) rmse_out[i] = (bs[i]->nF < 2) ? 0.f : H->rmse;
    if (iterations_out) iterations_out[i] = H->opt_iterations;
    if (accepts_out) accepts_out[i] = H->opt_accepts; }
  return SDV_OK;
}
float sdv_ba_last_kernel_ms(sdv_ctx* c) { return c ? c->ba_last_ms : 0.f; }
long long sdv_ba_host_wait_count(sdv_ctx* c) { if (!c) return 0; SDV_GUARD_BA(c); return c->ba_waits; }
int sdv_ba_optimize(sdv_ctx* c, int mnumOptIts, float* rmse_out, int32_t* iterations_out, int32_t* accepts_out) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG;
  int32_t w = -1; for (size_t i=0;i<c->ba_windows.size();i++) if (c->ba_windows[i] == c->ba) w = (int32_t)i;
  return sdv_ba_optimize_batch(c, 1, &w, mnumOptIts, rmse_out, iterations_out, accepts_out);
}

// ---- read-back (what the reference leaves in FrameHessian / PointHessian / PointFrameResidual / EnergyFunctional)
int sdv_ba_get_frames(sdv_ctx* c, double* T_evalPT7, double* state10, double* step10, float* frameEnergyTH, double* PRE_worldToCam7, double calib_value[4], double calib_step[4]) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  CK(cudaMemcpyAsync(b->hdr_host, b->hdr, offsetof(BAHeader, precalc), cudaMemcpyDeviceToHost, c->st_ba)); BA_WAIT();
  const BAHeader* H = b->hdr_host;
  for (int f=0; f<b->nF; f++) { const BAFrameDev& F = H->frames[f];
    if (T_evalPT7) se3_to7(F.evalPT, T_evalPT7 + 7*f); if (PRE_worldToCam7) se3_to7(F.PRE_w2c, PRE_worldToCam7 + 7*f);
    for (int i=0;i<10;i++) { if (state10) state10[10*f+i] = F.state[i]; if (step10) step10[10*f+i] = F.step[i]; }
    if (frameEnergyTH) frameEnergyTH[f] = F.frameEnergyTH; }
  for (int i=0;i<4;i++) { if (calib_value) calib_value[i] = H->calib.value[i]; if (calib_step) calib_step[i] = H->calib.step[i]; }
  return SDV_OK;
}
int sdv_ba_get_points(sdv_ctx* c, float* idepth, float* step, float* HdiF, float* bdSumF, float* maxRelBaseline, int32_t* numGoodResiduals, float* idepth_hessian) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; const int n = b->nP; const BAPointsDev& P = b->P;
#define DN(dst, src, T) do { if (dst && n > 0) CK(cudaMemcpyAsync(dst, src, (size_t)n*sizeof(T), cudaMemcpyDeviceToHost, c->st_ba)); } while (0)
  DN(idepth, P.idepth, float); DN(step, P.step, float); DN(HdiF, P.HdiF, float); DN(bdSumF, P.bdSumF, float); DN(maxRelBaseline, P.maxRelBaseline, float);
  DN(numGoodResiduals, P.numGoodResiduals, int); DN(idepth_hessian, P.idepth_hessian, float);
#undef DN
  BA_WAIT(); return SDV_OK;
}
int sdv_ba_get_residuals(sdv_ctx* c, int32_t* state_state, int32_t* state_NewState, float* energies3, int32_t* isActive, float* J24, float* efJ24,
                         float* JpJdF8, float* center3, int32_t* toRemove) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; const int n = b->nR; const BAResDev& R = b->R;
  if (n == 0) return SDV_OK;
  std::vector<float> e0(n), e1(n), e2(n);
#define DN(dst, src, cnt, T) do { if (dst) CK(cudaMemcpyAsync(dst, src, (size_t)(cnt)*sizeof(T), cudaMemcpyDeviceToHost, c->st_ba)); } while (0)
  DN(state_state, R.state_state, n, int); DN(state_NewState, R.state_NewState, n, int); DN(isActive, R.isActive, n, int); DN(toRemove, R.toRemove, n, int);
  DN(J24, R.J, (size_t)n*24, float); DN(efJ24, R.efJ, (size_t)n*24, float); DN(JpJdF8, R.JpJdF, (size_t)n*8, float); DN(center3, R.center, (size_t)n*3, float);
  DN(e0.data(), R.state_energy, n, float); DN(e1.data(), R.state_NewEnergy, n, float); DN(e2.data(), R.state_NewEnergyWithOutlier, n, float);
#undef DN
  BA_WAIT();
  if (energies3) for (int i=0;i<n;i++) { energies3[3*i] = e0[i]; energies3[3*i+1] = e1[i]; energies3[3*i+2] = e2[i]; }
  return SDV_OK;
}
// ------------------------------------------------------------------------------------------------ keyframe hand-over (FullSystem::makeKeyFrame, FullSystem.cpp:1152-1171)
// descriptors of n listed windows and the exclusive sum of their point counts (off, n+1 entries), staged for one copy; maxP sizes the grids
static int stage_windows(sdv_ctx* c, int n, BAState* const* bs, const BAWinDev** Wd, int** off_h, const int** off_d, int* maxP) {
  BAWinDev* Wh; BAWinDev* W; int* oh; int* od; stage2(c, n, &Wh, &W); stage2(c, (size_t)n + 1, &oh, &od);
  int mp = 1; oh[0] = 0;
  for (int i=0;i<n;i++) { Wh[i] = win_of(bs[i]); oh[i+1] = oh[i] + bs[i]->nP; mp = std::max(mp, bs[i]->nP); }
  *Wd = W; *off_h = oh; *off_d = od; *maxP = mp; return SDV_OK;
}
static int ba_list_points(sdv_ctx* c, const char* who, int n, const int32_t* windows, std::vector<BAState*>& bs) {
  { int rc = ba_list(c, who, n, windows, &bs); if (rc) return rc; }
  for (int i=0;i<n;i++) if (bs[i]->nP <= 0) return ctx_fail(c, SDV_ERR_STATE, "%s: window %d has no points (call sdv_ba_set_points)", who, windows[i]);
  return SDV_OK;
}

// FullSystem::flagPointsForRemoval, numeric part, for n windows: selected / status_out concatenated by the windows' point counts
int sdv_ba_flag_points_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* selected, int32_t* status_out) { SDV_GUARD_BA(c);
  const char* who = "sdv_ba_flag_points_batch";
  if (!c || n < 1 || !windows || !selected) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device)); cudaStream_t st = c->st_ba;
  std::vector<BAState*> bs; { int rc = ba_list_points(c, who, n, windows, bs); if (rc) return rc; }
  long long tot = 0; for (BAState* b : bs) tot += b->nP;
  { int rc = stage_reserve(c, need(n, sizeof(BAWinDev)) + need((size_t)n + 1, 4), need(tot, 4), 0, who); if (rc) return rc; }
  const BAWinDev* W; int* oh; const int* od; int maxP; stage_windows(c, n, bs.data(), &W, &oh, &od, &maxP);
  int* buf = c->ba_scr.take<int>(tot);
  { int rc = stage_up(c); if (rc) return rc; }
  CK(cudaMemcpyAsync(buf, selected, (size_t)tot*sizeof(int32_t), cudaMemcpyHostToDevice, st));
  launch_ba_status_copy(W, n, maxP, od, buf, 1, st);
  launch_ba_marg_flag(W, n, maxP, st); c->launches += 2;
  if (status_out) { launch_ba_status_copy(W, n, maxP, od, buf, 0, st); c->launches += 1;
    CK(cudaMemcpyAsync(status_out, buf, (size_t)tot*sizeof(int32_t), cudaMemcpyDeviceToHost, st)); }
  BA_WAIT(); CK(cudaGetLastError());
  return SDV_OK;
}
int sdv_ba_flag_points(sdv_ctx* c, const int32_t* selected, int32_t* status_out) { SDV_GUARD_BA(c);
  if (!c || !c->ba || !selected) return SDV_ERR_ARG;
  const int32_t w = ba_index(c, c->ba); return sdv_ba_flag_points_batch(c, 1, &w, selected, status_out);
}

// EnergyFunctional::marginalizePointsF for n windows; status (concatenated) == NULL: each window's device-resident status of the flag call
int sdv_ba_marginalize_points_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* status) { SDV_GUARD_BA(c);
  const char* who = "sdv_ba_marginalize_points_batch";
  if (!c || n < 1 || !windows) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device)); cudaStream_t st = c->st_ba;
  std::vector<BAState*> bs; { int rc = ba_list_points(c, who, n, windows, bs); if (rc) return rc; }
  long long tot = 0; for (BAState* b : bs) tot += b->nP;
  { int rc = stage_reserve(c, need(n, sizeof(BAWinDev)) + need((size_t)n + 1, 4), need(tot, 4), 0, who); if (rc) return rc; }
  const BAWinDev* W; int* oh; const int* od; int maxP; stage_windows(c, n, bs.data(), &W, &oh, &od, &maxP);
  int* buf = c->ba_scr.take<int>(tot);
  { int rc = stage_up(c); if (rc) return rc; }
  if (status) { CK(cudaMemcpyAsync(buf, status, (size_t)tot*sizeof(int32_t), cudaMemcpyHostToDevice, st)); launch_ba_status_copy(W, n, maxP, od, buf, 1, st); c->launches += 1; }
  launch_ba_marg_points(W, n, maxP, st); c->launches += 4;
  BA_WAIT(); CK(cudaGetLastError());
  return SDV_OK;
}
int sdv_ba_marginalize_points(sdv_ctx* c, const int32_t* status) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG;
  const int32_t w = ba_index(c, c->ba); return sdv_ba_marginalize_points_batch(c, 1, &w, status);
}

// EnergyFunctional::marginalizeFrame, repeated: window i eliminates idx[k_begin[i] .. k_begin[i+1]) in order, each index into the window as the previous
// eliminations left it.  Round k runs the k-th elimination of every window in one launch.  The priors come back in one copy.
int sdv_ba_marginalize_frames_batch(sdv_ctx* c, int n, const int32_t* windows, const int32_t* k_begin, const int32_t* idx, double* HM_out, double* bM_out) { SDV_GUARD_BA(c);
  const char* who = "sdv_ba_marginalize_frames_batch";
  if (!c || n < 1 || !windows || !k_begin) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device)); cudaStream_t st = c->st_ba;
  std::vector<BAState*> bs; { int rc = ba_list(c, who, n, windows, &bs); if (rc) return rc; }
  { int rc = check_offsets(c, n, k_begin, who, "k_begin"); if (rc) return rc; }
  int rounds = 0;
  for (int i=0;i<n;i++) { const int k = k_begin[i+1] - k_begin[i];
    if (k > 0 && !idx) return SDV_ERR_ARG;
    int nF = bs[i]->nF;
    for (int j=k_begin[i]; j<k_begin[i+1]; j++, nF--)
      if (idx[j] < 0 || idx[j] >= nF || nF < 2) return ctx_fail(c, SDV_ERR_ARG, "%s: window %d: marginalize_frame: frame %d of %d", who, windows[i], idx[j], nF);
    rounds = std::max(rounds, k); }
  std::vector<long long> off(2*(size_t)n); long long tot = 0;
  for (int i=0;i<n;i++) { const int N = kCP + 6*(bs[i]->nF - (k_begin[i+1] - k_begin[i])); off[2*i] = tot; tot += (long long)N*N; off[2*i+1] = tot; tot += N; }
  const bool prior = HM_out || bM_out;
  { int rc = stage_reserve(c, need(n, sizeof(BAWinDev)) + need((size_t)n*std::max(rounds, 1), 4) + need(2*(size_t)n, 8), need(tot, 8), need(tot, 8), who); if (rc) return rc; }
  BAWinDev *Wh, *Wd; int *Ih, *Id; long long *Oh, *Od;
  stage2(c, n, &Wh, &Wd); stage2(c, (size_t)n*std::max(rounds, 1), &Ih, &Id); stage2(c, 2*(size_t)n, &Oh, &Od);
  for (int i=0;i<n;i++) { Wh[i] = win_of(bs[i]); Oh[2*i] = off[2*i]; Oh[2*i+1] = off[2*i+1];
    for (int r=0;r<rounds;r++) Ih[(size_t)r*n + i] = (k_begin[i] + r < k_begin[i+1]) ? idx[k_begin[i] + r] : -1; }
  { int rc = stage_up(c); if (rc) return rc; }
  double* out_d = c->ba_scr.take<double>(tot); double* out_h = c->ba_scr_host.take<double>(tot);
  for (int r=0;r<rounds;r++) launch_ba_marg_frame(Wd, n, Id + (size_t)r*n, st);
  c->launches += rounds;
  if (prior) { launch_ba_prior_gather(Wd, n, Od, out_d, st); c->launches += 1; CK(cudaMemcpyAsync(out_h, out_d, (size_t)tot*sizeof(double), cudaMemcpyDeviceToHost, st)); }
  BA_WAIT(); CK(cudaGetLastError());
  long long hm = 0, bm = 0;
  for (int i=0;i<n;i++) { BAState* b = bs[i]; const int k = k_begin[i+1] - k_begin[i];
    for (int j=k_begin[i]; j<k_begin[i+1]; j++) { const int x = idx[j];
      if (x < b->n_pinned) { { SDV_GUARD_TRK(c); frame_unpin(c, b->pinned[x]); } for (int m=x; m+1<b->n_pinned; m++) b->pinned[m] = b->pinned[m+1]; b->n_pinned--; } }
    if (k > 0) { b->nF -= k; b->nP = 0; b->nR = 0; }                     // points/residuals are stale: the caller re-flattens the window (sdv_ba_set_points)
    const long long N = kCP + 6*b->nF;
    if (HM_out) memcpy(HM_out + hm, out_h + off[2*i], (size_t)(N*N)*sizeof(double));
    if (bM_out) memcpy(bM_out + bm, out_h + off[2*i+1], (size_t)N*sizeof(double));
    hm += N*N; bm += N; }
  return SDV_OK;
}
int sdv_ba_marginalize_frame(sdv_ctx* c, int idx) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG;
  const int32_t w = ba_index(c, c->ba), kb[2] = {0, 1}, x = idx;
  return sdv_ba_marginalize_frames_batch(c, 1, &w, kb, &x, nullptr, nullptr);
}
int sdv_ba_get_prior(sdv_ctx* c, int* dim, double* HM, double* bM) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; const int N = kCP + 6*b->nF;
  if (dim) *dim = N;
  if (HM) CK(cudaMemcpyAsync(HM, b->hdr->HM, (size_t)N*N*sizeof(double), cudaMemcpyDeviceToHost, c->st_ba));
  if (bM) CK(cudaMemcpyAsync(bM, b->hdr->bM, (size_t)N*sizeof(double), cudaMemcpyDeviceToHost, c->st_ba));
  BA_WAIT(); return SDV_OK;
}
int sdv_ba_get_linearized(sdv_ctx* c, float* res_toZero2, int32_t* isLinearized) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  if (res_toZero2) CK(cudaMemcpyAsync(res_toZero2, b->R.res_toZero, (size_t)b->nR*2*sizeof(float), cudaMemcpyDeviceToHost, c->st_ba));
  if (isLinearized) CK(cudaMemcpyAsync(isLinearized, b->R.isLinearized, (size_t)b->nR*sizeof(int32_t), cudaMemcpyDeviceToHost, c->st_ba));
  BA_WAIT(); return SDV_OK;
}
int sdv_ba_get_system(sdv_ctx* c, double* HA, double* bA, double* Hsc, double* bsc, double* lastHS, double* lastbS) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; const int N = kCP + 6*b->nF;
#define DN(dst, src, cnt) do { if (dst) CK(cudaMemcpyAsync(dst, b->hdr->src, (size_t)(cnt)*sizeof(double), cudaMemcpyDeviceToHost, c->st_ba)); } while (0)
  DN(HA, HA, N*N); DN(bA, bA, N); DN(Hsc, Hsc, N*N); DN(bsc, bsc, N); DN(lastHS, lastHS, N*N); DN(lastbS, lastbS, N);
#undef DN
  BA_WAIT(); return SDV_OK;
}
int sdv_ba_get_precalc(sdv_ctx* c, int host, int target, float out27[27], double adHost36[36], double adTarget36[36], float adHTdelta6[6]) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; const int nF = b->nF;
  if (host < 0 || target < 0 || host >= nF || target >= nF) return SDV_ERR_ARG;
  PrecalcDev p; CK(cudaMemcpy(&p, &b->hdr->precalc[host*nF+target], sizeof(p), cudaMemcpyDeviceToHost));
  for (int i=0;i<9;i++) { out27[i] = p.KRKi[i]; out27[12+i] = p.R0[i]; } for (int i=0;i<3;i++) { out27[9+i] = p.Kt[i]; out27[21+i] = p.t0[i]; }
  out27[24] = p.aff[0]; out27[25] = p.aff[1]; out27[26] = p.b0;
  const int idx = host + target*nF;
  CK(cudaMemcpy(adHost36, b->hdr->adHost + idx*36, 36*sizeof(double), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(adTarget36, b->hdr->adTarget + idx*36, 36*sizeof(double), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(adHTdelta6, b->hdr->adHTdeltaF + idx*6, 6*sizeof(float), cudaMemcpyDeviceToHost));
  return SDV_OK;
}

} // extern "C"
