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
#include <cmath>

using namespace sdv;

namespace sdv {
void ba_destroy(sdv_ctx* c) {
  if (!c) return;
  for (BAState* b : c->ba_windows) { if (!b) continue;
    for (int i=0;i<b->n_pinned;i++) frame_unpin(c, b->pinned[i]);
    cudaFree(b->hdr); cudaFreeHost(b->hdr_host); cudaFree(b->pool); cudaFree(b->partials); cudaFree(b->thbuf); cudaFree(b->thcount); delete b; }
  c->ba_windows.clear(); c->ba = nullptr;
  c->ba_wins_dev.release(); c->ba_wins_host.release();
  if (c->ba_graph) { cudaGraphExecDestroy(c->ba_graph); c->ba_graph = nullptr; }
}
}

static int ba_select(sdv_ctx* c, int window) {
  if (window < 0 || window > 1<<20) return SDV_ERR_ARG;
  if ((int)c->ba_windows.size() <= window) c->ba_windows.resize(window+1, nullptr);
  if (!c->ba_windows[window]) {
    BAState* b = new BAState(); memset(b, 0, sizeof(*b)); c->ba_windows[window] = b;
    CK(cudaMalloc(&b->hdr, sizeof(BAHeader))); CK(cudaMemset(b->hdr, 0, sizeof(BAHeader)));
    CK(cudaMallocHost(&b->hdr_host, sizeof(BAHeader))); memset(b->hdr_host, 0, sizeof(BAHeader));
    CK(cudaMalloc(&b->thcount, sizeof(int))); CK(cudaMemset(b->thcount, 0, sizeof(int)));
  }
  c->ba = c->ba_windows[window]; return SDV_OK;
}
static int ba_get(sdv_ctx* c, BAState** out) {
  if (!c->ba) { int rc = ba_select(c, 0); if (rc) return rc; }
  *out = c->ba; return SDV_OK;
}

template <typename T> static T* bump(char*& p, size_t n) { T* r = reinterpret_cast<T*>(p); p += ((n*sizeof(T) + 255)/256)*256; return r; }

static size_t ba_layout(BAState* b, char* base, int cp, int cr) {
  char* p = base;
  BAPointsDev& P = b->P; BAResDev& R = b->R;
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
static int ba_alloc(sdv_ctx* c, BAState* b, int nP, int nR, int nF) {
  if (nP <= b->capP && nR <= b->capR) return SDV_OK;
  int cp = nP + nP/4 + 256, cr = nR + nR/4 + 1024;
  cudaFree(b->pool); cudaFree(b->partials); cudaFree(b->thbuf); b->pool = nullptr; b->partials = nullptr; b->thbuf = nullptr; b->capP = b->capR = 0;
  size_t bytes = ba_layout(b, nullptr, cp, cr);
  CK(cudaMalloc(&b->pool, bytes)); CK(cudaMemset(b->pool, 0, bytes)); b->pool_bytes = bytes;
  ba_layout(b, (char*)b->pool, cp, cr);
  CK(cudaMalloc(&b->partials, (size_t)((cr + 127)/128 + 1)*sizeof(double)));
  CK(cudaMalloc(&b->thbuf, (size_t)cr*sizeof(float)));
  b->capP = cp; b->capR = cr; (void)nF;
  return SDV_OK;
}

static BAWinDev win_of(const BAState* b) { BAWinDev w; w.hdr = b->hdr; w.P = b->P; w.R = b->R; w.partials = b->partials; w.thbuf = b->thbuf; w.thcount = b->thcount; return w; }
// device array of window descriptors for one (batched) launch sequence; maxP/maxR size the grids
static int ba_wins(sdv_ctx* c, int n, BAState* const* bs, const BAWinDev** out, int* maxP, int* maxR) {
  const size_t bytes = Scratch::need(n, sizeof(BAWinDev));
  if (c->ba_wins_dev.reserve(bytes, c->st_ba) || c->ba_wins_host.reserve(bytes, c->st_ba)) return ctx_fail(c, SDV_ERR_CUDA, "BA: descriptors of %d windows", n);
  c->ba_wins_dev.reset(); c->ba_wins_host.reset(); BAWinDev* d = c->ba_wins_dev.take<BAWinDev>(n); BAWinDev* h = c->ba_wins_host.take<BAWinDev>(n); int mp = 1, mr = 1;
  CK(cudaStreamSynchronize(c->st_ba));                                          // the pinned staging array may still feed a previous launch sequence
  for (int i=0;i<n;i++) { h[i] = win_of(bs[i]); if (bs[i]->nP > mp) mp = bs[i]->nP; if (bs[i]->nR > mr) mr = bs[i]->nR; }
  CK(cudaMemcpyAsync(d, h, (size_t)n*sizeof(BAWinDev), cudaMemcpyHostToDevice, c->st_ba));
  *out = d; if (maxP) *maxP = mp; if (maxR) *maxR = mr;
  return SDV_OK;
}
#define WIN1() const BAWinDev* wins; int maxP, maxR; { int rcw = ba_wins(c, 1, &b, &wins, &maxP, &maxR); if (rcw) return rcw; }

static int ba_pull_scalars(sdv_ctx* c, BAState* b) {                        // energyP .. end of header
  const size_t off = offsetof(BAHeader, energyP), len = sizeof(BAHeader) - off;
  CK(cudaMemcpyAsync((char*)b->hdr_host + off, (char*)b->hdr + off, len, cudaMemcpyDeviceToHost, c->st_ba));
  CK(cudaStreamSynchronize(c->st_ba)); CK(cudaGetLastError());
  return SDV_OK;
}

extern "C" {

int sdv_ba_set_window(sdv_ctx* c, int nF, const uint64_t* frame_ids, const double* T_evalPT7, const double* state10, const double* state_zero10,
                      const float* ab_exposure, const int32_t* frameID, const float* frameEnergyTH, const double calib_value_scaled[4],
                      const double* HM, const double* bM) { SDV_GUARD_BA(c);
  if (!c || nF < 1 || nF > SDV_MAX_FRAMES_WINDOW || !frame_ids || !T_evalPT7 || !state10 || !state_zero10 || !calib_value_scaled) return SDV_ERR_ARG;
  SDV_GUARD_TRK(c);                                                           // frame table, pins, level-0 texel pool and the ingest join belong to the tracker domain
  CK(cudaSetDevice(c->device));
  BAState* b; int rc = ba_get(c, &b); if (rc) return rc;
  FrameDev* Fr[SDV_MAX_FRAMES_WINDOW]; int cam0 = -1;                         // one size per window: BAHeader::w/h are the window's frames' size
  for (int f=0; f<nF; f++) { int rcf = job_frame(c, "sdv_ba_set_window", f, frame_ids[f], -1, -1, nullptr, &Fr[f]); if (rcf) return rcf;
    const int cam = Fr[f]->cam; if (cam0 < 0) cam0 = cam;
    if (!same_size(c, cam, cam0)) return ctx_fail(c, SDV_ERR_ARG, "BA frame %d is %dx%d but frame 0 is %dx%d: one window holds frames of one size", f, c->cam_w[cam], c->cam_h[cam], c->cam_w[cam0], c->cam_h[cam0]); }
  for (int i=0;i<b->n_pinned;i++) frame_unpin(c, b->pinned[i]);          // the window is being replaced: drop its references, take the new ones
  b->n_pinned = nF; for (int f=0; f<nF; f++) { b->pinned[f] = frame_ids[f]; frame_pin(c, frame_ids[f]); }
  BAHeader* H = b->hdr_host; memset(H, 0, sizeof(BAHeader));
  H->nF = nF; H->w = c->cam_w[cam0]; H->h = c->cam_h[cam0]; H->dim = kCP + 6*nF; b->nF = nF;
  BASettingsDev& s = H->set;
  s.huberTH = c->set.huberTH; s.outlierTHSumComponent = c->set.outlierTHSumComponent; s.idepthFixPrior = c->set.idepthFixPrior;
  s.initialRotPrior = 1e11f; s.initialTransPrior = 1e10f; s.initialCalibHessian = 5e9f;            // settings.cpp:23-27
  s.frameEnergyTHConstWeight = 0.5f; s.frameEnergyTHN = 0.7f; s.frameEnergyTHFacMedian = 1.5f; s.overallEnergyTHWeight = 1;   // :108-111
  s.thOptIterations = 1.2f; s.minOptIterations = 1; s.solverModeDelta = 0.00001;                  // :56-57, :35
  BACalibDev& cal = H->calib;                                                                       // CalibHessian ctor: setValueScaled + value_zero = value
  const float SFI = 1.0f/50.0f;
  for (int i=0;i<4;i++) { cal.value_scaled[i] = calib_value_scaled[i]; cal.sf[i] = (float)calib_value_scaled[i]; cal.value[i] = SFI*calib_value_scaled[i];
    cal.value_zero[i] = cal.value[i]; cal.vmvz[i] = 0; cal.step[i] = 0; cal.value_backup[i] = cal.value[i]; }
  cal.si[0] = 1.0f/cal.sf[0]; cal.si[1] = 1.0f/cal.sf[1]; cal.si[2] = -cal.sf[2]/cal.sf[0]; cal.si[3] = -cal.sf[3]/cal.sf[1];
  for (int f=0; f<nF; f++) {
    BAFrameDev& F = H->frames[f];
    F.evalPT = se3_from7(T_evalPT7 + 7*f);
    for (int i=0;i<10;i++) { F.state[i] = state10[10*f+i]; F.state_zero[i] = state_zero10[10*f+i]; F.state_backup[i] = F.state[i]; F.step[i] = 0; }
    F.ab_exposure = ab_exposure ? ab_exposure[f] : 1.0f; F.frameID = frameID ? frameID[f] : f; F.frameEnergyTH = frameEnergyTH ? frameEnergyTH[f] : 8*8*8;
    { int rc0 = ensure_lvl0(c, *Fr[f]); if (rc0) return rc0; }
    F.img0 = Fr[f]->lvl[0];
  }
  const int N = H->dim;
  if (HM) memcpy(H->HM, HM, (size_t)N*N*sizeof(double));
  if (bM) memcpy(H->bM, bM, (size_t)N*sizeof(double));
  { int rcj = join_ingest(c); if (rcj) return rcj; }                          // the keyframes' pyramids (ingest stream) and level-0 texels (tracker stream) are complete
  CK(cudaEventRecord(c->ev_xdom, c->st)); CK(cudaStreamWaitEvent(c->st_ba, c->ev_xdom, 0));   // before the back-end stream reads them; pinned frames cannot change afterwards
  CK(cudaMemcpyAsync(b->hdr, H, sizeof(BAHeader), cudaMemcpyHostToDevice, c->st_ba));
  CK(cudaStreamSynchronize(c->st_ba));
  return SDV_OK;
}

int sdv_ba_set_points(sdv_ctx* c, int nP, const float* uv, const float* idepth, const float* idepth_zero, const float* color8, const float* weights8,
                      const int32_t* host, const int32_t* hasDepthPrior, const int32_t* isFromSensor, const int32_t* res_begin,
                      int nR, const int32_t* r_point, const int32_t* r_host, const int32_t* r_target, const int32_t* r_hasMatcher,
                      const float* r_matcher, const int32_t* r_isNew) { SDV_GUARD_BA(c);
  if (!c || !c->ba || nP < 0 || nR < 0) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  BAState* b = c->ba; const int nF = b->nF;
  int rc = ba_alloc(c, b, nP, nR, nF); if (rc) return rc;
  // ---- makeIDX mirror (EnergyFunctional.cpp:761-782): validate the flattening and build the index lists the kernels walk
  std::vector<int> rot((size_t)nP*kMaxF, -1), pair_begin(kMaxF*kMaxF+1, 0), pair_res(nR), host_begin(kMaxF+1, 0);
  if (nP > 0 && (!uv || !idepth || !idepth_zero || !color8 || !weights8 || !host || !hasDepthPrior || !isFromSensor || !res_begin)) return SDV_ERR_ARG;
  if (nR > 0 && (!r_point || !r_host || !r_target || !r_hasMatcher || !r_matcher || !r_isNew)) return SDV_ERR_ARG;
  // the CSR must be sane BEFORE any residual is indexed through it: [0 .. nR], monotone
  if (nP > 0 && (res_begin[0] != 0 || res_begin[nP] != nR)) return ctx_fail(c, SDV_ERR_ARG, "res_begin must span all residuals (res_begin[0]=%d, res_begin[nP]=%d, nR=%d)", res_begin[0], res_begin[nP], nR);
  if (nP == 0 && nR != 0) return ctx_fail(c, SDV_ERR_ARG, "residuals without points");
  for (int p=0;p<nP;p++) if (res_begin[p] > res_begin[p+1]) return ctx_fail(c, SDV_ERR_ARG, "res_begin not monotone at point %d", p);
  for (int p=0;p<nP;p++) {
    if (host[p] < 0 || host[p] >= nF || (p > 0 && host[p] < host[p-1])) return ctx_fail(c, SDV_ERR_ARG, "points must be grouped by host frame in frame order (ef->allPoints order)");
    for (int r=res_begin[p]; r<res_begin[p+1]; r++) {
      if (r_point[r] != p || r_host[r] != host[p] || r_target[r] < 0 || r_target[r] >= nF || r_target[r] == host[p]) return ctx_fail(c, SDV_ERR_ARG, "residual %d inconsistent with its point", r);
      if (rot[(size_t)p*kMaxF + r_target[r]] >= 0) return ctx_fail(c, SDV_ERR_ARG, "two residuals of point %d share a target", p);
      rot[(size_t)p*kMaxF + r_target[r]] = r;
    }
    host_begin[host[p]+1] = p+1;
  }
  for (int f=1; f<=nF; f++) if (host_begin[f] < host_begin[f-1]) host_begin[f] = host_begin[f-1];
  for (int r=0;r<nR;r++) pair_begin[r_host[r] + nF*r_target[r] + 1]++;
  for (int k=0;k<nF*nF;k++) pair_begin[k+1] += pair_begin[k];
  { std::vector<int> cur(pair_begin.begin(), pair_begin.end()-1); for (int r=0;r<nR;r++) pair_res[cur[r_host[r] + nF*r_target[r]]++] = r; }
  BAPointsDev& P = b->P; BAResDev& R = b->R; cudaStream_t st = c->st_ba;
#define UP(dst, src, n, T) do { if ((n) > 0) CK(cudaMemcpyAsync(dst, src, (size_t)(n)*sizeof(T), cudaMemcpyHostToDevice, st)); } while (0)
  UP(P.uv, uv, (size_t)nP*2, float); UP(P.idepth, idepth, nP, float); UP(P.idepth_zero, idepth_zero, nP, float); UP(P.idepth_backup, idepth, nP, float);
  UP(P.color, color8, (size_t)nP*8, float); UP(P.weights, weights8, (size_t)nP*8, float);
  UP(P.host, host, nP, int); UP(P.hasDepthPrior, hasDepthPrior, nP, int); UP(P.isFromSensor, isFromSensor, nP, int); UP(P.res_begin, res_begin, nP+1, int);
  UP(P.res_of_target, rot.data(), (size_t)nP*kMaxF, int);
  UP(R.point, r_point, nR, int); UP(R.host, r_host, nR, int); UP(R.target, r_target, nR, int); UP(R.hasMatcher, r_hasMatcher, nR, int);
  UP(R.matcher, r_matcher, (size_t)nR*2, float); UP(R.isNew, r_isNew, nR, int);
  UP(R.pair_begin, pair_begin.data(), nF*nF+1, int); UP(R.pair_res, pair_res.data(), nR, int); UP(R.host_begin, host_begin.data(), nF+1, int);
#undef UP
  if (nP > 0) { CK(cudaMemsetAsync(P.step, 0, (size_t)nP*sizeof(float), st)); CK(cudaMemsetAsync(P.maxRelBaseline, 0, (size_t)nP*sizeof(float), st)); CK(cudaMemsetAsync(P.numGoodResiduals, 0, (size_t)nP*sizeof(int), st)); }
  if (nR > 0) { CK(cudaMemsetAsync(R.isActive, 0, (size_t)nR*sizeof(int), st)); CK(cudaMemsetAsync(R.toRemove, 0, (size_t)nR*sizeof(int), st));
    CK(cudaMemsetAsync(R.J, 0, (size_t)nR*24*sizeof(float), st)); CK(cudaMemsetAsync(R.efJ, 0, (size_t)nR*24*sizeof(float), st)); CK(cudaMemsetAsync(R.JpJdF, 0, (size_t)nR*8*sizeof(float), st));
    CK(cudaMemsetAsync(R.center, 0, (size_t)nR*3*sizeof(float), st)); }
  b->nP = nP; b->nR = nR;
  b->hdr_host->nP = nP; b->hdr_host->nR = nR;
  CK(cudaMemcpyAsync(&b->hdr->nP, &b->hdr_host->nP, 2*sizeof(int), cudaMemcpyHostToDevice, st));
  { WIN1(); launch_ba_setup(wins, 1, maxP, st); launch_ba_reset_oob(wins, 1, maxR, st); }
  CK(cudaStreamSynchronize(st)); CK(cudaGetLastError());
  c->launches += 3;
  return SDV_OK;
}

int sdv_ba_clear(sdv_ctx* c) { SDV_GUARD_BA(c);               // empties the selected window and drops its references to frame images
  if (!c) return SDV_ERR_ARG; if (!c->ba) return SDV_OK; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  CK(cudaStreamSynchronize(c->st_ba));
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
  CK(cudaMemcpyAsync(&b->hdr->calib, &cal, sizeof(BACalibDev), cudaMemcpyHostToDevice, c->st_ba)); CK(cudaStreamSynchronize(c->st_ba));
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
int sdv_ba_apply_res(sdv_ctx* c) { SDV_GUARD_BA(c); if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; WIN1(); launch_ba_apply(wins, 1, maxR, GATE_ALWAYS, c->st_ba); c->launches++; CK(cudaStreamSynchronize(c->st_ba)); return SDV_OK; }
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
  CK(cudaStreamSynchronize(c->st_ba)); CK(cudaGetLastError());
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
        CK(cudaStreamSynchronize(st));
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
  CK(cudaStreamSynchronize(st)); CK(cudaGetLastError());
  CK(cudaEventElapsedTime(&c->ba_last_ms, c->ba_ev0, c->ba_ev1));
  for (int i=0;i<n;i++) { const BAHeader* H = bs[i]->hdr_host;
    if (rmse_out) rmse_out[i] = (bs[i]->nF < 2) ? 0.f : H->rmse;
    if (iterations_out) iterations_out[i] = H->opt_iterations;
    if (accepts_out) accepts_out[i] = H->opt_accepts; }
  return SDV_OK;
}
float sdv_ba_last_kernel_ms(sdv_ctx* c) { return c ? c->ba_last_ms : 0.f; }
int sdv_ba_optimize(sdv_ctx* c, int mnumOptIts, float* rmse_out, int32_t* iterations_out, int32_t* accepts_out) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG;
  int32_t w = -1; for (size_t i=0;i<c->ba_windows.size();i++) if (c->ba_windows[i] == c->ba) w = (int32_t)i;
  return sdv_ba_optimize_batch(c, 1, &w, mnumOptIts, rmse_out, iterations_out, accepts_out);
}

// ---- read-back (what the reference leaves in FrameHessian / PointHessian / PointFrameResidual / EnergyFunctional)
int sdv_ba_get_frames(sdv_ctx* c, double* T_evalPT7, double* state10, double* step10, float* frameEnergyTH, double* PRE_worldToCam7, double calib_value[4], double calib_step[4]) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  CK(cudaMemcpyAsync(b->hdr_host, b->hdr, offsetof(BAHeader, precalc), cudaMemcpyDeviceToHost, c->st_ba)); CK(cudaStreamSynchronize(c->st_ba));
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
  CK(cudaStreamSynchronize(c->st_ba)); return SDV_OK;
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
  CK(cudaStreamSynchronize(c->st_ba));
  if (energies3) for (int i=0;i<n;i++) { energies3[3*i] = e0[i]; energies3[3*i+1] = e1[i]; energies3[3*i+2] = e2[i]; }
  return SDV_OK;
}
// ------------------------------------------------------------------------------------------------ keyframe hand-over (FullSystem::makeKeyFrame, FullSystem.cpp:1152-1171)
int sdv_ba_flag_points(sdv_ctx* c, const int32_t* selected, int32_t* status_out) { SDV_GUARD_BA(c);
  if (!c || !c->ba || !selected) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  if (b->nP <= 0) return ctx_fail(c, SDV_ERR_STATE, "flag_points: window has no points (call sdv_ba_set_points)");
  WIN1();
  CK(cudaMemcpyAsync(b->P.marg_status, selected, (size_t)b->nP*sizeof(int32_t), cudaMemcpyHostToDevice, c->st_ba));
  launch_ba_marg_flag(wins, 1, maxP, c->st_ba); c->launches += 1;
  if (status_out) CK(cudaMemcpyAsync(status_out, b->P.marg_status, (size_t)b->nP*sizeof(int32_t), cudaMemcpyDeviceToHost, c->st_ba));
  CK(cudaStreamSynchronize(c->st_ba)); CK(cudaGetLastError());
  return SDV_OK;
}
int sdv_ba_marginalize_points(sdv_ctx* c, const int32_t* status) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  if (b->nP <= 0) return ctx_fail(c, SDV_ERR_STATE, "marginalize_points: window has no points");
  WIN1();
  if (status) CK(cudaMemcpyAsync(b->P.marg_status, status, (size_t)b->nP*sizeof(int32_t), cudaMemcpyHostToDevice, c->st_ba));
  launch_ba_marg_points(wins, 1, maxP, c->st_ba); c->launches += 4;
  CK(cudaStreamSynchronize(c->st_ba)); CK(cudaGetLastError());
  return SDV_OK;
}
int sdv_ba_marginalize_frame(sdv_ctx* c, int idx) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  if (idx < 0 || idx >= b->nF || b->nF < 2) return ctx_fail(c, SDV_ERR_ARG, "marginalize_frame: frame %d of %d", idx, b->nF);
  WIN1();
  launch_ba_marg_frame(wins, 1, idx, c->st_ba); c->launches += 1;
  CK(cudaStreamSynchronize(c->st_ba)); CK(cudaGetLastError());
  if (idx < b->n_pinned) { { SDV_GUARD_TRK(c); frame_unpin(c, b->pinned[idx]); } for (int i=idx; i+1<b->n_pinned; i++) b->pinned[i] = b->pinned[i+1]; b->n_pinned--; }
  b->nF -= 1; b->nP = 0; b->nR = 0;                                          // points/residuals are stale: the caller re-flattens the window (sdv_ba_set_points)
  return SDV_OK;
}
int sdv_ba_get_prior(sdv_ctx* c, int* dim, double* HM, double* bM) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; const int N = kCP + 6*b->nF;
  if (dim) *dim = N;
  if (HM) CK(cudaMemcpyAsync(HM, b->hdr->HM, (size_t)N*N*sizeof(double), cudaMemcpyDeviceToHost, c->st_ba));
  if (bM) CK(cudaMemcpyAsync(bM, b->hdr->bM, (size_t)N*sizeof(double), cudaMemcpyDeviceToHost, c->st_ba));
  CK(cudaStreamSynchronize(c->st_ba)); return SDV_OK;
}
int sdv_ba_get_linearized(sdv_ctx* c, float* res_toZero2, int32_t* isLinearized) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba;
  if (res_toZero2) CK(cudaMemcpyAsync(res_toZero2, b->R.res_toZero, (size_t)b->nR*2*sizeof(float), cudaMemcpyDeviceToHost, c->st_ba));
  if (isLinearized) CK(cudaMemcpyAsync(isLinearized, b->R.isLinearized, (size_t)b->nR*sizeof(int32_t), cudaMemcpyDeviceToHost, c->st_ba));
  CK(cudaStreamSynchronize(c->st_ba)); return SDV_OK;
}
int sdv_ba_get_system(sdv_ctx* c, double* HA, double* bA, double* Hsc, double* bsc, double* lastHS, double* lastbS) { SDV_GUARD_BA(c);
  if (!c || !c->ba) return SDV_ERR_ARG; CK(cudaSetDevice(c->device)); BAState* b = c->ba; const int N = kCP + 6*b->nF;
#define DN(dst, src, cnt) do { if (dst) CK(cudaMemcpyAsync(dst, b->hdr->src, (size_t)(cnt)*sizeof(double), cudaMemcpyDeviceToHost, c->st_ba)); } while (0)
  DN(HA, HA, N*N); DN(bA, bA, N); DN(Hsc, Hsc, N*N); DN(bsc, bsc, N); DN(lastHS, lastHS, N*N); DN(lastbS, lastbS, N);
#undef DN
  CK(cudaStreamSynchronize(c->st_ba)); return SDV_OK;
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
