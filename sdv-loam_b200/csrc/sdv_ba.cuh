// sdv_ba.cuh — device layout of the sliding-window back-end (EnergyFunctional + FullSystem::optimize) — DESIGN.md §5.
//
// The reference's pointer graph (FrameHessian -> PointHessian -> PointFrameResidual, EFFrame/EFPoint/EFResidual mirrors) is
// flattened by the caller into the reference's own iteration order: frames = ef->frames, points = ef->allPoints
// (EnergyFunctional.cpp:761-782; contiguous per host frame), residuals grouped per point in residualsAll order.
#pragma once
#include <cuda_runtime.h>
#include <cstddef>
#include "sdv_math.cuh"

namespace sdv {

constexpr int kMaxF = 8;                 // SDV_MAX_FRAMES_WINDOW
constexpr int kCP = 4;                   // CPARS
constexpr int kMaxDim = kCP + 6*kMaxF;   // 52
constexpr int kNTop = 66;                // per (host,target) bucket: 55 (10x10 upper) + 10 (gradient column) + 1 (r.r)   AccumulatorApprox
enum { RS_IN = 0, RS_OOB = 1, RS_OUTLIER = 2 };

struct BAFrameDev {
  SE3d evalPT; double state[10], state_zero[10], state_backup[10], step[10], state_scaled[10];
  SE3d PRE_w2c, PRE_c2w;
  double nullspaces_pose[36], nullspaces_scale[6];
  double prior[6], delta[6], delta_prior[6];
  float ab_exposure; int frameID; float frameEnergyTH; int pad;
  const float4* img0;                    // target->dI  (level 0 texels {I,dx,dy,.})
};
struct BACalibDev { double value[4], value_zero[4], value_scaled[4], step[4], value_backup[4], vmvz[4], cPrior[4]; float sf[4], si[4], cDeltaF[4]; };
struct PrecalcDev { float KRKi[9], Kt[3], R0[9], t0[3], aff[2], b0; };        // FrameFramePrecalc (HessianBlocks.h:51-79), the fields linearize reads

struct BASettingsDev {
  float huberTH, outlierTHSumComponent, idepthFixPrior, initialRotPrior, initialTransPrior, initialCalibHessian;
  float frameEnergyTHConstWeight, frameEnergyTHN, frameEnergyTHFacMedian, overallEnergyTHWeight, thOptIterations;
  int minOptIterations; double solverModeDelta;
};

struct BAHeader {                        // one per window, lives in device memory; small enough to stay L2/L1 resident
  int nF, nP, nR, w, h, dim;
  BASettingsDev set;
  BACalibDev calib;
  BAFrameDev frames[kMaxF];
  PrecalcDev precalc[kMaxF*kMaxF];       // [host*nF + target]
  double adHost[kMaxF*kMaxF*36], adTarget[kMaxF*kMaxF*36];      // [h + t*nF]
  float  adHostF[kMaxF*kMaxF*36], adTargetF[kMaxF*kMaxF*36], adHTdeltaF[kMaxF*kMaxF*6];
  double HM[kMaxDim*kMaxDim], bM[kMaxDim];
  // accumulators written by the accumulate kernels (float sums in the reference's order, incl. 1k/1M tiers)
  float  accTop[kMaxF*kMaxF*kNTop]; int accTopNum[kMaxF*kMaxF];
  float  accD[kMaxF*kMaxF*kMaxF*36]; int accDNum[kMaxF*kMaxF*kMaxF];   // [h + nF*t1 + nF^2*t2] 6x6 (rows/cols 6,7 of the 8x8 are identically 0)
  float  accE[kMaxF*kMaxF*24], accEB[kMaxF*kMaxF*6], accHcc[16], accbc[4];
  // solve outputs
  double HA[kMaxDim*kMaxDim], bA[kMaxDim], Hsc[kMaxDim*kMaxDim], bsc[kMaxDim], lastHS[kMaxDim*kMaxDim], lastbS[kMaxDim], lastX[kMaxDim];
  float  xAd[kMaxF*kMaxF*6], xF[kMaxDim];
  // scalars
  double energyP, energyL, energyM; int resInA; int canbreak; float sums[8];
  unsigned int ticket;
  // device-resident Gauss-Newton control (FullSystem::optimize, FullSystemOptimize.cpp:391-458): set by ba_decide_kernel
  int flags;                             // BA_ACTIVE | BA_APPLY | BA_RELOAD
  int mnumOptIts, iteration, opt_iterations, opt_accepts;
  double lambda, lastEnergy, lastEnergyL, lastEnergyM;
  float rmse;
  // cached orthonormal basis of the pose+scale nullspaces (valid while the evaluation points do not change)
  int ortho_valid; double orthoU[7*kMaxDim]; double orthoS[7];
  // stitch scratch: AH*M and AT*M per top bucket, AH_ij*D and AT_ij*D per Schur bucket (fp64, reference operation order)
  double topT1[kMaxF*kMaxF*36], topT3[kMaxF*kMaxF*36], scT1[kMaxF*kMaxF*kMaxF*36], scT3[kMaxF*kMaxF*kMaxF*36];
};
enum { BA_ACTIVE = 1, BA_APPLY = 2, BA_RELOAD = 4 };
enum { GATE_ALWAYS = 0, GATE_ACTIVE = 1, GATE_APPLY = 2, GATE_RELOAD = 4 };

struct BAPointsDev {                     // SoA over points
  float2* uv; float* idepth; float* idepth_zero; float* idepth_backup; float* step;
  float* color; float* weights;          // [nP*8]
  int* host; int* hasDepthPrior; int* isFromSensor; int* res_begin;            // res_begin[nP+1]
  float* priorF; float* deltaF; float* HdiF; float* bdSumF; float* Hdd_accAF; float* bd_accAF; float* Hcd_accAF;   // Hcd [nP*4]
  float* idepth_hessian; float* maxRelBaseline; int* numGoodResiduals; int* ngood;
  int* res_of_target;                    // [nP*kMaxF] residual index towards target t or -1
  int* marg_status;                      // keyframe hand-over: 0 keep / 1 PS_DROP / 2 PS_MARGINALIZE (flagPointsForRemoval)
};
struct BAResDev {                        // SoA over residuals
  int* point; int* host; int* target; int* hasMatcher; float2* matcher; int* isNew;
  int* state_state; int* state_NewState; float* state_energy; float* state_NewEnergy; float* state_NewEnergyWithOutlier;
  int* isActive; int* toRemove;
  float* J; float* efJ;                  // [nR*24] {resF[2], Jpdxi[0][6], Jpdxi[1][6], Jpdc[0][4], Jpdc[1][4], Jpdd[2]}
  float* JpJdF;                          // [nR*8]
  float* center;                         // [nR*3] centerProjectedTo
  float2* res_toZero; int* isLinearized; // EFResidual::res_toZeroF / isLinearized (fixLinearizationF)
  int* pair_begin; int* pair_res;        // residual indices grouped by (host + nF*target), in residual order
  int* host_begin;                       // point range per host frame [nF+1]
};

struct BAWinDev {                        // one window as the batched kernels see it (blockIdx.y selects the window)
  BAHeader* hdr; BAPointsDev P; BAResDev R; double* partials; float* thbuf; int* thcount;
};

struct BAState {
  BAHeader* hdr; BAHeader* hdr_host;     // device / pinned host mirror
  BAPointsDev P; BAResDev R; int capP, capR; int nF, nP, nR;
  void* pool; size_t pool_bytes;         // one allocation backing P and R
  double* partials; float* thbuf; int* thcount;
  int opt_iterations, opt_accepts;
  float last_ms;
  unsigned long long pinned[kMaxF]; int n_pinned;   // frame handles whose level-0 texels this window's header points at (sdv_ctx::pins)
};

// launchers (sdv_ba_kernels.cu): every kernel is batched over windows (grid.y = window); `gate` = flags the window must have set
void launch_ba_setup(const BAWinDev* wins, int W, int maxP, cudaStream_t st);                 // setState/Zero, takeData, adjoints, precalc, deltas
void launch_ba_reset_oob(const BAWinDev* wins, int W, int maxR, cudaStream_t st);
void launch_ba_linearize(const BAWinDev* wins, int W, int maxR, int fix, int gate, cudaStream_t st);
void launch_ba_apply(const BAWinDev* wins, int W, int maxR, int gate, cudaStream_t st);
void launch_ba_energies(const BAWinDev* wins, int W, int gate, cudaStream_t st);
void launch_ba_accumulate(const BAWinDev* wins, int W, int maxP, int gate, cudaStream_t st);
void launch_ba_solve(const BAWinDev* wins, int W, int maxP, int iteration, double lambda, int use_hdr_ctl, int gate, cudaStream_t st);
void launch_ba_backup(const BAWinDev* wins, int W, int maxP, int gate, cudaStream_t st);
void launch_ba_step(const BAWinDev* wins, int W, float stepfac, int load_backup, int gate, cudaStream_t st);
void launch_ba_reanchor(const BAWinDev* wins, int W, int maxP, cudaStream_t st);
// keyframe hand-over (FullSystem::makeKeyFrame, FullSystem.cpp:1152-1171)
void launch_ba_marg_flag(const BAWinDev* wins, int W, int maxP, cudaStream_t st);           // flagPointsForRemoval numeric part; P.marg_status in: selected, out: status
void launch_ba_marg_points(const BAWinDev* wins, int W, int maxP, cudaStream_t st);         // marginalizePointsF
void launch_ba_marg_frame(const BAWinDev* wins, int W, const int* idx, cudaStream_t st);    // marginalizeFrame (frame idx[w] of window w; -1: none)
void launch_ba_decide(const BAWinDev* wins, int W, int stage, cudaStream_t st);              // 0 init, 1 after step+linearize, 2 after reload, 3 final rmse

// ---- batched window install (sdv_ba_install.cu): insertFrame / makeIDX / setPrecalcValues for n windows in fixed launches
constexpr size_t kHdrPrefix = offsetof(BAHeader, precalc);   // what the host sets in a header besides HM / bM; the rest starts at zero
struct BAHdrInstall { BAHeader* hdr; long long src; int hm_n, bm_n; };   // staging byte offset of the prefix, then hm_n + bm_n doubles of HM / bM
// header w := its staged prefix, HM[0..hm_n), bM[0..bm_n), zero elsewhere (the bytes a full-header copy of a zeroed host header leaves)
void launch_ba_hdr_install(const BAHdrInstall* d, int n, const char* stage, cudaStream_t st);
// rows of window w in the concatenated point / residual arrays of one call: points p0 .. p0+nP, residuals r0 .. r0+nR, res_begin at p0 + w
struct BAPtsInstall { int p0, r0, nP, nR, nF; };
struct BAPtsStage {                      // the call's rows on the device, concatenated in window order
  const float2* uv; const float* idepth; const float* idepth_zero; const float* color; const float* weights;
  const int* host; const int* hasDepthPrior; const int* isFromSensor; const int* res_begin;
  const int* r_point; const int* r_host; const int* r_target; const int* r_hasMatcher; const float2* r_matcher; const int* r_isNew;
  int* rot;                              // [8 per point] res_of_target, written by the check
  int* cnt;                              // [kPairCnt per window] residuals per (host + nF*target) at 0..63, points per host at 64..71
  unsigned* key_in; unsigned* key; int* val_in; int* pair_res;   // pair sort: key = window*64 + pair, value = residual (window-local)
};
constexpr int kPairCnt = kMaxF*kMaxF + kMaxF;
// refusal code of a window (low 4 bits of its err word; ~0 = none) and the point / residual it names (see ba_err_*)
enum { BA_ERR_SPAN = 1, BA_ERR_MONO = 2, BA_ERR_HOST = 3, BA_ERR_RES = 4, BA_ERR_DUP = 5 };
__host__ __device__ inline int ba_err_code(unsigned long long e) { return (int)(e & 15); }
__host__ __device__ inline int ba_err_point(unsigned long long e) { return (int)((e >> 34) & ((1u << 28) - 1)); }
__host__ __device__ inline int ba_err_res(unsigned long long e) { return (int)((e >> 4) & ((1u << 30) - 1)) - 1; }
constexpr int kMaxPtsWin = (1 << 28) - 1, kMaxResWin = (1 << 30) - 2;   // what the err word can name
// the makeIDX checks of every point (err[w]: the window's first failure), res_of_target and the per-pair / per-host counts; err and cnt start at ~0 / 0
void launch_ba_pts_check(const BAPtsInstall* D, int n, int totP, const BAPtsStage& S, unsigned long long* err, cudaStream_t st);
// after the check passed: the pair lists (stable sort, before any window is written), pair_begin / host_begin / header nP, nR, the rows into each
// window's pool.  Returns the launches, or -1 when the sort could not be enqueued (no window written then).
int  launch_ba_pts_install(const BAWinDev* wins, const BAPtsInstall* D, int n, int totR, int maxP, int maxR, const BAPtsStage& S, void* sort_tmp, size_t sort_bytes,
                           cudaStream_t st);
size_t ba_pts_sort_bytes(int n, int totR);
// P.marg_status of window w <-> buf[off[w] .. off[w+1])  (to_window: 1 copy in, 0 copy out)
void launch_ba_status_copy(const BAWinDev* wins, int n, int maxP, const int* off, int* buf, int to_window, cudaStream_t st);
// (HM, bM) of window w (dim = header dim) -> out + off[2w] / out + off[2w+1]
void launch_ba_prior_gather(const BAWinDev* wins, int n, const long long* off, double* out, cudaStream_t st);

} // namespace sdv
