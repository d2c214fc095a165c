// sdv_ba_kernels.cu — sm_90a (H100) kernels of the sliding-window back-end (compiled with --fmad=false).
//
//   ba_frames_kernel        FrameHessian::setState/setStateZero, EFFrame::takeData, EnergyFunctional::setAdjointsF/setDeltaF,
//                           FrameFramePrecalc::set           HessianBlocks.h:141-183, HessianBlocks.cpp:52-82,169-195, EnergyFunctional.cpp:21-71,131-156
//   ba_linearize_kernel     PointFrameResidual::linearize (+ applyRes when fixing)       Residuals.cpp:60-224, 252-274
//   ba_energy_th_kernel     FullSystem::setNewFrameEnergyTH (exact k-th element by radix select)   FullSystemOptimize.cpp:63-97
//   ba_point_acc_kernel     per-point part of AccumulatedTopHessianSSE::addPoint<0> + head of AccumulatedSCHessianSSE::addPoint
//   ba_acc_top_kernel       AccumulatorApprox buckets per (host,target)                  AccumulatedTopHessian.cpp:13-112, MatrixAccumulators.h:560-932
//   ba_acc_sc_kernel        accD/accE/accEB/accHcc/accbc                                  AccumulatedSCHessian.cpp:10-62
//   ba_solve_kernel         stitchDouble*, solveSystemF, orthogonalize, resubstituteF_MT head   AccumulatedTopHessian.cpp:181-242, AccumulatedSCHessian.cpp:64-135,
//                                                                                         EnergyFunctional.cpp:650-759, 615-648, 221-248
//   ba_resub_kernel         EnergyFunctional::resubstituteFPt                             EnergyFunctional.cpp:250-282
//   ba_step_* / ba_backup   FullSystem::doStepFromBackup / backupState / loadSateBackup   FullSystemOptimize.cpp:165-321
//
// Accumulation kernels are "entry-parallel, item-sequential": one thread owns one accumulator cell and walks the items in the
// reference's order with the reference's 1 / 1k / 1M float tiers, so every float sum is bit-identical to the CPU path's.
#include "sdv_ba.cuh"
#include "sdv_core_common.cuh"

namespace sdv {

#define BA_WIN(gate) const BAWinDev& Wn = wins[blockIdx.y]; BAHeader* __restrict__ H = Wn.hdr; \
  if (((gate) != 0) && ((H->flags & (gate)) != (gate))) return; BAPointsDev P = Wn.P; BAResDev R = Wn.R; const int nP = H->nP, nR = H->nR; (void)P; (void)R; (void)nP; (void)nR;

// ================================================================================================ frames / pairs
__device__ void frame_set_state(BAFrameDev& f) {                          // HessianBlocks.h:141-153
  for (int i=0;i<3;i++) f.state_scaled[i] = 0.5f*f.state[i];
  for (int i=3;i<6;i++) f.state_scaled[i] = 1.0f*f.state[i];
  f.state_scaled[6] = 10.0f*f.state[6]; f.state_scaled[7] = 1000.0f*f.state[7]; f.state_scaled[8] = 10.0f*f.state[8]; f.state_scaled[9] = 1000.0f*f.state[9];
  f.PRE_w2c = se3_mul(se3_exp(f.state_scaled), f.evalPT);
  f.PRE_c2w = se3_inv(f.PRE_w2c);
}
__device__ void frame_set_state_zero(BAFrameDev& f) {                     // HessianBlocks.cpp:52-82
  SE3d T = f.evalPT, Ti = se3_inv(T);
  for (int i=0;i<6;i++) {
    double e[6]={0,0,0,0,0,0}, m[6]={0,0,0,0,0,0}; e[i]=1e-3; m[i]=-1e-3;
    SE3d P = se3_mul(se3_mul(T, se3_exp(e)), Ti), M = se3_mul(se3_mul(T, se3_exp(m)), Ti);
    double lp[6], lm[6]; se3_log(P, lp); se3_log(M, lm);
    for (int r=0;r<6;r++) f.nullspaces_pose[r*6+i] = (lp[r]-lm[r])/(2e-3);
  }
  SE3d P = T; for (int i=0;i<3;i++) P.t[i] *= 1.00001; P = se3_mul(P, Ti);
  SE3d M = T; for (int i=0;i<3;i++) M.t[i] /= 1.00001; M = se3_mul(M, Ti);
  double lp[6], lm[6]; se3_log(P, lp); se3_log(M, lm);
  for (int r=0;r<6;r++) f.nullspaces_scale[r] = (lp[r]-lm[r])/(2e-3);
}

// flags: 1 setState, 2 setStateZero, 4 takeData(prior), 8 adjoints, 16 precalc+deltas, 32 re-anchor newest frame first,
//        64 = this is doStepFromBackup/loadSateBackup: first apply calib/frame steps (stepfac) or restore the backups
__global__ void __launch_bounds__(64) ba_frames_kernel(const BAWinDev* __restrict__ wins, int flags, float stepfac, int load_backup, int gate) {
  BA_WIN(gate)
  const int tid = threadIdx.x; const int nF = H->nF;
  if (flags & 64) {
    if (tid == 0) {
      BACalibDev& c = H->calib; double v[4];
      for (int i=0;i<4;i++) v[i] = load_backup ? c.value_backup[i] : c.value_backup[i] + stepfac*c.step[i];
      for (int i=0;i<4;i++) c.value[i] = v[i];                              // CalibHessian::setValue (HessianBlocks.h:305-320)
      c.value_scaled[0] = 50.0f*v[0]; c.value_scaled[1] = 50.0f*v[1]; c.value_scaled[2] = 50.0f*v[2]; c.value_scaled[3] = 50.0f*v[3];
      for (int i=0;i<4;i++) c.sf[i] = (float)c.value_scaled[i];
      c.si[0] = 1.0f/c.sf[0]; c.si[1] = 1.0f/c.sf[1]; c.si[2] = -c.sf[2]/c.sf[0]; c.si[3] = -c.sf[3]/c.sf[1];
      for (int i=0;i<4;i++) c.vmvz[i] = c.value[i] - c.value_zero[i];
      if (!load_backup) {                                                   // doStepFromBackup sums (FullSystemOptimize.cpp:173-249)
        float sumT = 0, sumR = 0;
        for (int f=0; f<nF; f++) { const double* s = H->frames[f].step;
          sumT += s[0]*s[0]+s[1]*s[1]+s[2]*s[2]; sumR += s[3]*s[3]+s[4]*s[4]+s[5]*s[5]; }
        sumR /= nF; sumT /= nF;
        float sumNID = H->sums[1] / H->sums[2];                             // sumNID /= numID   (sums[] filled by ba_step_points_kernel)
        H->canbreak = (sqrtf(sumR) < 0.00005*H->set.thOptIterations && sqrtf(sumT)*sumNID < 0.00005*H->set.thOptIterations) ? 1 : 0;
      }
    }
    if (tid < nF) { BAFrameDev& f = H->frames[tid];
      if (load_backup) { for (int i=0;i<10;i++) f.state[i] = f.state_backup[i]; }
      else { for (int i=6;i<10;i++) f.step[i] = 0; for (int i=0;i<10;i++) f.state[i] = f.state_backup[i] + (double)stepfac*f.step[i]; } }
    __syncthreads();
  }
  if ((flags & 32) && tid == nF-1) {                                        // optimize() tail: setEvalPT(PRE_worldToCam, [0..,a,b,0,0])  (FullSystemOptimize.cpp:460-464)
    BAFrameDev& f = H->frames[tid]; double a = f.state[6], b = f.state[7];
    f.evalPT = f.PRE_w2c;
    for (int i=0;i<10;i++) { f.state[i] = 0; f.state_zero[i] = 0; }
    f.state[6] = a; f.state[7] = b; f.state_zero[6] = a; f.state_zero[7] = b;
    frame_set_state(f); frame_set_state_zero(f);
  }
  if (tid < nF) {
    BAFrameDev& f = H->frames[tid];
    if (flags & 1) frame_set_state(f);
    if (flags & 2) frame_set_state_zero(f);
    if (flags & 4) {                                                        // EFFrame::takeData + getPrior (HessianBlocks.h:220-252)
      for (int i=0;i<6;i++) f.prior[i] = 0;
      if (f.frameID == 0) { for (int i=0;i<3;i++) f.prior[i] = H->set.initialTransPrior; for (int i=3;i<6;i++) f.prior[i] = H->set.initialRotPrior; }
    }
    for (int i=0;i<6;i++) { f.delta[i] = f.state[i] - f.state_zero[i]; f.delta_prior[i] = f.state[i]; }
  }
  if (tid == 0) { for (int i=0;i<4;i++) { H->calib.cDeltaF[i] = (float)H->calib.vmvz[i]; H->calib.cPrior[i] = H->set.initialCalibHessian; }
    if (flags & (2|32)) H->ortho_valid = 0; }
  __syncthreads();
  if (tid < nF*nF) {
    const int h = tid % nF, t = tid / nF; const int idx = h + t*nF;
    const BAFrameDev& host = H->frames[h]; const BAFrameDev& target = H->frames[t];
    if (flags & 8) {                                                        // setAdjointsF (EnergyFunctional.cpp:30-52,61-66)
      SE3d hostToTarget = se3_mul(target.evalPT, se3_inv(host.evalPT));
      double Ad[36]; se3_adj(hostToTarget, Ad);
      double* AH = H->adHost + idx*36; double* AT = H->adTarget + idx*36;
      for (int r=0;r<6;r++) for (int c=0;c<6;c++) { AH[r*6+c] = -Ad[c*6+r]; AT[r*6+c] = (r==c) ? 1.0 : 0.0; }
      for (int r=0;r<3;r++) for (int c=0;c<6;c++) { AH[r*6+c] *= 0.5f; AT[r*6+c] *= 0.5f; }
      for (int r=3;r<6;r++) for (int c=0;c<6;c++) { AH[r*6+c] *= 1.0f; AT[r*6+c] *= 1.0f; }
      for (int i=0;i<36;i++) { H->adHostF[idx*36+i] = (float)AH[i]; H->adTargetF[idx*36+i] = (float)AT[i]; }
    }
    if (flags & 16) {                                                       // FrameFramePrecalc::set (HessianBlocks.cpp:169-195)
      PrecalcDev& p = H->precalc[h*nF + t];
      const BACalibDev& c = H->calib;
      float K[9] = {c.sf[0],0,c.sf[2], 0,c.sf[1],c.sf[3], 0,0,1}, Ki[9]; inv3f(K, Ki);
      SE3d l0 = se3_mul(target.evalPT, se3_inv(host.evalPT));
      double R0[9]; qmat(l0.q, R0); for (int i=0;i<9;i++) p.R0[i] = (float)R0[i]; for (int i=0;i<3;i++) p.t0[i] = (float)l0.t[i];
      SE3d l = se3_mul(target.PRE_w2c, host.PRE_c2w);
      double Rd[9]; qmat(l.q, Rd); float R[9], tl[3], KR[9]; for (int i=0;i<9;i++) R[i] = (float)Rd[i]; for (int i=0;i<3;i++) tl[i] = (float)l.t[i];
      for (int i=0;i<3;i++) for (int j=0;j<3;j++) KR[i*3+j] = (K[i*3]*R[j] + K[i*3+1]*R[3+j]) + K[i*3+2]*R[6+j];
      for (int i=0;i<3;i++) for (int j=0;j<3;j++) p.KRKi[i*3+j] = (KR[i*3]*Ki[j] + KR[i*3+1]*Ki[3+j]) + KR[i*3+2]*Ki[6+j];
      for (int i=0;i<3;i++) p.Kt[i] = (K[i*3]*tl[0] + K[i*3+1]*tl[1]) + K[i*3+2]*tl[2];
      double aff[2]; aff_from_to(host.ab_exposure, target.ab_exposure, host.state_scaled[6], host.state_scaled[7], target.state_scaled[6], target.state_scaled[7], aff);
      p.aff[0] = (float)aff[0]; p.aff[1] = (float)aff[1];
      p.b0 = (float)(host.state_zero[7]*1000.0f);
      // setDeltaF (EnergyFunctional.cpp:135-142)
      float dh[6], dt[6];
      for (int i=0;i<6;i++) { dh[i] = (float)(host.state[i]-host.state_zero[i]); dt[i] = (float)(target.state[i]-target.state_zero[i]); }
      for (int j=0;j<6;j++) { float s1 = 0, s2 = 0;
        for (int i=0;i<6;i++) { s1 += dh[i]*H->adHostF[idx*36+i*6+j]; s2 += dt[i]*H->adTargetF[idx*36+i*6+j]; }
        H->adHTdeltaF[idx*6+j] = s1 + s2; }
    }
  }
}

__global__ void ba_points_setup_kernel(const BAWinDev* __restrict__ wins, int take_data) {
  BA_WIN(0)
  int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= nP) return;
  if (take_data) P.priorF[i] = P.hasDepthPrior[i] ? H->set.idepthFixPrior*1.0f*1.0f : 0.0f;       // EFPoint::takeData (EnergyFunctionalStructs.cpp:40-46)
  P.deltaF[i] = P.idepth[i] - P.idepth_zero[i];
}

__global__ void ba_reset_oob_kernel(const BAWinDev* __restrict__ wins) {      // PointFrameResidual::resetOOB (Residuals.h:66-73)
  BA_WIN(0)
  int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= nR) return;
  R.state_NewEnergy[i] = 0; R.state_energy[i] = 0; R.state_NewState[i] = RS_OUTLIER; R.state_state[i] = RS_IN;
}

// ================================================================================================ linearize
__device__ __forceinline__ void apply_res(BAResDev& R, int r) {            // Residuals.cpp:252-274 (copyJacobians = true) + takeDataF
  if (R.state_state[r] == RS_OOB) return;
  if (R.state_NewState[r] == RS_IN) {
    R.isActive[r] = 1;
    float J[24];
#pragma unroll
    for (int k=0;k<24;k++) { J[k] = R.J[(size_t)r*24+k]; R.efJ[(size_t)r*24+k] = J[k]; }
#pragma unroll
    for (int i=0;i<6;i++) R.JpJdF[(size_t)r*8+i] = J[2+i]*J[22] + J[8+i]*J[23];
    R.JpJdF[(size_t)r*8+6] = 0; R.JpJdF[(size_t)r*8+7] = 0;
  } else R.isActive[r] = 0;
  R.state_state[r] = R.state_NewState[r]; R.state_energy[r] = R.state_NewEnergy[r];
}

// PointFrameResidual::linearize (Residuals.cpp:60-224) for residual r; returns the energy the caller sums (state_energy for OOB residuals).
// thbuf != nullptr: also collect the setNewFrameEnergyTH candidates (linearizeAll_Reductor, FullSystemOptimize.cpp:23-29).
__device__ __forceinline__ double lin_residual(BAHeader* __restrict__ H, BAPointsDev& P, BAResDev& R, int r, float* __restrict__ thbuf, int* __restrict__ thcount) {
  double energy = 0;
  R.state_NewEnergyWithOutlier[r] = -1;
  bool done = false;
  if (R.state_state[r] == RS_OOB) { R.state_NewState[r] = RS_OOB; energy = R.state_energy[r]; done = true; }
  const int nF = H->nF; const int hI = R.host[r], tI = R.target[r], pI = R.point[r];
  const PrecalcDev& pc = H->precalc[hI*nF + tI];
  const float wM3G = (float)(H->w - 3), hM3G = (float)(H->h - 3);
  const float fxl = H->calib.sf[0], fyl = H->calib.sf[1], cxl = H->calib.sf[2], cyl = H->calib.sf[3], fxli = H->calib.si[0], fyli = H->calib.si[1];
  float J[24]; float Ku = 0, Kv = 0;
  if (!done && !R.hasMatcher[r]) { R.state_NewState[r] = RS_OOB; energy = R.state_energy[r]; done = true; }
  const float2 uv = P.uv[pI];
  if (!done) {
    const float idz = P.idepth_zero[pI]*1.0f;                                     // idepth_zero_scaled
    float KliP0 = (uv.x+0-cxl)*fxli, KliP1 = (uv.y+0-cyl)*fyli, KliP2 = 1;
    float p0 = ((pc.R0[0]*KliP0 + pc.R0[1]*KliP1) + pc.R0[2]*KliP2) + pc.t0[0]*idz;
    float p1 = ((pc.R0[3]*KliP0 + pc.R0[4]*KliP1) + pc.R0[5]*KliP2) + pc.t0[1]*idz;
    float p2 = ((pc.R0[6]*KliP0 + pc.R0[7]*KliP1) + pc.R0[8]*KliP2) + pc.t0[2]*idz;
    float drescale = 1.0f/p2; float new_idepth = idz*drescale;
    float u = p0*drescale, v = p1*drescale;
    Ku = u*fxl + cxl; Kv = v*fyl + cyl;
    if (!(drescale > 0) || !(Ku > 1.1f && Kv > 1.1f && Ku < wM3G && Kv < hM3G)) { R.state_NewState[r] = RS_OOB; energy = R.state_energy[r]; done = true; }
    else {
      R.center[(size_t)r*3] = Ku; R.center[(size_t)r*3+1] = Kv; R.center[(size_t)r*3+2] = new_idepth;
      float d_d_x = drescale * (pc.t0[0]-pc.t0[2]*u)*1.0f*fxl;
      float d_d_y = drescale * (pc.t0[1]-pc.t0[2]*v)*1.0f*fyl;
      float cx2 = drescale*(pc.R0[6]*u-pc.R0[0]);
      float cx3 = fxl * drescale*(pc.R0[7]*u-pc.R0[1]) * fyli;
      float cx0 = KliP0*cx2, cx1 = KliP1*cx3;
      float cy2 = fyl * drescale*(pc.R0[6]*v-pc.R0[3]) * fxli;
      float cy3 = drescale*(pc.R0[7]*v-pc.R0[4]);
      float cy0 = KliP0*cy2, cy1 = KliP1*cy3;
      cx0 = (cx0+u)*50.0f; cx1 *= 50.0f; cx2 = (cx2+1)*50.0f; cx3 *= 50.0f;
      cy0 *= 50.0f; cy1 = (cy1+v)*50.0f; cy2 *= 50.0f; cy3 = (cy3+1)*50.0f;
      J[2] = new_idepth*fxl; J[3] = 0; J[4] = -new_idepth*u*fxl; J[5] = -u*v*fxl; J[6] = (1+u*u)*fxl; J[7] = -v*fxl;
      J[8] = 0; J[9] = new_idepth*fyl; J[10] = -new_idepth*v*fyl; J[11] = -(1+v*v)*fyl; J[12] = u*v*fyl; J[13] = u*fyl;
      J[14] = cx0; J[15] = cx1; J[16] = cx2; J[17] = cx3; J[18] = cy0; J[19] = cy1; J[20] = cy2; J[21] = cy3;
      J[22] = d_d_x; J[23] = d_d_y;
    }
  }
  if (!done) {
    // photometric 8-pattern outlier gate at the CURRENT pose (Residuals.cpp:157-194)
    const float4* __restrict__ img = H->frames[tI].img0; const int wI = H->w;
    const float ids = P.idepth[pI]*1.0f; const float a0 = pc.aff[0], a1 = pc.aff[1];
    float wJI2_sum = 0, energyLeft2 = 0.0f;
    // (Tried in round 2: all 8 projections first, then the footprints of 4 pixels fetched together — 16 independent loads in flight per thread — and accumulated in
    // order.  Bit-identical, but 184 registers instead of 96 cut the resident warps by more than the extra memory parallelism gave: slower.)
    for (int idx = 0; idx < 8; idx++) {
      float x = uv.x + staticPattern[idx][0], y = uv.y + staticPattern[idx][1];
      float q0 = ((pc.KRKi[0]*x + pc.KRKi[1]*y) + pc.KRKi[2]*1.0f) + pc.Kt[0]*ids;
      float q1 = ((pc.KRKi[3]*x + pc.KRKi[4]*y) + pc.KRKi[5]*1.0f) + pc.Kt[1]*ids;
      float q2 = ((pc.KRKi[6]*x + pc.KRKi[7]*y) + pc.KRKi[8]*1.0f) + pc.Kt[2]*ids;
      float Ku2 = q0/q2, Kv2 = q1/q2;
      if (!(Ku2 > 1.1f && Kv2 > 1.1f && Ku2 < wM3G && Kv2 < hM3G)) break;
      int ix = (int)Ku2, iy = (int)Kv2; float dx = Ku2-ix, dy = Kv2-iy, dxdy = dx*dy;
      const float4* bp = img + ix + iy*wI;
      float4 p00 = __ldg(bp), p10 = __ldg(bp+1), p01 = __ldg(bp+wI), p11 = __ldg(bp+1+wI);
      float w11 = dxdy, w01 = dy-dxdy, w10 = dx-dxdy, w00 = 1-dx-dy+dxdy;
      float h0 = ((w11*p11.x + w01*p01.x) + w10*p10.x) + w00*p00.x;
      float h1 = ((w11*p11.y + w01*p01.y) + w10*p10.y) + w00*p00.y;
      float h2 = ((w11*p11.z + w01*p01.z) + w10*p10.z) + w00*p00.z;
      float residual = h0 - (a0*P.color[(size_t)pI*8+idx] + a1);
      if (!isfinite(h0)) break;
      float wgt = sqrtf(H->set.outlierTHSumComponent / (H->set.outlierTHSumComponent + (h1*h1 + h2*h2)));
      wgt = 0.5f*(wgt + P.weights[(size_t)pI*8+idx]);
      float hw = fabsf(residual) < H->set.huberTH ? 1 : H->set.huberTH / fabsf(residual);
      energyLeft2 += wgt*wgt*hw*residual*residual*(2-hw);
      if (hw < 1) hw = sqrtf(hw);
      hw = hw*wgt; h1 *= hw; h2 *= hw;
      wJI2_sum += hw*hw*(h1*h1 + h2*h2);
    }
    const float2 m = R.matcher[r];
    float res0 = Ku - m.x, res1 = Kv - m.y;
    float nrm = sqrtf(res0*res0 + res1*res1);
    float hw = fabsf(nrm) < H->set.huberTH ? 1 : H->set.huberTH / fabsf(nrm);
    float energyLeft = hw * (res0*res0 + res1*res1)*(2-hw);
    if (hw < 1) hw = sqrtf(hw);
    J[0] = res0*hw; J[1] = res1*hw;
#pragma unroll
    for (int k=2;k<24;k++) J[k] = J[k]*hw;
#pragma unroll
    for (int k=0;k<24;k++) R.J[(size_t)r*24+k] = J[k];
    R.state_NewEnergyWithOutlier[r] = energyLeft2;
    float th = fmaxf(H->frames[hI].frameEnergyTH, H->frames[tI].frameEnergyTH);
    if (energyLeft2 > th || wJI2_sum < 2) { R.state_NewEnergy[r] = th; R.state_NewState[r] = RS_OUTLIER; }
    else { R.state_NewEnergy[r] = energyLeft2; R.state_NewState[r] = RS_IN; }
    energy = energyLeft;
    if (thbuf && tI == nF-1) { int slot = atomicAdd(thcount, 1); thbuf[slot] = energyLeft2; }       // setNewFrameEnergyTH candidates (order-free)
  }
  return energy;
}

constexpr int kLinThreads = 128;
__global__ void __launch_bounds__(kLinThreads) ba_linearize_kernel(const BAWinDev* __restrict__ wins, int fix, int gate) {
  BA_WIN(gate)
  const int nblocks = (nR + kLinThreads - 1)/kLinThreads < 1 ? 1 : (nR + kLinThreads - 1)/kLinThreads;
  if ((int)blockIdx.x >= nblocks) return;                                   // grid.x is sized for the largest window of the batch
  double* __restrict__ partials = Wn.partials; float* __restrict__ thbuf = Wn.thbuf; int* __restrict__ thcount = Wn.thcount;
  const int r = blockIdx.x*kLinThreads + threadIdx.x;
  double energy = 0;
  if (r < nR) {
    energy = lin_residual(H, P, R, r, thbuf, thcount);
    const int nF = H->nF; const int hI = R.host[r], tI = R.target[r], pI = R.point[r];
    const PrecalcDev& pc = H->precalc[hI*nF + tI]; const float2 uv = P.uv[pI]; (void)tI;
    if (fix) {                                                              // linearizeAll_Reductor, fixLinearization branch (FullSystemOptimize.cpp:30-53)
      apply_res(R, r);
      if (R.isActive[r]) {
        if (R.isNew[r]) {
          const float ids = P.idepth[pI]*1.0f;
          float i0 = (pc.KRKi[0]*uv.x + pc.KRKi[1]*uv.y) + pc.KRKi[2]*1.0f, i1 = (pc.KRKi[3]*uv.x + pc.KRKi[4]*uv.y) + pc.KRKi[5]*1.0f, i2 = (pc.KRKi[6]*uv.x + pc.KRKi[7]*uv.y) + pc.KRKi[8]*1.0f;
          float q0 = i0 + pc.Kt[0]*ids, q1 = i1 + pc.Kt[1]*ids, q2 = i2 + pc.Kt[2]*ids;
          float ddx = i0/i2 - q0/q2, ddy = i1/i2 - q1/q2;
          float relBS = (float)(0.01*(double)sqrtf(ddx*ddx + ddy*ddy));
          atomicMax(reinterpret_cast<int*>(P.maxRelBaseline + pI), __float_as_int(relBS));   // non-negative floats: int order == float order
          atomicAdd(P.numGoodResiduals + pI, 1);
        }
      } else R.toRemove[r] = 1;
    }
  }
  // deterministic energy reduction (double): warp butterfly -> block -> last block sums the block partials in order
  __shared__ double wsum[kLinThreads/32]; __shared__ bool is_last;
  for (int o=16;o>0;o>>=1) energy += __shfl_xor_sync(0xffffffffu, energy, o);
  if ((threadIdx.x & 31) == 0) wsum[threadIdx.x>>5] = energy;
  __syncthreads();
  if (threadIdx.x == 0) {
    double s = 0; for (int k=0;k<kLinThreads/32;k++) s += wsum[k];
    partials[blockIdx.x] = s; __threadfence();
    unsigned int t = atomicAdd(&H->ticket, 1u); is_last = (t == (unsigned int)nblocks-1);
    if (is_last) { __threadfence(); double tot = 0; for (int b=0;b<nblocks;b++) tot += __ldcg(partials+b); H->energyP = tot; H->ticket = 0; }
  }
}

// exact k-th smallest (std::nth_element value) of n non-negative floats by 4x8-bit radix select, then the threshold formula
__global__ void __launch_bounds__(1024) ba_energy_th_kernel(const BAWinDev* __restrict__ wins, int gate) {
  BA_WIN(gate)
  const float* __restrict__ buf = Wn.thbuf; int* __restrict__ count = Wn.thcount;
  __shared__ unsigned int hist[256]; __shared__ unsigned int prefix, kk, sel_mask;
  const int n = *count; BAFrameDev& nf = H->frames[H->nF-1];
  if (n == 0) { if (threadIdx.x == 0) { nf.frameEnergyTH = 12*12*8; *count = 0; } return; }
  if (threadIdx.x == 0) { prefix = 0; sel_mask = 0; kk = (unsigned int)(int)(H->set.frameEnergyTHN * n); }
  __syncthreads();
  for (int shift = 24; shift >= 0; shift -= 8) {
    for (int i = threadIdx.x; i < 256; i += blockDim.x) hist[i] = 0;
    __syncthreads();
    const unsigned int pf = prefix, mk = sel_mask;
    for (int i = threadIdx.x; i < n; i += blockDim.x) { unsigned int key = __float_as_uint(buf[i]); if ((key & mk) == pf) atomicAdd(&hist[(key >> shift) & 255u], 1u); }
    __syncthreads();
    if (threadIdx.x == 0) { unsigned int k = kk, b = 0; for (; b < 256; b++) { if (k < hist[b]) break; k -= hist[b]; }
      kk = k; prefix = pf | (b << shift); sel_mask = mk | (255u << shift); }
    __syncthreads();
  }
  if (threadIdx.x == 0) {
    float nthElement = sqrtf(__uint_as_float(prefix));                       // FullSystemOptimize.cpp:91-96
    float th = nthElement*H->set.frameEnergyTHFacMedian;
    th = 26.0f*H->set.frameEnergyTHConstWeight + th*(1-H->set.frameEnergyTHConstWeight);
    th = th*th; th *= H->set.overallEnergyTHWeight*H->set.overallEnergyTHWeight;
    nf.frameEnergyTH = th; *count = 0;
  }
}

__global__ void ba_apply_kernel(const BAWinDev* __restrict__ wins, int gate) { BA_WIN(gate) int r = blockIdx.x*blockDim.x + threadIdx.x; if (r < nR) apply_res(R, r); }

// ================================================================================================ energies
__global__ void __launch_bounds__(256) ba_energies_kernel(const BAWinDev* __restrict__ wins, int gate) {
  BA_WIN(gate)
  __shared__ double sh[256];
  const int tid = threadIdx.x; const int nF = H->nF, N = H->dim;
  // calcLEnergyPt: chunks of 50 points, float Accumulator11 per chunk (EnergyFunctional.cpp:295-331)
  double mine = 0; const int nchunks = (nP + 49)/50;
  for (int c = tid; c < nchunks; c += 256) { float acc = 0; for (int i = c*50; i < min(c*50+50, nP); i++) acc += P.deltaF[i]*P.deltaF[i]*P.priorF[i]; mine += (double)((acc + 0.0f) + 0.0f); }
  sh[tid] = mine; __syncthreads();
  for (int o = 128; o > 0; o >>= 1) { if (tid < o) sh[tid] += sh[tid+o]; __syncthreads(); }
  if (tid == 0) {
    double E = 0;
    for (int f=0; f<nF; f++) for (int i=0;i<6;i++) E += (H->frames[f].delta_prior[i]*H->frames[f].prior[i])*H->frames[f].delta_prior[i];
    float s = 0; for (int i=0;i<4;i++) s += (H->calib.cDeltaF[i]*(float)H->calib.cPrior[i])*H->calib.cDeltaF[i];
    H->energyL = (E + s) + sh[0];
  }
  __syncthreads();
  // calcMEnergyF: delta . (2 bM + HM delta)   (:284-293)
  double d_i = 0, row = 0;
  if (tid < N) {
    for (int j=0;j<N;j++) { double dj = (j < 4) ? (double)H->calib.cDeltaF[j] : H->frames[(j-4)/6].delta[(j-4)%6]; row += H->HM[tid*N+j]*dj; }
    d_i = (tid < 4) ? (double)H->calib.cDeltaF[tid] : H->frames[(tid-4)/6].delta[(tid-4)%6];
    sh[tid] = d_i*(2*H->bM[tid] + row);
  }
  __syncthreads();
  if (tid == 0) { double e = 0; for (int i=0;i<N;i++) e += sh[i]; H->energyM = e; }
}

// ================================================================================================ accumulation
// per point: Hdd/bd/Hcd sums over its active residuals in order (addPoint<0>), then HdiF / bdSumF (SC addPoint head)
// mode 0: addPoint<0> + addPoint(p, shiftPriorToZero=true) over all points (solveSystemF).
// mode 2: addPoint<2> + addPoint(p, false) over the PS_MARGINALIZE points (marginalizePointsF, EnergyFunctional.cpp:527,543-547): resApprox =
//         res_toZeroF, priorF *= setting_idepthFixPriorMargFac, no prior shift; the "L" sums are stored in the A slots (only A+L is ever read).
__global__ void ba_point_acc_kernel(const BAWinDev* __restrict__ wins, int gate, int mode) {
  BA_WIN(gate)
  int p = blockIdx.x*blockDim.x + threadIdx.x; if (p >= nP) return;
  if (mode == 2) { if (P.marg_status[p] != 2) { P.ngood[p] = 0; return; } P.priorF[p] *= 600.0f*600.0f; }
  float bd = 0, Hdd = 0, Hcd[4] = {0,0,0,0}; int ngood = 0;
  for (int r = P.res_begin[p]; r < P.res_begin[p+1]; r++) {
    if (!R.isActive[r]) continue;
    const float* J = R.efJ + (size_t)r*24; ngood++;
    const float2 rz = (mode == 2) ? R.res_toZero[r] : make_float2(J[0], J[1]);
    bd += rz.x*J[22] + rz.y*J[23];
    Hdd += J[22]*J[22] + J[23]*J[23];
    for (int i=0;i<4;i++) Hcd[i] += J[14+i]*J[22] + J[18+i]*J[23];
  }
  P.Hdd_accAF[p] = Hdd; P.bd_accAF[p] = bd; for (int i=0;i<4;i++) P.Hcd_accAF[(size_t)p*4+i] = Hcd[i];
  P.ngood[p] = ngood;
  if (ngood == 0) { P.HdiF[p] = 0; P.bdSumF[p] = 0; P.idepth_hessian[p] = 0; P.maxRelBaseline[p] = 0; return; }   // AccumulatedSCHessian.cpp:12-21
  float Hh = Hdd + 0.0f + P.priorF[p]; if (Hh < 1e-10) Hh = 1e-10;
  P.idepth_hessian[p] = Hh; P.HdiF[p] = (float)(1.0 / (double)Hh);
  float bs = bd + 0.0f; if (mode != 2) bs += P.priorF[p]*P.deltaF[p]; P.bdSumF[p] = bs;
}

struct Tier { float d, d1k, d1m, n1, n1k; };
__device__ __forceinline__ void tier_shift(Tier& t) {                       // shiftUp(false) after numIn1++ (MatrixAccumulators.h:897-931)
  if (t.n1 > 1000) { t.d1k = t.d + t.d1k; t.n1k += t.n1; t.n1 = 0; t.d = 0; }
  if (t.n1k > 1000) { t.d1m = t.d1k + t.d1m; t.n1k = 0; t.d1k = 0; }
}
__device__ __forceinline__ float tier_finish(Tier& t) { t.d1k = t.d + t.d1k; t.d1m = t.d1k + t.d1m; return t.d1m; }

// one CTA per (host,target) bucket; thread e < 66 owns one cell of AccumulatorApprox and walks the pair's residuals in order
constexpr int kTopChunk = 96;                 // residuals staged per pass (one per thread for the activity flags); fewer latency-bound gather stages per bucket
__global__ void __launch_bounds__(96) ba_acc_top_kernel(const BAWinDev* __restrict__ wins, int gate, int mode) {
  BA_WIN(gate)
  if ((int)blockIdx.x >= H->nF*H->nF) return;
  const int pair = blockIdx.x; const int e = threadIdx.x;
  __shared__ float sJ[kTopChunk][24]; __shared__ int sAct[kTopChunk];
  int ei = 0, ej = 0;                                                        // cell (j row, i col) of the 10x10 upper triangle, Data[] order
  if (e < 55) { int k = e; int j = 0; while (k >= 10 - j) { k -= 10 - j; j++; } ej = j; ei = j + k; }
  else if (e < 65) { ei = e - 55; }
  Tier t = {0,0,0,0,0}; int num = 0;
  const int b0 = R.pair_begin[pair], b1 = R.pair_begin[pair+1];
  for (int base = b0; base < b1; base += kTopChunk) {
    const int cnt = min(kTopChunk, b1 - base);
    __syncthreads();
    for (int k = threadIdx.x; k < cnt*24; k += 96) { int q = k/24, c = k - q*24; int r = R.pair_res[base+q];
      float v = R.efJ[(size_t)r*24+c]; if (mode == 2 && c < 2) { const float2 rz = R.res_toZero[r]; v = c ? rz.y : rz.x; } sJ[q][c] = v; }
    if (threadIdx.x < cnt) { int r = R.pair_res[base+threadIdx.x]; int a = R.isActive[r]; if (mode == 2 && P.marg_status[R.point[r]] != 2) a = 0; sAct[threadIdx.x] = a; }
    __syncthreads();
    if (e < kNTop) {
      for (int q = 0; q < cnt; q++) {
        if (!sAct[q]) continue;
        const float* J = sJ[q]; num++;
        // x = [Jpdc[0](4) ; Jpdxi[0](6)], y = [Jpdc[1] ; Jpdxi[1]]
        if (e < 55) {
          float xi = (ei < 4) ? J[14+ei] : J[2+ei-4], xj = (ej < 4) ? J[14+ej] : J[2+ej-4];
          float yi = (ei < 4) ? J[18+ei] : J[8+ei-4], yj = (ej < 4) ? J[18+ej] : J[8+ej-4];
          t.d += 1.0f*xi*xj + 1.0f*yi*yj + 0.0f*(xi*yj + yi*xj);            // update(x4,x6,y4,y6, a=1,b=0,c=1)
          t.n1 += 1; tier_shift(t);
        } else {
          t.n1 += 1; tier_shift(t);                                          // the tier shift happens inside update(), before TopRight/BotRight are touched
          if (e < 65) { float xi = (ei < 4) ? J[14+ei] : J[2+ei-4], yi = (ei < 4) ? J[18+ei] : J[8+ei-4]; t.d += xi*J[0] + yi*J[1]; }
          else t.d += J[0]*J[0] + J[1]*J[1];
        }
      }
    }
  }
  if (e < kNTop) H->accTop[pair*kNTop + e] = tier_finish(t);
  if (e == 0) H->accTopNum[pair] = num;
}

// one CTA per host frame: thread (t1,t2) owns the whole 6x6 accD[(h,t1,t2)] bucket in registers, thread nF^2+t1 owns accE[(h,t1)] (6x4)
// and accEB[(h,t1)] (6).  The host's points are staged through shared memory 32 at a time (activity mask over targets, JpJdF per
// target, HdiF, bdSumF, Hcd) and walked in order; a bucket is touched only by the points whose residuals towards t1 and t2 are active,
// i.e. exactly the (r1,r2) loops of AccumulatedSCHessian.cpp:46-61.  Float sums, their order and the 1k/1M tiers match the CPU path.
constexpr int kScChunk = 64;
__global__ void __launch_bounds__(96) ba_acc_sc_kernel(const BAWinDev* __restrict__ wins, int gate) {
  BA_WIN(gate)
  const int nF = H->nF; const int nF2 = nF*nF; const int h = blockIdx.x;
  if (blockIdx.x == kMaxF) {                                                  // extra CTA: accHcc (4x4) and accbc (4) over ALL points of the window, in point order.
    // Points are staged through shared memory 256 at a time; threads 0..19 own one cell each and walk the staged chunk (a walk over global memory was the
    // critical path of the whole kernel: 1687 dependent L2 round trips per cell).
    constexpr int kHcChunk = 256;
    __shared__ float hHdi[kHcChunk], hBd[kHcChunk], hHcd[kHcChunk][4]; __shared__ int hOk[kHcChunk];
    const int e2 = threadIdx.x; Tier tt = {0,0,0,0,0};
    for (int base = 0; base < nP; base += kHcChunk) {
      const int cnt = min(kHcChunk, nP - base);
      __syncthreads();
      for (int q = threadIdx.x; q < cnt; q += 96) { const int p = base + q; const int ok = !(P.ngood[p] == 0 || P.isFromSensor[p]); hOk[q] = ok;
        hHdi[q] = P.HdiF[p]; hBd[q] = P.bdSumF[p]; for (int c = 0; c < 4; c++) hHcd[q][c] = P.Hcd_accAF[(size_t)p*4 + c] + 0.0f; }
      __syncthreads();
      if (e2 < 20) for (int q = 0; q < cnt; q++) { if (!hOk[q]) continue;
        const float Hdi = hHdi[q];
        if (e2 < 16) tt.d += (Hdi*hHcd[q][e2/4])*hHcd[q][e2%4];
        else tt.d += (hBd[q]*Hdi)*hHcd[q][e2-16];
        tt.n1 += 1; tier_shift(tt); }
    }
    if (e2 < 20) { const float v = tier_finish(tt); if (e2 < 16) H->accHcc[e2] = v; else H->accbc[e2-16] = v; }
    return;
  }
  if (h >= nF) return;
  const int p0 = R.host_begin[h], p1 = R.host_begin[h+1];
  const int e = threadIdx.x;
  const int role = (e < nF2) ? 0 : ((e < nF2 + nF) ? 1 : 2);
  const int t1 = (role == 0) ? e / nF : ((role == 1) ? e - nF2 : 0), t2 = (role == 0) ? e % nF : 0;
  __shared__ float sJ[kScChunk][kMaxF][6]; __shared__ int sMask[kScChunk]; __shared__ float sHdi[kScChunk], sBd[kScChunk], sHcd[kScChunk][4];
  float d[36], d1k[36], d1m[36]; float n1 = 0, n1k = 0; int num = 0;
#pragma unroll
  for (int k = 0; k < 36; k++) { d[k] = 0; d1k[k] = 0; d1m[k] = 0; }
  for (int base = p0; base < p1; base += kScChunk) {
    const int cnt = min(kScChunk, p1 - base);
    __syncthreads();
    if (e < cnt) sMask[e] = 0;
    __syncthreads();
    for (int k = e; k < cnt*nF; k += 96) { int q = k / nF, tt = k - q*nF; int p = base + q;
      int r = P.res_of_target[(size_t)p*kMaxF + tt]; int act = (r >= 0) ? R.isActive[r] : 0;
      if (act) { atomicOr(&sMask[q], 1 << tt); for (int c=0;c<6;c++) sJ[q][tt][c] = R.JpJdF[(size_t)r*8+c]; } }
    if (e < cnt) { int p = base + e; sHdi[e] = P.HdiF[p]; sBd[e] = P.bdSumF[p];
      for (int c=0;c<4;c++) sHcd[e][c] = P.Hcd_accAF[(size_t)p*4+c] + 0.0f; }
    __syncthreads();
    if (e < cnt) { int p = base + e; if (P.ngood[p] == 0 || P.isFromSensor[p]) sMask[e] = 0; }   // such points never reach the accumulators
    __syncthreads();
    for (int q = 0; q < cnt; q++) {
      const int mask = sMask[q]; if (mask == 0) continue;
      bool upd = false;
      if (role == 0) {
        if (((mask >> t1) & 1) && ((mask >> t2) & 1)) { upd = true;
          const float Hdi = sHdi[q];
#pragma unroll
          for (int i = 0; i < 6; i++) { const float wl = Hdi*sJ[q][t1][i];
#pragma unroll
            for (int j = 0; j < 6; j++) d[i*6+j] += wl*sJ[q][t2][j]; }            // accD.update(r1->JpJdF, r2->JpJdF, HdiF): A += (w*L)*R^T
        }
      } else if (role == 1) {
        if ((mask >> t1) & 1) { upd = true;
          const float Hdi = sHdi[q]; const float w2 = Hdi*sBd[q];
#pragma unroll
          for (int i = 0; i < 6; i++) { const float wl = Hdi*sJ[q][t1][i];
#pragma unroll
            for (int c = 0; c < 4; c++) d[i*4+c] += wl*sHcd[q][c];                // accE.update(r1->JpJdF, Hcd, HdiF)
            d[24+i] += w2*sJ[q][t1][i]; }                                         // accEB.update(r1->JpJdF, HdiF*bdSumF)
        }
      }
      if (upd) { num++; n1 += 1;
        if (n1 > 1000) {                                                          // tier shift (MatrixAccumulators.h:49-65)
#pragma unroll
          for (int k = 0; k < 36; k++) { d1k[k] += d[k]; d[k] = 0; }
          n1k += n1; n1 = 0;
          if (n1k > 1000) {
#pragma unroll
            for (int k = 0; k < 36; k++) { d1m[k] += d1k[k]; d1k[k] = 0; }
            n1k = 0; } } }
    }
  }
  // finish(): shiftUp(true)  ->  A1k += A ; A1m += A1k
  if (role == 0) { const int b = h + nF*t1 + nF2*t2;
#pragma unroll
    for (int k = 0; k < 36; k++) { float v1k = d1k[k] + d[k]; H->accD[b*36 + k] = d1m[k] + v1k; }
    H->accDNum[b] = num; }
  else if (role == 1) {
#pragma unroll
    for (int k = 0; k < 24; k++) { float v1k = d1k[k] + d[k]; H->accE[(h + nF*t1)*24 + k] = d1m[k] + v1k; }
#pragma unroll
    for (int k = 0; k < 6; k++) { float v1k = d1k[24+k] + d[24+k]; H->accEB[(h + nF*t1)*6 + k] = d1m[24+k] + v1k; } }
}

// ================================================================================================ stitch + solve (single CTA per window)
// Stitching is GATHER-style: one thread owns one element of the output system and walks the contributing (host,target) buckets in
// the reference's order (AccumulatedTopHessian.cpp:181-242, AccumulatedSCHessian.cpp:64-135), so every fp64 sum has the reference's
// order without a barrier per bucket.  The two system matrices live in shared memory.
__device__ __forceinline__ double tri10(const float* a, int r, int c) { int lo = min(r,c), hi = max(r,c); return (double)a[lo*10 - lo*(lo-1)/2 + (hi-lo)]; }
// element (i,j) of A1 * M * A2^T with M(p,q) supplied by a functor; evaluated as (A1*M) then * A2^T, inner indices ascending
template <typename MF> __device__ __forceinline__ double triple66(const double* A1, const double* A2, int i, int j, MF M) {
  double s = 0;
#pragma unroll
  for (int q = 0; q < 6; q++) { double t = 0;
#pragma unroll
    for (int p = 0; p < 6; p++) t += A1[i*6+p]*M(p, q);
    s += t*A2[j*6+q]; }
  return s;
}

constexpr int kSolveThreads = 512;
#ifdef SDV_BA_PROFILE
__device__ long long g_ba_prof[16];
#define BA_PROF_T(var) const long long var = clock64()
#define BA_PROF_ADD(slot, a, b) do { if (blockIdx.y == 0 && threadIdx.x == 0) g_ba_prof[slot] += (b) - (a); } while (0)
#else
#define BA_PROF_T(var) do {} while (0)
#define BA_PROF_ADD(slot, a, b) do {} while (0)
#endif
// Stitch the accumulated top (sA, sbA) and Schur (sS, sbS) systems from the per-bucket float accumulators.
//   MARG = false: stitchDoubleMT as solveSystemF calls it (buckets walked k = h + nF*t ascending, priors and deltas added)
//                 AccumulatedTopHessian.cpp:181-242 + .h:63-114, AccumulatedSCHessian.cpp:64-135 + .h:68-111
//   MARG = true : the single-threaded stitchDouble of marginalizePointsF (h outer / t inner, no priors)
//                 AccumulatedTopHessian.cpp:118-179, AccumulatedSCHessian.cpp:136-195
template <bool MARG>
__device__ __forceinline__ void ba_stitch(BAHeader* __restrict__ H, const int tid, const int nF, const int N, const int nF2,
                                          double* __restrict__ sA, double* __restrict__ sS, double* __restrict__ sbA, double* __restrict__ sbS) {
#define BK(kk) (MARG ? ((kk)/nF + nF*((kk)%nF)) : (kk))
  BA_PROF_T(ts0);
  // ---- products shared by many output elements, in the reference's operation order: T1 = AH*M, T3 = AT*M (top buckets), AH_ij*D, AT_ij*D (Schur buckets)
  for (int task = tid; task < nF2*72; task += kSolveThreads) {
    const int k = task/72, e = task%72, which = e/36, i = (e%36)/6, q = e%6; if (H->accTopNum[k] == 0) continue;
    const float* m = H->accTop + k*kNTop; const double* A1 = (which ? H->adTarget : H->adHost) + k*36;
    double t = 0; for (int p = 0; p < 6; p++) t += A1[i*6+p]*tri10(m, 4+p, 4+q);
    (which ? H->topT3 : H->topT1)[k*36 + i*6 + q] = t;
  }
  for (int task = tid; task < nF2*nF*72; task += kSolveThreads) {
    const int bk = task/72, e = task%72, which = e/36, i = (e%36)/6, q = e%6; if (H->accDNum[bk] == 0) continue;
    const int k = bk % nF2; const float* d = H->accD + bk*36; const double* A1 = (which ? H->adTarget : H->adHost) + k*36;
    double t = 0; for (int p = 0; p < 6; p++) t += A1[i*6+p]*(double)d[p*6+q];
    (which ? H->scT3 : H->scT1)[bk*36 + i*6 + q] = t;
  }
  __syncthreads();
  BA_PROF_T(ts1); BA_PROF_ADD(8, ts0, ts1);
  // ---- top: frame-frame blocks (raw), frame-calib blocks, calib block, gradient
  for (int task = tid; task < nF2*36; task += kSolveThreads) {
    const int blk = task/36, e = task%36, a = blk/nF, b = blk%nF, i = e/6, j = e%6; double acc = 0;
    auto term = [&](int k) {                                               // the contribution of bucket k = h + nF*t to cell (a,b), in the reference's order hh, tt, ht
      const int h = k % nF, t = k / nF;
      if (H->accTopNum[k] == 0) return;                                    // empty bucket contributes exact zeros
      const double* AH = H->adHost + k*36; const double* AT = H->adTarget + k*36; const double* T1 = H->topT1 + k*36 + i*6; const double* T3 = H->topT3 + k*36 + i*6;
      if (a == h && b == h) { double s2 = 0; for (int q=0;q<6;q++) s2 += T1[q]*AH[j*6+q]; acc += s2; }
      if (a == t && b == t) { double s2 = 0; for (int q=0;q<6;q++) s2 += T3[q]*AT[j*6+q]; acc += s2; }
      if (a == h && b == t) { double s2 = 0; for (int q=0;q<6;q++) s2 += T1[q]*AT[j*6+q]; acc += s2; }
    };
    if (MARG) {
      for (int kk = 0; kk < nF2; kk++) { const int k = BK(kk); const int h = k % nF, t = k / nF; if (!((a == h || a == t) && (b == h || b == t))) continue; term(k); }
    } else if (a != b) {                                                   // only the buckets (a,b) and (b,a) touch an off-diagonal cell: visit them in ascending k
      const int k1 = a + nF*b, k2 = b + nF*a; term(k1 < k2 ? k1 : k2); term(k1 < k2 ? k2 : k1);
    } else {                                                               // diagonal cell: buckets with h == a or t == a, ascending k = h + nF*t
      for (int t = 0; t < a; t++) term(a + nF*t);
      for (int h = 0; h < nF; h++) term(h + nF*a);
      for (int t = a+1; t < nF; t++) term(a + nF*t);
    }
    if (!MARG && a == b && i == j) acc += H->frames[a].prior[i];
    sA[(kCP+a*6+i)*N + kCP+b*6+j] = acc;
  }
  for (int task = tid; task < nF*24; task += kSolveThreads) {              // H[frame a, calib] (6x4)
    const int a = task/24, r = (task%24)/4, c = task%4; double acc = 0;
    for (int kk = 0; kk < nF2; kk++) { const int k = BK(kk); const int h = k % nF, t = k / nF; if (a != h && a != t) continue; if (H->accTopNum[k] == 0) continue;
      const float* m = H->accTop + k*kNTop;
      if (a == h) { const double* AH = H->adHost + k*36; double s1 = 0; for (int q=0;q<6;q++) s1 += AH[r*6+q]*tri10(m, 4+q, c); acc += s1; }
      if (a == t) { const double* AT = H->adTarget + k*36; double s2 = 0; for (int q=0;q<6;q++) s2 += AT[r*6+q]*tri10(m, 4+q, c); acc += s2; } }
    sA[(kCP+a*6+r)*N + c] = acc;
  }
  if (tid < 16) { const int r = tid/4, c = tid%4; double acc = 0; int resInA = 0;
    for (int kk = 0; kk < nF2; kk++) { const int k = BK(kk); resInA += H->accTopNum[k]; if (H->accTopNum[k] == 0) continue; acc += tri10(H->accTop + k*kNTop, r, c); }
    if (!MARG && r == c) acc += H->calib.cPrior[r];
    sA[r*N + c] = acc; if (!MARG && tid == 0) H->resInA = resInA; }
  for (int task = tid; task < N; task += kSolveThreads) {                  // bA
    double acc = 0;
    if (task < kCP) { for (int kk = 0; kk < nF2; kk++) { const int k = BK(kk); if (H->accTopNum[k] == 0) continue; acc += (double)H->accTop[k*kNTop + 55 + task]; }
      if (!MARG) acc += H->calib.cPrior[task]*(double)H->calib.cDeltaF[task]; }
    else { const int a = (task-kCP)/6, r = (task-kCP)%6;
      for (int kk = 0; kk < nF2; kk++) { const int k = BK(kk); const int h = k % nF, t = k / nF; if (a != h && a != t) continue; if (H->accTopNum[k] == 0) continue;
        const float* m = H->accTop + k*kNTop;
        if (a == h) { const double* AH = H->adHost + k*36; double s1 = 0; for (int q=0;q<6;q++) s1 += AH[r*6+q]*(double)m[55+4+q]; acc += s1; }
        if (a == t) { const double* AT = H->adTarget + k*36; double s2 = 0; for (int q=0;q<6;q++) s2 += AT[r*6+q]*(double)m[55+4+q]; acc += s2; } }
      if (!MARG) acc += H->frames[a].prior[r]*H->frames[a].delta_prior[r]; }
    sbA[task] = acc;
  }
  __syncthreads();
  BA_PROF_T(ts2); BA_PROF_ADD(9, ts1, ts2);
  // symmetrise (AccumulatedTopHessian.h:100-113): calib row-blocks = transposed column-blocks; (h,t) += (t,h)^T for t>h, then mirror
  for (int task = tid; task < nF*24; task += kSolveThreads) { const int a = task/24, r = (task%24)/6, c = task%6; sA[r*N + kCP+a*6+c] = sA[(kCP+a*6+c)*N + r]; }
  for (int task = tid; task < nF2*36; task += kSolveThreads) { const int blk = task/36, e = task%36, a = blk/nF, b = blk%nF, r = e/6, c = e%6;
    if (b > a) sA[(kCP+a*6+r)*N + kCP+b*6+c] += sA[(kCP+b*6+c)*N + kCP+a*6+r]; }
  __syncthreads();
  for (int task = tid; task < nF2*36; task += kSolveThreads) { const int blk = task/36, e = task%36, a = blk/nF, b = blk%nF, r = e/6, c = e%6;
    if (b > a) sA[(kCP+b*6+r)*N + kCP+a*6+c] = sA[(kCP+a*6+c)*N + kCP+b*6+r]; }
  BA_PROF_T(ts3); BA_PROF_ADD(10, ts2, ts3);
  // ---- Schur complement: frame-frame blocks
  for (int task = tid; task < nF2*36; task += kSolveThreads) {
    const int blk = task/36, e = task%36, a = blk/nF, b = blk%nF, i = e/6, j = e%6; double acc = 0;
    auto term = [&](int fi, int fj, int k2) {                              // bucket (k = fi + nF*fj, k2) -> cell (a,b), conditions in the reference's order
      const int k = fi + nF*fj;
      const bool c1 = (a == fi && b == fi), c2 = (a == fj && b == k2), c3 = (a == fj && b == fi), c4 = (a == fi && b == k2);
      if (!(c1 || c2 || c3 || c4)) return;
      const int bk = k + k2*nF2; if (H->accDNum[bk] == 0) return;
      const int ik = fi + nF*k2;
      const double* AHik = H->adHost + ik*36 + j*6; const double* ATik = H->adTarget + ik*36 + j*6;
      const double* T1 = H->scT1 + bk*36 + i*6; const double* T3 = H->scT3 + bk*36 + i*6;
      if (c1) { double s2 = 0; for (int q=0;q<6;q++) s2 += T1[q]*AHik[q]; acc += s2; }
      if (c2) { double s2 = 0; for (int q=0;q<6;q++) s2 += T3[q]*ATik[q]; acc += s2; }
      if (c3) { double s2 = 0; for (int q=0;q<6;q++) s2 += T3[q]*AHik[q]; acc += s2; }
      if (c4) { double s2 = 0; for (int q=0;q<6;q++) s2 += T1[q]*ATik[q]; acc += s2; }
    };
    if (MARG) {
      for (int kk = 0; kk < nF2; kk++) { const int k = BK(kk); const int fi = k % nF, fj = k / nF; if (a != fi && a != fj) continue;
        for (int k2 = 0; k2 < nF; k2++) term(fi, fj, k2); }
    } else {
      // same visiting order as the full scan (fj outer, fi inner, k2 innermost), restricted to the (fi, fj, k2) that can satisfy one of the four conditions:
      //   fi == a: c1 needs b == a (any k2), c4 needs k2 == b;   fj == a: c2 needs k2 == b, c3 needs fi == b (any k2)
      for (int fj = 0; fj < nF; fj++) {
        if (fj != a) {                                                     // only fi == a can match (c1 / c4)
          if (a == b) { for (int k2 = 0; k2 < nF; k2++) term(a, fj, k2); } else term(a, fj, b);
        } else {
          for (int fi = 0; fi < nF; fi++) {
            const bool all_k2 = (fi == b) || (fi == a && a == b);          // c3, or c1
            if (all_k2) { for (int k2 = 0; k2 < nF; k2++) term(fi, fj, k2); } else term(fi, fj, b);   // c2 (and c4 when fi == a) at k2 == b only
          }
        }
      }
    }
    sS[(kCP+a*6+i)*N + kCP+b*6+j] = acc;
  }
  BA_PROF_T(ts4); BA_PROF_ADD(11, ts3, ts4);
  for (int task = tid; task < nF*24; task += kSolveThreads) {              // Hsc[frame a, calib]
    const int a = task/24, r = (task%24)/4, c = task%4; double acc = 0;
    for (int kk = 0; kk < nF2; kk++) { const int k = BK(kk); const int fi = k % nF, fj = k / nF; if (a != fi && a != fj) continue;
      if (a == fi) { const double* AH = H->adHost + k*36; double s1 = 0; for (int q=0;q<6;q++) s1 += AH[r*6+q]*(double)H->accE[k*24+q*4+c]; acc += s1; }
      if (a == fj) { const double* AT = H->adTarget + k*36; double s2 = 0; for (int q=0;q<6;q++) s2 += AT[r*6+q]*(double)H->accE[k*24+q*4+c]; acc += s2; } }
    sS[(kCP+a*6+r)*N + c] = acc;
  }
  if (tid < 16) sS[(tid/4)*N + tid%4] = (double)H->accHcc[tid];
  for (int task = tid; task < N; task += kSolveThreads) {                  // bsc
    double acc = 0;
    if (task < kCP) acc = (double)H->accbc[task];
    else { const int a = (task-kCP)/6, r = (task-kCP)%6;
      for (int kk = 0; kk < nF2; kk++) { const int k = BK(kk); const int fi = k % nF, fj = k / nF; if (a != fi && a != fj) continue;
        if (a == fi) { const double* AH = H->adHost + k*36; double s1 = 0; for (int q=0;q<6;q++) s1 += AH[r*6+q]*(double)H->accEB[k*6+q]; acc += s1; }
        if (a == fj) { const double* AT = H->adTarget + k*36; double s2 = 0; for (int q=0;q<6;q++) s2 += AT[r*6+q]*(double)H->accEB[k*6+q]; acc += s2; } } }
    sbS[task] = acc;
  }
  __syncthreads();
  for (int task = tid; task < nF*24; task += kSolveThreads) { const int a = task/24, r = (task%24)/6, c = task%6; sS[r*N + kCP+a*6+c] = sS[(kCP+a*6+c)*N + r]; }
  __syncthreads();
#undef BK
}

__global__ void __launch_bounds__(kSolveThreads) ba_solve_kernel(const BAWinDev* __restrict__ wins, int iteration_arg, double lambda_arg, int use_hdr_ctl, int gate) {
  BA_WIN(gate)
  const int iteration = use_hdr_ctl ? H->iteration : iteration_arg; const double lambda = use_hdr_ctl ? H->lambda : lambda_arg;
  const int tid = threadIdx.x; const int nF = H->nF, N = H->dim, nF2 = nF*nF;
  __shared__ double sA[kMaxDim*kMaxDim];                                    // HA -> HFinal (scaled) -> LDLT in place
  __shared__ double sS[kMaxDim*kMaxDim];                                    // Hsc -> nullspace basis
  __shared__ double sv[kMaxDim], sb[kMaxDim], sx[kMaxDim], stmp[kMaxDim], sbA[kMaxDim], sbS[kMaxDim];
  __shared__ int sperm[kMaxDim]; __shared__ int spiv; __shared__ double srot[4];
  BA_PROF_T(tb0);
  ba_stitch<false>(H, tid, nF, N, nF2, sA, sS, sbA, sbS);
  BA_PROF_T(tb1); BA_PROF_ADD(0, tb0, tb1);
  // ---- publish HA/bA/Hsc/bsc (read-back for tests), HFinal / bFinal, damping, diagonal pre-scaling (EnergyFunctional.cpp:668-744)
  for (int i = tid; i < N*N; i += kSolveThreads) { H->HA[i] = sA[i]; H->Hsc[i] = sS[i]; double v = sA[i] + H->HM[i] - sS[i]; H->lastHS[i] = v; sA[i] = v; }
  if (tid < N) {
    H->bA[tid] = sbA[tid]; H->bsc[tid] = sbS[tid];
    double s = 0; for (int j=0;j<N;j++) { double dj = (j < 4) ? (double)H->calib.cDeltaF[j] : H->frames[(j-4)/6].delta[(j-4)%6]; s += H->HM[tid*N+j]*dj; }
    double bf = sbA[tid] + (H->bM[tid] + s) - sbS[tid]; H->lastbS[tid] = bf; sb[tid] = bf;
  }
  __syncthreads();
  if (tid < N) { sA[tid*N+tid] *= (1+lambda); }
  __syncthreads();
  if (tid < N) sv[tid] = 1.0/sqrt(sA[tid*N+tid] + 10);
  __syncthreads();
  for (int i = tid; i < N*N; i += kSolveThreads) { int r = i/N, c = i%N; sA[i] = sv[r]*sA[i]*sv[c]; }
  if (tid < N) sb[tid] = sv[tid]*sb[tid];
  __syncthreads();
  BA_PROF_T(tb2); BA_PROF_ADD(1, tb1, tb2);
  // ---- pivoted LDLT, left-looking like Eigen's unblocked kernel: every dot product is evaluated by ONE thread in index order.
  // Only the first two warps take part (one matrix row per thread, N <= 52) and meet at a 64-thread named barrier; the pivot search is a warp arg-max
  // (first index among equal maxima, like the sequential `a > big` scan).  The other warps wait at the block barrier behind the solve.
#define BAR64() asm volatile("bar.sync 1, 64;" ::: "memory")
  if (tid < 64) {
    for (int k = 0; k < N; k++) {
      if (tid < 32) {
        double best = -1.0; int bi = k;
#pragma unroll
        for (int rep = 0; rep < 2; rep++) { const int i = k + tid + 32*rep;
          if (i < N) { const double v = fabs(sA[i*N+i]); const double a = (i == k) ? v : ((v == v) ? v : -1.0);     // a NaN diagonal entry never replaces the running maximum (a > big is false)
            if (i == k || a > best) { best = a; bi = i; } } }
#pragma unroll
        for (int off = 16; off > 0; off >>= 1) {
          const double ob = __shfl_down_sync(0xffffffffu, best, off); const int oi = __shfl_down_sync(0xffffffffu, bi, off);
          if (ob > best || (ob == best && oi < bi)) { best = ob; bi = oi; } }
        if (tid == 0) { spiv = bi; sperm[k] = bi; }
      }
      BAR64();
      const int piv = spiv;
      if (piv != k) {
        if (tid < k) { double s = sA[k*N+tid]; sA[k*N+tid] = sA[piv*N+tid]; sA[piv*N+tid] = s; }
        else if (tid > piv && tid < N) { double s = sA[tid*N+k]; sA[tid*N+k] = sA[tid*N+piv]; sA[tid*N+piv] = s; }
        else if (tid > k && tid < piv) { double s = sA[tid*N+k]; sA[tid*N+k] = sA[piv*N+tid]; sA[piv*N+tid] = s; }
        else if (tid == k) { double s = sA[k*N+k]; sA[k*N+k] = sA[piv*N+piv]; sA[piv*N+piv] = s; }
        BAR64();
      }
      if (tid < k) stmp[tid] = sA[tid*N+tid]*sA[k*N+tid];
      BAR64();
      if (tid >= k && tid < N && k > 0) {                                      // row k: the diagonal update, rows below: the column update — same loop, same order
        const double* row = sA + tid*N; double s2 = 0;
#pragma unroll 4
        for (int j = 0; j < k; j++) s2 += row[j]*stmp[j];
        sA[tid*N+k] -= s2;
      }
      BAR64();
      const double akk = sA[k*N+k];
      if (tid > k && tid < N && fabs(akk) > 0) sA[tid*N+k] /= akk;
      BAR64();
    }
    BA_PROF_T(tb3); BA_PROF_ADD(2, tb2, tb3);
    // ---- solve: P, L^-1, D^+, L^-T, P^T.  L^-1 column by column: thread i owns y_i and subtracts L_ij*y_j for j ascending — the row-wise order of the sequential loop;
    // L^-T stays sequential (row i needs y_{i+1} first), its products do not sit on the dependency chain.
    if (tid == 0) { for (int i=0;i<N;i++) sx[i] = sb[i]; for (int k=0;k<N;k++) { double s = sx[k]; sx[k] = sx[sperm[k]]; sx[sperm[k]] = s; } }
    BAR64();
    { double yi = (tid < N) ? sx[tid] : 0.0;
      for (int j2 = 0; j2 < N; j2++) {
        if (tid == j2) sx[j2] = yi;
        BAR64();
        if (tid > j2 && tid < N) yi -= sA[tid*N+j2]*sx[j2];
      } }
    BAR64();
    if (tid < 32) {
      double dm = 0;
      for (int i = tid; i < N; i += 32) dm = fmax(dm, fabs(sA[i*N+i]));
#pragma unroll
      for (int off = 16; off > 0; off >>= 1) dm = fmax(dm, __shfl_xor_sync(0xffffffffu, dm, off));
      const double tol = fmax(dm*2.220446049250313e-16, 1.0/1.7976931348623157e308);
      for (int i = tid; i < N; i += 32) { const double d = sA[i*N+i]; sx[i] = (fabs(d) > tol) ? sx[i]/d : 0.0; }
    }
    BAR64();
    if (tid == 0) {
      for (int i=N-1;i>=0;i--) { double s = sx[i];
#pragma unroll 4
        for (int j2=i+1;j2<N;j2++) s -= sA[j2*N+i]*sx[j2];
        sx[i] = s; }
      for (int k=N-1;k>=0;k--) { double s = sx[k]; sx[k] = sx[sperm[k]]; sx[sperm[k]] = s; }
    }
    BAR64();
    if (tid < N) sx[tid] = sv[tid]*sx[tid];
  }
#undef BAR64
  __syncthreads();
  BA_PROF_T(tb4); BA_PROF_ADD(3, tb2, tb4);
  // ---- orthogonalize x against the pose+scale nullspaces for iteration >= 2 (EnergyFunctional.cpp:615-648, 746-750).  The basis only
  // depends on the evaluation points, so it is computed once per linearisation point (one-sided Jacobi, same operation order as the
  // oracle: each dot product by one thread, row updates in parallel) and cached in the header.
  if (iteration >= 2) {
    const int m = 7; double* A = sS;                                        // N x 7, column i at A[i*N ..]
    if (!H->ortho_valid) {
      for (int e = tid; e < N*m; e += kSolveThreads) { int r = e % N, i = e / N; double v = 0;
        if (r >= kCP) { int f = (r-kCP)/6, q = (r-kCP)%6; v = (i < 6) ? H->frames[f].nullspaces_pose[q*6+i] : H->frames[f].nullspaces_scale[q]; v *= (q < 3) ? (double)(1.0f/0.5f) : (double)(1.0f/1.0f); }
        A[i*N + r] = v; }
      __syncthreads();
      if (tid < m) { double nr = 0; for (int r=0;r<N;r++) nr += A[tid*N+r]*A[tid*N+r]; nr = sqrt(nr); for (int r=0;r<N;r++) A[tid*N+r] /= nr; }
      __syncthreads();
      // one-sided Jacobi on the first two warps (row updates: one row per thread, N <= 52), 64-thread named barrier instead of block barriers
      if (tid < 64) {
        for (int sweep = 0; sweep < 60; sweep++) {
          if (tid == 0) srot[3] = 0;
          for (int p=0;p<m;p++) for (int q=p+1;q<m;q++) {
            asm volatile("bar.sync 1, 64;" ::: "memory");
            if (tid == 0) { double al = 0;
#pragma unroll 4
              for (int r=0;r<N;r++) al += A[p*N+r]*A[p*N+r]; srot[0] = al; }
            else if (tid == 32) { double be = 0, ga = 0;                      // two independent chains, each in index order
#pragma unroll 4
              for (int r=0;r<N;r++) { const double aq = A[q*N+r]; be += aq*aq; ga += A[p*N+r]*aq; }
              srot[1] = be; srot[2] = ga; }
            asm volatile("bar.sync 1, 64;" ::: "memory");
            const double al = srot[0], be = srot[1], ga = srot[2];
            if (fabs(ga) <= 1e-300 || fabs(ga) <= 1e-17*sqrt(al*be)) continue;
            if (tid == 0) srot[3] = fmax(srot[3], fabs(ga)/sqrt(al*be + 1e-300));
            const double zeta = (be-al)/(2*ga), tt = ((zeta >= 0) ? 1.0 : -1.0)/(fabs(zeta) + sqrt(1+zeta*zeta)), c = 1/sqrt(1+tt*tt), sn = c*tt;
            if (tid < N) { double ap = A[p*N+tid], aq = A[q*N+tid]; A[p*N+tid] = c*ap - sn*aq; A[q*N+tid] = sn*ap + c*aq; }
          }
          asm volatile("bar.sync 1, 64;" ::: "memory");
          if (srot[3] < 1e-15) break;
          asm volatile("bar.sync 1, 64;" ::: "memory");
        }
      }
      __syncthreads();
      if (tid < m) { double nr = 0; for (int r=0;r<N;r++) nr += A[tid*N+r]*A[tid*N+r]; H->orthoS[tid] = sqrt(nr); }
      for (int e = tid; e < N*m; e += kSolveThreads) H->orthoU[e] = A[e];
      __syncthreads();
      if (tid == 0) H->ortho_valid = 1;
    } else {
      for (int e = tid; e < N*m; e += kSolveThreads) A[e] = H->orthoU[e];
      __syncthreads();
    }
    if (tid == 0) {
      double maxSv = 0; for (int i=0;i<m;i++) maxSv = fmax(maxSv, H->orthoS[i]);
      for (int r=0;r<N;r++) stmp[r] = 0;
      for (int i=0;i<m;i++) { const double svi = H->orthoS[i]; if (!(svi > H->set.solverModeDelta*maxSv)) continue;
        double dot = 0; for (int r=0;r<N;r++) dot += (A[i*N+r]/svi)*sx[r];
        for (int r=0;r<N;r++) stmp[r] += (A[i*N+r]/svi)*dot; }
      for (int r=0;r<N;r++) sx[r] -= stmp[r];
    }
    __syncthreads();
  }
  BA_PROF_T(tb5); BA_PROF_ADD(4, tb4, tb5);
  // ---- lastX, steps, xAd (resubstituteF_MT head, EnergyFunctional.cpp:221-248)
  if (tid < N) { H->lastX[tid] = sx[tid]; H->xF[tid] = (float)sx[tid]; }
  if (tid < 4) H->calib.step[tid] = -sx[tid];
  if (tid >= 32 && tid < 32 + nF) { BAFrameDev& f = H->frames[tid-32]; for (int i=0;i<6;i++) f.step[i] = -sx[kCP + 6*(tid-32) + i]; for (int i=6;i<10;i++) f.step[i] = 0; }
  __syncthreads();
  for (int e = tid; e < nF2*6; e += kSolveThreads) { int pr = e/6, j = e%6, h = pr / nF, t = pr % nF;       // xAd[nF*h + t]
    float s1 = 0, s2 = 0; for (int i=0;i<6;i++) { s1 += (float)sx[kCP+6*h+i]*H->adHostF[(h+nF*t)*36+i*6+j]; s2 += (float)sx[kCP+6*t+i]*H->adTargetF[(h+nF*t)*36+i*6+j]; }
    H->xAd[(nF*h+t)*6+j] = s1 + s2; }
  BA_PROF_T(tb6); BA_PROF_ADD(5, tb5, tb6); BA_PROF_ADD(6, tb0, tb6);
#ifdef SDV_BA_PROFILE
  if (blockIdx.y == 0 && tid == 0) g_ba_prof[7] += 1;
#endif
}
#ifdef SDV_BA_PROFILE
extern "C" int sdv_debug_ba_profile(long long* out16, int reset) {
  long long z[16] = {0};
  if (out16) cudaMemcpyFromSymbol(out16, g_ba_prof, sizeof(z));
  if (reset) cudaMemcpyToSymbol(g_ba_prof, z, sizeof(z));
  return 0;
}
#endif

__global__ void ba_resub_kernel(const BAWinDev* __restrict__ wins, int gate) {     // resubstituteFPt (:250-282)
  BA_WIN(gate)
  int p = blockIdx.x*blockDim.x + threadIdx.x; if (p >= nP) return;
  if (P.ngood[p] == 0) { P.step[p] = 0; return; }
  const int nF = H->nF;
  float b = P.bdSumF[p];
  { float s = 0; for (int i=0;i<4;i++) s += H->xF[i]*P.Hcd_accAF[(size_t)p*4+i]; b -= s; }
  for (int r = P.res_begin[p]; r < P.res_begin[p+1]; r++) { if (!R.isActive[r]) continue;
    const float* xa = H->xAd + (R.host[r]*nF + R.target[r])*6; float s = 0; for (int i=0;i<6;i++) s += xa[i]*R.JpJdF[(size_t)r*8+i]; b -= s; }
  P.step[p] = P.isFromSensor[p] ? 0.0f : -b*P.HdiF[p];
}

// ================================================================================================ backup / step
__global__ void ba_backup_kernel(const BAWinDev* __restrict__ wins, int gate) {
  BA_WIN(gate)
  int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i < nP) P.idepth_backup[i] = P.idepth[i];
  if (i < H->nF) for (int k=0;k<10;k++) H->frames[i].state_backup[k] = H->frames[i].state[k];
  if (i == 0) for (int k=0;k<4;k++) H->calib.value_backup[k] = H->calib.value[k];
}
// points part of doStepFromBackup / loadSateBackup + the float sums the break test needs (single CTA keeps the reduction fixed-order)
__global__ void __launch_bounds__(1024) ba_step_points_kernel(const BAWinDev* __restrict__ wins, float stepfac, int load_backup, int gate) {
  BA_WIN(gate)
  __shared__ float s1[1024], s2[1024];
  float sumID = 0, sumNID = 0;
  for (int i = threadIdx.x; i < nP; i += 1024) {
    float nv = load_backup ? P.idepth_backup[i] : P.idepth_backup[i] + stepfac*P.step[i];
    P.idepth[i] = nv; P.idepth_zero[i] = nv; P.deltaF[i] = nv - nv;
    sumID += P.step[i]*P.step[i]; sumNID += fabsf(P.idepth_backup[i]);
  }
  s1[threadIdx.x] = sumID; s2[threadIdx.x] = sumNID; __syncthreads();
  for (int o = 512; o > 0; o >>= 1) { if (threadIdx.x < o) { s1[threadIdx.x] += s1[threadIdx.x+o]; s2[threadIdx.x] += s2[threadIdx.x+o]; } __syncthreads(); }
  if (threadIdx.x == 0) { H->sums[0] = s1[0]; H->sums[1] = s2[0]; H->sums[2] = (float)nP; }
}

// ================================================================================================ device-resident GN control
// stage 0: after the initial linearizeAll + energies (optimize :373-381)         -> lastEnergy*, lambda, APPLY
// stage 1: after backup/solve/step/linearize/energies of one iteration (:395-454) -> accept (APPLY, lambda/4) or reject (RELOAD, lambda*100)
// stage 2: after the reload path of a rejected step                               -> lastEnergy* from the re-linearisation; break test (:457)
// stage 3: after the final linearizeAll(true)                                     -> rmse (:501)
__global__ void ba_decide_kernel(const BAWinDev* __restrict__ wins, int W, int stage) {
  const int wi = blockIdx.x*blockDim.x + threadIdx.x; if (wi >= W) return;
  BAHeader* H = wins[wi].hdr;
  if (stage == 0) {
    int m = H->mnumOptIts; if (H->nF < 3) m = 100; if (H->nF < 4) m = 75;                // FullSystemOptimize.cpp:347-349 (sequential ifs)
    H->mnumOptIts = m; H->iteration = 0; H->opt_iterations = 0; H->opt_accepts = 0; H->lambda = 1e-1;
    H->lastEnergy = H->energyP; H->lastEnergyL = H->energyL; H->lastEnergyM = H->energyM;
    H->flags = (H->nF >= 2) ? BA_ACTIVE : 0;
  } else if (stage == 1) {
    if (!(H->flags & BA_ACTIVE)) return;
    H->opt_iterations++;
    const double newE = H->energyP, newL = H->energyL, newM = H->energyM;
    if (newE + 0 + newL + newM < H->lastEnergy + 0 + H->lastEnergyL + H->lastEnergyM) {
      H->opt_accepts++; H->lastEnergy = newE; H->lastEnergyL = newL; H->lastEnergyM = newM; H->lambda *= 0.25; H->flags |= BA_APPLY;
    } else { H->lambda *= 1e2; H->flags |= BA_RELOAD; }
  } else if (stage == 2) {
    if (!(H->flags & BA_ACTIVE)) return;
    if (H->flags & BA_RELOAD) { H->lastEnergy = H->energyP; H->lastEnergyL = H->energyL; H->lastEnergyM = H->energyM; }
    H->flags &= ~(BA_APPLY | BA_RELOAD);
    const int it = H->iteration; H->iteration = it + 1;
    if ((H->canbreak && it >= H->set.minOptIterations) || it + 1 >= H->mnumOptIts) H->flags &= ~BA_ACTIVE;
  } else {
    H->rmse = sqrtf((float)(H->energyP / H->resInA));
  }
}

// ================================================================================================ keyframe hand-over: marginalisation
// FullSystem::flagPointsForRemoval, numeric part (FullSystem.cpp:764-797).  P.marg_status[p] holds the host-side predicate on entry
// ((isOOB || host flagged) && isInlierNew — graph bookkeeping) and the resulting EFPointStatus on exit.  One thread per point: its
// residuals are re-linearised at the current state (resetOOB, linearize, applyRes(true)) and frozen by fixLinearizationF.
__global__ void __launch_bounds__(128) ba_marg_flag_kernel(const BAWinDev* __restrict__ wins) {
  BA_WIN(0)
  const int p = blockIdx.x*blockDim.x + threadIdx.x; if (p >= nP) return;
  if (!P.marg_status[p]) return;
  const int nF = H->nF; const float deltaF = P.deltaF[p];
  for (int r = P.res_begin[p]; r < P.res_begin[p+1]; r++) {
    if (R.toRemove[r]) continue;                                             // dropped by linearizeAll(fix) (the reference deleted it, FullSystemOptimize.cpp:129-157): it is not in ph->residuals any more
    R.state_NewEnergy[r] = 0; R.state_energy[r] = 0; R.state_NewState[r] = RS_OUTLIER; R.state_state[r] = RS_IN;
    lin_residual(H, P, R, r, nullptr, nullptr);
    R.isLinearized[r] = 0;
    apply_res(R, r);
    if (R.isActive[r]) {                                                     // EFResidual::fixLinearizationF (EnergyFunctionalStructs.cpp:46-55)
      const float* J = R.efJ + (size_t)r*24; const float* dp = H->adHTdeltaF + (R.host[r] + nF*R.target[r])*6;
      float dx0 = 0, dx1 = 0, dc0 = 0, dc1 = 0;
      for (int i=0;i<6;i++) { dx0 += J[2+i]*dp[i]; dx1 += J[8+i]*dp[i]; }
      for (int i=0;i<4;i++) { dc0 += J[14+i]*H->calib.cDeltaF[i]; dc1 += J[18+i]*H->calib.cDeltaF[i]; }
      const float Jp_delta_x = dx0 + dc0 + J[22]*deltaF, Jp_delta_y = dx1 + dc1 + J[23]*deltaF;
      R.res_toZero[r] = make_float2(J[0] - Jp_delta_x, J[1] - Jp_delta_y);
      R.isLinearized[r] = 1;
    }
  }
  P.marg_status[p] = (P.idepth_hessian[p] > 50.0f) ? 2 : 1;                  // setting_minIdepthH_marg (settings.cpp:42)
}

// EnergyFunctional::marginalizePointsF, tail (EnergyFunctional.cpp:549-567): stitch M, Msc, then HM += margWeightFac*(M - Msc).
// M/Mb/Msc/Mbsc are published in the HA/bA/Hsc/bsc slots of the header for read-back.
__global__ void __launch_bounds__(kSolveThreads) ba_marg_stitch_kernel(const BAWinDev* __restrict__ wins) {
  BA_WIN(0)
  const int tid = threadIdx.x; const int nF = H->nF, N = H->dim, nF2 = nF*nF;
  __shared__ double sA[kMaxDim*kMaxDim]; __shared__ double sS[kMaxDim*kMaxDim]; __shared__ double sbA[kMaxDim], sbS[kMaxDim];
  ba_stitch<true>(H, tid, nF, N, nF2, sA, sS, sbA, sbS);
  const double fac = (double)(0.5f*0.5f);                                    // setting_margWeightFac (settings.cpp:71)
  for (int i = tid; i < N*N; i += kSolveThreads) { H->HA[i] = sA[i]; H->Hsc[i] = sS[i]; const double d = sA[i] - sS[i]; H->HM[i] += fac*d; }
  if (tid < N) { H->bA[tid] = sbA[tid]; H->bsc[tid] = sbS[tid]; const double d = sbA[tid] - sbS[tid]; H->bM[tid] += fac*d; }
  if (tid == 0) H->ortho_valid = 0;
}

// EnergyFunctional::marginalizeFrame (EnergyFunctional.cpp:434-512): fp64, one CTA.  The frame's 6 unknowns are moved to the end, its
// prior added, the system is diagonally pre-scaled, the 6x6 block inverted (partial-pivot LU) and eliminated, the result un-scaled and
// symmetrised.  idxs[w] names window w's frame (-1: none this round).  Frame idx is then dropped from the header (frames[], nF, dim); points/residuals of the window are stale afterwards.
__global__ void __launch_bounds__(kSolveThreads) ba_marg_frame_kernel(const BAWinDev* __restrict__ wins, const int* __restrict__ idxs) {
  BA_WIN(0)
  const int idx = idxs[blockIdx.y];
  const int tid = threadIdx.x; const int nF = H->nF, odim = H->dim, ndim = odim - 6;
  if (idx < 0 || idx >= nF) return;
  __shared__ double sH[kMaxDim*kMaxDim]; __shared__ double sb[kMaxDim], SV[kMaxDim], SVI[kMaxDim]; __shared__ double hpi[36], bli[kMaxDim*6]; __shared__ int ord[kMaxDim];
  if (tid < odim) { int o; if (tid < ndim) o = (tid < kCP + 6*idx) ? tid : tid + 6; else o = kCP + 6*idx + (tid - ndim); ord[tid] = o; }
  __syncthreads();
  for (int i = tid; i < odim*odim; i += kSolveThreads) { const int r = i/odim, c = i%odim; double v = H->HM[ord[r]*odim + ord[c]];
    if (r == c && r >= ndim) v += H->frames[idx].prior[r-ndim];
    sH[i] = v; }
  if (tid < odim) { double v = H->bM[ord[tid]]; if (tid >= ndim) v += H->frames[idx].prior[tid-ndim]*H->frames[idx].delta_prior[tid-ndim]; sb[tid] = v; }
  __syncthreads();
  if (tid < odim) { SV[tid] = sqrt(fabs(sH[tid*odim+tid]) + 10.0); SVI[tid] = 1.0/SV[tid]; }
  __syncthreads();
  for (int i = tid; i < odim*odim; i += kSolveThreads) { const int r = i/odim, c = i%odim; sH[i] = (SVI[r]*sH[i])*SVI[c]; }
  if (tid < odim) sb[tid] = SVI[tid]*sb[tid];
  __syncthreads();
  if (tid == 0) {                                                            // hpi = bottomRightCorner<6,6>().inverse()
    double L[36]; int perm[6];
    for (int i=0;i<6;i++) { perm[i] = i; for (int j=0;j<6;j++) { double v = sH[(ndim+i)*odim + ndim+j]; L[i*6+j] = 0.5*(v+v); } }
    for (int k=0;k<6;k++) {
      int piv = k; double big = fabs(L[k*6+k]); for (int i=k+1;i<6;i++) { double a = fabs(L[i*6+k]); if (a > big) { big = a; piv = i; } }
      if (piv != k) { for (int j=0;j<6;j++) { double t = L[k*6+j]; L[k*6+j] = L[piv*6+j]; L[piv*6+j] = t; } int t = perm[k]; perm[k] = perm[piv]; perm[piv] = t; }
      for (int i=k+1;i<6;i++) L[i*6+k] /= L[k*6+k];
      for (int i=k+1;i<6;i++) for (int j=k+1;j<6;j++) L[i*6+j] -= L[i*6+k]*L[k*6+j];
    }
    for (int c=0;c<6;c++) { double y[6]; for (int i=0;i<6;i++) y[i] = (perm[i] == c) ? 1.0 : 0.0;
      for (int k=0;k<6;k++) for (int i=k+1;i<6;i++) y[i] -= L[i*6+k]*y[k];
      for (int k=5;k>=0;k--) { y[k] /= L[k*6+k]; for (int i=0;i<k;i++) y[i] -= L[i*6+k]*y[k]; }
      for (int i=0;i<6;i++) hpi[i*6+c] = 0.5*(y[i]+y[i]); }
  }
  __syncthreads();
  for (int t = tid; t < ndim*6; t += kSolveThreads) { const int i = t/6, j = t%6; double s = 0; for (int k=0;k<6;k++) s += sH[(ndim+k)*odim + i]*hpi[k*6+j]; bli[t] = s; }
  __syncthreads();
  for (int t = tid; t < ndim*ndim; t += kSolveThreads) { const int i = t/ndim, j = t%ndim; double s = 0; for (int k=0;k<6;k++) s += bli[i*6+k]*sH[(ndim+k)*odim + j]; sH[i*odim+j] -= s; }
  __syncthreads();                                                           // (the bottom rows read above are not written by the update)
  if (tid < ndim) { double s = 0; for (int k=0;k<6;k++) s += bli[tid*6+k]*sb[ndim+k]; sb[tid] -= s; }
  __syncthreads();
  for (int t = tid; t < ndim*ndim; t += kSolveThreads) { const int i = t/ndim, j = t%ndim; sH[i*odim+j] = (SV[i]*sH[i*odim+j])*SV[j]; }
  if (tid < ndim) sb[tid] = SV[tid]*sb[tid];
  __syncthreads();
  for (int t = tid; t < ndim*ndim; t += kSolveThreads) { const int i = t/ndim, j = t%ndim; H->HM[i*ndim+j] = 0.5*(sH[i*odim+j] + sH[j*odim+i]); }
  if (tid < ndim) H->bM[tid] = sb[tid];
  __syncthreads();
  if (tid == 0) { for (int f = idx; f+1 < nF; f++) H->frames[f] = H->frames[f+1]; H->nF = nF-1; H->dim = ndim; H->nP = 0; H->nR = 0; H->ortho_valid = 0; }
}

// ================================================================================================ launchers
static inline dim3 g2(int n, int per, int W) { int gx = (n + per - 1)/per; if (gx < 1) gx = 1; return dim3(gx, W); }
void launch_ba_setup(const BAWinDev* wins, int W, int maxP, cudaStream_t st) {
  ba_frames_kernel<<<dim3(1, W), 64, 0, st>>>(wins, 1|2|4|8|16, 0.f, 0, GATE_ALWAYS);
  ba_points_setup_kernel<<<g2(maxP, 256, W), 256, 0, st>>>(wins, 1);
}
void launch_ba_reset_oob(const BAWinDev* wins, int W, int maxR, cudaStream_t st) { ba_reset_oob_kernel<<<g2(maxR, 256, W), 256, 0, st>>>(wins); }
void launch_ba_linearize(const BAWinDev* wins, int W, int maxR, int fix, int gate, cudaStream_t st) {
  ba_linearize_kernel<<<g2(maxR, kLinThreads, W), kLinThreads, 0, st>>>(wins, fix, gate);
  ba_energy_th_kernel<<<dim3(1, W), 1024, 0, st>>>(wins, gate);
}
void launch_ba_apply(const BAWinDev* wins, int W, int maxR, int gate, cudaStream_t st) { ba_apply_kernel<<<g2(maxR, 256, W), 256, 0, st>>>(wins, gate); }
void launch_ba_energies(const BAWinDev* wins, int W, int gate, cudaStream_t st) { ba_energies_kernel<<<dim3(1, W), 256, 0, st>>>(wins, gate); }
static void accumulate_mode(const BAWinDev* wins, int W, int maxP, int gate, int mode, cudaStream_t st) {
  ba_point_acc_kernel<<<g2(maxP, 128, W), 128, 0, st>>>(wins, gate, mode);
  ba_acc_top_kernel<<<dim3(kMaxF*kMaxF, W), 96, 0, st>>>(wins, gate, mode);
  ba_acc_sc_kernel<<<dim3(kMaxF + 1, W), 96, 0, st>>>(wins, gate);          // kMaxF host CTAs + one CTA for the calibration block
}
void launch_ba_accumulate(const BAWinDev* wins, int W, int maxP, int gate, cudaStream_t st) { accumulate_mode(wins, W, maxP, gate, 0, st); }
void launch_ba_solve(const BAWinDev* wins, int W, int maxP, int iteration, double lambda, int use_hdr_ctl, int gate, cudaStream_t st) {
  ba_solve_kernel<<<dim3(1, W), kSolveThreads, 0, st>>>(wins, iteration, lambda, use_hdr_ctl, gate);
  ba_resub_kernel<<<g2(maxP, 128, W), 128, 0, st>>>(wins, gate);
}
void launch_ba_backup(const BAWinDev* wins, int W, int maxP, int gate, cudaStream_t st) { ba_backup_kernel<<<g2(maxP > kMaxF ? maxP : kMaxF, 256, W), 256, 0, st>>>(wins, gate); }
void launch_ba_step(const BAWinDev* wins, int W, float stepfac, int load_backup, int gate, cudaStream_t st) {
  ba_step_points_kernel<<<dim3(1, W), 1024, 0, st>>>(wins, stepfac, load_backup, gate);
  ba_frames_kernel<<<dim3(1, W), 64, 0, st>>>(wins, 64|1|16, stepfac, load_backup, gate);
}
void launch_ba_reanchor(const BAWinDev* wins, int W, int maxP, cudaStream_t st) {
  ba_frames_kernel<<<dim3(1, W), 64, 0, st>>>(wins, 32|8|16, 0.f, 0, GATE_ALWAYS);
  ba_points_setup_kernel<<<g2(maxP, 256, W), 256, 0, st>>>(wins, 0);
}
void launch_ba_marg_flag(const BAWinDev* wins, int W, int maxP, cudaStream_t st) { ba_marg_flag_kernel<<<g2(maxP, 128, W), 128, 0, st>>>(wins); }
void launch_ba_marg_points(const BAWinDev* wins, int W, int maxP, cudaStream_t st) {
  accumulate_mode(wins, W, maxP, GATE_ALWAYS, 2, st);
  ba_marg_stitch_kernel<<<dim3(1, W), kSolveThreads, 0, st>>>(wins);
}
void launch_ba_marg_frame(const BAWinDev* wins, int W, const int* idx, cudaStream_t st) { ba_marg_frame_kernel<<<dim3(1, W), kSolveThreads, 0, st>>>(wins, idx); }
void launch_ba_decide(const BAWinDev* wins, int W, int stage, cudaStream_t st) { ba_decide_kernel<<<(W + 127)/128, 128, 0, st>>>(wins, W, stage); }

} // namespace sdv
