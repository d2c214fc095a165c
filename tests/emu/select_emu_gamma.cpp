// select_emu_gamma.cpp — TEST INFRASTRUCTURE: the candidate-management engine of sdv-loam_b200/csrc/sdv_select_core.cuh compiled for the host (tests/emu/cuda_emu.hpp),
// with entry points whose jobs carry their frame camera's gamma weights (HistJob::gw2, MapsJobHost::gw2, NewTracesJob::gw2: gamma_w2 of sdv_core_common.cuh; NULL: none),
// for tests/test_select_emu_gamma_cpu.py.  "Device" pointers are host pointers here; selector slots are the SelectorSlot objects of tests/emu/select_emu.cpp.
#define SDV_EMU 1
#define SDV_EMU_IMPL 1
#include "cuda_emu.hpp"
#include "../../sdv-loam_b200/csrc/sdv_select_core.cuh"
using namespace sdv::sel;

extern "C" {
void* emu_gamma_engine_create(int w, int h, const unsigned char* rp) {
  SelEngine* e = new SelEngine(); SelSet S; S.minGradHistCut = 0.5f; S.minGradHistAdd = 3; S.gradDownweightPerLevel = 0.75f; S.selectDirectionDistribution = 1;
  S.outlierTH = 12*12; S.outlierTHSumComponent = 50*50; S.overallEnergyTHWeight = 1; e->init(w, h, S, rp, nullptr);
  e->walk_threads = 64;
  return e; }
void emu_gamma_engine_destroy(void* e) { ((SelEngine*)e)->destroy(); delete (SelEngine*)e; }
const char* emu_gamma_engine_error(void* e) { return ((SelEngine*)e)->err.c_str(); }
// gamma_w2 itself, for the rounding edges and the undefined conversions
float emu_gamma_w2(float I, const float* gw2) { return sdv::gamma_w2(I, gw2); }
int emu_gamma_make_hists(void* ep, const float* I0, int w, int h, const float* gw2, float* ths_out, float* thsSm_out) {
  SelEngine* e = (SelEngine*)ep; size_t tf = e->ths_floats(w, h); std::vector<float> a(tf, 0.f), b(tf, 0.f); HistJob J{I0, a.data(), b.data(), w, h, gw2};
  int rc = e->make_hists(1, &J); int n = (w/32)*(h/32); memcpy(ths_out, a.data(), n*4); memcpy(thsSm_out, b.data(), n*4); return rc; }
// one job per frame, all LiDAR (cloud3[j], n[j]) or all dense (cloud3 == nullptr); gw2[j]: job j's table or NULL; maps_out: the jobs' maps back to back
int emu_gamma_make_maps(void* ep, int nj, const float* const* I0, const float4* const* L1, const float4* const* L2, const float* const* gw2, const int* w, const int* h,
                        const double* const* cloud3, const int* n, const float* density, const int* rec, const float* thFactor, int* pot_io, unsigned char* maps_out, int* numHaveSub) {
  SelEngine* e = (SelEngine*)ep; const bool lidar = cloud3 != nullptr; std::vector<std::vector<float>> th(nj); std::vector<HistJob> H(nj); std::vector<MapsJobHost> M(nj); size_t o = 0;
  for (int j = 0; j < nj; j++) { const size_t tf = e->ths_floats(w[j], h[j]); th[j].assign(2*tf, 0.f); H[j] = HistJob{I0[j], th[j].data(), th[j].data() + tf, w[j], h[j], gw2[j]};
    M[j].img = FrameImg{I0[j], L1[j], L2[j]}; M[j].gw2 = gw2[j]; M[j].w = w[j]; M[j].h = h[j]; M[j].thsSm = th[j].data() + tf; M[j].cloud_dev = lidar ? cloud3[j] : nullptr;
    M[j].n = lidar ? n[j] : 0; M[j].map = maps_out + o; M[j].density = density[j]; M[j].recursionsLeft = rec[j]; M[j].thFactor = thFactor[j]; M[j].currentPotential = pot_io + j;
    M[j].numHaveSub = 0; M[j].passes = 0;
    o += lidar ? (size_t)std::max(n[j], 1) : (size_t)w[j]*h[j]; }
  if (e->make_hists(nj, H.data())) return -1;
  int rc = e->make_maps(M, lidar);
  for (int j = 0; j < nj; j++) numHaveSub[j] = M[j].numHaveSub;
  return rc;
}
int emu_gamma_make_new_traces(void* ep, int nj, void** slots, const float* const* I0, const float4* const* L1, const float4* const* L2, const float* const* gw2, const int* w, const int* h,
                              const double* const* cloud3, const int* n, const float* densL, const float* densD, const int* add, void* out, void* imm, int cap, int* n_out, int* numPoints2) {
  SelEngine* e = (SelEngine*)ep; std::vector<SelEngine::NewTracesJob> J(nj);
  for (int j = 0; j < nj; j++) { J[j].img = FrameImg{I0[j], L1[j], L2[j]}; J[j].gw2 = gw2[j]; J[j].w = w[j]; J[j].h = h[j]; J[j].cloud_host = cloud3[j]; J[j].n = n[j]; J[j].slot = (SelectorSlot*)slots[j];
    J[j].densityLidar = densL[j]; J[j].densityDense = densD[j]; J[j].addFeaturePoint = add[j]; J[j].out_host = (NewTrace*)out + (size_t)j*cap; J[j].imm_host = (ImmPt*)imm + (size_t)j*cap; J[j].cap = cap; }
  int rc = e->make_new_traces(J);
  for (int j = 0; j < nj; j++) { n_out[j] = J[j].n_out; numPoints2[2*j] = J[j].numPoints[0]; numPoints2[2*j+1] = J[j].numPoints[1]; }
  return rc;
}
}
