// select_emu_mixed.cpp — TEST INFRASTRUCTURE: the candidate-management engine of sdv-loam_b200/csrc/sdv_select_core.cuh compiled for the host (tests/emu/cuda_emu.hpp),
// with entry points whose jobs carry their own frame sizes, for tests/test_select_emu_mixed_cpu.py.  "Device" pointers are host pointers here; selector slots are the
// SelectorSlot objects of tests/emu/select_emu.cpp (emu_slot_create), a plain struct both libraries share.
#define SDV_EMU 1
#define SDV_EMU_IMPL 1
#include "cuda_emu.hpp"
#include "../../sdv-loam_b200/csrc/sdv_select_core.cuh"
using namespace sdv::sel;

extern "C" {
void* emu_mixed_engine_create(int w, int h, const unsigned char* rp) {
  SelEngine* e = new SelEngine(); SelSet S; S.minGradHistCut = 0.5f; S.minGradHistAdd = 3; S.gradDownweightPerLevel = 0.75f; S.selectDirectionDistribution = 1;
  S.outlierTH = 12*12; S.outlierTHSumComponent = 50*50; S.overallEnergyTHWeight = 1; e->init(w, h, S, rp, nullptr);
  e->walk_threads = 64;                               // one OS thread per CUDA thread here: keep the emulated CTA small (the result does not depend on the CTA size)
  return e; }
void emu_mixed_engine_destroy(void* e) { ((SelEngine*)e)->destroy(); delete (SelEngine*)e; }
const char* emu_mixed_engine_error(void* e) { return ((SelEngine*)e)->err.c_str(); }
// ---- mixed sizes: every job carries its own frame size w[j] x h[j] (<= the engine's, whose pattern every job indexes by its prefix)
int emu_mixed_make_hists(void* ep, const float* I0, int w, int h, float* ths_out, float* thsSm_out) {
  SelEngine* e = (SelEngine*)ep; size_t tf = e->ths_floats(w, h); std::vector<float> a(tf, 0.f), b(tf, 0.f); HistJob J{I0, a.data(), b.data(), w, h};
  int rc = e->make_hists(1, &J); int n = (w/32)*(h/32); memcpy(ths_out, a.data(), n*4); memcpy(thsSm_out, b.data(), n*4); return rc; }
// one job per frame, all LiDAR (cloud3[j], n[j]) or all dense (cloud3 == nullptr); maps_out: the jobs' maps back to back (n[j] or w[j]*h[j] bytes)
int emu_mixed_make_maps(void* ep, int nj, const float* const* I0, const float4* const* L1, const float4* const* L2, const int* w, const int* h, const double* const* cloud3, const int* n,
                     const float* density, const int* rec, const float* thFactor, int* pot_io, unsigned char* maps_out, int* numHaveSub, int* passes) {
  SelEngine* e = (SelEngine*)ep; const bool lidar = cloud3 != nullptr; std::vector<std::vector<float>> th(nj); std::vector<HistJob> H(nj); std::vector<MapsJobHost> M(nj); size_t o = 0;
  for (int j = 0; j < nj; j++) { const size_t tf = e->ths_floats(w[j], h[j]); th[j].assign(2*tf, 0.f); H[j] = HistJob{I0[j], th[j].data(), th[j].data() + tf, w[j], h[j]};
    M[j].img = FrameImg{I0[j], L1[j], L2[j]}; M[j].w = w[j]; M[j].h = h[j]; M[j].thsSm = th[j].data() + tf; M[j].cloud_dev = lidar ? cloud3[j] : nullptr; M[j].n = lidar ? n[j] : 0; M[j].map = maps_out + o;
    M[j].density = density[j]; M[j].recursionsLeft = rec[j]; M[j].thFactor = thFactor[j]; M[j].currentPotential = pot_io + j; M[j].numHaveSub = 0; M[j].passes = 0;
    o += lidar ? (size_t)std::max(n[j], 1) : (size_t)w[j]*h[j]; }
  if (e->make_hists(nj, H.data())) return -1;
  int rc = e->make_maps(M, lidar);
  for (int j = 0; j < nj; j++) { numHaveSub[j] = M[j].numHaveSub; passes[j] = M[j].passes; }
  return rc;
}
int emu_mixed_make_new_traces(void* ep, int nj, void** slots, const float* const* I0, const float4* const* L1, const float4* const* L2, const int* w, const int* h, const double* const* cloud3, const int* n,
                           const float* densL, const float* densD, const int* add, void* out, void* imm, int cap, int* n_out, int* numPoints2, int* passes2) {
  SelEngine* e = (SelEngine*)ep; std::vector<SelEngine::NewTracesJob> J(nj);
  for (int j = 0; j < nj; j++) { J[j].img = FrameImg{I0[j], L1[j], L2[j]}; J[j].w = w[j]; J[j].h = h[j]; J[j].cloud_host = cloud3[j]; J[j].n = n[j]; J[j].slot = (SelectorSlot*)slots[j]; J[j].densityLidar = densL[j];
    J[j].densityDense = densD[j]; J[j].addFeaturePoint = add[j]; J[j].out_host = (NewTrace*)out + (size_t)j*cap; J[j].imm_host = (ImmPt*)imm + (size_t)j*cap; J[j].cap = cap; }
  int rc = e->make_new_traces(J);
  for (int j = 0; j < nj; j++) { n_out[j] = J[j].n_out; numPoints2[2*j] = J[j].numPoints[0]; numPoints2[2*j+1] = J[j].numPoints[1]; passes2[2*j] = J[j].passes[0]; passes2[2*j+1] = J[j].passes[1]; }
  return rc;
}
// nj sequences with the same sources and candidates, sequence j at image size w[j] x h[j] (its level-1 map (w[j]/2) x (h[j]/2)); map_out: the maps back to back
int emu_mixed_activate(void* ep, int nj, const int* w, const int* h, int nHosts, const int* pt_begin, const float* KRKi, const float* Kt, const float* uvid, int nCandHosts, const int* cand_begin,
                    const float* cKRKi, const float* cKt, const float* cand4, float minActDist, int* decision, float* map_out) {
  SelEngine* e = (SelEngine*)ep; std::vector<SelEngine::ActJob> J(nj); const int nc = nCandHosts ? cand_begin[nCandHosts] : 0; size_t o = 0;
  for (int j = 0; j < nj; j++) { J[j] = SelEngine::ActJob{nHosts, pt_begin, KRKi, Kt, uvid, nCandHosts, cand_begin, cKRKi, cKt, cand4, minActDist, decision ? decision + (size_t)j*nc : nullptr, map_out + o,
                                                          w[j] >> 1, h[j] >> 1};
    o += (size_t)(w[j] >> 1)*(h[j] >> 1); }
  return e->activate(J);
}
}
