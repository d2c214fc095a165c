// lidar_emu_rows.cpp — TEST INFRASTRUCTURE: the LiDAR front-end of sdv-loam_b200/csrc/sdv_lidar_core.cuh compiled for the host (tests/emu/cuda_emu.hpp), driven through its
// device-output path (LidarEngine::handle_rows: rows into row-set blocks, the running pixel box read from and written back to "device" memory, a header per sweep),
// for tests/test_lidar_emu_rows_cpu.py.  "Device" pointers are host pointers here.
#define SDV_EMU 1
#define SDV_EMU_IMPL 1
#include "cuda_emu.hpp"
#include "../../sdv-loam_b200/csrc/sdv_lidar_core.cuh"
using sdv::lidar::LidarEngine;

extern "C" {
void* emu_rows_create(int n_scan, int horizon, float ang_res_x, float ang_res_y, float ang_bottom, int groundScanInd) {
  LidarEngine* e = new LidarEngine(); e->init(n_scan, horizon, ang_res_x, ang_res_y, ang_bottom, groundScanInd, nullptr); return e; }
void emu_rows_destroy(void* e) { ((LidarEngine*)e)->destroy(); delete (LidarEngine*)e; }
const char* emu_rows_error(void* e) { return ((LidarEngine*)e)->err.c_str(); }
int emu_rows_header_bytes() { return (int)sizeof(sdv::lidar::RowsHdr); }
// nj sweeps in one call, shared extrinsics / intrinsics / image size.  boxes: nj x 4 ints (each sweep's slot box, read and updated); blocks: sweep j's rows at
// blocks + j*block_stride doubles (room for cap rows); hdrs: nj headers; stats5: NULL (no wait) or nj x 5
int emu_rows_handle(void* ep, int nj, const float* const* xyzi, const int* n, const double* R9, const double* t3, const float* K4, int w, int h, int* boxes, double* blocks,
                    long long block_stride, void* hdrs, int cap, int* stats5) {
  LidarEngine* e = (LidarEngine*)ep; std::vector<LidarEngine::Sweep> S(nj);
  for (int j = 0; j < nj; j++) { LidarEngine::Sweep& s = S[j]; s.xyzi_host = xyzi[j]; s.n = n[j]; for (int k = 0; k < 9; k++) s.R[k] = R9[k]; for (int k = 0; k < 3; k++) s.t[k] = t3[k];
    for (int k = 0; k < 4; k++) s.K[k] = K4[k];
    s.w = w; s.h = h; s.cap = cap; s.out3_host = nullptr; s.box_dev = boxes + 4*j; s.hdr_dev = (sdv::lidar::RowsHdr*)hdrs + j; s.out3_dev = blocks + (size_t)j*block_stride; }
  return e->handle_rows(S, stats5);
}
}
