// sdv_lidar.cu — C-ABI of the LiDAR front-end (SURVEY.md §8f rank 3, second half): the node's lidarCloudHandler (src/main.cpp:785-858 -> projectPointCloud :563-607,
// groundRemoval :609-655, cloudSegmentation :657-783, pixel projection :806-849) for a batch of raw sweeps, one per resident sequence.  Kernels + host engine live in
// sdv_lidar_core.cuh (which the CPU suite also compiles for the host, tests/emu); this file binds them to the context and its tracker-domain stream.
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "sdv_ctx.cuh"
#include "sdv_lidar_core.cuh"

using namespace sdv;
#define CK(call) do { cudaError_t e_ = (call); if (e_ != cudaSuccess) return ctx_fail(c, SDV_ERR_CUDA, "%s:%d %s -> %s", __FILE__, __LINE__, #call, cudaGetErrorString(e_)); } while (0)

namespace sdv {
struct LidarState { lidar::LidarEngine eng; };
void lidar_destroy(sdv_ctx* c) { LidarState* s = (LidarState*)c->lidar; if (!s) return; s->eng.destroy(); delete s; c->lidar = nullptr; }
}

extern "C" {

int sdv_lidar_init(sdv_ctx* c, int n_scan, int horizon_scan, float ang_res_x, float ang_res_y, float ang_bottom, int ground_scan_ind) { SDV_GUARD_TRK(c);
  if (!c) return SDV_ERR_ARG;
  if (n_scan < 2 || n_scan > 128 || horizon_scan < 2 || horizon_scan > 65536 || !(ang_res_x > 0) || !(ang_res_y > 0) || ground_scan_ind < 0 || ground_scan_ind >= n_scan)
    return ctx_fail(c, SDV_ERR_ARG, "lidar_init: rings 2..128, azimuth bins 2..65536, positive resolutions, groundScanInd < rings");
  CK(cudaSetDevice(c->device));
  lidar_destroy(c);
  LidarState* s = new LidarState(); c->lidar = s; s->eng.init(n_scan, horizon_scan, ang_res_x, ang_res_y, ang_bottom, ground_scan_ind, c->st);
  return SDV_OK;
}

int sdv_lidar_handler_batch_cams(sdv_ctx* c, int n, const int32_t* sweep_begin, const float* xyzi, const double* Rlc9, const double* tlc3, const float* K4, const int32_t* cams,
                                 int32_t* lrud_io, int cap, double* cloud3_out, int32_t* n_out, int32_t* add_feature_point_out, int32_t* stats_out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!sweep_begin || !Rlc9 || !tlc3 || !K4 || !lrud_io || !cloud3_out || !n_out || cap < 1))) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK;
  LidarState* s = (LidarState*)c->lidar; if (!s) return ctx_fail(c, SDV_ERR_STATE, "lidar_handler: sdv_lidar_init has not been called");
  if (sweep_begin[0] != 0) return ctx_fail(c, SDV_ERR_ARG, "lidar_handler: sweep_begin[0] must be 0");
  for (int j = 0; j < n; j++) { if (sweep_begin[j+1] < sweep_begin[j]) return ctx_fail(c, SDV_ERR_ARG, "lidar_handler: sweep_begin is not ascending at sweep %d", j);
    if (sweep_begin[j+1] > sweep_begin[j] && !xyzi) return SDV_ERR_ARG;
    if (cams && (cams[j] < 0 || cams[j] >= SDV_MAX_CAMERAS)) return ctx_fail(c, SDV_ERR_ARG, "lidar_handler: sweep %d names camera %d (valid: 0..%d)", j, cams[j], SDV_MAX_CAMERAS - 1); }
  CK(cudaSetDevice(c->device));
  std::vector<lidar::LidarEngine::Sweep> S(n);
  for (int j = 0; j < n; j++) { auto& w = S[j]; w.xyzi_host = xyzi ? xyzi + 4*(size_t)sweep_begin[j] : nullptr; w.n = sweep_begin[j+1] - sweep_begin[j];
    for (int k = 0; k < 9; k++) w.R[k] = Rlc9[9*j+k]; for (int k = 0; k < 3; k++) w.t[k] = tlc3[3*j+k]; for (int k = 0; k < 4; k++) { w.K[k] = K4[4*j+k]; w.lrud[k] = lrud_io[4*j+k]; }
    const int cam = cams ? cams[j] : 0; w.w = c->cam_w[cam]; w.h = c->cam_h[cam]; w.out3_host = cloud3_out + 3*(size_t)j*cap; w.cap = cap; }
  const long long l0 = s->eng.launches;
  CK(cudaEventRecord(c->ev0, c->st));
  { int rc = s->eng.handle(S); if (rc) return ctx_fail(c, rc == -2 ? SDV_ERR_CAPACITY : SDV_ERR_CUDA, "lidar_handler: %s", s->eng.err.c_str()); }
  CK(cudaEventRecord(c->ev1, c->st)); CK(cudaStreamSynchronize(c->st)); CK(cudaEventElapsedTime(&c->last_ms, c->ev0, c->ev1));
  if (s->eng.have_ev) c->last_ms = s->eng.last_kernel_ms;                                  // sdv_last_kernel_ms: the nine kernels of the front-end, copies excluded
  c->launches += s->eng.launches - l0;
  for (int j = 0; j < n; j++) { n_out[j] = S[j].n_out; for (int k = 0; k < 4; k++) lrud_io[4*j+k] = S[j].lrud[k]; if (add_feature_point_out) add_feature_point_out[j] = S[j].addFeaturePoint;
    if (stats_out) { stats_out[2*j] = S[j].numGround; stats_out[2*j+1] = S[j].n_segmented; } }
  return SDV_OK;
}
int sdv_lidar_handler_batch(sdv_ctx* c, int n, const int32_t* sweep_begin, const float* xyzi, const double* Rlc9, const double* tlc3, const float* K4, int32_t* lrud_io, int cap,
                            double* cloud3_out, int32_t* n_out, int32_t* add_feature_point_out, int32_t* stats_out) {
  return sdv_lidar_handler_batch_cams(c, n, sweep_begin, xyzi, Rlc9, tlc3, K4, nullptr, lrud_io, cap, cloud3_out, n_out, add_feature_point_out, stats_out);
}

}  // extern "C"
