// sdv_lidar.cu — C-ABI of the LiDAR front-end (SURVEY.md §8f rank 3, second half): the node's lidarCloudHandler (src/main.cpp:785-858 -> projectPointCloud :563-607,
// groundRemoval :609-655, cloudSegmentation :657-783, pixel projection :806-849) for a batch of raw sweeps, one per resident sequence.  Kernels + host engine live in
// sdv_lidar_core.cuh (which the CPU suite also compiles for the host, tests/emu); this file binds them to the context and its tracker-domain stream.
// Row sets (sdv_lidar_handler_rows_batch, sdv_lidar_rows_*): FullSystem::qCloudPixel kept on the device, one block per frame handle, so that the rows go from the
// handler to makeNewTraces (sdv_make_new_traces_rows_store_batch) without a host round trip.
#include <cuda_runtime.h>
#include <stdint.h>
#include <vector>
#include "sdv_ctx.cuh"
#include "sdv_pool.cuh"
#include "sdv_lidar_core.cuh"

using namespace sdv;

namespace sdv {
struct LidarState { lidar::LidarEngine eng; };
void lidar_destroy(sdv_ctx* c) { LidarState* s = (LidarState*)c->lidar; if (!s) return; s->eng.destroy(); delete s; c->lidar = nullptr; }

// ---- row sets: one block per frame handle = header (lidar::RowsHdr, 64 B) | room for `cap` rows {Ku, Kv, depth}.  Block::n = the room the last deposit asked for.
struct RowBlock {
  char* p = nullptr; int n = 0, cap = 0;
  char* base() const { return p; }
  lidar::RowsHdr* hdr() const { return (lidar::RowsHdr*)p; }
  double* rows() const { return (double*)(p + sizeof(lidar::RowsHdr)); }
  static size_t bytes(int cap) { return sizeof(lidar::RowsHdr) + 3*(size_t)cap*sizeof(double); }
  static RowBlock layout(char* p, int cap) { RowBlock b; b.p = p; b.cap = cap; return b; }
};
static_assert(sizeof(lidar::RowsHdr) == 64, "row-set header");
struct RowStore : BlockPool<RowBlock> {};
static RowStore* rows_store(sdv_ctx* c) { if (!c->lidar_rows) c->lidar_rows = new RowStore(); return (RowStore*)c->lidar_rows; }
void lidar_rows_destroy(sdv_ctx* c) { RowStore* R = (RowStore*)c->lidar_rows; if (!R) return; R->release(); delete R; c->lidar_rows = nullptr; }
__global__ void __launch_bounds__(128) lf_rows_hdr_gather_kernel(const lidar::RowsHdr* const* __restrict__ src, int n, lidar::RowsHdr* __restrict__ dst) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i < n) dst[i] = *src[i];
}
int lidar_rows_fetch(sdv_ctx* c, int n, const uint64_t* frames, const double** rows_dev, LidarRowsInfo* info, const char* who) {
  RowStore* R = (RowStore*)c->lidar_rows; std::vector<const lidar::RowsHdr*> src(n);
  for (int j = 0; j < n; j++) { auto it = R ? R->blocks.find(frames[j]) : decltype(R->blocks.end())();
    if (!R || it == R->blocks.end()) return ctx_fail(c, SDV_ERR_NOFRAME, "%s: frame %llu has no LiDAR row set", who, (unsigned long long)frames[j]);
    src[j] = it->second.hdr(); rows_dev[j] = it->second.rows(); info[j].room = it->second.n; }
  if (n == 0) return SDV_OK;
  if (c->scr.reserve(Scratch::need(n, sizeof(void*)) + Scratch::need(n, sizeof(lidar::RowsHdr)), c->st)) return ctx_fail(c, SDV_ERR_CUDA, "%s: scratch", who);
  c->scr.reset(); const lidar::RowsHdr** dsrc = c->scr.take<const lidar::RowsHdr*>(n); lidar::RowsHdr* dh = c->scr.take<lidar::RowsHdr>(n); std::vector<lidar::RowsHdr> h(n);
  CK(cudaMemcpyAsync(dsrc, src.data(), n*sizeof(void*), cudaMemcpyHostToDevice, c->st));
  lf_rows_hdr_gather_kernel<<<(n + 127)/128, 128, 0, c->st>>>(dsrc, n, dh); c->launches += 1; CK(cudaGetLastError());
  CK(cudaMemcpyAsync(h.data(), dh, n*sizeof(lidar::RowsHdr), cudaMemcpyDeviceToHost, c->st)); CK(cudaStreamSynchronize(c->st));
  for (int j = 0; j < n; j++) { LidarRowsInfo& o = info[j]; const lidar::RowsHdr& q = h[j]; o.rows = q.rows; o.overflow = q.overflow;
    o.lrud[0] = q.left; o.lrud[1] = q.right; o.lrud[2] = q.up; o.lrud[3] = q.down; o.addFeaturePoint = q.addFeaturePoint; o.numGround = q.numGround; o.n_segmented = q.n_segmented; }
  return SDV_OK;
}
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
  { int rc = check_offsets(c, n, sweep_begin, "lidar_handler", "sweep_begin"); if (rc) return rc; }
  if (sweep_begin[n] > 0 && !xyzi) return SDV_ERR_ARG;
  { int rc = check_cams(c, n, cams, "lidar_handler", "sweep"); if (rc) return rc; }
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

int sdv_lidar_handler_rows_batch(sdv_ctx* c, int n, const int32_t* slots, const uint64_t* frames, const int32_t* sweep_begin, const float* xyzi, const double* Rlc9,
                                 const double* tlc3, const float* K4, int cap, int32_t* stats_out) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && (!slots || !frames || !sweep_begin || !Rlc9 || !tlc3 || !K4))) return SDV_ERR_ARG;
  if (n == 0) return SDV_OK;
  LidarState* s = (LidarState*)c->lidar; if (!s) return ctx_fail(c, SDV_ERR_STATE, "lidar_handler_rows: sdv_lidar_init has not been called");
  const int ns = sel_n_slots(c); if (ns < 0) return ctx_fail(c, SDV_ERR_STATE, "lidar_handler_rows: sdv_selector_init has not been called (the pixel box lives with the selector slot)");
  if (cap < 1) return ctx_fail(c, SDV_ERR_ARG, "lidar_handler_rows: cap %d (>= 1)", cap);
  { int rc = check_offsets(c, n, sweep_begin, "lidar_handler_rows", "sweep_begin"); if (rc) return rc; }
  if (sweep_begin[n] > 0 && !xyzi) return SDV_ERR_ARG;
  // a slot named twice would leave the order of its box updates ambiguous
  { int rc = check_ids(c, n, slots, ns, "lidar_handler_rows", "selector slot"); if (rc) return rc; }
  { int rc = check_distinct(c, n, frames, "lidar_handler_rows", "frame"); if (rc) return rc; }
  CK(cudaSetDevice(c->device));
  RowStore* R = rows_store(c); std::vector<int> room(n, cap); std::vector<RowStore::Plan> P;
  { int rc = R->plan(c, n, frames, room.data(), P, "lidar row sets", "rows"); if (rc) return rc; }
  std::vector<lidar::LidarEngine::Sweep> S(n);
  for (int j = 0; j < n; j++) { auto& w = S[j]; w.xyzi_host = xyzi ? xyzi + 4*(size_t)sweep_begin[j] : nullptr; w.n = sweep_begin[j+1] - sweep_begin[j];
    for (int k = 0; k < 9; k++) w.R[k] = Rlc9[9*j+k]; for (int k = 0; k < 3; k++) w.t[k] = tlc3[3*j+k]; for (int k = 0; k < 4; k++) w.K[k] = K4[4*j+k];
    int cam = 0; sel_slot_box(c, slots[j], &cam, &w.box_dev); w.w = c->cam_w[cam]; w.h = c->cam_h[cam];
    w.hdr_dev = P[j].b.hdr(); w.out3_dev = P[j].b.rows(); w.cap = cap; w.out3_host = nullptr; }
  const long long l0 = s->eng.launches; s->eng.st_up = c->st_cp;
  if (s->eng.handle_rows(S, stats_out)) { R->abandon(P); return ctx_fail(c, SDV_ERR_CUDA, "lidar_handler_rows: %s", s->eng.err.c_str()); }
  R->commit(P);
  c->launches += s->eng.launches - l0;
  if (stats_out && s->eng.have_ev) c->last_ms = s->eng.last_kernel_ms;                   // sdv_last_kernel_ms: the nine kernels of the front-end (only when the call waited)
  return SDV_OK;
}
int sdv_lidar_rows_get(sdv_ctx* c, uint64_t frame, int cap, double* cloud3_out, int32_t* n_out, int32_t* lrud_out, int32_t* add_feature_point_out) { SDV_GUARD_TRK(c);
  if (!c || cap < 0) return SDV_ERR_ARG;
  CK(cudaSetDevice(c->device));
  const double* rows = nullptr; LidarRowsInfo I;
  { int rc = lidar_rows_fetch(c, 1, &frame, &rows, &I, "lidar_rows_get"); if (rc) return rc; }
  if (n_out) *n_out = I.rows;
  if (lrud_out) for (int k = 0; k < 4; k++) lrud_out[k] = I.lrud[k];
  if (add_feature_point_out) *add_feature_point_out = I.addFeaturePoint;
  if (I.overflow) return ctx_fail(c, SDV_ERR_CAPACITY, "lidar_rows_get: the sweep of frame %llu left %d pixel rows, its row set holds %d", (unsigned long long)frame, I.rows, I.room);
  if (!cloud3_out || I.rows == 0) return SDV_OK;
  if (cap < I.rows) return ctx_fail(c, SDV_ERR_CAPACITY, "lidar_rows_get: frame %llu holds %d rows, room for %d", (unsigned long long)frame, I.rows, cap);
  CK(cudaMemcpyAsync(cloud3_out, rows, 3*(size_t)I.rows*sizeof(double), cudaMemcpyDeviceToHost, c->st)); CK(cudaStreamSynchronize(c->st));
  return SDV_OK;
}
int sdv_lidar_rows_drop(sdv_ctx* c, int n, const uint64_t* frames) { SDV_GUARD_TRK(c);
  if (!c || n < 0 || (n && !frames)) return SDV_ERR_ARG;
  RowStore* R = (RowStore*)c->lidar_rows;
  for (int i = 0; i < n; i++) if (!R || !R->blocks.count(frames[i])) return ctx_fail(c, SDV_ERR_NOFRAME, "lidar_rows_drop: frame %llu has no LiDAR row set", (unsigned long long)frames[i]);
  for (int i = 0; i < n; i++) R->drop(frames[i]);                                         // a frame named twice is dropped once
  return SDV_OK;
}

}  // extern "C"
