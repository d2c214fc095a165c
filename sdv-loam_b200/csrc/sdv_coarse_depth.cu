// sdv_coarse_depth.cu — CoarseTracker::makeCoarseDepthL0 (CoarseTracker.cpp:258-425) for a batch of tracker slots: sdv_tracker_set_ref_batch,
// sdv_tracker_set_ref (one job) and the initialiser's reference install.  Every job has the size and depth of its slot's camera; jobs of different
// cameras share the launches.  DESIGN.md Round 13 gives the order argument and the chunk budget.
#include "sdv_ctx.cuh"
#include <cub/device/device_radix_sort.cuh>
#include <cub/device/device_scan.cuh>
#include <algorithm>

namespace sdv {

// one job of a chunk.  Its planes are float2 {idepth, weightSums} cells at plane + off[l]; level 0 of every job of the chunk comes first, so one memset
// clears it.  Its rows are rows[row_begin, row_begin + n) of the chunk, its tiles of 1024 cells tile_begin[l] .. tile_begin[l+1] at level l
// (tile_begin[l] = the job's end for l >= L).
struct CdJob {
  const float* img[kLevels]; float4* out[kLevels]; long long off[kLevels]; int cap[kLevels]; int tile_begin[kLevels + 1];
  int w, h, L, row_begin, n, out_index;
};

constexpr int kCdThreads = 256, kCdItems = 4, kCdTile = kCdThreads*kCdItems;   // 1024 cells per tile, contiguous per thread
// bytes of {idepth, weightSums} planes one chunk may hold: at most 8 bytes x 1.33 x w x h per job (KITTI 1200x360: 4.6 MB, ~110 jobs per chunk)
constexpr size_t kCdPlaneBudget = size_t(512) << 20;

// the last job k of nj with begin(k) <= x: the owner of row / tile x (a job without rows or tiles has the begin of the next one)
template <class Begin> __device__ __forceinline__ int cd_owner(int nj, int x, Begin begin) {
  int lo = 0, hi = nj - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (begin(mid) <= x) lo = mid; else hi = mid - 1; }
  return lo;
}

// (a) one splat row: its cell (the job's level-0 plane offset + u + w*v) and its terms new_idepth*weight, weight (:264-294).  The product is rounded
//     on its own, as the reference's `idepth += new_idepth*weight` without FMA.
__global__ void cd_prep_kernel(const CdJob* __restrict__ J, int nj, const float* __restrict__ pts4, const int* __restrict__ round_half, int nrows,
                               unsigned* __restrict__ key, int* __restrict__ row, float2* __restrict__ term) {
  const int r = blockIdx.x*blockDim.x + threadIdx.x; if (r >= nrows) return;
  const CdJob& q = J[cd_owner(nj, r, [&](int k) { return J[k].row_begin; })];
  const float pu = pts4[4*r], pv = pts4[4*r+1], id = pts4[4*r+2], HdiF = pts4[4*r+3];
  const int u = round_half[r] ? (int)(pu + 0.5f) : (int)pu;
  const int v = round_half[r] ? (int)(pv + 0.5f) : (int)pv;
  const float weight = sqrtf((float)(1e-3 / ((double)HdiF + 1e-12)));      // sqrtf(1e-3 / (HdiF+1e-12)): double division, float sqrt (:273)
  key[r] = (unsigned)(q.off[0] + u + q.w*v); row[r] = r; term[r] = make_float2(__fmul_rn(id, weight), weight);
}
// (b) after a stable sort by cell, the rows of one cell are a run in row order: its first element adds the run from the memset +0.0f, in that order
__global__ void cd_splat_kernel(const unsigned* __restrict__ key, const int* __restrict__ row, const float2* __restrict__ term, int nrows, float2* plane) {
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= nrows) return;
  const unsigned k = key[i]; if (i > 0 && key[i-1] == k) return;
  float id = 0.f, ws = 0.f;
  for (int m = i; m < nrows && key[m] == k; m++) { const float2 t = term[row[m]]; id = __fadd_rn(id, t.x); ws = __fadd_rn(ws, t.y); }
  plane[k] = make_float2(id, ws);
}
// (c) sum-pool level l of every job from its un-dilated level l-1 (:296-322); blockIdx.y = job
__global__ void cd_pool_kernel(const CdJob* __restrict__ J, float2* plane, int l) {
  const CdJob& q = J[blockIdx.y]; if (l >= q.L) return;
  const int wl = q.w >> l, hl = q.h >> l, wlm1 = q.w >> (l-1);
  const int idx = blockIdx.x*blockDim.x + threadIdx.x; if (idx >= wl*hl) return;
  const int y = idx / wl, x = idx - y*wl; const float2* s = plane + q.off[l-1] + 2*x + 2*y*wlm1;
  const float2 a = s[0], b = s[1], c = s[wlm1], d = s[wlm1+1];
  plane[q.off[l] + idx] = make_float2(__fadd_rn(__fadd_rn(__fadd_rn(a.x, b.x), c.x), d.x), __fadd_rn(__fadd_rn(__fadd_rn(a.y, b.y), c.y), d.y));
}
// (d) cell i of a w x h level after the 1-px dilation into empty cells (:324-375), from the un-dilated plane P: the dilation never feeds another
//     level, so the count and emit passes form it on the fly.  diag: the 4 diagonal neighbours (levels 0, 1), else the 4 axis neighbours.  The
//     reference updates idepth in place but only reads cells with weight > 0 and writes cells with weight <= 0, so reading the un-dilated plane is
//     equivalent.  It reads one element past either end of the plane for the first / last cell of its loop (i = w: i-1-w = -1; i = n-w-1:
//     i+1+w = n), undefined there; here such a neighbour counts as empty.  Both cells lie in the 2 px border the cloud drops.
__device__ __forceinline__ float2 cd_dilated(const float2* __restrict__ P, int i, int w, int n, bool diag) {
  float2 c = P[i];
  if (i >= w && i < n - w && c.y <= 0) {
    const int o0 = diag ? 1+w : 1, o1 = diag ? -1-w : -1, o2 = diag ? w-1 : w, o3 = diag ? -w+1 : -w;
    float sum = 0, num = 0, numn = 0;
#define CD_NB(o) { const int j = i + (o); if (j >= 0 && j < n) { const float2 e = P[j]; if (e.y > 0) { sum += e.x; num += e.y; numn++; } } }
    CD_NB(o0) CD_NB(o1) CD_NB(o2) CD_NB(o3)
#undef CD_NB
    if (numn > 0) { c.x = sum/numn; c.y = num/numn; }
  }
  return c;
}
// (e) a cloud point (:377-423): outside the 2 px border, weight > 0, idepth/weight > 0 and a finite reference colour
__device__ __forceinline__ bool cd_valid(const float2* __restrict__ P, const float* __restrict__ ref, int i, int w, int h, bool diag, float& idn, float& col) {
  const int y = i / w, x = i - y*w;
  if (x < 2 || x >= w-2 || y < 2 || y >= h-2) return false;
  const float2 c = cd_dilated(P, i, w, w*h, diag);
  if (!(c.y > 0)) return false;
  idn = c.x / c.y; col = ref[i];
  return isfinite(col) && (idn > 0);
}
// the (job, level) of tile t and its first cell
__device__ __forceinline__ const CdJob& cd_tile(const CdJob* __restrict__ J, int nj, int t, int& l, int& base) {
  const CdJob& q = J[cd_owner(nj, t, [&](int k) { return J[k].tile_begin[0]; })];
  l = 0; while (l + 1 < q.L && q.tile_begin[l+1] <= t) l++;
  base = (t - q.tile_begin[l])*kCdTile + threadIdx.x*kCdItems;
  return q;
}
// (f) raster compaction of every (job, level) segment: tile counts -> one exclusive scan over the chunk -> emit at the offset within the segment
__global__ void __launch_bounds__(kCdThreads) cd_count_kernel(const CdJob* __restrict__ J, int nj, const float2* __restrict__ plane, int ntiles, int* tileCounts) {
  __shared__ int s[kCdThreads/32];
  int l, base; const CdJob& q = cd_tile(J, nj, blockIdx.x, l, base);
  const int w = q.w >> l, h = q.h >> l, n = w*h; const float2* P = plane + q.off[l]; int c = 0;
  for (int j = 0; j < kCdItems; j++) { const int i = base + j; float a, b; if (i < n && cd_valid(P, q.img[l], i, w, h, l < 2, a, b)) c++; }
  for (int o = 16; o > 0; o >>= 1) c += __shfl_xor_sync(0xffffffffu, c, o);
  if ((threadIdx.x & 31) == 0) s[threadIdx.x >> 5] = c;
  __syncthreads();
  if (threadIdx.x == 0) { int t = 0; for (int k = 0; k < kCdThreads/32; k++) t += s[k]; tileCounts[blockIdx.x] = t; if (blockIdx.x == 0) tileCounts[ntiles] = 0; }
}
// totals[out_index*SDV_PYR_LEVELS + l] = the true cloud size; nothing is written past cap[l] (the host compares the totals with the capacities)
__global__ void __launch_bounds__(kCdThreads) cd_emit_kernel(const CdJob* __restrict__ J, int nj, const float2* __restrict__ plane, const int* __restrict__ tileOffsets, int* totals) {
  __shared__ int s[kCdThreads/32];
  int l, base; const CdJob& q = cd_tile(J, nj, blockIdx.x, l, base);
  const int w = q.w >> l, h = q.h >> l, n = w*h; const float2* P = plane + q.off[l];
  const int seg0 = tileOffsets[q.tile_begin[l]];
  if (threadIdx.x == 0 && (int)blockIdx.x == q.tile_begin[l]) totals[q.out_index*SDV_PYR_LEVELS + l] = tileOffsets[q.tile_begin[l+1]] - seg0;
  float idn[kCdItems], col[kCdItems]; bool ok[kCdItems]; int c = 0;
  for (int j = 0; j < kCdItems; j++) { const int i = base + j; ok[j] = (i < n) && cd_valid(P, q.img[l], i, w, h, l < 2, idn[j], col[j]); c += ok[j]; }
  const int lane = threadIdx.x & 31, warp = threadIdx.x >> 5; int incl = c;
  for (int o = 1; o < 32; o <<= 1) { const int t = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += t; }
  if (lane == 31) s[warp] = incl;
  __syncthreads();
  int woff = 0; for (int k = 0; k < warp; k++) woff += s[k];
  int pos = tileOffsets[blockIdx.x] - seg0 + woff + incl - c;
  float4* out = q.out[l]; const int cap = q.cap[l];
  for (int j = 0; j < kCdItems; j++) if (ok[j]) { const int i = base + j; const int y = i / w, x = i - y*w; if (pos < cap) out[pos] = make_float4((float)x, (float)y, idn[j], col[j]); pos++; }
}

namespace {
struct CdChunk { int j0, j1, rows, tiles, maxL; long long cells, cells0; int maxpix[kLevels]; };
}

int set_ref_build(sdv_ctx* c, int nj, const int32_t* slots, FrameDev* const* F, const uint64_t* ref_frames, const int32_t* pt_begin, const float* pts4,
                  const int32_t* round_half, cudaMemcpyKind kind, const double* ref_ab, int32_t* npts_out, int* launches) {
  const char* who = "sdv_tracker_set_ref_batch";
  // chunks: consecutive jobs whose planes fit kCdPlaneBudget (a chunk holds at least one job); the sort keys are 32-bit plane offsets
  std::vector<CdChunk> ch; std::vector<CdJob> H(nj);
  for (int j = 0; j < nj; j++) {
    const int cam = c->slots[slots[j]].cam, w = c->cam_w[cam], h = c->cam_h[cam], L = c->cam_levels[cam];
    long long cells = 0; int tiles = 0; for (int l = 0; l < L; l++) { const int px = (w>>l)*(h>>l); cells += px; tiles += (px + kCdTile - 1)/kCdTile; }
    if (ch.empty() || ch.back().j1 - ch.back().j0 >= 65535 || (size_t)(ch.back().cells + cells)*sizeof(float2) > kCdPlaneBudget)
      ch.push_back(CdChunk{j, j, 0, 0, 1, 0, 0, {0}});
    CdChunk& k = ch.back(); k.j1 = j + 1; k.rows += pt_begin[j+1] - pt_begin[j]; k.tiles += tiles; k.cells += cells; k.cells0 += (long long)w*h; k.maxL = std::max(k.maxL, L);
    for (int l = 0; l < L; l++) k.maxpix[l] = std::max(k.maxpix[l], (w>>l)*(h>>l));
    if (k.cells >= (1ll << 32)) return ctx_fail(c, SDV_ERR_ARG, "%s: job %d's planes (%lld cells) exceed 32-bit offsets", who, j, k.cells);
  }
  int max_rows = 1, max_tiles = 1; long long max_cells = 1;
  for (const CdChunk& k : ch) { max_rows = std::max(max_rows, k.rows); max_tiles = std::max(max_tiles, k.tiles); max_cells = std::max(max_cells, k.cells); }
  size_t sort_tmp = 0, scan_tmp = 0;
  CK(cub::DeviceRadixSort::SortPairs(nullptr, sort_tmp, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, max_rows, 0, 32, c->st));
  CK(cub::DeviceScan::ExclusiveSum(nullptr, scan_tmp, (const int*)nullptr, (int*)nullptr, max_tiles + 1, c->st));
  const size_t nrows = (size_t)pt_begin[nj];
  const size_t dev_bytes = Scratch::need(4*std::max(nrows, (size_t)1), 4) + Scratch::need(std::max(nrows, (size_t)1), 4) + Scratch::need(nj, sizeof(CdJob))
                         + Scratch::need((size_t)nj*SDV_PYR_LEVELS, 4) + Scratch::need(max_cells, sizeof(float2)) + 4*Scratch::need(max_rows, 4)
                         + Scratch::need(max_rows, sizeof(float2)) + 2*Scratch::need(max_tiles + 1, 4) + Scratch::need(std::max(sort_tmp, scan_tmp), 1);
  const size_t host_bytes = Scratch::need(nj, sizeof(CdJob)) + Scratch::need((size_t)nj*SDV_PYR_LEVELS, 4);
  if (c->scr.reserve(dev_bytes, c->st) || c->scr_host.reserve(host_bytes, c->st)) return ctx_fail(c, SDV_ERR_CUDA, "%s: scratch of %d jobs, %zu rows", who, nj, nrows);
  Scratch& S = c->scr; S.reset(); c->scr_host.reset();
  float* rows4 = S.take<float>(4*std::max(nrows, (size_t)1)); int* rows_rh = S.take<int>(std::max(nrows, (size_t)1));
  CdJob* Jd = S.take<CdJob>(nj); int* totals = S.take<int>((size_t)nj*SDV_PYR_LEVELS);
  float2* plane = S.take<float2>(max_cells); unsigned* key_in = S.take<unsigned>(max_rows); unsigned* key = S.take<unsigned>(max_rows);
  int* row_in = S.take<int>(max_rows); int* row = S.take<int>(max_rows); float2* term = S.take<float2>(max_rows);
  int* tileCounts = S.take<int>(max_tiles + 1); int* tileOffsets = S.take<int>(max_tiles + 1); void* tmp = S.take<char>(std::max(sort_tmp, scan_tmp));
  CdJob* Jh = c->scr_host.take<CdJob>(nj); int* totals_h = c->scr_host.take<int>((size_t)nj*SDV_PYR_LEVELS);
  for (const CdChunk& k : ch) {                                        // descriptors of every chunk, uploaded once
    long long off0 = 0, offl = k.cells0; int tile = 0;
    for (int j = k.j0; j < k.j1; j++) {
      const TrackerSlot& t = c->slots[slots[j]]; const int cam = t.cam; CdJob& q = Jh[j]; memset(&q, 0, sizeof(q));
      q.w = c->cam_w[cam]; q.h = c->cam_h[cam]; q.L = c->cam_levels[cam]; q.row_begin = pt_begin[j] - pt_begin[k.j0]; q.n = pt_begin[j+1] - pt_begin[j]; q.out_index = j;
      for (int l = 0; l < q.L; l++) {
        const int px = (q.w>>l)*(q.h>>l);
        q.img[l] = F[j]->img[l]; q.out[l] = t.pts[l]; q.cap[l] = t.cap[l];
        if (l == 0) { q.off[0] = off0; off0 += px; } else { q.off[l] = offl; offl += px; }
        q.tile_begin[l] = tile; tile += (px + kCdTile - 1)/kCdTile;
      }
      for (int l = q.L; l <= kLevels; l++) q.tile_begin[l] = tile;
    }
  }
  { int rcj = join_ingest(c); if (rcj) return rcj; }
  if (nrows) {
    CK(cudaMemcpyAsync(rows4, pts4, 4*nrows*sizeof(float), kind, c->st));
    CK(cudaMemcpyAsync(rows_rh, round_half, nrows*sizeof(int), kind, c->st));
  }
  CK(cudaMemcpyAsync(Jd, Jh, (size_t)nj*sizeof(CdJob), cudaMemcpyHostToDevice, c->st));
  CK(cudaMemsetAsync(totals, 0, (size_t)nj*SDV_PYR_LEVELS*sizeof(int), c->st));        // levels past a camera's depth stay 0
  int nl = 0;
  for (const CdChunk& k : ch) {
    const CdJob* J = Jd + k.j0; const int n = k.j1 - k.j0, r0 = pt_begin[k.j0];
    CK(cudaMemsetAsync(plane, 0, (size_t)k.cells0*sizeof(float2), c->st));           // the pool writes every cell of levels >= 1
    if (k.rows) {
      cd_prep_kernel<<<(k.rows + 255)/256, 256, 0, c->st>>>(J, n, rows4 + 4*(size_t)r0, rows_rh + r0, k.rows, key_in, row_in, term);
      size_t tb = sort_tmp;
      CK(cub::DeviceRadixSort::SortPairs(tmp, tb, key_in, key, row_in, row, k.rows, 0, 32, c->st));   // stable: equal cells keep row order
      cd_splat_kernel<<<(k.rows + 255)/256, 256, 0, c->st>>>(key, row, term, k.rows, plane);
      nl += 3;
    }
    for (int l = 1; l < k.maxL; l++) cd_pool_kernel<<<dim3((k.maxpix[l] + 255)/256, n), 256, 0, c->st>>>(J, plane, l);
    cd_count_kernel<<<k.tiles, kCdThreads, 0, c->st>>>(J, n, plane, k.tiles, tileCounts);
    size_t sb = scan_tmp;
    CK(cub::DeviceScan::ExclusiveSum(tmp, sb, tileCounts, tileOffsets, k.tiles + 1, c->st));
    cd_emit_kernel<<<k.tiles, kCdThreads, 0, c->st>>>(J, n, plane, tileOffsets, totals);
    nl += k.maxL - 1 + 3;
  }
  CK(cudaGetLastError());
  CK(cudaMemcpyAsync(totals_h, totals, (size_t)nj*SDV_PYR_LEVELS*sizeof(int), cudaMemcpyDeviceToHost, c->st));
  CK(cudaStreamSynchronize(c->st));
  if (launches) *launches += nl;
  int over = -1, over_l = 0;
  for (int j = 0; j < nj; j++) {
    TrackerSlot& t = c->slots[slots[j]]; const int* T = totals_h + (size_t)j*SDV_PYR_LEVELS; const int L = c->cam_levels[t.cam]; int bad = -1;
    if (npts_out) for (int l = 0; l < SDV_PYR_LEVELS; l++) npts_out[(size_t)j*SDV_PYR_LEVELS + l] = T[l];
    for (int l = 0; l < L && bad < 0; l++) if (T[l] > t.cap[l]) bad = l;
    if (bad >= 0) {                    // the emit never wrote past cap[l], but the slot's clouds are a truncated mix now: it has no reference
      t.ref_frame = ~0ull; t.has_totals = false; for (int l = 0; l < c->levels; l++) t.npts[l] = 0;
      if (over < 0) { over = j; over_l = bad; }
      continue;
    }
    for (int l = 0; l < c->levels; l++) t.npts[l] = l < L ? T[l] : 0;                     // levels past the camera's depth are never read
    t.ref_frame = ref_frames[j]; t.ref_a = ref_ab ? ref_ab[2*j] : 0.0; t.ref_b = ref_ab ? ref_ab[2*j+1] : 0.0; t.refExposure = F[j]->exposure; t.has_totals = false;
  }
  if (over >= 0) {
    const TrackerSlot& t = c->slots[slots[over]];
    return ctx_fail(c, SDV_ERR_CAPACITY, "%s: job %d: level %d cloud (%d) exceeds capacity %d (max_ref_points); slot %d has no reference now", who, over, over_l,
                    totals_h[(size_t)over*SDV_PYR_LEVELS + over_l], t.cap[over_l], slots[over]);
  }
  return SDV_OK;
}

}  // namespace sdv
