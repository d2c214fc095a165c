// sdv_select_core.cuh — candidate management at keyframe rate on the device (SURVEY.md §8f rank 4 and the caller half of rank 2):
//
//   PixelSelector::makeHists                    /root/reference/src/FullSystem/PixelSelector2.cpp:47-106    -> sel_hist_kernel, sel_smooth_kernel
//   PixelSelector::selectFromLidar / select     PixelSelector2.cpp:451-622 / :202-352                       -> sel_point_kernel, sel_scatter_kernel, sel_cell_kernel, sel_n2_kernel, sel_block_kernel
//   PixelSelector::makeMapsFromLidar / makeMaps PixelSelector2.cpp:354-449 / :108-200                       -> host loop of SelEngine::make_maps + sel_sub_*_kernel
//   FullSystem::shiTomasiScore, makeNewTraces   FullSystem/FullSystem.cpp:1540-1583, 1261-1356              -> nt_* kernels
//   CoarseDistanceMap::makeDistanceMap / growDistBFS / addIntoDistFinal   FullSystem/CoarseTracker.cpp:1139-1282   -> dm_* kernels
//   candidate walk of FullSystem::activatePointsMT                        FullSystem/FullSystem.cpp:600-671        -> act_project_kernel, act_walk_kernel
//
// The selector is a scan over the image whose only cross-cell coupling is the running count n2 of level-2 picks: it indexes the random direction table, so the
// direction a cell is judged with depends on how many cells before it produced a pick.  On the device that chain is cut like this: (1) every pot x pot cell
// evaluates, for all 16 directions, whether it WOULD produce a pick (16-bit mask, exact incl. the reference's `bestIdx > 0` quirk); (2) one CTA walks the cells in the
// reference's visiting order and resolves n2 — a plain prefix sum wherever the masks are all-ones / all-zeros, a sequential table walk only through cells whose
// answer depends on the direction; (3) one thread per 4x4-cell block replays the reference's three-level state machine with the now-known directions.
// The distance map is a multi-source BFS with alternating 4/8-connectivity (39 rings): pull sweeps for makeDistanceMap, a frontier BFS with atomicMin claims for the
// single-source updates of the greedy activation walk, which stays sequential per sequence (one CTA each) and parallel over sequences.
// Everything is integer / short float expressions in the reference's operation order (--fmad=false): results are bit-identical to the CPU code.
//
// This header holds the kernels AND the host engine, and depends on nothing but the CUDA runtime: the build container has no GPU, so tests/emu/ compiles this very file
// for the host against a small CUDA emulation (tests/emu/cuda_emu.hpp) and checks it against the oracle (tests/test_select_emu_cpu.py); sdv_select.cu compiles it
// with nvcc and binds it to the context (frames, streams) behind the C-ABI.
#pragma once
#include "sdv_core_common.cuh"

namespace sdv { namespace sel {

struct FrameImg { const float* I0; const float4* L1; const float4* L2; };              // level-0 plane, packed {I,dx,dy,|grad|^2} texels of levels 1 and 2
struct SelSet { float minGradHistCut, minGradHistAdd, gradDownweightPerLevel; int selectDirectionDistribution;     // util/settings.cpp:119-122
                float outlierTH, outlierTHSumComponent, overallEnergyTHWeight; };                                   // :64-65, :111 (ImmaturePoint constructor)
struct PtRec { float dx, dy, ag0, ag1, ag2, th0; int valid, out; };                     // what the three tests of a candidate need; out = index written into the map
struct NewTrace { float u, v, my_type, score, idepth_fromSensor; int32_t isFromSensor, type; };   // = sdv_new_trace (include/sdv_b200.h)
struct ImmPt { float u, v, idepth_min, idepth_max, color[8], weights[8], gradH[4], energyTH, quality, lastTraceUV[2], lastTracePixelInterval; int32_t lastTraceStatus; };   // = sdv_immature_pt

struct SelJob {                          // one select pass of one frame
  FrameImg img; const float* thsSm; const double* cloud; int n;       // cloud == nullptr: dense pass over all pixels
  int w, h;                              // the frame's (its camera's) size
  int pot, nbx4, nby4, numPotW, numPotH, nslots; float thFactor; int active;
  int *cnt, *off, *slot_of, *list, *mask, *n2start; PtRec* rec;
  unsigned char* map;                    // n bytes (LiDAR) or w*h bytes (dense): 0 / 1 / 2 / 4
  int* counters;                         // [0] n2 [1] n3 [2] n4 [3] sub-selected away
  int charTH;                            // random sub-selection threshold, -1 = none
  const float* gw2 = nullptr;            // the frame camera's gamma weights of level 0 (gamma_w2; levels 1, 2 carry them in the texels); nullptr: no gamma set
};

SDV_DEVCONST float kSelDirs[16][2] = {{0,1.0000f},{0.3827f,0.9239f},{0.1951f,0.9808f},{0.9239f,0.3827f},{0.7071f,0.7071f},{0.3827f,-0.9239f},{0.8315f,0.5556f},{0.8315f,-0.5556f},
                                      {0.5556f,-0.8315f},{0.9808f,0.1951f},{0.9239f,-0.3827f},{0.7071f,-0.7071f},{0.5556f,0.8315f},{0.9808f,-0.1951f},{1.0000f,0.0000f},{0.1951f,-0.9808f}};

__device__ __forceinline__ int slot_of_cell(int cx, int cy, int nbx4) {                 // position of cell (cx,cy) in the reference's visiting order (4x4 block, 2x2 sub-block, cell)
  return (((cy>>2)*nbx4 + (cx>>2)) << 4) | (((cy>>1)&1) << 3) | (((cx>>1)&1) << 2) | ((cy&1) << 1) | (cx&1);
}
// the inputs of the three threshold tests for a candidate at float position (xf,yf) whose level-0 values are read at flat index idx
__device__ __forceinline__ PtRec make_rec(const FrameImg& F, const float* __restrict__ gw2, const float* __restrict__ thsSm, int w, int h, float xf, float yf, int idx, int out) {
  PtRec r; r.valid = 1; r.out = out;
  const int w32 = w/32, w1 = w>>1, w2 = w>>2;
  r.th0 = __ldg(thsSm + ((int)xf>>5) + ((int)yf>>5)*w32);
  planar_grad(F.I0, idx, w, h, r.dx, r.dy); r.ag0 = r.dx*r.dx + r.dy*r.dy;
  if (gw2) r.ag0 *= gamma_w2(__ldg(F.I0 + idx), gw2);
  r.ag1 = __ldg(&F.L1[(int)(xf*0.5f+0.25f) + (int)(yf*0.5f+0.25f)*w1].w);
  r.ag2 = __ldg(&F.L2[(int)((double)(xf*0.25f)+0.125) + (int)((double)(yf*0.25f)+0.125)*w2].w);
  return r;
}
struct Best { int i2, i3, i4; float v2, v3, v4; };
__device__ __forceinline__ void test_rec(const PtRec& r, float thF, float dw1, float dw2, int dirDist, const float* d2, const float* d3, const float* d4, Best& B) {
  const float th1 = r.th0*dw1, th2 = th1*dw2;
  if (r.ag0 > r.th0*thF) {
    float dn = fabsf(r.dx*d2[0] + r.dy*d2[1]); if (!dirDist) dn = r.ag0;
    if (dn > B.v2) { B.v2 = dn; B.i2 = r.out; B.i3 = -2; B.i4 = -2; }
  }
  if (B.i3 == -2) return;
  if (r.ag1 > th1*thF) {
    float dn = fabsf(r.dx*d3[0] + r.dy*d3[1]); if (!dirDist) dn = r.ag1;
    if (dn > B.v3) { B.v3 = dn; B.i3 = r.out; B.i4 = -2; }
  }
  if (B.i4 == -2) return;
  if (r.ag2 > th2*thF) {
    float dn = fabsf(r.dx*d4[0] + r.dy*d4[1]); if (!dirDist) dn = r.ag2;
    if (dn > B.v4) { B.v4 = dn; B.i4 = r.out; }
  }
}

// ---------------------------------------------------------------------------------------------- makeHists
struct HistJob { const float* I0; float* ths; float* thsSm; int w = 0, h = 0;             // w, h: the frame's (its camera's) size; 0: the engine's
                 const float* gw2 = nullptr; };                                          // the frame camera's gamma weights (gamma_w2); nullptr: no gamma set
// G: some job of the launch has gamma weights (the host picks the instantiation, so a batch without them runs no gamma code)
template <bool G> __global__ void __launch_bounds__(128) sel_hist_kernel(const HistJob* __restrict__ jobs, SelSet S) {      // CTA per 32x32 block of the largest job
  const HistJob J = jobs[blockIdx.y]; const float* gw2 = G ? J.gw2 : nullptr; const int w = J.w, h = J.h, w32 = w/32; if ((int)blockIdx.x >= w32*(h/32)) return;
  const int bx = blockIdx.x % w32, by = blockIdx.x / w32;
  __shared__ int hist[64];
  if (threadIdx.x < 64) hist[threadIdx.x] = 0;
  __syncthreads();
  for (int k = threadIdx.x; k < 1024; k += blockDim.x) {
    const int it = (k&31) + 32*bx, jt = (k>>5) + 32*by;
    if (it > w-2 || jt > h-2 || it < 1 || jt < 1) continue;
    float dx, dy; planar_grad(J.I0, it + jt*w, w, h, dx, dy);
    float ab = dx*dx + dy*dy; if (gw2) ab *= gamma_w2(__ldg(J.I0 + it + jt*w), gw2);
    int g = (int)sqrtf(ab); if (g > 48) g = 48;
    atomicAdd(&hist[g+1], 1); atomicAdd(&hist[0], 1);
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    int th = (int)(hist[0]*S.minGradHistCut + 0.5f), q = 90;
    for (int i = 0; i < 90; i++) { th -= (i+1 < 50) ? hist[i+1] : 0; if (th < 0) { q = i; break; } }
    J.ths[bx + by*w32] = q + S.minGradHistAdd;
  }
}
__global__ void __launch_bounds__(128) sel_smooth_kernel(const HistJob* __restrict__ jobs) {                             // thread per block
  const HistJob J = jobs[blockIdx.y]; const int w32 = J.w/32, h32 = J.h/32, i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= w32*h32) return;
  const int x = i % w32, y = i / w32; const float* ths = J.ths; float sum = 0, num = 0;
  if (x > 0)     { if (y > 0) { num++; sum += ths[x-1+(y-1)*w32]; } if (y < h32-1) { num++; sum += ths[x-1+(y+1)*w32]; } num++; sum += ths[x-1+y*w32]; }
  if (x < w32-1) { if (y > 0) { num++; sum += ths[x+1+(y-1)*w32]; } if (y < h32-1) { num++; sum += ths[x+1+(y+1)*w32]; } num++; sum += ths[x+1+y*w32]; }
  if (y > 0) { num++; sum += ths[x+(y-1)*w32]; }
  if (y < h32-1) { num++; sum += ths[x+(y+1)*w32]; }
  num++; sum += ths[x+y*w32];
  J.thsSm[x+y*w32] = (sum/num)*(sum/num);
}

// ---------------------------------------------------------------------------------------------- one select pass
// LiDAR pixels -> records + cell histogram (thread per cloud row)
template <bool G> __global__ void __launch_bounds__(128) sel_point_kernel(const SelJob* __restrict__ jobs) {
  const SelJob J = jobs[blockIdx.y]; if (!J.active || !J.cloud) return;
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= J.n) return;
  const int w = J.w, h = J.h;
  const double cu = J.cloud[3*i], cv = J.cloud[3*i+1]; const float xf = (float)cu, yf = (float)cv;
  PtRec r; r.valid = 0; r.out = i; r.dx = r.dy = r.ag0 = r.ag1 = r.ag2 = r.th0 = 0;
  int slot = -1;
  if (!(xf < 4 || xf >= w-5 || yf < 4 || yf > h-4) && cu == cu && cv == cv) {          // PixelSelector2.cpp:548 (also rejects NaN rows)
    const int idx = (int)(xf + (float)w*yf);                                             // sic: the float product of a fractional row with the width (:547)
    r = make_rec(J.img, G ? J.gw2 : nullptr, J.thsSm, w, h, xf, yf, idx, i);
    slot = slot_of_cell((int)cu / J.pot, (int)cv / J.pot, J.nbx4);
    atomicAdd(&J.cnt[slot], 1);
  }
  J.rec[i] = r; J.slot_of[i] = slot;
}
__global__ void __launch_bounds__(256) sel_scan_kernel(const SelJob* __restrict__ jobs) {                                 // CTA per job: off = exclusive scan of cnt over the slots
  const SelJob J = jobs[blockIdx.x]; if (!J.active || !J.cloud) return;
  __shared__ int sm[512]; __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int s0 = 0; s0 < J.nslots; s0 += blockDim.x*8) {                                  // 8 consecutive slots per thread
    const int s = s0 + threadIdx.x*8; int loc[8], sum = 0;
    for (int k = 0; k < 8; k++) { loc[k] = (s+k < J.nslots) ? J.cnt[s+k] : 0; sum += loc[k]; }
    int total; int ex = block_excl_scan(sum, sm, total) + base;
    for (int k = 0; k < 8; k++) { if (s+k < J.nslots) J.off[s+k] = ex; ex += loc[k]; }
    __syncthreads();
    if (threadIdx.x == 0) base += total;
    __syncthreads();
  }
}
__global__ void __launch_bounds__(128) sel_scatter_kernel(const SelJob* __restrict__ jobs) {                              // thread per cloud row
  const SelJob J = jobs[blockIdx.y]; if (!J.active || !J.cloud) return;
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= J.n) return;
  const int s = J.slot_of[i]; if (s < 0) return;
  J.list[atomicAdd(&J.off[s], 1)] = i;                                                   // off[s] ends as the END of the cell's segment
}
// candidate k of a cell: LiDAR = k-th entry of its (index-sorted) list; dense = k-th pixel of the cell in raster order
template <bool LIDAR, bool G> struct CellIter {
  const SelJob& J; int w, h; int beg, cnt; int x0, y0, mx, my;
  __device__ CellIter(const SelJob& J_, int slot, int cx, int cy) : J(J_), w(J_.w), h(J_.h) {
    if (LIDAR) { cnt = J.cnt[slot]; beg = J.off[slot] - cnt; x0 = y0 = mx = my = 0; }
    else { x0 = cx*J.pot; y0 = cy*J.pot; mx = imin_(J.pot, w - x0); my = imin_(J.pot, h - y0); cnt = mx*my; beg = 0; }
  }
  __device__ bool get(int k, PtRec& r) const {
    if (LIDAR) { r = J.rec[J.list[beg + k]]; return true; }
    const int y1 = k / mx, x1 = k - y1*mx, xf = x0 + x1, yf = y0 + y1;
    if (xf < 4 || xf >= w-5 || yf < 4 || yf > h-4) return false;                          // PixelSelector2.cpp:276
    r = make_rec(J.img, G ? J.gw2 : nullptr, J.thsSm, w, h, (float)xf, (float)yf, xf + w*yf, xf + w*yf); return true;
  }
};
// per cell: would it produce a level-2 pick, for each of the 16 directions (bit d)?  Exact: arg-max of |grad . dir_d| over the candidates above the level-0
// threshold, first one wins ties, and the pick only counts when the winner's index is > 0 (PixelSelector2.cpp:319, :592)
template <bool LIDAR, bool G> __global__ void __launch_bounds__(128) sel_cell_kernel(const SelJob* __restrict__ jobs, int dirDist) {
  const SelJob J = jobs[blockIdx.y]; if (!J.active || (J.cloud != nullptr) != LIDAR) return;
  const int slot = blockIdx.x*blockDim.x + threadIdx.x; if (slot >= J.nslots) return;
  const int blk = slot >> 4, bx = blk % J.nbx4, by = blk / J.nbx4, cx = bx*4 + ((slot>>2)&1)*2 + (slot&1), cy = by*4 + ((slot>>3)&1)*2 + ((slot>>1)&1);
  int m = 0;
  if (cx < J.numPotW && cy < J.numPotH) {
    CellIter<LIDAR, G> it(J, slot, cx, cy);
    if (LIDAR && it.cnt > 1) {                                                           // atomics filled the segment in arbitrary order: restore cloud order
      int* L = J.list + it.beg;
      for (int a = 1; a < it.cnt; a++) { const int v = L[a]; int b = a-1; while (b >= 0 && L[b] > v) { L[b+1] = L[b]; b--; } L[b+1] = v; }
    }
    float bv[16]; int bi[16];
#pragma unroll
    for (int d = 0; d < 16; d++) { bv[d] = 0; bi[d] = -1; }
    for (int k = 0; k < it.cnt; k++) {
      PtRec r; if (!it.get(k, r)) continue;
      if (!(r.ag0 > r.th0*J.thFactor)) continue;
#pragma unroll
      for (int d = 0; d < 16; d++) { float dn = fabsf(r.dx*kSelDirs[d][0] + r.dy*kSelDirs[d][1]); if (!dirDist) dn = r.ag0; if (dn > bv[d]) { bv[d] = dn; bi[d] = r.out; } }
    }
#pragma unroll
    for (int d = 0; d < 16; d++) if (bi[d] > 0) m |= 1 << d;
  }
  J.mask[slot] = m;
}
// n2 at the start of every cell, in visiting order.  CTA per job.  Where no cell of a chunk depends on the direction this is a prefix sum of "cell picks";
// a chunk holding such a cell is walked by one thread: d = randomPattern[n2] & 15, n2 += (mask >> d) & 1
__global__ void __launch_bounds__(256) sel_n2_kernel(const SelJob* __restrict__ jobs, const unsigned char* __restrict__ rp) {
  const SelJob J = jobs[blockIdx.x]; if (!J.active) return;
  __shared__ int sm[512]; __shared__ int base; __shared__ int smm[2048], smn[2048];      // masks / resolved counts of one chunk for the sequential walk
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int chunk = blockDim.x*8;                                                        // 8 consecutive cells per thread
  for (int s0 = 0; s0 < J.nslots; s0 += chunk) {
    const int s = s0 + threadIdx.x*8; int m[8], fullc = 0, partial = 0;
    for (int k = 0; k < 8; k++) { m[k] = (s+k < J.nslots) ? J.mask[s+k] : 0; const int full = (m[k] == 0xFFFF); fullc += full; partial |= (m[k] != 0 && !full); }
    if (!__syncthreads_or(partial)) {
      int total; int ex = block_excl_scan(fullc, sm, total) + base;
      for (int k = 0; k < 8; k++) { if (s+k < J.nslots) J.n2start[s+k] = ex; ex += (m[k] == 0xFFFF); }
      __syncthreads();
      if (threadIdx.x == 0) base += total;
    } else {                                                                             // a direction-dependent cell in this chunk: one thread walks the chunk from shared memory
      for (int k = 0; k < 8; k++) smm[threadIdx.x*8 + k] = m[k];
      __syncthreads();
      if (threadIdx.x == 0) { int b = base; const int e = imin_(chunk, J.nslots - s0);
        for (int t = 0; t < e; t++) { const int mm = smm[t]; smn[t] = b; if (mm) b += (mm == 0xFFFF) ? 1 : ((mm >> (rp[b] & 0xF)) & 1); }
        base = b; }
      __syncthreads();
      for (int k = 0; k < 8; k++) if (s+k < J.nslots) J.n2start[s+k] = smn[threadIdx.x*8 + k];
    }
    __syncthreads();
  }
  if (threadIdx.x == 0) J.counters[0] = base;
}
// thread per 4x4-cell block: the three-level state machine of select / selectFromLidar with the directions now known
template <bool LIDAR, bool G> __global__ void __launch_bounds__(128) sel_block_kernel(const SelJob* __restrict__ jobs, const unsigned char* __restrict__ rp, int dirDist, float dw1) {
  const SelJob J = jobs[blockIdx.y]; if (!J.active || (J.cloud != nullptr) != LIDAR) return;
  const int blk = blockIdx.x*blockDim.x + threadIdx.x; if (blk >= J.nbx4*J.nby4) return;
  const int bx = blk % J.nbx4, by = blk / J.nbx4; const float dw2 = dw1*dw1;
  Best B; B.i4 = -1; B.v4 = 0; int n3 = 0, n4 = 0;
  const float* dir4 = kSelDirs[rp[J.n2start[blk << 4]] & 0xF];
  for (int sub = 0; sub < 4; sub++) {
    const int scx = bx*4 + (sub&1)*2, scy = by*4 + (sub>>1)*2; if (scx >= J.numPotW || scy >= J.numPotH) continue;
    B.i3 = -1; B.v3 = 0;
    const float* dir3 = kSelDirs[rp[J.n2start[(blk << 4) | (sub << 2)]] & 0xF];
    for (int c = 0; c < 4; c++) {
      const int cx = scx + (c&1), cy = scy + (c>>1); if (cx >= J.numPotW || cy >= J.numPotH) continue;
      const int slot = (blk << 4) | (sub << 2) | c;
      B.i2 = -1; B.v2 = 0;
      const float* dir2 = kSelDirs[rp[J.n2start[slot]] & 0xF];
      CellIter<LIDAR, G> it(J, slot, cx, cy);
      for (int k = 0; k < it.cnt; k++) { PtRec r; if (!it.get(k, r)) continue; test_rec(r, J.thFactor, dw1, dw2, dirDist, dir2, dir3, dir4, B); }
      if (B.i2 > 0) { J.map[B.i2] = 1; B.v3 = 1e10f; }
    }
    if (B.i3 > 0) { J.map[B.i3] = 2; B.v4 = 1e10f; n3++; }
  }
  if (B.i4 > 0) { J.map[B.i4] = 4; n4++; }
  if (n3) atomicAdd(&J.counters[1], n3);
  if (n4) atomicAdd(&J.counters[2], n4);
}
// Dense pass (select over all pixels), one WARP per 4x4-cell block: the block's (4 pot)^2 pixels are walked in the reference's order in chunks of 32 — every lane
// gathers the record of one pixel (threshold, level-0 gradient, the two coarser gradient magnitudes: the scattered loads, now 32 wide), then all lanes replay the
// three-level state machine over the chunk from shared memory, redundantly and identically (no divergence; lane 0 writes).  A thread-per-block version walks 144 pixels per
// thread with dependent loads.
template <bool G> __global__ void __launch_bounds__(32) sel_block_dense_kernel(const SelJob* __restrict__ jobs, const unsigned char* __restrict__ rp, int dirDist, float dw1) {
  const SelJob J = jobs[blockIdx.y]; if (!J.active || J.cloud != nullptr) return;
  const int blk = blockIdx.x; if (blk >= J.nbx4*J.nby4) return;
  const int w = J.w, h = J.h;
  const int bx = blk % J.nbx4, by = blk / J.nbx4, pot = J.pot, pp = pot*pot, npx = 16*pp, lane = threadIdx.x; const float dw2 = dw1*dw1;
  __shared__ PtRec recs[32];
  Best B; B.i2 = B.i3 = B.i4 = -1; B.v2 = B.v3 = B.v4 = 0; int n3 = 0, n4 = 0;
  const float* dir4 = kSelDirs[rp[J.n2start[blk << 4]] & 0xF]; const float* dir3 = dir4; const float* dir2 = dir4;
  for (int p0 = 0; p0 < npx; p0 += 32) {
    { const int p = p0 + lane; PtRec r; r.valid = 0; r.out = 0; r.dx = r.dy = r.ag0 = r.ag1 = r.ag2 = r.th0 = 0;
      if (p < npx) { const int ci = p / pp, k = p - ci*pp, y1 = k / pot, x1 = k - y1*pot;
        const int cx = bx*4 + ((ci>>2)&1)*2 + (ci&1), cy = by*4 + (ci>>3)*2 + ((ci>>1)&1), xf = cx*pot + x1, yf = cy*pot + y1;
        if (xf < w && yf < h && !(xf < 4 || xf >= w-5 || yf < 4 || yf > h-4)) r = make_rec(J.img, G ? J.gw2 : nullptr, J.thsSm, w, h, (float)xf, (float)yf, xf + w*yf, xf + w*yf); }
      recs[lane] = r; }
    __syncthreads();
    const int cnt = imin_(32, npx - p0);
    for (int l = 0; l < cnt; l++) {
      const int p = p0 + l, ci = p / pp, k = p - ci*pp;
      if (k == 0) {                                                                      // a cell begins (and with it, possibly, a sub-block)
        if ((ci & 3) == 0) { B.i3 = -1; B.v3 = 0; dir3 = kSelDirs[rp[J.n2start[(blk << 4) | ci]] & 0xF]; }
        B.i2 = -1; B.v2 = 0; dir2 = kSelDirs[rp[J.n2start[(blk << 4) | ci]] & 0xF];
      }
      if (recs[l].valid) test_rec(recs[l], J.thFactor, dw1, dw2, dirDist, dir2, dir3, dir4, B);
      if (k == pp-1) {                                                                   // the cell ends
        if (B.i2 > 0) { if (lane == 0) J.map[B.i2] = 1; B.v3 = 1e10f; }
        if ((ci & 3) == 3) { if (B.i3 > 0) { if (lane == 0) J.map[B.i3] = 2; B.v4 = 1e10f; n3++; } }
      }
    }
    __syncthreads();
  }
  if (B.i4 > 0) { if (lane == 0) J.map[B.i4] = 4; n4++; }
  if (lane == 0) { if (n3) atomicAdd(&J.counters[1], n3); if (n4) atomicAdd(&J.counters[2], n4); }
}
// random sub-selection (PixelSelector2.cpp:405-423 LiDAR: the pattern is indexed by the pixel; :156-172 dense: by the rank among the selected pixels)
// A w_c x h_c camera's pattern (PixelSelector::PixelSelector(w_c, h_c) re-seeds and draws w_c*h_c bytes) is the first w_c*h_c bytes of the context's: rp serves every job.
__global__ void __launch_bounds__(128) sel_sub_lidar_kernel(const SelJob* __restrict__ jobs, const unsigned char* __restrict__ rp) {
  const SelJob J = jobs[blockIdx.y]; if (J.charTH < 0 || !J.cloud) return;
  const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= J.n) return;
  if (J.map[i] == 0) return;
  const int rn = (int)(J.cloud[3*i] + J.cloud[3*i+1]*J.w);
  if ((int)rp[rn] > J.charTH) { J.map[i] = 0; atomicAdd(&J.counters[3], 1); }
}
__global__ void __launch_bounds__(128) sel_rowcount_kernel(const SelJob* __restrict__ jobs, int rs, int* __restrict__ rowcnt /* jobs x rs >= every job's h */) {   // thread per image row
  const SelJob J = jobs[blockIdx.y]; if (J.charTH < 0 || J.cloud) return;
  const int w = J.w, y = blockIdx.x*blockDim.x + threadIdx.x; if (y >= J.h) return;
  int n = 0; for (int x = 0; x < w; x++) n += J.map[y*w + x] != 0;
  rowcnt[blockIdx.y*rs + y] = n;
}
__global__ void __launch_bounds__(128) sel_sub_dense_kernel(const SelJob* __restrict__ jobs, const unsigned char* __restrict__ rp, int rs, const int* __restrict__ rowcnt) {
  const SelJob J = jobs[blockIdx.y]; if (J.charTH < 0 || J.cloud) return;
  const int w = J.w, y = blockIdx.x*blockDim.x + threadIdx.x; if (y >= J.h) return;
  int rn = 0; for (int r = 0; r < y; r++) rn += rowcnt[blockIdx.y*rs + r];
  int drop = 0;
  for (int x = 0; x < w; x++) if (J.map[y*w + x] != 0) { if ((int)rp[rn] > J.charTH) { J.map[y*w + x] = 0; drop++; } rn++; }
  if (drop) atomicAdd(&J.counters[3], drop);
}

// ---------------------------------------------------------------------------------------------- makeNewTraces
struct TraceJob {
  FrameImg img; const double* cloud; int n; const unsigned char* mapL; unsigned char* mapD;        // LiDAR selection (n bytes), persistent monocular selection (w*h bytes)
  int w, h;                                                                                         // the frame's (its camera's) size
  int pot;                                                                                         // PixelSelector::currentPotential after both makeMaps calls (setMask)
  float* score; int* flag; int* pos;                                                                // per cloud row
  unsigned char* occ; unsigned char* state; int* cand; int ncand_cap;                              // occupancy mask, per-pixel state of the monocular candidates, their list
  NewTrace* out; ImmPt* imm; int cap;
  int* counts;                                                                                      // [0] LiDAR points kept [1] monocular points kept [2] monocular candidates [3] max score bits
};
__device__ float shi_tomasi(const float* __restrict__ I, int w, int h, int u, int v) {            // FullSystem.cpp:1540-1583; (*ptr)[0] is the intensity channel
  float dXX = 0, dYY = 0, dXY = 0; const int x_min = u-4, x_max = u+4, y_min = v-4, y_max = v+4;
  if (x_min < 1 || x_max >= w-1 || y_min < 1 || y_max >= h-1) return 0.0f;
  for (int y = y_min; y < y_max; y++) for (int x = 0; x < 8; x++) {
    const float dx = __ldg(I + w*y + x_min+1+x) - __ldg(I + w*y + x_min-1+x), dy = __ldg(I + w*(y+1) + x_min+x) - __ldg(I + w*(y-1) + x_min+x);
    dXX += dx*dx; dYY += dy*dy; dXY += dx*dy;
  }
  dXX = (float)(dXX / (2.0*64)); dYY = (float)(dYY / (2.0*64)); dXY = (float)(dXY / (2.0*64));
  const float disc = sqrtf((dXX+dYY)*(dXX+dYY) - 4*(dXX*dYY - dXY*dXY));                         // FullSystem.h:19 includes <math.h>: sqrt(float) is the float overload
  const float l1 = (float)(0.5*(dXX + dYY - disc)), l2 = (float)(0.5*(dXX + dYY + disc));
  const float k = 0.04f;
  return (l1*l2 - k*(l1+l2)*(l1+l2));
}
__device__ __forceinline__ void paint_mask(unsigned char* occ, int w, int h, int Ku, int Kv, int pot) {        // FullSystem::setMask :1261-1271
  for (int i = Ku-pot; i <= Ku+pot; i++) for (int j = Kv-1; j <= Kv+1; j++) if (j < h && j >= 0 && i < w && i >= 0) occ[j*w + i] = 1;
}
__device__ __forceinline__ int float_order_bits(float f) { int b = __float_as_int(f); return b >= 0 ? b : (b ^ 0x7FFFFFFF); }     // monotone float -> int (atomicMax of the scores)
__device__ __forceinline__ float float_from_order_bits(int b) { return __int_as_float(b >= 0 ? b : (b ^ 0x7FFFFFFF)); }
// LiDAR loop, part 1 (thread per cloud row): score of every selected pixel, whether its candidate survives (finite pattern), the maximum score
__global__ void __launch_bounds__(128) nt_lidar_score_kernel(const TraceJob* __restrict__ jobs, SelSet S) {
  const TraceJob J = jobs[blockIdx.y]; const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= J.n) return;
  const int w = J.w, h = J.h;
  int keep = 0; float sc = 0;
  if (J.mapL[i] != 0) {
    const int u = (int)J.cloud[3*i], v = (int)J.cloud[3*i+1];
    sc = shi_tomasi(J.img.I0, w, h, u, v); atomicMax(&J.counts[3], float_order_bits(sc));
    ImmPt p; keep = imm_construct(J.img.I0, w, u, v, S, p) ? 1 : 0;
  }
  J.score[i] = sc; J.flag[i] = keep;
}
__global__ void __launch_bounds__(256) nt_scan_kernel(const TraceJob* __restrict__ jobs) {                       // CTA per job: pos = exclusive scan of flag over the cloud rows
  const TraceJob J = jobs[blockIdx.x];
  __shared__ int sm[512]; __shared__ int base;
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  for (int s0 = 0; s0 < J.n; s0 += blockDim.x*8) {
    const int s = s0 + threadIdx.x*8; int loc[8], sum = 0;
    for (int k = 0; k < 8; k++) { loc[k] = (s+k < J.n) ? J.flag[s+k] : 0; sum += loc[k]; }
    int total; int ex = block_excl_scan(sum, sm, total) + base;
    for (int k = 0; k < 8; k++) { if (s+k < J.n) J.pos[s+k] = ex; ex += loc[k]; }
    __syncthreads();
    if (threadIdx.x == 0) base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) J.counts[0] = base;
}
// LiDAR loop, part 2: the kept candidates in cloud order -> records, CORNER / EDGELET by score > 0.01f * maxScore (:1328-1335), occupancy mask
__global__ void __launch_bounds__(128) nt_lidar_emit_kernel(const TraceJob* __restrict__ jobs, SelSet S) {
  const TraceJob J = jobs[blockIdx.y]; const int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= J.n || !J.flag[i]) return;
  const int w = J.w, h = J.h;
  const int u = (int)J.cloud[3*i], v = (int)J.cloud[3*i+1], m = J.pos[i];
  const float maxScore = float_from_order_bits(J.counts[3]), threshold = 0.01f;
  if (m < J.cap) {
    NewTrace t; t.u = (float)u; t.v = (float)v; t.my_type = (float)J.mapL[i]; t.score = J.score[i]; t.idepth_fromSensor = (float)(1.0 / J.cloud[3*i+2]); t.isFromSensor = 1;
    t.type = (t.score > threshold*maxScore) ? 0 : 1; J.out[m] = t;
    ImmPt p; imm_construct(J.img.I0, w, u, v, S, p); J.imm[m] = p;
  }
  paint_mask(J.occ, w, h, u, v, J.pot);
}
// monocular loop (:1337-1353): candidates = selected pixels of the persistent map inside the pattern padding, in raster order.  A candidate is dropped when its
// pattern is not finite or the occupancy mask is set at its pixel — by a LiDAR point, or by a monocular candidate accepted EARLIER in raster order (greedy).
__global__ void __launch_bounds__(128) nt_dense_state_kernel(const TraceJob* __restrict__ jobs, SelSet S) {   // thread per pixel: state of the monocular candidates
  const TraceJob J = jobs[blockIdx.y]; const int w = J.w, h = J.h, i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= w*h) return;
  const int y = i / w, x = i - y*w; unsigned char st = 0;
  if (y >= 3 && y < h-4 && x >= 3 && x < w-4 && J.mapD[i] != 0) { ImmPt p; st = (imm_construct(J.img.I0, w, x, y, S, p) && J.occ[i] == 0) ? 1 : 3; }
  J.state[i] = st;
}
__global__ void __launch_bounds__(256) nt_dense_resolve_kernel(const TraceJob* __restrict__ jobs, SelSet S) {   // CTA per job
  const TraceJob J = jobs[blockIdx.x]; const int w = J.w, h = J.h;
  __shared__ int sm[512]; __shared__ int base;
  // (1) candidate list in raster order: chunked compaction of state != 0
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int wh = w*h;
  for (int s0 = 0; s0 < wh; s0 += blockDim.x*8) {
    const int s = s0 + threadIdx.x*8; int loc[8], sum = 0;
    for (int k = 0; k < 8; k++) { loc[k] = (s+k < wh && J.state[s+k] != 0) ? 1 : 0; sum += loc[k]; }
    int total; int ex = block_excl_scan(sum, sm, total) + base;
    for (int k = 0; k < 8; k++) if (loc[k]) { if (ex < J.ncand_cap) J.cand[ex] = s+k; ex++; }
    __syncthreads();
    if (threadIdx.x == 0) base += total;
    __syncthreads();
  }
  const int nc = imin_(base, J.ncand_cap);
  // (2) greedy raster-order suppression, resolved in rounds: a candidate is final once every earlier candidate whose mask rectangle covers it is final
  volatile unsigned char* st = J.state;
  for (int round = 0; round < 4096; round++) {
    int undecided = 0;
    for (int c = threadIdx.x; c < nc; c += blockDim.x) {
      const int i = J.cand[c]; if (st[i] != 1) continue;
      const int y = i / w, x = i - y*w; int acc = 0, und = 0;
      for (int xx = x-J.pot; xx <= x+J.pot; xx++) if (xx >= 0 && xx < w) { const unsigned char a = st[(y-1)*w + xx]; acc |= (a == 2); und |= (a == 1); }   // y >= 3
      for (int xx = x-J.pot; xx < x; xx++) if (xx >= 0) { const unsigned char a = st[y*w + xx]; acc |= (a == 2); und |= (a == 1); }
      if (acc) st[i] = 3; else if (!und) st[i] = 2; else undecided = 1;
    }
    if (!__syncthreads_or(undecided)) break;
  }
  __syncthreads();
  // (3) accepted candidates, raster order, appended after the LiDAR points
  if (threadIdx.x == 0) base = 0;
  __syncthreads();
  const int m0 = J.counts[0];
  for (int c0 = 0; c0 < nc; c0 += blockDim.x) {
    const int c = c0 + threadIdx.x; const int i = (c < nc) ? J.cand[c] : 0; const int ok = (c < nc && st[i] == 2) ? 1 : 0;
    int total; const int ex = block_excl_scan(ok, sm, total) + base;
    if (ok) { const int m = m0 + ex, y = i / w, x = i - y*w;
      if (m < J.cap) { NewTrace t; t.u = (float)x; t.v = (float)y; t.my_type = (float)J.mapD[i]; t.score = 0; t.idepth_fromSensor = 0; t.isFromSensor = 0; t.type = -1; J.out[m] = t;
        ImmPt p; imm_construct(J.img.I0, w, x, y, S, p); J.imm[m] = p; } }
    __syncthreads();
    if (threadIdx.x == 0) base += total;
    __syncthreads();
  }
  if (threadIdx.x == 0) { J.counts[1] = base; J.counts[2] = nc; }
}

// ---------------------------------------------------------------------------------------------- CoarseDistanceMap + activation walk
struct DistJob {
  int* d; int w1, h1;                                          // fwdWarpedIDDistFinal at level-1 resolution (1000 = far)
  int nHosts; const int* pt_begin; const float* KRKi; const float* Kt; const float* uvid;       // sources: ACTIVE points grouped by host, K[1] R K[0]^-1 and K[1] t per host
  int nCandHosts; const int* cand_begin; const float* cKRKi; const float* cKt; const float* cand4;   // candidates {u, v, 0.5f*(idepth_max+idepth_min), my_type} grouped by host
  float minActDist; int* proj;                                 // per candidate: u | v<<16 (or -1 outside), then frac, then thr — 3 ints (floats as bits)
  int* decision;
};
__device__ __forceinline__ bool dm_project(const float* M, const float* t, float pu, float pv, float id, int w1, int h1, int& u, int& v, float& px) {
  float ptp[3];
#pragma unroll
  for (int r = 0; r < 3; r++) ptp[r] = ((M[3*r]*pu + M[3*r+1]*pv) + M[3*r+2]*1.0f) + t[r]*id;
  u = (int)(ptp[0] / ptp[2] + 0.5f); v = (int)(ptp[1] / ptp[2] + 0.5f); px = ptp[0];
  return (u > 0 && v > 0 && u < w1 && v < h1);
}
__global__ void __launch_bounds__(256) dm_fill_kernel(const DistJob* __restrict__ jobs) {
  const DistJob J = jobs[blockIdx.y]; const int n = J.w1*J.h1;
  for (int i = blockIdx.x*blockDim.x + threadIdx.x; i < n; i += gridDim.x*blockDim.x) J.d[i] = 1000;
}
__global__ void __launch_bounds__(128) dm_source_kernel(const DistJob* __restrict__ jobs) {                      // thread per ACTIVE point (CoarseTracker.cpp:1160-1169)
  const DistJob J = jobs[blockIdx.y]; const int p = blockIdx.x*blockDim.x + threadIdx.x; if (p >= J.pt_begin[J.nHosts]) return;
  int hI = 0; while (p >= J.pt_begin[hI+1]) hI++;
  int u, v; float px;
  if (dm_project(J.KRKi + 9*hI, J.Kt + 3*hI, J.uvid[3*p], J.uvid[3*p+1], J.uvid[3*p+2], J.w1, J.h1, u, v, px)) J.d[u + J.w1*v] = 0;
}
// ring k of growDistBFS (:1179-1270) as a pull sweep: a pixel farther than k takes k when a 4-neighbour (odd k: 8-neighbour) that is not on the image border holds k-1.
// Valid for the fresh map of makeDistanceMap, where every pixel holding k-1 was set by this BFS.  In-place is safe: values only change from > k to k.
__global__ void __launch_bounds__(256) dm_ring_kernel(const DistJob* __restrict__ jobs, int k) {
  const DistJob J = jobs[blockIdx.y]; const int w1 = J.w1, h1 = J.h1, n = w1*h1;
  for (int i = blockIdx.x*blockDim.x + threadIdx.x; i < n; i += gridDim.x*blockDim.x) {
    if (J.d[i] <= k) continue;
    const int y = i / w1, x = i - y*w1; bool hit = false;
    for (int dy = -1; dy <= 1 && !hit; dy++) for (int dx = -1; dx <= 1; dx++) {
      if ((dx == 0 && dy == 0) || ((k&1) == 0 && dx != 0 && dy != 0)) continue;
      const int qx = x+dx, qy = y+dy; if (qx <= 0 || qy <= 0 || qx >= w1-1 || qy >= h1-1) continue;         // the expanding pixel must be interior (:1190)
      if (J.d[qx + qy*w1] == k-1) { hit = true; break; }
    }
    if (hit) J.d[i] = k;
  }
}
__global__ void __launch_bounds__(128) act_project_kernel(const DistJob* __restrict__ jobs) {                   // thread per candidate (FullSystem.cpp:648-651)
  const DistJob J = jobs[blockIdx.y]; const int c = blockIdx.x*blockDim.x + threadIdx.x; if (c >= J.cand_begin[J.nCandHosts]) return;
  int hI = 0; while (c >= J.cand_begin[hI+1]) hI++;
  int u, v; float px;
  const bool in = dm_project(J.cKRKi + 9*hI, J.cKt + 3*hI, J.cand4[4*c], J.cand4[4*c+1], J.cand4[4*c+2], J.w1, J.h1, u, v, px);
  J.proj[3*c] = in ? (u | (v << 16)) : -1;
  J.proj[3*c+1] = __float_as_int(px - floorf(px)); J.proj[3*c+2] = __float_as_int(J.minActDist*J.cand4[4*c+3]);
}
// the greedy walk (:653-664): candidates in order; one whose distance-map value + sub-pixel offset reaches its threshold is accepted and becomes a new BFS source
// (addIntoDistFinal) before the next one is judged.  CTA per sequence; a chunk of candidates is judged in parallel, the first accept wins, the BFS runs
// block-wide over an explicit frontier (atomicMin claims a pixel exactly once), then the rest of the chunk is judged again.
__global__ void __launch_bounds__(64) act_walk_kernel(const DistJob* __restrict__ jobs) {
  const DistJob J = jobs[blockIdx.x]; const int w1 = J.w1, h1 = J.h1, nc = J.cand_begin[J.nCandHosts];
  __shared__ int listA[1024], listB[1024]; __shared__ int nA, nB, first;
  for (int c0 = 0; c0 < nc; c0 += blockDim.x) {
    const int c = c0 + threadIdx.x; bool live = c < nc; int uv = -1; float frac = 0, thr = 0;
    if (live) { uv = J.proj[3*c]; frac = __int_as_float(J.proj[3*c+1]); thr = __int_as_float(J.proj[3*c+2]); if (uv < 0) { J.decision[c] = -1; live = false; } }
    for (;;) {
      if (threadIdx.x == 0) first = INT_MAX;
      __syncthreads();
      bool pass = false;
      if (live) { const float dist = (float)__ldcg(&J.d[(uv & 0xFFFF) + w1*(uv >> 16)]) + frac; pass = dist >= thr; if (pass) atomicMin(&first, (int)threadIdx.x); }
      __syncthreads();
      const int f = first;
      if (f == INT_MAX) { if (live) J.decision[c] = 0; break; }
      if (live && (int)threadIdx.x < f) { J.decision[c] = 0; live = false; }
      if ((int)threadIdx.x == f) { J.decision[c] = 1; live = false; J.d[(uv & 0xFFFF) + w1*(uv >> 16)] = 0; listA[0] = uv; nA = 1; }
      __syncthreads();
      int* A = listA; int* Bq = listB;
      for (int k = 1; k < 40; k++) {                                                     // growDistBFS(1)
        if (threadIdx.x == 0) nB = 0;
        __syncthreads();
        const int na = nA;
        for (int i = threadIdx.x; i < na; i += blockDim.x) {
          const int x = A[i] & 0xFFFF, y = A[i] >> 16; if (x == 0 || y == 0 || x == w1-1 || y == h1-1) continue;
          for (int dy = -1; dy <= 1; dy++) for (int dx = -1; dx <= 1; dx++) {
            if ((dx == 0 && dy == 0) || ((k&1) == 0 && dx != 0 && dy != 0)) continue;
            if (atomicMin(&J.d[(x+dx) + (y+dy)*w1], k) > k) { const int q = atomicAdd(&nB, 1); if (q < 1024) Bq[q] = (x+dx) | ((y+dy) << 16); }
          }
        }
        __syncthreads();
        if (threadIdx.x == 0) nA = imin_(nB, 1024);
        __syncthreads();
        int* T = A; A = Bq; Bq = T;
        if (nA == 0) break;
      }
      __syncthreads();
    }
    __syncthreads();
  }
}

// The same walk with the distance map in SHARED memory (one byte per level-1 pixel: 105 KB for KITTI, two CTAs per SM): the judge reads and the ring claims no longer
// make an L2 round trip each (in the global-memory version those round trips dominate the keyframe-rate device time).  A claim is a compare-and-swap
// on the 32-bit word holding the byte, so every pixel is still taken exactly once per ring.  255 stands for "farther than 39" (1000 in the reference).
__device__ __forceinline__ int smap_get(const unsigned int* m, int cell) { return (m[cell >> 2] >> ((cell & 3)*8)) & 255; }
__device__ __forceinline__ bool smap_claim(unsigned int* m, int cell, int k) {
  unsigned int* wp = m + (cell >> 2); const int sh = (cell & 3)*8;
  for (;;) { const unsigned int old = *(volatile unsigned int*)wp; if ((int)((old >> sh) & 255u) <= k) return false;
    const unsigned int nw = (old & ~(255u << sh)) | ((unsigned int)k << sh); if (atomicCAS(wp, old, nw) == old) return true; }
}
// (A one-warp walk with 128 threads for the map load / store — tried because most of the issue cycles of this kernel sit at the block barrier — is slower: the second
// warp does shorten the frontier and judge loops.)
__global__ void __launch_bounds__(256) act_walk_smem_kernel(const DistJob* __restrict__ jobs, int build_map) {
  const DistJob J = jobs[blockIdx.x]; const int w1 = J.w1, h1 = J.h1, n1 = w1*h1, nc = J.cand_begin[J.nCandHosts];
  SDV_DYN_SMEM(unsigned int, dsm);
  unsigned int* smap = dsm; int* listA = (int*)(dsm + ((n1 + 3) >> 2)); int* listB = listA + 1024;
  __shared__ int nA, nB, first;
  if (build_map) {                                                                       // makeDistanceMap in shared memory: fill, sources, 39 pull rings (same rule as dm_ring_kernel)
    unsigned char* bm = reinterpret_cast<unsigned char*>(smap);
    for (int i = threadIdx.x; i < ((n1 + 3) >> 2); i += blockDim.x) smap[i] = 0xFFFFFFFFu;
    __syncthreads();
    const int np = J.pt_begin[J.nHosts];
    for (int p = threadIdx.x; p < np; p += blockDim.x) { int hI = 0; while (p >= J.pt_begin[hI+1]) hI++;
      int u, v; float px; if (dm_project(J.KRKi + 9*hI, J.Kt + 3*hI, J.uvid[3*p], J.uvid[3*p+1], J.uvid[3*p+2], w1, h1, u, v, px)) bm[u + w1*v] = 0; }
    __syncthreads();
    for (int k = 1; k < 40; k++) {
      for (int i = threadIdx.x; i < n1; i += blockDim.x) {
        if ((int)bm[i] <= k) continue;
        const int y = i / w1, x = i - y*w1; bool hit = false;
        for (int dy = -1; dy <= 1 && !hit; dy++) for (int dx = -1; dx <= 1; dx++) {
          if ((dx == 0 && dy == 0) || ((k&1) == 0 && dx != 0 && dy != 0)) continue;
          const int qx = x+dx, qy = y+dy; if (qx <= 0 || qy <= 0 || qx >= w1-1 || qy >= h1-1) continue;
          if ((int)bm[qx + qy*w1] == k-1) { hit = true; break; }
        }
        if (hit) bm[i] = (unsigned char)k;
      }
      __syncthreads();
    }
  } else {
    for (int i = threadIdx.x; i < ((n1 + 3) >> 2); i += blockDim.x) {                     // four cells per word
      unsigned int wv = 0; for (int b = 0; b < 4; b++) { const int c = 4*i + b; const int d = (c < n1) ? J.d[c] : 1000; wv |= (unsigned int)(d > 254 ? 255 : d) << (8*b); }
      smap[i] = wv; }
  }
  __syncthreads();
  for (int c0 = 0; c0 < nc; c0 += blockDim.x) {
    const int c = c0 + threadIdx.x; bool live = c < nc; int uv = -1; float frac = 0, thr = 0;
    if (live) { uv = J.proj[3*c]; frac = __int_as_float(J.proj[3*c+1]); thr = __int_as_float(J.proj[3*c+2]); if (uv < 0) { J.decision[c] = -1; live = false; } }
    for (;;) {
      if (threadIdx.x == 0) first = INT_MAX;
      __syncthreads();
      if (live) { const int b = smap_get(smap, (uv & 0xFFFF) + w1*(uv >> 16)); const float dist = (float)(b == 255 ? 1000 : b) + frac; if (dist >= thr) atomicMin(&first, (int)threadIdx.x); }
      __syncthreads();
      const int f = first;
      if (f == INT_MAX) { if (live) J.decision[c] = 0; break; }
      if (live && (int)threadIdx.x < f) { J.decision[c] = 0; live = false; }
      if ((int)threadIdx.x == f) { J.decision[c] = 1; live = false; const int cell = (uv & 0xFFFF) + w1*(uv >> 16); const int sh = (cell & 3)*8; smap[cell >> 2] &= ~(255u << sh); listA[0] = uv; nA = 1; }
      __syncthreads();
      int* A = listA; int* Bq = listB;
      for (int k = 1; k < 40; k++) {
        if (threadIdx.x == 0) nB = 0;
        __syncthreads();
        const int na = nA;
        for (int i = threadIdx.x; i < na; i += blockDim.x) {
          const int x = A[i] & 0xFFFF, y = A[i] >> 16; if (x == 0 || y == 0 || x == w1-1 || y == h1-1) continue;
          for (int dy = -1; dy <= 1; dy++) for (int dx = -1; dx <= 1; dx++) {
            if ((dx == 0 && dy == 0) || ((k&1) == 0 && dx != 0 && dy != 0)) continue;
            if (smap_claim(smap, (x+dx) + (y+dy)*w1, k)) { const int q = atomicAdd(&nB, 1); if (q < 1024) Bq[q] = (x+dx) | ((y+dy) << 16); }
          }
        }
        __syncthreads();
        if (threadIdx.x == 0) nA = imin_(nB, 1024);
        __syncthreads();
        int* T = A; A = Bq; Bq = T;
        if (nA == 0) break;
      }
      __syncthreads();
    }
    __syncthreads();
  }
  for (int i = threadIdx.x; i < n1; i += blockDim.x) { const int b = smap_get(smap, i); J.d[i] = (b == 255) ? 1000 : b; }
}

// ================================================================================================ host engine
// host-side state of one PixelSelector (one per resident sequence): currentPotential + the persistent monocular selection map
struct SelectorSlot { int currentPotential = 3; unsigned char* mapD = nullptr; };

struct MapsJobHost {                     // one makeMaps / makeMapsFromLidar call
  FrameImg img; int w = 0, h = 0; const float* thsSm; const double* cloud_dev; int n; unsigned char* map; float density; int recursionsLeft; float thFactor; int* currentPotential;
  int numHaveSub;                       // out
  int passes;                            // out: select passes run (1, or 2 after a recursion)
  const float* gw2 = nullptr;            // the frame camera's gamma weights (SelJob::gw2)
};

struct SelEngine {
  int w = 0, h = 0;                        // the largest image (the pattern's size); every job carries its own size w_j <= w, h_j <= h (a job whose size is 0 has w x h)
  SelSet S; cudaStream_t st = nullptr; std::string err;
  unsigned char* rp = nullptr;           // randomPattern (device)
  Scratch scr, scr2; long long launches = 0;
  cudaEvent_t ev0 = nullptr, ev1 = nullptr; bool have_ev = false; float last_kernel_ms = 0.f;   // device time of the launches of the last activate() (copies excluded)
  size_t max_scratch = (size_t)1 << 30;
  int walk_threads = 64;                    // CTA size of the shared-memory walk kernel (64 / 128 / 256 measured equal: the walk is a latency chain)
  bool fuse_map = false;                    // build the distance map inside the walk kernel (fill, sources, 39 rings in shared memory; SDV_FUSE_MAP=1).  Correct (GPU tests green) but
                                            // slower: full-map sweeps by one CTA per sequence lose against 39 grid-wide launches
  size_t max_walk_smem = 200*1024;          // the activation walk keeps its distance map in shared memory up to this size (227 KB per CTA on sm_90)

  int init(int w_, int h_, const SelSet& S_, const unsigned char* random_pattern_host, cudaStream_t st_) {
    w = w_; h = h_; S = S_; st = st_;
    if (!have_ev) have_ev = (cudaEventCreate(&ev0) == cudaSuccess && cudaEventCreate(&ev1) == cudaSuccess);
    if (rp) cudaFree(rp);
    SEL_CK(cudaMalloc((void**)&rp, (size_t)w*h)); SEL_CK(cudaMemcpyAsync(rp, random_pattern_host, (size_t)w*h, cudaMemcpyHostToDevice, st)); SEL_CK(cudaStreamSynchronize(st));
    return 0;
  }
  void destroy() { if (rp) cudaFree(rp); rp = nullptr; scr.release(); scr2.release(); if (have_ev) { cudaEventDestroy(ev0); cudaEventDestroy(ev1); have_ev = false; } }
  static size_t ths_floats(int w, int h) { const int w32 = w/32, h32 = h/32; return (size_t)w32*(h32+1) + 101; }   // thsSmoothed is read up to one block row / column past its end (zero there)
  size_t ths_floats() const { return ths_floats(w, h); }
  template <class J> void size_or_engine(J& j) const { if (!j.w) { j.w = w; j.h = h; } }

  // PixelSelector::makeHists for nj frames: ths / thsSm are device arrays of ths_floats(w_j, h_j) floats per job, zero-initialised by the caller
  int make_hists(int nj, const HistJob* jobs_host) {
    if (nj <= 0) return 0;
    if (scr2.reserve(Scratch::need(nj, sizeof(HistJob)), st)) { err = "scratch"; return -1; }
    scr2.reset(); HistJob* d = scr2.take<HistJob>(nj);
    std::vector<HistJob> H(jobs_host, jobs_host + nj); int nb = 0; bool g = false;
    for (auto& J : H) { size_or_engine(J); nb = std::max(nb, (J.w/32)*(J.h/32)); g |= J.gw2 != nullptr; }
    SEL_CK(cudaMemcpyAsync(d, H.data(), nj*sizeof(HistJob), cudaMemcpyHostToDevice, st));
    auto hist = g ? sel_hist_kernel<true> : sel_hist_kernel<false>;
    SDV_LAUNCH_SYNC(hist, dim3(nb, nj), dim3(128), st, d, S);
    SDV_LAUNCH(sel_smooth_kernel, dim3((nb + 127)/128, nj), dim3(128), st, d);
    launches += 2; SEL_CK(cudaGetLastError());
    SEL_CK(cudaStreamSynchronize(st));                                                   // jobs_host / scr2 may be reused by the caller
    return 0;
  }

  static size_t pass_bytes(int pot, int n, bool lidar, int w, int h) {
    const int nbx4 = (w + 4*pot-1)/(4*pot), nby4 = (h + 4*pot-1)/(4*pot); const size_t ns = (size_t)nbx4*nby4*16;
    size_t b = 2*Scratch::need(ns, 4);                                                   // mask, n2start
    if (lidar) b += 2*Scratch::need(ns, 4) + 2*Scratch::need(n, 4) + Scratch::need(n, sizeof(PtRec));
    return b + 512;
  }
  // one select pass for the jobs listed in idx (all LiDAR or all dense), counters read back into n3[j][0..2]
  int select_pass(const std::vector<MapsJobHost*>& jobs, bool lidar, std::vector<int>& n3 /* 4 per job */) {
    const int nj = (int)jobs.size(); n3.assign((size_t)nj*4, 0);
    for (int j0 = 0; j0 < nj; ) {                                                        // chunks bounded by the scratch budget
      size_t bytes = Scratch::need(nj, sizeof(SelJob)) + Scratch::need((size_t)nj*4, 4); int j1 = j0;
      while (j1 < nj) { const size_t b = pass_bytes(*jobs[j1]->currentPotential, jobs[j1]->n, lidar, jobs[j1]->w, jobs[j1]->h); if (j1 > j0 && bytes + b > max_scratch) break; bytes += b; j1++; }
      if (scr.reserve(bytes, st)) { err = "scratch"; return -1; }
      scr.reset(); const int nc = j1 - j0; std::vector<SelJob> H(nc);
      SelJob* d = scr.take<SelJob>(nc); int* counters = scr.take<int>((size_t)nc*4);
      int maxSlots = 0, maxN = 0, maxBlk = 0; bool g = false; const size_t zero_from = scr.used;
      for (int k = 0; k < nc; k++) { MapsJobHost& M = *jobs[j0+k]; SelJob& J = H[k]; const int pot = *M.currentPotential, w = M.w, h = M.h;
        J.img = M.img; J.w = w; J.h = h; J.thsSm = M.thsSm; J.cloud = lidar ? M.cloud_dev : nullptr; J.n = lidar ? M.n : 0; J.pot = pot; J.thFactor = M.thFactor; J.active = 1; J.charTH = -1;
        J.numPotW = (w + pot-1)/pot; J.numPotH = (h + pot-1)/pot; J.nbx4 = (w + 4*pot-1)/(4*pot); J.nby4 = (h + 4*pot-1)/(4*pot); J.nslots = J.nbx4*J.nby4*16;
        J.mask = scr.take<int>(J.nslots); J.n2start = scr.take<int>(J.nslots); J.cnt = J.off = J.slot_of = J.list = nullptr; J.rec = nullptr;
        if (lidar) { J.cnt = scr.take<int>(J.nslots); J.off = scr.take<int>(J.nslots); J.slot_of = scr.take<int>(M.n); J.list = scr.take<int>(M.n); J.rec = scr.take<PtRec>(M.n); }
        J.map = M.map; J.counters = counters + 4*k; J.gw2 = M.gw2; g |= M.gw2 != nullptr;
        maxSlots = std::max(maxSlots, J.nslots); maxN = std::max(maxN, J.n); maxBlk = std::max(maxBlk, J.nbx4*J.nby4);
        SEL_CK(cudaMemsetAsync(J.map, 0, lidar ? (size_t)std::max(M.n, 1) : (size_t)w*h, st)); }
      SEL_CK(cudaMemsetAsync(counters, 0, (size_t)nc*4*sizeof(int), st));
      if (lidar) SEL_CK(cudaMemsetAsync(scr.p + zero_from, 0, scr.used - zero_from, st));  // cell histograms start at zero
      SEL_CK(cudaMemcpyAsync(d, H.data(), nc*sizeof(SelJob), cudaMemcpyHostToDevice, st));
      const int dd = S.selectDirectionDistribution;
      if (lidar) {
        auto point = g ? sel_point_kernel<true> : sel_point_kernel<false>;
        auto cell = g ? sel_cell_kernel<true, true> : sel_cell_kernel<true, false>;
        auto block = g ? sel_block_kernel<true, true> : sel_block_kernel<true, false>;
        if (maxN > 0) SDV_LAUNCH(point, dim3((maxN + 127)/128, nc), dim3(128), st, d);
        SDV_LAUNCH_SYNC(sel_scan_kernel, dim3(nc), dim3(256), st, d);
        if (maxN > 0) SDV_LAUNCH(sel_scatter_kernel, dim3((maxN + 127)/128, nc), dim3(128), st, d);
        SDV_LAUNCH(cell, dim3((maxSlots + 127)/128, nc), dim3(128), st, d, dd);
        SDV_LAUNCH_SYNC(sel_n2_kernel, dim3(nc), dim3(256), st, d, rp);
        SDV_LAUNCH(block, dim3((maxBlk + 127)/128, nc), dim3(128), st, d, rp, dd, S.gradDownweightPerLevel);
        launches += 6;
      } else {
        auto cell = g ? sel_cell_kernel<false, true> : sel_cell_kernel<false, false>;
        auto block = g ? sel_block_dense_kernel<true> : sel_block_dense_kernel<false>;
        SDV_LAUNCH(cell, dim3((maxSlots + 127)/128, nc), dim3(128), st, d, dd);
        SDV_LAUNCH_SYNC(sel_n2_kernel, dim3(nc), dim3(256), st, d, rp);
        SDV_LAUNCH_SYNC(block, dim3(maxBlk, nc), dim3(32), st, d, rp, dd, S.gradDownweightPerLevel);
        launches += 3;
      }
      SEL_CK(cudaGetLastError());
      SEL_CK(cudaMemcpyAsync(n3.data() + (size_t)j0*4, counters, (size_t)nc*4*sizeof(int), cudaMemcpyDeviceToHost, st));
      SEL_CK(cudaStreamSynchronize(st));
      j0 = j1;
    }
    return 0;
  }
  // makeMaps / makeMapsFromLidar for a batch (all LiDAR or all dense): the potential adaptation of :366-397 / :116-150 on the host (a handful of float operations per job),
  // the passes and the sub-selection on the device
  int make_maps(std::vector<MapsJobHost>& jobs, bool lidar) {
    const int nj = (int)jobs.size(); if (!nj) return 0;
    for (auto& M : jobs) size_or_engine(M);
    std::vector<float> numHave(nj, 0), quotia(nj, 0); std::vector<int> ideal(nj, 0), rec(nj); std::vector<MapsJobHost*> act;
    for (int j = 0; j < nj; j++) { rec[j] = jobs[j].recursionsLeft; jobs[j].passes = 0; act.push_back(&jobs[j]); }
    std::vector<int> actIdx(nj); for (int j = 0; j < nj; j++) actIdx[j] = j;
    while (!act.empty()) {
      std::vector<int> n3; if (select_pass(act, lidar, n3)) return -1;
      std::vector<MapsJobHost*> next; std::vector<int> nextIdx;
      for (size_t a = 0; a < act.size(); a++) { const int j = actIdx[a]; MapsJobHost& M = jobs[j]; M.passes++;
        int& cp = *M.currentPotential;
        numHave[j] = (float)(n3[4*a] + n3[4*a+1] + n3[4*a+2]);
        const float numWant = M.density; quotia[j] = numWant / numHave[j];
        const float K = numHave[j] * (cp+1) * (cp+1);
        int idealPotential = (int)(sqrtf(K/numWant)-1);
        if (idealPotential < 1) idealPotential = 1;
        ideal[j] = idealPotential;
        if (rec[j] > 0 && quotia[j] > 1.25 && cp > 1) { if (idealPotential >= cp) idealPotential = cp-1; cp = idealPotential; rec[j]--; next.push_back(&M); nextIdx.push_back(j); }
        else if (rec[j] > 0 && quotia[j] < 0.25) { if (idealPotential <= cp) idealPotential = cp+1; cp = idealPotential; rec[j]--; next.push_back(&M); nextIdx.push_back(j); }
      }
      act.swap(next); actIdx.swap(nextIdx);
    }
    // random sub-selection
    std::vector<SelJob> H(nj); bool any = false; int maxN = 0;
    for (int j = 0; j < nj; j++) { SelJob& J = H[j]; J = SelJob(); J.cloud = lidar ? jobs[j].cloud_dev : nullptr; J.n = lidar ? jobs[j].n : 0; J.map = jobs[j].map; J.charTH = -1;
      J.w = jobs[j].w; J.h = jobs[j].h;
      if (quotia[j] < 0.95) { J.charTH = (int)(unsigned char)(255*quotia[j]); any = true; } maxN = std::max(maxN, J.n); }
    std::vector<int> sub((size_t)nj*4, 0);
    if (any) {
      if (scr.reserve(Scratch::need(nj, sizeof(SelJob)) + Scratch::need((size_t)nj*4, 4) + Scratch::need((size_t)nj*h, 4), st)) { err = "scratch"; return -1; }
      scr.reset(); SelJob* d = scr.take<SelJob>(nj); int* counters = scr.take<int>((size_t)nj*4); int* rowcnt = scr.take<int>((size_t)nj*h);
      for (int j = 0; j < nj; j++) H[j].counters = counters + 4*j;
      SEL_CK(cudaMemsetAsync(counters, 0, (size_t)nj*4*sizeof(int), st));
      SEL_CK(cudaMemcpyAsync(d, H.data(), nj*sizeof(SelJob), cudaMemcpyHostToDevice, st));
      if (lidar) { if (maxN > 0) SDV_LAUNCH(sel_sub_lidar_kernel, dim3((maxN + 127)/128, nj), dim3(128), st, d, rp); launches += 1; }
      else { int maxH = 0; for (int j = 0; j < nj; j++) maxH = std::max(maxH, H[j].h);                                 // rowcnt rows at the stride h
        SDV_LAUNCH(sel_rowcount_kernel, dim3((maxH + 127)/128, nj), dim3(128), st, d, h, rowcnt); SDV_LAUNCH(sel_sub_dense_kernel, dim3((maxH + 127)/128, nj), dim3(128), st, d, rp, h, rowcnt); launches += 2; }
      SEL_CK(cudaGetLastError());
      SEL_CK(cudaMemcpyAsync(sub.data(), counters, (size_t)nj*4*sizeof(int), cudaMemcpyDeviceToHost, st));
      SEL_CK(cudaStreamSynchronize(st));
    }
    for (int j = 0; j < nj; j++) { jobs[j].numHaveSub = (int)numHave[j] - sub[4*j+3]; *jobs[j].currentPotential = ideal[j]; }
    return 0;
  }

  // ---- FullSystem::makeNewTraces for a batch of new keyframes (one per resident sequence)
  struct NewTracesJob {
    FrameImg img; int w = 0, h = 0; const double* cloud_host; int n; SelectorSlot* slot; float densityLidar, densityDense; int addFeaturePoint;   // w, h: the frame's size (= the slot's map)
    NewTrace* out_host; ImmPt* imm_host; int cap;                  // cap: room for the returned points (LiDAR + monocular)
    const double* cloud_dev = nullptr;                              // device-input path: the n rows are already on the device (cloud_host unused, nothing copied)
    int n_out, numPoints[2], passes[2];                             // out: points created, {numPointLidar, numPointMonocular}, select passes of the two makeMaps calls
    const float* gw2 = nullptr;                                     // the frame camera's gamma weights (SelJob::gw2)
    const NewTrace* out_dev = nullptr; const ImmPt* imm_dev = nullptr;   // out: the n_out records on the device (engine scratch, valid until the next engine call);
                                                                    // out_host == nullptr: they stay there (device-output path)
  };
  Scratch io;
  int make_new_traces(std::vector<NewTracesJob>& jobs) {
    const int nj = (int)jobs.size(); if (!nj) return 0;
    for (auto& N : jobs) size_or_engine(N);
    std::vector<size_t> o_ths(nj + 1, 0), o_occ(nj + 1, 0);                                 // per-job ths / thsSm pairs and occupancy masks, each at the job's size
    for (int j = 0; j < nj; j++) { o_ths[j+1] = o_ths[j] + 2*ths_floats(jobs[j].w, jobs[j].h); o_occ[j+1] = o_occ[j] + (size_t)jobs[j].w*jobs[j].h; }
    size_t bytes = Scratch::need(nj, sizeof(TraceJob)) + Scratch::need(nj, sizeof(HistJob)) + Scratch::need(o_ths[nj], 4) + Scratch::need(o_occ[nj], 1) + 8192;
    for (auto& j : jobs) bytes += (j.cloud_dev ? 0 : Scratch::need((size_t)3*j.n, 8)) + Scratch::need(std::max(j.n, 1), 1) + 3*Scratch::need(j.n, 4) + Scratch::need((size_t)j.w*j.h, 1)
                              + Scratch::need(j.cap, 4) + Scratch::need(j.cap, sizeof(NewTrace)) + Scratch::need(j.cap, sizeof(ImmPt)) + Scratch::need(4, 4);
    if (io.reserve(bytes, st)) { err = "scratch"; return -1; }
    io.reset(); std::vector<TraceJob> T(nj); std::vector<HistJob> Hj(nj); std::vector<MapsJobHost> ML, MD;
    TraceJob* dT = io.take<TraceJob>(nj);
    // per-type arrays of all jobs back to back: one memset / one upload per call instead of one per keyframe
    float* ths_all = io.take<float>(o_ths[nj]); unsigned char* occ_all = io.take<unsigned char>(o_occ[nj]); int* counts_all = io.take<int>((size_t)4*nj);
    size_t tot_cl = 0; for (auto& j : jobs) if (!j.cloud_dev) tot_cl += (size_t)3*std::max(j.n, 0);
    double* cl_all = io.take<double>(std::max(tot_cl, (size_t)1)); size_t off = 0;
    SEL_CK(cudaMemsetAsync(ths_all, 0, o_ths[nj]*sizeof(float), st)); SEL_CK(cudaMemsetAsync(occ_all, 0, o_occ[nj], st));
    std::vector<int> c0((size_t)4*nj, 0); for (int j = 0; j < nj; j++) c0[4*j+3] = float_order_bits_host(-1000.0f);
    SEL_CK(cudaMemcpyAsync(counts_all, c0.data(), c0.size()*sizeof(int), cudaMemcpyHostToDevice, st));
    int maxWH = 0;
    for (int j = 0; j < nj; j++) { NewTracesJob& N = jobs[j]; TraceJob& J = T[j]; const size_t wh = (size_t)N.w*N.h, tf = ths_floats(N.w, N.h); maxWH = std::max(maxWH, (int)wh);
      if (!N.slot->mapD) { SEL_CK(cudaMalloc((void**)&N.slot->mapD, wh)); SEL_CK(cudaMemsetAsync(N.slot->mapD, 0, wh, st)); }   // FullSystem::selectionMap: persistent; zero at birth (the reference: uninitialised)
      const double* cl = N.cloud_dev ? N.cloud_dev : cl_all + off; unsigned char* mapL = io.take<unsigned char>(std::max(N.n, 1)); float* ths = ths_all + o_ths[j]; float* thsSm = ths + tf;
      if (N.n && !N.cloud_dev) {                              // clouds that follow each other in host memory (the C-ABI's layout) travel in ONE copy
        const bool starts_run = (j == 0) || !(jobs[j-1].n > 0 && jobs[j-1].cloud_host + 3*(size_t)jobs[j-1].n == N.cloud_host);
        if (starts_run) { int j2 = j; size_t run = (size_t)3*N.n; while (j2 + 1 < nj && jobs[j2+1].n > 0 && jobs[j2].cloud_host + 3*(size_t)jobs[j2].n == jobs[j2+1].cloud_host) { j2++; run += (size_t)3*jobs[j2].n; }
          SEL_CK(cudaMemcpyAsync(cl_all + off, N.cloud_host, run*sizeof(double), cudaMemcpyHostToDevice, st)); }
        off += (size_t)3*std::max(N.n, 0);
      }
      J.img = N.img; J.w = N.w; J.h = N.h; J.cloud = cl; J.n = N.n; J.mapL = mapL; J.mapD = N.slot->mapD; J.score = io.take<float>(N.n); J.flag = io.take<int>(N.n); J.pos = io.take<int>(N.n);
      J.occ = occ_all + o_occ[j]; J.state = io.take<unsigned char>(wh); J.cand = io.take<int>(N.cap); J.ncand_cap = N.cap;
      J.out = io.take<NewTrace>(N.cap); J.imm = io.take<ImmPt>(N.cap); J.cap = N.cap; J.counts = counts_all + 4*j;
      Hj[j] = HistJob{N.img.I0, ths, thsSm, N.w, N.h, N.gw2};
      MapsJobHost M; M.img = N.img; M.w = N.w; M.h = N.h; M.thsSm = thsSm; M.cloud_dev = cl; M.n = N.n; M.map = mapL; M.density = N.densityLidar; M.recursionsLeft = 1; M.thFactor = 1; M.currentPotential = &N.slot->currentPotential; M.gw2 = N.gw2;
      M.numHaveSub = 0; M.passes = 0; ML.push_back(M);
    }
    if (make_hists(nj, Hj.data())) return -1;
    if (make_maps(ML, true)) return -1;                                                   // makeMapsFromLidar(newFrame, ..., density, 1, false, 1, vCloudPixel)   FullSystem.cpp:1290
    std::vector<int> dj;
    for (int j = 0; j < nj; j++) { jobs[j].numPoints[0] = ML[j].numHaveSub; jobs[j].passes[0] = ML[j].passes; jobs[j].numPoints[1] = 0; jobs[j].passes[1] = 0;
      if (jobs[j].addFeaturePoint) { MapsJobHost M = ML[j]; M.map = jobs[j].slot->mapD; M.density = jobs[j].densityDense; MD.push_back(M); dj.push_back(j); } }
    if (make_maps(MD, false)) return -1;                                                  // makeMaps(newFrame, selectionMap, setting_desiredImmatureDensity)   :1293
    for (size_t k = 0; k < dj.size(); k++) { jobs[dj[k]].numPoints[1] = MD[k].numHaveSub; jobs[dj[k]].passes[1] = MD[k].passes; }
    int maxN = 0;
    for (int j = 0; j < nj; j++) { T[j].pot = jobs[j].slot->currentPotential; maxN = std::max(maxN, T[j].n); }
    SEL_CK(cudaMemcpyAsync(dT, T.data(), nj*sizeof(TraceJob), cudaMemcpyHostToDevice, st));
    if (maxN > 0) SDV_LAUNCH(nt_lidar_score_kernel, dim3((maxN + 127)/128, nj), dim3(128), st, dT, S);
    SDV_LAUNCH_SYNC(nt_scan_kernel, dim3(nj), dim3(256), st, dT);
    if (maxN > 0) SDV_LAUNCH(nt_lidar_emit_kernel, dim3((maxN + 127)/128, nj), dim3(128), st, dT, S);
    SDV_LAUNCH(nt_dense_state_kernel, dim3((maxWH + 127)/128, nj), dim3(128), st, dT, S);
    SDV_LAUNCH_SYNC(nt_dense_resolve_kernel, dim3(nj), dim3(256), st, dT, S);
    launches += 5; SEL_CK(cudaGetLastError());
    std::vector<int> counts((size_t)nj*4);
    SEL_CK(cudaMemcpyAsync(counts.data(), counts_all, counts.size()*sizeof(int), cudaMemcpyDeviceToHost, st));
    SEL_CK(cudaStreamSynchronize(st));
    for (int j = 0; j < nj; j++) { NewTracesJob& N = jobs[j]; N.n_out = counts[4*j] + counts[4*j+1];
      if (counts[4*j+2] >= N.cap || N.n_out > N.cap) { err = "make_new_traces: output capacity too small"; return -2; }
      N.out_dev = T[j].out; N.imm_dev = T[j].imm;
      if (N.n_out && N.out_host) { SEL_CK(cudaMemcpyAsync(N.out_host, T[j].out, (size_t)N.n_out*sizeof(NewTrace), cudaMemcpyDeviceToHost, st));
                     if (N.imm_host) SEL_CK(cudaMemcpyAsync(N.imm_host, T[j].imm, (size_t)N.n_out*sizeof(ImmPt), cudaMemcpyDeviceToHost, st)); } }
    SEL_CK(cudaStreamSynchronize(st));
    return 0;
  }
  static int float_order_bits_host(float f) { int b; memcpy(&b, &f, 4); return b >= 0 ? b : (b ^ 0x7FFFFFFF); }

  // ---- CoarseDistanceMap::makeDistanceMap + the candidate walk of activatePointsMT for a batch of sequences
  struct ActJob {
    int nHosts; const int* pt_begin; const float* KRKi; const float* Kt; const float* uvid;                        // host arrays; sources grouped by host keyframe
    int nCandHosts; const int* cand_begin; const float* cKRKi; const float* cKt; const float* cand4; float minActDist;
    int32_t* decision_host; float* map_host;                                                                       // out: per candidate 1 / 0 / -1; optional w1*h1 map after the walk
    int w1 = 0, h1 = 0;                                                                                            // level-1 size of the sequence's camera
    const float* cand4_dev = nullptr;                                                                              // device-input path: the cand4 rows already on the device
  };
  int activate(std::vector<ActJob>& jobs) {
    const int nj = (int)jobs.size(); if (!nj) return 0;
    for (auto& a : jobs) if (!a.w1) { a.w1 = w >> 1; a.h1 = h >> 1; }
    size_t n1max = 0; for (auto& a : jobs) n1max = std::max(n1max, (size_t)a.w1*a.h1);
    size_t bytes = Scratch::need(nj, sizeof(DistJob)) + 1024;
    for (auto& a : jobs) { const int np = a.pt_begin[a.nHosts], nc = a.nCandHosts ? a.cand_begin[a.nCandHosts] : 0;
      bytes += Scratch::need((size_t)a.w1*a.h1, 4) + Scratch::need(a.nHosts+1, 4) + Scratch::need(12*(size_t)a.nHosts, 4) + Scratch::need(3*(size_t)np, 4)
             + Scratch::need(a.nCandHosts+1, 4) + Scratch::need(12*(size_t)a.nCandHosts, 4) + Scratch::need(4*(size_t)nc, 4) + Scratch::need(3*(size_t)nc, 4) + Scratch::need(nc, 4) + 4096; }
    if (io.reserve(bytes, st)) { err = "scratch"; return -1; }
    io.reset(); std::vector<DistJob> D(nj); DistJob* dD = io.take<DistJob>(nj); int maxP = 0, maxC = 0;
    auto up = [&](const void* src, size_t n) -> void* { char* d = io.take<char>(std::max(n, (size_t)4)); if (n) cudaMemcpyAsync(d, src, n, cudaMemcpyHostToDevice, st); return d; };
    static const int zero1[1] = {0};
    for (int j = 0; j < nj; j++) { ActJob& a = jobs[j]; DistJob& J = D[j]; const int np = a.pt_begin[a.nHosts], nc = a.nCandHosts ? a.cand_begin[a.nCandHosts] : 0;
      J.d = io.take<int>((size_t)a.w1*a.h1); J.w1 = a.w1; J.h1 = a.h1; J.nHosts = a.nHosts;
      J.pt_begin = (const int*)up(a.pt_begin, (a.nHosts+1)*sizeof(int)); J.KRKi = (const float*)up(a.KRKi, 9*a.nHosts*sizeof(float)); J.Kt = (const float*)up(a.Kt, 3*a.nHosts*sizeof(float));
      J.uvid = (const float*)up(a.uvid, 3*(size_t)np*sizeof(float));
      J.nCandHosts = a.nCandHosts; J.cand_begin = (const int*)up(a.nCandHosts ? (const void*)a.cand_begin : (const void*)zero1, (a.nCandHosts+1)*sizeof(int));
      J.cKRKi = (const float*)up(a.cKRKi, 9*a.nCandHosts*sizeof(float)); J.cKt = (const float*)up(a.cKt, 3*a.nCandHosts*sizeof(float)); J.cand4 = a.cand4_dev ? a.cand4_dev : (const float*)up(a.cand4, 4*(size_t)nc*sizeof(float));
      J.minActDist = a.minActDist; J.proj = io.take<int>(3*(size_t)std::max(nc, 1)); J.decision = io.take<int>(std::max(nc, 1));
      maxP = std::max(maxP, np); maxC = std::max(maxC, nc); }
    SEL_CK(cudaMemcpyAsync(dD, D.data(), nj*sizeof(DistJob), cudaMemcpyHostToDevice, st));
    const int gpx = (int)std::min<size_t>((n1max + 255)/256, 1024);
    if (have_ev) cudaEventRecord(ev0, st);
    const size_t walk_smem = (((n1max + 3) >> 2) + 2048)*sizeof(int);                      // byte map + the two frontier lists, for the largest job
    const bool smem_ok = walk_smem <= max_walk_smem && SDV_SET_SMEM(act_walk_smem_kernel, walk_smem) == 0, fused = smem_ok && fuse_map;
    if (maxC > 0) SDV_LAUNCH(act_project_kernel, dim3((maxC + 127)/128, nj), dim3(128), st, dD);
    if (fused) {                                                                         // ONE kernel per call: distance map built, walked and written back from shared memory
      SDV_LAUNCH_SYNC_SMEM(act_walk_smem_kernel, dim3(nj), dim3(walk_threads), walk_smem, st, dD, 1); launches += 2;
    } else {                                                                             // 41 launches for the map (all SMs per ring), then the walk
      SDV_LAUNCH(dm_fill_kernel, dim3(gpx, nj), dim3(256), st, dD);
      if (maxP > 0) SDV_LAUNCH(dm_source_kernel, dim3((maxP + 127)/128, nj), dim3(128), st, dD);
      for (int k = 1; k < 40; k++) SDV_LAUNCH(dm_ring_kernel, dim3(gpx, nj), dim3(256), st, dD, k);
      launches += 41;
      if (maxC > 0) {
        if (smem_ok) SDV_LAUNCH_SYNC_SMEM(act_walk_smem_kernel, dim3(nj), dim3(walk_threads), walk_smem, st, dD, 0);
        else SDV_LAUNCH_SYNC(act_walk_kernel, dim3(nj), dim3(64), st, dD);               // image too large for the shared-memory map: global-memory walk
        launches += 2; }
    }
    if (have_ev) cudaEventRecord(ev1, st);
    SEL_CK(cudaGetLastError());
    std::vector<std::vector<int>> maps(nj);
    for (int j = 0; j < nj; j++) { ActJob& a = jobs[j]; const int nc = a.nCandHosts ? a.cand_begin[a.nCandHosts] : 0;
      if (nc && a.decision_host) SEL_CK(cudaMemcpyAsync(a.decision_host, D[j].decision, (size_t)nc*sizeof(int), cudaMemcpyDeviceToHost, st));
      if (a.map_host) { maps[j].resize((size_t)a.w1*a.h1); SEL_CK(cudaMemcpyAsync(maps[j].data(), D[j].d, maps[j].size()*sizeof(int), cudaMemcpyDeviceToHost, st)); } }
    SEL_CK(cudaStreamSynchronize(st));
    for (int j = 0; j < nj; j++) if (jobs[j].map_host) for (size_t i = 0; i < maps[j].size(); i++) jobs[j].map_host[i] = (float)maps[j][i];
    if (have_ev) cudaEventElapsedTime(&last_kernel_ms, ev0, ev1);
    return 0;
  }
};

}}  // namespace sdv::sel
