// sdv_kernels.cu — hand-written sm_90a (H100) kernels of the tracker path (compiled with --fmad=false; see DESIGN.md §4).
//
//   pyr_fused_kernel / grad_texel_kernel   FrameHessian::makeImages           HessianBlocks.cpp:107-167
//   coarse_res_gs_kernel                   CoarseTracker::calcRes + calcGSSSE  CoarseTracker.cpp:486-634, 427-484 (one fused pass)
//   track_cluster_kernel                   CoarseTracker::trackNewestCoarse    CoarseTracker.cpp:662-838 (whole coarse-to-fine LM
//                                          device-resident: one thread-block cluster per call, DSMEM all-reduce, per-CTA redundant solve)
//   (CoarseTracker::makeCoarseDepthL0, CoarseTracker.cpp:258-425, is sdv_coarse_depth.cu)
#include "sdv_kernels.cuh"
#include "sdv_warp_solve.cuh"
#include <cooperative_groups.h>
#include <atomic>
#include <cstdlib>
namespace cg = cooperative_groups;

namespace sdv {

// SM count of the current device (132 on an H100 SXM, 114 on an H100 PCIe): grid caps of the streaming kernels and of the step-wise calcRes+GS partials.
// Cached per device; every caller runs after cudaSetDevice(context device), so a context sizes its partials buffer and caps its grid with the same value.
static int num_sms() {
  static std::atomic<int> cache[64];
  int dev = 0; if (cudaGetDevice(&dev) != cudaSuccess) dev = 0;
  int n = (dev >= 0 && dev < 64) ? cache[dev].load(std::memory_order_relaxed) : 0;
  if (n <= 0) {
    if (cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev) != cudaSuccess || n <= 0) n = 1;
    if (dev >= 0 && dev < 64) cache[dev].store(n, std::memory_order_relaxed);
  }
  return n;
}

// ================================================================================================ pyramid
// Every level of a frame is a planar float intensity plane (level 0: the frame's I0; levels >= 1: the frame's `pyr` allocation, level l after levels
// 1..l-1 of the frame's own size).
// Packed {I,dx,dy,|grad|^2} texels are a derived cache that only keyframe-rate consumers build (grad_texel_kernel).
struct PyrBatch { const void* src; float* I0; float* pyr; int flags; int cam; int w, h; };   // per frame: level-0 input (float/u8; may equal I0), level-0 plane, planes of levels >= 1; flags bit0: photometric response applies (exposure > 0); cam: Undistort camera of a RAW input; w x h: the frame's (its camera's) size
static_assert(sizeof(PyrBatch) == sizeof(PyrBatchHost), "PyrBatch mirrors PyrBatchHost");

template <typename T> __device__ __forceinline__ float px_load(const T* p, int i);
template <> __device__ __forceinline__ float px_load<float>(const float* p, int i) { return __ldg(p + i); }
template <> __device__ __forceinline__ float px_load<unsigned char>(const unsigned char* p, int i) { return (float)__ldg(p + i); }
template <typename T> __device__ __forceinline__ float4 px_load4(const T* p, int i);         // 4 consecutive pixels, i a multiple of 4 on an aligned plane
template <> __device__ __forceinline__ float4 px_load4<float>(const float* p, int i) { return __ldg(reinterpret_cast<const float4*>(p + i)); }
template <> __device__ __forceinline__ float4 px_load4<unsigned char>(const unsigned char* p, int i) {
  const uchar4 v = __ldg(reinterpret_cast<const uchar4*>(p + i)); return make_float4((float)v.x, (float)v.y, (float)v.z, (float)v.w);
}

// gradient + pack of one texel of a planar intensity image (HessianBlocks.cpp:147-165); |grad|^2 carries the camera's gamma weight (gw2 == nullptr: none)
__device__ __forceinline__ float4 grad_texel(const float* __restrict__ I, int idx, int w, int h, const float* __restrict__ gw2) {
  const float c = __ldg(I + idx); float dx, dy, ab = 0.f;
  if (planar_grad(I, idx, w, h, dx, dy)) { ab = dx*dx + dy*dy; if (gw2) ab *= gamma_w2(c, gw2); }
  return make_float4(c, dx, dy, ab);
}
// packed texels of one level from its planar intensity, on demand (keyframes entering the BA window or the selector, debugging read-back); G: gw2 is set
template <bool G> __global__ void __launch_bounds__(256) grad_texel_kernel(const float* __restrict__ I, float4* __restrict__ out, int w, int h, const float* __restrict__ gw2_) {
  const int n = w*h; const float* gw2 = G ? gw2_ : nullptr;
  for (int idx = blockIdx.x*blockDim.x + threadIdx.x; idx < n; idx += gridDim.x*blockDim.x) out[idx] = grad_texel(I, idx, w, h, gw2);
}

// Undistort::undistort<unsigned char> (util/Undistort.cpp:341-435) fused with PhotometricUndistorter::processFrame (:177-214): one rectified level-0 pixel from the
// RAW mono8 wire image.  remapX/remapY are the tables of Undistort::readFromFile (:842-886; -1 = outside), the four taps go through the photometric stage
// (factor*v, or G[v] (* vignetteMapInv) with a response calibration and exposure > 0) and are blended in the reference's order (fmad off):
//   xxyy*src[1+wOrg] + (yy-xxyy)*src[wOrg] + (xx-xxyy)*src[1] + (1-xx-yy+xxyy)*src[0]
__device__ __forceinline__ float undist_tap(const unsigned char* __restrict__ raw, int i, const UndistortDev& U, bool photo) {
  const unsigned char v = __ldg(raw + i);
  if (!photo) return U.factor * (float)v;
  float r = __ldg(U.G + v);
  if (U.vignette) r *= __ldg(U.vignette + i);
  return r;
}
__device__ __forceinline__ float undist_px(const unsigned char* __restrict__ raw, int idx, const UndistortDev& U, bool photo) {
  float xx = __ldg(U.remapX + idx), yy = __ldg(U.remapY + idx);
  if (xx < 0) return 0.f;
  const int xxi = (int)xx, yyi = (int)yy;
  xx -= xxi; yy -= yyi;
  const float xxyy = xx*yy;
  const int o = xxi + yyi*U.wOrg;
  const float s0 = undist_tap(raw, o, U, photo), s1 = undist_tap(raw, o+1, U, photo), sw = undist_tap(raw, o+U.wOrg, U, photo), sw1 = undist_tap(raw, o+1+U.wOrg, U, photo);
  return xxyy*sw1 + (yy-xxyy)*sw + (xx-xxyy)*s1 + (1-xx-yy+xxyy)*s0;
}
// Each CTA serves one frame and reads that frame's camera entry once (the table is a __grid_constant__ parameter: indexed in place, never copied per thread).
__global__ void __launch_bounds__(256) pyr_remap0_kernel(const PyrBatch* __restrict__ batch, const __grid_constant__ UndistortCams cams) {
  const PyrBatch b = batch[blockIdx.y]; const UndistortDev U = cams.cam[b.cam]; const bool photo = (b.flags & 1) && U.G; const int n = b.w*b.h;
  for (int idx = blockIdx.x*blockDim.x + threadIdx.x; idx < n; idx += gridDim.x*blockDim.x) b.I0[idx] = undist_px(reinterpret_cast<const unsigned char*>(b.src), idx, U, photo);
}

// The whole pyramid of a frame in one pass (FrameHessian::makeImages, HessianBlocks.cpp:137-145): one CTA per (band of 2^(levels-1) level-0 rows, frame).
// The CTA reads its band of the level-0 input once, keeps levels 1..levels-2 of the band in shared memory and writes every level >= 1 to the frame's planes.
// Each pixel is 0.25f*(((a+b)+c)+d) of its 2x2 parent quad in the flat-index layout of the per-level filter (parent row 2y, columns 2x, 2x+1 of a level of
// width wlm1 at 2x + 2y*wlm1), so odd intermediate sizes drop the last column / row exactly as that filter did; a band past the last row of a coarse level
// simply has fewer (or no) rows there.  Level 0 comes from a float plane (resident or adopted), mono8, or RAW mono8 through its camera's Undistort tables (RAW),
// and is written to the frame's I0 plane whenever the input is not that plane already.
// Each frame has its own size b.w x b.h (its camera's); the grid covers the bands of the tallest frame, and the CTAs past a frame's last band exit.  Level l
// is written after levels 1..l-1 of that size, so a frame fits storage of its own size (a camera's pool) as well as the context's.
// P = level-1 pixels per work item: 2 reads each parent row as one 16-byte (float) / 4-byte (mono8) vector, 1 reads scalars (unaligned input or w % 4 != 0).
// The second bound keeps the register count of the offsets of the frame's own size at the parent layout's: 32 (8 CTAs per SM) for the plane inputs, 40 for RAW.
constexpr int kPyrThreads = 256;
template <typename T, bool RAW, int P>
__global__ void __launch_bounds__(kPyrThreads, RAW ? 6 : 8) pyr_fused_kernel(const PyrBatch* __restrict__ batch, const __grid_constant__ UndistortCams cams, int levels) {
  extern __shared__ float pyr_band[];                       // levels 1..levels-2 of the band: [R1][w1] [R1/2][w2] ...
  const PyrBatch b = batch[blockIdx.y];
  const int w = b.w, R1 = 1 << (levels - 2);                // R1: level-1 rows per band
  const int w1 = w >> 1, h1 = b.h >> 1, y1 = blockIdx.x*R1, n1 = min(R1, h1 - y1);
  if (n1 <= 0) return;                                      // past this frame's last band (a taller frame sized the grid)
  UndistortDev U{};
  if constexpr (RAW) U = cams.cam[b.cam];                   // RAW: this frame's camera
  const T* src = reinterpret_cast<const T*>(b.src);
  float* I0 = (RAW || reinterpret_cast<const void*>(b.I0) != b.src) ? b.I0 : nullptr;
  const bool photo = RAW && (b.flags & 1) && U.G;
  const bool keep = levels > 2;
  {
    const int items = w1 / P;
    for (int k = threadIdx.x; k < n1*items; k += kPyrThreads) {
      const int rr = k / items, x = (k - rr*items)*P, y = y1 + rr;
      const int bi = 2*x + 2*y*w;
      float t[2*P], u[2*P];                                 // parent rows 2y and 2y+1, columns 2x .. 2x+2P-1
      if constexpr (RAW) {
#pragma unroll
        for (int j = 0; j < 2*P; j++) { t[j] = undist_px(reinterpret_cast<const unsigned char*>(src), bi + j, U, photo); u[j] = undist_px(reinterpret_cast<const unsigned char*>(src), bi + w + j, U, photo); }
      } else if constexpr (P == 2) {
        const float4 a = px_load4<T>(src, bi), c = px_load4<T>(src, bi + w);
        t[0] = a.x; t[1] = a.y; t[2] = a.z; t[3] = a.w; u[0] = c.x; u[1] = c.y; u[2] = c.z; u[3] = c.w;
      } else {
#pragma unroll
        for (int j = 0; j < 2*P; j++) { t[j] = px_load<T>(src, bi + j); u[j] = px_load<T>(src, bi + w + j); }
      }
      float v[P];
#pragma unroll
      for (int j = 0; j < P; j++) v[j] = 0.25f * (((t[2*j] + t[2*j+1]) + u[2*j]) + u[2*j+1]);
      if constexpr (P == 2) {
        *reinterpret_cast<float2*>(b.pyr + y*w1 + x) = make_float2(v[0], v[1]);
        if (keep) *reinterpret_cast<float2*>(pyr_band + rr*w1 + x) = make_float2(v[0], v[1]);
      } else {
        b.pyr[y*w1 + x] = v[0];
        if (keep) pyr_band[rr*w1 + x] = v[0];
      }
      if (I0) {
        if constexpr (P == 2) { *reinterpret_cast<float4*>(I0 + bi) = make_float4(t[0], t[1], t[2], t[3]); *reinterpret_cast<float4*>(I0 + bi + w) = make_float4(u[0], u[1], u[2], u[3]); }
        else {
#pragma unroll
          for (int j = 0; j < 2*P; j++) { I0[bi + j] = t[j]; I0[bi + w + j] = u[j]; }
        }
      }
    }
  }
  const float* prev = pyr_band; float* cur = pyr_band + (size_t)R1*w1;
  int wp = w1, hp = h1; size_t off = (size_t)w1*h1;          // off: level l's offset in the frame's pyr
  for (int l = 2; l < levels; l++) {
    __syncthreads();
    const int wl = wp >> 1, hl = hp >> 1, Rl = R1 >> (l - 1), yl = blockIdx.x*Rl, nl = min(Rl, hl - yl);
    const bool keep_l = l + 1 < levels;
    float* out = b.pyr + off;
    for (int k = threadIdx.x; k < nl*wl; k += kPyrThreads) {
      const int rr = k / wl, x = k - rr*wl;
      const float* s = prev + 2*rr*wp + 2*x;                // band-local parent rows 2rr, 2rr+1
      const float v = 0.25f * (((s[0] + s[1]) + s[wp]) + s[wp+1]);
      out[(size_t)(yl + rr)*wl + x] = v;
      if (keep_l) cur[rr*wl + x] = v;
    }
    prev = cur; cur += (size_t)Rl*wl; off += (size_t)wl*hl; wp = wl; hp = hl;
  }
}
static size_t pyr_band_bytes(int w, int levels) {
  size_t n = 0; const int R1 = 1 << (levels - 2);
  for (int l = 1; l + 1 < levels; l++) n += (size_t)(R1 >> (l - 1))*(w >> l);
  return n*sizeof(float);
}
template <typename T, bool RAW, int P>
static void launch_pyr_fused(const PyrBatch* batch_dev, int nframes, int max_w, int max_h, int levels, const UndistortCams& U, cudaStream_t st) {
  const size_t smem = pyr_band_bytes(max_w, levels);
  if (smem > 48*1024) cudaFuncSetAttribute(pyr_fused_kernel<T, RAW, P>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);   // very wide images; a refusal surfaces as the launch error
  const int R1 = 1 << (levels - 2);
  dim3 g(((max_h >> 1) + R1 - 1)/R1, nframes);
  pyr_fused_kernel<T, RAW, P><<<g, kPyrThreads, smem, st>>>(batch_dev, U, levels);
}

// batch_dev: nframes PyrBatch descriptors in device memory.  src_u8: level-0 input is mono8 (sensor_msgs/Image wire format) instead of float.
// vec: every level-0 input (and I0 plane written) of the batch is 16-byte aligned and every frame's w % 4 == 0 (the 4-pixel vector path).
// Requires even w,h whenever levels > 1 (pyrLevelsUsed only halves even sizes, globalCalib.cpp:24).
void launch_pyramid_batch(const void* batch_dev_v, int nframes, bool src_u8, bool vec, int max_w, int max_h, int levels, cudaStream_t st, const UndistortCams* und) {
  const PyrBatch* batch_dev = reinterpret_cast<const PyrBatch*>(batch_dev_v);
  if (nframes <= 0 || levels < 2) return;
  const UndistortCams U = und ? *und : UndistortCams{};
  if (und) launch_pyr_fused<unsigned char, true, 1>(batch_dev, nframes, max_w, max_h, levels, U, st);
  else if (src_u8) { if (vec) launch_pyr_fused<unsigned char, false, 2>(batch_dev, nframes, max_w, max_h, levels, U, st); else launch_pyr_fused<unsigned char, false, 1>(batch_dev, nframes, max_w, max_h, levels, U, st); }
  else             { if (vec) launch_pyr_fused<float, false, 2>(batch_dev, nframes, max_w, max_h, levels, U, st);         else launch_pyr_fused<float, false, 1>(batch_dev, nframes, max_w, max_h, levels, U, st); }
}
// levels == 1: the level-0 plane still has to be materialised from a foreign / mono8 source
template <typename T> __global__ void pyr_copy0_kernel(const PyrBatch* __restrict__ batch) {
  const PyrBatch b = batch[blockIdx.y]; if (reinterpret_cast<const void*>(b.I0) == b.src) return;
  const int n = b.w*b.h;
  for (int idx = blockIdx.x*blockDim.x + threadIdx.x; idx < n; idx += gridDim.x*blockDim.x) b.I0[idx] = px_load<T>(reinterpret_cast<const T*>(b.src), idx);
}
void launch_pyramid_copy0(const void* batch_dev_v, int nframes, bool src_u8, int max_w, int max_h, cudaStream_t st, const UndistortCams* und) {
  const PyrBatch* batch_dev = reinterpret_cast<const PyrBatch*>(batch_dev_v); if (nframes <= 0) return;
  const int n = max_w*max_h;
  dim3 g((n + 255)/256 > 1024 ? 1024 : (n + 255)/256, nframes);
  if (und) pyr_remap0_kernel<<<g, 256, 0, st>>>(batch_dev, *und);
  else if (src_u8) pyr_copy0_kernel<unsigned char><<<g, 256, 0, st>>>(batch_dev); else pyr_copy0_kernel<float><<<g, 256, 0, st>>>(batch_dev);
}
void launch_grad_texels(const float* I, float4* out, int w, int h, const float* gw2, cudaStream_t st) {
  int n = w*h; int grid = (n + 255)/256; if (grid > num_sms()*16) grid = num_sms()*16;
  if (gw2) grad_texel_kernel<true><<<grid, 256, 0, st>>>(I, out, w, h, gw2); else grad_texel_kernel<false><<<grid, 256, 0, st>>>(I, out, w, h, nullptr);
}

__global__ void unpack_level_kernel(const float4* __restrict__ in, float* dI3, float* ab, int n) {
  int i = blockIdx.x*blockDim.x + threadIdx.x; if (i >= n) return;
  float4 t = in[i];
  if (dI3) { dI3[3*i] = t.x; dI3[3*i+1] = t.y; dI3[3*i+2] = t.z; }
  if (ab) ab[i] = t.w;
}
void launch_unpack_level(const float4* in, float* dI3, float* ab, int n, cudaStream_t st) {
  unpack_level_kernel<<<(n+255)/256, 256, 0, st>>>(in, dI3, ab, n);
}

// ================================================================================================ reductions
// Deterministic CTA reduction of the 51 per-thread partial sums: transpose through shared memory, each warp owns rows,
// 8 serial adds + xor-butterfly in double.  Fixed order => bit-reproducible run to run.
template <int THREADS>
__device__ __forceinline__ void block_reduce_acc(const float (&acc)[kNAcc], float* red, double* out) {
  const int tid = threadIdx.x;
#pragma unroll
  for (int k = 0; k < kNAcc; k++) red[k*THREADS + tid] = acc[k];
  __syncthreads();
  const int warp = tid >> 5, lane = tid & 31; constexpr int NW = THREADS/32;
  for (int k = warp; k < kNAcc; k += NW) {
    double s = 0;
#pragma unroll
    for (int j = 0; j < NW; j++) s += (double)red[k*THREADS + lane + 32*j];
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
    if (lane == 0) out[k] = s;
  }
  __syncthreads();
}

// ================================================================================================ step-wise fused calcRes+calcGSSSE
// grid-stride over the reference cloud; per-block partials -> global; the last block to finish (ticket) sums the block
// partials in block order and writes the 51 totals.  One launch per calcRes.
template <int THREADS>
__global__ void __launch_bounds__(THREADS) coarse_res_gs_kernel(const float4* __restrict__ pts, int n, const float* __restrict__ I,
                                                               LevelGeom g, EvalParams ep, double* __restrict__ partials,
                                                               unsigned int* __restrict__ ticket, double* __restrict__ totals) {
  extern __shared__ __align__(16) unsigned char smem_raw[];
  float* red = reinterpret_cast<float*>(smem_raw);
  __shared__ double bsum[kNAcc];
  __shared__ bool is_last;
  float acc[kNAcc];
#pragma unroll
  for (int k = 0; k < kNAcc; k++) acc[k] = 0.f;
  {
    const int stride = gridDim.x*THREADS; int i = blockIdx.x*THREADS + threadIdx.x;
    const float4 zero4 = make_float4(0.f, 0.f, 0.f, 0.f);
    float4 pc = (i < n) ? __ldg(pts + i) : zero4;
    float4 pn = (i + stride < n) ? __ldg(pts + i + stride) : zero4;
    for (; i < n; i += stride) {
      const float4 pn2 = (i + 2*stride < n) ? __ldg(pts + i + 2*stride) : zero4;
      eval_point(pc, i, g, ep, I, acc);
      pc = pn; pn = pn2;
    }
  }
  block_reduce_acc<THREADS>(acc, red, bsum);
  if (threadIdx.x < kNAcc) partials[(size_t)blockIdx.x*kNAcc + threadIdx.x] = bsum[threadIdx.x];
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) { unsigned int t = atomicAdd(ticket, 1u); is_last = (t == gridDim.x - 1); }
  __syncthreads();
  if (is_last) {
    __threadfence();
    if (threadIdx.x < kNAcc) {
      double s = 0; for (unsigned int b = 0; b < gridDim.x; b++) s += __ldcg(partials + (size_t)b*kNAcc + threadIdx.x);
      totals[threadIdx.x] = s;
    }
    if (threadIdx.x == 0) *ticket = 0;
  }
}

constexpr int kStepThreads = 256;
int step_kernel_max_grid() { return num_sms()*4; }
void launch_coarse_res_gs(const float4* pts, int n, const float* I, const LevelGeom& g, const EvalParams& ep,
                          double* partials, unsigned int* ticket, double* totals, cudaStream_t st) {
  size_t smem = (size_t)kNAcc*kStepThreads*sizeof(float);                // opt-in size set per device by kernels_init_device()
  int grid = (n + kStepThreads - 1)/kStepThreads; if (grid < 1) grid = 1; if (grid > step_kernel_max_grid()) grid = step_kernel_max_grid();
  coarse_res_gs_kernel<kStepThreads><<<grid, kStepThreads, smem, st>>>(pts, n, I, g, ep, partials, ticket, totals);
}

// ================================================================================================ device-resident LM
constexpr int kMaxCluster = 16;

// ================================================================================================ device-resident LM
// One trackNewestCoarse per cluster of CTAs, the whole coarse-to-fine LM on the device.  THREADS x MINB is chosen so that several jobs are resident per SM:
// one job's (single-warp, latency-bound) LM control step overlaps the point sweeps of the others.  <128,4> is the batched-throughput configuration
// (cluster size 1); <256,1> with a cluster of 8-16 CTAs is the low-latency single-sequence configuration.  No load ever stalls a warp on HBM:
//   * the reference cloud streams through shared memory in chunks: one elected thread issues cp.async.bulk (TMA bulk copy, SASS UBLKCP) per
//     2 KB block of float4 points, completion is signalled on an mbarrier (expect_tx), two chunks in flight;
//   * the 12-tap planar footprint of point k+1 (bilinear 2x2 plus the neighbours its central differences need) is gathered by per-thread cp.async
//     (SASS LDGSTS) into a private shared-memory slot while point k is accumulated — the gather needs no registers and is complete one full iteration later;
//   * the level-0 flow indicators (every 32nd point, CoarseTracker.cpp:538-566) are a dense pre-pass (all lanes busy) instead of a divergent branch
//     that cost one lane's 6 divisions per warp iteration;
//   * the LM control flow is a state machine around ONE instance of the sweep.
__device__ __forceinline__ uint32_t smem_u32(const void* p) { return (uint32_t)__cvta_generic_to_shared(p); }
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) { asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" :: "r"(smem_u32(bar)), "r"(count) : "memory"); }
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
  asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" :: "r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
#if defined(SDV_MBAR_SPIN)          // non-blocking test_wait poll
  uint32_t done = 0;
  while (!done) asm volatile("{\n\t.reg .pred p;\n\tmbarrier.test_wait.parity.shared::cta.b64 p, [%1], %2;\n\tselp.u32 %0, 1, 0, p;\n\t}" : "=r"(done) : "r"(smem_u32(bar)), "r"(parity) : "memory");
#elif defined(SDV_MBAR_HINT_NS)     // try_wait with an explicit suspend-time hint
  asm volatile("{\n\t.reg .pred p;\n\tSDV_WAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1, %2;\n\t@p bra SDV_DONE_%=;\n\tbra SDV_WAIT_%=;\n\tSDV_DONE_%=:\n\t}"
               :: "r"(smem_u32(bar)), "r"(parity), "r"((uint32_t)SDV_MBAR_HINT_NS) : "memory");
#else
  asm volatile("{\n\t.reg .pred p;\n\tSDV_WAIT_%=:\n\tmbarrier.try_wait.parity.shared::cta.b64 p, [%0], %1;\n\t@p bra SDV_DONE_%=;\n\tbra SDV_WAIT_%=;\n\tSDV_DONE_%=:\n\t}"
               :: "r"(smem_u32(bar)), "r"(parity) : "memory");
#endif
}
__device__ __forceinline__ void bulk_g2s(void* dst, const void* src, uint32_t bytes, uint64_t* bar) {
  asm volatile("cp.async.bulk.shared::cluster.global.mbarrier::complete_tx::bytes [%0], [%1], %2, [%3];"
               :: "r"(smem_u32(dst)), "l"(src), "r"(bytes), "r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void cp_async4(uint32_t s, const void* g)  { asm volatile("cp.async.ca.shared.global [%0], [%1], 4;" :: "r"(s), "l"(g) : "memory"); }
__device__ __forceinline__ void cp_async_commit() { asm volatile("cp.async.commit_group;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait1()  { asm volatile("cp.async.wait_group 1;" ::: "memory"); }
__device__ __forceinline__ void cp_async_wait0()  { asm volatile("cp.async.wait_group 0;" ::: "memory"); }

struct PtState { ProjPt q; float dx, dy, col; bool ok; };    // what the accumulate stage needs of a projected point (its taps are in the thread's smem slot)

// calcRes, first half (CoarseTracker.cpp:525-575): projection + bounds, then launch the gather of the 12-tap planar footprint into `slot`.
constexpr int kTaps = 12;
template <int THREADS>
__device__ __forceinline__ PtState stage_project(const float4 p, const LevelGeom& g, const EvalParams& ep, const float* __restrict__ I, uint32_t slot) {
  PtState s; s.col = p.w;
  s.q = project_point(p, g, ep);
  s.ok = proj_inside(s.q, g);
  s.dx = 0.f; s.dy = 0.f;
  if (s.ok) {
    const int ix = (int)s.q.Ku, iy = (int)s.q.Kv, w = g.w;
    s.dx = s.q.Ku - ix; s.dy = s.q.Kv - iy;
    const float* b = I + ix + iy*w;                         // rows -1..2 in accumulate_point's tap order
    cp_async4(slot + 0*THREADS*4, b - w);       cp_async4(slot + 1*THREADS*4, b - w + 1);
    cp_async4(slot + 2*THREADS*4, b - 1);       cp_async4(slot + 3*THREADS*4, b);         cp_async4(slot + 4*THREADS*4, b + 1);     cp_async4(slot + 5*THREADS*4, b + 2);
    cp_async4(slot + 6*THREADS*4, b + w - 1);   cp_async4(slot + 7*THREADS*4, b + w);     cp_async4(slot + 8*THREADS*4, b + w + 1); cp_async4(slot + 9*THREADS*4, b + w + 2);
    cp_async4(slot + 10*THREADS*4, b + 2*w);    cp_async4(slot + 11*THREADS*4, b + 2*w + 1);
  }
  return s;
}
// calcRes second half + calcGSSSE for one point whose taps have landed (CoarseTracker.cpp:576-601, 442-466)
template <int THREADS>
__device__ __forceinline__ void stage_accumulate(const PtState s, const LevelGeom& g, const EvalParams& ep, const float* slot, float (&acc)[kNAcc]) {
  if (!s.ok) return;
  accumulate_point([&](int k) { return slot[k*THREADS]; }, s.dx, s.dy, s.q, s.col, g, ep, acc);
}

#ifdef SDV_TRACK_PROFILE
__device__ long long g_track_prof[16];
#ifndef SDV_PROF_MASK
#define SDV_PROF_MASK 0xffff
#endif
#define SDV_PROF_T(var) long long var = ((SDV_PROF_MASK >> __COUNTER__) & 1) ? clock64() : 0
#define SDV_PROF_ADD(slot, t0, t1) do { if (blockIdx.x == 0 && threadIdx.x == 0) g_track_prof[slot] += (t1) - (t0); } while (0)
#else
#define SDV_PROF_T(var) do {} while (0)
#define SDV_PROF_ADD(slot, t0, t1) do {} while (0)
#endif
#ifndef SDV_TRACK_STAGGER_DEFAULT_NS
#define SDV_TRACK_STAGGER_DEFAULT_NS 0
#endif
constexpr int kPtChunk = 4;                                 // sweep iterations (blocks of THREADS points) per TMA-staged chunk.  Larger chunks cost the 4th resident CTA; per-WARP
                                                            // streams with __syncwarp instead of the block barrier let the warps drift apart

struct Ctl2 {                                               // per-CTA LM state (every CTA of a cluster computes it redundantly and identically)
  SE3d cur; double a_cur, b_cur;
  SE3d cand; double a_cand, b_cand;
  double H[64], b[8];
  double resOld[6], resNew[6];
  double lastRes[5], flow[3];
  double incn;
  float lambda, lcr;                                        // LM damping, levelCutoffRepeat
  int lvl, mode, iteration, haveRepeated, aborted, done;
  long long evals[kLevels]; int iters[kLevels], accs[kLevels];
  EvalParams ep;
};
__constant__ unsigned char kAccRow[45] = {0,0,0,0,0,0,0,0,0, 1,1,1,1,1,1,1,1, 2,2,2,2,2,2,2, 3,3,3,3,3,3, 4,4,4,4,4, 5,5,5,5, 6,6,6, 7,7, 8};
__constant__ unsigned char kAccCol[45] = {0,1,2,3,4,5,6,7,8, 1,2,3,4,5,6,7,8, 2,3,4,5,6,7,8, 3,4,5,6,7,8, 4,5,6,7,8, 5,6,7,8, 6,7,8, 7,8, 8};

template <int THREADS, int MINB>
__global__ void __launch_bounds__(THREADS, MINB) track_cluster_kernel(TrackJob* __restrict__ jobs, const TrackConst* __restrict__ tc_g, const GeomRow* __restrict__ geom_tab,
                                                                unsigned stagger_ns) {
  cg::cluster_group cluster = cg::this_cluster();
  const int C = (int)cluster.num_blocks();
  const int rank = (int)cluster.block_rank();
  const int tid = threadIdx.x;
  TrackJob& J = jobs[blockIdx.x / C];
  // Phase stagger: the MINB jobs co-resident on an SM run the same program on similar data and would reach their single-warp LM control steps
  // together, leaving the SM idle; CTAs are dealt round-robin over the SMs, so wave j of the grid (blockIdx / #SMs-worth) starts j*stagger_ns late
  // and one job's control step overlaps the other jobs' sweeps.
  if (stagger_ns && C == 1) {                               // only the first resident set is delayed; CTAs that start later are desynchronised by their predecessors
    unsigned nsm; asm("mov.u32 %0, %%nsmid;" : "=r"(nsm));
    const unsigned wave = (blockIdx.x < nsm*MINB) ? (blockIdx.x / nsm) % MINB : 0u;
    for (unsigned k = 0; k < wave; k++) __nanosleep(stagger_ns);
  }

  // dynamic smem: [ tap ring 2 x kTaps x THREADS x 4 B | point chunks 2 x kPtChunk x THREADS x 16 B ] aliased by the reduction scratch [kNAcc][THREADS] floats,
  // then the DSMEM gather buffers and the reduced sums
  extern __shared__ __align__(128) unsigned char smem_raw[];
  constexpr size_t kRingBytes = (size_t)2*kTaps*THREADS*4, kPtsBytes = (size_t)2*kPtChunk*THREADS*16, kRedBytes = (size_t)kNAcc*THREADS*sizeof(float);
  constexpr size_t kStageBytes = (kRingBytes + kPtsBytes) > kRedBytes ? (kRingBytes + kPtsBytes) : kRedBytes;
  unsigned char* ring = smem_raw;
  float4* pbuf   = reinterpret_cast<float4*>(smem_raw + kRingBytes);
  float*  red    = reinterpret_cast<float*>(smem_raw);
  double* gather = reinterpret_cast<double*>(smem_raw + kStageBytes);                    // [2][C][kNAcc] — sized by the launch's cluster size (13 KB at 16 CTAs, 0.8 KB at 1)
  double* bsum   = gather + 2*C*kNAcc;                                                   // [kNAcc]
  double* tot    = bsum + kNAcc;                                                         // [kNAcc]
  __shared__ Ctl2 ctl;
  __shared__ TrackConst tc;
  __shared__ GeomRow geom;                                  // the job's row of the geometry table: the K of its tracker slot at every level
  __shared__ __align__(8) uint64_t full_bar[2];
  for (int i = tid; i < (int)(sizeof(TrackConst)/4); i += THREADS) reinterpret_cast<int*>(&tc)[i] = reinterpret_cast<const int*>(tc_g)[i];
  { const int* __restrict__ row = reinterpret_cast<const int*>(geom_tab + J.geom_row);
    for (int i = tid; i < (int)(sizeof(GeomRow)/4); i += THREADS) reinterpret_cast<int*>(&geom)[i] = row[i]; }
  if (tid == 0) {
    ctl.cur = se3_from7(J.T); ctl.a_cur = J.ab[0]; ctl.b_cur = J.ab[1];
    for (int i = 0; i < 5; i++) ctl.lastRes[i] = nan("");
    for (int i = 0; i < 3; i++) ctl.flow[i] = 1000.0;
    for (int i = 0; i < kLevels; i++) { ctl.evals[i] = 0; ctl.iters[i] = 0; ctl.accs[i] = 0; }
    ctl.lvl = J.coarsest; ctl.mode = 0; ctl.iteration = 0; ctl.haveRepeated = 0; ctl.aborted = 0; ctl.done = 0; ctl.lcr = 1.0f; ctl.lambda = 0.01f; ctl.incn = 0;
    mbar_init(&full_bar[0], 1); mbar_init(&full_bar[1], 1);
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
  }
  __syncthreads();
  if (tid == 0) make_eval_params(ctl.cur, ctl.a_cur, ctl.b_cur, J.refExposure, J.newExposure, J.ref_a, J.ref_b, geom.g[ctl.lvl], ctl.lvl,
                                 tc.coarseCutoffTH*ctl.lcr, tc.huberTH, ctl.ep);
  __syncthreads();
  if (C > 1) cluster.sync();                                // every CTA of the cluster must be running before the first distributed-shared-memory write

  int evalCount = 0;
  uint32_t bar_phase = 0;                                   // bit b = parity the next wait on full_bar[b] expects
  const int stride = C*THREADS;
  const uint32_t slot_base = smem_u32(ring) + tid*4;        // [slot][tap 0..11][tid] float
  constexpr uint32_t kSlotStride = kTaps*THREADS*4;

  while (true) {
    const int lvl = ctl.lvl; int n_eval = 0;
    // ------------------------------------------------------------------ one calcRes + calcGSSSE sweep at ctl.ep
    float acc[kNAcc];
#pragma unroll
    for (int k = 0; k < kNAcc; k++) acc[k] = 0.f;
    {
      const float4* __restrict__ pts = J.pts[lvl]; const int n = J.npts[lvl];
      const float* __restrict__ I = J.img[lvl];
      // the sweep's operands as register copies: the cp.async / mbarrier asm below clobbers "memory", which would reload them from shared memory for every point
      const LevelGeom g = geom.g[lvl];
      const EvalParams ep = ctl.ep;
      const int K = (n + stride - 1)/stride;                // sweep iterations (uniform over the CTA)
      const int NC = (K + kPtChunk - 1)/kPtChunk;           // point chunks
      auto issue_chunk = [&](int c) {                       // thread 0: TMA bulk copies of chunk c's (<= kPtChunk) blocks into buffer c&1
        const int b = c & 1; uint32_t bytes = 0; int cnt[kPtChunk];
#pragma unroll
        for (int j = 0; j < kPtChunk; j++) {
          const int base = (c*kPtChunk + j)*stride + rank*THREADS; int m = n - base; m = m < 0 ? 0 : (m > THREADS ? THREADS : m);
          cnt[j] = m; bytes += (uint32_t)m*16u;
        }
        mbar_expect_tx(&full_bar[b], bytes);
#pragma unroll
        for (int j = 0; j < kPtChunk; j++) if (cnt[j] > 0)
          bulk_g2s(pbuf + (b*kPtChunk + j)*THREADS, pts + (size_t)(c*kPtChunk + j)*stride + rank*THREADS, (uint32_t)cnt[j]*16u, &full_bar[b]);
      };
      SDV_PROF_T(tp0);
#ifndef SDV_PTS_LDG
      if (tid == 0) { if (NC > 0) issue_chunk(0); if (NC > 1) issue_chunk(1); }
#endif
      SDV_PROF_T(tp1); SDV_PROF_ADD(0, tp0, tp1);
      if (lvl == 0) {                                       // dense flow-indicator pre-pass: point indices 0, 32, 64, ...
        for (int j = rank*THREADS + tid; 32*j < n; j += stride) flow_point(__ldg(pts + 32*j), g, ep, acc);
      }
      PtState sN; sN.ok = false; sN.q.u = sN.q.v = sN.q.nid = sN.dx = sN.dy = sN.col = 0.f;
      auto project = [&](int m) {                           // stage A for sweep iteration m (its chunk has landed)
        const int i = m*stride + rank*THREADS + tid;
        PtState s; s.ok = false; s.q.u = s.q.v = s.q.nid = s.dx = s.dy = s.col = 0.f;
        if (i < n) {
#ifdef SDV_PTS_LDG
          const float4 p = __ldg(pts + i);
#else
          const float4 p = pbuf[(((m/kPtChunk) & 1)*kPtChunk + (m % kPtChunk))*THREADS + tid];
#endif
          const uint32_t so = (uint32_t)(m & 1)*kSlotStride;
          s = stage_project<THREADS>(p, g, ep, I, slot_base + so);
        }
        return s;
      };
      SDV_PROF_T(tp2); SDV_PROF_ADD(1, tp1, tp2);
#ifdef SDV_PTS_LDG
      if (K > 0) sN = project(0);
#else
      if (K > 0) { mbar_wait(&full_bar[0], bar_phase & 1u); bar_phase ^= 1u; sN = project(0); }
#endif
      cp_async_commit();
      SDV_PROF_T(tp3); SDV_PROF_ADD(2, tp2, tp3);
      for (int k = 0; k < K; k++) {
        const PtState sC = sN;
        const int m = k + 1;
        if (m < K) {
#ifndef SDV_PTS_LDG
          if (m % kPtChunk == 0) {                          // entering chunk c: everyone is done reading chunk c-1, its buffer can take chunk c+1
            const int c = m / kPtChunk;
            __syncthreads();
            if (tid == 0 && c + 1 < NC) issue_chunk(c + 1);
            mbar_wait(&full_bar[c & 1], (bar_phase >> (c & 1)) & 1u); bar_phase ^= (1u << (c & 1));
          }
#endif
          sN = project(m);
        }
        cp_async_commit();
        cp_async_wait1();                                   // the gather of iteration k (committed one iteration ago) has landed in this thread's slot
        stage_accumulate<THREADS>(sC, g, ep, reinterpret_cast<const float*>(ring + (size_t)(k & 1)*kSlotStride) + tid, acc);
      }
      SDV_PROF_T(tp4); SDV_PROF_ADD(3, tp3, tp4);
      cp_async_wait0();
      __syncthreads();                                      // the reduction scratch aliases the tap ring / point chunks
      SDV_PROF_T(tp5); SDV_PROF_ADD(4, tp4, tp5);
      block_reduce_acc<THREADS>(acc, red, bsum);
      if (C > 1) {
        const int buf = evalCount & 1;
        for (int k = tid; k < kNAcc*C; k += THREADS) {
          int r = k / kNAcc, e = k - r*kNAcc;
          double* dst = cluster.map_shared_rank(gather, r);
          dst[(buf*C + rank)*kNAcc + e] = bsum[e];
        }
        cluster.sync();
        if (tid < kNAcc) { double s = 0; for (int r = 0; r < C; r++) s += gather[(buf*C + r)*kNAcc + tid]; tot[tid] = s; }
      } else {
        if (tid < kNAcc) tot[tid] = bsum[tid];
      }
      __syncthreads();
      evalCount++;
      n_eval = n;                                             // ctl.evals is updated by lane 0 inside the control block: a lane-0-only store HERE left warp 0 split 1 + 31 with
                                                            // nothing to reconverge it before the control step (every control instruction issued twice)
      SDV_PROF_T(tp6); SDV_PROF_ADD(5, tp5, tp6);
#ifdef SDV_TRACK_PROFILE
      if (blockIdx.x == 0 && tid == 0) g_track_prof[8] += 1;
#endif
    }
    SDV_PROF_T(tc0);
    // ------------------------------------------------------------------ LM control (warp 0), CoarseTracker.cpp:679-812 as a state machine
    // All 32 lanes execute the SAME instruction stream on the same values (SIMT: no extra cost) and only lane 0's stores to `ctl` are predicated.  A lane-0-only
    // branch in front of the warp-cooperative LDLT left the warp diverged at the shuffles (the solve executed twice per call, every __shfl_sync a rendezvous of
    // two groups).
    if (tid < 32) {
      __syncwarp();                                          // converge warp 0 before anything warp-cooperative
      const bool L0 = (tid == 0);
      const float lambdaExtrapolationLimit = 0.001f;         // :680
      const int maxIt = (lvl == 0) ? 10 : ((lvl == 1) ? 20 : 50);   // maxIterations[] = {10,20,50,50,50}  (:679)
      const int mode = ctl.mode; float lcr = ctl.lcr; float lambda = ctl.lambda; int iteration = ctl.iteration;
      SE3d cur = ctl.cur; double a_cur = ctl.a_cur, b_cur = ctl.b_cur;
      double resOld[6];
#pragma unroll
      for (int i = 0; i < 6; i++) resOld[i] = ctl.resOld[i];
      bool propose = false, level_end = false, repeat_entry = false;
      __syncwarp();
      if (mode == 0) {                                       // level entry: resOld at the current pose (:690-702)
        finalize_res(tot, resOld);
        if (resOld[5] > 0.6 && lcr < 50) { lcr *= 2; repeat_entry = true; }
        else { finalize_gs_warp(tot, ctl.H, ctl.b, tid); lambda = 0.01f; iteration = 0; propose = true; }
      } else {                                               // candidate evaluated: accept / reject (:770-806)
        double resNew[6]; finalize_res(tot, resNew);
        const bool accept = (resNew[0]/resNew[1]) < (resOld[0]/resOld[1]);
        if (accept) {
          finalize_gs_warp(tot, ctl.H, ctl.b, tid);
#pragma unroll
          for (int i = 0; i < 6; i++) resOld[i] = resNew[i];
          cur = ctl.cand; a_cur = ctl.a_cand; b_cur = ctl.b_cand;
          lambda *= 0.5f;
        } else {
          lambda *= 4;
          if (lambda < lambdaExtrapolationLimit) lambda = lambdaExtrapolationLimit;
        }
        if (L0 && accept) ctl.accs[lvl]++;
        iteration++;
        if (!(ctl.incn > 1e-3) || iteration >= maxIt) level_end = true; else propose = true;
      }
      __syncwarp();                                          // ctl.H / ctl.b (lane 0's stores) before every lane reads them
      SDV_PROF_T(tq1); SDV_PROF_ADD(9, tc0, tq1);
      int next_lvl = lvl, next_mode = mode, done = 0, aborted = 0, haveRepeated = ctl.haveRepeated;
      double incn_out = ctl.incn; SE3d cand = cur; double a_cand = a_cur, b_cand = b_cur;
      bool new_ep = false; SE3d ep_pose = cur; double ep_a = a_cur, ep_b = b_cur; int ep_lvl = lvl; float ep_lcr = lcr;
      double lastRes_l = 0;
      if (repeat_entry) { new_ep = true; next_mode = 0; }
      if (level_end) {                                       // :808-822
        lastRes_l = sqrtf((float)(resOld[0]/resOld[1]));
        if (lastRes_l > 1.5*J.minRes[lvl]) { aborted = 1; done = 1; }
        else {
          int nl = lvl;
          if (lcr > 1 && !haveRepeated) { nl++; haveRepeated = 1; }
          nl--;
          if (nl < 0) done = 1;
          else { next_lvl = nl; next_mode = 0; lcr = 1.0f; new_ep = true; ep_lvl = nl; ep_lcr = 1.0f; }
        }
      }
      if (propose) {                                         // propose the LM step (:722-765) — warp-cooperative, every lane converged
        const int r = tid & 7;
        const bool fixA = tc.affineOptModeA < 0, fixB = tc.affineOptModeB < 0;
        const int nv = (!fixA && !fixB) ? 8 : ((fixA && fixB) ? 6 : 7);
        const bool stitch = fixA && !fixB;                   // fix a only: b takes slot 6 (:736-748)
        const int rr = (stitch && r == 6) ? 7 : r;
        double a[8];
#pragma unroll
        for (int j = 0; j < 8; j++) {
          const int cc = (stitch && j == 6) ? 7 : j;
          double hv = ctl.H[rr*8 + cc];
          if (rr == cc) hv *= (1 + lambda);
          a[j] = (r < nv && j < nv) ? hv : ((r == j) ? 1.0 : 0.0);
        }
        double rhs = (r < nv) ? -ctl.b[rr] : 0.0;
        const double x = warp_ldlt_solve8(a, rhs);
        SDV_PROF_T(tq2); SDV_PROF_ADD(10, tq1, tq2);
        double inc[8];
#pragma unroll
        for (int j = 0; j < 8; j++) inc[j] = __shfl_sync(0xffffffffu, x, j, 8);
        if (fixA && fixB) { inc[6] = 0; inc[7] = 0; }
        else if (!fixA && fixB) { inc[7] = 0; }
        else if (stitch) { inc[7] = inc[6]; inc[6] = 0; }
        float extrapFac = 1;
        if (lambda < lambdaExtrapolationLimit) extrapFac = sqrtf(sqrtf(lambdaExtrapolationLimit / lambda));
#pragma unroll
        for (int i = 0; i < 8; i++) inc[i] *= extrapFac;
        double incScaled[8];
#pragma unroll
        for (int i = 0; i < 3; i++) incScaled[i] = inc[i]*1.0f;        // SCALE_XI_ROT   (:755)
#pragma unroll
        for (int i = 3; i < 6; i++) incScaled[i] = inc[i]*0.5f;        // SCALE_XI_TRANS (:756)
        incScaled[6] = inc[6]*10.0f; incScaled[7] = inc[7]*1000.0f;    // SCALE_A, SCALE_B
        double ssum = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) ssum += incScaled[i];
        if (!isfinite(ssum)) {
#pragma unroll
          for (int i = 0; i < 8; i++) incScaled[i] = 0;
        }
        double incn = 0;
#pragma unroll
        for (int i = 0; i < 8; i++) incn += inc[i]*inc[i];
        incn_out = sqrt(incn);
        cand = se3_mul(se3_exp(incScaled), cur); a_cand = a_cur + incScaled[6]; b_cand = b_cur + incScaled[7];
        next_mode = 1; new_ep = true; ep_pose = cand; ep_a = a_cand; ep_b = b_cand;
        SDV_PROF_T(tq3); SDV_PROF_ADD(11, tq2, tq3);
      }
      SDV_PROF_T(tq4);
      EvalParams ep;
      if (new_ep) make_eval_params(ep_pose, ep_a, ep_b, J.refExposure, J.newExposure, J.ref_a, J.ref_b, geom.g[ep_lvl], ep_lvl, tc.coarseCutoffTH*ep_lcr, tc.huberTH, ep);
      __syncwarp();                                          // every lane has read the old control state (racecheck: warp-level WAR on ctl.incn / ctl.haveRepeated otherwise)
      if (L0) {                                              // publish (plain predicated stores; nothing collective follows inside this block)
        ctl.cur = cur; ctl.a_cur = a_cur; ctl.b_cur = b_cur; ctl.cand = cand; ctl.a_cand = a_cand; ctl.b_cand = b_cand;
#pragma unroll
        for (int i = 0; i < 6; i++) ctl.resOld[i] = resOld[i];
        ctl.lambda = lambda; ctl.lcr = lcr; ctl.iteration = iteration; ctl.incn = incn_out; ctl.mode = next_mode; ctl.lvl = next_lvl;
        ctl.haveRepeated = haveRepeated; ctl.done = done; ctl.aborted = aborted;
        if (propose) ctl.iters[lvl]++;
        ctl.evals[lvl] += n_eval;
        if (level_end) { ctl.lastRes[lvl] = lastRes_l; ctl.flow[0] = resOld[2]; ctl.flow[1] = resOld[3]; ctl.flow[2] = resOld[4]; }
        if (new_ep) ctl.ep = ep;
      }
      SDV_PROF_T(tq5); SDV_PROF_ADD(12, tq4, tq5);
    }
    __syncthreads();
    SDV_PROF_T(tc1); SDV_PROF_ADD(6, tc0, tc1);
    if (ctl.done) break;
  }

  if (rank == 0 && tid == 0) {
    int good = 0;
    if (!ctl.aborted) {
      se3_to7(ctl.cur, J.T);
      double a_out = ctl.a_cur, b_out = ctl.b_cur;
      good = 1;
      if ((tc.affineOptModeA != 0 && (fabsf((float)a_out) > 1.2f)) || (tc.affineOptModeB != 0 && (fabsf((float)b_out) > 200))) good = 0;
      if (good) {
        double rel[2]; aff_from_to(J.refExposure, J.newExposure, J.ref_a, J.ref_b, a_out, b_out, rel);
        float r0 = (float)rel[0], r1 = (float)rel[1];
        if ((tc.affineOptModeA == 0 && (fabsf(logf(r0)) > 1.5f)) || (tc.affineOptModeB == 0 && (fabsf(r1) > 200))) good = 0;
        if (good) { if (tc.affineOptModeA < 0) a_out = 0; if (tc.affineOptModeB < 0) b_out = 0; }
      }
      J.ab[0] = a_out; J.ab[1] = b_out;
    }
    J.good = good;
    for (int i = 0; i < 5; i++) J.lastRes[i] = ctl.lastRes[i];
    for (int i = 0; i < 3; i++) J.flow[i] = ctl.flow[i];
    for (int i = 0; i < kLevels; i++) { J.point_evals[i] = ctl.evals[i]; J.iterations[i] = ctl.iters[i]; J.accepts[i] = ctl.accs[i]; }
  }
  if (C > 1) cluster.sync();                                // keep every CTA's shared memory alive until all remote writes/reads are done
}

template <int THREADS>
static size_t track_kernel_smem(int cluster_size = kMaxCluster) {
  size_t stage = (size_t)2*kTaps*THREADS*4 + (size_t)2*kPtChunk*THREADS*16, red = (size_t)kNAcc*THREADS*sizeof(float);
  return (stage > red ? stage : red) + (size_t)(2*cluster_size*kNAcc + 2*kNAcc)*sizeof(double);
}

static unsigned track_stagger_ns() { static long v = -1; if (v < 0) { const char* e = getenv("SDV_TRACK_STAGGER_NS"); v = e ? atol(e) : SDV_TRACK_STAGGER_DEFAULT_NS; if (v < 0) v = 0; } return (unsigned)v; }
template <typename Kern, typename... Extra>
static cudaError_t launch_track_kern(Kern kern, size_t smem, int threads, TrackJob* jobs_dev, int njobs, const TrackConst* tc_dev, const GeomRow* geom_dev, int cluster_size, cudaStream_t st,
                                     Extra... extra) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3((unsigned)(njobs*cluster_size)); cfg.blockDim = dim3(threads); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeClusterDimension; at[0].val.clusterDim.x = (unsigned)cluster_size; at[0].val.clusterDim.y = 1; at[0].val.clusterDim.z = 1;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kern, jobs_dev, tc_dev, geom_dev, extra...);
}
template <int THREADS, int MINB>
static cudaError_t launch_track_t(TrackJob* jobs_dev, int njobs, const TrackConst* tc_dev, const GeomRow* geom_dev, int cluster_size, cudaStream_t st) {
  // stagger only when the grid fills the co-resident slots of the chip (otherwise there is nothing to desynchronise)
  const unsigned stag = (cluster_size == 1 && njobs > num_sms()) ? track_stagger_ns() : 0u;
  return launch_track_kern(track_cluster_kernel<THREADS, MINB>, track_kernel_smem<THREADS>(cluster_size), THREADS, jobs_dev, njobs, tc_dev, geom_dev, cluster_size, st, stag);
}
template <typename Kern>
static cudaError_t track_attrs(Kern kern, size_t smem) {
  cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem); if (e != cudaSuccess) return e;
  return cudaFuncSetAttribute(kern, cudaFuncAttributeNonPortableClusterSizeAllowed, 1);
}
// threads: 128 (throughput, 4 jobs resident per SM) or 256 (latency)
#ifndef SDV_TRACK_MINB
#define SDV_TRACK_MINB 4                    // H100: 4 (128 regs, 80 B spilled at the time) 2.57 ms per 1 056 jobs against 3 (160 regs, no spills) 2.93 ms; DESIGN.md §6
#endif
cudaError_t launch_track_cluster(TrackJob* jobs_dev, int njobs, const TrackConst* tc_dev, const GeomRow* geom_dev, int cluster_size, int threads, cudaStream_t st) {
  if (threads == 256) return launch_track_t<256, 1>(jobs_dev, njobs, tc_dev, geom_dev, cluster_size, st);
  if (threads == 64)  return launch_track_t<64, 8>(jobs_dev, njobs, tc_dev, geom_dev, cluster_size, st);
  return launch_track_t<128, SDV_TRACK_MINB>(jobs_dev, njobs, tc_dev, geom_dev, cluster_size, st);
}

// Function attributes (opt-in dynamic shared memory, non-portable cluster sizes) belong to the CURRENT DEVICE's copy of a kernel: sdv_create calls this
// after cudaSetDevice, so a second context on another device of the same process gets them too (a process-wide "already set" flag did not).
cudaError_t kernels_init_device() {
  cudaError_t e = cudaFuncSetAttribute(coarse_res_gs_kernel<kStepThreads>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)((size_t)kNAcc*kStepThreads*sizeof(float)));
  if (e != cudaSuccess) return e;
#define SDV_TRACK_ATTRS(T, M) \
  if ((e = track_attrs(track_cluster_kernel<T, M>, track_kernel_smem<T>())) != cudaSuccess) return e;
  SDV_TRACK_ATTRS(256, 1) SDV_TRACK_ATTRS(64, 8) SDV_TRACK_ATTRS(128, SDV_TRACK_MINB)
#undef SDV_TRACK_ATTRS
  return cudaSuccess;
}

#ifdef SDV_TRACK_PROFILE
extern "C" int sdv_debug_track_profile(long long* out16, int reset) {
  long long z[16] = {0};
  if (out16 && cudaMemcpyFromSymbol(out16, g_track_prof, sizeof(z)) != cudaSuccess) return -1;
  if (reset && cudaMemcpyToSymbol(g_track_prof, z, sizeof(z)) != cudaSuccess) return -1;
  return 0;
}
#endif
__global__ void h2d_words_kernel(uint4* __restrict__ dst, const uint4* __restrict__ src, size_t n16) {
  for (size_t i = (size_t)blockIdx.x*blockDim.x + threadIdx.x; i < n16; i += (size_t)gridDim.x*blockDim.x) dst[i] = src[i];
}
void launch_h2d_words(void* dst_dev, const void* src_pinned, size_t bytes, cudaStream_t st) {      // bytes is rounded up to 16: both buffers are allocated with slack
  const size_t n16 = (bytes + 15)/16; if (!n16) return;
  int blocks = (int)((n16 + 255)/256); if (blocks > num_sms()*2) blocks = num_sms()*2;
  h2d_words_kernel<<<blocks, 256, 0, st>>>(reinterpret_cast<uint4*>(dst_dev), reinterpret_cast<const uint4*>(src_pinned), n16);
}

__global__ void pack_cloud_kernel(const float* u, const float* v, const float* id, const float* col, int n, float4* out) {
  int i = blockIdx.x*blockDim.x + threadIdx.x; if (i < n) out[i] = make_float4(u[i], v[i], id[i], col[i]);
}
void launch_pack_cloud(const float* u, const float* v, const float* id, const float* col, int n, float4* out, cudaStream_t st) {
  if (n > 0) pack_cloud_kernel<<<(n+255)/256, 256, 0, st>>>(u, v, id, col, n, out);
}

} // namespace sdv
