// sdv_ba_install.cu — sm_90a kernels of the batched back-end install and hand-over (sdv_ba_set_window_batch, sdv_ba_set_points_batch,
// sdv_ba_flag_points_batch, sdv_ba_marginalize_frames_batch): the header install, the makeIDX mirror (EnergyFunctional.cpp:761-782) as a check
// kernel plus a stable radix sort, and the scatter of the staged rows into each window's pool.  Every launch serves all windows of the call.
#include "sdv_ba.cuh"
#include <cub/device/device_radix_sort.cuh>

namespace sdv {

static_assert(kHdrPrefix % 8 == 0 && offsetof(BAHeader, HM) % 8 == 0 && offsetof(BAHeader, bM) % 8 == 0 && sizeof(BAHeader) % 8 == 0, "header copied in 8-byte words");

// blockIdx.y = window: every 8-byte word of its header, from the staged prefix / HM / bM or zero
__global__ void __launch_bounds__(256) ba_hdr_install_kernel(const BAHdrInstall* __restrict__ D, const char* __restrict__ stage) {
  const BAHdrInstall d = D[blockIdx.y];
  const unsigned long long* __restrict__ s = reinterpret_cast<const unsigned long long*>(stage + d.src);
  unsigned long long* h = reinterpret_cast<unsigned long long*>(d.hdr);
  constexpr int kPre = (int)(kHdrPrefix/8), kHM = (int)(offsetof(BAHeader, HM)/8), kbM = (int)(offsetof(BAHeader, bM)/8), kAll = (int)(sizeof(BAHeader)/8);
  for (int i = blockIdx.x*blockDim.x + threadIdx.x; i < kAll; i += gridDim.x*blockDim.x) {
    unsigned long long v = 0;
    if (i < kPre) v = s[i];
    else if (i >= kHM && i < kHM + d.hm_n) v = s[kPre + (i - kHM)];
    else if (i >= kbM && i < kbM + d.bm_n) v = s[kPre + d.hm_n + (i - kbM)];
    h[i] = v;
  }
}
void launch_ba_hdr_install(const BAHdrInstall* d, int n, const char* stage, cudaStream_t st) { ba_hdr_install_kernel<<<dim3(32, n), 256, 0, st>>>(d, stage); }

// the last window k with begin(k) <= x: the owner of row x (a window without rows has the begin of the next one)
template <class Begin> __device__ __forceinline__ int ba_owner(int n, int x, Begin begin) {
  int lo = 0, hi = n - 1;
  while (lo < hi) { const int mid = (lo + hi + 1) >> 1; if (begin(mid) <= x) lo = mid; else hi = mid - 1; }
  return lo;
}

// refusal word: ordered as the host loop of the single install met the failures — the span of res_begin (stage 0), its monotonicity over all
// points (stage 1), then point by point its host frame and its residuals in order (stage 2)
__device__ __forceinline__ unsigned long long ba_err(unsigned stage, int p, int sub, int code) {
  return ((unsigned long long)stage << 62) | ((unsigned long long)p << 34) | ((unsigned long long)sub << 4) | (unsigned long long)code;
}

// one thread per (window, point): the makeIDX checks, res_of_target, the residual count of each (host, target) pair and the point count per host
__global__ void __launch_bounds__(256) ba_pts_check_kernel(const BAPtsInstall* __restrict__ D, int n, int totP, const BAPtsStage S, unsigned long long* err) {
  const int g = blockIdx.x*blockDim.x + threadIdx.x; if (g >= totP) return;
  const int w = ba_owner(n, g, [&](int k) { return D[k].p0; });
  const BAPtsInstall q = D[w]; const int p = g - q.p0, nF = q.nF;
  const int* rb = S.res_begin + q.p0 + w;
  unsigned long long e = ~0ull;
  if (p == 0 && (rb[0] != 0 || rb[q.nP] != q.nR)) e = ba_err(0, 0, 0, BA_ERR_SPAN);
  const int a = rb[p], b = rb[p+1];
  if (a > b) e = min(e, ba_err(1, p, 0, BA_ERR_MONO));
  else if (a >= 0 && b <= q.nR) {                                            // else the span test has failed: no residual is indexed through it
    const int h = S.host[g];
    if (h < 0 || h >= nF || (p > 0 && h < S.host[g-1])) e = min(e, ba_err(2, p, 0, BA_ERR_HOST));
    else {
      unsigned seen = 0; bool ok = true;
      for (int r = a; r < b; r++) {
        const int R = q.r0 + r, t = S.r_target[R];
        if (S.r_point[R] != p || S.r_host[R] != h || t < 0 || t >= nF || t == h) { e = min(e, ba_err(2, p, r + 1, BA_ERR_RES)); ok = false; break; }
        if (seen & (1u << t)) { e = min(e, ba_err(2, p, r + 1, BA_ERR_DUP)); ok = false; break; }
        seen |= 1u << t; S.rot[(size_t)g*kMaxF + t] = r;
      }
      if (ok) {
        int* cnt = S.cnt + (size_t)w*kPairCnt;
        for (int r = a; r < b; r++) atomicAdd(cnt + h + nF*S.r_target[q.r0 + r], 1);
        atomicAdd(cnt + kMaxF*kMaxF + h, 1);
      }
    }
  }
  if (e != ~0ull) atomicMin(err + w, e);
}
void launch_ba_pts_check(const BAPtsInstall* D, int n, int totP, const BAPtsStage& S, unsigned long long* err, cudaStream_t st) {
  if (totP > 0) ba_pts_check_kernel<<<(totP + 255)/256, 256, 0, st>>>(D, n, totP, S, err);
}

// one thread per window: pair_begin and host_begin (exclusive scans of the counts), the header's nP / nR
__global__ void ba_pts_begin_kernel(const BAWinDev* __restrict__ wins, const BAPtsInstall* __restrict__ D, int n, const int* __restrict__ cnt) {
  const int w = blockIdx.x*blockDim.x + threadIdx.x; if (w >= n) return;
  const BAPtsInstall q = D[w]; const BAWinDev& W = wins[w]; const int* c = cnt + (size_t)w*kPairCnt; const int nF = q.nF;
  int s = 0; for (int k = 0; k < nF*nF; k++) { W.R.pair_begin[k] = s; s += c[k]; } W.R.pair_begin[nF*nF] = s;
  s = 0; for (int f = 0; f < nF; f++) { W.R.host_begin[f] = s; s += c[kMaxF*kMaxF + f]; } W.R.host_begin[nF] = s;
  W.hdr->nP = q.nP; W.hdr->nR = q.nR;
}
// one thread per residual of the call: its pair key and its window-local index
__global__ void ba_pair_key_kernel(const BAPtsInstall* __restrict__ D, int n, int totR, const int* __restrict__ r_host, const int* __restrict__ r_target,
                                   unsigned* __restrict__ key, int* __restrict__ val) {
  const int j = blockIdx.x*blockDim.x + threadIdx.x; if (j >= totR) return;
  const int w = ba_owner(n, j, [&](int k) { return D[k].r0; });
  key[j] = (unsigned)(w*(kMaxF*kMaxF) + r_host[j] + D[w].nF*r_target[j]); val[j] = j - D[w].r0;
}
// blockIdx.y = window, thread i: point row i, res_begin[i], residual row i of the window and the zero-fills of sdv_ba_set_points
__global__ void __launch_bounds__(256) ba_pts_scatter_kernel(const BAWinDev* __restrict__ wins, const BAPtsInstall* __restrict__ D, const BAPtsStage S) {
  const BAPtsInstall q = D[blockIdx.y]; BAPointsDev P = wins[blockIdx.y].P; BAResDev R = wins[blockIdx.y].R;
  const int i = blockIdx.x*blockDim.x + threadIdx.x;
  if (i < q.nP) { const int g = q.p0 + i;
    P.uv[i] = S.uv[g]; const float id = S.idepth[g]; P.idepth[i] = id; P.idepth_backup[i] = id; P.idepth_zero[i] = S.idepth_zero[g];
    for (int k = 0; k < 8; k++) { P.color[(size_t)i*8 + k] = S.color[(size_t)g*8 + k]; P.weights[(size_t)i*8 + k] = S.weights[(size_t)g*8 + k]; }
    for (int k = 0; k < kMaxF; k++) P.res_of_target[(size_t)i*kMaxF + k] = S.rot[(size_t)g*kMaxF + k];
    P.host[i] = S.host[g]; P.hasDepthPrior[i] = S.hasDepthPrior[g]; P.isFromSensor[i] = S.isFromSensor[g];
    P.step[i] = 0.f; P.maxRelBaseline[i] = 0.f; P.numGoodResiduals[i] = 0;
  }
  if (i <= q.nP) P.res_begin[i] = S.res_begin[q.p0 + blockIdx.y + i];
  if (i < q.nR) { const int j = q.r0 + i;
    R.point[i] = S.r_point[j]; R.host[i] = S.r_host[j]; R.target[i] = S.r_target[j]; R.hasMatcher[i] = S.r_hasMatcher[j]; R.matcher[i] = S.r_matcher[j];
    R.isNew[i] = S.r_isNew[j]; R.pair_res[i] = S.pair_res[j];
    R.isActive[i] = 0; R.toRemove[i] = 0;
    for (int k = 0; k < 24; k++) { R.J[(size_t)i*24 + k] = 0.f; R.efJ[(size_t)i*24 + k] = 0.f; }
    for (int k = 0; k < 8; k++) R.JpJdF[(size_t)i*8 + k] = 0.f;
    for (int k = 0; k < 3; k++) R.center[(size_t)i*3 + k] = 0.f;
  }
}

static int key_bits(int n) { int b = 1; while ((1ll << b) < (long long)n*kMaxF*kMaxF) b++; return b; }
size_t ba_pts_sort_bytes(int n, int totR) {
  size_t b = 0;
  if (totR > 0) cub::DeviceRadixSort::SortPairs(nullptr, b, (const unsigned*)nullptr, (unsigned*)nullptr, (const int*)nullptr, (int*)nullptr, totR, 0, key_bits(n));
  return b;
}
int launch_ba_pts_install(const BAWinDev* wins, const BAPtsInstall* D, int n, int totR, int maxP, int maxR, const BAPtsStage& S, void* sort_tmp, size_t sort_bytes,
                          cudaStream_t st) {
  int nl = 2;
  if (totR > 0) {                                                            // stable: the residuals of one pair keep their order, which the accumulators' sums follow
    ba_pair_key_kernel<<<(totR + 255)/256, 256, 0, st>>>(D, n, totR, S.r_host, S.r_target, S.key_in, S.val_in);
    size_t tb = sort_bytes;                                                  // (staging only: a failure here has written no window)
    if (cub::DeviceRadixSort::SortPairs(sort_tmp, tb, S.key_in, S.key, S.val_in, S.pair_res, totR, 0, key_bits(n), st) != cudaSuccess) return -1;
    nl += 2;
  }
  ba_pts_begin_kernel<<<(n + 127)/128, 128, 0, st>>>(wins, D, n, S.cnt);
  const int m = (maxP + 1 > maxR ? maxP + 1 : maxR);
  ba_pts_scatter_kernel<<<dim3((m + 255)/256, n), 256, 0, st>>>(wins, D, S);
  return nl;
}

__global__ void ba_status_copy_kernel(const BAWinDev* __restrict__ wins, const int* __restrict__ off, int* buf, int to_window) {
  const int w = blockIdx.y, p = blockIdx.x*blockDim.x + threadIdx.x; const int o = off[w]; if (p >= off[w+1] - o) return;
  int* s = wins[w].P.marg_status;
  if (to_window) s[p] = buf[o + p]; else buf[o + p] = s[p];
}
void launch_ba_status_copy(const BAWinDev* wins, int n, int maxP, const int* off, int* buf, int to_window, cudaStream_t st) {
  ba_status_copy_kernel<<<dim3((maxP + 255)/256 > 0 ? (maxP + 255)/256 : 1, n), 256, 0, st>>>(wins, off, buf, to_window);
}

__global__ void __launch_bounds__(256) ba_prior_gather_kernel(const BAWinDev* __restrict__ wins, const long long* __restrict__ off, double* out) {
  const BAHeader* H = wins[blockIdx.y].hdr; const int N = H->dim;
  double* hm = out + off[2*blockIdx.y]; double* bm = out + off[2*blockIdx.y + 1];
  for (int i = blockIdx.x*blockDim.x + threadIdx.x; i < N*N; i += gridDim.x*blockDim.x) { hm[i] = H->HM[i]; if (i < N) bm[i] = H->bM[i]; }
}
void launch_ba_prior_gather(const BAWinDev* wins, int n, const long long* off, double* out, cudaStream_t st) {
  ba_prior_gather_kernel<<<dim3(4, n), 256, 0, st>>>(wins, off, out);
}

}  // namespace sdv
