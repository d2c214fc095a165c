// sdv_pool.cuh — device blocks keyed by frame handle, reused in place or from a spare list (the immature-point store, sdv_trace.cu; the LiDAR row sets, sdv_lidar.cu).
// Room for keys that are about to receive new contents is planned in two phases so that a refused call changes no block.  plan picks, per key, its own block
// if large enough, else the smallest free spare that fits, else a new allocation with 25 % headroom; before allocating it frees the spares too small for the
// request (a drive whose sizes grow does not keep every block it outgrew).  Nothing visible changes until commit; on failure the new allocations become spares.
// Stream-ordered reuse: every reader and writer of a block runs on the context's tracker stream.
// Block: int n, cap; char* base() (the one allocation); static size_t bytes(int cap); static Block layout(char* p, int cap).
#pragma once
#include <unordered_map>
#include <vector>
#include <algorithm>
#include "sdv_ctx.cuh"

namespace sdv {

template <class Block> struct BlockPool {
  std::unordered_map<uint64_t, Block> blocks; std::vector<Block> spare;                 // spare: blocks of dropped keys, reused before allocating
  struct Plan { uint64_t key; int n; Block b; bool own; };
  // room for n[j] elements under keys[j]; store / unit name the store and its element in error messages
  int plan(sdv_ctx* c, int nk, const uint64_t* keys, const int* n, std::vector<Plan>& P, const char* store, const char* unit) {
    P.assign(nk, Plan()); std::vector<char> taken(spare.size(), 0); std::vector<Block> fresh;
    auto fail = [&](int rc) { for (auto& b : fresh) spare.push_back(b); return rc; };
    for (int j = 0; j < nk; j++) {
      Plan& q = P[j]; q.key = keys[j]; q.n = n[j]; auto it = blocks.find(keys[j]);
      if (it != blocks.end() && it->second.cap >= n[j]) { q.b = it->second; q.own = true; continue; }
      q.own = false; int best = -1;
      for (int k = 0; k < (int)spare.size(); k++) if (!taken[k] && spare[k].cap >= n[j] && (best < 0 || spare[k].cap < spare[best].cap)) best = k;
      if (best >= 0) { taken[best] = 1; q.b = spare[best]; continue; }
      bool small = false; for (int k = 0; k < (int)spare.size(); k++) small |= !taken[k] && spare[k].cap < n[j];
      if (small) {                                                                       // spares this request outgrew: give their memory back first
        if (cudaStreamSynchronize(c->st) != cudaSuccess) return fail(ctx_fail(c, SDV_ERR_CUDA, "%s: stream synchronise", store));
        std::vector<Block> keep; std::vector<char> kt;
        for (int k = 0; k < (int)spare.size(); k++) { if (!taken[k] && spare[k].cap < n[j]) cudaFree(spare[k].base()); else { keep.push_back(spare[k]); kt.push_back(taken[k]); } }
        spare.swap(keep); taken.swap(kt);
      }
      const int cap = std::max(256, n[j] + n[j]/4); char* p = nullptr;
      if (cudaMalloc((void**)&p, Block::bytes(cap)) != cudaSuccess) { cudaGetLastError(); return fail(ctx_fail(c, SDV_ERR_CUDA, "%s: cudaMalloc of %d %s", store, cap, unit)); }
      q.b = Block::layout(p, cap); fresh.push_back(q.b);
    }
    for (int k = (int)taken.size() - 1; k >= 0; k--) if (taken[k]) spare.erase(spare.begin() + k);   // the spares now in a plan
    return SDV_OK;
  }
  // the plan's blocks and counts become the keys' blocks; a key that moved leaves its old block as a spare
  void commit(std::vector<Plan>& P) {
    for (Plan& q : P) {
      auto it = blocks.find(q.key); q.b.n = q.n;
      if (it == blocks.end()) blocks[q.key] = q.b;
      else { if (!q.own) spare.push_back(it->second); it->second = q.b; }
    }
  }
  // a failed call after plan: blocks it took from the spares or allocated go back to the spares
  void abandon(std::vector<Plan>& P) { for (Plan& q : P) if (!q.own) spare.push_back(q.b); }
  void drop(uint64_t key) { auto it = blocks.find(key); if (it == blocks.end()) return; spare.push_back(it->second); blocks.erase(it); }
  void release() { for (auto& kv : blocks) cudaFree(kv.second.base()); for (auto& b : spare) cudaFree(b.base()); blocks.clear(); spare.clear(); }
};

}  // namespace sdv
