// Content-addressed set dictionary of a run (DevDict): the group-cooperative lookup-or-insert shared by every kernel
// that turns a sorted transcript-id list into a set handle (resolve_kernel, the multi-GPU import, cfc_select_kernel).
#pragma once
#include "kb_device.cuh"

namespace kb {
namespace {

__device__ __forceinline__ unsigned long long ld_acquire_u64(const unsigned long long* p) {
  unsigned long long v;
  asm volatile("ld.acquire.gpu.global.u64 %0, [%1];" : "=l"(v) : "l"(p) : "memory");
  return v;
}

__device__ __forceinline__ bool bsearch_contains(const uint32_t* s, uint32_t n, uint32_t v, uint32_t* rank) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    const uint32_t x = __ldcg(s + mid);
    if (x < v) lo = mid + 1; else hi = mid;
  }
  if (rank) *rank = lo;
  return lo < n && __ldcg(s + lo) == v;
}

// Lane groups: G consecutive lanes of a warp (G = 32, 16, 8 or 4) work on one item; the groups of a warp are
// independent of each other (every collective below names only the group's lanes).
template <int G>
__device__ __forceinline__ unsigned group_mask(unsigned lane_in_warp) {
  return G == 32 ? 0xFFFFFFFFu : (((1u << (G & 31)) - 1u) << (lane_in_warp & ~(unsigned)(G - 1)));
}

// Group-cooperative lookup-or-insert of a sorted transcript-id list in the content-addressed set
// dictionary (ecmapinv semantics: equal sets share one handle).  `src` may be shared or global memory
// readable by all lanes of the group; `lane` is the lane's index inside its group, `gmask` the group's lanes.
// Returns the handle, or KB_H_UNMAPPED after flagging an error.
template <int G = 32>
__device__ __forceinline__ int32_t dict_insert_warp(const DevDict& dd, const uint32_t* src, uint32_t nres, unsigned lane,
                                                    unsigned gmask = 0xFFFFFFFFu) {
  uint64_t sum = 0;
  for (uint32_t i = lane; i < nres; i += G) sum += kb_mix64((uint64_t)src[i] + 0x9E3779B97F4A7C15ULL);
  for (int o = G / 2; o > 0; o >>= 1) sum += __shfl_xor_sync(gmask, sum, o);
  const uint64_t hsh = kb_mix64(sum ^ nres);
  const unsigned long long tag = hsh >> 56;
  uint64_t s = hsh & dd.dmask;
  unsigned long long my_word = ~0ULL;   // pool space is allocated lazily
  uint64_t visited = 0;
  for (;;) {
    unsigned long long word = 0;
    if (lane == 0) word = ld_acquire_u64(&dd.dslots[s]);
    word = __shfl_sync(gmask, word, 0, G);
    if (word == ~0ULL) {
      if (my_word == ~0ULL) {
        unsigned long long off = 0;
        if (lane == 0) off = atomicAdd(dd.pool_top, (unsigned long long)nres);
        off = __shfl_sync(gmask, off, 0, G);
        if (off + nres > dd.pool_cap || off + nres > 0xFFFFFFFFULL) {
          if (lane == 0) atomicOr(dd.error, KB_DEVERR_POOL_FULL);
          return KB_H_UNMAPPED;
        }
        for (uint32_t i = lane; i < nres; i += G) dd.pool[off + i] = src[i];
        __threadfence();
        __syncwarp(gmask);
        my_word = off | ((unsigned long long)nres << 32) | (tag << 56);
      }
      unsigned long long old = 0;
      if (lane == 0) old = atomicCAS(&dd.dslots[s], ~0ULL, my_word);
      old = __shfl_sync(gmask, old, 0, G);
      if (old == ~0ULL) return (int32_t)s;
      word = old;   // somebody else took the slot: compare against theirs
    }
    if ((word >> 56) == tag && ((word >> 32) & 0xFFFFFFu) == nres) {
      const uint32_t* S = dd.pool + (uint32_t)word;
      bool eq = true;
      for (uint32_t i = lane; i < nres; i += G) eq = eq && (__ldcg(S + i) == src[i]);
      if (__all_sync(gmask, eq)) return (int32_t)s;
    }
    s = (s + 1) & dd.dmask;
    if (++visited > dd.dmask) {
      if (lane == 0) atomicOr(dd.error, KB_DEVERR_DICT_FULL);
      return KB_H_UNMAPPED;
    }
  }
}

}  // namespace
}  // namespace kb
