// Device-side construction of the flat k-mer table and the initial set dictionary.
//
// Replaces, for query purposes only, Bifrost's minimizer index + BBHash MPHF
// (ext/bifrost/src/CompactedDBG.tcc:999-1119, MinimizerIndex.cpp:370-395, BooPHF.h:787-822):
// every k-mer of every unitig is enumerated once, canonicalised and inserted in an
// open-addressing table whose 32-byte slot carries everything KmerIndex::match needs from
// `dbg.find` + `Node::get_mc_contig` + `Node::ec[dist]` (src/KmerIndex.cpp:1753-1788).
#include "kb_device.cuh"
#include "kernels.hpp"

namespace kb {

__global__ void __launch_bounds__(256) build_table_kernel(TableBuildArgs a) {
  const uint64_t g = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (g >= a.n_kmers) return;
  // unitig containing global k-mer g: last u with kstart[u] <= g
  uint32_t lo = 0, hi = a.n_unitigs;   // invariant: kstart[lo] <= g < kstart[hi]
  while (hi - lo > 1) {
    const uint32_t mid = (lo + hi) >> 1;
    if (a.kstart[mid] <= g) lo = mid; else hi = mid;
  }
  const uint32_t u = lo;
  const uint32_t dist = (uint32_t)(g - a.kstart[u]);
  const int k = a.k;
  uint64_t fwd;
  if (u < a.n_long) {
    const uint8_t* s = a.useq + a.useq_byteoff[u];
    fwd = 0;
    for (int j = 0; j < k; ++j) {
      const uint32_t i = dist + j;
      fwd = (fwd << 2) | ((s[i >> 2] >> ((i & 3) * 2)) & 3);
    }
  } else {
    fwd = a.skmer[u - a.n_long];
  }
  const uint64_t rc = kb_revcomp(fwd, k);
  const uint64_t canon = fwd < rc ? fwd : rc;
  // EC block containing dist: last block with lb <= dist (blocks tile the unitig)
  uint64_t blo = a.blk_off[u], bhi = a.blk_off[u + 1];
  while (bhi - blo > 1) {
    const uint64_t mid = (blo + bhi) >> 1;
    if (a.blk_lb[mid] <= dist) blo = mid; else bhi = mid;
  }
  KmerSlot* slots = a.slots;
  const uint64_t hsh = kb_mix64(canon);
  if (a.filter) {
    const uint32_t fi = (uint32_t)(hsh >> 32) & a.filter_mask;
    atomicOr(&a.filter[fi >> 5], 1u << (fi & 31));
  }
  uint64_t h = hsh & a.mask;
  for (;;) {
    const unsigned long long old =
        atomicCAS((unsigned long long*)&slots[h].key, (unsigned long long)KB_EMPTY_KEY, (unsigned long long)canon);
    if (old == KB_EMPTY_KEY) break;
    if (old == canon) { atomicOr(a.error, KB_DEVERR_TABLE_DUP); return; }
    h = (h + 1) & a.mask;
  }
  slots[h].unitig = u;
  slots[h].blk = (uint32_t)blo;
  slots[h].ec = a.blk_ec[blo];
  slots[h].dist_flag = dist | (fwd == canon ? 0x80000000u : 0u);
  slots[h].lb = a.blk_lb[blo];
  slots[h].ub = a.blk_ub[blo];
}

// One thread per index EC set: register it in the content-addressed dictionary.
__global__ void __launch_bounds__(256) dict_init_kernel(DictInitArgs a) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= a.n_ec) return;
  const uint32_t off = a.ec_off[e];
  const uint32_t len = a.ec_off[e + 1] - off;
  uint64_t sum = 0;
  for (uint32_t i = 0; i < len; ++i) sum += kb_mix64((uint64_t)a.pool[off + i] + 0x9E3779B97F4A7C15ULL);
  const uint64_t hsh = kb_mix64(sum ^ len);
  const unsigned long long word = (unsigned long long)off | ((unsigned long long)len << 32) | ((hsh >> 56) << 56);
  uint64_t h = hsh & a.dmask;
  for (;;) {
    const unsigned long long old = atomicCAS(&a.dslots[h], ~0ULL, word);
    if (old == ~0ULL) break;
    h = (h + 1) & a.dmask;
  }
  a.ec_handle[e] = (int32_t)h;
}

__global__ void fill_u64_kernel(unsigned long long* p, uint64_t n, unsigned long long v) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}
__global__ void fill_memo2_kernel(Memo2Entry* p, uint64_t n) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    Memo2Entry e;
    e.key = ~0ULL; e.val = KB_H_NOTREADY; e.pad = 0;
    p[i] = e;
  }
}
__global__ void fill_i32_kernel(int32_t* p, uint64_t n, int32_t v) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) p[i] = v;
}
__global__ void fill_slots_kernel(KmerSlot* p, uint64_t n) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += stride) {
    KmerSlot s;
    s.key = KB_EMPTY_KEY; s.unitig = 0; s.blk = 0; s.ec = 0; s.dist_flag = 0; s.lb = 0; s.ub = 0;
    p[i] = s;
  }
}

void launch_fill_u64(unsigned long long* p, uint64_t n, unsigned long long v, cudaStream_t st) {
  if (n == 0) return;
  fill_u64_kernel<<<device_sm_count() * 8, 256, 0, st>>>(p, n, v);
}
void launch_fill_memo2(Memo2Entry* p, uint64_t n, cudaStream_t st) {
  if (n == 0) return;
  fill_memo2_kernel<<<device_sm_count() * 8, 256, 0, st>>>(p, n);
}
void launch_fill_i32(int32_t* p, uint64_t n, int32_t v, cudaStream_t st) {
  if (n == 0) return;
  fill_i32_kernel<<<device_sm_count() * 8, 256, 0, st>>>(p, n, v);
}
void launch_build_table(const TableBuildArgs& a, cudaStream_t st) {
  fill_slots_kernel<<<device_sm_count() * 8, 256, 0, st>>>(a.slots, a.mask + 1);
  if (a.n_kmers == 0) return;
  const uint64_t blocks = (a.n_kmers + 255) / 256;
  build_table_kernel<<<(unsigned)blocks, 256, 0, st>>>(a);
}
void launch_dict_init(const DictInitArgs& a, cudaStream_t st) {
  if (a.n_ec == 0) return;
  dict_init_kernel<<<(a.n_ec + 255) / 256, 256, 0, st>>>(a);
}

}  // namespace kb
