// Device-side construction of the EM problem straight from the run's set dictionary: no EC table
// ever travels to the host on the quant path.
//
// Replaces MasterProcessor::update's id assignment (EC ids = order of first occurrence, what the
// reference produces with -t 1; src/ProcessReads.cpp:323-334,424-483) and calc_weights
// (src/weights.cpp:220-246), and lays the equivalence classes out twice: CSR by EC for the
// denominator pass, CSC by transcript (entries in increasing EC id) for the numerator pass of
// em_kernel.  Sorting / scanning uses CUB device primitives (library plumbing, not a hot path:
// ~1e6 keys once per run); the gather / weight / transpose kernels are ours.
#include <cstdlib>

#include <cub/cub.cuh>

#include "kb_device.cuh"
#include "kernels.hpp"

namespace kb {

namespace {

__global__ void gather_used_kernel(DevDict dd, const uint32_t* used, uint32_t n, unsigned long long* first, uint32_t* idx) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  first[i] = dd.first[used[i]];
  idx[i] = i;
}

// After the sort: EC id e <- used[order[e]]
__global__ void ec_meta_kernel(DevDict dd, const uint32_t* used, const uint32_t* order, uint32_t n, uint32_t* handle,
                               uint32_t* count, uint32_t* len, uint32_t* multi_len, uint32_t* is_multi, uint32_t* minkey) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n) return;
  const uint32_t h = used[order[e]];
  const unsigned long long word = dd.dslots[h];
  const uint32_t l = (uint32_t)((word >> 32) & 0xFFFFFFu);
  handle[e] = h;
  count[e] = dd.count[h];
  len[e] = l;
  multi_len[e] = l > 1 ? l : 0;
  is_multi[e] = l > 1 ? 1u : 0u;
  minkey[e] = l > 0 ? dd.pool[(uint32_t)word] : 0u;     // smallest transcript id of the set (lists are sorted)
}

// Rows of the EM matrices = the multi-transcript ECs, laid out in order of their SMALLEST TRANSCRIPT ID instead of EC
// id: ECs of one gene (adjacent transcript ids) become adjacent rows, so the alpha gathers of neighbouring rows and
// the norm gathers of neighbouring transcripts fall into the same 32-byte sectors.  The arithmetic does not change:
// a row is still accumulated in its own order and a transcript's entries stay in increasing EC id.
__global__ void multi_compact_kernel(const uint32_t* is_multi, const uint32_t* multi_index, const uint32_t* minkey, uint32_t n,
                                     uint32_t* ckey, uint32_t* cval) {
  const uint32_t e = blockIdx.x * blockDim.x + threadIdx.x;
  if (e >= n || !is_multi[e]) return;
  const uint32_t r0 = multi_index[e];
  ckey[r0] = minkey[e];
  cval[r0] = e;
}
__global__ void row_len_kernel(const uint32_t* multi_ec, const uint32_t* len, uint32_t n_multi, uint32_t* rlen, uint32_t* rowpos) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r > n_multi) return;
  if (r == n_multi) { rlen[r] = 0; return; }     // the scan runs over n_multi + 1 items
  const uint32_t e = multi_ec[r];
  rlen[r] = len[e];
  rowpos[e] = r;
}

// One warp per EC: copy its transcript ids, compute the weights, count transcript degrees.
__global__ void ec_fill_kernel(DevDict dd, EmPrep p) {
  const uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned lane = threadIdx.x & 31;
  if (e >= p.n_ec) return;
  const uint32_t h = p.handle[e];
  const uint32_t off = (uint32_t)dd.dslots[h];
  const uint32_t l = p.len[e];
  const uint32_t* src = dd.pool + off;
  // the EC table itself (ids in order of first occurrence)
  const uint32_t eo = p.ec_off[e];
  for (uint32_t j = lane; j < l; j += 32) p.ec_tid[eo + j] = src[j];
  if (l == 1) {
    if (lane == 0) p.t_single[src[0]] = (int32_t)e;
    return;
  }
  const uint32_t r = p.multi_index[e];     // row of this EC (rows are ordered by smallest transcript id)
  const uint32_t mo = p.m_rowoff[r];
  const double c = (double)p.count[e];
  for (uint32_t j = lane; j < l; j += 32) {
    const uint32_t t = src[j];
    p.m_tid[mo + j] = t;
    p.m_w[mo + j] = __ddiv_rn(c, p.eff[t]);        // calc_weights: counts[ec] / eff_lens[tr]
    p.m_row[mo + j] = r;
    p.m_iota[mo + j] = mo + j;
    p.k64_in[mo + j] = ((unsigned long long)t << 32) | e;    // CSC order: transcript, then EC id
    atomicAdd(&p.t_deg[t], 1u);
  }
}

// EC table only (export to other ranks): one warp per EC copies its transcript ids
__global__ void ec_table_kernel(DevDict dd, EmPrep p) {
  const uint32_t e = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const unsigned lane = threadIdx.x & 31;
  if (e >= p.n_ec) return;
  const uint32_t* src = dd.pool + (uint32_t)dd.dslots[p.handle[e]];
  const uint32_t l = p.len[e], eo = p.ec_off[e];
  for (uint32_t j = lane; j < l; j += 32) p.ec_tid[eo + j] = src[j];
}

// CSC entries in (transcript, EC id) order from the stable sort of (tid, entry index)
__global__ void csc_fill_kernel(EmPrep p, const uint32_t* sorted_entry, uint32_t nnz) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= nnz) return;
  const uint32_t j = sorted_entry[i];
  p.t_midx[i] = p.m_row[j];
  p.t_w[i] = p.m_w[j];
}

__global__ void stats_kernel(const uint32_t* count, const uint32_t* len, uint32_t n, unsigned long long* out) {
  unsigned long long a = 0, u = 0;
  for (uint32_t e = blockIdx.x * blockDim.x + threadIdx.x; e < n; e += gridDim.x * blockDim.x) {
    a += count[e];
    if (len[e] == 1) u += count[e];
  }
  for (int o = 16; o > 0; o >>= 1) {
    a += __shfl_xor_sync(0xFFFFFFFFu, a, o);
    u += __shfl_xor_sync(0xFFFFFFFFu, u, o);
  }
  if ((threadIdx.x & 31) == 0) {
    atomicAdd(&out[0], a);
    atomicAdd(&out[1], u);
  }
}

}  // namespace

size_t emprep_sort_bytes(uint32_t n_used, uint32_t nnz_max) {
  size_t a = 0, b = 0, c = 0, d = 0;
  const int big = (int)std::max(n_used, nnz_max);
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const unsigned long long*)nullptr, (unsigned long long*)nullptr,
                                  (const uint32_t*)nullptr, (uint32_t*)nullptr, big);
  cub::DeviceRadixSort::SortPairs(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, big);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (const uint32_t*)nullptr, (uint32_t*)nullptr, big + 1);
  (void)d;
  return std::max(a, std::max(b, c)) + 256;
}

void emprep_sort_by_first(const DevDict& dd, const uint32_t* used, uint32_t n_used, unsigned long long* key_in,
                          unsigned long long* key_out, uint32_t* idx_in, uint32_t* order_out, void* tmp, size_t tmp_bytes,
                          cudaStream_t st) {
  if (n_used == 0) return;
  gather_used_kernel<<<(n_used + 255) / 256, 256, 0, st>>>(dd, used, n_used, key_in, idx_in);
  cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, key_in, key_out, idx_in, order_out, (int)n_used, 0, 64, st);
}

void emprep_meta(const DevDict& dd, const uint32_t* used, const uint32_t* order, uint32_t n, const EmPrep& p,
                 uint32_t* multi_len, uint32_t* is_multi, void* tmp, size_t tmp_bytes, cudaStream_t st) {
  if (n == 0) return;
  ec_meta_kernel<<<(n + 255) / 256, 256, 0, st>>>(dd, used, order, n, p.handle, p.count, p.len, multi_len, is_multi, p.minkey);
  // n + 1 items so that the totals land in [n]
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, p.len, p.ec_off, (int)n + 1, st);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, multi_len, p.m_off, (int)n + 1, st);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, is_multi, p.multi_index, (int)n + 1, st);
}

// Row order of the EM matrices: multi-transcript ECs sorted by their smallest transcript id (stable: ties in EC id
// order).  Fills multi_ec (row -> EC id), m_rowoff (n_multi + 1) and overwrites multi_index (EC id -> row).
void emprep_rows(const EmPrep& p, const uint32_t* is_multi, uint32_t* ckey, uint32_t* cval, uint32_t* ckey_out, uint32_t* rlen,
                 void* tmp, size_t tmp_bytes, cudaStream_t st) {
  if (p.n_multi == 0) return;
  multi_compact_kernel<<<(p.n_ec + 255) / 256, 256, 0, st>>>(is_multi, p.multi_index, p.minkey, p.n_ec, ckey, cval);
  int bits = 1;
  while ((1u << bits) < p.n_targets && bits < 32) ++bits;
  cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, ckey, ckey_out, cval, p.multi_ec, (int)p.n_multi, 0, bits, st);
  row_len_kernel<<<(p.n_multi + 1 + 255) / 256, 256, 0, st>>>(p.multi_ec, p.len, p.n_multi, rlen, p.multi_index);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, rlen, p.m_rowoff, (int)p.n_multi + 1, st);
}

void emprep_fill_table(const DevDict& dd, const EmPrep& p, cudaStream_t st) {
  if (p.n_ec == 0) return;
  const uint64_t threads = (uint64_t)p.n_ec * 32;
  ec_table_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(dd, p);
}

void emprep_fill(const DevDict& dd, const EmPrep& p, uint32_t nnz, unsigned long long* sort_keys_out, uint32_t* sort_vals_out,
                 void* tmp, size_t tmp_bytes, unsigned long long* stats2, cudaStream_t st) {
  if (p.n_ec == 0) return;
  const uint64_t threads = (uint64_t)p.n_ec * 32;
  ec_fill_kernel<<<(unsigned)((threads + 255) / 256), 256, 0, st>>>(dd, p);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, p.t_deg, p.t_off, (int)p.n_targets + 1, st);
  if (nnz) {
    int bits = 1;
    while ((1u << bits) < p.n_targets && bits < 32) ++bits;
    // (transcript, EC id) order: a transcript's entries are accumulated in increasing EC id (EMAlgorithm.h:125-169
    // walks the ECs in id order), whatever the row order of the matrices
    cub::DeviceRadixSort::SortPairs(tmp, tmp_bytes, p.k64_in, sort_keys_out, p.m_iota, sort_vals_out, (int)nnz, 0, 32 + bits, st);
    csc_fill_kernel<<<(nnz + 255) / 256, 256, 0, st>>>(p, sort_vals_out, nnz);
  }
  cudaMemsetAsync(stats2, 0, 16, st);
  stats_kernel<<<device_sm_count(), 256, 0, st>>>(p.count, p.len, p.n_ec, stats2);
}

// ---------------------------------------------------------------------------------------------
// Component layout of one EM problem (em_component_kernel, kernels_em.cu).  Built from the CSR / CSC of EmProblem,
// which stay as they are (the bootstrap reuses them).
namespace {

// Roots only ever get hooked under a smaller root, so parent pointers decrease and every walk ends.  A stale read is
// harmless: it can only show a root that has since been hooked, and the CAS on it then fails and the walk restarts.
__device__ __forceinline__ uint32_t uf_find(const uint32_t* parent, uint32_t x) {
  for (;;) {
    const uint32_t q = __ldcg(parent + x);
    if (q == x) return x;
    x = q;
  }
}

__global__ void comp_init_kernel(EmCompWs w, uint32_t T) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  w.parent[t] = t;
  w.rfirst[t] = 0;
  w.csize[t] = 0;
}

// Thread per row: every transcript of the row joins the component of the row's first transcript.
__global__ void comp_union_kernel(EmProblem p, EmCompWs w) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_multi) return;
  const uint32_t e0 = p.m_off[r], e1 = p.m_off[r + 1];
  if (e0 == e1) return;
  const uint32_t t0 = p.m_tid[e0];
  atomicAdd(&w.rfirst[t0], 1u);
  for (uint32_t j = e0 + 1; j < e1; ++j) {
    uint32_t a = t0, b = p.m_tid[j];
    for (;;) {
      a = uf_find(w.parent, a);
      b = uf_find(w.parent, b);
      if (a == b) break;
      if (a < b) { const uint32_t x = a; a = b; b = x; }
      if (atomicCAS(&w.parent[a], a, b) == a) break;
    }
  }
}

// After the unions: parent[t] <- root (the component's smallest transcript id).  Concurrent walks see either the old
// parent or the root, both ancestors.
__global__ void comp_compress_kernel(EmCompWs w, uint32_t T) {
  const uint32_t t = blockIdx.x * blockDim.x + threadIdx.x;
  if (t >= T) return;
  w.parent[t] = uf_find(w.parent, t);
  w.iota[t] = t;
}

__global__ void comp_rows_kernel(EmProblem p, EmCompWs w) {
  const uint32_t r = blockIdx.x * blockDim.x + threadIdx.x;
  if (r >= p.n_multi) return;
  w.rcomp[r] = w.parent[p.m_tid[p.m_off[r]]];
  w.iota[r] = r;
}

// Size carried by the transcript at each pos: itself, its entries and the rows it is the first transcript of.
__global__ void comp_size_kernel(EmProblem p, EmCompWs w) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > p.n_targets) return;
  if (i == p.n_targets) { w.tsize[i] = 0; return; }      // the scan runs over T + 1 items
  const uint32_t t = w.t_id[i];
  const unsigned long long s = 1ull + (p.t_off[t + 1] - p.t_off[t]) + w.rfirst[t];
  w.tsize[i] = s;
  atomicAdd(&w.csize[w.tkey[i]], s);
}

// Component heads record where their component starts; the slice target size is ceil(total / slices), and a component
// goes to slice floor(start / target), so there are at most `slices` slices (some may be empty).
__global__ void comp_heads_kernel(EmProblem p, EmCompWs w, uint32_t slices) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i == 0) {
    const unsigned long long total = w.tscan[p.n_targets];
    const unsigned long long target = (total + slices - 1) / slices;
    w.stats[0] = total;
    w.stats[1] = target;
    w.stats[2] = (total - 1) / target + 1;
  }
  if (i >= p.n_targets) return;
  const uint32_t c = w.tkey[i];
  if (i == 0 || w.tkey[i - 1] != c) {
    w.cstart[c] = w.tscan[i];
    atomicMax(&w.stats[3], w.csize[c]);
  }
}

// first index of `key` (sorted by component) whose component lies in slice `s` or later
__device__ __forceinline__ uint32_t slice_lower_bound(const uint32_t* key, uint32_t n, const unsigned long long* cstart,
                                                      unsigned long long target, uint32_t s) {
  uint32_t lo = 0, hi = n;
  while (lo < hi) {
    const uint32_t mid = (lo + hi) >> 1;
    if (cstart[key[mid]] / target < s) lo = mid + 1; else hi = mid;
  }
  return lo;
}

// Thread per slice: its first pos and row pos, and the shared memory em_component_kernel needs for it.
__global__ void comp_bounds_kernel(EmProblem p, EmCompWs w) {
  const uint32_t s = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t n = (uint32_t)w.stats[2];
  if (s >= n) return;
  const unsigned long long target = w.stats[1];
  const uint32_t t0 = slice_lower_bound(w.tkey, p.n_targets, w.cstart, target, s);
  const uint32_t t1 = slice_lower_bound(w.tkey, p.n_targets, w.cstart, target, s + 1);
  const uint32_t r0 = slice_lower_bound(w.rkey, p.n_multi, w.cstart, target, s);
  const uint32_t r1 = slice_lower_bound(w.rkey, p.n_multi, w.cstart, target, s + 1);
  w.s_t0[s] = t0;
  w.s_r0[s] = r0;
  if (s + 1 == n) { w.s_t0[n] = t1; w.s_r0[n] = r1; }
  atomicMax(&w.stats[4], emcomp_smem_bytes(t1 - t0, r1 - r0));
  // a slice holds whole components, so its size is its transcripts, its rows and its entries
  const unsigned long long ne = (w.tscan[t1] - w.tscan[t0]) - (t1 - t0) - (r1 - r0);
  atomicMax(&w.stats[6], emcomp_resident_bytes(t1 - t0, r1 - r0, ne));
}

// Thread per row and per transcript: counts the entries of the CSR and the CSC whose weight emcomp_weight does not
// rebuild bit for bit from the row's count and the transcript's effective length.
__global__ void comp_check_weights_kernel(EmProblem p, EmCompWs w) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  unsigned long long bad = 0;
  if (i < p.n_multi) {
    const double c = (double)p.cnt_row[i];
    for (uint32_t j = p.m_off[i]; j < p.m_off[i + 1]; ++j) {
      const double e = w.eff[p.m_tid[j]];
      bad += __double_as_longlong(emcomp_weight(c, e, __drcp_rn(e))) != __double_as_longlong(p.m_w[j]);
    }
  }
  if (i < p.n_targets) {
    const double e = w.eff[i], y = __drcp_rn(e);
    for (uint32_t j = p.t_off[i]; j < p.t_off[i + 1]; ++j)
      bad += __double_as_longlong(emcomp_weight((double)p.cnt_row[p.t_midx[j]], e, y)) != __double_as_longlong(p.t_w[j]);
  }
  if (bad) atomicAdd(&w.stats[5], bad);
}

// Slice-local positions, per-pos counts and entry counts (thread per pos and per row pos).
__global__ void comp_local_kernel(EmProblem p, EmCompWs w, bool resident) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  const unsigned long long target = w.stats[1];
  if (i < p.n_targets) {
    const uint32_t t = w.t_id[i];
    w.tloc[t] = i - w.s_t0[w.cstart[w.tkey[i]] / target];
    w.t_single[i] = p.single_cnt[t];
    if (resident) w.t_eff[i] = w.eff[t];
    w.t_len[i] = p.t_off[t + 1] - p.t_off[t];
  } else if (i == p.n_targets) {
    w.t_len[i] = 0;
  }
  if (i < p.n_multi) {
    const uint32_t r = w.r_id[i];
    w.rloc[r] = i - w.s_r0[w.cstart[w.rkey[i]] / target];
    w.r_cnt[i] = p.cnt_row[r];
    w.r_len[i] = p.m_off[r + 1] - p.m_off[r];
  } else if (i == p.n_multi) {
    w.r_len[i] = 0;
  }
}

// Entries in slice order; the order inside a row and inside a transcript's list is kept.
__global__ void comp_entries_kernel(EmProblem p, EmCompWs w, bool resident) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i < p.n_targets) {
    const uint32_t t = w.t_id[i];
    const uint32_t s0 = p.t_off[t], n = p.t_off[t + 1] - s0, d0 = w.t_off[i];
    for (uint32_t j = 0; j < n; ++j) {
      w.t_row[d0 + j] = (uint16_t)w.rloc[p.t_midx[s0 + j]];
      if (!resident) w.t_w[d0 + j] = p.t_w[s0 + j];
    }
  }
  if (i < p.n_multi) {
    const uint32_t r = w.r_id[i];
    const uint32_t s0 = p.m_off[r], n = p.m_off[r + 1] - s0, d0 = w.r_off[i];
    for (uint32_t j = 0; j < n; ++j) {
      w.r_tid[d0 + j] = (uint16_t)w.tloc[p.m_tid[s0 + j]];
      if (!resident) w.r_w[d0 + j] = p.m_w[s0 + j];
    }
  }
}

int key_bits(uint32_t n) {
  int bits = 1;
  while ((1u << bits) < n && bits < 32) ++bits;
  return bits;
}

}  // namespace

size_t emcomp_tmp_bytes(uint32_t n_targets, uint32_t n_multi) {
  const int big = (int)std::max(n_targets, n_multi) + 1;
  size_t a = 0, b = 0, c = 0;
  cub::DeviceRadixSort::SortPairs(nullptr, a, (const uint32_t*)nullptr, (uint32_t*)nullptr, (const uint32_t*)nullptr,
                                  (uint32_t*)nullptr, big);
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const unsigned long long*)nullptr, (unsigned long long*)nullptr, big);
  cub::DeviceScan::ExclusiveSum(nullptr, c, (const uint32_t*)nullptr, (uint32_t*)nullptr, big);
  return std::max(a, std::max(b, c)) + 256;
}

unsigned long long emcomp_cap() {
  if (const char* s = getenv("KB_EM_COMP_CAP")) return strtoull(s, nullptr, 10);   // test knob
  return ~0ull;
}

unsigned long long emcomp_smem_budget() {
  if (const char* s = getenv("KB_EM_COMP_SMEM")) return strtoull(s, nullptr, 10);   // test knob
  return ~0ull;
}

void emcomp_cut(const EmProblem& p, const EmCompWs& w, uint32_t slices, unsigned long long* stats_host, cudaStream_t st) {
  const uint32_t T = p.n_targets, R = p.n_multi;
  const int bits = key_bits(T);
  cudaMemsetAsync(w.stats, 0, 8 * sizeof(unsigned long long), st);
  comp_init_kernel<<<(T + 255) / 256, 256, 0, st>>>(w, T);
  if (R) comp_union_kernel<<<(R + 255) / 256, 256, 0, st>>>(p, w);
  comp_compress_kernel<<<(T + 255) / 256, 256, 0, st>>>(w, T);
  size_t tb = w.tmp_bytes;
  cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.parent, w.tkey, w.iota, w.t_id, (int)T, 0, bits, st);
  if (R) {
    comp_rows_kernel<<<(R + 255) / 256, 256, 0, st>>>(p, w);
    tb = w.tmp_bytes;
    cub::DeviceRadixSort::SortPairs(w.tmp, tb, w.rcomp, w.rkey, w.iota, w.r_id, (int)R, 0, bits, st);
  }
  comp_size_kernel<<<(T + 1 + 255) / 256, 256, 0, st>>>(p, w);
  tb = w.tmp_bytes;
  cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.tsize, w.tscan, (int)T + 1, st);
  comp_heads_kernel<<<(T + 255) / 256, 256, 0, st>>>(p, w, slices);
  comp_bounds_kernel<<<(slices + 127) / 128, 128, 0, st>>>(p, w);
  if (w.eff) comp_check_weights_kernel<<<(std::max(T, R) + 255) / 256, 256, 0, st>>>(p, w);
  cudaMemcpyAsync(stats_host, w.stats, 8 * sizeof(unsigned long long), cudaMemcpyDeviceToHost, st);
  cudaStreamSynchronize(st);
}

void emcomp_fill(const EmProblem& p, const EmCompWs& w, bool resident, cudaStream_t st) {
  const uint32_t T = p.n_targets, R = p.n_multi;
  const uint32_t n = std::max(T, R) + 1;
  comp_local_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, w, resident);
  size_t tb = w.tmp_bytes;
  cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.t_len, w.t_off, (int)T + 1, st);
  tb = w.tmp_bytes;
  cub::DeviceScan::ExclusiveSum(w.tmp, tb, w.r_len, w.r_off, (int)R + 1, st);
  comp_entries_kernel<<<(n + 255) / 256, 256, 0, st>>>(p, w, resident);
}

}  // namespace kb
