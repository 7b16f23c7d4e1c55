// K6: BUS record path of `kallisto bus` (BUSProcessor::processBuffer, src/ProcessReads.cpp:1380-1832).
//
//   bus_fields_kernel   per read set: slice barcode / UMI out of the technology's files
//                       (BUSOptionSubstr{fileno,start,stop}, :1486-1627), 2-bit encode them with the N
//                       bookkeeping of stringToBinary (src/BUSData.cpp:8-36), histogram the observed
//                       lengths, flag the sets the reference skips (:1505-1521, :1592-1602).
//   (pack / match / resolve kernels run on the cDNA read exactly as for `quant --single`)
//   bus_newec_kernel    + scan: equivalence classes first seen in this batch get the next ids, in
//                       read order -- the ids MasterProcessor::update hands out with -t 1
//                       (src/ProcessReads.cpp:603-624).
//   bus_records_kernel  + scan: one 32-byte BUSData (src/BUSData.h:30-38) per pseudoaligned read, in
//                       read order, ready to be appended to output.bus.
//   bus --devices (a member of a kb_bus_group): bus_newlen_kernel + scan + bus_export_kernel lay the sets new
//                       on the member out as CSR for the host's run-wide numbering, and bus_newid_gid_kernel
//                       writes the ids it chose instead of next_id + rank.
#include <cub/cub.cuh>

#include "kb_device.cuh"
#include "kernels.hpp"

namespace kb {

namespace {

struct Enc {
  uint64_t r = 0;
  int n = 0;        // characters consumed (only the first 32 are encoded)
  int numN = 0;
  int posN = 0;
  __device__ __forceinline__ void push(uint32_t c) {   // stringToBinary, one character
    if (n < 32) {
      const uint64_t x = (c & 4) >> 1;
      if ((c & 3) == 2) {
        if (numN == 0) posN = n;
        ++numN;
      }
      r = (r << 2) | (x + ((x ^ (c & 2)) >> 1));
    }
    ++n;
  }
  __device__ __forceinline__ uint32_t flag() const {
    if (numN == 0) return 0;
    const int nn = numN > 3 ? 3 : numN;
    return (uint32_t)(nn & 3) | ((uint32_t)(posN & 31) << 2);
  }
};

// `back`: letters in front of the slice that are encoded with it (the tag sequence in front of the first UMI piece,
// src/ProcessReads.cpp:1512-1514); the fit test is the slice's own
__device__ __forceinline__ bool slice(const BusArgs& a, uint32_t i, int fileno, int start, int stop, Enc& e, int back = 0) {
  const uint32_t o0 = a.off[fileno][i], o1 = a.off[fileno][i + 1];
  const int l = (int)(o1 - o0);
  const int n = (stop == 0) ? l - start : stop - start;
  if (l < start + n || n <= 0) return false;
  const uint8_t* s = a.bases[fileno] + o0 + start - back;
  for (int j = 0; j < n + back; ++j) e.push(s[j]);
  return true;
}

}  // namespace

__global__ void __launch_bounds__(256) bus_fields_kernel(BusArgs a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  bool valid = false;
  if (i < a.n_sets) {
    const BusSpec& sp = a.spec;
    // UMI first (a bad UMI skips the set before the barcode is looked at)
    Enc u;
    bool ok = true;
    if (sp.no_umi) {
      u.n = 1;       // "bulk_like" (:1477-1482): a one-letter dummy UMI, never encoded: the record carries umi_binary = -1
      u.r = ~0ull;
    } else {
      for (int p = 0; p < sp.n_umi && ok; ++p) ok = slice(a, i, sp.umi_f[p], sp.umi_a[p], sp.umi_b[p], u, p == 0 ? sp.tag_len : 0);
    }
    bool tag_missing = false;
    if (ok && sp.tag_len) {
      // --tag / SMARTSEQ3 (:1512-1530): the letters in front of the UMI must be the tag (one mismatch allowed when it is
      // longer than 5); then the UMI is what follows it, else the read set has no UMI at all
      const int rest = u.n - sp.tag_len;                       // letters of the UMI proper
      const unsigned long long head = (2 * rest < 64) ? (u.r >> (2 * rest)) : 0ull;
      unsigned long long df = head ^ sp.tag_bin;
      int d = 0;
      for (int j = 0; j < sp.tag_len; ++j, df >>= 2) d += (df & 3ull) != 0;
      if (d <= (sp.tag_len <= 5 ? 0 : 1)) {
        if (rest < 32) u.r &= ~(~0ull << (2 * rest));
        u.n = rest;
      } else {
        tag_missing = true;
        u.r = ~0ull;
        u.n = 99;                                              // no UMI length is recorded for it
      }
    }
    if (ok) {
      if (u.n <= 32) atomicAdd(&a.umi_hist[u.n], 1u);
      Enc b;
      if (sp.n_bc == 0) {
        b.n = 16;   // BUSFORMAT_FAKE_BARCODE_LEN: 16 x 'A' (binary 0), or the sample's id in batch mode
        b.r = sp.fake_bc;
      } else {
        for (int p = 0; p < sp.n_bc && ok; ++p) ok = slice(a, i, sp.bc_f[p], sp.bc_a[p], sp.bc_b[p], b);
      }
      if (ok) {
        if (b.n <= 32) atomicAdd(&a.bc_hist[b.n], 1u);
        uint32_t bf = b.flag();
        if (sp.batch_bc) {
          // --batch-barcodes (:1617-1626): binaryToString(batch, 32 - blen) + binaryToString(stringToBinary(bc), blen),
          // re-encoded: 32 letters with the sample's number in front, an N already turned into G, so no N flag.  Past
          // 32 letters the reference's 32 - blen wraps around; such a set stops the run on the host instead.
          if (b.n > 32) atomicAdd(a.n_long_bc, 1ull);
          else if (b.n < 32) b.r |= (sp.bc_prefix & ((1ull << (64 - 2 * b.n)) - 1)) << (2 * b.n);
          bf = 0;
        }
        a.barcode[i] = b.r;
        a.umi[i] = u.r;
        // without a UMI stringToBinary runs once only, so the UMI half of the flags repeats the barcode's (:1736-1743)
        const uint32_t uf = (sp.no_umi || sp.tag_len) ? bf : u.flag();
        a.flags[i] = sp.num_flag ? (uint32_t)(a.set_base + i) : (bf | (uf << 8));
        valid = true;
      }
    }
    a.skip[i] = valid ? 0 : 1;
    if (a.notag) a.notag[i] = (valid && tag_missing) ? 1 : 0;
  }
  const unsigned m = __ballot_sync(0xFFFFFFFFu, valid);
  if ((threadIdx.x & 31) == 0 && m) atomicAdd(a.n_valid, (unsigned long long)__popc(m));
}

// flag the fragment that is the first occurrence of its set handle
__global__ void bus_newflag_kernel(DevDict dd, const int32_t* handle, uint32_t n, uint64_t base, uint32_t* is_new,
                                   uint32_t* is_mapped) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  const int32_t h = handle[f];
  is_mapped[f] = h >= 0 ? 1u : 0u;
  is_new[f] = (h >= 0 && dd.first[h] == base + f) ? 1u : 0u;
}

__global__ void bus_newid_kernel(const int32_t* handle, uint32_t n, const uint32_t* is_new, const uint32_t* new_rank,
                                 uint32_t next_id, int32_t* id_of) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  if (is_new[f]) id_of[handle[f]] = (int32_t)(next_id + new_rank[f]);
}

// bus --devices: the run-wide ids of the sets new on this run, chosen by the group on the host (gid, by new_rank)
__global__ void bus_newid_gid_kernel(const int32_t* handle, uint32_t n, const uint32_t* is_new, const uint32_t* new_rank,
                                     const int32_t* gid, int32_t* id_of) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n) return;
  if (is_new[f]) id_of[handle[f]] = gid[new_rank[f]];
}

// bus --devices: per fragment, the length of its set when the fragment is that set's first occurrence on this run
__global__ void bus_newlen_kernel(DevDict dd, const int32_t* handle, uint32_t n, const uint32_t* is_new, uint32_t* len) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > n) return;
  len[f] = (f < n && is_new[f]) ? (uint32_t)((__ldcg(&dd.dslots[handle[f]]) >> 32) & 0xFFFFFFu) : 0u;
}

// bus --devices: the new sets as CSR in new_rank order (out_off: n_new + 1 entries, out_tid: their transcript ids).
// eoff is the exclusive scan of bus_newlen_kernel's lengths over n + 1 items, so eoff[n] is the total; ids that would
// pass `cap` are not written (the host sees the total and gathers again into a larger buffer).
__global__ void bus_export_kernel(DevDict dd, const int32_t* handle, uint32_t n, const uint32_t* is_new,
                                  const uint32_t* new_rank, const uint32_t* eoff, uint32_t cap, uint32_t* out_off,
                                  uint32_t* out_tid) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f > n) return;
  if (f == n) { out_off[new_rank[n]] = eoff[n]; return; }
  if (!is_new[f]) return;
  const uint32_t o = eoff[f];
  out_off[new_rank[f]] = o;
  const unsigned long long word = __ldcg(&dd.dslots[handle[f]]);
  const uint32_t l = (uint32_t)((word >> 32) & 0xFFFFFFu);
  if ((uint64_t)o + l > cap) return;
  const uint32_t* src = dd.pool + (uint32_t)word;
  for (uint32_t j = 0; j < l; ++j) out_tid[o + j] = __ldcg(src + j);
}

__global__ void bus_records_kernel(const int32_t* handle, uint32_t n, const uint32_t* is_mapped, const uint32_t* rank,
                                   const int32_t* id_of, const uint64_t* barcode, const uint64_t* umi, const uint32_t* flags,
                                   BusRecord* out) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= n || !is_mapped[f]) return;
  BusRecord r;
  r.barcode = barcode[f];
  r.umi = umi[f];
  r.ec = id_of[handle[f]];
  r.count = 1;
  r.flags = flags[f];
  r.pad = 0;
  out[rank[f]] = r;
}

size_t bus_scan_bytes(uint32_t n) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n + 1);
  return b + 256;
}

void launch_bus_fields(const BusArgs& a, cudaStream_t st) {
  if (a.n_sets == 0) return;
  bus_fields_kernel<<<(a.n_sets + 255) / 256, 256, 0, st>>>(a);
}

// After match + resolve: ids for the new ECs, then the compacted records.  Totals (new ECs, records)
// land in new_rank[n] and rank[n].
void launch_bus_records(const DevDict& dd, const int32_t* handle, uint32_t n, uint64_t base, uint32_t next_id,
                        int32_t* id_of, uint32_t* is_new, uint32_t* new_rank, uint32_t* is_mapped, uint32_t* rank,
                        const uint64_t* barcode, const uint64_t* umi, const uint32_t* flags, BusRecord* out, void* tmp,
                        size_t tmp_bytes, cudaStream_t st) {
  if (n == 0) return;
  const unsigned g = (n + 255) / 256;
  cudaMemsetAsync(is_new + n, 0, 4, st);
  cudaMemsetAsync(is_mapped + n, 0, 4, st);
  bus_newflag_kernel<<<g, 256, 0, st>>>(dd, handle, n, base, is_new, is_mapped);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, is_new, new_rank, (int)n + 1, st);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, is_mapped, rank, (int)n + 1, st);
  bus_newid_kernel<<<g, 256, 0, st>>>(handle, n, is_new, new_rank, next_id, id_of);
  bus_records_kernel<<<g, 256, 0, st>>>(handle, n, is_mapped, rank, id_of, barcode, umi, flags, out);
}

// bus --devices, first half: the flags and ranks of launch_bus_records, then the sets new on this run as CSR
// (launch_bus_export_gather).  Totals land in new_rank[n] (new sets), eoff[n] (their ids) and rank[n] (records).
void launch_bus_new_sets(const DevDict& dd, const int32_t* handle, uint32_t n, uint64_t base, uint32_t* is_new,
                         uint32_t* new_rank, uint32_t* is_mapped, uint32_t* rank, uint32_t* len, uint32_t* eoff,
                         uint32_t cap, uint32_t* out_off, uint32_t* out_tid, void* tmp, size_t tmp_bytes, cudaStream_t st) {
  if (n == 0) return;
  const unsigned g = (n + 255) / 256, g1 = (n + 256) / 256;
  cudaMemsetAsync(is_new + n, 0, 4, st);
  cudaMemsetAsync(is_mapped + n, 0, 4, st);
  bus_newflag_kernel<<<g, 256, 0, st>>>(dd, handle, n, base, is_new, is_mapped);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, is_new, new_rank, (int)n + 1, st);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, is_mapped, rank, (int)n + 1, st);
  bus_newlen_kernel<<<g1, 256, 0, st>>>(dd, handle, n, is_new, len);
  cub::DeviceScan::ExclusiveSum(tmp, tmp_bytes, len, eoff, (int)n + 1, st);
  launch_bus_export_gather(dd, handle, n, is_new, new_rank, eoff, cap, out_off, out_tid, st);
}

void launch_bus_export_gather(const DevDict& dd, const int32_t* handle, uint32_t n, const uint32_t* is_new,
                              const uint32_t* new_rank, const uint32_t* eoff, uint32_t cap, uint32_t* out_off,
                              uint32_t* out_tid, cudaStream_t st) {
  if (n == 0) return;
  bus_export_kernel<<<(n + 256) / 256, 256, 0, st>>>(dd, handle, n, is_new, new_rank, eoff, cap, out_off, out_tid);
}

// bus --devices, second half: the run-wide ids of the new sets (gid, n_new of them, by new_rank), then the records
void launch_bus_group_records(const int32_t* handle, uint32_t n, const uint32_t* is_new, const uint32_t* new_rank,
                              const int32_t* gid, int32_t* id_of, const uint32_t* is_mapped, const uint32_t* rank,
                              const uint64_t* barcode, const uint64_t* umi, const uint32_t* flags, BusRecord* out,
                              cudaStream_t st) {
  if (n == 0) return;
  const unsigned g = (n + 255) / 256;
  bus_newid_gid_kernel<<<g, 256, 0, st>>>(handle, n, is_new, new_rank, gid, id_of);
  bus_records_kernel<<<g, 256, 0, st>>>(handle, n, is_mapped, rank, id_of, barcode, umi, flags, out);
}

}  // namespace kb
