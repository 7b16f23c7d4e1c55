// Translated search (bus --aa, src/ProcessReads.cpp:1652-1695): every read set is matched in its six reading frames
// against an index built over proteins in comma-free code (cfc), and the frame with the smallest non-empty set wins.
//
//   cfc_len_kernel / cfc_frames_kernel   the six frames of every set as ASCII cfc reads (one thread per set, frame
//                                        and group of codons); they go through pack_kernel -> match_kernel ->
//                                        resolve_kernel as 6n unpaired, unstranded fragments that are not counted
//   cfc_select_kernel                    per set: the winning frame (MinCollector::intersectKmersCFC,
//                                        src/MinCollector.cpp:44-119), the frame-0 strand filter
//                                        (doStrandSpecificity, src/ProcessReads.cpp:61-110, with v = frame 0's hits)
//                                        and the accounting of the set
//
// Frame j of a sequence s of length L reads from (j < 3 ? s : revcomp(s)) + j % 3 and has l_j = L - j % 3 letters.
// The reference translates it with nn_to_cfc (src/KmerIndex.cpp:19-85,118-138): every full triplet becomes the three
// letters of its amino acid's code, a stop codon or a triplet with a letter other than A/C/G/T (either case) becomes
// NNN, and the l_j mod 3 letters of a trailing partial triplet are dropped.  match() then walks the cfc string of
// 3 floor(l_j / 3) letters, but bounds its jumps with the NUCLEOTIDE length l_j (l - k, src/KmerIndex.cpp:1795-1820).
// Here the frame is written with its partial triplet replaced by l_j mod 3 letters N, so it has exactly l_j letters and
// match_kernel's bounds, which use the read length, are the reference's.  The tail changes no k-mer walk: the
// reference's KmerIterator (ext/bifrost/src/KmerIterator.cpp:40-63) becomes invalid both where the string ends and
// where no window without a letter other than A/C/G/T is left, and a window that reaches into the N tail is such a
// window, so match_kernel's next_valid answers -1 exactly where the reference's iterator ends.
#include <cub/cub.cuh>

#include "kb_device.cuh"
#include "kb_dict.cuh"
#include "kernels.hpp"

namespace kb {

namespace {

// The comma-free code of every codon (nn_to_cfc's cfc_map), codon = b0 * 16 + b1 * 4 + b2 with A 0, C 1, G 2, T 3;
// NNN for the three stop codons.
__constant__ char kCfc[64 * 3 + 1] =
    "CGCCGACGCCGACTTCTTCTTCTTTGTCTATGTCTAATAATAATCATAAGGAGTAGGAGTCTCCTCCTCCTCTGTTGTTGTTGTACAACAACAACACGGCGTCGGCG"
    "TAGAAGAAGAAGATGGTGGTGGTGGATTATTATTATTNNNAGCNNNAGCCTACTACTACTANNNTGATGCTGAACAACCACAACC";

__device__ __forceinline__ int base2(uint8_t c) {
  switch (c) {
    case 'A': case 'a': return 0;
    case 'C': case 'c': return 1;
    case 'G': case 'g': return 2;
    case 'T': case 't': return 3;
    default: return -1;
  }
}

// length of set i's sequence, 0 for a skipped set
__device__ __forceinline__ uint32_t seq_len(const CfcArgs& a, uint32_t i, uint64_t& off) {
  const uint32_t o0 = a.off[i], o1 = a.off[i + 1];
  off = (uint64_t)o0 + a.start;
  if (a.skip && a.skip[i]) return 0;
  return o1 - o0 > a.start ? o1 - o0 - a.start : 0;
}

__device__ __forceinline__ uint32_t frame_len(uint32_t L, int j) { return L > (uint32_t)(j % 3) ? L - (uint32_t)(j % 3) : 0; }

constexpr int kCodonsPerThread = 4;

}  // namespace

// letters of the six frames of every set into foff[0 .. n_sets), 0 into foff[n_sets] (the scan's last input)
__global__ void cfc_len_kernel(CfcArgs a) {
  const uint32_t i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i > a.n_sets) return;
  uint32_t tot = 0;
  if (i < a.n_sets) {
    uint64_t off;
    const uint32_t L = seq_len(a, i, off);
    for (int j = 0; j < 6; ++j) tot += frame_len(L, j);
  }
  a.foff[i] = tot;
}

// One thread per (set, frame, kCodonsPerThread codons); the first thread of a frame also writes the frame's offset.
__global__ void __launch_bounds__(256) cfc_frames_kernel(CfcArgs a, uint32_t groups) {
  const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  if (gid >= (uint64_t)a.n_sets * 6 * groups) return;
  const uint32_t g = (uint32_t)(gid % groups);
  const uint32_t f = (uint32_t)(gid / groups);
  const uint32_t i = f / 6;
  const int j = (int)(f - 6 * i);
  uint64_t off;
  const uint32_t L = seq_len(a, i, off);
  const uint32_t lj = frame_len(L, j);
  uint32_t dst = a.set_off[i];
  for (int jj = 0; jj < j; ++jj) dst += frame_len(L, jj);
  if (g == 0) {
    a.foff[f] = dst;
    if (f == 6 * a.n_sets - 1) a.foff[f + 1] = a.set_off[a.n_sets];
  }
  const uint8_t* s = a.bases + off;
  const bool rc = j >= 3;
  const uint32_t sh = (uint32_t)(j % 3);
  for (int c = 0; c < kCodonsPerThread; ++c) {
    const uint32_t q = 3 * (g * kCodonsPerThread + c);
    if (q >= lj) break;
    uint8_t* out = a.fbases + dst + q;
    if (q + 3 > lj) {                     // the partial triplet: N up to the nucleotide length
      for (uint32_t x = q; x < lj; ++x) out[x - q] = 'N';
      break;
    }
    int code = 0;
    bool ok = true;
#pragma unroll
    for (int t = 0; t < 3; ++t) {
      const uint32_t y = sh + q + (uint32_t)t;                 // position in the frame's source string
      int b = base2(rc ? s[L - 1 - y] : s[y]);
      if (rc && b >= 0) b = 3 - b;                              // revcomp (src/common.cpp:36-53)
      ok = ok && b >= 0;
      code = code * 4 + (b & 3);
    }
    if (ok) {
      out[0] = (uint8_t)kCfc[3 * code]; out[1] = (uint8_t)kCfc[3 * code + 1]; out[2] = (uint8_t)kCfc[3 * code + 2];
    } else {
      out[0] = out[1] = out[2] = 'N';
    }
  }
}

// G lanes per read set (grid-stride over the sets, ra.scratch as per-group scratch).
template <int G>
__global__ void __launch_bounds__(128) cfc_select_kernel(DevIndex ix, DevDict dd, BatchArgs ba, ResolveArgs ra, uint32_t n_sets,
                                                         uint32_t n_groups, int strand_mode, int32_t* handle_out,
                                                         unsigned long long* clashes) {
  const unsigned lane = threadIdx.x & (G - 1);
  const unsigned gmask = group_mask<G>(threadIdx.x & 31);
  const unsigned gshift = (threadIdx.x & 31) & ~(unsigned)(G - 1);
  const uint32_t grp = (blockIdx.x * blockDim.x + threadIdx.x) / G;
  if (grp >= n_groups) return;
  uint32_t* scratch = ra.scratch + (size_t)grp * ra.scratch_stride;
  unsigned long long n_clash = 0;
  for (uint32_t i = grp; i < n_sets; i += n_groups) {
    // the six frames' set handles and sizes
    int32_t h = KB_H_UNMAPPED;
    uint32_t sz = 0;
    if (lane < 6) {
      h = ba.handle_out[6 * i + lane];
      if (h >= 0) sz = (uint32_t)((dd.dslots[h] >> 32) & 0xFFFFFFu);
    }
    // intersectKmersCFC: the smallest non-empty set, the lowest frame on a tie; a clash for every later frame as small
    // as the smallest set before it
    int32_t win = KB_H_UNMAPPED;
    uint32_t best = 0xFFFFFFFFu;
    for (int j = 0; j < 6; ++j) {
      const uint32_t s = __shfl_sync(gmask, sz, j, G);
      const int32_t hj = __shfl_sync(gmask, h, j, G);
      if (s > 0 && s < best) { best = s; win = hj; }
      else if (s > 0 && s == best) ++n_clash;
    }
    int32_t handle = win;
    // doStrandSpecificity with v = frame 0's hits, whichever frame won: u &= the EC of the block of frame 0's first
    // mapping k-mer, keeping the members whose sense agrees with the strand (src/ProcessReads.cpp:1728-1735,61-110)
    const uint32_t fh = (win >= 0 && strand_mode != 0) ? ba.first_hit[6 * i] : 0xFFFFFFFFu;
    if (fh != 0xFFFFFFFFu) {
      const uint32_t blk = fh >> 1;
      const bool um_strand = (fh & 1u) != 0;
      const bool want = strand_mode == 1;
      const unsigned long long bword = dd.dslots[ix.blk_ec[blk]];
      const uint32_t* B = dd.pool + (uint32_t)bword;
      const uint32_t blen = (uint32_t)((bword >> 32) & 0xFFFFFFu);
      const uint8_t* sb = ix.strand + ix.blk_strand_off[blk];
      const uint32_t* A = dd.pool + (uint32_t)dd.dslots[win];
      uint32_t n_v = 0;
      for (uint32_t base = 0; base < best; base += G) {
        const uint32_t x = base + lane;
        const uint32_t a = x < best ? __ldcg(A + x) : 0;
        uint32_t rank = 0;
        bool keep = x < best && bsearch_contains(B, blen, a, &rank);
        if (keep) {
          const uint8_t sense = sb[rank];
          keep = ((um_strand == (sense != 0)) == want) || sense == 2;
        }
        const unsigned bv = (__ballot_sync(gmask, keep) >> gshift);
        if (keep) scratch[n_v + __popc(bv & ((1u << lane) - 1))] = a;
        n_v += __popc(bv);
      }
      __syncwarp(gmask);
      if (n_v == 0) handle = KB_H_UNMAPPED;
      else if (n_v < best) handle = dict_insert_warp<G>(dd, scratch, n_v, lane, gmask);
    }
    if (lane == 0) {
      handle_out[i] = handle;
      if (handle >= 0) {
        atomicAdd(&dd.count[handle], 1u);
        atomicMin(&dd.first[handle], (unsigned long long)(ba.frag_base + i));
      }
    }
    __syncwarp(gmask);
  }
  if (lane == 0 && n_clash) atomicAdd(clashes, n_clash);
}

size_t cfc_scan_bytes(uint32_t n_sets) {
  size_t b = 0;
  cub::DeviceScan::ExclusiveSum(nullptr, b, (const uint32_t*)nullptr, (uint32_t*)nullptr, (int)n_sets + 1);
  return b + 256;
}

void launch_cfc_frames(const CfcArgs& a, cudaStream_t st) {
  if (a.n_sets == 0) return;
  cfc_len_kernel<<<(a.n_sets + 1 + 255) / 256, 256, 0, st>>>(a);
  size_t tb = a.tmp_bytes;
  cub::DeviceScan::ExclusiveSum(a.tmp, tb, a.foff, a.set_off, (int)a.n_sets + 1, st);
  const uint32_t groups = (a.max_len + 3 * kCodonsPerThread - 1) / (3 * kCodonsPerThread);
  const uint64_t total = (uint64_t)a.n_sets * 6 * (groups ? groups : 1);
  cfc_frames_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(a, groups ? groups : 1);
}

void launch_cfc_select(const DevIndex& ix, const DevDict& dd, const BatchArgs& ba, const ResolveArgs& ra, uint32_t n_sets,
                       int strand_mode, int32_t* handle_out, unsigned long long* clashes, cudaStream_t st) {
  if (n_sets == 0) return;
  constexpr int G = 8;      // the sets are short: 8 lanes hold a set, a warp serves four
  const uint32_t n_groups = n_sets < ra.n_warps ? n_sets : ra.n_warps;
  cfc_select_kernel<G><<<(n_groups * G + 127) / 128, 128, 0, st>>>(ix, dd, ba, ra, n_sets, n_groups, strand_mode, handle_out,
                                                                  clashes);
}

}  // namespace kb
