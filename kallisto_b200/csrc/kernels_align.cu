// K1: per-fragment pseudoalignment on the device.
//
//   match_kernel    one thread per fragment (read pair or single read).  Restates
//                   KmerIndex::match (src/KmerIndex.cpp:1698-1940: k-mer iteration, skip-ahead to the
//                   end of the EC block, middle probe, one-step back-off) on the flat 32-byte-slot
//                   table, then the pair combination of MinCollector::intersectKmers /
//                   intersectECs (src/MinCollector.cpp:160-218, 425-496) reduced to its net effect:
//                   the intersection of the distinct non-empty EC sets hit by the two mates.
//                   Fragments whose hits fall in a single EC set, or whose tuple of EC sets has been
//                   seen before (memo tables), are finished here; the others are queued.
//   resolve_kernel  one warp per queued fragment: warp-cooperative sorted-list intersection
//                   (lanes own elements of the smallest set and binary-search the others), the strand
//                   filter of doStrandSpecificity (src/ProcessReads.cpp:61-124), content-addressed
//                   dictionary insert (ecmapinv semantics) and memo publication.
//
// Per-fragment result = a set handle; per-handle counters (count, first fragment index) replace
// MasterProcessor::update + MinCollector::increaseCount (src/ProcessReads.cpp:424-483,
// src/MinCollector.cpp:251-269): EC ids are assigned afterwards in order of first occurrence,
// which is what the reference produces with -t 1.
#include "kb_device.cuh"
#include "kb_dict.cuh"
#include "kernels.hpp"

#ifndef KB_MATCH_MIN_BLOCKS
// 3 blocks of 256 lanes per SM (1 536 lanes, two lookup chains each) at up to 80 registers, with no local memory; at 4
// blocks the 64 registers still do not hold the two chains' state and the lookup loop spills
#define KB_MATCH_MIN_BLOCKS 3
#endif
#ifdef KB_MATCH_STATS
#include <cstdio>
#endif

namespace kb {

#ifdef KB_MATCH_STATS
// Instrumented build (-DKB_MATCH_STATS, tools/match_stats.py): per-launch counters of match_kernel, printed to stderr
// by launch_pseudoalign.  The counters and the host synchronisation slow the kernel; only their ratios mean something.
enum : int {
  MS_WARP_ITERS, MS_SERVICE_ROUNDS, MS_LANE_ITERS, MS_CHAIN_ITERS,
  MS_MAIN_HIT, MS_MAIN_MISS_FILTER, MS_MAIN_MISS_SLOT, MS_JUMP, MS_MIDDLE, MS_BACKOFF, MS_COLLISION,
  MS_CYCLES_LOOKUP, MS_CYCLES_SERVICE,
  // split of a lane-iteration's cycles, summed over lanes (cycles_lookup and cycles_service are lane 0's): keys and hashes
  // up to the filter loads, the wait for the filter and slot loads, and the state transitions (with the handle dedup)
  MS_CYCLES_KEY, MS_CYCLES_WAIT, MS_CYCLES_STEP,
  // chain iterations settled on the straight-line path (collision, MAIN miss on a mate without N), and the passes of the
  // general transition per warp-iteration (summed over warps; a warp runs as many as its busiest lane needs)
  MS_STRAIGHT, MS_GEN_PASSES,
  MS_RUN_HIST, MS_N = MS_RUN_HIST + 9     // MAIN miss runs of 1, 2, 3, 4, 5-8, 9-16, 17-32, 33-64, 65+ positions
};
__device__ unsigned long long kb_match_stats[MS_N];
static const char* const kMatchStatNames[MS_N] = {
  "warp_iters", "service_rounds", "lane_iters", "chain_iters",
  "main_hit", "main_miss_filter", "main_miss_slot", "jump", "middle", "backoff", "collision",
  "cycles_lookup", "cycles_service", "cycles_key", "cycles_wait", "cycles_step", "straight", "gen_passes",
  "run_1", "run_2", "run_3", "run_4", "run_5_8", "run_9_16", "run_17_32", "run_33_64", "run_65_"};
__device__ __forceinline__ int run_bin(int n) {
  return n <= 4 ? n - 1 : (n <= 8 ? 4 : (n <= 16 ? 5 : (n <= 32 ? 6 : (n <= 64 ? 7 : 8))));
}
#define KB_MS(i, n) (ms[i] += (unsigned long long)(n))
#define KB_MS_ONLY(x) x
#else
#define KB_MS(i, n) ((void)0)
#define KB_MS_ONLY(x)
#endif

namespace {

__device__ __forceinline__ int32_t ld_relaxed_s32(const int32_t* p) {
  int32_t v;
  asm volatile("ld.relaxed.gpu.global.s32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// One 32-byte read-only load as two 128-bit loads (sm_90a has no 256-bit global load): a whole
// k-mer slot, half a packed read, or a block of memo entries.  The address must be 32-byte aligned,
// so both halves fall in the same 32-byte sector and the probe still costs one sector of traffic.
__device__ __forceinline__ void ld256_nc(const void* p, uint32_t (&w)[8]) {
  asm volatile("ld.global.nc.v4.b32 {%0,%1,%2,%3}, [%8]; ld.global.nc.v4.b32 {%4,%5,%6,%7}, [%8+16];"
               : "=r"(w[0]), "=r"(w[1]), "=r"(w[2]), "=r"(w[3]), "=r"(w[4]), "=r"(w[5]), "=r"(w[6]), "=r"(w[7])
               : "l"(p));
}
// Per-lane view of the read being matched: 2-bit bases in shared memory as 32-bit words (base i in
// bits 30-2*(i&15) of word i>>4), word w of lane t at [w * stride + t] (bank-conflict free).
// Bases other than A/C/G/T are rare, so the lane keeps only a flag in a register; a read that has
// one consults the invalid-base masks of its packed form in global memory (bit i&31 of word i>>5;
// positions past the end of the read are marked invalid there as well).
struct ReadView {
  const uint32_t* bw;
  const uint32_t* gmask;
  int n_mask;
  int stride;
  int len;
  int k;
  bool has_invalid;

  __device__ __forceinline__ uint64_t kmer(int p) const {
    const int w = p >> 4, s = (p & 15) * 2;
    uint64_t x = (uint64_t)bw[w * stride] << 32;
    if (s + 2 * k > 32) x |= bw[(w + 1) * stride];
    x <<= s;
    if (s + 2 * k > 64) x |= (uint64_t)(bw[(w + 2) * stride] >> (32 - s));   // s > 0 here: 2k <= 62
    return x >> (64 - 2 * k);
  }
  // first start position >= p whose k-window holds only A/C/G/T, or -1
  // (KmerIterator::operator++ / operator+=, ext/bifrost/src/KmerIterator.cpp:6-63)
  __device__ __forceinline__ int next_valid(int p) const {
    if (!has_invalid) return p <= len - k ? p : -1;
    const uint64_t wmask = (1ULL << k) - 1;
    while (p <= len - k) {
      const int w = p >> 5, s = p & 31;
      const uint64_t lo = __ldg(gmask + w);
      const uint64_t hi = (w + 1 < n_mask) ? __ldg(gmask + w + 1) : 0xFFFFFFFFu;
      const uint64_t x = (((hi << 32) | lo) >> s) & wmask;      // s + k <= 63
      if (x == 0) return p;
      p += 64 - __clzll((long long)x);
    }
    return -1;
  }
};

__device__ __forceinline__ uint64_t tuple_hash(const uint32_t* w, int n, int stride) {
  uint64_t h = 0x243F6A8885A308D3ULL ^ (uint64_t)n;
  for (int i = 0; i < n; ++i) h = kb_mix64(h ^ ((uint64_t)w[i * stride] + 0x9E3779B97F4A7C15ULL * (i + 1)));
  return h;
}

// Memo lookups used by the resolve kernel (one lane).  Return KB_H_NOTREADY on a miss.
__device__ __forceinline__ int32_t memo2_lookup(const DevDict& dd, uint32_t e0, uint32_t e1) {
  const unsigned long long key = ((unsigned long long)e0 << 32) | e1;
  uint64_t s = kb_mix64(key) & dd.m2_mask;
  for (;;) {
    const unsigned long long kk = __ldcg(&dd.m2[s].key);
    if (kk == key) return ld_relaxed_s32(&dd.m2[s].val);
    if (kk == ~0ULL) return KB_H_NOTREADY;
    s = (s + 1) & dd.m2_mask;
  }
}
__device__ __forceinline__ bool tuple_equal(const DevDict& dd, uint32_t toff, const uint32_t* w, int n, int stride) {
  const uint32_t* t = dd.tpool + toff;
  bool eq = __ldcg(t) == (uint32_t)n;
  for (int i = 0; eq && i < n; ++i) eq = __ldcg(t + 1 + i) == w[i * stride];
  return eq;
}
__device__ __forceinline__ int32_t memon_lookup(const DevDict& dd, const uint32_t* w, int n, int stride) {
  const uint64_t th = tuple_hash(w, n, stride);
  const uint32_t tag = (uint32_t)(th >> 32);
  uint64_t s = th & dd.mn_mask;
  for (;;) {
    const unsigned long long word = ld_acquire_u64(&dd.mn_key[s]);
    if (word == ~0ULL) return KB_H_NOTREADY;
    if ((uint32_t)(word >> 32) == tag && tuple_equal(dd, (uint32_t)word, w, n, stride)) return ld_relaxed_s32(&dd.mn_val[s]);
    s = (s + 1) & dd.mn_mask;
  }
}

// Location of read `ridx` of a batch (mates interleaved in one buffer, or one buffer per mate).
__device__ __forceinline__ void read_span(const BatchArgs& ba, uint32_t ridx, const uint8_t*& base, uint64_t& off, int& len) {
  base = ba.bases;
  const uint32_t* offs = ba.off;
  uint32_t i = ridx;
  if (ba.bases2) {
    i = ridx >> 1;
    if (ridx & 1) { base = ba.bases2; offs = ba.off2; }
  }
  if (offs) {
    const uint32_t o0 = offs[i], o1 = offs[i + 1];
    off = o0;
    len = (int)(o1 - o0);
  } else {
    off = (uint64_t)i * ba.fixed_len;
    len = (int)ba.fixed_len;
  }
  const bool second = ba.paired && (ridx & 1);
  uint32_t st = second ? ba.start2 : ba.start;
  if (ba.notag && ba.notag[ba.paired ? (ridx >> 1) : ridx]) st = second ? ba.alt_start2 : ba.alt_start;
  if (st) {
    off += st;
    len -= (int)st;
    if (len < 0) len = 0;
  }
  if (ba.skip && ba.skip[ba.paired ? (ridx >> 1) : ridx]) len = 0;
}

// States of a lookup chain of match_kernel.
enum : int {
  S_MAIN = 0, S_JUMP = 1, S_MIDDLE = 2, S_BACKOFF = 3,   // k-mer table lookups (KmerIndex::match control flow)
  S_FIN = 4,                                             // chain ended; the fragment waits for the next service round once both have
  S_EMPTY = 5                                            // no fragment assigned
};
// What a chain's next lookup does to its k-mer before the probe.
enum : int {
  P_NONE = 0,      // nothing: the same key at the next slot (linear probing)
  P_BUILD = 1,     // read it from the packed bases at the state's position
  P_ROLL = 2       // shift in one base: the lookup is at p + 1 of the k-mer the chain holds
};
// Cold words of a chain in shared memory: word w of chain c of a lane is its per-lane word KB_MAX_E + 2 * w + c.  The
// first three (the chain's first hit) are overwritten when a finalised tuple grows past KB_MAX_E.  The rest are only
// read when a JUMP or MIDDLE key is formed and in the transitions out of those states: the reference's nextPos, the
// second hit of a jump (unitig, set handle), the jump and middle positions, the distance to the end of the EC block and
// the hit the jump started from (unitig, set handle).
enum : int { C_BLK = 0, C_DS = 1, C_POS = 2, C_NP = 3, C_H2U = 4, C_H2E = 5, C_P2 = 6, C_P3 = 7, C_DIST = 8, C_HU = 9, C_HE = 10 };
static_assert(C_HE + 1 == KB_CHAIN_WORDS, "match_lane_words counts every cold word of a chain");

}  // namespace

// ---------------------------------------------------------------------------------------------
// pack_kernel: ASCII reads -> 2-bit bases + invalid-base masks, one thread per (read, 32-base word).
// Streaming and convergent: nine aligned 32-bit loads per thread (whatever the byte offset of the read; never past
// the word that holds the read's last base), then 4 bases at a time with SWAR arithmetic
//   idx   = (c >> 1) & 3                      A 0, C 1, T 2, G 3
//   code  = idx ^ (idx >> 1)                  == Kmer::set_kmer (Kmer.cpp:92-107) on A/C/G/T
//   valid = (c & 0xDF) == "ACTG"[idx]         == isDNA(c & 0xDF)  (KmerIterator.cpp:12-14); the four expected letters
//                                             of a group come from ONE byte permute of the constant "ACTG" with the
//                                             indices as selector, so a group costs 13 instructions; the per-base mask
//                                             is only assembled for words that hold a non-ACGT letter or the read's end
// Packed read = nb 64-bit base words, then nb 32-bit invalid masks, padded (with "invalid") to a
// multiple of 32 bytes.  Bases past the end of the read are packed as A and marked invalid.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) pack_kernel(BatchArgs ba, uint32_t n_reads, uint32_t* out) {
  const uint32_t gid = blockIdx.x * blockDim.x + threadIdx.x;     // launch_pseudoalign: n_reads * nb < 2^32
  const uint32_t nb = ba.nb;
  if (gid >= n_reads * nb) return;
  const uint32_t r = gid / nb, w = gid - r * nb;
  uint64_t off;
  int len;
  const uint8_t* src_bases;
  read_span(ba, r, src_bases, off, len);
  if (w == 0) ba.rlen[r] = (uint32_t)len;
  const int base = (int)w * 32;
  uint32_t hi = 0, lo = 0, inv32 = ~0u;
  if (base < len) {
    const int n = min(32, len - base);
    const uint64_t a = off + (uint64_t)base;
    const uint32_t* wp = reinterpret_cast<const uint32_t*>(src_bases + (a & ~3ull));
    const int sh = (int)(a & 3) * 8;
    const int last = ((int)(a & 3) + n - 1) >> 2;       // index of the aligned word holding base n-1
    uint32_t wd[9];
#pragma unroll
    for (int q = 0; q < 9; ++q) wd[q] = __ldg(wp + min(q, last));
    uint32_t d[8], pr[8];
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      const uint32_t four = __funnelshift_r(wd[q], wd[q + 1], sh);
      uint32_t x = (four >> 1) & 0x03030303u;
      const uint32_t y = (x | (x >> 4)) & 0x00330033u;                  // index nibbles of bytes 0,1 and of bytes 2,3
      d[q] = (four & 0xDFDFDFDFu) ^ __byte_perm(0x47544341u, 0u, y | (y >> 8));   // 0 where the letter is the expected one
      x ^= (x >> 1) & 0x01010101u;
      pr[q] = x * 0x40100401u;                                          // byte 3 = b0<<6 | b1<<4 | b2<<2 | b3
    }
    hi = __byte_perm(__byte_perm(pr[3], pr[2], 0x0073u), __byte_perm(pr[1], pr[0], 0x0073u), 0x5410u);
    lo = __byte_perm(__byte_perm(pr[7], pr[6], 0x0073u), __byte_perm(pr[5], pr[4], 0x0073u), 0x5410u);
    const bool full = (n == 32);
    uint32_t any = full ? (d[0] | d[1] | d[2] | d[3] | d[4] | d[5] | d[6] | d[7]) : 1u;
    inv32 = 0;
    if (any) {
      const int ng = (n + 3) >> 2;    // a warp whose only lanes here are read ends (4 bases of a 100-base read) leaves after one group
#pragma unroll
      for (int q = 0; q < 8; ++q) {
        if (q >= ng) break;
        uint32_t t = (d[q] & 0x7F7F7F7Fu) + 0x7F7F7F7Fu;
        t = (t | d[q]) & 0x80808080u;                                   // bit 7 of a byte = letter differs
        inv32 |= (((t >> 7) * 0x01020408u) >> 24) << (4 * q);           // bit j = base j invalid
      }
    }
    if (!full) {                      // n in [1, 31]: bases n.. are not part of the read
      inv32 |= ~0u << n;
      if (n > 16) lo &= ~0u << (64 - 2 * n);
      else { lo = 0; if (n < 16) hi &= ~0u << (32 - 2 * n); }
    }
  }
  uint32_t* dst = out + (size_t)r * ba.pstride;
  reinterpret_cast<uint2*>(dst)[w] = make_uint2(lo, hi);
  dst[2 * nb + w] = inv32;
  for (uint32_t j = 3 * nb + w; j < ba.pstride; j += nb) dst[j] = ~0u;   // padding reads as "invalid"
}

// ---------------------------------------------------------------------------------------------
// dlist_scan_kernel: the D-list rule of KmerIndex::match (src/KmerIndex.cpp:1818-1826, 1928-1939).  The reference
// appends a hit on the dummy unitig -- whose equivalence class is the single off-list target -- to a read's hit list
// when any of the read's k-mers is a distinguishing flanking k-mer; the intersection with the on-list targets
// (ProcessReads.cpp:1072) is then empty.  Net effect with default flags: a fragment holding a D-list k-mer in either
// mate is not pseudoaligned.  One thread per (read, window of 32 k-mer start positions) over the packed 2-bit reads;
// a hit marks the fragment in the skip array match_kernel honours.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) dlist_scan_kernel(DevIndex ix, BatchArgs ba, uint32_t n_reads) {
  const uint64_t gid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t nb = ba.nb;
  if (gid >= (uint64_t)n_reads * nb) return;
  const uint32_t r = (uint32_t)(gid / nb), w = (uint32_t)(gid % nb);
  const uint32_t frag = ba.paired ? (r >> 1) : r;
  uint64_t off;
  int len;
  const uint8_t* unused;
  read_span(ba, r, unused, off, len);
  const int k = ix.k;
  const int p0 = (int)w * 32;
  if (len < k || p0 > len - k) return;
  const uint32_t* pk = ba.packed + (size_t)r * ba.pstride;
  const unsigned long long* bw = reinterpret_cast<const unsigned long long*>(pk);
  const unsigned long long w0 = bw[w], w1 = (w + 1 < nb) ? bw[w + 1] : 0ull;
  const unsigned long long inv = (unsigned long long)pk[2 * nb + w] | ((w + 1 < nb) ? ((unsigned long long)pk[2 * nb + w + 1] << 32) : 0xFFFFFFFF00000000ull);
  const unsigned long long wmask = (1ull << k) - 1;
  for (int j = 0; j < 32; ++j) {
    const int p = p0 + j;
    if (p > len - k) break;
    if ((inv >> j) & wmask) continue;                       // a base other than A/C/G/T in the window
    unsigned long long x = w0 << (2 * j);
    if (j) x |= w1 >> (64 - 2 * j);
    const uint64_t fwd = x >> (64 - 2 * k);
    const uint64_t rc = kb_revcomp(fwd, k);
    const uint64_t canon = fwd < rc ? fwd : rc;
    uint64_t h = kb_mix64(canon) & ix.dfk_mask;
    for (;;) {
      const unsigned long long key = __ldg(ix.dfk + h);
      if (key == canon) { ba.skip_w[frag] = 1; return; }
      if (key == KB_EMPTY_KEY) break;
      h = (h + 1) & ix.dfk_mask;
    }
  }
}

// ---------------------------------------------------------------------------------------------
// match_kernel: persistent warps, 32 independent fragment state machines per warp, two lookup chains per lane.
//
// KmerIndex::match (src/KmerIndex.cpp:1698-1940, default flags, empty D-list) is a chain of
// dependent k-mer lookups whose length varies from 2 (clean read inside one EC block) to >100
// (unmappable read: every k-mer is probed).  As straight-line per-thread code a warp pays the
// maximum over its lanes, and lanes sitting at different call sites serialise.  Here each lane
// keeps an explicit state per chain -- chain m matches mate m of the lane's fragment; single-end
// reads use chain 0 only -- and every iteration of the warp's loop performs ONE lookup per live
// chain through a single convergent site: the canonical k-mers + hashes of both chains (a k-mer one
// position after the chain's previous one is rolled from it by one base), both presence-filter
// loads, then both 32-byte slot loads (two 128-bit loads of the same sector on sm_90a), and only
// then the reference's control flow as a state transition.  Collisions and MAIN misses on mates
// without N are settled for both chains by straight-line code; the other outcomes go through one
// copy of the transition, a pass per chain that needs it, chain 0 first
//   MAIN     the k-mer at p.  Miss: next valid k-mer.  Hit: record it, distance to the end of its EC
//            block (1780-1788); if >= 2 go to JUMP.
//   JUMP     the jump target (1793-1827).  Absent or same (unitig, EC set): accepted, scanning resumes
//            after the target.  Otherwise MIDDLE (dist > 4) or BACKOFF.
//   MIDDLE   the middle k-mer (1831-1873).
//   BACKOFF  the k-mer after p, once (1876-1925: the outer nextPos is never updated, so the back-off
//            loop runs a single iteration), then MAIN.
// (linear-probing collisions cost that chain one more iteration in the same state).  The reference
// matches the two mates independently and only then intersects their hits (ProcessReads.cpp:
// index.match(s1), index.match(s2), MinCollector::intersectKmers), so a pair costs as many
// iterations as its longer mate instead of the sum, with two independent lookups in flight per
// lane.  Both chains push into the fragment's one tuple of EC-set handles; it is a set, sorted
// before use.  Lanes whose fragment is finished (both chains ended) wait until `refill_min` of
// them can be served together: the rare, expensive steps -- pair combination, memo lookup,
// accounting, loading the next packed reads -- then run convergent over many lanes instead of
// once per lane.  The lookups executed are exactly the reference's, in the same order per read.
// `partial` (single-end early exit) does not change the result and is not modelled; the pushes of
// the anchor hit at synthetic positions (1820, 1824) add no new EC set and are dropped.
// ---------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256, KB_MATCH_MIN_BLOCKS) match_kernel(DevIndex ix, DevDict dd, BatchArgs ba) {
  extern __shared__ uint32_t smem[];
  const int tid = threadIdx.x, nt = blockDim.x;
  const unsigned lane = tid & 31;
  const int nb = (int)ba.nb, nw = 2 * nb;
  const int k = ix.k;
  // shared memory per lane (32-bit words, word w of lane t at [w * nt + t]; match_lane_words): the tuple of EC-set
  // handles, the cold words of both chains (C_*), the 2-bit bases of both mates.  When a fragment is finalised the
  // handle tuple may grow by up to 6 words over the chain words that follow it; their contents are in registers by then.
  uint32_t* elist = smem + tid;                                  // [KB_MAX_E]
  uint32_t* cold = elist + (size_t)KB_MAX_E * nt;                // [2 * KB_CHAIN_WORDS]
  uint32_t* s_bw = cold + (size_t)2 * KB_CHAIN_WORDS * nt;       // [mate][nw]
  uint32_t* spill = ba.spill + ((size_t)blockIdx.x * nt + tid) * KB_SPILL;   // handles beyond KB_MAX_E (global memory)
  // the cold words after the first hit (C_NP .. C_HE) are in enum order
  static_assert(C_BLK < C_POS && C_DS < C_POS && C_POS == 2 && C_NP == C_POS + 1 && C_HE == KB_CHAIN_WORDS - 1,
                "a tuple grown by 6 words past KB_MAX_E overwrites exactly the first-hit words of both chains");
  auto cw = [&](int w, int c) -> uint32_t& { return cold[(size_t)(2 * w + c) * nt]; };

  // fragments are handed out at each refill from one counter for the whole grid, as many as the warp has idle lanes: a
  // warp whose fragments were quick takes more, so the warps run out of work together instead of each draining a
  // fixed share (and the blocks of a launch that become resident late take only what is left)
  bool work_left = true;     // warp-uniform: the counter has not passed n_frag yet
  const int n_mates = ba.paired ? 2 : 1;
  const int n_chunks = (int)(ba.pstride >> 3);   // 32-byte pieces per packed read

  // the block's totals of lookups, slot visits and memo hits, added to by each warp's service rounds
  __shared__ unsigned long long s_tot[3];
  if (tid < 3) s_tot[tid] = 0;
  __syncthreads();

  // per fragment
  uint32_t frag = 0;
  int n_e = 0;
  bool overflow = false;
  unsigned inv_flags = 0;    // bit m: mate m holds a base other than A/C/G/T
  // per chain (index = mate); the state of a jump or middle probe and the first hit live in `cold`.  The arrays are
  // only indexed by compile-time constants (unrolled loops); code that picks a chain at run time does so by selects.
  int st[2] = {S_EMPTY, S_EMPTY};
  int p[2] = {-1, -1}, len[2] = {0, 0};
  int prep[2] = {P_NONE, P_NONE};
  unsigned hv = 0, hs = 0;     // bit m: mate m has a hit / a hit on a non-empty EC set
  // the k-mer of the chain's current lookup and its reverse complement (the key is the smaller of the two)
  uint64_t fwd[2] = {0, 0}, rc[2] = {0, 0};
  uint32_t slot[2] = {0, 0};   // the table has at most 2^32 slots (KmerIndex load)
  const uint32_t slot_mask = (uint32_t)ix.mask;
  const uint64_t kmask = (1ULL << (2 * k)) - 1;
  uint32_t pv = 0;          // counter of the current fragment: lookups in the low half, slot visits in the high half
#ifdef KB_MATCH_STATS
  unsigned long long ms[MS_N] = {};
  int run[2] = {0, 0};      // current MAIN miss run of each chain, in positions
  long long t_mark = clock64();
  long long t_step = -1;    // >= 0: the lane's state transitions of this lookup iteration started at this clock
  auto end_run = [&](int c) { if (run[c] > 0) { KB_MS(MS_RUN_HIST + run_bin(run[c]), 1); run[c] = 0; } };
#endif
  // view of mate c of the lane's fragment, of length l (the caller reads len[c]: a run-time index into the array would
  // put it in local memory)
  auto view = [&](int c, int l) {
    ReadView rv;
    rv.bw = s_bw + (size_t)c * nw * nt;
    rv.gmask = ba.packed + (size_t)(ba.paired ? 2 * frag + c : frag) * ba.pstride + nw;
    rv.n_mask = nb;
    rv.stride = nt;
    rv.len = l;
    rv.k = k;
    rv.has_invalid = ((inv_flags >> c) & 1u) != 0;
    return rv;
  };

  KB_MS_ONLY(bool in_service = true;)
  for (;;) {
#ifdef KB_MATCH_STATS
    {
      const long long t_now = clock64();
      KB_MS(in_service ? MS_CYCLES_SERVICE : MS_CYCLES_LOOKUP, t_now - t_mark);
      if (t_step >= 0) KB_MS(MS_CYCLES_STEP, t_now - t_step);
      t_mark = t_now;
      t_step = -1;
    }
#endif
    // ------------------------------------------------------------------ service round
    const bool done = st[0] == S_FIN && st[1] == S_FIN;
    const unsigned fin = __ballot_sync(0xFFFFFFFFu, done);
    const unsigned idle = fin | __ballot_sync(0xFFFFFFFFu, st[0] == S_EMPTY);
    if (idle == 0xFFFFFFFFu && fin == 0 && !work_left) break;
    KB_MS_ONLY(in_service = false;)
    if (idle == 0xFFFFFFFFu || (work_left && __popc(idle) >= ba.refill_min)) {
      KB_MS(MS_SERVICE_ROUNDS, 1);
      KB_MS_ONLY(in_service = true;)
      if (done) {
        bool memo_hit = false;
        // ---- MinCollector::intersectKmers, net effect (MinCollector.cpp:160-218) ----
        const bool v0 = hv & 1u, s0 = hs & 1u, v1 = hv & 2u, s1 = hs & 2u;
        // first hit of each mate, before the tuple may grow over it
        uint32_t f_blk[2], f_ds[2], f_pos[2];
#pragma unroll
        for (int c = 0; c < 2; ++c) { f_blk[c] = cw(C_BLK, c); f_ds[c] = cw(C_DS, c); f_pos[c] = cw(C_POS, c); }
        bool mapped = v0 || v1;
        if ((v0 && !s0) || (v1 && !s1)) mapped = false;
        if (mapped && n_e == 0) mapped = false;
        int32_t handle = KB_H_UNMAPPED;
        if (mapped) {
          // single-end reads / pairs with one mate mapped, known mean fragment length: the transcripts
          // whose ends the fragment would overhang are filtered per fragment (ProcessReads.cpp:1095-1136)
          const bool want_fp = ba.fp_fl >= 0 && (!ba.paired || !v0 || !v1);
          // words that follow the set handles in the tuple: (block, orientation) of each mate's first hit for the
          // strand filter; block, orientation, read position and unitig offset of the mapped mate's first hit for
          // the position filter
          const bool stranded = ba.strand_mode != 0;
          uint32_t xs0 = 0xFFFFFFFFu, xs1 = 0xFFFFFFFFu;
          if (stranded) {
            xs0 = v0 ? (f_blk[0] * 2u + (f_ds[0] >> 31)) : 0xFFFFFFFFu;
            xs1 = v1 ? (f_blk[1] * 2u + (f_ds[1] >> 31)) : 0xFFFFFFFFu;
            // a fragment without the UMI tag is not strand-filtered (doStrandSpecificityIfPossible = false,
            // ProcessReads.cpp:1526): "no first hit" for both mates makes resolve_kernel skip the filter
            if (ba.notag && ba.notag[frag]) xs0 = xs1 = 0xFFFFFFFFu;
          }
          // the second mate's first hit; the first mate's when the second has none
          const uint32_t x_blk = v1 ? f_blk[1] : f_blk[0], x_ds = v1 ? f_ds[1] : f_ds[0], x_pos = v1 ? f_pos[1] : f_pos[0];
          const uint32_t xf0 = x_blk;
          const uint32_t xf1 = x_ds >> 31;
          const uint32_t xf2 = x_pos;
          const uint32_t xf3 = x_ds & 0x7FFFFFFFu;
          const int nx = (stranded ? 2 : 0) + (want_fp ? 4 : 0);
          // appends the extra words to a tuple stored with stride `st` starting at index `at`
          auto put_extras = [&](uint32_t* dst, int at, int st) {
            if (stranded) { dst[at * st] = xs0; dst[(at + 1) * st] = xs1; at += 2; }
            if (want_fp) { dst[at * st] = xf0; dst[(at + 1) * st] = xf1; dst[(at + 2) * st] = xf2; dst[(at + 3) * st] = xf3; }
          };
          if (overflow) {
            atomicOr(dd.error, KB_DEVERR_E_OVERFLOW);
          } else if (n_e > KB_MAX_E) {
            // ---- rare: more distinct EC sets than the shared-memory tuple holds (reads crossing many short EC
            //      blocks).  The tail of the list lives in this lane's spill area in global memory; the tuple is
            //      sorted through an accessor and handed to the resolve kernel through the wide queue, unmemoised.
            auto E = [&](int i) -> uint32_t { return i < KB_MAX_E ? elist[i * nt] : spill[i - KB_MAX_E]; };
            auto S = [&](int i, uint32_t x) { if (i < KB_MAX_E) elist[i * nt] = x; else spill[i - KB_MAX_E] = x; };
            for (int i = 1; i < n_e; ++i) {
              const uint32_t x = E(i);
              int j = i - 1;
              while (j >= 0 && E(j) > x) { S(j + 1, E(j)); --j; }
              S(j + 1, x);
            }
            const uint32_t q = atomicAdd(ba.qbig_count, 1u);
            if (q >= ba.qbig_cap) {
              atomicOr(dd.error, KB_DEVERR_E_OVERFLOW);
            } else {
              uint32_t* e = ba.qbig_entries + (size_t)q * KB_QBIG_STRIDE;
              e[0] = frag;
              e[1] = (uint32_t)(n_e + nx) | (want_fp ? 0x80000000u : 0u) | 0x40000000u;   // bit 30: never memoised
              for (int i = 0; i < n_e; ++i) e[2 + i] = E(i);
              put_extras(e + 2, n_e, 1);
              handle = KB_H_PENDING;
            }
          } else {
            for (int i = 1; i < n_e; ++i) {   // sort the distinct set handles (<= 16 entries)
              const uint32_t x = elist[i * nt];
              int j = i - 1;
              while (j >= 0 && elist[j * nt] > x) { elist[(j + 1) * nt] = elist[j * nt]; --j; }
              elist[(j + 1) * nt] = x;
            }
            if (ba.strand_mode == 0 && n_e == 1 && !want_fp) {
              handle = (int32_t)elist[0];            // a single EC set: its handle is stored in the slot
            } else {
              const int n = n_e + nx;
              int32_t r;
              if (ba.strand_mode == 0 && n_e == 2 && !want_fp) {
                r = memo2_lookup(dd, elist[0], elist[nt]);
              } else {
                put_extras(elist, n_e, nt);
                // position-filtered fragments depend on the read itself: never memoised
                r = want_fp ? KB_H_NOTREADY : memon_lookup(dd, elist, n, nt);
              }
              if (r == KB_H_NOTREADY) {
                handle = KB_H_PENDING;
                const uint32_t q = atomicAdd(ba.q_count, 1u);
                uint32_t* e = ba.q_entries + (size_t)q * KB_Q_STRIDE;
                e[0] = frag;
                e[1] = (uint32_t)n | (want_fp ? 0x80000000u : 0u);
                for (int i = 0; i < n; ++i) e[2 + i] = elist[i * nt];
              } else {
                handle = r;
                memo_hit = true;
              }
            }
          }
        }
        ba.handle_out[frag] = handle;
        if (ba.tl_out) {
          // KmerIndex::mapPair (KmerIndex.cpp:1622-1693): the first k-mer found by a linear scan is
          // the first hit of match(); same unitig, same EC set, opposite strands, same block end --
          // i.e. the same EC block of the index (blocks tile their unitig and carry one EC set).
          uint16_t tl = 0;
          if (ba.paired && v0 && v1) {
            int q[2];
            bool strand[2];
#pragma unroll
            for (int c = 0; c < 2; ++c) {
              const int d = (int)(f_ds[c] & 0x7FFFFFFFu);
              strand[c] = (f_ds[c] >> 31) != 0;
              q[c] = strand[c] ? d - (int)f_pos[c] : d + k + (int)f_pos[c];
            }
            if (f_blk[0] == f_blk[1] && strand[0] != strand[1]) {
              const int d = q[0] > q[1] ? q[0] - q[1] : q[1] - q[0];
              if (d > 0 && d < 1000) tl = (uint16_t)d;
            }
          }
          if (ba.notag && !ba.notag[frag]) tl = 0;     // tag runs: only fragments without the tag are sampled (getFragLenIfPaired, :1525)
          ba.tl_out[frag] = tl;
        }
        // per-handle accounting, aggregated over the lanes finalised in this round
        if (ba.first_hit) ba.first_hit[frag] = v0 ? f_blk[0] * 2u + (f_ds[0] >> 31) : 0xFFFFFFFFu;
        const unsigned grp = __match_any_sync(fin, handle);
        const uint32_t fmin = __reduce_min_sync(grp, frag);
        if (handle >= 0 && !ba.no_count && lane == (unsigned)(__ffs(grp) - 1)) {
          atomicAdd(&dd.count[handle], (uint32_t)__popc(grp));
          atomicMin(&dd.first[handle], (unsigned long long)(ba.frag_base + fmin));
        }
        // statistics of the round's fragments (a fragment executes at most a few hundred lookups)
        const uint32_t r_probes = __reduce_add_sync(fin, pv & 0xFFFFu), r_visits = __reduce_add_sync(fin, pv >> 16);
        const uint32_t r_memo = __popc(__ballot_sync(fin, memo_hit));
        pv = 0;
        if (lane == (unsigned)(__ffs(fin) - 1)) {
          atomicAdd(&s_tot[0], (unsigned long long)r_probes);
          atomicAdd(&s_tot[1], (unsigned long long)r_visits);
          if (r_memo) atomicAdd(&s_tot[2], (unsigned long long)r_memo);
        }
        st[0] = st[1] = S_EMPTY;
      }
      __syncwarp();
      // ---- refill: the idle lanes claim the next fragments with one atomic of lane 0 and copy their packed reads
      //      (pack_kernel output) into shared memory with 32-byte loads (ld256_nc)
      if (work_left) {
        const uint32_t n_idle = __popc(idle);
        uint32_t f0 = 0;
        if (lane == 0) f0 = atomicAdd(ba.take, n_idle);
        f0 = __shfl_sync(0xFFFFFFFFu, f0, 0);
        const uint32_t avail = f0 < ba.n_frag ? ba.n_frag - f0 : 0u;
        if (avail <= n_idle) work_left = false;
        const bool is_idle = (idle >> lane) & 1u;
        const uint32_t rank = __popc(idle & ((1u << lane) - 1));
        if (is_idle && rank < avail) {
          const uint32_t fidx = f0 + rank;
          unsigned inv = 0;
#pragma unroll
          for (int mt = 0; mt < 2; ++mt) {
            len[mt] = 0;
            if (mt >= n_mates) continue;
            const uint32_t ridx = ba.paired ? 2 * fidx + mt : fidx;
            // read_span's length, as pack_kernel found it; the D-list marks come after packing
            int l = (ba.skip && ba.skip[fidx]) ? 0 : (int)ba.rlen[ridx];
            if (l > nb * 32) l = nb * 32;   // cannot happen: the host sizes nb from the longest read
            len[mt] = l;
            const uint32_t* src = ba.packed + (size_t)ridx * ba.pstride;
            uint32_t* dbw = s_bw + (size_t)mt * nw * nt;
            uint32_t bad = 0;
            for (int c = 0; c < n_chunks; ++c) {
              uint32_t v[8];
              ld256_nc(src + c * 8, v);
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                // packed stream: nb 64-bit base words (little-endian halves: the high half holds the
                // first 16 bases), then nb 32-bit invalid masks, then padding
                const int g = c * 8 + i;
                if (g < nw) {
                  dbw[(g ^ 1) * nt] = v[i];
                } else if (g < nw + nb) {
                  const int first = (g - nw) * 32;           // mask of bases [first, first + 32)
                  const uint32_t in_read = l >= first + 32 ? 0xFFFFFFFFu : (l > first ? ((1u << (l - first)) - 1u) : 0u);
                  bad |= v[i] & in_read;
                }
              }
            }
            if (bad) inv |= 1u << mt;
          }
          frag = fidx;
          n_e = 0;
          overflow = false;
          inv_flags = inv;
          hv = hs = 0;
#pragma unroll
          for (int c = 0; c < 2; ++c) {
            prep[c] = P_BUILD;
            st[c] = S_FIN;     // no second mate, or a mate without a valid k-mer: the chain ends here
            if (c < n_mates) {
              p[c] = view(c, len[c]).next_valid(0);
              if (p[c] >= 0) st[c] = S_MAIN;
            }
          }
        }
      }
      continue;
    }
    // ------------------------------------------------------------------ one lookup per live chain
    const bool live[2] = {st[0] <= S_BACKOFF, st[1] <= S_BACKOFF};
    KB_MS(MS_WARP_ITERS, 1);
    KB_MS_ONLY(int n_pass = 0;)
    if (live[0] || live[1]) {
      KB_MS(MS_LANE_ITERS, 1);
      // keys of both chains and their presence-filter words (L2 resident) before either is used
      uint32_t fword[2] = {0xFFFFFFFFu, 0xFFFFFFFFu}, fbit[2] = {0, 0};
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (live[c] && prep[c] != P_NONE) {
          const bool filtered = st[c] == S_MAIN || st[c] == S_BACKOFF;
          if (prep[c] == P_ROLL) {
            // the k-mer at p from the one at p - 1: its last base enters at the low end of the forward k-mer and,
            // complemented, at the high end of the reverse complement
            const int q = p[c] + k - 1;
            const uint64_t b = (s_bw[((size_t)c * nw + (q >> 4)) * nt] >> (30 - 2 * (q & 15))) & 3u;
            fwd[c] = ((fwd[c] << 2) | b) & kmask;
            rc[c] = (rc[c] >> 2) | ((b ^ 3u) << (2 * k - 2));
          } else {
            const int pq = filtered ? p[c] : (int)cw(st[c] == S_JUMP ? C_P2 : C_P3, c);
            fwd[c] = view(c, len[c]).kmer(pq);
            rc[c] = kb_revcomp(fwd[c], k);
          }
          const uint64_t hsh = kb_mix64(fwd[c] < rc[c] ? fwd[c] : rc[c]);
          slot[c] = (uint32_t)hsh & slot_mask;
          prep[c] = P_NONE;
          ++pv;
          // a clear bit means the k-mer is not in the index -- no HBM sector is touched.  The jump target and the
          // middle k-mer lie in the EC block of the hit before them and are nearly always present: their slot is
          // loaded without the filter word, which would only add an L2 round trip and an L2 request
          if (ix.filter && filtered) {
            const uint32_t fidx = (uint32_t)(hsh >> 32) & ix.filter_mask;
            fword[c] = __ldg(ix.filter + (fidx >> 5));
            fbit[c] = fidx & 31;
          }
        }
      }
#ifdef KB_MATCH_STATS
      const long long t_key = clock64();
#endif
      // both slot loads before either is used
      uint32_t v[2][8];
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        if (live[c] && ((fword[c] >> fbit[c]) & 1u)) {
          ld256_nc(ix.slots + slot[c], v[c]);
          pv += 0x10000u;
        } else {
          v[c][0] = v[c][1] = 0xFFFFFFFFu;     // reads as an empty slot: a miss
        }
      }
#ifdef KB_MATCH_STATS
      {
        // the clock is read once both slots (and so both filter words) have arrived: the read is under a branch on the
        // loaded words, and a volatile read cannot be hoisted above it (the untaken side, a key pair that spells
        // 0x0BADF00D, only loses that iteration's wait)
        long long t_wait = t_key;
        if (((v[0][0] ^ v[0][1]) ^ 3u * (v[1][0] ^ v[1][1])) != 0x0BADF00Du) t_wait = clock64();
        KB_MS(MS_CYCLES_KEY, t_key - t_mark);
        KB_MS(MS_CYCLES_WAIT, t_wait - t_key);
        t_step = t_wait;
      }
#endif
      // the common outcomes first, for both chains and without branches: a collision moves to the next slot (linear
      // probing), and a MAIN miss on a mate without bases other than A/C/G/T moves to the next position, whose k-mer is
      // then rolled from this one.  Only a hit, a JUMP, MIDDLE or BACKOFF lookup, or a miss on a mate with such a base
      // is left to the general transition below.
      bool f[2];
      unsigned todo = 0;     // bit c: chain c takes the general transition
#pragma unroll
      for (int c = 0; c < 2; ++c) {
        const uint64_t key = (uint64_t)v[c][0] | ((uint64_t)v[c][1] << 32);
        f[c] = key == (fwd[c] < rc[c] ? fwd[c] : rc[c]);
        const bool coll = live[c] && !f[c] && key != KB_EMPTY_KEY;
        const bool step = live[c] && !f[c] && !coll && st[c] == S_MAIN && !((inv_flags >> c) & 1u);
#ifdef KB_MATCH_STATS
        if (live[c]) {
          KB_MS(MS_CHAIN_ITERS, 1);
          if (coll || step) KB_MS(MS_STRAIGHT, 1);
          if (coll) {
            KB_MS(MS_COLLISION, 1);
          } else if (st[c] == S_MAIN) {
            if (f[c]) { KB_MS(MS_MAIN_HIT, 1); end_run(c); }
            else { KB_MS(((fword[c] >> fbit[c]) & 1u) ? MS_MAIN_MISS_SLOT : MS_MAIN_MISS_FILTER, 1); ++run[c]; }
          } else {
            KB_MS(st[c] == S_JUMP ? MS_JUMP : (st[c] == S_MIDDLE ? MS_MIDDLE : MS_BACKOFF), 1);
          }
        }
#endif
        if (coll) slot[c] = (slot[c] + 1) & slot_mask;
        if (step) {
          ++p[c];
          prep[c] = P_ROLL;
          if (p[c] > len[c] - k) st[c] = S_FIN;
          KB_MS_ONLY(if (st[c] == S_FIN) end_run(c);)
        }
        if (live[c] && !coll && !step) todo |= 1u << c;
      }
      // the general transition (KmerIndex::match's control flow), one copy for both chains: each pass takes the lane's
      // lowest chain that still needs it, its fields picked by selects.  A warp runs as many passes as its busiest lane
      // needs, and chain 1's handle dedup sees what chain 0 pushed in the same iteration.
      while (todo) {
        KB_MS_ONLY(++n_pass;)
        const bool c1 = !(todo & 1u);
        const int c = c1 ? 1 : 0;
        todo &= todo - 1;
        const int s = c1 ? st[1] : st[0];
        const int pc = c1 ? p[1] : p[0];
        const int l = c1 ? len[1] : len[0];
        const bool fc = c1 ? f[1] : f[0];
        const bool is_canon = c1 ? fwd[1] < rc[1] : fwd[0] < rc[0];
        // hit fields: h[0] unitig, h[1] blk, h[2] ec (set handle), h[3] dist|flag, h[4] lb, h[5] ub
        uint32_t h[6];
#pragma unroll
        for (int i = 0; i < 6; ++i) h[i] = c1 ? v[1][i + 2] : v[0][i + 2];
        const uint32_t r_unitig = h[0], r_ec = h[2];
        const bool r_strand = (is_canon == ((h[3] >> 31) != 0));
        const ReadView rv = view(c, l);
        int ns = s, np_ = pc, npr = P_BUILD;     // the chain's next state, position and key preparation
        bool push = false, end_chain = false, to_backoff = false;
        int nv_from = -1;      // >= 0: continue with p = next_valid(nv_from) in MAIN (or BACKOFF)
        if (s == S_MAIN) {
          if (!fc) {
            nv_from = pc + 1;
          } else {
            push = true;
            const int r_dist = (int)(h[3] & 0x7FFFFFFFu);
            const int off = r_dist - (int)h[4], blen = (int)(h[5] - h[4]);
            const int dist = r_strand ? (blen - 1 - off) : off;               // 1780-1788
            if (dist >= 2) {
              const int np = (pc + dist >= l - k) ? (l - k) : (pc + dist);      // 1793-1798
              const int p2 = rv.next_valid(np);                               // kit2 += nextPos-pos (adv 0: p itself)
              if (p2 < 0) {
                end_chain = true;                                           // 1882-1886
              } else {
                cw(C_NP, c) = (uint32_t)np;
                cw(C_P2, c) = (uint32_t)p2;
                cw(C_DIST, c) = (uint32_t)dist;
                cw(C_HU, c) = r_unitig; cw(C_HE, c) = r_ec;
                ns = S_JUMP;
              }
            } else {
              nv_from = pc + 1;
            }
          }
        } else if (s == S_JUMP) {
          const bool found2 = !fc || (cw(C_HU, c) == r_unitig && cw(C_HE, c) == r_ec);   // 1807-1815
          const int dist = (int)cw(C_DIST, c);
          const int found2pos = !fc ? pc : pc + dist;
          if (found2) {
            if (found2pos >= l - k) end_chain = true;                       // "fake position", break (1819-1822)
            else nv_from = (int)cw(C_P2, c) + 1;                            // kit = kit2; ++kit
          } else {
            cw(C_H2U, c) = r_unitig; cw(C_H2E, c) = r_ec;
            if (dist > 4) {
              const int middlePos = (pc + (int)cw(C_NP, c)) / 2;
              const int p3 = rv.next_valid(middlePos);                      // kit3 += middlePos-pos
              if (p3 >= 0) { cw(C_P3, c) = (uint32_t)p3; ns = S_MIDDLE; }
              else to_backoff = true;
            } else {
              to_backoff = true;
            }
          }
        } else if (s == S_MIDDLE) {
          const bool foundMiddle = fc && ((cw(C_HU, c) == r_unitig && cw(C_HE, c) == r_ec) ||
                                          (cw(C_H2U, c) == r_unitig && cw(C_H2E, c) == r_ec));
          if (foundMiddle) {
            push = true;
            if ((int)cw(C_NP, c) >= l - k) end_chain = true;               // 1867
            else nv_from = (int)cw(C_P2, c) + 1;                            // kit = kit2; ++kit
          } else {
            to_backoff = true;
          }
        } else {   // S_BACKOFF: the single probe of the back-off loop
          push = fc;
          nv_from = pc + 1;
        }
        if (push) {
          if (!((hv >> c) & 1u)) {
            hv |= 1u << c;   // only a MAIN hit can be the first hit of a read
            cw(C_BLK, c) = h[1];
            cw(C_DS, c) = (h[3] & 0x7FFFFFFFu) | (r_strand ? 0x80000000u : 0u);
            cw(C_POS, c) = (uint32_t)pc;
          }
          if (r_ec != ba.empty_ec) {               // "Don't intersect empty EC", MinCollector.cpp:468-469
            hs |= 1u << c;
            // the tuple is shared by both chains: a handle the other chain pushed (also in this iteration) is a duplicate
            bool dup = false;
            const int n_sh = n_e < KB_MAX_E ? n_e : KB_MAX_E;
            for (int i = 0; i < n_sh; ++i) dup |= (elist[i * nt] == r_ec);
            for (int i = KB_MAX_E; i < n_e; ++i) dup |= (spill[i - KB_MAX_E] == r_ec);     // rare: spilled tail
            if (!dup) {
              if (n_e < KB_MAX_E) { elist[n_e * nt] = r_ec; ++n_e; }
              else if (n_e < KB_MAX_E + KB_SPILL) { spill[n_e - KB_MAX_E] = r_ec; ++n_e; }
              else overflow = true;
            }
          }
        }
        if (to_backoff) nv_from = pc + 1;          // ++kit; backOff = true
        if (nv_from >= 0) {
          // where the k-mer the chain holds starts: the next one is rolled from it when it starts one base later
          const int key_pos = (s == S_MAIN || s == S_BACKOFF) ? pc : (int)cw(s == S_JUMP ? C_P2 : C_P3, c);
          np_ = rv.next_valid(nv_from);
          if (np_ < 0) end_chain = true;
          else { ns = to_backoff ? S_BACKOFF : S_MAIN; npr = np_ == key_pos + 1 ? P_ROLL : P_BUILD; }
        }
        if (end_chain) ns = S_FIN;
        KB_MS_ONLY(if (ns == S_FIN) end_run(c);)
        if (c1) { st[1] = ns; p[1] = np_; prep[1] = npr; }
        else { st[0] = ns; p[0] = np_; prep[0] = npr; }
      }
    }
#ifdef KB_MATCH_STATS
    KB_MS(MS_GEN_PASSES, __reduce_max_sync(0xFFFFFFFFu, n_pass));   // the warp's passes of the general transition
#endif
  }
  // statistics: lookups, slot visits, memo hits (every warp leaves the loop with all its fragments finalised)
  __syncthreads();
  if (tid < 3 && s_tot[tid]) atomicAdd(&dd.stats[tid == 0 ? 0 : (tid == 1 ? 3 : 2)], s_tot[tid]);
#ifdef KB_MATCH_STATS
  for (int i = 0; i < MS_N; ++i) {
    const bool per_warp = i == MS_WARP_ITERS || i == MS_SERVICE_ROUNDS || i == MS_CYCLES_LOOKUP || i == MS_CYCLES_SERVICE ||
                          i == MS_GEN_PASSES;
    unsigned long long x = ms[i];
    if (!per_warp)
      for (int o = 16; o > 0; o >>= 1) x += __shfl_xor_sync(0xFFFFFFFFu, x, o);
    if (lane == 0 && x) atomicAdd(&kb_match_stats[i], x);
  }
#endif
}

// One group of G lanes per queued fragment (ra.n_warps counts groups).  The kernel is a chain of dependent memory
// accesses per fragment (queue entry -> memo -> set descriptors -> set elements -> binary searches -> dictionary ->
// memo), so what sets its speed is the number of fragments in flight: the sets are short (2.5 ids on average), 8
// lanes hold them, and a warp then carries four fragments instead of one.
template <int G>
__global__ void __launch_bounds__(128, 8) resolve_kernel(DevIndex ix, DevDict dd, BatchArgs ba, ResolveArgs ra) {
  const unsigned lane = threadIdx.x & (G - 1);                          // lane inside its group
  const unsigned gmask = group_mask<G>(threadIdx.x & 31);
  const unsigned gshift = (threadIdx.x & 31) & ~(unsigned)(G - 1);      // the group's first lane of the warp
  const uint32_t warp = (blockIdx.x * blockDim.x + threadIdx.x) / G;    // group index
  if (warp >= ra.n_warps) return;
  uint32_t* scratch = ra.scratch + (size_t)warp * ra.scratch_stride;
  const uint32_t* pool = dd.pool;

  // pass 0: the regular queue; pass 1: the wide queue (fragments with more than KB_MAX_E distinct EC sets)
  for (int pass = 0; pass < 2; ++pass) {
  const uint32_t nq = pass == 0 ? *ba.q_count : min(*ba.qbig_count, ba.qbig_cap);
  const uint32_t* entries = pass == 0 ? ba.q_entries : ba.qbig_entries;
  const size_t stride = pass == 0 ? (size_t)KB_Q_STRIDE : (size_t)KB_QBIG_STRIDE;
  if (warp == 0 && lane == 0 && nq) atomicAdd(&dd.stats[1], (unsigned long long)nq);   // fragments finished here
  for (uint32_t q = warp; q < nq; q += ra.n_warps) {
    const uint32_t* e = entries + (size_t)q * stride;
    const uint32_t f = e[0];
    const bool has_fp = (e[1] >> 31) != 0;
    const bool no_memo = has_fp || ((e[1] >> 30) & 1u) != 0;
    const int n = (int)(e[1] & 0xFFFFu);
    const uint32_t* w = e + 2;
    const bool stranded = ba.strand_mode != 0;
    const int n_e = n - (stranded ? 2 : 0) - (has_fp ? 4 : 0);
    const bool use_m2 = (!stranded && !no_memo && n_e == 2);

    // 1. has somebody else resolved the same tuple in the meantime?
    int32_t handle = KB_H_NOTREADY;
    if (lane == 0 && !no_memo) handle = use_m2 ? memo2_lookup(dd, w[0], w[1]) : memon_lookup(dd, w, n, 1);
    handle = __shfl_sync(gmask, handle, 0, G);

    if (handle == KB_H_NOTREADY) {
      // 2. intersection of the n_e sets: lanes own elements of the smallest one
      // the tuple holds set handles: dslots[h] = offset | len << 32 | tag << 56
      int sm = 0;
      uint32_t sm_len = (uint32_t)((dd.dslots[w[0]] >> 32) & 0xFFFFFFu);
      for (int j = 1; j < n_e; ++j) {
        const uint32_t len = (uint32_t)((dd.dslots[w[j]] >> 32) & 0xFFFFFFu);
        if (len < sm_len) { sm_len = len; sm = j; }
      }
      const uint32_t* A = pool + (uint32_t)dd.dslots[w[sm]];
      uint32_t nres = 0;
      for (uint32_t base = 0; base < sm_len; base += G) {
        const uint32_t i = base + lane;
        bool alive = i < sm_len;
        const uint32_t a = alive ? __ldcg(A + i) : 0;
        for (int j = 0; j < n_e; ++j) {
          if (j == sm) continue;
          const unsigned long long bw_ = dd.dslots[w[j]];
          const uint32_t* B = pool + (uint32_t)bw_;
          const uint32_t blen = (uint32_t)((bw_ >> 32) & 0xFFFFFFu);
          if (alive) alive = bsearch_contains(B, blen, a, nullptr);
        }
        const unsigned bal = (__ballot_sync(gmask, alive) >> gshift);
        if (alive) scratch[nres + __popc(bal & ((1u << lane) - 1))] = a;
        nres += __popc(bal);
      }
      __syncwarp(gmask);
      // 2b. fragment-position filter (ProcessReads.cpp:1095-1136 with KmerIndex::findPosition,
      //     KmerIndex.cpp:2188-2292): keep the transcripts the fragment fits into
      if (has_fp && nres > 0) {
        const uint32_t* fw = w + n - 4;
        const uint32_t blk = fw[0];
        const bool csense = fw[1] != 0;
        const long long pp = (long long)fw[2], udist = (long long)fw[3];
        const long long usize = (long long)ix.blk_usize[blk], kk = (long long)ix.k, fl = (long long)ba.fp_fl;
        const unsigned long long bword = dd.dslots[ix.blk_ec[blk]];
        const uint32_t* B = pool + (uint32_t)bword;
        const uint32_t blen = (uint32_t)((bword >> 32) & 0xFFFFFFu);
        const uint4* info = ix.fp_info + ix.blk_strand_off[blk];
        uint32_t n_v = 0;
        for (uint32_t base = 0; base < nres; base += G) {
          const uint32_t i = base + lane;
          bool keep = false;
          const uint32_t tr = i < nres ? scratch[i] : 0;
          if (i < nres) {
            uint32_t rank = 0;
            if (bsearch_contains(B, blen, tr, &rank)) {
              const uint4 c = info[rank];
              const long long trpos = (long long)(c.x & 0x7FFFFFFFu);
              const bool trsense = (c.x >> 31) == 0;
              long long x;
              bool s;
              if (trsense) {
                if (csense) { x = trpos - pp + udist + 1 - (long long)c.y; s = true; }           // case I
                else { x = trpos + pp + kk + udist - (long long)c.z; s = false; }                // case III
              } else {
                if (csense) { x = trpos - udist + usize - (long long)c.w + pp; s = false; }      // case IV
                else { x = trpos + usize - udist - (long long)c.w - kk + 1 - pp; s = true; }     // case II
              }
              const int xi = (int)x;
              keep = (s && xi + (int)fl <= (int)ix.target_len[tr]) || (!s && xi - (int)fl >= 0);
            }
          }
          const unsigned bv = (__ballot_sync(gmask, keep) >> gshift);
          if (keep) scratch[ra.scratch_stride / 2 + n_v + __popc(bv & ((1u << lane) - 1))] = tr;
          n_v += __popc(bv);
        }
        __syncwarp(gmask);
        if (n_v < nres) {
          for (uint32_t i = lane; i < n_v; i += G) scratch[i] = scratch[ra.scratch_stride / 2 + i];
          nres = n_v;
        }
        __syncwarp(gmask);
      }
      // 3. doStrandSpecificity (ProcessReads.cpp:61-124), first mate then second mate
      if (stranded) {
        for (int mate = 0; mate < 2 && nres > 0; ++mate) {
          const uint32_t sw = w[n_e + mate];
          if (sw == 0xFFFFFFFFu) continue;            // v empty for this mate
          const uint32_t blk = sw >> 1;
          const bool um_strand = (sw & 1) != 0;
          const bool want = (mate == 0) ? (ba.strand_mode == 1) : (ba.strand_mode == 2);
          // EC set of the first-hit block: recover its id from the tuple?  Not possible in general
          // (empty sets are not in the tuple), so the block's set is looked up via blk_ec.
          const unsigned long long bword = dd.dslots[ix.blk_ec[blk]];   // blk_ec holds set handles
          const uint32_t* B = pool + (uint32_t)bword;
          const uint32_t blen = (uint32_t)((bword >> 32) & 0xFFFFFFu);
          const uint8_t* sb = ix.strand + ix.blk_strand_off[blk];
          // u &= ec ; vtmp = strand-compatible subset
          uint32_t n_u = 0, n_v = 0;
          // two passes over scratch, compacting in place: first u &= ec (keeping a flag per kept
          // element in the top of the scratch area is avoided by recomputing the predicate)
          for (uint32_t base = 0; base < nres; base += G) {
            const uint32_t i = base + lane;
            bool in_u = i < nres;
            const uint32_t a = in_u ? scratch[i] : 0;
            uint32_t rank = 0;
            if (in_u) in_u = bsearch_contains(B, blen, a, &rank);
            bool in_v = false;
            if (in_u) {
              const uint8_t sense = sb[rank];
              in_v = ((um_strand == (sense != 0)) == want) || sense == 2;
            }
            const unsigned bu = (__ballot_sync(gmask, in_u) >> gshift);
            const unsigned bv = (__ballot_sync(gmask, in_v) >> gshift);
            __syncwarp(gmask);
            // u goes to the front of scratch (in place: n_u <= base), v to the second half
            if (in_u) scratch[n_u + __popc(bu & ((1u << lane) - 1))] = a;
            if (in_v) scratch[ra.scratch_stride / 2 + n_v + __popc(bv & ((1u << lane) - 1))] = a;
            n_u += __popc(bu);
            n_v += __popc(bv);
            __syncwarp(gmask);
          }
          if (n_v < n_u) {
            for (uint32_t i = lane; i < n_v; i += G) scratch[i] = scratch[ra.scratch_stride / 2 + i];
            nres = n_v;
          } else {
            nres = n_u;
          }
          __syncwarp(gmask);
        }
      }
      // 4. set -> handle through the content-addressed dictionary
      handle = nres == 0 ? KB_H_UNMAPPED : dict_insert_warp<G>(dd, scratch, nres, lane, gmask);
      // 5. publish tuple -> handle (not for position-filtered fragments: the result depends on the read)
      if (lane == 0 && !no_memo) {
        if (use_m2) {
          const unsigned long long key = ((unsigned long long)w[0] << 32) | w[1];
          uint64_t s = kb_mix64(key) & dd.m2_mask;
          uint64_t visited = 0;
          for (;;) {
            const unsigned long long old = atomicCAS(&dd.m2[s].key, ~0ULL, key);
            if (old == ~0ULL || old == key) { atomicExch(&dd.m2[s].val, handle); break; }
            s = (s + 1) & dd.m2_mask;
            if (++visited > dd.m2_mask) { atomicOr(dd.error, KB_DEVERR_MEMO_FULL); break; }
          }
        } else {
          const uint64_t th = tuple_hash(w, n, 1);
          const uint32_t tag = (uint32_t)(th >> 32);
          const unsigned long long toff = atomicAdd(dd.tpool_top, (unsigned long long)(n + 1));
          if (toff + n + 1 > dd.tpool_cap) {
            atomicOr(dd.error, KB_DEVERR_TPOOL_FULL);
          } else {
            dd.tpool[toff] = (uint32_t)n;
            for (int i = 0; i < n; ++i) dd.tpool[toff + 1 + i] = w[i];
            __threadfence();
            const unsigned long long word = ((unsigned long long)tag << 32) | toff;
            uint64_t s = th & dd.mn_mask;
            uint64_t visited = 0;
            for (;;) {
              unsigned long long old = atomicCAS(&dd.mn_key[s], ~0ULL, word);
              bool mine = (old == ~0ULL);
              if (!mine && (uint32_t)(old >> 32) == tag) {
                const uint32_t* t = dd.tpool + (uint32_t)old;
                bool eq = __ldcg(t) == (uint32_t)n;
                for (int i = 0; eq && i < n; ++i) eq = __ldcg(t + 1 + i) == w[i];
                mine = eq;
              }
              if (mine) { atomicExch(&dd.mn_val[s], handle); break; }
              s = (s + 1) & dd.mn_mask;
              if (++visited > dd.mn_mask) { atomicOr(dd.error, KB_DEVERR_MEMO_FULL); break; }
            }
          }
        }
      }
    }
    // 6. account for this fragment
    if (lane == 0) {
      ba.handle_out[f] = handle;
      if (handle >= 0 && !ba.no_count) {
        atomicAdd(&dd.count[handle], 1u);
        atomicMin(&dd.first[handle], (unsigned long long)(ba.frag_base + f));
      }
    }
    __syncwarp(gmask);
  }
  }
}

// A fragment contributes to the fragment-length distribution only if its EC has a single
// transcript (ProcessReads.cpp:1174).
__global__ void fld_finalize_kernel(DevDict dd, BatchArgs ba) {
  const uint32_t f = blockIdx.x * blockDim.x + threadIdx.x;
  if (f >= ba.n_frag) return;
  const int32_t h = ba.handle_out[f];
  if (h < 0) { ba.tl_out[f] = 0; return; }
  const unsigned long long word = dd.dslots[h];
  if (((word >> 32) & 0xFFFFFFu) != 1) ba.tl_out[f] = 0;
}

__global__ void collect_used_kernel(DevDict dd, uint32_t* used, uint32_t* n_used) {
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t h = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; h <= dd.dmask; h += stride) {
    if (dd.count[h] > 0) used[atomicAdd(n_used, 1u)] = (uint32_t)h;
  }
}

void launch_pseudoalign(const DevIndex& ix, const DevDict& dd, const BatchArgs& ba, const ResolveArgs& ra,
                        int tpb, cudaStream_t st, cudaEvent_t* ev, cudaEvent_t packed) {
  if (ba.n_frag == 0) return;
  cudaMemsetAsync(ba.q_count, 0, sizeof(uint32_t) * KB_BATCH_COUNTER_WORDS, st);   // q_count, qbig_count, take
  // persistent grid: as many blocks as fit on the device at once
  const size_t smem = (size_t)tpb * 4 * match_lane_words(ba.nb);
  const int sms = device_sm_count();
  cudaFuncSetAttribute(match_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  int per_sm = 0;
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, match_kernel, tpb, smem);
  if (per_sm < 1) per_sm = 1;
  unsigned blocks = (unsigned)(sms * per_sm);
  const unsigned need = (ba.n_frag + tpb - 1) / tpb;   // never more lanes than fragments
  if (blocks > need) blocks = need;
  if (ev) cudaEventRecord(ev[0], st);
  {
    const uint32_t n_reads = ba.paired ? 2 * ba.n_frag : ba.n_frag;
    const uint64_t total = (uint64_t)n_reads * ba.nb;     // < 2^32: engine.cu bounds a batch by 2^31 bases
    pack_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ba, n_reads, const_cast<uint32_t*>(ba.packed));
    if (ix.dfk && ba.skip_w) dlist_scan_kernel<<<(unsigned)((total + 255) / 256), 256, 0, st>>>(ix, ba, n_reads);
  }
  if (packed) cudaEventRecord(packed, st);    // the batch's input buffers are not read after this point
  if (ev) cudaEventRecord(ev[1], st);
#ifdef KB_MATCH_STATS
  void* ms_dev = nullptr;
  cudaGetSymbolAddress(&ms_dev, kb_match_stats);
  cudaMemsetAsync(ms_dev, 0, sizeof(unsigned long long) * MS_N, st);
#endif
  match_kernel<<<blocks, tpb, smem, st>>>(ix, dd, ba);
#ifdef KB_MATCH_STATS
  {
    unsigned long long h[MS_N];
    cudaMemcpyAsync(h, ms_dev, sizeof(h), cudaMemcpyDeviceToHost, st);
    cudaStreamSynchronize(st);
    fprintf(stderr, "kb_match_stats {\"n_frag\": %u", ba.n_frag);
    for (int i = 0; i < MS_N; ++i) fprintf(stderr, ", \"%s\": %llu", kMatchStatNames[i], h[i]);
    fprintf(stderr, "}\n");
  }
#endif
  if (ev) cudaEventRecord(ev[2], st);
  switch (ra.group) {      // lanes per fragment (engine.cu: KB_RESOLVE_G, default 32)
    case 4: resolve_kernel<4><<<(ra.n_warps * 4 + 127) / 128, 128, 0, st>>>(ix, dd, ba, ra); break;
    case 8: resolve_kernel<8><<<(ra.n_warps * 8 + 127) / 128, 128, 0, st>>>(ix, dd, ba, ra); break;
    case 16: resolve_kernel<16><<<(ra.n_warps * 16 + 127) / 128, 128, 0, st>>>(ix, dd, ba, ra); break;
    default: resolve_kernel<32><<<(ra.n_warps * 32 + 127) / 128, 128, 0, st>>>(ix, dd, ba, ra); break;
  }
  if (ev) cudaEventRecord(ev[3], st);
}

// Multi-GPU merge: equivalence classes exported by another rank (CSR of transcript ids, counts, first
// fragment index) are folded into this rank's dictionary -- the content-keyed reduction that replaces
// a dense all-reduce, since EC ids are discovered independently on every rank.  One warp per set.
__global__ void __launch_bounds__(128) import_sets_kernel(DevDict dd, uint32_t n_sets, const uint32_t* off, const uint32_t* tids,
                                                         const uint32_t* counts, const unsigned long long* first,
                                                         unsigned long long first_offset) {
  const unsigned lane = threadIdx.x & 31;
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nw = (gridDim.x * blockDim.x) >> 5;
  for (uint32_t s = w; s < n_sets; s += nw) {
    const uint32_t o0 = off[s], n = off[s + 1] - o0;
    if (n == 0) continue;
    const int32_t h = dict_insert_warp(dd, tids + o0, n, lane);
    if (lane == 0 && h >= 0) {
      atomicAdd(&dd.count[h], counts[s]);
      atomicMin(&dd.first[h], first[s] + first_offset);
    }
    __syncwarp();
  }
}

struct ImportSegs {
  int n;
  uint32_t prefix[KB_IMPORT_SEGS + 1];
  ImportSeg seg[KB_IMPORT_SEGS];
};
__global__ void __launch_bounds__(128) import_segments_kernel(DevDict dd, ImportSegs a) {
  const unsigned lane = threadIdx.x & 31;
  const uint32_t w = (blockIdx.x * blockDim.x + threadIdx.x) >> 5;
  const uint32_t nw = (gridDim.x * blockDim.x) >> 5;
  const uint32_t total = a.prefix[a.n];
  for (uint32_t g = w; g < total; g += nw) {
    int k = 0;
    while (g >= a.prefix[k + 1]) ++k;
    const ImportSeg& sg = a.seg[k];
    const uint32_t s = g - a.prefix[k];
    const uint32_t o0 = sg.off[s], n = sg.off[s + 1] - o0;
    if (n == 0) continue;
    const int32_t h = dict_insert_warp(dd, sg.tids + o0, n, lane);
    if (lane == 0 && h >= 0) {
      atomicAdd(&dd.count[h], sg.counts[s]);
      atomicMin(&dd.first[h], sg.first[s]);
    }
    __syncwarp();
  }
}

int device_sm_count() {
  static int sms[64] = {0};
  int dev = 0;
  cudaGetDevice(&dev);
  if (dev < 0 || dev >= 64) dev = 0;
  if (sms[dev] == 0) {
    int v = 0;
    cudaDeviceGetAttribute(&v, cudaDevAttrMultiProcessorCount, dev);
    sms[dev] = v > 0 ? v : 1;
  }
  return sms[dev];
}

void launch_import_segments(const DevDict& dd, const ImportSeg* segs, int n_segs, cudaStream_t st) {
  if (n_segs <= 0) return;
  ImportSegs a;
  a.n = n_segs;
  a.prefix[0] = 0;
  for (int i = 0; i < n_segs; ++i) { a.seg[i] = segs[i]; a.prefix[i + 1] = a.prefix[i] + segs[i].n_sets; }
  if (a.prefix[n_segs] == 0) return;
  const unsigned warps_needed = a.prefix[n_segs];
  unsigned blocks = (unsigned)device_sm_count() * 16;
  if (blocks > (warps_needed + 3) / 4) blocks = (warps_needed + 3) / 4;
  import_segments_kernel<<<blocks, 128, 0, st>>>(dd, a);
}

void launch_import_sets(const DevDict& dd, uint32_t n_sets, const uint32_t* off, const uint32_t* tids, const uint32_t* counts,
                        const unsigned long long* first, unsigned long long first_offset, cudaStream_t st) {
  if (n_sets == 0) return;
  import_sets_kernel<<<device_sm_count() * 8, 128, 0, st>>>(dd, n_sets, off, tids, counts, first, first_offset);
}

void launch_fld_finalize(const DevDict& dd, const BatchArgs& ba, cudaStream_t st) {
  if (ba.n_frag == 0 || !ba.tl_out) return;
  fld_finalize_kernel<<<(ba.n_frag + 255) / 256, 256, 0, st>>>(dd, ba);
}

void launch_collect_used(const DevDict& dd, uint32_t* used, uint32_t* n_used, cudaStream_t st) {
  cudaMemsetAsync(n_used, 0, sizeof(uint32_t), st);
  collect_used_kernel<<<device_sm_count() * 8, 256, 0, st>>>(dd, used, n_used);
}

}  // namespace kb
