// Device-side data layout shared by the kallisto_b200 CUDA kernels (sm_90a).
//
// Everything the per-read pseudoalignment loop of the reference touches through
// pointer-rich host structures (CompactedDBG<Node>::find -> UnitigMap, Node::ec BlockArray,
// SparseVector/Roaring; see DESIGN.md) is flattened here into HBM-resident arrays:
//
//   * KmerSlot[cap]   open-addressing table, one 32-byte slot (= one DRAM sector) per canonical
//                     k-mer of the compacted dBG; a probe returns unitig identity, EC-block bounds,
//                     EC-set id and orientation with no dependent load.
//   * set pool        sorted u32 transcript-id lists: the index's de-duplicated EC sets first,
//                     then sets discovered at run time (intersections).
//   * set dictionary  content-addressed (set -> handle), so that an intersection result that
//                     equals an existing set gets the same handle (ecmapinv semantics,
//                     src/KmerIndex.h:131, src/MinCollector.cpp:251-269).
//   * memo tables     (sorted tuple of EC-set ids hit by a fragment) -> handle.
#pragma once
#include <cstdint>
#include <cuda_runtime.h>

namespace kb {

static constexpr uint64_t KB_EMPTY_KEY = ~0ULL;
static constexpr int KB_MAX_E = 16;          // distinct EC sets tracked per fragment on the fast path
static constexpr int32_t KB_H_UNMAPPED = -1;
static constexpr int32_t KB_H_PENDING = -2;  // fragment queued for the resolve kernel
static constexpr int32_t KB_H_NOTREADY = -3; // memo slot claimed, value not yet published

struct __align__(32) KmerSlot {
  uint64_t key;        // canonical k-mer, right-aligned 2k bits; KB_EMPTY_KEY = free
  uint32_t unitig;     // global unitig id (long, then short, then abundant)
  uint32_t blk;        // global EC-block id
  uint32_t ec;         // EC set of that block, as its dictionary handle (equal handles <=> equal transcript sets)
  uint32_t dist_flag;  // bits 0..30: k-mer offset in unitig-forward coordinates; bit 31: forward k-mer is the canonical one
  uint32_t lb, ub;     // EC block [lb, ub) in k-mer coordinates of the unitig
};
static_assert(sizeof(KmerSlot) == 32, "slot must be one 32-byte sector");

struct DevIndex {
  const KmerSlot* slots;
  uint64_t mask;             // capacity - 1 (capacity is a power of two)
  // presence filter of the k-mer table, kept in L2 (persisting window): bit ((mix64(kmer) >> 32) & filter_mask) is set
  // for every k-mer of the table.  69 % of KmerIndex::match's lookups are misses; a clear bit answers them without
  // touching HBM.  nullptr = no filter.
  const uint32_t* filter;
  uint32_t filter_mask;      // bits - 1 (a power of two)
  // D-list (distinguishing flanking k-mers, src/KmerIndex.cpp:1385-1403): open-addressing set of canonical k-mers
  // (KB_EMPTY_KEY = free); nullptr = the index has none
  const unsigned long long* dfk;
  uint64_t dfk_mask;
  int k;
  uint32_t n_ec;             // index EC sets
  uint32_t n_targets;
  const uint32_t* ec_off;    // n_ec + 1 offsets into pool (index sets occupy pool[0 .. ec_off[n_ec]))
  const int32_t* ec_handle;  // n_ec: handle (dictionary slot) of each index set
  const uint32_t* blk_ec;    // per block: set handle of its EC (strand filter)
  const uint64_t* blk_strand_off;  // per block offset into strand bytes (stranded modes)
  const uint8_t* strand;
  // single-end fragment-position filter (findPosition): per (block, member) constants, unitig length per
  // block, target lengths; null unless the index was loaded with positions
  const uint4* fp_info;
  const uint32_t* blk_usize;
  const uint32_t* target_len;
};

struct __align__(16) Memo2Entry {
  unsigned long long key;   // ~0 = free
  int32_t val;              // KB_H_NOTREADY until published
  uint32_t pad;
};

// Run-time state of one quantification run, resident on the device.
struct DevDict {
  uint32_t* pool;            // transcript-id lists
  unsigned long long* pool_top;   // next free entry in pool
  uint64_t pool_cap;
  unsigned long long* dslots;     // set dictionary: off(32) | len(24)<<32 | tag(8)<<56 ; ~0 = free
  uint64_t dmask;
  uint32_t* count;           // per handle
  unsigned long long* first; // per handle: smallest global fragment index that produced it
  // memo for tuples of exactly two EC sets: key = lo<<32|hi ; 16-byte entries, two per 32-byte block
  Memo2Entry* m2;
  uint64_t m2_mask;
  // memo for longer tuples (and tuples carrying strand words): word = tag(32)<<32 | tuple offset
  unsigned long long* mn_key;
  int32_t* mn_val;
  uint64_t mn_mask;
  uint32_t* tpool;           // tuple pool: [n, w0..w(n-1)]
  unsigned long long* tpool_top;
  uint64_t tpool_cap;
  int* error;                // sticky error flags (KB_DEVERR_*)
  unsigned long long* stats; // [0]=probes, [1]=fragments resolved by the warp kernel, [2]=memo hits, [3]=slot visits
};

enum {
  KB_DEVERR_POOL_FULL = 1,
  KB_DEVERR_DICT_FULL = 2,
  KB_DEVERR_MEMO_FULL = 4,
  KB_DEVERR_E_OVERFLOW = 8,     // more than KB_MAX_E + KB_SPILL distinct EC sets in one fragment, or wide queue full
  KB_DEVERR_TABLE_DUP = 16,     // duplicate k-mer while building the table (corrupt index)
  KB_DEVERR_TPOOL_FULL = 32,
};

__host__ __device__ __forceinline__ uint64_t kb_mix64(uint64_t x) {
  x ^= x >> 33;
  x *= 0xFF51AFD7ED558CCDULL;
  x ^= x >> 33;
  x *= 0xC4CEB9FE1A85EC53ULL;
  x ^= x >> 33;
  return x;
}

__host__ __device__ __forceinline__ uint64_t kb_revcomp(uint64_t x, int k) {
  x = ~x;
  x = ((x >> 2) & 0x3333333333333333ULL) | ((x & 0x3333333333333333ULL) << 2);
  x = ((x >> 4) & 0x0F0F0F0F0F0F0F0FULL) | ((x & 0x0F0F0F0F0F0F0F0FULL) << 4);
#ifdef __CUDA_ARCH__
  x = ((uint64_t)__byte_perm((uint32_t)x, 0, 0x0123) << 32) | (uint64_t)__byte_perm((uint32_t)(x >> 32), 0, 0x0123);
#else
  x = __builtin_bswap64(x);
#endif
  return x >> (64 - 2 * k);
}

}  // namespace kb
