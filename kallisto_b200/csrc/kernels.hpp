// Host-visible kernel argument blocks and launch wrappers (plain structs, no torch types).
#pragma once
#include <cstdint>
#include <cuda_runtime.h>
#include "kb_device.cuh"

namespace kb {

struct TableBuildArgs {
  const uint8_t* useq;
  const uint64_t* useq_byteoff;
  const uint64_t* skmer;
  const uint64_t* kstart;     // n_unitigs + 1: number of k-mers before each unitig
  const uint64_t* blk_off;
  const uint32_t* blk_lb;
  const uint32_t* blk_ub;
  const uint32_t* blk_ec;     // per block: set handle
  uint32_t n_long, n_unitigs;
  int k;
  uint64_t n_kmers;
  KmerSlot* slots;
  uint64_t mask;
  uint32_t* filter;         // optional presence filter (zeroed by the caller)
  uint32_t filter_mask;
  int* error;
};

struct DictInitArgs {
  const uint32_t* ec_off;
  const uint32_t* pool;
  uint32_t n_ec;
  unsigned long long* dslots;
  uint64_t dmask;
  int32_t* ec_handle;
};

// One batch of reads for the pseudoalignment kernels (ReadProcessor::processBuffer's `seqs`,
// src/ProcessReads.cpp:968-1046): concatenated ASCII bases, mates interleaved when paired.
// The caller of Quant::run_batch fills the batch's input and its layout: bases, off, bases2, off2, fixed_len, start,
// start2, skip, notag, alt_start and alt_start2 (zero or nullptr when not in play).  run_batch fills in the rest.
struct BatchArgs {
  const uint8_t* bases;
  const uint32_t* off;      // n_reads + 1 offsets into bases, or nullptr when every read has fixed_len bases
  const uint8_t* bases2;    // optional: second-mate buffer (then `bases`/`off` hold the first mates only and
  const uint32_t* off2;     //           read 2f+m is entry f of buffer m); nullptr = mates interleaved in `bases`
  uint32_t fixed_len;
  uint32_t n_frag;          // pairs (paired) or reads (single)
  int paired;
  int strand_mode;          // 0 unstranded, 1 FR (--fr-stranded), 2 RF (--rf-stranded)
  uint64_t frag_base;       // global index of fragment 0
  int32_t* handle_out;      // per fragment: set handle, or KB_H_UNMAPPED
  uint16_t* tl_out;         // per fragment fragment-length candidate (mapPair), or nullptr
  uint32_t* q_count;        // resolve queue
  uint32_t* q_entries;      // stride KB_Q_STRIDE
  uint32_t* spill;          // KB_SPILL words per resident lane of match_kernel: set handles beyond KB_MAX_E
  uint32_t* qbig_count;     // wide resolve queue (fragments that hit more than KB_MAX_E distinct EC sets)
  uint32_t* qbig_entries;   // stride KB_QBIG_STRIDE
  uint32_t qbig_cap;        // entries
  const uint32_t* packed;   // pack_kernel output: per read, nb 64-bit base words then nb 32-bit invalid masks
  uint32_t* rlen;           // pack_kernel output: per read, the length read_span gives it (match_kernel reads no input)
  uint32_t* take;           // match_kernel's hand-out counter: fragments claimed so far (zeroed with the queue counts)
  uint32_t nb;              // 32-base words per packed read = ceil(max_read_len / 32)
  uint32_t pstride;         // 32-bit words per packed read (multiple of 8 = 32 bytes)
  uint32_t empty_ec;        // handle of the empty index EC set, or 0xFFFFFFFF
  int refill_min;           // finished lanes of a warp that trigger a finalise + refill round
  const uint8_t* skip;      // optional per fragment: 1 = treat as having no sequence (bus: bad barcode/UMI; D-list hit)
  uint8_t* skip_w;          // the same array, writable: set when the index has a D-list (dlist_scan_kernel marks fragments)
  int fp_fl;                // >= 0: apply the fragment-position filter of ProcessReads.cpp:1095-1136 with this mean fragment length
  uint32_t start;           // first base of every read that is matched (bus: BUSOptionSubstr.start of the sequence)
  uint32_t start2;          // the same for the second mate of a pair (paired bus technologies, e.g. STORM-seq: 14)
  // UMI tag sequences (bus --tag / SMARTSEQ3, src/ProcessReads.cpp:1512-1530): notag[f] = 1 marks a fragment without the
  // tag ("ignore_umi"): its reads start at alt_start / alt_start2, the strand filter is off for it, and ONLY such
  // fragments sample fragment lengths.  nullptr = no tag sequence in play.
  const uint8_t* notag;
  uint32_t alt_start, alt_start2;
  // Translated search (bus --aa): the fragments are the six reading frames of each read set, and cfc_select_kernel
  // accounts for the set.  no_count != 0: match_kernel and resolve_kernel leave dd.count and dd.first alone.
  // first_hit (optional): per fragment, block * 2 + orientation of the first k-mer found (the first mapping k-mer of
  // doStrandSpecificity), or 0xFFFFFFFF when there is none.
  int no_count;
  uint32_t* first_hit;
};
// The counters of one batch, one 128-byte line each (they are zeroed together): q_count at word 0, qbig_count at word
// KB_BATCH_COUNTER_LINE, match_kernel's hand-out counter `take` at word 2 * KB_BATCH_COUNTER_LINE.
static constexpr int KB_BATCH_COUNTER_LINE = 32;
static constexpr int KB_BATCH_COUNTER_WORDS = 3 * KB_BATCH_COUNTER_LINE;
static constexpr int KB_Q_STRIDE = 2 + KB_MAX_E + 6;   // frag, n|flags, handles, 2 strand words, 4 position-filter words
static constexpr int KB_SPILL = 112;                   // a fragment may hit KB_MAX_E + KB_SPILL = 128 distinct EC sets
static constexpr int KB_QBIG_STRIDE = 2 + KB_MAX_E + KB_SPILL + 6;
static constexpr uint32_t KB_QBIG_CAP = 1u << 16;      // wide-queue entries per batch
// match_kernel's shared memory per lane, in 32-bit words: the handle tuple, 11 words per lookup chain (first hit, the
// reference's nextPos, the second hit of a jump, the jump and middle positions, the distance to the end of the EC block
// and the anchor hit of a jump), then the 2-bit bases of both mates (2 x 2 nb words).  At 2 x 100 bp (nb = 4) that is
// 54 words = 216 B per lane, so four blocks of 256 lanes (55.3 KB each + 1 KB reserved per block) fit in an SM's 228 KB
static constexpr int KB_CHAIN_WORDS = 11;
__host__ __device__ constexpr size_t match_lane_words(uint32_t nb) { return (size_t)KB_MAX_E + 2 * KB_CHAIN_WORDS + 4 * (size_t)nb; }

struct ResolveArgs {
  uint32_t* scratch;        // per lane group: scratch_stride entries
  uint32_t scratch_stride;
  uint32_t n_warps;         // number of lane groups (one fragment each at a time)
  uint32_t group;           // lanes per group: 32, 16, 8 or 4
};

void launch_fill_u64(unsigned long long* p, uint64_t n, unsigned long long v, cudaStream_t st);
void launch_fill_i32(int32_t* p, uint64_t n, int32_t v, cudaStream_t st);
void launch_fill_memo2(Memo2Entry* p, uint64_t n, cudaStream_t st);
void launch_build_table(const TableBuildArgs& a, cudaStream_t st);
void launch_dict_init(const DictInitArgs& a, cudaStream_t st);

// Pseudoalignment of one batch: match kernel (thread per fragment) + resolve kernel (warp per
// queued fragment) [+ fragment-length finalisation].
// ev (optional): four events recorded before pack_kernel, before match_kernel, between the kernels, after
// resolve_kernel.  packed (optional): recorded once the kernels that read the batch's input (bases, offsets) are done;
// the later kernels read only what they wrote to ba's work buffers.
void launch_pseudoalign(const DevIndex& ix, const DevDict& dd, const BatchArgs& ba, const ResolveArgs& ra,
                        int threads_per_block, cudaStream_t st, cudaEvent_t* ev = nullptr, cudaEvent_t packed = nullptr);
void launch_fld_finalize(const DevDict& dd, const BatchArgs& ba, cudaStream_t st);
void launch_import_sets(const DevDict& dd, uint32_t n_sets, const uint32_t* off, const uint32_t* tids, const uint32_t* counts,
                        const unsigned long long* first, unsigned long long first_offset, cudaStream_t st);
// Same for the tables of several ranks at once (Quant::merge_to_root): one launch, warp per incoming set.
struct ImportSeg {
  uint32_t n_sets;
  const uint32_t* off;
  const uint32_t* tids;
  const uint32_t* counts;
  const unsigned long long* first;
};
static constexpr int KB_IMPORT_SEGS = 16;
void launch_import_segments(const DevDict& dd, const ImportSeg* segs, int n_segs, cudaStream_t st);
int device_sm_count();
// Compact the handles with count > 0: used[0..*n_used)
void launch_collect_used(const DevDict& dd, uint32_t* used, uint32_t* n_used, cudaStream_t st);

// ---- EM / bootstrap (kernels_em.cu) ----
struct EmProblem {
  // structure shared by all problems of a batch
  uint32_t n_ec, n_targets;
  // ECs with >= 2 members and their members, CSR in EC-id order (denominator pass)
  uint32_t n_multi;
  const uint32_t* multi_ec;     // n_multi: EC id
  const uint32_t* m_off;        // n_multi + 1
  const uint32_t* m_tid;        // nnz
  const double* m_w;            // nnz: counts_orig[ec] / eff_len[tid]  (calc_weights, src/weights.cpp:220-246)
  // CSC by transcript over the same nnz, entries in increasing EC id (numerator pass)
  const uint32_t* t_off;        // n_targets + 1
  const uint32_t* t_midx;       // nnz: index into the multi arrays (row of the EC)
  const double* t_w;            // nnz
  const int32_t* t_single;      // n_targets: EC id of the singleton EC {t}, or -1
  // per problem (nb of them)
  int nb;
  const uint32_t* counts;       // nb x n_ec
  double* alpha;                // nb x n_targets (in/out)
  double* norm;                 // nb x n_multi scratch: counts/denom or 0
  int* rounds;                  // nb: iterations run (the reference's "ran for i rounds")
  unsigned* bar;                // arrival counter of the kernel's grid barrier (zeroed by launch_em)
  // filled by launch_em before the EM kernel starts (one dependent load less per row and per round):
  uint32_t* cnt_row;            // nb x n_multi: counts of the multi-transcript ECs in row order
  double* single_cnt;           // nb x n_targets: count of the singleton EC {t}, or 0
  int* fstate;                  // nb: final state (2 finished, 3 finished + host must zero small alphas)
  unsigned int* chcount;        // nb x 2 (double-buffered) change counters
  int max_iter, min_rounds;
  // 0: the weights m_w / t_w are shared by all problems (quant, bootstrap); nnz: problem b has its own at [b * w_stride]
  // (quant-tcc: the weights are the SAMPLE's counts / eff_len, src/weights.cpp:220-246)
  uint64_t w_stride;
  // optional, with w_stride != 0: problem b reads weight set w_set[b] instead of set b (quant-tcc bootstrap: the B
  // resampled problems of a row share that row's weights).  nullptr: set b.
  const uint32_t* w_set;
};
// Most problems one launch_em may carry: em_kernel keeps an int of state per problem in dynamic shared memory (32 KB
// here, under the 48 KB a launch gets without opting in).  The bootstrap and quant-tcc also launch their resample /
// fill kernels for at most this many samples at a time: the samples sit on gridDim.y (at most 65 535).
static constexpr int KB_EM_MAX_BATCH = 8192;
// co-resident blocks of em_kernel for `nb` problems (the cooperative launch's limit)
int em_max_blocks(int threads_per_block, int nb);
// quant-tcc helpers: dense per-sample count vectors from the sparse TCC rows, and per-sample weights in CSR and CSC order
struct TccFill {
  uint32_t n_ec, n_targets, nb;        // samples in this chunk
  const unsigned long long* row_off;    // chunk's rows: nb + 1 offsets into ec_ids / vals
  const uint32_t* ec_ids;
  const uint32_t* vals;
  uint32_t* counts;                     // nb x n_ec (zeroed by the launcher)
  // entry -> (EC id, transcript) of the CSR (m_*) and CSC (t_*) layouts
  uint64_t nnz;
  const uint32_t* m_ec; const uint32_t* m_tid; const uint32_t* t_ec; const uint32_t* t_tid;
  const double* eff; uint64_t eff_stride;   // nb x n_targets when eff_stride == n_targets, shared when 0
  double* m_w; double* t_w;             // nb x nnz
};
void launch_tcc_fill(const TccFill& a, cudaStream_t st);

// Component layout of one problem (kernels_emprep.cu builds it, em_component_kernel runs on it).  The bipartite graph of
// multi-transcript ECs and transcripts falls apart into connected components that never exchange a value; they are
// sorted by (component, id) and cut at component boundaries into slices, one per block.  Size of a component or a
// slice = transcripts + rows + entries.  Positions ("pos") are indices into the sorted order; every array below is
// workspace of at least the size given (T transcripts, R multi-transcript ECs, nnz entries).
struct EmCompWs {
  uint32_t* parent;               // T: union-find forest, then the component (its smallest transcript id) of every transcript
  uint32_t* rfirst;               // T: rows whose first transcript this is
  unsigned long long* csize;      // T: size of the component rooted here
  unsigned long long* cstart;     // T: size of all components before the one rooted here
  uint32_t* iota;                 // max(T, R)
  uint32_t* tkey;                 // T: component of the transcript at each pos
  uint32_t* t_id;                 // T: pos -> transcript
  uint32_t* tloc;                 // T: transcript -> pos inside its slice
  unsigned long long* tsize;      // T + 1: size carried by each pos (itself, its entries, the rows it heads), then its scan
  unsigned long long* tscan;      // T + 1
  uint32_t* rcomp;                // R: component of each row
  uint32_t* rkey;                 // R: component of the row at each row pos
  uint32_t* r_id;                 // R: row pos -> row
  uint32_t* rloc;                 // R: row -> row pos inside its slice
  uint32_t* r_cnt;                // R: count of the row at each row pos
  uint32_t* r_len;                // R + 1
  uint32_t* r_off;                // R + 1: entries of the row at each row pos (CSR in slice order)
  uint16_t* r_tid;                // nnz: slice-local transcript pos
  double* r_w;                    // nnz
  double* t_single;               // T: singleton count of the transcript at each pos
  uint32_t* t_len;                // T + 1
  uint32_t* t_off;                // T + 1: entries of the transcript at each pos (CSC in slice order)
  uint16_t* t_row;                // nnz: slice-local row pos
  double* t_w;                    // nnz
  uint32_t* s_t0;                 // slices + 1: first pos of each slice
  uint32_t* s_r0;                 // slices + 1: first row pos of each slice
  const double* eff;              // T, by transcript id: effective lengths the weights were formed from; nullptr: the
                                  //    resident kernel is off
  double* t_eff;                  // T: effective length of the transcript at each pos
  unsigned long long* stats;      // 8: [0] total size, [1] slice target size, [2] slices, [3] largest component,
                                  //    [4] largest slice's shared memory (bytes), [5] entries whose weight
                                  //    emcomp_weight does not rebuild bit for bit, [6] largest slice's shared memory
                                  //    in the resident layout (bytes)
  unsigned* sync;                 // 2 x sync_rounds: per round, blocks that changed an estimate, blocks that arrived
  int sync_rounds;
  int max_slices;                 // capacity of s_t0 / s_r0 minus one
  void* tmp;
  size_t tmp_bytes;
};
// Shared memory of em_component_kernel for a slice of nt transcripts and nr rows: alpha and the singleton count per
// transcript, norm per row (doubles), then the count per row and the entry offsets of rows and transcripts (uint32).
__host__ __device__ inline unsigned long long emcomp_smem_bytes(uint32_t nt, uint32_t nr) {
  return 20ull * nt + 16ull * nr + 8;
}
// The resident layout of the same slice with ne entries: also the effective length and its reciprocal per transcript
// (doubles), and every entry's two 16-bit indices; the weights are rebuilt from the counts (emcomp_weight).
__host__ __device__ inline unsigned long long emcomp_resident_bytes(uint32_t nt, uint32_t nr, unsigned long long ne) {
  return emcomp_smem_bytes(nt, nr) + 16ull * nt + 4ull * ne;
}
// The weight of an entry, count c / eff, from y = __drcp_rn(eff): q = c y is within an ulp of c / eff, the residual
// c - q eff is exact in one fma, and q + r y is then the correctly rounded quotient (Markstein), i.e.
// __ddiv_rn(c, eff), which is how the weights are formed (calc_weights).  emcomp_cut checks every entry anyway.
__device__ __forceinline__ double emcomp_weight(double c, double eff, double y) {
  const double q = __dmul_rn(c, y);
  return __fma_rn(__fma_rn(-q, eff, c), y, q);
}
size_t emcomp_tmp_bytes(uint32_t n_targets, uint32_t n_multi);
// Largest component the component kernel takes: KB_EM_COMP_CAP (test knob, in the size units above), else unlimited.
unsigned long long emcomp_cap();
// Shared memory the resident layout may take per block: KB_EM_COMP_SMEM (test knob, bytes; 0 keeps the weights
// streamed), else whatever the device grants a block.
unsigned long long emcomp_smem_budget();
// Components, slices and the slice bounds, and the check of the weights against emcomp_weight when w.eff is set;
// returns stats[0..6] through one device-to-host read.
void emcomp_cut(const EmProblem& p, const EmCompWs& w, uint32_t slices, unsigned long long* stats_host, cudaStream_t st);
// Per-slice copies of counts, offsets and entries with slice-local 16-bit indices; with `resident`, the effective
// lengths per pos instead of the weights per entry.
void emcomp_fill(const EmProblem& p, const EmCompWs& w, bool resident, cudaStream_t st);

// The start state of nb problems over T targets, alpha[b * T + t]: prior[t] when `prior` (T doubles, device) is given,
// else `uniform` (the caller's 1.0 / T, EMAlgorithm.h:38).
void launch_em_start(double* alpha, uint32_t nb, uint32_t T, const double* prior, double uniform, cudaStream_t st);

// Returns the number of blocks of em_component_kernel it launched, 0 when one of the grid-wide kernels ran.
// `cw` (optional, one problem): workspace of the component layout.  `resident` (optional): set to whether the
// component kernel held the entries in shared memory.
int launch_em(const EmProblem& p, int threads_per_block, cudaStream_t st, const EmCompWs* cw = nullptr,
              bool* resident = nullptr);

// Device-side EM problem construction (kernels_emprep.cu)
struct EmPrep {
  uint32_t n_ec, n_multi, n_targets;
  // per EC (id = order of first occurrence); arrays of n_ec + 1 where a scan total is stored
  uint32_t* handle;
  uint32_t* count;
  uint32_t* len;           // n_ec + 1
  uint32_t* ec_off;        // n_ec + 1: offsets of the EC table
  uint32_t* m_off;         // n_ec + 1: offsets into the multi-EC entry arrays (0-length for singletons)
  uint32_t* multi_index;   // n_ec + 1: after the scan the rank among the multi-transcript ECs, after emprep_rows the ROW of the EC
  uint32_t* minkey;        // n_ec: smallest transcript id of the EC
  uint32_t* ec_tid;        // EC table entries
  // multi-transcript ECs, CSR
  uint32_t* multi_ec;      // n_multi
  uint32_t* m_rowoff;      // n_multi + 1
  uint32_t* m_tid;
  double* m_w;
  uint32_t* m_row;         // entry -> row
  uint32_t* m_iota;        // entry -> entry (values of the CSC sort)
  unsigned long long* k64_in;   // entry -> tid << 32 | EC id (keys of the CSC sort)
  // CSC
  uint32_t* t_deg;         // n_targets + 1 (zeroed by the caller)
  uint32_t* t_off;         // n_targets + 1
  uint32_t* t_midx;
  double* t_w;
  int32_t* t_single;       // n_targets (filled with -1 by the caller)
  const double* eff;       // n_targets
};
size_t emprep_sort_bytes(uint32_t n_used, uint32_t nnz_max);
void emprep_sort_by_first(const DevDict& dd, const uint32_t* used, uint32_t n_used, unsigned long long* key_in,
                          unsigned long long* key_out, uint32_t* idx_in, uint32_t* order_out, void* tmp, size_t tmp_bytes,
                          cudaStream_t st);
void emprep_meta(const DevDict& dd, const uint32_t* used, const uint32_t* order, uint32_t n, const EmPrep& p,
                 uint32_t* multi_len, uint32_t* is_multi, void* tmp, size_t tmp_bytes, cudaStream_t st);
void emprep_rows(const EmPrep& p, const uint32_t* is_multi, uint32_t* ckey, uint32_t* cval, uint32_t* ckey_out, uint32_t* rlen,
                 void* tmp, size_t tmp_bytes, cudaStream_t st);
void emprep_fill_table(const DevDict& dd, const EmPrep& p, cudaStream_t st);
void emprep_fill(const DevDict& dd, const EmPrep& p, uint32_t nnz, unsigned long long* sort_keys_out, uint32_t* sort_vals_out,
                 void* tmp, size_t tmp_bytes, unsigned long long* stats2, cudaStream_t st);

// ---- BUS (kernels_bus.cu) ----
struct BusRecord {      // BUSData, src/BUSData.h:30-38
  uint64_t barcode, umi;
  int32_t ec;
  uint32_t count, flags, pad;
};
struct BusSpec {        // BUSOptions (src/common.h:38-91): where barcode / UMI / sequence sit in the files of a read set
  int nfiles;
  int n_bc, n_umi;
  int bc_f[4], bc_a[4], bc_b[4];
  int umi_f[4], umi_a[4], umi_b[4];
  int seq_file, seq_start;
  int num_flag;         // --num: flags = read number
  int paired;           // busopt.paired: two sequence reads, pseudoaligned as a pair (src/ProcessReads.cpp:1550-1567)
  int seq2_file, seq2_start;
  int no_umi;           // umi[0].fileno == -1 ("bulk_like", :1393): UMI field = ~0, one count in umi_len[1]
  unsigned long long fake_bc;   // n_bc == 0: the barcode every record gets (0 = 16 x 'A'; batch mode: the sample's id, :1603-1607)
  int tag_len;                  // --tag: length of the tag sequence that precedes the UMI (0 = none); umi_a[0] is already advanced by it
  unsigned long long tag_bin;   // stringToBinary(tag)
  int batch_bc;                 // --batch-barcodes with a barcode read: the sample's number goes in front of the barcode
  unsigned long long bc_prefix; // batch_bc: the sample's number (batch_id_mapping[id], src/ProcessReads.cpp:1617-1626)
};
struct BusArgs {
  const uint8_t* bases[4];
  const uint32_t* off[4];
  uint32_t n_sets;
  uint64_t set_base;
  BusSpec spec;
  uint64_t* barcode;
  uint64_t* umi;
  uint32_t* flags;
  uint8_t* skip;
  uint8_t* notag;       // tag runs: 1 = the read set does not carry the tag
  uint32_t* bc_hist;    // 33 bins
  uint32_t* umi_hist;   // 33 bins
  unsigned long long* n_valid;
  unsigned long long* n_long_bc;   // batch_bc: read sets whose barcode has more than 32 letters (the run must stop)
};
size_t bus_scan_bytes(uint32_t n);
void launch_bus_fields(const BusArgs& a, cudaStream_t st);
void launch_bus_records(const DevDict& dd, const int32_t* handle, uint32_t n, uint64_t base, uint32_t next_id,
                        int32_t* id_of, uint32_t* is_new, uint32_t* new_rank, uint32_t* is_mapped, uint32_t* rank,
                        const uint64_t* barcode, const uint64_t* umi, const uint32_t* flags, BusRecord* out, void* tmp,
                        size_t tmp_bytes, cudaStream_t st);
// bus --devices (kb_bus_group_*): launch_bus_records in two halves around the host's choice of run-wide EC ids.
// launch_bus_new_sets flags the fragments as launch_bus_records does, and lays the sets new on this run out as CSR in
// new_rank order: out_off[0 .. n_new], out_tid[0 .. total) (ids past `cap` are left out; the total is eoff[n]).
// len / eoff: n + 1 words each.  launch_bus_export_gather repeats the gather once the host has a large enough buffer.
void launch_bus_new_sets(const DevDict& dd, const int32_t* handle, uint32_t n, uint64_t base, uint32_t* is_new,
                         uint32_t* new_rank, uint32_t* is_mapped, uint32_t* rank, uint32_t* len, uint32_t* eoff,
                         uint32_t cap, uint32_t* out_off, uint32_t* out_tid, void* tmp, size_t tmp_bytes, cudaStream_t st);
void launch_bus_export_gather(const DevDict& dd, const int32_t* handle, uint32_t n, const uint32_t* is_new,
                              const uint32_t* new_rank, const uint32_t* eoff, uint32_t cap, uint32_t* out_off,
                              uint32_t* out_tid, cudaStream_t st);
// id_of[handle] = gid[new_rank] for the new sets, then the records of launch_bus_records
void launch_bus_group_records(const int32_t* handle, uint32_t n, const uint32_t* is_new, const uint32_t* new_rank,
                              const int32_t* gid, int32_t* id_of, const uint32_t* is_mapped, const uint32_t* rank,
                              const uint64_t* barcode, const uint64_t* umi, const uint32_t* flags, BusRecord* out,
                              cudaStream_t st);

// ---- translated search, bus --aa (kernels_cfc.cu) ----
// The six reading frames of every read set in comma-free code, fragment 6 i + j = frame j of set i.
struct CfcArgs {
  const uint8_t* bases;     // the sequence file of the batch
  const uint32_t* off;      // n_sets + 1
  uint32_t start;           // first base of the sequence in its read
  const uint8_t* skip;      // per set: 1 = no sequence (bad barcode / UMI): its frames are empty
  uint32_t n_sets;
  uint32_t max_len;         // longest sequence (after `start`)
  uint32_t* set_off;        // n_sets + 1: frame letters before each set (filled by launch_cfc_frames)
  uint8_t* fbases;          // frame letters
  uint32_t* foff;           // 6 n_sets + 1 frame offsets
  void* tmp;
  size_t tmp_bytes;         // cfc_scan_bytes(n_sets)
};
size_t cfc_scan_bytes(uint32_t n_sets);
void launch_cfc_frames(const CfcArgs& a, cudaStream_t st);
// After the frames went through launch_pseudoalign with ba.no_count and ba.first_hit: per set, the winning frame's set
// (smallest non-empty, lowest frame on a tie), the frame-0 strand filter when strand_mode != 0, the accounting
// (dd.count, dd.first = ba.frag_base + set) and the set's handle in handle_out[set].  clashes += frames whose set is as
// small as the smallest one before them.
void launch_cfc_select(const DevIndex& ix, const DevDict& dd, const BatchArgs& ba, const ResolveArgs& ra, uint32_t n_sets,
                       int strand_mode, int32_t* handle_out, unsigned long long* clashes, cudaStream_t st);

struct ResampleArgs {
  const double* cp;          // n_ec cumulative probabilities (discrete_distribution::_M_cp)
  uint32_t n_ec;
  uint64_t n_draws;          // N = sum(counts)
  int nb;
  const uint32_t* x0;        // nb initial minstd_rand0 states
  uint32_t* samp;            // nb x n_ec output counts (zeroed by the launcher)
};
void launch_resample(const ResampleArgs& a, cudaStream_t st);

// quant-tcc bootstrap: problem p of a launch is global problem g = first + p, i.e. bootstrap g % B of row g / B.  Every
// row has a cumulative table over its NON-ZERO ECs (plus the sentinel of the last EC, see tcc_bootstrap in engine.cu);
// the draws of all problems form one flat list of 64-draw chunks, chunk_off being its prefix sum per problem.
struct TccResampleArgs {
  uint32_t n_ec;
  uint32_t nb;                          // problems in this launch
  uint64_t first;                       // global index of problem 0
  uint32_t B;                           // bootstraps per row
  const uint32_t* x0;                   // B initial minstd_rand0 states (the same for every row)
  const unsigned long long* cp_off;     // rows + 1: offsets of each row's table (indexed by global row)
  const double* cp;                     // partial sums, the last of each row 1.0
  const uint32_t* cp_ec;                // EC id of each table entry
  const unsigned long long* n_draws;    // per global row: the row's total count
  const unsigned long long* chunk_off;  // nb + 1: prefix sum of ceil(n_draws / 64) over the launch's problems
  uint64_t n_chunks;                    // chunk_off[nb]
  uint32_t* samp;                      // nb x n_ec output counts (zeroed by the launcher)
};
void launch_tcc_resample(const TccResampleArgs& a, cudaStream_t st);

// quant-tcc gene-level output (src/main.cpp:3026-3058, plaintext_writer_gene src/PlaintextWriter.cpp:67-112): per problem,
// tpm = counts_to_tpm(alpha, eff_lens), then for every transcript with alpha > 0 in increasing id, gene_counts[gene] +=
// alpha and gene_tpm[gene] += tpm.  The genes come as a CSR of member transcripts in increasing id, so a (problem, gene)
// thread adds in the reference's order; the total mass is a sequential sum in target order, one thread per problem.
struct TccGeneArgs {
  uint32_t nb, n_targets, n_genes;
  const double* alpha;                  // nb x n_targets
  const int* fstate;                    // nb: 3 -> alphas below 1e-8 count as 0 (the host zeroes them, EMAlgorithm.h:213-216)
  const double* eff; uint64_t eff_stride;   // problem b's eff_lens: eff + (w_set ? w_set[b] : b) * eff_stride
  const uint32_t* w_set;                // nb or nullptr
  const uint32_t* g_off;                // n_genes + 1
  const uint32_t* g_tid;                // member transcripts, increasing within a gene
  double* total;                        // nb scratch: sum of alpha / eff_len
  double* gene_counts;                  // nb x n_genes
  double* gene_tpm;                     // nb x n_genes
};
void launch_tcc_genes(const TccGeneArgs& a, cudaStream_t st);

}  // namespace kb
