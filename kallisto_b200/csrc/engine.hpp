// Host-side engine: owns the device tables of one index and the device state of one
// quantification run.  This is the C++ layer right under the C ABI (include/kallisto_b200.h);
// it mirrors the reference objects that sit on the hot path:
//
//   kb::Index  <->  KmerIndex after KmerIndex::load            (src/KmerIndex.cpp:1330-1559)
//   kb::Quant  <->  MinCollector + MasterProcessor/ReadProcessor (src/MinCollector.h:17-119,
//                   src/ProcessReads.cpp:307-483, 934-1237) followed by EMAlgorithm / Bootstrap
//
// There is no CPU implementation of any of the per-read or per-iteration work in here:
// without a CUDA device every entry point throws.
#pragma once
#include <cstdint>
#include <functional>
#include <memory>
#include <stdexcept>
#include <string>
#include <unordered_map>
#include <vector>

#include "index_v13.hpp"
#include "kernels.hpp"

namespace kb {

struct Error : std::runtime_error {
  using std::runtime_error::runtime_error;
};

template <class T>
struct DBuf {
  T* p = nullptr;
  size_t n = 0;
  DBuf() = default;
  DBuf(const DBuf&) = delete;
  DBuf& operator=(const DBuf&) = delete;
  ~DBuf() { release(); }
  void alloc(size_t count);
  // grow-only: at least `need` elements (contents are lost when it grows); `slack` over-allocates by that fraction
  void grow(size_t need, double slack = 0.0) { if (n < need) alloc(need + (size_t)((double)need * slack)); }
  void release();
  void upload(const T* src, size_t count, cudaStream_t st = 0);
  void download(T* dst, size_t count, size_t offset = 0, cudaStream_t st = 0) const;
  void zero(cudaStream_t st = 0);
};

// Everything one batch's kernels write that the next batch's would overwrite.  A run keeps two: batch i uses
// BatchWs::slot[i & 1] on the run's internal stream i & 1 (Quant::run_batch), so that batch i + 1 can run while batch i
// drains, and stream order alone keeps batch i + 2 off the buffers until batch i is done with them.
struct BatchSlot {
  DBuf<uint32_t> d_counters;        // KB_BATCH_COUNTER_WORDS: the queue counts and match_kernel's hand-out counter
  DBuf<uint32_t> d_qentries, d_scratch, d_packed, d_rlen;
  DBuf<uint32_t> d_spill, d_qbig;   // fragments with more than KB_MAX_E distinct EC sets (d_spill: per resident lane)
  DBuf<int32_t> d_handles;
  DBuf<uint16_t> d_tl;
  DBuf<uint8_t> d_skip;             // per fragment: holds a D-list k-mer (only when the index has a D-list)
};

// Grow-only device work buffers.  They belong to the Index and are lent to one run at a time, so that
// consecutive runs on the same index (the normal case) do not pay cudaMalloc again; a second run
// created while the first is still alive gets private ones.
struct BatchWs {
  // input staging of the host entry points (Quant::stage), up to four files per slot: the quant runs alternate between
  // the slots, so that the copy of batch i+1 overlaps the kernels of batch i; the bus runs use slot 0
  DBuf<uint8_t> stage_b[2][4];
  DBuf<uint32_t> stage_o[2][4];
  BatchSlot slot[2];
};

// The per-problem device state of launch_em for up to `cap` problems (grow-only), and the one host-side driver of every
// EM batch: launch() starts the problems from the given priors (or a uniform alpha) with zeroed round counts, final
// states and change counters; fetch() downloads their estimates and round counts and applies the state-3 zeroing.
// Bootstraps always start uniform (Bootstrap::run_em builds a fresh EMAlgorithm, src/Bootstrap.cpp:4-13): their
// callers pass no priors.
struct EmState {
  DBuf<double> alpha, norm, single_cnt;
  DBuf<uint32_t> cnt_row;
  DBuf<int> emi;                    // rounds in [0, cap), final states in [cap, 2 cap)
  DBuf<unsigned int> chcount, bar;  // two change counters per problem; the grid barrier's arrival counter
  std::vector<int> h_emi;
  size_t cap = 0;
  void reserve(size_t nb, uint32_t T, size_t n_multi);
  // p: the shared structure filled in by the caller (n_ec .. w_set, max_iter, min_rounds); its per-problem fields are
  // pointed at this state.  `start` (optional) is recorded right before launch_em.  `prior` (optional, device, n_targets
  // doubles): the start of every problem instead of the uniform 1 / n_targets.  Returns what launch_em returns.
  int launch(EmProblem& p, int nb, const uint32_t* counts, int threads_per_block, cudaStream_t st,
             const EmCompWs* cw = nullptr, cudaEvent_t start = nullptr, bool* comp_resident = nullptr,
             const double* prior = nullptr);
  // Enqueues the download of p's nb x n_targets estimates and nb rounds behind whatever the caller enqueued since
  // launch(), synchronises the stream once and zeroes the small estimates of problems that stopped in state 3.
  void fetch(const EmProblem& p, double* alpha_out, int* rounds_out, cudaStream_t st);
};

struct EmWs {   // grow-only device workspace of Quant::number_ecs and of what run_em_device builds on its numbering
  DBuf<uint32_t> used, scal, idx_in, order, handle, count, len, multi_len, is_multi, ec_off, m_off, multi_index;
  DBuf<unsigned long long> key_in, key_out;
  DBuf<uint8_t> tmp;
  DBuf<uint32_t> ec_tid, multi_ec, m_rowoff, m_tid, m_row, m_iota, sortv, t_deg, t_off, t_midx;
  DBuf<uint32_t> minkey, ckey, cval, ckey_out, rlen;     // row order of the EM matrices (emprep_rows)
  DBuf<unsigned long long> k64_in, k64_out;              // CSC sort keys
  // bootstrap over the same matrices (run_bootstrap_device)
  DBuf<uint32_t> bs_counts, bs_x0;
  DBuf<double> bs_cp;
  DBuf<double> m_w, t_w, eff;
  DBuf<int32_t> t_single;
  EmState em;                                            // per-problem state of run_em_device and the bootstrap
  // The two sizings (slack: see DBuf::grow): what number_ecs touches for n ECs, and the EM matrices and single-problem
  // state of n ECs (n_multi of them with >= 2 targets, nnz entries in those) over T targets.  ec_tid, the EC table's
  // entries, is sized by whoever fills it.
  void reserve_numbering(size_t dict_cap, size_t n, double slack);
  void reserve_matrices(size_t n, uint32_t T, size_t n_multi, size_t nnz, double slack);
  // the shared structure of the EM matrices run_em_device built here (n_ec ECs, n_multi of them with >= 2 targets)
  EmProblem problem(uint32_t n_ec, uint32_t T, uint32_t n_multi, int max_iter, int min_rounds) const;
  // component layout of the single-problem EM (EmCompWs, kernels.hpp)
  DBuf<uint32_t> c_parent, c_rfirst, c_iota, c_tkey, c_tid, c_tloc, c_rcomp, c_rkey, c_rid, c_rloc, c_rcnt, c_rlen, c_roff;
  DBuf<uint32_t> c_tlen, c_toff, c_st0, c_sr0;
  DBuf<unsigned long long> c_csize, c_cstart, c_tsize, c_tscan, c_stats;
  DBuf<uint16_t> c_rtid, c_trow;
  DBuf<double> c_rw, c_tw, c_tsingle, c_teff;
  DBuf<unsigned> c_sync;
  DBuf<uint8_t> c_tmp;
  // grows the buffers to T transcripts, R rows, nnz entries and max_iter rounds and hands them out; `eff`: the
  // effective lengths the weights were formed from (EmCompWs::eff)
  EmCompWs comp(uint32_t T, uint32_t R, size_t nnz, int max_iter, const double* eff);
};

// What Quant::number_ecs found: n ECs with n_entries transcript ids in all, n_multi of them with >= 2 transcripts and
// multi_entries ids in those; `prep` points at their handle / count / len / offsets in the EmWs (ec_tid and the
// matrices are for the caller to size and fill).
struct EcNumbering {
  uint32_t n = 0, n_entries = 0, multi_entries = 0, n_multi = 0;
  EmPrep prep{};
};

class Index {
 public:
  static std::unique_ptr<Index> load(const std::string& path, int device, bool load_positions, int threads);
  ~Index();

  FlatIndex flat;
  int device = 0;
  DevIndex dev{};
  uint64_t table_cap = 0;
  uint64_t dict_cap = 0;          // set-dictionary capacity used by every run on this index
  uint32_t empty_ec = 0xFFFFFFFFu;
  uint32_t max_set_len = 0;
  uint32_t n_index_tids = 0;      // pool entries occupied by the index's own EC sets
  double load_seconds = 0, build_seconds = 0;

  DBuf<KmerSlot> slots;
  DBuf<unsigned long long> dfk;   // D-list k-mer set
  DBuf<uint32_t> filter;          // presence filter of the k-mer table (L2-resident, see DevIndex)
  size_t l2_persist_bytes = 0;    // persisting-L2 carve-out set aside for it
  DBuf<uint32_t> ec_off;
  DBuf<uint32_t> index_pool;      // the index's EC sets (copied to the front of every run's pool)
  DBuf<unsigned long long> dslots_init;
  DBuf<int32_t> ec_handle;
  std::vector<int32_t> h_ec_handle;   // host copy: index EC-set id -> dictionary handle
  DBuf<uint32_t> blk_ec;
  DBuf<uint64_t> blk_strand_off;
  DBuf<uint8_t> strand;
  BatchWs shared_bws;
  EmWs* shared_emws = nullptr;
  bool ws_in_use = false;
  DBuf<uint4> fp_info;            // only when loaded with positions
  DBuf<uint32_t> blk_usize, target_len;
};

// One NCCL communicator per process/GPU plus the receive area of the merge (csrc/comm.cu).
struct CommImpl;
class Comm {
 public:
  static void unique_id(void* out128);                                  // ncclGetUniqueId (rank 0, then broadcast by the caller)
  Comm(int n_ranks, int rank, const void* id128, int device);            // ncclCommInitRank
  Comm(void* nccl_comm, int n_ranks, int rank, int device, bool take_ownership);   // an existing ncclComm_t
  static std::vector<Comm*> init_all(const std::vector<int>& devices);   // one process, one communicator per device
  ~Comm();
  Comm(const Comm&) = delete;
  Comm& operator=(const Comm&) = delete;
  void reserve(size_t n_sets_per_rank, size_t n_entries_per_rank);       // root: size the receive area ahead of time
  int n_ranks = 1, rank = 0, device = 0;
  CommImpl* impl_ = nullptr;
};

struct QuantOptions {
  int paired = 1;          // !opt.single_end
  int strand_mode = 0;     // 0 unstranded, 1 --fr-stranded, 2 --rf-stranded
  int collect_fld = 1;     // opt.fld == 0: estimate the fragment-length distribution from the data
  uint32_t max_batch_reads = 1u << 22;     // staging capacity (reads per batch)
  uint64_t max_batch_bases = 1ull << 29;   // staging capacity (bases per batch)
  int threads_per_block = 256;
  int fp_fl = -1;          // >= 0: fragment-position filter with this mean fragment length (!single_overhang && -l given)
  bool bus = false;        // `kallisto bus` run: records instead of (only) counts
  BusSpec bus_spec{};
  int refill_min = 16;     // match_kernel: finished lanes per warp that trigger a finalise + refill round
};

// Equivalence classes of a finished run, ids in order of first occurrence (== reference -t 1).
struct EcTable {
  std::vector<uint64_t> off;      // n_ec + 1
  std::vector<uint32_t> tid;
  std::vector<uint32_t> count;
  std::vector<int32_t> handle;    // device handle of each EC (to translate per-fragment results)
  uint32_t n() const { return (uint32_t)count.size(); }
};

struct EmResult {
  std::vector<double> alpha;      // est_counts
  std::vector<double> eff_lens;
  int rounds = 0;
  double seconds = 0;
};

struct Stats {
  uint64_t n_processed = 0, n_pseudoaligned = 0, n_unique = 0;
  uint64_t n_probes = 0, n_slot_visits = 0, n_resolved = 0, n_memo_hits = 0;
};

class Quant {
 public:
  Quant(Index& ix, const QuantOptions& opt);
  ~Quant();

  // One batch of reads (mates interleaved when paired).  `off` has n_reads+1 entries or is null
  // when every read has `fixed_len` bases.  Pointers are HOST memory; the copy to the device, the
  // kernels and (if handles_out != null) the copy back of one handle per fragment happen inside.
  void pseudoalign_host(const char* bases, const uint32_t* off, uint32_t n_reads, uint32_t fixed_len,
                        int32_t* handles_out);
  // Paired batch with one buffer per mate (what a FASTQ reader produces: R1 and R2 parsed
  // separately), n_pairs fragments; off1/off2 have n_pairs + 1 entries or are null with fixed_len.
  void pseudoalign_host_pe(const char* bases1, const uint32_t* off1, const char* bases2, const uint32_t* off2,
                           uint32_t n_pairs, uint32_t fixed_len, int32_t* handles_out);
  // `kallisto bus`: one batch of read sets (bases[k]/offs[k] = file k of the technology, n_sets + 1
  // offsets each).  Writes the BUS records of the pseudoaligned sets, in read order, EC ids final.
  void bus_batch_host(const char* const* bases, const uint32_t* const* offs, uint32_t n_sets, BusRecord* records_out,
                      uint32_t* n_records_out);
  uint32_t bus_batch_device(const uint8_t* const* d_bases, const uint32_t* const* d_offs, uint32_t n_sets, uint32_t max_seq_len);
  const BusRecord* bus_records_device() const { return bus_rec_.p; }
  void bus_lengths(uint32_t* bc_hist, uint32_t* umi_hist);
  // Batch mode (`bus -x BULK` / `bus --batch`, src/ProcessReads.cpp:371-404,1603-1626): the read sets that follow belong
  // to sample `barcode` (the fake barcode of their records without a barcode read, else the prefix of set_batch_barcodes);
  // its fragment-length sampling and --num read numbers start again.
  void bus_begin_sample(uint64_t barcode);
  // `bus --batch --batch-barcodes` with a barcode read: every barcode gets the sample's number (bus_begin_sample) in
  // front of it, 32 letters in all (src/ProcessReads.cpp:1617-1626).  Before the first batch.
  void set_batch_barcodes(bool on);
  // `bus --aa` (src/ProcessReads.cpp:1652-1695): every read set is matched in its six reading frames, translated into
  // comma-free code, against a protein index; the smallest non-empty frame set wins.  Before the first batch; refused
  // for paired technologies, tag sequences and indices with a D-list.
  void set_aa(bool on);
  // cardinality_clashes of the run: frames whose set was as small as the winning frame's before them
  uint64_t frame_clashes();
  // ---- `bus --devices`: this run as a member of a BusGroup (several runs, one run-wide EC numbering) ----
  // Stages one batch whose first read set has the run-wide index `base`, in a sample whose first read set has the
  // run-wide index `sample_base`, and enqueues its work up to the export of the sets new on this run.  Returns once
  // the host buffers may be reused.  One batch at a time: bus_group_finish ends it.
  void bus_group_submit(const char* const* bases, const uint32_t* const* offs, uint32_t n_sets, uint64_t base,
                        uint64_t sample_base);
  // Waits for the submitted batch and returns its new sets in order of first occurrence (off: n_new + 1 entries)
  void bus_group_new_sets(std::vector<uint32_t>& off, std::vector<uint32_t>& tids);
  // Gives the new sets the run-wide ids `gid` (one per new set, in that order) and returns the batch's records
  void bus_group_finish(const int32_t* gid, BusRecord* records_out, uint32_t* n_records_out);
  bool bus_fresh() const { return n_frag_total_ == 0 && !grp_pending_; }
  bool aa() const { return aa_; }
  // Same, inputs already resident in device memory; handles stay on the device
  // (device_handles(), valid until the next batch).  The call returns once the kernels are enqueued; the caller may
  // overwrite its input in the run's stream order, since that stream waits for the kernels that read it.
  void pseudoalign_device(const uint8_t* d_bases, const uint32_t* d_off, uint32_t n_reads, uint32_t fixed_len,
                          uint32_t max_read_len);
  // the last batch's handles, complete in the run's stream order
  const int32_t* device_handles() { join(); return bws_->slot[last_slot_].d_handles.p; }
  void sync();

  // MasterProcessor tail flush + EC id assignment: the table export_prepare lays out on the device (ids from
  // number_ecs), downloaded.
  const EcTable& finalize_ecs();
  const std::vector<uint32_t>& flens() const { return flens_; }
  void set_flens(const uint32_t* f);     // e.g. after an all-reduce across ranks
  Stats stats();

  // Effective lengths from the fragment-length distribution (or a given mean/sd), then the EM.
  std::vector<double> mean_fl_trunc(double fld_mean, double fld_sd) const;
  EmResult run_em(const EcTable& ecs, const std::vector<double>& fl_trunc, int max_iter = 10000, int min_rounds = 50);
  // Same result, EC table built and kept on the device (the `quant` fast path).
  EmResult run_em_device(const std::vector<double>& fl_trunc, int max_iter = 10000, int min_rounds = 50);
  // ---- multi-GPU: ship this rank's equivalence classes to another rank / fold another rank's in ----
  // export_prepare numbers the ECs (number_ecs) and lays the table out on the device; returns
  // {n_sets, n_entries}.  export_copy then fills caller-provided DEVICE buffers (e.g. torch tensors
  // about to go through NCCL): off[n_sets+1], tids[n_entries], counts[n_sets], first[n_sets].
  void export_prepare(uint32_t* n_sets, uint32_t* n_entries);
  void export_copy(uint32_t* d_off, uint32_t* d_tids, uint32_t* d_counts, unsigned long long* d_first);
  void import_sets_device(uint32_t n_sets, const uint32_t* d_off, const uint32_t* d_tids, const uint32_t* d_counts,
                          const unsigned long long* d_first, unsigned long long first_offset);
  void add_processed(uint64_t n) { n_frag_total_ += n; }
  // The whole exchange in one collective call (csrc/comm.cu): tables gathered to rank 0 with NCCL send/recv and
  // folded in by content with one kernel launch, fragment-length samples completed in rank order.  Returns the
  // number of fragments processed by all ranks.
  uint64_t merge_to_root(Comm& comm, uint64_t first_stride);
  // Same merge when all runs live in THIS process (one host thread drives several GPUs, `kallisto_b200 quant --devices`):
  // the other runs' tables are copied with cudaMemcpyPeerAsync (NVLink) -- no communicator to set up.  Called on the root.
  uint64_t merge_local(const std::vector<Quant*>& others, uint64_t first_stride);
  // Global index of the first fragment of the NEXT batch (multi-GPU drivers that deal batches of one read
  // stream to several runs: first-occurrence order then is the order of the stream).  Default: running count.
  void set_frag_base(uint64_t base) { frag_base_ = base; have_frag_base_ = true; }
  // Size the EM / EC-numbering workspace ahead of time (no cudaMalloc on the first kb_em_run).
  void reserve_em(size_t n_ecs, size_t n_entries);

  // --priors (EMAlgorithm::set_priors, src/EMAlgorithm.h:83-93): n_targets start values of every later run_em /
  // run_em_device, uploaded once; nullptr goes back to the uniform start.  Bootstraps ignore them.
  void set_priors(const double* priors);
  bool has_priors() const { return has_priors_; }

  // Same result on the EM matrices run_em_device left on the device (no EC table on the host, no second set-up);
  // the B problems are solved `chunk` at a time so that their alpha / norm vectors stay in L2.  ms_out (optional):
  // {resample ms, EM ms} measured with CUDA events.
  std::vector<int> run_bootstrap_device(const std::vector<double>& fl_trunc, uint64_t seed, int B, std::vector<double>& alpha_out,
                                        std::vector<uint32_t>* samples_out = nullptr, double* ms_out = nullptr);
  bool dev_problem_valid() const { return dev_problem_valid_; }
  // Run on a caller-provided stream (e.g. the framework's current stream) instead of the run's own.
  void set_stream(cudaStream_t st);
  // Per-kernel device time, measured with CUDA events on the launching stream.
  struct Timings { double match_ms = 0, resolve_ms = 0, pack_ms = 0; uint64_t match_launches = 0, resolve_launches = 0; };
  void enable_timing(bool on) { timing_ = on; }
  Timings timings();

  Index& index() { return ix_; }
  const QuantOptions& options() const { return opt_; }
  cudaStream_t stream() const { return stream_; }
  double last_em_seconds = 0, last_prep_seconds = 0, last_bs_resample_ms = 0, last_bs_em_ms = 0;
  uint64_t n_kernel_launches = 0;   // launches of this library's own kernels by this run (CUB's are not counted)
  int last_em_comp_blocks = 0;      // last single-problem EM: blocks of em_component_kernel, 0 for the grid-wide kernels
  bool last_em_comp_resident = false;   // ... and whether that kernel held the entries in shared memory
  // filled by run_em_device
  bool dev_stats_valid_ = false, dev_problem_valid_ = false;
  uint32_t dev_n_multi_ = 0;
  uint64_t dev_n_ecs_ = 0, dev_nnz_ = 0, dev_pseudoaligned_ = 0, dev_unique_ = 0;

 private:
  // `in`: the batch's input and layout, the fields of BatchArgs its caller fills (kernels.hpp); run_batch fills the rest
  void run_batch(BatchArgs in, uint32_t n_reads, uint32_t max_read_len);
  // A host batch on the device: per file, its bases, its offsets (nullptr without) and its longest read.
  struct Staged {
    const uint8_t* bases[4];
    const uint32_t* off[4];
    uint32_t maxlen[4];
  };
  // The one host-to-device copy of reads: the files k < nf of a batch of n reads each (bases [0, offs[k][n]), or
  // n x fixed_len without offsets, since offsets are positions in bases[k] and need not start at 0) into staging slot s
  // on copy_stream_, after the kernels that last read the slot (ev_done_[s]); the run's stream waits for the copy
  // (ev_copied_[s]).  A buffer that is too small is reallocated to at least min_bases / min_offs.
  Staged stage(int s, int nf, const char* const* bases, const uint32_t* const* offs, uint32_t n, uint32_t fixed_len,
               uint64_t min_bases, size_t min_offs);
  // pseudoalign_host (nf = 1: one buffer of n reads) and pseudoalign_host_pe (nf = 2: one buffer of n reads per mate)
  // after their checks
  void pseudoalign_staged(int nf, const char* const* bases, const uint32_t* const* offs, uint32_t n, uint32_t fixed_len,
                          int32_t* handles_out);
  void check_device_errors();
  // Makes the run's stream wait for the batches enqueued on the internal streams since the last join.  Every entry point
  // that reads or changes run state on the run's stream calls it first.
  void join();
  // The one EC numbering of every path: the used sets, ids in order of first occurrence, with their handles, counts,
  // lengths and table offsets in emws_.  Synchronises the stream.
  EcNumbering number_ecs();
  void apply_l2_window();
  uint32_t bus_core(const uint8_t* const* db, const uint32_t* const* dofs, uint32_t n_sets, uint32_t maxlen);
  // bus_core up to the records: read-set fields and pseudoalignment of a batch whose first read set has the index
  // `base` (the dictionary's first-occurrence keys) and the read number `set_base` (--num); returns the set handles
  const int32_t* bus_enqueue(const uint8_t* const* db, const uint32_t* const* dofs, uint32_t n_sets, uint32_t maxlen,
                             uint64_t base, uint64_t set_base);
  // the host batch staged for bus_enqueue (slot 0: the bus paths do not overlap batches); returns its longest cDNA read
  uint32_t bus_stage(const char* const* bases, const uint32_t* const* offs, uint32_t n_sets, Staged& g);

  Index& ix_;
  QuantOptions opt_;
  cudaStream_t stream_ = nullptr;
  bool own_stream_ = true;
  // batch i runs on bstream_[i & 1] with BatchWs::slot[i & 1]: forked from stream_ by ev_fork_, stream_ waits for its
  // input to be read (ev_packed_) and, at the next join(), for all of it (ev_last_)
  cudaStream_t bstream_[2] = {nullptr, nullptr};
  cudaEvent_t ev_fork_ = nullptr, ev_packed_[2] = {nullptr, nullptr}, ev_last_[2] = {nullptr, nullptr};
  uint64_t n_batches_ = 0;
  int last_slot_ = 0;
  bool pending_ = false;      // batches enqueued since the last join()
  bool timing_ = false;
  std::vector<cudaEvent_t> events_;   // triples
  Timings tacc_;
  DevDict dd_{};
  // run state on the device
  DBuf<uint32_t> pool_;
  DBuf<Memo2Entry> m2_;
  DBuf<unsigned long long> dslots_, first_, mn_key_, counters_;   // counters_: pool_top, tpool_top, stats[4], one 128-byte line each
  DBuf<uint32_t> count_, tpool_;
  DBuf<int32_t> mn_val_;
  DBuf<int> error_;
  // batch staging
  BatchWs* bws_ = nullptr;
  bool own_ws_ = false;
  cudaStream_t copy_stream_ = nullptr;
  cudaEvent_t ev_copied_[2] = {nullptr, nullptr}, ev_done_[2] = {nullptr, nullptr};
  int stage_idx_ = 0;
  uint32_t n_resolve_warps_ = 0, scratch_stride_ = 0, resolve_group_ = 32;
  uint32_t* h_off_pinned_ = nullptr;
  // host-side run state
  uint64_t n_frag_total_ = 0;
  std::vector<uint32_t> flens_;
  uint32_t tlencount_ = 0;
  std::vector<uint16_t> tl_list_;        // the samples behind flens_, in read order (shipped to rank 0 by merge_to_root)
  uint64_t frag_base_ = 0;
  bool have_frag_base_ = false;
  std::vector<uint16_t> h_tl_;
  EcTable ecs_;
  bool ecs_valid_ = false;
  DBuf<double> priors_;
  bool has_priors_ = false;
  struct EmWs* emws_ = nullptr;
  // bus mode
  DBuf<uint8_t> bus_skip_, bus_notag_;
  DBuf<uint32_t> bus_flags_, bus_hist_, bus_isnew_, bus_newrank_, bus_ismapped_, bus_rank_;
  DBuf<unsigned long long> bus_bc_, bus_umi_, bus_nvalid_;
  DBuf<int32_t> bus_idof_;
  DBuf<BusRecord> bus_rec_;
  DBuf<uint8_t> bus_tmp_;
  uint32_t exp_n_ = 0, exp_nnz_ = 0;
  DBuf<uint32_t> lm_off_, lm_tids_, lm_counts_;       // merge_local: receive area on the root
  DBuf<unsigned long long> lm_first_;
  uint32_t bus_next_id_ = 0;
  uint64_t bus_valid_total_ = 0, bus_sample_base_ = 0;
  // bus --aa: the frames of a batch (6 per read set), frame 0's first hit per set, the sets' handles, the clash count
  bool aa_ = false;
  DBuf<uint8_t> cfc_b_, cfc_tmp_;
  DBuf<uint32_t> cfc_o_, cfc_set_off_, cfc_first_;
  DBuf<int32_t> cfc_handles_;
  DBuf<unsigned long long> cfc_clashes_;
  // bus group member: the submitted batch's set handles and size, its new sets as CSR (grp_len_ / grp_eoff_: per
  // fragment, grp_off_ / grp_tid_: per new set), the run-wide ids of those sets, and the batch's totals (pinned:
  // n_new, total ids, records, valid sets, long barcodes)
  bool grp_pending_ = false;
  const int32_t* grp_handles_ = nullptr;
  uint32_t grp_n_ = 0;
  DBuf<uint32_t> grp_len_, grp_eoff_, grp_off_, grp_tid_;
  DBuf<int32_t> grp_gid_;
  unsigned long long* h_grp_ = nullptr;
};

// `bus --devices` (kb_bus_group_*): several bus runs, each on its own index replica, fed batches of one read stream,
// whose records carry one run-wide EC numbering -- the ids of a single run fed the whole stream.  Batches complete in
// the order they were submitted; each member's new sets are committed to a content-keyed registry (transcript list ->
// id) on the host: a known set keeps its id, an unknown one takes the next.  One host thread drives a group.
class BusGroup {
 public:
  explicit BusGroup(std::vector<Quant*> members);
  // returns the batch's ticket; the host buffers may be reused on return
  uint64_t submit(int member, const char* const* bases, const uint32_t* const* offs, uint32_t n_sets);
  // the oldest outstanding batch (ticket must name it): its records with run-wide EC ids
  void complete(uint64_t ticket, BusRecord* records_out, uint32_t* n_records_out);
  void begin_sample(uint64_t barcode);
  size_t outstanding() const { return queue_.size(); }
  uint64_t n_sets_total() const { return n_sets_total_; }
  // the run-wide table, ids in order; counts summed over the members (refreshed by every call)
  const EcTable& ec_table();
  Stats stats();
  int n_members() const { return (int)m_.size(); }
  Quant& member(int i) { return *m_[i]; }

 private:
  struct VecHash {
    size_t operator()(const std::vector<uint32_t>& v) const {
      uint64_t h = 1469598103934665603ULL ^ v.size();
      for (uint32_t x : v) h = (h ^ x) * 1099511628211ULL;
      return (size_t)h;
    }
  };
  std::vector<Quant*> m_;
  std::vector<int> queue_;          // members of the outstanding batches, oldest first
  std::vector<bool> busy_;
  uint64_t next_ticket_ = 0, done_tickets_ = 0, n_sets_total_ = 0, sample_base_ = 0;
  std::unordered_map<std::vector<uint32_t>, int32_t, VecHash> reg_;
  EcTable table_;                   // off / tid in id order; count filled by ec_table()
};

std::vector<double> mean_fl_trunc_of(const uint32_t* flens /* 1000 */, double fld_mean, double fld_sd);

// `kallisto quant-tcc` (src/main.cpp:2802-3220): one EM per sample (row of a transcript-compatibility-count matrix) over
// one shared equivalence-class table (the lines of matrix.ec), on the device in chunks of samples.
struct TccInput {
  uint32_t n_ecs = 0;
  const uint64_t* ec_off = nullptr;     // n_ecs + 1
  const uint32_t* tids = nullptr;       // sorted transcript ids of every EC
  uint32_t n_samples = 0;
  const uint64_t* row_off = nullptr;    // n_samples + 1 offsets into ec_ids / counts
  const uint32_t* ec_ids = nullptr;
  const uint32_t* counts = nullptr;
  const double* eff_lens = nullptr;     // n_targets, or n_samples x n_targets when per_sample_eff
  bool per_sample_eff = false;
  // gene-level output (-g / -G): the gene of every target (-1: none), genes 0 .. n_genes - 1.  n_genes == 0: none is
  // computed and nothing for it is allocated.
  const int32_t* gene_of = nullptr;
  uint32_t n_genes = 0;
  // --priors: the start of every sample's EM (n_targets values, host), nullptr for the uniform start.  tcc_bootstrap
  // ignores it: bootstraps start uniform, as the reference's do.
  const double* priors = nullptr;
};
// gene_counts_out / gene_tpm_out (n_samples x n_genes) are filled when in.n_genes > 0.
std::vector<int> tcc_run(Index& ix, const TccInput& in, std::vector<double>& alpha_out /* n_samples x n_targets */,
                         std::vector<double>* gene_counts_out = nullptr, std::vector<double>* gene_tpm_out = nullptr);
// The B bootstraps of every sample (src/main.cpp:3109-3178), problem g = sample * B + b, handed to `sink` chunk by chunk
// in order: (first problem, count, est_counts count x n_targets, rounds, resampled counts count x n_ecs or nullptr,
// gene counts and gene TPM count x n_genes or nullptr without genes).  Host memory is bounded by one chunk, whatever
// n_samples x B.
using TccBootstrapSink = std::function<void(uint64_t first, uint32_t count, const double* est, const int* rounds,
                                            const uint32_t* samples, const double* gene_counts, const double* gene_tpm)>;
void tcc_bootstrap(Index& ix, const TccInput& in, uint64_t seed, int B, bool want_samples, const TccBootstrapSink& sink);

}  // namespace kb
