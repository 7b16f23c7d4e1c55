/* kallisto_b200 -- C ABI of the H100-native `kallisto quant` / `kallisto bus` hot path.
 *
 * kallisto (the reference, /root/reference) has no plugin or FFI layer: the hot path sits between
 * its CLI, its index file and its output files (SURVEY.md section 8b).  This header is the boundary a
 * maintainer would bind to from the reference's own C++ (see INTEGRATION.md): every entry point
 * names the reference function whose work it takes over.  Plain pointers and sizes only; all
 * buffers are caller-allocated HOST memory unless the name says `_device`; opaque handles are
 * freed with the matching `_free`.  Every function returns 0 on success and a negative code on
 * failure; kb_last_error() then returns a message for the calling thread.  There is no CPU
 * implementation behind any of these calls: without a CUDA device they fail with KB_ERR_NO_DEVICE.
 */
#ifndef KALLISTO_B200_H
#define KALLISTO_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define KB_OK 0
#define KB_ERR_INVALID (-1)   /* bad argument */
#define KB_ERR_INDEX (-2)     /* unreadable / unsupported index file */
#define KB_ERR_NO_DEVICE (-3) /* no CUDA device: there is no CPU path */
#define KB_ERR_CUDA (-4)      /* CUDA runtime or device-side failure */
#define KB_ERR_IO (-5)        /* file could not be read or written */

typedef struct kb_index kb_index; /* KmerIndex after load(), resident in HBM */
typedef struct kb_quant kb_quant; /* MinCollector + MasterProcessor state of one run */

const char* kb_last_error(void);
const char* kb_version(void);

/* ---- index: replaces KmerIndex::load (src/KmerIndex.cpp:1330-1559) ---------------------------
 * Reads an index file written by the reference `kallisto index` (format v13), flattens the
 * compacted de Bruijn graph + mosaic equivalence classes and builds the k-mer table on the
 * device.  load_positions != 0 keeps per-transcript positions (needed only by single-end quant
 * without --single-overhang, KmerIndex.h:78). */
int kb_index_load(const char* path, int device, int load_positions, int threads, kb_index** out);
void kb_index_free(kb_index* ix);

typedef struct kb_index_info {
  int32_t k;
  uint32_t n_targets;
  uint32_t n_unitigs;
  uint32_t n_ec_blocks;
  uint32_t n_ec_sets;      /* distinct transcript sets among the blocks */
  uint64_t n_kmers;        /* "[index] number of k-mers" */
  uint64_t table_slots;    /* capacity of the device k-mer table (32 B per slot) */
  double load_seconds;     /* file parse */
  double build_seconds;    /* device upload + table build */
} kb_index_info;
int kb_index_get_info(const kb_index* ix, kb_index_info* info);
/* Host-only: parse the file and report its sizes without touching a device (tooling, CI). */
int kb_index_inspect(const char* path, kb_index_info* info);
/* target_names_ / target_lens_ (src/KmerIndex.h:136-138) */
const char* kb_index_target_name(const kb_index* ix, uint32_t i);
int kb_index_target_lens(const kb_index* ix, uint32_t* lens_out /* n_targets */);

/* ---- a quantification run ------------------------------------------------------------------- */
typedef struct kb_quant_opts {
  int32_t paired;            /* 1: reads come as interleaved mate pairs (kallisto quant default); 0: --single */
  int32_t strand_mode;       /* 0 unstranded, 1 --fr-stranded, 2 --rf-stranded (ProgramOptions::StrandType) */
  int32_t collect_fld;       /* 1: estimate the fragment-length distribution from the first 10000 unique pairs */
  uint32_t max_batch_reads;  /* largest batch (reads) that will be submitted; 0 = default (4 Mi) */
  uint64_t max_batch_bases;  /* largest batch (bases); 0 = default (512 Mi) */
  int32_t single_overhang;   /* --single-overhang: skip the fragment-position filter (ProcessReads.cpp:1095-1136) */
  double fld_mean;           /* -l (0 = not given); with !single_overhang the filter runs for single-end reads and for
                                pairs with one mate mapped, and needs an index loaded with load_positions = 1 */
} kb_quant_opts;
int kb_quant_create(kb_index* ix, const kb_quant_opts* opts, kb_quant** out);
void kb_quant_free(kb_quant* q);

/* Replaces ReadProcessor::processBuffer (src/ProcessReads.cpp:968-1237) for one batch of parsed
 * reads, i.e. per fragment KmerIndex::match x2 (src/KmerIndex.cpp:1698-1940) +
 * MinCollector::intersectKmers (src/MinCollector.cpp:160-218) + [doStrandSpecificity] + the
 * ecmapinv lookup / count (ProcessReads.cpp:1148-1161) + KmerIndex::mapPair fragment-length
 * sampling (1174-1181).
 *   bases    concatenated ASCII read sequences (as in the reference's `seqs` buffer, without the NULs)
 *   offsets  n_reads + 1 offsets into bases, or NULL if every read has exactly fixed_len bases
 *   n_reads  reads in the batch; mates interleaved (r1,r2,r1,r2,...) when the run is paired
 *   ec_out   optional: one int32 per fragment, an opaque set handle >= 0, or -1 if not pseudoaligned
 *            (translate with kb_quant_ec_table after the run)
 * Host buffers; the host->device copy, the kernels and the copy back are all inside the call. */
int kb_pseudoalign_batch(kb_quant* q, const char* bases, const uint32_t* offsets, uint32_t n_reads,
                         uint32_t fixed_len, int32_t* ec_out);
/* Paired batch with one buffer per mate, as a FASTQ reader produces them (R1 and R2 parsed
 * separately, FastqSequenceReader::fetchSequences, src/ProcessReads.cpp:3128-3267): n_pairs
 * fragments, offsetsN with n_pairs + 1 entries each (or both NULL with fixed_len). */
int kb_pseudoalign_batch_pe(kb_quant* q, const char* bases1, const uint32_t* offsets1, const char* bases2,
                            const uint32_t* offsets2, uint32_t n_pairs, uint32_t fixed_len, int32_t* ec_out);
/* Page-locked host memory for batch buffers (so that the copies inside kb_pseudoalign_batch* run at
 * full PCIe speed without the caller linking against CUDA). */
void* kb_host_alloc(size_t bytes);
void kb_host_free(void* p);
/* Same with DEVICE pointers (inputs already resident in HBM); asynchronous on the run's stream.  The kernels run on
 * the run's internal streams, two batches at a time; the run's stream waits only until the inputs have been read, so
 * the caller may overwrite them in that stream's order.  Everything that reads results waits for the batches. */
int kb_pseudoalign_batch_device(kb_quant* q, const void* d_bases, const uint32_t* d_offsets, uint32_t n_reads,
                                uint32_t fixed_len, uint32_t max_read_len);
int kb_quant_sync(kb_quant* q);
/* Run the kernels of this run on the caller's CUDA stream (cudaStream_t) instead of a private one. */
int kb_quant_set_stream(kb_quant* q, void* cuda_stream);
/* Per-kernel device time measured with CUDA events on the launching stream (for the roofline). */
typedef struct kb_kernel_timings {
  double match_ms, resolve_ms, em_ms, em_prep_ms;
  uint64_t match_launches, resolve_launches;
  uint64_t kernel_launches;   /* launches of the library's own kernels by this run so far (pack, match, resolve,
                                 fld, EC numbering / CSR / CSC construction, EM); CUB sort/scan launches not counted */
  double bs_resample_ms, bs_em_ms;   /* last kb_bootstrap_run: multinomial resampling, batched EM (CUDA events) */
  double pack_ms;             /* pack_kernel (+ dlist_scan_kernel with a D-list index), same launches as match_ms */
  uint64_t em_comp_blocks;    /* last single-problem EM: blocks of the per-component kernel, 0 for the grid-wide kernel */
  uint64_t em_comp_resident;  /* ... 1 when that kernel held the entries in shared memory, 0 when it streamed them */
} kb_kernel_timings;
int kb_quant_enable_timing(kb_quant* q, int on);
int kb_quant_get_timings(kb_quant* q, kb_kernel_timings* out);

/* Replaces MasterProcessor::update + the tail flush + MinCollector::increaseCount
 * (src/ProcessReads.cpp:323-334,424-483; src/MinCollector.cpp:251-269): equivalence classes in
 * order of first occurrence (the ids the reference assigns with -t 1), their transcript sets and counts. */
typedef struct kb_run_stats {
  uint64_t n_processed, n_pseudoaligned, n_unique;
  uint64_t n_ecs, n_ec_entries;
  uint64_t n_probes;        /* k-mer table lookups executed (dbg.find equivalents) */
  uint64_t n_slot_visits;   /* 32-byte slots touched by those lookups */
  uint64_t n_resolved;      /* fragments finished by the warp-level intersection kernel */
  uint64_t n_memo_hits;
} kb_run_stats;
int kb_quant_finalize(kb_quant* q, kb_run_stats* stats);
int kb_quant_ec_table(kb_quant* q, uint64_t* ec_offsets /* n_ecs+1 */, uint32_t* tids /* n_ec_entries */,
                      uint32_t* counts /* n_ecs */, int32_t* handles /* n_ecs, may be NULL */);
/* tc.flens (fragment-length histogram, 1000 bins) */
int kb_quant_get_flens(kb_quant* q, uint32_t* flens_out);
int kb_quant_set_flens(kb_quant* q, const uint32_t* flens_in);

/* ---- multi-GPU: reads are sharded across ranks (one kb_quant per GPU, index replicated); before the
 * single EM the per-rank equivalence classes are merged by CONTENT on one rank -- the multi-rank
 * form of MasterProcessor::update's merge under writer_lock (src/ProcessReads.cpp:424-483).
 * export: number this rank's ECs and copy them into caller-provided DEVICE buffers (which the caller
 * moves with NCCL): off[n_sets+1], tids[n_entries], counts[n_sets], first[n_sets] (fragment index of
 * first occurrence).  import: fold such a table into this run's dictionary; first_offset orders the
 * ranks' fragment indices (rank r: r << 40), n_processed adds the other rank's fragment count. */
int kb_quant_export_prepare(kb_quant* q, uint32_t* n_sets, uint32_t* n_entries);
int kb_quant_export_device(kb_quant* q, uint32_t* d_off, uint32_t* d_tids, uint32_t* d_counts, uint64_t* d_first);
int kb_quant_import_device(kb_quant* q, uint32_t n_sets, const uint32_t* d_off, const uint32_t* d_tids,
                           const uint32_t* d_counts, const uint64_t* d_first, uint64_t first_offset, uint64_t n_processed);

/* The same exchange as ONE collective call in C++ over NCCL (csrc/comm.cu) -- what `kallisto_b200 quant --devices`
 * and bench.py use.  Every rank calls kb_quant_merge_nccl after its last batch: a 4-word meta record per rank is
 * all-gathered, ranks != 0 ncclSend their tables (and their ordered fragment-length samples) to rank 0, which
 * folds all of them into its dictionary by content with one kernel launch and completes the fragment-length
 * histogram in rank order (first 10000 unique pairs of the whole input, ProcessReads.cpp:985-1004).  Afterwards
 * rank 0 runs kb_em_run.  first_stride: rank r's first-occurrence keys are offset by r * first_stride (ranks own
 * consecutive slices of the input); 0 if the runs were fed global fragment indices (kb_quant_set_frag_base).
 * NCCL is bound at run time (libnccl.so.2); the id is the 128-byte ncclUniqueId, created on rank 0 and
 * distributed by the caller (torch.distributed / MPI / a file). */
typedef struct kb_comm kb_comm;
int kb_comm_unique_id(void* id_out /* 128 bytes */);
int kb_comm_create(int n_ranks, int rank, const void* id /* 128 bytes */, int device, kb_comm** out);
/* Wrap an existing ncclComm_t (not destroyed by kb_comm_free). */
int kb_comm_create_from_nccl(void* nccl_comm, int n_ranks, int rank, int device, kb_comm** out);
/* One process driving several GPUs (one host thread per GPU): ncclCommInitAll. out[] receives n_devices handles. */
int kb_comm_create_all(const int* devices, int n_devices, kb_comm** out);
/* Rank 0: size the receive area ahead of time (sets / entries expected per peer). */
int kb_comm_reserve(kb_comm* c, uint64_t n_sets_per_rank, uint64_t n_entries_per_rank);
void kb_comm_free(kb_comm* c);
int kb_quant_merge_nccl(kb_quant* q, kb_comm* c, uint64_t first_stride, uint64_t* n_processed_total);
/* The same merge when all runs belong to THIS process (one host thread per GPU or one thread driving all): the other
 * runs' tables are copied to the root's device with cudaMemcpyPeerAsync (NVLink) and folded in by content; no
 * communicator.  The runs must have been fed global fragment indices (kb_quant_set_frag_base) and only the root
 * collects the fragment-length distribution. */
int kb_quant_merge_local(kb_quant* root, kb_quant* const* others, int32_t n_others, uint64_t* n_processed_total);
/* Global index of the first fragment of the NEXT batch (several runs fed from one read stream). */
int kb_quant_set_frag_base(kb_quant* q, uint64_t base);
/* Size the EC-numbering / EM workspace ahead of time (kb_quant_create reserves for 2x the index's own EC sets). */
int kb_quant_reserve(kb_quant* q, uint64_t n_ecs, uint64_t n_ec_entries);

/* Replaces compute_mean_frag_lens_trunc / init_mean_fl_trunc + get_frag_len_means + calc_eff_lens +
 * calc_weights + EMAlgorithm::run(10000, 50) (src/MinCollector.cpp:629-651, src/weights.cpp,
 * src/EMAlgorithm.h:95-221).  fld_mean == 0 uses the estimated distribution, otherwise the
 * truncated Gaussian of -l/-s.  Outputs have n_targets entries. */
int kb_em_run(kb_quant* q, double fld_mean, double fld_sd, double* est_counts_out, double* eff_lens_out,
              int32_t* rounds_out, double* seconds_out);
/* Same, on an explicit EC table (e.g. the table merged across ranks). */
int kb_em_run_table(kb_quant* q, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids,
                    const uint32_t* counts, double fld_mean, double fld_sd, double* est_counts_out,
                    double* eff_lens_out, int32_t* rounds_out, double* seconds_out);

/* --priors (EMAlgorithm::read_priors, src/EMAlgorithm.h:52-81).  Host-only.  Reads one value per line with std::stod
 * (leading blanks skipped, anything after the number ignored) and sums them in file order.  A sum >= 1 + 1e-3 means
 * raw counts: each value becomes (value + 1) / (sum + n).  Otherwise the values are returned as they are.
 * Two calls: with out == NULL or cap < n only *n_out is set.  Returns KB_ERR_IO when the file cannot be opened and
 * KB_ERR_INVALID when a line is not a number std::stod accepts (kb_last_error() names the line). */
int kb_read_priors(const char* path, double* out, uint64_t cap, uint64_t* n_out);
/* EMAlgorithm::set_priors (src/EMAlgorithm.h:83-93): every later kb_em_run / kb_em_run_table of q starts from these
 * n == n_targets values instead of the uniform 1 / n_targets (the values are copied).  Any other n returns
 * KB_ERR_INVALID and changes nothing; priors == NULL goes back to the uniform start.  kb_bootstrap_run always starts
 * uniform, as the reference's bootstraps do. */
int kb_em_set_priors(kb_quant* q, const double* priors, uint32_t n);

/* Replaces the bootstrap loop of main.cpp:2743-2782 (seeds from mt19937_64(seed); per bootstrap
 * Multinomial::sample + Bootstrap::run_em).  est_counts_out is n_bootstrap x n_targets, row-major;
 * samples_out (optional) n_bootstrap x n_ecs resampled counts; rounds_out (optional) n_bootstrap. */
int kb_bootstrap_run(kb_quant* q, double fld_mean, double fld_sd, uint64_t seed, int32_t n_bootstrap,
                     double* est_counts_out, uint32_t* samples_out, int32_t* rounds_out);

/* ---- `kallisto quant-tcc` (src/main.cpp:2802-3220): one EM per sample (row of a transcript-compatibility-count matrix)
 * over ONE shared equivalence-class table (the lines of matrix.ec, EC id = line number), batched on the device; a
 * sample's weights are its own counts / eff_len (calc_weights, src/weights.cpp:220-246).  The TCC matrix comes as
 * CSR (row_offsets / ec_ids / counts); eff_lens has n_targets entries, or n_samples x n_targets with
 * per_sample_eff != 0 (one fragment-length distribution per sample).  est_counts_out: n_samples x n_targets. */
int kb_tcc_run(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids, uint32_t n_samples,
               const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts, const double* eff_lens,
               int32_t per_sample_eff, double* est_counts_out, int32_t* rounds_out);
/* Bootstraps of quant-tcc (src/main.cpp:3109-3178): n_bootstrap per sample, each the sample's counts resampled
 * (Multinomial::sample with the seeds of mt19937_64(seed), the same seeds for every sample) and run through the EM with
 * the sample's ORIGINAL counts / eff_len as weights.  Problem g = sample * n_bootstrap + b.  The results are handed to
 * `cb` in chunks, in order: problems first .. first + count - 1, est_counts (count x n_targets, row-major), rounds
 * (count) and, when want_samples != 0, the resampled counts (count x n_ecs); the pointers are valid during the call
 * only.  A non-zero return from cb stops the run (KB_ERR_INVALID).  Arguments as kb_tcc_run, except that the EC ids
 * of a row must be strictly increasing; a row's total count must fit an int32. */
typedef int (*kb_tcc_bootstrap_cb)(void* user, uint64_t first, uint32_t count, const double* est_counts,
                                   const int32_t* rounds, const uint32_t* samples);
int kb_tcc_bootstrap_run(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids, uint32_t n_samples,
                         const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts, const double* eff_lens,
                         int32_t per_sample_eff, uint64_t seed, int32_t n_bootstrap, int32_t want_samples,
                         kb_tcc_bootstrap_cb cb, void* user);
/* Gene-level output of quant-tcc (-g / -G; src/main.cpp:3026-3058, plaintext_writer_gene src/PlaintextWriter.cpp:67-112),
 * summed on the device.  gene_of_target (n_targets) is the gene of every target, -1 for none; genes are 0 .. n_genes - 1.
 * For every problem, tpm = counts_to_tpm(est_counts, eff_lens); every target with est_counts > 0, in increasing id, adds
 * its est_counts to its gene's count and its tpm to its gene's TPM.  The values equal the reference's bit for bit.
 * kb_tcc_run_genes = kb_tcc_run plus gene_counts_out and gene_tpm_out (n_samples x n_genes each, row-major).
 * kb_tcc_bootstrap_run_genes = kb_tcc_bootstrap_run, with the bootstraps' gene counts and gene TPM (count x n_genes each,
 * computed with the eff_lens of the problem's sample) handed to cb next to est_counts.  With n_genes == 0 both behave
 * as kb_tcc_run / kb_tcc_bootstrap_run (gene_of_target may be NULL; cb gets NULL gene arrays). */
int kb_tcc_run_genes(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids, uint32_t n_samples,
                     const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts, const double* eff_lens,
                     int32_t per_sample_eff, const int32_t* gene_of_target, uint32_t n_genes, double* est_counts_out,
                     int32_t* rounds_out, double* gene_counts_out, double* gene_tpm_out);
/* kb_tcc_run_genes with --priors (src/main.cpp:2984-2987,3019): every sample's EM starts from priors (n_targets values)
 * instead of the uniform 1 / n_targets; priors == NULL is kb_tcc_run_genes.  The bootstrap entry points take no priors:
 * bootstraps start uniform. */
int kb_tcc_run_priors(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids, uint32_t n_samples,
                      const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts, const double* eff_lens,
                      int32_t per_sample_eff, const int32_t* gene_of_target, uint32_t n_genes, const double* priors,
                      double* est_counts_out, int32_t* rounds_out, double* gene_counts_out, double* gene_tpm_out);
typedef int (*kb_tcc_bootstrap_genes_cb)(void* user, uint64_t first, uint32_t count, const double* est_counts,
                                         const int32_t* rounds, const uint32_t* samples, const double* gene_counts,
                                         const double* gene_tpm);
int kb_tcc_bootstrap_run_genes(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids,
                               uint32_t n_samples, const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts,
                               const double* eff_lens, int32_t per_sample_eff, const int32_t* gene_of_target, uint32_t n_genes,
                               uint64_t seed, int32_t n_bootstrap, int32_t want_samples, kb_tcc_bootstrap_genes_cb cb,
                               void* user);
/* mean_fl_trunc -> eff_lens exactly as the reference forms them (get_frag_len_means + calc_eff_lens, src/weights.cpp:7-28,
 * 58-79): fld_mean > 0: truncated Gaussian (-l/-s); else the histogram flens[1000]; both 0/NULL: eff_len = 1 for every
 * target (quant-tcc without fragment-length information).  Host arithmetic. */
int kb_eff_lens(const kb_index* ix, const uint32_t* flens, double fld_mean, double fld_sd, double* eff_lens_out,
                double* mean_fl_out, double* sd_fl_out);

/* ---- `kallisto bus`: replaces BUSProcessor::processBuffer (src/ProcessReads.cpp:1380-1832) + the
 * record writing / EC id assignment of MasterProcessor::update (:603-624) ------------------------ */
typedef struct kb_bus_substr { int32_t fileno, start, stop; } kb_bus_substr;   /* BUSOptionSubstr, src/common.h:29-36 */
typedef struct kb_bus_opts {
  int32_t nfiles;                 /* files per read set (technology), <= 4 */
  int32_t n_bc;  kb_bus_substr bc[4];    /* n_bc == 0: no barcode (fake barcode of 16 A, or the sample of kb_bus_begin_sample) */
  int32_t n_umi; kb_bus_substr umi[4];   /* n_umi == 1 and umi[0].fileno == -1: no UMI ("bulk_like", src/ProcessReads.cpp:1393):
                                          * the records carry UMI = ~0 */
  kb_bus_substr seq;              /* the read that is pseudoaligned; stop must be 0 (to the end of the read) */
  int32_t strand_mode;            /* 0 unstranded, 1 --fr-stranded (default of the 10x technologies), 2 --rf-stranded */
  int32_t num;                    /* --num: flags = read number */
  uint32_t max_batch_sets;        /* 0 = default */
  uint64_t max_batch_bases;
  int32_t paired;                 /* busopt.paired (src/main.cpp:1366-1395,1424-1426; `bus -x BULK --paired`): seq and seq2 are
                                   * pseudoaligned as a pair (match x 2 + intersectKmers + mapPair, :1646-1650,1747-1756);
                                   * the fragment-length histogram is read with kb_quant_get_flens */
  kb_bus_substr seq2;             /* second sequence read when paired; stop must be 0 */
  const char* tag;                /* UMI tag sequence (`--tag`, SMARTSEQ3: "ATTGCGCAATG"; src/main.cpp:1447-1475,
                                   * src/ProcessReads.cpp:1497-1530) or NULL.  umi[0] must then cover tag + UMI, as the user
                                   * of the reference gives it; a read set whose UMI is not preceded by the tag (one mismatch
                                   * allowed when it is longer than 5) is an internal read: UMI ~0, the sequence starts where
                                   * the tag would have, no strand filter, and only those sample fragment lengths. */
} kb_bus_opts;
typedef struct kb_bus_record {    /* BUSData, src/BUSData.h:30-38: 32 bytes, as written to output.bus */
  uint64_t barcode, umi;
  int32_t ec;
  uint32_t count, flags, pad;
} kb_bus_record;
int kb_bus_create(kb_index* ix, const kb_bus_opts* opts, kb_quant** out);
/* One batch of read sets: bases[f] / offsets[f] (n_sets + 1 entries) for each file f of the technology.
 * records_out (capacity n_sets) receives one record per pseudoaligned set, in read order, with final
 * EC ids (order of first occurrence = the ids of the reference with -t 1). */
int kb_bus_batch(kb_quant* q, const char* const* bases, const uint32_t* const* offsets, uint32_t n_sets,
                 kb_bus_record* records_out, uint32_t* n_records_out);
/* Same with the files of the batch already resident in DEVICE memory (offsets too); the records stay on the device:
 * *d_records_out points to n_records records, valid until the next batch.  max_seq_len = longest read of the
 * sequence file in the batch. */
int kb_bus_batch_device(kb_quant* q, const void* const* d_bases, const uint32_t* const* d_offsets, uint32_t n_sets,
                        uint32_t max_seq_len, uint32_t* n_records_out, const kb_bus_record** d_records_out);
/* Batch mode (`kallisto bus -x BULK` or `--batch`: one sample per file set, src/ProcessReads.cpp:371-404): the read sets
 * of the following batches belong to the sample `barcode`.  Without a barcode read (n_bc == 0) it is their records' fake
 * barcode (BUSProcessor writes binaryToString(batch_id_mapping[id], 16), :1603-1607; pass 0 for the 16 x 'A' of a
 * technology run without --batch-barcodes).  With a barcode read it goes in front of the barcode when batch barcodes are
 * on (kb_bus_set_batch_barcodes), and is unused otherwise.  The fragment-length sampling restarts from an empty
 * histogram (batchFlens[id] / tlencounts[id], :486-493) -- read the finished sample's with kb_quant_get_flens first --
 * and --num read numbers start again from 0. */
int kb_bus_begin_sample(kb_quant* q, uint64_t barcode);
/* `kallisto bus --batch --batch-barcodes` (src/ProcessReads.cpp:1617-1626): on != 0 gives every record of a technology
 * with a barcode read of blen <= 32 letters the barcode binaryToString(sample, 32 - blen) + the barcode (an N read as G),
 * with no N flag in the barcode half of the flags, nor in the UMI half where it repeats the barcode's (no UMI, or a tag).
 * Call before the first batch.  Fails when the technology's fixed barcode pieces exceed 32 letters; kb_bus_batch fails for a batch
 * with a read set whose variable-length barcode exceeds 32 letters (kb_last_error() says so) and returns no records.  Without a barcode read it changes nothing: the barcode is kb_bus_begin_sample's. */
int kb_bus_set_batch_barcodes(kb_quant* q, int32_t on);
/* Observed barcode / UMI length histograms (33 bins), for the header of output.bus
 * (src/main.cpp:2470-2508). */
int kb_bus_lengths(kb_quant* q, uint32_t* bc_hist, uint32_t* umi_hist);
/* `kallisto bus --aa` (src/ProcessReads.cpp:1652-1695, MinCollector::intersectKmersCFC src/MinCollector.cpp:44-119):
 * on != 0 matches every read set's sequence in its six reading frames, translated into comma-free code, against an
 * index built with `kallisto index --aa`; the frame with the smallest non-empty set wins (the lowest frame on a tie), and
 * with a strand mode the set is then filtered by the strand of frame 0's first mapping k-mer.  Call before the first
 * batch.  Fails for a paired technology, a tag sequence and an index with a D-list. */
int kb_bus_set_aa(kb_quant* q, int32_t on);
/* --aa: cardinality_clashes of the run so far ("n_frame_clashes" of run_info.json): per read set, the frames whose set
 * is as small as the smallest one before them. */
int kb_bus_frame_clashes(kb_quant* q, uint64_t* n_out);

/* ---- `kallisto bus --devices`: batches of one read stream dealt to several bus runs (one index replica each, on one GPU
 * or several), with the records and the EC table a single run fed the whole stream would produce.  Every batch is
 * numbered run-wide on its member (first-occurrence keys, --num read numbers); when a batch completes, the sets that
 * were new on its member are committed in order of first occurrence to the group's registry (transcript list -> id): a
 * set the registry knows keeps its id, an unknown one takes the next.  One host thread drives a group; it is not
 * thread-safe.  Refusals return KB_ERR_INVALID. */
typedef struct kb_bus_group kb_bus_group;
/* members: n >= 1 fresh kb_bus_create handles (no batch run yet, none listed twice), with identical kb_bus_opts, --aa and
 * batch-barcode settings, on indices with the same k and target count.  The same device may appear more than once.  The
 * group does not own the members: free it before them. */
int kb_bus_group_create(kb_quant* const* members, int32_t n, kb_bus_group** out);
void kb_bus_group_free(kb_bus_group* g);
/* Stages one batch (as kb_bus_batch) on `member` and enqueues its work; returns once the host buffers may be reused.
 * *ticket numbers the batches of the group in submission order.  A member takes one batch at a time: a member with a
 * batch outstanding is refused. */
int kb_bus_group_submit(kb_bus_group* g, int32_t member, const char* const* bases, const uint32_t* const* offsets,
                        uint32_t n_sets, uint64_t* ticket);
/* Finishes the oldest outstanding batch, whose ticket must be given (any other is refused): records_out (capacity: its
 * n_sets) receives its records, in read order, with run-wide EC ids.  A batch kb_bus_batch would fail (--batch-barcodes
 * with a barcode over 32 letters) fails here. */
int kb_bus_group_complete(kb_bus_group* g, uint64_t ticket, kb_bus_record* records_out, uint32_t* n_records_out);
/* kb_bus_begin_sample on every member, and --num read numbers restart run-wide.  Refused while a batch is outstanding. */
int kb_bus_group_begin_sample(kb_bus_group* g, uint64_t barcode);
/* n_processed, n_pseudoaligned, n_unique and the lookup counters summed over the members; n_ecs / n_ec_entries of the
 * group's numbering. */
int kb_bus_group_finalize(kb_bus_group* g, kb_run_stats* stats);
/* The group's EC table (layout of kb_quant_ec_table, ids in run-wide order), counts summed over the members. */
int kb_bus_group_ec_table(kb_bus_group* g, uint64_t* ec_offsets /* n_ecs+1 */, uint32_t* tids /* n_ec_entries */,
                          uint32_t* counts /* n_ecs */);
/* Barcode / UMI length histograms summed over the members (kb_bus_lengths). */
int kb_bus_group_lengths(kb_bus_group* g, uint32_t* bc_hist, uint32_t* umi_hist);
/* --aa: frame clashes summed over the members (kb_bus_frame_clashes). */
int kb_bus_group_frame_clashes(kb_bus_group* g, uint64_t* n_out);
/* Fragment lengths are those of member 0 (kb_quant_get_flens on it): a driver that wants the first 10000 pairs of each
 * sample gives member 0 the sample's batches until its histogram holds 10000. */

/* Host-only: parse a FASTA/FASTQ file (plain or gzip) with the library's reader (kseq_read grammar,
 * src/kseq.h) and report the number of records, of bases, and an FNV-1a hash of the sequences
 * (0xFF after each record).  Tooling / tests. */
int kb_fastx_summary(const char* path, uint64_t* n_reads, uint64_t* n_bases, uint64_t* fnv1a);
/* Same through the command-line front end's ingest path: with threads > 1 a plain (uncompressed) regular
 * file is mapped and parsed by `threads` host threads (csrc/fastx.hpp: segment starts are guessed, then
 * proven by the parse of the preceding segment), otherwise the sequential zlib reader is used.  The
 * result is the sequential parse in every case (replaces the serial fetchSequences + kseq_read under
 * reader_lock, src/ProcessReads.cpp:945,3128-3267). */
int kb_fastx_summary_mt(const char* path, int threads, uint64_t* n_reads, uint64_t* n_bases, uint64_t* fnv1a);

/* Host-only: decompress a gzip file with the command-line front end's decoder (csrc/fast_inflate.hpp, which
 * stands in for zlib's gzread on the reference's input path, src/common.h:216-225) and report the number of
 * bytes and their CRC-32.  Tooling / tests: the decoder must produce what zlib produces. */
int kb_gz_summary(const char* path, uint64_t* n_bytes, uint32_t* crc32_out);

/* counts_to_tpm (src/PlaintextWriter.cpp:5-27) -- host arithmetic, here so that callers format
 * identical numbers. */
int kb_counts_to_tpm(const double* est_counts, const double* eff_lens, uint32_t n, double* tpm_out);

#ifdef __cplusplus
}
#endif
#endif /* KALLISTO_B200_H */
