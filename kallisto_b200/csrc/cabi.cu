// extern "C" boundary: include/kallisto_b200.h implemented on top of kb::Index / kb::Quant.
#include <cmath>
#include <cstring>
#include <exception>
#include <limits>
#include <string>

#include "../../include/kallisto_b200.h"
#include "engine.hpp"
#include "fastx.hpp"
#include "priors.hpp"

namespace {
thread_local std::string g_err;

int fail(int code, const std::string& msg) {
  g_err = msg;
  return code;
}

template <class F> int guarded(F&& f) {
  try {
    f();
    return KB_OK;
  } catch (const kb::Error& e) {
    const std::string m = e.what();
    int code = KB_ERR_CUDA;
    if (m.find("no CUDA device") != std::string::npos) code = KB_ERR_NO_DEVICE;
    return fail(code, m);
  } catch (const std::bad_alloc&) {
    return fail(KB_ERR_CUDA, "out of host memory");
  } catch (const std::exception& e) {
    return fail(KB_ERR_INDEX, e.what());
  }
}

// guarded, with the refusals of a call's preconditions (std::invalid_argument) returned as KB_ERR_INVALID
template <class F> int guarded_invalid(F&& f) {
  try {
    f();
    return KB_OK;
  } catch (const std::invalid_argument& e) {
    return fail(KB_ERR_INVALID, e.what());
  } catch (...) {
    return guarded([] { throw; });
  }
}
}  // namespace

struct kb_index {
  std::unique_ptr<kb::Index> ix;
};
struct kb_quant {
  std::unique_ptr<kb::Quant> q;
  kb_index* owner;
};
struct kb_bus_group {
  std::unique_ptr<kb::BusGroup> g;
};

extern "C" {

const char* kb_last_error(void) { return g_err.c_str(); }
const char* kb_version(void) { return "kallisto_b200 0.1.0 (reference: kallisto 0.51.1, index format 13)"; }

int kb_index_load(const char* path, int device, int load_positions, int threads, kb_index** out) {
  if (!path || !out) return fail(KB_ERR_INVALID, "kb_index_load: null argument");
  *out = nullptr;
  return guarded([&] {
    auto ix = kb::Index::load(path, device, load_positions != 0, threads > 0 ? threads : 1);
    kb_index* h = new kb_index();
    h->ix = std::move(ix);
    *out = h;
  });
}

void kb_index_free(kb_index* ix) { delete ix; }

int kb_index_get_info(const kb_index* ix, kb_index_info* info) {
  if (!ix || !info) return fail(KB_ERR_INVALID, "kb_index_get_info: null argument");
  const kb::FlatIndex& f = ix->ix->flat;
  info->k = f.k;
  info->n_targets = f.num_targets();
  info->n_unitigs = f.n_unitigs();
  info->n_ec_blocks = (uint32_t)f.blk_lb.size();
  info->n_ec_sets = f.n_ec();
  info->n_kmers = f.n_kmers;
  info->table_slots = ix->ix->table_cap;
  info->load_seconds = ix->ix->load_seconds;
  info->build_seconds = ix->ix->build_seconds;
  return KB_OK;
}

int kb_index_inspect(const char* path, kb_index_info* info) {
  if (!path || !info) return fail(KB_ERR_INVALID, "kb_index_inspect: null argument");
  return guarded([&] {
    kb::FlatIndex f;
    kb::load_index_v13(path, f, false, 1);
    info->k = f.k;
    info->n_targets = f.num_targets();
    info->n_unitigs = f.n_unitigs();
    info->n_ec_blocks = (uint32_t)f.blk_lb.size();
    info->n_ec_sets = f.n_ec();
    info->n_kmers = f.n_kmers;
    info->table_slots = 0;
    info->load_seconds = 0;
    info->build_seconds = 0;
  });
}

const char* kb_index_target_name(const kb_index* ix, uint32_t i) {
  if (!ix || i >= ix->ix->flat.num_targets()) return nullptr;
  return ix->ix->flat.target_name[i].c_str();
}

int kb_index_target_lens(const kb_index* ix, uint32_t* lens_out) {
  if (!ix || !lens_out) return fail(KB_ERR_INVALID, "kb_index_target_lens: null argument");
  const auto& v = ix->ix->flat.target_len;
  memcpy(lens_out, v.data(), v.size() * sizeof(uint32_t));
  return KB_OK;
}

int kb_quant_create(kb_index* ix, const kb_quant_opts* opts, kb_quant** out) {
  if (!ix || !out) return fail(KB_ERR_INVALID, "kb_quant_create: null argument");
  *out = nullptr;
  return guarded([&] {
    kb::QuantOptions o;
    if (opts) {
      o.paired = opts->paired;
      o.strand_mode = opts->strand_mode;
      o.collect_fld = opts->collect_fld;
      // ProcessReads.cpp:1095: !single_overhang && tc.has_mean_fl  (has_mean_fl <=> -l given, MinCollector.h:37-41)
      if (!opts->single_overhang && opts->fld_mean > 0.0) o.fp_fl = (int)opts->fld_mean;
      if (opts->max_batch_reads) o.max_batch_reads = opts->max_batch_reads;
      if (opts->max_batch_bases) o.max_batch_bases = opts->max_batch_bases;
    }
    if (o.strand_mode < 0 || o.strand_mode > 2) throw std::invalid_argument("kb_quant_create: bad strand_mode");
    kb_quant* h = new kb_quant();
    h->owner = ix;
    h->q.reset(new kb::Quant(*ix->ix, o));
    *out = h;
  });
}

void kb_quant_free(kb_quant* q) { delete q; }

int kb_pseudoalign_batch(kb_quant* q, const char* bases, const uint32_t* offsets, uint32_t n_reads,
                         uint32_t fixed_len, int32_t* ec_out) {
  if (!q || (!bases && n_reads)) return fail(KB_ERR_INVALID, "kb_pseudoalign_batch: null argument");
  if (!offsets && fixed_len == 0 && n_reads) return fail(KB_ERR_INVALID, "kb_pseudoalign_batch: need offsets or fixed_len");
  return guarded([&] { q->q->pseudoalign_host(bases, offsets, n_reads, fixed_len, ec_out); });
}

int kb_pseudoalign_batch_pe(kb_quant* q, const char* bases1, const uint32_t* offsets1, const char* bases2,
                            const uint32_t* offsets2, uint32_t n_pairs, uint32_t fixed_len, int32_t* ec_out) {
  if (!q || ((!bases1 || !bases2) && n_pairs)) return fail(KB_ERR_INVALID, "kb_pseudoalign_batch_pe: null argument");
  if (!offsets1 && fixed_len == 0 && n_pairs) return fail(KB_ERR_INVALID, "kb_pseudoalign_batch_pe: need offsets or fixed_len");
  return guarded([&] { q->q->pseudoalign_host_pe(bases1, offsets1, bases2, offsets2, n_pairs, fixed_len, ec_out); });
}

void* kb_host_alloc(size_t bytes) {
  void* p = nullptr;
  if (cudaMallocHost(&p, bytes) != cudaSuccess) {
    cudaGetLastError();
    return nullptr;
  }
  return p;
}
void kb_host_free(void* p) {
  if (p) cudaFreeHost(p);
}

int kb_pseudoalign_batch_device(kb_quant* q, const void* d_bases, const uint32_t* d_offsets, uint32_t n_reads,
                                uint32_t fixed_len, uint32_t max_read_len) {
  if (!q || (!d_bases && n_reads)) return fail(KB_ERR_INVALID, "kb_pseudoalign_batch_device: null argument");
  return guarded([&] {
    q->q->pseudoalign_device((const uint8_t*)d_bases, d_offsets, n_reads, fixed_len,
                             d_offsets ? max_read_len : fixed_len);
  });
}

int kb_quant_sync(kb_quant* q) {
  if (!q) return fail(KB_ERR_INVALID, "kb_quant_sync: null argument");
  return guarded([&] { q->q->sync(); });
}

int kb_quant_set_stream(kb_quant* q, void* cuda_stream) {
  if (!q) return fail(KB_ERR_INVALID, "kb_quant_set_stream: null argument");
  return guarded([&] { q->q->set_stream((cudaStream_t)cuda_stream); });
}

int kb_quant_enable_timing(kb_quant* q, int on) {
  if (!q) return fail(KB_ERR_INVALID, "kb_quant_enable_timing: null argument");
  q->q->enable_timing(on != 0);
  return KB_OK;
}

int kb_quant_get_timings(kb_quant* q, kb_kernel_timings* out) {
  if (!q || !out) return fail(KB_ERR_INVALID, "kb_quant_get_timings: null argument");
  return guarded([&] {
    const kb::Quant::Timings t = q->q->timings();
    out->match_ms = t.match_ms;
    out->resolve_ms = t.resolve_ms;
    out->match_launches = t.match_launches;
    out->resolve_launches = t.resolve_launches;
    out->em_ms = q->q->last_em_seconds * 1e3;
    out->em_prep_ms = q->q->last_prep_seconds * 1e3;
    out->kernel_launches = q->q->n_kernel_launches;
    out->bs_resample_ms = q->q->last_bs_resample_ms;
    out->bs_em_ms = q->q->last_bs_em_ms;
    out->pack_ms = t.pack_ms;
    out->em_comp_blocks = (uint64_t)q->q->last_em_comp_blocks;
    out->em_comp_resident = q->q->last_em_comp_resident ? 1 : 0;
  });
}

int kb_quant_finalize(kb_quant* q, kb_run_stats* stats) {
  if (!q) return fail(KB_ERR_INVALID, "kb_quant_finalize: null argument");
  return guarded([&] {
    const bool fast = q->q->dev_stats_valid_;   // kb_em_run already numbered the ECs on the device
    if (!fast) q->q->finalize_ecs();
    if (stats) {
      const kb::Stats s = q->q->stats();
      stats->n_processed = s.n_processed;
      stats->n_pseudoaligned = s.n_pseudoaligned;
      stats->n_unique = s.n_unique;
      stats->n_ecs = fast ? q->q->dev_n_ecs_ : q->q->finalize_ecs().n();
      stats->n_ec_entries = fast ? q->q->dev_nnz_ : q->q->finalize_ecs().tid.size();
      stats->n_probes = s.n_probes;
      stats->n_slot_visits = s.n_slot_visits;
      stats->n_resolved = s.n_resolved;
      stats->n_memo_hits = s.n_memo_hits;
    }
  });
}

int kb_quant_ec_table(kb_quant* q, uint64_t* ec_offsets, uint32_t* tids, uint32_t* counts, int32_t* handles) {
  if (!q || !ec_offsets || !tids || !counts) return fail(KB_ERR_INVALID, "kb_quant_ec_table: null argument");
  return guarded([&] {
    const kb::EcTable& e = q->q->finalize_ecs();
    memcpy(ec_offsets, e.off.data(), e.off.size() * sizeof(uint64_t));
    memcpy(tids, e.tid.data(), e.tid.size() * sizeof(uint32_t));
    memcpy(counts, e.count.data(), e.count.size() * sizeof(uint32_t));
    if (handles) memcpy(handles, e.handle.data(), e.handle.size() * sizeof(int32_t));
  });
}

int kb_quant_get_flens(kb_quant* q, uint32_t* flens_out) {
  if (!q || !flens_out) return fail(KB_ERR_INVALID, "kb_quant_get_flens: null argument");
  memcpy(flens_out, q->q->flens().data(), 1000 * sizeof(uint32_t));
  return KB_OK;
}

int kb_quant_set_flens(kb_quant* q, const uint32_t* flens_in) {
  if (!q || !flens_in) return fail(KB_ERR_INVALID, "kb_quant_set_flens: null argument");
  q->q->set_flens(flens_in);
  return KB_OK;
}

static void em_common(kb_quant* q, const kb::EcTable& ecs, double fld_mean, double fld_sd, double* est, double* eff,
                      int32_t* rounds, double* seconds) {
  const auto fl = q->q->mean_fl_trunc(fld_mean, fld_sd);
  kb::EmResult r = q->q->run_em(ecs, fl);
  if (est) memcpy(est, r.alpha.data(), r.alpha.size() * sizeof(double));
  if (eff) memcpy(eff, r.eff_lens.data(), r.eff_lens.size() * sizeof(double));
  if (rounds) *rounds = r.rounds;
  if (seconds) *seconds = r.seconds;
}

int kb_em_run(kb_quant* q, double fld_mean, double fld_sd, double* est_counts_out, double* eff_lens_out,
              int32_t* rounds_out, double* seconds_out) {
  if (!q) return fail(KB_ERR_INVALID, "kb_em_run: null argument");
  return guarded([&] {
    const auto fl = q->q->mean_fl_trunc(fld_mean, fld_sd);
    kb::EmResult r = q->q->run_em_device(fl);
    if (est_counts_out) memcpy(est_counts_out, r.alpha.data(), r.alpha.size() * sizeof(double));
    if (eff_lens_out) memcpy(eff_lens_out, r.eff_lens.data(), r.eff_lens.size() * sizeof(double));
    if (rounds_out) *rounds_out = r.rounds;
    if (seconds_out) *seconds_out = r.seconds;
  });
}

int kb_em_run_table(kb_quant* q, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids,
                    const uint32_t* counts, double fld_mean, double fld_sd, double* est_counts_out,
                    double* eff_lens_out, int32_t* rounds_out, double* seconds_out) {
  if (!q || !ec_offsets || (!tids && n_ecs) || (!counts && n_ecs))
    return fail(KB_ERR_INVALID, "kb_em_run_table: null argument");
  return guarded([&] {
    kb::EcTable t;
    t.off.assign(ec_offsets, ec_offsets + n_ecs + 1);
    t.tid.assign(tids, tids + ec_offsets[n_ecs]);
    t.count.assign(counts, counts + n_ecs);
    const uint32_t T = q->q->index().flat.num_targets();
    for (uint32_t v : t.tid)
      if (v >= T) throw std::invalid_argument("kb_em_run_table: transcript id out of range");
    em_common(q, t, fld_mean, fld_sd, est_counts_out, eff_lens_out, rounds_out, seconds_out);
  });
}

int kb_read_priors(const char* path, double* out, uint64_t cap, uint64_t* n_out) {
  if (!path || !n_out) return fail(KB_ERR_INVALID, "kb_read_priors: null argument");
  std::vector<double> v;
  uint64_t line = 0;
  const int r = kb::read_priors_file(path, v, &line);
  if (r == 1) return fail(KB_ERR_IO, std::string("could not open priors file ") + path);
  if (r == 2)
    return fail(KB_ERR_INVALID, "line " + std::to_string(line) + " of priors file " + path + " is not a number");
  *n_out = v.size();
  if (out && cap >= v.size() && !v.empty()) memcpy(out, v.data(), v.size() * sizeof(double));
  return KB_OK;
}

int kb_em_set_priors(kb_quant* q, const double* priors, uint32_t n) {
  if (!q) return fail(KB_ERR_INVALID, "kb_em_set_priors: null argument");
  const uint32_t T = q->q->index().flat.num_targets();
  if (priors && n != T)
    return fail(KB_ERR_INVALID, "kb_em_set_priors: " + std::to_string(n) + " priors for " + std::to_string(T) + " targets");
  return guarded([&] { q->q->set_priors(priors); });
}

int kb_bootstrap_run(kb_quant* q, double fld_mean, double fld_sd, uint64_t seed, int32_t n_bootstrap,
                     double* est_counts_out, uint32_t* samples_out, int32_t* rounds_out) {
  if (!q || !est_counts_out || n_bootstrap < 0) return fail(KB_ERR_INVALID, "kb_bootstrap_run: bad argument");
  return guarded([&] {
    const auto fl = q->q->mean_fl_trunc(fld_mean, fld_sd);
    std::vector<double> alpha;
    std::vector<uint32_t> samples;
    // on the matrices kb_em_run left on the device (built now if it has not run yet)
    double ms[2] = {0, 0};
    std::vector<int> rounds = q->q->run_bootstrap_device(fl, seed, n_bootstrap, alpha, samples_out ? &samples : nullptr, ms);
    q->q->last_bs_resample_ms = ms[0];
    q->q->last_bs_em_ms = ms[1];
    memcpy(est_counts_out, alpha.data(), alpha.size() * sizeof(double));
    if (samples_out) memcpy(samples_out, samples.data(), samples.size() * sizeof(uint32_t));
    if (rounds_out)
      for (int b = 0; b < n_bootstrap; ++b) rounds_out[b] = rounds[b];
  });
}

int kb_quant_export_prepare(kb_quant* q, uint32_t* n_sets, uint32_t* n_entries) {
  if (!q || !n_sets || !n_entries) return fail(KB_ERR_INVALID, "kb_quant_export_prepare: null argument");
  return guarded([&] { q->q->export_prepare(n_sets, n_entries); });
}
int kb_quant_export_device(kb_quant* q, uint32_t* d_off, uint32_t* d_tids, uint32_t* d_counts, uint64_t* d_first) {
  if (!q || !d_off || !d_tids || !d_counts || !d_first) return fail(KB_ERR_INVALID, "kb_quant_export_device: null argument");
  return guarded([&] { q->q->export_copy(d_off, d_tids, d_counts, (unsigned long long*)d_first); });
}
int kb_quant_import_device(kb_quant* q, uint32_t n_sets, const uint32_t* d_off, const uint32_t* d_tids, const uint32_t* d_counts,
                           const uint64_t* d_first, uint64_t first_offset, uint64_t n_processed) {
  if (!q || (n_sets && (!d_off || !d_tids || !d_counts || !d_first))) return fail(KB_ERR_INVALID, "kb_quant_import_device: null argument");
  return guarded([&] {
    q->q->import_sets_device(n_sets, d_off, d_tids, d_counts, (const unsigned long long*)d_first, first_offset);
    q->q->add_processed(n_processed);
  });
}

struct kb_comm {
  std::unique_ptr<kb::Comm> c;
};

int kb_comm_unique_id(void* id_out) {
  if (!id_out) return fail(KB_ERR_INVALID, "kb_comm_unique_id: null argument");
  return guarded([&] { kb::Comm::unique_id(id_out); });
}
int kb_comm_create(int n_ranks, int rank, const void* id, int device, kb_comm** out) {
  if (!id || !out) return fail(KB_ERR_INVALID, "kb_comm_create: null argument");
  *out = nullptr;
  return guarded([&] {
    kb_comm* h = new kb_comm();
    h->c.reset(new kb::Comm(n_ranks, rank, id, device));
    *out = h;
  });
}
int kb_comm_create_from_nccl(void* nccl_comm, int n_ranks, int rank, int device, kb_comm** out) {
  if (!nccl_comm || !out) return fail(KB_ERR_INVALID, "kb_comm_create_from_nccl: null argument");
  *out = nullptr;
  return guarded([&] {
    kb_comm* h = new kb_comm();
    h->c.reset(new kb::Comm(nccl_comm, n_ranks, rank, device, false));
    *out = h;
  });
}
int kb_comm_create_all(const int* devices, int n_devices, kb_comm** out) {
  if (!devices || !out || n_devices < 1) return fail(KB_ERR_INVALID, "kb_comm_create_all: bad argument");
  return guarded([&] {
    std::vector<kb::Comm*> cs = kb::Comm::init_all(std::vector<int>(devices, devices + n_devices));
    for (int i = 0; i < n_devices; ++i) {
      out[i] = new kb_comm();
      out[i]->c.reset(cs[i]);
    }
  });
}
int kb_comm_reserve(kb_comm* c, uint64_t n_sets, uint64_t n_entries) {
  if (!c) return fail(KB_ERR_INVALID, "kb_comm_reserve: null argument");
  return guarded([&] { c->c->reserve(n_sets, n_entries); });
}
void kb_comm_free(kb_comm* c) { delete c; }
int kb_quant_merge_nccl(kb_quant* q, kb_comm* c, uint64_t first_stride, uint64_t* n_processed_total) {
  if (!q || !c) return fail(KB_ERR_INVALID, "kb_quant_merge_nccl: null argument");
  return guarded([&] {
    const uint64_t t = q->q->merge_to_root(*c->c, first_stride);
    if (n_processed_total) *n_processed_total = t;
  });
}
int kb_quant_merge_local(kb_quant* root, kb_quant* const* others, int32_t n_others, uint64_t* n_processed_total) {
  if (!root || (n_others > 0 && !others) || n_others < 0) return fail(KB_ERR_INVALID, "kb_quant_merge_local: bad argument");
  return guarded([&] {
    std::vector<kb::Quant*> o;
    for (int i = 0; i < n_others; ++i) {
      if (!others[i]) throw std::invalid_argument("kb_quant_merge_local: null run");
      o.push_back(others[i]->q.get());
    }
    const uint64_t t = root->q->merge_local(o, 0);
    if (n_processed_total) *n_processed_total = t;
  });
}
int kb_quant_set_frag_base(kb_quant* q, uint64_t base) {
  if (!q) return fail(KB_ERR_INVALID, "kb_quant_set_frag_base: null argument");
  q->q->set_frag_base(base);
  return KB_OK;
}
int kb_quant_reserve(kb_quant* q, uint64_t n_ecs, uint64_t n_entries) {
  if (!q) return fail(KB_ERR_INVALID, "kb_quant_reserve: null argument");
  return guarded([&] { q->q->reserve_em(n_ecs, n_entries); });
}

int kb_tcc_run_priors(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids, uint32_t n_samples,
                      const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts, const double* eff_lens,
                      int32_t per_sample_eff, const int32_t* gene_of_target, uint32_t n_genes, const double* priors,
                      double* est_counts_out, int32_t* rounds_out, double* gene_counts_out, double* gene_tpm_out) {
  if (!ix || !ec_offsets || !row_offsets || !eff_lens || !est_counts_out || (n_ecs && !tids) ||
      (n_genes && (!gene_of_target || !gene_counts_out || !gene_tpm_out)))
    return fail(KB_ERR_INVALID, "kb_tcc_run: null argument");
  return guarded([&] {
    kb::TccInput in;
    in.n_ecs = n_ecs; in.ec_off = ec_offsets; in.tids = tids; in.n_samples = n_samples; in.row_off = row_offsets;
    in.ec_ids = ec_ids; in.counts = counts; in.eff_lens = eff_lens; in.per_sample_eff = per_sample_eff != 0;
    in.gene_of = gene_of_target; in.n_genes = n_genes; in.priors = priors;
    std::vector<double> alpha, gc, gt;
    const std::vector<int> rounds = kb::tcc_run(*ix->ix, in, alpha, &gc, &gt);
    memcpy(est_counts_out, alpha.data(), alpha.size() * sizeof(double));
    if (n_genes) {
      memcpy(gene_counts_out, gc.data(), gc.size() * sizeof(double));
      memcpy(gene_tpm_out, gt.data(), gt.size() * sizeof(double));
    }
    if (rounds_out)
      for (uint32_t i = 0; i < n_samples; ++i) rounds_out[i] = rounds[i];
  });
}

int kb_tcc_run_genes(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids, uint32_t n_samples,
                     const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts, const double* eff_lens,
                     int32_t per_sample_eff, const int32_t* gene_of_target, uint32_t n_genes, double* est_counts_out,
                     int32_t* rounds_out, double* gene_counts_out, double* gene_tpm_out) {
  return kb_tcc_run_priors(ix, n_ecs, ec_offsets, tids, n_samples, row_offsets, ec_ids, counts, eff_lens, per_sample_eff,
                           gene_of_target, n_genes, nullptr, est_counts_out, rounds_out, gene_counts_out, gene_tpm_out);
}

int kb_tcc_run(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids, uint32_t n_samples,
               const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts, const double* eff_lens,
               int32_t per_sample_eff, double* est_counts_out, int32_t* rounds_out) {
  return kb_tcc_run_priors(ix, n_ecs, ec_offsets, tids, n_samples, row_offsets, ec_ids, counts, eff_lens, per_sample_eff,
                           nullptr, 0, nullptr, est_counts_out, rounds_out, nullptr, nullptr);
}

int kb_tcc_bootstrap_run_genes(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids,
                               uint32_t n_samples, const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts,
                               const double* eff_lens, int32_t per_sample_eff, const int32_t* gene_of_target, uint32_t n_genes,
                               uint64_t seed, int32_t n_bootstrap, int32_t want_samples, kb_tcc_bootstrap_genes_cb cb,
                               void* user) {
  if (!ix || !ec_offsets || !row_offsets || !eff_lens || !cb || (n_ecs && !tids) || n_bootstrap < 0 ||
      (n_genes && !gene_of_target))
    return fail(KB_ERR_INVALID, "kb_tcc_bootstrap_run: bad argument");
  return guarded([&] {
    kb::TccInput in;
    in.n_ecs = n_ecs; in.ec_off = ec_offsets; in.tids = tids; in.n_samples = n_samples; in.row_off = row_offsets;
    in.ec_ids = ec_ids; in.counts = counts; in.eff_lens = eff_lens; in.per_sample_eff = per_sample_eff != 0;
    in.gene_of = gene_of_target; in.n_genes = n_genes;
    kb::tcc_bootstrap(*ix->ix, in, seed, n_bootstrap, want_samples != 0,
                      [&](uint64_t first, uint32_t count, const double* est, const int* rounds, const uint32_t* samples,
                          const double* gene_counts, const double* gene_tpm) {
                        static_assert(sizeof(int) == sizeof(int32_t), "rounds are handed out as int32_t");
                        if (cb(user, first, count, est, reinterpret_cast<const int32_t*>(rounds), samples, gene_counts,
                               gene_tpm) != 0)
                          throw std::invalid_argument("kb_tcc_bootstrap_run: stopped by the callback");
                      });
  });
}

namespace {
struct TccBootstrapCbAdapter {     // kb_tcc_bootstrap_cb behind a kb_tcc_bootstrap_genes_cb that ignores the genes
  kb_tcc_bootstrap_cb cb;
  void* user;
  static int call(void* self, uint64_t first, uint32_t count, const double* est, const int32_t* rounds,
                  const uint32_t* samples, const double*, const double*) {
    const auto* a = static_cast<const TccBootstrapCbAdapter*>(self);
    return a->cb(a->user, first, count, est, rounds, samples);
  }
};
}  // namespace

int kb_tcc_bootstrap_run(kb_index* ix, uint32_t n_ecs, const uint64_t* ec_offsets, const uint32_t* tids, uint32_t n_samples,
                         const uint64_t* row_offsets, const uint32_t* ec_ids, const uint32_t* counts, const double* eff_lens,
                         int32_t per_sample_eff, uint64_t seed, int32_t n_bootstrap, int32_t want_samples,
                         kb_tcc_bootstrap_cb cb, void* user) {
  if (!cb) return fail(KB_ERR_INVALID, "kb_tcc_bootstrap_run: bad argument");
  TccBootstrapCbAdapter a{cb, user};
  return kb_tcc_bootstrap_run_genes(ix, n_ecs, ec_offsets, tids, n_samples, row_offsets, ec_ids, counts, eff_lens,
                                    per_sample_eff, nullptr, 0, seed, n_bootstrap, want_samples, &TccBootstrapCbAdapter::call,
                                    &a);
}

int kb_eff_lens(const kb_index* ix, const uint32_t* flens, double fld_mean, double fld_sd, double* eff_out, double* mean_out,
                double* sd_out) {
  if (!ix || !eff_out) return fail(KB_ERR_INVALID, "kb_eff_lens: null argument");
  const auto& tl = ix->ix->flat.target_len;
  const size_t T = tl.size();
  if (!flens && fld_mean == 0.0) {
    // no fragment-length information: fl_means = target lengths, so every effective length is len - len + 1 (main.cpp:3025-3027)
    for (size_t t = 0; t < T; ++t) {
      const double len = static_cast<double>(tl[t]);
      double e = len - len + 1;
      if (e < 1.0) e = len;
      eff_out[t] = e;
    }
    return KB_OK;
  }
  static const uint32_t zeros[1000] = {0};
  const uint32_t* fl = flens ? flens : zeros;
  const std::vector<double> trunc = kb::mean_fl_trunc_of(fl, fld_mean, fld_sd);
  const double marginal = trunc[999];
  for (size_t t = 0; t < T; ++t) {
    const double mean = tl[t] >= 1000 ? marginal : trunc[tl[t]];
    const double len = static_cast<double>(tl[t]);
    double e = len - mean + 1;
    if (e < 1.0) e = len;
    eff_out[t] = e;
  }
  // MinCollector::get_mean_frag_len(true) / get_sd_frag_len (src/MinCollector.cpp:583-627)
  double mean_fl;
  if (fld_mean != 0.0) {
    mean_fl = trunc[999];
  } else {
    auto total_counts = 0;
    double total_mass = 0.0;
    for (size_t i = 0; i < 1000; ++i) {
      total_counts += fl[i];
      total_mass += static_cast<double>(fl[i] * i);
    }
    mean_fl = total_counts == 0 ? std::numeric_limits<double>::max() : total_mass / static_cast<double>(total_counts);
  }
  if (mean_out) *mean_out = mean_fl;
  if (sd_out) {
    const uint32_t* sf = fld_mean != 0.0 ? zeros : fl;     // with -l the collector's histogram stays empty
    size_t total_counts = 0;
    double total_mass = 0.0;
    const double m = mean_fl;
    for (size_t i = 0; i < 1000; ++i) {
      total_counts += sf[i];
      total_mass += sf[i] * (i - m) * (i - m);
    }
    *sd_out = std::sqrt(total_mass / total_counts);
  }
  return KB_OK;
}

int kb_bus_create(kb_index* ix, const kb_bus_opts* o, kb_quant** out) {
  if (!ix || !o || !out) return fail(KB_ERR_INVALID, "kb_bus_create: null argument");
  *out = nullptr;
  return guarded([&] {
    if (o->nfiles < 1 || o->nfiles > 4 || o->n_bc < 0 || o->n_bc > 4 || o->n_umi < 1 || o->n_umi > 4)
      throw std::invalid_argument("kb_bus_create: unsupported technology layout");
    if (o->seq.stop != 0 || o->seq.fileno < 0 || o->seq.fileno >= o->nfiles || o->seq.start < 0)
      throw std::invalid_argument("kb_bus_create: the sequence must run to the end of its read (stop == 0)");
    if (o->paired && (o->seq2.stop != 0 || o->seq2.fileno < 0 || o->seq2.fileno >= o->nfiles || o->seq2.start < 0 ||
                      o->seq2.fileno == o->seq.fileno))
      throw std::invalid_argument("kb_bus_create: the second sequence of a paired technology must be another file, running to the end of its read");
    const bool no_umi = o->n_umi == 1 && o->umi[0].fileno == -1;
    kb::QuantOptions q;
    q.paired = o->paired ? 1 : 0;
    q.strand_mode = o->strand_mode;
    q.collect_fld = o->paired ? 1 : 0;     // findFragmentLength = tcount < 10000 && busopt.paired (src/ProcessReads.cpp:1400)
    q.bus = true;
    if (o->max_batch_sets) q.max_batch_reads = o->max_batch_sets;
    if (o->max_batch_bases) q.max_batch_bases = o->max_batch_bases;
    kb::BusSpec& s = q.bus_spec;
    s.nfiles = o->nfiles;
    s.n_bc = o->n_bc;
    s.n_umi = o->n_umi;
    auto chk = [&](const kb_bus_substr& x) {
      if (x.fileno < 0 || x.fileno >= o->nfiles || x.start < 0 || x.stop < 0)
        throw std::invalid_argument("kb_bus_create: bad barcode/UMI location");
    };
    for (int i = 0; i < o->n_bc; ++i) { chk(o->bc[i]); s.bc_f[i] = o->bc[i].fileno; s.bc_a[i] = o->bc[i].start; s.bc_b[i] = o->bc[i].stop; }
    s.no_umi = no_umi ? 1 : 0;
    if (no_umi) s.n_umi = 0;
    else
      for (int i = 0; i < o->n_umi; ++i) { chk(o->umi[i]); s.umi_f[i] = o->umi[i].fileno; s.umi_a[i] = o->umi[i].start; s.umi_b[i] = o->umi[i].stop; }
    s.seq_file = o->seq.fileno;
    s.seq_start = o->seq.start;
    s.num_flag = o->num;
    s.paired = o->paired ? 1 : 0;
    s.seq2_file = o->paired ? o->seq2.fileno : 0;
    s.seq2_start = o->paired ? o->seq2.start : 0;
    s.fake_bc = 0;
    s.tag_len = 0;
    s.tag_bin = 0;
    if (o->tag && o->tag[0]) {
      const size_t tl = strlen(o->tag);
      if (no_umi || tl > 31) throw std::invalid_argument("kb_bus_create: a tag sequence needs a UMI and at most 31 letters");
      // opt.busOptions.umi[0].start += tag length; it must stay in front of the stop (src/main.cpp:1467-1475)
      s.umi_a[0] += (int)tl;
      if (s.umi_b[0] != 0 && s.umi_a[0] >= s.umi_b[0]) throw std::invalid_argument("Error: Tag sequence must be shorter than UMI sequence");
      unsigned long long r = 0;                       // stringToBinary (src/BUSData.cpp:8-36)
      for (size_t i = 0; i < tl; ++i) {
        const unsigned c = (unsigned char)o->tag[i];
        const unsigned long long x = (c & 4) >> 1;
        r = (r << 2) | (x + ((x ^ (c & 2)) >> 1));
      }
      s.tag_len = (int)tl;
      s.tag_bin = r;
    }
    kb_quant* h = new kb_quant();
    h->owner = ix;
    h->q.reset(new kb::Quant(*ix->ix, q));
    *out = h;
  });
}

int kb_bus_batch(kb_quant* q, const char* const* bases, const uint32_t* const* offsets, uint32_t n_sets,
                 kb_bus_record* records_out, uint32_t* n_records_out) {
  if (!q || !bases || !offsets || (!records_out && n_sets)) return fail(KB_ERR_INVALID, "kb_bus_batch: null argument");
  static_assert(sizeof(kb_bus_record) == sizeof(kb::BusRecord), "record layout");
  return guarded([&] { q->q->bus_batch_host(bases, offsets, n_sets, (kb::BusRecord*)records_out, n_records_out); });
}

int kb_bus_batch_device(kb_quant* q, const void* const* d_bases, const uint32_t* const* d_offsets, uint32_t n_sets,
                        uint32_t max_seq_len, uint32_t* n_records_out, const kb_bus_record** d_records_out) {
  if (!q || !d_bases || !d_offsets) return fail(KB_ERR_INVALID, "kb_bus_batch_device: null argument");
  return guarded([&] {
    const uint32_t n = q->q->bus_batch_device((const uint8_t* const*)d_bases, d_offsets, n_sets, max_seq_len);
    if (n_records_out) *n_records_out = n;
    if (d_records_out) *d_records_out = (const kb_bus_record*)q->q->bus_records_device();
  });
}

int kb_bus_begin_sample(kb_quant* q, uint64_t barcode) {
  if (!q) return fail(KB_ERR_INVALID, "kb_bus_begin_sample: null argument");
  return guarded([&] { q->q->bus_begin_sample(barcode); });
}

int kb_bus_set_batch_barcodes(kb_quant* q, int32_t on) {
  if (!q) return fail(KB_ERR_INVALID, "kb_bus_set_batch_barcodes: null argument");
  return guarded([&] { q->q->set_batch_barcodes(on != 0); });
}

int kb_bus_lengths(kb_quant* q, uint32_t* bc_hist, uint32_t* umi_hist) {
  if (!q || !bc_hist || !umi_hist) return fail(KB_ERR_INVALID, "kb_bus_lengths: null argument");
  return guarded([&] { q->q->bus_lengths(bc_hist, umi_hist); });
}

int kb_bus_set_aa(kb_quant* q, int32_t on) {
  if (!q) return fail(KB_ERR_INVALID, "kb_bus_set_aa: null argument");
  return guarded([&] { q->q->set_aa(on != 0); });
}

int kb_bus_frame_clashes(kb_quant* q, uint64_t* n_out) {
  if (!q || !n_out) return fail(KB_ERR_INVALID, "kb_bus_frame_clashes: null argument");
  return guarded([&] { *n_out = q->q->frame_clashes(); });
}

int kb_bus_group_create(kb_quant* const* members, int32_t n, kb_bus_group** out) {
  if (!members || !out || n < 1) return fail(KB_ERR_INVALID, "kb_bus_group_create: null argument or no members");
  *out = nullptr;
  std::vector<kb::Quant*> ms;
  for (int32_t i = 0; i < n; ++i) {
    if (!members[i]) return fail(KB_ERR_INVALID, "kb_bus_group_create: null member");
    kb::Quant* q = members[i]->q.get();
    for (kb::Quant* o : ms)
      if (o == q) return fail(KB_ERR_INVALID, "kb_bus_group_create: a member is listed twice");
    if (!q->options().bus) return fail(KB_ERR_INVALID, "kb_bus_group_create: member " + std::to_string(i) + " is not a bus run");
    if (!q->bus_fresh()) return fail(KB_ERR_INVALID, "kb_bus_group_create: member " + std::to_string(i) + " has run a batch already");
    ms.push_back(q);
  }
  const kb::Quant& a = *ms[0];
  for (int32_t i = 1; i < n; ++i) {
    const kb::Quant& b = *ms[i];
    const kb::QuantOptions &x = a.options(), &y = b.options();
    const kb::BusSpec &s = x.bus_spec, &t = y.bus_spec;
    bool same = x.paired == y.paired && x.strand_mode == y.strand_mode && x.collect_fld == y.collect_fld &&
                x.max_batch_reads == y.max_batch_reads && x.max_batch_bases == y.max_batch_bases && a.aa() == b.aa() &&
                s.nfiles == t.nfiles && s.n_bc == t.n_bc && s.n_umi == t.n_umi && s.seq_file == t.seq_file &&
                s.seq_start == t.seq_start && s.num_flag == t.num_flag && s.paired == t.paired && s.seq2_file == t.seq2_file &&
                s.seq2_start == t.seq2_start && s.no_umi == t.no_umi && s.fake_bc == t.fake_bc && s.tag_len == t.tag_len &&
                s.tag_bin == t.tag_bin && s.batch_bc == t.batch_bc && s.bc_prefix == t.bc_prefix;
    for (int j = 0; j < 4; ++j)
      same = same && s.bc_f[j] == t.bc_f[j] && s.bc_a[j] == t.bc_a[j] && s.bc_b[j] == t.bc_b[j] && s.umi_f[j] == t.umi_f[j] &&
             s.umi_a[j] == t.umi_a[j] && s.umi_b[j] == t.umi_b[j];
    if (!same) return fail(KB_ERR_INVALID, "kb_bus_group_create: member " + std::to_string(i) + " has other bus options than member 0");
    kb::Index &ia = members[0]->q->index(), &ib = members[i]->q->index();
    if (ia.flat.k != ib.flat.k || ia.flat.num_targets() != ib.flat.num_targets())
      return fail(KB_ERR_INVALID, "kb_bus_group_create: member " + std::to_string(i) + " has an index with another k or target count");
  }
  return guarded([&] {
    kb_bus_group* h = new kb_bus_group();
    h->g.reset(new kb::BusGroup(ms));
    *out = h;
  });
}

void kb_bus_group_free(kb_bus_group* g) { delete g; }

int kb_bus_group_submit(kb_bus_group* g, int32_t member, const char* const* bases, const uint32_t* const* offsets,
                        uint32_t n_sets, uint64_t* ticket) {
  if (!g || !bases || !offsets || !ticket) return fail(KB_ERR_INVALID, "kb_bus_group_submit: null argument");
  return guarded_invalid([&] { *ticket = g->g->submit(member, bases, offsets, n_sets); });
}

int kb_bus_group_complete(kb_bus_group* g, uint64_t ticket, kb_bus_record* records_out, uint32_t* n_records_out) {
  if (!g || !records_out) return fail(KB_ERR_INVALID, "kb_bus_group_complete: null argument");
  return guarded_invalid([&] { g->g->complete(ticket, (kb::BusRecord*)records_out, n_records_out); });
}

int kb_bus_group_begin_sample(kb_bus_group* g, uint64_t barcode) {
  if (!g) return fail(KB_ERR_INVALID, "kb_bus_group_begin_sample: null argument");
  return guarded_invalid([&] { g->g->begin_sample(barcode); });
}

int kb_bus_group_finalize(kb_bus_group* g, kb_run_stats* stats) {
  if (!g || !stats) return fail(KB_ERR_INVALID, "kb_bus_group_finalize: null argument");
  return guarded([&] {
    const kb::Stats s = g->g->stats();
    const kb::EcTable& e = g->g->ec_table();
    stats->n_processed = s.n_processed;
    stats->n_pseudoaligned = s.n_pseudoaligned;
    stats->n_unique = s.n_unique;
    stats->n_ecs = e.off.size() - 1;
    stats->n_ec_entries = e.tid.size();
    stats->n_probes = s.n_probes;
    stats->n_slot_visits = s.n_slot_visits;
    stats->n_resolved = s.n_resolved;
    stats->n_memo_hits = s.n_memo_hits;
  });
}

int kb_bus_group_ec_table(kb_bus_group* g, uint64_t* ec_offsets, uint32_t* tids, uint32_t* counts) {
  if (!g || !ec_offsets || !tids || !counts) return fail(KB_ERR_INVALID, "kb_bus_group_ec_table: null argument");
  return guarded([&] {
    const kb::EcTable& e = g->g->ec_table();
    memcpy(ec_offsets, e.off.data(), e.off.size() * sizeof(uint64_t));
    memcpy(tids, e.tid.data(), e.tid.size() * sizeof(uint32_t));
    memcpy(counts, e.count.data(), e.count.size() * sizeof(uint32_t));
  });
}

int kb_bus_group_lengths(kb_bus_group* g, uint32_t* bc_hist, uint32_t* umi_hist) {
  if (!g || !bc_hist || !umi_hist) return fail(KB_ERR_INVALID, "kb_bus_group_lengths: null argument");
  return guarded([&] {
    memset(bc_hist, 0, 33 * sizeof(uint32_t));
    memset(umi_hist, 0, 33 * sizeof(uint32_t));
    for (int m = 0; m < g->g->n_members(); ++m) {
      uint32_t b[33], u[33];
      g->g->member(m).bus_lengths(b, u);
      for (int i = 0; i < 33; ++i) { bc_hist[i] += b[i]; umi_hist[i] += u[i]; }
    }
  });
}

int kb_bus_group_frame_clashes(kb_bus_group* g, uint64_t* n_out) {
  if (!g || !n_out) return fail(KB_ERR_INVALID, "kb_bus_group_frame_clashes: null argument");
  return guarded([&] {
    uint64_t n = 0;
    for (int m = 0; m < g->g->n_members(); ++m) n += g->g->member(m).frame_clashes();
    *n_out = n;
  });
}

int kb_fastx_summary(const char* path, uint64_t* n_reads, uint64_t* n_bases, uint64_t* fnv1a) {
  return kb_fastx_summary_mt(path, 1, n_reads, n_bases, fnv1a);
}

int kb_fastx_summary_mt(const char* path, int threads, uint64_t* n_reads, uint64_t* n_bases, uint64_t* fnv1a) {
  if (!path || !n_reads || !n_bases || !fnv1a) return fail(KB_ERR_INVALID, "kb_fastx_summary: null argument");
  try {
    kb::FastxReader f(path, threads);
    kb::ReadBatch b;
    std::vector<char> bases((size_t)(1u << 22) + kb::FastxFile::kMaxRead);
    std::vector<uint32_t> off(65537);
    b.bases = bases.data(); b.off = off.data(); b.cap_bases = bases.size(); b.cap_reads = 65536;
    uint64_t nr = 0, nbz = 0, h = 1469598103934665603ULL;
    for (;;) {
      b.clear();
      if (!f.fill(b, 65536)) break;
      nr += b.n;
      nbz += b.n_bases();
      for (size_t i = 0; i < b.n; ++i) {
        for (uint32_t j = b.off[i]; j < b.off[i + 1]; ++j) { h ^= (unsigned char)b.bases[j]; h *= 1099511628211ULL; }
        h ^= 0xFF; h *= 1099511628211ULL;   // record separator
      }
    }
    *n_reads = nr; *n_bases = nbz; *fnv1a = h;
    return KB_OK;
  } catch (const std::exception& e) {
    return fail(KB_ERR_IO, e.what());
  }
}

int kb_gz_summary(const char* path, uint64_t* n_bytes, uint32_t* crc) {
  if (!path || !n_bytes || !crc) return fail(KB_ERR_INVALID, "kb_gz_summary: null argument");
  try {
    kb::FastGz g(path);
    const char* p = nullptr;
    size_t n = 0;
    uint64_t tot = 0;
    uint32_t c = 0;
    while (g.next_chunk(p, n)) {
      tot += n;
      c = kb::fast_crc32(c, (const uint8_t*)p, n);
    }
    *n_bytes = tot;
    *crc = c;
    return KB_OK;
  } catch (const std::exception& e) {
    return fail(KB_ERR_IO, e.what());
  }
}

int kb_counts_to_tpm(const double* est_counts, const double* eff_lens, uint32_t n, double* tpm_out) {
  if (!est_counts || !eff_lens || !tpm_out) return fail(KB_ERR_INVALID, "kb_counts_to_tpm: null argument");
  const double MILLION = 1e6;
  double total_mass = 0.0;
  for (uint32_t i = 0; i < n; ++i) {
    tpm_out[i] = est_counts[i] / eff_lens[i];
    total_mass += tpm_out[i];
  }
  for (uint32_t i = 0; i < n; ++i) tpm_out[i] = (tpm_out[i] / total_mass) * MILLION;
  return KB_OK;
}

}  // extern "C"
