// Host-side engine: see engine.hpp.
#include "engine.hpp"

#include <algorithm>
#include <chrono>
#include <cmath>
#include <cstring>
#include <numeric>
#include <random>
#include <thread>

namespace kb {

namespace {

inline void ck(cudaError_t e, const char* what) {
  if (e != cudaSuccess) throw Error(std::string("CUDA error in ") + what + ": " + cudaGetErrorString(e));
}
#define KB_CK(x) ck((x), #x)

inline uint64_t pow2_ge(uint64_t v) {
  uint64_t p = 1;
  while (p < v) p <<= 1;
  return p;
}

double now_s() {
  return std::chrono::duration<double>(std::chrono::steady_clock::now().time_since_epoch()).count();
}

}  // namespace

template <class T> void DBuf<T>::alloc(size_t count) {
  release();
  n = count;
  if (count) KB_CK(cudaMalloc((void**)&p, count * sizeof(T)));
}
template <class T> void DBuf<T>::release() {
  if (p) cudaFree(p);
  p = nullptr;
  n = 0;
}
template <class T> void DBuf<T>::upload(const T* src, size_t count, cudaStream_t st) {
  if (count > n) alloc(count);
  if (count) KB_CK(cudaMemcpyAsync(p, src, count * sizeof(T), cudaMemcpyHostToDevice, st));
}
template <class T> void DBuf<T>::download(T* dst, size_t count, size_t offset, cudaStream_t st) const {
  if (count) KB_CK(cudaMemcpyAsync(dst, p + offset, count * sizeof(T), cudaMemcpyDeviceToHost, st));
}
template <class T> void DBuf<T>::zero(cudaStream_t st) {
  if (n) KB_CK(cudaMemsetAsync(p, 0, n * sizeof(T), st));
}


// ------------------------------------------------------------------------------------------
// Index
// ------------------------------------------------------------------------------------------
Index::~Index() { delete shared_emws; }

std::unique_ptr<Index> Index::load(const std::string& path, int device, bool load_positions, int threads) {
  std::unique_ptr<Index> ix(new Index());
  ix->device = device;
  const double t0 = now_s();
  // the file is parsed on its own thread while this one initialises the driver and brings the CUDA context up
  // (0.3 s + 0.3-0.5 s in a fresh process)
  std::exception_ptr parse_err;
  std::thread parser([&] {
    try {
      load_index_v13(path, ix->flat, load_positions, threads);
    } catch (...) {
      parse_err = std::current_exception();
    }
  });
  int ndev = 0;
  const bool have_dev = cudaGetDeviceCount(&ndev) == cudaSuccess && ndev > 0;
  if (!have_dev || device < 0 || device >= ndev) {
    parser.join();
    if (!have_dev) throw Error("kallisto_b200: no CUDA device available (this build has no CPU path)");
    throw Error("kallisto_b200: invalid CUDA device ordinal");
  }
  cudaError_t init_err = cudaSetDevice(device);
  if (init_err == cudaSuccess) init_err = cudaFree(0);
  if (init_err == cudaSuccess) {
    // The k-mer table probes touch one random 32-byte sector each.  With the default L2 fetch granularity
    // every miss pulls 64-128 bytes from HBM (ncu: 5.2 GB per 2 M pairs against 1.5 GB algorithmic); with
    // 32 bytes the DRAM traffic equals the algorithmic bytes (1.85 GB) at the same probe rate -- the rate is
    // bounded by the random-sector throughput of the L2-miss path (tools/randbench), not by bytes.
    size_t gran = 32;
    if (const char* s = getenv("KB_L2_FETCH")) gran = (size_t)atoi(s);    // 0: leave the device default
    if (gran > 0 && cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, gran) != cudaSuccess) cudaGetLastError();
  }
  parser.join();
  if (parse_err) std::rethrow_exception(parse_err);
  KB_CK(init_err);
  const double t1 = now_s();
  ix->load_seconds = t1 - t0;
  FlatIndex& f = ix->flat;
  if (f.graphless) {      // index.saved: targets only; nothing to build on the device, only quant-tcc can use it
    ix->build_seconds = 0;
    return ix;
  }
  if (f.onlist.size() != f.target_len.size())
    throw Error("kallisto_b200: indices whose on-list does not cover every target are not supported yet");
  if (f.ec_tid.size() >= 0xFFFFFFFFull) throw Error("kallisto_b200: index EC sets exceed 2^32 entries");
  if (f.num_targets() >= (1u << 24)) throw Error("kallisto_b200: more than 2^24 targets are not supported");

  const uint32_t nU = f.n_unitigs();
  std::vector<uint64_t> kstart(nU + 1, 0);
  for (uint32_t u = 0; u < nU; ++u) kstart[u + 1] = kstart[u] + (f.ulen[u] - f.k + 1);
  if (kstart[nU] != f.n_kmers) throw Error("kallisto_b200: k-mer count mismatch");

  cudaStream_t st = 0;
  // permanent arrays
  std::vector<uint32_t> ec_off32(f.ec_off.size());
  for (size_t i = 0; i < f.ec_off.size(); ++i) ec_off32[i] = (uint32_t)f.ec_off[i];
  ix->ec_off.upload(ec_off32.data(), ec_off32.size(), st);
  ix->n_index_tids = (uint32_t)f.ec_tid.size();
  ix->index_pool.alloc(std::max<size_t>(1, f.ec_tid.size()));
  ix->index_pool.upload(f.ec_tid.data(), f.ec_tid.size(), st);
  ix->blk_strand_off.upload(f.blk_strand_off.data(), f.blk_strand_off.size(), st);
  ix->strand.alloc(std::max<size_t>(1, f.strand.size()));
  ix->strand.upload(f.strand.data(), f.strand.size(), st);
  if (f.has_positions) {
    ix->fp_info.alloc(std::max<size_t>(1, f.fp_info.size() / 4));
    if (!f.fp_info.empty())
      KB_CK(cudaMemcpyAsync(ix->fp_info.p, f.fp_info.data(), f.fp_info.size() * 4, cudaMemcpyHostToDevice, st));
    std::vector<uint32_t> busize(f.blk_lb.size());
    for (uint32_t u = 0; u < f.n_unitigs(); ++u)
      for (uint64_t b = f.blk_off[u]; b < f.blk_off[u + 1]; ++b) busize[b] = f.ulen[u];
    ix->blk_usize.upload(busize.data(), busize.size(), st);
    ix->target_len.upload(f.target_len.data(), f.target_len.size(), st);
    KB_CK(cudaStreamSynchronize(st));
  }
  for (uint32_t e = 0; e < f.n_ec(); ++e) {
    const uint32_t len = (uint32_t)(f.ec_off[e + 1] - f.ec_off[e]);
    if (len == 0) ix->empty_ec = e;
    ix->max_set_len = std::max(ix->max_set_len, len);
  }

  cudaStream_t st0 = st;
  // set dictionary, initial state: the index's own EC sets.  Done first: the k-mer slots store the
  // dictionary handle of their block's set, not its index-local id.
  ix->dict_cap = pow2_ge((uint64_t)f.n_ec() * 4 + (1u << 20));
  ix->dslots_init.alloc(ix->dict_cap);
  launch_fill_u64(ix->dslots_init.p, ix->dict_cap, ~0ULL, st0);
  ix->ec_handle.alloc(std::max<uint32_t>(1, f.n_ec()));
  {
    DictInitArgs a{};
    a.ec_off = ix->ec_off.p; a.pool = ix->index_pool.p; a.n_ec = f.n_ec();
    a.dslots = ix->dslots_init.p; a.dmask = ix->dict_cap - 1; a.ec_handle = ix->ec_handle.p;
    launch_dict_init(a, st0);
    KB_CK(cudaGetLastError());
  }
  ix->h_ec_handle.resize(f.n_ec());
  ix->ec_handle.download(ix->h_ec_handle.data(), f.n_ec(), 0, st0);
  KB_CK(cudaStreamSynchronize(st0));
  {
    std::vector<uint32_t> blk_handle(f.blk_ec.size());
    for (size_t i = 0; i < blk_handle.size(); ++i) blk_handle[i] = (uint32_t)ix->h_ec_handle[f.blk_ec[i]];
    ix->blk_ec.upload(blk_handle.data(), blk_handle.size(), st0);
    KB_CK(cudaStreamSynchronize(st0));
  }
  if (ix->empty_ec != 0xFFFFFFFFu) ix->empty_ec = (uint32_t)ix->h_ec_handle[ix->empty_ec];

  // k-mer table.  Every probe costs one random 32-byte sector whatever the table size, and the sector rate of the
  // L2-miss path is the bound of match_kernel (tools/randbench), so HBM capacity is traded for shorter probe
  // sequences: slots >= 4 x k-mers (load 0.14-0.27: 1.14 visits per lookup) when that
  // leaves three quarters of the free device memory to the run, else 2 x (load <= 0.5; 1.37 visits measured at
  // 0.27).  KB_TABLE_FACTOR overrides.
  double factor = 4.0;
  {
    size_t free_b = 0, total_b = 0;
    KB_CK(cudaMemGetInfo(&free_b, &total_b));
    const uint64_t cap4 = pow2_ge(std::max<uint64_t>(1024, f.n_kmers * 4));
    if (cap4 * sizeof(KmerSlot) > free_b / 4) factor = 2.0;
  }
  if (const char* s = getenv("KB_TABLE_FACTOR")) { const double v = atof(s); if (v >= 1.25 && v <= 64.0) factor = v; }
  ix->table_cap = pow2_ge(std::max<uint64_t>(1024, (uint64_t)((double)f.n_kmers * factor)));
  // match_kernel keeps a probe's slot index in 32 bits (128 GB of slots)
  if (ix->table_cap > (1ull << 32)) throw Error("kallisto_b200: k-mer table larger than 2^32 slots");
  ix->slots.alloc(ix->table_cap);
  // presence filter: 2^KB_FILTER_LOG2 bits (default: about 3.5 bits per k-mer, at most 2^28 bits = 32 MB so that it
  // fits the persisting part of the H100's 50 MB L2; 0 = off).  Single hash: a miss passes it with probability
  // 1 - exp(-n / bits).
  uint32_t filter_bits = 0;
  {
    int lg = 0;
    while ((1ull << lg) < f.n_kmers * 3 && lg < 28) ++lg;
    if (lg < 16) lg = 16;
    if (const char* s = getenv("KB_FILTER_LOG2")) lg = atoi(s);
    if (lg >= 10 && lg <= 32) filter_bits = lg == 32 ? 0 : (1u << lg);
    if (lg == 32) filter_bits = 0;
  }
  if (filter_bits) {
    ix->filter.alloc(filter_bits / 32);
    ix->filter.zero(st);
  }
  DBuf<int> err;
  err.alloc(1);
  err.zero(st);
  {
    DBuf<uint8_t> d_useq;
    DBuf<uint64_t> d_byteoff, d_skmer, d_kstart, d_blkoff;
    DBuf<uint32_t> d_lb, d_ub;
    d_useq.upload(f.useq.data(), f.useq.size(), st);
    d_byteoff.upload(f.useq_byteoff.data(), f.useq_byteoff.size(), st);
    d_skmer.alloc(std::max<size_t>(1, f.skmer.size()));
    d_skmer.upload(f.skmer.data(), f.skmer.size(), st);
    d_kstart.upload(kstart.data(), kstart.size(), st);
    d_blkoff.upload(f.blk_off.data(), f.blk_off.size(), st);
    d_lb.upload(f.blk_lb.data(), f.blk_lb.size(), st);
    d_ub.upload(f.blk_ub.data(), f.blk_ub.size(), st);
    TableBuildArgs a{};
    a.useq = d_useq.p; a.useq_byteoff = d_byteoff.p; a.skmer = d_skmer.p; a.kstart = d_kstart.p;
    a.blk_off = d_blkoff.p; a.blk_lb = d_lb.p; a.blk_ub = d_ub.p; a.blk_ec = ix->blk_ec.p;
    a.n_long = f.n_long; a.n_unitigs = nU; a.k = f.k; a.n_kmers = f.n_kmers;
    a.slots = ix->slots.p; a.mask = ix->table_cap - 1; a.error = err.p;
    a.filter = filter_bits ? ix->filter.p : nullptr; a.filter_mask = filter_bits ? filter_bits - 1 : 0;
    launch_build_table(a, st);
    KB_CK(cudaGetLastError());
    KB_CK(cudaStreamSynchronize(st));
  }
  int herr = 0;
  err.download(&herr, 1, 0, st);
  KB_CK(cudaStreamSynchronize(st));
  if (herr & KB_DEVERR_TABLE_DUP) throw Error("kallisto_b200: corrupt index (a k-mer occurs in two unitigs)");

  DevIndex& d = ix->dev;
  d.slots = ix->slots.p;
  d.mask = ix->table_cap - 1;
  d.filter = filter_bits ? ix->filter.p : nullptr;
  d.filter_mask = filter_bits ? filter_bits - 1 : 0;
  if (filter_bits) {
    // keep the filter in L2: persisting carve-out as large as the device allows (the access window itself is set on the
    // stream of every run, Quant::apply_l2_window)
    int max_persist = 0;
    cudaDeviceGetAttribute(&max_persist, cudaDevAttrMaxPersistingL2CacheSize, device);
    size_t want = std::min<size_t>((size_t)filter_bits / 8, (size_t)std::max(0, max_persist));
    if (const char* s = getenv("KB_L2_PERSIST_MB")) want = std::min<size_t>((size_t)atoll(s) << 20, (size_t)std::max(0, max_persist));
    if (want > 0 && cudaDeviceSetLimit(cudaLimitPersistingL2CacheSize, want) == cudaSuccess) ix->l2_persist_bytes = want;
    else cudaGetLastError();
  }
  d.k = f.k;
  d.n_ec = f.n_ec();
  d.n_targets = f.num_targets();
  d.ec_off = ix->ec_off.p;
  d.ec_handle = ix->ec_handle.p;
  d.blk_ec = ix->blk_ec.p;
  d.blk_strand_off = ix->blk_strand_off.p;
  d.strand = ix->strand.p;
  d.fp_info = f.has_positions ? ix->fp_info.p : nullptr;
  d.blk_usize = f.has_positions ? ix->blk_usize.p : nullptr;
  d.target_len = f.has_positions ? ix->target_len.p : nullptr;
  if (f.dlist_n) {
    // D-list k-mers: open-addressing set, built on the host (the list is a small fraction of the k-mer table)
    const uint64_t cap = pow2_ge(2 * f.dlist_n + 16);
    std::vector<unsigned long long> tab(cap, ~0ULL);
    for (uint64_t km : f.dlist) {
      uint64_t h = kb_mix64(km) & (cap - 1);
      while (tab[h] != ~0ULL && tab[h] != km) h = (h + 1) & (cap - 1);
      tab[h] = km;
    }
    ix->dfk.upload(tab.data(), cap, st);
    KB_CK(cudaStreamSynchronize(st));
    d.dfk = ix->dfk.p;
    d.dfk_mask = cap - 1;
  }
  ix->build_seconds = now_s() - t1;
  return ix;
}

// ------------------------------------------------------------------------------------------
// Quant
// ------------------------------------------------------------------------------------------
Quant::Quant(Index& ix, const QuantOptions& opt) : ix_(ix), opt_(opt), flens_(1000, 0) {
  if (ix.flat.graphless) throw Error("kallisto_b200: this index has no k-mers (an index.saved written by `bus`): only quant-tcc can use it");
  if (!ix_.ws_in_use) {   // borrow the index's work buffers
    ix_.ws_in_use = true;
    if (!ix_.shared_emws) ix_.shared_emws = new EmWs();
    bws_ = &ix_.shared_bws;
    emws_ = ix_.shared_emws;
  } else {
    own_ws_ = true;
    bws_ = new BatchWs();
    emws_ = new EmWs();
  }
  if (opt_.fp_fl >= 0 && !ix_.flat.has_positions)
    throw Error("kallisto_b200: the fragment-position filter needs an index loaded with positions (load_positions = 1)");
  if (const char* s = getenv("KB_REFILL_MIN")) opt_.refill_min = std::max(1, std::min(32, atoi(s)));   // tuning knob
  KB_CK(cudaSetDevice(ix_.device));
  KB_CK(cudaStreamCreateWithFlags(&stream_, cudaStreamNonBlocking));
  KB_CK(cudaStreamCreateWithFlags(&copy_stream_, cudaStreamNonBlocking));
  for (int i = 0; i < 2; ++i) {
    KB_CK(cudaEventCreateWithFlags(&ev_copied_[i], cudaEventDisableTiming));
    KB_CK(cudaEventCreateWithFlags(&ev_done_[i], cudaEventDisableTiming));
    KB_CK(cudaStreamCreateWithFlags(&bstream_[i], cudaStreamNonBlocking));
    KB_CK(cudaEventCreateWithFlags(&ev_packed_[i], cudaEventDisableTiming));
    KB_CK(cudaEventCreateWithFlags(&ev_last_[i], cudaEventDisableTiming));
  }
  KB_CK(cudaEventCreateWithFlags(&ev_fork_, cudaEventDisableTiming));
  cudaStream_t st = stream_;
  apply_l2_window();
  const uint64_t nE = ix_.flat.n_ec();
  // pools and tables of this run
  const uint64_t pool_cap =
      std::min<uint64_t>(0xFFFFFFF0ull, (uint64_t)ix_.n_index_tids + std::max<uint64_t>(1u << 24, 4ull * ix_.n_index_tids));
  pool_.alloc(pool_cap);
  KB_CK(cudaMemcpyAsync(pool_.p, ix_.index_pool.p, (size_t)ix_.n_index_tids * 4, cudaMemcpyDeviceToDevice, st));
  dslots_.alloc(ix_.dict_cap);
  KB_CK(cudaMemcpyAsync(dslots_.p, ix_.dslots_init.p, ix_.dict_cap * 8, cudaMemcpyDeviceToDevice, st));
  count_.alloc(ix_.dict_cap);
  count_.zero(st);
  first_.alloc(ix_.dict_cap);
  launch_fill_u64(first_.p, ix_.dict_cap, ~0ULL, st);
  const uint64_t m2_cap = pow2_ge(nE * 8 + (1u << 20));
  const uint64_t mn_cap = pow2_ge(nE * 4 + (1u << 20));
  m2_.alloc(m2_cap);
  launch_fill_memo2(m2_.p, m2_cap, st);
  mn_key_.alloc(mn_cap);
  launch_fill_u64(mn_key_.p, mn_cap, ~0ULL, st);
  mn_val_.alloc(mn_cap);
  launch_fill_i32(mn_val_.p, mn_cap, KB_H_NOTREADY, st);
  const uint64_t tpool_cap = mn_cap * 8;
  tpool_.alloc(tpool_cap);
  // pool_top, tpool_top and the statistics live in separate 128-byte lines: atomics on one line are served one after
  // the other by the L2, and resolve_kernel allocates from both pools once per fragment (with the counters side by
  // side, and a statistics increment per fragment on the same line, those atomics were 30 % of the kernel's time)
  counters_.alloc(48);
  {
    unsigned long long init[48] = {};
    init[0] = ix_.n_index_tids;
    KB_CK(cudaMemcpyAsync(counters_.p, init, sizeof(init), cudaMemcpyHostToDevice, st));
    KB_CK(cudaStreamSynchronize(st));   // init is a stack array
  }
  error_.alloc(1);
  error_.zero(st);

  dd_.pool = pool_.p; dd_.pool_top = counters_.p + 0; dd_.pool_cap = pool_cap;
  dd_.dslots = dslots_.p; dd_.dmask = ix_.dict_cap - 1;
  dd_.count = count_.p; dd_.first = first_.p;
  dd_.m2 = m2_.p; dd_.m2_mask = m2_cap - 1;
  dd_.mn_key = mn_key_.p; dd_.mn_val = mn_val_.p; dd_.mn_mask = mn_cap - 1;
  dd_.tpool = tpool_.p; dd_.tpool_top = counters_.p + 16; dd_.tpool_cap = tpool_cap;
  dd_.error = error_.p; dd_.stats = counters_.p + 32;

  // batch work buffers, both slots (BatchSlot)
  const uint32_t max_frag = opt_.max_batch_reads;
  int sms = 0, tpsm = 0;
  KB_CK(cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, ix_.device));
  KB_CK(cudaDeviceGetAttribute(&tpsm, cudaDevAttrMaxThreadsPerMultiProcessor, ix_.device));
  for (BatchSlot& w : bws_->slot) {
    w.d_handles.grow(max_frag);
    w.d_tl.grow(max_frag);
    w.d_counters.grow(KB_BATCH_COUNTER_WORDS);
    w.d_qentries.grow((size_t)max_frag * KB_Q_STRIDE);
    w.d_rlen.grow(2 * (size_t)max_frag);
    // rare path: fragments with more than KB_MAX_E distinct EC sets (spill area per resident lane + wide queue)
    w.d_qbig.grow((size_t)KB_QBIG_CAP * KB_QBIG_STRIDE);
    w.d_spill.grow((size_t)sms * (size_t)tpsm * KB_SPILL);
  }
  // resolve-kernel scratch: 2 x max_set_len words per lane group, at most ~0.5 GiB per slot
  {
    const char* e = getenv("KB_RESOLVE_G");
    const int g = e ? atoi(e) : 32;
    resolve_group_ = (g == 4 || g == 8 || g == 16 || g == 32) ? (uint32_t)g : 32u;
  }
  const uint64_t stride = std::max<uint64_t>(64, 2ull * ix_.max_set_len);
  uint64_t warps = (1ull << 27) / stride;
  // the kernel is latency-bound: fill the SMs (32 warps each), every warp split into 32 / group lane groups
  warps = std::min<uint64_t>((uint64_t)device_sm_count() * 32 * (32 / resolve_group_), std::max<uint64_t>(64, warps));
  n_resolve_warps_ = (uint32_t)(warps / 16 * 16);
  for (BatchSlot& w : bws_->slot) w.d_scratch.grow((size_t)n_resolve_warps_ * stride);
  scratch_stride_ = (uint32_t)stride;
  // EM workspace: sized once per index for the EC tables runs on it normally end with (twice the index's own sets),
  // so that the timed EM tail of a run does not allocate; it still grows on demand
  if (!opt_.bus) reserve_em(2 * (size_t)nE + (1u << 16), 4 * (size_t)ix_.n_index_tids + (1u << 20));
  KB_CK(cudaStreamSynchronize(st));
}

void Quant::reserve_em(size_t n_ecs, size_t nnz) {
  KB_CK(cudaSetDevice(ix_.device));
  EmWs& w = *emws_;
  const uint32_t T = ix_.flat.num_targets();
  w.reserve_numbering(ix_.dict_cap, n_ecs, 0.0);
  w.ec_tid.grow(std::max<size_t>(1, nnz));
  w.reserve_matrices(n_ecs, T, n_ecs, nnz, 0.0);
  w.comp(T, (uint32_t)std::min<size_t>(n_ecs, UINT32_MAX - 1), nnz, 10000, nullptr);
}

void EmWs::reserve_numbering(size_t dict_cap, size_t n, double slack) {
  const size_t n1 = n + 1;      // the scans run over n + 1 items
  used.grow(dict_cap); scal.grow(8);
  key_in.grow(n1, slack); key_out.grow(n1, slack);
  for (auto* b : {&idx_in, &order, &handle, &count, &len, &multi_len, &is_multi, &ec_off, &m_off, &multi_index, &minkey})
    b->grow(n1, slack);
  tmp.grow(emprep_sort_bytes((uint32_t)n1, 0));
}

void EmWs::reserve_matrices(size_t n, uint32_t T, size_t n_multi, size_t nnz, double slack) {
  const size_t n1 = n + 1, t1 = (size_t)T + 1, nz = std::max<size_t>(1, nnz);
  tmp.grow(emprep_sort_bytes((uint32_t)n1, (uint32_t)std::max(nnz, t1)));
  for (auto* b : {&ckey, &cval, &ckey_out}) b->grow(n1, slack);
  rlen.grow(n1 + 1, slack); multi_ec.grow(n_multi + 1, slack); m_rowoff.grow(n_multi + 2, slack);
  for (auto* b : {&m_tid, &m_row, &m_iota, &sortv, &t_midx}) b->grow(nz, slack);
  k64_in.grow(nz, slack); k64_out.grow(nz, slack);
  m_w.grow(nz, slack); t_w.grow(nz, slack); eff.grow(T, slack);
  t_deg.grow(t1, slack); t_off.grow(t1, slack); t_single.grow(T, slack);
  em.reserve(1, T, n_multi);
}

EmCompWs EmWs::comp(uint32_t T, uint32_t R, size_t nnz, int max_iter, const double* eff) {
  const size_t t1 = (size_t)T + 1, r1 = (size_t)R + 1, nz = std::max<size_t>(1, nnz);
  const size_t slices = (size_t)device_sm_count() + 1;
  c_parent.grow(t1); c_rfirst.grow(t1); c_iota.grow(std::max(t1, r1)); c_tkey.grow(t1); c_tid.grow(t1); c_tloc.grow(t1);
  c_rcomp.grow(r1); c_rkey.grow(r1); c_rid.grow(r1); c_rloc.grow(r1); c_rcnt.grow(r1); c_rlen.grow(r1); c_roff.grow(r1);
  c_tlen.grow(t1); c_toff.grow(t1); c_st0.grow(slices); c_sr0.grow(slices);
  c_csize.grow(t1); c_cstart.grow(t1); c_tsize.grow(t1); c_tscan.grow(t1); c_stats.grow(8);
  c_rtid.grow(nz); c_trow.grow(nz); c_rw.grow(nz); c_tw.grow(nz); c_tsingle.grow(t1); c_teff.grow(t1);
  c_sync.grow(2 * (size_t)std::max(1, max_iter));
  c_tmp.grow(emcomp_tmp_bytes(T, R));
  EmCompWs c{};
  c.parent = c_parent.p; c.rfirst = c_rfirst.p; c.csize = c_csize.p; c.cstart = c_cstart.p; c.iota = c_iota.p;
  c.tkey = c_tkey.p; c.t_id = c_tid.p; c.tloc = c_tloc.p; c.tsize = c_tsize.p; c.tscan = c_tscan.p;
  c.rcomp = c_rcomp.p; c.rkey = c_rkey.p; c.r_id = c_rid.p; c.rloc = c_rloc.p; c.r_cnt = c_rcnt.p; c.r_len = c_rlen.p;
  c.r_off = c_roff.p; c.r_tid = c_rtid.p; c.r_w = c_rw.p; c.t_single = c_tsingle.p; c.t_len = c_tlen.p; c.t_off = c_toff.p;
  c.t_row = c_trow.p; c.t_w = c_tw.p; c.s_t0 = c_st0.p; c.s_r0 = c_sr0.p; c.stats = c_stats.p; c.sync = c_sync.p;
  c.eff = eff; c.t_eff = c_teff.p;
  c.sync_rounds = (int)(c_sync.n / 2);
  c.max_slices = (int)(std::min(c_st0.n, c_sr0.n) - 1);
  c.tmp = c_tmp.p;
  c.tmp_bytes = c_tmp.n;
  return c;
}

Quant::~Quant() {
  for (cudaStream_t b : bstream_)
    if (b) cudaStreamSynchronize(b);
  if (stream_) cudaStreamSynchronize(stream_);
  if (own_ws_) { delete emws_; delete bws_; } else { ix_.ws_in_use = false; }
  if (h_off_pinned_) cudaFreeHost(h_off_pinned_);
  if (h_grp_) cudaFreeHost(h_grp_);
  for (auto ev : events_) cudaEventDestroy(ev);
  for (int i = 0; i < 2; ++i) {
    if (ev_copied_[i]) cudaEventDestroy(ev_copied_[i]);
    if (ev_done_[i]) cudaEventDestroy(ev_done_[i]);
  }
  for (int i = 0; i < 2; ++i) {
    if (ev_packed_[i]) cudaEventDestroy(ev_packed_[i]);
    if (ev_last_[i]) cudaEventDestroy(ev_last_[i]);
    if (bstream_[i]) cudaStreamDestroy(bstream_[i]);
  }
  if (ev_fork_) cudaEventDestroy(ev_fork_);
  if (copy_stream_) cudaStreamDestroy(copy_stream_);
  if (stream_ && own_stream_) cudaStreamDestroy(stream_);
}

void Quant::set_stream(cudaStream_t st) {
  join();
  KB_CK(cudaStreamSynchronize(stream_));
  if (stream_ && own_stream_) cudaStreamDestroy(stream_);
  stream_ = st;
  own_stream_ = false;
  apply_l2_window();
}

// Kernels launched on the run's streams treat the presence filter as persisting in L2; everything else streams.  The
// window is a stream attribute: match_kernel runs on the internal streams, so they carry it too.
void Quant::apply_l2_window() {
  if (!ix_.filter.p || ix_.l2_persist_bytes == 0) return;
  int max_win = 0;
  cudaDeviceGetAttribute(&max_win, cudaDevAttrMaxAccessPolicyWindowSize, ix_.device);
  const size_t bytes = std::min<size_t>(ix_.filter.n * 4, (size_t)std::max(0, max_win));
  if (bytes == 0) return;
  cudaStreamAttrValue v{};
  v.accessPolicyWindow.base_ptr = (void*)ix_.filter.p;
  v.accessPolicyWindow.num_bytes = bytes;
  v.accessPolicyWindow.hitRatio = (float)std::min(1.0, (double)ix_.l2_persist_bytes / (double)bytes);
  v.accessPolicyWindow.hitProp = cudaAccessPropertyPersisting;
  v.accessPolicyWindow.missProp = cudaAccessPropertyStreaming;
  for (cudaStream_t s : {stream_, bstream_[0], bstream_[1]})
    if (cudaStreamSetAttribute(s, cudaStreamAttributeAccessPolicyWindow, &v) != cudaSuccess) cudaGetLastError();
}

Quant::Timings Quant::timings() {
  join();
  KB_CK(cudaStreamSynchronize(stream_));
  for (size_t i = 0; i + 3 < events_.size(); i += 4) {
    // with batches overlapping, each is a span on its own stream that other batches' kernels may share
    float a = 0, b = 0, c = 0;
    KB_CK(cudaEventElapsedTime(&c, events_[i], events_[i + 1]));
    KB_CK(cudaEventElapsedTime(&a, events_[i + 1], events_[i + 2]));
    KB_CK(cudaEventElapsedTime(&b, events_[i + 2], events_[i + 3]));
    tacc_.pack_ms += c;
    tacc_.match_ms += a;
    tacc_.resolve_ms += b;
    ++tacc_.match_launches;
    ++tacc_.resolve_launches;
  }
  for (auto ev : events_) cudaEventDestroy(ev);
  events_.clear();
  return tacc_;
}

void Quant::sync() {
  join();
  KB_CK(cudaStreamSynchronize(stream_));
}

void Quant::join() {
  if (!pending_) return;
  for (cudaEvent_t e : ev_last_) KB_CK(cudaStreamWaitEvent(stream_, e, 0));
  pending_ = false;
}

void Quant::check_device_errors() {
  join();
  int herr = 0;
  error_.download(&herr, 1, 0, stream_);
  KB_CK(cudaStreamSynchronize(stream_));
  if (herr == 0) return;
  std::string m = "kallisto_b200: device-side failure:";
  if (herr & KB_DEVERR_POOL_FULL) m += " set pool exhausted;";
  if (herr & KB_DEVERR_DICT_FULL) m += " set dictionary full;";
  if (herr & KB_DEVERR_MEMO_FULL) m += " memo table full;";
  if (herr & KB_DEVERR_TPOOL_FULL) m += " tuple pool exhausted;";
  if (herr & KB_DEVERR_E_OVERFLOW) m += " a fragment hit more than 128 distinct EC sets, or more than 65536 fragments of a batch hit more than 16;";
  throw Error(m);
}

void Quant::run_batch(BatchArgs ba, uint32_t n_reads, uint32_t max_read_len) {
  const uint32_t n_frag = opt_.paired ? n_reads / 2 : n_reads;
  if (opt_.paired && (n_reads & 1)) throw Error("kallisto_b200: odd number of reads in a paired batch");
  const int b = (int)(n_batches_ & 1);
  BatchSlot& w = bws_->slot[b];
  if (n_frag > w.d_handles.n) throw Error("kallisto_b200: batch larger than max_batch_reads");
  if (n_frag == 0) return;
  // the batch runs on internal stream b, after what the caller enqueued on the run's stream so far; stream b last ran
  // batch i - 2, the one that used these buffers before
  const cudaStream_t bs = bstream_[b];
  ++n_batches_;
  last_slot_ = b;
  pending_ = true;
  KB_CK(cudaEventRecord(ev_fork_, stream_));
  KB_CK(cudaStreamWaitEvent(bs, ev_fork_, 0));
  ecs_valid_ = false;
  dev_stats_valid_ = false;
  dev_problem_valid_ = false;
  ba.n_frag = n_frag;
  ba.paired = opt_.paired;
  ba.strand_mode = aa_ ? 0 : opt_.strand_mode;     // --aa: the frames are matched unstranded, cfc_select_kernel filters the set
  ba.frag_base = have_frag_base_ ? frag_base_ : n_frag_total_;
  have_frag_base_ = false;
  ba.handle_out = w.d_handles.p;
  const bool want_fld = opt_.paired && opt_.collect_fld && tlencount_ < 10000;   // ProcessReads.cpp:981-1017
  ba.tl_out = want_fld ? w.d_tl.p : nullptr;
  ba.q_count = w.d_counters.p;
  ba.qbig_count = w.d_counters.p + KB_BATCH_COUNTER_LINE;
  ba.take = w.d_counters.p + 2 * KB_BATCH_COUNTER_LINE;
  ba.q_entries = w.d_qentries.p;
  ba.spill = w.d_spill.p;
  ba.qbig_entries = w.d_qbig.p;
  ba.qbig_cap = KB_QBIG_CAP;
  ba.nb = std::max<uint32_t>(1, (max_read_len + 31) / 32);
  ba.pstride = (3 * ba.nb + 7) & ~7u;
  {
    const size_t need = (size_t)n_reads * ba.pstride;
    if ((uint64_t)n_reads * ba.nb >= (1ull << 32))      // pack_kernel / dlist_scan_kernel index (read, word) with 32 bits
      throw Error("kallisto_b200: batch too large for its longest read (reads x ceil(max length / 32) must be < 2^32)");
    if (w.d_packed.n < need) w.d_packed.alloc(std::max(need, (size_t)opt_.max_batch_reads * 2 * 16));
    if (w.d_rlen.n < n_reads) w.d_rlen.alloc(n_reads);
  }
  ba.packed = w.d_packed.p;
  ba.rlen = w.d_rlen.p;
  ba.empty_ec = ix_.empty_ec;
  ba.refill_min = opt_.refill_min;
  ba.skip_w = nullptr;
  if (ix_.dev.dfk) {
    // D-list: fragments holding a distinguishing flanking k-mer are marked by dlist_scan_kernel (after packing)
    if (ba.skip) {
      ba.skip_w = const_cast<uint8_t*>(ba.skip);            // bus: the scan adds to the bad-barcode marks
    } else {
      if (w.d_skip.n < n_frag) w.d_skip.alloc(std::max<size_t>(n_frag, opt_.max_batch_reads));
      KB_CK(cudaMemsetAsync(w.d_skip.p, 0, n_frag, bs));
      ba.skip = ba.skip_w = w.d_skip.p;
    }
  }
  ba.fp_fl = opt_.fp_fl;
  ba.no_count = aa_ ? 1 : 0;
  ba.first_hit = aa_ ? cfc_first_.p : nullptr;
  ResolveArgs ra{};
  ra.scratch = w.d_scratch.p;
  ra.scratch_stride = scratch_stride_;
  ra.n_warps = n_resolve_warps_;
  ra.group = resolve_group_;

  int tpb = opt_.threads_per_block;
  const size_t per_thread = 4 * match_lane_words(ba.nb);   // match_kernel's shared memory per lane
  while (tpb > 32 && per_thread * tpb > 200 * 1024) tpb >>= 1;
  if (per_thread * tpb > 200 * 1024) throw Error("kallisto_b200: read too long for the short-read kernel");
  cudaEvent_t* ev = nullptr;
  if (timing_) {
    const size_t base = events_.size();
    events_.resize(base + 4);
    for (int i = 0; i < 4; ++i) KB_CK(cudaEventCreate(&events_[base + i]));
    ev = events_.data() + base;
  }
  launch_pseudoalign(ix_.dev, dd_, ba, ra, tpb, bs, ev, ev_packed_[b]);
  KB_CK(cudaGetLastError());
  // the caller may overwrite its input in its stream order once pack_kernel (and dlist_scan_kernel) have read it
  KB_CK(cudaStreamWaitEvent(stream_, ev_packed_[b], 0));
  n_kernel_launches += 3 + (ba.skip_w ? 1 : 0);   // pack_kernel, [dlist_scan_kernel,] match_kernel, resolve_kernel
  if (aa_) {
    launch_cfc_select(ix_.dev, dd_, ba, ra, n_frag / 6, opt_.strand_mode, cfc_handles_.p, cfc_clashes_.p, bs);
    KB_CK(cudaGetLastError());
    ++n_kernel_launches;
  }
  if (want_fld) launch_fld_finalize(dd_, ba, bs);
  KB_CK(cudaEventRecord(ev_last_[b], bs));
  if (want_fld) {
    ++n_kernel_launches;
    h_tl_.resize(n_frag);
    w.d_tl.download(h_tl_.data(), n_frag, 0, bs);
    KB_CK(cudaStreamSynchronize(bs));
    // first (10000 - tlencount) qualifying fragments of this batch, in read order
    int goal = 10000 - (int)tlencount_;
    uint32_t local = 0;
    for (uint32_t i = 0; i < n_frag && goal > 0; ++i) {
      const uint16_t tl = h_tl_[i];
      if (tl > 0) { ++flens_[tl]; tl_list_.push_back(tl); --goal; ++local; }
    }
    tlencount_ += local;
  }
  n_frag_total_ += aa_ ? n_frag / 6 : n_frag;     // --aa: read sets are counted, not their frames
}

void Quant::pseudoalign_device(const uint8_t* d_bases, const uint32_t* d_off, uint32_t n_reads, uint32_t fixed_len,
                               uint32_t max_read_len) {
  KB_CK(cudaSetDevice(ix_.device));
  BatchArgs in{};
  in.bases = d_bases;
  in.off = d_off;
  in.fixed_len = fixed_len;
  run_batch(in, n_reads, max_read_len);
}

Quant::Staged Quant::stage(int s, int nf, const char* const* bases, const uint32_t* const* offs, uint32_t n,
                           uint32_t fixed_len, uint64_t min_bases, size_t min_offs) {
  Staged g{};
  KB_CK(cudaStreamWaitEvent(copy_stream_, ev_done_[s], 0));      // kernels that last read this slot
  for (int k = 0; k < nf; ++k) {
    const uint32_t* off = offs[k];
    const uint64_t n_bases = off ? off[n] : (uint64_t)n * fixed_len;
    DBuf<uint8_t>& db = bws_->stage_b[s][k];
    if (db.n < n_bases + 16) { KB_CK(cudaStreamSynchronize(stream_)); db.alloc(std::max<uint64_t>(n_bases + 16, min_bases)); }
    KB_CK(cudaMemcpyAsync(db.p, bases[k], n_bases, cudaMemcpyHostToDevice, copy_stream_));
    g.bases[k] = db.p;
    g.maxlen[k] = fixed_len;
    if (off) {
      DBuf<uint32_t>& dofs = bws_->stage_o[s][k];
      if (dofs.n < (size_t)n + 1) { KB_CK(cudaStreamSynchronize(stream_)); dofs.alloc(std::max<size_t>((size_t)n + 1, min_offs)); }
      KB_CK(cudaMemcpyAsync(dofs.p, off, ((size_t)n + 1) * 4, cudaMemcpyHostToDevice, copy_stream_));
      g.off[k] = dofs.p;
      g.maxlen[k] = 0;
      for (uint32_t i = 0; i < n; ++i) g.maxlen[k] = std::max(g.maxlen[k], off[i + 1] - off[i]);
    }
  }
  KB_CK(cudaEventRecord(ev_copied_[s], copy_stream_));
  KB_CK(cudaStreamWaitEvent(stream_, ev_copied_[s], 0));
  return g;
}

void Quant::pseudoalign_staged(int nf, const char* const* bases, const uint32_t* const* offs, uint32_t n,
                               uint32_t fixed_len, int32_t* handles_out) {
  // batches alternate between the two staging slots, so that the copy of one overlaps the previous batch's kernels
  const int s = stage_idx_;
  stage_idx_ ^= 1;
  // first allocations: one buffer holds a whole batch, a mate's buffer half of it
  const Staged g = nf == 1 ? stage(s, 1, bases, offs, n, fixed_len, opt_.max_batch_bases, 2 * (size_t)opt_.max_batch_reads + 1)
                           : stage(s, 2, bases, offs, n, fixed_len, opt_.max_batch_bases / 2 + 16, (size_t)opt_.max_batch_reads + 1);
  BatchArgs in{};
  in.bases = g.bases[0];
  in.off = g.off[0];
  in.bases2 = g.bases[1];
  in.off2 = g.off[1];
  in.fixed_len = fixed_len;
  const uint32_t n_reads = (uint32_t)nf * n;
  run_batch(in, n_reads, std::max(g.maxlen[0], g.maxlen[1]));
  KB_CK(cudaEventRecord(ev_done_[s], stream_));
  if (handles_out) {
    join();
    bws_->slot[last_slot_].d_handles.download(handles_out, opt_.paired ? n_reads / 2 : n_reads, 0, stream_);
    KB_CK(cudaStreamSynchronize(stream_));
  } else {
    // the caller may reuse its buffers once the copy is done; the kernels keep running
    KB_CK(cudaEventSynchronize(ev_copied_[s]));
  }
}

void Quant::pseudoalign_host(const char* bases, const uint32_t* off, uint32_t n_reads, uint32_t fixed_len,
                             int32_t* handles_out) {
  KB_CK(cudaSetDevice(ix_.device));
  if (n_reads == 0) return;
  if (off && off[0] != 0) throw Error("kallisto_b200: offsets must start at 0");
  pseudoalign_staged(1, &bases, &off, n_reads, fixed_len, handles_out);
}

void Quant::pseudoalign_host_pe(const char* bases1, const uint32_t* off1, const char* bases2, const uint32_t* off2,
                                uint32_t n_pairs, uint32_t fixed_len, int32_t* handles_out) {
  KB_CK(cudaSetDevice(ix_.device));
  if (n_pairs == 0) return;
  if (!opt_.paired) throw Error("kallisto_b200: per-mate buffers need a paired run");
  if ((off1 == nullptr) != (off2 == nullptr)) throw Error("kallisto_b200: give offsets for both mates or for neither");
  const char* bases[2] = {bases1, bases2};
  const uint32_t* offs[2] = {off1, off2};
  pseudoalign_staged(2, bases, offs, n_pairs, fixed_len, handles_out);
}

void Quant::bus_batch_host(const char* const* bases, const uint32_t* const* offs, uint32_t n_sets, BusRecord* records_out,
                           uint32_t* n_records_out) {
  KB_CK(cudaSetDevice(ix_.device));
  if (!opt_.bus) throw Error("kallisto_b200: not a bus run");
  if (n_records_out) *n_records_out = 0;
  if (n_sets == 0) return;
  if (grp_pending_) throw Error("kallisto_b200: this bus run has a group batch outstanding");
  Staged g{};
  const uint32_t maxlen = bus_stage(bases, offs, n_sets, g);
  const uint32_t n_rec = bus_core(g.bases, g.off, n_sets, maxlen);
  if (n_rec && records_out) {
    bus_rec_.download(records_out, n_rec, 0, stream_);
    KB_CK(cudaStreamSynchronize(stream_));
  }
  if (n_records_out) *n_records_out = n_rec;
}

uint32_t Quant::bus_stage(const char* const* bases, const uint32_t* const* offs, uint32_t n_sets, Staged& g) {
  const BusSpec& sp = opt_.bus_spec;
  for (int k = 0; k < sp.nfiles; ++k)
    if (!bases[k] || !offs[k]) throw Error("kallisto_b200: bus batch needs bases and offsets for every file of the technology");
  // This path does not overlap batches, so it stages into slot 0 only, once the run's stream is done with the batch
  // before: bus_fields, cfc_frames and pack_kernel all read the staged files, and that batch may have failed part way.
  KB_CK(cudaEventRecord(ev_done_[0], stream_));
  g = stage(0, sp.nfiles, bases, offs, n_sets, 0, opt_.max_batch_bases / 2 + 16, (size_t)opt_.max_batch_reads + 1);
  // longest cDNA read of the batch (sizes the packed-read layout)
  return std::max(g.maxlen[sp.seq_file], sp.paired ? g.maxlen[sp.seq2_file] : 0u);
}

void Quant::bus_group_submit(const char* const* bases, const uint32_t* const* offs, uint32_t n_sets, uint64_t base,
                             uint64_t sample_base) {
  KB_CK(cudaSetDevice(ix_.device));
  if (!opt_.bus) throw Error("kallisto_b200: not a bus run");
  if (grp_pending_) throw Error("kallisto_b200: this group member has a batch outstanding");
  grp_n_ = n_sets;
  if (n_sets == 0) { grp_pending_ = true; return; }
  Staged g{};
  const uint32_t maxlen = bus_stage(bases, offs, n_sets, g);
  set_frag_base(base);                       // run_batch's first-occurrence keys: the run-wide index too
  grp_handles_ = bus_enqueue(g.bases, g.off, n_sets, maxlen, base, base - sample_base);
  cudaStream_t st = stream_;
  const size_t n1 = (size_t)n_sets + 1;
  auto grow = [&](auto& b, size_t need) { if (b.n < need) b.alloc(std::max<size_t>(need, (size_t)opt_.max_batch_reads + 1)); };
  grow(grp_len_, n1); grow(grp_eoff_, n1); grow(grp_off_, n1); grow(grp_tid_, 1);
  if (!h_grp_) KB_CK(cudaMallocHost((void**)&h_grp_, 8 * sizeof(unsigned long long)));
  launch_bus_new_sets(dd_, grp_handles_, n_sets, base, bus_isnew_.p, bus_newrank_.p, bus_ismapped_.p, bus_rank_.p,
                      grp_len_.p, grp_eoff_.p, (uint32_t)std::min<size_t>(grp_tid_.n, 0xFFFFFFFFu), grp_off_.p, grp_tid_.p,
                      bus_tmp_.p, bus_tmp_.n, st);
  KB_CK(cudaGetLastError());
  n_kernel_launches += 4;      // bus_fields, bus_newflag, bus_newlen, bus_export
  // the batch's totals, read by bus_group_new_sets: n_new, entries, records, valid sets, long barcodes
  uint32_t* h32 = reinterpret_cast<uint32_t*>(h_grp_);
  KB_CK(cudaMemcpyAsync(h32 + 0, bus_newrank_.p + n_sets, 4, cudaMemcpyDeviceToHost, st));
  KB_CK(cudaMemcpyAsync(h32 + 1, grp_eoff_.p + n_sets, 4, cudaMemcpyDeviceToHost, st));
  KB_CK(cudaMemcpyAsync(h32 + 2, bus_rank_.p + n_sets, 4, cudaMemcpyDeviceToHost, st));
  KB_CK(cudaMemcpyAsync(h_grp_ + 2, bus_nvalid_.p, 16, cudaMemcpyDeviceToHost, st));
  grp_pending_ = true;
  // the caller may reuse its buffers once the copy is done; the kernels keep running
  KB_CK(cudaEventSynchronize(ev_copied_[0]));
}

void Quant::bus_group_new_sets(std::vector<uint32_t>& off, std::vector<uint32_t>& tids) {
  if (!grp_pending_) throw Error("kallisto_b200: no group batch outstanding on this member");
  off.assign(1, 0);
  tids.clear();
  if (grp_n_ == 0) return;
  KB_CK(cudaSetDevice(ix_.device));
  cudaStream_t st = stream_;
  KB_CK(cudaStreamSynchronize(st));
  const uint32_t* h32 = reinterpret_cast<const uint32_t*>(h_grp_);
  const uint32_t n_new = h32[0], n_ent = h32[1];
  if (h_grp_[3]) {
    grp_pending_ = false;
    throw Error("kallisto_b200: --batch-barcodes: " + std::to_string(h_grp_[3]) + " read set(s) of this batch have a barcode of "
                "more than 32 letters, which cannot take the sample's number in front of it");
  }
  if (n_ent > grp_tid_.n) {       // the first gather ran out of room: gather again into a buffer of the right size
    grp_tid_.alloc((size_t)n_ent + n_ent / 4);
    launch_bus_export_gather(dd_, grp_handles_, grp_n_, bus_isnew_.p, bus_newrank_.p, grp_eoff_.p,
                             (uint32_t)std::min<size_t>(grp_tid_.n, 0xFFFFFFFFu), grp_off_.p, grp_tid_.p, st);
    KB_CK(cudaGetLastError());
    ++n_kernel_launches;
  }
  off.resize((size_t)n_new + 1);
  tids.resize(n_ent);
  grp_off_.download(off.data(), (size_t)n_new + 1, 0, st);
  if (n_ent) grp_tid_.download(tids.data(), n_ent, 0, st);
  KB_CK(cudaStreamSynchronize(st));
}

void Quant::bus_group_finish(const int32_t* gid, BusRecord* records_out, uint32_t* n_records_out) {
  if (!grp_pending_) throw Error("kallisto_b200: no group batch outstanding on this member");
  grp_pending_ = false;
  if (n_records_out) *n_records_out = 0;
  if (grp_n_ == 0) return;
  KB_CK(cudaSetDevice(ix_.device));
  cudaStream_t st = stream_;
  const uint32_t* h32 = reinterpret_cast<const uint32_t*>(h_grp_);
  const uint32_t n_new = h32[0], n_rec = h32[2];
  grp_gid_.grow(std::max<size_t>(1, n_new), 0.25);
  if (n_new) grp_gid_.upload(gid, n_new, st);
  launch_bus_group_records(grp_handles_, grp_n_, bus_isnew_.p, bus_newrank_.p, grp_gid_.p, bus_idof_.p, bus_ismapped_.p,
                           bus_rank_.p, (const uint64_t*)bus_bc_.p, (const uint64_t*)bus_umi_.p, bus_flags_.p, bus_rec_.p, st);
  KB_CK(cudaGetLastError());
  n_kernel_launches += 2;      // bus_newid_gid, bus_records
  if (n_rec && records_out) bus_rec_.download(records_out, n_rec, 0, st);
  KB_CK(cudaStreamSynchronize(st));
  bus_valid_total_ += h_grp_[2];
  if (n_records_out) *n_records_out = n_rec;
}

// Same with the files of the batch already resident in device memory; the records stay on the device
// (bus_records_device(), valid until the next batch).
uint32_t Quant::bus_batch_device(const uint8_t* const* d_bases, const uint32_t* const* d_offs, uint32_t n_sets,
                                 uint32_t max_seq_len) {
  KB_CK(cudaSetDevice(ix_.device));
  if (!opt_.bus) throw Error("kallisto_b200: not a bus run");
  if (n_sets == 0) return 0;
  for (int k = 0; k < opt_.bus_spec.nfiles; ++k)
    if (!d_bases[k] || !d_offs[k]) throw Error("kallisto_b200: bus batch needs bases and offsets for every file of the technology");
  return bus_core(d_bases, d_offs, n_sets, max_seq_len);
}

uint32_t Quant::bus_core(const uint8_t* const* db, const uint32_t* const* dofs, uint32_t n_sets, uint32_t maxlen) {
  cudaStream_t st = stream_;
  const uint64_t base = n_frag_total_;
  // --num: read numbers restart with every sample (one reader per batch)
  const int32_t* handles = bus_enqueue(db, dofs, n_sets, maxlen, base, n_frag_total_ - bus_sample_base_);
  launch_bus_records(dd_, handles, n_sets, base, bus_next_id_, bus_idof_.p, bus_isnew_.p, bus_newrank_.p,
                     bus_ismapped_.p, bus_rank_.p, (const uint64_t*)bus_bc_.p, (const uint64_t*)bus_umi_.p, bus_flags_.p,
                     bus_rec_.p, bus_tmp_.p, bus_tmp_.n, st);
  KB_CK(cudaGetLastError());
  n_kernel_launches += 4;      // bus_fields, bus_newflag, bus_newid, bus_records (CUB scans not counted)
  uint32_t n_new = 0, n_rec = 0;
  unsigned long long n_valid[2] = {0, 0};
  bus_newrank_.download(&n_new, 1, n_sets, st);
  bus_rank_.download(&n_rec, 1, n_sets, st);
  bus_nvalid_.download(n_valid, 2, 0, st);
  KB_CK(cudaStreamSynchronize(st));
  if (n_valid[1])
    throw Error("kallisto_b200: --batch-barcodes: " + std::to_string(n_valid[1]) + " read set(s) of this batch have a barcode of "
                "more than 32 letters, which cannot take the sample's number in front of it");
  bus_next_id_ += n_new;
  bus_valid_total_ += n_valid[0];
  return n_rec;
}

const int32_t* Quant::bus_enqueue(const uint8_t* const* db, const uint32_t* const* dofs, uint32_t n_sets, uint32_t maxlen,
                                  uint64_t base, uint64_t set_base) {
  const BusSpec& sp = opt_.bus_spec;
  cudaStream_t st = stream_;
  BusArgs a{};
  for (int k = 0; k < sp.nfiles; ++k) { a.bases[k] = db[k]; a.off[k] = dofs[k]; }
  const size_t n1 = (size_t)n_sets + 1;
  auto grow = [&](auto& b, size_t need) { if (b.n < need) b.alloc(std::max<size_t>(need, (size_t)opt_.max_batch_reads + 1)); };
  grow(bus_bc_, n1); grow(bus_umi_, n1); grow(bus_flags_, n1); grow(bus_skip_, n1);
  if (sp.tag_len) grow(bus_notag_, n1);
  grow(bus_isnew_, n1); grow(bus_newrank_, n1); grow(bus_ismapped_, n1); grow(bus_rank_, n1); grow(bus_rec_, n1);
  if (bus_hist_.n < 66) { bus_hist_.alloc(66); bus_hist_.zero(st); }
  bus_nvalid_.grow(2);      // [0] valid read sets, [1] --batch-barcodes sets with more than 32 barcode letters
  if (bus_idof_.n < ix_.dict_cap) { bus_idof_.alloc(ix_.dict_cap); launch_fill_i32(bus_idof_.p, ix_.dict_cap, -1, st); }
  const size_t tb = bus_scan_bytes(n_sets);
  if (bus_tmp_.n < tb) bus_tmp_.alloc(std::max(tb, bus_scan_bytes(opt_.max_batch_reads)));
  bus_nvalid_.zero(st);
  a.n_sets = n_sets;
  a.set_base = set_base;
  a.spec = sp;
  a.barcode = (uint64_t*)bus_bc_.p; a.umi = (uint64_t*)bus_umi_.p; a.flags = bus_flags_.p; a.skip = bus_skip_.p;
  a.notag = sp.tag_len ? bus_notag_.p : nullptr;
  a.bc_hist = bus_hist_.p; a.umi_hist = bus_hist_.p + 33; a.n_valid = bus_nvalid_.p; a.n_long_bc = bus_nvalid_.p + 1;
  launch_bus_fields(a, st);
  KB_CK(cudaGetLastError());
  // the cDNA read(s): single-read or paired pseudoalignment with the strand filter of the technology
  BatchArgs in{};
  in.bases = db[sp.seq_file];
  in.off = dofs[sp.seq_file];
  in.start = (uint32_t)sp.seq_start;
  in.skip = bus_skip_.p;
  uint32_t min_start = (uint32_t)(sp.paired ? std::min(sp.seq_start, sp.seq2_start) : sp.seq_start);
  if (sp.tag_len) {
    // a read set without the tag has no UMI: the sequence read that shares the UMI's file starts where the tag would
    // have started (src/ProcessReads.cpp:1547,1553-1554), the other one where the technology says
    const int at = sp.umi_a[0] - sp.tag_len;
    in.notag = bus_notag_.p;
    in.alt_start = (uint32_t)(sp.umi_f[0] == sp.seq_file ? at : sp.seq_start);
    in.alt_start2 = (uint32_t)(sp.paired && sp.umi_f[0] == sp.seq2_file ? at : sp.seq2_start);
    min_start = std::min(min_start, sp.paired ? std::min(in.alt_start, in.alt_start2) : in.alt_start);
  }
  maxlen = maxlen > min_start ? maxlen - min_start : 1;
  if (aa_) {
    // the six reading frames of every set in comma-free code (kernels_cfc.cu), 6 n_sets unpaired fragments; a skipped
    // set has empty frames
    const uint64_t bound = 6ull * n_sets * maxlen;
    if (bound >= (1ull << 32)) throw Error("kallisto_b200: bus --aa batch too large (6 x read sets x longest read must be < 2^32)");
    auto grow_to = [&](auto& b, size_t need, size_t dflt) { if (b.n < need) b.alloc(std::max(need, dflt)); };
    grow_to(cfc_b_, bound + 16, 0);
    grow_to(cfc_o_, 6 * (size_t)n_sets + 1, 6 * (size_t)opt_.max_batch_reads + 1);
    grow_to(cfc_first_, 6 * (size_t)n_sets, 6 * (size_t)opt_.max_batch_reads);
    grow_to(cfc_set_off_, n1, (size_t)opt_.max_batch_reads + 1);
    grow_to(cfc_handles_, n1, (size_t)opt_.max_batch_reads + 1);
    grow_to(cfc_tmp_, cfc_scan_bytes(n_sets), cfc_scan_bytes(opt_.max_batch_reads));
    CfcArgs c{};
    c.bases = db[sp.seq_file];
    c.off = dofs[sp.seq_file];
    c.start = (uint32_t)sp.seq_start;
    c.skip = bus_skip_.p;
    c.n_sets = n_sets;
    c.max_len = maxlen;
    c.set_off = cfc_set_off_.p;
    c.fbases = cfc_b_.p;
    c.foff = cfc_o_.p;
    c.tmp = cfc_tmp_.p;
    c.tmp_bytes = cfc_tmp_.n;
    launch_cfc_frames(c, st);
    KB_CK(cudaGetLastError());
    n_kernel_launches += 2;      // cfc_len, cfc_frames
    BatchArgs fr{};              // the frames, from their first base and without skip marks: a skipped set's are empty
    fr.bases = cfc_b_.p;
    fr.off = cfc_o_.p;
    run_batch(fr, 6 * n_sets, maxlen);
  } else if (sp.paired) {
    // two sequence reads (busopt.paired, src/ProcessReads.cpp:1550-1567,1646-1650): the pair goes through the same
    // match x 2 / intersectKmers / strand filter / mapPair path as `quant` (one buffer per mate)
    in.bases2 = db[sp.seq2_file];
    in.off2 = dofs[sp.seq2_file];
    in.start2 = (uint32_t)sp.seq2_start;
    run_batch(in, 2 * n_sets, maxlen);
  } else {
    run_batch(in, n_sets, maxlen);
  }
  // the records need the whole batch, and the batch's read-set fields (barcodes, skip and tag marks) are rewritten by
  // the next one: this path does not overlap batches
  join();
  return aa_ ? cfc_handles_.p : bws_->slot[last_slot_].d_handles.p;
}

void Quant::bus_begin_sample(uint64_t barcode) {
  if (!opt_.bus) throw Error("kallisto_b200: not a bus run");
  if (opt_.bus_spec.n_bc == 0) opt_.bus_spec.fake_bc = barcode;
  else opt_.bus_spec.bc_prefix = barcode;      // in front of the barcode only with --batch-barcodes (batch_bc)
  bus_sample_base_ = n_frag_total_;
  // per-sample fragment-length histogram and quota (batchFlens[id] / tlencounts[id], src/ProcessReads.cpp:486-493)
  std::fill(flens_.begin(), flens_.end(), 0u);
  tl_list_.clear();
  tlencount_ = 0;
}

void Quant::set_batch_barcodes(bool on) {
  if (!opt_.bus) throw Error("kallisto_b200: --batch-barcodes needs a bus run");
  if (n_frag_total_ != 0) throw Error("kallisto_b200: --batch-barcodes must be chosen before the first batch");
  const BusSpec& sp = opt_.bus_spec;
  if (on && sp.n_bc > 0) {
    int fixed = 0;      // letters of the pieces with a stop; a piece to the end of its read adds to them
    for (int p = 0; p < sp.n_bc; ++p)
      if (sp.bc_b[p] != 0) fixed += sp.bc_b[p] - sp.bc_a[p];
    // the reference forms a barcode of 32 - blen batch letters there, with 32 - blen wrapped around (size_t)
    if (fixed > 32)
      throw Error("kallisto_b200: --batch-barcodes needs a barcode of at most 32 letters; the technology's has " +
                  std::to_string(fixed));
  }
  // a technology without a barcode read takes the sample's number as its barcode (kb_bus_begin_sample) either way
  opt_.bus_spec.batch_bc = (on && sp.n_bc > 0) ? 1 : 0;
}

void Quant::set_aa(bool on) {
  KB_CK(cudaSetDevice(ix_.device));
  if (!opt_.bus) throw Error("kallisto_b200: --aa needs a bus run");
  if (n_frag_total_ != 0) throw Error("kallisto_b200: --aa must be chosen before the first batch");
  if (on) {
    if (opt_.paired || opt_.bus_spec.paired)
      throw Error("kallisto_b200: --aa translates single-end reads only; a paired technology or --paired is not supported");
    if (opt_.bus_spec.tag_len) throw Error("kallisto_b200: --aa with a UMI tag sequence (--tag) is not supported");
    if (ix_.dev.dfk)
      throw Error("kallisto_b200: --aa with an index that has a D-list is not supported: there the reference keeps the off-list "
                  "target in every frame's intersection (dfk_onlist), which makes the result depend on the order of the hits");
    // 6 frames per read set go through the pseudoalignment buffers
    const size_t frames = 6 * (size_t)opt_.max_batch_reads;
    for (BatchSlot& w : bws_->slot) {
      w.d_handles.grow(frames);
      w.d_qentries.grow(frames * KB_Q_STRIDE);
      w.d_rlen.grow(frames);
    }
    cfc_clashes_.grow(1);
    cfc_clashes_.zero(stream_);
  }
  aa_ = on;
}

uint64_t Quant::frame_clashes() {
  unsigned long long c = 0;
  join();
  if (aa_) {
    cfc_clashes_.download(&c, 1, 0, stream_);
    KB_CK(cudaStreamSynchronize(stream_));
  }
  return c;
}

void Quant::bus_lengths(uint32_t* bc_hist, uint32_t* umi_hist) {
  uint32_t h[66] = {0};
  join();
  if (bus_hist_.n >= 66) {
    bus_hist_.download(h, 66, 0, stream_);
    KB_CK(cudaStreamSynchronize(stream_));
  }
  memcpy(bc_hist, h, 33 * 4);
  memcpy(umi_hist, h + 33, 33 * 4);
}

BusGroup::BusGroup(std::vector<Quant*> members) : m_(std::move(members)), busy_(m_.size(), false) {
  table_.off.assign(1, 0);
}

uint64_t BusGroup::submit(int member, const char* const* bases, const uint32_t* const* offs, uint32_t n_sets) {
  if (member < 0 || member >= (int)m_.size()) throw std::invalid_argument("kb_bus_group_submit: no such member");
  if (busy_[member]) throw std::invalid_argument("kb_bus_group_submit: the member has a batch outstanding; complete it first");
  // every member numbers read sets run-wide: the dictionary's first-occurrence keys and --num read numbers
  m_[member]->bus_group_submit(bases, offs, n_sets, n_sets_total_, sample_base_);
  busy_[member] = true;
  queue_.push_back(member);
  n_sets_total_ += n_sets;
  return next_ticket_++;
}

// The commit rule.  A set that is new run-wide in this batch is, among the sets new run-wide, in order of first
// occurrence within the batch, and it is new on the member too (an earlier batch on the member would have committed
// it); a set the member saw before keeps the id an earlier batch committed.  So handing out the next ids in the
// member's new_rank order, after every earlier ticket, gives the ids of one run fed the whole stream.
void BusGroup::complete(uint64_t ticket, BusRecord* records_out, uint32_t* n_records_out) {
  if (queue_.empty()) throw std::invalid_argument("kb_bus_group_complete: no batch outstanding");
  if (ticket != done_tickets_)
    throw std::invalid_argument("kb_bus_group_complete: ticket " + std::to_string(ticket) + " is not the oldest outstanding batch (" +
                                std::to_string(done_tickets_) + ")");
  const int d = queue_.front();
  queue_.erase(queue_.begin());
  busy_[d] = false;
  ++done_tickets_;
  Quant& q = *m_[d];
  std::vector<uint32_t> off, tids;
  q.bus_group_new_sets(off, tids);
  const size_t n_new = off.size() - 1;
  std::vector<int32_t> gid(n_new);
  std::vector<uint32_t> key;
  for (size_t i = 0; i < n_new; ++i) {
    key.assign(tids.begin() + off[i], tids.begin() + off[i + 1]);
    auto it = reg_.find(key);
    if (it == reg_.end()) {
      const int32_t id = (int32_t)(table_.off.size() - 1);
      table_.tid.insert(table_.tid.end(), key.begin(), key.end());
      table_.off.push_back(table_.tid.size());
      it = reg_.emplace(std::move(key), id).first;
      key = std::vector<uint32_t>();
    }
    gid[i] = it->second;
  }
  q.bus_group_finish(gid.data(), records_out, n_records_out);
}

void BusGroup::begin_sample(uint64_t barcode) {
  if (!queue_.empty()) throw std::invalid_argument("kb_bus_group_begin_sample: complete the outstanding batches first");
  for (Quant* q : m_) q->bus_begin_sample(barcode);
  sample_base_ = n_sets_total_;
}

const EcTable& BusGroup::ec_table() {
  const size_t n = table_.off.size() - 1;
  table_.count.assign(n, 0);
  std::vector<uint32_t> key;
  for (Quant* q : m_) {
    const EcTable& e = q->finalize_ecs();
    for (uint32_t i = 0; i < e.n(); ++i) {
      key.assign(e.tid.begin() + e.off[i], e.tid.begin() + e.off[i + 1]);
      auto it = reg_.find(key);
      if (it == reg_.end()) throw Error("kallisto_b200: a member's equivalence class was never committed to its group");
      table_.count[it->second] += e.count[i];
    }
  }
  return table_;
}

Stats BusGroup::stats() {
  Stats s;
  for (Quant* q : m_) {
    const Stats t = q->stats();
    s.n_processed += t.n_processed;
    s.n_pseudoaligned += t.n_pseudoaligned;
    s.n_unique += t.n_unique;
    s.n_probes += t.n_probes;
    s.n_slot_visits += t.n_slot_visits;
    s.n_resolved += t.n_resolved;
    s.n_memo_hits += t.n_memo_hits;
  }
  return s;
}

void Quant::set_flens(const uint32_t* f) {
  flens_.assign(f, f + 1000);
  tl_list_.clear();
  tlencount_ = 0;
  for (int i = 0; i < 1000; ++i) tlencount_ += flens_[i];
}

const EcTable& Quant::finalize_ecs() {
  if (ecs_valid_) return ecs_;
  uint32_t n = 0, n_entries = 0;
  export_prepare(&n, &n_entries);
  const EmWs& w = *emws_;
  // 32-bit offsets on the device (a set's offset into the pool is 32-bit, and the used sets are distinct sets of that
  // pool, so all their entries together fit), widened to EcTable's 64-bit ones here
  std::vector<uint32_t> off(n + 1, 0);
  ecs_ = EcTable();
  ecs_.tid.resize(n_entries);
  ecs_.count.resize(n);
  ecs_.handle.resize(n);
  if (n) {
    w.ec_off.download(off.data(), (size_t)n + 1, 0, stream_);
    w.ec_tid.download(ecs_.tid.data(), n_entries, 0, stream_);
    w.count.download(ecs_.count.data(), n, 0, stream_);
    w.handle.download(reinterpret_cast<uint32_t*>(ecs_.handle.data()), n, 0, stream_);
    KB_CK(cudaStreamSynchronize(stream_));
  }
  ecs_.off.assign(off.begin(), off.end());
  ecs_valid_ = true;
  return ecs_;
}

Stats Quant::stats() {
  Stats s;
  s.n_processed = n_frag_total_;   // bus: read sets with a bad barcode/UMI are skipped but still counted as processed (ProcessReads.cpp:1372)
  if (dev_stats_valid_) {   // computed on the device by run_em_device: no EC table on the host needed
    s.n_pseudoaligned = dev_pseudoaligned_;
    s.n_unique = dev_unique_;
  } else {
    const EcTable& e = finalize_ecs();
    for (uint32_t i = 0; i < e.n(); ++i) {
      s.n_pseudoaligned += e.count[i];
      if (e.off[i + 1] - e.off[i] == 1) s.n_unique += e.count[i];
    }
  }
  unsigned long long st[4];
  sync();
  KB_CK(cudaMemcpy(st, dd_.stats, sizeof(st), cudaMemcpyDeviceToHost));
  s.n_probes = st[0];
  s.n_resolved = st[1];
  s.n_memo_hits = st[2];
  s.n_slot_visits = st[3];
  return s;
}

// MinCollector::compute_mean_frag_lens_trunc (src/MinCollector.cpp:629-651) when fld_mean == 0,
// MinCollector::init_mean_fl_trunc + trunc_gaussian_fld (src/MinCollector.cpp:583-627,
// src/weights.cpp:248-296) otherwise.
std::vector<double> mean_fl_trunc_of(const uint32_t* flens, double fld_mean, double fld_sd) {
  const int MAXF = 1000;
  std::vector<double> out(MAXF, 0.0);
  if (fld_mean == 0.0) {
    std::vector<int> counts(MAXF, 0);
    std::vector<double> mass(MAXF, 0.0);
    counts[0] = (int)flens[0];
    for (size_t i = 1; i < (size_t)MAXF; ++i) {
      mass[i] = static_cast<double>(flens[i] * i) + mass[i - 1];
      counts[i] = (int)flens[i] + counts[i - 1];
      if (counts[i] > 0) out[i] = mass[i] / static_cast<double>(counts[i]);
    }
  } else {
    // trunc_gaussian_fld(0, MAX_FRAG_LEN, mean, sd), src/weights.cpp:248-271
    std::vector<double> mean_fl(MAXF, 0.0);
    double total_mass = 0.0, total_density = 0.0;
    for (size_t i = 0; i < (size_t)MAXF; ++i) {
      double x = static_cast<double>(0 + i);
      x = (x - fld_mean) / fld_sd;
      const double cur_density = std::exp(-0.5 * x * x) / fld_sd;
      total_mass += cur_density * i;
      total_density += cur_density;
      if (total_mass > 0) mean_fl[i] = total_mass / total_density;
    }
    out = mean_fl;
  }
  return out;
}

std::vector<double> Quant::mean_fl_trunc(double fld_mean, double fld_sd) const {
  return mean_fl_trunc_of(flens_.data(), fld_mean, fld_sd);
}

namespace {
int em_tpb() {
  if (const char* s = getenv("KB_EM_TPB")) return std::max(32, std::min(1024, atoi(s)));   // tuning knob
  return 1024;     // one block per SM: fewest participants in the grid barrier (20.8 vs 21.6 us per round with 4 x 256)
}

// get_frag_len_means + calc_eff_lens (src/weights.cpp:7-28,58-79)
std::vector<double> eff_lens(const FlatIndex& f, const std::vector<double>& fl_trunc) {
  const uint32_t T = f.num_targets();
  std::vector<double> eff(T);
  const double marginal = fl_trunc[999];
  for (uint32_t t = 0; t < T; ++t) {
    const double mean = f.target_len[t] >= 1000 ? marginal : fl_trunc[f.target_len[t]];
    const double len = static_cast<double>(f.target_len[t]);
    double e = len - mean + 1;
    if (e < 1.0) e = len;
    eff[t] = e;
  }
  return eff;
}

// The minstd_rand0 seeds of B bootstraps: the first B outputs of the 64-bit Mersenne Twister seeded with `seed`
// (src/main.cpp:2746-2752, 3125-3130), reduced as libstdc++'s linear_congruential_engine::seed reduces them.
std::vector<uint32_t> minstd_seeds(uint64_t seed, int B) {
  std::mt19937_64 rnd;
  rnd.seed(seed);
  std::vector<uint32_t> x0(B);
  for (uint32_t& x : x0) {
    x = (uint32_t)(rnd() % 2147483647ull);
    if (x == 0) x = 1;
  }
  return x0;
}

// Problems per EM launch: `fit` (what the caller's memory budget allows), or the positive value of the tuning knob
// `env`, clamped to [1, min(total, KB_EM_MAX_BATCH)].
uint64_t em_chunk(uint64_t fit, uint64_t total, const char* env) {
  if (const char* s = getenv(env)) { const long long v = atoll(s); if (v > 0) fit = (uint64_t)v; }
  return std::max<uint64_t>(1, std::min<uint64_t>({fit, total, (uint64_t)KB_EM_MAX_BATCH}));
}
struct StreamGuard {    // a private non-blocking stream, destroyed on every way out
  cudaStream_t s = nullptr;
  StreamGuard() { KB_CK(cudaStreamCreateWithFlags(&s, cudaStreamNonBlocking)); }
  ~StreamGuard() { if (s) cudaStreamDestroy(s); }
  StreamGuard(const StreamGuard&) = delete;
  StreamGuard& operator=(const StreamGuard&) = delete;
};
struct EventGuard {     // a timing event, destroyed on every way out
  cudaEvent_t e = nullptr;
  EventGuard() { KB_CK(cudaEventCreate(&e)); }
  ~EventGuard() { if (e) cudaEventDestroy(e); }
  EventGuard(const EventGuard&) = delete;
  EventGuard& operator=(const EventGuard&) = delete;
};
float elapsed_ms(const EventGuard& a, const EventGuard& b) {
  float ms = 0;
  KB_CK(cudaEventElapsedTime(&ms, a.e, b.e));
  return ms;
}

template <class T> void upload_new(DBuf<T>& d, const T* h, size_t n, cudaStream_t st) {
  d.alloc(std::max<size_t>(1, n));
  d.upload(h, n, st);
}

// The structure of an EC table given on the host (n_ec, ec_off, tids; EC ids = positions in the table), on the device:
// CSR of the multi-transcript ECs in EC-id order, CSC by transcript, singletons, and the (EC id, transcript) of every
// entry of both layouts, which launch_tcc_fill forms the weights from.  An EC without transcripts gets no row: it
// would add to no sum.  The transcript ids must have been checked against T.
struct EmShape {
  uint32_t n_ec = 0, n_targets = 0, n_multi = 0;
  uint64_t nnz = 0;
  DBuf<uint32_t> multi_ec, m_off, m_tid, m_ec, t_off, t_midx, t_ec, t_tid;
  DBuf<int32_t> t_single;

  void build(uint32_t nE, const uint64_t* ec_off, const uint32_t* tids, uint32_t T, cudaStream_t st) {
    std::vector<uint32_t> h_multi_ec, h_m_off{0}, h_m_tid, h_m_ec, h_t_off(T + 1, 0);
    std::vector<int32_t> h_single(T, -1);
    for (uint32_t e = 0; e < nE; ++e) {
      const uint64_t b = ec_off[e], n = ec_off[e + 1] - b;
      if (n == 1) h_single[tids[b]] = (int32_t)e;
      if (n < 2) continue;
      h_multi_ec.push_back(e);
      for (uint64_t j = 0; j < n; ++j) {
        h_m_tid.push_back(tids[b + j]);
        h_m_ec.push_back(e);
        ++h_t_off[tids[b + j] + 1];
      }
      h_m_off.push_back((uint32_t)h_m_tid.size());
    }
    n_ec = nE; n_targets = T;
    nnz = h_m_tid.size();
    n_multi = (uint32_t)h_multi_ec.size();
    for (uint32_t t = 0; t < T; ++t) h_t_off[t + 1] += h_t_off[t];
    std::vector<uint32_t> h_t_midx(nnz), h_t_ec(nnz), h_t_tid(nnz), fill(h_t_off.begin(), h_t_off.end() - 1);
    for (uint32_t r = 0; r < n_multi; ++r)
      for (uint32_t j = h_m_off[r]; j < h_m_off[r + 1]; ++j) {
        const uint32_t t = h_m_tid[j], at = fill[t]++;
        h_t_midx[at] = r; h_t_ec[at] = h_multi_ec[r]; h_t_tid[at] = t;
      }
    auto up = [&](DBuf<uint32_t>& d, const std::vector<uint32_t>& h) { upload_new(d, h.data(), h.size(), st); };
    up(multi_ec, h_multi_ec); up(m_off, h_m_off); up(m_tid, h_m_tid); up(m_ec, h_m_ec);
    up(t_off, h_t_off); up(t_midx, h_t_midx); up(t_ec, h_t_ec); up(t_tid, h_t_tid);
    upload_new(t_single, h_single.data(), T, st);
    KB_CK(cudaStreamSynchronize(st));     // the host vectors go out of scope
  }
  // the shared structure of an EmProblem; the weights are the caller's (shared by all problems unless it sets w_stride)
  EmProblem problem(int max_iter, int min_rounds) const {
    EmProblem p{};
    p.n_ec = n_ec; p.n_targets = n_targets; p.n_multi = n_multi;
    p.multi_ec = multi_ec.p; p.m_off = m_off.p; p.m_tid = m_tid.p;
    p.t_off = t_off.p; p.t_midx = t_midx.p; p.t_single = t_single.p;
    p.max_iter = max_iter; p.min_rounds = min_rounds;
    return p;
  }
  // weights of `nb` rows of counts (row_off: their nb + 1 offsets into ec_ids / vals) into counts / m_w / t_w
  TccFill fill(int nb, const unsigned long long* row_off, const uint32_t* ec_ids, const uint32_t* vals, uint32_t* counts,
               const double* eff, uint64_t eff_stride, double* m_w, double* t_w) const {
    TccFill f{};
    f.n_ec = n_ec; f.n_targets = n_targets; f.nb = (uint32_t)nb; f.row_off = row_off; f.ec_ids = ec_ids; f.vals = vals;
    f.counts = counts; f.nnz = nnz; f.m_ec = m_ec.p; f.m_tid = m_tid.p; f.t_ec = t_ec.p; f.t_tid = t_tid.p;
    f.eff = eff; f.eff_stride = eff_stride; f.m_w = m_w; f.t_w = t_w;
    return f;
  }
};
}  // namespace

void EmState::reserve(size_t nb, uint32_t T, size_t n_multi) {
  const size_t nm = nb * std::max<size_t>(1, n_multi);
  alpha.grow(nb * T); single_cnt.grow(nb * T); norm.grow(nm); cnt_row.grow(nm); bar.grow(1);
  if (cap < nb) {
    cap = nb;
    emi.alloc(2 * cap);
    chcount.alloc(2 * cap);
    h_emi.resize(2 * cap);
  }
}

int EmState::launch(EmProblem& p, int nb, const uint32_t* counts, int threads_per_block, cudaStream_t st,
                    const EmCompWs* cw, cudaEvent_t start, bool* comp_resident, const double* prior) {
  const uint32_t T = p.n_targets;
  reserve((size_t)nb, T, p.n_multi);
  launch_em_start(alpha.p, (uint32_t)nb, T, prior, 1.0 / T, st);   // priors, or the uniform start (EMAlgorithm.h:38)
  emi.zero(st);
  chcount.zero(st);
  p.nb = nb; p.counts = counts; p.alpha = alpha.p; p.norm = norm.p; p.cnt_row = cnt_row.p; p.single_cnt = single_cnt.p;
  p.rounds = emi.p; p.fstate = emi.p + cap; p.chcount = chcount.p; p.bar = bar.p;
  if (start) KB_CK(cudaEventRecord(start, st));
  const int blocks = launch_em(p, threads_per_block, st, cw, comp_resident);
  KB_CK(cudaGetLastError());
  return blocks;
}

void EmState::fetch(const EmProblem& p, double* alpha_out, int* rounds_out, cudaStream_t st) {
  const size_t T = p.n_targets;
  alpha.download(alpha_out, (size_t)p.nb * T, 0, st);
  emi.download(h_emi.data(), cap + p.nb, 0, st);
  KB_CK(cudaStreamSynchronize(st));
  for (int b = 0; b < p.nb; ++b) {
    rounds_out[b] = h_emi[b];
    if (h_emi[cap + b] == 3)   // stop detected on the last allowed iteration: zero small alphas (EMAlgorithm.h:213-216)
      for (size_t t = 0; t < T; ++t)
        if (alpha_out[b * T + t] < 1e-7 / 10.0) alpha_out[b * T + t] = 0.0;
  }
}

EmProblem EmWs::problem(uint32_t n_ec, uint32_t T, uint32_t n_multi, int max_iter, int min_rounds) const {
  EmProblem p{};
  p.n_ec = n_ec; p.n_targets = T; p.n_multi = n_multi;
  p.multi_ec = multi_ec.p; p.m_off = m_rowoff.p; p.m_tid = m_tid.p; p.m_w = m_w.p;
  p.t_off = t_off.p; p.t_midx = t_midx.p; p.t_w = t_w.p; p.t_single = t_single.p;
  p.max_iter = max_iter; p.min_rounds = min_rounds;
  return p;
}

EmResult Quant::run_em(const EcTable& ecs, const std::vector<double>& fl_trunc, int max_iter, int min_rounds) {
  KB_CK(cudaSetDevice(ix_.device));
  join();
  const FlatIndex& f = ix_.flat;
  const uint32_t T = f.num_targets(), nE = ecs.n();
  cudaStream_t st = stream_;
  EmResult r;
  r.eff_lens = eff_lens(f, fl_trunc);
  EmShape sh;
  sh.build(nE, ecs.off.data(), ecs.tid.data(), T, st);
  // calc_weights (src/weights.cpp:220-246) on the device: the table's counts are the one row launch_tcc_fill weights,
  // a count for every EC in id order.  The weights stay shared (w_stride == 0): the single-problem kernels take it.
  std::vector<uint32_t> ids(nE);
  std::iota(ids.begin(), ids.end(), 0u);
  const unsigned long long row[2] = {0, nE};
  DBuf<unsigned long long> d_row;
  DBuf<uint32_t> d_ids, d_val, d_counts;
  DBuf<double> d_eff, d_mw, d_tw;
  upload_new(d_row, row, 2, st); upload_new(d_ids, ids.data(), nE, st); upload_new(d_val, ecs.count.data(), nE, st);
  upload_new(d_eff, r.eff_lens.data(), T, st);
  d_counts.alloc(std::max<uint32_t>(1, nE));
  d_mw.alloc(std::max<uint64_t>(1, sh.nnz)); d_tw.alloc(std::max<uint64_t>(1, sh.nnz));
  launch_tcc_fill(sh.fill(1, d_row.p, d_ids.p, d_val.p, d_counts.p, d_eff.p, 0, d_mw.p, d_tw.p), st);
  KB_CK(cudaGetLastError());
  EmProblem p = sh.problem(max_iter, min_rounds);
  p.m_w = d_mw.p; p.t_w = d_tw.p;
  EventGuard e0, e1;
  const EmCompWs cw = emws_->comp(T, p.n_multi, sh.nnz, max_iter, d_eff.p);
  EmState s;
  last_em_comp_blocks = s.launch(p, 1, d_counts.p, 256, st, &cw, e0.e, &last_em_comp_resident, has_priors_ ? priors_.p : nullptr);
  KB_CK(cudaEventRecord(e1.e, st));
  r.alpha.resize(T);
  s.fetch(p, r.alpha.data(), &r.rounds, st);
  r.seconds = elapsed_ms(e0, e1) * 1e-3;
  last_em_seconds = r.seconds;
  return r;
}

void Quant::set_priors(const double* priors) {
  KB_CK(cudaSetDevice(ix_.device));
  has_priors_ = false;
  if (!priors) return;
  const uint32_t T = ix_.flat.num_targets();
  priors_.grow(std::max<uint32_t>(1, T));
  priors_.upload(priors, T, stream_);
  KB_CK(cudaStreamSynchronize(stream_));     // the caller's buffer may go away
  has_priors_ = true;
}

// Used handles, sorted by first occurrence; their lengths and offsets.  First-occurrence keys are distinct per set.
EcNumbering Quant::number_ecs() {
  join();
  cudaStream_t st = stream_;
  EmWs& w = *emws_;
  EcNumbering nu;
  w.reserve_numbering(ix_.dict_cap, 0, 0.0);      // `used` and the scalar; the rest once n is known
  launch_collect_used(dd_, w.used.p, w.scal.p, st);
  w.scal.download(&nu.n, 1, 0, st);
  KB_CK(cudaStreamSynchronize(st));
  const uint32_t n = nu.n;
  if (n == 0) return nu;
  w.reserve_numbering(ix_.dict_cap, n, 0.25);
  // the scans run over n + 1 items: the extra item must be zero
  KB_CK(cudaMemsetAsync(w.len.p + n, 0, 4, st));
  KB_CK(cudaMemsetAsync(w.multi_len.p + n, 0, 4, st));
  KB_CK(cudaMemsetAsync(w.is_multi.p + n, 0, 4, st));
  emprep_sort_by_first(dd_, w.used.p, n, w.key_in.p, w.key_out.p, w.idx_in.p, w.order.p, w.tmp.p, w.tmp.n, st);
  EmPrep& ep = nu.prep;
  ep.n_ec = n; ep.n_targets = ix_.flat.num_targets();
  ep.handle = w.handle.p; ep.count = w.count.p; ep.len = w.len.p; ep.ec_off = w.ec_off.p; ep.m_off = w.m_off.p;
  ep.multi_index = w.multi_index.p; ep.minkey = w.minkey.p;
  emprep_meta(dd_, w.used.p, w.order.p, n, ep, w.multi_len.p, w.is_multi.p, w.tmp.p, w.tmp.n, st);
  w.ec_off.download(&nu.n_entries, 1, n, st);
  w.m_off.download(&nu.multi_entries, 1, n, st);
  w.multi_index.download(&nu.n_multi, 1, n, st);
  KB_CK(cudaStreamSynchronize(st));
  return nu;
}

// The whole tail of `kallisto quant` without the EC table ever visiting the host: EC ids by first
// occurrence, CSR/CSC + weights on the device (kernels_emprep.cu), then em_kernel.
EmResult Quant::run_em_device(const std::vector<double>& fl_trunc, int max_iter, int min_rounds) {
  KB_CK(cudaSetDevice(ix_.device));
  check_device_errors();
  // the EM works out of L2: give it the part that the k-mer presence filter held as persisting lines during pseudoalignment
  if (ix_.l2_persist_bytes) cudaCtxResetPersistingL2Cache();
  const FlatIndex& f = ix_.flat;
  const uint32_t T = f.num_targets();
  cudaStream_t st = stream_;
  EmWs& w = *emws_;
  EmResult res;
  res.eff_lens = eff_lens(f, fl_trunc);
  const bool trace = getenv("KB_EM_TRACE") != nullptr;     // host wall clock of the set-up steps on stderr
  double t_last = now_s();
  auto mark = [&](const char* what) {
    if (!trace) return;
    const double t = now_s();
    fprintf(stderr, "[em-trace] %s: %.3f ms\n", what, (t - t_last) * 1e3);
    t_last = t;
  };
  EventGuard e0, e1, e2;
  KB_CK(cudaEventRecord(e0.e, st));
  mark("eff lens + events");
  const EcNumbering nu = number_ecs();
  mark("number ECs: drain stream, collect used handles, sort by first occurrence, scans");
  res.alpha.assign(T, 0.0);
  const uint32_t n = nu.n, nnz_all = nu.n_entries, nnz = nu.multi_entries, n_multi = nu.n_multi;
  if (n == 0) {
    res.rounds = 0;
    return res;
  }
  // ---- EC table, CSR, weights, CSC
  w.ec_tid.grow(std::max<uint32_t>(1, nnz_all), 0.25);
  w.reserve_matrices(n, T, n_multi, nnz, 0.25);
  mark("phase-2 buffers");
  KB_CK(cudaMemsetAsync(w.t_deg.p, 0, ((size_t)T + 1) * 4, st));
  launch_fill_i32(w.t_single.p, T, -1, st);
  KB_CK(cudaMemsetAsync(w.m_rowoff.p, 0, 4, st));   // n_multi == 0: offsets [0]
  w.eff.upload(res.eff_lens.data(), T, st);
  EmPrep ep = nu.prep;
  ep.n_multi = n_multi;
  ep.ec_tid = w.ec_tid.p; ep.multi_ec = w.multi_ec.p; ep.m_rowoff = w.m_rowoff.p; ep.m_tid = w.m_tid.p; ep.m_w = w.m_w.p;
  ep.m_row = w.m_row.p; ep.m_iota = w.m_iota.p; ep.t_deg = w.t_deg.p; ep.t_off = w.t_off.p; ep.t_midx = w.t_midx.p;
  ep.t_w = w.t_w.p; ep.t_single = w.t_single.p; ep.eff = w.eff.p; ep.k64_in = w.k64_in.p;
  emprep_rows(ep, w.is_multi.p, w.ckey.p, w.cval.p, w.ckey_out.p, w.rlen.p, w.tmp.p, w.tmp.n, st);
  emprep_fill(dd_, ep, nnz, w.k64_out.p, w.sortv.p, w.tmp.p, w.tmp.n, (unsigned long long*)w.key_in.p, st);
  KB_CK(cudaGetLastError());
  // ---- EM
  EmProblem p = w.problem(n, T, n_multi, max_iter, min_rounds);
  const EmCompWs cw = w.comp(T, n_multi, nnz, max_iter, w.eff.p);
  mark("fill launches + uploads");
  // collect_used, gather_used, ec_meta, multi_compact, row_len, ec_fill, csc_fill, stats, fill_i32, em_start,
  // em_gather_counts + em_kernel
  n_kernel_launches += 11 + 1;
  last_em_comp_blocks = w.em.launch(p, 1, w.count.p, em_tpb(), st, &cw, e1.e, &last_em_comp_resident,
                                    has_priors_ ? priors_.p : nullptr);
  KB_CK(cudaEventRecord(e2.e, st));
  unsigned long long s2[2] = {0, 0};
  w.key_in.download(s2, 2, 0, st);
  w.em.fetch(p, res.alpha.data(), &res.rounds, st);
  mark("EM kernel + results");
  res.seconds = elapsed_ms(e1, e2) * 1e-3;
  last_em_seconds = res.seconds;
  last_prep_seconds = elapsed_ms(e0, e1) * 1e-3;
  dev_stats_valid_ = true;
  dev_problem_valid_ = true;
  dev_n_multi_ = n_multi;
  dev_n_ecs_ = n; dev_nnz_ = nnz_all; dev_pseudoaligned_ = s2[0]; dev_unique_ = s2[1];
  return res;
}

std::vector<int> Quant::run_bootstrap_device(const std::vector<double>& fl_trunc, uint64_t seed, int B, std::vector<double>& alpha_out,
                                             std::vector<uint32_t>* samples_out, double* ms_out) {
  KB_CK(cudaSetDevice(ix_.device));
  join();
  std::vector<int> rounds;
  if (B <= 0) { alpha_out.clear(); return rounds; }
  if (!dev_problem_valid_) run_em_device(fl_trunc);      // builds the matrices (and runs the main EM once)
  const uint32_t T = ix_.flat.num_targets();
  alpha_out.assign((size_t)B * T, 0.0);
  rounds.assign(B, 0);
  if (!dev_problem_valid_) return rounds;                // nothing pseudoaligned
  if (ix_.l2_persist_bytes) cudaCtxResetPersistingL2Cache();
  cudaStream_t st = stream_;
  EmWs& w = *emws_;
  const uint32_t nE = (uint32_t)dev_n_ecs_, n_multi = dev_n_multi_;
  const std::vector<uint32_t> x0 = minstd_seeds(seed, B);
  // std::discrete_distribution<int>(counts): normalised probabilities and their partial sums, in the host's own
  // sequential double arithmetic (a parallel scan would round differently)
  std::vector<uint32_t> cnt(nE);
  w.count.download(cnt.data(), nE, 0, st);
  KB_CK(cudaStreamSynchronize(st));
  uint64_t N = 0;
  for (uint32_t e = 0; e < nE; ++e) N += cnt[e];
  const int n_draws = (int)N;   // Multinomial::n_ is an int
  w.bs_counts.grow((size_t)B * nE);
  EventGuard e0, e1, e2;
  KB_CK(cudaEventRecord(e0.e, st));
  if (nE >= 2) {
    std::vector<double> prob(cnt.begin(), cnt.end());
    const double sum = std::accumulate(prob.begin(), prob.end(), 0.0);
    for (auto& v : prob) v /= sum;
    std::vector<double> cp(nE);
    std::partial_sum(prob.begin(), prob.end(), cp.begin());
    cp[nE - 1] = 1.0;
    w.bs_cp.grow(nE); w.bs_x0.grow(B);
    w.bs_cp.upload(cp.data(), nE, st);
    w.bs_x0.upload(x0.data(), B, st);
    for (int b0 = 0; b0 < B; b0 += KB_EM_MAX_BATCH) {
      ResampleArgs ra{};
      ra.cp = w.bs_cp.p; ra.n_ec = nE; ra.n_draws = n_draws > 0 ? (uint64_t)n_draws : 0; ra.nb = std::min(KB_EM_MAX_BATCH, B - b0);
      ra.x0 = w.bs_x0.p + b0; ra.samp = w.bs_counts.p + (size_t)b0 * nE;
      launch_resample(ra, st);
      KB_CK(cudaGetLastError());
      ++n_kernel_launches;
    }
    KB_CK(cudaStreamSynchronize(st));     // cp / x0 are local vectors
  } else {
    // a single class: discrete_distribution returns 0 without consuming the engine
    std::vector<uint32_t> s1((size_t)B * nE, 0);
    for (int b = 0; b < B && nE == 1; ++b) s1[b] = n_draws > 0 ? (uint32_t)n_draws : 0;
    w.bs_counts.upload(s1.data(), s1.size(), st);
    KB_CK(cudaStreamSynchronize(st));
  }
  KB_CK(cudaEventRecord(e1.e, st));
  if (samples_out) {
    samples_out->resize((size_t)B * nE);
    w.bs_counts.download(samples_out->data(), samples_out->size(), 0, st);
    KB_CK(cudaStreamSynchronize(st));
  }
  // the B problems, `chunk` at a time: alpha + norm + counts of a chunk are meant to stay in L2 next to the shared
  // matrices, so a chunk's vectors take at most half of the device's L2 (25 MB on an H100)
  int chunk;
  {
    const size_t per = ((size_t)T + n_multi) * 8 + (size_t)nE * 4;
    int l2 = 0;
    if (cudaDeviceGetAttribute(&l2, cudaDevAttrL2CacheSize, ix_.device) != cudaSuccess || l2 <= 0) {
      cudaGetLastError();
      l2 = 50 << 20;
    }
    const size_t budget = (size_t)l2 / 2;
    chunk = (int)em_chunk(budget / std::max<size_t>(1, per), (uint64_t)B, "KB_BS_CHUNK");
  }
  w.em.reserve((size_t)chunk, T, n_multi);
  EmProblem p = w.problem(nE, T, n_multi, 10000, 50);
  for (int b0 = 0; b0 < B; b0 += chunk) {
    const int nb = std::min(chunk, B - b0);
    w.em.launch(p, nb, w.bs_counts.p + (size_t)b0 * nE, em_tpb(), st);
    n_kernel_launches += 2;
    w.em.fetch(p, alpha_out.data() + (size_t)b0 * T, rounds.data() + b0, st);
  }
  KB_CK(cudaEventRecord(e2.e, st));
  KB_CK(cudaEventSynchronize(e2.e));
  if (ms_out) {
    ms_out[0] = elapsed_ms(e0, e1);
    ms_out[1] = elapsed_ms(e1, e2);
  }
  return rounds;
}

void Quant::export_prepare(uint32_t* n_sets, uint32_t* n_entries) {
  KB_CK(cudaSetDevice(ix_.device));
  check_device_errors();
  EmWs& w = *emws_;
  const EcNumbering nu = number_ecs();
  exp_n_ = nu.n;
  exp_nnz_ = nu.n_entries;
  if (nu.n) {
    w.ec_tid.grow(std::max<uint32_t>(1, nu.n_entries), 0.25);
    EmPrep ep = nu.prep;
    ep.ec_tid = w.ec_tid.p;
    emprep_fill_table(dd_, ep, stream_);
    KB_CK(cudaGetLastError());
  }
  *n_sets = exp_n_;
  *n_entries = exp_nnz_;
}

void Quant::export_copy(uint32_t* d_off, uint32_t* d_tids, uint32_t* d_counts, unsigned long long* d_first) {
  KB_CK(cudaSetDevice(ix_.device));
  join();
  EmWs& w = *emws_;
  cudaStream_t st = stream_;
  if (exp_n_) {
    KB_CK(cudaMemcpyAsync(d_off, w.ec_off.p, ((size_t)exp_n_ + 1) * 4, cudaMemcpyDeviceToDevice, st));
    KB_CK(cudaMemcpyAsync(d_tids, w.ec_tid.p, (size_t)exp_nnz_ * 4, cudaMemcpyDeviceToDevice, st));
    KB_CK(cudaMemcpyAsync(d_counts, w.count.p, (size_t)exp_n_ * 4, cudaMemcpyDeviceToDevice, st));
    KB_CK(cudaMemcpyAsync(d_first, w.key_out.p, (size_t)exp_n_ * 8, cudaMemcpyDeviceToDevice, st));
  } else {
    KB_CK(cudaMemsetAsync(d_off, 0, 4, st));
  }
  KB_CK(cudaStreamSynchronize(st));
}

uint64_t Quant::merge_local(const std::vector<Quant*>& others, uint64_t first_stride) {
  uint64_t total = n_frag_total_;
  size_t sum_n = 0, sum_nnz = 0;
  std::vector<std::pair<uint32_t, uint32_t>> sizes;
  for (Quant* o : others) {
    uint32_t n = 0, nnz = 0;
    o->export_prepare(&n, &nnz);                 // numbers o's ECs on ITS device (synchronises o's stream)
    sizes.push_back({n, nnz});
    sum_n += n;
    sum_nnz += nnz;
    total += o->n_frag_total_;
  }
  KB_CK(cudaSetDevice(ix_.device));
  check_device_errors();
  lm_off_.grow(sum_n + others.size() + 1);
  lm_counts_.grow(sum_n + 1);
  lm_first_.grow(sum_n + 1);
  lm_tids_.grow(sum_nnz + 1);
  std::vector<ImportSeg> segs;
  size_t o_off = 0, o_n = 0, o_nnz = 0;
  for (size_t i = 0; i < others.size(); ++i) {
    Quant* o = others[i];
    const uint32_t n = sizes[i].first, nnz = sizes[i].second;
    if (n) {
      EmWs& w = *o->emws_;
      const int src = o->ix_.device, dst = ix_.device;
      KB_CK(cudaMemcpyPeerAsync(lm_off_.p + o_off, dst, w.ec_off.p, src, ((size_t)n + 1) * 4, stream_));
      KB_CK(cudaMemcpyPeerAsync(lm_tids_.p + o_nnz, dst, w.ec_tid.p, src, (size_t)nnz * 4, stream_));
      KB_CK(cudaMemcpyPeerAsync(lm_counts_.p + o_n, dst, w.count.p, src, (size_t)n * 4, stream_));
      KB_CK(cudaMemcpyPeerAsync(lm_first_.p + o_n, dst, w.key_out.p, src, (size_t)n * 8, stream_));
      ImportSeg sg;
      sg.n_sets = n; sg.off = lm_off_.p + o_off; sg.tids = lm_tids_.p + o_nnz; sg.counts = lm_counts_.p + o_n; sg.first = lm_first_.p + o_n;
      segs.push_back(sg);
      if (first_stride) throw Error("kallisto_b200: merge_local expects runs fed with global fragment indices");
    }
    o_off += (size_t)n + 1; o_n += n; o_nnz += nnz;
  }
  ecs_valid_ = false;
  dev_stats_valid_ = false;
  dev_problem_valid_ = false;
  for (size_t i = 0; i < segs.size(); i += KB_IMPORT_SEGS) {
    launch_import_segments(dd_, segs.data() + i, (int)std::min<size_t>(KB_IMPORT_SEGS, segs.size() - i), stream_);
    KB_CK(cudaGetLastError());
    ++n_kernel_launches;
  }
  KB_CK(cudaStreamSynchronize(stream_));
  n_frag_total_ = total;
  return total;
}

void Quant::import_sets_device(uint32_t n_sets, const uint32_t* d_off, const uint32_t* d_tids, const uint32_t* d_counts,
                               const unsigned long long* d_first, unsigned long long first_offset) {
  KB_CK(cudaSetDevice(ix_.device));
  join();
  ecs_valid_ = false;
  dev_stats_valid_ = false;
  dev_problem_valid_ = false;
  launch_import_sets(dd_, n_sets, d_off, d_tids, d_counts, d_first, first_offset, stream_);
  KB_CK(cudaGetLastError());
  KB_CK(cudaStreamSynchronize(stream_));
}

namespace {
// What every quant-tcc problem shares: the structure of the EC table (EC ids = line numbers of matrix.ec) and the TCC
// rows themselves, on the device.
struct TccShape : EmShape {
  DBuf<uint32_t> ecid, val;

  TccShape(uint32_t T, const TccInput& in, cudaStream_t st) {
    const uint64_t n_rows = in.row_off[in.n_samples];
    for (uint64_t j = in.ec_off[0]; j < in.ec_off[in.n_ecs]; ++j)
      if (in.tids[j] >= T) throw Error("kallisto_b200: equivalence class file has a transcript id out of range");
    for (uint64_t i = 0; i < n_rows; ++i)
      if (in.ec_ids[i] >= in.n_ecs) throw Error("kallisto_b200: TCC file refers to an equivalence class that is not in the EC file");
    upload_new(ecid, in.ec_ids, n_rows, st);
    upload_new(val, in.counts, n_rows, st);
    build(in.n_ecs, in.ec_off, in.tids, T, st);
  }
  // weights of `nb` rows (row_off: their nb + 1 offsets into ecid / val) into counts / m_w / t_w
  TccFill fill(int nb, const unsigned long long* row_off, uint32_t* counts, const double* eff, uint64_t eff_stride,
               double* m_w, double* t_w) const {
    return EmShape::fill(nb, row_off, ecid.p, val.p, counts, eff, eff_stride, m_w, t_w);
  }
  EmProblem problem() const {     // every problem has its own weights
    EmProblem p = EmShape::problem(10000, 50);
    p.w_stride = nnz;
    return p;
  }
};

// Gene-level output: gene -> member transcripts (CSR, increasing id) from in.gene_of, and the gene sums of up to `nb_max`
// problems at a time.  Without genes (in.n_genes == 0) nothing is allocated and run() does nothing.
struct TccGenes {
  uint32_t G = 0;
  DBuf<uint32_t> g_off, g_tid;
  DBuf<double> total, counts, tpm;

  TccGenes(uint32_t T, const TccInput& in, uint64_t nb_max, cudaStream_t st) : G(in.n_genes) {
    if (!G) return;
    if (!in.gene_of) throw Error("kallisto_b200: n_genes > 0 without a gene of every target");
    std::vector<uint32_t> off(G + 1, 0), tid;
    for (uint32_t t = 0; t < T; ++t) {
      const int32_t g = in.gene_of[t];
      if (g < -1 || (g >= 0 && (uint32_t)g >= G)) throw Error("kallisto_b200: a target's gene id is out of range");
      if (g >= 0) ++off[g + 1];
    }
    for (uint32_t g = 0; g < G; ++g) off[g + 1] += off[g];
    tid.resize(off[G]);
    {
      std::vector<uint32_t> fill(off.begin(), off.end() - 1);
      for (uint32_t t = 0; t < T; ++t)
        if (in.gene_of[t] >= 0) tid[fill[in.gene_of[t]]++] = t;
    }
    g_off.alloc(G + 1); g_off.upload(off.data(), G + 1, st);
    g_tid.alloc(std::max<size_t>(1, tid.size())); g_tid.upload(tid.data(), tid.size(), st);
    total.alloc(nb_max); counts.alloc(nb_max * G); tpm.alloc(nb_max * G);
    KB_CK(cudaStreamSynchronize(st));     // the host vectors go out of scope
  }
  // bytes per problem, for the sizing of chunks
  static size_t per_problem(const TccInput& in) { return in.n_genes ? (size_t)in.n_genes * 16 + 8 : 0; }
  // the gene sums of nb problems whose estimates are in alpha (their final states in fstate), into counts / tpm
  void run(uint32_t nb, uint32_t T, const double* alpha, const int* fstate, const double* eff, uint64_t eff_stride,
           const uint32_t* w_set, cudaStream_t st) {
    if (!G) return;
    TccGeneArgs a{};
    a.nb = nb; a.n_targets = T; a.n_genes = G; a.alpha = alpha; a.fstate = fstate;
    a.eff = eff; a.eff_stride = eff_stride; a.w_set = w_set; a.g_off = g_off.p; a.g_tid = g_tid.p;
    a.total = total.p; a.gene_counts = counts.p; a.gene_tpm = tpm.p;
    launch_tcc_genes(a, st);
    KB_CK(cudaGetLastError());
  }
};
}  // namespace

std::vector<int> tcc_run(Index& ix, const TccInput& in, std::vector<double>& alpha_out, std::vector<double>* gene_counts_out,
                         std::vector<double>* gene_tpm_out) {
  KB_CK(cudaSetDevice(ix.device));
  const uint32_t T = ix.flat.num_targets(), nE = in.n_ecs, S = in.n_samples, G = in.n_genes;
  alpha_out.assign((size_t)S * T, 0.0);
  if (G && (!gene_counts_out || !gene_tpm_out)) throw Error("kallisto_b200: gene-level output without its buffers");
  if (G) { gene_counts_out->assign((size_t)S * G, 0.0); gene_tpm_out->assign((size_t)S * G, 0.0); }
  std::vector<int> rounds(S, 0);
  if (S == 0) return rounds;
  StreamGuard sg;
  const cudaStream_t st = sg.s;
  const TccShape sh(T, in, st);
  const uint64_t nnz = sh.nnz;
  const uint32_t n_multi = sh.n_multi;
  DBuf<uint32_t> d_counts;
  DBuf<unsigned long long> d_rowoff;
  DBuf<double> d_eff, d_mw, d_tw;
  EmState em;
  // samples per chunk: weights dominate (16 bytes per entry and sample); ~2 GB of work space
  const size_t per = (size_t)nnz * 16 + (size_t)nE * 4 + ((size_t)T + n_multi) * 8 + TccGenes::per_problem(in);
  const int chunk = (int)em_chunk(((size_t)2 << 30) / std::max<size_t>(1, per), S, "KB_TCC_CHUNK");
  TccGenes genes(T, in, (uint64_t)chunk, st);
  d_counts.alloc((size_t)chunk * std::max<uint32_t>(1, nE));
  d_mw.alloc(std::max<size_t>(1, (size_t)chunk * nnz)); d_tw.alloc(std::max<size_t>(1, (size_t)chunk * nnz));
  em.reserve((size_t)chunk, T, n_multi);
  d_eff.alloc(in.per_sample_eff ? (size_t)chunk * T : (size_t)T);
  if (!in.per_sample_eff) d_eff.upload(in.eff_lens, T, st);
  d_rowoff.alloc((size_t)chunk + 1);
  std::vector<unsigned long long> ro((size_t)chunk + 1);
  DBuf<double> d_prior;
  if (in.priors) {
    d_prior.alloc(std::max<uint32_t>(1, T));
    d_prior.upload(in.priors, T, st);
  }
  EmProblem p = sh.problem();
  p.m_w = d_mw.p; p.t_w = d_tw.p;
  for (uint32_t s0 = 0; s0 < S; s0 += (uint32_t)chunk) {
    const int nb = (int)std::min<uint32_t>((uint32_t)chunk, S - s0);
    for (int b = 0; b <= nb; ++b) ro[b] = in.row_off[s0 + b];
    d_rowoff.upload(ro.data(), (size_t)nb + 1, st);
    if (in.per_sample_eff) d_eff.upload(in.eff_lens + (size_t)s0 * T, (size_t)nb * T, st);
    launch_tcc_fill(sh.fill(nb, d_rowoff.p, d_counts.p, d_eff.p, in.per_sample_eff ? T : 0, d_mw.p, d_tw.p), st);
    KB_CK(cudaGetLastError());
    em.launch(p, nb, d_counts.p, em_tpb(), st, nullptr, nullptr, nullptr, in.priors ? d_prior.p : nullptr);
    genes.run((uint32_t)nb, T, p.alpha, p.fstate, d_eff.p, in.per_sample_eff ? T : 0, nullptr, st);
    if (G) {
      genes.counts.download(gene_counts_out->data() + (size_t)s0 * G, (size_t)nb * G, 0, st);
      genes.tpm.download(gene_tpm_out->data() + (size_t)s0 * G, (size_t)nb * G, 0, st);
    }
    em.fetch(p, alpha_out.data() + (size_t)s0 * T, rounds.data() + s0, st);
  }
  return rounds;
}

void tcc_bootstrap(Index& ix, const TccInput& in, uint64_t seed, int B, bool want_samples, const TccBootstrapSink& sink) {
  KB_CK(cudaSetDevice(ix.device));
  const uint32_t T = ix.flat.num_targets(), nE = in.n_ecs, S = in.n_samples;
  if (S == 0 || B <= 0) return;
  StreamGuard sg;
  const cudaStream_t st = sg.s;
  const TccShape sh(T, in, st);      // checks the EC ids
  const uint64_t nnz = sh.nnz;
  const uint32_t n_multi = sh.n_multi;
  // Multinomial::sample of every row (src/Multinomial.hpp): std::discrete_distribution<int> over the row's DENSE counts
  // (n_ecs of them).  libstdc++ normalises by the sum, takes partial sums in order and sets the LAST dense entry to
  // 1.0; a draw is the first index whose partial sum is >= u.  The table here keeps the non-zero ECs only, in the same
  // sequential double arithmetic: a zero count adds 0.0 to the sum and to the partial sum, which changes neither.
  //   - A zero-count EC e never wins a draw: its partial sum equals that of the EC before it, which comes first in the
  //     search; for e = 0 it is 0.0, and u > 0 always (generate_canonical over minstd_rand0: u = 0 needs two
  //     consecutive engine outputs of 1, and 16807 * 1 != 1).  So dropping those entries changes no draw ...
  //   - ... except for the last EC: its entry is forced to 1.0 even when its count is 0, and a u above the row's last
  //     partial sum (below 1 by rounding) lands on it.  If EC n_ecs - 1 has count 0 the table ends with a sentinel
  //     entry (EC n_ecs - 1, 1.0); otherwise the row's own last entry is set to 1.0.
  // With one EC (n_ecs == 1) libstdc++ keeps no table and returns 0 for every draw; the one-entry table does the same.
  std::vector<unsigned long long> cp_off(S + 1, 0), n_draws(S, 0);
  std::vector<double> cp;
  std::vector<uint32_t> cp_ec;
  for (uint32_t r = 0; r < S; ++r) {
    const uint64_t a = in.row_off[r], z = in.row_off[r + 1];
    double sum = 0.0;
    uint64_t N = 0;
    for (uint64_t i = a; i < z; ++i) {
      if (i > a && in.ec_ids[i] <= in.ec_ids[i - 1])
        throw Error("kallisto_b200: the EC ids of a TCC row must be strictly increasing for bootstrapping");
      sum += (double)in.counts[i];
      N += in.counts[i];
    }
    if (N > 2147483647ull) throw Error("kallisto_b200: a TCC row holds more than 2^31 - 1 counts (Multinomial::n_ is an int)");
    n_draws[r] = N;
    if (N) {
      double acc = 0.0;
      for (uint64_t i = a; i < z; ++i) {
        if (!in.counts[i]) continue;
        acc += (double)in.counts[i] / sum;
        cp.push_back(acc);
        cp_ec.push_back(in.ec_ids[i]);
      }
      if (cp_ec.back() == nE - 1) cp.back() = 1.0;
      else { cp.push_back(1.0); cp_ec.push_back(nE - 1); }
    }
    cp_off[r + 1] = cp.size();
  }
  const std::vector<uint32_t> x0 = minstd_seeds(seed, B);   // the same B for every row
  // problems per chunk (a chunk may split a row's B bootstraps): the per-problem vectors plus the weights of the rows the
  // chunk touches fit ~2 GB of work space
  const uint64_t P = (uint64_t)S * B;
  auto rows_of = [&](uint64_t c) { return std::min<uint64_t>(S, (c + B - 2) / B + 1); };   // most rows c problems touch
  const size_t per_prob = (size_t)nE * 4 + (size_t)T * 16 + (size_t)n_multi * 12 + 32 + TccGenes::per_problem(in);
  const size_t per_row = (size_t)nnz * 16 + (size_t)nE * 4 + (in.per_sample_eff ? (size_t)T * 8 : 0) + 16;
  auto fits = [&](uint64_t c) { return c * per_prob + rows_of(c) * per_row <= ((size_t)2 << 30); };
  uint64_t fit = std::min<uint64_t>(P, KB_EM_MAX_BATCH);
  if (!fits(fit)) {
    uint64_t lo = 1, hi = fit;     // largest chunk that fits (1 if none does)
    while (hi - lo > 1) { const uint64_t mid = (lo + hi) / 2; if (fits(mid)) lo = mid; else hi = mid; }
    fit = lo;
  }
  const uint64_t chunk = em_chunk(fit, P, "KB_TCC_BS_CHUNK");
  const uint64_t rmax = rows_of(chunk);
  const uint32_t G = in.n_genes;
  TccGenes genes(T, in, chunk, st);
  std::vector<double> gcounts(chunk * G), gtpm(chunk * G);
  DBuf<uint32_t> d_counts, d_samp, d_x0, d_cp_ec, d_wset;
  DBuf<unsigned long long> d_rowoff, d_cp_off, d_ndraws, d_chunkoff;
  DBuf<double> d_eff, d_mw, d_tw, d_cp;
  EmState em;
  d_counts.alloc(rmax * std::max<uint32_t>(1, nE));
  d_mw.alloc(std::max<size_t>(1, rmax * nnz)); d_tw.alloc(std::max<size_t>(1, rmax * nnz));
  d_eff.alloc(in.per_sample_eff ? rmax * T : (size_t)T);
  if (!in.per_sample_eff) d_eff.upload(in.eff_lens, T, st);
  d_rowoff.alloc(rmax + 1);
  d_samp.alloc(chunk * std::max<uint32_t>(1, nE));
  em.reserve(chunk, T, n_multi);
  d_wset.alloc(chunk); d_chunkoff.alloc(chunk + 1);
  d_x0.alloc(B); d_x0.upload(x0.data(), B, st);
  d_cp_off.alloc(S + 1); d_cp_off.upload(cp_off.data(), S + 1, st);
  d_ndraws.alloc(S); d_ndraws.upload(n_draws.data(), S, st);
  d_cp.alloc(std::max<size_t>(1, cp.size())); d_cp.upload(cp.data(), cp.size(), st);
  d_cp_ec.alloc(std::max<size_t>(1, cp_ec.size())); d_cp_ec.upload(cp_ec.data(), cp_ec.size(), st);
  std::vector<unsigned long long> ro(rmax + 1), coff(chunk + 1);
  std::vector<uint32_t> wset(chunk), samp(want_samples ? chunk * nE : 0);
  std::vector<double> est(chunk * T);
  std::vector<int> rounds(chunk);
  EmProblem p = sh.problem();
  p.m_w = d_mw.p; p.t_w = d_tw.p; p.w_set = d_wset.p;
  for (uint64_t g0 = 0; g0 < P; g0 += chunk) {
    const int nb = (int)std::min<uint64_t>(chunk, P - g0);
    const uint64_t r0 = g0 / B, nr = (g0 + nb - 1) / B - r0 + 1;
    // the original counts of the chunk's rows -> their weights (calc_weights(tc_.counts, ...), src/weights.cpp:220-246)
    for (uint64_t i = 0; i <= nr; ++i) ro[i] = in.row_off[r0 + i];
    d_rowoff.upload(ro.data(), nr + 1, st);
    if (in.per_sample_eff) d_eff.upload(in.eff_lens + r0 * T, nr * T, st);
    launch_tcc_fill(sh.fill((int)nr, d_rowoff.p, d_counts.p, d_eff.p, in.per_sample_eff ? T : 0, d_mw.p, d_tw.p), st);
    KB_CK(cudaGetLastError());
    // resampled counts
    coff[0] = 0;
    for (int i = 0; i < nb; ++i) {
      const uint64_t r = (g0 + i) / B;
      wset[i] = (uint32_t)(r - r0);
      coff[i + 1] = coff[i] + (n_draws[r] + 63) / 64;
    }
    d_wset.upload(wset.data(), nb, st);
    d_chunkoff.upload(coff.data(), (size_t)nb + 1, st);
    TccResampleArgs ra{};
    ra.n_ec = nE; ra.nb = (uint32_t)nb; ra.first = g0; ra.B = (uint32_t)B; ra.x0 = d_x0.p;
    ra.cp_off = d_cp_off.p; ra.cp = d_cp.p; ra.cp_ec = d_cp_ec.p; ra.n_draws = d_ndraws.p;
    ra.chunk_off = d_chunkoff.p; ra.n_chunks = coff[nb]; ra.samp = d_samp.p;
    launch_tcc_resample(ra, st);
    KB_CK(cudaGetLastError());
    // the EMs, with the weights of the problem's row
    em.launch(p, nb, d_samp.p, em_tpb(), st);
    genes.run((uint32_t)nb, T, p.alpha, p.fstate, d_eff.p, in.per_sample_eff ? T : 0, d_wset.p, st);
    if (want_samples) d_samp.download(samp.data(), (size_t)nb * nE, 0, st);
    if (G) {
      genes.counts.download(gcounts.data(), (size_t)nb * G, 0, st);
      genes.tpm.download(gtpm.data(), (size_t)nb * G, 0, st);
    }
    em.fetch(p, est.data(), rounds.data(), st);
    sink(g0, (uint32_t)nb, est.data(), rounds.data(), want_samples ? samp.data() : nullptr, G ? gcounts.data() : nullptr,
         G ? gtpm.data() : nullptr);
  }
}

template struct DBuf<uint8_t>;
template struct DBuf<uint16_t>;
template struct DBuf<uint32_t>;
template struct DBuf<int32_t>;
template struct DBuf<uint64_t>;
template struct DBuf<unsigned long long>;
template struct DBuf<double>;
template struct DBuf<KmerSlot>;
template struct DBuf<Memo2Entry>;
template struct DBuf<BusRecord>;
template struct DBuf<uint4>;


}  // namespace kb
