// TEST INFRASTRUCTURE: the stand-in library of stub_batch.cpp plus the kb_bus_group_* entry points, so that the command
// line's handling of `bus --devices` runs on a CPU-only box (tests/test_cli_bus_devices_host.py).  A group copies every
// submitted batch and hands it to member 0's kb_bus_batch when the batch completes, so its records equal a one-device
// run's exactly when the command line completes the batches in submission order.  It refuses what the library refuses:
// a second batch on a busy member, a ticket that is not the oldest, a sample switch with batches outstanding.  It says
// on stderr how many members it has and how many batches each one was given.  Never linked into the product.
#include <deque>

#include "stub_batch.cpp"

struct kb_bus_group {
  std::vector<kb_quant*> m;
  std::vector<int> busy;
  std::vector<uint64_t> per_member;
  struct Batch {
    uint64_t ticket;
    int member;
    uint32_t n;
    std::vector<std::string> bases;
    std::vector<std::vector<uint32_t>> offs;
  };
  std::deque<Batch> q;
  uint64_t next = 0;
};

extern "C" {
int kb_bus_group_create(kb_quant* const* members, int32_t n, kb_bus_group** out) {
  if (n < 1) return KB_ERR_INVALID;
  kb_bus_group* g = new kb_bus_group();
  g->m.assign(members, members + n);
  g->busy.assign(n, 0);
  g->per_member.assign(n, 0);
  fprintf(stderr, "stub: group of %d\n", n);
  *out = g;
  return KB_OK;
}
void kb_bus_group_free(kb_bus_group* g) {
  if (!g) return;
  fprintf(stderr, "stub: batches per member");
  for (uint64_t c : g->per_member) fprintf(stderr, " %llu", (unsigned long long)c);
  fprintf(stderr, "\n");
  delete g;
}
int kb_bus_group_submit(kb_bus_group* g, int32_t member, const char* const* bases, const uint32_t* const* offs, uint32_t n_sets,
                        uint64_t* ticket) {
  if (member < 0 || member >= (int32_t)g->m.size() || g->busy[member]) { g_err = "stub: member busy"; return KB_ERR_INVALID; }
  kb_bus_group::Batch b;
  b.ticket = g->next++;
  b.member = member;
  b.n = n_sets;
  const int nf = g->m[0]->nfiles;
  for (int f = 0; f < nf; ++f) {
    b.offs.emplace_back(offs[f], offs[f] + n_sets + 1);
    b.bases.emplace_back(bases[f], bases[f] + offs[f][n_sets]);
  }
  g->q.push_back(std::move(b));
  g->busy[member] = 1;
  ++g->per_member[member];
  *ticket = g->q.back().ticket;
  return KB_OK;
}
int kb_bus_group_complete(kb_bus_group* g, uint64_t ticket, kb_bus_record* rec, uint32_t* n_rec) {
  if (g->q.empty() || g->q.front().ticket != ticket) { g_err = "stub: ticket out of order"; return KB_ERR_INVALID; }
  kb_bus_group::Batch b = std::move(g->q.front());
  g->q.pop_front();
  g->busy[b.member] = 0;
  std::vector<const char*> bp;
  std::vector<const uint32_t*> op;
  for (size_t f = 0; f < b.bases.size(); ++f) { bp.push_back(b.bases[f].data()); op.push_back(b.offs[f].data()); }
  return kb_bus_batch(g->m[0], bp.data(), op.data(), b.n, rec, n_rec);
}
int kb_bus_group_begin_sample(kb_bus_group* g, uint64_t barcode) {
  if (!g->q.empty()) { g_err = "stub: batches outstanding"; return KB_ERR_INVALID; }
  for (kb_quant* q : g->m) kb_bus_begin_sample(q, barcode);
  return KB_OK;
}
int kb_bus_group_finalize(kb_bus_group* g, kb_run_stats* st) { return kb_quant_finalize(g->m[0], st); }
int kb_bus_group_ec_table(kb_bus_group* g, uint64_t* off, uint32_t* tids, uint32_t* counts) {
  return kb_quant_ec_table(g->m[0], off, tids, counts, nullptr);
}
int kb_bus_group_lengths(kb_bus_group* g, uint32_t* bc, uint32_t* umi) { return kb_bus_lengths(g->m[0], bc, umi); }
int kb_bus_group_frame_clashes(kb_bus_group* g, uint64_t* n) { return kb_bus_frame_clashes(g->m[0], n); }
}
