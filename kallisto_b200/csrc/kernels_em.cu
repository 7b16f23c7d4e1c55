// K4/K5: fp64 EM over the sparse EC x transcript layout, and bootstrap resampling.
//
// EMAlgorithm::run (src/EMAlgorithm.h:95-221) restated as two segmented passes per iteration
// inside ONE persistent kernel with a hand-rolled grid barrier (no dense contraction, no tensor cores):
//   pass A  per multi-transcript EC (CSR by EC):     denom = sum_j alpha[t_j] * w_j ; norm = count/denom
//   pass B  per transcript (CSC, entries by EC id):  next[t] = count(singleton {t}) + sum (w*alpha[t]) * norm
//           + the convergence test and alpha <- next
// Every row is accumulated sequentially in the reference's own order (transcript ids ascending
// inside an EC, EC ids ascending inside a transcript) with separate IEEE multiply and add
// (the reference is built without FMA contraction: no -march on src/), so alpha is
// bit-identical to the CPU result, iteration count included.  A batch dimension runs the B
// bootstrap EMs of Bootstrap::run_em (src/Bootstrap.cpp:4-13) concurrently over the same structure.
#include <algorithm>
#include <cstdlib>

#include "kb_device.cuh"
#include "kernels.hpp"

namespace kb {

namespace {
constexpr double kAlphaLimit = 1e-7;          // EMAlgorithm.h:101
constexpr double kAlphaChangeLimit = 1e-2;    // :102
constexpr double kAlphaChange = 1e-2;         // :103
constexpr double kTolerance = 4.9406564584124654e-324;   // std::numeric_limits<double>::denorm_min()
}

// Grid-wide barrier of the persistent kernel: a monotonically increasing arrival counter in global memory
// (zeroed by the launcher), one atomic per block and one spinning thread per block.  The kernel is launched
// cooperatively only for the co-residency guarantee; cooperative_groups' grid.sync() cost ~5 us of a 26 us round
// with 592 blocks, this one well under 2.  The fences around the spin order the other threads' plain loads and
// stores (and drop stale L1 lines) exactly as grid.sync() does.
__device__ __forceinline__ unsigned ld_acquire_u32(const unsigned* p) {
  unsigned v;
  asm volatile("ld.acquire.gpu.global.u32 %0, [%1];" : "=r"(v) : "l"(p) : "memory");
  return v;
}
// `add_to` (optional): the block's contribution *s_add is added to it by the arriving thread (one global atomic per
// block instead of one per warp) and *s_add is cleared.
__device__ __forceinline__ void grid_barrier(unsigned* bar, unsigned& gen, unsigned* add_to = nullptr, unsigned* s_add = nullptr) {
  __syncthreads();
  ++gen;
  if (threadIdx.x == 0) {
    if (add_to) {
      const unsigned v = *s_add;
      if (v) atomicAdd(add_to, v);
      *s_add = 0;
    }
    __threadfence();
    atomicAdd(bar, 1u);
    const unsigned target = gen * gridDim.x;
    while (ld_acquire_u32(bar) < target) {}
    __threadfence();
  }
  __syncthreads();
}

// OCC = 2 (KB_EM_OCC=2, experiment): compiled for 2048 resident threads per SM (32 registers, 16 bytes of spill).
// Measured slower than the 62-register build at every launch shape (27-36 vs 21 us per round, tools/em_sweep.py):
// not the default.
template <int TPB, int OCC>
__global__ void __launch_bounds__(TPB, OCC * (TPB >= 1024 ? 1 : (TPB >= 512 ? 2 : 4))) em_kernel(EmProblem p) {
  extern __shared__ int s_state[];    // per problem: 0 running, 1 final round, >= 2 finished (every block keeps its own, identical copy)
  const uint64_t gtid = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t gstride = (uint64_t)gridDim.x * blockDim.x;
  const unsigned lane = threadIdx.x & 31;
  const uint64_t nA = (uint64_t)p.nb * p.n_multi;
  const uint64_t nB = (uint64_t)p.nb * p.n_targets;
  const double zero_below = kAlphaLimit / 10.0;
  unsigned gen = 0;
  __shared__ unsigned s_changed;
  if (threadIdx.x == 0) s_changed = 0;
  for (int b = threadIdx.x; b < p.nb; b += blockDim.x) s_state[b] = 0;

  for (int it = 0;; ++it) {
    // ---------------- state machine per problem (:202-221), evaluated redundantly by every block from the change
    // counters of the iteration that just finished
    if (it > 0) {
      const int i = it - 1;                                         // the iteration that just ran
      for (int b = threadIdx.x; b < p.nb; b += blockDim.x) {
        int st = s_state[b];
        if (st < 2) {
          const unsigned ch = __ldcg(&p.chcount[2 * b + (i & 1)]);
          if (st == 1) { st = 2; if (blockIdx.x == 0) p.rounds[b] = i; }     // if (finalRound) break;
          else if (ch == 0 && i > p.min_rounds) st = 1;             // stopEM -> finalRound
          if (st < 2 && i + 1 == p.max_iter) {
            // loop runs out: i == n_iter.  If the stop was detected on the very last iteration the
            // reference still zeroes the small alphas (:213-216); the host does that for state 3.
            if (blockIdx.x == 0) p.rounds[b] = p.max_iter;
            st = (st == 1) ? 3 : 2;
          }
          if (st >= 2 && blockIdx.x == 0) p.fstate[b] = st;
          s_state[b] = st;
        }
      }
    }
    __syncthreads();
    bool mine_done = true;
    for (int b = threadIdx.x; b < p.nb; b += blockDim.x) mine_done = mine_done && s_state[b] >= 2;
    if (__syncthreads_and(mine_done)) break;
    // ---------------- pass A: denominators ----------------
    for (uint64_t i = gtid; i < nA; i += gstride) {
      const uint32_t b = (uint32_t)(i / p.n_multi), r = (uint32_t)(i % p.n_multi);
      const int st = s_state[b];
      if (st >= 2) continue;
      // count and row bounds are independent loads; the row is only walked when it has reads
      const uint32_t c = p.cnt_row[i];
      const uint32_t e0 = p.m_off[r], e1 = p.m_off[r + 1];
      double nrm = 0.0;
      if (c != 0) {
        const double* al = p.alpha + (size_t)b * p.n_targets;
        const double* mw = p.m_w + (size_t)(p.w_set ? p.w_set[b] : b) * p.w_stride;
        double denom = 0.0;
        for (uint32_t j = e0; j < e1; ++j) {
          double a = al[p.m_tid[j]];
          if (st == 1 && a < zero_below) a = 0.0;          // alpha zeroed before the final round (:213-216)
          denom = __dadd_rn(denom, __dmul_rn(a, mw[j]));
        }
        if (!(denom < kTolerance)) nrm = __ddiv_rn((double)c, denom);
      }
      p.norm[(size_t)b * p.n_multi + r] = nrm;
    }
    // the other parity of the change counters was consumed by every block before it arrives here
    grid_barrier(p.bar, gen);
    if (blockIdx.x == 0)
      for (int b = threadIdx.x; b < p.nb; b += blockDim.x) p.chcount[2 * b + ((it + 1) & 1)] = 0;
    // ---------------- pass B: numerators, convergence test, alpha <- next ----------------
    unsigned n_changed = 0;       // nb == 1: counted per thread, reduced per block
    for (uint64_t i0 = gtid - lane; i0 < nB; i0 += gstride) {
      const uint64_t i = i0 + lane;
      bool changed = false;
      uint32_t b = 0;
      if (i < nB) {
        b = (uint32_t)(i / p.n_targets);
        const uint32_t t = (uint32_t)(i % p.n_targets);
        const int st = s_state[b];
        if (st < 2) {
          double* al = p.alpha + (size_t)b * p.n_targets;
          double a = al[t];
          if (st == 1 && a < zero_below) a = 0.0;
          double acc = p.single_cnt[i];                                             // :119-123
          const double* nr = p.norm + (size_t)b * p.n_multi;
          const double* tw = p.t_w + (size_t)(p.w_set ? p.w_set[b] : b) * p.w_stride;
          const uint32_t e0 = p.t_off[t], e1 = p.t_off[t + 1];
          for (uint32_t j = e0; j < e1; ++j)
            acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(tw[j], a), nr[p.t_midx[j]]));   // :154-156
          changed = acc > kAlphaChangeLimit && (fabs(__dadd_rn(acc, -a)) / acc) > kAlphaChange;   // :178
          al[t] = acc;
        }
      }
      if (p.nb == 1) {
        n_changed += changed ? 1u : 0u;
      } else {
        // one atomic per warp when the warp sits inside one problem (the common case)
        const uint32_t b0 = __shfl_sync(0xFFFFFFFFu, b, 0), b31 = __shfl_sync(0xFFFFFFFFu, b, 31);
        const bool full = (i0 + 31 < nB) && b0 == b31;
        if (full) {
          const unsigned m = __ballot_sync(0xFFFFFFFFu, changed);
          if (lane == 0 && m) atomicAdd(&p.chcount[2 * b0 + (it & 1)], (unsigned)__popc(m));
        } else if (changed) {
          atomicAdd(&p.chcount[2 * b + (it & 1)], 1u);
        }
      }
    }
    if (p.nb == 1) {
      // one global atomic per block, issued by the thread that arrives at the grid barrier
      for (int o = 16; o > 0; o >>= 1) n_changed += __shfl_xor_sync(0xFFFFFFFFu, n_changed, o);
      if (lane == 0 && n_changed) atomicAdd(&s_changed, n_changed);
      grid_barrier(p.bar, gen, &p.chcount[it & 1], &s_changed);
    } else {
      grid_barrier(p.bar, gen);
    }
  }
}

// One problem (the main EM of `quant`): the same two passes and the same stop logic without the batch dimension --
// no 64-bit div/mod per row, no per-problem state in shared memory, 32-bit indices -- so that more threads fit an SM
// (the round time follows the number of resident threads, tools/em_sweep.py).  Bit-identical to em_kernel with nb == 1.
template <int TPB, int MINB>
__global__ void __launch_bounds__(TPB, MINB) em_single_kernel(EmProblem p) {
  const uint32_t gtid = blockIdx.x * blockDim.x + threadIdx.x;
  const uint32_t gstride = gridDim.x * blockDim.x;
  const unsigned lane = threadIdx.x & 31;
  const uint32_t nA = p.n_multi, nB = p.n_targets;
  const double zero_below = kAlphaLimit / 10.0;
  unsigned gen = 0;
  __shared__ unsigned s_changed;
  if (threadIdx.x == 0) s_changed = 0;
  int st = 0;      // 0 running, 1 final round, >= 2 finished: every thread evolves it from the same counters
  for (int it = 0;; ++it) {
    if (it > 0) {   // (:202-221) from the change counter of the iteration that just ran
      const int i = it - 1;
      const unsigned ch = __ldcg(&p.chcount[i & 1]);
      if (st == 1) { st = 2; if (gtid == 0) p.rounds[0] = i; }
      else if (ch == 0 && i > p.min_rounds) st = 1;
      if (st < 2 && i + 1 == p.max_iter) {
        if (gtid == 0) p.rounds[0] = p.max_iter;
        st = (st == 1) ? 3 : 2;
      }
      if (st >= 2 && gtid == 0) p.fstate[0] = st;
    }
    if (st >= 2) break;
    const bool fin = st == 1;
    // ---------------- pass A: denominators ----------------
    for (uint32_t r = gtid; r < nA; r += gstride) {
      const uint32_t c = p.cnt_row[r];
      const uint32_t e0 = p.m_off[r], e1 = p.m_off[r + 1];
      double nrm = 0.0;
      if (c != 0) {
        double denom = 0.0;
        for (uint32_t j = e0; j < e1; ++j) {
          double a = p.alpha[p.m_tid[j]];
          if (fin && a < zero_below) a = 0.0;
          denom = __dadd_rn(denom, __dmul_rn(a, p.m_w[j]));
        }
        if (!(denom < kTolerance)) nrm = __ddiv_rn((double)c, denom);
      }
      p.norm[r] = nrm;
    }
    grid_barrier(p.bar, gen);
    if (gtid == 0) p.chcount[(it + 1) & 1] = 0;
    // ---------------- pass B: numerators, convergence test, alpha <- next ----------------
    unsigned n_changed = 0;
    for (uint32_t t = gtid; t < nB; t += gstride) {
      double a = p.alpha[t];
      if (fin && a < zero_below) a = 0.0;
      double acc = p.single_cnt[t];
      const uint32_t e0 = p.t_off[t], e1 = p.t_off[t + 1];
      for (uint32_t j = e0; j < e1; ++j)
        acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(p.t_w[j], a), p.norm[p.t_midx[j]]));
      n_changed += (acc > kAlphaChangeLimit && (fabs(__dadd_rn(acc, -a)) / acc) > kAlphaChange) ? 1u : 0u;
      p.alpha[t] = acc;
    }
    for (int o = 16; o > 0; o >>= 1) n_changed += __shfl_xor_sync(0xFFFFFFFFu, n_changed, o);
    if (lane == 0 && n_changed) atomicAdd(&s_changed, n_changed);
    grid_barrier(p.bar, gen, &p.chcount[it & 1], &s_changed);
  }
}

// One problem whose components fit a block each (kernels.hpp, EmCompWs): every block solves one slice of whole
// components with its alpha, norm, counts and offsets in shared memory.  Streamed (RES = false), the entries (16-bit
// slice-local indices and the weights) come from the slice's contiguous part of the layout in every round.  Resident
// (RES = true), the block also holds the entries' indices and the effective lengths (and their reciprocals) of its
// transcripts, and rebuilds each weight count / eff with emcomp_weight -- the bits calc_weights produced, which
// emcomp_cut checked for every entry -- so a round touches no global memory.  Pass A and pass B are
// em_single_kernel's, statement for statement, with slice-local indices, so every row and every transcript sums
// exactly what it summed there.
//
// Components exchange no value, so there is no grid barrier.  Only the stop rule is global (EMAlgorithm.h:170-221):
// after round i a block adds 1 to sync[2i] if it changed an estimate, then 1 to sync[2i + 1].  A block that changed
// something knows that the global count is not zero and goes on; only a block without a change (past min_rounds) waits
// until every block has arrived at round i and reads the count.  A block only waits for a round it has reported itself,
// and all blocks are co-resident (cooperative launch), so no cycle of waits can form.  All blocks see a zero count in
// the same round, so they evolve the same state and stop after the same round.
template <int TPB, bool RES>
__global__ void __launch_bounds__(TPB, 1) em_component_kernel(EmProblem p, EmCompWs w) {
  extern __shared__ double s_d[];
  __shared__ int s_zero;
  const uint32_t b = blockIdx.x;
  const uint32_t t0 = w.s_t0[b], nt = w.s_t0[b + 1] - t0;
  const uint32_t r0 = w.s_r0[b], nr = w.s_r0[b + 1] - r0;
  double* s_alpha = s_d;
  double* s_single = s_alpha + nt;
  double* s_norm = s_single + nt;
  double* s_eff = s_norm + nr;                        // resident: nt each
  double* s_rcp = s_eff + nt;
  uint32_t* s_cnt = (uint32_t*)(RES ? s_rcp + nt : s_eff);
  uint32_t* s_roff = s_cnt + nr;          // nr + 1
  uint32_t* s_toff = s_roff + nr + 1;     // nt + 1
  uint16_t* s_rtid = (uint16_t*)(s_toff + nt + 1);    // resident: the slice's entries, CSR then CSC
  // resident: offsets relative to the slice's first entry
  const uint32_t tb = RES ? w.t_off[t0] : 0, rb = RES ? w.r_off[r0] : 0;
  for (uint32_t i = threadIdx.x; i <= nt; i += TPB) {
    s_toff[i] = w.t_off[t0 + i] - tb;
    if (i < nt) {
      s_alpha[i] = p.alpha[w.t_id[t0 + i]];
      s_single[i] = w.t_single[t0 + i];
      if (RES) {
        const double e = w.t_eff[t0 + i];
        s_eff[i] = e;
        s_rcp[i] = __drcp_rn(e);
      }
    }
  }
  for (uint32_t k = threadIdx.x; k <= nr; k += TPB) {
    s_roff[k] = w.r_off[r0 + k] - rb;
    if (k < nr) s_cnt[k] = w.r_cnt[r0 + k];
  }
  const uint32_t ne = RES ? w.r_off[r0 + nr] - rb : 0;
  uint16_t* s_trow = s_rtid + ne;
  for (uint32_t j = threadIdx.x; j < ne; j += TPB) {
    s_rtid[j] = w.r_tid[rb + j];
    s_trow[j] = w.t_row[tb + j];
  }
  const uint16_t* e_tid = RES ? s_rtid : w.r_tid;
  const uint16_t* e_row = RES ? s_trow : w.t_row;
  __syncthreads();
  const double zero_below = kAlphaLimit / 10.0;
  const bool lead = b == 0 && threadIdx.x == 0;
  int st = 0;      // 0 running, 1 final round, >= 2 finished
  for (int it = 0;; ++it) {
    const bool fin = st == 1;
    // ---------------- pass A: denominators ----------------
    for (uint32_t k = threadIdx.x; k < nr; k += TPB) {
      const uint32_t c = s_cnt[k];
      const uint32_t e0 = s_roff[k], e1 = s_roff[k + 1];
      double nrm = 0.0;
      if (c != 0) {
        const double cd = (double)c;
        double denom = 0.0;
#pragma unroll 4
        for (uint32_t j = e0; j < e1; ++j) {
          const uint32_t t = e_tid[j];
          double a = s_alpha[t];
          if (fin && a < zero_below) a = 0.0;
          const double wt = RES ? emcomp_weight(cd, s_eff[t], s_rcp[t]) : w.r_w[j];
          denom = __dadd_rn(denom, __dmul_rn(a, wt));
        }
        if (!(denom < kTolerance)) nrm = __ddiv_rn((double)c, denom);
      }
      s_norm[k] = nrm;
    }
    __syncthreads();
    // ---------------- pass B: numerators, convergence test, alpha <- next ----------------
    bool changed = false;
    for (uint32_t i = threadIdx.x; i < nt; i += TPB) {
      double a = s_alpha[i];
      if (fin && a < zero_below) a = 0.0;
      double acc = s_single[i];
      const uint32_t e0 = s_toff[i], e1 = s_toff[i + 1];
      const double ef = RES ? s_eff[i] : 0.0, y = RES ? s_rcp[i] : 0.0;
#pragma unroll 4
      for (uint32_t j = e0; j < e1; ++j) {
        const uint32_t k = e_row[j];
        const double wt = RES ? emcomp_weight((double)s_cnt[k], ef, y) : w.t_w[j];
        acc = __dadd_rn(acc, __dmul_rn(__dmul_rn(wt, a), s_norm[k]));
      }
      changed = changed || (acc > kAlphaChangeLimit && (fabs(__dadd_rn(acc, -a)) / acc) > kAlphaChange);
      s_alpha[i] = acc;
    }
    const bool any = __syncthreads_or(changed);
    // ---------------- stop rule (:202-221) for the round that just ran ----------------
    if (threadIdx.x == 0) {
      if (any) atomicAdd(&w.sync[2 * it], 1u);
      // release: the change count is visible before the arrival (a full fence here would stall thread 0, and with it
      // the block's next round)
      asm volatile("red.release.gpu.global.add.u32 [%0], 1;" ::"l"(&w.sync[2 * it + 1]) : "memory");
    }
    if (st == 1) {
      st = 2;
      if (lead) p.rounds[0] = it;
    } else if (!any && it > p.min_rounds) {
      if (threadIdx.x == 0) {
        while (ld_acquire_u32(&w.sync[2 * it + 1]) < gridDim.x) {}
        s_zero = ld_acquire_u32(&w.sync[2 * it]) == 0;
      }
      __syncthreads();
      if (s_zero) st = 1;
    }
    if (st < 2 && it + 1 == p.max_iter) {
      if (lead) p.rounds[0] = p.max_iter;
      st = (st == 1) ? 3 : 2;
    }
    if (st >= 2) {
      if (lead) p.fstate[0] = st;
      break;
    }
  }
  for (uint32_t i = threadIdx.x; i < nt; i += TPB) p.alpha[w.t_id[t0 + i]] = s_alpha[i];
}

// Start state of every problem of a launch: the caller's priors broadcast to each problem (EMAlgorithm::set_priors,
// EMAlgorithm.h:83-93), or the uniform 1 / T.
__global__ void em_start_kernel(double* alpha, uint32_t nb, uint32_t T, const double* prior, double uniform) {
  for (uint32_t b = blockIdx.y; b < nb; b += gridDim.y)
    for (uint32_t t = blockIdx.x * blockDim.x + threadIdx.x; t < T; t += gridDim.x * blockDim.x)
      alpha[(size_t)b * T + t] = prior ? prior[t] : uniform;
}
void launch_em_start(double* alpha, uint32_t nb, uint32_t T, const double* prior, double uniform, cudaStream_t st) {
  if (nb == 0 || T == 0) return;
  const unsigned gx = (unsigned)std::min<uint32_t>(256, (T + 255) / 256);
  const unsigned gy = std::min<uint32_t>(nb, 65535);
  em_start_kernel<<<dim3(gx, gy), 256, 0, st>>>(alpha, nb, T, prior, uniform);
}

// Row-ordered copies of the counts the passes need: cnt_row[b][r] = counts[b][multi_ec[r]],
// single_cnt[b][t] = counts[b][t_single[t]] (as a double) or 0.
__global__ void em_gather_counts_kernel(EmProblem p) {
  const uint64_t nA = (uint64_t)p.nb * p.n_multi, nB = (uint64_t)p.nb * p.n_targets;
  const uint64_t stride = (uint64_t)gridDim.x * blockDim.x;
  for (uint64_t i = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; i < nA + nB; i += stride) {
    if (i < nA) {
      const uint32_t b = (uint32_t)(i / p.n_multi), r = (uint32_t)(i % p.n_multi);
      p.cnt_row[i] = p.counts[(size_t)b * p.n_ec + p.multi_ec[r]];
    } else {
      const uint64_t k = i - nA;
      const uint32_t b = (uint32_t)(k / p.n_targets), t = (uint32_t)(k % p.n_targets);
      const int32_t s = p.t_single[t];
      p.single_cnt[k] = s >= 0 ? (double)p.counts[(size_t)b * p.n_ec + s] : 0.0;
    }
  }
}

namespace {
int em_occ() {
  if (const char* s = getenv("KB_EM_OCC")) return atoi(s) >= 2 ? 2 : 1;   // tuning knob
  return 1;
}
void* em_fn(int tpb, int occ) {
  if (occ >= 2) return tpb == 1024 ? (void*)em_kernel<1024, 2> : (tpb == 512 ? (void*)em_kernel<512, 2> : (void*)em_kernel<256, 2>);
  return tpb == 1024 ? (void*)em_kernel<1024, 1> : (tpb == 512 ? (void*)em_kernel<512, 1> : (void*)em_kernel<256, 1>);
}
// launch shapes of the single-problem kernel: threads per block x blocks per SM (KB_EM_SHAPE: 0..3; -1: use em_kernel)
struct SingleShape { void* fn; int tpb; };
SingleShape em_single_shape() {
  int sh = 0;
  if (const char* s = getenv("KB_EM_SHAPE")) sh = atoi(s);
  switch (sh) {
    case 1: return {(void*)em_single_kernel<512, 3>, 512};     // 1536 threads per SM, 42 registers
    case 2: return {(void*)em_single_kernel<768, 2>, 768};     // 1536 threads per SM
    case 3: return {(void*)em_single_kernel<1024, 2>, 1024};   // 2048 threads per SM, 32 registers
    case -1: return {nullptr, 0};
    default: return {(void*)em_single_kernel<1024, 1>, 1024};  // 1024 threads per SM
  }
}
}  // namespace

int em_max_blocks(int tpb, int nb) {
  int dev = 0, sms = 0, per_sm = 0;
  cudaGetDevice(&dev);
  cudaDeviceGetAttribute(&sms, cudaDevAttrMultiProcessorCount, dev);
  const int t = tpb >= 1024 ? 1024 : (tpb >= 512 ? 512 : 256);
  cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, em_fn(t, em_occ()), t, (size_t)nb * sizeof(int));
  return sms * per_sm;
}

namespace {
constexpr int kCompTpb = 1024;

// Whether n_slices blocks of the component kernel `fn` with `smem` bytes of shared memory each can all be resident.
bool comp_fits(const void* fn, unsigned long long smem, unsigned long long n_slices) {
  if (cudaFuncSetAttribute(fn, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)std::min<unsigned long long>(smem, 1u << 30)) !=
      cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  int per_sm = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, fn, kCompTpb, (size_t)smem) != cudaSuccess) {
    cudaGetLastError();
    return false;
  }
  return (unsigned long long)per_sm * device_sm_count() >= n_slices;
}

// The component layout and em_component_kernel, when the problem's components fit: returns the blocks launched, or 0
// (nothing launched) when a component is larger than KB_EM_COMP_CAP, a slice does not fit one block's shared memory
// or the slices cannot all be resident at once.  The resident kernel runs when the effective lengths are known, every
// weight is rebuilt bit for bit and the largest slice's resident layout fits KB_EM_COMP_SMEM and the block; the
// streamed kernel otherwise.
int launch_em_components(const EmProblem& p, const EmCompWs& w, cudaStream_t st, bool* resident) {
  if (p.n_targets == 0 || p.max_iter < 1 || p.max_iter > w.sync_rounds) return 0;
  const uint32_t slices = (uint32_t)std::min(device_sm_count(), w.max_slices);
  unsigned long long s[8];
  emcomp_cut(p, w, slices, s, st);
  const unsigned long long n_slices = s[2];
  if (s[3] > emcomp_cap()) return 0;
  const void* fn_res = (const void*)em_component_kernel<kCompTpb, true>;
  const bool res = w.eff && s[5] == 0 && s[6] <= emcomp_smem_budget() && comp_fits(fn_res, s[6], n_slices);
  const void* fn = res ? fn_res : (const void*)em_component_kernel<kCompTpb, false>;
  const unsigned long long smem = res ? s[6] : s[4];
  if (!res && !comp_fits(fn, smem, n_slices)) return 0;
  emcomp_fill(p, w, res, st);
  cudaMemsetAsync(w.sync, 0, 2 * (size_t)p.max_iter * sizeof(unsigned), st);
  EmProblem pp = p;
  EmCompWs ww = w;
  void* args[] = {&pp, &ww};
  cudaLaunchCooperativeKernel(fn, dim3((unsigned)n_slices), dim3(kCompTpb), args, (size_t)smem, st);
  if (resident) *resident = res;
  return (int)n_slices;
}
}  // namespace

int launch_em(const EmProblem& p, int tpb_req, cudaStream_t st, const EmCompWs* cw, bool* resident) {
  if (resident) *resident = false;
  EmProblem pp = p;
  cudaMemsetAsync(pp.bar, 0, sizeof(unsigned), st);
  {
    const uint64_t n = (uint64_t)p.nb * ((uint64_t)p.n_multi + p.n_targets);
    const unsigned g = (unsigned)std::min<uint64_t>((uint64_t)device_sm_count() * 8, (n + 255) / 256);
    if (g) em_gather_counts_kernel<<<g, 256, 0, st>>>(pp);
  }
  void* args[] = {&pp};
  const SingleShape ss = em_single_shape();
  if (p.nb == 1 && p.w_stride == 0 && ss.fn) {
    // an explicit KB_EM_SHAPE keeps the grid-wide kernels
    if (cw && !getenv("KB_EM_SHAPE")) {
      const int blocks = launch_em_components(p, *cw, st, resident);
      if (blocks) return blocks;
    }
    int per_sm = 0;
    cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, ss.fn, ss.tpb, 0);
    int blocks = device_sm_count() * std::max(1, per_sm);
    const uint32_t work = p.n_multi > p.n_targets ? p.n_multi : p.n_targets;
    blocks = std::max(1, std::min<int>(blocks, (int)((work + ss.tpb - 1) / ss.tpb)));
    cudaLaunchCooperativeKernel(ss.fn, dim3(blocks), dim3(ss.tpb), args, 0, st);
    return 0;
  }
  const int tpb = tpb_req >= 1024 ? 1024 : (tpb_req >= 512 ? 512 : 256);
  const int maxb = em_max_blocks(tpb, p.nb);
  const uint64_t work = (uint64_t)p.nb * (p.n_multi > p.n_targets ? p.n_multi : p.n_targets);
  int blocks = (int)((work + tpb - 1) / tpb);
  if (blocks > maxb) blocks = maxb;
  if (const char* s = getenv("KB_EM_BLOCKS")) { const int v = atoi(s); if (v > 0) blocks = std::min(maxb, v); }   // tuning knob
  if (blocks < 1) blocks = 1;
  cudaLaunchCooperativeKernel(em_fn(tpb, em_occ()), dim3(blocks), dim3(tpb), args, (size_t)pp.nb * sizeof(int), st);
  return 0;
}

// ---------------------------------------------------------------------------------------------
// quant-tcc (src/main.cpp:2802-3220): every sample (row of the TCC matrix) is its own EM over the SAME equivalence
// classes; its weights are its own counts / eff_len (calc_weights), so they are formed per sample here and the
// batched em_kernel reads them through w_stride.
__global__ void tcc_scatter_kernel(TccFill a) {
  const uint32_t b = blockIdx.y;
  const unsigned long long r0 = a.row_off[b], r1 = a.row_off[b + 1];
  for (unsigned long long i = r0 + (unsigned long long)blockIdx.x * blockDim.x + threadIdx.x; i < r1;
       i += (unsigned long long)gridDim.x * blockDim.x)
    a.counts[(size_t)b * a.n_ec + a.ec_ids[i]] = a.vals[i];
}
__global__ void tcc_weights_kernel(TccFill a) {
  const uint32_t b = blockIdx.y;
  const uint32_t* cnt = a.counts + (size_t)b * a.n_ec;
  const double* eff = a.eff + (size_t)b * a.eff_stride;
  for (uint64_t j = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; j < a.nnz; j += (uint64_t)gridDim.x * blockDim.x) {
    a.m_w[(size_t)b * a.nnz + j] = __ddiv_rn((double)cnt[a.m_ec[j]], eff[a.m_tid[j]]);
    a.t_w[(size_t)b * a.nnz + j] = __ddiv_rn((double)cnt[a.t_ec[j]], eff[a.t_tid[j]]);
  }
}
void launch_tcc_fill(const TccFill& a, cudaStream_t st) {
  if (a.nb == 0) return;
  cudaMemsetAsync(a.counts, 0, (size_t)a.nb * a.n_ec * sizeof(uint32_t), st);
  tcc_scatter_kernel<<<dim3(64, a.nb), 256, 0, st>>>(a);
  if (a.nnz) {
    const unsigned gx = (unsigned)std::min<uint64_t>(1024, (a.nnz + 255) / 256);
    tcc_weights_kernel<<<dim3(gx, a.nb), 256, 0, st>>>(a);
  }
}

// ---------------------------------------------------------------------------------------------
// Multinomial::sample (src/Multinomial.hpp:33-51): N draws of std::discrete_distribution<int>
// driven by std::default_random_engine (libstdc++: minstd_rand0, x <- 16807 x mod 2^31-1), two
// engine calls per draw (generate_canonical<double,53>).  The engine is a pure multiplicative
// LCG, so draw i starts from 16807^(2i) x0: every thread jumps to its own chunk of the stream
// and the result is bit-identical to the sequential CPU loop.
namespace {
constexpr uint32_t kM = 2147483647u;
__device__ __forceinline__ uint32_t mulmod(uint32_t a, uint32_t b) {
  uint64_t p = (uint64_t)a * b;
  p = (p & kM) + (p >> 31);
  p = (p & kM) + (p >> 31);
  return p >= kM ? (uint32_t)(p - kM) : (uint32_t)p;
}
__device__ __forceinline__ uint32_t powmod(uint32_t a, uint64_t e) {
  uint32_t r = 1;
  while (e) {
    if (e & 1) r = mulmod(r, a);
    a = mulmod(a, a);
    e >>= 1;
  }
  return r;
}
// The next draw of generate_canonical<double, 53> from engine state x: two engine steps, then
// (x1 - 1 + (x2 - 1) R) / R^2 with R = 2^31 - 2, kept below 1.0.
__device__ __forceinline__ double next_draw(uint32_t& x) {
  const double R = 2147483646.0;
  x = mulmod(x, 16807u);
  const double u0 = (double)(x - 1);
  x = mulmod(x, 16807u);
  const double u1 = (double)(x - 1);
  const double u = __ddiv_rn(__dadd_rn(u0, __dmul_rn(u1, R)), __dmul_rn(R, R));
  return u >= 1.0 ? 0.99999999999999988897769753748 : u;   // nextafter(1.0, 0.0)
}
constexpr int kDrawsPerThread = 64;
}

__global__ void __launch_bounds__(256) resample_kernel(ResampleArgs a) {
  const uint32_t b = blockIdx.y;
  const uint64_t chunk = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x;
  const uint64_t d0 = chunk * kDrawsPerThread;
  if (d0 >= a.n_draws) return;
  const uint64_t d1 = min(a.n_draws, d0 + kDrawsPerThread);
  uint32_t x = mulmod(a.x0[b], powmod(16807u, 2 * d0));
  uint32_t* samp = a.samp + (size_t)b * a.n_ec;
  for (uint64_t d = d0; d < d1; ++d) {
    const double u = next_draw(x);
    // std::lower_bound(cp.begin(), cp.end(), u): first index with cp[idx] >= u
    uint32_t lo = 0, hi = a.n_ec;
    while (lo < hi) {
      const uint32_t mid = (lo + hi) >> 1;
      if (a.cp[mid] < u) lo = mid + 1; else hi = mid;
    }
    atomicAdd(&samp[lo], 1u);
  }
}

void launch_resample(const ResampleArgs& a, cudaStream_t st) {
  cudaMemsetAsync(a.samp, 0, (size_t)a.nb * a.n_ec * sizeof(uint32_t), st);
  if (a.n_draws == 0 || a.nb == 0) return;
  const uint64_t chunks = (a.n_draws + kDrawsPerThread - 1) / kDrawsPerThread;
  dim3 grid((unsigned)((chunks + 255) / 256), (unsigned)a.nb);
  resample_kernel<<<grid, 256, 0, st>>>(a);
}

// The same draws for the (row, bootstrap) problems of quant-tcc, each over its row's sparse cumulative table.  Rows
// hold from 0 to tens of millions of draws, so the problems are not a grid dimension: every thread takes 64-draw
// chunks of one flat list (grid-stride) and finds its problem by binary search in the chunk prefix sum.
__global__ void __launch_bounds__(256) tcc_resample_kernel(TccResampleArgs a) {
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < a.n_chunks; w += (uint64_t)gridDim.x * blockDim.x) {
    uint32_t lo = 0, hi = a.nb;                 // last problem with chunk_off[p] <= w
    while (hi - lo > 1) {
      const uint32_t mid = (lo + hi) >> 1;
      if (a.chunk_off[mid] <= w) lo = mid; else hi = mid;
    }
    const uint32_t p = lo;
    const uint64_t g = a.first + p;
    const uint64_t row = g / a.B;
    const uint32_t b = (uint32_t)(g % a.B);
    const uint64_t d0 = (w - a.chunk_off[p]) * kDrawsPerThread;
    const uint64_t d1 = min((uint64_t)a.n_draws[row], d0 + kDrawsPerThread);
    const uint64_t t0 = a.cp_off[row], t1 = a.cp_off[row + 1];
    uint32_t* samp = a.samp + (size_t)p * a.n_ec;
    uint32_t x = mulmod(a.x0[b], powmod(16807u, 2 * d0));
    for (uint64_t d = d0; d < d1; ++d) {
      const double u = next_draw(x);
      // lower_bound over the row's table: its last entry is 1.0 > u, so the search ends inside the table
      uint64_t l = t0, h = t1;
      while (l < h) {
        const uint64_t mid = (l + h) >> 1;
        if (a.cp[mid] < u) l = mid + 1; else h = mid;
      }
      atomicAdd(&samp[a.cp_ec[l]], 1u);
    }
  }
}

void launch_tcc_resample(const TccResampleArgs& a, cudaStream_t st) {
  if (a.nb == 0) return;
  cudaMemsetAsync(a.samp, 0, (size_t)a.nb * a.n_ec * sizeof(uint32_t), st);
  if (a.n_chunks == 0) return;
  const unsigned g = (unsigned)std::min<uint64_t>((uint64_t)device_sm_count() * 16, (a.n_chunks + 255) / 256);
  tcc_resample_kernel<<<g, 256, 0, st>>>(a);
}

// Gene sums of quant-tcc.  Every operation is a separate IEEE double operation (no contraction), in the order of
// counts_to_tpm (src/PlaintextWriter.cpp:5-27): tpm[i] = alpha[i] / eff[i]; total += tpm[i]; tpm[i] = (tpm[i] / total)
// * 1e6.  The total is one sequential sum per problem, so it takes one thread per problem.
namespace {
__device__ __forceinline__ double gene_alpha(const TccGeneArgs& a, uint32_t b, uint32_t t) {
  const double x = a.alpha[(size_t)b * a.n_targets + t];
  return (a.fstate[b] == 3 && x < 1e-7 / 10.0) ? 0.0 : x;
}
__device__ __forceinline__ const double* gene_eff(const TccGeneArgs& a, uint32_t b) {
  return a.eff + (size_t)(a.w_set ? a.w_set[b] : b) * a.eff_stride;
}
}  // namespace

__global__ void tcc_gene_total_kernel(TccGeneArgs a) {
  const uint32_t b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= a.nb) return;
  const double* eff = gene_eff(a, b);
  double tot = 0.0;
  for (uint32_t t = 0; t < a.n_targets; ++t) tot = __dadd_rn(tot, __ddiv_rn(gene_alpha(a, b, t), eff[t]));
  a.total[b] = tot;
}

__global__ void __launch_bounds__(256) tcc_gene_sum_kernel(TccGeneArgs a) {
  const uint64_t n = (uint64_t)a.nb * a.n_genes;
  for (uint64_t w = (uint64_t)blockIdx.x * blockDim.x + threadIdx.x; w < n; w += (uint64_t)gridDim.x * blockDim.x) {
    const uint32_t b = (uint32_t)(w / a.n_genes), g = (uint32_t)(w % a.n_genes);
    const double* eff = gene_eff(a, b);
    const double tot = a.total[b];
    double gc = 0.0, gt = 0.0;
    for (uint32_t m = a.g_off[g]; m < a.g_off[g + 1]; ++m) {
      const uint32_t t = a.g_tid[m];
      const double x = gene_alpha(a, b, t);
      if (x > 0.0) {
        gc = __dadd_rn(gc, x);
        gt = __dadd_rn(gt, __dmul_rn(__ddiv_rn(__ddiv_rn(x, eff[t]), tot), 1e6));
      }
    }
    a.gene_counts[w] = gc;
    a.gene_tpm[w] = gt;
  }
}

void launch_tcc_genes(const TccGeneArgs& a, cudaStream_t st) {
  if (a.nb == 0 || a.n_genes == 0) return;
  tcc_gene_total_kernel<<<(a.nb + 127) / 128, 128, 0, st>>>(a);
  const uint64_t n = (uint64_t)a.nb * a.n_genes;
  const unsigned g = (unsigned)std::min<uint64_t>((uint64_t)device_sm_count() * 16, (n + 255) / 256);
  tcc_gene_sum_kernel<<<g, 256, 0, st>>>(a);
}

}  // namespace kb
