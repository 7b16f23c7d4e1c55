// kallisto_b200 -- command-line front end: same sub-commands, flags, messages and output files as
// `kallisto quant` (src/main.cpp:211-392 ParseOptionsEM, 1600-1805 CheckOptionsEM, 2620-2798 the
// command body), with the read pipeline, EC bookkeeping, EM and bootstrap running on the GPU through
// the C ABI (include/kallisto_b200.h).  Host work here: option parsing, FASTQ parsing, text output.
#include <getopt.h>
#include <fcntl.h>
#include <sys/mman.h>
#include <sys/stat.h>
#include <unistd.h>

#include <atomic>
#include <algorithm>
#include <charconv>
#include <cmath>
#include <chrono>
#include <condition_variable>
#include <cstdio>
#include <cstdlib>
#include <ctime>
#include <fstream>
#include <iomanip>
#include <iostream>
#include <mutex>
#include <sstream>
#include <string>
#include <thread>
#include <unordered_map>
#include <vector>

#include <zlib.h>

#include "../../include/kallisto_b200.h"
// Bound weakly: the command line also links against stand-ins of the library that carry only the entry points of the
// host pipeline (tests/stub); there `quant-tcc -b`, `quant-tcc -g / -G` and --priors report the missing entry point
// instead of failing to link; so do `bus --aa`, `bus --batch-barcodes` and `bus --devices`.
#pragma weak kb_tcc_bootstrap_run
#pragma weak kb_tcc_run_genes
#pragma weak kb_tcc_bootstrap_run_genes
#pragma weak kb_read_priors
#pragma weak kb_em_set_priors
#pragma weak kb_tcc_run_priors
#pragma weak kb_bus_set_aa
#pragma weak kb_bus_set_batch_barcodes
#pragma weak kb_bus_frame_clashes
#pragma weak kb_bus_group_create
#pragma weak kb_bus_group_free
#pragma weak kb_bus_group_submit
#pragma weak kb_bus_group_complete
#pragma weak kb_bus_group_begin_sample
#pragma weak kb_bus_group_finalize
#pragma weak kb_bus_group_ec_table
#pragma weak kb_bus_group_lengths
#pragma weak kb_bus_group_frame_clashes
#include "fastx.hpp"
#include "h5_reader.hpp"
#include "h5_writer.hpp"

using std::cerr;
using std::endl;

namespace {

const char* KALLISTO_VERSION = "0.51.1";   // the reference version whose behaviour is reproduced
const char* ERROR_STR = "Error:";   // src/main.cpp:29

void write_index_saved(const std::string& in_path, const std::string& out_path, int k);

// --priors file through kb_read_priors (EMAlgorithm::read_priors, src/EMAlgorithm.h:52-81).  An unreadable file and a line
// std::stod rejects are errors here; the reference runs uniform on the first and aborts on the second.
bool read_priors(const std::string& path, std::vector<double>& out) {
  if (!kb_read_priors) { cerr << "Error: this libkallisto_b200 has no kb_read_priors" << endl; return false; }
  uint64_t n = 0;
  int r = kb_read_priors(path.c_str(), nullptr, 0, &n);
  if (r == KB_OK) {
    out.resize(n);
    r = kb_read_priors(path.c_str(), out.data(), n, &n);
  }
  if (r != KB_OK) { cerr << ERROR_STR << " " << kb_last_error() << endl; return false; }
  return true;
}

// EMAlgorithm::set_priors (src/EMAlgorithm.h:83-93): a count other than the number of targets falls back to the uniform
// start with two lines on stderr (an empty file silently).  Returns whether the priors apply.
bool priors_apply(const std::vector<double>& priors, uint32_t n_targets) {
  if (priors.size() == n_targets) return true;
  if (!priors.empty())
    cerr << "[   em] number of priors does not match number of transcripts." << endl
         << "        defaulting to uniform priors." << endl;
  return false;
}

struct Options {
  int threads = 1;
  std::string index, output;
  double fld = 0.0, sd = 0.0;
  int bootstrap = 0;
  size_t seed = 42;
  bool plaintext = false, single_end = false, single_overhang = false, verbose = false, write_index = false;
  int strand = 0;   // 0 none, 1 FR, 2 RF
  int device = 0;
  std::vector<int> devices;   // --devices=0,1,...: reads are dealt to several GPUs, merged over NCCL (csrc/comm.cu)
  std::vector<std::string> files;
  std::string priors;         // -p / --priors: start of the EM (EMAlgorithm::read_priors / set_priors)
};

// Outputs are written and flushed: leave without tearing down the CUDA context, the k-mer table and the pinned rings
// one by one (a noticeable share of a short run).  KB_CLI_CLEANUP=1 keeps the orderly release (sanitizer runs).
[[noreturn]] void finish(int code) {
  std::cout.flush();
  cerr.flush();
  fflush(nullptr);
  _exit(code);
}

std::string pretty_num(size_t n) {   // src/common.cpp pretty_num
  std::string s = std::to_string(n);
  for (int i = (int)s.size() - 3; i > 0; i -= 3) s.insert(i, ",");
  return s;
}

std::string to_json(const std::string& id, const std::string& val, bool quote, bool comma = true, int level = 1) {
  std::string out;   // src/PlaintextWriter.cpp:114-138
  for (int i = 0; i < level; ++i) out += "\t";
  out += '"';
  out += id;
  out += "\": ";
  if (quote) out += '"';
  out += val;
  if (quote) out += '"';
  if (comma) out += ',';
  return out;
}

void usage_quant() {
  std::cout << "kallisto_b200 " << KALLISTO_VERSION << " (H100 build)" << endl
            << "Computes equivalence classes for reads and quantifies abundances" << endl << endl
            << "Usage: kallisto_b200 quant [arguments] FASTQ-files" << endl << endl
            << "Required arguments:" << endl
            << "-i, --index=STRING            Filename for the kallisto index to be used for" << endl
            << "                              quantification" << endl
            << "-o, --output-dir=STRING       Directory to write output to" << endl << endl
            << "Optional arguments:" << endl
            << "-b, --bootstrap-samples=INT   Number of bootstrap samples (default: 0)" << endl
            << "    --seed=INT                Seed for the bootstrap sampling (default: 42)" << endl
            << "    --plaintext               Output plaintext instead of HDF5" << endl
            << "    --single                  Quantify single-end reads" << endl
            << "    --single-overhang         Include reads where unobserved rest of fragment is" << endl
            << "                              predicted to lie outside a transcript" << endl
            << "    --fr-stranded             Strand specific reads, first read forward" << endl
            << "    --rf-stranded             Strand specific reads, first read reverse" << endl
            << "-l, --fragment-length=DOUBLE  Estimated average fragment length" << endl
            << "-s, --sd=DOUBLE               Estimated standard deviation of fragment length" << endl
            << "                              (default: -l, -s values are estimated from paired" << endl
            << "                               end data, but are required when using --single)" << endl
            << "-p, --priors                  Priors for the EM algorithm, either as raw counts or as" << endl
            << "                              probabilities. Pseudocounts are added to raw reads to" << endl
            << "                              prevent zero valued priors. Supplied in the same order" << endl
            << "                              as the transcripts in the transcriptome" << endl
            << "-t, --threads=INT             Number of host threads parsing input (default: 1)" << endl
            << "    --device=INT              CUDA device ordinal (default: 0)" << endl
            << "    --devices=LIST            Comma-separated CUDA devices: batches of reads are dealt to all of them," << endl
            << "                              index replicated, equivalence classes merged over NCCL before the EM" << endl
            << "    --verbose                 Print out progress information every 1M proccessed reads" << endl
            << "    --write-index             Also write counts.txt (reads per equivalence class) and index.saved" << endl << endl
            << "Limits of this build (a run stops with an error, never with a wrong answer): reads longer than ~12.6 kb," << endl
            << "more than 128 distinct equivalence classes hit by one fragment, more than 16.7 M targets." << endl;
}

void parse_quant(int argc, char** argv, Options& opt) {
  int verbose_flag = 0, plaintext_flag = 0, single_flag = 0, single_overhang_flag = 0, fr = 0, rf = 0, write_index_flag = 0;
  const char* opt_string = "t:i:l:s:o:b:d:D:p:";
  static struct option long_options[] = {
      {"verbose", no_argument, &verbose_flag, 1},
      {"write-index", no_argument, &write_index_flag, 1},
      {"plaintext", no_argument, &plaintext_flag, 1},
      {"single", no_argument, &single_flag, 1},
      {"single-overhang", no_argument, &single_overhang_flag, 1},
      {"fr-stranded", no_argument, &fr, 1},
      {"rf-stranded", no_argument, &rf, 1},
      {"seed", required_argument, 0, 'd'},
      {"threads", required_argument, 0, 't'},
      {"index", required_argument, 0, 'i'},
      {"fragment-length", required_argument, 0, 'l'},
      {"sd", required_argument, 0, 's'},
      {"output-dir", required_argument, 0, 'o'},
      {"bootstrap-samples", required_argument, 0, 'b'},
      {"priors", required_argument, 0, 'p'},
      {"device", required_argument, 0, 'D'},
      {"devices", required_argument, 0, 'G'},
      {0, 0, 0, 0}};
  int c, option_index = 0;
  while ((c = getopt_long(argc, argv, opt_string, long_options, &option_index)) != -1) {
    switch (c) {
      case 't': std::stringstream(optarg) >> opt.threads; break;
      case 'i': opt.index = optarg; break;
      case 'l': std::stringstream(optarg) >> opt.fld; break;
      case 's': std::stringstream(optarg) >> opt.sd; break;
      case 'o': opt.output = optarg; break;
      case 'b': std::stringstream(optarg) >> opt.bootstrap; break;
      case 'd': std::stringstream(optarg) >> opt.seed; break;
      case 'p': opt.priors = optarg; break;
      case 'D': std::stringstream(optarg) >> opt.device; break;
      case 'G': {
        std::stringstream ss(optarg);
        std::string tok;
        while (std::getline(ss, tok, ',')) {
          int v = -1;
          std::stringstream(tok) >> v;
          opt.devices.push_back(v);
        }
        break;
      }
      default: break;
    }
  }
  for (int i = optind; i < argc; i++) opt.files.push_back(argv[i]);
  if (!opt.devices.empty()) opt.device = opt.devices[0];
  opt.verbose = verbose_flag;
  opt.plaintext = plaintext_flag;
  opt.write_index = write_index_flag;
  opt.single_end = single_flag;
  opt.single_overhang = single_overhang_flag;
  if (fr) opt.strand = 1;
  if (rf) opt.strand = 2;
}

bool check_quant(Options& opt) {   // CheckOptionsEM, src/main.cpp:1600-1805
  bool ret = true;
  cerr << endl;
  struct stat st;
  if (opt.index.empty()) {
    cerr << ERROR_STR << " kallisto index file missing" << endl;
    ret = false;
  } else if (stat(opt.index.c_str(), &st) != 0) {
    cerr << ERROR_STR << " kallisto index file not found " << opt.index << endl;
    ret = false;
  }
  if (opt.files.empty()) {
    cerr << ERROR_STR << " Missing read files" << endl;
    ret = false;
  } else {
    for (auto& fn : opt.files)
      if (stat(fn.c_str(), &st) != 0) {
        cerr << ERROR_STR << " file not found " << fn << endl;
        ret = false;
      }
  }
  if (!opt.single_end && opt.files.size() % 2 != 0) {
    cerr << "Error: paired-end mode requires an even number of input files" << endl
         << "       (use --single for processing single-end reads)" << endl;
    ret = false;
  }
  if ((opt.fld != 0.0 && opt.sd == 0.0) || (opt.sd != 0.0 && opt.fld == 0.0)) {
    cerr << "Error: cannot supply mean/sd without supplying both -l and -s" << endl;
    ret = false;
  }
  if (opt.single_end && (opt.fld == 0.0 || opt.sd == 0.0)) {
    cerr << "Error: fragment length mean and sd must be supplied for single-end reads using -l and -s" << endl;
    ret = false;
  } else if (opt.fld == 0.0 && ret) {
    cerr << "[quant] fragment length distribution will be estimated from the data" << endl;
  } else if (ret && opt.fld > 0.0 && opt.sd > 0.0) {
    cerr << "[quant] fragment length distribution is truncated gaussian with mean = " << opt.fld << ", sd = " << opt.sd << endl;
  }
  if (!opt.single_end && (opt.fld > 0.0 && opt.sd > 0.0)) {
    cerr << "[~warn] you specified using a gaussian but have paired end data" << endl;
    cerr << "[~warn] we suggest omitting these parameters and let us estimate the distribution from data" << endl;
  }
  if (opt.fld < 0.0) { cerr << "Error: invalid value for mean fragment length " << opt.fld << endl; ret = false; }
  if (opt.sd < 0.0) { cerr << "Error: invalid value for fragment length standard deviation " << opt.sd << endl; ret = false; }
  if (opt.output.empty()) {
    cerr << "Error: need to specify output directory " << opt.output << endl;
    ret = false;
  } else if (stat(opt.output.c_str(), &st) == 0) {
    if (!S_ISDIR(st.st_mode)) {
      cerr << "Error: file " << opt.output << " exists and is not a directory" << endl;
      ret = false;
    }
  } else if (mkdir(opt.output.c_str(), 0777) == -1) {
    cerr << "Error: could not create directory " << opt.output << endl;
    ret = false;
  }
  if (opt.threads <= 0) {
    cerr << "Error: invalid number of threads " << opt.threads << endl;
    ret = false;
  }
  if (opt.bootstrap < 0) {
    cerr << "Error: number of bootstrap samples must be a non-negative integer." << endl;
    ret = false;
  }
  // (a reference built without HDF5 drops the bootstraps here unless --plaintext is given, src/main.cpp:1796-1803; this
  // build writes abundance.h5 itself -- csrc/h5_writer.hpp -- and so behaves like the reference built WITH HDF5)
  return ret;
}

// plaintext_writer, src/PlaintextWriter.cpp:29-65.  The reference streams every value with operator<< and
// ends every line with std::endl (one write() per transcript); the bytes are reproduced here -- default
// ostream formatting of a double is printf's %g with 6 significant digits, which is what
// std::to_chars(general, 6) is specified to produce -- but formatted into one buffer and written once.
void append_double(std::string& s, double v) {
  char buf[64];
  const auto r = std::to_chars(buf, buf + sizeof(buf), v, std::chars_format::general, 6);
  s.append(buf, r.ptr);
}
void write_abundance(const std::string& path, const std::vector<std::string>& names, const std::vector<uint32_t>& lens,
                     const double* eff, const double* est) {
  std::ofstream of(path, std::ios::out | std::ios::binary);
  if (!of.is_open()) {
    cerr << "Error: Couldn't open file: " << path << endl;
    exit(1);
  }
  std::vector<double> tpm(names.size());
  kb_counts_to_tpm(est, eff, (uint32_t)names.size(), tpm.data());
  std::string out;
  out.reserve(names.size() * 72 + 64);
  out += "target_id\tlength\teff_length\test_counts\ttpm\n";
  for (size_t i = 0; i < names.size(); ++i) {
    out += names[i];
    out += '\t';
    out += std::to_string(lens[i]);
    out += '\t';
    append_double(out, eff[i]);
    out += '\t';
    append_double(out, est[i]);
    out += '\t';
    append_double(out, tpm[i]);
    out += '\n';
  }
  of.write(out.data(), (std::streamsize)out.size());
}

// plaintext_aux, src/PlaintextWriter.cpp:140-199
// frame_clashes: `bus --aa` only, the last field "n_frame_clashes" (src/PlaintextWriter.cpp:189-195)
void write_run_info(const std::string& path, size_t n_targets, int n_bootstrap, uint64_t n_processed, uint64_t n_aln,
                    uint64_t n_unique, int index_version, int k, const std::string& start_time, const std::string& call,
                    const std::string& frame_clashes = "") {
  std::ofstream of(path);
  double p_uniq = 0.0, p_aln = 0.0;
  if (n_processed > 0) {
    p_uniq = 100.0 * (double)n_unique / (double)n_processed;
    p_aln = 100.0 * (double)n_aln / (double)n_processed;
  }
  std::stringstream ss;
  ss << std::fixed << std::setprecision(1) << p_uniq;
  const std::string p_uniq_s = ss.str();
  ss.str("");
  ss << std::fixed << std::setprecision(1) << p_aln;
  const std::string p_aln_s = ss.str();
  of << "{" << std::endl
     << to_json("n_targets", std::to_string(n_targets), false) << std::endl
     << to_json("n_bootstraps", std::to_string(n_bootstrap), false) << std::endl
     << to_json("n_processed", std::to_string(n_processed), false) << std::endl
     << to_json("n_pseudoaligned", std::to_string(n_aln), false) << std::endl
     << to_json("n_unique", std::to_string(n_unique), false) << std::endl
     << to_json("p_pseudoaligned", p_aln_s, false) << std::endl
     << to_json("p_unique", p_uniq_s, false) << std::endl
     << to_json("kallisto_version", KALLISTO_VERSION, true) << std::endl
     << to_json("index_version", std::to_string(index_version), false) << std::endl
     << to_json("k-mer length", std::to_string(k), false) << std::endl
     << to_json("start_time", start_time, true) << std::endl;
  if (!frame_clashes.empty())
    of << to_json("call", call, true) << std::endl << to_json("n_frame_clashes", frame_clashes, false, false) << std::endl;
  else
    of << to_json("call", call, true, false) << std::endl;
  of << "}" << std::endl;
}

#define KB_TRY(x)                                                     \
  do {                                                                \
    if ((x) != KB_OK) {                                               \
      cerr << "Error: " << kb_last_error() << endl;                   \
      exit(1);                                                        \
    }                                                                 \
  } while (0)

// KB_CLI_TIMING=1: wall-clock phases on stderr
struct PhaseTimer {
  bool on = getenv("KB_CLI_TIMING") != nullptr;
  bool verbose = on && atoi(getenv("KB_CLI_TIMING")) > 1;      // 2: also every round
  std::chrono::steady_clock::time_point t0 = std::chrono::steady_clock::now(), last = t0;
  void mark(const char* what) {
    if (!on) return;
    const auto now = std::chrono::steady_clock::now();
    cerr << endl << "[timing] " << what << ": " << std::chrono::duration<double>(now - last).count() << " s (at "
         << std::chrono::duration<double>(now - t0).count() << " s)";
    last = now;
  }
};

// One parser thread per input stream, handing filled batches to the GPU thread through a small ring.
struct Stream {
  std::vector<kb::ReadBatch> ring;
  std::vector<int> state;   // 0 free, 1 filled
  size_t head = 0, tail = 0;
  bool done = false;
  std::string error;
  std::mutex m;
  std::condition_variable cv;
};

void reader_thread(std::vector<std::string> files, Stream* s, size_t max_reads, int parse_threads) {
  try {
    // the ring of pinned batch buffers is allocated here, so that it happens on all streams at once and
    // while the main thread is still loading the index
    for (auto& b : s->ring) {
      b.bases = (char*)kb_host_alloc(b.cap_bases + 64);
      b.off = (uint32_t*)kb_host_alloc((b.cap_reads + 1) * sizeof(uint32_t));
      if (!b.bases || !b.off) throw std::runtime_error("Error: could not allocate pinned host memory");
      b.clear();
    }
    size_t slot = 0;
    for (auto& fn : files) {
      kb::FastxReader f(fn, parse_threads);   // plain files: mapped and parsed by parse_threads threads
      for (;;) {
        {
          std::unique_lock<std::mutex> lk(s->m);
          s->cv.wait(lk, [&] { return s->state[slot] == 0; });
        }
        kb::ReadBatch& b = s->ring[slot];
        b.clear();
        const bool any = f.fill(b, max_reads);
        if (!any) b.eof = true;     // end of this file: an empty marker batch, so that the consumer keeps file sets in step
        {
          std::lock_guard<std::mutex> lk(s->m);
          s->state[slot] = 1;
        }
        s->cv.notify_all();
        slot = (slot + 1) % s->ring.size();
        if (!any) break;
      }
    }
  } catch (const std::exception& e) {
    std::lock_guard<std::mutex> lk(s->m);
    s->error = e.what();
  }
  {
    std::lock_guard<std::mutex> lk(s->m);
    s->done = true;
  }
  s->cv.notify_all();
}

// `bus --inleaved` (src/main.cpp:583,739-741,1000-1012): ONE file holds the reads of a set one after the other (file 0's
// read, file 1's read, ...).  One parser thread reads it and deals record j to stream j % n_streams, so the consumer sees
// the same per-file streams as with separate files.  A trailing incomplete set is dropped.
void interleaved_reader_thread(std::string file, std::vector<Stream>* streams, size_t max_reads, int parse_threads) {
  const size_t nf = streams->size();
  std::string error;
  try {
    for (auto& s : *streams)
      for (auto& b : s.ring) {
        b.bases = (char*)kb_host_alloc(b.cap_bases + 64);
        b.off = (uint32_t*)kb_host_alloc((b.cap_reads + 1) * sizeof(uint32_t));
        if (!b.bases || !b.off) throw std::runtime_error("Error: could not allocate pinned host memory");
        b.clear();
      }
    kb::ReadBatch tmp;
    tmp.cap_reads = max_reads * nf;
    tmp.cap_bases = (*streams)[0].ring[0].cap_bases;
    std::vector<char> tb(tmp.cap_bases + 64);
    std::vector<uint32_t> to(tmp.cap_reads + 1);
    tmp.bases = tb.data();
    tmp.off = to.data();
    tmp.clear();
    kb::FastxReader f(file, parse_threads);
    size_t slot = 0;
    bool more = true;
    while (more) {
      more = f.fill(tmp, max_reads * nf);                      // appends to what was carried over
      const size_t n_sets = tmp.n / nf;
      if (n_sets) {
        for (size_t s = 0; s < nf; ++s) {
          Stream& st = (*streams)[s];
          {
            std::unique_lock<std::mutex> lk(st.m);
            st.cv.wait(lk, [&] { return st.state[slot] == 0; });
          }
          kb::ReadBatch& b = st.ring[slot];
          b.clear();
          for (size_t i = 0; i < n_sets; ++i) {
            const size_t r = i * nf + s;
            const uint32_t len = tmp.off[r + 1] - tmp.off[r];
            memcpy(b.bases + b.off[b.n], tmp.bases + tmp.off[r], len);
            b.off[b.n + 1] = b.off[b.n] + len;
            b.max_len = std::max(b.max_len, len);
            ++b.n;
          }
          {
            std::lock_guard<std::mutex> lk(st.m);
            st.state[slot] = 1;
          }
          st.cv.notify_all();
        }
        slot = (slot + 1) % (*streams)[0].ring.size();
      }
      // reads of an incomplete set stay for the next round
      const size_t used = n_sets * nf, rest = tmp.n - used;
      const uint32_t base = tmp.off[used];
      memmove(tmp.bases, tmp.bases + base, tmp.off[tmp.n] - base);
      for (size_t i = 0; i <= rest; ++i) tmp.off[i] = tmp.off[used + i] - base;
      tmp.n = rest;
    }
    for (size_t s = 0; s < nf; ++s) {                          // the end-of-file marker of every stream
      Stream& st = (*streams)[s];
      {
        std::unique_lock<std::mutex> lk(st.m);
        st.cv.wait(lk, [&] { return st.state[slot] == 0; });
      }
      st.ring[slot].clear();
      st.ring[slot].eof = true;
      {
        std::lock_guard<std::mutex> lk(st.m);
        st.state[slot] = 1;
      }
      st.cv.notify_all();
    }
  } catch (const std::exception& e) {
    error = e.what();
  }
  for (auto& st : *streams) {
    {
      std::lock_guard<std::mutex> lk(st.m);
      if (!error.empty()) st.error = error;
      st.done = true;
    }
    st.cv.notify_all();
  }
}

// Reads per batch of stream s.  KB_CLI_BATCH_READS="a,b,..." (tests) gives the streams different batch sizes, the
// situation that otherwise only arises when one file's batches fill up by bytes before they fill up by reads.
size_t stream_batch_reads(int s, size_t dflt) {
  const char* e = getenv("KB_CLI_BATCH_READS");
  if (!e || !*e) return dflt;
  std::vector<size_t> v;
  std::stringstream ss(e);
  std::string tok;
  while (std::getline(ss, tok, ',')) {
    const long long x = atoll(tok.c_str());
    if (x > 0) v.push_back(std::min<size_t>((size_t)x, dflt));
  }
  return v.empty() ? dflt : v[(size_t)s % v.size()];
}

// Starts one parser thread per input stream (file i of every group of n_streams files goes to stream i).  Called
// before the index is loaded: parsing does not need it, so the first batches are ready when the device is.
void start_streams(std::vector<Stream>& streams, std::vector<std::thread>& readers, const std::vector<std::string>& all_files,
                   size_t max_bases, size_t max_reads, int threads) {
  const int n_streams = (int)streams.size();
  for (int s = 0; s < n_streams; ++s) {
    streams[s].ring.resize(3);      // pinned memory is slow to pin and to release: keep the rings small
    streams[s].state.assign(3, 0);
    for (auto& b : streams[s].ring) {
      b.cap_bases = max_bases;
      b.cap_reads = max_reads;
    }
    std::vector<std::string> files;
    for (size_t i = s; i < all_files.size(); i += n_streams) files.push_back(all_files[i]);
    readers.emplace_back(reader_thread, files, &streams[s], stream_batch_reads(s, max_reads), std::max(1, threads / n_streams));
  }
}

void free_streams(std::vector<Stream>& streams) {
  for (auto& s : streams)
    for (auto& b : s.ring) {
      kb_host_free(b.bases);
      kb_host_free(b.off);
      b.bases = nullptr;
      b.off = nullptr;
    }
}

// Lock-step consumer of the parser streams.  The streams cut their batches independently (by read count
// or by bytes, whichever fills first), so a round hands out the reads that are available in EVERY stream
// and leaves the rest of a longer batch for the next round.
class LockStep {
 public:
  explicit LockStep(std::vector<Stream>& s) : st_(s), cur_(s.size(), 0), used_(s.size(), 0) {}

  // false at the end of the input.  Every input file ends with a marker batch.  When one stream reaches the end of
  // its file, what the other streams still hold of THEIR current file is dropped and all streams move on to the
  // next file set together -- FastqSequenceReader::fetchSequences (src/ProcessReads.cpp:3178-3262) stops a file set
  // at its shortest file (all_l) and reopens the next set in step.
  bool next(size_t& n, const char** bases, const uint32_t** off) {
    for (;;) {
      size_t with_data = 0;
      bool any_eof = false;
      n = (size_t)-1;
      for (size_t i = 0; i < st_.size(); ++i) {
        if (!wait_slot(i)) continue;
        ++with_data;
        const kb::ReadBatch& b = st_[i].ring[cur_[i]];
        if (b.eof) { any_eof = true; continue; }
        n = std::min(n, b.n - used_[i]);
        bases[i] = b.bases;
        off[i] = b.off + used_[i];          // offsets are absolute positions in `bases`
      }
      if (with_data == 0) return false;
      if (with_data != st_.size()) {
        cerr << endl << "Error: input files hold different numbers of reads" << endl;
        exit(1);
      }
      if (!any_eof) {
        n_ = n;
        return true;
      }
      for (size_t i = 0; i < st_.size(); ++i) {
        while (wait_slot(i) && !st_[i].ring[cur_[i]].eof) advance(i);     // rest of a longer file
        if (wait_slot(i)) advance(i);                                      // the marker itself
      }
      ++set_;
    }
  }
  // index of the file set (one file per stream) the reads of the last round came from
  size_t file_set() const { return set_; }
  // the reads of the last round have been consumed
  void release() {
    for (size_t i = 0; i < st_.size(); ++i) {
      used_[i] += n_;
      if (used_[i] == st_[i].ring[cur_[i]].n) advance(i);
    }
  }

 private:
  // waits for stream i's current slot; false when the stream has ended
  bool wait_slot(size_t i) {
    Stream& s = st_[i];
    std::unique_lock<std::mutex> lk(s.m);
    s.cv.wait(lk, [&] { return s.state[cur_[i]] == 1 || s.done; });
    if (!s.error.empty()) {
      cerr << endl << s.error << endl;
      exit(1);
    }
    return s.state[cur_[i]] == 1;
  }
  // hands stream i's current slot back to its reader
  void advance(size_t i) {
    Stream& s = st_[i];
    {
      std::lock_guard<std::mutex> lk(s.m);
      s.state[cur_[i]] = 0;
    }
    s.cv.notify_all();
    cur_[i] = (cur_[i] + 1) % s.ring.size();
    used_[i] = 0;
  }

  std::vector<Stream>& st_;
  std::vector<size_t> cur_, used_;
  size_t n_ = 0, set_ = 0;
};

// The driver initialises every VISIBLE GPU when the first CUDA call is made (about 0.1 s apiece on an 8-GPU node):
// unless the caller set CUDA_VISIBLE_DEVICES already, only the devices this run uses are made visible, and `device` /
// `devices` are renumbered to match.
void restrict_visible_devices(int& device, std::vector<int>& devices) {
  if (getenv("CUDA_VISIBLE_DEVICES")) return;
  std::string vis;
  if (devices.empty()) {
    vis = std::to_string(device);
    device = 0;
  } else {
    std::vector<int> uniq;                     // a device may be listed twice (two runs on one GPU)
    for (size_t i = 0; i < devices.size(); ++i) {
      size_t j = 0;
      while (j < uniq.size() && uniq[j] != devices[i]) ++j;
      if (j == uniq.size()) {
        uniq.push_back(devices[i]);
        vis += (vis.empty() ? "" : ",") + std::to_string(devices[i]);
      }
      devices[i] = (int)j;
    }
    device = devices[0];
  }
  setenv("CUDA_VISIBLE_DEVICES", vis.c_str(), 1);
}

// Loads the index once per device of `devices` (device 0 of the list first), in parallel; false after an error message
bool load_replicas(const std::string& path, const std::vector<int>& devices, int need_positions, int threads,
                   std::vector<kb_index*>& ixs) {
  const int n_dev = (int)devices.size();
  ixs.assign(n_dev, nullptr);
  std::vector<std::string> errs(n_dev);
  std::vector<std::thread> loaders;
  const int lt = std::max(1, std::min(16, std::max(1, threads)) / n_dev);
  for (int d = 0; d < n_dev; ++d)
    loaders.emplace_back([&, d] {
      if (kb_index_load(path.c_str(), devices[d], need_positions, lt, &ixs[d]) != KB_OK) errs[d] = kb_last_error();
    });
  for (auto& t : loaders) t.join();
  for (int d = 0; d < n_dev; ++d)
    if (!errs[d].empty()) { cerr << endl << "Error: " << errs[d] << endl; return false; }
  return true;
}

int cmd_quant(int argc, char** argv, const std::string& call, const std::string& start_time) {
  Options opt;
  parse_quant(argc, argv, opt);
  if (!check_quant(opt)) {
    cerr << endl;
    usage_quant();
    return 1;
  }
  // read before any device work, so that a bad file stops the run at once
  std::vector<double> priors;
  if (!opt.priors.empty() && !read_priors(opt.priors, priors)) return 1;
  PhaseTimer pt;
  restrict_visible_devices(opt.device, opt.devices);
  const bool paired = !opt.single_end;
  const size_t max_reads = 1u << 19;                 // reads per batch and mate (pinned rings: 3 x 2 x ~70 MB)
  const size_t max_bases = (size_t)max_reads * 136 + kb::FastxFile::kMaxRead;
  const int n_streams = paired ? 2 : 1;
  std::vector<Stream> streams(n_streams);
  std::vector<std::thread> readers;
  start_streams(streams, readers, opt.files, max_bases, max_reads, opt.threads);
  kb_index* ix = nullptr;
  // positions are needed only by the fragment-position filter (KmerIndex.h:78: load_positional_info)
  const int need_positions = (!opt.single_overhang && opt.fld > 0.0) ? 1 : 0;
  // --devices: the index is replicated (one load per device, in parallel); device 0 of the list is the root
  const int n_dev = std::max<int>(1, (int)opt.devices.size());
  std::vector<kb_index*> ixs(n_dev, nullptr);
  {
    std::vector<std::string> errs(n_dev);
    std::vector<std::thread> loaders;
    const int lt = std::max(1, std::min(16, std::max(1, opt.threads)) / n_dev);
    for (int d = 1; d < n_dev; ++d)
      loaders.emplace_back([&, d] {
        if (kb_index_load(opt.index.c_str(), opt.devices[d], need_positions, lt, &ixs[d]) != KB_OK) errs[d] = kb_last_error();
      });
    KB_TRY(kb_index_load(opt.index.c_str(), opt.device, need_positions, n_dev > 1 ? lt : std::min(16, std::max(1, opt.threads)), &ix));
    ixs[0] = ix;
    for (auto& t : loaders) t.join();
    for (int d = 1; d < n_dev; ++d)
      if (!errs[d].empty()) { cerr << endl << "Error: " << errs[d] << endl; return 1; }
  }
  pt.mark("index load");
  kb_index_info info;
  kb_index_get_info(ix, &info);
  if (pt.on) cerr << endl << "[timing] index load detail: file parse || CUDA context " << info.load_seconds << " s, uploads + table build "
                  << info.build_seconds << " s";
  cerr << "[index] k-mer length: " << info.k << endl;
  cerr << "[index] number of targets: " << pretty_num(info.n_targets) << endl;
  cerr << "[index] number of k-mers: " << pretty_num(info.n_kmers) << endl;
  cerr << (paired ? "[quant] running in paired-end mode" : "[quant] running in single-end mode") << endl;
  for (size_t i = 0; i < opt.files.size(); i += paired ? 2 : 1) {
    if (paired)
      cerr << "[quant] will process pair " << (i / 2 + 1) << ": " << opt.files[i] << endl
           << "                             " << opt.files[i + 1] << endl;
    else
      cerr << "[quant] will process file " << i + 1 << ": " << opt.files[i] << endl;
  }
  cerr << "[quant] finding pseudoalignments for the reads ...";
  cerr.flush();

  kb_quant_opts qo{};
  qo.paired = paired;
  qo.strand_mode = opt.strand;
  qo.collect_fld = opt.fld == 0.0;
  qo.single_overhang = opt.single_overhang;
  qo.fld_mean = opt.fld;
  qo.max_batch_reads = (uint32_t)max_reads;
  qo.max_batch_bases = 2 * max_bases;
  kb_quant* q = nullptr;
  KB_TRY(kb_quant_create(ix, &qo, &q));
  if (pt.on) kb_quant_enable_timing(q, 1);
  std::vector<kb_quant*> qs(n_dev, nullptr);
  qs[0] = q;
  for (int d = 1; d < n_dev; ++d) {
    kb_quant_opts qd = qo;
    qd.collect_fld = 0;        // the fragment-length samples are the first 10000 of the stream: device 0 sees them (below)
    KB_TRY(kb_quant_create(ixs[d], &qd, &qs[d]));
  }

  pt.mark("run set-up");
  uint64_t n_done = 0;
  {
    LockStep ls(streams);
    const char* bp[2] = {nullptr, nullptr};
    const uint32_t* op[2] = {nullptr, nullptr};
    size_t n = 0;
    size_t round = 0;
    bool fld_done = !(paired && opt.fld == 0.0) || n_dev == 1;
    while (ls.next(n, bp, op)) {
      const auto c0 = std::chrono::steady_clock::now();
      // batches are dealt round-robin once the root has its 10000 fragment-length samples (ProcessReads.cpp:985-1004:
      // they are the first qualifying pairs of the input); every batch carries its global fragment index, so EC ids
      // come out in the order of the input whatever device saw a fragment first
      kb_quant* qq = q;
      if (n_dev > 1) {
        if (fld_done) qq = qs[round % n_dev];
        kb_quant_set_frag_base(qq, n_done);
      }
      if (paired) KB_TRY(kb_pseudoalign_batch_pe(qq, bp[0], op[0], bp[1], op[1], (uint32_t)n, 0, nullptr));
      else KB_TRY(kb_pseudoalign_batch(qq, bp[0], op[0], (uint32_t)n, 0, nullptr));
      ++round;
      if (!fld_done) {
        uint32_t fl[1000];
        kb_quant_get_flens(q, fl);
        uint64_t c = 0;
        for (int i = 0; i < 1000; ++i) c += fl[i];
        fld_done = c >= 10000;
      }
      if (pt.verbose) cerr << endl << "[timing] round of " << n << " reads: call " << std::chrono::duration<double>(std::chrono::steady_clock::now() - c0).count()
                      << " s, at " << std::chrono::duration<double>(std::chrono::steady_clock::now() - pt.t0).count() << " s";
      n_done += n;
      if (opt.verbose) cerr << endl << "[quant] processed " << pretty_num(n_done) << " reads";
      ls.release();
    }
  }
  for (auto& t : readers) t.join();
  pt.mark("read + pseudoalign loop");
  if (n_dev > 1) {
    // the one exchange: every device's equivalence classes copied to the root over NVLink and folded in by content
    // (all runs live in this process, so no NCCL communicator is needed; multi-process drivers use kb_quant_merge_nccl)
    KB_TRY(kb_quant_merge_local(qs[0], qs.data() + 1, n_dev - 1, nullptr));
    pt.mark("merge (peer copies)");
  }
  cerr << " done" << endl;
  if (opt.write_index) {
    // --write-index: counts.txt = "id <tab> count" per equivalence class in id order (MinCollector::write,
    // src/MinCollector.h:74-78, src/ProcessReads.cpp:242-249) and the stripped index (src/main.cpp:2658-2661)
    kb_run_stats s0{};
    KB_TRY(kb_quant_finalize(q, &s0));
    std::vector<uint64_t> eo(s0.n_ecs + 1);
    std::vector<uint32_t> et(std::max<uint64_t>(1, s0.n_ec_entries)), ec(std::max<uint64_t>(1, s0.n_ecs));
    KB_TRY(kb_quant_ec_table(q, eo.data(), et.data(), ec.data(), nullptr));
    std::ofstream cf(opt.output + "/counts.txt");
    for (uint64_t i = 0; i < s0.n_ecs; ++i) cf << i << "\t" << ec[i] << "\n";
    cf.close();
    write_index_saved(opt.index, opt.output + "/index.saved", info.k);
  }

  const uint32_t T = info.n_targets;
  std::vector<double> est(T), eff(T);
  int32_t rounds = 0;
  uint32_t flens[1000];
  kb_quant_get_flens(q, flens);
  if (opt.fld == 0.0) {
    uint64_t c = 0;
    for (int i = 0; i < 1000; ++i) c += flens[i];
    if (c == 0 && paired) {
      // MinCollector::get_mean_frag_len (src/MinCollector.cpp:583-607) would stop here as well
    }
  }
  // the run that solves the EM (the root with --devices) starts from the priors (src/main.cpp:2683-2689)
  std::string priors_msg;
  if (!opt.priors.empty()) {
    priors_msg = "[   em] reading priors from file " + opt.priors + "\n";
    if (priors.size() == T) {
      if (!kb_em_set_priors) { cerr << "Error: this libkallisto_b200 has no kb_em_set_priors" << endl; return 1; }
      KB_TRY(kb_em_set_priors(q, priors.data(), T));
    }
  }
  KB_TRY(kb_em_run(q, opt.fld, opt.sd, est.data(), eff.data(), &rounds, nullptr));
  pt.mark("EM");
  if (pt.on) {
    kb_kernel_timings kt{};
    kb_quant_get_timings(q, &kt);
    cerr << endl << "[timing] device: match " << kt.match_ms << " ms in " << kt.match_launches << " launches, resolve " << kt.resolve_ms
         << " ms in " << kt.resolve_launches << " launches, EM " << kt.em_ms << " ms, EM set-up " << kt.em_prep_ms << " ms";
  }
  kb_run_stats st{};
  KB_TRY(kb_quant_finalize(q, &st));
  cerr << "[quant] processed " << pretty_num(st.n_processed) << " reads, " << pretty_num(st.n_pseudoaligned)
       << " reads pseudoaligned" << endl;
  if (st.n_pseudoaligned == 0) cerr << "[~warn] no reads pseudoaligned." << endl;
  if (opt.fld == 0.0) {
    // compute_mean_frag_lens_trunc(verbose): mean over the whole histogram
    double mass = 0;
    uint64_t cnt = 0;
    for (size_t i = 0; i < 1000; ++i) { mass += (double)(flens[i] * i); cnt += flens[i]; }
    cerr << "[quant] estimated average fragment length: " << (cnt ? mass / (double)cnt : 0.0) << endl;
  }
  if (!opt.priors.empty()) {
    cerr << priors_msg;
    priors_apply(priors, T);
  }
  cerr << "[   em] quantifying the abundances ... done" << endl;
  cerr << "[   em] the Expectation-Maximization algorithm ran for " << pretty_num((size_t)rounds) << " rounds" << endl;

  std::vector<std::string> names(T);
  std::vector<uint32_t> lens(T);
  for (uint32_t i = 0; i < T; ++i) names[i] = kb_index_target_name(ix, i);
  kb_index_target_lens(ix, lens.data());
  if (st.n_pseudoaligned == 0) cerr << "[~warn] Warning, zero reads pseudoaligned check your input files and index" << endl;
  write_run_info(opt.output + "/run_info.json", T, opt.bootstrap, st.n_processed, st.n_pseudoaligned, st.n_unique, 13,
                 info.k, start_time, call);
  write_abundance(opt.output + "/abundance.tsv", names, lens, eff.data(), est.data());
  pt.mark("finalize + write abundance.tsv");
  if (pt.on) cerr << endl;
  // without --plaintext the estimates (and the bootstraps) also go into abundance.h5, as in a reference built with HDF5
  // (H5Writer::init / write_main / write_bootstrap, src/H5Writer.cpp:4-71; src/main.cpp:2693-2702,2732-2776)
  kb::H5Writer h5;
  int h5_aux = -1, h5_bs = -1;
  if (!opt.plaintext) {
    h5.add_f64(0, "est_counts", est.data(), T);
    h5_aux = h5.group("aux");
    if (opt.bootstrap > 0) h5_bs = h5.group("bootstrap");
    const int32_t nb = opt.bootstrap, np = (int32_t)st.n_processed, iv = 13;
    h5.add_i32(h5_aux, "num_bootstrap", &nb, 1);
    h5.add_i32(h5_aux, "num_processed", &np, 1);
    std::vector<int32_t> fld(1000, 0);
    if (opt.fld == 0.0) {
      for (int i = 0; i < 1000; ++i) fld[i] = (int32_t)flens[i];
    } else {      // trunc_gaussian_counts(0, MAX_FRAG_LEN, mean, sd, 10000), src/weights.cpp:273-296
      double total_mass = 0.0;
      for (int i = 0; i < 1000; ++i) { const double x = ((double)i - opt.fld) / opt.sd; total_mass += std::exp(-0.5 * x * x) / opt.sd; }
      for (int i = 0; i < 1000; ++i) {
        const double x = ((double)i - opt.fld) / opt.sd;
        fld[i] = (int)std::round(std::exp(-0.5 * x * x) / opt.sd * 10000 / total_mass);
      }
    }
    h5.add_i32(h5_aux, "fld", fld.data(), fld.size());
    const std::vector<int32_t> bias_obs(4096, 1);        // no --bias in this build: the reference's untouched vectors
    const std::vector<double> bias_norm(4096, 1.0);      // (src/main.cpp:2676, src/EMAlgorithm.h:37)
    h5.add_i32(h5_aux, "bias_observed", bias_obs.data(), bias_obs.size());
    h5.add_f64(h5_aux, "bias_normalized", bias_norm.data(), bias_norm.size());
    h5.add_str(h5_aux, "kallisto_version", {KALLISTO_VERSION});
    h5.add_i32(h5_aux, "index_version", &iv, 1);
    h5.add_str(h5_aux, "call", {call});
    h5.add_str(h5_aux, "start_time", {start_time});
    h5.add_str(h5_aux, "ids", names);
    h5.add_f64(h5_aux, "eff_lengths", eff.data(), T);
    std::vector<int32_t> l32(lens.begin(), lens.end());
    h5.add_i32(h5_aux, "lengths", l32.data(), T);
  }
  auto emit_bs = [&](int b, const double* alpha) {
    if (opt.plaintext) write_abundance(opt.output + "/bs_abundance_" + std::to_string(b) + ".tsv", names, lens, eff.data(), alpha);
    else h5.add_f64(h5_bs, "bs" + std::to_string(b), alpha, T);
  };
  if (opt.bootstrap > 0 && st.n_pseudoaligned == 0) {
    for (int b = 0; b < opt.bootstrap; ++b) emit_bs(b, est.data());
  } else if (opt.bootstrap > 0) {
    std::vector<double> bs((size_t)opt.bootstrap * T);
    cerr << "[bstrp] running EM for " << opt.bootstrap << " bootstraps on the device" << endl;
    KB_TRY(kb_bootstrap_run(q, opt.fld, opt.sd, opt.seed, opt.bootstrap, bs.data(), nullptr, nullptr));
    if (opt.plaintext) {
      // one text file per sample (0.06 s of formatting each for a human transcriptome): written by several threads
      std::atomic<int> next{0};
      auto work = [&] {
        for (int b; (b = next.fetch_add(1)) < opt.bootstrap;) emit_bs(b, bs.data() + (size_t)b * T);
      };
      const int nt = std::max(1, std::min({opt.threads, opt.bootstrap, 32}));
      std::vector<std::thread> pool;
      for (int t = 1; t < nt; ++t) pool.emplace_back(work);
      work();
      for (auto& th : pool) th.join();
    } else {
      for (int b = 0; b < opt.bootstrap; ++b) emit_bs(b, bs.data() + (size_t)b * T);
    }
  }
  if (!opt.plaintext && !h5.write(opt.output + "/abundance.h5")) {
    cerr << "Error: could not write " << opt.output << "/abundance.h5" << endl;
    exit(1);
  }
  cerr << endl;
  if (!getenv("KB_CLI_CLEANUP")) finish(st.n_pseudoaligned == 0 ? 1 : 0);
  free_streams(streams);
  for (int d = 0; d < n_dev; ++d) {
    kb_quant_free(qs[d]);
    kb_index_free(ixs[d]);
  }
  return st.n_pseudoaligned == 0 ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// kallisto bus (src/main.cpp:541-776 ParseOptionsBus, 923-1526 CheckOptionsBus, 2336-2617 body)
// ------------------------------------------------------------------------------------------------
struct Tech {
  const char* name;
  int nfiles;
  std::vector<kb_bus_substr> bc, umi;
  kb_bus_substr seq;
  int strand;   // default strand of the technology: 0 none, 1 FR, 2 RF
  kb_bus_substr seq2 = {-1, 0, 0};   // paired technologies: the second sequence read
};

const std::vector<Tech>& tech_table() {   // src/main.cpp:1283-1407.
                                          // SMARTSEQ2 grows a fourth file with --paired (cmd_bus).  "STORM-seq" cannot be
                                          // selected in the reference either: -x is upper-cased (:619) before it is compared
                                          // with the mixed-case name (:1358); its layout is -x -1,-1,-1:1,0,8:0,0,0,1,14,0
  static const std::vector<Tech> t = {
      {"SMARTSEQ2", 3, {{0, 0, 0}, {1, 0, 0}}, {{-1, -1, -1}}, {2, 0, 0}, 0},
      {"SMARTSEQ3", 4, {{0, 0, 0}, {1, 0, 0}}, {{2, 0, 19}}, {2, 22, 0}, 1, {3, 0, 0}},      // + the default tag sequence, below
      {"BDWTA", 2, {{0, 0, 9}, {0, 21, 30}, {0, 43, 52}}, {{0, 52, 60}}, {1, 0, 0}, 1},
      {"VASA-SEQ", 1, {{0, 6, 14}}, {{0, 0, 6}}, {0, 14, 0}, 1},
      {"10XV1", 3, {{0, 0, 14}}, {{1, 0, 10}}, {2, 0, 0}, 1},
      {"10XV2", 2, {{0, 0, 16}}, {{0, 16, 26}}, {1, 0, 0}, 1},
      {"10XV3", 2, {{0, 0, 16}}, {{0, 16, 28}}, {1, 0, 0}, 1},
      {"VISIUM", 2, {{0, 0, 16}}, {{0, 16, 28}}, {1, 0, 0}, 1},
      {"SURECELL", 2, {{0, 0, 6}, {0, 21, 27}, {0, 42, 48}}, {{0, 51, 59}}, {1, 0, 0}, 1},
      {"DROPSEQ", 2, {{0, 0, 12}}, {{0, 12, 20}}, {1, 0, 0}, 0},
      {"INDROPSV1", 2, {{0, 0, 11}, {0, 30, 38}}, {{0, 42, 48}}, {1, 0, 0}, 0},
      {"INDROPSV2", 2, {{1, 0, 11}, {1, 30, 38}}, {{1, 42, 48}}, {0, 0, 0}, 0},
      {"INDROPSV3", 3, {{0, 0, 8}, {1, 0, 8}}, {{1, 8, 14}}, {2, 0, 0}, 0},
      {"CELSEQ", 2, {{0, 0, 8}}, {{0, 8, 12}}, {1, 0, 0}, 1},
      {"CELSEQ2", 2, {{0, 6, 12}}, {{0, 0, 6}}, {1, 0, 0}, 1},
      {"SPLIT-SEQ", 2, {{1, 10, 18}, {1, 48, 56}, {1, 78, 86}}, {{1, 0, 10}}, {0, 0, 0}, 1},
      {"SCRBSEQ", 2, {{0, 0, 6}}, {{0, 6, 16}}, {1, 0, 0}, 0},
  };
  return t;
}

bool parse_triplets(const std::string& s, std::vector<kb_bus_substr>& out) {
  std::vector<int> v;
  std::stringstream ss(s);
  std::string tok;
  while (std::getline(ss, tok, ',')) {
    try { v.push_back(std::stoi(tok)); } catch (...) { return false; }
  }
  if (v.empty() || v.size() % 3) return false;
  for (size_t i = 0; i < v.size(); i += 3) out.push_back(kb_bus_substr{v[i], v[i + 1], v[i + 2]});
  return true;
}

// index.saved of `kallisto bus` (KmerIndex::write(fn, false), src/KmerIndex.cpp:1226-1327): the index without graph,
// D-list and nodes -- what `quant-tcc` needs next to matrix.ec: version, three empty sections, then the number of real
// targets followed by the input file's own tail (target lengths, names, on-list), which the reference re-serialises
// unchanged.  The tail is found by walking the sections of the v13 file (SURVEY.md appendix B).
void write_index_saved(const std::string& in_path, const std::string& out_path, int k) {
  // the file is mapped and walked by pointer: a human index has ~10^6 node records to step over
  const int fd = open(in_path.c_str(), O_RDONLY);
  struct stat sb;
  const uint8_t* base = nullptr;
  if (fd >= 0 && fstat(fd, &sb) == 0 && sb.st_size > 0) {
    void* m = mmap(nullptr, (size_t)sb.st_size, PROT_READ, MAP_PRIVATE, fd, 0);
    if (m != MAP_FAILED) base = (const uint8_t*)m;
  }
  if (fd >= 0) close(fd);
  const uint64_t size = base ? (uint64_t)sb.st_size : 0;
  uint64_t o = 0;
  bool ok = base != nullptr;
  auto rd64 = [&]() -> uint64_t {
    uint64_t v = 0;
    if (ok && o + 8 <= size) memcpy(&v, base + o, 8); else ok = false;
    o += 8;
    return v;
  };
  auto skip = [&](uint64_t n) { if (ok && n <= size - std::min(o, size)) o += n; else ok = false; };
  const uint64_t version = rd64();
  const uint64_t dbg_bytes = rd64() & ~(1ull << 63);
  skip(dbg_bytes);
  if (dbg_bytes) skip(rd64());      // the MPHF section exists only next to a graph (src/KmerIndex.cpp:1365-1383)
  const uint64_t dlist_n = rd64();
  rd64();      // D-list overhang
  skip(dlist_n * 8);
  const uint64_t n_nodes = rd64();
  for (uint64_t i = 0; i < n_nodes && ok; ++i) {
    skip((uint64_t)k);
    uint32_t nb = 0;
    if (ok && o + 4 <= size) memcpy(&nb, base + o, 4); else ok = false;
    o += 4;
    skip(nb);
  }
  int32_t num_trans = 0;
  if (ok && o + 4 <= size) memcpy(&num_trans, base + o, 4); else ok = false;
  o += 4;
  if (!ok || version != 13) {
    cerr << "Error: could not read " << in_path << " to write index.saved" << endl;
    exit(1);
  }
  num_trans -= (int32_t)dlist_n;
  std::ofstream out(out_path, std::ios::binary);
  const uint64_t head[5] = {13, 0, 0, 1, 0};      // version, graph bytes, D-list size, D-list overhang, nodes
  out.write((const char*)head, sizeof(head));
  out.write((const char*)&num_trans, 4);
  out.write((const char*)base + o, (std::streamsize)(size - o));
  munmap((void*)base, (size_t)size);
}

void usage_bus() {
  std::cout << "kallisto_b200 " << KALLISTO_VERSION << " (H100 build)" << endl
            << "Generates BUS files for single-cell sequencing" << endl << endl
            << "Usage: kallisto_b200 bus [arguments] FASTQ-files" << endl << endl
            << "Required arguments:" << endl
            << "-i, --index=STRING            Filename for the kallisto index to be used for" << endl
            << "                              pseudoalignment" << endl
            << "-o, --output-dir=STRING       Directory to write output to" << endl
            << "-x, --technology=STRING       Single-cell technology used (10xv1, 10xv2, 10xv3, visium, surecell," << endl
            << "                              dropseq, indropsv1/2/3, celseq, celseq2, split-seq, scrbseq, bdwta," << endl
            << "                              vasa-seq, smartseq2, smartseq3), a custom bc:umi:seq string of file,start,stop" << endl
            << "                              triplets, or bulk (every file or file pair is a sample of its own)" << endl << endl
            << "Optional arguments:" << endl
            << "-t, --threads=INT             Number of host threads (default: 1)" << endl
            << "-n, --num                     Output number of read in flag column" << endl
            << "    --paired                  Treat reads as paired (bulk, smartseq2, custom technologies with two" << endl
            << "                              sequence reads)" << endl
            << "    --inleaved                Specifies that input is an interleaved FASTQ file" << endl
            << "    --tag=STRING              5' tag sequence to identify UMI reads for certain technologies" << endl
            << "    --batch=FILE              Process files listed in FILE (lines: id file1 [file2 ...], as many files" << endl
            << "                              as the technology reads), one sample per line; lines with the same id are" << endl
            << "                              one sample" << endl
            << "    --batch-barcodes          With --batch and a technology: write the sample's number into the barcode," << endl
            << "                              in front of the technology's barcode (32 letters in all; at most 32" << endl
            << "                              barcode letters), so that equal barcodes of different samples stay apart" << endl
            << "    --fr-stranded / --rf-stranded / --unstranded   Strand specificity" << endl
            << "    --aa                      Align to index generated from a FASTA-file containing amino acid sequences" << endl
            << "                              (single-end reads; not with --tag or an index with a D-list)" << endl
            << "    --device=INT              CUDA device ordinal (default: 0)" << endl
            << "    --devices=LIST            Comma-separated CUDA devices (a device may be listed twice): batches of" << endl
            << "                              read sets are dealt to all of them; output as with one device" << endl;
}

int cmd_bus(int argc, char** argv, const std::string& call, const std::string& start_time) {
  Options opt;
  std::string technology, tagsequence, batch_file;
  int num_flag = 0, fr = 0, rf = 0, unstranded = 0, verbose_flag = 0, paired_flag = 0, interleaved_flag = 0;
  int aa_flag = 0, union_flag = 0, no_jump_flag = 0, batch_barcodes_flag = 0;
  const char* opt_string = "i:o:x:t:nD:T:B:";
  static struct option long_options[] = {{"verbose", no_argument, &verbose_flag, 1},
                                         {"paired", no_argument, &paired_flag, 1},
                                         {"inleaved", no_argument, &interleaved_flag, 1},
                                         {"aa", no_argument, &aa_flag, 1},
                                         {"union", no_argument, &union_flag, 1},
                                         {"no-jump", no_argument, &no_jump_flag, 1},
                                         {"tag", required_argument, 0, 'T'},
                                         {"batch", required_argument, 0, 'B'},
                                         {"batch-barcodes", no_argument, &batch_barcodes_flag, 1},
                                         {"num", no_argument, 0, 'n'},
                                         {"fr-stranded", no_argument, &fr, 1},
                                         {"rf-stranded", no_argument, &rf, 1},
                                         {"unstranded", no_argument, &unstranded, 1},
                                         {"index", required_argument, 0, 'i'},
                                         {"output-dir", required_argument, 0, 'o'},
                                         {"technology", required_argument, 0, 'x'},
                                         {"threads", required_argument, 0, 't'},
                                         {"device", required_argument, 0, 'D'},
                                         {"devices", required_argument, 0, 'G'},
                                         {0, 0, 0, 0}};
  int c, oi = 0;
  bool bad_devices = false;
  while ((c = getopt_long(argc, argv, opt_string, long_options, &oi)) != -1) {
    switch (c) {
      case 'i': opt.index = optarg; break;
      case 'o': opt.output = optarg; break;
      case 'x': technology = optarg; break;
      case 'G': {
        std::stringstream ss(optarg);
        std::string tok;
        opt.devices.clear();
        while (std::getline(ss, tok, ',')) {
          int v = -1;
          const auto r = std::from_chars(tok.data(), tok.data() + tok.size(), v);
          if (r.ec != std::errc() || r.ptr != tok.data() + tok.size() || v < 0) bad_devices = true;
          opt.devices.push_back(v);
        }
        if (opt.devices.empty()) bad_devices = true;
        break;
      }
      case 't': std::stringstream(optarg) >> opt.threads; break;
      case 'n': num_flag = 1; break;
      case 'D': std::stringstream(optarg) >> opt.device; break;
      case 'T': std::stringstream(optarg) >> tagsequence; break;
      case 'B': batch_file = optarg; break;
      default: break;
    }
  }
  for (int i = optind; i < argc; i++) opt.files.push_back(argv[i]);
  if (!opt.devices.empty()) opt.device = opt.devices[0];
  // ---- CheckOptionsBus
  bool ret = true;
  struct stat stt;
  cerr << endl;
  if (bad_devices) { cerr << "Error: --devices needs a comma-separated list of device ordinals (e.g. 0,1 or 0,0)" << endl; ret = false; }
  if (opt.index.empty()) { cerr << ERROR_STR << " kallisto index file missing" << endl; ret = false; }
  else if (stat(opt.index.c_str(), &stt) != 0) { cerr << ERROR_STR << " kallisto index file not found " << opt.index << endl; ret = false; }
  if (opt.threads <= 0) { cerr << "Error: invalid number of threads " << opt.threads << endl; ret = false; }
  if (interleaved_flag) {      // src/main.cpp:1000-1012
    if (opt.files.size() > 1) { cerr << ERROR_STR << " interleaved input cannot consist of more than one input" << endl; ret = false; }
    if (!batch_file.empty()) { cerr << ERROR_STR << " interleaved input cannot be specified with a batch file" << endl; ret = false; }
  }
  std::string tech_upper = technology;
  for (auto& ch : tech_upper) ch = (char)toupper(ch);
  const bool from_batch_file = !batch_file.empty() && (technology.empty() || tech_upper == "BULK");
  // --batch with a technology (src/main.cpp:1221-1273): "id file1 file2 ...", as many files per line as the first line has
  const bool tech_batch = !batch_file.empty() && !from_batch_file;
  size_t tech_batch_nfiles = 0;
  std::vector<std::string> batch_files;       // the files of its lines, in order
  std::vector<std::string> sample_names;      // --batch: the ids of the lines (matrix.cells)
  std::vector<uint64_t> sample_barcode;       // batch_id_mapping: lines with the same id share a barcode (src/ProcessReads.h:211-224)
  auto sample_number = [&](const std::string& id) {
    for (size_t j = 0; j < sample_barcode.size(); ++j)
      if (sample_names[j] == id) return sample_barcode[j];
    uint64_t n = 0;
    for (uint64_t v : sample_barcode) n = std::max(n, v + 1);
    return n;
  };
  if (tech_batch) {
    cerr << "[bus] will try running read files supplied in batch file" << endl;
    if (!opt.files.empty()) { cerr << ERROR_STR << " cannot specify batch mode and supply read files" << endl; ret = false; }
    if (stat(batch_file.c_str(), &stt) != 0) { cerr << ERROR_STR << " file not found " << batch_file << endl; ret = false; }
    std::ifstream bfile(batch_file);
    std::string line;
    bool first = true;
    std::vector<std::string> line_files;
    while (std::getline(bfile, line)) {
      if (line.empty()) continue;
      std::stringstream ss(line);
      std::string id, f;
      ss >> id;
      if (id.empty() || id[0] == '#') continue;
      const uint64_t bcv = sample_number(id);
      sample_names.push_back(id);
      sample_barcode.push_back(bcv);
      line_files.clear();
      while (ss >> f) {
        if (stat(f.c_str(), &stt) != 0) { cerr << ERROR_STR << " file not found " << f << endl; ret = false; }
        line_files.push_back(f);
      }
      if (first) { tech_batch_nfiles = line_files.size(); first = false; }
      if (line_files.size() != tech_batch_nfiles) { cerr << ERROR_STR << " batch file malformatted" << endl; ret = false; break; }
      batch_files.insert(batch_files.end(), line_files.begin(), line_files.end());
    }
    if (!ret) {      // CheckOptionsBus returns here (src/main.cpp:1274)
      usage_bus();
      return 1;
    }
  }
  if (from_batch_file) {
    // src/main.cpp:1108-1180: "id file1 [file2]" per line, '#' lines skipped, the first line decides single / paired
    cerr << "[bus] will try running read files supplied in batch file" << endl;
    if (paired_flag) cerr << "[bus] --paired ignored; single/paired-end is inferred from number of files supplied" << endl;
    if (!opt.files.empty()) { cerr << ERROR_STR << " cannot specify batch mode and supply read files" << endl; ret = false; }
    else {
      if (stat(batch_file.c_str(), &stt) != 0) { cerr << ERROR_STR << " file not found " << batch_file << endl; ret = false; }
      std::ifstream bfile(batch_file);
      std::string line;
      bool first = true, single = true;
      std::vector<std::pair<std::string, uint64_t>> seen;
      while (std::getline(bfile, line)) {
        if (line.empty()) continue;
        std::stringstream ss(line);
        std::string id, f1, f2;
        ss >> id;
        if (id.empty() || id[0] == '#') continue;
        ss >> f1 >> f2;
        if (first) { single = f2.empty(); first = false; }
        sample_names.push_back(id);
        uint64_t bcv = seen.size();
        for (auto& pr : seen) if (pr.first == id) bcv = pr.second;
        if (bcv == seen.size()) seen.push_back({id, bcv});
        sample_barcode.push_back(bcv);
        if (stat(f1.c_str(), &stt) != 0) { cerr << ERROR_STR << " file not found " << f1 << endl; ret = false; }
        opt.files.push_back(f1);
        if (single) {
          if (!f2.empty()) { cerr << ERROR_STR << " batch file malformatted" << endl; ret = false; break; }
        } else {
          if (f2.empty()) { cerr << ERROR_STR << " batch file malformatted" << endl; ret = false; break; }
          if (stat(f2.c_str(), &stt) != 0) { cerr << ERROR_STR << " file not found " << f2 << endl; ret = false; }
          opt.files.push_back(f2);
        }
      }
      paired_flag = single ? 0 : 1;
    }
  }
  if (tech_batch) opt.files = batch_files;      // read files next to --batch were refused above
  if (opt.files.empty() && !from_batch_file && !tech_batch) { cerr << ERROR_STR << " Missing read files" << endl; ret = false; }
  if (!from_batch_file && !tech_batch)
    for (auto& fn : opt.files)
      if (stat(fn.c_str(), &stt) != 0) { cerr << ERROR_STR << " file not found " << fn << endl; ret = false; }
  kb_bus_opts bo{};
  bo.seq2 = kb_bus_substr{-1, 0, 0};
  int tech_strand = 0;
  bool batch_mode = false;      // -x BULK / --batch: every file (pair) is a sample of its own (src/main.cpp:1050-1214)
  if (technology.empty() && !from_batch_file) {
    if (ret) cerr << "Error: the technology must be specified via -x, use \"bulk\" for regular RNA-seq reads" << endl;   // src/main.cpp:1058
    ret = false;
  } else if (tech_upper == "BULK" || from_batch_file) {
    // batch mode without a technology (:1050-1107, 1190-1214): no barcode read, no UMI, the whole read(s) are the sequence
    batch_mode = true;
    if (ret && !from_batch_file && paired_flag && opt.files.size() % 2 != 0 && !interleaved_flag) {
      cerr << "Error: paired-end mode requires an even number of input files" << endl;
      ret = false;
    }
    bo.nfiles = paired_flag ? 2 : 1;
    bo.n_bc = 0;
    bo.n_umi = 1;
    bo.umi[0] = kb_bus_substr{-1, -1, -1};
    bo.seq = kb_bus_substr{0, 0, 0};
    if (paired_flag) { bo.paired = 1; bo.seq2 = kb_bus_substr{1, 0, 0}; }
    if (!tagsequence.empty()) {      // src/main.cpp:1191-1194
      cerr << "Error: --tag not supported in this mode" << endl;
      ret = false;
    }
  } else {
    std::string up = technology;
    for (auto& ch : up) ch = (char)toupper(ch);
    const Tech* found = nullptr;
    for (auto& t : tech_table())
      if (up == t.name) found = &t;
    std::vector<kb_bus_substr> bc, umi, seq;
    if (found) {
      bo.nfiles = found->nfiles;
      bc = found->bc; umi = found->umi; seq = {found->seq};
      tech_strand = found->strand;
      if (found->seq2.fileno >= 0) seq.push_back(found->seq2);
      if (up == "SMARTSEQ2" && paired_flag) {      // src/main.cpp:1386-1392
        bo.nfiles++;
        seq.push_back(kb_bus_substr{3, 0, 0});
      }
      if (bc.size() == 1 && bc[0].fileno == -1) bc.clear();
    } else if (technology.find(':') != std::string::npos) {
      std::vector<std::string> parts;
      std::stringstream ss(technology);
      std::string part;
      while (std::getline(ss, part, ':')) parts.push_back(part);
      const size_t n_colons = (size_t)std::count(technology.begin(), technology.end(), ':');
      if (n_colons != 2) {
        cerr << "Error: technology string must contain two colons (:), " << (n_colons == 1 ? "only one found" : "three found") << ": \""
             << tech_upper << "\"" << endl;
        ret = false;
      } else if (parts.size() != 3 || !parse_triplets(parts[0], bc) || !parse_triplets(parts[1], umi) || !parse_triplets(parts[2], seq)) {
        cerr << "Error: could not parse technology string " << technology << endl;
        ret = false;
      } else {
        int nf = 0;
        for (auto* v : {&bc, &umi, &seq}) for (auto& x : *v) nf = std::max(nf, x.fileno + 1);
        bo.nfiles = nf;
        if (bc.size() == 1 && bc[0].fileno == -1) bc.clear();   // no barcode
      }
    } else {
      // ParseTechnology, src/main.cpp:778-794: anything that is not a known name is read as a bc:umi:seq string
      cerr << "Error: technology string must contain two colons (:), none found: \"" << tech_upper << "\"" << endl;
      ret = false;
    }
    if (ret) {
      // two sequence reads are a pair when the technology says so or with --paired (src/main.cpp:1424-1426); without
      // --paired the reference glues them together with an N in between (:1568-1580), which this build does not do
      const bool tech_paired = found && found->seq2.fileno >= 0;
      const bool two = seq.size() == 2 && (tech_paired || paired_flag);
      bool bad = (seq.size() != 1 && !two) || bc.size() > 4 || umi.empty() || umi.size() > 4 || bo.nfiles > 4;
      for (auto& x : seq) bad = bad || x.stop != 0 || x.fileno < 0;
      if (two && seq[0].fileno == seq[1].fileno) bad = true;
      for (auto& x : umi) if (x.fileno < 0 && umi.size() != 1) bad = true;
      if (bad) {
        cerr << "Error: this build handles technologies with one sequence read, or two that form a pair, running to the end of their files" << endl;
        ret = false;
      } else {
        bo.n_bc = (int)bc.size();
        for (size_t i = 0; i < bc.size(); ++i) bo.bc[i] = bc[i];
        bo.n_umi = (int)umi.size();
        for (size_t i = 0; i < umi.size(); ++i) bo.umi[i] = umi[i];
        bo.seq = seq[0];
        if (two) { bo.paired = 1; bo.seq2 = seq[1]; }
      }
    }
    if (ret && tagsequence.empty() && up == "SMARTSEQ3") {      // src/main.cpp:1447-1450
      tagsequence = "ATTGCGCAATG";
      cerr << "[bus] Using " << tagsequence << " as UMI tag sequence" << endl;
    }
    if (ret && paired_flag && !bo.paired) {      // src/main.cpp:1472-1475
      cerr << "Error: Paired reads are not compatible with the specified technology" << endl;
      ret = false;
    }
    // the reference only warns here ("Wrong number of files per batch for technology", src/main.cpp:1439-1441) and then
    // reads outside the line's files; this build refuses the batch file
    if (ret && tech_batch && tech_batch_nfiles != (size_t)bo.nfiles) {
      cerr << "Error: the lines of batch file " << batch_file << " have " << tech_batch_nfiles << " files, technology "
           << tech_upper << " reads " << bo.nfiles << endl;
      ret = false;
    }
    // --batch-barcodes puts 32 - blen letters of the sample's number in front of a barcode of blen letters; the reference
    // wraps 32 - blen around for blen > 32 (:1617-1626).  This build refuses a barcode whose fixed pieces exceed 32
    // letters before any work, and stops the run when a read set's variable-length barcode does.
    if (ret && tech_batch && batch_barcodes_flag) {
      int fixed = 0;
      for (int i = 0; i < bo.n_bc; ++i)
        if (bo.bc[i].stop != 0) fixed += bo.bc[i].stop - bo.bc[i].start;
      if (fixed > 32) {
        cerr << "Error: --batch-barcodes needs a barcode of at most 32 letters; technology " << tech_upper << " has " << fixed
             << endl;
        ret = false;
      }
    }
  }
  if (ret && !interleaved_flag && opt.files.size() % bo.nfiles != 0) {
    cerr << "Error: Number of files (" << opt.files.size() << ") does not match number of input files required by "
         << "technology " << tech_upper << " (" << bo.nfiles << ")" << endl;
    ret = false;
  }
  int strand = 0;
  if (fr) strand = 1;
  else if (rf) strand = 2;
  else if (unstranded) strand = 0;
  else if (ret && !batch_mode) {      // -x BULK leaves CheckOptionsBus before the technology defaults (:1214): unstranded
    strand = tech_strand;
    if (strand == 1) cerr << "[bus] Note: Strand option was not specified; setting it to --fr-stranded for specified technology" << endl;
    else if (strand == 2) cerr << "[bus] Note: Strand option was not specified; setting it to --rf-stranded for specified technology" << endl;
    else cerr << "[bus] Note: Strand option was not specified; setting it to --unstranded for specified technology" << endl;
  }
  if (!tagsequence.empty() && !batch_mode && bo.n_umi > 0) {      // src/main.cpp:1467-1475: the UMI starts after the tag
    if (bo.umi[0].fileno < 0 || bo.umi[0].start + (int)tagsequence.size() >= bo.umi[0].stop || tagsequence.size() > 31) {
      cerr << "Error: Tag sequence must be shorter than UMI sequence" << endl;
      ret = false;
    } else {
      bo.tag = tagsequence.c_str();
    }
  }
  // --union / --no-jump are not built here; with --aa the reference refuses them as well (src/main.cpp:969-976)
  if (union_flag) { cerr << (aa_flag ? "--union is not compatible with this mode" : "Error: --union is not supported by this build") << endl; ret = false; }
  if (no_jump_flag) { cerr << (aa_flag ? "--no-jump is not compatible with this mode" : "Error: --no-jump is not supported by this build") << endl; ret = false; }
  if (aa_flag) {
    // the reference turns --paired off with a note and matches the first sequence read alone (src/main.cpp:761-770);
    // this build says so instead of dropping a read
    if (paired_flag || bo.paired) {
      cerr << "Error: --aa supports single-end reads only: --paired and technologies with two sequence reads are not supported" << endl;
      ret = false;
    }
    if (!tagsequence.empty()) { cerr << "Error: --aa with a UMI tag sequence (--tag) is not supported" << endl; ret = false; }
  }
  if (opt.output.empty()) { cerr << "Error: need to specify output directory " << opt.output << endl; ret = false; }
  else if (stat(opt.output.c_str(), &stt) == 0) {
    if (!S_ISDIR(stt.st_mode)) { cerr << "Error: file " << opt.output << " exists and is not a directory" << endl; ret = false; }
  } else if (ret && mkdir(opt.output.c_str(), 0777) == -1) { cerr << "Error: could not create directory " << opt.output << endl; ret = false; }
  // --devices with two entries or more: one run per entry, one index replica each, driven as a kb_bus_group
  const int n_dev = opt.devices.size() > 1 ? (int)opt.devices.size() : 1;
  if (ret && n_dev > 1 &&
      (!kb_bus_group_create || !kb_bus_group_free || !kb_bus_group_submit || !kb_bus_group_complete || !kb_bus_group_begin_sample ||
       !kb_bus_group_finalize || !kb_bus_group_ec_table || !kb_bus_group_lengths || !kb_bus_group_frame_clashes)) {
    cerr << "Error: this libkallisto_b200 has no kb_bus_group_create (bus --devices)" << endl;
    return 1;
  }
  if (!ret) {
    usage_bus();
    return 1;
  }
  kb_index* ix = nullptr;
  std::vector<kb_index*> ixs;
  if (n_dev > 1) {
    restrict_visible_devices(opt.device, opt.devices);
    if (!load_replicas(opt.index, opt.devices, 0, opt.threads, ixs)) return 1;
    ix = ixs[0];
  } else {
    KB_TRY(kb_index_load(opt.index.c_str(), opt.device, 0, std::min(16, std::max(1, opt.threads)), &ix));
  }
  kb_index_info info;
  kb_index_get_info(ix, &info);
  cerr << "[index] k-mer length: " << info.k << endl;
  cerr << "[index] number of targets: " << pretty_num(info.n_targets) << endl;
  cerr << "[index] number of k-mers: " << pretty_num(info.n_kmers) << endl;
  cerr << "[quant] will process sample 1: ";
  for (size_t i = 0; i < opt.files.size(); ++i) cerr << (i ? "\n                               " : "") << opt.files[i];
  cerr << endl << "[quant] finding pseudoalignments for the reads ...";
  cerr.flush();

  const size_t max_reads = 1u << 20;
  const size_t max_bases = (size_t)max_reads * 160 + kb::FastxFile::kMaxRead;
  bo.strand_mode = strand;
  bo.num = num_flag;
  bo.max_batch_sets = (uint32_t)max_reads;
  bo.max_batch_bases = 2 * max_bases;
  kb_quant* q = nullptr;
  // --batch-barcodes changes nothing without --batch or with -x bulk (src/main.cpp:2409, src/ProcessReads.cpp:1603-1626)
  const bool batch_barcodes = tech_batch && batch_barcodes_flag;
  std::vector<kb_quant*> qs(n_dev, nullptr);
  for (int d = 0; d < n_dev; ++d) {
    KB_TRY(kb_bus_create(n_dev > 1 ? ixs[d] : ix, &bo, &qs[d]));
    if (aa_flag) {
      if (!kb_bus_set_aa || !kb_bus_frame_clashes) { cerr << "Error: this libkallisto_b200 has no kb_bus_set_aa" << endl; return 1; }
      KB_TRY(kb_bus_set_aa(qs[d], 1));      // refuses an index with a D-list
    }
    if (batch_barcodes && bo.n_bc > 0) {
      if (!kb_bus_set_batch_barcodes) { cerr << "Error: this libkallisto_b200 has no kb_bus_set_batch_barcodes" << endl; return 1; }
      KB_TRY(kb_bus_set_batch_barcodes(qs[d], 1));
    }
  }
  q = qs[0];
  kb_bus_group* grp = nullptr;
  if (n_dev > 1) KB_TRY(kb_bus_group_create(qs.data(), n_dev, &grp));
  auto spec_len = [](const kb_bus_substr* v, int n) {   // BUSOptions::getBCLength / getUMILength
    int r = 0;
    for (int i = 0; i < n; ++i) {
      if (v[i].start < 0 || v[i].stop == 0) return 0;
      r += v[i].stop - v[i].start;
    }
    return r;
  };
  uint32_t bclen = (uint32_t)spec_len(bo.bc, bo.n_bc), umilen = (uint32_t)spec_len(bo.umi, bo.n_umi);
  if (bo.tag && umilen > 0) umilen -= (uint32_t)tagsequence.size();      // getUMILength() of the advanced UMI location
  if (batch_mode) umilen = 1;      // writeBUSHeader(busf_out, BUSFORMAT_FAKE_BARCODE_LEN, 1), src/ProcessReads.h:241-242
  // a --batch run with a technology writes getBCLength() (0 without a barcode read or with a variable-length one), 16 for
  // batch barcodes without a barcode read, and keeps it (src/ProcessReads.h:240-253): with batch barcodes the records
  // carry 32 letters all the same
  const uint32_t hdr_bclen = tech_batch ? ((batch_barcodes && bo.n_bc == 0) ? 16u : bclen) : (bo.n_bc == 0 ? 16u : bclen);
  const std::string busfile = opt.output + "/output.bus";
  std::ofstream busf(busfile, std::ios::out | std::ios::binary);
  {   // writeBUSHeader, src/BUSTools.cpp:5-14
    const uint32_t version = 1;
    busf.write("BUS\0", 4);
    busf.write((const char*)&version, 4);
    busf.write((const char*)&hdr_bclen, 4);
    busf.write((const char*)&umilen, 4);
    const std::string text = "BUS file produced by kallisto";
    const uint32_t tl = (uint32_t)text.size();
    busf.write((const char*)&tl, 4);
    busf.write(text.c_str(), tl);
  }
  const int n_streams = bo.nfiles;
  std::vector<Stream> streams(n_streams);
  std::vector<std::thread> readers;
  if (interleaved_flag) {
    for (auto& st : streams) {
      st.ring.resize(3);
      st.state.assign(3, 0);
      for (auto& b : st.ring) { b.cap_bases = max_bases; b.cap_reads = max_reads; }
    }
    const size_t per_stream = std::max<size_t>(1, stream_batch_reads(0, max_reads / (size_t)n_streams));
    readers.emplace_back(interleaved_reader_thread, opt.files[0], &streams, per_stream, std::max(1, opt.threads));
  } else {
    start_streams(streams, readers, opt.files, max_bases, max_reads, opt.threads);
  }
  std::vector<kb_bus_record> recs(max_reads);
  const bool by_sample = batch_mode || tech_batch;      // one sample per file set
  const size_t n_samples = (by_sample && !interleaved_flag) ? std::max<size_t>(1, opt.files.size() / (size_t)bo.nfiles) : 1;
  std::vector<std::vector<uint32_t>> sample_flens(n_samples, std::vector<uint32_t>(1000, 0));
  size_t cur_sample = (size_t)-1;
  // --devices: the outstanding batches (ticket, member), oldest first; records are written in ticket order, so
  // output.bus is the one-device file
  std::vector<std::pair<uint64_t, int>> outstanding;
  std::vector<char> busy(n_dev, 0);
  auto complete_oldest = [&]() {
    uint32_t nrec = 0;
    const std::pair<uint64_t, int> t = outstanding.front();
    outstanding.erase(outstanding.begin());
    busy[t.second] = 0;
    KB_TRY(kb_bus_group_complete(grp, t.first, recs.data(), &nrec));
    busf.write((const char*)recs.data(), (std::streamsize)nrec * sizeof(kb_bus_record));
  };
  auto drain = [&]() {
    while (!outstanding.empty()) complete_oldest();
  };
  // Paired runs sample fragment lengths from the first 10000 qualifying pairs of each sample: member 0 takes the
  // sample's batches, one at a time, until its histogram holds them; after that (and in unpaired runs from the start)
  // batches are dealt round-robin, one per member in flight.
  bool fld_done = !bo.paired;
  size_t rr = 0;
  {
    LockStep ls(streams);
    const char* bp[4] = {nullptr, nullptr, nullptr, nullptr};
    const uint32_t* op[4] = {nullptr, nullptr, nullptr, nullptr};
    size_t n = 0;
    while (ls.next(n, bp, op)) {
      if (by_sample && ls.file_set() != cur_sample) {
        // the reads of the next file set are the next sample: it samples its own fragment lengths and numbers its reads
        // from 0; its id is the fake barcode of its records without a technology or, with --batch-barcodes, goes into
        // the barcode; a technology without a barcode read gives 16 x 'A' otherwise (src/ProcessReads.cpp:371-404,
        // 486-493,1583-1627)
        if (grp) drain();
        if (cur_sample != (size_t)-1) KB_TRY(kb_quant_get_flens(q, sample_flens[cur_sample].data()));
        cur_sample = ls.file_set();
        const uint64_t id = sample_barcode.empty() ? (uint64_t)cur_sample : sample_barcode[cur_sample];
        const uint64_t bc = (tech_batch && !batch_barcodes && bo.n_bc == 0) ? 0 : id;
        if (grp) {
          KB_TRY(kb_bus_group_begin_sample(grp, bc));
          fld_done = !bo.paired;
          rr = 0;
        } else {
          KB_TRY(kb_bus_begin_sample(q, bc));
        }
      }
      if (!grp) {
        uint32_t nrec = 0;
        KB_TRY(kb_bus_batch(q, bp, op, (uint32_t)n, recs.data(), &nrec));
        busf.write((const char*)recs.data(), (std::streamsize)nrec * sizeof(kb_bus_record));
        ls.release();
        continue;
      }
      const int m = fld_done ? (int)(rr++ % (size_t)n_dev) : 0;
      while (busy[m]) complete_oldest();
      uint64_t ticket = 0;
      KB_TRY(kb_bus_group_submit(grp, m, bp, op, (uint32_t)n, &ticket));
      outstanding.push_back({ticket, m});
      busy[m] = 1;
      ls.release();      // the batch is on the device: the parsers may refill its ring slots
      if (!fld_done) {
        drain();
        uint32_t fl[1000];
        KB_TRY(kb_quant_get_flens(q, fl));
        uint64_t cnt = 0;
        for (int i = 0; i < 1000; ++i) cnt += fl[i];
        fld_done = cnt >= 10000;
      }
    }
    if (grp) drain();
  }
  for (auto& t : readers) t.join();
  busf.close();
  cerr << " done" << endl;
  if (bo.paired) KB_TRY(kb_quant_get_flens(q, sample_flens[by_sample ? (cur_sample == (size_t)-1 ? 0 : cur_sample) : 0].data()));
  if (by_sample) {
    // src/main.cpp:2406-2449: sample names (every line's id), their fake barcodes (without a technology, or with
    // --batch-barcodes), the stripped index, one fragment-length line per sample
    std::ofstream cf(opt.output + "/matrix.cells");
    std::ofstream bf;
    if (batch_mode || batch_barcodes) bf.open(opt.output + "/matrix.sample.barcodes");
    for (size_t j = 0; j < n_samples; ++j) {
      if (sample_names.empty()) cf << "batch" << j << "\n";
      else cf << sample_names[j] << "\n";
      const uint64_t v = sample_barcode.empty() ? (uint64_t)j : sample_barcode[j];
      std::string b(16, 'A');      // binaryToString(v, 16), src/BUSData.cpp:38-51
      for (int p = 0; p < 16; ++p) b[15 - p] = "ACGT"[(v >> (2 * p)) & 3];
      if (bf.is_open()) bf << b << "\n";
    }
  }
  if (batch_mode || bo.paired || (bo.n_umi == 1 && bo.umi[0].fileno == -1))
    write_index_saved(opt.index, opt.output + "/index.saved", info.k);      // :2414-2417, 2517, 2560-2563
  // with a technology, a --batch run writes flens.txt only when --paired was given (!opt.single_end, :2418-2420)
  if (tech_batch ? (bool)paired_flag : (bool)bo.paired) {      // :2418-2449 (one line per sample) / :2511-2526
    std::ofstream ff(opt.output + "/flens.txt");
    for (size_t j = 0; j < n_samples; ++j) {
      for (size_t i = 0; i < 1000; ++i) ff << (i ? " " : "") << sample_flens[j][i];
      ff << "\n";
    }
  }
  // barcode / UMI lengths of the header when the technology does not fix them (src/main.cpp:2470-2508); never in a
  // batch run
  if (!by_sample) {
    uint32_t bh[33], uh[33];
    if (grp) KB_TRY(kb_bus_group_lengths(grp, bh, uh));
    else KB_TRY(kb_bus_lengths(q, bh, uh));
    uint32_t bl = 0, ul = 0;
    for (uint32_t i = 0; i <= 32; ++i) {
      if (bh[i] > bh[bl]) bl = i;
      if (uh[i] > uh[ul]) ul = i;
    }
    bool write = false;
    uint32_t wb = hdr_bclen, wu = umilen;
    if (bclen == 0 && bo.n_bc > 0) { if (bl > 0) { write = true; } wb = bl; }
    if (bclen == 0 && bo.n_bc == 0) { if (bl > 0) write = true; wb = bl; }
    if (umilen == 0) { if (ul > 0) write = true; wu = ul; }
    if (write) {
      std::FILE* fp = std::fopen(busfile.c_str(), "r+b");
      if (fp) {
        std::fseek(fp, 8, SEEK_SET);
        std::fwrite(&wb, 4, 1, fp);
        std::fwrite(&wu, 4, 1, fp);
        std::fclose(fp);
      }
    }
  }
  kb_run_stats st{};
  if (grp) KB_TRY(kb_bus_group_finalize(grp, &st));
  else KB_TRY(kb_quant_finalize(q, &st));
  cerr << "[quant] processed " << pretty_num(st.n_processed) << " reads, " << pretty_num(st.n_pseudoaligned)
       << " reads pseudoaligned" << endl;
  if (st.n_pseudoaligned == 0) cerr << "[~warn] no reads pseudoaligned." << endl;
  {   // writeECList, src/PlaintextWriter.cpp:235-266
    std::vector<uint64_t> eo(st.n_ecs + 1);
    std::vector<uint32_t> et(std::max<uint64_t>(1, st.n_ec_entries)), ec(std::max<uint64_t>(1, st.n_ecs));
    if (grp) KB_TRY(kb_bus_group_ec_table(grp, eo.data(), et.data(), ec.data()));
    else KB_TRY(kb_quant_ec_table(q, eo.data(), et.data(), ec.data(), nullptr));
    std::ofstream ecof(opt.output + "/matrix.ec");
    for (uint64_t i = 0; i < st.n_ecs; ++i) {
      ecof << i << "\t";
      for (uint64_t j = eo[i]; j < eo[i + 1]; ++j) ecof << (j > eo[i] ? "," : "") << et[j];
      ecof << "\n";
    }
  }
  {
    std::ofstream tf(opt.output + "/transcripts.txt");
    for (uint32_t i = 0; i < info.n_targets; ++i) tf << kb_index_target_name(ix, i) << "\n";
  }
  std::string frame_clashes;
  if (aa_flag) {
    uint64_t nc = 0;
    if (grp) KB_TRY(kb_bus_group_frame_clashes(grp, &nc));
    else KB_TRY(kb_bus_frame_clashes(q, &nc));
    frame_clashes = std::to_string(nc);
  }
  write_run_info(opt.output + "/run_info.json", info.n_targets, 0, st.n_processed, st.n_pseudoaligned, st.n_unique, 13, info.k,
                 start_time, call, frame_clashes);
  cerr << endl;
  if (!getenv("KB_CLI_CLEANUP")) finish(st.n_pseudoaligned == 0 ? 1 : 0);
  free_streams(streams);
  if (grp) kb_bus_group_free(grp);
  for (kb_quant* m : qs) kb_quant_free(m);
  if (n_dev > 1)
    for (kb_index* x : ixs) kb_index_free(x);
  else
    kb_index_free(ix);
  return st.n_pseudoaligned == 0 ? 1 : 0;
}

// ------------------------------------------------------------------------------------------------
// kallisto quant-tcc (src/main.cpp:394-513 ParseOptionsTCCQuant, 1807-1967 CheckOptionsTCCQuant, 2802-3220 body):
// abundances from pre-computed transcript-compatibility counts.  Every row of the TCC matrix is one EM over the
// equivalence classes of the EC file; all rows are solved on the device by the batched EM kernel (kb_tcc_run), and
// their bootstraps (-b) likewise, every (row, bootstrap) pair its own problem (kb_tcc_bootstrap_run).
// Supported: -i, -e (required here), -o, -l/-s, -f, -t, -b, -d/--seed, -g/--genemap, -G/--gtf, --matrix-to-files,
// --matrix-to-directories, --plaintext, -p/--priors.  Gene-level output is summed on the device (kb_tcc_run_genes,
// kb_tcc_bootstrap_run_genes).  Priors start every sample's EM (kb_tcc_run_priors); bootstraps start uniform, as in the
// reference.  --long, -T and a per-sample abundance.h5 are refused loudly.
// Deliberate differences from the reference:
//   - -b on a matrix file without --matrix-to-files / --matrix-to-directories, or without --plaintext, is refused: the
//     reference (built without HDF5) runs and silently writes no bootstraps there.
//   - -b on a non-matrix file whose counts are all zero is an error; the reference aborts (Multinomial::sample(0)).
//   - --priors (here and in quant): a file that cannot be opened is an error ("Error: could not open priors file
//     <path>", exit 1); the reference silently starts uniform.  A line std::stod rejects (an empty line, `abc`, `1e999`)
//     is an error naming the line, exit 1; the reference aborts with an uncaught exception.
// ------------------------------------------------------------------------------------------------
void usage_tcc() {
  std::cout << "kallisto_b200 " << KALLISTO_VERSION << " (H100 build)" << endl
            << "Quantifies abundance from pre-computed transcript-compatibility counts" << endl << endl
            << "Usage: kallisto_b200 quant-tcc [arguments] transcript-compatibility-counts-file" << endl << endl
            << "Required arguments:" << endl
            << "-o, --output-dir=STRING       Directory to write output to" << endl
            << "-i, --index=STRING            Filename for the kallisto index to be used" << endl
            << "-e, --ec-file=FILE            File containing equivalence classes (matrix.ec of kallisto bus)" << endl << endl
            << "Optional arguments:" << endl
            << "-f, --fragment-file=FILE      File containing fragment length distribution" << endl
            << "                              (default: effective length normalization is not performed)" << endl
            << "-l, --fragment-length=DOUBLE  Estimated average fragment length" << endl
            << "-s, --sd=DOUBLE               Estimated standard deviation of fragment length" << endl
            << "-p, --priors                  Priors for the EM algorithm, either as raw counts or as" << endl
            << "                              probabilities. Pseudocounts are added to raw reads to" << endl
            << "                              prevent zero valued priors. Supplied in the same order" << endl
            << "                              as the transcripts in the transcriptome" << endl
            << "-t, --threads=INT             Number of host threads (default: 1)" << endl
            << "-b, --bootstrap-samples=INT   Number of bootstrap samples (default: 0); with a matrix file only" << endl
            << "                              together with --matrix-to-files or --matrix-to-directories and --plaintext" << endl
            << "    --seed=INT                Seed for the bootstrap sampling (default: 42)" << endl
            << "-g, --genemap                 File for mapping transcripts to genes" << endl
            << "                              (required for obtaining gene-level abundances)" << endl
            << "-G, --gtf=FILE                GTF file for transcriptome information" << endl
            << "                              (can be used instead of --genemap for obtaining gene-level abundances)" << endl
            << "    --matrix-to-files         Reorganize matrix output into abundance tsv files" << endl
            << "    --matrix-to-directories   Reorganize matrix output into abundance tsv files across" << endl
            << "                              multiple directories" << endl
            << "    --plaintext               Output plaintext only (quant-tcc writes no HDF5 in this build)" << endl
            << "    --device=INT              CUDA device ordinal (default: 0)" << endl;
}

void write_sparse_matrix(const std::string& path, const std::vector<std::vector<std::pair<int, double>>>& data, size_t cols) {
  // writeSparseBatchMatrix, src/PlaintextWriter.h:72-105
  uint64_t n = 0;
  for (auto& v : data)
    for (auto& x : v)
      if (x.second != 0.0) ++n;
  std::string out = "%%MatrixMarket matrix coordinate real general\n";
  out += std::to_string(data.size()) + "\t" + std::to_string(cols) + "\t" + std::to_string(n) + "\n";
  for (size_t j = 0; j < data.size(); ++j)
    for (auto& x : data[j])
      if (x.second != 0.0) {
        out += std::to_string(j + 1) + "\t" + std::to_string(x.first + 1) + "\t";
        append_double(out, x.second);
        out += "\n";
      }
  std::ofstream of(path, std::ios::out | std::ios::binary);
  of.write(out.data(), (std::streamsize)out.size());
}

// The gene model of quant-tcc's gene-level output (Transcriptome, src/GeneModel.cpp), reduced to what that output reads:
// the genes in id order with their common names, and the gene of every target (-1: none, left out of every sum).
struct GeneModel {
  std::vector<std::string> name, common;
  std::vector<int32_t> gene_of;
};

std::unordered_map<std::string, int32_t> target_ids(const std::vector<std::string>& targets) {
  std::unordered_map<std::string, int32_t> m;
  for (size_t i = 0; i < targets.size(); ++i) m.insert({targets[i], (int32_t)i});
  return m;
}

// Transcriptome::parseGeneMap (src/GeneModel.cpp:580-632): every non-empty line is `transcript gene [common name]`
// (further columns ignored); genes are numbered in order of first appearance, and a later line for a transcript
// reassigns it.  Prints the reference's message and returns false on an error.
bool parse_genemap(const std::string& fn, const std::vector<std::string>& targets, GeneModel& gm) {
  const auto tr = target_ids(targets);
  std::unordered_map<std::string, int32_t> gid;
  gm.gene_of.assign(targets.size(), -1);
  std::ifstream in(fn);
  if (!in.is_open()) { cerr << "Error: could not open file " << fn << endl; return false; }
  std::string line;
  while (getline(in, line)) {
    if (line.empty()) continue;
    std::stringstream ss(line);
    std::string txp, gene, common;
    ss >> txp >> gene >> common;
    if (gene.empty()) { cerr << "Error: No gene associated with transcript " << txp << " in " << fn << endl; return false; }
    const auto it = tr.find(txp);
    if (it == tr.end()) { cerr << "Error: Invalid transcript: " << txp << " in " << fn << endl; return false; }
    auto g = gid.find(gene);
    if (g == gid.end()) {
      g = gid.insert({gene, (int32_t)gm.name.size()}).first;
      gm.name.push_back(gene);
      gm.common.push_back(common);
    }
    gm.gene_of[it->second] = g->second;
  }
  return true;
}

// Transcriptome::parseGTF / addGTFLine (src/GeneModel.cpp:268-578) with every chromosome accepted, as quant-tcc calls it;
// plain or gzip (zlib's gzread, like the reference).  Only `gene` and `transcript` lines carry what gene-level output
// reads.  Their quirks are kept:
//   - a `gene` line appends ".<gene_version>" to a gene_id without a '.'; a duplicate gene adds a second entry to the
//     gene list, but its name keeps the id of the first;
//   - a `transcript` line looks its transcript up with ".<transcript_version>" (when the id has no '.') and then bare,
//     and its gene with ".<gene_version>" appended whether or not the id has a '.' (src/GeneModel.cpp:450 tests the
//     empty gene model of the line), then bare; a gene that has had no `gene` line yet gives -1;
//   - the first `transcript` line of a target decides its gene;
//   - attributes are read until a `gene` line's third counted key is gene_id, or a `transcript` line has counted four of
//     gene_id, gene_version, transcript_id, transcript_version.
bool parse_gtf(const std::string& fn, const std::vector<std::string>& targets, GeneModel& gm) {
  const auto tr = target_ids(targets);
  std::unordered_map<std::string, int32_t> gid;
  std::vector<char> seen(targets.size(), 0);
  gm.gene_of.assign(targets.size(), -1);
  std::string text;
  {
    gzFile f = gzopen(fn.c_str(), "r");
    if (!f) { cerr << "Error: could not open file " << fn << endl; return false; }
    char buf[1 << 16];
    int n;
    while ((n = gzread(f, buf, sizeof(buf))) > 0) text.append(buf, (size_t)n);
    const bool bad = n < 0;
    gzclose(f);
    if (bad) { cerr << "Error: could not read file " << fn << endl; return false; }
  }
  size_t missing = 0;
  const size_t npos = std::string::npos;
  for (size_t a = 0; a < text.size();) {
    size_t e = text.find('\n', a);
    if (e == npos) e = text.size();
    const std::string line = text.substr(a, e - a);
    a = e + 1;
    if (line.empty() || line[0] == '#') continue;
    const size_t t1 = line.find('\t'), t2 = t1 == npos ? npos : line.find('\t', t1 + 1);
    if (t2 == npos) continue;
    size_t t = line.find('\t', t2 + 1);
    const std::string type = line.substr(t2 + 1, t == npos ? npos : t - t2 - 1);
    const bool is_gene = type == "gene";
    if (!is_gene && type != "transcript") continue;
    for (int i = 0; i < 5 && t != npos; ++i) t = line.find('\t', t + 1);    // start, stop, score, strand, phase
    if (t == npos) { cerr << "Error: malformed GTF line in " << fn << ": " << line << endl; return false; }
    std::string gene, gversion, txp, tversion, common;
    int keycount = 0;
    for (size_t p = t + 1; p != npos;) {
      const size_t q = line.find('"', p);
      if (q == npos) break;
      const size_t s = line.find('"', q + 1);
      if (s == npos) break;
      const std::string key = line.substr(p, q - p - 1), value = line.substr(q + 1, s - q - 1);
      if (key == "gene_id") { ++keycount; gene = value; }
      else if (key == "gene_version") { ++keycount; gversion = value; }
      if (is_gene) {
        if (key == "gene_name") { ++keycount; common = value; }
        else if (key == "gene_id" && keycount == 3) break;
      } else {
        if (key == "transcript_id") { ++keycount; txp = value; }
        else if (key == "transcript_version") { ++keycount; tversion = value; }
        if (keycount == 4) break;
      }
      if ((p = line.find(' ', s)) != npos && ++p >= line.size()) break;
    }
    if (is_gene) {
      if (!gversion.empty() && gene.find('.') == npos) gene += "." + gversion;
      gid.insert({gene, (int32_t)gm.name.size()});
      gm.name.push_back(gene);
      gm.common.push_back(common);
      continue;
    }
    auto it = tr.end();
    if (!tversion.empty() && txp.find('.') == npos) it = tr.find(txp + "." + tversion);
    if (it == tr.end()) it = tr.find(txp);
    if (it == tr.end()) { ++missing; continue; }
    auto g = gid.end();
    if (!gversion.empty()) g = gid.find(gene + "." + gversion);
    if (g == gid.end()) g = gid.find(gene);
    if (!seen[it->second]) {
      seen[it->second] = 1;
      gm.gene_of[it->second] = g == gid.end() ? -1 : g->second;
    }
  }
  if (missing) cerr << "Warning: " << missing << " transcripts were defined in GTF file, but not in the index" << endl;
  return true;
}

// plaintext_writer_gene (src/PlaintextWriter.cpp:67-112): every gene, zero or not
void write_gene_abundance(const std::string& path, const GeneModel& gm, const double* gc, const double* gt) {
  std::ofstream of(path, std::ios::out | std::ios::binary);
  if (!of.is_open()) {
    cerr << "Error: Couldn't open file: " << path << endl;
    exit(1);
  }
  std::string out = "gene_id\tgene_name\test_counts\ttpm\n";
  for (size_t g = 0; g < gm.name.size(); ++g) {
    out += gm.name[g];
    out += '\t';
    out += gm.common[g];
    out += '\t';
    append_double(out, gc[g]);
    out += '\t';
    append_double(out, gt[g]);
    out += '\n';
  }
  of.write(out.data(), (std::streamsize)out.size());
}

// The bootstrap files of quant-tcc, written chunk by chunk as the device hands the (row, bootstrap) problems over
struct TccBsCtx {
  const std::string* output;
  bool is_matrix, dirs, per_sample;
  int B, threads;
  uint32_t T;
  const std::vector<std::string>* names;
  const std::vector<uint32_t>* lens;
  const std::vector<double>* eff;
  const std::vector<double>* est;
  const std::vector<char>* empty_row;
  const GeneModel* genes;                 // gene files next to every matrix row's bootstrap file, or nullptr
  const std::vector<double>* gene_counts; // the rows' own gene sums (an empty row's bootstraps are copies of them)
  const std::vector<double>* gene_tpm;
};

int write_tcc_bs_chunk(void* user, uint64_t first, uint32_t count, const double* bs_est, const int32_t*, const uint32_t*,
                       const double* bs_gc, const double* bs_gt) {
  const TccBsCtx& c = *static_cast<const TccBsCtx*>(user);
  const size_t G = c.genes ? c.genes->name.size() : 0;
  auto write_one = [&](uint32_t i) {
    const uint64_t g = first + i, r = g / c.B, b = g % c.B;
    std::string path, gpath;
    if (!c.is_matrix) path = *c.output + "/bs_abundance_" + std::to_string(b) + ".tsv";
    else if (c.dirs) {
      path = *c.output + "/abundance_" + std::to_string(r + 1) + "/bs_abundance_" + std::to_string(b) + ".tsv";
      gpath = *c.output + "/abundance_" + std::to_string(r + 1) + "/bs_abundance.gene_" + std::to_string(b) + ".tsv";
    } else {
      path = *c.output + "/bs_abundance_" + std::to_string(r + 1) + "_" + std::to_string(b) + ".tsv";
      gpath = *c.output + "/bs_abundance.gene_" + std::to_string(r + 1) + "_" + std::to_string(b) + ".tsv";
    }
    const bool empty = (*c.empty_row)[r];
    const double* a = empty ? c.est->data() + r * c.T : bs_est + (size_t)i * c.T;
    write_abundance(path, *c.names, *c.lens, c.eff->data() + (c.per_sample ? r : 0) * (size_t)c.T, a);
    if (c.genes && c.is_matrix)
      write_gene_abundance(gpath, *c.genes, empty ? c.gene_counts->data() + r * G : bs_gc + (size_t)i * G,
                           empty ? c.gene_tpm->data() + r * G : bs_gt + (size_t)i * G);
  };
  const uint32_t nt = (uint32_t)std::min<int64_t>(c.threads, count);
  std::vector<std::thread> pool;
  for (uint32_t t = 1; t < nt; ++t)
    pool.emplace_back([&, t] { for (uint32_t i = t; i < count; i += nt) write_one(i); });
  for (uint32_t i = 0; i < count; i += nt) write_one(i);
  for (auto& th : pool) th.join();
  return 0;
}

int cmd_quant_tcc(int argc, char** argv) {
  std::string index, ecfile, output, fldfile, tccfile, genemap, gtf, priors, txnames;
  double fld = 0.0, sd = 0.0;
  int threads = 1, device = 0, bootstrap = 0;
  size_t seed = 42;
  int matrix_to_files = 0, matrix_to_dirs = 0, plaintext = 0, long_flag = 0;
  const char* opt_string = "o:i:T:e:f:P:l:s:t:g:G:b:d:p:D:";
  static struct option long_options[] = {{"plaintext", no_argument, &plaintext, 1},
                                         {"matrix-to-files", no_argument, &matrix_to_files, 1},
                                         {"matrix-to-directories", no_argument, &matrix_to_dirs, 1},
                                         {"index", required_argument, 0, 'i'},
                                         {"txnames", required_argument, 0, 'T'},
                                         {"threads", required_argument, 0, 't'},
                                         {"fragment-file", required_argument, 0, 'f'},
                                         {"long", no_argument, &long_flag, 1},
                                         {"platform", required_argument, 0, 'P'},
                                         {"fragment-length", required_argument, 0, 'l'},
                                         {"sd", required_argument, 0, 's'},
                                         {"output-dir", required_argument, 0, 'o'},
                                         {"ec-file", required_argument, 0, 'e'},
                                         {"genemap", required_argument, 0, 'g'},
                                         {"gtf", required_argument, 0, 'G'},
                                         {"bootstrap-samples", required_argument, 0, 'b'},
                                         {"seed", required_argument, 0, 'd'},
                                         {"priors", required_argument, 0, 'p'},
                                         {"device", required_argument, 0, 'D'},
                                         {0, 0, 0, 0}};
  int c, oi = 0;
  while ((c = getopt_long(argc, argv, opt_string, long_options, &oi)) != -1) {
    switch (c) {
      case 't': std::stringstream(optarg) >> threads; break;
      case 'f': fldfile = optarg; break;
      case 'l': std::stringstream(optarg) >> fld; break;
      case 's': std::stringstream(optarg) >> sd; break;
      case 'o': output = optarg; break;
      case 'i': index = optarg; break;
      case 'e': ecfile = optarg; break;
      case 'g': genemap = optarg; break;
      case 'G': gtf = optarg; break;
      case 'b': std::stringstream(optarg) >> bootstrap; break;
      case 'd': std::stringstream(optarg) >> seed; break;
      case 'T': txnames = optarg; break;
      case 'p': priors = optarg; break;
      case 'D': std::stringstream(optarg) >> device; break;
      default: break;
    }
  }
  if (optind < argc) tccfile = argv[optind];
  if (matrix_to_dirs) matrix_to_files = 1;     // --matrix-to-directories implies --matrix-to-files (src/main.cpp:499-502)
  // ---- CheckOptionsTCCQuant
  bool ret = true;
  struct stat stt;
  cerr << endl;
  if (index.empty()) {
    cerr << ERROR_STR << " a kallisto index file needs to be supplied (a transcripts file alone, -T, is not supported by this build)" << endl;
    ret = false;
  } else if (stat(index.c_str(), &stt) != 0) {
    cerr << ERROR_STR << " kallisto index file not found " << index << endl;
    ret = false;
  }
  if (tccfile.empty()) { cerr << ERROR_STR << " transcript-compatibility counts file missing" << endl; ret = false; }
  else if (stat(tccfile.c_str(), &stt) != 0) { cerr << ERROR_STR << " transcript-compatibility counts file not found " << tccfile << endl; ret = false; }
  if (ecfile.empty()) { cerr << ERROR_STR << " equivalence class file must be supplied (-e)" << endl; ret = false; }
  else if (stat(ecfile.c_str(), &stt) != 0) { cerr << ERROR_STR << " equivalence class file not found " << ecfile << endl; ret = false; }
  if (!fldfile.empty() && stat(fldfile.c_str(), &stt) != 0) { cerr << ERROR_STR << " fragment length distribution file not found " << fldfile << endl; ret = false; }
  if (!genemap.empty() && !gtf.empty()) { cerr << ERROR_STR << " Cannot supply both --genemap and --gtf" << endl; ret = false; }
  if (!gtf.empty() && stat(gtf.c_str(), &stt) != 0) { cerr << ERROR_STR << " GTF file not found " << gtf << endl; ret = false; }
  if (!genemap.empty() && stat(genemap.c_str(), &stt) != 0) { cerr << ERROR_STR << " file for mapping transcripts to genes not found " << genemap << endl; ret = false; }
  if (long_flag || !txnames.empty()) { cerr << ERROR_STR << " --long and --txnames are not supported by this build" << endl; ret = false; }
  if (bootstrap > 0 && (!matrix_to_files || !plaintext) && !tccfile.empty()) {
    std::ifstream in(tccfile);
    std::string first;
    if (getline(in, first) && first.rfind("%%MatrixMarket", 0) == 0) {
      cerr << ERROR_STR << " bootstraps of a TCC matrix are not supported without --matrix-to-files (or --matrix-to-directories)"
           << " and --plaintext" << endl;
      ret = false;
    }
  }
  if ((fld != 0.0 || sd != 0.0) && !fldfile.empty()) { cerr << ERROR_STR << " cannot supply mean or sd while also supplying a fragment length distribution file" << endl; ret = false; }
  if ((fld != 0.0 && sd == 0.0) || (sd != 0.0 && fld == 0.0)) { cerr << ERROR_STR << " cannot supply mean/sd without supplying both -l and -s" << endl; ret = false; }
  if (ret && fld > 0.0 && sd > 0.0) cerr << "[tcc] fragment length distribution is truncated gaussian with mean = " << fld << ", sd = " << sd << endl;
  if (fld < 0.0) { cerr << ERROR_STR << " invalid value for mean fragment length " << fld << endl; ret = false; }
  if (sd < 0.0) { cerr << ERROR_STR << " invalid value for fragment length standard deviation " << sd << endl; ret = false; }
  if (output.empty()) { cerr << ERROR_STR << " need to specify output directory " << output << endl; ret = false; }
  else if (stat(output.c_str(), &stt) == 0) {
    if (!S_ISDIR(stt.st_mode)) { cerr << ERROR_STR << " file " << output << " exists and is not a directory" << endl; ret = false; }
  } else if (mkdir(output.c_str(), 0777) == -1) { cerr << ERROR_STR << " could not create directory " << output << endl; ret = false; }
  if (threads <= 0) { cerr << ERROR_STR << " invalid number of threads " << threads << endl; ret = false; }
  if (bootstrap < 0) { cerr << "Error: number of bootstrap samples must be a non-negative integer." << endl; ret = false; }
  if (!ret) { cerr << endl; usage_tcc(); return 1; }
  // the priors file is read once, before any device work (src/main.cpp:2984-2987)
  std::vector<double> prior_v;
  if (!priors.empty() && !read_priors(priors, prior_v)) return 1;

  kb_index* ix = nullptr;
  KB_TRY(kb_index_load(index.c_str(), device, 0, std::min(16, std::max(1, threads)), &ix));
  kb_index_info info;
  kb_index_get_info(ix, &info);
  const uint32_t T = info.n_targets;
  // ---- EC file (KmerIndex::loadECsFromFile, src/KmerIndex.cpp:1561-1600)
  std::vector<uint64_t> ec_off{0};
  std::vector<uint32_t> ec_tids;
  {
    std::ifstream in(ecfile);
    if (!in.is_open()) { cerr << "Error: could not open file " << ecfile << endl; return 1; }
    std::string line;
    int32_t i = 0;
    std::vector<uint32_t> tmp;
    while (getline(in, line)) {
      std::stringstream ss(line);
      int ec;
      std::string transcripts;
      ss >> ec >> transcripts;
      if (i != ec) {
        cerr << "Error: equivalence class file has a misplaced equivalence class. Found " << ec << ", expected " << i << endl;
        return 1;
      }
      tmp.clear();
      std::stringstream ss2(transcripts);
      while (ss2.good()) {
        std::string v;
        getline(ss2, v, ',');
        const int x = std::atoi(v.c_str());
        if (x < 0 || x >= (int)T) {
          cerr << "Error: equivalence class file has invalid value: " << v << " in " << transcripts << endl;
          return 1;
        }
        tmp.push_back((uint32_t)x);
      }
      std::sort(tmp.begin(), tmp.end());                       // a Roaring set: sorted, no duplicates
      tmp.erase(std::unique(tmp.begin(), tmp.end()), tmp.end());
      ec_tids.insert(ec_tids.end(), tmp.begin(), tmp.end());
      ec_off.push_back(ec_tids.size());
      ++i;
    }
    cerr << "[index] number of equivalence classes loaded from file: " << pretty_num(ec_off.size() - 1) << endl;
  }
  const uint32_t n_ecs = (uint32_t)(ec_off.size() - 1);
  // ---- TCC file (src/main.cpp:2817-2903)
  std::vector<uint64_t> row_off;
  std::vector<uint32_t> ids, vals;
  bool is_matrix = false;
  size_t nrow = 0, ncol = 0, nlines = 0;
  {
    std::ifstream in(tccfile);
    if (!in.is_open()) { cerr << "Error: could not open file " << tccfile << endl; return 1; }
    std::vector<std::vector<std::pair<uint32_t, uint32_t>>> rows;
    std::string line;
    bool first = true;
    size_t i = 0;
    int prev_row = 0, prev_col = 0;
    while (getline(in, line)) {
      if (first) {
        first = false;
        if (line.rfind("%%MatrixMarket", 0) == 0) {
          cerr << "[tcc] Parsing transcript-compatibility counts (TCC) file as a matrix file" << endl;
          is_matrix = true;
          while (getline(in, line) && line.rfind("%", 0) == 0) {}
          std::stringstream ss(line);
          ss >> nrow >> ncol >> nlines;
          cerr << "[tcc] Matrix dimensions: " << pretty_num(nrow) << " x " << pretty_num(ncol) << endl;
          rows.assign(nrow, {});
          continue;
        }
        cerr << "[tcc] Transcript-compatibility counts (TCC) file is not in matrix format; it will not be parsed as a matrix file" << endl;
        rows.assign(1, {});
      }
      std::stringstream ss(line);
      int row, col, val;
      if (is_matrix) {
        if (i >= nlines) {
          cerr << "[tcc] Warning: TCC matrix file contains additional lines which will not be read; only " << pretty_num(nlines)
               << " entries, as specified on the first line, will be read." << endl;
          break;
        }
        ss >> row >> col >> val;
        if ((size_t)row > nrow || (size_t)col > ncol) {
          cerr << "Error: TCC matrix file is malformed; row numbers or column numbers exceed the dimensions of the matrix." << endl;
          return 1;
        }
      } else {
        ss >> col >> val;
        col += 1;
        row = 1;
        nrow = 1;
        if (ncol < (size_t)col) ncol = col;
      }
      if (row <= 0 || col <= 0) { cerr << "Error: Invalid indices in TCC file." << endl; return 1; }
      if (row < prev_row || (row == prev_row && col <= prev_col)) { cerr << "Error: TCC file is not sorted." << endl; return 1; }
      prev_row = row;
      prev_col = col;
      if ((uint32_t)(col - 1) >= n_ecs) { cerr << "Error: TCC file refers to equivalence class " << col - 1 << ", the EC file holds " << n_ecs << endl; return 1; }
      rows[row - 1].push_back({(uint32_t)(col - 1), (uint32_t)val});
      ++i;
    }
    if (is_matrix && i < nlines) {
      cerr << "Error: Found only " << pretty_num(i) << " entries in TCC matrix file, expected " << pretty_num(nlines) << endl;
      return 1;
    }
    row_off.push_back(0);
    for (auto& r : rows) {
      for (auto& x : r) { ids.push_back(x.first); vals.push_back(x.second); }
      row_off.push_back(ids.size());
    }
    nrow = rows.size();
  }
  if (bootstrap > 0 && !is_matrix && std::all_of(vals.begin(), vals.end(), [](uint32_t v) { return v == 0; })) {
    cerr << "Error: cannot bootstrap a TCC file without any counts" << endl;
    return 1;
  }
  // ---- effective lengths (src/main.cpp:2998-3028)
  const bool calc_eff = !fldfile.empty() || fld != 0.0;
  std::vector<std::vector<uint32_t>> flds;
  if (!fldfile.empty()) {
    std::ifstream in(fldfile);
    if (!in.is_open()) { cerr << "Error: could not open file " << fldfile << endl; return 1; }
    std::string line;
    while (getline(in, line)) {
      if (line.empty() || line.rfind("#", 0) == 0) continue;
      std::vector<uint32_t> v;
      std::stringstream ss(line);
      while (ss.good()) {
        std::string tv;
        getline(ss, tv, ' ');
        const int x = std::atoi(tv.c_str());
        if (x < 0) { cerr << "Error: Fragment length distribution file contains invalid value: " << x << endl; return 1; }
        v.push_back((uint32_t)x);
      }
      if (v.size() != 1000) { cerr << "Error: Fragment length distribution file contains a line with " << v.size() << " values; expected: 1000" << endl; return 1; }
      flds.push_back(v);
    }
    if (flds.size() != 1 && flds.size() != nrow) {
      cerr << "Error: Fragment length distribution file contains " << flds.size() << " valid lines; expected: " << nrow << endl;
      return 1;
    }
  }
  const bool per_sample = flds.size() > 1;
  std::vector<double> eff((per_sample ? nrow : 1) * (size_t)T);
  std::vector<std::pair<double, double>> fld_mat(nrow, {0.0, 0.0});
  for (size_t r = 0; r < (per_sample ? nrow : 1); ++r) {
    double m = 0, s = 0;
    const uint32_t* fl = flds.empty() ? nullptr : flds[per_sample ? r : 0].data();
    KB_TRY(kb_eff_lens(ix, fl, fld, sd, eff.data() + r * T, &m, &s));
    if (per_sample) fld_mat[r] = {m, s};
    else for (auto& x : fld_mat) x = {m, s};
  }
  std::vector<std::string> names(T);
  std::vector<uint32_t> lens(T);
  for (uint32_t i = 0; i < T; ++i) names[i] = kb_index_target_name(ix, i);
  kb_index_target_lens(ix, lens.data());
  // ---- gene model (src/main.cpp:2975-2980)
  const bool gene_level = !genemap.empty() || !gtf.empty();
  GeneModel gm;
  if (!genemap.empty() && !parse_genemap(genemap, names, gm)) return 1;
  if (!gtf.empty() && !parse_gtf(gtf, names, gm)) return 1;
  const uint32_t G = (uint32_t)gm.name.size();
  cerr << "[quant] Running EM algorithm..." << endl;
  std::vector<double> est(nrow * (size_t)T), gene_counts(gene_level ? nrow * (size_t)G : 0), gene_tpm(gene_counts.size());
  std::vector<int32_t> rounds(nrow + 1);
  // every sample's EM starts from the priors (src/main.cpp:3019): a count mismatch is reported once per sample
  bool use_priors = false;
  if (!priors.empty()) {
    cerr << "[   em] reading priors from file " << priors << endl;
    for (size_t r = 0; r < nrow; ++r) use_priors = priors_apply(prior_v, T);
  }
  if (use_priors) {
    if (!kb_tcc_run_priors) { cerr << "Error: this libkallisto_b200 has no kb_tcc_run_priors" << endl; return 1; }
    KB_TRY(kb_tcc_run_priors(ix, n_ecs, ec_off.data(), ec_tids.empty() ? nullptr : ec_tids.data(), (uint32_t)nrow,
                             row_off.data(), ids.empty() ? nullptr : ids.data(), vals.empty() ? nullptr : vals.data(),
                             eff.data(), per_sample ? 1 : 0, gene_level ? gm.gene_of.data() : nullptr, G, prior_v.data(),
                             est.data(), rounds.data(), gene_level ? gene_counts.data() : nullptr,
                             gene_level ? gene_tpm.data() : nullptr));
  } else if (gene_level) {
    if (!kb_tcc_run_genes) { cerr << "Error: this libkallisto_b200 has no kb_tcc_run_genes" << endl; return 1; }
    KB_TRY(kb_tcc_run_genes(ix, n_ecs, ec_off.data(), ec_tids.empty() ? nullptr : ec_tids.data(), (uint32_t)nrow,
                            row_off.data(), ids.empty() ? nullptr : ids.data(), vals.empty() ? nullptr : vals.data(),
                            eff.data(), per_sample ? 1 : 0, gm.gene_of.data(), G, est.data(), rounds.data(),
                            gene_counts.data(), gene_tpm.data()));
  } else {
    KB_TRY(kb_tcc_run(ix, n_ecs, ec_off.data(), ec_tids.empty() ? nullptr : ec_tids.data(), (uint32_t)nrow, row_off.data(),
                      ids.empty() ? nullptr : ids.data(), vals.empty() ? nullptr : vals.data(), eff.data(), per_sample ? 1 : 0,
                      est.data(), rounds.data()));
  }
  cerr << " done" << endl << endl;
  // ---- outputs (src/main.cpp:2928-2946, 3040-3215)
  {
    std::string out;
    for (uint32_t i = 0; i < T; ++i) { out += names[i]; out += "\n"; }
    std::ofstream of(output + "/transcripts.txt", std::ios::binary);
    of.write(out.data(), (std::streamsize)out.size());
  }
  if (is_matrix) {
    std::vector<std::vector<std::pair<int, double>>> ab(nrow), tpm_m(nrow), el(nrow), ab_g(nrow), tpm_g(nrow);
    std::vector<double> tpm(T);
    for (size_t r = 0; r < nrow; ++r) {
      const double* a = est.data() + r * T;
      const double* e = eff.data() + (per_sample ? r : 0) * (size_t)T;
      const double* gc = gene_counts.data() + r * G;
      const double* gt = gene_tpm.data() + r * G;
      kb_counts_to_tpm(a, e, T, tpm.data());
      for (uint32_t i = 0; i < T; ++i)
        if (a[i] > 0.0) {
          ab[r].push_back({(int)i, a[i]});
          tpm_m[r].push_back({(int)i, tpm[i]});
          if (calc_eff) el[r].push_back({(int)i, e[i]});
        }
      if (gene_level)
        for (uint32_t g = 0; g < G; ++g)
          if (gc[g] > 0.0) {
            ab_g[r].push_back({(int)g, gc[g]});
            tpm_g[r].push_back({(int)g, gt[g]});
          }
      if (matrix_to_dirs) {
        const std::string dir = output + "/abundance_" + std::to_string(r + 1);     // src/main.cpp:3063-3084
        struct stat ds;
        if (stat(dir.c_str(), &ds) == 0) {
          if (!S_ISDIR(ds.st_mode)) { cerr << "Error: file " << dir << " exists and is not a directory" << endl; return 1; }
        } else if (mkdir(dir.c_str(), 0777) == -1) {
          cerr << "Error: could not create directory " << dir << endl;
          return 1;
        }
        write_abundance(dir + "/abundance.tsv", names, lens, e, a);
        if (gene_level) write_gene_abundance(dir + "/abundance.gene.tsv", gm, gc, gt);
      } else if (matrix_to_files) {
        write_abundance(output + "/abundance_" + std::to_string(r + 1) + ".tsv", names, lens, e, a);
        if (gene_level) write_gene_abundance(output + "/abundance.gene_" + std::to_string(r + 1) + ".tsv", gm, gc, gt);
      }
    }
    write_sparse_matrix(output + "/matrix.abundance.mtx", ab, T);
    write_sparse_matrix(output + "/matrix.abundance.tpm.mtx", tpm_m, T);
    if (calc_eff) write_sparse_matrix(output + "/matrix.efflens.mtx", el, T);
    if (gene_level) {
      write_sparse_matrix(output + "/matrix.abundance.gene.mtx", ab_g, G);
      write_sparse_matrix(output + "/matrix.abundance.gene.tpm.mtx", tpm_g, G);
      std::string out;                                              // writeGeneList(..., true), src/PlaintextWriter.cpp:300-315
      for (auto& n : gm.name) { out += n; out += "\n"; }
      std::ofstream of(output + "/genes.txt", std::ios::binary);
      of.write(out.data(), (std::streamsize)out.size());
    }
  } else {
    write_abundance(output + "/abundance.tsv", names, lens, eff.data(), est.data());
    if (gene_level) write_gene_abundance(output + "/abundance.gene.tsv", gm, gene_counts.data(), gene_tpm.data());
  }
  if (bootstrap > 0) {
    // src/main.cpp:3109-3178: bs_abundance_<b>.tsv (non-matrix file), bs_abundance_<row>_<b>.tsv (--matrix-to-files) or
    // abundance_<row>/bs_abundance_<b>.tsv (--matrix-to-directories), rows numbered from 1, each written with its row's
    // eff_lens.  A matrix row without any non-zero estimate gets B copies of that (zero) estimate.  The device hands the
    // (row, bootstrap) problems over chunk by chunk; up to -t threads write a chunk's files.  With genes, a matrix row's
    // bootstraps also get bs_abundance.gene_<row>_<b>.tsv or abundance_<row>/bs_abundance.gene_<b>.tsv, summed on the
    // device; a non-matrix file gets no gene bootstrap files, as in the reference.
    cerr << "[bstrp] running EM for " << pretty_num((size_t)nrow * bootstrap) << " bootstraps" << endl;
    std::vector<char> empty_row(nrow, 0);
    if (is_matrix)
      for (size_t r = 0; r < nrow; ++r)
        empty_row[r] = std::none_of(est.begin() + r * T, est.begin() + (r + 1) * T, [](double x) { return x > 0.0; });
    const bool bs_genes = gene_level && is_matrix;
    TccBsCtx ctx{&output, is_matrix, matrix_to_dirs != 0, per_sample, bootstrap, threads, T, &names, &lens, &eff, &est,
                 &empty_row, bs_genes ? &gm : nullptr, &gene_counts, &gene_tpm};
    if (bs_genes) {
      if (!kb_tcc_bootstrap_run_genes) { cerr << "Error: this libkallisto_b200 has no kb_tcc_bootstrap_run_genes" << endl; return 1; }
      KB_TRY(kb_tcc_bootstrap_run_genes(ix, n_ecs, ec_off.data(), ec_tids.empty() ? nullptr : ec_tids.data(), (uint32_t)nrow,
                                        row_off.data(), ids.empty() ? nullptr : ids.data(), vals.empty() ? nullptr : vals.data(),
                                        eff.data(), per_sample ? 1 : 0, gm.gene_of.data(), G, (uint64_t)seed, bootstrap, 0,
                                        write_tcc_bs_chunk, &ctx));
    } else {
      auto write_chunk = [](void* user, uint64_t first, uint32_t count, const double* bs_est, const int32_t* rounds,
                            const uint32_t* samples) -> int {
        return write_tcc_bs_chunk(user, first, count, bs_est, rounds, samples, nullptr, nullptr);
      };
      if (!kb_tcc_bootstrap_run) { cerr << "Error: this libkallisto_b200 has no kb_tcc_bootstrap_run" << endl; return 1; }
      KB_TRY(kb_tcc_bootstrap_run(ix, n_ecs, ec_off.data(), ec_tids.empty() ? nullptr : ec_tids.data(), (uint32_t)nrow, row_off.data(),
                                  ids.empty() ? nullptr : ids.data(), vals.empty() ? nullptr : vals.data(), eff.data(),
                                  per_sample ? 1 : 0, (uint64_t)seed, bootstrap, 0, write_chunk, &ctx));
    }
    cerr << " done" << endl << endl;
  }
  if (calc_eff) {
    std::ofstream of(output + "/matrix.fld.tsv");                 // writeFLD, src/PlaintextWriter.cpp:287-298
    for (size_t j = 0; j < fld_mat.size(); ++j) of << j << "\t" << fld_mat[j].first << "\t" << fld_mat[j].second << "\n";
    std::ofstream tl(output + "/transcript_lengths.txt");
    for (uint32_t i = 0; i < T; ++i) tl << names[i] << " " << lens[i] << "\n";
  }
  kb_index_free(ix);
  return 0;
}

// ------------------------------------------------------------------------------------------------
// kallisto h5dump (src/main.cpp:883-921 ParseOptionsH5Dump, 2027-2072 CheckOptionsH5Dump, 3223-3241; H5Converter,
// src/H5Writer.cpp:75-200): abundance.h5 -> abundance.tsv, bs_abundance_<b>.tsv, run_info.json.  Host only; the file is
// read by csrc/h5_reader.hpp.
// ------------------------------------------------------------------------------------------------
void usage_h5dump() {
  std::cout << "kallisto_b200 " << KALLISTO_VERSION << endl
            << "Converts HDF5-formatted results to plaintext" << endl << endl
            << "Usage:  kallisto_b200 h5dump [arguments] abundance.h5" << endl << endl
            << "Required argument:" << endl
            << "-o, --output-dir=STRING       Directory to write output to" << endl << endl;
}

int cmd_h5dump(int argc, char** argv) {
  std::string output;
  std::vector<std::string> files;
  int peek_flag = 0;
  static struct option long_options[] = {{"peek", no_argument, &peek_flag, 1}, {"output-dir", required_argument, 0, 'o'}, {0, 0, 0, 0}};
  int c, oi = 0;
  while ((c = getopt_long(argc, argv, "o:", long_options, &oi)) != -1)
    if (c == 'o') output = optarg;
  for (int i = optind; i < argc; i++) files.push_back(argv[i]);
  bool ret = true;
  struct stat stt;
  if (!peek_flag) {
    if (output.empty()) { cerr << "Error: You must specify an output directory." << endl; ret = false; }
    else if (stat(output.c_str(), &stt) == 0) {
      if (!S_ISDIR(stt.st_mode)) { cerr << "Error: tried to open " << output << " but another file already exists there" << endl; ret = false; }
    } else if (mkdir(output.c_str(), 0777) == -1) { cerr << "Error: could not create directory " << output << endl; ret = false; }
  } else if (!output.empty()) {
    cerr << "Error: Cannot specify output directory and '--peek'. Please specify only one." << endl;
    ret = false;
  }
  if (files.empty()) { cerr << "Error: Missing H5 files" << endl; ret = false; }
  else if (files.size() > 1) { cerr << "Error: Please specify only one H5 file" << endl; ret = false; }
  else if (stat(files[0].c_str(), &stt) != 0) { cerr << "Error: H5 file not found " << files[0] << endl; ret = false; }
  if (!ret) {
    usage_h5dump();
    return 1;
  }
  try {
    kb::H5Reader h5(files[0]);
    // H5Converter::H5Converter
    const std::vector<std::string> ids = h5.read_str("/aux/ids");
    cerr << "[h5dump] number of targets: " << ids.size() << endl;
    const std::vector<int64_t> lengths = h5.read_int("/aux/lengths");
    const std::vector<double> eff = h5.read_f64("/aux/eff_lengths");
    if (lengths.size() != ids.size() || eff.size() != ids.size()) throw std::runtime_error("Error: /aux/ids, /aux/lengths and /aux/eff_lengths differ in size");
    const int64_t n_bs = h5.read_int("/aux/num_bootstrap").at(0), n_proc = h5.read_int("/aux/num_processed").at(0);
    cerr << "[h5dump] number of bootstraps: " << n_bs << endl;
    const std::string version = h5.read_str("/aux/kallisto_version").at(0);
    cerr << "[h5dump] kallisto version: " << version << endl;
    const int64_t index_version = h5.read_int("/aux/index_version").at(0);
    cerr << "[h5dump] index version: " << index_version << endl;
    const std::string start_time = h5.read_str("/aux/start_time").at(0);
    cerr << "[h5dump] start time: " << start_time << endl;
    const std::string call = h5.read_str("/aux/call").at(0);
    cerr << "[h5dump] shell call: " << call << endl;
    if (peek_flag) return 0;
    std::vector<uint32_t> lens(lengths.begin(), lengths.end());
    // H5Converter::write_aux: the number of pseudoaligned reads is the rounded sum of the estimated counts, the number of
    // unique reads and the k-mer length are not in the file ("-1", "dummy k-mer length")
    std::vector<double> alpha = h5.read_f64("/est_counts");
    if (alpha.size() != ids.size()) throw std::runtime_error("Error: /est_counts and /aux/ids differ in size");
    double sum = 0.0;
    for (double x : alpha) sum += x;
    const int n_paln = (int)std::round(sum);
    {
      std::ofstream of(output + "/run_info.json");
      double p_uniq = 0.0, p_aln = 0.0;
      if ((double)n_proc > 0) {
        p_uniq = 100.0 * -1.0 / (double)n_proc;
        p_aln = 100.0 * (double)n_paln / (double)n_proc;
      }
      std::stringstream ss;
      ss << std::fixed << std::setprecision(1) << p_uniq;
      const std::string p_uniq_s = ss.str();
      ss.str("");
      ss << std::fixed << std::setprecision(1) << p_aln;
      const std::string p_aln_s = ss.str();
      of << "{" << std::endl
         << to_json("n_targets", std::to_string(ids.size()), false) << std::endl
         << to_json("n_bootstraps", std::to_string(n_bs), false) << std::endl
         << to_json("n_processed", std::to_string(n_proc), false) << std::endl
         << to_json("n_pseudoaligned", std::to_string(n_paln), false) << std::endl
         << to_json("n_unique", "-1", false) << std::endl
         << to_json("p_pseudoaligned", p_aln_s, false) << std::endl
         << to_json("p_unique", p_uniq_s, false) << std::endl
         << to_json("kallisto_version", version, true) << std::endl
         << to_json("index_version", std::to_string(index_version), false) << std::endl
         << to_json("k-mer length", "dummy k-mer length", false) << std::endl
         << to_json("start_time", start_time, true) << std::endl
         << to_json("call", call, true, false) << std::endl
         << "}" << std::endl;
    }
    // H5Converter::convert
    cerr << "[h5dump] writing abundance file: " << output << "/abundance.tsv" << endl;
    write_abundance(output + "/abundance.tsv", ids, lens, eff.data(), alpha.data());
    if (n_bs > 0) cerr << "[h5dump] writing bootstrap abundance files: " << output << "/bs_abundance_*.tsv" << endl;
    int64_t i = 0;
    for (; i < n_bs; ++i) {
      if (i % 50 == 0 && i > 0) cerr << endl;
      cerr << ".";
      alpha = h5.read_f64("/bootstrap/bs" + std::to_string(i));
      if (alpha.size() != ids.size()) throw std::runtime_error("Error: a bootstrap dataset and /aux/ids differ in size");
      write_abundance(output + "/bs_abundance_" + std::to_string(i) + ".tsv", ids, lens, eff.data(), alpha.data());
    }
    if (i > 0) cerr << endl;
  } catch (const std::exception& e) {
    cerr << e.what() << endl;
    return 1;
  }
  return 0;
}

}  // namespace

int main(int argc, char** argv) {
  // start time and call line, as in src/main.cpp:2260-2291
  std::time_t t = std::time(nullptr);
  char tbuf[64];
  std::strftime(tbuf, sizeof(tbuf), "%a %b %e %H:%M:%S %Y", std::localtime(&t));   // std::asctime layout, no newline
  std::string call;
  for (int i = 0; i < argc; ++i) {
    if (i) call += " ";
    call += argv[i];
  }
  if (argc < 2) {
    std::cout << "kallisto_b200 " << KALLISTO_VERSION << endl << endl
              << "Usage: kallisto_b200 <CMD> [arguments] .." << endl << endl
              << "Where <CMD> can be one of:" << endl << endl
              << "    quant         Runs the quantification algorithm (GPU)" << endl
              << "    bus           Generate BUS files for single-cell data (GPU)" << endl
              << "    quant-tcc     Runs quantification on transcript-compatibility counts (GPU)" << endl
              << "    h5dump        Converts HDF5-formatted results to plaintext" << endl
              << "    version       Prints version information" << endl << endl
              << "Indices are built with the reference `kallisto index` (format v13)." << endl;
    return 1;
  }
  const std::string cmd = argv[1];
  if (cmd == "version") {
    std::cout << "kallisto_b200, version " << KALLISTO_VERSION << " (" << kb_version() << ")" << endl;
    return 0;
  }
  if (cmd == "quant") {
    if (argc == 2) {
      usage_quant();
      return 0;
    }
    return cmd_quant(argc - 1, argv + 1, call, tbuf);
  }
  if (cmd == "bus") {
    if (argc == 2) {
      usage_bus();
      return 0;
    }
    return cmd_bus(argc - 1, argv + 1, call, tbuf);
  }
  if (cmd == "quant-tcc") {
    if (argc == 2) {
      usage_tcc();
      return 0;
    }
    return cmd_quant_tcc(argc - 1, argv + 1);
  }
  if (cmd == "h5dump") {
    if (argc == 2) {
      usage_h5dump();
      return 1;
    }
    return cmd_h5dump(argc - 1, argv + 1);
  }
  cerr << "Error: invalid command " << cmd << endl;
  return 1;
}
