// TEST INFRASTRUCTURE: the stand-in library of stub_abi.cpp plus the --priors entry points, so that the command line's
// handling of -p/--priors runs on a CPU-only box (tests/test_oracle_priors.py).  kb_read_priors is the library's own
// parser (csrc/priors.hpp); kb_em_set_priors checks the count against the stand-in's 3 targets and changes nothing else.
// Never linked into the product.
#include "stub_abi.cpp"
#include "priors.hpp"

extern "C" {
int kb_read_priors(const char* path, double* out, uint64_t cap, uint64_t* n_out) {
  std::vector<double> v;
  uint64_t line = 0;
  const int r = kb::read_priors_file(path, v, &line);
  if (r == 1) { g_err = std::string("could not open priors file ") + path; return KB_ERR_IO; }
  if (r == 2) { g_err = "line " + std::to_string(line) + " of priors file " + path + " is not a number"; return KB_ERR_INVALID; }
  *n_out = v.size();
  if (out && cap >= v.size() && !v.empty()) memcpy(out, v.data(), v.size() * sizeof(double));
  return KB_OK;
}
int kb_em_set_priors(kb_quant*, const double*, uint32_t n) {
  if (n != 3) { g_err = "kb_em_set_priors: wrong count"; return KB_ERR_INVALID; }
  return KB_OK;
}
}
