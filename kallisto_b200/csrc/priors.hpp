// --priors file (EMAlgorithm::read_priors, src/EMAlgorithm.h:52-81): one value per line, each line through std::stod (leading
// blanks skipped, whatever follows the number ignored), summed in file order.  A sum >= 1 + 1e-3 means raw counts: every value
// becomes (value + 1) / (sum + number of values).  Otherwise the values are used as they are.  Host code, shared by
// kb_read_priors and the stand-in library of the command-line tests.
#pragma once
#include <cstdint>
#include <fstream>
#include <stdexcept>
#include <string>
#include <vector>

namespace kb {

// 0: read; 1: the file cannot be opened; 2: line `*bad_line` (1-based) is not a number std::stod accepts (the reference
// aborts there with an uncaught exception).
inline int read_priors_file(const std::string& path, std::vector<double>& out, uint64_t* bad_line) {
  out.clear();
  std::ifstream f(path);
  if (!f) return 1;
  std::string line;
  double sum = 0.0;
  uint64_t n = 0;
  while (std::getline(f, line)) {
    ++n;
    double p;
    try {
      p = std::stod(line);
    } catch (const std::logic_error&) {   // std::invalid_argument, std::out_of_range
      if (bad_line) *bad_line = n;
      out.clear();
      return 2;
    }
    out.push_back(p);
    sum += p;
  }
  if (sum >= 1. + 1e-3) {
    sum += out.size();
    for (double& v : out) v = (v + 1.) / sum;
  }
  return 0;
}

}  // namespace kb
