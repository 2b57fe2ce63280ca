// Host build of the scanners' scoring (kai_action.cuh: node_key, binpack_score, better), the code the solver also runs
// on the host to answer small restricted sweeps from its node mirror.  Reads one case per line on stdin and prints the
// result, so tests/test_host_score.py can compare it bit for bit with the oracle's scoring:
//   K R strategy res gpu_task best_effort nominated n mn mx a_gpu a_cpu gpu_count nflags req[R] I[R] L[R]
//       -> "K <fits> <fit_i> <score as %a>"
//   P mn mx cur overall      -> "P <binpack_score as %a>"
//   B sa ra sb rb            -> "B <better(sa, ra, sb, rb)>"
// Doubles are read with strtod (hexadecimal floats are exact).  No GPU is needed: nothing is launched.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "../../kai_scheduler_b200/csrc/kai_host_seq.cuh"

using namespace kai;

static std::vector<std::string> split(const char *line) {
  std::vector<std::string> out;
  const char *p = line;
  while (*p) {
    while (*p == ' ' || *p == '\t' || *p == '\n') p++;
    if (!*p) break;
    const char *b = p;
    while (*p && *p != ' ' && *p != '\t' && *p != '\n') p++;
    out.emplace_back(b, p - b);
  }
  return out;
}

int main() {
  char line[8192];
  while (fgets(line, sizeof(line), stdin)) {
    std::vector<std::string> f = split(line);
    if (f.empty()) continue;
    auto D = [&](size_t i) { return strtod(f.at(i).c_str(), nullptr); };
    auto I = [&](size_t i) { return atoll(f.at(i).c_str()); };
    if (f[0] == "P") {
      printf("P %a\n", binpack_score(D(1), D(2), D(3), D(4)));
    } else if (f[0] == "B") {
      printf("B %d\n", better(D(1), (uint32_t)I(2), D(3), (uint32_t)I(4)) ? 1 : 0);
    } else if (f[0] == "K") {
      const int R = (int)I(1);
      if (R < 1 || R > KAI_MAX_RES || f.size() != 14 + 3 * (size_t)R) {
        printf("FAIL bad case line\n");
        return 1;
      }
      Decision d;
      memset(&d, 0, sizeof(d));
      d.strategy = (int)I(2);
      d.res = (int)I(3);
      d.gpu_task = (int)I(4);
      d.best_effort = (int)I(5);
      d.nominated = (int)I(6);
      const int n = (int)I(7);
      d.mn = D(8);
      d.mx = D(9);
      const double a_gpu = D(10), a_cpu = D(11), gpu_count = D(12);
      const uint32_t nflags = (uint32_t)I(13);
      std::vector<double> row(2 * R);
      for (int r = 0; r < R; r++) {
        d.req[r] = D(14 + r);
        row[r] = D(14 + R + r);
        row[R + r] = D(14 + 2 * R + r);
      }
      double score = 0;
      bool fit_i = false;
      const bool fits = node_key(d, R, row.data(), row.data() + R, 1, a_gpu, a_cpu, gpu_count, nflags, n, score, fit_i);
      printf("K %d %d %a\n", fits ? 1 : 0, fits && fit_i ? 1 : 0, fits ? score : 0.0);
    } else {
      printf("FAIL unknown case kind %s\n", f[0].c_str());
      return 1;
    }
  }
  printf("OK\n");
  return 0;
}
