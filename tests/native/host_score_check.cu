// Host build of the scanners' scoring (kai_action.cuh: node_key, repeat_row, binpack_score, better), the code the solver
// also runs on the host to answer small restricted sweeps from its node mirror.  Reads one case per line on stdin and
// prints the result, so tests/test_host_score.py can compare it bit for bit with the oracle's scoring:
//   K R strategy res gpu_task best_effort nominated n mn mx a_gpu a_cpu gpu_count nflags req[R] I[R] L[R]
//       -> "K <fits> <fit_i> <score as %a>"
//   A R ... (as K) ... L[R] pipeline_only k win
//       -> "A <to_idle> <repeat ok> <fits> <fit_i> <score as %a>": repeat_row's row after k placements (no topology term),
//          then row_fits / row_score on it
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
    } else if (f[0] == "K" || f[0] == "A") {
      const bool adv = f[0] == "A";
      const int R = (int)I(1);
      if (R < 1 || R > KAI_MAX_RES || f.size() != 14 + 3 * (size_t)R + (adv ? 3 : 0)) {
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
      double a_gpu = D(10), a_cpu = D(11), gpu_count = D(12);
      uint32_t nflags = (uint32_t)I(13);
      std::vector<double> row(2 * R);
      for (int r = 0; r < R; r++) {
        d.req[r] = D(14 + r);
        row[r] = D(14 + R + r);
        row[R + r] = D(14 + 2 * R + r);
      }
      double score = 0;
      bool fit_i = false;
      if (!adv) {
        const bool fits = node_key(d, R, row.data(), row.data() + R, 1, a_gpu, a_cpu, gpu_count, nflags, n, score, fit_i);
        printf("K %d %d %a\n", fits ? 1 : 0, fits && fit_i ? 1 : 0, fits ? score : 0.0);
        continue;
      }
      const size_t a = 14 + 3 * (size_t)R;
      d.pipeline_only = (int)I(a);
      Tile tl;
      memset(&tl, 0, sizeof(tl));
      int node = n, rank = 0;
      tl.I = row.data();
      tl.L = row.data() + R;
      tl.Agpu = &a_gpu;
      tl.Acpu = &a_cpu;
      tl.gpu_count = &gpu_count;
      tl.rank = &rank;
      tl.flags = &nflags;
      tl.node = &node;
      tl.npc = tl.count = 1;
      tl.R = R;
      double Ik[KAI_MAX_RES], Lk[KAI_MAX_RES];
      bool to_idle = false, fits_k = false;
      const bool ok = repeat_row(tl, d, 0, (int)I(a + 1), D(a + 2), 0.0, Ik, Lk, to_idle, fits_k);
      row_fits(d.req, R, Ik, Lk, 1, fit_i);
      if (fits_k) score = row_score(d, Ik, Lk, 1, a_gpu, a_cpu, gpu_count, nflags, n, fit_i);
      printf("A %d %d %d %d %a\n", to_idle ? 1 : 0, ok ? 1 : 0, fits_k ? 1 : 0, fits_k && fit_i ? 1 : 0, fits_k ? score : 0.0);
    } else {
      printf("FAIL unknown case kind %s\n", f[0].c_str());
      return 1;
    }
  }
  printf("OK\n");
  return 0;
}
