// The solver's heap (kai_solver.cuh: HeapGo, the sift code every JobsOrder heap runs on its arena range) against a
// plain restatement of Go's container/heap (Push / Pop / Fix / up / down, as in the Go sources) under the same random
// push / pop / fix sequences.  The comparator is a random relation that is neither antisymmetric nor transitive, as the
// queue-order comparators can be, so only the exact sift sequence reproduces the pop order.  The solver's heap lives
// inside a larger buffer at an offset, as a JobsOrder range does.  Usage: heap_go_check <seed> <rounds>; prints OK or
// the first difference.  No GPU is needed: nothing is launched.
#include <cstdio>
#include <cstdlib>
#include <random>
#include <vector>

#include "../../kai_scheduler_b200/csrc/kai_solver.cuh"

namespace {

// container/heap restated: the heap is h (a slice), Less(i, j) compares h[i] and h[j]
struct GoHeap {
  std::vector<int> h;
  const std::vector<std::vector<char>> *rel;
  bool Less(int i, int j) const { return (*rel)[h[i]][h[j]] != 0; }
  void Swap(int i, int j) { std::swap(h[i], h[j]); }
  void up(int j) {
    for (;;) {
      int i = (j - 1) / 2;  // parent (Go's integer division truncates toward zero, like C++'s)
      if (i == j || !Less(j, i)) break;
      Swap(i, j);
      j = i;
    }
  }
  bool down(int i0, int n) {
    int i = i0;
    for (;;) {
      int j1 = 2 * i + 1;
      if (j1 >= n || j1 < 0) break;
      int j = j1;
      int j2 = j1 + 1;
      if (j2 < n && Less(j2, j1)) j = j2;
      if (!Less(j, i)) break;
      Swap(i, j);
      i = j;
    }
    return i > i0;
  }
  void Push(int x) {
    h.push_back(x);
    up((int)h.size() - 1);
  }
  int Pop() {
    int n = (int)h.size() - 1;
    Swap(0, n);
    down(0, n);
    int x = h.back();
    h.pop_back();
    return x;
  }
  void Fix(int i) {
    if (!down(i, (int)h.size())) up(i);
  }
};

}  // namespace

int main(int argc, char **argv) {
  const unsigned seed = argc > 1 ? (unsigned)atoi(argv[1]) : 1u;
  const int rounds = argc > 2 ? atoi(argv[2]) : 2000;
  std::mt19937 rng(seed);
  const int V = 2 + (int)(rng() % 60);  // value domain; small domains give many equal values
  std::vector<std::vector<char>> rel(V, std::vector<char>(V));
  const unsigned p_true = 20 + rng() % 60;  // per cent of pairs for which less(a, b) holds; both directions may hold
  for (int a = 0; a < V; a++)
    for (int b = 0; b < V; b++) rel[a][b] = (char)(rng() % 100 < p_true);
  auto less = [&](int a, int b) { return rel[a][b] != 0; };

  GoHeap ref;
  ref.rel = &rel;
  const int off = 7, cap = rounds + 1;
  std::vector<int> buf((size_t)off + cap + 5, -1);
  int *a = buf.data() + off;
  int n = 0;
  for (int step = 0; step < rounds; step++) {
    const unsigned op = rng() % 10;
    if (op < 5 || n == 0) {
      const int x = (int)(rng() % V);
      ref.Push(x);
      kai::HeapGo::push(a, n, x, less);
    } else if (op < 8) {
      const int x = ref.Pop(), y = kai::HeapGo::pop(a, n, less);
      if (x != y) {
        printf("FAIL seed %u step %d: pop gives %d, container/heap gives %d\n", seed, step, y, x);
        return 1;
      }
    } else {
      const int i = (int)(rng() % n), x = (int)(rng() % V);
      ref.h[i] = x;
      a[i] = x;
      ref.Fix(i);
      kai::HeapGo::fix(a, n, i, less);
    }
    if (n != (int)ref.h.size()) {
      printf("FAIL seed %u step %d: length %d, container/heap %zu\n", seed, step, n, ref.h.size());
      return 1;
    }
    for (int i = 0; i < n; i++)
      if (a[i] != ref.h[i]) {
        printf("FAIL seed %u step %d: entry %d is %d, container/heap has %d\n", seed, step, i, a[i], ref.h[i]);
        return 1;
      }
  }
  while (n > 0) {
    const int x = ref.Pop(), y = kai::HeapGo::pop(a, n, less);
    if (x != y) {
      printf("FAIL seed %u drain: pop gives %d, container/heap gives %d\n", seed, y, x);
      return 1;
    }
  }
  if (buf[off - 1] != -1 || buf[(size_t)off + cap] != -1) {
    printf("FAIL seed %u: wrote outside the heap's range\n", seed);
    return 1;
  }
  printf("OK\n");
  return 0;
}
