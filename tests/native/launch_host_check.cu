// Host-only check of the launch transport's host side (kai_host_seq.cuh): (1) a decision record is packed into the
// LaunchRec a k_record launch carries exactly as the scanners decode it (folded node deltas, repeat counts, extended
// entries), (2) the merged candidate lists of several GPUs are merged with the cut rule applied across ranks, negative
// and -0.0 scores included, (3) the integer sort key of k_merge_cluster orders every score as the comparator does,
// (4) single-row and min-max answer lines are taken only under their full 64-bit sequence number, and a line that
// changes while it is read fails the action.
// Built and run by tests/test_launch_host.py (nvcc, no GPU needed: nothing is launched).
#include <algorithm>
#include <cfloat>
#include <cmath>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <vector>

#include <signal.h>
#include <sys/mman.h>
#include <unistd.h>

#include "../../kai_scheduler_b200/csrc/kai_host_seq.cuh"

using namespace kai;

static unsigned long long rng_state = 0x0C42ULL;
static unsigned int rnd() {
  rng_state = rng_state * 6364136223846793005ULL + 1442695040888963407ULL;
  return (unsigned int)(rng_state >> 33);
}

static LaunchRec g_last;
static int g_launches = 0;
static bool fake_launch(void *, const LaunchRec &rec) {
  g_last = rec;
  g_launches++;
  return true;
}

#define CHECK(cond, ...)            \
  do {                              \
    if (!(cond)) {                  \
      printf("FAIL %s:%d ", __FILE__, __LINE__); \
      printf(__VA_ARGS__);          \
      printf("\n");                 \
      return 1;                     \
    }                               \
  } while (0)

// ---------------------------------------------------------------- (4) answer lines
// A line as the last CTA of k_record writes it: payload words, the sequence number in the last word.
static void put_line(unsigned long long *line, const unsigned long long *payload, unsigned long long seq_no) {
  for (int i = 0; i < kLineWords - 1; i++) line[i] = payload[i];
  line[kLineWords - 1] = seq_no;
}
static unsigned long long dbits(double d) {
  unsigned long long u;
  memcpy(&u, &d, 8);
  return u;
}

// A line whose number changes between the wait and the re-check: the payload sits at the end of a page that is not
// readable yet, the sequence word at the start of the next page.  The wait sees the wanted number; the first payload
// load faults, and the handler rewrites the sequence word (as the GPU would for a later record) and makes the payload
// readable, so the re-check sees the new number.
static unsigned long long *g_moving_seq = nullptr;
static unsigned char *g_payload_page = nullptr;
static size_t g_page = 0;
static void move_on(int, siginfo_t *, void *) {
  *g_moving_seq += 2;
  mprotect(g_payload_page, g_page, PROT_READ | PROT_WRITE);
}

static int check_answer_lines(HostBackend &hb) {
  std::vector<int> rank_to_node(64);
  for (int i = 0; i < 64; i++) rank_to_node[i] = 1000 + i;
  hb.rank_to_node = rank_to_node.data();
  hb.failed = false;
  hb.error_msg[0] = 0;
  memset(&hb.ctl.trk, 0, sizeof(hb.ctl.trk));
  for (int S = 1; S <= 3; S++) {
    hb.n_ranks = S;
    std::vector<unsigned long long> slots((size_t)2 * S * kLineWords, 0), mm((size_t)2 * S * kLineWords, 0);
    hb.h_slots = slots.data();
    hb.h_mm = mm.data();
    // single-row lines above 2^32: rank r answers rank 10 + r with score 3 - r (rank 0 wins) and one repeat
    const unsigned long long seq_no = (3ull << 32) + 17 + (unsigned long long)S;
    for (int r = 0; r < S; r++) {
      const unsigned long long meta = ((unsigned long long)SLOT_TO_IDLE << 32) | (1ull << 24) | (unsigned long long)(10 + r);
      const unsigned long long w[kLineWords - 1] = {dbits(3.0 - r), meta, dbits(0.5), dbits(0.25), 0x2aull, 0, 0};
      put_line(slots.data() + ((seq_no & 1) * S + r) * kLineWords, w, seq_no);
    }
    hb.ctl.seq = seq_no;
    hb.gather_candidates();
    CHECK(!hb.failed && hb.ctl.seq == seq_no + 1, "S=%d: single-row lines at seq %llu", S, seq_no);
    CHECK(hb.ctl.win.score == 3.0 && hb.ctl.win.rank == 10 && hb.ctl.win.node == 1010 && hb.ctl.win.flags == SLOT_TO_IDLE,
          "S=%d: winner score %g rank %u node %d flags %u", S, hb.ctl.win.score, hb.ctl.win.rank, hb.ctl.win.node, hb.ctl.win.flags);
    CHECK(hb.ctl.batch.valid && hb.ctl.batch.left == 1 && hb.ctl.batch.node == 1010 && hb.ctl.batch.fl == 0x2aull, "S=%d: repeat", S);
    // min/max lines above 2^32: rank r reports gpu [1 + r, 8 - r] with counts (r + 1, 2), cpu [5, 5] with (1, 1)
    const unsigned long long mm_seq = seq_no + 1;
    for (int r = 0; r < S; r++) {
      const unsigned long long w[kLineWords - 1] = {dbits(1.0 + r), dbits(8.0 - r), dbits(5.0), dbits(5.0),
                                                     (unsigned long long)(r + 1) | (2ull << 32), 1ull | (1ull << 32), 0};
      put_line(mm.data() + ((mm_seq & 1) * S + r) * kLineWords, w, mm_seq);
    }
    hb.gather_minmax();
    CHECK(!hb.failed && hb.ctl.seq == mm_seq + 1, "S=%d: min/max lines at seq %llu", S, mm_seq);
    CHECK(hb.ctl.trk[0].mn == 1.0 && hb.ctl.trk[0].cnt_mn == 1 && hb.ctl.trk[0].mx == 8.0 && hb.ctl.trk[0].cnt_mx == 2,
          "S=%d: gpu tracker %g x%d .. %g x%d", S, hb.ctl.trk[0].mn, hb.ctl.trk[0].cnt_mn, hb.ctl.trk[0].mx, hb.ctl.trk[0].cnt_mx);
    CHECK(hb.ctl.trk[1].mn == 5.0 && hb.ctl.trk[1].cnt_mn == S && hb.ctl.trk[1].mx == 5.0 && hb.ctl.trk[1].cnt_mx == S,
          "S=%d: cpu tracker", S);
  }
  // a stale line whose number agrees with the wanted one in its low 24 or low 32 bits is never taken
  const double keep_timeout = hb.timeout_s;
  hb.timeout_s = 0.05;
  hb.n_ranks = 1;
  const unsigned long long wanted = (1ull << 32) + (7ull << 24) + 12345;
  const unsigned long long stale[2] = {wanted - (1ull << 24) * 2, wanted - (1ull << 32) * 2};  // same parity
  for (int i = 0; i < 2; i++)
    for (int kind = 0; kind < 2; kind++) {
      std::vector<unsigned long long> lines((size_t)2 * kLineWords, 0);
      const unsigned long long w[kLineWords - 1] = {dbits(1.0), 7ull, 0, 0, 0, 0, 0};
      put_line(lines.data() + (wanted & 1) * kLineWords, w, stale[i]);
      hb.h_slots = hb.h_mm = lines.data();
      hb.failed = false;
      hb.ctl.seq = wanted;
      if (kind == 0)
        hb.gather_candidates();
      else
        hb.gather_minmax();
      CHECK(hb.failed && (kind == 1 || hb.ctl.win.node == -1), "stale line %llu taken for %llu (%s)", stale[i], wanted,
            kind == 0 ? "single row" : "min/max");
    }
  hb.timeout_s = keep_timeout;
  // a line that moves on to a later record between the wait and the re-check fails the action and names the record
  g_page = (size_t)sysconf(_SC_PAGESIZE);
  unsigned char *pages = (unsigned char *)mmap(nullptr, 2 * g_page, PROT_READ | PROT_WRITE, MAP_PRIVATE | MAP_ANONYMOUS, -1, 0);
  CHECK(pages != MAP_FAILED, "mmap");
  unsigned long long *line = (unsigned long long *)(pages + g_page) - (kLineWords - 1);
  const unsigned long long w[kLineWords - 1] = {dbits(2.0), 3ull, 0, 0, 0, 0, 0};
  const unsigned long long moving = 4242;
  put_line(line, w, moving);
  g_moving_seq = line + kLineWords - 1;
  g_payload_page = pages;
  struct sigaction sa, old;
  memset(&sa, 0, sizeof(sa));
  sa.sa_sigaction = &move_on;
  sa.sa_flags = SA_SIGINFO;
  sigaction(SIGSEGV, &sa, &old);
  mprotect(pages, g_page, PROT_NONE);
  unsigned long long payload[kLineWords - 1];
  hb.failed = false;
  hb.error_msg[0] = 0;
  const bool ok = hb.read_line(line, moving, payload);
  sigaction(SIGSEGV, &old, nullptr);
  CHECK(!ok && hb.failed && *g_moving_seq == moving + 2, "a line that changed while it was read was accepted");
  CHECK(strstr(hb.error_msg, "record 4242") != nullptr, "error message names the record: %s", hb.error_msg);
  munmap(pages, 2 * g_page);
  return 0;
}

int main() {
  // ---------------------------------------------------------------- (1) record packing
  const int N = 64, T = 40, R = 4;
  std::vector<int> name_rank(N), rank_to_node(4096);
  for (int n = 0; n < N; n++) name_rank[n] = (n * 37) % N;  // a permutation (37 is odd, N a power of two)
  for (int i = 0; i < 4096; i++) rank_to_node[i] = i;
  std::vector<double> t_req((size_t)T * R);
  for (int t = 0; t < T; t++)
    for (int r = 0; r < R; r++) t_req[(size_t)t * R + r] = (double)(1 + (t / 4) % 3) * (r + 1);  // runs of 4 identical requests
  DevSnap s;
  memset(&s, 0, sizeof(s));
  s.R = R;
  s.N = N;
  s.T = T;
  s.name_rank = name_rank.data();
  s.t_req = t_req.data();
  HostBackend hb;
  std::vector<unsigned long long> delta_buf((size_t)2 * kMaxDelta * 2, 0);
  memset(&hb.ctl, 0, sizeof(hb.ctl));
  memset(&hb.seq, 0, sizeof(hb.seq));
  hb.seq.s = &s;
  hb.seq.ctl = &hb.ctl;
  hb.seq.delta_base = delta_buf.data();
  hb.seq.host_backend = &hb;
  hb.launch_fn = &fake_launch;
  hb.rank_to_node = rank_to_node.data();
  hb.ctl.seq = 7;
  hb.ctl.dec.nominated = hb.ctl.dec.pred_class = -1;
  // what the scanners must see: (rank | code << 28, first task, repeat count)
  struct Want {
    unsigned int key, task;
    int count;
  };
  std::vector<Want> want;
  auto expect = [&](int node, int code, int t) {
    const unsigned int key = (unsigned int)(name_rank[node] | (code << 28));
    if (!want.empty() && code < ND_FEAS_SET && want.back().key == key && want.back().count < 255 && !(want.back().key & 0x80000000u)) {
      bool same = true;
      for (int r = 0; r < R; r++) same = same && t_req[(size_t)want.back().task * R + r] == t_req[(size_t)t * R + r];
      if (same) {
        want.back().count++;
        return;
      }
    }
    want.push_back({key, (unsigned int)t, 1});
  };
  // four identical pods on node 5 (fold to one entry, count 4), a different request on the same node, another node,
  // a removal, a feasible-set bit, an extended entry, then again node 5
  for (int t = 0; t < 4; t++) {
    emit_delta(hb.seq, 5, ND_ADD, t);
    expect(5, ND_ADD, t);
  }
  emit_delta(hb.seq, 5, ND_ADD, 4);
  expect(5, ND_ADD, 4);
  emit_delta(hb.seq, 9, ND_ADD_PIPELINED, 5);
  expect(9, ND_ADD_PIPELINED, 5);
  emit_delta(hb.seq, 9, ND_REM_PIPELINED, 5);
  expect(9, ND_REM_PIPELINED, 5);
  emit_delta(hb.seq, 11, ND_FEAS_SET, 0);
  want.push_back({(unsigned int)(name_rank[11] | (ND_FEAS_SET << 28)), 0u, 1});
  emit_ext(hb.seq, EXT_SCORE, 17u, 3u);
  want.push_back({0x80000000u | ((unsigned int)EXT_SCORE << 28) | 17u, 3u, 1});
  emit_delta(hb.seq, 5, ND_ADD, 8);
  want.push_back({(unsigned int)(name_rank[5] | (ND_ADD << 28)), 8u, 1});
  emit_delta(hb.seq, 5, ND_ADD, 9);  // same request as task 8: folds
  want.back().count++;
  for (int r = 0; r < KAI_MAX_RES; r++) hb.ctl.dec.req[r] = r < R ? t_req[r] : 0.0;
  hb.ctl.dec.gpu_task = 1;
  hb.ctl.dec.res = KAI_RES_GPU;
  hb.ctl.xbits = XB_SINGLE;
  hb.publish(DK_SCAN);
  CHECK(g_launches == 1, "one launch per record, got %d", g_launches);
  CHECK(g_last.seq == 7u && g_last.n_delta == (int)want.size(), "seq %llu n_delta %d (want %zu)", (unsigned long long)g_last.seq,
        g_last.n_delta, want.size());
  CHECK((int)(g_last.dw[0] & 0xff) == DK_SCAN && (int)((g_last.dw[0] >> 32) & 0xffff) == (int)want.size(), "record word 0");
  CHECK(((unsigned int)(g_last.dw[0] >> 48) & XB_SINGLE) != 0, "xbits");
  for (size_t e = 0; e < want.size(); e++)
    CHECK(g_last.dkey[e] == want[e].key && g_last.dtask[e] == want[e].task && (int)g_last.dcount[e] == want[e].count - 1,
          "delta %zu: key %08x task %u count-1 %d, want %08x %u %d", e, g_last.dkey[e], g_last.dtask[e], (int)g_last.dcount[e], want[e].key,
          want[e].task, want[e].count - 1);
  // a full list flushes by a launch of its own, without waiting and without taking a sequence number
  hb.ctl.seq = 8;
  hb.ctl.n_delta = 0;
  hb.ctl.last_dcount = 0;
  for (int i = 0; i < kMaxDelta + 3; i++) emit_delta(hb.seq, i % N, ND_ADD, (i * 5) % T);  // neighbours differ: no folding
  CHECK(g_launches == 2 && (int)(g_last.dw[0] & 0xff) == DK_FLUSH && g_last.n_delta == kMaxDelta, "flush launch: %d launches, kind %d, n_delta %d",
        g_launches, (int)(g_last.dw[0] & 0xff), g_last.n_delta);
  CHECK(g_last.seq == 8u && hb.ctl.seq == 8u && hb.ctl.n_delta == 3, "after the flush: record seq %llu, next seq %llu, n_delta %d",
        (unsigned long long)g_last.seq, (unsigned long long)hb.ctl.seq, hb.ctl.n_delta);
  // past 2^32 the record still carries the whole number, and the folded repeat counts are intact
  hb.ctl.seq = (5ull << 32) + 9;
  hb.ctl.n_delta = 0;
  hb.ctl.last_dcount = 0;
  for (int t = 0; t < 4; t++) emit_delta(hb.seq, 5, ND_ADD, t);
  hb.publish(DK_SCAN);
  CHECK(g_last.seq == (5ull << 32) + 9 && g_last.n_delta == 1 && g_last.dcount[0] == 3, "record at seq 2^32 * 5 + 9: seq %llu n_delta %d count-1 %d",
        (unsigned long long)g_last.seq, g_last.n_delta, (int)g_last.dcount[0]);

  // ---------------------------------------------------------------- (2) merging the GPUs' lists
  for (int trial = 0; trial < 200; trial++) {
    const int S = 1 + (int)(rnd() % 4);
    std::vector<unsigned long long> clist((size_t)S * 2 * kCListWords, 0);
    hb.h_clist = clist.data();
    hb.n_ranks = S;
    hb.failed = false;
    const unsigned long long seq_no = 100 + (unsigned long long)trial;
    hb.ctl.seq = seq_no;
    struct Ent {
      double score;
      unsigned int rank;
    };
    std::vector<Ent> all;
    bool have_cut = false;
    Ent cut{0, 0};
    auto before = [](const Ent &a, const Ent &b) { return a.score > b.score || (a.score == b.score && a.rank < b.rank); };
    std::vector<unsigned int> ranks(2048);
    for (unsigned int i = 0; i < 2048; i++) ranks[i] = i;
    for (int i = 2047; i > 0; i--) std::swap(ranks[i], ranks[rnd() % (i + 1)]);
    size_t next_rank = 0;
    for (int r = 0; r < S; r++) {
      const int n = (int)(rnd() % 40);
      std::vector<Ent> mine;
      // few score levels, many ties; negative idle GPUs (over-committed nodes) and -0.0 (== +0.0: the rank decides)
      static const double levels[] = {4.0, 2.0, 1.0, 0.0, -0.0, -1.0, -3.0};
      for (int i = 0; i < n; i++) mine.push_back({levels[rnd() % 7], ranks[next_rank++]});
      std::sort(mine.begin(), mine.end(), before);
      const bool more = (rnd() & 1) != 0;
      unsigned long long *cl = clist.data() + ((size_t)r * 2 + (seq_no & 1)) * kCListWords;
      for (int i = 0; i < n; i++) {
        unsigned long long *e = cl + 2 + (size_t)i * kCEntryWords;
        memcpy(&e[0], &mine[i].score, 8);
        e[1] = (unsigned long long)mine[i].rank | (2ull << 24) | ((unsigned long long)LF_TO_IDLE << 32);  // cap 3
        double v = 1.0 + i;
        for (int q = 0; q < 4; q++) memcpy(&e[2 + q], &v, 8);
      }
      cl[0] = (unsigned long long)(unsigned int)n | (more ? (1ull << 31) : 0ull);
      cl[1] = seq_no;
      for (auto &m : mine) all.push_back(m);
      if (more && n > 0 && (!have_cut || before(mine.back(), cut))) {
        have_cut = true;
        cut = mine.back();
      }
    }
    std::sort(all.begin(), all.end(), before);
    size_t valid = all.size();
    if (have_cut)
      for (size_t i = 0; i < all.size(); i++)
        if (before(cut, all[i])) {  // strictly worse than the cut row: an unseen row could sit before it
          valid = i;
          break;
        }
    hb.gather_list();
    CHECK(!hb.failed, "trial %d: wait failed", trial);
    CHECK(hb.list.size() == all.size(), "trial %d: %zu entries, want %zu", trial, hb.list.size(), all.size());
    CHECK(hb.list_valid == valid, "trial %d (S=%d): valid prefix %zu, want %zu", trial, S, hb.list_valid, valid);
    CHECK(hb.list_more == have_cut, "trial %d: more flag", trial);
    for (size_t i = 0; i < valid; i++)
      CHECK(hb.list[i].score == all[i].score && hb.list[i].rank == all[i].rank && hb.list[i].cap == 3 &&
                hb.list[i].node == (int)all[i].rank,
            "trial %d entry %zu", trial, i);
    CHECK(hb.ctl.seq == seq_no + 1 && hb.ctl.n_delta == 0, "trial %d: sequence", trial);
  }

  // ---------------------------------------------------------------- (3) the list merge's sort key
  // k_merge_cluster sorts candidates by (list_key(score), rank << 32 | source) as unsigned integers; that order must be
  // the comparator's (score desc, rank asc) for every score a list can carry, and every real key must precede the
  // empty slot (~0ull).
  {
    auto dbl = [](unsigned long long u) {
      double d;
      memcpy(&d, &u, 8);
      return d;
    };
    const double specials[] = {0.0, -0.0, 1.0, -1.0, 8.0, -3.0, 0.5, -0.5, DBL_MAX, -DBL_MAX, DBL_MIN, -DBL_MIN,
                               dbl(1), dbl(0x8000000000000001ull), dbl(0x000fffffffffffffull), dbl(0x800fffffffffffffull),
                               HUGE_VAL, -HUGE_VAL, 1e300, -1e300, 2.0 - 1e-15, 2.0 + 4e-16};
    const int n_spec = (int)(sizeof(specials) / sizeof(specials[0]));
    for (int v = 0; v < n_spec; v++)
      CHECK(list_key(specials[v]) < ~0ull, "key of %a reaches the empty slot", specials[v]);
    CHECK(list_key(0.0) == list_key(-0.0), "-0.0 and +0.0 keys differ");
    CHECK(list_key(2.0) == ~kbits(2.0) - (1ull << 63), "non-negative keys keep their order: ~bits with the top bit cleared");
    long long pairs = 0;
    for (int trial = 0; trial < 300; trial++) {
      const int n = 1 + (int)(rnd() % 600);
      struct C {
        double v;
        unsigned int rank, src;
      };
      std::vector<C> c(n);
      std::vector<unsigned int> rk(n);
      for (int i = 0; i < n; i++) rk[i] = (unsigned int)i;
      for (int i = n - 1; i > 0; i--) std::swap(rk[i], rk[rnd() % (i + 1)]);
      for (int i = 0; i < n; i++) {
        double v;
        switch (rnd() % 6) {
          case 0: v = specials[rnd() % n_spec]; break;
          case 1: v = (double)((int)(rnd() % 9) - 4); break;  // exact ties around 0
          case 2: v = (rnd() & 1) ? 0.0 : -0.0; break;
          case 3: v = dbl(((unsigned long long)rnd() << 32 | rnd()) & 0x800fffffffffffffull); break;  // subnormal
          case 4: v = ((double)rnd() - 2147483648.0) * 1e-3; break;
          default: {  // any finite bit pattern
            unsigned long long u;
            do u = (unsigned long long)rnd() << 32 | rnd();
            while (((u >> 52) & 0x7ff) == 0x7ff);
            v = dbl(u);
          }
        }
        c[i] = {v, rk[i], (unsigned int)i};
      }
      std::vector<int> want_p(n), got_p(n);
      for (int i = 0; i < n; i++) want_p[i] = got_p[i] = i;
      std::sort(want_p.begin(), want_p.end(), [&](int a, int b) { return c[a].v > c[b].v || (c[a].v == c[b].v && c[a].rank < c[b].rank); });
      std::sort(got_p.begin(), got_p.end(), [&](int a, int b) {
        const unsigned long long ha = list_key(c[a].v), hb_ = list_key(c[b].v);
        const unsigned long long la = (unsigned long long)c[a].rank << 32 | c[a].src, lb = (unsigned long long)c[b].rank << 32 | c[b].src;
        return ha < hb_ || (ha == hb_ && la < lb);
      });
      for (int i = 0; i < n; i++)
        CHECK(want_p[i] == got_p[i], "key trial %d: position %d holds %a (rank %u), want %a (rank %u)", trial, i, c[got_p[i]].v,
              c[got_p[i]].rank, c[want_p[i]].v, c[want_p[i]].rank);
      for (int i = 0; i < n; i++) CHECK(list_key(c[i].v) < ~0ull, "key trial %d: %a reaches the empty slot", trial, c[i].v);
      pairs += n;
    }
    printf("OK record packing (%zu deltas, flush), 200 multi-GPU list merges and the list sort key (%lld candidates)",
           want.size(), pairs);
  }
  if (int rc = check_answer_lines(hb)) return rc;
  printf(", answer lines\n");
  return 0;
}
