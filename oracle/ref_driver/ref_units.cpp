// ref_units -- TEST INFRASTRUCTURE ONLY.
//
// Table-driven harness around the UNMODIFIED reference classes (linked from oracle/_ref/obj):
// market::Order, market::AskBook/BidBook/BookUtils, market::Market, RollingMean<double>,
// rl::State (tiles()/hash_UNH), and the C++/C runtime generators the reference consumes
// (std::mt19937_64 + distributions, glibc rand()).  It replays (a) the scenarios of the
// reference's own Catch tests (test/test_Order.cpp, test_Market.cpp, test_Accumulators.cpp,
// test_Book.cpp single-order cases) and (b) seeded random scripts, and prints one JSON document.
// tools/make_golden.py stores that document as tests/golden/units.json; the oracle port and the
// CUDA device entry points are then checked against it on machines where /root/reference and
// this binary do not exist.
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <random>
#include <string>
#include <vector>

#include "market/book.h"
#include "market/market.h"
#include "market/measures.h"
#include "market/order.h"
#include "rl/state.h"
#include "utilities/accumulators.h"

using namespace std;

static uint64_t lcg_state = 12345;
static uint32_t lcg() { lcg_state = lcg_state * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(lcg_state >> 33); }

static void p_d(double d) { uint64_t u; memcpy(&u, &d, 8); printf("\"%016llx\"", (unsigned long long)u); }  // exact bits

int main() {
  printf("{\n");
  // ---------------------------------------------------------------- Order scripts
  // op: 0 doTransaction, 1 doCancellation, 2 addVolumeBehind, 3 clearQueues
  struct Script { long size, qh; vector<pair<int, long>> ops; };
  vector<Script> scripts = {
      {100, 0, {{1, 50}}},                         // test_Order.cpp:103-113  0:100:0 cancel 50 -> queue ahead stays 0
      {100, 100, {{1, 50}}},                       // :115-125  -> 50
      {100, 100, {{1, 100}}},                      // :127-133  -> 0
      {100, 100, {{2, 500}, {1, 50}}},             // :185-204  100:100:500 cancel 50 -> 91:459
      {100, 100, {{2, 500}, {1, 100}}},            // :206-213  -> 83:417
      {100, 100, {{2, 500}, {1, 600}}},            // :215-222  -> 0:0
      {100, 100, {{2, 500}, {1, 1000}}},           // :224-231  -> 0:0
      {100, 100, {{2, 5000}, {1, 50}}},            // :238-245  -> 99:4951
      {100, 100, {{2, 5000}, {1, 100}}},           // :247-254  -> 98:4902
      {100, 100, {{2, 5000}, {1, 10000}}},         // :256-263  -> 0:0
      {100, 50, {{0, 25}, {0, 25}, {0, 60}, {0, 100}}},
      {100, 100, {{2, 30}, {2, -60}, {1, 20}}},    // negative q_tail (SURVEY Appendix A4)
      {100, 20, {{2, -20}, {1, 5}}},               // q_head + q_tail == 0: division by zero path (A5)
      {100, 10, {{2, -30}, {1, 4}}},               // SURVEY 8c extra vector -> 12:0
  };
  for (int k = 0; k < 40; ++k) {  // seeded random scripts
    Script s; s.size = 1 + lcg() % 200; s.qh = lcg() % 1000;
    int n = 1 + lcg() % 8;
    for (int i = 0; i < n; ++i) {
      int op = lcg() % 4;
      long arg = (op == 2) ? (long)(lcg() % 1200) - 400 : (long)(lcg() % 600);
      s.ops.push_back({op, arg});
    }
    scripts.push_back(s);
  }
  printf("\"orders\": [\n");
  for (size_t k = 0; k < scripts.size(); ++k) {
    auto& s = scripts[k];
    market::Order o(1.0, s.size, s.qh);
    printf("  {\"size\": %ld, \"q_head\": %ld, \"ops\": [", s.size, s.qh);
    for (size_t i = 0; i < s.ops.size(); ++i) printf("%s[%d, %ld]", i ? ", " : "", s.ops[i].first, s.ops[i].second);
    printf("], \"out\": [");
    for (size_t i = 0; i < s.ops.size(); ++i) {
      long ret = 0;
      switch (s.ops[i].first) {
        case 0: ret = o.doTransaction(s.ops[i].second); break;
        case 1: o.doCancellation(s.ops[i].second); break;
        case 2: o.addVolumeBehind(s.ops[i].second); break;
        case 3: o.clearQueues(); break;
      }
      printf("%s[%ld, %ld, %ld, %ld]", i ? ", " : "", o.getQueueAhead(), o.getQueueBehind(), o.getTotalExecutedVolume(), ret);
    }
    printf("]}%s\n", k + 1 < scripts.size() ? "," : "");
  }
  printf("],\n");

  // ---------------------------------------------------------------- Market (test/test_Market.cpp)
  printf("\"market\": [\n");
  const char* syms[][2] = {{"AAL", "L"}, {"BAES", "L"}, {"X", "AS"}, {"X", "BR"}, {"X", "CO"}, {"X", "DE"}, {"X", "HE"}, {"X", "I"},
                           {"X", "MC"}, {"X", "MI"}, {"X", "OL"}, {"X", "PA"}, {"X", "S"}, {"X", "VX"}, {"X", "ST"}, {"X", "VI"}};
  const int n_syms = (int)(sizeof(syms) / sizeof(syms[0]));
  for (int si = 0; si < n_syms; ++si) {
    market::Market* m = market::Market::make_market(syms[si][0], syms[si][1]);
    vector<double> px = {2750.0, 2750.5, 702.1, 702.5, 1000.0, 999.9, 999.95, 4999.5, 5000.0, 5001.0, 0.5, 0.00005, 1.0, 12.345,
                         49.99, 50.0, 99.999, 100.0, 123.45, 499.95, 500.0, 9999.0, 10000.0, 10002.5, 52500.0, 52501.0, 52487.0,
                         20000.0, 45020.0, 85040.0, 123400.0};
    for (int i = 0; i < 60; ++i) px.push_back((lcg() % 6000000) / 1000.0 + 0.001 * (lcg() % 7));
    printf("  {\"symbol\": \"%s.%s\", \"px\": [", syms[si][0], syms[si][1]);
    for (size_t i = 0; i < px.size(); ++i) { printf("%s", i ? ", " : ""); p_d(px[i]); }
    printf("], \"ticks\": [");
    vector<int> tk;
    for (size_t i = 0; i < px.size(); ++i) { int t = m->ToTicks(px[i]); tk.push_back(t); printf("%s%d", i ? ", " : "", t); }
    printf("], \"tick_size\": [");
    for (size_t i = 0; i < px.size(); ++i) { printf("%s", i ? ", " : ""); p_d(m->tick_size(px[i])); }
    vector<int> tq = {1, 10000, 10001, 18000, 49000, 49001, 52500, 52501, 57000, 57001, 62000, 46021, 46025};
    for (int i = 0; i < 40; ++i) tq.push_back(1 + lcg() % 62000);
    printf("], \"tq\": [");
    for (size_t i = 0; i < tq.size(); ++i) printf("%s%d", i ? ", " : "", tq[i]);
    printf("], \"price\": [");
    for (size_t i = 0; i < tq.size(); ++i) { printf("%s", i ? ", " : ""); p_d(m->ToPrice(tq[i])); }
    printf("], \"open\": %ld, \"close\": %ld}%s\n", m->open_time(), m->close_time(), si + 1 < n_syms ? "," : "");
    delete m;
  }
  printf("],\n");

  // ---------------------------------------------------------------- RollingMean<double> (test/test_Accumulators.cpp)
  printf("\"rolling\": [\n");
  for (int k = 0; k < 6; ++k) {
    int w = (k == 0) ? 3 : (k == 1 ? 5 : 1 + (int)(lcg() % 60));
    int n = (k < 2) ? 8 : 150;
    vector<double> v;
    for (int i = 0; i < n; ++i) v.push_back(k == 0 ? (double)(i + 1) : (k == 1 ? (double)(3 + i % 3) : 52000.0 + (lcg() % 4000) * 0.5));
    RollingMean<double> r(w);
    printf("  {\"window\": %d, \"vals\": [", w);
    for (int i = 0; i < n; ++i) { printf("%s", i ? ", " : ""); p_d(v[i]); }
    printf("], \"mean_var\": [");
    for (int i = 0; i < n; ++i) { r.push(v[i]); printf("%s[", i ? ", " : ""); p_d(r.mean()); printf(", "); p_d(r.var()); printf("]"); }
    printf("]}%s\n", k < 5 ? "," : "");
  }
  printf("],\n");

  // ---------------------------------------------------------------- tiles via rl::State (src/rl/state.cpp:53-65)
  // One entry per (memory_size, n_actions, n_vars); features[a*96 + i] = State::getFeatures(a)[i].
  printf("\"tiles\": [\n");
  auto tile_entry = [](long mem, int n_actions, int n_vars, const vector<vector<float>>& states, bool last) {
    rl::State st(mem, n_actions, 32);
    printf("  {\"memory_size\": %ld, \"n_actions\": %d, \"n_vars\": %d, \"cases\": [\n", mem, n_actions, n_vars);
    for (size_t k = 0; k < states.size(); ++k) {
      vector<float> v = states[k];
      st.newState(v, 0.0);
      printf("    {\"vars\": [");
      for (int i = 0; i < n_vars; ++i) { uint32_t u; memcpy(&u, &v[i], 4); printf("%s%u", i ? ", " : "", u); }
      printf("], \"features\": [");
      for (int a = 0; a < n_actions; ++a) {
        auto& f = st.getFeatures(a);
        for (int i = 0; i < 96; ++i) printf("%s%d", (a || i) ? ", " : "", f[i]);
      }
      printf("]}%s\n", k + 1 < states.size() ? "," : "");
    }
    printf("  ]}%s\n", last ? "" : ",");
  };
  long mems[3] = {65536, 20000000, 5003};
  for (int mi = 0; mi < 3; ++mi) {
    vector<vector<float>> states;
    for (int k = 0; k < 6; ++k) {
      vector<float> v(8);
      if (k == 0) v = {0.5f, -100.0f, -100.0f, 0.0f, 1.0f, 0.0f, 0.0f, 0.0f};
      else for (int i = 0; i < 8; ++i) v[i] = (float)((int)(lcg() % 4000) - 2000) / 97.0f;
      states.push_back(v);
    }
    tile_entry(mems[mi], 9, 8, states, false);
  }
  // The edges of the learner's index arithmetic: tables smaller than a step's 32 tiles per group (M = 1 has no
  // magic-number reciprocal; 1 and 2 are powers of two), both sides of the 2^27 limit of the packed tile table, and
  // tables above 2^30, where the sum of two indices below M no longer fits an int.  Every action count meets every
  // state size over the sweep.  A generator of its own keeps the vectors of the other sections as they were.
  {
    uint64_t s = 977;
    auto next = [&s]() -> uint32_t { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); };
    const long edge[8] = {1, 2, 3, 1L << 27, (1L << 27) + 1, (1L << 30) + 3, 3L << 29, 2147483647L};
    const int acts[3] = {1, 5, 9}, nvars[3] = {4, 8, 13};
    for (int mi = 0; mi < 8; ++mi)
      for (int c = 0; c < 3; ++c) {
        const int nv = nvars[(c + mi) % 3];
        vector<vector<float>> states;
        for (int k = 0; k < 2; ++k) {
          vector<float> v(nv);
          for (int i = 0; i < nv; ++i) v[i] = (float)((int)(next() % 40000) - 20000) / 97.0f;
          states.push_back(v);
        }
        tile_entry(edge[mi], acts[c], nv, states, mi == 7 && c == 2);
      }
  }
  printf("],\n");

  // ---------------------------------------------------------------- generators
  printf("\"rng\": {\n");
  {
    unsigned seeds[3] = {1994, 0, 4000000007u};
    printf("  \"cases\": [\n");
    for (int s = 0; s < 3; ++s) {
      std::mt19937_64 g(seeds[s]);
      printf("    {\"seed\": %u, \"mt\": [", seeds[s]);
      for (int i = 0; i < 320; ++i) printf("%s\"%llu\"", i ? ", " : "", (unsigned long long)g());
      std::mt19937_64 g2(seeds[s]);
      std::uniform_real_distribution<double> ur(0.0, 1.0);
      printf("], \"real\": [");
      for (int i = 0; i < 40; ++i) { printf("%s", i ? ", " : ""); p_d(ur(g2)); }
      std::mt19937_64 g3(seeds[s]);
      std::uniform_int_distribution<unsigned> ui(0, 8);
      printf("], \"int9\": [");
      for (int i = 0; i < 200; ++i) printf("%s%u", i ? ", " : "", ui(g3));
      srand(seeds[s]);
      printf("], \"rand\": [");
      for (int i = 0; i < 100; ++i) printf("%s%d", i ? ", " : "", rand());
      printf("]}%s\n", s < 2 ? "," : "");
    }
    printf("  ]\n");
  }
  printf("},\n");

  // ---------------------------------------------------------------- Book scenarios, one order per side
  // Seeded random walks over: snapshot, place order (both sides), prints, adverse selection.
  printf("\"book\": [\n");
  for (int sc = 0; sc < 12; ++sc) {
    market::AskBook<5> ask; market::BidBook<5> bid;
    double bb = 2750.0 + 0.5 * (lcg() % 20);
    int spread = 1 + lcg() % 3;
    long av[5], bv[5];
    for (int l = 0; l < 5; ++l) { av[l] = 100 + lcg() % 900; bv[l] = 100 + lcg() % 900; }
    printf("  {\"steps\": [\n");
    int nsteps = 30;
    for (int stp = 0; stp < nsteps; ++stp) {
      // prints against the current book (none on the first snapshot)
      std::map<double, long, FloatComparator<>> tx;
      double mp = 0;
      printf("    {");
      if (stp > 0) {
        mp = market::measure::midprice(ask, bid);
        int n = lcg() % 3;
        for (int i = 0; i < n; ++i) {
          bool buy = lcg() & 1; int deep = (lcg() % 4 == 0);
          double p = buy ? ask.price(0) + 0.5 * deep : bid.price(0) - 0.5 * deep;
          tx[p] += 1 + lcg() % 400;
        }
        printf("\"tx\": [");
        int c = 0;
        for (auto& kv : tx) { printf("%s[", c++ ? ", " : ""); p_d(kv.first); printf(", %ld]", kv.second); }
        printf("], \"ref\": "); p_d(mp);
        auto au = ask.ApplyTransactions(tx, mp);
        auto bu = bid.ApplyTransactions(tx, mp);
        printf(", \"au\": [%ld, ", get<0>(au)); p_d(get<1>(au)); printf(", "); p_d(get<2>(au));
        printf("], \"bu\": [%ld, ", get<0>(bu)); p_d(get<1>(bu)); printf(", "); p_d(get<2>(bu)); printf("], ");
      }
      // new snapshot
      int mv = (int)(lcg() % 3) - 1;
      if (lcg() % 5 == 0) spread = 1 + lcg() % 3;
      bb += 0.5 * mv;
      std::array<double, 5> ap, bp; std::array<long, 5> avv, bvv;
      for (int l = 0; l < 5; ++l) {
        long da = (long)(lcg() % 81) - 40, db = (long)(lcg() % 81) - 40;
        av[l] = std::max(1L, av[l] + da); bv[l] = std::max(1L, bv[l] + db);
        ap[l] = bb + 0.5 * (spread + l); bp[l] = bb - 0.5 * l; avv[l] = av[l]; bvv[l] = bv[l];
      }
      ask.StashState(); bid.StashState();
      ask.ApplyChanges(ap, avv, tx); bid.ApplyChanges(bp, bvv, tx);
      printf("\"ap\": ["); for (int l = 0; l < 5; ++l) { printf("%s", l ? ", " : ""); p_d(ap[l]); }
      printf("], \"av\": [%ld, %ld, %ld, %ld, %ld], \"bp\": [", avv[0], avv[1], avv[2], avv[3], avv[4]);
      for (int l = 0; l < 5; ++l) { printf("%s", l ? ", " : ""); p_d(bp[l]); }
      printf("], \"bv\": [%ld, %ld, %ld, %ld, %ld]", bvv[0], bvv[1], bvv[2], bvv[3], bvv[4]);
      if (stp > 0) {
        auto as = market::BookUtils::HandleAdverseSelection(ask, bid);
        printf(", \"as\": [%ld, ", get<0>(as)); p_d(get<1>(as)); printf(", "); p_d(get<2>(as)); printf("]");
      }
      // (re)place one order per side every few steps, like RiskManager::PlaceOrder with ORDER_LIMIT 1
      if (stp % 3 == 0) {
        double apx = ask.price(0) + 0.5 * ((int)(lcg() % 4) - 1), bpx = bid.price(0) - 0.5 * ((int)(lcg() % 4) - 1);
        long sz = 1 + lcg() % 50;
        if (ask.order_count() > 0) ask.CancelWorst();
        ask.PlaceOrder(apx, sz);
        if (bid.order_count() > 0) bid.CancelWorst();
        bid.PlaceOrder(bpx, sz);
        printf(", \"place\": ["); p_d(apx); printf(", "); p_d(bpx); printf(", %ld]", sz);
      }
      // observable order state
      for (int s = 0; s < 2; ++s) {
        printf(", \"%s\": ", s == 0 ? "ask_o" : "bid_o");
        bool live = s == 0 ? ask.order_count() > 0 : bid.order_count() > 0;
        if (!live) printf("null");
        else {
          double p = s == 0 ? ask.best_open_order_price() : bid.best_open_order_price();
          long qa = s == 0 ? ask.queue_ahead(p) : bid.queue_ahead(p);
          long qb = s == 0 ? ask.queue_behind(p) : bid.queue_behind(p);
          long rem = s == 0 ? ask.order_remaining_volume(p) : bid.order_remaining_volume(p);
          printf("["); p_d(p); printf(", %ld, %ld, %ld]", qa, qb, rem);
        }
      }
      printf(", \"ntr\": [%d, %d], \"tv\": [%ld, %ld]}%s\n", ask.n_transacted(), bid.n_transacted(), ask.total_volume(), bid.total_volume(),
             stp + 1 < nsteps ? "," : "");
    }
    printf("  ]}%s\n", sc < 11 ? "," : "");
  }
  printf("]\n}\n");
  return 0;
}
