// ref_q_values -- TEST INFRASTRUCTURE ONLY (fixture generator; never on the product path).
//
// Agent::getQ / DoubleAgent::getQb of the UNMODIFIED reference: rl::QLearn and rl::DoubleQLearn build their tables with
// learning.random_init (agent.cpp:37-39,190-192) from debug.random_seed; each case prints getQ (and getQb) of every action
// for a list of states made by State::newState(vars, 0.0) (state.cpp:45-51): exact tile boundaries, negatives, large
// values, infinities, NaN and seeded values.  One JSON document on stdout, doubles as exact bit patterns.
// tools/make_golden.py --q-values compiles this file against the reference objects oracle/Makefile builds into
// oracle/_ref/obj and stores the output as tests/golden/q_values.json.
#include <unistd.h>

#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <limits>
#include <memory>
#include <string>
#include <vector>

#include "rl/agent.h"
#include "rl/policy.h"
#include "rl/state.h"
#include "utilities/config.h"

using namespace std;

static void p_d(double d) { uint64_t u; memcpy(&u, &d, 8); printf("\"%016llx\"", (unsigned long long)u); }  // exact bits

int main() {
  struct Case { const char* algo; long mem; int n_actions, n_vars; unsigned seed; };
  const Case cases[] = {
      {"q_learn", 4096, 9, 8, 11},         {"q_learn", 5003, 5, 4, 12},         {"double_q_learn", 4096, 5, 13, 13},
      {"double_q_learn", 5003, 9, 8, 14},  {"q_learn", 5003, 9, 13, 15},        {"double_q_learn", 4096, 9, 4, 16},
      {"q_learn", 4096, 3, 13, 17},        {"double_q_learn", 5003, 2, 8, 18},
  };
  const int n_cases = (int)(sizeof(cases) / sizeof(cases[0]));
  uint64_t s = 31337;
  auto next = [&s]() -> uint32_t { s = s * 6364136223846793005ull + 1442695040888963407ull; return (uint32_t)(s >> 33); };
  const float nan = std::numeric_limits<float>::quiet_NaN(), inf = std::numeric_limits<float>::infinity();
  const char* tmp = getenv("TMPDIR");
  const string path_s = string(tmp && *tmp ? tmp : "/tmp") + "/ref_q_values_" + to_string((long)getpid()) + ".yaml";
  const char* path = path_s.c_str();
  printf("{\"cases\": [\n");
  for (int ci = 0; ci < n_cases; ++ci) {
    const Case& cs = cases[ci];
    FILE* f = fopen(path, "w");
    if (!f) { perror(path); return 1; }
    fprintf(f, "debug:\n  random_seed: %u\nlearning:\n  memory_size: %ld\n  n_tilings: 32\n  n_actions: %d\n  random_init: true\n"
               "  group_weights: [0.65, 0.25, 0.10]\n  gamma: 0.975\n  lambda: 0.85\n", cs.seed, cs.mem, cs.n_actions);
    fclose(f);
    Config c(path);
    remove(path);
    const bool dbl = strcmp(cs.algo, "double_q_learn") == 0;
    std::unique_ptr<rl::Policy> pol(new rl::Greedy(cs.n_actions, cs.seed));
    rl::Agent* m = dbl ? (rl::Agent*)new rl::DoubleQLearn(std::move(pol), c) : (rl::Agent*)new rl::QLearn(std::move(pol), c);
    vector<vector<float>> states;
    const int nv = cs.n_vars;
    auto fill = [&](float x) { vector<float> v(nv, x); return v; };
    states.push_back(fill(0.0f));
    states.push_back(fill(1.0f / 32.0f));   // exact tile boundaries: q = floor(v * 32) lands on an integer
    states.push_back(fill(-1.0f / 32.0f));
    states.push_back(fill(-0.0f));
    {
      vector<float> v(nv);
      for (int i = 0; i < nv; ++i) v[i] = (float)((int)i - 5) / 32.0f;
      states.push_back(v);
    }
    {
      vector<float> v(nv);
      for (int i = 0; i < nv; ++i) v[i] = (float)((int)i * 7 - 20) * 0.5f - (float)i / 64.0f;  // negatives, half-tile offsets
      states.push_back(v);
    }
    states.push_back(fill(1.0e8f));   // large: v * 32 still converts
    states.push_back(fill(-3.0e9f));  // v * 32 out of int range: x86's integer indefinite
    states.push_back(fill(nan));
    states.push_back(fill(inf));
    {
      vector<float> v(nv);
      const float odd[6] = {nan, -inf, 6.7e7f, -1.0e30f, 0.015625f, 123.456f};
      for (int i = 0; i < nv; ++i) v[i] = (i % 2) ? odd[(i / 2) % 6] : (float)((int)(next() % 4000) - 2000) / 97.0f;
      states.push_back(v);
    }
    for (int k = 0; k < 13; ++k) {
      vector<float> v(nv);
      for (int i = 0; i < nv; ++i) v[i] = (float)((int)(next() % 40000) - 20000) / 97.0f;
      states.push_back(v);
    }
    printf("  {\"algorithm\": \"%s\", \"memory_size\": %ld, \"n_actions\": %d, \"n_vars\": %d, \"random_seed\": %u, "
           "\"group_weights\": [0.65, 0.25, 0.10], \"queries\": [\n", cs.algo, cs.mem, cs.n_actions, nv, cs.seed);
    rl::State st(cs.mem, cs.n_actions, 32);
    for (size_t k = 0; k < states.size(); ++k) {
      vector<float> v = states[k];
      st.newState(v, 0.0);
      printf("    {\"vars\": [");
      for (int i = 0; i < nv; ++i) { uint32_t u; memcpy(&u, &states[k][i], 4); printf("%s%u", i ? ", " : "", u); }
      printf("], \"q\": [");
      for (int a = 0; a < cs.n_actions; ++a) { printf("%s", a ? ", " : ""); p_d(m->getQ(st, a)); }
      if (dbl) {
        printf("], \"qb\": [");
        for (int a = 0; a < cs.n_actions; ++a) { printf("%s", a ? ", " : ""); p_d(((rl::DoubleAgent*)m)->getQb(st, a)); }
      }
      printf("]}%s\n", k + 1 < states.size() ? "," : "");
    }
    printf("  ]}%s\n", ci + 1 < n_cases ? "," : "");
    delete m;
  }
  printf("]}\n");
  return 0;
}

