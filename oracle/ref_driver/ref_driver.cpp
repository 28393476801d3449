// ref_driver -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// Drives the UNMODIFIED reference (tspooner/rl_markets, compiled from
// /root/reference by oracle/Makefile into oracle/_ref/) for ONE environment
// and ONE agent on a pair of reference-format CSV files, and dumps one
// rlm_step_record per learner step.  It replaces src/main.cpp (which needs
// Boost): policy / agent construction follows src/main.cpp:82-189 for a
// single thread, the episode loop follows experiment::serial::Runner::
// RunEpisode and Learner::_step (src/experiment/serial.cpp:18-34,53-70).
// Everything else -- Intraday, Base, RiskManager, Book, Order, Market, the
// accumulators, State/tiles, Traces, QLearn/SARSA/DoubleQLearn, the policies,
// the CSV streamers -- is the reference's own object code.
//
// Subclasses are used only to READ protected members for the dump and to
// capture the TD error returned by the (virtual) UpdateWeights.
#include <algorithm>
#include <chrono>
#include <cstdint>
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <fstream>
#include <iostream>
#include <memory>
#include <string>
#include <vector>

#include <spdlog/spdlog.h>
#include <spdlog/sinks/null_sink.h>

#include "rl/agent.h"
#include "rl/policy.h"
#include "rl/state.h"
#include "environment/intraday.h"
#include "market/market.h"
#include "market/measures.h"

#include "rlm_record.h"

using namespace std;

namespace {

struct EnvSpy : public environment::Intraday<> {
  using environment::Intraday<>::Intraday;

  void fill(rlm_step_record& r) {
    r.time_ms = (int32_t)market->time();
    r.terminal = isTerminal() ? 1 : 0;
    r.position = risk_manager_.exposure();
    r.ask_quote = ask_quote;
    r.bid_quote = bid_quote;
    r.ask_level = ask_level;
    r.bid_level = bid_level;
    r.pnl_step = pnl_step;
    r.ep_pnl = episode_stats.pnl;
    r.ep_reward = episode_stats.reward;
    r.ep_bandh = episode_stats.bandh;
    r.midprice = market::measure::midprice(ask_book_, bid_book_);
    r.spread = market::measure::spread(ask_book_, bid_book_);
    r.bandh_step = last_bandh;
    fill_order(ask_book_, r.ask);
    fill_order(bid_book_, r.bid);
    r.ask_transactions = ask_book_.n_transacted();
    r.bid_transactions = bid_book_.n_transacted();
    r.market_buys = trade_stats.market_buys;
    r.market_sells = trade_stats.market_sells;
    r.lo_vol_step = lo_vol_step;
  }

  template <class B>
  static void fill_order(B& book, rlm_order_rec& o) {
    memset(&o, 0, sizeof(o));
    if (book.order_count() > 0) {
      double p = book.best_open_order_price();
      o.exists = 1;
      o.price = p;
      o.q_head = book.queue_ahead(p);
      o.q_tail = book.queue_behind(p);
      o.executed = book.order_size(p) - book.order_remaining_volume(p);
    }
  }

  long n_ticks_total() { return tick_stats.total_ticks; }

  // the bandh_step column of the profit_log row (a local of performAction, base.cpp:333)
  double last_bandh = 0.0;
  void LogProfit(int action, double pnl, double bandh) override {
    last_bandh = bandh;
    environment::Intraday<>::LogProfit(action, pnl, bandh);
  }
};

// Captures delta and exposes theta / traces of any concrete agent.
template <class A>
struct AgentSpy : public A {
  AgentSpy(std::unique_ptr<rl::Policy> p, Config& c) : A(std::move(p), c) {}
  double last_delta = 0.0;

  double UpdateWeights(rl::State& f, int a, double r, rl::State& t) override {
    last_delta = A::UpdateWeights(f, a, r, t);
    return last_delta;
  }
};

struct AgentView {
  rl::Agent* agent = nullptr;
  std::function<double()> delta;
  std::function<double*()> theta;
  std::function<double*()> theta_b;  // may return nullptr
  std::function<rl::Traces*()> traces;
  long memory_size = 0;
};

// theta_b is private in DoubleAgent; it is only reachable through getQb.  The
// dump therefore hashes theta (table A) for all agents and, for double
// agents, additionally folds in table B via a one-feature State probe.
template <class A>
struct Access : public AgentSpy<A> {
  using AgentSpy<A>::AgentSpy;
  double* th() { return this->theta; }
  rl::Traces* tr() { return &this->traces; }
};

template <class A>
AgentView make_agent(std::unique_ptr<rl::Policy> p, Config& c) {
  auto* a = new Access<A>(std::move(p), c);
  AgentView v;
  v.agent = a;
  v.delta = [a]() { return a->last_delta; };
  v.theta = [a]() { return a->th(); };
  v.traces = [a]() { return a->tr(); };
  v.memory_size = c["learning"]["memory_size"].as<long>();
  return v;
}

uint64_t bits_of(double d) { uint64_t u; memcpy(&u, &d, 8); return u; }
uint32_t bits_of(float f) { uint32_t u; memcpy(&u, &f, 4); return u; }

void usage() {
  fprintf(stderr,
          "usage: ref_driver --config cfg.yaml --symbol AAL.L --md md.csv --tas tas.csv\n"
          "                  [--algo q_learn|sarsa|double_q_learn] [--steps N] [--dump out.bin]\n"
          "                  [--theta out_theta.bin] [--quiet]\n"
          "                  [--episodes N]   N training episodes on ONE Intraday + ONE Learner-equivalent (the States and the\n"
          "                                   agent are reused, LoadData + RunEpisode per episode: main.cpp:45-60, serial.cpp:72-95)\n"
          "                  [--test-md md.csv --test-tas tas.csv [--test-symbol T] --dump-test out.bin]...\n"
          "                                   evaluation phase of main.cpp:216-244, one group per test day: ONE Intraday for\n"
          "                                   every day, LoadData + a new Backtester per day; --test-symbol defaults to --symbol\n"
          "                  [--log-dir d]   evaluation phase writes d/profit_log.csv, d/order_log.csv (Backtester ctor) and\n"
          "                                  d/test_stats.csv (env.writeStats after the last day, main.cpp:244)\n");
}

}  // namespace

int main(int argc, char** argv) {
  string cfg, symbol = "AAL.L", md, tas, algo, dump, theta_out, log_dir;
  vector<string> test_md, test_tas, test_symbol, dump_test;  // one entry per test day
  long max_steps = -1;
  int n_episodes = 1;
  bool quiet = false;
  for (int i = 1; i < argc; ++i) {
    string a = argv[i];
    auto next = [&]() -> string { if (i + 1 >= argc) { usage(); exit(2); } return argv[++i]; };
    if (a == "--config") cfg = next();
    else if (a == "--symbol") symbol = next();
    else if (a == "--md") md = next();
    else if (a == "--tas") tas = next();
    else if (a == "--algo") algo = next();
    else if (a == "--steps") max_steps = atol(next().c_str());
    else if (a == "--dump") dump = next();
    else if (a == "--theta") theta_out = next();
    else if (a == "--test-md") test_md.push_back(next());
    else if (a == "--test-tas") test_tas.push_back(next());
    else if (a == "--test-symbol") test_symbol.push_back(next());
    else if (a == "--dump-test") dump_test.push_back(next());
    else if (a == "--log-dir") log_dir = next();
    else if (a == "--episodes") n_episodes = atoi(next().c_str());
    else if (a == "--quiet") quiet = true;
    else { usage(); return 2; }
  }
  if (cfg.empty() || md.empty() || tas.empty()) { usage(); return 2; }
  const size_t n_test = test_md.size();
  if (test_tas.size() != n_test || (!dump_test.empty() && dump_test.size() != n_test) ||
      (!test_symbol.empty() && test_symbol.size() != n_test)) { usage(); return 2; }

  try {
    Config c(cfg);

    // agent.cpp:95-100 and serial.cpp:81 dereference these loggers unconditionally.
    if (!spdlog::get("model_log")) spdlog::create<spdlog::sinks::null_sink_mt>("model_log");
    if (!spdlog::get("training_log")) spdlog::create<spdlog::sinks::null_sink_mt>("training_log");

    // main.cpp:84-88
    unsigned seed = c["debug"]["random_seed"].as<unsigned>(
        chrono::system_clock::now().time_since_epoch().count());
    srand(seed);

    // main.cpp:137-165
    unsigned int n_actions = c["learning"]["n_actions"].as<unsigned int>();
    std::unique_ptr<rl::Policy> p;
    string policy_type = c["policy"]["type"].as<string>("");
    if (policy_type == "greedy")
      p = std::unique_ptr<rl::Policy>(new rl::Greedy(n_actions, seed));
    else if (policy_type == "random")
      p = std::unique_ptr<rl::Policy>(new rl::Random(n_actions, seed));
    else if (policy_type == "epsilon_greedy") {
      float eps = c["policy"]["eps_init"].as<float>(), eps_floor = c["policy"]["eps_floor"].as<float>();
      unsigned int eps_T = c["policy"]["eps_T"].as<unsigned int>();
      p = std::unique_ptr<rl::Policy>(new rl::EpsilonGreedy(n_actions, eps, eps_floor, eps_T, seed));
    } else if (policy_type == "boltzmann") {
      float tau = c["policy"]["tau_init"].as<float>(), tau_floor = c["policy"]["tau_floor"].as<float>();
      unsigned int tau_T = c["policy"]["tau_T"].as<unsigned int>();
      p = std::unique_ptr<rl::Policy>(new rl::Boltzmann(n_actions, tau, tau_floor, tau_T, seed));
    } else
      throw runtime_error("Please specify a valid policy!");

    // main.cpp:167-189 (the -a override of main.cpp:345 is --algo here)
    string algorithm = algo.empty() ? c["learning"]["algorithm"].as<string>("") : algo;
    AgentView av;
    if (algorithm == "q_learn") av = make_agent<rl::QLearn>(std::move(p), c);
    else if (algorithm == "double_q_learn") av = make_agent<rl::DoubleQLearn>(std::move(p), c);
    else if (algorithm == "sarsa") av = make_agent<rl::SARSA>(std::move(p), c);
    else if (algorithm == "r_learn") av = make_agent<rl::RLearn>(std::move(p), c);
    else if (algorithm == "online_r_learn") av = make_agent<rl::OnlineRLearn>(std::move(p), c);
    else if (algorithm == "double_r_learn") av = make_agent<rl::DoubleRLearn>(std::move(p), c);
    else throw runtime_error("Please specify a valid learning algorithm!");
    rl::Agent* m = av.agent;

    EnvSpy env(c);

    // experiment::serial::Runner::Runner (serial.cpp:9-16): ONE pair of States for every episode of this driver, exactly
    // like `experiment::serial::Learner experiment(c, env)` of main.cpp:47-48 lives across the while(true) of train()
    rl::State state1(c), state2(c);
    rl::State* state = &state1;
    rl::State* last_state = &state2;

    FILE* fd = dump.empty() ? nullptr : fopen(dump.c_str(), "wb");
    if (!dump.empty() && !fd) throw runtime_error("cannot open dump file " + dump);

    auto t_start = chrono::steady_clock::now();

    long steps = 0;
    double sum_reward = 0.0;
    long hist[16] = {0};
    bool terminal = false;
    for (int episode = 0; episode < n_episodes; ++episode) {
      env.LoadData(symbol, md, tas);  // main.cpp:55 (the same day again: what rlm_reset's rewound stream stands for)
      // Learner::RunEpisode serial.cpp:72-76, Runner::RunEpisode serial.cpp:18-34
      env.resetStats();
      if (!env.Initialise()) throw runtime_error("Initialise() failed: not enough data");
      last_state->newState(env);

      long ep_steps = 0;
      terminal = false;
      while (true) {
        // Learner::_step, serial.cpp:53-70
        swap(state, last_state);
        if (env.isTerminal()) { terminal = true; break; }
        int action = m->action(*last_state);
        if (!env.performAction(action)) { terminal = true; break; }
        state->newState(env);
        double reward = env.getReward();
        m->HandleTransition(*last_state, action, reward, *state);

        sum_reward += reward;
        if (action >= 0 && action < 16) hist[action]++;

        if (fd) {
          rlm_step_record r;
          memset(&r, 0, sizeof(r));
          r.step = (int32_t)ep_steps;
          r.action = action;
          env.fill(r);
          r.reward = reward;
          auto& sv = state->toVector();
          r.n_state = (int32_t)sv.size();
          for (size_t i = 0; i < sv.size() && i < RLM_N_STATE_MAX; ++i) r.state[i] = sv[i];
          r.delta = av.delta();
          rl::Traces* tr = av.traces();
          double* th = av.theta();
          r.n_traces = tr->n_nonzero_traces;
          uint64_t h = 0;
          for (int k = 0; k < tr->n_nonzero_traces; ++k) {
            int f = tr->nonzero_traces[k];
            h += rlm_trace_mix((uint32_t)f, bits_of(tr->eligibility[f]), bits_of(th[f]));
          }
          r.trace_hash = h;
          fwrite(&r, sizeof(r), 1, fd);
        }

        ++steps;
        ++ep_steps;
        if (max_steps >= 0 && steps >= max_steps) break;
      }
      if (terminal) {
        env.ClearInventory();              // serial.cpp:31
        m->HandleTerminal(episode);        // serial.cpp:79: HandleTerminal(_episode_counter++)
      }
      if (max_steps >= 0 && steps >= max_steps) break;
    }
    auto t_end = chrono::steady_clock::now();
    double secs = chrono::duration<double>(t_end - t_start).count();
    if (fd) fclose(fd);

    // Evaluation phase, main.cpp:216-244: greedy agent, ONE new Intraday object for every test day; per day LoadData,
    // a new Backtester (Runner::RunEpisode serial.cpp:18-34 + Backtester::_step serial.cpp:121-137).  The env object
    // keeps what Initialise does not clear (window sums, position, experiment statistics) from one day to the next.
    struct DaySummary { long steps; rlm_step_record last; };
    vector<DaySummary> days;
    if (n_test > 0) {
      m->GoGreedy();
      EnvSpy env2(c);
      for (size_t day = 0; day < n_test; ++day) {
        env2.LoadData(test_symbol.empty() ? symbol : test_symbol[day], test_md[day], test_tas[day]);
        if (!log_dir.empty()) {
          // Backtester::Backtester, serial.cpp:97-119 (pattern "%v": main.cpp:254).  From the second day on the
          // loggers exist: rotating_logger_mt throws and the ctor swallows it, so the files keep one header.
          spdlog::set_pattern("%v");
          try {
            spdlog::rotating_logger_mt("profit_log", log_dir + "/profit_log.csv", 1u << 30, 1);
            spdlog::get("profit_log")->info("episode,step,action,position,midprice,spread,quoted_ask,quoted_bid,ask_level,bid_level,pnl_step,bandh_step");
          } catch (const std::exception&) {}
          try {
            spdlog::rotating_logger_mt("trade_log", log_dir + "/order_log.csv", 1u << 30, 1);
            spdlog::get("trade_log")->info("episode,step,position,side,action,price,size,pnl");
          } catch (const std::exception&) {}
          env2.start_logging();
        }
        rl::State b1(c), b2(c);  // Runner ctor, serial.cpp:9-16
        rl::State* bstate = &b1;
        rl::State* blast = &b2;
        FILE* ft2 = dump_test.empty() ? nullptr : fopen(dump_test[day].c_str(), "wb");
        if (!dump_test.empty() && !ft2) throw runtime_error("cannot open dump file " + dump_test[day]);
        if (!env2.Initialise()) throw runtime_error("Initialise() failed on the test data");
        blast->newState(env2);
        long test_steps = 0;
        while (true) {
          if (env2.isTerminal()) break;
          bstate->newState(env2);
          int action = m->action(*bstate);
          if (!env2.performAction(action)) break;
          rlm_step_record r;
          memset(&r, 0, sizeof(r));
          r.step = (int32_t)test_steps;
          r.action = action;
          env2.fill(r);
          r.reward = env2.getReward();
          auto& sv = bstate->toVector();
          r.n_state = (int32_t)sv.size();
          for (size_t i = 0; i < sv.size() && i < RLM_N_STATE_MAX; ++i) r.state[i] = sv[i];
          r.n_traces = av.traces()->n_nonzero_traces;
          if (ft2) fwrite(&r, sizeof(r), 1, ft2);
          ++test_steps;
        }
        env2.ClearInventory();
        DaySummary ds;
        ds.steps = test_steps;
        memset(&ds.last, 0, sizeof(ds.last));
        env2.fill(ds.last);
        days.push_back(ds);
        if (ft2) fclose(ft2);
      }
      if (!log_dir.empty()) {
        spdlog::get("profit_log")->flush();
        spdlog::get("trade_log")->flush();
        env2.writeStats(log_dir + "/test_stats.csv");  // main.cpp:244
      }
    }
    const long test_steps = days.empty() ? 0 : days.back().steps;
    rlm_step_record test_last;
    memset(&test_last, 0, sizeof(test_last));
    if (!days.empty()) test_last = days.back().last;

    if (!theta_out.empty()) {
      // sparse dump: (int64 index, double value) for every nonzero weight of table A
      FILE* ft = fopen(theta_out.c_str(), "wb");
      if (!ft) throw runtime_error("cannot open theta file " + theta_out);
      double* th = av.theta();
      for (long i = 0; i < av.memory_size; ++i) {
        if (th[i] != 0.0) {
          int64_t idx = i;
          fwrite(&idx, 8, 1, ft);
          fwrite(&th[i], 8, 1, ft);
        }
      }
      fclose(ft);
    }

    if (!quiet) {
      rlm_step_record r;
      memset(&r, 0, sizeof(r));
      env.fill(r);
      printf("{\"steps\": %ld, \"terminal\": %d, \"seconds\": %.6f, \"steps_per_s\": %.1f, "
             "\"time_ms\": %d, \"position\": %lld, \"ep_pnl\": %.10g, \"ep_reward\": %.10g, "
             "\"sum_reward\": %.10g, \"ask_tx\": %d, \"bid_tx\": %d, \"actions\": [",
             steps, terminal ? 1 : 0, secs, steps / std::max(secs, 1e-12), r.time_ms, (long long)r.position,
             r.ep_pnl, r.ep_reward, sum_reward, r.ask_transactions, r.bid_transactions);
      for (unsigned a = 0; a < n_actions && a < 16; ++a) printf("%s%ld", a ? ", " : "", hist[a]);
      // one summary per test day after a multi-day evaluation; the test_* fields before it are the last day's
      auto day_json = [](long n, const rlm_step_record& l) {
        char buf[512];
        snprintf(buf, sizeof(buf), "\"test_steps\": %ld, \"test_position\": %lld, \"test_ep_pnl\": %.17g, \"test_ep_reward\": %.17g, "
                 "\"test_ask_tx\": %d, \"test_bid_tx\": %d, \"test_market_buys\": %d, \"test_market_sells\": %d",
                 n, (long long)l.position, l.ep_pnl, l.ep_reward, l.ask_transactions, l.bid_transactions, l.market_buys, l.market_sells);
        return string(buf);
      };
      printf("], %s", day_json(test_steps, test_last).c_str());
      if (days.size() > 1) {
        printf(", \"test_days\": [");
        for (size_t d = 0; d < days.size(); ++d) printf("%s{%s}", d ? ", " : "", day_json(days[d].steps, days[d].last).c_str());
        printf("]");
      }
      printf("}\n");
    }
    delete m;
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ref_driver: exception: %s\n", e.what());
    return 1;
  }
}
