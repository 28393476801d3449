// serial_driver.cpp -- the reference's driver (src/main.cpp:45-80,216-244 + src/experiment/serial.cpp) on the GPU library
// through the class surface of include/rlm_facade.hpp: one env, one agent, N training episodes, then optionally the test
// phase.
//
//   g++ -std=c++17 -Iinclude examples/serial_driver.cpp -Lrl_markets_b200 -lrlm -Wl,-rpath,$PWD/rl_markets_b200 -o examples/serial_driver
//   examples/serial_driver [--episodes N] [--algo q_learn|sarsa|double_q_learn] [--memory-size M] [--open-ticks T] [--theta out.bin]
//                          [--flow-seed S] [--eps-T T] [--train-log-dir D]
//                          [--md depth.csv --tas trades.csv [--symbol AAL.L] [--seed S] [--env E]]
//                          [--test-seed S]... [--test-md depth.csv --test-tas trades.csv]...
//
// Without --md/--tas every episode replays the synthetic day of the config (a short day of --open-ticks rows).  With them
// every episode is Intraday::LoadData(symbol, md, tas) + RunEpisode on that CSV pair (tape source), like src/main.cpp's
// loop over its file sample; --seed sets debug.random_seed and --env the env index the seeds are derived from.
// Prints one JSON line per episode (steps, reward, pnl) and optionally dumps theta; tests/test_gpu_facade.py and
// tests/test_gpu_tape.py check it against the fused rlm_run_ticks path.  --flow-seed sets the synthetic day's flow seed
// (default 41), --eps-T policy.eps_T.  --train-log-dir D writes D/model_log.csv and D/training_log.csv as main.cpp does
// into its output_dir with logging.log_learning on (tests/test_gpu_facade_training_logs.py).
//
// Test days (main.cpp:216-244): GoGreedy, ONE new Intraday, then per test day LoadData + a Backtester's RunEpisode on that
// object.  --test-seed S (repeatable) is a synthetic day of flow seed S laid out like the training day; --test-md/--test-tas
// (repeatable, paired in order) a CSV pair, on a Session that trains on CSV pairs.  One JSON line per test day with
// main.cpp:229-237's numbers: steps, reward, mean_reward (getMeanEpisodeReward), pnl, transactions.
#include <cstdio>
#include <cstdlib>
#include <cstring>
#include <string>
#include <vector>

#include "rlm_facade.hpp"

int main(int argc, char** argv) {
  int episodes = 2, algo = RLM_ALGO_Q_LEARN, open_ticks = 400;
  long long memory_size = 8192, seed = -1, env_index = 0;
  long long flow_seed = 41, eps_T = -1;
  std::string theta_out, md, tas, symbol = "AAL.L", log_dir;
  std::vector<long long> test_seeds;
  std::vector<std::string> test_md, test_tas;
  for (int i = 1; i < argc; ++i) {
    std::string a = argv[i];
    auto next = [&]() { return std::string(i + 1 < argc ? argv[++i] : ""); };
    if (a == "--episodes") episodes = atoi(next().c_str());
    else if (a == "--memory-size") memory_size = atoll(next().c_str());
    else if (a == "--open-ticks") open_ticks = atoi(next().c_str());
    else if (a == "--theta") theta_out = next();
    else if (a == "--md") md = next();
    else if (a == "--tas") tas = next();
    else if (a == "--symbol") symbol = next();
    else if (a == "--seed") seed = atoll(next().c_str());
    else if (a == "--env") env_index = atoll(next().c_str());
    else if (a == "--flow-seed") flow_seed = atoll(next().c_str());
    else if (a == "--eps-T") eps_T = atoll(next().c_str());
    else if (a == "--train-log-dir") log_dir = next();
    else if (a == "--test-seed") test_seeds.push_back(atoll(next().c_str()));
    else if (a == "--test-md") test_md.push_back(next());
    else if (a == "--test-tas") test_tas.push_back(next());
    else if (a == "--algo") { std::string v = next(); algo = v == "sarsa" ? RLM_ALGO_SARSA : (v == "double_q_learn" ? RLM_ALGO_DOUBLE_Q_LEARN : RLM_ALGO_Q_LEARN); }
  }
  try {
    rlm_config c;
    rlm::check(rlm_config_default(&c));      // config/example.yaml
    c.algorithm = algo;
    c.memory_size = memory_size;
    c.flow.seed = (uint64_t)flow_seed;
    if (eps_T > 0) c.eps_T = (uint32_t)eps_T;
    c.flow.t0_ms = (int32_t)(c.close_ms - 30 * 60000 - (long long)open_ticks * c.flow.dt_ms);  // a short day: it closes after open_ticks rows
    if (seed >= 0) c.random_seed = (uint32_t)seed;
    c.env_index0 = env_index;
    const bool csv = !md.empty() || !tas.empty();
    if (csv && (md.empty() || tas.empty())) throw std::invalid_argument("--md and --tas go together");
    if (test_md.size() != test_tas.size()) throw std::invalid_argument("--test-md and --test-tas go together");
    if (csv ? !test_seeds.empty() : !test_md.empty())
      throw std::invalid_argument(csv ? "a Session that trains on CSV pairs tests on CSV pairs (--test-md/--test-tas)"
                                      : "a Session that trains on synthetic days tests on synthetic days (--test-seed)");
    rlm::Session session(c, csv ? RLM_SOURCE_TAPE : RLM_SOURCE_GENERATOR);
    rlm::environment::Intraday env(session);
    rlm::rl::Agent m(session, log_dir);                      // (log_dir empty: no logs, as with log_learning off)
    rlm::experiment::serial::Learner experiment(env, log_dir);
    for (int episode = 1; episode <= episodes; ++episode) {   // train(), main.cpp:53-78
      if (csv) env.LoadData(symbol, md, tas);
      else env.LoadData();
      if (experiment.RunEpisode(&m))
        printf("{\"episode\": %d, \"steps\": %ld, \"reward\": %.17g, \"pnl\": %.17g, \"transactions\": %d}\n", episode, experiment.steps(),
               env.getEpisodeReward(), env.getEpisodePnL(), env.getTotalTransactions());
    }
    if (!theta_out.empty()) {
      std::vector<double> th;
      m.write_theta(th);
      FILE* f = fopen(theta_out.c_str(), "wb");
      if (!f) throw std::runtime_error("cannot open " + theta_out);
      fwrite(th.data(), 8, th.size(), f);
      fclose(f);
    }
    const size_t n_test = csv ? test_md.size() : test_seeds.size();
    if (n_test > 0) {                                         // main.cpp:216-244
      m.GoGreedy();
      rlm::environment::Intraday test_env(session);
      for (size_t i = 0; i < n_test; ++i) {
        rlm_flow_params day = c.flow;
        if (csv) test_env.LoadData(symbol, test_md[i], test_tas[i]);
        else { day.seed = (uint64_t)test_seeds[i]; test_env.LoadData(&day); }
        rlm::experiment::serial::Backtester bt(test_env);
        if (bt.RunEpisode(&m)) {
          const rlm_env_stats s = test_env.stats();
          printf("{\"test_day\": %zu, \"steps\": %d, \"reward\": %.17g, \"mean_reward\": %.17g, \"pnl\": %.17g, \"transactions\": %d}\n",
                 i + 1, s.steps, test_env.getEpisodeReward(), test_env.getMeanEpisodeReward(), test_env.getEpisodePnL(),
                 test_env.getTotalTransactions());
        }
      }
    }
  } catch (const std::exception& e) {
    fprintf(stderr, "serial_driver: %s\n", e.what());
    return 1;
  }
  return 0;
}
