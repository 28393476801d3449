// ref_train_logs -- TEST INFRASTRUCTURE ONLY (never linked into the product).
//
// Trains the UNMODIFIED reference for N episodes with logging.log_learning on, so that the reference itself writes
// model_log.csv (Agent's ctor registers the logger, agent.cpp:52-59; HandleTransition logs, agent.cpp:86-101) and
// training_log.csv into the yaml's output_dir.  The episode loop is src/main.cpp's train() for one thread
// (main.cpp:45-60): LoadData of the episode's day, then experiment::serial::Learner::RunEpisode.  serial.cpp itself does
// not compile against the spdlog at hand (its fmt cannot format the std::atomic_int episode counter of serial.cpp:82),
// so Learner's ctor (serial.cpp:40-50), Runner::RunEpisode (:18-34), Learner::_step (:53-70) and Learner::RunEpisode
// (:72-94) are restated below line for line, the training_log call with the same format string and arguments.  Every
// object they call -- Intraday, the agents and their HandleTransition / HandleTerminal, the policies, State -- is the
// reference's own object code.  Policy and agent are built as main.cpp:137-189 builds them; the loggers use the
// pattern "%v" of main.cpp:254.
//
//   ref_train_logs --config cfg.yaml --episodes N (--symbol S --md md.csv --tas tas.csv)...
// Episode e runs on day e % n_days.  Prints one JSON line: the day and episode id of every episode.
#include <chrono>
#include <cstdio>
#include <cstdlib>
#include <memory>
#include <string>
#include <vector>

#include <spdlog/spdlog.h>

#include "environment/intraday.h"
#include "rl/state.h"
#include "rl/agent.h"
#include "rl/policy.h"

using namespace std;

int main(int argc, char** argv) {
  string cfg;
  int n_episodes = 1;
  vector<string> sym, md, tas;
  for (int i = 1; i + 1 < argc; i += 2) {
    const string a = argv[i], v = argv[i + 1];
    if (a == "--config") cfg = v;
    else if (a == "--episodes") n_episodes = atoi(v.c_str());
    else if (a == "--symbol") sym.push_back(v);
    else if (a == "--md") md.push_back(v);
    else if (a == "--tas") tas.push_back(v);
    else { fprintf(stderr, "ref_train_logs: unknown argument %s\n", a.c_str()); return 2; }
  }
  if (cfg.empty() || md.empty() || md.size() != tas.size() || md.size() != sym.size()) {
    fprintf(stderr, "usage: ref_train_logs --config cfg.yaml --episodes N (--symbol S --md md.csv --tas tas.csv)...\n");
    return 2;
  }
  try {
    Config c(cfg);
    spdlog::set_pattern("%v");  // main.cpp:254

    unsigned seed = c["debug"]["random_seed"].as<unsigned>(chrono::system_clock::now().time_since_epoch().count());
    srand(seed);  // main.cpp:84-88

    unsigned int n_actions = c["learning"]["n_actions"].as<unsigned int>();
    std::unique_ptr<rl::Policy> p;  // main.cpp:137-165
    const string policy_type = c["policy"]["type"].as<string>("");
    if (policy_type == "greedy")
      p = std::unique_ptr<rl::Policy>(new rl::Greedy(n_actions, seed));
    else if (policy_type == "random")
      p = std::unique_ptr<rl::Policy>(new rl::Random(n_actions, seed));
    else if (policy_type == "epsilon_greedy")
      p = std::unique_ptr<rl::Policy>(new rl::EpsilonGreedy(n_actions, c["policy"]["eps_init"].as<float>(), c["policy"]["eps_floor"].as<float>(),
                                                            c["policy"]["eps_T"].as<unsigned int>(), seed));
    else if (policy_type == "boltzmann")
      p = std::unique_ptr<rl::Policy>(new rl::Boltzmann(n_actions, c["policy"]["tau_init"].as<float>(), c["policy"]["tau_floor"].as<float>(),
                                                        c["policy"]["tau_T"].as<unsigned int>(), seed));
    else
      throw runtime_error("Please specify a valid policy!");

    const string algorithm = c["learning"]["algorithm"].as<string>("");  // main.cpp:167-189
    rl::Agent* m = nullptr;
    if (algorithm == "q_learn") m = new rl::QLearn(std::move(p), c);
    else if (algorithm == "double_q_learn") m = new rl::DoubleQLearn(std::move(p), c);
    else if (algorithm == "sarsa") m = new rl::SARSA(std::move(p), c);
    else if (algorithm == "r_learn") m = new rl::RLearn(std::move(p), c);
    else if (algorithm == "online_r_learn") m = new rl::OnlineRLearn(std::move(p), c);
    else if (algorithm == "double_r_learn") m = new rl::DoubleRLearn(std::move(p), c);
    else throw runtime_error("Please specify a valid learning algorithm!");

    environment::Intraday<> env(c);  // main.cpp:47-48

    // Learner::Learner (serial.cpp:40-50); Runner::Runner (serial.cpp:9-16)
    auto training_log = spdlog::rotating_logger_mt("training_log", c["output_dir"].as<string>() + "training_log.csv",
                                                   c["logging"]["max_size"].as<size_t>(), 1);
    training_log->info("episode,episode_id,reward,pnl,n_steps,epsilon");
    rl::State state1(c), state2(c);
    rl::State* state = &state1;
    rl::State* last_state = &state2;
    int episode_counter = 0;  // Learner::_episode_counter

    printf("{\"episodes\": [");
    for (int e = 0; e < n_episodes; ++e) {
      const size_t d = (size_t)e % md.size();
      env.LoadData(sym[d], md[d], tas[d]);
      // Learner::RunEpisode (serial.cpp:72-94)
      unsigned long step_counter = 0;
      env.resetStats();
      // Runner::RunEpisode (serial.cpp:18-34)
      if (!env.Initialise()) throw runtime_error("RunEpisode: Initialise() failed");
      last_state->newState(env);
      while (true) {
        // Learner::_step (serial.cpp:53-70)
        swap(state, last_state);
        if (env.isTerminal()) break;
        int action = m->action(*last_state);
        if (!env.performAction(action)) break;
        state->newState(env);
        m->HandleTransition(*last_state, action, env.getReward(), *state);
        step_counter++;
      }
      env.ClearInventory();
      m->HandleTerminal(episode_counter++);
      training_log->info("{},{},{},{},{},{}", episode_counter, env.getEpisodeId(), env.getEpisodeReward(), env.getEpisodePnL(),
                         step_counter, m->policy->descr());
      printf("%s{\"day\": %zu, \"episode_id\": \"%s\"}", e ? ", " : "", d, env.getEpisodeId().c_str());
    }
    printf("]}\n");
    spdlog::get("model_log")->flush();
    spdlog::get("training_log")->flush();
    delete m;
    return 0;
  } catch (const std::exception& e) {
    fprintf(stderr, "ref_train_logs: exception: %s\n", e.what());
    return 1;
  }
}
