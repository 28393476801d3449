// rlm_facade.hpp -- the reference's class surface for this hot path, batch = 1, over the C ABI of rlm.h.
//
// The reference driver names three things (src/main.cpp:45-80,168-189): an environment
// (environment::Intraday<>, include/environment/base.h:102-136), an agent (rl::Agent and its subclasses,
// include/rl/agent.h:15-67) and an experiment loop (experiment::serial::Learner, src/experiment/serial.cpp:18-95).
// These header-only classes give a C++ host the same three objects with the same member names and the same call
// order, so that the loop of serial.cpp reads unchanged (examples/serial_driver.cpp is that loop) while every call
// lands in librlm.so.  What differs, and why: env and agent of one trajectory share ONE library handle (the fused
// kernels own both), so they are built from a common `rlm::Session`; the two rl::State objects of Runner live inside
// the handle (SURVEY.md 8b), so newState()/HandleTransition() take no State arguments.
#ifndef RLM_FACADE_HPP
#define RLM_FACADE_HPP

#include <stdexcept>
#include <string>
#include <vector>

extern "C" {
#include "rlm.h"
}

namespace rlm {

inline void check(int rc) {  // the reference throws std::runtime_error / std::invalid_argument (SURVEY.md 8b "Error convention")
  if (rc == RLM_OK) return;
  const std::string msg = rlm_last_error();
  if (rc == RLM_ERR_INVALID_ARGUMENT) throw std::invalid_argument(msg);
  throw std::runtime_error(msg);
}

// one env + one agent + the Runner's States: a library handle with n_envs = 1.  source: RLM_SOURCE_GENERATOR (the synthetic
// day of cfg.flow) or RLM_SOURCE_TAPE (CSV pairs through Intraday::LoadData(symbol, md, tas))
class Session {
 public:
  explicit Session(const rlm_config& cfg, int source = RLM_SOURCE_GENERATOR) : cfg_(cfg) {
    cfg_.n_envs = 1;
    cfg_.source = source;
    check(rlm_create(&cfg_, &h_));
  }
  ~Session() { if (h_) rlm_destroy(h_); }
  Session(const Session&) = delete;
  Session& operator=(const Session&) = delete;
  rlm_handle handle() const { return h_; }
  const rlm_config& config() const { return cfg_; }

 private:
  rlm_config cfg_;
  rlm_handle h_ = nullptr;
};

namespace environment {

// environment::Base / Intraday<> (include/environment/base.h:102-136, include/environment/intraday.h:26-104)
class Intraday {
 public:
  explicit Intraday(Session& s) : s_(s) {}
  // Intraday::LoadData (intraday.cpp:141-150): the synthetic day is part of the config; another day replaces its flow
  // parameters on the same env objects (rlm_set_flow), and Initialise() starts it.  The env keeps what Initialise does
  // not clear, as the reference's does from one test day to the next (main.cpp:219-241).
  void LoadData(const rlm_flow_params* day = nullptr) {
    if (!day) return;
    check(rlm_set_flow(s_.handle(), day));
    started_ = true;  // (the next Initialise resets the envs onto the new day's flow)
  }
  // Intraday::LoadData(ticker, md_path, tas_path) (intraday.cpp:141-150) on a tape Session: the CSV pair is read by
  // rlm_ingest_csv and becomes a one-day library.  The venue's tick table is the config's (the reference derives it from
  // the ticker, market.cpp:206-245); the ticker is kept for getEpisodeId-style reporting only.
  void LoadData(const std::string& ticker, const std::string& md_path, const std::string& tas_path) {
    if (s_.config().source != RLM_SOURCE_TAPE) throw std::invalid_argument("Intraday::LoadData(ticker, md, tas) needs a Session with source RLM_SOURCE_TAPE");
    int64_t n = 0, ticks = 0;
    check(rlm_ingest_csv(md_path.c_str(), tas_path.c_str(), nullptr, 0, &n, &ticks));
    std::vector<rlm_tick_msg> msgs((size_t)(n > 0 ? n : 1));
    check(rlm_ingest_csv(md_path.c_str(), tas_path.c_str(), msgs.data(), n, &n, &ticks));
    const int64_t offsets[2] = {0, n};
    check(rlm_load_days(s_.handle(), msgs.data(), offsets, 1));
    ticker_ = ticker;
  }
  const std::string& ticker() const { return ticker_; }
  // Intraday::Initialise (intraday.cpp:103-138): rows until the open, then until every window is full
  bool Initialise() {
    if (started_) check(rlm_reset(s_.handle()));
    started_ = true;
    unsigned char term = 0;
    check(rlm_env_step(s_.handle(), nullptr, &reward_, &term));
    check(rlm_agent_update(s_.handle(), nullptr));  // Q(first from-state, .): nothing is learned here
    terminal_ = term == 1;
    return term == 0;                                // (2: the tape day ended before the env was ready, NextState false)
  }
  // Base::performAction (base.cpp:254-337): DoAction, then NextState until the midprice has moved.  false: the tape day
  // ran out inside the step (NextState returned false at the end of the data, base.cpp:289)
  bool performAction(int action) {
    int32_t a = action;
    unsigned char term = 0;
    check(rlm_env_step(s_.handle(), &a, &reward_, &term));
    terminal_ = term == 1;
    return term != 2;
  }
  double getReward() const { return reward_; }            // Base::getReward (base.cpp:166-237) of the last step
  bool isTerminal() const { return terminal_; }           // Intraday::isTerminal (intraday.cpp:152-157)
  void getState(std::vector<float>& out) const {          // Intraday::getState (intraday.cpp:411-416)
    out.resize(s_.config().n_state_vars);
    check(rlm_get_state(s_.handle(), out.data()));
  }
  void ClearInventory() {}                                // (done by the library when the episode ends, serial.cpp:31)
  double getEpisodeReward() const { return stats().episode_reward; }  // base.cpp:244-252
  double getEpisodePnL() const { return stats().episode_pnl; }
  int getTotalTransactions() const { const rlm_env_stats s = stats(); return s.ask_transactions + s.bid_transactions; }
  rlm_env_stats stats() const { rlm_env_stats s; check(rlm_get_stats(s_.handle(), 0, 1, &s)); return s; }

 private:
  Session& s_;
  double reward_ = 0.0;
  bool terminal_ = false, started_ = false;
  std::string ticker_;
};

}  // namespace environment

namespace rl {

// rl::Agent (include/rl/agent.h:15-67); the concrete algorithm and policy are rlm_config::algorithm / policy_type
class Agent {
 public:
  explicit Agent(Session& s) : s_(s) {}
  int action() {                                           // Agent::action(State&) (agent.cpp:60-74)
    int32_t a = -1;
    check(rlm_act(s_.handle(), &a));
    return a;
  }
  double HandleTransition() {                              // Agent::HandleTransition (agent.cpp:86-101); returns delta
    double d = 0.0;
    check(rlm_agent_update(s_.handle(), &d));
    return d;
  }
  void HandleTerminal(int episode) { check(rlm_handle_terminal(s_.handle(), episode)); }  // agent.cpp:103-109
  void GoGreedy() { check(rlm_go_greedy(s_.handle())); }                                     // agent.cpp:76-79
  void write_theta(std::vector<double>& out) const {      // Agent::write_theta (agent.cpp:176-181), to memory
    out.resize((size_t)s_.config().memory_size);
    check(rlm_read_theta(s_.handle(), 0, 0, out.data(), (int64_t)out.size()));
  }

 private:
  Session& s_;
};

}  // namespace rl

namespace experiment {
namespace serial {

// experiment::serial::Runner / Learner (src/experiment/serial.cpp:18-95), statement for statement
class Learner {
 public:
  Learner(environment::Intraday& env) : environment(env) {}
  bool RunEpisode(rl::Agent* m) {
    _step_counter = 0;
    if (!environment.Initialise()) return false;           // Runner::RunEpisode, serial.cpp:20-22
    bool is_terminal;
    do { is_terminal = _step(m); } while (!is_terminal);   // :27-29
    environment.ClearInventory();                          // :31
    m->HandleTerminal(_episode_counter++);                 // Learner::RunEpisode, :79
    return true;
  }
  long steps() const { return _step_counter; }

 private:
  bool _step(rl::Agent* m) {                               // Learner::_step, serial.cpp:53-70
    int action = m->action();                              // (isTerminal is folded into action(): -1 = the episode is over)
    if (action < 0) return true;
    if (!environment.performAction(action)) return true;
    m->HandleTransition();                                 // state->newState(environment) + HandleTransition
    _step_counter++;
    return false;
  }
  environment::Intraday& environment;
  long _step_counter = 0;
  int _episode_counter = 0;
};

}  // namespace serial
}  // namespace experiment
}  // namespace rlm

#endif  // RLM_FACADE_HPP
