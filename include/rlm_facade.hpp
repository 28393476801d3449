// rlm_facade.hpp -- the reference's class surface for this hot path, batch = 1, over the C ABI of rlm.h.
//
// The reference driver names three things (src/main.cpp:45-80,168-189): an environment
// (environment::Intraday<>, include/environment/base.h:102-136), an agent (rl::Agent and its subclasses,
// include/rl/agent.h:15-67) and an experiment loop (experiment::serial::Learner for training and Backtester for the test
// phase, src/experiment/serial.cpp:18-137).
// These header-only classes give a C++ host the same three objects with the same member names and the same call
// order, so that the loop of serial.cpp reads unchanged (examples/serial_driver.cpp is that loop) while every call
// lands in librlm.so.  What differs, and why: env and agent of one trajectory share ONE library handle (the fused
// kernels own both), so they are built from a common `rlm::Session`; the two rl::State objects of Runner live inside
// the handle (SURVEY.md 8b), so newState()/HandleTransition() take no State arguments.
#ifndef RLM_FACADE_HPP
#define RLM_FACADE_HPP

#include <charconv>
#include <cmath>
#include <cstdio>
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

// A number as the training logs print it: fmt's "{}" through spdlog's "%v" pattern, i.e. the shortest string that reads
// back to the same double, integral values below 1e15 without a decimal point, exponents as e-05 / e+16 -- the rendering
// of rl_markets_b200/backtest.py's _num, which the reference's files are checked against.
inline std::string log_num(double x) {
  if (std::isnan(x)) return "nan";
  if (std::isinf(x)) return x < 0 ? "-inf" : "inf";
  if (x == std::trunc(x) && std::fabs(x) < 1e15) return std::to_string((long long)x);
  char buf[64];
  const auto r = std::to_chars(buf, buf + sizeof(buf), x, std::chars_format::scientific);  // shortest d.ddde+XX
  const std::string sci(buf, r.ptr);
  const size_t e = sci.find('e');
  const int ex = std::stoi(sci.substr(e + 1));
  const bool neg = sci[0] == '-';
  std::string digits;
  for (size_t i = neg ? 1 : 0; i < e; ++i) if (sci[i] != '.') digits += sci[i];
  std::string out = neg ? "-" : "";
  if (ex < -4 || ex >= 16) {  // repr's scientific form
    out += digits.substr(0, 1);
    if (digits.size() > 1) out += "." + digits.substr(1);
    char eb[16];
    snprintf(eb, sizeof(eb), "e%c%02d", ex < 0 ? '-' : '+', ex < 0 ? -ex : ex);
    return out + eb;
  }
  if (ex < 0) return out + "0." + std::string((size_t)(-ex - 1), '0') + digits;
  if ((size_t)ex + 1 >= digits.size()) return out + digits + std::string((size_t)ex + 1 - digits.size(), '0') + ".0";
  return out + digits.substr(0, (size_t)ex + 1) + "." + digits.substr((size_t)ex + 1);
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
  // `environment::Intraday<> env(c)`: the Session's first env object is the one rlm_create built; every later one is a new
  // env object for the same agent (rlm_new_env), as main.cpp:219 builds one for the test phase
  void attach_env() {
    if (n_env_objects_++ > 0) check(rlm_new_env(h_, nullptr));
  }

 private:
  rlm_config cfg_;
  rlm_handle h_ = nullptr;
  int n_env_objects_ = 0;
};

namespace environment {

// environment::Base / Intraday<> (include/environment/base.h:102-136, include/environment/intraday.h:26-104)
class Intraday {
 public:
  // A second Intraday on a Session is a new env object (Session::attach_env): the env state starts from scratch and the
  // agent keeps theta.  Only the newest object of a Session is meant to be driven, as main.cpp drives the test env only.
  explicit Intraday(Session& s) : s_(s) { s_.attach_env(); }
  // Intraday::LoadData (intraday.cpp:141-150): the synthetic day is part of the config; another day replaces its flow
  // parameters on the same env objects (rlm_set_flow), and Initialise() starts it.  The env keeps what Initialise does
  // not clear, as the reference's does from one test day to the next (main.cpp:219-241).
  void LoadData(const rlm_flow_params* day = nullptr) {
    if (!day) return;
    check(rlm_set_flow(s_.handle(), day));
    date_ = day->date;
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
    date_ = n > 0 ? msgs[0].date : 0;
  }
  const std::string& ticker() const { return ticker_; }
  // Intraday::getEpisodeId (intraday.cpp:160): to_string(init_date), the date of the day the episode runs on
  std::string getEpisodeId() const { return std::to_string(date_); }
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
  double getMeanEpisodeReward() const { const rlm_env_stats s = stats(); return s.episode_reward / s.total_ticks; }  // base.cpp:249-252
  double getEpisodePnL() const { return stats().episode_pnl; }
  int getTotalTransactions() const { const rlm_env_stats s = stats(); return s.ask_transactions + s.bid_transactions; }
  rlm_env_stats stats() const { rlm_env_stats s; check(rlm_get_stats(s_.handle(), 0, 1, &s)); return s; }
  Session& session() const { return s_; }

 private:
  Session& s_;
  double reward_ = 0.0;
  bool terminal_ = false, started_ = false;
  std::string ticker_;
  int date_ = s_.config().flow.date;  // (a generator Session's day; LoadData replaces it)
};

}  // namespace environment

namespace rl {

// rl::Agent (include/rl/agent.h:15-67); the concrete algorithm and policy are rlm_config::algorithm / policy_type
class Agent {
 public:
  explicit Agent(Session& s) : s_(s) {}
  // Agent::Agent with logging.log_learning on (agent.cpp:52-59): `output_dir` + "model_log.csv" receives _agg_delta / 1000
  // on every 1000th update (agent.cpp:86-101).  The values are accumulated on the device (rlm_set_model_log) and written
  // out by FlushModelLog, which Learner::RunEpisode calls after every episode.  Build the Agent on a fresh Session for a
  // file equal to the reference's.
  Agent(Session& s, const std::string& output_dir) : s_(s) {
    if (output_dir.empty()) return;
    check(rlm_set_model_log(s_.handle(), kModelLogCap));
    model_log_ = output_dir + "/model_log.csv";
    FILE* f = fopen(model_log_.c_str(), "w");
    if (!f) throw std::runtime_error("cannot open " + model_log_);
    fclose(f);
  }
  void FlushModelLog() {
    if (model_log_.empty()) return;
    std::vector<double> rows(kModelLogCap);
    int32_t n = 0;
    check(rlm_read_model_log(s_.handle(), 0, 1, rows.data(), &n));
    FILE* f = fopen(model_log_.c_str(), "a");
    if (!f) throw std::runtime_error("cannot open " + model_log_);
    for (int32_t i = 0; i < n; ++i) fprintf(f, "%s\n", log_num(rows[i]).c_str());
    fclose(f);
  }
  double descr() const {                                   // Policy::descr() of the agent's policy (policy.cpp:18,77,117)
    double d = 0.0;
    check(rlm_get_policy_descr(s_.handle(), &d));
    return d;
  }
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
  // Agent::getQ (agent.cpp:117-135) and DoubleAgent::getQb (:211-230) with State::newState(vars, .) (state.cpp:45-51) folded
  // in: the State objects live in the Session, so the state comes as its variables.  getQb needs a double agent.
  double getQ(const std::vector<float>& vars, int action) const { return q(vars, action, 0); }
  double getQb(const std::vector<float>& vars, int action) const { return q(vars, action, 1); }

 private:
  double q(const std::vector<float>& vars, int action, int table) const {
    const rlm_config& c = s_.config();
    const int T = (c.algorithm == RLM_ALGO_DOUBLE_Q_LEARN || c.algorithm == RLM_ALGO_DOUBLE_R_LEARN) ? 2 : 1;
    if ((int)vars.size() != c.n_state_vars) throw std::invalid_argument("Agent::getQ: vars must hold n_state_vars values");
    if (action < 0 || action >= c.n_actions) throw std::invalid_argument("Agent::getQ: action out of range");
    if (table >= T) throw std::invalid_argument("Agent::getQb: the agent has one table (not a double agent)");
    double out[2 * RLM_MAX_ACTIONS];
    check(rlm_eval_q(s_.handle(), vars.data(), nullptr, 1, out));
    return out[table * c.n_actions + action];
  }
  static constexpr int64_t kModelLogCap = 1 << 16;  // values kept between two flushes (one per 1000 updates)
  Session& s_;
  std::string model_log_;
};

}  // namespace rl

namespace experiment {
namespace serial {

// experiment::serial::Runner / Learner (src/experiment/serial.cpp:18-95), statement for statement
class Learner {
 public:
  Learner(environment::Intraday& env) : environment(env) {}
  // Learner::Learner with logging.log_learning on (serial.cpp:40-50): `output_dir` + "training_log.csv" gets the header,
  // then one row per episode (:81-88).  Pair it with rl::Agent(session, output_dir) for the model_log.
  Learner(environment::Intraday& env, const std::string& output_dir) : environment(env) {
    if (output_dir.empty()) return;
    training_log_ = output_dir + "/training_log.csv";
    FILE* f = fopen(training_log_.c_str(), "w");
    if (!f) throw std::runtime_error("cannot open " + training_log_);
    fprintf(f, "episode,episode_id,reward,pnl,n_steps,epsilon\n");
    fclose(f);
  }
  bool RunEpisode(rl::Agent* m) {
    _step_counter = 0;
    if (!environment.Initialise()) return false;           // Runner::RunEpisode, serial.cpp:20-22
    bool is_terminal;
    do { is_terminal = _step(m); } while (!is_terminal);   // :27-29
    environment.ClearInventory();                          // :31
    m->HandleTerminal(_episode_counter++);                 // Learner::RunEpisode, :79
    if (!training_log_.empty()) {                          // :81-88
      FILE* f = fopen(training_log_.c_str(), "a");
      if (!f) throw std::runtime_error("cannot open " + training_log_);
      fprintf(f, "%d,%s,%s,%s,%ld,%s\n", _episode_counter, environment.getEpisodeId().c_str(), log_num(environment.getEpisodeReward()).c_str(),
              log_num(environment.getEpisodePnL()).c_str(), _step_counter, log_num(m->descr()).c_str());
      fclose(f);
    }
    m->FlushModelLog();
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
  std::string training_log_;
};

// experiment::serial::Backtester (src/experiment/serial.cpp:97-137): the greedy evaluation of main.cpp:216-244.  The
// constructor puts the Session in backtest mode, where it stays -- the facade's counterpart of the reference's constructor,
// which sets up the evaluation loggers (:97-122): rlm_read_records then yields the profit_log rows and rlm_get_stats the
// test_stats counters (rl_markets_b200/backtest.py renders both files).  A Learner is not meant to run after it, as in
// main.cpp, where evaluation is the last phase.  Backtester does not override RunEpisode: no HandleTerminal, no episode or
// step counter (Intraday::stats().steps counts the steps of the day).
class Backtester {
 public:
  Backtester(environment::Intraday& env) : environment(env) { check(rlm_set_mode(env.session().handle(), RLM_MODE_BACKTEST)); }
  bool RunEpisode(rl::Agent* m) {                          // Runner::RunEpisode, serial.cpp:18-34
    if (!environment.Initialise()) return false;           // :21-22, and last_state->newState(environment) (:25)
    bool is_terminal;
    do { is_terminal = _step(m); } while (!is_terminal);   // :27-29
    environment.ClearInventory();                          // :31
    return true;
  }

 private:
  bool _step(rl::Agent* m) {                               // Backtester::_step, serial.cpp:124-137
    // isTerminal is folded into action(): -1 = the episode is over.  state->newState(environment) (:129) was made by the
    // previous step's newState() below, or by Initialise for the first step.
    int action = m->action();                              // :131
    if (action < 0) return true;
    if (!environment.performAction(action)) return true;   // :133
    newState();
    return false;
  }
  // State::newState(environment) of the next _step: the greedy evaluation step (Q of the env's state; theta is only read)
  void newState() { check(rlm_agent_update(environment.session().handle(), nullptr)); }
  environment::Intraday& environment;
};

}  // namespace serial
}  // namespace experiment
}  // namespace rlm

#endif  // RLM_FACADE_HPP
