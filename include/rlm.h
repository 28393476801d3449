/* rlm.h -- C ABI of the H100-native batched limit-order-book RL environment.
 *
 * Drop-in boundary for the hot path of tspooner/rl_markets (SURVEY.md section 8b).
 * The reference has no FFI; its seam is the shared library `rl_engine`
 * (src/CMakeLists.txt:5) and the C++ classes the driver uses by name.  Each
 * entry point below names the reference interface it replaces, batched over
 * `n_envs` independent environments:
 *
 *   rlm_create            environment::Intraday<>::Intraday(Config&)      include/environment/intraday.h:58
 *                         + rl::QLearn/SARSA/DoubleQLearn(policy, Config&) include/rl/agent.h:106-131
 *                         + rl::EpsilonGreedy/Greedy/Random(...)           include/rl/policy.h:31-66
 *   rlm_load_ticks        Intraday::LoadData / data::Streamer<R>           include/data/streamer.h:16-56
 *   rlm_load_days         Intraday::LoadData for a library of days          src/environment/intraday.cpp:141-150
 *   rlm_assign_days       ... and which day each env replays                 src/main.cpp:45-80 (sample a day per episode)
 *   rlm_set_day_markets   ... under the market of the day's ticker          src/environment/intraday.cpp:141-150
 *   rlm_set_flow          ... of another synthetic day, on the same env objects src/environment/intraday.cpp:141-150
 *   rlm_reset             Intraday::Initialise                             src/environment/intraday.cpp:103-138
 *   rlm_run_ticks         experiment::serial::Learner::_step               src/experiment/serial.cpp:53-70
 *                         = Agent::action + Base::performAction + State::newState
 *                           + Agent::HandleTransition, repeated while ticks remain
 *   rlm_get_state         Intraday::getState                               src/environment/intraday.cpp:411-416
 *   rlm_get_reward        Base::getReward                                  src/environment/base.cpp:166-237
 *   rlm_handle_terminal   Agent::HandleTerminal + Policy::HandleTerminal   src/rl/agent.cpp:103-109, policy.cpp:79-82
 *   rlm_go_greedy         Agent::GoGreedy                                  src/rl/agent.cpp:76-79
 *   rlm_read_theta        Agent::write_theta (raw double[MEMORY_SIZE])     src/rl/agent.cpp:176-181
 *   rlm_get_stats         Base::getEpisodeReward/getEpisodePnL/...         src/environment/base.cpp:244-252,458-473
 *
 * Conventions: plain C types only; every call returns 0 on success or a
 * negative rlm_status; rlm_last_error() holds the message (the reference's
 * C++ exceptions never cross this boundary); handles are opaque; the library
 * owns all device memory; one host thread per handle.  There is NO CPU
 * fallback: rlm_create fails with RLM_ERR_NO_DEVICE when no CUDA device is
 * usable.
 */
#ifndef RLM_H
#define RLM_H

#include <stdint.h>
#include "rlm_flow.h"
#include "rlm_record.h"

#ifdef __cplusplus
extern "C" {
#endif

#define RLM_ABI_VERSION 4

typedef enum rlm_status {
  RLM_OK = 0,
  RLM_ERR_INVALID_ARGUMENT = -1, /* std::invalid_argument in the reference (market.cpp:58,86,112,135) */
  RLM_ERR_RUNTIME = -2,          /* std::runtime_error   (book.cpp:74-77, order.cpp:22-27, ...)       */
  RLM_ERR_NO_DEVICE = -3,        /* CUDA device / extension unavailable: there is no CPU fallback     */
  RLM_ERR_CUDA = -4,
  RLM_ERR_UNSUPPORTED = -5,      /* configuration outside the CUDA path (e.g. n_tilings != 32)        */
  RLM_ERR_END_OF_DATA = -6       /* stream exhausted (performAction returning false, base.cpp:289)    */
} rlm_status;

/* learning.algorithm (src/main.cpp:169-189) */
enum { RLM_ALGO_Q_LEARN = 0, RLM_ALGO_SARSA = 1, RLM_ALGO_DOUBLE_Q_LEARN = 2,
       RLM_ALGO_R_LEARN = 3, RLM_ALGO_ONLINE_R_LEARN = 4, RLM_ALGO_DOUBLE_R_LEARN = 5 };
/* policy.type (src/main.cpp:141-165) */
enum { RLM_POLICY_GREEDY = 0, RLM_POLICY_RANDOM = 1, RLM_POLICY_EPSILON_GREEDY = 2, RLM_POLICY_BOLTZMANN = 3 };
/* reward.measure (src/environment/base.cpp:55-75) */
enum { RLM_REWARD_NONE = 0, RLM_REWARD_PNL, RLM_REWARD_PNL_DAMPED, RLM_REWARD_SPREAD, RLM_REWARD_NORMED,
       RLM_REWARD_LOVOL, RLM_REWARD_MM_LINEAR, RLM_REWARD_MM_EXP, RLM_REWARD_MM_DIV };
/* state.variables (include/environment/intraday.h:17-23) */
enum { RLM_VAR_POS = 0, RLM_VAR_SPD, RLM_VAR_MPM, RLM_VAR_IMB, RLM_VAR_SVL, RLM_VAR_VOL, RLM_VAR_RSI,
       RLM_VAR_VWAP, RLM_VAR_A_DIST, RLM_VAR_A_QUEUE, RLM_VAR_B_DIST, RLM_VAR_B_QUEUE, RLM_VAR_LAST_ACTION };
/* market.target_price.type AS WRITTEN IN THE YAML.  The reference's selector is
 * inverted (src/environment/base.cpp:101-112): "midprice" instantiates
 * tp::MicroPrice, every other string instantiates tp::MidPrice; the string
 * "book" additionally switches the quote rule (intraday.cpp:64-71). */
enum { RLM_TP_YAML_MIDPRICE = 0, RLM_TP_YAML_MICROPRICE = 1, RLM_TP_YAML_VWAP = 2, RLM_TP_YAML_BOOK = 3 };
/* where ticks come from */
enum { RLM_SOURCE_GENERATOR = 0, /* rlm_flow.h generator evaluated inside the tick kernel                 */
       RLM_SOURCE_STREAM = 1,    /* rlm_tick_msg chunks uploaded with rlm_load_ticks (tick-major, tick-aligned) */
       RLM_SOURCE_TAPE = 2 };    /* a device-resident library of whole days (rlm_load_days), one cursor per env */

#define RLM_MAX_BANDS 32 /* power of two (band search); the longest upstream table, NasdaqNordic / Oslo, has 17 bands */
#define RLM_MAX_ACTIONS 9
#define RLM_N_TILINGS 32

typedef struct rlm_config {
  /* ---- batch / placement (new; the reference is one env per thread) ---- */
  int32_t n_envs;        /* environments owned by this handle (this GPU)                           */
  int32_t device;        /* CUDA device ordinal                                                    */
  int64_t env_index0;    /* global index of local env 0; seeds and flow streams use env_index0 + b */
  int32_t shared_policy; /* 0: one theta per env (B reference processes); 1: one theta per handle  */
  int32_t source;        /* RLM_SOURCE_*                                                           */
  /* ---- learning.* (src/rl/agent.cpp:14-50, src/rl/state.cpp:22-24) ---- */
  int64_t memory_size;
  int32_t n_tilings;
  int32_t n_actions;
  int32_t algorithm;
  int32_t random_init;
  double group_weights[3];
  double gamma, lambda, omega, alpha_start, alpha_floor, beta;
  /* ---- policy.* (src/main.cpp:137-165; eps/tau are read as float there) ---- */
  int32_t policy_type;
  float eps_init, eps_floor;
  uint32_t eps_T;
  float tau_init, tau_floor;
  uint32_t tau_T;
  int32_t spread_lookback;
  /* ---- reward.* (src/environment/base.cpp:28-32,46-47,55-75) ---- */
  int32_t reward_measure;
  float damping_factor, pos_weight, trd_weight, pnl_weight;
  int32_t pnl_lookback;
  /* ---- state.* (src/environment/intraday.cpp:52-62, base.cpp:35-50) ---- */
  int32_t n_state_vars;
  int32_t state_vars[RLM_N_STATE_MAX];
  int32_t lb_mpm, lb_vlt, lb_svl, lb_rsi, lb_vwap;
  /* ---- market.* (base.cpp:18-25,101-112) ---- */
  int64_t pos_lb, pos_ub;
  int32_t order_size;
  int32_t target_price_type; /* RLM_TP_YAML_* */
  int32_t tp_lookback;
  /* ---- venue: Market::pts_ (price -> tick size), ascending (src/market/market.cpp:11-38,206-245) ---- */
  int32_t n_bands;
  double band_px[RLM_MAX_BANDS];
  double band_ts[RLM_MAX_BANDS];
  int64_t open_ms, close_ms; /* Market::mo_, mc_ */
  /* ---- debug.random_seed (main.cpp:84-88, agent.cpp:30): env b uses random_seed + env_index0 + b ---- */
  uint32_t random_seed;
  /* ---- synthetic flow (RLM_SOURCE_GENERATOR) ---- */
  rlm_flow_params flow;
  /* ---- capacity / debugging ---- */
  int32_t trace_cap;    /* max nonzero traces kept per env; 0 = derive from gamma*lambda (traces.h:13) */
  int32_t record_envs;  /* first N envs write one rlm_step_record per learner step (parity tests)    */
  int32_t record_cap;   /* records kept per recorded env                                              */
  int32_t reserved[5];
} rlm_config;

typedef struct rlm_handle_s* rlm_handle;

/* Aggregate counters since rlm_create (all envs of the handle). */
typedef struct rlm_counters {
  int64_t ticks;        /* NextState() calls                                   */
  int64_t steps;        /* completed learner steps (Learner::_step)             */
  int64_t sum_traces;   /* sum over steps of n_nonzero_traces after the update  */
  int64_t terminal_envs;/* envs currently terminal                              */
  int64_t kernel_launches;
} rlm_counters;

/* Per-env statistics (Base getters, src/environment/base.cpp:244-252,458-473). */
typedef struct rlm_env_stats {
  double episode_reward, episode_pnl, episode_bandh;
  int64_t position;
  int32_t ask_transactions, bid_transactions, market_buys, market_sells;
  int32_t total_ticks, steps;
  int32_t terminal, phase;
} rlm_env_stats;

const char* rlm_last_error(void);
int rlm_abi_version(void);

/* config/example.yaml defaults + LSE tick table for AAL (market.cpp:216-227). */
int rlm_config_default(rlm_config* cfg);

int rlm_create(const rlm_config* cfg, rlm_handle* out);
int rlm_destroy(rlm_handle h);

/* Intraday::Initialise for every env: books/windows cleared, stream rewound. */
int rlm_reset(rlm_handle h);

/* Which experiment::serial step the handle runs (src/experiment/serial.cpp):
 *   RLM_MODE_TRAIN    Learner::_step    :53-70   act on the previous state, performAction, newState, HandleTransition
 *   RLM_MODE_BACKTEST Backtester::_step :121-137 newState, act, performAction; theta and traces are never touched.
 * In backtest mode rlm_read_records yields one row per step with every column of Intraday::LogProfit's profit_log
 * (intraday.cpp:437-451) and rlm_get_stats the counters Base::writeStats dumps (base.cpp:451-456).
 * Both modes exist for independent and for shared policies.  On a shared_policy handle in backtest mode every env reads
 * policy 0 and nothing is reduced, so each env is exactly one reference process that loaded that table: results are
 * bitwise the reference's (shared-policy TRAINING is held to 1e-5, the order of the dtheta sum being free).
 * Backtest mode runs on the tick-synchronous engine (RLM_ERR_UNSUPPORTED under RLM_ENGINE=f|p). */
enum { RLM_MODE_TRAIN = 0, RLM_MODE_BACKTEST = 1 };
int rlm_set_mode(rlm_handle h, int32_t mode);

/* `environment::Intraday<> env(c)` of src/main.cpp:219: every env object is rebuilt from scratch (window sums,
 * statistics, position, book, records) while the agents keep theta, traces, generator positions and schedules.
 * `flow` (may be NULL = keep) replaces the synthetic-flow parameters of the new object's first day (generator source;
 * a tape handle takes NULL only and changes days with rlm_assign_days).
 * main.cpp:219-241 builds that object ONCE and evaluates every test day on it, so rlm_new_env stands for the FIRST test
 * day only.  Each later day is LoadData + Initialise on the same env objects, which keep what Base::Initialise does not
 * clear (the window sums of Accumulator::clear / RollingMean, position, the experiment statistics) -- per source:
 *   generator  rlm_set_flow(h, &next_day) + rlm_reset(h)
 *   stream     rlm_reset(h) + rlm_load_ticks(h, next_day, n)
 *   tape       rlm_assign_days(h, 0, n_envs, next_days) + rlm_reset(h)
 * (A new env object per test day is what one reference process per test day computes, not main.cpp's sequence.) */
int rlm_new_env(rlm_handle h, const rlm_flow_params* flow);

/* RLM_SOURCE_GENERATOR only: Intraday::LoadData of another synthetic day (intraday.cpp:141-150) -- `flow` replaces the
 * synthetic-flow parameters and nothing else changes; follow with rlm_reset (Initialise), which starts every env on the
 * new day.  The call waits for the handle's work.  Stream handles load the next day with rlm_load_ticks, tape handles
 * with rlm_assign_days (RLM_ERR_INVALID_ARGUMENT here). */
int rlm_set_flow(rlm_handle h, const rlm_flow_params* flow);

/* RLM_SOURCE_STREAM only: append `n_ticks` messages per env, host layout msgs[t][env] (tick-major).
 * The copy is issued on the handle's copy stream; the buffer must stay valid until rlm_sync. */
int rlm_load_ticks(rlm_handle h, const rlm_tick_msg* msgs, int32_t n_ticks);

/* RLM_SOURCE_TAPE: a library of whole trading days, copied to device memory once and replayed by every run call.
 * `msgs` is the concatenation of per-day message streams exactly as rlm_ingest_csv emits them (multi-message ticks
 * included); day d is msgs[day_offsets[d] .. day_offsets[d+1]), with day_offsets[0] = 0, non-decreasing offsets and at
 * most 2^31 - 1 messages in all.  The call waits for the handle's work, replaces any previous library, assigns env b to
 * day b % n_days and rewinds every env to the start of its day.  Each env reads its own day through its own cursor, one
 * message per tick-kernel pass that ticks it (a multi-message tick takes one pass per message, as on the stream source).
 * An env that needs a message past the end of its day stops there, inside performAction, and consumes nothing more
 * until it is reassigned or rewound; this is not an error (rlm_env_step reports it with terminal_out = 2).
 * rlm_reset and rlm_new_env(h, NULL) rewind every env to the start of its assigned day.
 * Engines: tick-synchronous, round-paced and shared policy; RLM_ENGINE=F|f|p makes rlm_create fail (unsupported). */
int rlm_load_days(rlm_handle h, const rlm_tick_msg* msgs, const int64_t* day_offsets /* [n_days + 1] */, int32_t n_days);
/* Intraday::LoadData per env: env env0 + i replays day[i] from its first message (follow with rlm_reset, Initialise). */
int rlm_assign_days(rlm_handle h, int32_t env0, int32_t n, const int32_t* day);
/* messages of its assigned day each env has consumed since it was last assigned or rewound */
int rlm_get_tape_pos(rlm_handle h, int64_t* out /* [n_envs] */);

/* One venue's Market (src/market/market.cpp:11-38,67-70): the same fields and rules as rlm_config's venue block. */
typedef struct rlm_market {
  int32_t n_bands; int32_t pad;
  double band_px[RLM_MAX_BANDS];
  double band_ts[RLM_MAX_BANDS];
  int64_t open_ms, close_ms;
} rlm_market;
/* RLM_SOURCE_TAPE: day d of the loaded library runs under markets[day_market[d]] (Intraday::LoadData building the
 * ticker's market, src/environment/intraday.cpp:141-150) -- its tick table decides ToTicks / ToPrice, its hours the
 * warm-up start and the terminal step.  n_days must equal the library's day count.
 * - Tape handles only, with a library loaded.  The call waits for the handle's work and, like rlm_load_days, rewinds
 *   every env to the start of its assigned day: follow it with rlm_reset.
 * - An env's market follows its day, through rlm_load_days' b % n_days assignment and through rlm_assign_days.
 * - rlm_load_days replaces the library and drops the day markets: every day runs under the config's market again.
 * - Every market gets the checks rlm_create applies to the config's (1..RLM_MAX_BANDS bands, ascending band_px,
 *   positive band_ts) and every index must lie in [0, n_markets); otherwise RLM_ERR_INVALID_ARGUMENT, nothing changed.
 * - Training and backtest, independent and shared policies and the split surface all read the env's market. */
int rlm_set_day_markets(rlm_handle h, const rlm_market* markets, int32_t n_markets, const int32_t* day_market, int32_t n_days);

/* Advance every env by n_ticks market ticks.  Each env runs warm-up, performAction's inner NextState loop, and --
 * whenever its midprice has moved -- the complete learner step.  On return every env has consumed exactly n_ticks
 * messages and sits inside performAction's loop, whatever order the engine ran the envs' ticks in (they never interact);
 * on the tape source an env whose day ends earlier has consumed the rest of its day.
 * Calls shorter than 128 ticks only enqueue work (asynchronous; see rlm_sync); longer calls of independent policies on
 * up to 16 384 envs run round by round and return when the device is nearly done with them (the host follows the
 * device to learn when the last env has finished; RLM_ROUNDS=0 keeps every call asynchronous). */
int rlm_run_ticks(rlm_handle h, int32_t n_ticks);

int rlm_sync(rlm_handle h);

int rlm_get_counters(rlm_handle h, rlm_counters* out);
int rlm_get_stats(rlm_handle h, int32_t env0, int32_t n, rlm_env_stats* out);
int rlm_get_state(rlm_handle h, float* out /* [n_envs][n_state_vars] */);
int rlm_get_reward(rlm_handle h, double* out /* [n_envs] last reward handed to the agent */);
int rlm_get_actions(rlm_handle h, int32_t* out /* [n_envs] last action */);
/* rho of the R-learning agents (RLearn / OnlineRLearn / DoubleRLearn private member, include/rl/agent.h:131,145,157;
   the reference never prints it -- exposed here so that parity of the average-reward estimate can be checked) */
int rlm_get_rho(rlm_handle h, double* out /* [n_envs] */);
/* theta (both tables of a double agent) of every policy of `src` -> `dst`, device to device: the B-env form of handing one
   trained `Agent*` to the next phase (src/main.cpp:196-222 keeps `m` across training episodes and into evaluation).  The
   handles must agree in device, n_envs / shared_policy, memory_size and algorithm family; traces and env state of `dst`
   are untouched. */
int rlm_copy_theta(rlm_handle dst, rlm_handle src);
/* Diagnostic (no reference counterpart): number of weights of env b's table A that are not +0.0, i.e. how far the
   table has filled up (independent policies). */
int rlm_get_occupancy(rlm_handle h, int32_t* out /* [n_envs] */);

int rlm_handle_terminal(rlm_handle h, int32_t episode);
int rlm_go_greedy(rlm_handle h);

/* theta access: policy = env index (independent) or 0 (shared); table 0 = A, 1 = B (double agents). */
int rlm_read_theta(rlm_handle h, int32_t policy, int32_t table, double* out, int64_t n);
int rlm_write_theta(rlm_handle h, int32_t policy, int32_t table, const double* in, int64_t n);

/* parity dump of recorded envs (cfg.record_envs / record_cap) */
int rlm_read_records(rlm_handle h, int32_t env, rlm_step_record* out, int32_t cap, int32_t* n_out);

/* raw device pointers, for torch.distributed / NCCL plumbing on the shared-policy path */
int rlm_device_ptrs(rlm_handle h, void** theta, void** dtheta, int64_t* n_doubles);
/* Shared policy (cfg.shared_policy = 1; reference analogue: threads sharing one rl::Agent*,
 * src/main.cpp:196-206).  One training tick across GPUs is
 *   rlm_shared_tick_accumulate(h)   env tick + learner steps under theta_t, updates summed into dtheta
 *   all-reduce(dtheta, SUM)         caller's collective (torch.distributed / NCCL) on rlm_device_ptrs()
 *   rlm_apply_dtheta(h)             theta += dtheta; dtheta = 0; Q(from,.) under theta_{t+1}; next actions
 * On one GPU rlm_run_ticks does the same without the collective.
 * Evaluation (RLM_MODE_BACKTEST) never writes theta, so it needs no collective on any number of GPUs: every rank calls
 * rlm_run_ticks and evaluates its own shard of envs (env_index0) against its replica of theta.  In that mode these two
 * calls return RLM_ERR_INVALID_ARGUMENT; theta, dtheta and the trace lists stay bit for bit as they were, and
 * rlm_set_mode(h, RLM_MODE_TRAIN) resumes training. */
int rlm_shared_tick_accumulate(rlm_handle h);
int rlm_apply_dtheta(rlm_handle h);
/* ---- split surface: the reference's Environment::step / Agent::update seam, batched ------------------------------
 * rlm_run_ticks fuses the whole of experiment::serial::Learner::_step (src/experiment/serial.cpp:53-70).  These three
 * calls expose its parts, so that an external policy can supply the actions and an external consumer can read every
 * transition; driven in the order below they reproduce rlm_run_ticks bit for bit (tests/test_gpu_split.py):
 *
 *   rlm_env_step(h, NULL, ..)        Runner::RunEpisode: environment.Initialise()              serial.cpp:18-25
 *   rlm_agent_update(h, NULL)        ... Q(first from-state, .) for the first action
 *   repeat:
 *     rlm_act(h, actions)            int action = m->action(*last_state)                       serial.cpp:60,  include/rl/agent.h:60
 *     rlm_env_step(h, actions, r, t) environment.performAction(action) + getReward()           serial.cpp:61,66, include/environment/base.h:132
 *     rlm_agent_update(h, delta)     state->newState(env); m->HandleTransition(...)            serial.cpp:64-67, include/rl/agent.h:62-67
 *
 * Every env advances by ONE learner step per rlm_env_step (its own K >= 1 market ticks, base.cpp:285-305); envs are
 * therefore not tick-aligned afterwards, which is why this surface needs source = generator or tape (not stream).
 * actions_out[b] / the action applied is -1 for an env whose episode is over or whose tape day has run out.
 * terminal_out[b]: 1 = the episode is over (Intraday::isTerminal), 2 = tape source: the env needed a message past the end
 * of its day and stopped inside performAction (the reference's performAction returning false at the end of its files).  rlm_env_step(h, actions != NULL) without a preceding rlm_act
 * is the "external policy" form: no generator draw is consumed.  Independent policies only. */
int rlm_act(rlm_handle h, int32_t* actions_out /* [n_envs] */);
int rlm_env_step(rlm_handle h, const int32_t* actions /* [n_envs] or NULL = the agent's own */, double* reward_out /* [n_envs] or NULL */,
                 uint8_t* terminal_out /* [n_envs] or NULL */);
int rlm_agent_update(rlm_handle h, double* delta_out /* [n_envs] TD error of each env's last transition, or NULL */);

/* measurement hooks (bench.py): CUDA-event durations of the env-tick and agent kernels, summed over launches */
int rlm_set_profiling(rlm_handle h, int32_t on);
int rlm_get_kernel_times(rlm_handle h, double* env_ms, double* agent_ms, int64_t* env_launches, int64_t* agent_launches);
/* run on a caller-provided CUDA stream (cudaStream_t as void*); 0 = the handle's own stream */
int rlm_set_stream(rlm_handle h, void* cuda_stream);

/* Real-data ingestion (host code, no GPU needed): a reference-format CSV pair -- market depth
 * (date,HH:MM:SS.mmm,AP1..5,AV1..5,BP1..5,BV1..5) and time-and-sales (date,time,price,size) -- becomes the packed message
 * stream rlm_load_ticks takes, with exactly the row filtering, print aggregation and row grouping of the reference's
 * data layer (data::basic::MarketDepth / TimeAndSales src/data/basic.cpp:20-202, Streamer::LoadUntil
 * src/data/streamer.cpp:57-81, Intraday::UpdateBookProfiles src/environment/intraday.cpp:274-313): depth rows that
 * share a timestamp or follow an invalid book state are flagged RLM_TICK_PARTIAL, ticks with more than RLM_N_TX_MAX
 * distinct print prices lead with RLM_TICK_TX_MORE messages (include/rlm_flow.h).  Call with out == NULL to size the
 * buffer: *n_msgs = messages, *n_ticks = market ticks (NextState calls) they make up. */
int rlm_ingest_csv(const char* md_path, const char* tas_path, rlm_tick_msg* out, int64_t cap, int64_t* n_msgs, int64_t* n_ticks);

/* host-side synthetic flow (same integer process as the in-kernel generator) */
int rlm_flow_generate(const rlm_flow_params* p, int64_t env_index, int64_t first_tick, int32_t n_ticks,
                      rlm_tick_msg* out);

/* ---- unit-level device entry points for the golden vectors of the reference's tests ---- */
/* Market::ToTicks / ToPrice (test/test_Market.cpp) evaluated ON THE DEVICE; out = -1 (-1.0) where the reference throws.
 * rlm_test_to_ticks converts px[0..n) in order in one thread and carries one band hint from each price to the next,
 * as an env does (starting from band 0), so an order that jumps between bands exercises hint misses; the hint never
 * changes a result. */
int rlm_test_to_ticks(const rlm_config* cfg, const double* px, int32_t n, int32_t* out);
int rlm_test_to_price(const rlm_config* cfg, const int32_t* ticks, int32_t n, double* out);
/* tiles() (src/rl/tiles.cpp:31-75) for n states of n_vars floats, all actions: out[n][n_actions][96] */
int rlm_test_tiles(const rlm_config* cfg, const float* vars, int32_t n, int32_t* out);
/* TEST ONLY.  The same tile indices as each learner kernel derives them (cfg sets memory_size, n_actions, n_state_vars):
 *   RLM_TILES_THREE_WARP    tile_base_sum + tile_index (rlm_agent3_kernel, round-1 kernels)      out[n][n_actions][96]
 *   RLM_TILES_ONE_WARP      ln_hash + ln_tile (rlm_learn_kernel, the fused 'F' engine)           out[n][n_actions][96]
 *   RLM_TILES_STAGED        the 16-bit index rows of rlm_learn_staged_kernel (memory_size <= 8192) out[n][n_actions][96]
 *   RLM_TILES_TRACE_GROUP0  group 0 rebuilt from the stored base (base mod M + action term) mod M, as the trace passes
 *                           and tile tables do                                                    out[n][n_actions][32]
 * Writes only `out`.  Returns RLM_ERR_UNSUPPORTED for RLM_TILES_STAGED above 8192. */
enum { RLM_TILES_THREE_WARP = 0, RLM_TILES_ONE_WARP = 1, RLM_TILES_STAGED = 2, RLM_TILES_TRACE_GROUP0 = 3 };
int rlm_test_learner_tiles(const rlm_config* cfg, int32_t form, const float* vars, int32_t n, int32_t* out);
/* Order script (test/test_Order.cpp): op codes see rlm_order_op */
typedef struct rlm_order_op { int32_t op; int32_t pad; int64_t arg; } rlm_order_op; /* 0=doTransaction 1=doCancellation 2=addVolumeBehind 3=clearQueues */
typedef struct rlm_order_state { int64_t size, q_head, q_tail, executed, ret; } rlm_order_state;
int rlm_test_order(int64_t size, int64_t q_head, const rlm_order_op* ops, int32_t n_ops, rlm_order_state* out /*[n_ops]*/);
/* RollingMean<double> (test/test_Accumulators.cpp): out[i] = {mean,var} after push i */
int rlm_test_rolling_mean(int32_t window, const double* vals, int32_t n, double* out /*[n][2]*/);

#ifdef __cplusplus
}
#endif
#endif /* RLM_H */
