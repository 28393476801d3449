/* lob_oracle.h -- C ABI of the CPU restatement.  TEST INFRASTRUCTURE ONLY.
 *
 * oracle/ is the checker, never the product: only tests/, __graft_entry__.smoke()
 * and bench.py's cpu_baseline / --impl reference legs may load this library.
 * It restates, one env at a time and in the reference's own operation order,
 * the hot path of tspooner/rl_markets (SURVEY.md section 8a); every function in
 * lob_oracle.cpp cites the reference file:line it follows.
 *
 * PARITY PINNING: the restatement is pinned against the reference itself,
 * compiled unmodified into oracle/_ref/ref_driver (oracle/Makefile), on the
 * same synthetic streams (tests/test_oracle_vs_ref.py, tests/golden/), and
 * against the golden vectors of the reference's own unit tests
 * (test/test_Order.cpp, test_Book.cpp, test_Market.cpp, test_Accumulators.cpp).
 */
#ifndef LOB_ORACLE_H
#define LOB_ORACLE_H

#include <stdint.h>
#include "rlm.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct lobo_env lobo_env;

lobo_env* lobo_create(const rlm_config* cfg, int64_t env_index);
void lobo_destroy(lobo_env* e);

/* Feed `n_msgs` ticks.  Runs Initialise (first call), then learner steps until
 * the messages are exhausted, the env is terminal, or max_steps further steps
 * were taken (max_steps < 0: no cap).  Writes up to rec_cap step records.
 * Returns the number of learner steps completed in this call; *n_consumed =
 * messages consumed.  Unlike the reference (whose streamer ends the episode at
 * end-of-file) a drained buffer just pauses the env mid-performAction. */
int64_t lobo_run(lobo_env* e, const rlm_tick_msg* msgs, int64_t n_msgs, int64_t max_steps,
                 rlm_step_record* recs, int64_t rec_cap, int64_t* n_consumed);

int lobo_is_terminal(lobo_env* e);
void lobo_stats(lobo_env* e, rlm_env_stats* out);
int64_t lobo_total_steps(lobo_env* e);
int64_t lobo_total_ticks(lobo_env* e);
int64_t lobo_sum_traces(lobo_env* e);
const double* lobo_theta(lobo_env* e, int table);
void lobo_handle_terminal(lobo_env* e, int episode);
void lobo_go_greedy(lobo_env* e);
void lobo_reset(lobo_env* e);
void lobo_set_backtest(lobo_env* e, int on);
void lobo_new_env(lobo_env* e);
double lobo_rho(lobo_env* e);

/* Run n_envs independent envs (env_index0 + b), each for `n_ticks` generated ticks, on
 * `n_threads` host threads; returns total learner steps.  Used as the "port" CPU baseline. */
int64_t lobo_run_batch(const rlm_config* cfg, int32_t n_envs, int64_t n_ticks, int32_t n_threads,
                       int64_t* total_ticks, double* seconds);

/* ---- shared-policy batch (SURVEY section 8e): synchronous formulation, see lob_oracle.cpp ---- */
typedef struct lobo_batch lobo_batch;
lobo_batch* lobo_batch_create(const rlm_config* cfg);
void lobo_batch_destroy(lobo_batch* b);
void lobo_batch_accumulate(lobo_batch* b, const rlm_tick_msg* msgs /* [n_envs] */, rlm_step_record* recs, int32_t* rec_count, int32_t rec_cap);
double* lobo_batch_dtheta(lobo_batch* b, int table);
double* lobo_batch_theta(lobo_batch* b, int table);
void lobo_batch_apply(lobo_batch* b);
/* Contribution log: with it on, every addition a batch env makes into dtheta during lobo_batch_accumulate is also
 * recorded as (table, feature, value), value being exactly the double added (scaled_update * eligibility[f]).  The
 * log holds the last accumulate's entries in the order they were added; switching it on or off clears it.  With the
 * log off nothing is recorded and every number is what it was without it. */
typedef struct lobo_contrib { int32_t table; int32_t feature; double value; } lobo_contrib;
void lobo_batch_log(lobo_batch* b, int on);
const lobo_contrib* lobo_batch_log_entries(lobo_batch* b, int64_t* n);
int64_t lobo_batch_steps(lobo_batch* b);
int64_t lobo_batch_sum_traces(lobo_batch* b);  /* trace entries summed over every step of every env (rlm_counters) */
void lobo_batch_stats(lobo_batch* b, int32_t env, rlm_env_stats* out);

/* ---- unit-level entry points (golden vectors) ---- */
int32_t lobo_to_ticks(const rlm_config* cfg, double px);
double lobo_to_price(const rlm_config* cfg, int32_t ticks);
double lobo_tick_size(const rlm_config* cfg, double px);
void lobo_tiles(const rlm_config* cfg, const float* vars, int32_t* out /* [n_actions][96] */);
void lobo_order_script(int64_t size, int64_t q_head, const rlm_order_op* ops, int32_t n_ops, rlm_order_state* out);
void lobo_rolling_mean(int32_t window, const double* vals, int32_t n, double* out /* [n][2] */);
uint64_t lobo_mt19937_64(uint64_t seed, int32_t n_skip);       /* value number n_skip (0-based) */
int32_t lobo_glibc_rand(uint32_t seed, int32_t n_skip);
double lobo_uniform_real(uint64_t seed, int32_t n_skip);
uint32_t lobo_uniform_int(uint64_t seed, uint32_t n, int32_t n_skip);

/* Book scenario replay (test/test_Book.cpp): a tiny interpreter, see tests/test_golden_book.py */
typedef struct lobo_book_op {
  int32_t op;      /* 0 ApplyChanges(prices,vols)+Stash  1 PlaceOrder(side,price,size)  2 ApplyTransactions(side,ref)
                      3 AdverseSelection  4 WalkTheBook(side,ref,size)  5 CancelAll(side)
                      6 set the prints (px,vol,n) handed to the following ApplyChanges calls */
  int32_t side;    /* 0 ask, 1 bid */
  double px[5];    /* op0: prices of `side`; op2: tx prices */
  int64_t vol[5];  /* op0: volumes; op2: tx volumes */
  int32_t n;       /* op0: depth used (<=5); op2: number of prints */
  int32_t pad;
  double a;        /* price / ref */
  int64_t b;       /* size */
} lobo_book_op;
typedef struct lobo_book_result {
  int64_t r_volume; double r_proxy; double r_value; int32_t r_ok; int32_t n_transacted;
  rlm_order_rec order; double obs_value; int64_t obs_volume; int64_t total_volume;
} lobo_book_result;
void lobo_book_script(const lobo_book_op* ops, int32_t n_ops, lobo_book_result* out);

#ifdef __cplusplus
}
#endif
#endif
