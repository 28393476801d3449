// rlm_types.h -- device-side data layout of the batched LOB environment + agent.
//
// One `EnvHdr` (+ its window rings) per environment, array-of-structs in HBM.
// The env kernel (one thread per env) copies the header into thread-local
// memory -- lane-interleaved, i.e. SoA across the warp -- for the scalar market
// logic; the agent kernel (one warp per env) stages only the AgentD block into
// shared memory.  The big per-env arrays (theta, the compact trace list, the
// Mersenne Twister state) stay in HBM and are touched sparsely.
#pragma once
#include <stdint.h>
#include "rlm.h"

#define RLM_NWIN 10
enum { W_MID = 0, W_VLT, W_VNUM, W_VDEN, W_SPREAD, W_TP, W_ASKTX, W_BIDTX, W_PNLUP, W_PNLDN };

enum { PH_PREOPEN = 0, PH_WARMUP = 1, PH_RUN = 2, PH_DONE = 3 };

// error bits accumulated per env (reported by rlm_sync as RLM_ERR_RUNTIME / INVALID_ARGUMENT)
enum {
  ERR_BAD_PRICE = 1,       // book.cpp:74-77 / order.cpp:22 (non-positive price or volume)
  ERR_TICK_RANGE = 2,      // market.cpp:86,112 invalid price / tick for conversion
  ERR_TRACE_OVERFLOW = 4,  // more nonzero traces than trace_cap (traces.h:13 MAX_NONZERO_TRACES analogue)
  ERR_INVALID_STATE = 8,   // BookUtils::IsValidState false (the reference would merge rows)
  ERR_STREAM_UNDERRUN = 16,
  ERR_MODEL_LOG_GAP = 32   // model_log: an env completed more than one update between two accumulation passes
};

struct OrderD {  // market::Order (include/market/order.h:11-51); one per side (ORDER_LIMIT == 1, base.cpp:21)
  double price;
  long long size, q_head, q_tail, executed, initial_queue;
  int live;
  int transactions;
};

struct SideD {  // market::Book<C,5> (include/market/book.h:22-110)
  double px[RLM_DEPTH];
  double last_px[RLM_DEPTH];
  int vol[RLM_DEPTH];
  int last_vol[RLM_DEPTH];
  long long total_vol, last_total_vol;
  double obs_value;
  long long obs_volume;
  int n_transacted;
  int has_cur, has_last;  // levels / last_levels non-empty
  int pad;
  OrderD ord;
};

// Agent-side per-env state.  The agent kernel stages exactly this block (16-byte aligned) into
// shared memory; everything the learner step needs from the env is in here.
struct alignas(16) AgentD {
  double q_from[RLM_MAX_ACTIONS];   // Q_A(from, .) under the current theta
  double qb_from[RLM_MAX_ACTIONS];  // Q_B(from, .) (double agents)
  double last_reward, last_delta;
  long long n_steps, sum_traces;
  float from_vars[RLM_N_STATE_MAX + 3];  // state variables of the from-state
  float to_vars[RLM_N_STATE_MAX + 3];    // state variables of the to-state (written by the env tick)
  int from_base0[32];  // from-state, feature group 0: lane j's partial tile hash sum mod M
  int crand_r[31];     // glibc rand() state
  int crand_f, crand_b;
  int mt_pol_idx, mt_agt_idx;  // std::mt19937_64::_M_p
  int null_from;   // from-state is the never-populated State of serial.cpp:14-15,55 (all features 0)
  int n_traces, cur_action;
  int need_begin;  // the next env tick starts with Learner::_step's action selection (serial.cpp:55-61)
  int kind;        // why the env is in the ready list: 0 learner step, 1 end of warm-up
  int ep_step, err;
  int n_occ;   // independent policies: bits set in this env's occupancy bitmap; > M/4 => treat theta as dense
  double rho;  // R-learning average reward (agent.h:131,145,157); lives as long as theta does
  // from-state of the last completed transition: Runner's two State objects survive RunEpisode (serial.h:17-23), so the
  // next episode's first action is chosen from -- and its first transition starts at -- this state (serial.cpp:24-25,55,60)
  float prev_vars[RLM_N_STATE_MAX + 3];
  int prev_null;
  int hs_valid;  // the tick kernel has stored the to-state's tile-hash sums in DevPtrs::hsum (and prefetched the tiles into L2)
  int pad[2];
};

struct FillD { long long volume; double proxy, value; };  // what Ask/BidBook::ApplyTransactions returns (book.cpp:382-427)

struct EnvHdr {
  SideD side[2];  // 0 = ask, 1 = bid
  long long position;  // RiskManager::position_
  double pnl_step, momentum_pnl_step, ask_quote, bid_quote;  // Base members (base.h:55-63)
  double agg_r, agg_pnl, agg_mpm;                            // locals of performAction kept across ticks
  double tp_val, ewma_up, ewma_dn;
  double ep_reward, ep_pnl, ep_bandh;
  double w_sum[RLM_NWIN], w_mean[RLM_NWIN], w_s[RLM_NWIN];
  long long n_ticks;
  int w_head[RLM_NWIN], w_count[RLM_NWIN];
  int phase, last_action, lo_vol_step;
  int ask_level, bid_level, date, last_date, time_ms;
  int market_buys, market_sells;
  int ts_total, ts_ask, ts_bid, ts_both, ts_pos, ts_long, ts_short;
  int err;
  // multi-message ticks of ingested real data (RLM_TICK_PARTIAL / RLM_TICK_TX_MORE, rlm_flow.h): the tick's prints and the
  // fills of its ApplyTransactions, kept until the last depth row of the tick has been applied
  int tick_open, txn;
  // round-paced engine (rlm_env_round_kernel): ticks of run call `run_id` this env has consumed
  int run_id, run_pos;
  // Market::ToTicks of the last midprice (next_state_tail): the midprice moves on fewer than a third of the ticks
  double tk_px;
  int tk_ticks, tk_band;  // (tk_band: band of the last conversion, to_ticks' hint)
  float tx_px[RLM_TX_CAP];
  int tx_vol[RLM_TX_CAP];
  FillD tick_au, tick_bu;
  rlm_flow_state flow;
  AgentD ag;
};

struct VenueD {
  int n;
  int cum_full[RLM_MAX_BANDS];   // ticks after fully traversing bands 0..k-1 (market.cpp:88-99 chain)
  int tts_tick[RLM_MAX_BANDS];   // Market::tts_ keys (market.cpp:27-37)
  double px[RLM_MAX_BANDS], ts[RLM_MAX_BANDS];
  double inv_ts[RLM_MAX_BANDS];     // 1 / ts where ts is a power of two (x / ts == x * inv_ts exactly), else 0
  double cum_price[RLM_MAX_BANDS];  // price after fully traversing tts_ bands 0..k-1 (market.cpp:115-125 chain)
  long long open_lo, close_hi;      // IsOpen bounds: mo+30min, mc-30min (market.cpp:67-70)
};

struct DevParams {
  int n_envs, n_actions, algorithm, policy_type, reward_measure, n_state_vars;
  int state_vars[RLM_N_STATE_MAX];
  int tp_is_micro, l2p_book, order_size, source, shared_policy, is_double;
  long long pos_lb, pos_ub, memory_size;
  unsigned long long m_magic;  // floor(2^64 / M)
  int m_pow2;
  int ra_m[RLM_MAX_ACTIONS];  // rndseq[(a + 449*4) & 2047] mod M: the action term of a group-0 tile hash
  unsigned rg[3][RLM_MAX_ACTIONS];  // rndseq[(g*A + a + 449*(nf_g + 1)) & 2047]: the action term of group g's tile hash (tiles.cpp:65-68)
  float gl;  // (float)(gamma*lambda): Traces::decay(float rate)
  double gw[3], gamma, beta;
  float damping, pos_weight, trd_weight, pnl_weight;
  double ewma_alpha;
  int win_size[RLM_NWIN], win_off[RLM_NWIN];
  int ring_total;       // doubles per env
  int env_stride;       // bytes per env record in HBM (multiple of 16)
  int trace_cap, record_envs, record_cap;
  int scratch_bytes;    // per-warp shared-memory scratch (depends on is_double)
  int occ_words;        // 32-bit words of the occupancy bitmap per policy
  int occ_smem_words;   // > 0: the learner kernel stages an env's whole bitmap in shared memory (small memory_size)
  long long env_index0;
  VenueD venue;
  rlm_flow_params flow;
};

struct DynParams {  // changes between launches (HandleTerminal / GoGreedy)
  double alpha, eps, tau;
  int greedy;
  int n_ticks;
  int stream_ticks;   // ticks in the resident stream chunk
  int stream_off;     // first tick of the chunk this launch consumes
  int env0;           // tick-synchronous engine: first env of the sub-batch this launch covers
  int backtest;       // 1: Backtester::_step (serial.cpp:121-137): act on the current state, never learn
  int n_sub;          // ... and its size (0 = the whole batch).  Sub-batches run on their own streams (rlm_api.cu)
  int sub_idx;        // index of the sub-batch (timeline probe of the RLM_TIMING build)
  int debug_flags;    // RLM_TIMING build only (RLM_DEBUG_FLAGS): what-if switches of tools/timeline_probe.py; results are wrong with any set
  int env_hash;       // tick kernel hashes the to-state and prefetches its tiles at a step end (RLM_ENV_HASH=1; measured slower)
  int round_cap;      // round-paced engine: most ticks an env runs in one round (RLM_ROUND_CAP; 0 = up to its step end)
  int ctl_stream;     // tick-synchronous engine under a CUDA graph, STREAM source: stream pointer / offset / length come from *DevPtrs::runctl
  int hold;           // split surface (rlm_env_step): envs whose step has ended, or whose next action is not applied yet, do not tick
  int tape_l2;        // tape source: the warp-per-env tick kernels ask L2 for each env's next message (RLM_TAPE_PREFETCH, default 1)
};

// ready counters: [RLM_MAX_SUB][RLM_READY_CAP] ints, followed by as many live counters (round-paced engine)
#define RLM_MAX_SUB 8
#define RLM_READY_CAP 256
#define RLM_LIVE_OFF (RLM_MAX_SUB * RLM_READY_CAP)

// per-call parameters of the round-paced engine, in device memory so that its CUDA graphs do not depend on them
struct RunCtl { int run_id, n_ticks, stream_off, stream_ticks; const rlm_tick_msg* stream; long long pad; };

struct DevPtrs {
  unsigned char* env;       // [n_envs][env_stride]
  double* theta;            // [n_policies][M]
  double* theta_b;          // [n_policies][M] or null
  double* dtheta;           // shared policy: accumulated delta, [M]
  int* trace_f;             // [n_envs][trace_cap]
  float* trace_e;           // [n_envs][trace_cap]
  unsigned long long* mt_pol;  // [n_envs][312]
  unsigned long long* mt_agt;  // [n_envs][312] or null
  const rlm_tick_msg* stream;  // [stream_ticks][n_envs]
  rlm_step_record* records;    // [record_envs][record_cap]
  int* record_count;           // [record_envs]
  unsigned long long* counters;  // [8]: ticks, steps, sum_traces, terminal, err
  unsigned* occ;                 // [n_policies][occ_words] occupancy bitmap: bit f set <=> theta[f] was ever updated
  unsigned long long* hsum;      // [n_envs][3][32] partial tile-hash sums of the to-state (lane j = tiling j), written by the tick kernel
  int* ready;                    // [n_envs] env indices that need the agent kernel this tick
  int* ready_count;              // [ticks of the current run call]
  // persistent engine
  int* q_slots;                  // [q_size] env ids handed from env threads to agent warps (-1 = empty)
  unsigned* q_head;              // consumer tickets
  unsigned* q_tail;              // producer tickets
  unsigned* env_warps_done;
  int* q_done;                   // set when every env warp has finished
  int* ag_done;                  // [n_envs] agent -> env completion flags
  int q_size;                    // power of two >= n_envs
  int pad;
  RunCtl* runctl;                // round-paced engine: the current run call
  // tape source (rlm_load_days): the day library and each env's read position in it.  The cursor lives here and not in
  // the env record so that a tick kernel can form the message address without waiting for the record's stage-in.
  const rlm_tick_msg* tape;      // [n_msgs] concatenated days
  int2* tape_cur;                // [n_envs] {next message, end of the env's day} (absolute message indices)
  int* tape_lo;                  // [n_envs] first message of the env's day (rlm_reset / rlm_new_env rewind to it)
};

// model_log (rlm_set_model_log, rlm_model_log.cu): per env the state of Agent::_agg_delta / _update_counter
// (include/rl/agent.h:40-41) and the rows it has logged since the last read
struct ModelLogAcc {
  double agg;      // _agg_delta
  long long seen;  // AgentD::n_steps at the last pass
  int count;       // _update_counter
  int pad;
};
struct ModelLogPtrs {
  ModelLogAcc* acc;    // [n_envs]
  long long* written;  // [n_envs] rows logged since the last read (the first `cap` of them are kept)
  double* rows;        // [n_envs][cap]
  long long cap;
};

// Tape days with markets of their own (rlm_set_day_markets).  A __constant__ block of its own (rlm_env.cuh: PM), uploaded
// with DevParams: only the kernels that read an env's market see it, every other kernel keeps its parameters.
struct DevMarkets {
  const VenueD* markets;  // [n_markets]; null while every day runs under the config's market
  int* env_market;        // [n_envs] market of the env's current day (-1: the config's)
  int* rec_fixed;         // [record_envs] records whose terminal flag already accounts for the env's market
};
