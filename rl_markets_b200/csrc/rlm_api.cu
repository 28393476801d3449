// rlm_api.cu -- host side of the C ABI declared in include/rlm.h.
//
// Owns device memory, derives the constant tables the kernels need (venue tick chains,
// window layout, modulo magic), and maps the reference's exception classes to rlm_status
// codes.  There is deliberately NO CPU execution path here: without a CUDA device
// rlm_create fails with RLM_ERR_NO_DEVICE.
#include <cuda_runtime.h>
#include <math.h>
#include <stdio.h>
#include <string.h>
#include <algorithm>
#include <mutex>
#include <string>
#include <vector>

#include "rlm.h"
#include "rlm_flow_tables.h"
#include "rlm_rndseq.h"
#include "rlm_kernels.h"
#include <limits.h>
#include <stddef.h>
#include <stdlib.h>

static thread_local std::string g_err;
static int fail(int code, const std::string& msg) { g_err = msg; return code; }
int rlm_set_error_(int code, const std::string& msg) { return fail(code, msg); }  // for the host-only translation units
#define CK(expr)                                                                                      \
  do {                                                                                                \
    cudaError_t _e = (expr);                                                                          \
    if (_e != cudaSuccess) return fail((_e == cudaErrorNoDevice || _e == cudaErrorInsufficientDriver) ? RLM_ERR_NO_DEVICE : RLM_ERR_CUDA, \
                                       std::string(#expr) + ": " + cudaGetErrorString(_e));          \
  } while (0)

struct rlm_handle_s {
  rlm_config cfg;
  DevParams hp;
  DevPtrs ptr;
  DynParams dyn;
  cudaStream_t stream = nullptr;
  bool own_stream = true;
  int n_sms = 132;
  int engine = 1;        // 1 tick-synchronous (two launches per tick), 0 persistent queue (rlm_run_kernel), 2 fused (warp per env)
  int n_agent_ctas = 0;  // persistent engine: CTAs in the agent role
  int env_variant = 0;   // env tick kernel: 0 = warp per env, 1 = thread per env
  int agent_variant = 4; // learner kernel: 4 = rlm_learn_kernel (one warp per env, round 2), 3 = three warps per env, 1 = round-1 one-warp kernel
  unsigned* d_qctl = nullptr;  // [4]: q_head, q_tail, env_warps_done, q_done
  DynParams shared_dyn;
  bool in_run = false;
  // optional per-kernel timing (bench.py roofline leg): CUDA events around every launch of a run call
  bool profile = false;
  std::vector<cudaEvent_t> ev;
  double prof_env_ms = 0, prof_agent_ms = 0;
  long long prof_env_launches = 0, prof_agent_launches = 0;
  int ready_cap = 0;  // ticks per run call the ready counters can hold
  int n_policies = 1;
  size_t env_bytes = 0;
  // STREAM source: two device chunks; rlm_load_ticks fills the idle one on a copy stream while the kernels of
  // earlier rlm_run_ticks calls still read the other (upload of chunk k+1 overlaps compute of chunk k)
  rlm_tick_msg* d_stream[2] = {nullptr, nullptr};
  size_t stream_cap[2] = {0, 0};  // messages
  int stream_buf = 0;
  cudaStream_t copy_stream = nullptr;
  cudaEvent_t ev_copied[2] = {nullptr, nullptr}, ev_consumed[2] = {nullptr, nullptr};
  bool consumed_valid[2] = {false, false};
  int stream_ticks = 0, stream_cursor = 0;
  // TAPE source: the day library (ptr.tape, ptr.tape_cur, ptr.tape_lo) and its day boundaries on the host
  std::vector<int64_t> day_off;  // [n_days + 1]; empty until rlm_load_days
  std::vector<int32_t> env_day;  // [n_envs] the day each env replays
  // day markets (rlm_set_day_markets): the market of each day (empty: every day runs under the config's), each env's current
  // market (-1: the config's; mirrors ptr.env_market, which exists once day markets were first set) and the config's
  // VenueD, whose IsOpen bounds the uploaded copy gives up while day markets are on (see day_markets_on)
  std::vector<int32_t> day_market;
  std::vector<int32_t> env_mkt;
  VenueD cfg_venue;
  DevMarkets dm = {};  // uploaded with hp (rlm_env.cuh: PM)
  bool rec_dirty = false;  // learner work was enqueued since rlm_fix_terminal_kernel last ran (fix_records)
  void* d_gather = nullptr; void* h_gather = nullptr; size_t gather_cap = 0;  // rlm_get_reward/actions/state staging
  long long launches = 0;
  double alpha = 0, eps = 0, tau = 1.0;
  // tick-synchronous engine: the batch is cut into n_sub sub-batches, each ticking on its own stream, so that the
  // DRAM-bound gather burst of one sub-batch's learner kernel overlaps the issue-bound scalar tick kernel of another
  int n_sub = 1;
  // CUDA graphs of the tick-synchronous engine (generator source, one stream): one instantiated graph per chunk length,
  // valid as long as the per-launch parameters it was captured with are unchanged
  struct TickGraph { int chunk; DynParams d; cudaGraphExec_t exec; };
  std::vector<TickGraph> graphs;
  bool use_graphs = true, graph_warm = false;
  bool staged = false;  // learner: whole-table staging (memory_size * 8 <= 64 KB, independent single-table policies)
  cudaStream_t sub_stream[RLM_MAX_SUB] = {};
  cudaEvent_t ev_fork = nullptr, ev_join[RLM_MAX_SUB] = {};
  // round-paced engine (independent policies, warp-per-env ticks): see run_rounds
  bool rounds = false;       // forced (RLM_ROUNDS=1)
  bool in_rounds = false;    // run_rounds is enqueueing (learner launches see more steps)
  bool rounds_auto = false;  // default: run calls of at least RLM_ROUNDS_MIN_TICKS ticks
  int run_seq = 0;
  int round_streams = 1;  // sub-batches of the round-paced engine, each on its own stream (RLM_ROUND_STREAMS)
  int* h_live = nullptr;  // pinned [RLM_MAX_SUB][2]: ready count of the last round of each group in flight
  cudaEvent_t ev_live[RLM_MAX_SUB][2] = {};
  long long rounds_launched = 0, rounds_calls = 0;
};

// The kernels read their per-handle constants from ONE __constant__ block (rlm_env.cuh: P).  g_params_owner says whose
// they are; another handle takes the block over only after everything launched so far has finished (device-wide
// synchronisation), and every entry point that launches kernels holds g_api_mu while it does so -- so two handles on
// one GPU, from one or several host threads, are safe; alternating between them costs a device synchronisation per switch.
static const rlm_handle_s* g_params_owner = nullptr;
static std::recursive_mutex g_api_mu;
#define API_LOCK std::lock_guard<std::recursive_mutex> api_lock_(g_api_mu)

// pinned + device staging area for per-env columns (grown on demand)
static int split_scratch(rlm_handle_s* h, size_t bytes) {
  if (bytes > h->gather_cap) {
    CK(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gather); if (h->h_gather) cudaFreeHost(h->h_gather);
    h->d_gather = nullptr; h->h_gather = nullptr; h->gather_cap = 0;
    CK(cudaMalloc(&h->d_gather, bytes));
    CK(cudaMallocHost(&h->h_gather, bytes));
    h->gather_cap = bytes;
  }
  return RLM_OK;
}

extern "C" {

const char* rlm_last_error(void) { return g_err.c_str(); }
int rlm_abi_version(void) { return RLM_ABI_VERSION; }

int rlm_config_default(rlm_config* c) {
  if (!c) return fail(RLM_ERR_INVALID_ARGUMENT, "null config");
  memset(c, 0, sizeof(*c));
  c->n_envs = 1; c->device = 0; c->env_index0 = 0; c->shared_policy = 0; c->source = RLM_SOURCE_GENERATOR;
  // config/example.yaml
  c->memory_size = 20000000; c->n_tilings = 32; c->n_actions = 9; c->algorithm = RLM_ALGO_DOUBLE_Q_LEARN;
  c->group_weights[0] = 0.65; c->group_weights[1] = 0.25; c->group_weights[2] = 0.10;
  c->gamma = 0.975; c->lambda = 0.85; c->omega = 1.0; c->alpha_start = 0.001; c->alpha_floor = 0.001; c->beta = 0.005;
  c->policy_type = RLM_POLICY_EPSILON_GREEDY; c->eps_init = 0.8f; c->eps_floor = 0.0001f; c->eps_T = 800;
  c->tau_init = 1.0f; c->tau_floor = 1.0f; c->tau_T = 1;
  c->spread_lookback = 45;
  c->reward_measure = RLM_REWARD_PNL_DAMPED; c->damping_factor = 0.15f; c->pos_weight = 0.0f; c->trd_weight = 0.0f; c->pnl_weight = 1.0f;
  c->pnl_lookback = 0;
  const int vars[8] = {RLM_VAR_POS, RLM_VAR_A_DIST, RLM_VAR_B_DIST, RLM_VAR_MPM, RLM_VAR_SPD, RLM_VAR_VOL, RLM_VAR_IMB, RLM_VAR_SVL};
  c->n_state_vars = 8;
  for (int i = 0; i < 8; ++i) c->state_vars[i] = vars[i];
  c->lb_mpm = 15; c->lb_vlt = 60; c->lb_svl = 60; c->lb_rsi = 0; c->lb_vwap = 0;
  c->pos_lb = -50; c->pos_ub = 50; c->order_size = 10;
  c->target_price_type = RLM_TP_YAML_MIDPRICE; c->tp_lookback = 1;
  // LondonStockExchange, symbol group of AAL (src/market/market.cpp:206-227)
  const double px[10] = {0., 1., 5., 10., 50., 100., 500., 1000., 5000., 10000.};
  const double ts[10] = {0.0001, 0.0005, 0.001, 0.005, 0.01, 0.05, 0.1, 0.5, 1, 5};
  c->n_bands = 10;
  for (int i = 0; i < 10; ++i) { c->band_px[i] = px[i]; c->band_ts[i] = ts[i]; }
  c->open_ms = 8LL * 3600000; c->close_ms = 16LL * 3600000 + 30LL * 60000;
  c->random_seed = 1994;
  rlm_flow_default_params(&c->flow, 1, 250);
  return RLM_OK;
}

// The VenueD of one Market (src/market/market.cpp:11-38, 67-70): the tick-table chains of market.cpp:27-37,78-128 in the
// reference's fp64 operation order, unused bands padded with px = +inf (to_ticks' band search and band hint rely on it),
// and the IsOpen bounds.  The config's market and every day market (rlm_set_day_markets) are built here.  false + why:
// the table is not one rlm_create accepts.
static bool venue_derive(VenueD& v, int n_bands, const double* band_px, const double* band_ts, int64_t open_ms, int64_t close_ms,
                         std::string& why) {
  memset(&v, 0, sizeof(v));
  if (n_bands < 1 || n_bands > RLM_MAX_BANDS) { why = "bad venue table"; return false; }
  v.n = n_bands;
  for (int i = 0; i < RLM_MAX_BANDS; ++i) { v.px[i] = INFINITY; v.ts[i] = 1.0; v.inv_ts[i] = 0.0; v.tts_tick[i] = INT_MAX; }
  for (int i = 0; i < n_bands; ++i) {
    v.px[i] = band_px[i]; v.ts[i] = band_ts[i];
    { int ex = 0; if (frexp(band_ts[i], &ex) == 0.5) v.inv_ts[i] = 1.0 / band_ts[i]; }  // power of two: exact reciprocal
    if (i > 0 && !(band_px[i] > band_px[i - 1])) { why = "venue bands must ascend"; return false; }
    if (!(band_ts[i] > 0)) { why = "venue tick sizes must be positive"; return false; }
  }
  {
    int ticks = 0;
    v.cum_full[0] = 0;
    for (int i = 0; i + 1 < v.n; ++i) {
      volatile double q = (v.px[i + 1] - v.px[i]) / v.ts[i];
      ticks = (int)((double)ticks + q);  // `int += double`
      v.cum_full[i + 1] = ticks;
    }
    long acc = 0;
    v.tts_tick[0] = 0;
    for (int i = 1; i < v.n; ++i) {
      volatile double q = (v.px[i] - v.px[i - 1]) / v.ts[i - 1];
      acc = (long)((double)acc + q);  // `long += double`
      v.tts_tick[i] = (int)acc;
    }
    double price = 0;
    v.cum_price[0] = 0.0;
    for (int i = 0; i + 1 < v.n; ++i) {
      volatile double prod = ((double)v.tts_tick[i + 1] - (double)v.tts_tick[i]) * v.ts[i];
      price += prod;
      v.cum_price[i + 1] = price;
    }
  }
  v.open_lo = open_ms + 30LL * 60000; v.close_hi = close_ms - 30LL * 60000;
  return true;
}

static int derive(rlm_handle_s* h) {
  const rlm_config& c = h->cfg;
  DevParams& p = h->hp;
  memset(&p, 0, sizeof(p));
  if (c.n_envs <= 0) return fail(RLM_ERR_INVALID_ARGUMENT, "n_envs must be positive");
  if (c.n_tilings != RLM_N_TILINGS) return fail(RLM_ERR_UNSUPPORTED, "the CUDA path maps tiling j to lane j: n_tilings must be 32");
  if (c.n_actions < 1 || c.n_actions > RLM_MAX_ACTIONS) return fail(RLM_ERR_UNSUPPORTED, "n_actions must be in 1..9 (Intraday::DoAction has 9 actions)");
  if (c.algorithm < RLM_ALGO_Q_LEARN || c.algorithm > RLM_ALGO_DOUBLE_R_LEARN)
    return fail(RLM_ERR_INVALID_ARGUMENT, "Please specify a valid learning algorithm!");  // main.cpp:188-189
  if (c.policy_type < RLM_POLICY_GREEDY || c.policy_type > RLM_POLICY_BOLTZMANN)
    return fail(RLM_ERR_INVALID_ARGUMENT, "Please specify a valid policy!");  // main.cpp:164-165
  if (c.shared_policy && c.algorithm >= RLM_ALGO_R_LEARN)
    return fail(RLM_ERR_UNSUPPORTED, "shared_policy is defined for q_learn, sarsa and double_q_learn (rho of the R-learning agents is per agent)");
  if (c.memory_size < 1 || c.memory_size > 2147483647LL) return fail(RLM_ERR_INVALID_ARGUMENT, "memory_size must fit the reference's int tile index");
  if (c.n_state_vars < 4 || c.n_state_vars > RLM_N_STATE_MAX) return fail(RLM_ERR_INVALID_ARGUMENT, "state.variables needs 4..13 entries (State::populateFeatures splits at 3)");
  if (c.n_bands < 1 || c.n_bands > RLM_MAX_BANDS) return fail(RLM_ERR_INVALID_ARGUMENT, "bad venue table");
  if (c.order_size <= 0) return fail(RLM_ERR_RUNTIME, "Order size must be non-zero and positive.");
  if (c.tp_lookback < 1) return fail(RLM_ERR_INVALID_ARGUMENT, "target_price.lookback must be >= 1");
  if (c.shared_policy && c.random_init) return fail(RLM_ERR_UNSUPPORTED, "shared_policy with random_init is not supported");
  if (c.shared_policy && (c.memory_size & 1)) return fail(RLM_ERR_UNSUPPORTED, "shared_policy needs an even memory_size");
  p.n_envs = c.n_envs; p.n_actions = c.n_actions; p.algorithm = c.algorithm; p.policy_type = c.policy_type;
  p.reward_measure = c.reward_measure; p.n_state_vars = c.n_state_vars;
  for (int i = 0; i < c.n_state_vars; ++i) {
    if (c.state_vars[i] < 0 || c.state_vars[i] > RLM_VAR_LAST_ACTION) return fail(RLM_ERR_INVALID_ARGUMENT, "Unknown state variable");
    p.state_vars[i] = c.state_vars[i];
  }
  // inverted selector of base.cpp:101-112: yaml "midprice" -> tp::MicroPrice, anything else -> tp::MidPrice
  p.tp_is_micro = (c.target_price_type == RLM_TP_YAML_MIDPRICE) ? 1 : 0;
  p.l2p_book = (c.target_price_type == RLM_TP_YAML_BOOK) ? 1 : 0;  // intraday.cpp:64
  p.order_size = c.order_size; p.source = c.source; p.shared_policy = c.shared_policy;
  p.is_double = (c.algorithm == RLM_ALGO_DOUBLE_Q_LEARN || c.algorithm == RLM_ALGO_DOUBLE_R_LEARN) ? 1 : 0;
  p.beta = c.beta;
  p.pos_lb = c.pos_lb; p.pos_ub = c.pos_ub; p.memory_size = c.memory_size;
  p.m_pow2 = ((c.memory_size & (c.memory_size - 1)) == 0) ? 1 : 0;
  p.m_magic = (unsigned long long)((((unsigned __int128)1) << 64) / (unsigned __int128)c.memory_size);
  if (c.memory_size == 1) p.m_magic = ~0ull;
  for (int a = 0; a < RLM_MAX_ACTIONS; ++a)  // hash_UNH term of the action integer for feature group 0 (3 floats + tiling + int)
    p.ra_m[a] = (int)((unsigned long long)rlm_rndseq_table[(a + 449 * 4) & 2047] % (unsigned long long)c.memory_size);
  for (int g = 0; g < 3; ++g) {
    const int nf = (g == 0) ? 3 : ((g == 1) ? c.n_state_vars - 3 : c.n_state_vars);
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) p.rg[g][a] = rlm_rndseq_table[(g * c.n_actions + a + 449 * (nf + 1)) & 2047];
  }
  p.scratch_bytes = (int)rlm_scratch_bytes(p.is_double);
  p.occ_words = (int)((c.memory_size + 31) / 32);
  // independent policies with a bitmap of <= 16 KB (memory_size <= 2^17): the 3-warp learner kernel keeps the env's
  // bitmap in shared memory for the step, so the 1728 bit tests never touch the global load path
  p.occ_smem_words = 0;  // round 2: the bitmap is maintained by the fallback kernels but never consulted
  p.gl = (float)(c.gamma * c.lambda);  // Traces::decay(float rate) narrows gamma*lambda (A11)
  for (int i = 0; i < 3; ++i) p.gw[i] = c.group_weights[i];
  p.gamma = c.gamma;
  p.damping = c.damping_factor; p.pos_weight = c.pos_weight; p.trd_weight = c.trd_weight; p.pnl_weight = c.pnl_weight;
  p.ewma_alpha = 2.0 / (std::max(c.lb_rsi, 1) + 1.0);  // accumulators.cpp:149-154
  // windows: base.cpp:35-50 (max(lookback,1)) + target price lookback
  int ws[RLM_NWIN];
  ws[W_MID] = std::max(c.lb_mpm, 1); ws[W_VLT] = std::max(c.lb_vlt, 1);
  ws[W_VNUM] = std::max(c.lb_vwap, 1); ws[W_VDEN] = std::max(c.lb_vwap, 1);
  ws[W_SPREAD] = std::max(c.spread_lookback, 1); ws[W_TP] = c.tp_lookback;
  ws[W_ASKTX] = std::max(c.lb_svl, 1); ws[W_BIDTX] = std::max(c.lb_svl, 1);
  ws[W_PNLUP] = std::max(c.pnl_lookback, 1); ws[W_PNLDN] = std::max(c.pnl_lookback, 1);
  int off = 0;
  for (int w = 0; w < RLM_NWIN; ++w) { p.win_size[w] = ws[w]; p.win_off[w] = off; off += ws[w]; }
  p.ring_total = off;
  p.env_stride = (int)((sizeof(EnvHdr) + (size_t)off * 8 + 15) & ~(size_t)15);
  // trace capacity: an entry survives k decays while (gamma*lambda)^k >= 0.01 (traces.cpp:30-38)
  int cap = c.trace_cap;
  if (cap <= 0) {
    double gl = (double)p.gl;
    int life = 1;
    if (gl > 0.0 && gl < 1.0) life = (int)ceil(log(0.01) / log(gl)) + 1;
    else if (gl >= 1.0) return fail(RLM_ERR_UNSUPPORTED, "gamma*lambda >= 1 needs an explicit trace_cap");
    cap = RLM_N_TILINGS * (life + 1);
    if (cap > 100000) return fail(RLM_ERR_UNSUPPORTED, "derived trace_cap exceeds MAX_NONZERO_TRACES (traces.h:10); set trace_cap");
  }
  p.trace_cap = (cap + 31) & ~31;
  p.record_envs = std::min(std::max(c.record_envs, 0), c.n_envs);
  p.record_cap = std::max(c.record_cap, 0);
  p.env_index0 = c.env_index0;
  p.flow = c.flow;
  std::string why;
  if (!venue_derive(p.venue, c.n_bands, c.band_px, c.band_ts, c.open_ms, c.close_ms, why)) return fail(RLM_ERR_INVALID_ARGUMENT, why);
  h->cfg_venue = p.venue;
  return RLM_OK;
}

static cudaError_t launch_agent_on(rlm_handle_s* h, const DevPtrs& ptr, const DynParams& d, int tslot, int stage, cudaStream_t st) {
  const int n = d.n_sub > 0 ? d.n_sub : h->cfg.n_envs;  // worst case: every env of the (sub-)batch is ready
  // backtest mode: the greedy evaluation step is the same for every algorithm and for independent and shared policies
  if (d.backtest) return rlm_launch_eval(ptr, d, n, h->hp.is_double, tslot, h->n_sms, st);
  // Q-learning / SARSA / Double-Q training: the one-warp-per-env learner (rlm_learn.cuh).  The R-learning agents' third
  // evaluation stays on the three-warp kernel's EXTRAS instantiation.
  if (h->agent_variant == 4 && h->cfg.algorithm < RLM_ALGO_R_LEARN) {
    // small per-env tables: the whole table is staged in shared memory by one bulk copy per step (rlm_learn_staged_kernel)
    if (h->staged && stage == 0) return rlm_launch_learn_staged(ptr, d, n, h->cfg.memory_size, tslot, h->n_sms, st);
    // steps a launch usually finds: ~29 % of the envs per tick, ~57 % per round of at most three ticks
    return rlm_launch_learn(ptr, d, n, h->hp.is_double, tslot, h->n_sms, stage, h->in_rounds ? (n * 3 + 4) / 5 : (n * 3 + 9) / 10, st);
  }
  if (h->agent_variant >= 3) {
    const int full = (h->cfg.algorithm >= RLM_ALGO_R_LEARN) ? 1 : 0;
    return rlm_launch_agent3(ptr, d, n, h->hp.is_double, h->hp.occ_smem_words, tslot, h->n_sms, stage, full, st);
  }
  return rlm_launch_agent(ptr, d, n, h->hp.scratch_bytes, tslot, h->n_sms, stage, st);
}
static cudaError_t launch_agent_any(rlm_handle_s* h, const DynParams& d, int tslot, int stage) {
  return launch_agent_on(h, h->ptr, d, tslot, stage, h->stream);
}

static int upload_params(rlm_handle_s* h) {
  if (g_params_owner != h) {
    CK(cudaDeviceSynchronize());  // kernels of the previous owner still read its constants
    CK(rlm_upload_params(&h->hp, &h->dm));
    g_params_owner = h;
  }
  return RLM_OK;
}

static int create_impl(const rlm_config* cfg, rlm_handle_s* h);

int rlm_create(const rlm_config* cfg, rlm_handle* out) {
  API_LOCK;
  if (!cfg || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  *out = nullptr;
  int ndev = 0;
  cudaError_t ce = cudaGetDeviceCount(&ndev);
  if (ce != cudaSuccess || ndev == 0)
    return fail(RLM_ERR_NO_DEVICE, std::string("no CUDA device: ") + (ce == cudaSuccess ? "device count is 0" : cudaGetErrorString(ce)) +
                                       " (this library has no CPU fallback)");
  if (cfg->device < 0 || cfg->device >= ndev) return fail(RLM_ERR_INVALID_ARGUMENT, "bad device ordinal");
  rlm_handle_s* h = new rlm_handle_s();
  h->cfg = *cfg;
  memset(&h->ptr, 0, sizeof(h->ptr));
  int rc = derive(h);
  if (rc != RLM_OK) { delete h; return rc; }
  rc = create_impl(cfg, h);
  if (rc != RLM_OK) {  // every stream, event and device buffer made so far goes back
    const std::string keep = g_err;
    rlm_destroy(h);
    g_err = keep;
    return rc;
  }
  *out = h;
  return RLM_OK;
}

static int create_impl(const rlm_config* cfg, rlm_handle_s* h) {
  CK(cudaSetDevice(cfg->device));
  {
    // theta dominates: fail with a readable message instead of an out-of-memory half way through the allocations
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    const double need = (double)(cfg->shared_policy ? 1 : cfg->n_envs) * (double)h->hp.memory_size * 8.0 * (h->hp.is_double ? 2 : 1) +
                        (double)cfg->n_envs * ((double)h->hp.env_stride + 8.0 * h->hp.trace_cap + 2.0 * 312 * 8 + 768);
    if (need > (double)free_b)
      return fail(RLM_ERR_INVALID_ARGUMENT, "n_envs x memory_size needs " + std::to_string((long long)(need / 1e6)) + " MB of device memory, " +
                                                std::to_string((long long)(free_b / 1e6)) + " MB are free");
  }
  CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking));
  const DevParams& p = h->hp;
  h->n_policies = cfg->shared_policy ? 1 : cfg->n_envs;
  h->env_bytes = (size_t)p.env_stride * cfg->n_envs;
  CK(cudaMalloc(&h->ptr.env, h->env_bytes));
  size_t th_bytes = (size_t)h->n_policies * (size_t)p.memory_size * 8;
  CK(cudaMalloc(&h->ptr.theta, th_bytes));
  CK(cudaMemsetAsync(h->ptr.theta, 0, th_bytes, h->stream));
  if (p.is_double) {
    CK(cudaMalloc(&h->ptr.theta_b, th_bytes));
    CK(cudaMemsetAsync(h->ptr.theta_b, 0, th_bytes, h->stream));
  }
  {
    // occupancy bitmap: clear = "theta entry is still exactly +0.0"; random_init makes every entry nonzero
    size_t obytes = (size_t)h->n_policies * (size_t)p.occ_words * 4;
    CK(cudaMalloc(&h->ptr.occ, obytes));
    CK(cudaMemsetAsync(h->ptr.occ, cfg->random_init ? 0xFF : 0x00, obytes, h->stream));
  }
  if (cfg->shared_policy) {
    size_t dbytes = (size_t)(p.is_double ? 2 : 1) * (size_t)p.memory_size * 8;
    CK(cudaMalloc(&h->ptr.dtheta, dbytes));
    CK(cudaMemsetAsync(h->ptr.dtheta, 0, dbytes, h->stream));
  }
  CK(cudaMalloc(&h->ptr.trace_f, (size_t)cfg->n_envs * p.trace_cap * 4));
  CK(cudaMalloc(&h->ptr.trace_e, (size_t)cfg->n_envs * p.trace_cap * 4));
  CK(cudaMalloc(&h->ptr.mt_pol, (size_t)cfg->n_envs * 312 * 8));
  if (p.is_double || cfg->random_init) CK(cudaMalloc(&h->ptr.mt_agt, (size_t)cfg->n_envs * 312 * 8));
  if (p.record_envs > 0 && p.record_cap > 0) {
    CK(cudaMalloc(&h->ptr.records, (size_t)p.record_envs * p.record_cap * sizeof(rlm_step_record)));
    CK(cudaMalloc(&h->ptr.record_count, (size_t)p.record_envs * 4));
    CK(cudaMemsetAsync(h->ptr.record_count, 0, (size_t)p.record_envs * 4, h->stream));
  } else {
    h->hp.record_envs = 0;
  }
  CK(cudaMalloc(&h->ptr.counters, 8 * 8));
  CK(cudaMemsetAsync(h->ptr.counters, 0, 8 * 8, h->stream));
  if (cfg->source == RLM_SOURCE_TAPE) {  // per-env cursors of the day library: every env is on an empty day until rlm_load_days
    CK(cudaMalloc(&h->ptr.tape_cur, (size_t)cfg->n_envs * sizeof(int2)));
    CK(cudaMalloc(&h->ptr.tape_lo, (size_t)cfg->n_envs * sizeof(int)));
    CK(cudaMemsetAsync(h->ptr.tape_cur, 0, (size_t)cfg->n_envs * sizeof(int2), h->stream));
    CK(cudaMemsetAsync(h->ptr.tape_lo, 0, (size_t)cfg->n_envs * sizeof(int), h->stream));
  }
  g_params_owner = nullptr;
  int rc = upload_params(h);
  if (rc != RLM_OK) return rc;
  CK(rlm_launch_init(h->ptr, cfg->n_envs, 0, h->stream));
  CK(rlm_launch_seed(h->ptr, cfg->n_envs, cfg->random_seed, h->stream));
  if (cfg->random_init) CK(rlm_launch_random_init(h->ptr, h->n_policies, h->stream));
  // Agent ctor: alpha(alpha_start) (agent.cpp:25); EpsilonGreedy ctor: eps(eps) (policy.cpp:63, main.cpp:149-154)
  h->alpha = cfg->alpha_start;
  h->eps = (double)cfg->eps_init;
  h->tau = (double)cfg->tau_init;  // Boltzmann ctor (policy.cpp:85-96, main.cpp:157-162)
  memset(&h->dyn, 0, sizeof(h->dyn));
#ifdef RLM_TIMING
  if (const char* s = getenv("RLM_DEBUG_FLAGS")) h->dyn.debug_flags = atoi(s);
#endif
  if (const char* s = getenv("RLM_ENV_HASH")) h->dyn.env_hash = atoi(s) != 0;
  if (const char* s = getenv("RLM_ROUND_CAP")) h->dyn.round_cap = std::max(0, atoi(s));
  CK(cudaDeviceGetAttribute(&h->n_sms, cudaDevAttrMultiProcessorCount, cfg->device));
  CK(cudaMalloc(&h->ptr.ready, (size_t)cfg->n_envs * 4));
  CK(cudaMalloc(&h->ptr.hsum, (size_t)cfg->n_envs * 3 * 32 * 8));
  h->ready_cap = RLM_READY_CAP;
  CK(cudaMalloc(&h->ptr.ready_count, (size_t)2 * RLM_LIVE_OFF * 4));  // ready counters + live counters (rlm_types.h)
  CK(cudaMemset(h->ptr.ready_count, 0, (size_t)2 * RLM_LIVE_OFF * 4));
  CK(cudaMalloc(&h->ptr.runctl, sizeof(RunCtl)));
  CK(cudaMemset(h->ptr.runctl, 0, sizeof(RunCtl)));
  CK(cudaMallocHost(&h->h_live, RLM_MAX_SUB * 2 * sizeof(int)));
  for (int s = 0; s < RLM_MAX_SUB; ++s)
    for (int i = 0; i < 2; ++i) CK(cudaEventCreateWithFlags(&h->ev_live[s][i], cudaEventDisableTiming));
  if (const char* s = getenv("RLM_ROUND_STREAMS")) { const int v = atoi(s); if (v >= 1 && v <= RLM_MAX_SUB) h->round_streams = v; }
  // sub-batches of the tick-synchronous engine (see rlm_handle_s::n_sub); RLM_SUBBATCHES overrides
  h->n_sub = 1;  // (co-resident tick and learner kernels slow each other down as much as they overlap)
  h->staged = !h->hp.is_double && !cfg->shared_policy && cfg->memory_size * 8 <= 65536 && (cfg->memory_size % 2) == 0;
  if (const char* s = getenv("RLM_STAGED")) h->staged = h->staged && atoi(s) != 0;
  // Large batches are throughput-bound: what counts is how many steps an SM keeps in flight.  The one-warp learner holds
  // 20 KB of shared memory per step (9 per SM); the round-1 three-warp kernel holds 7 KB and 64 registers (10 CTAs = 30
  // warps per SM) and measures 30 % faster at 65 536 envs (C2), so it takes over above 16 384 envs unless the table is
  // small enough to be staged whole.
  if (cfg->n_envs > 16384 && !h->staged) h->agent_variant = 3;
  if (const char* s = getenv("RLM_AGENT_VARIANT")) { const int v = atoi(s); h->agent_variant = (v == 1 || v == 3) ? v : 4; }
  // the one-warp learners pack (feature << 4 | action) into one word of their tile table (rlm_learn.cuh)
  if (cfg->memory_size > (1LL << 27) && h->agent_variant == 4) h->agent_variant = 3;
  if (const char* s = getenv("RLM_GRAPHS")) h->use_graphs = atoi(s) != 0;
  if (const char* s = getenv("RLM_SUBBATCHES")) { const int v = atoi(s); if (v >= 1 && v <= RLM_MAX_SUB) h->n_sub = cfg->shared_policy ? 1 : v; }
  if (std::max(h->n_sub, h->round_streams) > 1) {
    CK(cudaEventCreateWithFlags(&h->ev_fork, cudaEventDisableTiming));
    for (int s = 0; s < std::max(h->n_sub, h->round_streams); ++s) {
      CK(cudaStreamCreateWithFlags(&h->sub_stream[s], cudaStreamNonBlocking));
      CK(cudaEventCreateWithFlags(&h->ev_join[s], cudaEventDisableTiming));
    }
  }
  {
    int dev_smem = 0;
    CK(cudaDeviceGetAttribute(&dev_smem, cudaDevAttrMaxSharedMemoryPerBlockOptin, cfg->device));
    if (rlm_agent_smem_bytes(8, p.scratch_bytes) > (size_t)dev_smem) return fail(RLM_ERR_UNSUPPORTED, "agent kernel shared memory exceeds the device limit");
  }
  // persistent engine: queue + flags
  {
    // agent CTAs must all be resident; leave at least a quarter of the slots to env CTAs
    const int resident = rlm_run_max_resident_ctas(p.scratch_bytes, h->n_sms);
    const int n_env_ctas = (cfg->n_envs + 127) / 128;
    int want = (cfg->n_envs + 3) / 4;  // one agent warp per env at most
    int cap = resident - std::min(n_env_ctas, std::max(resident / 4, 1));
    h->n_agent_ctas = std::max(1, std::min(want, cap));
    if (const char* s = getenv("RLM_AGENT_CTAS")) { int v = atoi(s); if (v > 0 && v < resident) h->n_agent_ctas = v; }
    // Every agent warp holds one ticket while it waits, and ticket t waits on slot t % q_size: the ring needs a slot per
    // waiting warp as well as per env.  With fewer slots (1 or 2 envs: 4 agent warps) several warps spin on one slot and
    // more than one can take the same push -- two learner steps on one env at once.
    int q = 1;
    while (q < cfg->n_envs || q < h->n_agent_ctas * RLM_RUN_WARPS) q <<= 1;
    h->ptr.q_size = q;
    CK(cudaMalloc(&h->ptr.q_slots, (size_t)q * 4));
    CK(cudaMemsetAsync(h->ptr.q_slots, 0xFF, (size_t)q * 4, h->stream));
    CK(cudaMalloc(&h->ptr.ag_done, (size_t)cfg->n_envs * 4));
    CK(cudaMemsetAsync(h->ptr.ag_done, 0, (size_t)cfg->n_envs * 4, h->stream));
    CK(cudaMalloc(&h->d_qctl, 4 * 4));
    h->ptr.q_head = h->d_qctl; h->ptr.q_tail = h->d_qctl + 1; h->ptr.env_warps_done = h->d_qctl + 2; h->ptr.q_done = (int*)(h->d_qctl + 3);
    // engines: 's' tick-synchronous (two launches per tick), 'F' fused persistent round-2 kernel, 'f' round-1 fused kernel,
    // 'p' persistent queue
    if (const char* s = getenv("RLM_ENGINE")) h->engine = (s[0] == 'p') ? 0 : ((s[0] == 'f') ? 2 : ((s[0] == 'F') ? 3 : 1));
    // warp-per-env ticks minimise latency (small batches); thread-per-env ticks are ~2x cheaper in issue slots
    h->env_variant = (cfg->n_envs > 16384) ? 1 : 0;
    if (const char* s = getenv("RLM_ENV_VARIANT")) h->env_variant = atoi(s) ? 1 : 0;
    // The round-paced engine needs envs that never interact and the warp-per-env tick kernel.  With a cap on the ticks
    // an env runs per round (RLM_ROUND_CAP, default 3) it is the faster engine for long run calls: a round hands the
    // learner kernel ~2 300 steps instead of ~1 200 and pays the two launch gaps once per 2.2 ticks.  Without a cap the
    // round waits for the env with the longest run of unchanged midprices.  Short calls stay tick-synchronous: a call ends with a tail
    // of thinly populated rounds (envs drift apart by a few ticks), which only a long call amortises, and the
    // round-paced call returns only when the device is nearly done (no overlap with the next chunk's upload).
    // RLM_ROUNDS=1 forces it for every call, RLM_ROUNDS=0 (or an explicit RLM_ENGINE) switches it off.
    h->rounds = false;
    h->rounds_auto = !cfg->shared_policy && h->env_variant == 0 && h->engine == 1 && !getenv("RLM_ENGINE") && cfg->algorithm < RLM_ALGO_R_LEARN;
    if (const char* s = getenv("RLM_ROUNDS")) {
      h->rounds = atoi(s) != 0 && !cfg->shared_policy && h->env_variant == 0;
      h->rounds_auto = false;
    }
    if (!getenv("RLM_ROUND_CAP")) h->dyn.round_cap = 3;
    if (const char* s = getenv("RLM_PDL")) rlm_set_pdl(atoi(s));  // programmatic dependent launch of the per-tick kernels (default off: slower when measured)
    if (const char* s = getenv("RLM_AGENT_VARIANT")) { const int v = atoi(s); h->agent_variant = (v == 1 || v == 3) ? v : 4; }
    if (cfg->memory_size > (1LL << 27)) {  // (packed tile table of the one-warp learner step, also inside the fused engine)
      if (h->agent_variant == 4) h->agent_variant = 3;
      if (h->engine == 3) h->engine = 1;
    }
  }
  if (cfg->source == RLM_SOURCE_TAPE) {
    if (h->engine != 1) return fail(RLM_ERR_UNSUPPORTED, "the tape source runs on the tick-synchronous and round-paced engines (RLM_ENGINE=F|f|p read the stream source only)");
    h->dyn.tape_l2 = 1;
    if (const char* s = getenv("RLM_TAPE_PREFETCH")) h->dyn.tape_l2 = atoi(s) != 0;
  }
  // theta is gathered 8 bytes at a time from random addresses: do not let L2 promote misses to 64/128-byte fetches
  // (device-wide, and it stays for the lifetime of the hosting process)
  cudaDeviceSetLimit(cudaLimitMaxL2FetchGranularity, 32);
  CK(cudaStreamSynchronize(h->stream));
  return RLM_OK;
}

int rlm_destroy(rlm_handle h) {
  API_LOCK;
  if (!h) return RLM_OK;
  cudaSetDevice(h->cfg.device);
  cudaStreamSynchronize(h->stream);
  cudaFree(h->ptr.env); cudaFree(h->ptr.theta); cudaFree(h->ptr.theta_b); cudaFree(h->ptr.dtheta);
  cudaFree(h->ptr.trace_f); cudaFree(h->ptr.trace_e); cudaFree(h->ptr.mt_pol); cudaFree(h->ptr.mt_agt);
  cudaFree(h->ptr.records); cudaFree(h->ptr.record_count); cudaFree(h->ptr.counters);
  cudaFree(h->d_gather); if (h->h_gather) cudaFreeHost(h->h_gather);
  if (h->copy_stream) { cudaStreamSynchronize(h->copy_stream); cudaStreamDestroy(h->copy_stream); }
  for (int i = 0; i < 2; ++i) {
    cudaFree(h->d_stream[i]);
    if (h->ev_copied[i]) cudaEventDestroy(h->ev_copied[i]);
    if (h->ev_consumed[i]) cudaEventDestroy(h->ev_consumed[i]);
  }
  cudaFree(h->ptr.ready); cudaFree(h->ptr.ready_count); cudaFree(h->ptr.occ); cudaFree(h->ptr.hsum);
  cudaFree(h->ptr.runctl); if (h->h_live) cudaFreeHost(h->h_live);
  cudaFree((void*)h->ptr.tape); cudaFree(h->ptr.tape_cur); cudaFree(h->ptr.tape_lo);
  cudaFree((void*)h->dm.markets); cudaFree(h->dm.env_market); cudaFree(h->dm.rec_fixed);
  for (auto& es : h->ev_live) for (auto e : es) if (e) cudaEventDestroy(e);
  cudaFree(h->ptr.q_slots); cudaFree(h->ptr.ag_done); cudaFree(h->d_qctl);
  for (auto e : h->ev) cudaEventDestroy(e);
  for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
  if (h->ev_fork) cudaEventDestroy(h->ev_fork);
  for (int s = 0; s < RLM_MAX_SUB; ++s) {
    if (h->sub_stream[s]) { cudaStreamSynchronize(h->sub_stream[s]); cudaStreamDestroy(h->sub_stream[s]); }
    if (h->ev_join[s]) cudaEventDestroy(h->ev_join[s]);
  }
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  if (g_params_owner == h) g_params_owner = nullptr;
  delete h;
  return RLM_OK;
}

int rlm_set_stream(rlm_handle h, void* cuda_stream) {
  API_LOCK;
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  if (h->own_stream && h->stream) cudaStreamDestroy(h->stream);
  if (cuda_stream) { h->stream = (cudaStream_t)cuda_stream; h->own_stream = false; }
  else { CK(cudaStreamCreateWithFlags(&h->stream, cudaStreamNonBlocking)); h->own_stream = true; }
  return RLM_OK;
}

int rlm_reset(rlm_handle h) {
  API_LOCK;
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  int rc = upload_params(h);
  if (rc) return rc;
  CK(rlm_launch_init(h->ptr, h->cfg.n_envs, 1, h->stream));
  h->stream_cursor = 0; h->stream_ticks = 0;
  return RLM_OK;
}

int rlm_set_mode(rlm_handle h, int32_t mode) {
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  if (mode != RLM_MODE_TRAIN && mode != RLM_MODE_BACKTEST) return fail(RLM_ERR_INVALID_ARGUMENT, "unknown mode");
  if (mode == RLM_MODE_BACKTEST && h->engine != 1 && h->engine != 3) return fail(RLM_ERR_UNSUPPORTED, "backtest mode runs on the tick-synchronous engine only");
  if (h->dyn.backtest != mode) h->graph_warm = false;  // (the other mode's kernel: its first call launches directly, see run_ticks_impl)
  h->dyn.backtest = mode;
  return RLM_OK;
}

int rlm_new_env(rlm_handle h, const rlm_flow_params* flow) {
  API_LOCK;
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  if (flow && h->cfg.source == RLM_SOURCE_TAPE)
    return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_new_env: a tape handle replays its day library (rlm_assign_days changes days); pass flow = NULL");
  CK(cudaSetDevice(h->cfg.device));
  if (flow) {
    CK(cudaStreamSynchronize(h->stream));  // running kernels read the old parameters from constant memory
    h->cfg.flow = *flow;
    h->hp.flow = *flow;
    if (g_params_owner == h) g_params_owner = nullptr;  // force the re-upload (after a device-wide synchronisation)
  }
  int rc = upload_params(h);
  if (rc) return rc;
  CK(rlm_launch_init(h->ptr, h->cfg.n_envs, 2, h->stream));
  if (h->ptr.records) CK(cudaMemsetAsync(h->ptr.record_count, 0, (size_t)h->hp.record_envs * 4, h->stream));
  if (h->dm.rec_fixed) CK(cudaMemsetAsync(h->dm.rec_fixed, 0, (size_t)h->hp.record_envs * sizeof(int), h->stream));
  h->stream_cursor = 0; h->stream_ticks = 0;
  return RLM_OK;
}

int rlm_set_flow(rlm_handle h, const rlm_flow_params* flow) {
  API_LOCK;
  if (!h || !flow) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_set_flow: bad arguments");
  if (h->cfg.source != RLM_SOURCE_GENERATOR)
    return fail(RLM_ERR_INVALID_ARGUMENT, h->cfg.source == RLM_SOURCE_TAPE ? "rlm_set_flow: a tape handle changes days with rlm_assign_days"
                                                                           : "rlm_set_flow: a stream handle loads its next day with rlm_load_ticks");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));  // running kernels read the old parameters from constant memory
  h->cfg.flow = *flow;
  h->hp.flow = *flow;
  if (g_params_owner == h) g_params_owner = nullptr;  // rlm_reset uploads them again (after a device-wide synchronisation)
  return RLM_OK;
}

int rlm_load_ticks(rlm_handle h, const rlm_tick_msg* msgs, int32_t n_ticks) {
  API_LOCK;
  if (!h || !msgs || n_ticks <= 0) return fail(RLM_ERR_INVALID_ARGUMENT, "bad arguments");
  if (h->cfg.source != RLM_SOURCE_STREAM)
    return fail(RLM_ERR_INVALID_ARGUMENT, h->cfg.source == RLM_SOURCE_TAPE ? "rlm_load_ticks: a tape handle reads its day library (rlm_load_days)"
                                                                           : "handle was created with source = generator");
  CK(cudaSetDevice(h->cfg.device));
  size_t n = (size_t)n_ticks * h->cfg.n_envs;
  if (!h->copy_stream) {
    CK(cudaStreamCreateWithFlags(&h->copy_stream, cudaStreamNonBlocking));
    for (int i = 0; i < 2; ++i) {
      CK(cudaEventCreateWithFlags(&h->ev_copied[i], cudaEventDisableTiming));
      CK(cudaEventCreateWithFlags(&h->ev_consumed[i], cudaEventDisableTiming));
    }
  }
  const int nb = h->stream_buf ^ 1;
  if (n > h->stream_cap[nb]) {
    CK(cudaStreamSynchronize(h->stream));
    CK(cudaStreamSynchronize(h->copy_stream));
    cudaFree(h->d_stream[nb]);
    h->d_stream[nb] = nullptr; h->stream_cap[nb] = 0;
    CK(cudaMalloc(&h->d_stream[nb], n * sizeof(rlm_tick_msg)));
    h->stream_cap[nb] = n;
    h->consumed_valid[nb] = false;
  }
  // the idle chunk may still be read by kernels of an earlier run call
  if (h->consumed_valid[nb]) CK(cudaStreamWaitEvent(h->copy_stream, h->ev_consumed[nb], 0));
  CK(cudaMemcpyAsync(h->d_stream[nb], msgs, n * sizeof(rlm_tick_msg), cudaMemcpyHostToDevice, h->copy_stream));
  CK(cudaEventRecord(h->ev_copied[nb], h->copy_stream));
  CK(cudaStreamWaitEvent(h->stream, h->ev_copied[nb], 0));
  h->stream_buf = nb;
  h->ptr.stream = h->d_stream[nb];
  h->stream_ticks = n_ticks;
  h->stream_cursor = 0;
  return RLM_OK;
}

// ---- TAPE source -------------------------------------------------------------------------------------------------
static int tape_check(rlm_handle h) {
  if (h->cfg.source == RLM_SOURCE_TAPE && h->day_off.empty()) return fail(RLM_ERR_INVALID_ARGUMENT, "no day library loaded (rlm_load_days)");
  return RLM_OK;
}
// Day markets on: the learner kernels, which read the config's market from the __constant__ block, fill a record's
// terminal flag from it (fill_record).  That copy is made to never close, so the flag they write is the date change of
// Intraday::isTerminal alone, and rlm_fix_terminal_kernel adds the close of the env's own market.  The tick kernels read
// every env's market from ptr.markets (the MKT instantiations), so nothing else reads the constant copy's hours.
static void day_markets_on(rlm_handle h, bool on) {
  h->hp.venue = h->cfg_venue;
  if (on) { h->hp.venue.open_lo = LLONG_MIN; h->hp.venue.close_hi = LLONG_MAX; }
  g_params_owner = nullptr;  // upload again
}
// the records written since the last call get the close of their env's current market (day markets on, params uploaded;
// nothing to do unless learner work was enqueued since)
static int fix_records(rlm_handle h) {
  if (!h->dm.markets || h->hp.record_envs <= 0 || !h->rec_dirty) return RLM_OK;
  int rc = upload_params(h);
  if (rc) return rc;
  CK(rlm_launch_fix_terminal(h->ptr, h->hp.record_envs, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  h->rec_dirty = false;
  return RLM_OK;
}
// envs env0 .. env0+n-1 replay days day[0..n-1] from their first message, each under its day's market (the handle's
// work has finished).  remarket: the markets themselves were replaced (rlm_set_day_markets), so every env's market
// counts as changed even where its index stays the same.
static int tape_assign(rlm_handle h, int env0, int n, const int32_t* day, bool remarket = false) {
  std::vector<int2> cur(n);
  std::vector<int> lo(n);
  for (int i = 0; i < n; ++i) {
    lo[i] = (int)h->day_off[day[i]];
    cur[i] = make_int2(lo[i], (int)h->day_off[day[i] + 1]);
    h->env_day[env0 + i] = day[i];
  }
  CK(cudaMemcpy(h->ptr.tape_cur + env0, cur.data(), (size_t)n * sizeof(int2), cudaMemcpyHostToDevice));
  CK(cudaMemcpy(h->ptr.tape_lo + env0, lo.data(), (size_t)n * sizeof(int), cudaMemcpyHostToDevice));
  if (!h->dm.env_market) return RLM_OK;  // (day markets were never set: every env is on the config's market)
  std::vector<int32_t> mk(n);
  bool changed = remarket;
  for (int i = 0; i < n; ++i) {
    mk[i] = h->day_market.empty() ? -1 : h->day_market[day[i]];
    changed = changed || mk[i] != h->env_mkt[env0 + i];
  }
  if (!changed) return RLM_OK;
  int rc = fix_records(h);  // (records so far belong to the old markets)
  if (rc) return rc;
  rc = upload_params(h);
  if (rc) return rc;
  rc = split_scratch(h, (size_t)n * 4);
  if (rc) return rc;
  CK(cudaMemcpy(h->d_gather, mk.data(), (size_t)n * 4, cudaMemcpyHostToDevice));
  CK(rlm_launch_env_market(h->ptr, env0, n, (const int*)h->d_gather, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  for (int i = 0; i < n; ++i) h->env_mkt[env0 + i] = mk[i];
  return RLM_OK;
}

int rlm_load_days(rlm_handle h, const rlm_tick_msg* msgs, const int64_t* day_offsets, int32_t n_days) {
  API_LOCK;
  if (!h || !msgs || !day_offsets || n_days <= 0) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_load_days: bad arguments");
  if (h->cfg.source != RLM_SOURCE_TAPE) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_load_days needs a handle created with source = tape");
  if (day_offsets[0] != 0) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_load_days: day_offsets[0] must be 0");
  for (int d = 0; d < n_days; ++d)
    if (day_offsets[d + 1] < day_offsets[d])
      return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_load_days: day_offsets must not decrease (day " + std::to_string(d) + ")");
  const int64_t n_msgs = day_offsets[n_days];
  if (n_msgs <= 0) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_load_days: the library holds no message");
  if (n_msgs > INT_MAX) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_load_days: a day library holds at most 2^31 - 1 messages");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));  // kernels of earlier calls may still read the old library and cursors
  {
    size_t free_b = 0, total_b = 0;
    CK(cudaMemGetInfo(&free_b, &total_b));
    const double need = (double)n_msgs * sizeof(rlm_tick_msg);
    const double have = (double)free_b + (h->day_off.empty() ? 0.0 : (double)h->day_off.back() * sizeof(rlm_tick_msg));
    if (need > have)
      return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_load_days: the library needs " + std::to_string((long long)(need / 1e6)) + " MB of device memory, " +
                                                std::to_string((long long)(have / 1e6)) + " MB are free");
  }
  // a new library drops the day markets of the old one: every day runs under the config's market again
  if (h->dm.markets) {
    int rc = fix_records(h);
    if (rc) return rc;
    cudaFree((void*)h->dm.markets);
    h->dm.markets = nullptr;
    h->day_market.clear();
    day_markets_on(h, false);
  }
  // the cached CUDA graphs hold the old library's address (DevPtrs is captured by value)
  for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
  h->graphs.clear();
  cudaFree((void*)h->ptr.tape);
  h->ptr.tape = nullptr;
  h->day_off.clear();
  rlm_tick_msg* d_lib = nullptr;
  CK(cudaMalloc(&d_lib, (size_t)n_msgs * sizeof(rlm_tick_msg)));
  h->ptr.tape = d_lib;
  CK(cudaMemcpy(d_lib, msgs, (size_t)n_msgs * sizeof(rlm_tick_msg), cudaMemcpyHostToDevice));
  h->day_off.assign(day_offsets, day_offsets + n_days + 1);
  h->env_day.assign(h->cfg.n_envs, 0);
  std::vector<int32_t> day(h->cfg.n_envs);
  for (int b = 0; b < h->cfg.n_envs; ++b) day[b] = b % n_days;
  return tape_assign(h, 0, h->cfg.n_envs, day.data());
}

int rlm_assign_days(rlm_handle h, int32_t env0, int32_t n, const int32_t* day) {
  API_LOCK;
  if (!h || (n > 0 && !day)) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_assign_days: bad arguments");
  if (h->cfg.source != RLM_SOURCE_TAPE) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_assign_days needs a handle created with source = tape");
  int rc = tape_check(h);
  if (rc) return rc;
  if (env0 < 0 || n < 0 || (int64_t)env0 + n > h->cfg.n_envs) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_assign_days: env range out of bounds");
  const int n_days = (int)h->day_off.size() - 1;
  for (int i = 0; i < n; ++i)
    if (day[i] < 0 || day[i] >= n_days)
      return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_assign_days: day " + std::to_string(day[i]) + " of env " + std::to_string(env0 + i) +
                                                " is not in the library (" + std::to_string(n_days) + " days)");
  if (n == 0) return RLM_OK;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  return tape_assign(h, env0, n, day);
}

int rlm_set_day_markets(rlm_handle h, const rlm_market* markets, int32_t n_markets, const int32_t* day_market, int32_t n_days) {
  API_LOCK;
  if (!h || !markets || !day_market || n_markets <= 0) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_set_day_markets: bad arguments");
  if (h->cfg.source != RLM_SOURCE_TAPE) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_set_day_markets needs a handle created with source = tape");
  int rc = tape_check(h);
  if (rc) return rc;
  if (n_days != (int)h->day_off.size() - 1)
    return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_set_day_markets: n_days is " + std::to_string(n_days) + ", the library holds " +
                                              std::to_string(h->day_off.size() - 1) + " days");
  std::vector<VenueD> v(n_markets);
  for (int k = 0; k < n_markets; ++k) {
    const rlm_market& m = markets[k];
    std::string why;
    if (!venue_derive(v[k], m.n_bands, m.band_px, m.band_ts, m.open_ms, m.close_ms, why))
      return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_set_day_markets: market " + std::to_string(k) + ": " + why);
  }
  for (int d = 0; d < n_days; ++d)
    if (day_market[d] < 0 || day_market[d] >= n_markets)
      return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_set_day_markets: day " + std::to_string(d) + " has market " + std::to_string(day_market[d]) +
                                                ", not in [0, " + std::to_string(n_markets) + ")");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  rc = fix_records(h);  // (records so far belong to the old markets)
  if (rc) return rc;
  VenueD* d_v = nullptr;
  CK(cudaMalloc(&d_v, (size_t)n_markets * sizeof(VenueD)));
  CK(cudaMemcpy(d_v, v.data(), (size_t)n_markets * sizeof(VenueD), cudaMemcpyHostToDevice));
  if (!h->dm.env_market) {
    CK(cudaMalloc(&h->dm.env_market, (size_t)h->cfg.n_envs * sizeof(int)));
    CK(cudaMemset(h->dm.env_market, 0xFF, (size_t)h->cfg.n_envs * sizeof(int)));  // -1: the config's market
    h->env_mkt.assign(h->cfg.n_envs, -1);
    if (h->hp.record_envs > 0) CK(cudaMalloc(&h->dm.rec_fixed, (size_t)h->hp.record_envs * sizeof(int)));
  }
  if (!h->dm.markets && h->hp.record_envs > 0)  // the records written so far carry the config's close already
    CK(cudaMemcpy(h->dm.rec_fixed, h->ptr.record_count, (size_t)h->hp.record_envs * sizeof(int), cudaMemcpyDeviceToDevice));
  cudaFree((void*)h->dm.markets);
  h->dm.markets = d_v;
  h->day_market.assign(day_market, day_market + n_days);
  day_markets_on(h, true);
  // the cached CUDA graphs hold the tick kernels without day markets
  for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
  h->graphs.clear();
  // every env back to the start of its day, now under the day's market
  std::vector<int32_t> day(h->env_day);
  return tape_assign(h, 0, h->cfg.n_envs, day.data(), true);
}

int rlm_get_tape_pos(rlm_handle h, int64_t* out) {
  API_LOCK;
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  if (h->cfg.source != RLM_SOURCE_TAPE) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_get_tape_pos needs a handle created with source = tape");
  const int B = h->cfg.n_envs;
  std::vector<int2> cur(B);
  std::vector<int> lo(B);
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(cur.data(), h->ptr.tape_cur, (size_t)B * sizeof(int2), cudaMemcpyDeviceToHost));
  CK(cudaMemcpy(lo.data(), h->ptr.tape_lo, (size_t)B * sizeof(int), cudaMemcpyDeviceToHost));
  for (int b = 0; b < B; ++b) out[b] = (int64_t)cur[b].x - lo[b];
  return RLM_OK;
}

static int run_ticks_impl(rlm_handle h, int32_t n_ticks);
static int run_rounds(rlm_handle h, const DynParams& d, int n_ticks);
#define RLM_ROUNDS_MIN_TICKS 128

int rlm_run_ticks(rlm_handle h, int32_t n_ticks) {
  API_LOCK;
  if (!h || n_ticks < 0) return fail(RLM_ERR_INVALID_ARGUMENT, "bad arguments");
  if (n_ticks == 0) return RLM_OK;
  CK(cudaSetDevice(h->cfg.device));
  h->rec_dirty = true;  // (learner steps write records)
  int rc = run_ticks_impl(h, n_ticks);
  if (rc == RLM_OK && h->cfg.source == RLM_SOURCE_STREAM && h->copy_stream) {
    // the chunk these launches read may be overwritten by the load after next
    CK(cudaEventRecord(h->ev_consumed[h->stream_buf], h->stream));
    h->consumed_valid[h->stream_buf] = true;
  }
  return rc;
}

// Round-paced engine.  A round = rlm_env_round_kernel (every live env ticks until its step ends or its n_ticks are used
// up) + the learner kernel over the envs that came back ready.  How many rounds a call needs is only known on the
// device (the env with the most steps in these n_ticks decides), so rounds are enqueued in groups of G -- one CUDA
// graph each -- and after every group the ready count of its last round comes back through pinned memory: zero means
// that every env has finished.  The host stays one group ahead of the device and stops when the group before the one it
// has just enqueued reports zero; the rounds enqueued beyond the end find nothing to do (their CTAs return after one
// load).  Unlike the tick-synchronous path the call therefore returns only when the device is (nearly) done.
static int run_rounds_impl(rlm_handle h, const DynParams& d, int n_ticks);
static int run_rounds(rlm_handle h, const DynParams& d, int n_ticks) {
  h->in_rounds = true;
  const int rc = run_rounds_impl(h, d, n_ticks);
  h->in_rounds = false;
  return rc;
}
static int run_rounds_impl(rlm_handle h, const DynParams& d, int n_ticks) {
  const int B = h->cfg.n_envs;
  RunCtl rc = {++h->run_seq, n_ticks, d.stream_off, d.stream_ticks, h->ptr.stream, 0};
  CK(rlm_launch_runctl(h->ptr, rc, h->stream));
  // sub-batches on their own streams: the learner kernel of one (throughput-bound: more steps than resident warps)
  // runs while the tick kernel of another (latency-bound: a few serial ticks per env) does
  const int S = h->profile ? 1 : std::max(1, std::min(h->round_streams, (B + 255) / 256));
  int sub0[RLM_MAX_SUB + 1];
  {
    const int per = (((B + S - 1) / S) + 31) & ~31;
    for (int s = 0; s <= S; ++s) sub0[s] = std::min(B, s * per);
  }
  int G = n_ticks >= 512 ? 32 : (n_ticks >= 128 ? 16 : 8);
  G = std::min(std::min(G, n_ticks + 1), h->ready_cap);
  const bool graphs = h->use_graphs && h->graph_warm && !h->profile;
  h->graph_warm = true;  // (the first call launches directly: function attributes are set outside any capture)
  if (h->profile) while ((int)h->ev.size() < 3 * G) { cudaEvent_t e; CK(cudaEventCreate(&e)); h->ev.push_back(e); }
  DynParams dts[RLM_MAX_SUB];
  DevPtrs pss[RLM_MAX_SUB];
  cudaGraphExec_t exec[RLM_MAX_SUB] = {};
  if (S > 1) CK(cudaEventRecord(h->ev_fork, h->stream));
  for (int s = 0; s < S; ++s) {
    cudaStream_t st = S > 1 ? h->sub_stream[s] : h->stream;
    if (S > 1) CK(cudaStreamWaitEvent(st, h->ev_fork, 0));
    DynParams& dt = dts[s];
    dt = d;
    dt.n_ticks = 0; dt.stream_off = 0; dt.stream_ticks = 0; dt.env0 = sub0[s]; dt.n_sub = sub0[s + 1] - sub0[s]; dt.sub_idx = s;
    DevPtrs& ps = pss[s];
    ps = h->ptr;
    ps.stream = nullptr;  // (read from *runctl: rlm_load_ticks swaps buffers between calls, the graphs stay)
    ps.ready = h->ptr.ready + sub0[s];
    ps.ready_count = h->ptr.ready_count + (size_t)s * h->ready_cap;
    if (!graphs || dt.n_sub <= 0) continue;
    for (auto& g : h->graphs)
      if (g.chunk == -G && memcmp(&g.d, &dt, sizeof(DynParams)) == 0) exec[s] = g.exec;
    if (!exec[s]) {
      if (h->graphs.size() >= 24) {
        CK(cudaStreamSynchronize(h->stream));
        for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec);
        h->graphs.clear();
        for (int q = 0; q < s; ++q) exec[q] = nullptr;  // (re-captured below when launched directly this call)
      }
      cudaGraph_t graph = nullptr;
      CK(cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal));
      cudaError_t ce = cudaMemsetAsync(ps.ready_count, 0, (size_t)G * 4, st);
      if (ce == cudaSuccess) ce = cudaMemsetAsync(ps.ready_count + RLM_LIVE_OFF, 0, (size_t)G * 4, st);
      for (int r = 0; r < G && ce == cudaSuccess; ++r) {
        ce = rlm_launch_env_round(ps, dt, dt.n_sub, r, st);
        if (ce == cudaSuccess) ce = launch_agent_on(h, ps, dt, r, 0, st);
      }
      cudaError_t ce2 = cudaStreamEndCapture(st, &graph);
      if (ce != cudaSuccess || ce2 != cudaSuccess) { if (graph) cudaGraphDestroy(graph); CK(ce != cudaSuccess ? ce : ce2); }
      ce = cudaGraphInstantiate(&exec[s], graph, 0);
      cudaGraphDestroy(graph);
      CK(ce);
      h->graphs.push_back({-G, dt, exec[s]});
    }
  }
  const int max_groups = (n_ticks + 1 + G - 1) / G + 1;  // a round advances every live env by at least one tick
  bool live[RLM_MAX_SUB];
  int n_live = 0;
  for (int s = 0; s < S; ++s) { live[s] = sub0[s + 1] > sub0[s]; n_live += live[s] ? 1 : 0; }
  h->rounds_calls++;
  for (int k = 0; k <= max_groups && n_live > 0; ++k) {
    for (int s = 0; s < S && k < max_groups; ++s) {
      if (!live[s]) continue;
      cudaStream_t st = S > 1 ? h->sub_stream[s] : h->stream;
      if (exec[s]) CK(cudaGraphLaunch(exec[s], st));
      else {
        CK(cudaMemsetAsync(pss[s].ready_count, 0, (size_t)G * 4, st));
        CK(cudaMemsetAsync(pss[s].ready_count + RLM_LIVE_OFF, 0, (size_t)G * 4, st));
        for (int r = 0; r < G; ++r) {
          if (h->profile) CK(cudaEventRecord(h->ev[3 * r], st));
          CK(rlm_launch_env_round(pss[s], dts[s], dts[s].n_sub, r, st));
          if (h->profile) CK(cudaEventRecord(h->ev[3 * r + 1], st));
          CK(launch_agent_on(h, pss[s], dts[s], r, 0, st));
          if (h->profile) CK(cudaEventRecord(h->ev[3 * r + 2], st));
        }
        if (h->profile) {  // bench instrumentation: per-kernel times of the rounds that had work (S == 1, direct launches)
          std::vector<int> cnt(2 * G);
          CK(cudaStreamSynchronize(st));
          CK(cudaMemcpy(cnt.data(), pss[s].ready_count, (size_t)G * 4, cudaMemcpyDeviceToHost));
          CK(cudaMemcpy(cnt.data() + G, pss[s].ready_count + RLM_LIVE_OFF, (size_t)G * 4, cudaMemcpyDeviceToHost));
          for (int r = 0; r < G; ++r) {
            float a = 0, b = 0;
            CK(cudaEventElapsedTime(&a, h->ev[3 * r], h->ev[3 * r + 1]));
            CK(cudaEventElapsedTime(&b, h->ev[3 * r + 1], h->ev[3 * r + 2]));
            if (cnt[G + r] > 0) { h->prof_env_ms += a; h->prof_env_launches++; }
            if (cnt[r] > 0) { h->prof_agent_ms += b; h->prof_agent_launches++; }
          }
        }
      }
      h->launches += 2 * G;
      h->rounds_launched += G;
      CK(cudaMemcpyAsync(h->h_live + 2 * s + (k & 1), pss[s].ready_count + RLM_LIVE_OFF + (G - 1), sizeof(int), cudaMemcpyDeviceToHost, st));
      CK(cudaEventRecord(h->ev_live[s][k & 1], st));
    }
    if (k >= 1)
      for (int s = 0; s < S; ++s) {
        if (!live[s]) continue;
        CK(cudaEventSynchronize(h->ev_live[s][(k - 1) & 1]));
        if (h->h_live[2 * s + ((k - 1) & 1)] == 0) { live[s] = false; --n_live; }
      }
  }
  if (n_live > 0) return fail(RLM_ERR_CUDA, "round-paced engine: envs still live after the last possible round");
  if (S > 1)
    for (int s = 0; s < S; ++s) {
      CK(cudaEventRecord(h->ev_join[s], h->sub_stream[s]));
      CK(cudaStreamWaitEvent(h->stream, h->ev_join[s], 0));
    }
  return RLM_OK;
}

static int run_ticks_impl(rlm_handle h, int32_t n_ticks) {
  int rc = tape_check(h);  // (the tape source has no upload-length check: an env whose day ends stops there)
  if (rc) return rc;
  rc = upload_params(h);
  if (rc) return rc;
  DynParams d = h->dyn;
  d.alpha = h->alpha; d.eps = h->eps; d.tau = h->tau; d.n_ticks = n_ticks;
  if (h->cfg.source == RLM_SOURCE_STREAM) {
    if (h->stream_cursor + n_ticks > h->stream_ticks)
      return fail(RLM_ERR_END_OF_DATA, "rlm_run_ticks: not enough ticks loaded (performAction would return false, base.cpp:289)");
    d.stream_off = h->stream_cursor;
    d.stream_ticks = h->stream_ticks;
    h->stream_cursor += n_ticks;
  }
  if (h->cfg.shared_policy && !d.backtest) {
    // single-GPU shared policy: every tick = accumulate, apply (no all-reduce needed).  Evaluation (backtest mode) never
    // writes theta, so it needs neither stage: it takes the tick-synchronous path below with every env reading policy 0.
    const DynParams keep = h->dyn;
    h->in_run = true;
    for (int t = 0; t < n_ticks; ++t) {
      h->dyn = keep; h->dyn.stream_off = d.stream_off + t; h->dyn.stream_ticks = d.stream_ticks;
      int rc2 = rlm_shared_tick_accumulate(h);
      if (!rc2) rc2 = rlm_apply_dtheta(h);
      if (rc2) { h->dyn = keep; h->in_run = false; return rc2; }
    }
    h->dyn = keep;
    h->in_run = false;
    return RLM_OK;
  }
  if (h->engine == 2) {
    CK(rlm_launch_fused(h->ptr, d, h->cfg.n_envs, h->hp.is_double, h->stream));
    h->launches += 1;
    return RLM_OK;
  }
  if (h->engine == 3 && !d.backtest && h->cfg.algorithm < RLM_ALGO_R_LEARN) {
    // fused persistent engine, round 2 (rlm_fused2_kernel): one launch, no per-tick barrier
    CK(rlm_launch_fused2(h->ptr, d, h->cfg.n_envs, h->hp.is_double, h->stream));
    h->launches += 1;
    return RLM_OK;
  }
  if (h->engine == 0) {
    // persistent engine: one launch, no global barrier between ticks
    CK(cudaMemsetAsync(h->d_qctl, 0, 16, h->stream));
    CK(rlm_launch_run(h->ptr, d, h->cfg.n_envs, h->hp.scratch_bytes, h->n_agent_ctas, h->stream));
    h->launches += 1;
    return RLM_OK;
  }
  if ((h->rounds || (h->rounds_auto && n_ticks >= RLM_ROUNDS_MIN_TICKS)) && h->engine == 1 && !d.backtest && !d.hold && h->n_sub <= 1)
    return run_rounds(h, d, n_ticks);
  // two kernels per tick (env tick, then the learner step of the envs whose midprice moved), then one
  // trailing env pass that only runs the pending action selections, so that the observable state
  // after the call is "every env sits inside performAction's loop".  With n_sub > 1 every sub-batch does this on its own
  // stream (forked from and joined to the handle's stream), its own ready list and its own ready counters.
  const int S = (h->profile || h->n_sub < 1) ? 1 : h->n_sub;
  const int B = h->cfg.n_envs;
  int sub0[RLM_MAX_SUB + 1];
  {
    const int per = (((B + S - 1) / S) + 31) & ~31;  // whole warps of the thread-per-env kernel, whole CTAs of the warp-per-env one
    for (int s = 0; s <= S; ++s) sub0[s] = std::min(B, s * per);
  }
  if (S > 1) {
    CK(cudaEventRecord(h->ev_fork, h->stream));
    for (int s = 0; s < S; ++s) CK(cudaStreamWaitEvent(h->sub_stream[s], h->ev_fork, 0));
  }
  int done = 0;
  // One CUDA graph per chunk instead of 2 * chunk launches: every node's parameters are fixed (the generator source has
  // no stream offset), so the instantiated graph is reused until alpha / epsilon / the mode change.
  const bool graphs = h->use_graphs && h->graph_warm && S == 1 && !h->profile;
  const bool from_stream = h->cfg.source == RLM_SOURCE_STREAM;
  h->graph_warm = true;  // (the first call launches directly: function attributes are set outside any capture)
  while (graphs && done < n_ticks) {
    const int chunk = std::min(n_ticks - done, h->ready_cap);
    DynParams dt = d;
    dt.env0 = 0; dt.n_sub = B; dt.sub_idx = 0;
    DevPtrs pg = h->ptr;
    if (from_stream) {
      // STREAM source: what changes from call to call (buffer, offset, length) goes through device memory, so that the
      // graph of a chunk is reused by every call -- and by both buffers of the double-buffered upload
      dt.ctl_stream = 1; dt.stream_off = 0; dt.stream_ticks = 0;
      pg.stream = nullptr;
      RunCtl rc = {++h->run_seq, n_ticks, d.stream_off + done, d.stream_ticks, h->ptr.stream, 0};
      CK(rlm_launch_runctl(h->ptr, rc, h->stream));
    }
    rlm_handle_s::TickGraph* tg = nullptr;
    for (auto& g : h->graphs)
      if (g.chunk == chunk && memcmp(&g.d, &dt, sizeof(DynParams)) == 0) tg = &g;
    if (!tg) {
      if (h->graphs.size() >= 8) { for (auto& g : h->graphs) cudaGraphExecDestroy(g.exec); h->graphs.clear(); }
      cudaGraph_t graph = nullptr;
      CK(cudaStreamBeginCapture(h->stream, cudaStreamCaptureModeThreadLocal));
      cudaError_t ce = cudaMemsetAsync(h->ptr.ready_count, 0, (size_t)chunk * 4, h->stream);
      for (int t = 0; t < chunk && ce == cudaSuccess; ++t) {
        ce = rlm_launch_env(pg, dt, B, t, 0, h->env_variant, h->stream);
        if (ce == cudaSuccess) ce = launch_agent_on(h, pg, dt, t, 0, h->stream);
      }
      cudaError_t ce2 = cudaStreamEndCapture(h->stream, &graph);
      if (ce != cudaSuccess || ce2 != cudaSuccess) { if (graph) cudaGraphDestroy(graph); CK(ce != cudaSuccess ? ce : ce2); }
      cudaGraphExec_t exec = nullptr;
      ce = cudaGraphInstantiate(&exec, graph, 0);
      cudaGraphDestroy(graph);
      CK(ce);
      h->graphs.push_back({chunk, dt, exec});
      tg = &h->graphs.back();
    }
    CK(cudaGraphLaunch(tg->exec, h->stream));
    h->launches += 2 * chunk;
    done += chunk;
  }
  while (done < n_ticks) {
    const int chunk = std::min(n_ticks - done, h->ready_cap);
    if (h->profile) {
      while ((int)h->ev.size() < 3 * chunk) { cudaEvent_t e; CK(cudaEventCreate(&e)); h->ev.push_back(e); }
    }
    for (int s = 0; s < S; ++s)
      CK(cudaMemsetAsync(h->ptr.ready_count + (size_t)s * h->ready_cap, 0, (size_t)chunk * 4, S > 1 ? h->sub_stream[s] : h->stream));
    for (int t = 0; t < chunk; ++t) {
      for (int s = 0; s < S; ++s) {
        if (sub0[s + 1] <= sub0[s]) continue;
        cudaStream_t st = S > 1 ? h->sub_stream[s] : h->stream;
        DynParams dt = d;
        dt.stream_off = d.stream_off + done;
        dt.env0 = sub0[s];
        dt.n_sub = sub0[s + 1] - sub0[s];
        dt.sub_idx = s;
        DevPtrs ps = h->ptr;
        ps.ready = h->ptr.ready + sub0[s];
        ps.ready_count = h->ptr.ready_count + (size_t)s * h->ready_cap;
        if (h->profile) CK(cudaEventRecord(h->ev[3 * t], st));
        CK(rlm_launch_env(ps, dt, B, t, 0, h->env_variant, st));
        if (h->profile) CK(cudaEventRecord(h->ev[3 * t + 1], st));
        CK(launch_agent_on(h, ps, dt, t, 0, st));
        if (h->profile) CK(cudaEventRecord(h->ev[3 * t + 2], st));
        h->launches += 2;
      }
    }
    if (h->profile) {
      CK(cudaStreamSynchronize(h->stream));
      for (int t = 0; t < chunk; ++t) {
        float a = 0, b = 0;
        CK(cudaEventElapsedTime(&a, h->ev[3 * t], h->ev[3 * t + 1]));
        CK(cudaEventElapsedTime(&b, h->ev[3 * t + 1], h->ev[3 * t + 2]));
        h->prof_env_ms += a; h->prof_agent_ms += b;
        h->prof_env_launches++; h->prof_agent_launches++;
      }
    }
    done += chunk;
  }
  for (int s = 0; s < S; ++s) {
    if (sub0[s + 1] <= sub0[s]) continue;
    cudaStream_t st = S > 1 ? h->sub_stream[s] : h->stream;
    DynParams dt = d;
    dt.env0 = sub0[s];
    dt.n_sub = sub0[s + 1] - sub0[s];
    CK(rlm_launch_env(h->ptr, dt, B, 0, 1, h->env_variant, st));
    h->launches++;
    if (S > 1) {
      CK(cudaEventRecord(h->ev_join[s], st));
      CK(cudaStreamWaitEvent(h->stream, h->ev_join[s], 0));
    }
  }
  return RLM_OK;
}

int rlm_sync(rlm_handle h) {
  API_LOCK;
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  unsigned long long c[8];
  CK(cudaMemcpy(c, h->ptr.counters, sizeof(c), cudaMemcpyDeviceToHost));
  unsigned err = (unsigned)c[4];
  if (err) {
    char buf[256];
    snprintf(buf, sizeof(buf), "device error flags 0x%x:%s%s%s%s%s", err,
             (err & ERR_BAD_PRICE) ? " non-positive price/volume (book.cpp:74-77)" : "",
             (err & ERR_TICK_RANGE) ? " invalid price/ticks for conversion (market.cpp:86,112)" : "",
             (err & ERR_TRACE_OVERFLOW) ? " trace list overflow (raise trace_cap)" : "",
             (err & ERR_INVALID_STATE) ? " invalid book state (book.cpp:612-625)" : "",
             (err & ERR_STREAM_UNDERRUN) ? " stream underrun" : "");
    return fail((err & ERR_TICK_RANGE) ? RLM_ERR_INVALID_ARGUMENT : RLM_ERR_RUNTIME, buf);
  }
  return RLM_OK;
}

int rlm_get_counters(rlm_handle h, rlm_counters* out) {
  API_LOCK;
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  unsigned long long c[8];
  CK(cudaMemcpy(c, h->ptr.counters, sizeof(c), cudaMemcpyDeviceToHost));
  out->ticks = (int64_t)c[0]; out->steps = (int64_t)c[1]; out->sum_traces = (int64_t)c[2];
  out->terminal_envs = (int64_t)c[3]; out->kernel_launches = h->launches;
  return RLM_OK;
}

static int fetch_hdrs(rlm_handle h, int env0, int n, std::vector<EnvHdr>& out) {
  if (env0 < 0 || n < 0 || env0 + n > h->cfg.n_envs) return fail(RLM_ERR_INVALID_ARGUMENT, "env range out of bounds");
  out.resize(n);
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  if (n) CK(cudaMemcpy2D(out.data(), sizeof(EnvHdr), h->ptr.env + (size_t)env0 * h->hp.env_stride, h->hp.env_stride, sizeof(EnvHdr), n,
                         cudaMemcpyDeviceToHost));
  return RLM_OK;
}

int rlm_get_stats(rlm_handle h, int32_t env0, int32_t n, rlm_env_stats* out) {
  API_LOCK;
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  std::vector<EnvHdr> v;
  int rc = fetch_hdrs(h, env0, n, v);
  if (rc) return rc;
  for (int i = 0; i < n; ++i) {
    const EnvHdr& e = v[i];
    rlm_env_stats& s = out[i];
    s.episode_reward = e.ep_reward; s.episode_pnl = e.ep_pnl; s.episode_bandh = e.ep_bandh;
    s.position = e.position;
    s.ask_transactions = e.side[0].n_transacted; s.bid_transactions = e.side[1].n_transacted;
    s.market_buys = e.market_buys; s.market_sells = e.market_sells;
    s.total_ticks = e.ts_total; s.steps = e.ag.ep_step;
    s.terminal = e.phase == PH_DONE; s.phase = e.phase;
  }
  return RLM_OK;
}

// packed column read-back: gather kernel -> pinned staging -> caller's buffer (B values over PCIe, not B headers)
static int fetch_column(rlm_handle h, int what, void* out, size_t bytes) {
  API_LOCK;
  CK(cudaSetDevice(h->cfg.device));
  int rc = upload_params(h);
  if (rc) return rc;
  if (bytes > h->gather_cap) {
    CK(cudaStreamSynchronize(h->stream));
    cudaFree(h->d_gather); if (h->h_gather) cudaFreeHost(h->h_gather);
    h->d_gather = nullptr; h->h_gather = nullptr; h->gather_cap = 0;
    CK(cudaMalloc(&h->d_gather, bytes));
    CK(cudaMallocHost(&h->h_gather, bytes));
    h->gather_cap = bytes;
  }
  CK(rlm_launch_gather(h->ptr, h->cfg.n_envs, what, h->d_gather, h->stream));
  CK(cudaMemcpyAsync(h->h_gather, h->d_gather, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  memcpy(out, h->h_gather, bytes);
  return RLM_OK;
}

int rlm_get_state(rlm_handle h, float* out) {
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  return fetch_column(h, 2, out, (size_t)h->cfg.n_envs * h->cfg.n_state_vars * sizeof(float));
}
int rlm_get_reward(rlm_handle h, double* out) {
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  return fetch_column(h, 0, out, (size_t)h->cfg.n_envs * sizeof(double));
}
int rlm_get_occupancy(rlm_handle h, int32_t* out) {
  API_LOCK;
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  if (h->cfg.shared_policy) return fail(RLM_ERR_UNSUPPORTED, "rlm_get_occupancy is per env (independent policies)");
  CK(cudaSetDevice(h->cfg.device));
  const size_t bytes = (size_t)h->cfg.n_envs * sizeof(int32_t);
  int rc = split_scratch(h, bytes);
  if (rc) return rc;
  CK(rlm_launch_count_nonzero(h->ptr.theta, h->cfg.memory_size, h->cfg.n_envs, (int*)h->d_gather, h->stream));
  CK(cudaMemcpyAsync(h->h_gather, h->d_gather, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  memcpy(out, h->h_gather, bytes);
  return RLM_OK;
}
int rlm_get_rho(rlm_handle h, double* out) {
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  return fetch_column(h, 3, out, (size_t)h->cfg.n_envs * sizeof(double));
}
int rlm_get_actions(rlm_handle h, int32_t* out) {
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  return fetch_column(h, 1, out, (size_t)h->cfg.n_envs * sizeof(int32_t));
}

int rlm_handle_terminal(rlm_handle h, int32_t episode) {
  API_LOCK;
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  CK(cudaSetDevice(h->cfg.device));
  int rc = upload_params(h);
  if (rc) return rc;
  CK(rlm_launch_clear_traces(h->ptr, h->cfg.n_envs, h->stream));  // traces.decay(0.0), agent.cpp:105
  const rlm_config& c = h->cfg;
  h->alpha = std::max(c.alpha_floor, c.alpha_start * pow(c.omega, (double)episode));  // agent.cpp:106
  if (c.policy_type == RLM_POLICY_EPSILON_GREEDY) {                                   // policy.cpp:79-82
    double e0 = (double)c.eps_init, ef = (double)c.eps_floor;
    h->eps = e0 * pow(ef / e0, (double)episode / (double)(long)c.eps_T);
  }
  if (c.policy_type == RLM_POLICY_BOLTZMANN) {                                        // policy.cpp:119-122
    double t0 = (double)c.tau_init, tf = (double)c.tau_floor;
    h->tau = t0 * pow(tf / t0, (double)episode / (double)(long)c.tau_T);
  }
  return RLM_OK;
}

int rlm_go_greedy(rlm_handle h) {
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  h->dyn.greedy = 1;  // Agent::GoGreedy, agent.cpp:76-79
  return RLM_OK;
}

int rlm_read_theta(rlm_handle h, int32_t policy, int32_t table, double* out, int64_t n) {
  API_LOCK;
  if (!h || !out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  if (policy < 0 || policy >= h->n_policies || n < 0 || n > h->cfg.memory_size) return fail(RLM_ERR_INVALID_ARGUMENT, "bad policy index / length");
  double* src = table == 0 ? h->ptr.theta : h->ptr.theta_b;
  if (!src) return fail(RLM_ERR_INVALID_ARGUMENT, "no such table");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(out, src + (size_t)policy * h->cfg.memory_size, (size_t)n * 8, cudaMemcpyDeviceToHost));
  return RLM_OK;
}
int rlm_write_theta(rlm_handle h, int32_t policy, int32_t table, const double* in, int64_t n) {
  API_LOCK;
  if (!h || !in) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  if (policy < 0 || policy >= h->n_policies || n < 0 || n > h->cfg.memory_size) return fail(RLM_ERR_INVALID_ARGUMENT, "bad policy index / length");
  double* dst = table == 0 ? h->ptr.theta : h->ptr.theta_b;
  if (!dst) return fail(RLM_ERR_INVALID_ARGUMENT, "no such table");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  CK(cudaMemcpy(dst + (size_t)policy * h->cfg.memory_size, in, (size_t)n * 8, cudaMemcpyHostToDevice));
  CK(cudaMemset(h->ptr.occ + (size_t)policy * h->hp.occ_words, 0xFF, (size_t)h->hp.occ_words * 4));  // caller-provided weights: assume dense
  if (!h->cfg.shared_policy) {
    const int dense = (int)h->cfg.memory_size;
    CK(cudaMemcpy(h->ptr.env + (size_t)policy * h->hp.env_stride + offsetof(EnvHdr, ag) + offsetof(AgentD, n_occ), &dense, 4, cudaMemcpyHostToDevice));
  }
  CK(cudaDeviceSynchronize());
  return RLM_OK;
}

int rlm_copy_theta(rlm_handle dst, rlm_handle src) {
  API_LOCK;
  if (!dst || !src) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  if (dst->cfg.device != src->cfg.device || dst->n_policies != src->n_policies || dst->cfg.memory_size != src->cfg.memory_size ||
      dst->hp.is_double != src->hp.is_double || dst->cfg.shared_policy != src->cfg.shared_policy)
    return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_copy_theta: handles differ in device, policy count, memory_size or table count");
  CK(cudaSetDevice(dst->cfg.device));
  CK(cudaStreamSynchronize(src->stream));
  CK(cudaStreamSynchronize(dst->stream));
  const size_t tbytes = (size_t)src->n_policies * (size_t)src->cfg.memory_size * 8;
  CK(cudaMemcpy(dst->ptr.theta, src->ptr.theta, tbytes, cudaMemcpyDeviceToDevice));
  if (src->ptr.theta_b) CK(cudaMemcpy(dst->ptr.theta_b, src->ptr.theta_b, tbytes, cudaMemcpyDeviceToDevice));
  CK(cudaMemcpy(dst->ptr.occ, src->ptr.occ, (size_t)src->n_policies * (size_t)src->hp.occ_words * 4, cudaMemcpyDeviceToDevice));
  if (!src->cfg.shared_policy)  // per-env population count of the bitmap (AgentD::n_occ) travels with it
    CK(cudaMemcpy2D(dst->ptr.env + offsetof(EnvHdr, ag) + offsetof(AgentD, n_occ), dst->hp.env_stride,
                    src->ptr.env + offsetof(EnvHdr, ag) + offsetof(AgentD, n_occ), src->hp.env_stride, 4, src->cfg.n_envs,
                    cudaMemcpyDeviceToDevice));
  CK(cudaDeviceSynchronize());  // device-to-device copies do not block the host: dst may be run right away
  return RLM_OK;
}

int rlm_read_records(rlm_handle h, int32_t env, rlm_step_record* out, int32_t cap, int32_t* n_out) {
  API_LOCK;
  if (!h || !out || !n_out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  if (env < 0 || env >= h->hp.record_envs) return fail(RLM_ERR_INVALID_ARGUMENT, "env is not recorded (cfg.record_envs)");
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  int rc = fix_records(h);
  if (rc) return rc;
  int cnt = 0;
  CK(cudaMemcpy(&cnt, h->ptr.record_count + env, 4, cudaMemcpyDeviceToHost));
  int n = std::min(std::min(cnt, h->hp.record_cap), cap);
  if (n > 0) CK(cudaMemcpy(out, h->ptr.records + (size_t)env * h->hp.record_cap, (size_t)n * sizeof(rlm_step_record), cudaMemcpyDeviceToHost));
  *n_out = n;
  return RLM_OK;
}

int rlm_device_ptrs(rlm_handle h, void** theta, void** dtheta, int64_t* n_doubles) {
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  if (theta) *theta = h->ptr.theta;
  if (dtheta) *dtheta = h->ptr.dtheta;
  // dtheta holds table A then table B (double agents): all-reduce n_doubles values starting at *dtheta
  if (n_doubles) *n_doubles = h->cfg.shared_policy ? (int64_t)(h->hp.is_double ? 2 : 1) * h->cfg.memory_size : (int64_t)h->n_policies * h->cfg.memory_size;
  return RLM_OK;
}
static const char* const k_eval_no_collective =
    "backtest mode: evaluation never writes theta, so it needs no collective -- call rlm_run_ticks (every rank evaluates its own envs)";
// Shared policy, phase A of one tick: env tick + learner steps evaluated under theta_t, updates
// accumulated into dtheta.  The caller all-reduces dtheta (rlm_device_ptrs) across ranks when the policy
// spans GPUs, then calls rlm_apply_dtheta.
int rlm_shared_tick_accumulate(rlm_handle h) {
  API_LOCK;
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  if (!h->cfg.shared_policy) return fail(RLM_ERR_INVALID_ARGUMENT, "handle was not created with shared_policy");
  if (h->dyn.backtest) return fail(RLM_ERR_INVALID_ARGUMENT, k_eval_no_collective);
  h->rec_dirty = true;  // (learner steps write records)
  CK(cudaSetDevice(h->cfg.device));
  int rc = upload_params(h);
  if (rc) return rc;
  DynParams d = h->dyn;
  d.alpha = h->alpha; d.eps = h->eps; d.tau = h->tau; d.n_ticks = 1;
  rc = tape_check(h);
  if (rc) return rc;
  if (h->cfg.source == RLM_SOURCE_STREAM && !h->in_run) {
    if (h->stream_cursor + 1 > h->stream_ticks) return fail(RLM_ERR_END_OF_DATA, "not enough ticks loaded");
    d.stream_off = h->stream_cursor; d.stream_ticks = h->stream_ticks;
    h->stream_cursor += 1;
  }
  CK(cudaMemsetAsync(h->ptr.ready_count, 0, 4, h->stream));
  CK(rlm_launch_env(h->ptr, d, h->cfg.n_envs, 0, 0, h->env_variant, h->stream));
  CK(launch_agent_any(h, d, 0, 1));
  h->launches += 2;
  h->shared_dyn = d;
  return RLM_OK;
}

// Shared policy, phase B: theta += dtheta; dtheta = 0; Q(from, .) under the new theta for the envs that
// stepped; then their action selection (the trailing env pass).
int rlm_apply_dtheta(rlm_handle h) {
  API_LOCK;
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  if (!h->cfg.shared_policy) return fail(RLM_ERR_INVALID_ARGUMENT, "handle was not created with shared_policy");
  if (h->dyn.backtest) return fail(RLM_ERR_INVALID_ARGUMENT, k_eval_no_collective);
  h->rec_dirty = true;  // (learner steps write records)
  CK(cudaSetDevice(h->cfg.device));
  int rc = upload_params(h);
  if (rc) return rc;
  const long long n =(long long)(h->hp.is_double ? 2 : 1) * h->cfg.memory_size;
  CK(rlm_launch_apply_dtheta(h->ptr.theta, h->ptr.dtheta, h->cfg.memory_size, h->n_sms, h->stream));
  if (h->hp.is_double) CK(rlm_launch_apply_dtheta(h->ptr.theta_b, h->ptr.dtheta + h->cfg.memory_size, h->cfg.memory_size, h->n_sms, h->stream));
  (void)n;
  CK(launch_agent_any(h, h->shared_dyn, 0, 2));
  CK(rlm_launch_env(h->ptr, h->shared_dyn, h->cfg.n_envs, 0, 1, h->env_variant, h->stream));
  h->launches += 3;
  return RLM_OK;
}

// ---------------------------------------------------------------------------------------------
// Split surface: the reference's Environment::step / Agent::update seam (SURVEY.md 8b), batched.
static int split_check(rlm_handle h) {
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  if (h->cfg.shared_policy) return fail(RLM_ERR_UNSUPPORTED, "the split surface drives independent policies (shared policy: rlm_shared_tick_accumulate / rlm_apply_dtheta)");
  if (h->cfg.source == RLM_SOURCE_STREAM)
    return fail(RLM_ERR_UNSUPPORTED, "the split surface needs source = generator or tape: envs consume different numbers of ticks per step");
  if (h->dyn.backtest) return fail(RLM_ERR_UNSUPPORTED, "the split surface runs Learner::_step (train mode)");
  return tape_check(h);
}
static DynParams split_dyn(rlm_handle h) {
  DynParams d = h->dyn;
  d.alpha = h->alpha; d.eps = h->eps; d.tau = h->tau; d.n_ticks = 1;
  d.hold = 1;
  return d;
}

int rlm_act(rlm_handle h, int32_t* actions_out) {
  API_LOCK;
  int rc = split_check(h);
  if (rc) return rc;
  if (!actions_out) return fail(RLM_ERR_INVALID_ARGUMENT, "null argument");
  CK(cudaSetDevice(h->cfg.device));
  rc = upload_params(h);
  if (rc) return rc;
  const size_t bytes = (size_t)h->cfg.n_envs * 4;
  rc = split_scratch(h, bytes);
  if (rc) return rc;
  CK(rlm_launch_act(h->ptr, split_dyn(h), h->cfg.n_envs, (int*)h->d_gather, h->stream));
  CK(cudaMemcpyAsync(h->h_gather, h->d_gather, bytes, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  memcpy(actions_out, h->h_gather, bytes);
  h->launches += 1;
  return RLM_OK;
}

int rlm_env_step(rlm_handle h, const int32_t* actions, double* reward_out, uint8_t* terminal_out) {
  API_LOCK;
  int rc = split_check(h);
  if (rc) return rc;
  CK(cudaSetDevice(h->cfg.device));
  rc = upload_params(h);
  if (rc) return rc;
  const int B = h->cfg.n_envs;
  rc = split_scratch(h, (size_t)B * 16);
  if (rc) return rc;
  const DynParams d = split_dyn(h);
  int* d_actions = nullptr;
  if (actions) {
    d_actions = (int*)h->d_gather;
    memcpy(h->h_gather, actions, (size_t)B * 4);
    CK(cudaMemcpyAsync(d_actions, h->h_gather, (size_t)B * 4, cudaMemcpyHostToDevice, h->stream));
  }
  CK(rlm_launch_apply(h->ptr, d, B, d_actions, h->stream));
  h->launches += 1;
  // performAction's do-while for every env that is inside a step (or Initialise for envs that are warming up): tick
  // until each one has reached its step end.  Envs on hold do not tick; all step ends of this call share ONE ready list.
  CK(cudaMemsetAsync(h->ptr.ready_count, 0, 4, h->stream));
  for (int guard = 0; guard < (1 << 22); ++guard) {
    CK(cudaMemsetAsync(h->ptr.counters + 5, 0, 8, h->stream));
    CK(rlm_launch_env(h->ptr, d, B, 0, 0, h->env_variant, h->stream));
    h->launches += 1;
    unsigned long long running = 0;
    CK(cudaMemcpyAsync(&running, h->ptr.counters + 5, 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (running == 0) break;
  }
  if (reward_out || terminal_out) {
    double* d_rew = (double*)h->d_gather;
    unsigned char* d_term = (unsigned char*)h->d_gather + (size_t)B * 8;
    CK(rlm_launch_step_out(h->ptr, B, d_rew, d_term, nullptr, h->stream));
    CK(cudaMemcpyAsync(h->h_gather, h->d_gather, (size_t)B * 9, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (reward_out) memcpy(reward_out, h->h_gather, (size_t)B * 8);
    if (terminal_out) memcpy(terminal_out, (unsigned char*)h->h_gather + (size_t)B * 8, (size_t)B);
  }
  return RLM_OK;
}

int rlm_agent_update(rlm_handle h, double* delta_out) {
  API_LOCK;
  int rc = split_check(h);
  if (rc) return rc;
  h->rec_dirty = true;  // (learner steps write records)
  CK(cudaSetDevice(h->cfg.device));
  rc = upload_params(h);
  if (rc) return rc;
  const int B = h->cfg.n_envs;
  // State::newState + Agent::HandleTransition for the envs on the ready list of the last rlm_env_step
  CK(launch_agent_any(h, split_dyn(h), 0, 0));
  CK(cudaMemsetAsync(h->ptr.ready_count, 0, 4, h->stream));
  h->launches += 1;
  if (delta_out) {
    rc = split_scratch(h, (size_t)B * 8);
    if (rc) return rc;
    CK(rlm_launch_step_out(h->ptr, B, nullptr, nullptr, (double*)h->d_gather, h->stream));
    CK(cudaMemcpyAsync(h->h_gather, h->d_gather, (size_t)B * 8, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    memcpy(delta_out, h->h_gather, (size_t)B * 8);
  }
  return RLM_OK;
}

// bench instrumentation: CUDA-event time of every env / agent kernel launch of the tick-synchronous engine
int rlm_set_profiling(rlm_handle h, int32_t on) {
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  h->profile = on != 0;
  h->prof_env_ms = h->prof_agent_ms = 0; h->prof_env_launches = h->prof_agent_launches = 0;
  return RLM_OK;
}
int rlm_get_kernel_times(rlm_handle h, double* env_ms, double* agent_ms, int64_t* env_launches, int64_t* agent_launches) {
  if (!h) return fail(RLM_ERR_INVALID_ARGUMENT, "null handle");
  if (env_ms) *env_ms = h->prof_env_ms;
  if (agent_ms) *agent_ms = h->prof_agent_ms;
  if (env_launches) *env_launches = h->prof_env_launches;
  if (agent_launches) *agent_launches = h->prof_agent_launches;
  return RLM_OK;
}

int rlm_flow_generate(const rlm_flow_params* p, int64_t env_index, int64_t first_tick, int32_t n_ticks, rlm_tick_msg* out) {
  if (!p || !out || n_ticks < 0 || first_tick < 0) return fail(RLM_ERR_INVALID_ARGUMENT, "bad arguments");
  rlm_flow_state s;
  rlm_flow_init(&s, p, (uint64_t)env_index);
  rlm_tick_msg tmp;
  for (int64_t t = 0; t < first_tick; ++t) rlm_flow_next(&s, p, rlm_flow_skellam20_lut, rlm_flow_pois30_lut, rlm_flow_pois1p5_lut, &tmp);
  for (int32_t t = 0; t < n_ticks; ++t) rlm_flow_next(&s, p, rlm_flow_skellam20_lut, rlm_flow_pois30_lut, rlm_flow_pois1p5_lut, &out[t]);
  return RLM_OK;
}

// ---------------------------------------------------------------------------------------------
// unit-level device entry points
static int test_setup(const rlm_config* cfg, rlm_handle_s& tmp) {
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(RLM_ERR_NO_DEVICE, "no CUDA device (no CPU fallback)");
  tmp.cfg = *cfg;
  if (tmp.cfg.n_envs <= 0) tmp.cfg.n_envs = 1;
  int rc = derive(&tmp);
  if (rc) return rc;
  CK(cudaSetDevice(cfg->device));
  CK(cudaDeviceSynchronize());
  g_params_owner = nullptr;
  CK(rlm_upload_params(&tmp.hp, &tmp.dm));
  return RLM_OK;
}

int rlm_test_to_ticks(const rlm_config* cfg, const double* px, int32_t n, int32_t* out) {
  API_LOCK;
  rlm_handle_s tmp;
  int rc = test_setup(cfg, tmp);
  if (rc) return rc;
  double* d_in; int* d_out;
  CK(cudaMalloc(&d_in, n * 8)); CK(cudaMalloc(&d_out, n * 4));
  CK(cudaMemcpy(d_in, px, n * 8, cudaMemcpyHostToDevice));
  CK(rlm_launch_test_to_ticks(d_in, n, d_out));
  CK(cudaMemcpy(out, d_out, n * 4, cudaMemcpyDeviceToHost));
  cudaFree(d_in); cudaFree(d_out);
  return RLM_OK;
}
int rlm_test_to_price(const rlm_config* cfg, const int32_t* ticks, int32_t n, double* out) {
  API_LOCK;
  rlm_handle_s tmp;
  int rc = test_setup(cfg, tmp);
  if (rc) return rc;
  int* d_in; double* d_out;
  CK(cudaMalloc(&d_in, n * 4)); CK(cudaMalloc(&d_out, n * 8));
  CK(cudaMemcpy(d_in, ticks, n * 4, cudaMemcpyHostToDevice));
  CK(rlm_launch_test_to_price(d_in, n, d_out));
  CK(cudaMemcpy(out, d_out, n * 8, cudaMemcpyDeviceToHost));
  cudaFree(d_in); cudaFree(d_out);
  return RLM_OK;
}
int rlm_test_tiles(const rlm_config* cfg, const float* vars, int32_t n, int32_t* out) {
  API_LOCK;
  rlm_handle_s tmp;
  int rc = test_setup(cfg, tmp);
  if (rc) return rc;
  float* d_in; int* d_out;
  size_t nin = (size_t)n * cfg->n_state_vars, nout = (size_t)n * cfg->n_actions * 96;
  CK(cudaMalloc(&d_in, nin * 4)); CK(cudaMalloc(&d_out, nout * 4));
  CK(cudaMemcpy(d_in, vars, nin * 4, cudaMemcpyHostToDevice));
  CK(rlm_launch_test_tiles(d_in, n, d_out));
  CK(cudaMemcpy(out, d_out, nout * 4, cudaMemcpyDeviceToHost));
  cudaFree(d_in); cudaFree(d_out);
  return RLM_OK;
}
int rlm_test_learner_tiles(const rlm_config* cfg, int32_t form, const float* vars, int32_t n, int32_t* out) {
  API_LOCK;
  if (form < RLM_TILES_THREE_WARP || form > RLM_TILES_TRACE_GROUP0) return fail(RLM_ERR_INVALID_ARGUMENT, "unknown tile form");
  if (form == RLM_TILES_STAGED && cfg->memory_size > 8192) return fail(RLM_ERR_UNSUPPORTED, "the staged learner holds tables of at most 8192 weights");
  rlm_handle_s tmp;
  int rc = test_setup(cfg, tmp);
  if (rc) return rc;
  float* d_in; int* d_out;
  size_t nin = (size_t)n * cfg->n_state_vars, nout = (size_t)n * cfg->n_actions * (form == RLM_TILES_TRACE_GROUP0 ? 32 : 96);
  CK(cudaMalloc(&d_in, nin * 4)); CK(cudaMalloc(&d_out, nout * 4));
  CK(cudaMemcpy(d_in, vars, nin * 4, cudaMemcpyHostToDevice));
  CK(rlm_launch_test_learner_tiles(form, d_in, n, d_out));
  CK(cudaMemcpy(out, d_out, nout * 4, cudaMemcpyDeviceToHost));
  cudaFree(d_in); cudaFree(d_out);
  return RLM_OK;
}
int rlm_test_order(int64_t size, int64_t q_head, const rlm_order_op* ops, int32_t n_ops, rlm_order_state* out) {
  API_LOCK;
  int ndev = 0;
  if (cudaGetDeviceCount(&ndev) != cudaSuccess || ndev == 0) return fail(RLM_ERR_NO_DEVICE, "no CUDA device (no CPU fallback)");
  if (size <= 0) return fail(RLM_ERR_RUNTIME, "Order size must be non-zero and positive.");  // order.cpp:24-25
  if (q_head < 0) return fail(RLM_ERR_RUNTIME, "Order queue must be positive.");             // order.cpp:26-27
  for (int i = 0; i < n_ops; ++i)
    if ((ops[i].op == 0 || ops[i].op == 1) && ops[i].arg < 0)
      return fail(RLM_ERR_RUNTIME, ops[i].op == 0 ? "Transaction volume must be positive." : "Cancellation volume must be positive.");  // order.cpp:56-57,86-87
  rlm_order_op* d_ops; rlm_order_state* d_out;
  CK(cudaMalloc(&d_ops, n_ops * sizeof(rlm_order_op))); CK(cudaMalloc(&d_out, n_ops * sizeof(rlm_order_state)));
  CK(cudaMemcpy(d_ops, ops, n_ops * sizeof(rlm_order_op), cudaMemcpyHostToDevice));
  CK(rlm_launch_test_order(size, q_head, d_ops, n_ops, d_out));
  CK(cudaMemcpy(out, d_out, n_ops * sizeof(rlm_order_state), cudaMemcpyDeviceToHost));
  cudaFree(d_ops); cudaFree(d_out);
  return RLM_OK;
}
int rlm_test_rolling_mean(int32_t window, const double* vals, int32_t n, double* out) {
  API_LOCK;
  rlm_config cfg;
  rlm_config_default(&cfg);
  cfg.memory_size = 1024; cfg.algorithm = RLM_ALGO_Q_LEARN;
  cfg.lb_mpm = window;
  rlm_handle_s tmp;
  int rc = test_setup(&cfg, tmp);
  if (rc) return rc;
  double *d_in, *d_out, *d_ring; EnvHdr* d_e;
  CK(cudaMalloc(&d_in, n * 8)); CK(cudaMalloc(&d_out, n * 16)); CK(cudaMalloc(&d_ring, (size_t)tmp.hp.ring_total * 8)); CK(cudaMalloc(&d_e, sizeof(EnvHdr)));
  CK(cudaMemset(d_ring, 0, (size_t)tmp.hp.ring_total * 8)); CK(cudaMemset(d_e, 0, sizeof(EnvHdr)));
  CK(cudaMemcpy(d_in, vals, n * 8, cudaMemcpyHostToDevice));
  CK(rlm_launch_test_rolling_mean(d_in, n, d_out, d_ring, d_e));
  CK(cudaMemcpy(out, d_out, n * 16, cudaMemcpyDeviceToHost));
  cudaFree(d_in); cudaFree(d_out); cudaFree(d_ring); cudaFree(d_e);
  return RLM_OK;
}

}  // extern "C"
