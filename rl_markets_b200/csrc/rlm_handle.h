// rlm_handle.h -- the handle behind the C ABI and the host helpers its translation units share (rlm_api.cu,
// rlm_checkpoint.cu).  Not part of the public interface.
#pragma once
#include <cuda_runtime.h>
#include <mutex>
#include <string>
#include <vector>

#include "rlm.h"
#include "rlm_kernels.h"

// msg becomes the calling thread's rlm_last_error; returns code.  (rlm_ingest.cpp, built without CUDA, declares it itself.)
int fail(int code, const std::string& msg);
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
  int n_markets = 0;  // entries of dm.markets
  VenueD cfg_venue;
  DevMarkets dm = {};  // uploaded with hp (rlm_env.cuh: PM)
  bool rec_dirty = false;  // learner work was enqueued since rlm_fix_terminal_kernel last ran (fix_records)
  void* d_gather = nullptr; void* h_gather = nullptr; size_t gather_cap = 0;  // rlm_get_reward/actions/state staging
  long long launches = 0;
  double alpha = 0, eps = 0, tau = 1.0;
  // tick-synchronous engine: the batch is cut into n_sub sub-batches, each ticking on its own stream, so that the
  // DRAM-bound gather burst of one sub-batch's learner kernel overlaps the issue-bound scalar tick kernel of another
  int n_sub = 1;
  // CUDA graphs of the two-launch engines (see cached_graph): one instantiated graph per chunk length (a round group: -G),
  // valid as long as the per-launch parameters it was captured with are unchanged; `launches` kernels per replay
  struct TickGraph { int chunk; DynParams d; cudaGraphExec_t exec; long long launches; };
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
  // model_log (rlm_set_model_log): off while mlog.cap == 0; then one rlm_model_log_kernel pass follows every training
  // learner launch
  ModelLogPtrs mlog = {};
};

// Every entry point that launches kernels holds g_api_mu while it does so (rlm_api.cu: g_params_owner).
extern __attribute__((visibility("hidden"))) std::recursive_mutex g_api_mu;
#define API_LOCK std::lock_guard<std::recursive_mutex> api_lock_(g_api_mu)

// rlm_api.cu
int tape_check(rlm_handle h);
void day_markets_on(rlm_handle h, bool on);
int fix_records(rlm_handle h);
void drop_graphs(rlm_handle h);
