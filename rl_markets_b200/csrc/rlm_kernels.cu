// rlm_kernels.cu -- sm_90a (H100) kernels of the batched LOB environment + tile-coded TD agent (DESIGN.md section 3).
//
// Two kernels, driven by two engines (rlm_api.cu: run_ticks_impl / run_rounds); per env both run the same sequence
// begin_step / tick / ... / learner step, so their results are bit-identical:
//   tick-synchronous  two launches per market tick over all envs of the handle (short run calls, large batches, shared
//                     policies, backtest, the split surface), one CUDA graph per chunk of ticks;
//   round-paced       two launches per ROUND (the default for long run calls of up to 16 384 independent envs): every
//                     live env runs up to DynParams::round_cap of its own ticks, until its step ends.
//
//   env tick     rlm_env_kernel_w / rlm_env_round_kernel: one WARP per env (B <= 16384) -- record staged in shared
//                memory, Philox draws on three lanes, the generator's book update one level per lane, ask/bid book
//                updates on two lanes, rolling windows and state variables one per lane (their ToTicks conversions in
//                two convergent passes), quote placement at a step start on two lanes, the rest of the scalar market
//                logic (Intraday::NextState, src/environment/intraday.cpp:224-272, and rlm_env.cuh) on lane 0.
//                rlm_env_kernel<32>: one THREAD per env (B > 16384), the record in lane-interleaved local memory, SIMT
//                over 32 envs.  An env whose midprice moved (Base::performAction's do-while, base.cpp:285-305)
//                finishes the step, writes its state variables and reward, and appends itself to the ready list.
//   learner step rlm_learn_kernel (rlm_learn.cuh): ONE warp per ready env (lane j = tiling j of all three feature
//                groups, N_TILINGS == 32 == warp width): tile hashing, theta gathers, exact-order Q sums, the fused
//                trace-decay/clear/set/theta-update pass (Agent::HandleTransition, src/rl/agent.cpp:86-101) and
//                Q(from,.) for the next action selection.  rlm_learn_staged_kernel: the same step with the env's whole
//                weight table staged in shared memory by one TMA bulk copy (memory_size * 8 <= 64 KB).
//                rlm_agent3_kernel (round 1: one CTA of three warps per env, warp g = feature group g) serves the
//                R-learning agents and batches above 16 384 envs; rlm_agent_kernel<8> is older still.
//   evaluation   rlm_eval_kernel (rlm_learn.cuh): backtest mode's greedy step for every algorithm, independent or shared
//                policy -- one warp per ready env: hash, gathers, exact-order sums, Q(state, .); theta is only read.
//
// The next tick of a stepped env starts with Learner::_step's action selection and DoAction (serial.cpp:55-61,
// base.cpp:254-284; begin_step / begin_step_warp).  Alternative engines, all parity-green and all slower than the
// two-launch engines (DESIGN.md section 3.5): rlm_fused2_kernel (rlm_learn.cuh), rlm_run_kernel (persistent queue) and rlm_fused_kernel
// (RLM_ENGINE=F|p|f).
#include <cuda_runtime.h>
#include <stdint.h>
#define RLM_TABLE_QUAL static __device__ const
#include "rlm_flow_tables.h"
#include "rlm_rndseq.h"
#include "rlm_agent.cuh"
#include <cstdio>
#include "rlm_kernels.h"
#define RLM_ENVT_CARVEOUT_DEFAULT 30  // the thread-per-env tick kernel keeps its record copy in local memory: most of the array as L1
#define RLM_SMEM_CARVEOUT 88  // percent of the 228 KB L1/shared array configured as shared memory, for every per-tick kernel

// ---- one-warp-per-env learner (rlm_agent_kernel, fused and persistent engines): per warp [AgentD][scratch]
// (the 8 KB hashing table is read through L1)
// per-warp scratch: [q_pre_a, q_pre_b: 18 doubles][small set: 64 ints][vbuf: (1|2) * A_max * VROW doubles]
#define SCR_Q 0
#define SCR_SS (SCR_Q + 8 * 2 * RLM_MAX_ACTIONS)
#define SCR_IDX (SCR_SS + 4 * SS_SLOTS)                    // int idx[27][32]: tile indices of the to-state
#define SCR_VBUF (SCR_IDX + 4 * 3 * RLM_MAX_ACTIONS * 32)
#define AG_BYTES ((sizeof(AgentD) + 15) & ~(size_t)15)
size_t rlm_scratch_bytes(int is_double) {
  return ((size_t)SCR_VBUF + (size_t)(is_double ? 2 : 1) * RLM_MAX_ACTIONS * VROW * 8 + 15) & ~(size_t)15;
}
size_t rlm_agent_smem_bytes(int warps_per_cta, int scratch_bytes) {
  return (size_t)warps_per_cta * (AG_BYTES + (size_t)scratch_bytes);
}

// Programmatic dependent launch (the two per-tick kernels): the next kernel of the stream may be scheduled while this
// one drains -- its launch latency and CTA ramp-up overlap our tail -- but it touches nothing before
// griddepcontrol.wait, which returns only when the whole preceding grid has completed and flushed its writes.
#define PDL_PROLOGUE() do { asm volatile("griddepcontrol.launch_dependents;" ::: "memory"); asm volatile("griddepcontrol.wait;" ::: "memory"); } while (0)
static bool g_use_pdl = false;  // off: the early dependents crowd the tail of the preceding kernel
void rlm_set_pdl(int on) { g_use_pdl = on != 0; }
template <typename... KArgs, typename... Args>
static cudaError_t launch_pdl(void (*kernel)(KArgs...), int grid, int block, size_t smem, cudaStream_t st, Args... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = dim3(grid); cfg.blockDim = dim3(block); cfg.dynamicSmemBytes = smem; cfg.stream = st;
  cudaLaunchAttribute at[1];
  at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  at[0].val.programmaticStreamSerializationAllowed = g_use_pdl ? 1 : 0;
  cfg.attrs = at; cfg.numAttrs = 1;
  return cudaLaunchKernelEx(&cfg, kernel, args...);
}

#ifdef RLM_TIMING  // launch timeline: [tick slot][sub-batch][kernel: 0 env, 1 learner][0 first CTA start, 1 last CTA end], ns (globaltimer)
__device__ unsigned long long g_klog[256][8][2][2];
__device__ __forceinline__ unsigned long long gtime() { unsigned long long t; asm volatile("mov.u64 %0, %%globaltimer;" : "=l"(t)); return t; }
#define KLOG_BEGIN(kind) do { if (threadIdx.x == 0 && tslot < 256) atomicMin(&g_klog[tslot][D.sub_idx & 7][kind][0], gtime()); } while (0)
#define KLOG_END(kind) do { if (threadIdx.x == 0 && tslot < 256) atomicMax(&g_klog[tslot][D.sub_idx & 7][kind][1], gtime()); } while (0)
extern "C" int rlm_debug_klog(unsigned long long* out, int reset) {
  cudaDeviceSynchronize();
  if (out && cudaMemcpyFromSymbol(out, g_klog, sizeof(g_klog)) != cudaSuccess) return -1;
  if (reset) {
    static unsigned long long init[256][8][2][2];
    for (auto& a : init) for (auto& b : a) for (auto& c : b) { c[0] = ~0ull; c[1] = 0ull; }
    if (cudaMemcpyToSymbol(g_klog, init, sizeof(init)) != cudaSuccess) return -1;
  }
  return 0;
}
#else
#define KLOG_BEGIN(kind) do { } while (0)
#define KLOG_END(kind) do { } while (0)
#endif

// whether the uploaded block has day markets on: the launchers then pick the tick kernels' MKT instantiations
static bool g_day_markets = false;
cudaError_t rlm_upload_params(const DevParams* p, const DevMarkets* m) {
  g_day_markets = m->markets != nullptr;
  const cudaError_t e = cudaMemcpyToSymbol(P, p, sizeof(DevParams));
  return e != cudaSuccess ? e : cudaMemcpyToSymbol(PM, m, sizeof(DevMarkets));
}

// ---------------------------------------------------------------------------------------------
// init: Intraday ctor/Initialise state + RNG seeding, one thread per env.
// mode 0: full create; mode 1: episode reset (Base::Initialise base.cpp:123-135 keeps window sums, A13);
// mode 2: new env object, same agent
__global__ void rlm_init_kernel(DevPtrs ptr, int mode) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.n_envs) return;
  EnvHdr* e = (EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  double* ring = (double*)((unsigned char*)e + sizeof(EnvHdr));
  if (mode == 0 || mode == 2) {
    // mode 2: a NEW env object for the SAME agent (`environment::Intraday<> env(c)` of main.cpp:219): the agent block
    // (generator positions, rho, trace count, occupancy count) survives, everything else starts from scratch
    AgentD keep;
    if (mode == 2) keep = e->ag;
    unsigned char* raw = (unsigned char*)e;
    for (int i = 0; i < P.env_stride; ++i) raw[i] = 0;
    for (int i = 0; i < P.ring_total; ++i) ring[i] = 0.0;
    e->tp_val = -1.0;  // TargetPrice::val_ (target_price.cpp:8-10)
    if (mode == 2) e->ag = keep;
  }
  side_reset(e->side[0]);
  side_reset(e->side[1]);
  e->ask_quote = 0.0; e->bid_quote = 0.0;
  e->ep_reward = 0.0; e->ep_pnl = 0.0; e->ep_bandh = 0.0;
  e->market_buys = 0; e->market_sells = 0;
  e->ts_total = e->ts_ask = e->ts_bid = e->ts_both = e->ts_pos = e->ts_long = e->ts_short = 0;
  for (int w = 0; w < RLM_NWIN; ++w) { e->w_head[w] = 0; e->w_count[w] = 0; }
  e->last_date = 0; e->date = 0; e->time_ms = 0;
  e->phase = PH_PREOPEN;
  e->ag.ep_step = 0;
  if (mode == 1) {  // same Learner, next episode: the stale State is the from-state of the last completed transition
    for (int i = 0; i < RLM_N_STATE_MAX + 3; ++i) e->ag.from_vars[i] = e->ag.prev_vars[i];
    e->ag.null_from = e->ag.prev_null;
  } else {  // (mode 0: AgentD was zeroed above; mode 2: a new Runner's States are never-populated, serial.cpp:9-16)
    e->ag.null_from = 1;
    e->ag.prev_null = 1;
  }
  e->ag.need_begin = 0;
  e->ag.kind = 0;
  rlm_flow_init(&e->flow, &P.flow, (uint64_t)(P.env_index0 + b));
  if (P.source == RLM_SOURCE_TAPE) ptr.tape_cur[b].x = ptr.tape_lo[b];  // back to the first message of the env's day
}

__global__ void rlm_seed_kernel(DevPtrs ptr, unsigned random_seed) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.n_envs) return;
  EnvHdr* e = (EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  unsigned seed = random_seed + (unsigned)(P.env_index0 + b);
  // std::mt19937_64::seed(value)
  for (int g = 0; g < 2; ++g) {
    unsigned long long* x = g == 0 ? ptr.mt_pol : ptr.mt_agt;
    if (!x) continue;
    x += (size_t)b * 312;
    unsigned long long v = (unsigned long long)seed;
    x[0] = v;
    for (int i = 1; i < 312; ++i) { v = 6364136223846793005ull * (v ^ (v >> 62)) + (unsigned long long)i; x[i] = v; }
  }
  e->ag.mt_pol_idx = 312;
  e->ag.mt_agt_idx = 312;
  // glibc srandom_r, TYPE_3
  unsigned s = seed == 0 ? 1u : seed;
  e->ag.crand_r[0] = (int)s;
  for (int i = 1; i < 31; ++i) {
    long long hi = e->ag.crand_r[i - 1] / 127773, lo = e->ag.crand_r[i - 1] % 127773;
    long long word = 16807 * lo - 2836 * hi;
    if (word < 0) word += 2147483647;
    e->ag.crand_r[i] = (int)word;
  }
  e->ag.crand_f = 3; e->ag.crand_b = 0;
  for (int i = 0; i < 310; ++i) crand_next(e->ag);
}

// theta[i] = 2*U(0,1)-1 from the agent generator (agent.cpp:37-39,190-192), one thread per policy
__global__ void rlm_random_init_kernel(DevPtrs ptr, int n_policies) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_policies) return;
  EnvHdr* e = (EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  unsigned long long* x = ptr.mt_agt + (size_t)b * 312;
  double* th = ptr.theta + (size_t)b * P.memory_size;
  for (long long i = 0; i < P.memory_size; ++i) th[i] = 2.0 * mt_uniform_real(x, e->ag.mt_agt_idx) - 1.0;
  e->ag.n_occ = (int)P.memory_size;  // dense from the start
  if (ptr.theta_b) {
    double* tb = ptr.theta_b + (size_t)b * P.memory_size;
    for (long long i = 0; i < P.memory_size; ++i) tb[i] = 2.0 * mt_uniform_real(x, e->ag.mt_agt_idx) - 1.0;
  }
}

// Agent::HandleTerminal's traces.decay(0.0) (agent.cpp:105)
__global__ void rlm_clear_traces_kernel(DevPtrs ptr) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.n_envs) return;
  EnvHdr* e = (EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  e->ag.n_traces = 0;
}

// column read-back for rlm_get_reward / rlm_get_actions / rlm_get_state: one packed array instead of B headers
__global__ void rlm_gather_kernel(DevPtrs ptr, int what, void* out) {
  int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.n_envs) return;
  const EnvHdr* e = (const EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  if (what == 0) ((double*)out)[b] = e->ag.last_reward;
  else if (what == 1) ((int*)out)[b] = e->last_action;
  else if (what == 3) ((double*)out)[b] = e->ag.rho;
  else if (what == 4) ((int*)out)[b] = e->ag.n_occ;
  else
    for (int k = 0; k < P.n_state_vars; ++k) ((float*)out)[(size_t)b * P.n_state_vars + k] = e->ag.from_vars[k];
}

// rlm_get_occupancy: weights of table A that are not (bitwise) +0.0, one CTA per policy
__global__ void rlm_count_nonzero_kernel(const double* theta, long long M, int* out) {
  const double* th = theta + (size_t)blockIdx.x * (size_t)M;
  int n = 0;
  for (long long i = threadIdx.x; i < M; i += blockDim.x) n += (__double_as_longlong(__ldcs(th + i)) != 0ll) ? 1 : 0;
  for (int o = 16; o > 0; o >>= 1) n += __shfl_xor_sync(FULL, n, o);
  __shared__ int part[8];
  if ((threadIdx.x & 31) == 0) part[threadIdx.x >> 5] = n;
  __syncthreads();
  if (threadIdx.x == 0) { int t = 0; for (int w = 0; w < (int)(blockDim.x >> 5); ++w) t += part[w]; out[blockIdx.x] = t; }
}
cudaError_t rlm_launch_count_nonzero(const double* theta, long long M, int n_policies, int* out, cudaStream_t st) {
  rlm_count_nonzero_kernel<<<n_policies, 256, 0, st>>>(theta, M, out);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// parity record (include/rlm_record.h); lane 0 fills everything but the trace hash
// `vars`: the state written to the record (to-state of a learner step; decision state of a backtest step)
__device__ __noinline__ void fill_record(rlm_step_record* r, const EnvHdr& e, const AgentD& ag, unsigned long long thash,
                                         const float* vars) {
  r->step = ag.ep_step; r->action = ag.cur_action; r->time_ms = e.time_ms; r->terminal = is_terminal(e) ? 1 : 0;
  r->position = e.position; r->ask_quote = e.ask_quote; r->bid_quote = e.bid_quote;
  r->ask_level = e.ask_level; r->bid_level = e.bid_level;
  r->reward = ag.last_reward; r->pnl_step = e.pnl_step;
  r->ep_pnl = e.ep_pnl; r->ep_reward = e.ep_reward; r->ep_bandh = e.ep_bandh;
  r->midprice = m_midprice(e); r->spread = m_spread(e); r->bandh_step = e.agg_mpm;  // LogProfit, intraday.cpp:437-451
  for (int s = 0; s < 2; ++s) {
    rlm_order_rec& o = s == 0 ? r->ask : r->bid;
    const OrderD& d = e.side[s].ord;
    o.exists = d.live ? 1 : 0; o.pad = 0;
    o.price = d.live ? d.price : 0.0; o.q_head = d.live ? d.q_head : 0; o.q_tail = d.live ? d.q_tail : 0;
    o.executed = d.live ? (d.size - ord_remaining(d)) : 0;
  }
  r->ask_transactions = e.side[0].n_transacted; r->bid_transactions = e.side[1].n_transacted;
  r->market_buys = e.market_buys; r->market_sells = e.market_sells;
  r->lo_vol_step = e.lo_vol_step;
  r->n_state = P.n_state_vars;
  for (int i = 0; i < RLM_N_STATE_MAX + 1; ++i) r->state[i] = (i < P.n_state_vars) ? vars[i] : 0.0f;
  r->delta = ag.last_delta;
  r->n_traces = ag.n_traces; r->pad = 0;
  r->trace_hash = thash;
}

// Learner::_step up to the first NextState of performAction (serial.cpp:55-61, base.cpp:254-284), in its two halves:
//   begin_select  Agent::action(*last_state) -- or the end of the episode (isTerminal, ClearInventory serial.cpp:31)
//   begin_apply   Base::performAction(action) up to its do-while (DoAction, CheckOrders, UpdateStats, first reward term)
// Needs ag.q_from / qb_from.  begin_select returns the action, or -1 when the episode is over.
template <class... M>
__device__ __forceinline__ int begin_select_in(EnvHdr& e, unsigned long long* mt_pol, const DynParams& D, M... mk) {
  if (is_terminal(e, mk...)) {
    clear_inventory(e);  // Runner::RunEpisode, serial.cpp:31
    e.phase = PH_DONE;
    return -1;
  }
  return policy_action(e.ag, e.ag.q_from, e.ag.qb_from, mt_pol, D);
}
__device__ __noinline__ int begin_select(EnvHdr& e, unsigned long long* mt_pol, const DynParams& D) { return begin_select_in(e, mt_pol, D); }
__device__ __noinline__ int begin_select(EnvHdr& e, unsigned long long* mt_pol, const DynParams& D, EnvMarket mk) {
  return begin_select_in(e, mt_pol, D, mk);
}
template <class... M>
__device__ __forceinline__ void begin_apply_in(EnvHdr& e, int a, M... mk) {
  e.ag.cur_action = a;
  e.last_action = a;
  e.lo_vol_step = 0;
  e.pnl_step = 0.0;
  e.momentum_pnl_step = 0.0;
  do_action(e, a, mk...);
  check_orders(e);
  update_stats(e);
  e.agg_r = get_reward(e);
  e.agg_pnl = e.pnl_step;
  e.agg_mpm = 0.0;
  e.ag.kind = 3;  // inside performAction's loop (0 / 1 = the step / the warm-up has ended and waits for the learner)
}
__device__ __noinline__ void begin_apply(EnvHdr& e, int a) { begin_apply_in(e, a); }
__device__ __noinline__ void begin_apply(EnvHdr& e, int a, EnvMarket mk) { begin_apply_in(e, a, mk); }
template <class... M>
__device__ __forceinline__ bool begin_step(EnvHdr& e, unsigned long long* mt_pol, const DynParams& D, M... mk) {
  if (e.ag.kind == 4) { begin_apply(e, e.ag.cur_action, mk...); return true; }  // (rlm_act already drew the action)
  const int a = begin_select(e, mt_pol, D, mk...);
  if (a < 0) return false;
  begin_apply(e, a, mk...);
  return true;
}
// The same for the warp-per-env tick kernels: lane 0 selects the action and runs DoAction's book-keeping, the two quotes
// (Intraday::l2p_ + RiskManager::PlaceOrder, intraday.cpp:64-82,163-173) are priced and placed by lane 0 (ask) and lane 1
// (bid) side by side -- two ToTicks / ToPrice / queue look-ups instead of four in a row on the launch's critical path.
template <class... M>
__device__ __forceinline__ void begin_step_warp(EnvHdr& e, unsigned long long* mt_pol, const DynParams& D, int* flag, int lane, M... mk) {
  if (lane == 0) {
    int a;
    if (e.ag.kind == 4) a = e.ag.cur_action;  // (rlm_act already drew the action)
    else a = begin_select(e, mt_pol, D, mk...);
    int place = 0;
    if (a >= 0) {
      e.ag.cur_action = a;
      e.last_action = a;
      e.lo_vol_step = 0;
      e.pnl_step = 0.0;
      e.momentum_pnl_step = 0.0;
      int al = 0, bl = 0;
      place = 1;
      switch (a) {  // Intraday::DoAction (intraday.cpp:175-220), see do_action
        case 0: al = 1; bl = 1; break;
        case 1: clear_inventory(e); al = e.ask_level; bl = e.bid_level; break;
        case 2: al = 2; bl = 2; break;
        case 3: al = 3; bl = 3; break;
        case 4: al = 0; bl = 2; break;
        case 5: al = 2; bl = 0; break;
        case 6: al = 1; bl = 4; break;
        case 7: al = 4; bl = 1; break;
        case 8: al = 5; bl = 5; break;
        default: place = 0; break;
      }
      if (place) { e.ask_level = al; e.bid_level = bl; }
    }
    flag[0] = a;
    flag[1] = place;
  }
  __syncwarp();
  const int a = flag[0];
  if (a >= 0) {
    if (flag[1] && lane < 2) {  // place_orders, one side per lane
      int lerr = 0, hint = e.tk_band;
      const int lv = lane == 0 ? e.ask_level : -e.bid_level;
      double q;
      if (P.l2p_book) {
        q = to_price(mk..., to_ticks(mk..., e.side[lane].px[0], &lerr, &hint) + lv, &lerr);
      } else {
        const double tp = e.tp_val, half_spd = fmax(0.0, e.w_mean[W_SPREAD] / 2.0);
        const double px = lane == 0 ? tp + (double)e.ask_level * half_spd : tp - (double)e.bid_level * half_spd;
        q = to_price(mk..., to_ticks(mk..., px, &lerr, &hint), &lerr);
      }
      if (lane == 0) e.ask_quote = q; else e.bid_quote = q;
      side_replace_order(e.side[lane], q, P.order_size, &lerr);
      if (lerr) atomicOr(&e.err, lerr);
    }
    __syncwarp();
    if (lane == 0) {  // rest of begin_apply
      check_orders(e);
      update_stats(e);
      e.agg_r = get_reward(e);
      e.agg_pnl = e.pnl_step;
      e.agg_mpm = 0.0;
      e.ag.kind = 3;
    }
  }
  if (lane == 0) e.ag.need_begin = 0;
  __syncwarp();
}
// The market argument of env b's tick (rlm_env.cuh, EnvMarket): MKT = false, the config's market (no argument, and no
// load); MKT = true, the VenueD of the market of b's day.  on_market<MKT>(mk, f) calls f() or f(mk).
template <bool MKT>
__device__ __forceinline__ EnvMarket env_market_of(int b) {
  EnvMarket m{nullptr};
  if (MKT) m.v = PM.markets + PM.env_market[b];
  return m;
}
template <bool MKT, class F>
__device__ __forceinline__ decltype(auto) on_market(EnvMarket mk, F&& f) {
  if constexpr (MKT) return f(mk);
  else return f();
}
template <bool MKT>
__device__ __forceinline__ bool env_is_terminal(const EnvHdr& e, int b) {
  if constexpr (MKT) return is_terminal(e, env_market_of<true>(b));
  else return is_terminal(e);
}

// split surface: is this env waiting for rlm_agent_update (its step or its warm-up has ended) or for rlm_env_step to
// apply an action?  Such envs do not tick under DynParams::hold.
__device__ __forceinline__ bool env_on_hold(const EnvHdr& e) {
  return e.phase == PH_RUN && (e.ag.need_begin || e.ag.kind == 0 || e.ag.kind == 1);
}

// ---------------------------------------------------------------------------------------------
// Split surface (include/rlm.h: rlm_act / rlm_env_step / rlm_agent_update), one thread per env, straight on the
// record in HBM (this is the interoperability path, not the training loop).
// rlm_act: Agent::action for every env at a decision point; actions[b] = -1 elsewhere (and at the end of an episode).
template <bool MKT>
__global__ void rlm_act_kernel(DevPtrs ptr, DynParams D, int* actions) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.n_envs) return;
  EnvHdr& e = *(EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  int a = -1;
  if (e.phase == PH_RUN && e.ag.need_begin) {
    if (e.ag.kind == 4) a = e.ag.cur_action;  // already selected, not applied yet
    else {
      a = on_market<MKT>(env_market_of<MKT>(b), [&](auto... mk) { return begin_select(e, ptr.mt_pol + (size_t)b * 312, D, mk...); });
      if (a >= 0) { e.ag.cur_action = a; e.ag.kind = 4; }
      else e.ag.need_begin = 0;
    }
  }
  actions[b] = a;
}
// first half of rlm_env_step: Base::performAction(actions[b]) up to its do-while for every env at a decision point.
// actions == nullptr: the agent's own choice (rlm_act semantics, selected here if rlm_act was not called).
template <bool MKT>
__global__ void rlm_apply_kernel(DevPtrs ptr, DynParams D, const int* actions) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.n_envs) return;
  EnvHdr& e = *(EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  if (e.phase != PH_RUN || !e.ag.need_begin) return;
  const EnvMarket mk = env_market_of<MKT>(b);
  int a;
  if (e.ag.kind == 4) a = actions ? actions[b] : e.ag.cur_action;
  else if (actions) {  // external policy: Learner::_step without Agent::action (no generator draw)
    if (on_market<MKT>(mk, [&](auto... m) { return is_terminal(e, m...); })) { clear_inventory(e); e.phase = PH_DONE; e.ag.need_begin = 0; return; }
    a = actions[b];
  } else {
    a = on_market<MKT>(mk, [&](auto... m) { return begin_select(e, ptr.mt_pol + (size_t)b * 312, D, m...); });
    if (a < 0) { e.ag.need_begin = 0; return; }
  }
  if (a < 0 || a >= P.n_actions) { e.err |= ERR_BAD_PRICE; a = 0; }
  on_market<MKT>(mk, [&](auto... m) { begin_apply(e, a, m...); });
  e.ag.need_begin = 0;
}
// per-env outputs of rlm_env_step / rlm_agent_update
template <bool MKT>
__global__ void rlm_step_out_kernel(DevPtrs ptr, double* reward, unsigned char* terminal, double* delta) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.n_envs) return;
  const EnvHdr& e = *(const EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  if (reward) reward[b] = e.ag.last_reward;
  if (terminal) {
    // tape source: an env that is inside its step (not waiting for rlm_agent_update or for an action) with its day used up
    // has stopped inside performAction -- the reference's performAction returning false at the end of its files
    const int2 tc = P.source == RLM_SOURCE_TAPE ? ptr.tape_cur[b] : make_int2(0, 1);
    if (e.phase != PH_DONE && !env_on_hold(e) && tc.x >= tc.y) terminal[b] = 2;
    else terminal[b] = (e.phase == PH_DONE || (e.phase == PH_RUN && env_is_terminal<MKT>(e, b))) ? 1 : 0;
  }
  if (delta) delta[b] = e.ag.last_delta;
}
cudaError_t rlm_launch_act(const DevPtrs& ptr, const DynParams& D, int n_envs, int* actions, cudaStream_t st) {
  if (g_day_markets) rlm_act_kernel<true><<<(n_envs + 63) / 64, 64, 0, st>>>(ptr, D, actions);
  else rlm_act_kernel<false><<<(n_envs + 63) / 64, 64, 0, st>>>(ptr, D, actions);
  return cudaGetLastError();
}
cudaError_t rlm_launch_apply(const DevPtrs& ptr, const DynParams& D, int n_envs, const int* actions, cudaStream_t st) {
  if (g_day_markets) rlm_apply_kernel<true><<<(n_envs + 63) / 64, 64, 0, st>>>(ptr, D, actions);
  else rlm_apply_kernel<false><<<(n_envs + 63) / 64, 64, 0, st>>>(ptr, D, actions);
  return cudaGetLastError();
}
cudaError_t rlm_launch_step_out(const DevPtrs& ptr, int n_envs, double* reward, unsigned char* terminal, double* delta, cudaStream_t st) {
  if (g_day_markets) rlm_step_out_kernel<true><<<(n_envs + 127) / 128, 128, 0, st>>>(ptr, reward, terminal, delta);
  else rlm_step_out_kernel<false><<<(n_envs + 127) / 128, 128, 0, st>>>(ptr, reward, terminal, delta);
  return cudaGetLastError();
}

__device__ __noinline__ void flow_next_dev(rlm_flow_state* s, rlm_tick_msg* m) {
  rlm_flow_next(s, &P.flow, rlm_flow_skellam20_lut, rlm_flow_pois30_lut, rlm_flow_pois1p5_lut, m);
}
// warp version of rlm_flow_next (include/rlm_flow.h): lanes 0..2 evaluate the three Philox calls; the book part of
// rlm_flow_apply runs one LEVEL per lane -- lanes 0..4 = ask levels, 5..9 = bid levels: the shift of the level volumes, the
// Skellam add/cancel draw, the level's price and its slot in the message -- and the prints one PRICE per lane (lanes
// 0..3 = bid-1, bid, ask, ask+1).  Same integer arithmetic as the host function, statement by statement; the generated
// stream is compared with the host's bit for bit (tests/test_gpu_parity.py::test_stream_mode_equals_generator_mode).
__device__ __forceinline__ uint32_t flow_fresh3(uint32_t f0, uint32_t f1, uint32_t f2, int i) { return i == 0 ? f0 : (i == 1 ? f1 : f2); }
__device__ __noinline__ void flow_next_warp(rlm_flow_state* s, rlm_tick_msg* m, unsigned* r12 /* 12 words of shared memory */, int lane) {
  if (lane < 3) rlm_flow_draw(s, (uint32_t)lane, r12 + 4 * lane);
  __syncwarp();
  const rlm_flow_params* p = &P.flow;
  const uint32_t* r0 = r12;
  const uint32_t* r1 = r12 + 4;
  const uint32_t* r2 = r12 + 8;
  const int32_t tick = s->tick, bid_tick = s->bid_tick, spread = s->spread;
  // ---- prints against the PRE-update book: lane j < 4 sums the prints that land on price j (ascending price)
  const int32_t pa = bid_tick + spread, pb = bid_tick;
  const int n_prints = (tick == 0) ? 0 : (int)rlm_flow_pois1p5_lut[(r0[0] >> 24) & 0xFFu];
  int32_t agg = 0;
  if (lane < 4) {
#pragma unroll 1
    for (int i = 0; i < n_prints; ++i) {
      const uint32_t bits = (r0[1] >> (12 + 3 * i)) & 7u;
      const uint32_t u12 = (i < 2) ? ((r2[1] >> (12 * i)) & 0xFFFu) : ((r2[2] >> (12 * (i - 2))) & 0xFFFu);
      const int deep = ((int)(bits >> 1) < p->p_deep_u2) ? 1 : 0;
      const int slot = (bits & 1u) ? 2 + deep : 1 - deep;
      if (slot == lane) agg += 1 + (int32_t)rlm_flow_pois30_lut[u12];
    }
  }
  const unsigned txm = __ballot_sync(FULL, lane < 4 && agg > 0);
  // ---- evolve the book (not on the very first row): every lane derives the scalars, lanes 0..9 own one level each
  int move = 0, new_spread = spread;
  const bool evolve = tick > 0;
  if (evolve) {
    const uint32_t um = r0[0] & 0xFFFu;
    if ((int32_t)um < p->p_move_u12 / 2) move = -1;
    else if ((int32_t)um < p->p_move_u12) move = +1;
    if ((int32_t)((r0[0] >> 12) & 0xFFFu) < p->p_spread_u12) {
      const uint32_t us = r0[1] & 0xFFFu;
      new_spread = ((int32_t)us < p->spread_c1_u12) ? 1 : (((int32_t)us < p->spread_c2_u12) ? 2 : 3);
    }
    if (bid_tick + move - (RLM_DEPTH - 1) < p->tick_lo) move = +1;
    if (bid_tick + move + new_spread + (RLM_DEPTH - 1) > p->tick_hi) move = -1;
  }
  const int32_t new_bid = bid_tick + move;
  const bool is_bid = lane >= RLM_DEPTH;
  const int l = is_bid ? lane - RLM_DEPTH : lane;
  int32_t v = 0;
  if (lane < 2 * RLM_DEPTH) {
    const int32_t* vol = is_bid ? s->bid_vol : s->ask_vol;
    v = vol[l];
    if (evolve) {
      // rlm_flow_shift: bid best moves by `move` (d = -move), ask best by move + (new_spread - spread) (d = +shift)
      const int d = is_bid ? -move : move + (new_spread - spread);
      const uint32_t f0 = is_bid ? (r0[3] >> 16) : (r0[2] & 0xFFFFu);
      const uint32_t f1 = is_bid ? ((r0[3] >> 8) & 0xFFFFu) : (r0[2] >> 16);
      const uint32_t f2 = is_bid ? ((r0[2] >> 8) & 0xFFFFu) : (r0[3] & 0xFFFFu);
      if (d > 0) {
        const int src = l + d;
        v = (src < RLM_DEPTH) ? vol[src] : (int32_t)(100u + flow_fresh3(f0, f1, f2, (l + d - RLM_DEPTH) % 3) % 800u);
      } else if (d < 0) {
        const int src = l + d;
        v = (src >= 0) ? vol[src] : (int32_t)(100u + flow_fresh3(f0, f1, f2, l % 3) % 800u);
      }
      // depth add - cancel per level: draws 0..4 ask, 5..9 bid
      const uint32_t w = (lane < 8) ? r1[lane >> 1] : r2[0];
      const uint32_t u = (lane & 1) ? ((w >> 12) & 0xFFFu) : (w & 0xFFFu);
      v += (int32_t)rlm_flow_skellam20_lut[u];
      v = v < 1 ? 1 : v;
    }
  }
  __syncwarp();  // every lane has read the old level volumes and the old state scalars
  if (lane < 2 * RLM_DEPTH) {
    if (is_bid) { s->bid_vol[l] = v; m->bid_vol[l] = v; m->bid_px[l] = rlm_flow_px(p, new_bid - l); }
    else { s->ask_vol[l] = v; m->ask_vol[l] = v; m->ask_px[l] = rlm_flow_px(p, new_bid + new_spread + l); }
  }
  if (lane < RLM_N_TX_MAX) {  // aggregated prints, ascending price, compacted: {pb - 1, pb, pa, pa + 1}
    const int32_t agg_tick = lane == 0 ? pb - 1 : (lane == 1 ? pb : (lane == 2 ? pa : pa + 1));
    const int n_tx = __popc(txm);
    if (agg > 0) {
      const int pos = __popc(txm & ((1u << lane) - 1u));
      m->tx_px[pos] = rlm_flow_px(p, agg_tick);
      m->tx_vol[pos] = agg;
    }
    if (lane >= n_tx) { m->tx_px[lane] = 0.0f; m->tx_vol[lane] = 0; }
    if (lane == 0) {
      m->n_tx = n_tx;
      m->time_ms = p->t0_ms + (tick + 1) * p->dt_ms;
      m->date = p->date;
      m->flags = 0;
      s->bid_tick = new_bid;
      s->spread = new_spread;
      s->tick = tick + 1;
    }
  }
}

// One market tick of one env (thread-per-env).  Returns -1, or the ready kind: 0 = a learner step
// ended (state variables + reward are in e.ag), 1 = warm-up ended (Intraday::Initialise done).
template <class... M>
__device__ __forceinline__ int env_tick_in(EnvHdr& e, double* ring, const rlm_tick_msg& msg, int backtest, M... mk) {
  const int phase = e.phase;
  const bool multi = needs_multi(e, msg);  // ingested real data: this tick spans several messages (rlm_flow.h)
  if (phase == PH_PREOPEN) {  // intraday.cpp:111-116: rows before the open only update the book
    if (multi) {
      if (update_book_profiles_multi(e, msg, false) && market_is_open(e, mk...)) e.phase = PH_WARMUP;
      return -1;
    }
    rlm_tick_msg none = msg;
    none.n_tx = 0;
    update_book_profiles(e, none);
    if (market_is_open(e, mk...)) e.phase = PH_WARMUP;
    return -1;
  }
  double pushv[RLM_NWIN], oldv[RLM_NWIN];
#pragma unroll
  for (int w = 0; w < RLM_NWIN; ++w) oldv[w] = window_peek(e, ring, w);  // 10 independent loads, consumed after the book logic
  if (phase == PH_RUN) e.pnl_step = 0.0;  // base.cpp:286
  if (multi) { if (!next_state_multi(e, msg, pushv, mk...)) return -2; }  // (message consumed, tick not complete yet)
  else next_state_scalar(e, msg, pushv, mk...);  // Intraday::NextState
#pragma unroll 1
  for (int w = 0; w < 8; ++w) window_push(e, ring, w, pushv[w], oldv[w]);
  e.tp_val = e.w_mean[W_TP];
  if (phase == PH_WARMUP) {  // intraday.cpp:118-135
    bool full = true;
#pragma unroll 1
    for (int w = 0; w < 8; ++w) full = full && (e.w_count[w] == P.win_size[w]);
    if (!full) return -1;
    place_orders(e, 1, 1, mk...);
    e.phase = PH_RUN;
    e.ag.kind = 1;  // serial.cpp:24-25,55-60: the first from-state is the never-populated State
    if (backtest) {  // Backtester::_step builds its state from the env before every action (serial.cpp:126)
#pragma unroll 1
      for (int i = 0; i < P.n_state_vars; ++i) e.ag.to_vars[i] = (float)get_variable(e, ring, P.state_vars[i], mk...);
    }
    return 1;
  }
  // tail of one iteration of performAction's do-while (base.cpp:292-305)
  double mpm = m_midprice(e) - m_last_midprice(e);
  e.pnl_step += (double)e.position * mpm;
  e.momentum_pnl_step += (double)e.position * mpm;
  e.agg_r += get_reward(e);
  e.agg_pnl += e.pnl_step;
  e.agg_mpm += mpm;
  if (!is_terminal(e, mk...) && fabs(e.agg_mpm) < 1e-5) return -1;
  // base.cpp:317-331
  e.pnl_step = e.agg_pnl;
  window_push(e, ring, W_PNLUP, fmax(0.0, e.pnl_step), oldv[W_PNLUP]);
  window_push(e, ring, W_PNLDN, fabs(fmin(0.0, e.pnl_step)), oldv[W_PNLDN]);
  e.ep_reward += e.agg_r;
  e.ep_bandh += e.agg_mpm;
  // State::newState -> Intraday::getState (state.cpp:35-43, intraday.cpp:411-416); serial.cpp:64-65
#pragma unroll 1
  for (int i = 0; i < P.n_state_vars; ++i) e.ag.to_vars[i] = (float)get_variable(e, ring, P.state_vars[i], mk...);
  e.ag.last_reward = get_reward(e);
  e.ag.kind = 0;
  e.ag.hs_valid = 0;  // (one thread per env: the learner kernel hashes the to-state itself)
  return 0;
}

__device__ __noinline__ int env_tick(EnvHdr& e, double* ring, const rlm_tick_msg& msg, int backtest) { return env_tick_in(e, ring, msg, backtest); }
__device__ __noinline__ int env_tick(EnvHdr& e, double* ring, const rlm_tick_msg& msg, int backtest, EnvMarket mk) {
  return env_tick_in(e, ring, msg, backtest, mk);
}

// TAPE: instantiation for the tape source (the other sources' code is the same as without it); MKT: ... whose days run
// under markets of their own (rlm_set_day_markets)
template <int THREADS, bool TAPE, bool MKT = false>
__global__ void __launch_bounds__(THREADS) rlm_env_kernel(DevPtrs ptr, DynParams D, int tslot, int only_begin) {
  const int b = D.env0 + blockIdx.x * THREADS + threadIdx.x;
  const int lane = threadIdx.x & 31;
  if (!only_begin) KLOG_BEGIN(0);
  int ready = -1;
  unsigned ticked = 0, errs = 0;
  bool starved = false;  // tape source: this env needed a message past the end of its day
  if (b < (D.n_sub > 0 ? D.env0 + D.n_sub : P.n_envs)) {
    EnvHdr* g = (EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
    // tape source: the cursor comes from its own array, so its load is in flight together with the record copy below
    const int2 tc = (TAPE && !only_begin) ? ptr.tape_cur[b] : make_int2(0, 0);
    const EnvMarket mk = env_market_of<MKT>(b);
    const int ph = g->phase;
    const int nb = D.hold ? 0 : g->ag.need_begin;
    if (ph != PH_DONE && (!only_begin || nb) && !(D.hold && env_on_hold(*g))) {
      // thread-local copy: local memory is lane-interleaved == SoA across the warp.  The agent block (the last 700 of the
      // record's 2 000 bytes) only travels when this tick touches it: an action selection now, or a step end below.
      EnvHdr e;
      constexpr int HOT16 = (int)(offsetof(EnvHdr, ag) / 16), ALL16 = (int)(sizeof(EnvHdr) / 16);
      static_assert(offsetof(EnvHdr, ag) % 16 == 0 && sizeof(EnvHdr) % 16 == 0, "16-byte copies of the two halves of the record");
      bool ag_in = nb || D.hold || D.backtest;
      {
        const int4* src = (const int4*)g;
        int4* dst = (int4*)&e;
        for (int i = 0; i < HOT16; ++i) dst[i] = src[i];
        if (ag_in) for (int i = HOT16; i < ALL16; ++i) dst[i] = src[i];
        else e.ag.err = 0;
      }
      double* ring = (double*)((unsigned char*)g + sizeof(EnvHdr));
      if (nb) {
        on_market<MKT>(mk, [&](auto... m) { begin_step(e, ptr.mt_pol + (size_t)b * 312, D, m...); });
        e.ag.need_begin = 0;
      }
      if (!only_begin && e.phase != PH_DONE) {
        rlm_tick_msg msg;
        bool have = true;
        if (TAPE) {
          // the env's own day: message tc.x, then the cursor moves on; past the day's end the env waits inside performAction
          if (tc.x >= tc.y) { have = false; starved = true; }
          else {
            const int4* src = (const int4*)(ptr.tape + tc.x);
            int4* dst = (int4*)&msg;
#pragma unroll
            for (int i = 0; i < 8; ++i) dst[i] = __ldg(src + i);
            ptr.tape_cur[b].x = tc.x + 1;
          }
        } else if (P.source == RLM_SOURCE_GENERATOR) {
          flow_next_dev(&e.flow, &msg);
        } else {
          // tick-synchronous: every env consumes the same tick index.  Under a CUDA graph the call's stream pointer,
          // offset and length are read from device memory (the graph outlives rlm_load_ticks and the run calls)
          const rlm_tick_msg* sp = ptr.stream;
          int s_off = D.stream_off, s_n = D.stream_ticks;
          if (D.ctl_stream) {
            const int4 rc4 = __ldg((const int4*)ptr.runctl);
            s_off = rc4.z; s_n = rc4.w;
            sp = (const rlm_tick_msg*)__ldg((const unsigned long long*)ptr.runctl + 2);
          }
          const int pos = s_off + tslot;
          if (pos >= s_n) { e.err |= ERR_STREAM_UNDERRUN; have = false; }
          else {
            const int4* src = (const int4*)(sp + ((size_t)pos * P.n_envs + b));
            int4* dst = (int4*)&msg;
#pragma unroll
            for (int i = 0; i < 8; ++i) dst[i] = __ldg(src + i);
          }
        }
        if (have) {
          const int was = e.phase;
          ready = on_market<MKT>(mk, [&](auto... m) { return env_tick(e, ring, msg, D.backtest, m...); });
          if (was != PH_PREOPEN && ready != -2) ticked = 1;
          if (ready == -2) ready = -1;
        }
      }
      if (ready >= 0 && !ag_in) {
        // a step (or the warm-up) ended on an env whose agent block was not loaded: env_tick wrote the to-state, the
        // reward and the ready kind into the local copy -- put them on top of the block in HBM
        const int kind = e.ag.kind;
        const double rew = e.ag.last_reward;
        float tv[RLM_N_STATE_MAX];
        for (int i = 0; i < RLM_N_STATE_MAX; ++i) tv[i] = (i < P.n_state_vars) ? e.ag.to_vars[i] : 0.0f;
        const int4* src = (const int4*)g;
        int4* dst = (int4*)&e;
        for (int i = HOT16; i < ALL16; ++i) dst[i] = src[i];
        e.ag.kind = kind;
        if (kind == 0) {
          e.ag.last_reward = rew; e.ag.hs_valid = 0;
          for (int i = 0; i < RLM_N_STATE_MAX; ++i) if (i < P.n_state_vars) e.ag.to_vars[i] = tv[i];
        }
        ag_in = true;
      }
      errs = (unsigned)(e.err | e.ag.err);
      {
        int4* dst = (int4*)g;
        const int4* src = (const int4*)&e;
        for (int i = 0; i < HOT16; ++i) dst[i] = src[i];
        if (ag_in) for (int i = HOT16; i < ALL16; ++i) dst[i] = src[i];
      }
    }
  }
  if (D.hold) {  // split surface: envs still inside their step after this launch
    bool still = false;
    if (b < (D.n_sub > 0 ? D.env0 + D.n_sub : P.n_envs) && ready < 0 && !only_begin) {
      const EnvHdr* g = (const EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
      still = g->phase != PH_DONE && !env_on_hold(*g) && !starved;
    }
    const unsigned rm = __ballot_sync(FULL, still);
    if (rm && lane == 0) atomicAdd(&ptr.counters[5], (unsigned long long)__popc(rm));
  }
  // ready list: one atomic per warp
  const unsigned m = __ballot_sync(FULL, ready >= 0);
  if (m) {
    const int leader = __ffs(m) - 1;
    int base = 0;
    if (lane == leader) base = atomicAdd(&ptr.ready_count[tslot], __popc(m));
    base = __shfl_sync(FULL, base, leader);
    if (ready >= 0) ptr.ready[base + __popc(m & ((1u << lane) - 1u))] = b;
  }
  if (!only_begin) KLOG_END(0);
  const unsigned tm = __ballot_sync(FULL, ticked != 0);
  unsigned em = errs;
  for (int o = 16; o > 0; o >>= 1) em |= __shfl_xor_sync(FULL, em, o);
  if (lane == 0) {
    if (tm) atomicAdd(&ptr.counters[0], (unsigned long long)__popc(tm));
    if (em) atomicOr(&ptr.counters[4], (unsigned long long)em);
  }
}

// ---------------------------------------------------------------------------------------------
// Env tick, one WARP per env (the latency-oriented variant; default).  The env record is staged in
// shared memory with coalesced 16-byte copies; lane 0 runs the scalar market logic, lanes 0..9 own one
// rolling window each (ring loads are issued first so their HBM/L2 round trips overlap the book logic),
// lanes 0..7 each evaluate one state variable at a step end.  No env waits for another one: a warp whose
// env needs the learner step just appends it to the ready list.
#define ENVW_WARPS 8  // most warps per CTA (launch bounds)
#define ENVW_WARPS_DEFAULT 8
// per-warp shared memory of the tick: [EnvHdr][message 128][pushv, oldv: 2 x 10 doubles][flag 16, Philox 48, fills + errs 64]
__host__ __device__ inline size_t envw_hdr_bytes() { return (sizeof(EnvHdr) + 15) & ~(size_t)15; }
__host__ __device__ inline size_t envw_warp_bytes() { return envw_hdr_bytes() + 128 + 8 * 2 * RLM_NWIN + 128; }
struct EnvWarp {
  EnvHdr* e; rlm_tick_msg* msg; double* pushv; double* oldv; int* flag; unsigned* r12; Fill* fills;
};
__device__ __forceinline__ EnvWarp envw_carve(unsigned char* wbase) {
  EnvWarp w;
  const size_t hb = envw_hdr_bytes();
  w.e = (EnvHdr*)wbase;
  w.msg = (rlm_tick_msg*)(wbase + hb);
  w.pushv = (double*)(wbase + hb + 128);
  w.oldv = w.pushv + RLM_NWIN;
  w.flag = (int*)(w.oldv + RLM_NWIN);
  w.r12 = (unsigned*)(w.flag + 4);
  w.fills = (Fill*)(w.r12 + 12);  // 2 Fill + 2 ints
  return w;
}
// env record HBM <-> shared memory, coalesced 16-byte copies; the loads of one record are all in flight together
__device__ __forceinline__ void envw_stage_in(EnvHdr* dst_e, const EnvHdr* g, int lane) {
  const int4* src = (const int4*)g;
  int4* dst = (int4*)dst_e;
  const int n16 = (int)(envw_hdr_bytes() / 16);
  static_assert(sizeof(EnvHdr) <= 4 * 32 * 16, "four 16-byte loads per lane cover the env header");
  int4 t[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) { const int i = lane + 32 * k; if (i < n16) t[k] = src[i]; }
#pragma unroll
  for (int k = 0; k < 4; ++k) { const int i = lane + 32 * k; if (i < n16) dst[i] = t[k]; }
}
// envw_stage_in on the tape source.  The env's cursor is loaded first and this lane's word of the env's next message
// between the record's loads and their stores to shared memory: the message waits for the cursor only, never for the
// record.  l2_next: also ask L2 for the message after it (the next launch's), one 128-byte line.
__device__ __forceinline__ unsigned envw_stage_in_tape(EnvHdr* dst_e, const EnvHdr* g, const DevPtrs& ptr, int env, int lane, bool l2_next,
                                                       int2& tc) {
  tc = ptr.tape_cur[env];
  const int4* src = (const int4*)g;
  int4* dst = (int4*)dst_e;
  const int n16 = (int)(envw_hdr_bytes() / 16);
  int4 t[4];
#pragma unroll
  for (int k = 0; k < 4; ++k) { const int i = lane + 32 * k; if (i < n16) t[k] = src[i]; }
  unsigned word = 0;
  if (tc.x < tc.y) word = __ldg((const unsigned*)(ptr.tape + tc.x) + lane);
  if (l2_next && lane == 0 && tc.x + 1 < tc.y) asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr.tape + tc.x + 1));
#pragma unroll
  for (int k = 0; k < 4; ++k) { const int i = lane + 32 * k; if (i < n16) dst[i] = t[k]; }
  return word;
}
__device__ __forceinline__ void envw_stage_out(EnvHdr* g, const EnvHdr* src_e, int lane) {
  int4* dst = (int4*)g;
  const int4* src = (const int4*)src_e;
  for (int i = lane; i < (int)(envw_hdr_bytes() / 16); i += 32) dst[i] = src[i];
}

// One market tick of the env staged in `w`, by its warp.  stream_pos: index of this tick in the resident stream chunk.
// Tape source: stream_pos / stream_ticks are the env's cursor and the end of its day, and tape_word is this lane's word of
// message stream_pos, loaded by the caller ahead of the record's stage-in.
// Returns -1, or the ready kind (0: a learner step ended -- state variables and reward are in e.ag; 1: warm-up ended).
template <bool TAPE = false, class... M>
__device__ __forceinline__ int envw_tick(const EnvWarp& w, double* ring, const DevPtrs& ptr, const DynParams& D, int env, int stream_pos,
                                         int stream_ticks, int lane, unsigned& ticked, unsigned tape_word = 0, M... mk) {
  EnvHdr& e = *w.e;
  rlm_tick_msg& msg = *w.msg;
  double* pushv = w.pushv;
  double* oldv = w.oldv;
  int ready = -1;
  bool have = true;
  if (TAPE) {
    if (stream_pos >= stream_ticks) have = false;  // (callers only tick an env whose day has messages left)
    else ((unsigned*)&msg)[lane] = tape_word;
  } else if (P.source == RLM_SOURCE_GENERATOR) {
    flow_next_warp(&e.flow, &msg, w.r12, lane);
  } else {
    if (stream_pos >= stream_ticks) { if (lane == 0) e.err |= ERR_STREAM_UNDERRUN; have = false; }
    else ((unsigned*)&msg)[lane] = __ldg((const unsigned*)(ptr.stream + ((size_t)stream_pos * P.n_envs + env)) + lane);
  }
  if (lane < RLM_NWIN) oldv[lane] = window_peek(e, ring, lane);  // issued early, consumed after the book logic
  __syncwarp();
  const int phase = e.phase;
  const bool multi = have && needs_multi(e, msg);  // ingested real data: this tick spans several messages (rlm_flow.h)
  int complete = 1;
  if (multi && phase != PH_PREOPEN) {  // lane 0 runs the one-thread version; the tick may not be complete yet
    if (lane == 0) {
      if (phase == PH_RUN) e.pnl_step = 0.0;  // base.cpp:286
      complete = next_state_multi(e, msg, pushv, mk...) ? 1 : 0;
    }
    complete = __shfl_sync(FULL, complete, 0);
  }
  if (have && phase == PH_PREOPEN) {  // intraday.cpp:111-116
    if (lane == 0) {
      if (multi) {
        if (update_book_profiles_multi(e, msg, false) && market_is_open(e, mk...)) e.phase = PH_WARMUP;
      } else {
        msg.n_tx = 0;
        update_book_profiles(e, msg);
        if (market_is_open(e, mk...)) e.phase = PH_WARMUP;
      }
    }
  } else if (have && complete) {
    ticked += 1;
    if (!multi) {
      if (lane == 0 && phase == PH_RUN) e.pnl_step = 0.0;  // base.cpp:286
      __syncwarp();
      next_state_warp(e, msg, pushv, w.fills, lane, mk...);  // Intraday::NextState, ask side on lane 0, bid side on lane 1
    }
    __syncwarp();
    if (lane < 8) window_push(e, ring, lane, pushv[lane], oldv[lane]);
    __syncwarp();
    if (lane == 0) {
      int r = -1;
      e.tp_val = e.w_mean[W_TP];
      if (phase == PH_WARMUP) {  // intraday.cpp:118-135
        bool full = true;
        for (int k = 0; k < 8; ++k) full = full && (e.w_count[k] == P.win_size[k]);
        if (full) {
          place_orders(e, 1, 1, mk...);
          e.phase = PH_RUN;
          e.ag.kind = 1;  // serial.cpp:24-25,55-60: the first from-state is the never-populated (or the stale) State
          r = 1;
        }
      } else {
        // tail of one iteration of performAction's do-while (base.cpp:292-305)
        double mpm = m_midprice(e) - m_last_midprice(e);
        e.pnl_step += (double)e.position * mpm;
        e.momentum_pnl_step += (double)e.position * mpm;
        e.agg_r += get_reward(e);
        e.agg_pnl += e.pnl_step;
        e.agg_mpm += mpm;
        if (!(!is_terminal(e, mk...) && fabs(e.agg_mpm) < 1e-5)) {
          e.pnl_step = e.agg_pnl;  // base.cpp:317-331
          pushv[W_PNLUP] = fmax(0.0, e.pnl_step);
          pushv[W_PNLDN] = fabs(fmin(0.0, e.pnl_step));
          e.ep_reward += e.agg_r;
          e.ep_bandh += e.agg_mpm;
          r = 0;
        }
      }
      *w.flag = r;
    }
    __syncwarp();
    ready = *w.flag;
    if (ready == 0) {
      if (lane == W_PNLUP || lane == W_PNLDN) window_push(e, ring, lane, pushv[lane], oldv[lane]);
      __syncwarp();
      // State::newState -> Intraday::getState (state.cpp:35-43, intraday.cpp:411-416): one variable per lane.  The
      // variables built from two Market::ToTicks conversions (spd, mpm, a_dist, b_dist) make those calls together, in
      // two convergent passes, instead of eight calls one switch case after the other (this is the critical path of the
      // launch: the warps whose step ends are the last ones to finish)
      {
        const bool has = lane < P.n_state_vars;
        const int var = has ? P.state_vars[lane] : -1;
        double x0 = 0.0, x1 = 0.0;
        const bool two = has && var_tick_args(e, ring, var, x0, x1);
        int t0 = 0, t1 = 0, lerr = 0, hint = e.tk_band;
        if (two) { t0 = to_ticks(mk..., x0, &lerr, &hint); t1 = to_ticks(mk..., x1, &lerr, &hint); }
        if (lerr) atomicOr(&e.err, lerr);
        if (has) e.ag.to_vars[lane] = (float)(two ? var_from_ticks(var, t0, t1) : get_variable(e, ring, var, mk...));
      }
      if (lane == 31) { e.ag.last_reward = get_reward(e); e.ag.kind = 0; }
      if (D.env_hash && !D.backtest && !P.shared_policy && P.algorithm < RLM_ALGO_R_LEARN) {
        // OPTIONAL (RLM_ENV_HASH=1; off by default): hash the to-state here -- 31 lanes of this warp idle anyway -- hand
        // the sums to the learner kernel and ask L2 for the step's 864 sectors now.  At C1 one tick's 1.04 M sectors
        // occupy 1.04 M 128-byte L2 lines = 133 MB, more than L2 holds, so the learner kernel still misses and the
        // prefetches add DRAM traffic, while the extra instructions lengthen this latency-bound kernel.
        __syncwarp();
        const LnSums h = ln_hash(rlm_rndseq_table, e.ag.to_vars, false, lane);
        unsigned long long* hs = ptr.hsum + (size_t)env * 96;
        hs[lane] = h.s[0]; hs[32 + lane] = h.s[1]; hs[64 + lane] = h.s[2];
        const double* th_a = ptr.theta + (size_t)env * (size_t)P.memory_size;
        const double* th_b = ptr.theta_b ? ptr.theta_b + (size_t)env * (size_t)P.memory_size : nullptr;
#pragma unroll 1
        for (int g = 0; g < 3; ++g) {
#pragma unroll
          for (int a = 0; a < RLM_MAX_ACTIONS; ++a) {
            if (a < P.n_actions) {
              const int f = mod_m(h.s[g] + P.rg[g][a]);
              asm volatile("prefetch.global.L2 [%0];" ::"l"(th_a + f));
              if (th_b) asm volatile("prefetch.global.L2 [%0];" ::"l"(th_b + f));
            }
          }
        }
        if (lane == 0) e.ag.hs_valid = 1;
      }
    } else if (ready == 1 && D.backtest) {
      // Backtester::_step builds its state from the env before every action (serial.cpp:126), the first one included
      if (lane < P.n_state_vars) e.ag.to_vars[lane] = (float)get_variable(e, ring, P.state_vars[lane], mk...);
    }
  }
  __syncwarp();
  return ready;
}

template <bool TAPE, bool MKT = false>
__global__ void __launch_bounds__(ENVW_WARPS * 32) rlm_env_kernel_w(DevPtrs ptr, DynParams D, int tslot, int only_begin) {
  PDL_PROLOGUE();
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int env = D.env0 + blockIdx.x * (blockDim.x >> 5) + warp;  // (warps per CTA: rlm_launch_env, <= ENVW_WARPS)
  if (!only_begin) KLOG_BEGIN(0);
  if (env >= (D.n_sub > 0 ? D.env0 + D.n_sub : P.n_envs)) return;
  const EnvWarp w = envw_carve(smem + (size_t)warp * envw_warp_bytes());
  EnvHdr& e = *w.e;
  EnvHdr* g = (EnvHdr*)(ptr.env + (size_t)env * P.env_stride);
  double* ring = (double*)((unsigned char*)g + sizeof(EnvHdr));
  // the trailing begin-only pass touches few envs: look before staging.  A tick pass stages straight away -- one
  // memory round trip instead of two on every env's critical path -- and drops finished envs afterwards.
  if (only_begin && !g->ag.need_begin) return;
  const EnvMarket mk = env_market_of<MKT>(env);
  const bool tape = TAPE && !only_begin;
  int2 tc = make_int2(0, 0);
  unsigned tape_word = 0;
  if (tape) tape_word = envw_stage_in_tape(&e, g, ptr, env, lane, D.tape_l2 != 0, tc);
  else envw_stage_in(&e, g, lane);
  __syncwarp();
  if (e.phase == PH_DONE) return;
  if (D.hold && env_on_hold(e)) return;
  int ready = -1;
  unsigned ticked = 0;
  bool starved = false;  // tape source: this env needs a message past the end of its day
  if (e.ag.need_begin) on_market<MKT>(mk, [&](auto... m) { begin_step_warp(e, ptr.mt_pol + (size_t)env * 312, D, w.flag, lane, m...); });
  if (!only_begin && e.phase != PH_DONE) {
    if (tape) {
      starved = tc.x >= tc.y;
      if (!starved) {
        ready = on_market<MKT>(mk, [&](auto... m) { return envw_tick<true>(w, ring, ptr, D, env, tc.x, tc.y, lane, ticked, tape_word, m...); });
        if (lane == 0) ptr.tape_cur[env].x = tc.x + 1;
      }
    } else if (D.ctl_stream) {  // (see rlm_env_kernel: stream pointer, offset and length of this call live in *ptr.runctl)
      const int4 rc4 = __ldg((const int4*)ptr.runctl);
      DevPtrs pt = ptr;
      pt.stream = (const rlm_tick_msg*)__ldg((const unsigned long long*)ptr.runctl + 2);
      ready = envw_tick(w, ring, pt, D, env, rc4.z + tslot, rc4.w, lane, ticked);
    } else {
      ready = envw_tick(w, ring, ptr, D, env, D.stream_off + tslot, D.stream_ticks, lane, ticked);
    }
  }
  __syncwarp();
  envw_stage_out(g, &e, lane);
  if (!only_begin) KLOG_END(0);
  if (lane == 0) {
    if (ready >= 0) ptr.ready[atomicAdd(&ptr.ready_count[tslot], 1)] = env;
    if (D.hold && ready < 0 && e.phase != PH_DONE && !starved) atomicAdd(&ptr.counters[5], 1ull);  // still inside its step
    if (ticked) atomicAdd(&ptr.counters[0], 1ull);
    const unsigned errs = (unsigned)(e.err | e.ag.err);
    if (errs) atomicOr(&ptr.counters[4], (unsigned long long)errs);
  }
}

// Round-paced tick kernel (independent policies): every env runs its OWN ticks until a step ends (or the run call's
// ticks are used up), then waits for the learner kernel -- so a round is one learner step of EVERY live env instead of
// the ~30 % whose midprice happened to move this tick, and the two launches' latencies are paid once per env step
// instead of once per market tick.  Envs never exchange anything (own book, own stream, own weights), so the order in
// which their ticks run is not observable: per env the sequence begin_step / tick / ... / learner step is the same as
// in the tick-synchronous engine, bit for bit.  The per-call values live in *ptr.runctl (graphs are reused across calls).
template <bool TAPE, bool MKT = false>
__global__ void __launch_bounds__(ENVW_WARPS * 32, 4) rlm_env_round_kernel(DevPtrs ptr, DynParams D, int tslot) {
  PDL_PROLOGUE();
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int env = D.env0 + blockIdx.x * (blockDim.x >> 5) + warp;
  KLOG_BEGIN(0);
  if (env >= (D.n_sub > 0 ? D.env0 + D.n_sub : P.n_envs)) return;
  // live envs of a round = those that left it with a learner step due or with ticks of this call still to run (counted
  // behind the ready counters): none a round ago, nothing to do
  int* live_count = ptr.ready_count + RLM_LIVE_OFF;
  if (tslot > 0 && __ldcg(live_count + tslot - 1) == 0) return;
  const int4 rc4 = __ldg((const int4*)ptr.runctl);
  const RunCtl rc = {rc4.x, rc4.y, rc4.z, rc4.w, nullptr, 0};
  DevPtrs pt = ptr;
  pt.stream = (const rlm_tick_msg*)__ldg((const unsigned long long*)ptr.runctl + 2);
  const EnvWarp w = envw_carve(smem + (size_t)warp * envw_warp_bytes());
  EnvHdr& e = *w.e;
  EnvHdr* g = (EnvHdr*)(ptr.env + (size_t)env * P.env_stride);
  double* ring = (double*)((unsigned char*)g + sizeof(EnvHdr));
  const bool tape = TAPE;
  const EnvMarket mk = env_market_of<MKT>(env);
  int2 tc = make_int2(0, 0);
  unsigned tape_word = 0;
  if (tape) tape_word = envw_stage_in_tape(&e, g, ptr, env, lane, false, tc);
  else envw_stage_in(&e, g, lane);
  __syncwarp();
  if (e.phase == PH_DONE) return;
  int pos = e.run_id == rc.run_id ? e.run_pos : 0;
  if (pos >= rc.n_ticks && !e.ag.need_begin) return;
  int ready = -1;
  unsigned ticked = 0;
  // D.round_cap > 0 bounds the ticks of one round: an env whose step has not ended by then simply comes back in the
  // next round, so that a round's tick kernel does not wait for the env with the longest run of unchanged midprices
  const int cap = D.round_cap > 0 ? D.round_cap : 0x7fffffff;
  int n_run = 0;
  bool starved = false;  // tape source: the env's day has run out (it waits inside performAction, consuming nothing)
#pragma unroll 1
  for (;;) {
    if (e.ag.need_begin) on_market<MKT>(mk, [&](auto... m) { begin_step_warp(e, ptr.mt_pol + (size_t)env * 312, D, w.flag, lane, m...); });
    if (e.phase == PH_DONE || pos >= rc.n_ticks || n_run >= cap) break;
    if (tape) {
      if (tc.x >= tc.y) { starved = true; break; }
      const unsigned word = tape_word;
      if (tc.x + 1 < tc.y) tape_word = __ldg((const unsigned*)(ptr.tape + tc.x + 1) + lane);  // the next tick's, in flight during this one
      ready = on_market<MKT>(mk, [&](auto... m) { return envw_tick<true>(w, ring, pt, D, env, tc.x, tc.y, lane, ticked, word, m...); });
      ++tc.x;
    } else {
      ready = envw_tick(w, ring, pt, D, env, rc.stream_off + pos, rc.stream_ticks, lane, ticked);
    }
    ++pos; ++n_run;
    if (ready >= 0) break;
  }
  if (lane == 0) {
    e.run_id = rc.run_id; e.run_pos = pos;
    if (tape) {
      ptr.tape_cur[env].x = tc.x;
      if (D.tape_l2 && tc.x < tc.y) asm volatile("prefetch.global.L2 [%0];" ::"l"(ptr.tape + tc.x));  // the next round's first
    }
  }
  __syncwarp();
  envw_stage_out(g, &e, lane);
  KLOG_END(0);
  if (lane == 0) {
    if (ready >= 0) ptr.ready[atomicAdd(&ptr.ready_count[tslot], 1)] = env;
    if (ready >= 0 || (e.phase != PH_DONE && pos < rc.n_ticks && !starved)) atomicAdd(&live_count[tslot], 1);
    if (ticked) atomicAdd(&ptr.counters[0], (unsigned long long)ticked);
    const unsigned errs = (unsigned)(e.err | e.ag.err);
    if (errs) atomicOr(&ptr.counters[4], (unsigned long long)errs);
  }
}
__global__ void rlm_runctl_kernel(RunCtl* dst, RunCtl v) { *dst = v; }

// parity / profit-log record of one finished step (warp 0 of the CTA, or the env's warp).  Inlined into the training
// kernel on purpose: as a call it costs the hot path ~200 bytes of register spills (ptxas call ABI).
__device__ __forceinline__ void emit_record(const DevPtrs& ptr, const EnvHdr* g, int env, const AgentD& ag, const double* theta_a,
                                         const float* vars, int lane) {
  const int* tf = ptr.trace_f + (size_t)env * P.trace_cap;
  const float* te = ptr.trace_e + (size_t)env * P.trace_cap;
  unsigned long long h = trace_hash(tf, te, theta_a, ag.n_traces, lane);
  if (lane == 0) {
    int c = ptr.record_count[env];
    if (c < P.record_cap) {
      EnvHdr tmp;
      const int4* src = (const int4*)g;
      int4* dst = (int4*)&tmp;
      for (int i = 0; i < (int)(sizeof(EnvHdr) / 16); ++i) dst[i] = __ldcg(src + i);
      fill_record(&ptr.records[(size_t)env * P.record_cap + c], tmp, ag, h, vars);
    }
    ptr.record_count[env] = c + 1;
  }
}

__device__ __noinline__ void emit_record_ool(const DevPtrs& ptr, const EnvHdr* g, int env, const AgentD& ag, const double* theta_a,
                                             const float* vars, int lane) {
  emit_record(ptr, g, env, ag, theta_a, vars, lane);
}
// the same for a record that is resident in the warp's shared memory (fused engine)
__device__ __noinline__ void emit_record_res(const DevPtrs& ptr, const EnvHdr* e, int env, const AgentD& ag, const double* theta_a,
                                             const float* vars, int lane) {
  const int* tf = ptr.trace_f + (size_t)env * P.trace_cap;
  const float* te = ptr.trace_e + (size_t)env * P.trace_cap;
  const unsigned long long h = trace_hash(tf, te, theta_a, ag.n_traces, lane);
  if (lane == 0) {
    const int c = ptr.record_count[env];
    if (c < P.record_cap) fill_record(&ptr.records[(size_t)env * P.record_cap + c], *e, ag, h, vars);
    ptr.record_count[env] = c + 1;
  }
}

// TD error + trace decision of Agent::HandleTransition (agent.cpp:86-101); lane 0.
// out[0] = trace decay rate, out[1] = alpha*delta/N_TILINGS, out[2] = table (0 = A, 1 = B);
// R-learning agents also hand out[3] = Q(from, action) and out[4] = the bootstrap value to td_rho
__device__ __noinline__ void td_decision(AgentD& ag, const double* q_pre_a, const double* q_pre_b, unsigned long long* mt_pol,
                                         unsigned long long* mt_agt, const DynParams& D, double* out) {
  ASSUME_SHARED(&ag); ASSUME_SHARED(q_pre_a); ASSUME_SHARED(q_pre_b); ASSUME_SHARED(out); ASSUME_GLOBAL(mt_pol);
  const int action = ag.cur_action;
  const double reward = ag.last_reward;
  const double F_term = P.gamma * 0.0 - 0.0;  // potentials are 0 (base.cpp:239-242)
  float rate = P.gl;
  double delta;
  int table = 0;
  if (P.algorithm == RLM_ALGO_SARSA) {  // Agent::UpdateTraces :111-115, SARSA::UpdateWeights :300-311
    double Q1 = ag.q_from[action];
    int a2 = policy_action(ag, q_pre_a, q_pre_b, mt_pol, D);
    double Q2 = q_pre_a[a2];
    delta = reward + F_term + P.gamma * Q2 - Q1;
  } else if (P.algorithm == RLM_ALGO_Q_LEARN) {  // QLearn :272-292
    int amax = argmax_ties_fast(ag, ag.q_from);
    if (action != amax) rate = 0.0f;
    double Q = ag.q_from[action];
    int am2 = argmax_ties_fast(ag, q_pre_a);
    delta = reward + F_term + P.gamma * q_pre_a[am2] - Q;
  } else if (P.algorithm == RLM_ALGO_DOUBLE_Q_LEARN) {  // DoubleQLearn :319-353
    int amax = argmax_ties_fast(ag, ag.q_from);
    if (action != amax) rate = 0.0f;
    if (mt_uniform_real(mt_agt, ag.mt_agt_idx) > 0.5) {
      double Qa = ag.q_from[action];
      int am2 = argmax_ties_fast(ag, q_pre_a);
      delta = reward + F_term + P.gamma * q_pre_b[am2] - Qa;
      table = 0;
    } else {
      double Qb = ag.qb_from[action];
      int am2 = argmax_ties_fast(ag, q_pre_b);
      delta = reward + F_term + P.gamma * q_pre_a[am2] - Qb;
      table = 1;
    }
  } else if (P.algorithm == RLM_ALGO_R_LEARN) {  // RLearn :364-380
    int amax = argmax_ties_fast(ag, ag.q_from);
    if (action != amax) rate = 0.0f;
    double Q = ag.q_from[action];
    double mQ = q_pre_a[argmax_ties_fast(ag, q_pre_a)];
    delta = reward - ag.rho + mQ - Q;
    out[3] = Q; out[4] = mQ;
  } else if (P.algorithm == RLM_ALGO_ONLINE_R_LEARN) {  // Agent::UpdateTraces :111-115, OnlineRLearn :398-405
    double Q = ag.q_from[action];
    double gQ = q_pre_a[policy_action(ag, q_pre_a, q_pre_b, mt_pol, D)];
    delta = reward - ag.rho + gQ - Q;
    out[3] = Q; out[4] = gQ;
  } else {  // DoubleRLearn :422-451
    int amax = argmax_ties_fast(ag, ag.q_from);
    if (action != amax) rate = 0.0f;
    double Q, mQ;
    if (mt_uniform_real(mt_agt, ag.mt_agt_idx) > 0.5) {
      Q = ag.q_from[action];
      mQ = q_pre_b[argmax_ties_fast(ag, q_pre_a)];
      table = 0;
    } else {
      Q = ag.qb_from[action];
      mQ = q_pre_a[argmax_ties_fast(ag, q_pre_b)];
      table = 1;
    }
    delta = reward - ag.rho + mQ - Q;
    out[3] = Q; out[4] = mQ;
  }
  ag.last_delta = delta;
  out[0] = (double)rate;
  out[1] = (D.alpha * delta) * (1.0 / (double)RLM_N_TILINGS);  // Agent::updateQ: update / N_TILINGS (32: the reciprocal is exact)
  out[2] = (double)table;
}

// Second half of the R-learning agents' UpdateWeights (agent.cpp:382-386,407-411,453-465): rho moves when the
// updated Q(from, action) is (within 1e-7 of) the best value of the from-state under the UPDATED theta.
// q_post_a/b = Q_A/Q_B(from, .) after updateQ; lane 0.
__device__ __noinline__ void td_rho(AgentD& ag, const double* q_post_a, const double* q_post_b, const DynParams& D, const double* dec) {
  const double Q = dec[3];
  double boot = dec[4];
  const double nQ = Q + D.alpha * ag.last_delta;
  double best;
  if (P.algorithm == RLM_ALGO_DOUBLE_R_LEARN) {
    best = -1.7976931348623157e308;  // -DBL_MAX
    for (int i = 0; i < P.n_actions; i++) {
      double val = (q_post_a[i] + q_post_b[i]) / 2.0;
      if (val > best) best = val;
    }
    boot = best;  // agent.cpp:453-464 reuses `mQ` for the maximum, so the rho target is built from it
  } else {
    best = q_post_a[argmax_ties(ag, q_post_a)];  // maxQ(from_state), agent.cpp:171-174
  }
  if (nQ - best < 1e-7) ag.rho += P.beta * (ag.last_reward - ag.rho + boot - nQ);
}

#ifdef RLM_TIMING  // debug build only (see the Makefile): per-CTA phase timeline of the learner kernel
__device__ long long g_phase_clk[4096 * 16];
__device__ unsigned g_phase_sm[4096];
#define PH(i) do { if (tid == 0 && idx < 4096) { g_phase_clk[idx * 16 + (i)] = clock64(); if ((i) == 0) { unsigned s_; asm volatile("mov.u32 %0, %%smid;" : "=r"(s_)); g_phase_sm[idx] = s_; } } } while (0)
extern "C" int rlm_debug_read_phases(long long* clk, unsigned* sm) {
  cudaDeviceSynchronize();
  if (cudaMemcpyFromSymbol(clk, g_phase_clk, sizeof(long long) * 4096 * 16) != cudaSuccess) return -1;
  if (cudaMemcpyFromSymbol(sm, g_phase_sm, sizeof(unsigned) * 4096) != cudaSuccess) return -1;
  long long tp[8];
  if (cudaMemcpyFromSymbol(tp, g_tp_clk, sizeof(tp)) == cudaSuccess)
    printf("slowest trace_pass so far: %lld cycles = set build %lld + decay loop %lld + set() %lld; n=%lld decay=%lld\n", tp[0], tp[1], tp[2], tp[3],
           tp[4], tp[5]);
  return 0;
}
#else
#define PH(i) do { } while (0)
#endif

#include "rlm_learn.cuh"

// The learner step of one ready env, by one warp.  `ag` / `scratch` are this warp's shared memory.
// stage 0: the whole step (independent policies).  Shared policy (one theta per handle, SURVEY 8e):
// stage 1 = evaluate under theta_t and accumulate the update into dtheta; stage 2 (after
// theta += all-reduced dtheta) = Q(from, .) under theta_{t+1} for the next action selection.
struct AgentScratch { double* q_pre; int* sset; int* idx; double* vbuf; };
__device__ __forceinline__ AgentScratch std_scratch(unsigned char* scratch) {
  AgentScratch s;
  s.q_pre = (double*)(scratch + SCR_Q); s.sset = (int*)(scratch + SCR_SS); s.idx = (int*)(scratch + SCR_IDX);
  s.vbuf = (double*)(scratch + SCR_VBUF);
  return s;
}
// `resident` != nullptr: the env record (and `ag` = resident->ag) already lives in this warp's shared
// memory (fused kernel): nothing is staged or written back here.
__device__ __noinline__ void agent_process_env(const DevPtrs& ptr, const DynParams& D, int env, AgentD& ag, AgentScratch sc,
                                               int lane, unsigned long long& steps_done, unsigned long long& sum_z, int stage,
                                               const EnvHdr* resident) {
  const unsigned* s_rnd = rlm_rndseq_table;
  double* q_pre_a = sc.q_pre;
  double* q_pre_b = q_pre_a + RLM_MAX_ACTIONS;
  int* sset = sc.sset;
  int* idxc = sc.idx;
  double* vbuf = sc.vbuf;
  double* dec = vbuf;  // 3 doubles handed from lane 0 to the warp (vbuf is free between the evaluations)
  const int A = P.n_actions;
  EnvHdr* g = (EnvHdr*)(ptr.env + (size_t)env * P.env_stride);
  if (!resident) {  // stage the agent block: coalesced 16-byte L2 loads (the block was written by another SM)
    const int4* src = (const int4*)&g->ag;
    int4* dst = (int4*)&ag;
    for (int i = lane; i < (int)(AG_BYTES / 16); i += 32) dst[i] = __ldcg(src + i);
  }
  __syncwarp();
  const size_t pol = P.shared_policy ? 0 : (size_t)env;
  double* theta_a = ptr.theta + pol * (size_t)P.memory_size;
  double* theta_b = ptr.theta_b ? ptr.theta_b + pol * (size_t)P.memory_size : nullptr;
  unsigned* occ_w = ptr.occ + pol * (size_t)P.occ_words;
  // once a quarter of an env's table is nonzero the bitmap test costs more than it saves: gather directly
  const unsigned* occ = nullptr;  // (round 2: the occupancy bitmap is no longer consulted -- every gather goes to theta)
  unsigned long long bases[3];
  if (stage == 2) {
    if (ag.kind == 0) {
      if (lane < RLM_N_STATE_MAX + 3) { ag.prev_vars[lane] = ag.from_vars[lane]; ag.from_vars[lane] = ag.to_vars[lane]; }
      __syncwarp();
      double qa, qb;
      eval_q(s_rnd, theta_a, theta_b, ag.from_vars, P.n_state_vars, false, vbuf, lane, qa, qb, bases, false, idxc, occ);
      if (lane < A) { ag.q_from[lane] = qa; ag.qb_from[lane] = qb; }
      ag.from_base0[lane] = mod_m(bases[0]);
      if (lane == 0) { ag.prev_null = ag.null_from; ag.null_from = 0; ag.n_steps++; ag.ep_step++; ag.need_begin = 1; }
      steps_done++;
    }
  } else if (ag.kind == 1) {
    // end of warm-up: Q(first from-state, .) for the first action selection: the never-populated State in a Learner's
    // first episode, the previous episode's stale State afterwards (serial.cpp:24-25,55,60)
    double qa, qb;
    const bool nullf = ag.null_from != 0;
    eval_q(s_rnd, theta_a, theta_b, ag.from_vars, P.n_state_vars, nullf, vbuf, lane, qa, qb, bases, false, idxc, occ);
    if (lane < A) { ag.q_from[lane] = qa; ag.qb_from[lane] = qb; }
    if (!nullf) ag.from_base0[lane] = mod_m(bases[0]);
    if (lane == 0) { ag.need_begin = 1; ag.kind = 2; }
  } else {
    int* tf = ptr.trace_f + (size_t)env * P.trace_cap;
    float* te = ptr.trace_e + (size_t)env * P.trace_cap;
    if (stage == 1) {
      // shared theta moved since the action was selected: UpdateTraces / UpdateWeights read Q(from, .)
      // under the theta of NOW (agent.cpp:274,285 call getQ at update time), i.e. theta_t
      double qa, qb;
      eval_q(s_rnd, theta_a, theta_b, ag.from_vars, P.n_state_vars, ag.null_from != 0, vbuf, lane, qa, qb, bases, false, idxc, occ);
      if (lane < A) { ag.q_from[lane] = qa; ag.qb_from[lane] = qb; }
      __syncwarp();
    }
    {  // Q(to, .) under the current theta
      double qa, qb;
      eval_q(s_rnd, theta_a, theta_b, ag.to_vars, P.n_state_vars, false, vbuf, lane, qa, qb, bases, false, idxc, occ);
      if (lane < A) { q_pre_a[lane] = qa; q_pre_b[lane] = qb; }
    }
    __syncwarp();
    if (lane == 0)
      td_decision(ag, q_pre_a, q_pre_b, ptr.mt_pol + (size_t)env * 312, ptr.mt_agt ? ptr.mt_agt + (size_t)env * 312 : nullptr, D, dec);
    __syncwarp();
    {
      const float rate = (float)dec[0];
      const double scaled = dec[1];
      double* th = (dec[2] != 0.0) ? theta_b : theta_a;
      if (stage == 1) th = (dec[2] != 0.0) ? ptr.dtheta + P.memory_size : ptr.dtheta;  // accumulate, apply after the all-reduce
      __syncwarp();
      int nz = trace_pass(ag, sset, nullptr, tf, te, th, occ_w, nullptr, ag.cur_action, rate, scaled, lane);
      if (lane == 0) { ag.n_traces = nz; ag.sum_traces += nz; }
      sum_z += (lane == 0) ? (unsigned long long)nz : 0ull;
    }
    __syncwarp();
    __threadfence();  // theta updates (L2 atomics) are ordered before the re-evaluation below
    if (env < P.record_envs) {  // parity record: the env part is read back from HBM (published by the env thread)
      unsigned long long h = trace_hash(tf, te, theta_a, ag.n_traces, lane);
      if (lane == 0) {
        int c = ptr.record_count[env];
        if (c < P.record_cap) {
          if (resident) fill_record(&ptr.records[(size_t)env * P.record_cap + c], *resident, ag, h, ag.to_vars);
          else {
            EnvHdr tmp;
            const int4* src = (const int4*)g;
            int4* dst = (int4*)&tmp;
            for (int i = 0; i < (int)(sizeof(EnvHdr) / 16); ++i) dst[i] = __ldcg(src + i);
            fill_record(&ptr.records[(size_t)env * P.record_cap + c], tmp, ag, h, ag.to_vars);
          }
        }
        ptr.record_count[env] = c + 1;
      }
    }
    const bool r_learning = P.algorithm >= RLM_ALGO_R_LEARN;
    if (r_learning) {  // maxQ(from_state) under the updated theta, then rho (td_rho)
      double d3 = 0.0, d4 = 0.0;
      if (lane == 0) { d3 = dec[3]; d4 = dec[4]; }  // dec aliases vbuf, which the evaluation below reuses
      __syncwarp();
      unsigned long long bases_f[3];
      double qa, qb;
      eval_q(s_rnd, theta_a, theta_b, ag.from_vars, P.n_state_vars, ag.null_from != 0, vbuf, lane, qa, qb, bases_f, false, idxc, occ);
      if (lane < A) { q_pre_a[lane] = qa; q_pre_b[lane] = qb; }
      __syncwarp();
      if (lane == 0) { double dd[5] = {0.0, 0.0, 0.0, d3, d4}; td_rho(ag, q_pre_a, q_pre_b, D, dd); }
      __syncwarp();
    }
    if (stage == 0) {
      // the to-state becomes the from-state; Q(from, .) under the UPDATED theta (serial.cpp:55,60)
      if (lane < RLM_N_STATE_MAX + 3) { ag.prev_vars[lane] = ag.from_vars[lane]; ag.from_vars[lane] = ag.to_vars[lane]; }
      ag.from_base0[lane] = mod_m(bases[0]);
      if (lane == 0) { ag.prev_null = ag.null_from; ag.null_from = 0; ag.n_steps++; ag.ep_step++; ag.need_begin = 1; }
      __syncwarp();
      {
        double qa, qb;
        // (the R-learning agents' extra evaluation overwrote the cached indices of the to-state)
        eval_q(s_rnd, theta_a, theta_b, ag.from_vars, P.n_state_vars, false, vbuf, lane, qa, qb, bases, !r_learning, idxc, occ);
        if (lane < A) { ag.q_from[lane] = qa; ag.qb_from[lane] = qb; }
      }
      steps_done++;
    }
  }
  __syncwarp();
  if (!resident) {  // write the agent block back
    int4* dst = (int4*)&g->ag;
    const int4* src = (const int4*)&ag;
    for (int i = lane; i < (int)(AG_BYTES / 16); i += 32) __stcg(dst + i, src[i]);
  }
  __syncwarp();
}

// ---------------------------------------------------------------------------------------------
// Learner step with THREE warps per ready env (one CTA of 96 threads per env; default): warp g hashes
// feature group g and issues its 9 (18) theta gathers at once, so the three groups' DRAM round trips
// overlap and the hashing chain is a third as long; warp 0 then does the exact-order sums, the TD
// decision and the trace pass; the second evaluation re-gathers with the indices still in registers.
#define A3_WARPS 3
#define A3_Q 0                                             // q_pre_a, q_pre_b: 18 doubles
#define A3_SS (A3_Q + 8 * 2 * RLM_MAX_ACTIONS)             // small set
#define A3_DEC (A3_SS + 4 * SS_SLOTS)                      // 6 doubles
#define A3_V (A3_DEC + 48)                                 // V[table][g][a][VROW]
__host__ __device__ inline size_t a3_occ_offset(int is_double) {  // bytes from `sb` to the staged bitmap
  return ((size_t)A3_V + (size_t)(is_double ? 2 : 1) * 4 * RLM_MAX_ACTIONS * VROW * 8 + 15) & ~(size_t)15;
}
__host__ __device__ inline size_t a3_tt_offset(int is_double, int occ_smem_words) {  // bytes from `sb` to the tile table
  return a3_occ_offset(is_double) + (((size_t)occ_smem_words * 4 + 15) & ~(size_t)15);
}
size_t rlm_agent3_smem_bytes(int is_double, int occ_smem_words) {
  return AG_BYTES + a3_tt_offset(is_double, occ_smem_words) + (size_t)2 * TT_SLOTS * 4;
}

// indices of lane j's tiles of group g for every action (registers), and the partial hash sum
__device__ __forceinline__ unsigned long long a3_hash(const unsigned* rnd, const float* vars, int n, bool null_state, int g, int lane,
                                                      int* f) {
  const int A = P.n_actions;
  const float* gv = (g == 1) ? vars + 3 : vars;
  const int nf = (g == 0) ? 3 : ((g == 1) ? n - 3 : n);
  unsigned long long base = 0ull;
  if (!null_state) base = tile_base_sum(rnd, gv, nf, lane);
#pragma unroll
  for (int a = 0; a < RLM_MAX_ACTIONS; ++a) f[a] = (a < A && !null_state) ? tile_index(rnd, base, nf, g * A + a) : 0;
  return base;
}
// V[table][seg][a][VROW] holds the PRODUCTS w*theta[f] of agent.cpp:117-135's four loops -- seg 0 = (group 0, w0),
// 1 = (group 1, w1), 2 = (group 1, w2: the third loop starts at T, Appendix A8), 3 = (group 2, w2) -- so that the
// multiplications are done by the gathering lanes, in parallel, and only the additions remain on the serial chain.
#define A3_SEGS 4
// occ: bitmap to test (nullptr = dense table: gather everything); occ_sm: it is the shared-memory copy
__device__ __forceinline__ void a3_gather(const double* th_a, const double* th_b, const unsigned* occ, bool occ_sm, const int* f, int g, int lane,
                                          double* V) {
  const int A = P.n_actions;
  double va[RLM_MAX_ACTIONS], vb[RLM_MAX_ACTIONS];
  bool nz[RLM_MAX_ACTIONS];
  if (occ_sm) {
#pragma unroll
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) nz[a] = (a < A) && occ_test_s(occ, f[a]);
  } else {
#pragma unroll
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) nz[a] = (a < A) && (occ == nullptr || occ_test(occ, f[a]));
  }
#pragma unroll
  for (int a = 0; a < RLM_MAX_ACTIONS; ++a) va[a] = nz[a] ? __ldcg(th_a + f[a]) : 0.0;
  if (th_b) {
#pragma unroll
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) vb[a] = nz[a] ? __ldcg(th_b + f[a]) : 0.0;
  }
  const int seg0 = (g == 0) ? 0 : ((g == 1) ? 1 : 3);
  const double w = P.gw[g];
  double* Va = V + (size_t)seg0 * RLM_MAX_ACTIONS * VROW;
  double* Vb = V + (size_t)(A3_SEGS + seg0) * RLM_MAX_ACTIONS * VROW;
#pragma unroll
  for (int a = 0; a < RLM_MAX_ACTIONS; ++a) {
    if (a < A) {
      Va[a * VROW + lane] = w * va[a];
      if (th_b) Vb[a * VROW + lane] = w * vb[a];
    }
  }
  if (g == 1) {  // group 1 is summed a second time with w2
    const double w2 = P.gw[2];
#pragma unroll
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) {
      if (a < A) {
        Va[(RLM_MAX_ACTIONS + a) * VROW + lane] = w2 * va[a];
        if (th_b) Vb[(RLM_MAX_ACTIONS + a) * VROW + lane] = w2 * vb[a];
      }
    }
  }
}
// Second evaluation of a step (same state, theta after this env's own update): only the tiles the update touched
// -- flagged by the trace pass in `bloom` -- are read again; every other product row entry of V is still exact.
__device__ __forceinline__ void a3_regather_patch(const double* th_a, const double* th_b, const unsigned* occ, bool occ_sm, const unsigned* bloom,
                                                  const int* f, int g, int lane, double* V) {
  const int A = P.n_actions;
  const int seg0 = (g == 0) ? 0 : ((g == 1) ? 1 : 3);
  const double w = P.gw[g], w2 = P.gw[2];
  double* Va = V + (size_t)seg0 * RLM_MAX_ACTIONS * VROW;
  double* Vb = V + (size_t)(A3_SEGS + seg0) * RLM_MAX_ACTIONS * VROW;
#pragma unroll
  for (int a = 0; a < RLM_MAX_ACTIONS; ++a) {
    if (a < A && bloom_test(bloom, f[a])) {
      const bool nz = (occ == nullptr) || (occ_sm ? occ_test_s(occ, f[a]) : occ_test(occ, f[a]));
      const double va = nz ? __ldcg(th_a + f[a]) : 0.0;
      Va[a * VROW + lane] = w * va;
      if (g == 1) Va[(RLM_MAX_ACTIONS + a) * VROW + lane] = w2 * va;
      if (th_b) {
        const double vb = nz ? __ldcg(th_b + f[a]) : 0.0;
        Vb[a * VROW + lane] = w * vb;
        if (g == 1) Vb[(RLM_MAX_ACTIONS + a) * VROW + lane] = w2 * vb;
      }
    }
  }
}
// Exact-order sum of agent.cpp:117-135 for one action: the 4 x 32 products of V's rows, strictly left to right.
// Software-pipelined by hand -- block k+1 is loaded before block k is added, in a loop that is NOT unrolled: left to
// itself ptxas pairs every shared-memory load with its addition (~37 cycles per element instead of ~10).
__device__ __forceinline__ double a3_chain(const double* row0) {
  double acc = 0.0, cur[8], nxt[8];
#pragma unroll
  for (int j = 0; j < 8; ++j) cur[j] = row0[j];
#pragma unroll 1
  for (int blk = 1; blk <= 4 * A3_SEGS; ++blk) {
    const int nb = (blk < 4 * A3_SEGS) ? blk : 0;  // (the last iteration reloads block 0; its values are not used)
    const double* r = row0 + (size_t)(nb >> 2) * RLM_MAX_ACTIONS * VROW + (nb & 3) * 8;
#pragma unroll
    for (int j = 0; j < 8; ++j) nxt[j] = r[j];
#pragma unroll
    for (int j = 0; j < 8; ++j) acc += cur[j];
#pragma unroll
    for (int j = 0; j < 8; ++j) cur[j] = nxt[j];
  }
  return acc;
}
// exact-order sums over the four product rows; lanes < A of warp 0
__device__ __noinline__ void a3_sums(const double* V, bool has_b, int lane, double& qa_out, double& qb_out) {
  qa_out = a3_chain(V + (size_t)lane * VROW);
  qb_out = has_b ? a3_chain(V + ((size_t)A3_SEGS * RLM_MAX_ACTIONS + lane) * VROW) : 0.0;
}

// R-learning agents (whole CTA): maxQ(from_state) under the UPDATED theta, then the rho update (td_rho).
// Kept out of line so that its index registers do not weigh on the Q-learning / SARSA path.
__device__ __noinline__ void a3_rho_step(AgentD& ag, const double* theta_a, const double* theta_b, const unsigned* occ, bool occ_sm, double* V,
                                         double* q_post_a, double* q_post_b, const double* dec, const DynParams& D, int warp, int lane) {
  const int A = P.n_actions;
  __syncthreads();  // trace pass done, V free
  int f2[RLM_MAX_ACTIONS];
  a3_hash(rlm_rndseq_table, ag.from_vars, P.n_state_vars, ag.null_from != 0, warp, lane, f2);
  a3_gather(theta_a, theta_b, occ, occ_sm, f2, warp, lane, V);
  __syncthreads();
  if (warp == 0) {
    if (lane < A) { double qa, qb; a3_sums(V, theta_b != nullptr, lane, qa, qb); q_post_a[lane] = qa; q_post_b[lane] = qb; }
    __syncwarp();
    if (lane == 0) td_rho(ag, q_post_a, q_post_b, D, dec);
  }
  __syncthreads();  // every warp has read from_vars
}

// EXTRAS = false: the Q-learning / SARSA / Double-Q training kernel; EXTRAS = true adds the R-learning agents' third
// evaluation (separate instantiation so that it costs the training path no registers).
template <bool EXTRAS>
__global__ void __launch_bounds__(A3_WARPS * 32, 10) rlm_agent3_kernel(DevPtrs ptr, DynParams D, int tslot, int stage) {
  PDL_PROLOGUE();
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  AgentD& ag = *(AgentD*)smem;
  unsigned char* sb = smem + AG_BYTES;
  double* q_pre_a = (double*)(sb + A3_Q);
  double* q_pre_b = q_pre_a + RLM_MAX_ACTIONS;
  int* sset = (int*)(sb + A3_SS);
  double* dec = (double*)(sb + A3_DEC);
  double* V = (double*)(sb + A3_V);
  unsigned* occ_s = (unsigned*)(sb + a3_occ_offset(P.is_double));
  const unsigned* rnd = rlm_rndseq_table;
  const int A = P.n_actions;
  const int n_ready = ptr.ready_count[tslot];
  unsigned long long steps_done = 0, sum_z = 0;
#pragma unroll 1
  for (int idx = blockIdx.x; idx < n_ready; idx += gridDim.x) {
    PH(0);
    const int env = ptr.ready[idx];
    EnvHdr* g = (EnvHdr*)(ptr.env + (size_t)env * P.env_stride);
    __syncthreads();  // previous env's shared state is dead
    const size_t pol = P.shared_policy ? 0 : (size_t)env;
    unsigned* occ_w = ptr.occ + pol * (size_t)P.occ_words;
    {
      const int4* src = (const int4*)&g->ag;
      int4* dst = (int4*)&ag;
      for (int i = tid; i < (int)(AG_BYTES / 16); i += A3_WARPS * 32) dst[i] = __ldcg(src + i);
      // the env's whole occupancy bitmap (<= 16 KB, L2-resident) rides along: one coalesced copy per step instead of
      // 1728 scattered 4-byte loads on the step's critical path
      // LDGSTS (cp.async, L2-coherent .cg): no registers, and the copy is only waited for right before the first gather
      const int n4 = P.occ_smem_words >> 2;
      const int4* osrc = (const int4*)occ_w;
      const unsigned odst = (unsigned)__cvta_generic_to_shared(occ_s);
      for (int i = tid; i < n4; i += A3_WARPS * 32)
        asm volatile("cp.async.cg.shared.global [%0], [%1], 16;" ::"r"(odst + 16u * (unsigned)i), "l"(osrc + i) : "memory");
      asm volatile("cp.async.commit_group;" ::: "memory");
    }
    __syncthreads();
    PH(1);
    double* theta_a = ptr.theta + pol * (size_t)P.memory_size;
    double* theta_b = ptr.theta_b ? ptr.theta_b + pol * (size_t)P.memory_size : nullptr;
    // every path below hashes first and gathers second: A3_OCC_READY() sits between the two
#define A3_OCC_READY() do { if (P.occ_smem_words) { asm volatile("cp.async.wait_all;" ::: "memory"); __syncthreads(); } } while (0)
    // the bitmap test pays for itself as long as it filters enough gathers: against HBM-resident bitmaps up to a
    // quarter full, against the shared-memory copy (a test is one LDS) up to 15/16 full
    const bool dense = true;  // round 2: the occupancy bitmap is no longer consulted (dense tables are the regime that counts)
    const bool occ_sm = !dense && P.occ_smem_words > 0;
    const unsigned* occ = dense ? nullptr : (occ_sm ? occ_s : occ_w);
    const int kind = ag.kind;
    int f[RLM_MAX_ACTIONS];
    unsigned long long base = 0ull;
    if (stage == 2) {
      if (kind == 0) {  // shared policy, after theta += dtheta: Q(from = to-state, .) under theta_{t+1}
        base = a3_hash(rnd, ag.to_vars, P.n_state_vars, false, warp, lane, f);
        A3_OCC_READY();
        a3_gather(theta_a, theta_b, occ, occ_sm, f, warp, lane, V);
        __syncthreads();
        if (warp == 0) {
          double qa, qb;
          if (lane < A) { a3_sums(V, theta_b != nullptr, lane, qa, qb); ag.q_from[lane] = qa; ag.qb_from[lane] = qb; }
          if (lane < RLM_N_STATE_MAX + 3) { ag.prev_vars[lane] = ag.from_vars[lane]; ag.from_vars[lane] = ag.to_vars[lane]; }
          ag.from_base0[lane] = mod_m(base);
          if (lane == 0) { ag.prev_null = ag.null_from; ag.null_from = 0; ag.n_steps++; ag.ep_step++; ag.need_begin = 1; }
          steps_done++;
        }
      }
    } else if (kind == 1) {  // end of warm-up: Q(null state, .)
      const bool nullf = ag.null_from != 0;  // a Learner's first episode; afterwards the previous episode's stale State
      base = a3_hash(rnd, ag.from_vars, P.n_state_vars, nullf, warp, lane, f);
      A3_OCC_READY();
      a3_gather(theta_a, theta_b, occ, occ_sm, f, warp, lane, V);
      __syncthreads();
      if (warp == 0) {
        double qa, qb;
        if (lane < A) { a3_sums(V, theta_b != nullptr, lane, qa, qb); ag.q_from[lane] = qa; ag.qb_from[lane] = qb; }
        if (!nullf) ag.from_base0[lane] = mod_m(base);
        if (lane == 0) { ag.need_begin = 1; ag.kind = 2; }
      }
    } else if (kind == 0) {
      if (stage == 1) {  // shared policy: Q(from, .) under theta_t (agent.cpp:274,285 read theta at update time)
        a3_hash(rnd, ag.from_vars, P.n_state_vars, ag.null_from != 0, warp, lane, f);
        A3_OCC_READY();
        a3_gather(theta_a, theta_b, occ, occ_sm, f, warp, lane, V);
        __syncthreads();
        if (warp == 0 && lane < A) { double qa, qb; a3_sums(V, theta_b != nullptr, lane, qa, qb); ag.q_from[lane] = qa; ag.qb_from[lane] = qb; }
        __syncthreads();
      }
      base = a3_hash(rnd, ag.to_vars, P.n_state_vars, false, warp, lane, f);  // Q(to, .) under the current theta
      if (stage != 1) A3_OCC_READY();
      PH(2);
      a3_gather(theta_a, theta_b, occ, occ_sm, f, warp, lane, V);
      PH(3);
      __syncthreads();
      PH(4);
      if (warp == 0 && lane < A) { double qa, qb; a3_sums(V, theta_b != nullptr, lane, qa, qb); q_pre_a[lane] = qa; q_pre_b[lane] = qb; }
      int* tt = (int*)(sb + a3_tt_offset(P.is_double, P.occ_smem_words));
      __syncthreads();
      PH(5);
      if (warp != 0) {
        // the two idle warps list every tile of the from-state with its last writer while warp 0 computes the TD error
        tt_build(tt, ag, tid - 32, (A3_WARPS - 1) * 32);
        asm volatile("bar.sync 1, %0;" ::"n"((A3_WARPS - 1) * 32) : "memory");  // slots initialised before any insert
        if (!ag.null_from) tt_fill(tt, ag, tid - 32, (A3_WARPS - 1) * 32);
      } else if (lane == 0) {
        td_decision(ag, q_pre_a, q_pre_b, ptr.mt_pol + (size_t)env * 312, ptr.mt_agt ? ptr.mt_agt + (size_t)env * 312 : nullptr, D, dec);
      }
      __syncthreads();
      if (warp == 0) {
        int* tf = ptr.trace_f + (size_t)env * P.trace_cap;
        float* te = ptr.trace_e + (size_t)env * P.trace_cap;
        PH(6);
        const float rate = (float)dec[0];
        const double scaled = dec[1];
        double* th = (dec[2] != 0.0) ? theta_b : theta_a;
        if (stage == 1) th = (dec[2] != 0.0) ? ptr.dtheta + P.memory_size : ptr.dtheta;
#ifdef RLM_TIMING
        if (tid == 0 && idx < 4096) { g_phase_clk[idx * 16 + 13] = ag.n_traces; g_phase_clk[idx * 16 + 14] = (rate != 0.0f); }
#endif
        int nz = trace_pass(ag, sset, tt, tf, te, th, occ_w, occ_sm ? occ_s : nullptr, ag.cur_action, rate, scaled, lane);
        if (lane == 0) { ag.n_traces = nz; ag.sum_traces += nz; }
        sum_z += (lane == 0) ? (unsigned long long)nz : 0ull;
        __syncwarp();
        PH(7);
        __threadfence();
        PH(8);
        if (env < P.record_envs) emit_record(ptr, g, env, ag, theta_a, ag.to_vars, lane);
        if (!EXTRAS && stage == 0) {
          if (lane < RLM_N_STATE_MAX + 3) { ag.prev_vars[lane] = ag.from_vars[lane]; ag.from_vars[lane] = ag.to_vars[lane]; }
          ag.from_base0[lane] = mod_m(base);
          if (lane == 0) { ag.prev_null = ag.null_from; ag.null_from = 0; ag.n_steps++; ag.ep_step++; ag.need_begin = 1; }
          steps_done++;
        }
      }
      if (EXTRAS) {
        if (P.algorithm >= RLM_ALGO_R_LEARN) a3_rho_step(ag, theta_a, theta_b, occ, occ_sm, V, q_pre_a, q_pre_b, dec, D, warp, lane);
        if (warp == 0 && stage == 0) {  // (after the other warps have read from_vars in a3_rho_step)
          if (lane < RLM_N_STATE_MAX + 3) { ag.prev_vars[lane] = ag.from_vars[lane]; ag.from_vars[lane] = ag.to_vars[lane]; }
          ag.from_base0[lane] = mod_m(base);
          if (lane == 0) { ag.prev_null = ag.null_from; ag.null_from = 0; ag.n_steps++; ag.ep_step++; ag.need_begin = 1; }
          steps_done++;
        }
      }
      if (stage == 0) {  // Q(from = to-state, .) under the UPDATED theta (serial.cpp:55,60); indices are still in registers
        __syncthreads();
        PH(9);
        // (the R-learning agents' extra evaluation has overwritten the product rows: gather everything again)
        if (EXTRAS && P.algorithm >= RLM_ALGO_R_LEARN) a3_gather(theta_a, theta_b, occ, occ_sm, f, warp, lane, V);
        else a3_regather_patch(theta_a, theta_b, occ, occ_sm, (const unsigned*)sset, f, warp, lane, V);
        __syncthreads();
        PH(10);
        if (warp == 0 && lane < A) { double qa, qb; a3_sums(V, theta_b != nullptr, lane, qa, qb); ag.q_from[lane] = qa; ag.qb_from[lane] = qb; }
      }
    }
    asm volatile("cp.async.wait_all;" ::: "memory");  // (paths that gathered nothing)
    __syncthreads();
    PH(11);
    {
      int4* dst = (int4*)&g->ag;
      const int4* src = (const int4*)&ag;
      for (int i = tid; i < (int)(AG_BYTES / 16); i += A3_WARPS * 32) __stcg(dst + i, src[i]);
    }
    PH(12);
  }
  if (tid == 0 && (steps_done | sum_z)) {
    atomicAdd(&ptr.counters[1], steps_done);
    atomicAdd(&ptr.counters[2], sum_z);
  }
}

cudaError_t rlm_launch_agent3(const DevPtrs& ptr, const DynParams& D, int n_envs, int is_double, int occ_smem_words, int tslot, int n_sms,
                              int stage, int full, cudaStream_t st) {
  const size_t smem = rlm_agent3_smem_bytes(is_double, occ_smem_words);
  static size_t attr_smem[2] = {0, 0};
  if (smem > attr_smem[full ? 1 : 0]) {
    cudaError_t e = full ? cudaFuncSetAttribute(rlm_agent3_kernel<true>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem)
                         : cudaFuncSetAttribute(rlm_agent3_kernel<false>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr_smem[full ? 1 : 0] = smem;
  }
  int grid = n_envs;            // worst case: every env is ready
  const int cap = n_sms * 16;   // then the grid-stride loop takes over
  if (grid > cap) grid = cap;
  if (full) return launch_pdl(rlm_agent3_kernel<true>, grid, A3_WARPS * 32, smem, st, ptr, D, tslot, stage);
  return launch_pdl(rlm_agent3_kernel<false>, grid, A3_WARPS * 32, smem, st, ptr, D, tslot, stage);
}

// Tick-synchronous engine: one launch per tick after rlm_env_kernel.
template <int WARPS>
__global__ void __launch_bounds__(WARPS * 32) rlm_agent_kernel(DevPtrs ptr, DynParams D, int tslot, int stage) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  unsigned char* wbase = smem + (size_t)warp * (AG_BYTES + P.scratch_bytes);
  AgentD& ag = *(AgentD*)wbase;
  unsigned char* scratch = wbase + AG_BYTES;
  const int n_ready = ptr.ready_count[tslot];
  unsigned long long steps_done = 0, sum_z = 0;
#pragma unroll 1
  for (int idx = blockIdx.x * WARPS + warp; idx < n_ready; idx += gridDim.x * WARPS)
    agent_process_env(ptr, D, ptr.ready[idx], ag, std_scratch(scratch), lane, steps_done, sum_z, stage, nullptr);
  if (lane == 0 && (steps_done | sum_z)) {
    atomicAdd(&ptr.counters[1], steps_done);
    atomicAdd(&ptr.counters[2], sum_z);
  }
}

// theta += dtheta; dtheta = 0  (after the all-reduce of dtheta in shared-policy mode)
__global__ void rlm_apply_dtheta_kernel(double* theta, double* dtheta, long long n) {
  const long long stride = (long long)gridDim.x * blockDim.x * 2;
  for (long long i = ((long long)blockIdx.x * blockDim.x + threadIdx.x) * 2; i < n; i += stride) {
    double2 t = *(double2*)(theta + i), d = *(double2*)(dtheta + i);
    t.x += d.x; t.y += d.y;
    *(double2*)(theta + i) = t;
    *(double2*)(dtheta + i) = make_double2(0.0, 0.0);
  }
}
cudaError_t rlm_launch_apply_dtheta(double* theta, double* dtheta, long long n, int n_sms, cudaStream_t st) {
  if (n & 1) return cudaErrorInvalidValue;
  long long blocks = (n / 2 + 255) / 256;
  if (blocks > (long long)n_sms * 8) blocks = (long long)n_sms * 8;
  rlm_apply_dtheta_kernel<<<(int)blocks, 256, 0, st>>>(theta, dtheta, n);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Fused engine (RLM_ENGINE=f; not the default -- measured slower than two launches per tick, DESIGN.md 3.3):
// ONE launch, one warp per env for all `n_ticks` ticks.
// The env record stays in shared memory for the whole launch; the warp runs the tick (lane 0 scalar +
// lane-parallel windows / state variables) and, whenever its env's midprice has moved, the learner step
// inline -- so envs never wait for each other and the theta gathers of some warps overlap the book
// logic of others.  14 warps per CTA, 2 CTAs per SM: 3 696 resident envs on the 132 SMs of an H100.
#define FUSED_WARPS 14
#define FU_MSG 0
#define FU_PUSH (FU_MSG + 128)
#define FU_FLAG (FU_PUSH + 8 * 2 * RLM_NWIN)
#define FU_Q (FU_FLAG + 16)
#define FU_SS (FU_Q + 8 * 2 * RLM_MAX_ACTIONS)
#define FU_VBUF (FU_SS + 4 * SS_SLOTS)
size_t rlm_fused_smem_bytes(int is_double) {
  size_t per_warp = ((sizeof(EnvHdr) + 15) & ~(size_t)15) + (((size_t)FU_VBUF + (size_t)(is_double ? 2 : 1) * RLM_MAX_ACTIONS * VROW * 8 + 15) & ~(size_t)15);
  return FUSED_WARPS * per_warp;
}

__global__ void __launch_bounds__(FUSED_WARPS * 32, 2) rlm_fused_kernel(DevPtrs ptr, DynParams D) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  const int env = blockIdx.x * FUSED_WARPS + warp;
  if (env >= P.n_envs) return;
  const int hdr_bytes = (int)((sizeof(EnvHdr) + 15) & ~(size_t)15);
  const size_t per_warp = hdr_bytes + (((size_t)FU_VBUF + (size_t)(P.is_double ? 2 : 1) * RLM_MAX_ACTIONS * VROW * 8 + 15) & ~(size_t)15);
  unsigned char* wbase = smem + (size_t)warp * per_warp;
  EnvHdr& e = *(EnvHdr*)wbase;
  unsigned char* sb = wbase + hdr_bytes;
  rlm_tick_msg& msg = *(rlm_tick_msg*)(sb + FU_MSG);
  double* pushv = (double*)(sb + FU_PUSH);
  double* oldv = pushv + RLM_NWIN;
  int* flag = (int*)(sb + FU_FLAG);
  AgentScratch sc;
  sc.q_pre = (double*)(sb + FU_Q); sc.sset = (int*)(sb + FU_SS); sc.idx = nullptr; sc.vbuf = (double*)(sb + FU_VBUF);
  EnvHdr* g = (EnvHdr*)(ptr.env + (size_t)env * P.env_stride);
  double* ring = (double*)((unsigned char*)g + sizeof(EnvHdr));
  if (g->phase == PH_DONE) return;
  {
    const int4* src = (const int4*)g;
    int4* dst = (int4*)&e;
    for (int i = lane; i < hdr_bytes / 16; i += 32) dst[i] = src[i];
  }
  __syncwarp();
  unsigned long long ticked = 0, steps_done = 0, sum_z = 0;
  unsigned long long* mt_pol = ptr.mt_pol + (size_t)env * 312;
#pragma unroll 1
  for (int t = 0; t < D.n_ticks; ++t) {
    const int phase = e.phase;
    if (phase == PH_DONE) break;
    if (P.source == RLM_SOURCE_GENERATOR) {
      if (lane == 0) flow_next_dev(&e.flow, &msg);
    } else {
      const int pos = D.stream_off + t;
      if (pos >= D.stream_ticks) { if (lane == 0) e.err |= ERR_STREAM_UNDERRUN; break; }
      ((unsigned*)&msg)[lane] = __ldg((const unsigned*)(ptr.stream + ((size_t)pos * P.n_envs + env)) + lane);
    }
    if (lane < RLM_NWIN) oldv[lane] = window_peek(e, ring, lane);
    __syncwarp();
    const bool multi = needs_multi(e, msg);
    if (phase == PH_PREOPEN) {  // intraday.cpp:111-116
      if (lane == 0) {
        if (multi) {
          if (update_book_profiles_multi(e, msg, false) && market_is_open(e)) e.phase = PH_WARMUP;
        } else {
          msg.n_tx = 0;
          update_book_profiles(e, msg);
          if (market_is_open(e)) e.phase = PH_WARMUP;
        }
      }
      __syncwarp();
      continue;
    }
    if (lane == 0) {
      if (phase == PH_RUN) e.pnl_step = 0.0;  // base.cpp:286
      int done = 1;
      if (multi) done = next_state_multi(e, msg, pushv) ? 1 : 0;
      else next_state_scalar(e, msg, pushv);  // Intraday::NextState
      *flag = done;
    }
    __syncwarp();
    if (!*flag) { __syncwarp(); continue; }  // (a multi-message tick that is not complete yet)
    ticked++;
    if (lane < 8) window_push(e, ring, lane, pushv[lane], oldv[lane]);
    __syncwarp();
    if (lane == 0) {
      int r = -1;
      e.tp_val = e.w_mean[W_TP];
      if (phase == PH_WARMUP) {  // intraday.cpp:118-135
        bool full = true;
        for (int w = 0; w < 8; ++w) full = full && (e.w_count[w] == P.win_size[w]);
        if (full) { place_orders(e, 1, 1); e.phase = PH_RUN; e.ag.kind = 1; r = 1; }
      } else {  // tail of one iteration of performAction's do-while (base.cpp:292-305)
        double mpm = m_midprice(e) - m_last_midprice(e);
        e.pnl_step += (double)e.position * mpm;
        e.momentum_pnl_step += (double)e.position * mpm;
        e.agg_r += get_reward(e);
        e.agg_pnl += e.pnl_step;
        e.agg_mpm += mpm;
        if (!(!is_terminal(e) && fabs(e.agg_mpm) < 1e-5)) {
          e.pnl_step = e.agg_pnl;  // base.cpp:317-331
          pushv[W_PNLUP] = fmax(0.0, e.pnl_step);
          pushv[W_PNLDN] = fabs(fmin(0.0, e.pnl_step));
          e.ep_reward += e.agg_r;
          e.ep_bandh += e.agg_mpm;
          r = 0;
        }
      }
      *flag = r;
    }
    __syncwarp();
    const int ready = *flag;
    if (ready < 0) continue;
    if (ready == 0) {
      if (lane == W_PNLUP || lane == W_PNLDN) window_push(e, ring, lane, pushv[lane], oldv[lane]);
      __syncwarp();
      if (lane < P.n_state_vars) e.ag.to_vars[lane] = (float)get_variable(e, ring, P.state_vars[lane]);
      if (lane == 31) { e.ag.last_reward = get_reward(e); e.ag.kind = 0; }
      __syncwarp();
    }
    agent_process_env(ptr, D, env, e.ag, sc, lane, steps_done, sum_z, 0, &e);  // serial.cpp:64-65
    if (lane == 0) { begin_step(e, mt_pol, D); e.ag.need_begin = 0; }          // serial.cpp:55-61
    __syncwarp();
  }
  __syncwarp();
  {
    int4* dst = (int4*)g;
    const int4* src = (const int4*)&e;
    for (int i = lane; i < hdr_bytes / 16; i += 32) dst[i] = src[i];
  }
  if (lane == 0) {
    if (ticked) atomicAdd(&ptr.counters[0], ticked);
    if (steps_done | sum_z) { atomicAdd(&ptr.counters[1], steps_done); atomicAdd(&ptr.counters[2], sum_z); }
    const unsigned errs = (unsigned)(e.err | e.ag.err);
    if (errs) atomicOr(&ptr.counters[4], (unsigned long long)errs);
  }
}

cudaError_t rlm_launch_fused(const DevPtrs& ptr, const DynParams& D, int n_envs, int is_double, cudaStream_t st) {
  const size_t smem = rlm_fused_smem_bytes(is_double);
  static size_t attr_smem = 0;
  if (smem > attr_smem) {
    cudaError_t e = cudaFuncSetAttribute(rlm_fused_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr_smem = smem;
  }
  rlm_fused_kernel<<<(n_envs + FUSED_WARPS - 1) / FUSED_WARPS, FUSED_WARPS * 32, smem, st>>>(ptr, D);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Persistent engine: ONE launch runs `n_ticks` ticks of every env with no global barrier.
//   CTAs [0, n_agent_ctas)   agent role: warps pop env ids from a queue in HBM and run the learner step;
//   CTAs [n_agent_ctas, ...)  env role: one thread per env; an env whose step ended publishes its agent
//                             block, pushes its id and waits for the done flag while the other lanes of
//                             its warp keep ticking.  Envs advance at their own pace (their results do
//                             not depend on the schedule: all state is per env).
// Agent CTAs come first in the grid, so they are resident before any env CTA can wait on them.
#define RUN_WARPS RLM_RUN_WARPS
#define RUN_THREADS (RUN_WARPS * 32)

__device__ __forceinline__ void copy_ag_from_global(AgentD& dst, const AgentD* src) {
  const int4* s = (const int4*)src;
  int4* d = (int4*)&dst;
#pragma unroll 4
  for (int i = 0; i < (int)(sizeof(AgentD) / 16); ++i) d[i] = __ldcg(s + i);
}

__global__ void __launch_bounds__(RUN_THREADS, 4) rlm_run_kernel(DevPtrs ptr, DynParams D, int n_agent_ctas, int n_env_warps) {
  extern __shared__ __align__(16) unsigned char smem[];
  const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
  if ((int)blockIdx.x < n_agent_ctas) {
    // ------------------------------------------------------------------ agent role
    unsigned char* wbase = smem + (size_t)warp * (AG_BYTES + P.scratch_bytes);
    AgentD& ag = *(AgentD*)wbase;
    unsigned char* scratch = wbase + AG_BYTES;
    unsigned long long steps_done = 0, sum_z = 0;
    const unsigned qmask = (unsigned)ptr.q_size - 1u;
    while (true) {
      int env = -1;
      if (lane == 0) {
        const unsigned ticket = atomicAdd(ptr.q_head, 1u);
        volatile int* slot = ptr.q_slots + (ticket & qmask);
        while (true) {
          int v = *slot;
          if (v >= 0) { env = v; *slot = -1; break; }
          if (*(volatile int*)ptr.q_done) {
            const unsigned tail = *(volatile unsigned*)ptr.q_tail;
            if ((int)(ticket - tail) >= 0) { env = -2; break; }  // every push is already consumed or owned
          }
          __nanosleep(200);
        }
      }
      env = __shfl_sync(FULL, env, 0);
      if (env < 0) break;
      __threadfence();  // acquire: the env record published before the push
      agent_process_env(ptr, D, env, ag, std_scratch(scratch), lane, steps_done, sum_z, 0, nullptr);
      __threadfence();  // release: agent block, theta, traces
      if (lane == 0) *(volatile int*)(ptr.ag_done + env) = 1;
    }
    if (lane == 0 && (steps_done | sum_z)) {
      atomicAdd(&ptr.counters[1], steps_done);
      atomicAdd(&ptr.counters[2], sum_z);
    }
    return;
  }
  // -------------------------------------------------------------------- env role
  const int b = ((int)blockIdx.x - n_agent_ctas) * RUN_THREADS + tid;
  const bool valid = b < P.n_envs;
  EnvHdr* g = (EnvHdr*)(ptr.env + (size_t)(valid ? b : 0) * P.env_stride);
  double* ring = (double*)((unsigned char*)g + sizeof(EnvHdr));
  EnvHdr e;
  int ticks_left = 0, tick_idx = 0;
  bool waiting = false;
  unsigned ticked = 0;
  if (valid) {
    e = *g;  // thread-local copy (lane-interleaved local memory), kept for the whole launch
    if (e.phase != PH_DONE) ticks_left = D.n_ticks;
  }
  const unsigned qmask = (unsigned)ptr.q_size - 1u;
  while (true) {
    if (waiting && *(volatile int*)(ptr.ag_done + b)) {
      __threadfence();
      *(volatile int*)(ptr.ag_done + b) = 0;
      copy_ag_from_global(e.ag, &g->ag);
      waiting = false;
      begin_step(e, ptr.mt_pol + (size_t)b * 312, D);
      e.ag.need_begin = 0;
      if (e.phase == PH_DONE) ticks_left = 0;
    }
    bool push = false;
    if (!waiting && ticks_left > 0) {
      rlm_tick_msg msg;
      bool have = true;
      if (P.source == RLM_SOURCE_GENERATOR) {
        flow_next_dev(&e.flow, &msg);
      } else {
        const int pos = D.stream_off + tick_idx;
        if (pos >= D.stream_ticks) { e.err |= ERR_STREAM_UNDERRUN; have = false; ticks_left = 0; }
        else {
          const int4* src = (const int4*)(ptr.stream + ((size_t)pos * P.n_envs + b));
          int4* dst = (int4*)&msg;
#pragma unroll
          for (int i = 0; i < 8; ++i) dst[i] = __ldg(src + i);
        }
      }
      if (have) {
        const int was = e.phase;
        const int r = env_tick(e, ring, msg, 0);
        ticks_left--; tick_idx++;
        if (was != PH_PREOPEN && r != -2) ticked++;
        if (r >= 0) {
          // publish what the agent warp needs (the whole record for envs with a parity dump)
          if (b < P.record_envs) *g = e; else g->ag = e.ag;
          __threadfence();
          push = true;
          waiting = true;
        }
      }
    }
    const unsigned pm = __ballot_sync(FULL, push);
    if (pm) {
      const int leader = __ffs(pm) - 1;
      unsigned base = 0;
      if (lane == leader) base = atomicAdd(ptr.q_tail, (unsigned)__popc(pm));
      base = __shfl_sync(FULL, base, leader);
      if (push) *(volatile int*)(ptr.q_slots + ((base + __popc(pm & ((1u << lane) - 1u))) & qmask)) = b;
    }
    if (!__any_sync(FULL, waiting || ticks_left > 0)) break;
  }
  unsigned errs = 0;
  if (valid) { errs = (unsigned)(e.err | e.ag.err); *g = e; }
  for (int o = 16; o > 0; o >>= 1) { ticked += __shfl_xor_sync(FULL, ticked, o); errs |= __shfl_xor_sync(FULL, errs, o); }
  if (lane == 0) {
    if (ticked) atomicAdd(&ptr.counters[0], (unsigned long long)ticked);
    if (errs) atomicOr(&ptr.counters[4], (unsigned long long)errs);
    __threadfence();
    if (atomicAdd(ptr.env_warps_done, 1u) + 1u == (unsigned)n_env_warps) {
      __threadfence();
      *(volatile int*)ptr.q_done = 1;
    }
  }
}

cudaError_t rlm_launch_run(const DevPtrs& ptr, const DynParams& D, int n_envs, int scratch_bytes, int n_agent_ctas, cudaStream_t st) {
  size_t smem = rlm_agent_smem_bytes(RUN_WARPS, scratch_bytes);
  static size_t attr_smem = 0;
  if (smem > attr_smem) {
    cudaError_t e = cudaFuncSetAttribute(rlm_run_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr_smem = smem;
  }
  const int n_env_ctas = (n_envs + RUN_THREADS - 1) / RUN_THREADS;
  rlm_run_kernel<<<n_agent_ctas + n_env_ctas, RUN_THREADS, smem, st>>>(ptr, D, n_agent_ctas, n_env_ctas * RUN_WARPS);
  return cudaGetLastError();
}
int rlm_run_max_resident_ctas(int scratch_bytes, int n_sms) {
  int per_sm = 0;
  size_t smem = rlm_agent_smem_bytes(RUN_WARPS, scratch_bytes);
  cudaFuncSetAttribute(rlm_run_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&per_sm, rlm_run_kernel, RUN_THREADS, smem) != cudaSuccess) per_sm = 1;
  return per_sm * n_sms;
}

// ---------------------------------------------------------------------------------------------
// warps (= envs) per CTA of the warp-per-env tick kernels: 4 096 envs are 512 CTAs of 8 warps, i.e. 3 or 4 CTAs per SM --
// smaller CTAs spread them evenly (RLM_ENVW_WARPS = 1, 2, 4 or 8)
static int envw_warps_per_cta() {
  static int w = 0;
  if (!w) {
    w = ENVW_WARPS_DEFAULT;
    if (const char* e = getenv("RLM_ENVW_WARPS")) { const int v = atoi(e); if (v == 1 || v == 2 || v == 4 || v == 8) w = v; }
  }
  return w;
}
// L1 / shared-memory split of the warp-per-env tick kernels (percent shared; RLM_ENVW_CARVEOUT).  They need 79 KB per SM
// (four CTAs); the rest is better spent as L1 -- even though the SMs are then reconfigured between the two kernels of a tick.
static int envw_carveout() {
  static int c = -1;
  if (c < 0) { c = 40; if (const char* e = getenv("RLM_ENVW_CARVEOUT")) { const int v = atoi(e); if (v >= 35 && v <= 100) c = v; } }
  return c;
}
cudaError_t rlm_launch_env(const DevPtrs& ptr, const DynParams& D, int n_envs, int tslot, int only_begin, int variant, cudaStream_t st) {
  if (D.n_sub > 0) n_envs = D.n_sub;  // one sub-batch
  const bool tape = ptr.tape_cur != nullptr;  // (the cursors exist on the tape source only)
  const int kv = g_day_markets ? 2 : (tape ? 1 : 0);  // instantiation: generator / stream, tape, tape with day markets
  if (variant == 1) {  // one thread per env (SIMT over envs)
    const int T = 32;
    auto kern = kv == 2 ? rlm_env_kernel<T, true, true> : (kv == 1 ? rlm_env_kernel<T, true> : rlm_env_kernel<T, false>);
    static bool attr1[3] = {false, false, false};
    if (!attr1[kv]) {
      // this kernel uses no shared memory at all; its per-thread record copy lives in local memory, i.e. in L1 (RLM_ENVT_CARVEOUT)
      int c = RLM_ENVT_CARVEOUT_DEFAULT;
      if (const char* e = getenv("RLM_ENVT_CARVEOUT")) { const int v = atoi(e); if (v >= 0 && v <= 100) c = v; }
      cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, c);
      attr1[kv] = true;
    }
    kern<<<(n_envs + T - 1) / T, T, 0, st>>>(ptr, D, tslot, only_begin);
    return cudaGetLastError();
  }
  const int W = envw_warps_per_cta();
  const size_t smem = (size_t)W * envw_warp_bytes();
  auto kern = kv == 2 ? rlm_env_kernel_w<true, true> : (kv == 1 ? rlm_env_kernel_w<true> : rlm_env_kernel_w<false>);
  static bool attr[3] = {false, false, false};
  if (!attr[kv]) {
    if (smem > 48 * 1024) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
    }
    // the same L1/shared split as the learner kernel: CTAs of the two kernels (different sub-batches, different streams)
    // can then share an SM instead of waiting for it to drain and be reconfigured
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, envw_carveout());
    attr[kv] = true;
  }
  return launch_pdl(kern, (n_envs + W - 1) / W, W * 32, smem, st, ptr, D, tslot, only_begin);
}

cudaError_t rlm_launch_env_round(const DevPtrs& ptr, const DynParams& D, int n_envs, int tslot, cudaStream_t st) {
  const int W = envw_warps_per_cta();
  const size_t smem = (size_t)W * envw_warp_bytes();
  const bool tape = ptr.tape_cur != nullptr;
  const int kv = g_day_markets ? 2 : (tape ? 1 : 0);  // (as in rlm_launch_env)
  auto kern = kv == 2 ? rlm_env_round_kernel<true, true> : (kv == 1 ? rlm_env_round_kernel<true> : rlm_env_round_kernel<false>);
  static bool attr[3] = {false, false, false};
  if (!attr[kv]) {
    if (smem > 48 * 1024) {
      cudaError_t e = cudaFuncSetAttribute(kern, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
      if (e != cudaSuccess) return e;
    }
    cudaFuncSetAttribute(kern, cudaFuncAttributePreferredSharedMemoryCarveout, envw_carveout());
    attr[kv] = true;
  }
  return launch_pdl(kern, (n_envs + W - 1) / W, W * 32, smem, st, ptr, D, tslot);
}
cudaError_t rlm_launch_runctl(const DevPtrs& ptr, const RunCtl& v, cudaStream_t st) {
  rlm_runctl_kernel<<<1, 1, 0, st>>>(ptr.runctl, v);
  return cudaGetLastError();
}

cudaError_t rlm_launch_agent(const DevPtrs& ptr, const DynParams& D, int n_envs, int scratch_bytes, int tslot, int n_sms, int stage, cudaStream_t st) {
  const int W = 8;
  size_t smem = rlm_agent_smem_bytes(W, scratch_bytes);
  static size_t attr_smem = 0;
  if (smem > attr_smem) {
    cudaError_t e = cudaFuncSetAttribute(rlm_agent_kernel<W>, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem);
    if (e != cudaSuccess) return e;
    attr_smem = smem;
  }
  int grid = (n_envs + W - 1) / W;      // worst case: every env is ready
  int cap = n_sms * 6;                  // beyond ~6 CTAs per SM the grid-stride loop takes over
  if (grid > cap) grid = cap;
  rlm_agent_kernel<W><<<grid, W * 32, smem, st>>>(ptr, D, tslot, stage);
  return cudaGetLastError();
}

cudaError_t rlm_launch_init(const DevPtrs& ptr, int n_envs, int mode, cudaStream_t st) {
  rlm_init_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(ptr, mode);
  return cudaGetLastError();
}
cudaError_t rlm_launch_seed(const DevPtrs& ptr, int n_envs, unsigned seed, cudaStream_t st) {
  rlm_seed_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(ptr, seed);
  return cudaGetLastError();
}
cudaError_t rlm_launch_random_init(const DevPtrs& ptr, int n_policies, cudaStream_t st) {
  rlm_random_init_kernel<<<(n_policies + 63) / 64, 64, 0, st>>>(ptr, n_policies);
  return cudaGetLastError();
}
cudaError_t rlm_launch_gather(const DevPtrs& ptr, int n_envs, int what, void* out, cudaStream_t st) {
  rlm_gather_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(ptr, what, out);
  return cudaGetLastError();
}
cudaError_t rlm_launch_clear_traces(const DevPtrs& ptr, int n_envs, cudaStream_t st) {
  rlm_clear_traces_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(ptr);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Day markets (rlm_set_day_markets).  Envs env0 .. env0+n-1 take markets mk[0..n-1] (-1: the config's; the host launches
// this only when some env's market changes, or the markets themselves were replaced) and forget next_state_tail's
// midprice memo: it holds ToTicks under the old table, and the next day may open at
// the same midprice.  (The band hint needs no clearing: to_ticks checks it against the table, whose unused bands are +inf.)
__global__ void rlm_env_market_kernel(DevPtrs ptr, int env0, int n, const int* mk) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = env0 + i;
  PM.env_market[b] = mk[i];
  EnvHdr* e = (EnvHdr*)(ptr.env + (size_t)b * P.env_stride);
  e->tk_px = 0.0;
  e->tk_ticks = 0;
}
cudaError_t rlm_launch_env_market(const DevPtrs& ptr, int env0, int n, const int* mk, cudaStream_t st) {
  rlm_env_market_kernel<<<(n + 127) / 128, 128, 0, st>>>(ptr, env0, n, mk);
  return cudaGetLastError();
}
// Under day markets the learner kernels fill a record's terminal flag from the config's market, which the host then sets
// to never close (rlm_api.cu, day_markets_on): the flag they write is the date change of Intraday::isTerminal alone.  This
// kernel adds the env's own market's close to the records written since it last ran (every record env, one thread each);
// the host runs it before an env's market changes and before records are read.
__global__ void rlm_fix_terminal_kernel(DevPtrs ptr) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= P.record_envs) return;
  const int n = min(ptr.record_count[b], P.record_cap);
  const int k = PM.env_market[b];  // (-1 only between the first rlm_set_day_markets and its assignment, with no record due)
  if (k >= 0) {
    const VenueD* V = PM.markets + k;
    for (int i = PM.rec_fixed[b]; i < n; ++i) {
      rlm_step_record& r = ptr.records[(size_t)b * P.record_cap + i];
      if (!((long long)r.time_ms > V->open_lo && (long long)r.time_ms < V->close_hi)) r.terminal = 1;
    }
  }
  PM.rec_fixed[b] = max(n, PM.rec_fixed[b]);
}
cudaError_t rlm_launch_fix_terminal(const DevPtrs& ptr, int record_envs, cudaStream_t st) {
  if (record_envs <= 0) return cudaSuccess;
  rlm_fix_terminal_kernel<<<(record_envs + 127) / 128, 128, 0, st>>>(ptr);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// unit-level device entry points (golden vectors of the reference's tests)
// one thread, in order, carrying one band hint from price to price the way an env carries EnvHdr::tk_band (zeroed at
// creation), so that a sequence that jumps between bands exercises both the hinted and the searched band look-up
__global__ void k_test_to_ticks(const double* px, int n, int* out) {
  if (threadIdx.x || blockIdx.x) return;
  int hint = 0;
  for (int i = 0; i < n; ++i) {
    int err = 0;
    const int t = to_ticks(px[i], &err, &hint);
    out[i] = err ? -1 : t;
  }
}
__global__ void k_test_to_price(const int* ticks, int n, double* out) {
  int i = blockIdx.x * blockDim.x + threadIdx.x;
  int err = 0;
  if (i < n) { double p = to_price(ticks[i], &err); out[i] = err ? -1.0 : p; }
}
// one warp per state: all tile indices, out[s][a][96]
__global__ void k_test_tiles(const float* vars, int n, int* out) {
  const unsigned* s_rnd = rlm_rndseq_table;
  int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n) return;
  const float* v = vars + (size_t)warp * P.n_state_vars;
  const int A = P.n_actions, nv = P.n_state_vars;
  for (int g = 0; g < 3; ++g) {
    const float* gv = (g == 1) ? v + 3 : v;
    const int nf = (g == 0) ? 3 : ((g == 1) ? nv - 3 : nv);
    unsigned long long base = tile_base_sum(s_rnd, gv, nf, lane);
    for (int a = 0; a < A; ++a) out[((size_t)warp * A + a) * 96 + g * 32 + lane] = tile_index(s_rnd, base, nf, g * A + a);
  }
}
// one warp per state: the tile indices as each learner form derives them (rlm_test_learner_tiles in include/rlm.h)
__global__ void k_test_learner_tiles(int form, const float* vars, int n, int* out) {
  const int warp = (blockIdx.x * blockDim.x + threadIdx.x) >> 5, lane = threadIdx.x & 31;
  if (warp >= n) return;
  const float* v = vars + (size_t)warp * P.n_state_vars;
  const int A = P.n_actions;
  if (form == RLM_TILES_THREE_WARP) {
    for (int g = 0; g < 3; ++g) {
      const float* gv = (g == 1) ? v + 3 : v;
      const int nf = (g == 0) ? 3 : ((g == 1) ? P.n_state_vars - 3 : P.n_state_vars);
      const unsigned long long base = tile_base_sum(rlm_rndseq_table, gv, nf, lane);
      for (int a = 0; a < A; ++a) out[((size_t)warp * A + a) * 96 + g * 32 + lane] = tile_index(rlm_rndseq_table, base, nf, g * A + a);
    }
    return;
  }
  const LnSums h = ln_hash(rlm_rndseq_table, v, false, lane);
  if (form == RLM_TILES_TRACE_GROUP0) {  // EnvHdr::from_base0 and the group-0 tile rebuilt from it (trace passes, tile tables)
    const int b0 = mod_m(h.s[0]);
    for (int a = 0; a < A; ++a) out[((size_t)warp * A + a) * 32 + lane] = tile0_from_base(b0, a);
    return;
  }
  for (int k = 0; k < 3 * RLM_MAX_ACTIONS; ++k) {
    const int g = k / RLM_MAX_ACTIONS, a = k % RLM_MAX_ACTIONS;
    if (a >= A) continue;
    int f = P.m_pow2 ? ln_tile<true>(h, k) : ln_tile<false>(h, k);  // rlm_learn_kernel's gathers and ln_patch_local
    if (form == RLM_TILES_STAGED) f = (unsigned short)f;            // rlm_learn_staged_kernel's 16-bit index rows
    out[((size_t)warp * A + a) * 96 + g * 32 + lane] = f;
  }
}
__global__ void k_test_order(long long size, long long q_head, const rlm_order_op* ops, int n_ops, rlm_order_state* out) {
  if (threadIdx.x || blockIdx.x) return;
  OrderD o; o.live = 1; o.price = 1.0; o.size = size; o.q_head = q_head; o.q_tail = 0; o.executed = 0; o.initial_queue = q_head; o.transactions = 0;
  for (int i = 0; i < n_ops; ++i) {
    long long ret = 0;
    switch (ops[i].op) {
      case 0: ret = ord_do_transaction(o, ops[i].arg); break;
      case 1: ord_do_cancellation(o, ops[i].arg); break;
      case 2: o.q_tail += ops[i].arg; break;
      case 3: o.q_head = 0; o.q_tail = 0; break;
    }
    out[i].size = o.size; out[i].q_head = o.q_head; out[i].q_tail = o.q_tail; out[i].executed = o.executed; out[i].ret = ret;
  }
}
// RollingMean<double> through the production window_push, window slot W_MID
__global__ void k_test_rolling_mean(const double* vals, int n, double* out, double* ring_mem, EnvHdr* e) {
  if (threadIdx.x || blockIdx.x) return;
  for (int i = 0; i < n; ++i) {
    window_push(*e, ring_mem, W_MID, vals[i], window_peek(*e, ring_mem, W_MID));
    out[2 * i] = e->w_mean[W_MID];
    out[2 * i + 1] = e->w_s[W_MID] / (double)((unsigned long long)((long long)e->w_count[W_MID] - 1));
  }
}

cudaError_t rlm_launch_test_to_ticks(const double* px, int n, int* out) { k_test_to_ticks<<<1, 32>>>(px, n, out); return cudaGetLastError(); }
cudaError_t rlm_launch_test_to_price(const int* t, int n, double* out) { k_test_to_price<<<(n + 127) / 128, 128>>>(t, n, out); return cudaGetLastError(); }
cudaError_t rlm_launch_test_tiles(const float* vars, int n, int* out) { k_test_tiles<<<(n + 3) / 4, 128>>>(vars, n, out); return cudaGetLastError(); }
cudaError_t rlm_launch_test_learner_tiles(int form, const float* vars, int n, int* out) {
  k_test_learner_tiles<<<(n + 3) / 4, 128>>>(form, vars, n, out);
  return cudaGetLastError();
}
cudaError_t rlm_launch_test_order(long long size, long long q_head, const rlm_order_op* ops, int n_ops, rlm_order_state* out) { k_test_order<<<1, 32>>>(size, q_head, ops, n_ops, out); return cudaGetLastError(); }
cudaError_t rlm_launch_test_rolling_mean(const double* vals, int n, double* out, double* ring_mem, EnvHdr* e) { k_test_rolling_mean<<<1, 32>>>(vals, n, out, ring_mem, e); return cudaGetLastError(); }
