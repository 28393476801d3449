// rlm_agent.cuh -- warp-cooperative tile-coded TD agent (one warp per env, lane j = tiling j).
//
// Restates, for N_TILINGS == 32 == warp width:
//   tiles()/hash_UNH        src/rl/tiles.cpp:31-75,130-169
//   State::populateFeatures src/rl/state.cpp:53-65
//   Agent::getQ/argmaxQ     src/rl/agent.cpp:117-174   (DoubleAgent :202-264)
//   Traces                  src/rl/traces.cpp:30-101
//   QLearn/SARSA/DoubleQLearn UpdateTraces/UpdateWeights  src/rl/agent.cpp:268-353
//   Greedy/EpsilonGreedy/Random::Sample  src/rl/policy.cpp:27-75
//   std::mt19937_64, uniform_real/int_distribution (libstdc++ 13), glibc rand()
#pragma once
#include "rlm_env.cuh"

#define FULL 0xffffffffu
#define HS_EMPTY (-1)

// ------------------------------------------------------------------ RNGs (lane 0)
// std::mt19937_64, regenerated one word at a time: equivalent to the batch twist of
// libstdc++'s _M_gen_rand because word k only depends on old x[k], old-or-new x[k+1] and
// x[k+156 mod 312] exactly as they stand when the batch loop reaches k.
__device__ __noinline__ unsigned long long mt_next(unsigned long long* x, int& p) {
  int k = p; if (k >= 312) k -= 312;   // _M_p == 312 means "regenerate": start at word 0
  const unsigned long long UM = 0xFFFFFFFF80000000ull, LM = 0x7FFFFFFFull, A = 0xB5026F5AA96619E9ull;
  int k1 = k + 1; if (k1 == 312) k1 = 0;
  int km = k + 156; if (km >= 312) km -= 312;
  // L2-coherent accesses: the policy generator is drawn from by env CTAs and by agent CTAs of the
  // persistent kernel, which may run on different SMs
  unsigned long long y = (__ldcg(x + k) & UM) | (__ldcg(x + k1) & LM);
  unsigned long long z = __ldcg(x + km) ^ (y >> 1) ^ ((y & 1ull) ? A : 0ull);
  __stcg(x + k, z);
  p = k + 1;   // stays in 1..312; 312 wraps on the next call
  z ^= (z >> 29) & 0x5555555555555555ull;
  z ^= (z << 17) & 0x71D67FFFEDA60000ull;
  z ^= (z << 37) & 0xFFF7EEE000000000ull;
  z ^= z >> 43;
  return z;
}
// generate_canonical<double,53> on a 64-bit URBG + uniform_real_distribution(0,1)
__device__ __noinline__ double mt_uniform_real(unsigned long long* x, int& p) {
  double r = __ull2double_rn(mt_next(x, p)) / 18446744073709551616.0;
  if (r >= 1.0) r = 0.99999999999999988897769753748;  // nextafter(1,0)
  return r * (1.0 - 0.0) + 0.0;
}
// uniform_int_distribution<unsigned>(0,n-1): Lemire with a 128-bit product
__device__ __noinline__ unsigned mt_uniform_int(unsigned long long* x, int& p, unsigned n) {
  unsigned long long range = n;
  unsigned long long g = mt_next(x, p);
  unsigned long long low = g * range, hi = __umul64hi(g, range);
  if (low < range) {
    unsigned long long threshold = (0ull - range) % range;
    while (low < threshold) {
      g = mt_next(x, p);
      low = g * range; hi = __umul64hi(g, range);
    }
  }
  return (unsigned)hi;
}
// glibc rand() (random_r TYPE_3)
__device__ __noinline__ int crand_next(AgentD& e) {
  unsigned v = (unsigned)e.crand_r[e.crand_f] + (unsigned)e.crand_r[e.crand_b];
  e.crand_r[e.crand_f] = (int)v;
  int out = (int)(v >> 1);
  e.crand_f = e.crand_f + 1 == 31 ? 0 : e.crand_f + 1;
  e.crand_b = e.crand_b + 1 == 31 ? 0 : e.crand_b + 1;
  return out;
}

// ------------------------------------------------------------------ windows (lane w = window w)
// Accumulator<double>::push / RollingMean<double>::push (accumulators.cpp:17-27,86-109)
// `old` = ring slot about to be overwritten (the oldest element when the window is full); callers
// load the slots of all windows first so that the HBM/L2 round trips overlap.
__device__ __forceinline__ double window_peek(const EnvHdr& e, const double* ring, int w) {
  return ring[P.win_off[w] + e.w_head[w]];
}
__device__ __noinline__ void window_push(EnvHdr& e, double* ring, int w, double val, double old) {
  const int ws = P.win_size[w];
  double* r = ring + P.win_off[w];
  int head = e.w_head[w], cnt = e.w_count[w];
  double sum = e.w_sum[w], mean = e.w_mean[w], s = e.w_s[w];
  const bool overflow = (cnt == ws);
  r[head] = val;
  head = head + 1 == ws ? 0 : head + 1;
  sum += val;
  double n = (double)(cnt + 1);
  double old_mean = mean;
  mean += (val - mean) / n;
  s += (val - mean) * (val - old_mean);
  if (overflow) {
    sum -= old;
    double n2 = (double)ws;
    double old_mean2 = mean;
    mean -= (old - mean) / n2;
    s -= (old - mean) * (old - old_mean2);
  } else {
    cnt += 1;
  }
  e.w_head[w] = head; e.w_count[w] = cnt; e.w_sum[w] = sum; e.w_mean[w] = mean; e.w_s[w] = s;
}

// ------------------------------------------------------------------ tile coding
__device__ __forceinline__ int mod_m(unsigned long long sum) {  // (int)(sum % m), sum < 2^36
  if (P.m_pow2) return (int)(sum & (unsigned long long)(P.memory_size - 1));
  unsigned long long q = __umul64hi(sum, P.m_magic);
  unsigned long long r = sum - q * (unsigned long long)P.memory_size;
  while (r >= (unsigned long long)P.memory_size) r -= (unsigned long long)P.memory_size;
  return (int)r;
}

// (int) floor(float) as x86-64 evaluates it (cvttss2si): NaN and out-of-range values give INT_MIN ("integer
// indefinite"), where CUDA's cvt would give 0 / saturate.  A NaN state variable is reachable: vwap over an empty volume
// window is 0/0 (intraday.cpp:356-362) and tiles.cpp:56 quantises it like any other value.
__device__ __forceinline__ int f2i_x86(float v) {
  if (!(v >= -2147483648.0f && v < 2147483648.0f)) return (int)0x80000000;
  return (int)v;
}
// coordinate of tiling j for quantised value q at dimension i (tiles.cpp:56-63): base = j*(1+2i)
__device__ __forceinline__ int tile_coord(int q, int i, int j) {
  int base = j * (1 + 2 * i);
  if (q >= base) return q - ((q - base) % RLM_N_TILINGS);
  return q + 1 + ((base - q - 1) % RLM_N_TILINGS) - RLM_N_TILINGS;
}

// Partial hash sum (everything except the action-dependent integer) for lane j's tiling of one
// feature group: floats vars[0..nf) then the tiling index (tiles.cpp:65-68, hash_UNH :152-161).
__device__ __noinline__ unsigned long long tile_base_sum(const unsigned* rnd, const float* vars, int nf, int j) {
  // fully unrolled and predicated so that the table lookups (L1/L2 round trips) are all in flight together
  unsigned v[RLM_N_STATE_MAX];
#pragma unroll
  for (int i = 0; i < RLM_N_STATE_MAX; ++i) {
    v[i] = 0u;
    if (i < nf) {
      int q = f2i_x86(floorf(vars[i] * (float)RLM_N_TILINGS));
      int c = tile_coord(q, i, j);
      v[i] = __ldg(rnd + ((c + 449 * i) & 2047));
    }
  }
  unsigned long long sum = __ldg(rnd + ((j + 449 * nf) & 2047));
#pragma unroll
  for (int i = 0; i < RLM_N_STATE_MAX; ++i) sum += v[i];
  return sum;
}
__device__ __forceinline__ int tile_index(const unsigned* rnd, unsigned long long base, int nf, int h1) {
  return mod_m(base + __ldg(rnd + ((h1 + 449 * (nf + 1)) & 2047)));
}
// group-0 tile of action a from a stored base b0 = (partial hash sum) mod M: (b0 + ra_m[a]) mod M.  Both terms are below
// M <= 2^31 - 1, so their sum can pass INT_MAX once M > 2^30: it is formed unsigned (< 2^32) and reduced by one subtract.
__device__ __forceinline__ int tile0_from_base(int b0, int a) {
  unsigned f = (unsigned)b0 + (unsigned)P.ra_m[a];
  if (f >= (unsigned)P.memory_size) f -= (unsigned)P.memory_size;
  return (int)f;
}

// ---- tile hashing of one state.  sums[g] = lane's partial hash sum of group g (everything but the action term);
// tile (group g, tiling `lane`, action a) = (sums[g] + rg[g][a]) mod M.  The sums are what stays live across the step
// (6 registers); the 27 indices are re-derived where they are needed (2 instructions each for a power-of-two M).
struct LnSums { unsigned long long s[3]; bool null_state; };
__device__ __forceinline__ LnSums ln_hash(const unsigned* __restrict__ rnd, const float* vars, bool null_state, int lane) {
  const int n = P.n_state_vars;
  LnSums out;
  out.null_state = null_state;
#pragma unroll
  for (int g = 0; g < 3; ++g) {
    const float* gv = (g == 1) ? vars + 3 : vars;
    const int nf = (g == 0) ? 3 : ((g == 1) ? n - 3 : n);
    const int NF_MAX = (g == 0) ? 3 : ((g == 1) ? RLM_N_STATE_MAX - 3 : RLM_N_STATE_MAX);
    unsigned v[RLM_N_STATE_MAX];
#pragma unroll
    for (int i = 0; i < NF_MAX; ++i) {
      v[i] = 0u;
      if (i < nf) {
        const int q = f2i_x86(floorf(gv[i] * (float)RLM_N_TILINGS));
        v[i] = __ldg(rnd + ((tile_coord(q, i, lane) + 449 * i) & 2047));
      }
    }
    unsigned long long sum = __ldg(rnd + ((lane + 449 * nf) & 2047));
#pragma unroll
    for (int i = 0; i < NF_MAX; ++i) sum += v[i];
    out.s[g] = null_state ? 0ull : sum;
  }
  return out;
}
template <bool POW2>
__device__ __forceinline__ int ln_tile(const LnSums& h, int k) {  // k = g*9 + a
  if (POW2) {  // (sum + r) mod 2^k only needs the low words; null state: sums are 0 and so is every index (hash_UNH is skipped)
    const unsigned lo = (unsigned)h.s[k / RLM_MAX_ACTIONS] + P.rg[k / RLM_MAX_ACTIONS][k % RLM_MAX_ACTIONS];
    return h.null_state ? 0 : (int)(lo & (unsigned)(P.memory_size - 1));
  }
  return h.null_state ? 0 : mod_m(h.s[k / RLM_MAX_ACTIONS] + P.rg[k / RLM_MAX_ACTIONS][k % RLM_MAX_ACTIONS]);
}

// Exact-order Q(s,a) for all actions (agent.cpp:117-135): lanes gather theta for their tiling,
// values are transposed through shared memory and lanes 0..A-1 accumulate
//   Q += w0*th[f_i] (i<T);  Q += w1*th[f_i] (T<=i<2T);  Q += w2*th[f_i] (T<=i<3T)
// strictly left to right, so the result is bitwise the reference's.
// vars: state variables (n of them) in shared memory; vbuf: >= 2*A*32 doubles of scratch.
// If null_state, every feature index is 0 (the never-populated State of serial.cpp:14-15,55).
#define VROW 33  // padded row stride (doubles) of the transposition buffer: conflict-free for lanes 0..8
__device__ __forceinline__ double seg_sum(double acc, double w, const double* r) {
#pragma unroll 8
  for (int i = 0; i < 32; ++i) acc += w * r[i];
  return acc;
}
// bases[g]: lane j's partial hash sum of group g; computed when !reuse, reused otherwise (the two
// evaluations of one learner step -- before and after the weight update -- are on the same state).
//
// Software pipeline: the 9 (18 for double agents) gathers of group g+1 are issued -- back to back,
// after ALL their indices are known, so that no shared-memory wait sits between two of them --
// before group g is transposed and summed; the DRAM round trip of a group hides behind the
// 32..64 dependent multiply-adds of the previous one.
struct QGather { double a[RLM_MAX_ACTIONS]; double b[RLM_MAX_ACTIONS]; };

// theta starts at +0.0 and only trace_pass writes it, so an entry whose bit in the per-policy
// occupancy bitmap is clear is known to be exactly +0.0 and is not fetched.  The bitmap (M/8 bytes per
// policy, 32 MB for 4096 x 2^16) stays L2-resident, whereas theta (2 GB) does not: the test turns most
// of a step's 864 random DRAM sector reads -- the measured limiter of the agent kernel -- into L2 hits.
__device__ __forceinline__ bool occ_test(const unsigned* occ, int f) { return (__ldcg(occ + (f >> 5)) >> (f & 31)) & 1u; }
// the same test on a copy of the bitmap staged in shared memory (rlm_agent3_kernel, small memory_size)
__device__ __forceinline__ bool occ_test_s(const unsigned* occ_s, int f) { return (occ_s[f >> 5] >> (f & 31)) & 1u; }

// idx: this warp's [27][32] tile-index cache in shared memory (row g*9+a, column lane).  The first
// evaluation of a step fills it, the second one (same state, updated theta) just reads it back.
__device__ __forceinline__ void q_issue(const unsigned* rnd, const double* th_a, const double* th_b, const float* vars, int n,
                                        bool null_state, int g, int lane, unsigned long long* bases, bool reuse, int* idx,
                                        const unsigned* occ, QGather& out) {
  const int A = P.n_actions;
  int f[RLM_MAX_ACTIONS];
  if (reuse && idx) {
#pragma unroll
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) f[a] = (a < A) ? idx[(g * RLM_MAX_ACTIONS + a) * 32 + lane] : 0;
  } else {
    const float* gv = (g == 1) ? vars + 3 : vars;
    const int nf = (g == 0) ? 3 : ((g == 1) ? n - 3 : n);
    unsigned long long base = 0ull;
    if (!null_state) {
      if (reuse) base = bases[g];  // no index cache (fused kernel): reuse at least the partial hash sums
      else { base = tile_base_sum(rnd, gv, nf, lane); bases[g] = base; }
    }
#pragma unroll
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) {
      f[a] = (a < A && !null_state) ? tile_index(rnd, base, nf, g * A + a) : 0;
      if (a < A && idx) idx[(g * RLM_MAX_ACTIONS + a) * 32 + lane] = f[a];
    }
  }
  bool nz[RLM_MAX_ACTIONS];
#pragma unroll
  for (int a = 0; a < RLM_MAX_ACTIONS; ++a) nz[a] = (a < A) && (occ == nullptr || occ_test(occ, f[a]));  // occ == nullptr: dense table
#pragma unroll
  for (int a = 0; a < RLM_MAX_ACTIONS; ++a) out.a[a] = nz[a] ? __ldcg(th_a + f[a]) : 0.0;  // L2-coherent: theta is rewritten by trace_pass, possibly from another SM
  if (th_b) {
#pragma unroll
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) out.b[a] = nz[a] ? __ldcg(th_b + f[a]) : 0.0;
  }
}

__device__ __noinline__ void eval_q(const unsigned* rnd, const double* th_a, const double* th_b, const float* vars, int n,
                       bool null_state, double* vbuf, int lane, double& qa_out, double& qb_out,
                       unsigned long long* bases, bool reuse, int* idx, const unsigned* occ) {
  const int A = P.n_actions;
  double qa = 0.0, qb = 0.0;
  double* va = vbuf;
  double* vb = vbuf + RLM_MAX_ACTIONS * VROW;
  QGather cur, nxt;
  q_issue(rnd, th_a, th_b, vars, n, null_state, 0, lane, bases, reuse, idx, occ, cur);
#pragma unroll
  for (int g = 0; g < 3; ++g) {
    if (g < 2) q_issue(rnd, th_a, th_b, vars, n, null_state, g + 1, lane, bases, reuse, idx, occ, nxt);
#pragma unroll
    for (int a = 0; a < RLM_MAX_ACTIONS; ++a) {
      if (a < A) {
        va[a * VROW + lane] = cur.a[a];
        if (th_b) vb[a * VROW + lane] = cur.b[a];
      }
    }
    __syncwarp();
    if (lane < A) {
      const double* ra = va + lane * VROW;
      const double* rb = vb + lane * VROW;
      // g=0: w0 | g=1: w1 then w2 (the third loop starts at T, not 2T: SURVEY Appendix A8) | g=2: w2
      const int npass = (g == 1) ? 2 : 1;
#pragma unroll 1
      for (int pass = 0; pass < npass; ++pass) {
        const double w = P.gw[(g == 0) ? 0 : ((g == 1) ? 1 + pass : 2)];
        qa = seg_sum(qa, w, ra);
        if (th_b) qb = seg_sum(qb, w, rb);
      }
    }
    __syncwarp();
    if (g < 2) cur = nxt;
  }
  qa_out = qa;
  qb_out = qb;
}

// Address-space promises for the out-of-line learner functions: their pointer parameters are generic, and without
// these ptxas emits the generic forms (LD/ST with a window check, and for atomics a QSPC + shared/global CAS-spin
// fallback whose success predicate makes every atomicAdd wait for its L2 round trip).
#define ASSUME_SHARED(p) __builtin_assume(__isShared((const void*)(p)))
#define ASSUME_GLOBAL(p) __builtin_assume(__isGlobal((const void*)(p)))
// theta[f] += v as a reduction performed at L2 (one IEEE fp64 add, round-to-nearest: the same rounding as the
// reference's load-add-store); nothing is returned, so the warp does not wait for it
__device__ __forceinline__ void red_add_f64(double* p, double v) {
  asm volatile("red.global.add.f64 [%0], %1;" ::"l"(__cvta_generic_to_global(p)), "d"(v) : "memory");
}
__device__ __forceinline__ void red_or_b32(unsigned* p, unsigned v) {
  asm volatile("red.global.or.b32 [%0], %1;" ::"l"(__cvta_generic_to_global(p)), "r"(v) : "memory");
}

// argmax with rand() tie-breaks over q[0..A) (agent.cpp:144-169); lane 0
__device__ __noinline__ int argmax_ties(AgentD& e, const double* q) {
  ASSUME_SHARED(&e); ASSUME_SHARED(q);  // only the learner kernels call this: agent block and Q arrays are in shared memory
  int index = 0, n_ties = 1;
  double cur = q[0];
  for (int a = 1; a < P.n_actions; a++) {
    double val = q[a];
    if (val >= cur) {
      if (val > cur) { cur = val; index = a; }
      else {
        n_ties++;
        if (0 == crand_next(e) % n_ties) { cur = val; index = a; }
      }
    }
  }
  return index;
}
// The same scan, unrolled over values held in registers: the learner's serial TD step runs at ~25 cycles per
// instruction, so the loop-carried shared-memory loads and the call of the version above are worth removing.
// rand() is still drawn exactly when the reference draws it (only on ties with the running maximum).
__device__ __forceinline__ int argmax_ties_fast(AgentD& e, const double* q) {
  double v[RLM_MAX_ACTIONS];
#pragma unroll
  for (int a = 0; a < RLM_MAX_ACTIONS; ++a) v[a] = (a < P.n_actions) ? q[a] : 0.0;
  int index = 0, n_ties = 1;
  double cur = v[0];
#pragma unroll
  for (int a = 1; a < RLM_MAX_ACTIONS; ++a) {
    if (a < P.n_actions) {
      const double val = v[a];
      if (val > cur) { cur = val; index = a; }
      else if (val == cur) {
        n_ties++;
        if (0 == crand_next(e) % n_ties) { cur = val; index = a; }
      }
    }
  }
  return index;
}
// Greedy::Sample (policy.cpp:37-55); lane 0
__device__ __noinline__ int greedy_sample(AgentD& e, const double* qs) {
  int argmax = 0, n_ties = 1;
  for (int a = 1; a < P.n_actions; a++) {
    if (qs[a] > qs[argmax]) argmax = a;
    else if (qs[a] >= qs[argmax]) {
      n_ties++;
      if (0 == crand_next(e) % n_ties) argmax = a;
    }
  }
  return argmax;
}
// Agent::action / DoubleAgent::action + Policy::Sample; lane 0.  qa/qb: Q_A(s,.), Q_B(s,.)
__device__ __noinline__ int policy_action(AgentD& e, const double* qa, const double* qb, unsigned long long* mt, const DynParams& D) {
  double qs[RLM_MAX_ACTIONS];
  for (int a = 0; a < P.n_actions; ++a) qs[a] = P.is_double ? (qa[a] + qb[a]) / 2.0 : qa[a];
  int pt = D.greedy ? RLM_POLICY_GREEDY : P.policy_type;
  if (pt == RLM_POLICY_RANDOM) return (int)mt_uniform_int(mt, e.mt_pol_idx, (unsigned)P.n_actions);
  if (pt == RLM_POLICY_EPSILON_GREEDY) {
    if (mt_uniform_real(mt, e.mt_pol_idx) < D.eps) return (int)mt_uniform_int(mt, e.mt_pol_idx, (unsigned)P.n_actions);
  }
  if (pt == RLM_POLICY_BOLTZMANN) {  // Boltzmann::Sample (policy.cpp:98-115); exp() is CUDA's, the reference's is glibc's
    double pr[RLM_MAX_ACTIONS];
    double z = 0.0;
    for (int a = 0; a < P.n_actions; ++a) { pr[a] = exp(qs[a] / D.tau); z += pr[a]; }
    double acc = 0.0;
    const double r = mt_uniform_real(mt, e.mt_pol_idx);
    for (int a = 0; a < P.n_actions; ++a) {
      acc += pr[a] / z;
      if (r < acc) return a;
    }
    return P.n_actions - 1;
  }
  return greedy_sample(e, qs);
}

// ------------------------------------------------------------------ traces + weight update
// The reference keeps a dense float e[M] plus a nonzero list (traces.cpp); here only the list
// exists: (f, e) pairs, compact, per env.  One fused pass implements, in the reference's order,
//   Traces::decay(rate)            e *= rate; drop if e < 0.01                       traces.cpp:30-38
//   Traces::update(from, action)   for a = 0..A-1: clear / set the 32 group-0 tiles   traces.cpp:40-50
//   Agent::updateQ(alpha*delta)    theta[f] += (alpha*delta/32) * e[f]                agent.cpp:137-142
// update()'s outcome for a feature f touched by it is decided by the LAST action whose tile list
// contains f (set if that action is the one taken, cleared otherwise).  Tile (j, a) of the
// from-state is (b_j + r_a) mod M with b_j = lane j's partial hash sum mod M (EnvHdr::from_base0)
// and r_a = rndseq[(a + 449*4) & 2047] mod M (DevParams::ra_m), so "f is a tile of action a" is
// "(f - r_a) mod M is one of the 32 b_j": a 128-slot hash set of the b_j answers it with A probes.
#define SS_SLOTS 128
__device__ __forceinline__ unsigned ss_hash(int x) { return ((unsigned)x * 2654435761u) >> 25; }  // 7 bits
__device__ __forceinline__ bool ss_member(const int* ss, int x) {
  unsigned slot = ss_hash(x);
  while (true) {
    int k = ss[slot];
    if (k == x) return true;
    if (k == HS_EMPTY) return false;
    slot = (slot + 1) & (SS_SLOTS - 1);
  }
}
// last action whose group-0 tile list contains f, or -1
__device__ __forceinline__ int last_writer(const int* ss, int f, bool null_from, int a0 = 0) {
  const int A = P.n_actions;
  if (null_from) return f == 0 ? A - 1 : -1;  // every tile of every action is feature 0
  int la = -1;
#pragma unroll 1
  for (int a = a0; a < A; ++a) {
    int x = f - P.ra_m[a];
    if (x < 0) x += (int)P.memory_size;
    if (ss_member(ss, x)) la = a;
  }
  return la;
}

// The 3-warp learner kernel answers the same question with ONE probe: its two idle warps insert all A*32 tiles
// of the from-state into a 512-slot table  feature -> last action that lists it  (keys in tt[0..512), values in
// tt[512..1024)) while warp 0 computes the TD error; the serial trace pass then costs one lookup per entry instead
// of A membership tests (cold, serial code runs at ~25 cycles per instruction here: instruction count is time).
#define TT_SLOTS 512
__device__ __forceinline__ unsigned tt_hash(int f) { return ((unsigned)f * 2654435761u) >> 23; }  // 9 bits
__device__ __forceinline__ void tt_insert(int* tt, int f, int a) {
  unsigned slot = tt_hash(f);
  while (true) {
    int old = atomicCAS(&tt[slot], HS_EMPTY, f);
    if (old == HS_EMPTY || old == f) { atomicMax(&tt[TT_SLOTS + slot], a); return; }
    slot = (slot + 1) & (TT_SLOTS - 1);
  }
}
__device__ __forceinline__ int tt_last_writer(const int* tt, int f) {
  unsigned slot = tt_hash(f);
  while (true) {
    int k = tt[slot];
    if (k == f) return tt[TT_SLOTS + slot];
    if (k == HS_EMPTY) return -1;
    slot = (slot + 1) & (TT_SLOTS - 1);
  }
}
// building warps, thread t of n_threads: tt_build clears the slots; after a barrier among the builders, tt_fill
// inserts tiles t, t + n_threads, ... of the A*32 (tile j, action a) of the from-state
__device__ __forceinline__ void tt_build(int* tt, const AgentD& e, int t, int n_threads) {
  for (int i = t; i < 2 * TT_SLOTS; i += n_threads) tt[i] = (i < TT_SLOTS) ? HS_EMPTY : -1;
}
__device__ __forceinline__ void tt_fill(int* tt, const AgentD& e, int t, int n_threads) {
  const int n = P.n_actions * 32;
  for (int i = t; i < n; i += n_threads) {
    const int a = i >> 5, j = i & 31;
    tt_insert(tt, tile0_from_base(e.from_base0[j], a), a);
  }
}

// 4096-bit filter of the features whose weight this step's update touched (every entry that survives the trace pass).
// The learner kernel's second evaluation -- same state, theta after the update -- re-reads only the tiles the filter
// flags and keeps the first evaluation's products for the rest (a false positive is just a redundant load).
#define BLOOM_WORDS 128
__device__ __forceinline__ unsigned bloom_bit(int f) { return ((unsigned)f * 2654435761u) >> 20; }  // 12 bits
__device__ __forceinline__ void bloom_set(unsigned* bl, int f) { const unsigned h = bloom_bit(f); atomicOr(&bl[h >> 5], 1u << (h & 31)); }
__device__ __forceinline__ bool bloom_test(const unsigned* bl, int f) { const unsigned h = bloom_bit(f); return (bl[h >> 5] >> (h & 31)) & 1u; }

// occ: the policy's bitmap in HBM; occ_s: its shared-memory copy for this step, or nullptr
#ifdef RLM_TIMING
__device__ long long g_tp_clk[8];
#define TP(i) do { if (lane == 0) tp_[i] = clock64(); } while (0)
#else
#define TP(i) do { } while (0)
#endif
// tt: the prebuilt tile table (see above), or nullptr: build the 128-slot set of the b_j in `ss` here
__device__ __noinline__ int trace_pass(AgentD& e, int* ss, const int* tt, int* tf, float* te, double* theta, unsigned* occ, unsigned* occ_s,
                                       int action, float rate, double scaled_update, int lane) {
#ifdef RLM_TIMING
  long long tp_[5] = {0, 0, 0, 0, 0};
#endif
  TP(0);
  ASSUME_SHARED(&e); ASSUME_SHARED(ss); ASSUME_GLOBAL(tf); ASSUME_GLOBAL(te); ASSUME_GLOBAL(theta); ASSUME_GLOBAL(occ);
  if (occ_s) ASSUME_SHARED(occ_s);
  const bool null_from = e.null_from != 0;
  const int b0 = e.from_base0[lane];
  unsigned* bloom = nullptr;
  if (tt) {
    ASSUME_SHARED(tt);
    bloom = (unsigned*)ss;  // the small set is not needed on this path: its 512 bytes hold the filter
    for (int i = lane; i < BLOOM_WORDS; i += 32) bloom[i] = 0u;
    __syncwarp();
  } else {
    for (int i = lane; i < SS_SLOTS; i += 32) ss[i] = HS_EMPTY;
    __syncwarp();
    if (!null_from) {
      unsigned slot = ss_hash(b0);
      while (true) {
        int old = atomicCAS(&ss[slot], HS_EMPTY, b0);
        if (old == HS_EMPTY || old == b0) break;
        slot = (slot + 1) & (SS_SLOTS - 1);
      }
    }
    __syncwarp();
  }
  TP(1);
  const float tol = 0.01f;
  int w = 0;
  if (rate != 0.0f) {
    const int n = e.n_traces;
    // TR_AHEAD rounds of 32 entries are loaded at once (one memory round trip per chunk instead of one per
    // round); the list is compacted in place, and a chunk only ever writes below the entries it has read
#define TR_AHEAD 4
#pragma unroll 1
    for (int base = 0; base < n; base += 32 * TR_AHEAD) {
      int fq[TR_AHEAD];
      float eq[TR_AHEAD];
#pragma unroll
      for (int k = 0; k < TR_AHEAD; ++k) {
        const int i = base + 32 * k + lane;
        fq[k] = (i < n) ? __ldcg(tf + i) : 0;
        eq[k] = (i < n) ? __ldcg(te + i) : 0.0f;
      }
#pragma unroll
      for (int k = 0; k < TR_AHEAD; ++k) {
        if (base + 32 * k < n) {  // warp-uniform
          const int i = base + 32 * k + lane;
          const int f = fq[k];
          const float ev = eq[k] * rate;
          bool keep = (i < n) && !(ev < tol);
          if (keep) keep = ((tt && !null_from) ? tt_last_writer(tt, f) : last_writer(ss, f, null_from)) < 0;
          unsigned mask = __ballot_sync(FULL, keep);
          int pos = w + __popc(mask & ((1u << lane) - 1u));
          if (keep) {
            __stcg(tf + pos, f);
            __stcg(te + pos, ev);
            red_add_f64(theta + f, scaled_update * (double)ev);
            if (bloom) bloom_set(bloom, f);
          }
          w += __popc(mask);
        }
      }
    }
  }
  TP(2);
  // set(): the taken action's tiles that no later action cleared; one entry per distinct f
  {
    const int f = null_from ? 0 : tile0_from_base(b0, action);
    // f is a tile of `action` by construction: only later actions can still clear it
    bool add;
    if (null_from) add = (action == P.n_actions - 1);
    else if (tt) add = (tt_last_writer(tt, f) == action);  // f is listed by `action`; a later action would own the slot
    else add = (last_writer(ss, f, false, action + 1) < 0);
    unsigned same = __match_any_sync(FULL, f);
    add = add && ((__ffs(same) - 1) == lane);
    unsigned mask = __ballot_sync(FULL, add);
    int pos = w + __popc(mask & ((1u << lane) - 1u));
    int total = w + __popc(mask);
    if (total > P.trace_cap) {
      if (lane == 0) e.err |= ERR_TRACE_OVERFLOW;
      add = add && (pos < P.trace_cap);
      total = P.trace_cap;
    }
    bool fresh = false;
    if (add) {
      __stcg(tf + pos, f);
      __stcg(te + pos, 1.0f);
      const unsigned bit = 1u << (f & 31);
      // every list entry was appended here once: its bit is set
      if (occ_s) {
        fresh = !(atomicOr(occ_s + (f >> 5), bit) & bit);  // shared-memory copy answers; HBM gets a fire-and-forget OR
        red_or_b32(occ + (f >> 5), bit);
      } else {
        fresh = !(atomicOr(occ + (f >> 5), bit) & bit);
      }
      red_add_f64(theta + f, scaled_update * (double)1.0f);
      if (bloom) bloom_set(bloom, f);
    }
    const int n_fresh = __popc(__ballot_sync(FULL, fresh));
    if (lane == 0) e.n_occ += n_fresh;
    w = total;
  }
  __syncwarp();
  TP(3);
#ifdef RLM_TIMING
  if (lane == 0 && tp_[3] - tp_[0] > g_tp_clk[0]) {  // keep the slowest pass seen (racy, debug only)
    g_tp_clk[0] = tp_[3] - tp_[0]; g_tp_clk[1] = tp_[1] - tp_[0]; g_tp_clk[2] = tp_[2] - tp_[1]; g_tp_clk[3] = tp_[3] - tp_[2];
    g_tp_clk[4] = e.n_traces; g_tp_clk[5] = (rate != 0.0f);
  }
#endif
  return w;
}

// order-independent hash of {(f, e, theta[f])} for the parity record
__device__ __noinline__ unsigned long long trace_hash(const int* tf, const float* te, const double* theta, int n, int lane) {
  ASSUME_GLOBAL(tf); ASSUME_GLOBAL(te); ASSUME_GLOBAL(theta);
  unsigned long long h = 0;
  for (int i = lane; i < n; i += 32) {
    int f = __ldcg(tf + i);
    h += rlm_trace_mix((unsigned)f, __float_as_uint(__ldcg(te + i)), (unsigned long long)__double_as_longlong(__ldcg(theta + f)));
  }
  for (int o = 16; o > 0; o >>= 1) h += __shfl_xor_sync(FULL, h, o);
  return h;
}
