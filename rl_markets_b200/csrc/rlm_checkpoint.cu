// rlm_checkpoint.cu -- rlm_save / rlm_load (include/rlm.h): the file format, the pipeline that moves a handle's state
// through it, and the kernels that pack and unpack weight tables and fingerprint a tape day library.
//
// A packed table of `len` 64-bit words is a bitmap of the words that are not +0.0 -- bitwise, so -0.0 and every NaN
// payload count as set -- followed by those words in index order.  One chunk of work is `nt` tables of `len` words each,
// table t at src + t * tstride (whole tables of one weight array, or one slice of a table larger than a chunk).  Every
// block owns CK_TILE words of one table: warp w the 1024 words from w * 1024, 32 at a time, lane j one word of each.
// The tile is the unit of the two-level scan: a count pass writes each block's population, rlm_ck_scan_kernel turns the
// populations into exclusive offsets over the chunk, and the pack / unpack pass then moves each block's values at its
// offset.  The values of table t therefore start at off[t * bpt]: the chunk's tables lie back to back in table order.
// The kernels take every parameter by value (no __constant__ block), so no existing kernel changes.
#include <cuda_runtime.h>
#include <errno.h>
#include <fcntl.h>
#include <limits.h>
#include <stddef.h>
#include <string.h>
#include <sys/stat.h>
#include <unistd.h>
#include <algorithm>

#include "rlm_handle.h"

#define RLM_CK_TILE 8192  // words per block of the pack / unpack kernels
// device scratch of one chunk of packed tables
struct CkChunkDev {
  double* vals;       // the chunk's nonzero words, table after table
  unsigned* bits;     // [nt][ceil(len / 32)] bitmap words
  int* blk_cnt;       // [nt * bpt] population of each block's tile
  long long* off;     // [nt * bpt + 1] exclusive offsets of the tiles' values
  long long* cnt;     // [nt] values of each table
  long long* expect;  // [nt] unpack: the stored value count of each table
  int* err;           // unpack: nonzero = the bitmap does not match the stored counts
};

#define CK_WARPS 8

__device__ __forceinline__ unsigned ck_lanes_below() {
  unsigned m;
  asm("mov.u32 %0, %%lanemask_lt;" : "=r"(m));
  return m;
}

// sum of v over the block (every thread gets it); sh: CK_WARPS slots
__device__ __forceinline__ long long ck_block_sum(long long v, long long* sh) {
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  const int lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  if (lane == 0) sh[w] = v;
  __syncthreads();
  long long s = 0;
  for (int i = 0; i < CK_WARPS; ++i) s += sh[i];
  return s;
}

// Pack, pass 1: the bitmap words of each tile and the tile's population.  bits: [nt][bw] 32-bit words, bw = ceil(len / 32)
__global__ void __launch_bounds__(CK_WARPS * 32) rlm_pack_count_kernel(const unsigned long long* __restrict__ src, long long tstride,
                                                                       long long len, int bpt, long long bw, unsigned* __restrict__ bits,
                                                                       int* __restrict__ blk_cnt) {
  __shared__ long long sh[CK_WARPS];
  const int t = blockIdx.x / bpt, k = blockIdx.x % bpt, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned long long* s = src + (size_t)t * tstride;
  const long long i0 = (long long)k * RLM_CK_TILE + (long long)w * 1024;
  unsigned mine = 0;
  int cnt = 0;
  for (int j = 0; j < 32; ++j) {
    const long long i = i0 + j * 32 + lane;
    const unsigned m = __ballot_sync(0xffffffffu, i < len && s[i] != 0ull);
    if (lane == j) mine = m;
    cnt += __popc(m);
  }
  const long long wi = i0 / 32 + lane;
  if (wi < bw) bits[(size_t)t * bw + wi] = mine;
  const long long tot = ck_block_sum(lane == 0 ? cnt : 0, sh);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = (int)tot;
}

// Unpack, pass 1: each tile's population from the stored bitmap.  Bits at or past `len` must be clear: a set one is a
// corrupt bitmap (*err), and it is not counted.
__global__ void __launch_bounds__(CK_WARPS * 32) rlm_unpack_count_kernel(const unsigned* __restrict__ bits, long long len, int bpt, long long bw,
                                                                         int* __restrict__ blk_cnt, int* err) {
  __shared__ long long sh[CK_WARPS];
  const int t = blockIdx.x / bpt, k = blockIdx.x % bpt, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const long long i0 = (long long)k * RLM_CK_TILE + (long long)w * 1024, wi = i0 / 32 + lane;
  unsigned m = wi < bw ? bits[(size_t)t * bw + wi] : 0u;
  const long long first = wi * 32;
  const unsigned valid = first + 32 <= len ? 0xffffffffu : (first >= len ? 0u : (1u << (len - first)) - 1u);
  if (m & ~valid) atomicOr(err, 1);
  m &= valid;
  const long long tot = ck_block_sum(__popc(m), sh);
  if (threadIdx.x == 0) blk_cnt[blockIdx.x] = (int)tot;
}

// One block: exclusive offsets of the n block populations over the chunk (off[n] = the chunk's total) and each table's
// value count cnt[t].  expect != null: a table whose count differs from expect[t] sets *err.
__global__ void __launch_bounds__(1024) rlm_ck_scan_kernel(const int* __restrict__ blk_cnt, int n, int bpt, int nt, long long* __restrict__ off,
                                                           long long* __restrict__ cnt, const long long* __restrict__ expect, int* err) {
  __shared__ long long part[1024];
  const int per = (n + 1023) / 1024, a = min(n, (int)threadIdx.x * per), b = min(n, a + per);
  long long s = 0;
  for (int i = a; i < b; ++i) s += blk_cnt[i];
  part[threadIdx.x] = s;
  __syncthreads();
  for (int o = 1; o < 1024; o <<= 1) {  // inclusive Hillis-Steele scan of the thread partials
    const long long v = threadIdx.x >= o ? part[threadIdx.x - o] : 0;
    __syncthreads();
    part[threadIdx.x] += v;
    __syncthreads();
  }
  long long run = part[threadIdx.x] - s;
  for (int i = a; i < b; ++i) { off[i] = run; run += blk_cnt[i]; }
  if (threadIdx.x == 1023) off[n] = part[1023];
  __syncthreads();
  for (int t = threadIdx.x; t < nt; t += 1024) {
    const long long c = off[(t + 1) * bpt] - off[t * bpt];
    cnt[t] = c;
    if (expect && c != expect[t]) atomicOr(err, 2);
  }
}

// Pack, pass 2: every block writes its tile's nonzero words, in index order, from off[block].
__global__ void __launch_bounds__(CK_WARPS * 32) rlm_pack_kernel(const unsigned long long* __restrict__ src, long long tstride, long long len,
                                                                 int bpt, long long bw, const unsigned* __restrict__ bits,
                                                                 const long long* __restrict__ off, unsigned long long* __restrict__ vals) {
  __shared__ long long sh[CK_WARPS];
  const int t = blockIdx.x / bpt, k = blockIdx.x % bpt, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  const unsigned long long* s = src + (size_t)t * tstride;
  const long long i0 = (long long)k * RLM_CK_TILE + (long long)w * 1024, wi = i0 / 32 + lane;
  const unsigned m = wi < bw ? bits[(size_t)t * bw + wi] : 0u;
  // lane j's exclusive prefix over the warp's 32 bitmap words, then the warp's place in the block
  const int pc = __popc(m);
  int incl = pc;
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) sh[w] = incl;
  __syncthreads();
  long long base = off[blockIdx.x];
  for (int i = 0; i < w; ++i) base += sh[i];
  const int excl = incl - pc;
  const unsigned below = ck_lanes_below();
  for (int j = 0; j < 32; ++j) {
    const unsigned mj = __shfl_sync(0xffffffffu, m, j);
    const int pj = __shfl_sync(0xffffffffu, excl, j);
    if (!mj) continue;
    const long long i = i0 + j * 32 + lane;
    if ((mj >> lane) & 1u) vals[base + pj + __popc(mj & below)] = s[i];
  }
}

// Unpack, pass 2: every word of the tile, the stored value where its bit is set and +0.0 elsewhere.  Nothing is written
// when a count pass or the scan flagged the chunk (*err): the values would not line up with the bitmap.
__global__ void __launch_bounds__(CK_WARPS * 32) rlm_unpack_kernel(const unsigned* __restrict__ bits, long long len, int bpt, long long bw,
                                                                   const long long* __restrict__ off, const unsigned long long* __restrict__ vals,
                                                                   unsigned long long* __restrict__ dst, long long tstride, const int* err) {
  __shared__ long long sh[CK_WARPS];
  if (*err) return;
  const int t = blockIdx.x / bpt, k = blockIdx.x % bpt, lane = threadIdx.x & 31, w = threadIdx.x >> 5;
  unsigned long long* d = dst + (size_t)t * tstride;
  const long long i0 = (long long)k * RLM_CK_TILE + (long long)w * 1024, wi = i0 / 32 + lane;
  const long long first = wi * 32;
  const unsigned valid = first + 32 <= len ? 0xffffffffu : (first >= len ? 0u : (1u << (len - first)) - 1u);
  const unsigned m = (wi < bw ? bits[(size_t)t * bw + wi] : 0u) & valid;
  const int pc = __popc(m);
  int incl = pc;
  for (int o = 1; o < 32; o <<= 1) { const int v = __shfl_up_sync(0xffffffffu, incl, o); if (lane >= o) incl += v; }
  if (lane == 31) sh[w] = incl;
  __syncthreads();
  long long base = off[blockIdx.x];
  for (int i = 0; i < w; ++i) base += sh[i];
  const int excl = incl - pc;
  const unsigned below = ck_lanes_below();
  for (int j = 0; j < 32; ++j) {
    const unsigned mj = __shfl_sync(0xffffffffu, m, j);
    const int pj = __shfl_sync(0xffffffffu, excl, j);
    const long long i = i0 + j * 32 + lane;
    if (i < len) d[i] = ((mj >> lane) & 1u) ? vals[base + pj + __popc(mj & below)] : 0ull;
  }
}

// 64-bit fingerprint of n words: the sum, modulo 2^64, of a mix of every word with its index (order-free, so the
// reduction is deterministic).  *out must start at 0.
__device__ __forceinline__ unsigned long long ck_mix(unsigned long long x) {
  x += 0x9E3779B97F4A7C15ull;
  x = (x ^ (x >> 30)) * 0xBF58476D1CE4E5B9ull;
  x = (x ^ (x >> 27)) * 0x94D049BB133111EBull;
  return x ^ (x >> 31);
}
__global__ void __launch_bounds__(256) rlm_fingerprint_kernel(const unsigned long long* __restrict__ w, long long n, unsigned long long* out) {
  unsigned long long s = 0;
  for (long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x; i < n; i += (long long)gridDim.x * blockDim.x)
    s += ck_mix(w[i] ^ ((unsigned long long)i * 0xD6E8FEB86659FD93ull));
  for (int o = 16; o > 0; o >>= 1) s += __shfl_xor_sync(0xffffffffu, s, o);
  if ((threadIdx.x & 31) == 0) atomicAdd(out, s);
}

static long long ck_bw(long long len) { return (len + 31) / 32; }  // bitmap words of a table slice
static int ck_bpt(long long len) { return (int)((len + RLM_CK_TILE - 1) / RLM_CK_TILE); }  // blocks (tiles) of a table slice

static cudaError_t rlm_launch_pack(const CkChunkDev& c, const double* src, long long tstride, int nt, long long len, cudaStream_t st) {
  const int bpt = ck_bpt(len), n = nt * bpt;
  const long long bw = ck_bw(len);
  rlm_pack_count_kernel<<<n, CK_WARPS * 32, 0, st>>>((const unsigned long long*)src, tstride, len, bpt, bw, c.bits, c.blk_cnt);
  rlm_ck_scan_kernel<<<1, 1024, 0, st>>>(c.blk_cnt, n, bpt, nt, c.off, c.cnt, nullptr, c.err);
  rlm_pack_kernel<<<n, CK_WARPS * 32, 0, st>>>((const unsigned long long*)src, tstride, len, bpt, bw, c.bits, c.off,
                                               (unsigned long long*)c.vals);
  return cudaGetLastError();
}

static cudaError_t rlm_launch_unpack(const CkChunkDev& c, double* dst, long long tstride, int nt, long long len, int count_only, cudaStream_t st) {
  const int bpt = ck_bpt(len), n = nt * bpt;
  const long long bw = ck_bw(len);
  rlm_unpack_count_kernel<<<n, CK_WARPS * 32, 0, st>>>(c.bits, len, bpt, bw, c.blk_cnt, c.err);
  rlm_ck_scan_kernel<<<1, 1024, 0, st>>>(c.blk_cnt, n, bpt, nt, c.off, c.cnt, count_only ? nullptr : c.expect, c.err);
  if (!count_only)
    rlm_unpack_kernel<<<n, CK_WARPS * 32, 0, st>>>(c.bits, len, bpt, bw, c.off, (const unsigned long long*)c.vals, (unsigned long long*)dst,
                                                   tstride, c.err);
  return cudaGetLastError();
}

static cudaError_t rlm_launch_fingerprint(const void* data, long long n_words, unsigned long long* out, int n_sms, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(out, 0, 8, st);
  if (e != cudaSuccess || n_words <= 0) return e;
  const long long want = (n_words + 255) / 256;
  const int grid = (int)(want < (long long)n_sms * 8 ? want : (long long)n_sms * 8);
  rlm_fingerprint_kernel<<<grid, 256, 0, st>>>((const unsigned long long*)data, n_words, out);
  return cudaGetLastError();
}

// ---------------------------------------------------------------------------------------------
// Checkpoints: rlm_save / rlm_load (include/rlm.h).  Everything that carries from one call on a handle to the next, and
// whether a file holds it:
//   rlm_handle_s
//     cfg                  saved; a loading handle must match it field for field except `device`, and takes `flow` from it
//     hp, cfg_venue        derived from cfg (hp.flow restored with cfg.flow, hp.venue follows the day markets)
//     dyn                  greedy and backtest saved; the other fields are per-launch values or engine switches
//     shared_dyn           saved: rlm_apply_dtheta finishes the tick rlm_shared_tick_accumulate began with it
//     alpha, eps, tau      saved (the schedules of rlm_handle_terminal)
//     launches             saved
//     run_seq              saved: the round-paced engine tells its calls apart by EnvHdr::run_id == RunCtl::run_id, so a
//                          handle restarting at 0 would skip ticks
//     mlog                 acc, written, rows and cap saved: the log is on in the loaded handle if it was on when saved
//     day_off              saved, and must equal the loading handle's library (whose bytes are checked by fingerprint)
//     env_day, day_market, env_mkt, n_markets, dm   saved; dm's buffers are allocated or freed to match
//     stream_ticks, stream_cursor   equal at a save (every uploaded tick consumed); 0 after a load
//     d_stream, stream_cap, stream_buf, copy_stream, ev_copied, ev_consumed, consumed_valid   transient: the stream
//                          source's upload buffers, empty of unconsumed ticks at a save; the caller uploads after a load
//     rec_dirty            transient: records are fixed (fix_records) before they are saved
//     stream, own_stream, n_sms, engine, n_agent_ctas, env_variant, agent_variant, n_sub, staged, rounds, rounds_auto,
//     round_streams, use_graphs   the loading handle's own: its device and stream, and engine switches, under which every
//                          engine computes the same results
//     graphs, graph_warm   dropped and cleared by a load (the graphs captured the old buffers and parameters)
//     d_qctl               transient: persistent engine (RLM_ENGINE=p), which save and load refuse
//     in_rounds            transient: false between calls
//     profile, ev, prof_*  transient: measurement hooks
//     ready_cap, n_policies, env_bytes   derived from cfg
//     d_gather, h_gather, gather_cap, sub_stream, ev_fork, ev_join, h_live, ev_live   transient: staging and
//                          synchronisation objects
//   DevPtrs
//     env                  saved whole (env_stride bytes per env, window rings included)
//     theta, theta_b       saved packed, one table per policy
//     dtheta               saved packed: a save between rlm_shared_tick_accumulate and rlm_apply_dtheta keeps the update
//     trace_f, trace_e, mt_pol, mt_agt, counters, occ, hsum   saved
//     records, record_count   saved
//     ready, ready_count   saved: the ready list of rlm_env_step / rlm_shared_tick_accumulate is read by the next call
//     tape_cur, tape_lo    saved
//     tape                 not saved (a library can be gigabytes): the loading handle holds the same one
//     stream               transient (see d_stream)
//     runctl               transient: rewritten before every kernel that reads it (round-paced call, stream-source graph)
//     q_slots, q_head, q_tail, env_warps_done, q_done, ag_done, q_size   transient: persistent engine, refused
//
// File: a header (CkHeader), a section table, the raw sections in table order, then every weight table packed -- a
// bitmap of its words that are not +0.0, (M + 7) / 8 bytes, then those words in index order.  Tables cross PCIe packed
// (rlm_checkpoint.cu), in chunks of at most RLM_CK_CHUNK words through two device and two pinned buffers: the copy and
// the write of chunk k run while chunk k + 1 is packed (loading: the read of chunk k + 1 while chunk k is copied and
// unpacked), so device memory does not grow with n_envs x memory_size.
#define RLM_CK_VERSION 1
#define RLM_CK_CHUNK (1LL << 22)
#define RLM_CK_MAX_TABLES 4096

struct CkHeader {
  char magic[8];  // "RLMCKPT"
  uint32_t version, n_sections;
  uint64_t file_bytes;
  uint32_t header_bytes;  // header + section table: the first section's offset
  uint32_t env_stride, env_hdr_bytes, pad;
  int64_t model_log_cap;  // (offset 40, and the config at 48: rl_markets_b200/lib.py reads both)
  rlm_config cfg;
  double alpha, eps, tau;
  int64_t launches;
  int32_t run_seq, greedy, backtest, n_days, n_markets, has_env_market;
  uint64_t library_fp;  // tape: fingerprint of the day library's bytes (rlm_fingerprint_kernel)
  DynParams shared_dyn;
};
static_assert(offsetof(CkHeader, model_log_cap) == 40 && offsetof(CkHeader, cfg) == 48, "lib.py reads the header at fixed offsets");
static_assert(offsetof(CkHeader, library_fp) == 48 + sizeof(rlm_config) + 56, "tests/checkpoint_format.py reads library_fp after the config");
struct CkSection { uint32_t id, table; uint64_t offset, bytes, count; };  // count: values of a packed table
enum { CK_ENV = 1, CK_HSUM, CK_OCC, CK_TRACE_F, CK_TRACE_E, CK_MT_POL, CK_MT_AGT, CK_COUNTERS, CK_READY, CK_READY_COUNT, CK_RECORDS,
       CK_RECORD_COUNT, CK_TAPE_CUR, CK_TAPE_LO, CK_ENV_DAY, CK_DAY_OFF, CK_DAY_MARKET, CK_MARKETS, CK_ENV_MARKET, CK_REC_FIXED,
       CK_MLOG_ACC, CK_MLOG_WRITTEN, CK_MLOG_ROWS, CK_THETA = 64, CK_THETA_B, CK_DTHETA };

// what decides the layout beyond the config, and where the sections of a file come from or go to
struct CkView {
  long long mlog_cap;
  int n_days, n_markets, has_env_market;
  ModelLogPtrs mlog;
  VenueD* markets;
  int* rec_fixed;
  void *env_day, *day_off, *day_market, *env_mkt;  // host sections
};
struct CkRaw { uint32_t id; size_t bytes; void* dev; void* host; };
static std::vector<CkRaw> ck_raw(rlm_handle h, const CkView& v) {
  const size_t B = h->cfg.n_envs, R = h->hp.record_envs;
  std::vector<CkRaw> r;
  auto dev = [&](uint32_t id, size_t bytes, const void* p) { r.push_back({id, bytes, (void*)p, nullptr}); };
  auto host = [&](uint32_t id, size_t bytes, void* p) { r.push_back({id, bytes, nullptr, p}); };
  dev(CK_ENV, h->env_bytes, h->ptr.env);
  dev(CK_HSUM, B * 3 * 32 * 8, h->ptr.hsum);
  dev(CK_OCC, (size_t)h->n_policies * h->hp.occ_words * 4, h->ptr.occ);
  dev(CK_TRACE_F, B * h->hp.trace_cap * 4, h->ptr.trace_f);
  dev(CK_TRACE_E, B * h->hp.trace_cap * 4, h->ptr.trace_e);
  dev(CK_MT_POL, B * 312 * 8, h->ptr.mt_pol);
  if (h->ptr.mt_agt) dev(CK_MT_AGT, B * 312 * 8, h->ptr.mt_agt);
  dev(CK_COUNTERS, 8 * 8, h->ptr.counters);
  dev(CK_READY, B * 4, h->ptr.ready);
  dev(CK_READY_COUNT, (size_t)2 * RLM_LIVE_OFF * 4, h->ptr.ready_count);
  if (R > 0) {
    dev(CK_RECORDS, R * h->hp.record_cap * sizeof(rlm_step_record), h->ptr.records);
    dev(CK_RECORD_COUNT, R * 4, h->ptr.record_count);
  }
  if (h->cfg.source == RLM_SOURCE_TAPE) {
    dev(CK_TAPE_CUR, B * sizeof(int2), h->ptr.tape_cur);
    dev(CK_TAPE_LO, B * 4, h->ptr.tape_lo);
    host(CK_ENV_DAY, B * 4, v.env_day);
    host(CK_DAY_OFF, ((size_t)v.n_days + 1) * 8, v.day_off);
    if (v.n_markets > 0) {
      host(CK_DAY_MARKET, (size_t)v.n_days * 4, v.day_market);
      dev(CK_MARKETS, (size_t)v.n_markets * sizeof(VenueD), v.markets);
    }
    if (v.has_env_market) {
      host(CK_ENV_MARKET, B * 4, v.env_mkt);
      if (R > 0) dev(CK_REC_FIXED, R * 4, v.rec_fixed);
    }
  }
  if (v.mlog_cap > 0) {
    dev(CK_MLOG_ACC, B * sizeof(ModelLogAcc), v.mlog.acc);
    dev(CK_MLOG_WRITTEN, B * 8, v.mlog.written);
    dev(CK_MLOG_ROWS, B * (size_t)v.mlog_cap * 8, v.mlog.rows);
  }
  return r;
}
static CkView ck_view_of(rlm_handle h) {
  CkView v = {};
  v.mlog_cap = h->mlog.cap; v.mlog = h->mlog;
  v.n_days = h->cfg.source == RLM_SOURCE_TAPE ? (int)h->day_off.size() - 1 : 0;
  v.n_markets = h->dm.markets ? h->n_markets : 0;
  v.has_env_market = h->dm.env_market != nullptr;
  v.markets = (VenueD*)h->dm.markets; v.rec_fixed = h->dm.rec_fixed;
  v.env_day = h->env_day.data(); v.day_off = h->day_off.data(); v.day_market = h->day_market.data(); v.env_mkt = h->env_mkt.data();
  return v;
}

// the weight arrays ([n][M] tables each) and the chunks they are packed in: whole tables, or slices of one table that is
// larger than a chunk
struct CkArr { uint32_t id; double* base; int n; };
struct CkChunk { int arr, t0, nt; long long lo, len; };
static std::vector<CkArr> ck_arrays(rlm_handle h) {
  std::vector<CkArr> a;
  a.push_back({CK_THETA, h->ptr.theta, h->n_policies});
  if (h->ptr.theta_b) a.push_back({CK_THETA_B, h->ptr.theta_b, h->n_policies});
  if (h->ptr.dtheta) a.push_back({CK_DTHETA, h->ptr.dtheta, h->hp.is_double ? 2 : 1});
  return a;
}
static std::vector<CkChunk> ck_chunks(const std::vector<CkArr>& arrs, long long M) {
  std::vector<CkChunk> c;
  for (int a = 0; a < (int)arrs.size(); ++a) {
    if (M <= RLM_CK_CHUNK) {
      const int per = (int)std::min<long long>(RLM_CK_CHUNK / M, RLM_CK_MAX_TABLES);
      for (int t = 0; t < arrs[a].n; t += per) c.push_back({a, t, std::min(per, arrs[a].n - t), 0, M});
    } else {
      for (int t = 0; t < arrs[a].n; ++t)
        for (long long lo = 0; lo < M; lo += RLM_CK_CHUNK) c.push_back({a, t, 1, lo, std::min(RLM_CK_CHUNK, M - lo)});
    }
  }
  return c;
}

// two device and two pinned chunk buffers, the copy stream and the events of the pipeline; freed when it goes out of scope
struct CkScratch {
  CkChunkDev d[2] = {};
  unsigned char* dmem[2] = {};
  unsigned char* hmem[2] = {};
  double* h_vals[2] = {};
  unsigned* h_bits[2] = {};
  long long* h_cnt[2] = {};
  long long* h_expect[2] = {};
  int* h_err = nullptr;
  unsigned long long* d_fp = nullptr;
  size_t words = 0, bit_bytes = 0, pinned = 0;
  cudaStream_t cs = nullptr;
  cudaEvent_t ev_a[2] = {}, ev_b[2] = {};
  ~CkScratch() {
    if (cs) { cudaStreamSynchronize(cs); cudaStreamDestroy(cs); }
    for (int b = 0; b < 2; ++b) {
      if (ev_a[b]) cudaEventDestroy(ev_a[b]);
      if (ev_b[b]) cudaEventDestroy(ev_b[b]);
      cudaFree(dmem[b]);
      if (hmem[b]) cudaFreeHost(hmem[b]);
    }
    cudaFree(d_fp);
    if (h_err) cudaFreeHost(h_err);
  }
};
static size_t ck_al(size_t x) { return (x + 255) & ~(size_t)255; }
static int ck_scratch(rlm_handle h, CkScratch& s, const std::vector<CkChunk>& ch) {
  size_t words = 1, bits = 1, blocks = 1, nt = 1;
  for (const CkChunk& c : ch) {
    words = std::max(words, (size_t)(c.nt * c.len));
    bits = std::max(bits, (size_t)(c.nt * ck_bw(c.len)));
    blocks = std::max(blocks, (size_t)(c.nt * ck_bpt(c.len)));
    nt = std::max(nt, (size_t)c.nt);
  }
  s.words = words;
  s.bit_bytes = bits * 4;
  const size_t dbytes = ck_al(words * 8) + ck_al(bits * 4) + ck_al(blocks * 4) + ck_al((blocks + 1) * 8) + 2 * ck_al(nt * 8) + 256;
  s.pinned = ck_al(words * 8) + ck_al(bits * 4) + 2 * ck_al(nt * 8);
  CK(cudaStreamCreateWithFlags(&s.cs, cudaStreamNonBlocking));
  CK(cudaMalloc(&s.d_fp, 8));
  CK(cudaMallocHost(&s.h_err, 2 * sizeof(int)));
  for (int b = 0; b < 2; ++b) {
    CK(cudaEventCreateWithFlags(&s.ev_a[b], cudaEventDisableTiming));
    CK(cudaEventCreateWithFlags(&s.ev_b[b], cudaEventDisableTiming));
    CK(cudaMalloc(&s.dmem[b], dbytes));
    CK(cudaMallocHost(&s.hmem[b], s.pinned));
    unsigned char* p = s.dmem[b];
    s.d[b].vals = (double*)p; p += ck_al(words * 8);
    s.d[b].bits = (unsigned*)p; p += ck_al(bits * 4);
    s.d[b].blk_cnt = (int*)p; p += ck_al(blocks * 4);
    s.d[b].off = (long long*)p; p += ck_al((blocks + 1) * 8);
    s.d[b].cnt = (long long*)p; p += ck_al(nt * 8);
    s.d[b].expect = (long long*)p; p += ck_al(nt * 8);
    s.d[b].err = (int*)p;
    unsigned char* q = s.hmem[b];
    s.h_vals[b] = (double*)q; q += ck_al(words * 8);
    s.h_bits[b] = (unsigned*)q; q += ck_al(bits * 4);
    s.h_cnt[b] = (long long*)q; q += ck_al(nt * 8);
    s.h_expect[b] = (long long*)q;
    CK(cudaMemsetAsync(s.d[b].err, 0, sizeof(int), h->stream));
  }
  return RLM_OK;
}

static bool ck_pwrite(int fd, const void* p, size_t n, uint64_t off) {
  const char* c = (const char*)p;
  while (n > 0) {
    const ssize_t w = pwrite(fd, c, n, (off_t)off);
    if (w <= 0) return false;
    c += w; n -= (size_t)w; off += (uint64_t)w;
  }
  return true;
}
static bool ck_pread(int fd, void* p, size_t n, uint64_t off) {
  char* c = (char*)p;
  while (n > 0) {
    const ssize_t r = pread(fd, c, n, (off_t)off);
    if (r <= 0) return false;
    c += r; n -= (size_t)r; off += (uint64_t)r;
  }
  return true;
}
static int ck_io_fail(const char* what, const char* path) {
  return fail(RLM_ERR_RUNTIME, std::string(what) + " " + path + ": " + strerror(errno));
}

// raw device sections pass through pinned buffer 0
static int ck_raw_save(rlm_handle h, int fd, CkScratch& s, const CkRaw& r, uint64_t off, const char* path) {
  if (r.host) return ck_pwrite(fd, r.host, r.bytes, off) ? RLM_OK : ck_io_fail("rlm_save: cannot write", path);
  for (size_t done = 0; done < r.bytes;) {
    const size_t n = std::min(s.pinned, r.bytes - done);
    CK(cudaMemcpyAsync(s.hmem[0], (const unsigned char*)r.dev + done, n, cudaMemcpyDeviceToHost, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    if (!ck_pwrite(fd, s.hmem[0], n, off + done)) return ck_io_fail("rlm_save: cannot write", path);
    done += n;
  }
  return RLM_OK;
}
static int ck_raw_load(rlm_handle h, int fd, CkScratch& s, const CkRaw& r, uint64_t off, const char* path) {
  for (size_t done = 0; done < r.bytes;) {
    const size_t n = std::min(s.pinned, r.bytes - done);
    if (!ck_pread(fd, s.hmem[0], n, off + done)) return ck_io_fail("rlm_load: cannot read", path);
    CK(cudaMemcpyAsync((unsigned char*)r.dev + done, s.hmem[0], n, cudaMemcpyHostToDevice, h->stream));
    CK(cudaStreamSynchronize(h->stream));
    done += n;
  }
  return RLM_OK;
}

// Pack every table and write it from file offset *pos on; secs gets one section per table.  Chunk c packs into buffers
// c & 1 on the handle's stream while the copy stream brings chunk c - 1 to the host and the host writes chunk c - 2.
static int ck_tables_save(rlm_handle h, int fd, CkScratch& s, const std::vector<CkArr>& arrs, const std::vector<CkChunk>& ch,
                          uint64_t* pos, std::vector<CkSection>& secs, const char* path) {
  const long long M = h->cfg.memory_size, bmb = (M + 7) / 8;
  const size_t C = ch.size();
  CkSection cur = {};
  std::vector<long long> cnt[2];
  for (size_t c = 0; c <= C; ++c) {
    const int b = (int)(c & 1);
    if (c < C) {
      const CkChunk& k = ch[c];
      if (c >= 2) CK(cudaStreamWaitEvent(h->stream, s.ev_b[b], 0));  // (the copy of chunk c - 2 out of these buffers)
      CK(rlm_launch_pack(s.d[b], arrs[k.arr].base + (size_t)k.t0 * M + k.lo, M, k.nt, k.len, h->stream));
      CK(cudaMemcpyAsync(s.h_cnt[b], s.d[b].cnt, (size_t)k.nt * 8, cudaMemcpyDeviceToHost, h->stream));
      CK(cudaEventRecord(s.ev_a[b], h->stream));
    }
    if (c >= 1) {  // write chunk c - 1
      const int pb = b ^ 1;
      const CkChunk& k = ch[c - 1];
      CK(cudaEventSynchronize(s.ev_b[pb]));
      const long long bw = ck_bw(k.len);
      long long v0 = 0;
      for (int t = 0; t < k.nt; ++t) {
        if (k.lo == 0) cur = {arrs[k.arr].id, (uint32_t)(k.t0 + t), *pos, 0, 0};
        const long long n = cnt[pb][t];
        if (!ck_pwrite(fd, s.h_bits[pb] + (size_t)t * bw, (size_t)((k.len + 7) / 8), cur.offset + k.lo / 8) ||
            !ck_pwrite(fd, s.h_vals[pb] + v0, (size_t)n * 8, cur.offset + bmb + 8 * cur.count))
          return ck_io_fail("rlm_save: cannot write", path);
        v0 += n;
        cur.count += n;
        if (k.lo + k.len == M) {
          cur.bytes = bmb + 8 * cur.count;
          *pos = cur.offset + cur.bytes;
          secs.push_back(cur);
        }
      }
    }
    if (c < C) {  // the counts of chunk c size its copy
      const CkChunk& k = ch[c];
      CK(cudaEventSynchronize(s.ev_a[b]));
      cnt[b].assign(s.h_cnt[b], s.h_cnt[b] + k.nt);
      long long tot = 0;
      for (long long n : cnt[b]) tot += n;
      CK(cudaStreamWaitEvent(s.cs, s.ev_a[b], 0));
      CK(cudaMemcpyAsync(s.h_bits[b], s.d[b].bits, (size_t)(k.nt * ck_bw(k.len)) * 4, cudaMemcpyDeviceToHost, s.cs));
      if (tot) CK(cudaMemcpyAsync(s.h_vals[b], s.d[b].vals, (size_t)tot * 8, cudaMemcpyDeviceToHost, s.cs));
      CK(cudaEventRecord(s.ev_b[b], s.cs));
    }
  }
  return RLM_OK;
}

// Read every table back.  pass 1 (count_only): only the bitmaps go to the device, and sub[c][t] gets the population of
// chunk c's table t (the caller checks it against the stored counts).  pass 2: bitmaps and values, unpacked into the
// arrays; the scan checks each table against sub and the unpack kernel writes nothing on a mismatch.  The host reads
// chunk c + 1 while the copy stream uploads chunk c and the handle's stream unpacks it.
static int ck_tables_load(rlm_handle h, int fd, CkScratch& s, const std::vector<CkArr>& arrs, const std::vector<CkChunk>& ch,
                          const std::vector<const CkSection*>& sec_of, std::vector<std::vector<long long>>& sub, int count_only,
                          const char* path) {
  const long long M = h->cfg.memory_size, bmb = (M + 7) / 8;
  const size_t C = ch.size();
  std::vector<int> first(arrs.size() + 1, 0);  // section index of table 0 of each array
  for (size_t a = 0; a < arrs.size(); ++a) first[a + 1] = first[a] + arrs[a].n;
  std::vector<long long> run(sec_of.size(), 0);  // values read so far of each table (slices)
  if (count_only) sub.assign(C, {});
  for (size_t c = 0; c <= C; ++c) {
    const int b = (int)(c & 1);
    if (c < C) {
      const CkChunk& k = ch[c];
      if (c >= 2) CK(cudaEventSynchronize(s.ev_b[b]));  // chunk c - 2 is done with these buffers
      const long long bw = ck_bw(k.len);
      long long v0 = 0;
      for (int t = 0; t < k.nt; ++t) {
        const int si = first[k.arr] + k.t0 + t;
        const CkSection& sc = *sec_of[si];
        const size_t nb = (size_t)((k.len + 7) / 8);
        unsigned char* bits = (unsigned char*)(s.h_bits[b] + (size_t)t * bw);
        memset(bits + nb, 0, (size_t)bw * 4 - nb);
        if (!ck_pread(fd, bits, nb, sc.offset + k.lo / 8)) return ck_io_fail("rlm_load: cannot read", path);
        if (!count_only) {
          const long long n = sub[c][t];
          if (!ck_pread(fd, s.h_vals[b] + v0, (size_t)n * 8, sc.offset + bmb + 8 * run[si])) return ck_io_fail("rlm_load: cannot read", path);
          s.h_expect[b][t] = n;
          run[si] += n;
          v0 += n;
        }
      }
      CK(cudaMemcpyAsync(s.d[b].bits, s.h_bits[b], (size_t)(k.nt * bw) * 4, cudaMemcpyHostToDevice, s.cs));
      if (!count_only) {
        CK(cudaMemcpyAsync(s.d[b].expect, s.h_expect[b], (size_t)k.nt * 8, cudaMemcpyHostToDevice, s.cs));
        if (v0) CK(cudaMemcpyAsync(s.d[b].vals, s.h_vals[b], (size_t)v0 * 8, cudaMemcpyHostToDevice, s.cs));
      }
      CK(cudaEventRecord(s.ev_a[b], s.cs));
      CK(cudaStreamWaitEvent(h->stream, s.ev_a[b], 0));
      CK(rlm_launch_unpack(s.d[b], arrs[k.arr].base + (size_t)k.t0 * M + k.lo, M, k.nt, k.len, count_only, h->stream));
      if (count_only) CK(cudaMemcpyAsync(s.h_cnt[b], s.d[b].cnt, (size_t)k.nt * 8, cudaMemcpyDeviceToHost, h->stream));
      CK(cudaEventRecord(s.ev_b[b], h->stream));
    }
    if (c >= 1 && count_only) {
      CK(cudaEventSynchronize(s.ev_b[b ^ 1]));
      sub[c - 1].assign(s.h_cnt[b ^ 1], s.h_cnt[b ^ 1] + ch[c - 1].nt);
    }
  }
  CK(cudaStreamSynchronize(h->stream));
  for (int b = 0; b < 2; ++b) CK(cudaMemcpy(s.h_err + b, s.d[b].err, sizeof(int), cudaMemcpyDeviceToHost));
  return RLM_OK;
}

static int ck_library_fp(rlm_handle h, CkScratch& s, uint64_t* fp) {
  const long long words = h->day_off.back() * (long long)sizeof(rlm_tick_msg) / 8;
  CK(rlm_launch_fingerprint(h->ptr.tape, words, s.d_fp, h->n_sms, h->stream));
  CK(cudaMemcpyAsync(fp, s.d_fp, 8, cudaMemcpyDeviceToHost, h->stream));
  CK(cudaStreamSynchronize(h->stream));
  return RLM_OK;
}

// the config with the fields a loading handle may differ in (and the struct's padding) cleared
static rlm_config ck_norm(const rlm_config& in) {
  rlm_config c = in;
  c.device = 0;
  memset(&c.flow, 0, sizeof(c.flow));
  const size_t g1 = offsetof(rlm_config, lb_vwap) + sizeof(c.lb_vwap), g2 = offsetof(rlm_config, random_seed) + sizeof(c.random_seed);
  memset((char*)&c + g1, 0, offsetof(rlm_config, pos_lb) - g1);
  memset((char*)&c + g2, 0, offsetof(rlm_config, flow) - g2);
  return c;
}

static const char* const k_ck_engine = "checkpoints need the tick-synchronous or round-paced engine (RLM_ENGINE=F|f|p run every step inside one launch)";

int rlm_save(rlm_handle h, const char* path) {
  API_LOCK;
  if (!h || !path) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_save: null argument");
  if (h->engine != 1) return fail(RLM_ERR_UNSUPPORTED, std::string("rlm_save: ") + k_ck_engine);
  if (h->cfg.source == RLM_SOURCE_STREAM && h->stream_cursor < h->stream_ticks)
    return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_save: " + std::to_string(h->stream_ticks - h->stream_cursor) +
                                              " uploaded ticks are not consumed yet (run them, then save; upload the next ticks after rlm_load)");
  int rc = tape_check(h);
  if (rc) return rc;
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  rc = fix_records(h);
  if (rc) return rc;
  const CkView v = ck_view_of(h);
  const std::vector<CkRaw> raw = ck_raw(h, v);
  const std::vector<CkArr> arrs = ck_arrays(h);
  const std::vector<CkChunk> ch = ck_chunks(arrs, h->cfg.memory_size);
  int n_tables = 0;
  for (const CkArr& a : arrs) n_tables += a.n;
  CkScratch s;
  rc = ck_scratch(h, s, ch);
  if (rc) return rc;
  CkHeader hd;
  memset(&hd, 0, sizeof(hd));
  memcpy(hd.magic, "RLMCKPT", 8);
  hd.version = RLM_CK_VERSION;
  hd.n_sections = (uint32_t)(raw.size() + n_tables);
  hd.header_bytes = (uint32_t)(sizeof(CkHeader) + hd.n_sections * sizeof(CkSection));
  hd.env_stride = (uint32_t)h->hp.env_stride;
  hd.env_hdr_bytes = (uint32_t)sizeof(EnvHdr);
  hd.model_log_cap = v.mlog_cap;
  memcpy(&hd.cfg, &h->cfg, sizeof(rlm_config));
  hd.alpha = h->alpha; hd.eps = h->eps; hd.tau = h->tau;
  hd.launches = h->launches;
  hd.run_seq = h->run_seq; hd.greedy = h->dyn.greedy; hd.backtest = h->dyn.backtest;
  hd.n_days = v.n_days; hd.n_markets = v.n_markets; hd.has_env_market = v.has_env_market;
  memcpy(&hd.shared_dyn, &h->shared_dyn, sizeof(DynParams));
  if (h->cfg.source == RLM_SOURCE_TAPE) {
    rc = ck_library_fp(h, s, &hd.library_fp);
    if (rc) return rc;
  }
  const int fd = open(path, O_WRONLY | O_CREAT | O_TRUNC, 0644);
  if (fd < 0) return fail(RLM_ERR_INVALID_ARGUMENT, std::string("rlm_save: cannot create ") + path + ": " + strerror(errno));
  std::vector<CkSection> secs;
  uint64_t pos = hd.header_bytes;
  for (const CkRaw& r : raw) {
    secs.push_back({r.id, 0, pos, r.bytes, 0});
    rc = ck_raw_save(h, fd, s, r, pos, path);
    if (rc) break;
    pos += r.bytes;
  }
  if (!rc) rc = ck_tables_save(h, fd, s, arrs, ch, &pos, secs, path);
  if (!rc) {
    hd.file_bytes = pos;
    if (!ck_pwrite(fd, &hd, sizeof(hd), 0) || !ck_pwrite(fd, secs.data(), secs.size() * sizeof(CkSection), sizeof(hd)))
      rc = ck_io_fail("rlm_save: cannot write", path);
  }
  if (close(fd) != 0 && !rc) rc = ck_io_fail("rlm_save: cannot close", path);
  if (rc) unlink(path);  // (no partial checkpoint is left behind)
  return rc;
}

int rlm_load(rlm_handle h, const char* path) {
  API_LOCK;
  if (!h || !path) return fail(RLM_ERR_INVALID_ARGUMENT, "rlm_load: null argument");
  if (h->engine != 1) return fail(RLM_ERR_UNSUPPORTED, std::string("rlm_load: ") + k_ck_engine);
  const std::string P = std::string("rlm_load: ") + path + ": ";
  const int fd = open(path, O_RDONLY);
  if (fd < 0) return fail(RLM_ERR_INVALID_ARGUMENT, P + strerror(errno));
  struct Closer { int fd; ~Closer() { close(fd); } } closer{fd};
  struct stat st;
  if (fstat(fd, &st) != 0) return fail(RLM_ERR_INVALID_ARGUMENT, P + strerror(errno));
  const uint64_t size = (uint64_t)st.st_size;
  // ---- everything is checked before anything of the handle changes
  CkHeader hd;
  if (size < sizeof(hd) || !ck_pread(fd, &hd, sizeof(hd), 0)) return fail(RLM_ERR_INVALID_ARGUMENT, P + "truncated header");
  if (memcmp(hd.magic, "RLMCKPT", 8) != 0) return fail(RLM_ERR_INVALID_ARGUMENT, P + "not a checkpoint (bad magic)");
  if (hd.version != RLM_CK_VERSION || hd.env_hdr_bytes != sizeof(EnvHdr))
    return fail(RLM_ERR_INVALID_ARGUMENT, P + "layout version " + std::to_string(hd.version) + " / env header " + std::to_string(hd.env_hdr_bytes) +
                                              " bytes; this library writes " + std::to_string(RLM_CK_VERSION) + " / " + std::to_string(sizeof(EnvHdr)));
  if (hd.file_bytes != size) return fail(RLM_ERR_INVALID_ARGUMENT, P + "the file holds " + std::to_string(size) + " bytes, its header says " +
                                                                       std::to_string(hd.file_bytes) + " (truncated?)");
  {
    const rlm_config a = ck_norm(hd.cfg), b = ck_norm(h->cfg);
    if (memcmp(&a, &b, sizeof(a)) != 0 || hd.env_stride != (uint32_t)h->hp.env_stride)
      return fail(RLM_ERR_INVALID_ARGUMENT, P + "the handle's config differs from the saved one (every field but device and flow must match)");
  }
  const bool tape = h->cfg.source == RLM_SOURCE_TAPE;
  if (hd.model_log_cap < 0 || hd.model_log_cap > INT_MAX || hd.n_days < 0 || hd.n_markets < 0 || (hd.has_env_market & ~1) ||
      (!tape && (hd.n_days || hd.n_markets || hd.has_env_market)))
    return fail(RLM_ERR_INVALID_ARGUMENT, P + "corrupt header");
  if (tape) {
    int rc = tape_check(h);
    if (rc) return rc;
    if (hd.n_days != (int)h->day_off.size() - 1)
      return fail(RLM_ERR_INVALID_ARGUMENT, P + "saved with a library of " + std::to_string(hd.n_days) + " days, the handle holds " +
                                                std::to_string(h->day_off.size() - 1) + " (rlm_load_days the same library first)");
  }
  const int B = h->cfg.n_envs;
  std::vector<int32_t> env_day(tape ? B : 0), day_market(hd.n_markets > 0 ? hd.n_days : 0), env_mkt(hd.has_env_market ? B : 0);
  std::vector<int64_t> day_off(tape ? hd.n_days + 1 : 0);
  CkView v = {};
  v.mlog_cap = hd.model_log_cap; v.n_days = hd.n_days; v.n_markets = hd.n_markets; v.has_env_market = hd.has_env_market;
  v.env_day = env_day.data(); v.day_off = day_off.data(); v.day_market = day_market.data(); v.env_mkt = env_mkt.data();
  const std::vector<CkRaw> raw0 = ck_raw(h, v);
  const std::vector<CkArr> arrs = ck_arrays(h);
  const std::vector<CkChunk> ch = ck_chunks(arrs, h->cfg.memory_size);
  const long long M = h->cfg.memory_size, bmb = (M + 7) / 8;
  size_t n_tables = 0;
  for (const CkArr& a : arrs) n_tables += a.n;
  if (hd.n_sections != raw0.size() + n_tables || hd.header_bytes != sizeof(CkHeader) + hd.n_sections * sizeof(CkSection))
    return fail(RLM_ERR_INVALID_ARGUMENT, P + "the section table does not fit the handle's config");
  std::vector<CkSection> secs(hd.n_sections);
  if (!ck_pread(fd, secs.data(), secs.size() * sizeof(CkSection), sizeof(hd))) return fail(RLM_ERR_INVALID_ARGUMENT, P + "truncated section table");
  {
    uint64_t pos = hd.header_bytes;
    size_t i = 0;
    for (const CkRaw& r : raw0) {
      const CkSection& sc = secs[i++];
      if (sc.id != r.id || sc.offset != pos || sc.bytes != r.bytes) return fail(RLM_ERR_INVALID_ARGUMENT, P + "section " + std::to_string(i - 1) + " does not fit the handle");
      pos += sc.bytes;
    }
    for (const CkArr& a : arrs)
      for (int t = 0; t < a.n; ++t) {
        const CkSection& sc = secs[i++];
        if (sc.id != a.id || sc.table != (uint32_t)t || sc.offset != pos || sc.count > (uint64_t)M || sc.bytes != (uint64_t)bmb + 8 * sc.count)
          return fail(RLM_ERR_INVALID_ARGUMENT, P + "packed table section " + std::to_string(i - 1) + " is malformed");
        pos += sc.bytes;
      }
    if (pos != size) return fail(RLM_ERR_INVALID_ARGUMENT, P + "the sections do not add up to the file's length");
  }
  for (size_t i = 0; i < raw0.size(); ++i)  // host sections: small, read now and checked
    if (raw0[i].host && !ck_pread(fd, raw0[i].host, raw0[i].bytes, secs[i].offset)) return fail(RLM_ERR_INVALID_ARGUMENT, P + "cannot read");
  if (tape) {
    if (day_off != h->day_off) return fail(RLM_ERR_INVALID_ARGUMENT, P + "the handle's day library has other day offsets than the saved one");
    for (int32_t d : env_day) if (d < 0 || d >= hd.n_days) return fail(RLM_ERR_INVALID_ARGUMENT, P + "corrupt day assignment");
    for (int32_t k : day_market) if (k < 0 || k >= hd.n_markets) return fail(RLM_ERR_INVALID_ARGUMENT, P + "corrupt day markets");
    for (int32_t k : env_mkt) if (k < -1 || k >= hd.n_markets) return fail(RLM_ERR_INVALID_ARGUMENT, P + "corrupt env markets");
  }
  CK(cudaSetDevice(h->cfg.device));
  CK(cudaStreamSynchronize(h->stream));
  CkScratch s;
  int rc = ck_scratch(h, s, ch);
  if (rc) return rc;
  if (tape) {
    uint64_t fp = 0;
    rc = ck_library_fp(h, s, &fp);
    if (rc) return rc;
    if (fp != hd.library_fp) return fail(RLM_ERR_INVALID_ARGUMENT, P + "the handle's day library differs from the saved one (fingerprint)");
  }
  std::vector<const CkSection*> sec_of;
  for (size_t i = raw0.size(); i < secs.size(); ++i) sec_of.push_back(&secs[i]);
  std::vector<std::vector<long long>> sub;
  rc = ck_tables_load(h, fd, s, arrs, ch, sec_of, sub, 1, path);
  if (rc) return rc;
  {
    std::vector<long long> tot(sec_of.size(), 0);
    std::vector<int> first(arrs.size() + 1, 0);
    for (size_t a = 0; a < arrs.size(); ++a) first[a + 1] = first[a] + arrs[a].n;
    for (size_t c = 0; c < ch.size(); ++c)
      for (int t = 0; t < ch[c].nt; ++t) tot[first[ch[c].arr] + ch[c].t0 + t] += sub[c][t];
    bool bad = s.h_err[0] || s.h_err[1];
    for (size_t i = 0; i < tot.size(); ++i) bad = bad || tot[i] != (long long)sec_of[i]->count;
    if (bad) return fail(RLM_ERR_INVALID_ARGUMENT, P + "corrupt packed table (bitmap population differs from the stored value count)");
  }
  // ---- the new buffers, before anything is replaced
  ModelLogPtrs L = {};
  VenueD* d_markets = nullptr;
  int *d_env_market = nullptr, *d_rec_fixed = nullptr;
  {
    cudaError_t ce = cudaSuccess;
    if (hd.model_log_cap > 0) {
      L.cap = hd.model_log_cap;
      ce = cudaMalloc(&L.acc, (size_t)B * sizeof(ModelLogAcc));
      if (ce == cudaSuccess) ce = cudaMalloc(&L.written, (size_t)B * 8);
      if (ce == cudaSuccess) ce = cudaMalloc(&L.rows, (size_t)B * (size_t)L.cap * 8);
    }
    if (ce == cudaSuccess && hd.n_markets > 0) ce = cudaMalloc(&d_markets, (size_t)hd.n_markets * sizeof(VenueD));
    if (ce == cudaSuccess && hd.has_env_market && !h->dm.env_market) {
      ce = cudaMalloc(&d_env_market, (size_t)B * sizeof(int));
      if (ce == cudaSuccess && h->hp.record_envs > 0) ce = cudaMalloc(&d_rec_fixed, (size_t)h->hp.record_envs * sizeof(int));
    }
    if (ce != cudaSuccess) {
      cudaFree(L.acc); cudaFree(L.written); cudaFree(L.rows); cudaFree(d_markets); cudaFree(d_env_market); cudaFree(d_rec_fixed);
      CK(ce);
    }
  }
  // ---- commit
  drop_graphs(h);
  h->graph_warm = false;
  cudaFree(h->mlog.acc); cudaFree(h->mlog.written); cudaFree(h->mlog.rows);
  h->mlog = L;
  cudaFree((void*)h->dm.markets);
  h->dm.markets = d_markets;
  h->n_markets = hd.n_markets;
  if (!hd.has_env_market) {
    cudaFree(h->dm.env_market); cudaFree(h->dm.rec_fixed);
    h->dm.env_market = nullptr; h->dm.rec_fixed = nullptr;
  } else if (d_env_market) {
    h->dm.env_market = d_env_market; h->dm.rec_fixed = d_rec_fixed;
  }
  h->env_day = env_day; h->day_market = day_market; h->env_mkt = env_mkt;
  v = ck_view_of(h);
  const std::vector<CkRaw> raw = ck_raw(h, v);
  for (size_t i = 0; i < raw.size() && !rc; ++i)
    if (raw[i].dev) rc = ck_raw_load(h, fd, s, raw[i], secs[i].offset, path);
  if (!rc && hd.has_env_market) {
    CK(cudaMemcpy(h->dm.env_market, h->env_mkt.data(), (size_t)B * sizeof(int), cudaMemcpyHostToDevice));
  }
  if (!rc) rc = ck_tables_load(h, fd, s, arrs, ch, sec_of, sub, 0, path);
  if (!rc && (s.h_err[0] || s.h_err[1])) rc = fail(RLM_ERR_RUNTIME, P + "the file changed while it was loaded; the handle's state is undefined");
  if (rc) return rc;
  h->alpha = hd.alpha; h->eps = hd.eps; h->tau = hd.tau;
  h->launches = hd.launches;
  h->run_seq = hd.run_seq;
  h->dyn.greedy = hd.greedy; h->dyn.backtest = hd.backtest;
  memcpy(&h->shared_dyn, &hd.shared_dyn, sizeof(DynParams));
  memcpy(&h->cfg.flow, &hd.cfg.flow, sizeof(rlm_flow_params));
  h->hp.flow = h->cfg.flow;
  h->rec_dirty = false;
  h->stream_ticks = 0; h->stream_cursor = 0;
  day_markets_on(h, h->dm.markets != nullptr);  // (and the parameters are uploaded again before the next launch)
  return RLM_OK;
}
