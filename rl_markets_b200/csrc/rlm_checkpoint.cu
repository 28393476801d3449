// rlm_checkpoint.cu -- the device side of rlm_save / rlm_load (include/rlm.h): packing and unpacking weight tables, and
// the fingerprint of a tape day library.
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
#include "rlm_kernels.h"

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

static int ck_bpt(long long len) { return (int)((len + RLM_CK_TILE - 1) / RLM_CK_TILE); }

cudaError_t rlm_launch_pack(const CkChunkDev& c, const double* src, long long tstride, int nt, long long len, cudaStream_t st) {
  const int bpt = ck_bpt(len), n = nt * bpt;
  const long long bw = (len + 31) / 32;
  rlm_pack_count_kernel<<<n, CK_WARPS * 32, 0, st>>>((const unsigned long long*)src, tstride, len, bpt, bw, c.bits, c.blk_cnt);
  rlm_ck_scan_kernel<<<1, 1024, 0, st>>>(c.blk_cnt, n, bpt, nt, c.off, c.cnt, nullptr, c.err);
  rlm_pack_kernel<<<n, CK_WARPS * 32, 0, st>>>((const unsigned long long*)src, tstride, len, bpt, bw, c.bits, c.off,
                                               (unsigned long long*)c.vals);
  return cudaGetLastError();
}

cudaError_t rlm_launch_unpack(const CkChunkDev& c, double* dst, long long tstride, int nt, long long len, int count_only, cudaStream_t st) {
  const int bpt = ck_bpt(len), n = nt * bpt;
  const long long bw = (len + 31) / 32;
  rlm_unpack_count_kernel<<<n, CK_WARPS * 32, 0, st>>>(c.bits, len, bpt, bw, c.blk_cnt, c.err);
  rlm_ck_scan_kernel<<<1, 1024, 0, st>>>(c.blk_cnt, n, bpt, nt, c.off, c.cnt, count_only ? nullptr : c.expect, c.err);
  if (!count_only)
    rlm_unpack_kernel<<<n, CK_WARPS * 32, 0, st>>>(c.bits, len, bpt, bw, c.off, (const unsigned long long*)c.vals, (unsigned long long*)dst,
                                                   tstride, c.err);
  return cudaGetLastError();
}

cudaError_t rlm_launch_fingerprint(const void* data, long long n_words, unsigned long long* out, int n_sms, cudaStream_t st) {
  cudaError_t e = cudaMemsetAsync(out, 0, 8, st);
  if (e != cudaSuccess || n_words <= 0) return e;
  const long long want = (n_words + 255) / 256;
  const int grid = (int)(want < (long long)n_sms * 8 ? want : (long long)n_sms * 8);
  rlm_fingerprint_kernel<<<grid, 256, 0, st>>>((const unsigned long long*)data, n_words, out);
  return cudaGetLastError();
}
