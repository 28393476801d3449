// rlm_model_log.cu -- the reference's model_log (Agent::HandleTransition, src/rl/agent.cpp:86-101) on the device.
//
// The learner kernels leave each env's TD error of its last transition in AgentD::last_delta and count its updates in
// AgentD::n_steps.  One pass of rlm_model_log_kernel after a training learner launch folds the new update of every env
// into its own accumulator, exactly as HandleTransition does it:
//   _agg_delta += abs(delta);  if (++_update_counter % 1000 == 0) { log(_agg_delta / 1000); _agg_delta = 0; _update_counter = 0; }
// Every learner launch completes at most one step per env, so one pass per launch sees every delta, in the env's own
// step order.  A jump of more than one step (or a step count that went back) means deltas were never seen: the pass
// raises ERR_MODEL_LOG_GAP instead of logging a wrong mean.  The kernel has its own translation unit and takes every
// parameter by value (no __constant__ block), so no existing kernel changes.
#include <cuda_runtime.h>
#include "rlm_kernels.h"

__global__ void __launch_bounds__(128) rlm_model_log_kernel(ModelLogPtrs L, const unsigned char* __restrict__ env, int env_stride,
                                                            int env0, int n, unsigned long long* counters) {
  const int i = blockIdx.x * blockDim.x + threadIdx.x;
  if (i >= n) return;
  const int b = env0 + i;
  const AgentD* ag = (const AgentD*)(env + (size_t)b * env_stride + offsetof(EnvHdr, ag));
  const long long steps = ag->n_steps;
  ModelLogAcc a = L.acc[b];
  if (steps == a.seen) return;
  if (steps == a.seen + 1) {
    a.agg += fabs(ag->last_delta);
    if (++a.count == 1000) {
      const long long k = L.written[b];
      if (k < L.cap) L.rows[(size_t)b * L.cap + k] = a.agg / 1000.0;
      L.written[b] = k + 1;
      a.agg = 0.0;
      a.count = 0;
    }
  } else {
    atomicOr(&counters[4], (unsigned long long)ERR_MODEL_LOG_GAP);
  }
  a.seen = steps;
  L.acc[b] = a;
}

// seen = n_steps for every env: steps taken outside training (evaluation) neither count nor look like a gap
__global__ void __launch_bounds__(128) rlm_model_log_baseline_kernel(ModelLogPtrs L, const unsigned char* __restrict__ env,
                                                                     int env_stride, int n_envs) {
  const int b = blockIdx.x * blockDim.x + threadIdx.x;
  if (b >= n_envs) return;
  L.acc[b].seen = ((const AgentD*)(env + (size_t)b * env_stride + offsetof(EnvHdr, ag)))->n_steps;
}

cudaError_t rlm_launch_model_log(const ModelLogPtrs& L, const DevPtrs& ptr, int env_stride, int env0, int n, cudaStream_t st) {
  if (n <= 0) return cudaSuccess;
  rlm_model_log_kernel<<<(n + 127) / 128, 128, 0, st>>>(L, ptr.env, env_stride, env0, n, ptr.counters);
  return cudaGetLastError();
}

cudaError_t rlm_launch_model_log_baseline(const ModelLogPtrs& L, const DevPtrs& ptr, int env_stride, int n_envs, cudaStream_t st) {
  rlm_model_log_baseline_kernel<<<(n_envs + 127) / 128, 128, 0, st>>>(L, ptr.env, env_stride, n_envs);
  return cudaGetLastError();
}
