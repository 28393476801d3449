// rlm_kernels.h -- launch wrappers implemented in rlm_kernels.cu (host-callable).
#pragma once
#include <cuda_runtime.h>
#include "rlm_types.h"

size_t rlm_scratch_bytes(int is_double);
size_t rlm_agent_smem_bytes(int warps_per_cta, int scratch_bytes);
cudaError_t rlm_upload_params(const DevParams* p);
cudaError_t rlm_launch_env(const DevPtrs& ptr, const DynParams& D, int n_envs, int tslot, int only_begin, int variant, cudaStream_t st);
cudaError_t rlm_launch_env_round(const DevPtrs& ptr, const DynParams& D, int n_envs, int tslot, cudaStream_t st);
cudaError_t rlm_launch_runctl(const DevPtrs& ptr, const RunCtl& v, cudaStream_t st);
cudaError_t rlm_launch_agent(const DevPtrs& ptr, const DynParams& D, int n_envs, int scratch_bytes, int tslot, int n_sms, int stage, cudaStream_t st);
cudaError_t rlm_launch_agent3(const DevPtrs& ptr, const DynParams& D, int n_envs, int is_double, int occ_smem_words, int tslot, int n_sms, int stage, int full,
                              cudaStream_t st);
cudaError_t rlm_launch_learn(const DevPtrs& ptr, const DynParams& D, int n_envs, int is_double, int tslot, int n_sms, int stage, int expected_steps, cudaStream_t st);
cudaError_t rlm_launch_learn_staged(const DevPtrs& ptr, const DynParams& D, int n_envs, long long memory_size, int tslot, int n_sms, cudaStream_t st);
cudaError_t rlm_launch_fused2(const DevPtrs& ptr, const DynParams& D, int n_envs, int is_double, cudaStream_t st);
cudaError_t rlm_launch_apply_dtheta(double* theta, double* dtheta, long long n, int n_sms, cudaStream_t st);
size_t rlm_fused_smem_bytes(int is_double);
cudaError_t rlm_launch_fused(const DevPtrs& ptr, const DynParams& D, int n_envs, int is_double, cudaStream_t st);
cudaError_t rlm_launch_run(const DevPtrs& ptr, const DynParams& D, int n_envs, int scratch_bytes, int n_agent_ctas, cudaStream_t st);
#define RLM_RUN_WARPS 4  // warps per CTA of the persistent engine (rlm_run_kernel)
int rlm_run_max_resident_ctas(int scratch_bytes, int n_sms);
cudaError_t rlm_launch_act(const DevPtrs& ptr, const DynParams& D, int n_envs, int* actions, cudaStream_t st);
cudaError_t rlm_launch_apply(const DevPtrs& ptr, const DynParams& D, int n_envs, const int* actions, cudaStream_t st);
cudaError_t rlm_launch_step_out(const DevPtrs& ptr, int n_envs, double* reward, unsigned char* terminal, double* delta, cudaStream_t st);
cudaError_t rlm_launch_count_nonzero(const double* theta, long long M, int n_policies, int* out, cudaStream_t st);
cudaError_t rlm_launch_init(const DevPtrs& ptr, int n_envs, int mode, cudaStream_t st);
cudaError_t rlm_launch_seed(const DevPtrs& ptr, int n_envs, unsigned seed, cudaStream_t st);
cudaError_t rlm_launch_random_init(const DevPtrs& ptr, int n_policies, cudaStream_t st);
void rlm_set_pdl(int on);
cudaError_t rlm_launch_gather(const DevPtrs& ptr, int n_envs, int what, void* out, cudaStream_t st);
cudaError_t rlm_launch_clear_traces(const DevPtrs& ptr, int n_envs, cudaStream_t st);
cudaError_t rlm_launch_test_to_ticks(const double* px, int n, int* out);
cudaError_t rlm_launch_test_to_price(const int* t, int n, double* out);
cudaError_t rlm_launch_test_tiles(const float* vars, int n, int* out);
cudaError_t rlm_launch_test_learner_tiles(int form, const float* vars, int n, int* out);
cudaError_t rlm_launch_test_order(long long size, long long q_head, const rlm_order_op* ops, int n_ops, rlm_order_state* out);
cudaError_t rlm_launch_test_rolling_mean(const double* vals, int n, double* out, double* ring_mem, EnvHdr* e);
