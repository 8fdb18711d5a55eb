/* rexsim_agent.h -- C ABI of the device-side agent glue that sits either side of rexsim_step in a rollout
 * (SURVEY.md section 8(f) rows 1-2: the callers immediately before and after the hot path).
 *
 * The reference runs these as TensorFlow-1 graph ops around InGraphBatchEnv (rex_gym/agents/tools/simulate.py:57-76):
 *
 *   rexagent_perform            <- PPOAlgorithm.perform (rex_gym/agents/ppo/algorithm.py:105-135):
 *                                  StreamingNormalize.transform (agents/ppo/normalize.py:43-71) ->
 *                                  ForwardGaussianPolicy (agents/scripts/networks.py:66-110: policy MLP relu..relu->tanh
 *                                  mean, free logstd vector, value MLP) -> sample / mean, log-prob
 *   rexagent_experience         <- PPOAlgorithm._define_experience filter updates (algorithm.py:157-161;
 *                                  StreamingNormalize.update normalize.py:73-99) for observations and rewards
 *   rexagent_discounted_return  <- utility.discounted_return (agents/ppo/utility.py:72-82)
 *   rexagent_lambda_advantage   <- utility.lambda_advantage  (agents/ppo/utility.py:112-124)
 *   rexagent_gae_segments       <- the same two scans on a time-major [T][N] rollout with done flags (auto-reset
 *                                  batches: an episode boundary inside the buffer restarts the scan) -- ours
 *
 * The PPO learner itself (losses, Adam, KL penalty: algorithm.py:243-520) is out of scope.
 * Conventions as in rexsim.h: plain C, 0 / negative RexSimStatus, device pointers owned by the caller, everything
 * enqueued on the given stream, no host synchronisation except create / get_*.
 */
#ifndef REXSIM_AGENT_H
#define REXSIM_AGENT_H
#include <stdint.h>
#include "rexsim.h"

#ifdef __cplusplus
extern "C" {
#endif

typedef struct {
    int32_t obs_dim;            /* O <= 32 */
    int32_t action_dim;         /* A <= 8 */
    int32_t hidden1, hidden2;   /* policy_layers == value_layers == (200, 100) in every config.yaml the reference ships
                                 * (rex_gym/policies/<task>/config.yaml); hidden1 <= 256, hidden2 <= 128, both multiples of 4 */
    float observ_clip;          /* 5  (algorithm.py:49-53)  */
    float reward_clip;          /* 10 (algorithm.py:54-58) */
} RexAgentConfig;

typedef struct RexAgent RexAgent;

/* Packed parameter block (floats), TF variable order of networks.py:96-110, weights row-major [in][out] like
 * tf.contrib.layers.fully_connected:
 *   policy: W1[O][H1] b1[H1] W2[H1][H2] b2[H2] W3[H2][A] b3[A] logstd[A]   (padded with zeros to a multiple of 4 floats)
 *   value : W1[O][H1] b1[H1] W2[H1][H2] b2[H2] W3[H2][1] b3[1]             (padded likewise)                        */
int64_t rexagent_policy_floats(const RexAgentConfig* cfg);   /* padded size of the policy block */
int64_t rexagent_value_floats(const RexAgentConfig* cfg);    /* padded size of the value block  */
int rexagent_create(const RexAgentConfig* cfg, RexAgent** out);
void rexagent_destroy(RexAgent* a);
/* 0 (default): the networks in fp32 on the CUDA cores -- matches an fp32 reference to rounding.
 * 1: layer 2 (hidden1 x hidden2, 97 % of the flops) on the tensor cores: wgmma tf32 with fp32 accumulation in registers
 *    (operands rounded to 11 significant bits; error bounds in tests/test_gpu_agent.py).  Needs hidden1 % 8 == 0, obs_dim <= 16. */
int rexagent_set_precision(RexAgent* a, int32_t mode);
int rexagent_set_params(RexAgent* a, const float* host_params, int64_t n_floats);
int rexagent_get_params(RexAgent* a, float* host_params, int64_t n_floats);
/* device pointer to the packed block (a learner updates it in place) */
int rexagent_params_buffer(RexAgent* a, float** params);

/* streaming normaliser state; host arrays.  observ: count, mean[O], var_sum[O]; reward: count, mean, var_sum.
 * The counts are 64-bit: every filter update adds the whole batch, so at 65 536 envs a 32-bit count would wrap after
 * 32 768 control steps (the reference's int32 TF variable never gets near that at its 30 envs). */
int rexagent_set_filters(RexAgent* a, int64_t observ_count, const float* observ_mean, const float* observ_var_sum,
                         int64_t reward_count, float reward_mean, float reward_var_sum);
int rexagent_get_filters(RexAgent* a, int64_t* counts /*[2]*/, float* observ_mean, float* observ_var_sum,
                         float* reward_mean_var /*[2]*/);

/* raw device state for checkpoint / resume: filt dev [2*O + 2] f32 (observ mean[O], var_sum[O], reward mean, var_sum);
 * counters dev [4] i64 (observ count, reward count, step counter, internal ticket = 0 between launches) */
int rexagent_state_buffers(RexAgent* a, float** filt, int64_t** counters);

/* observ dev [n][O] -> action dev [n][A], mean dev [n][A], logprob dev [n], value dev [n]  (any output may be NULL).
 * training != 0: action = mean + exp(logstd) * eps, eps ~ N(0,1) from the counter-based generator keyed on
 * (seed, env_offset + env, step + device step counter, action index); training == 0: action = mean.
 * observ_copy (dev [n][O] or NULL) receives the raw observations (the `prevob` copy of simulate.py:66). */
int rexagent_perform(RexAgent* a, const float* observ, int32_t n, int32_t training, uint64_t seed, uint32_t step,
                     uint32_t env_offset, float* action, float* mean, float* logprob, float* value, float* observ_copy,
                     void* stream);
/* update both filters with one batch (observ dev [n][O], reward dev [n]); also advances the device step counter */
int rexagent_experience(RexAgent* a, const float* observ, const float* reward, int32_t n, void* stream);
/* Environment-sharded rollouts (one rank per GPU): the filters must see the WHOLE batch, so the update splits in two around
 * the one real exchange step of this path -- a sum all-reduce of 2*(O+1) floats:
 *   rexagent_experience_partial  -> sums dev [O+1][2] = (sum(x - mean), sum((x - mean)^2)) of this rank's batch, filters untouched
 *   ncclAllReduce(sums, sum)        (torch.distributed.all_reduce on the same stream)
 *   rexagent_experience_finalize -> applies the global sums with n_total = envs of all ranks; observ/reward: this rank's batch
 *                                   (only element 0 is read, for the count <= 1 corner of normalize.py:88) */
int rexagent_experience_partial(RexAgent* a, const float* observ, const float* reward, int32_t n, float* sums, void* stream);
int rexagent_experience_finalize(RexAgent* a, const float* sums, int32_t n_total, const float* observ, const float* reward, void* stream);
/* reward filter transform (scale by the running std, clip): in dev [n] -> out dev [n] */
int rexagent_transform_reward(RexAgent* a, const float* reward, int32_t n, float* out, void* stream);

/* episode-row scans with the reference's semantics: element (e, t) lives at base[e * stride_e + t * stride_t];
 * steps t >= length[e] are masked exactly as `mask * reward` does in utility.py */
int rexagent_discounted_return(const float* reward, const int32_t* length, int32_t episodes, int32_t max_length,
                               int64_t stride_e, int64_t stride_t, float discount, float* out, void* stream);
int rexagent_lambda_advantage(const float* reward, const float* value, const int32_t* length, int32_t episodes,
                              int32_t max_length, int64_t stride_e, int64_t stride_t, float discount, float* out,
                              void* stream);
/* time-major rollout of an auto-resetting batch: reward, done [T][N]; value [T+1][N] (last row = bootstrap value);
 * out_return, out_advantage [T][N] (either may be NULL).  delta_t = r_t + discount * v_{t+1} * (1 - done_t) - v_t,
 * adv_t = delta_t + discount * lambda * (1 - done_t) * adv_{t+1}; return_t = r_t + discount * (1 - done_t) * return_{t+1},
 * return_T = bootstrap value */
int rexagent_gae_segments(const float* reward, const float* value, const uint8_t* done, int32_t T, int32_t n,
                          float discount, float lambda, float* out_return, float* out_advantage, void* stream);
/* (its form that bootstraps episodes cut by the time limit, rexsim_gae_segments_bootstrap, is declared in rexsim.h) */
int64_t rexagent_launch_count(const RexAgent* a);

#ifdef __cplusplus
}
#endif
#endif
