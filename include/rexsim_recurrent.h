/* rexsim_recurrent.h -- C ABI of the reference's two other policy cells, beside the ForwardGaussianPolicy of rexsim_agent.h:
 *
 *   REXRNN_GRU     <- RecurrentGaussianPolicy (rex_gym/agents/scripts/networks.py:113-159): normalised observation -> dense
 *                     hidden1 ReLU (policy_layers[:-1]) -> GRUBlockCell(cell) -> dense action_dim tanh -> mean, free logstd
 *   REXRNN_LINEAR  <- LinearGaussianPolicy (networks.py:21-63): mean = tanh(observation . W + b), free logstd
 *
 * Both keep ForwardGaussianPolicy's value network.  A handle is created against an existing RexAgent, which keeps everything
 * but the policy: the observation and reward filters, the noise step counter, the value block, rexagent_experience* and
 * rexagent_transform_reward.  The handle owns the policy block and, for the GRU, one hidden-state row per environment:
 * PPOAlgorithm's _last_state (rex_gym/agents/ppo/algorithm.py:74), zero at create.
 *
 * GRUBlockCell (TensorFlow 1.15 op documentation), G = cell, x = the dense layer's output, h = the previous state:
 *   [r | u] = sigmoid([x, h] . w_ru + b_ru)      (r: the first G columns)
 *   c       = tanh([x, r * h] . w_c + b_c)
 *   h'      = u * h + (1 - u) * c                 (the cell's output and its new state)
 *
 * Conventions as in rexsim.h: plain C, 0 / negative RexSimStatus, device pointers owned by the caller, everything enqueued on
 * the given stream, no host synchronisation except create / get_* / set_*.  The RexAgent must outlive the handle.
 */
#ifndef REXSIM_RECURRENT_H
#define REXSIM_RECURRENT_H
#include <stdint.h>
#include "rexsim_agent.h"

#ifdef __cplusplus
extern "C" {
#endif

enum { REXRNN_GRU = 0, REXRNN_LINEAR = 1 };

typedef struct {
    int32_t kind;       /* REXRNN_GRU or REXRNN_LINEAR */
    int32_t hidden1;    /* GRU: the dense layer before the cell (policy_layers[:-1]), <= 256, a multiple of 4; linear: ignored */
    int32_t cell;       /* GRU: the cell width G (hard-coded to 100 in networks.py:132), <= 128, a multiple of 4; linear: ignored */
    int32_t num_envs;   /* rows of the hidden state; perform takes n <= num_envs */
} RexRnnConfig;

typedef struct RexRnn RexRnn;

/* Packed policy block (floats), TF variable order, weights row-major [in][out], padded with zeros to a multiple of 4 floats:
 *   GRU   : W1[O][H1] b1[H1] w_ru[H1+G][2G] b_ru[2G] w_c[H1+G][G] b_c[G] W3[G][A] b3[A] logstd[A]
 *   linear: W[O][A] b[A] logstd[A]
 * O, A from the agent's RexAgentConfig; the value block stays the agent's (rexagent_set_params). */
int64_t rexrnn_policy_floats(const RexAgentConfig* agent, const RexRnnConfig* cfg);
/* the acceptance rule of rexrnn_create, without touching the device: O <= 32, A <= 8 and the agent's own limits (INVALID /
 * UNSUPPORTED as rexagent_create); kind and num_envs > 0 (INVALID); GRU: hidden1 <= 256, cell <= 128, both positive multiples
 * of 4 (UNSUPPORTED) */
int rexrnn_check(const RexAgentConfig* agent, const RexRnnConfig* cfg);
int rexrnn_create(RexAgent* agent, const RexRnnConfig* cfg, RexRnn** out);
void rexrnn_destroy(RexRnn* r);
int rexrnn_set_params(RexRnn* r, const float* host_params, int64_t n_floats);
int rexrnn_get_params(RexRnn* r, float* host_params, int64_t n_floats);
/* device pointer to the hidden state dev [num_envs][G] f32 (NULL for the linear cell): checkpoint / resume, begin_episode */
int rexrnn_state_buffer(RexRnn* r, float** state);
/* rexagent_perform with the recurrent policy: the same arguments, observation filter, sampling keys and log-density, plus
 * begin dev [n] u8 (or NULL): rows with begin != 0 start from the zero state (PPOAlgorithm.begin_episode, algorithm.py:90-103).
 * When action, mean or logprob is asked for, the policy runs and the new state of rows 0..n-1 is written back (algorithm.py:129).
 * A call that asks only for the value runs the agent's value network alone and leaves the state untouched (a rollout's
 * bootstrap value); observ_copy then must be NULL. */
int rexrnn_perform(RexRnn* r, const float* observ, const uint8_t* begin, int32_t n, int32_t training, uint64_t seed, uint32_t step,
                   uint32_t env_offset, float* action, float* mean, float* logprob, float* value, float* observ_copy, void* stream);
int64_t rexrnn_launch_count(const RexRnn* r);

#ifdef __cplusplus
}
#endif
#endif
