/*
 * ovc_horizon.h — C ABI of the horizon bootstrap (csrc/libovc_horizon.so): PPO advantages that bootstrap from the learner's
 * value of each episode's last state where the episode was cut by the time limit, instead of counting that state terminal.
 *
 * Every Overcooked episode ends at the horizon, and no state of the MDP is terminal (Pardo et al., "Time Limits in
 * Reinforcement Learning", 2018).  The rollout evaluates the learner's value head on the terminal records between ovc_step
 * (without its auto-reset) and the reset, on the rows ovc_horizon_rows compacts, and ovc_gae_horizon uses those values as
 * the next value at the cut.
 *
 * Conventions are include/ovc_b200.h's: `extern "C"`, device pointers owned by the caller, `stream` a cudaStream_t passed as
 * void*, 0 on success or a negative OVC_E_* code with a message from ovc_horizon_last_error().  Launches are asynchronous.
 */
#ifndef OVC_HORIZON_H
#define OVC_HORIZON_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OVC_HORIZON_ABI_VERSION 1

int ovc_horizon_abi_version(void);
const char *ovc_horizon_last_error(void);

/*
 * ovc_horizon_rows: the learner rows of the environments whose episode just ended, compacted on the device.  For every
 * environment e with done[e] != 0 (int32 [n_envs], ovc_step's done), each of its learner views v gets one compact row r:
 *     two views (one_view = 0)   partner_seat NULL or partner_seat[e] < 0: views 0 and 1 (self-play), output row 2 e + v;
 *                                else view 1 - partner_seat[e] (the partner holds the other one), output row 2 e + v
 *     one view (one_view = 1)    view 1 - partner_seat[e] (partner_seat required: agent 1's player), output row e
 *   records[r] = state[e] (int32 [rows][state_words], rows = 2 n_envs, or n_envs with one_view), view[r] = v, jrow[r] = the
 *   output row (both int32 [rows]), range = (0, the row count) (int32 [2], device memory: the range of
 *   ovc_encode_linear_rows, ovc_wide_layers_range and ovc_policy_tail_joint).  The compact order is unspecified (rows are
 *   claimed with atomics); entries past the count are left as they were.  values (float32 [2 n_envs], or [n_envs] with
 *   one_view; nullable): every output row of every environment is set to 0, so that a value pass writing the learner rows
 *   of the ended environments afterwards leaves 0 everywhere else.  With no environment done the count is 0.
 *   state 16-byte aligned, state_words in {16, 32, 64, 128}; the int32 and float buffers 4-byte aligned.  n_envs < 2^30;
 *   n_envs = 0 writes nothing.
 */
int ovc_horizon_rows(const int32_t *state, int state_words, const int32_t *done, const int32_t *partner_seat, int one_view,
                     int64_t n_envs, int32_t *records, int32_t *view, int32_t *jrow, int32_t *range, float *values, void *stream);

/*
 * ovc_gae_horizon: generalized advantage estimation over a window of n_steps transitions of n_rows = 2 n_envs agent rows
 * that bootstraps at every episode end from terminal_values instead of counting the state after it terminal:
 *     rewards, values, terminal_values, advantages, value_targets float32 [n_steps][n_rows];  dones uint8 [n_steps][n_rows / 2]
 *     (one flag per environment, shared by its two rows);  last_values float32 [n_rows]
 *   from t = n_steps - 1 down to 0, with A = 0 after the window, every operation rounded to float32 on its own:
 *     d = dones[t][r / 2];  next_v = d ? terminal_values[t][r] : (t < n_steps - 1 ? values[t + 1][r] : last_values[r])
 *     delta = (rewards[t][r] + gamma * next_v) - values[t][r]
 *     A = delta + ((gamma * lambda) * (1 - d)) * A;   advantages[t][r] = A;   value_targets[t][r] = A + values[t][r]
 *   The lambda chain is cut at every episode end; only the bootstrap differs from ovc_gae.  With every terminal value 0
 *   the result is bit for bit ovc_gae's (gamma * 0 = +0 and r + 0 = r for every reward but -0, which the rollout's rewards
 *   never are).  Float buffers 8-byte aligned.
 * ovc_gae_horizon_view: the same over n_envs rows, one per environment (an agent pair's learner): every [n_rows] array is
 *   [n_envs], dones uint8 [n_steps][n_envs]; bit for bit ovc_gae_horizon on those rows of a two-row layout.  Float buffers
 *   4-byte aligned.
 */
int ovc_gae_horizon(const float *rewards, const float *values, const uint8_t *dones, const float *terminal_values,
                    const float *last_values, int64_t n_steps, int64_t n_rows, float gamma, float lambda, float *advantages,
                    float *value_targets, void *stream);
int ovc_gae_horizon_view(const float *rewards, const float *values, const uint8_t *dones, const float *terminal_values,
                         const float *last_values, int64_t n_steps, int64_t n_envs, float gamma, float lambda, float *advantages,
                         float *value_targets, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* OVC_HORIZON_H */
