/*
 * ovc_bc.h — C ABI of behaviour-cloning training (csrc/libovc_bc.so): K multilayer perceptrons trained by minibatch Adam
 * on featurize_state rows, one CTA per model, one call per epoch.  It trains the float32 network that BCPolicy holds
 * (human_aware_rl/imitation/behavior_cloning_tf2.py's default MLP); K10 plays it after BCPolicy.tables() rounds it to bf16.
 *
 * Conventions are include/ovc_b200.h's: `extern "C"`, device pointers owned by the caller, `stream` a cudaStream_t passed as
 * void*, 0 on success or a negative OVC_E_* code with a message from ovc_bc_last_error().  Launches are asynchronous.
 */
#ifndef OVC_BC_H
#define OVC_BC_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define OVC_BC_ABI_VERSION 1
#define OVC_BC_MAX_BATCH 128 /* the largest minibatch whose rows, activations and deltas fit in shared memory */

int ovc_bc_abi_version(void);
const char *ovc_bc_last_error(void);

/*
 * ovc_bc_train_epoch: one epoch of training for each of n_models models.
 *
 * Shapes (the ones K10 plays): n_features = 96 (featurize_state at num_pots = 2), hidden = 64, num_hidden_layers L in
 *   {1, 2}, num_actions A in [2, 7], batch in [1, OVC_BC_MAX_BATCH].  Anything else is refused with OVC_E_UNSUPPORTED.
 *
 * Data:  features float32 [n_rows][n_features] (16-byte aligned), labels int32 [n_rows], labels in [0, A).
 *   Model k trains on train_rows[k * row_stride + i], i < n_train[k], in that order (the epoch's shuffle is the caller's),
 *   and is validated on val_rows[k * row_stride + i], i < n_val[k].  n_train and n_val are int32 [n_models], clamped to
 *   [0, row_stride].  Every listed row must lie in [0, n_rows) and every label in [0, A): the kernel does not check them.
 *
 * Parameters: params float32 [n_models][P], one flat vector per model in torch.nn.Linear's layout,
 *     for l = 0 .. L-1:  W_l [hidden][in_l] (out, in; in_0 = n_features, in_l = hidden), then b_l [hidden];
 *     then W_out [A][hidden], then b_out [A];
 *   P = n_features*hidden + hidden + (L-1)*(hidden*hidden + hidden) + A*hidden + A (10 758 at L = 2, A = 6).
 *   adam_m, adam_v float32 [n_models][P] (the same layout), step int32 [n_models] (Adam's step count t, 0 before the first
 *   update), lr float32 [n_models].  active uint8 [n_models]: a model whose flag is 0 is neither read nor written (its
 *   stats row included).  params, adam_m and adam_v 4-byte aligned, stats 8-byte aligned.
 *
 * Per minibatch: the next `batch` rows of train_rows[k] (the last minibatch holds the n_train % batch rows left over, if
 *   any), n of them, all in float32:
 *     a_0 = x;  a_{l+1} = relu(W_l a_l + b_l) for l < L;  z = W_out a_L + b_out     (each dot product a chain of FFMAs
 *       over the inputs in order, from 0, then + the bias)
 *     per row: m = max_a z_a;  s = sum_a exp(z_a - m);  lse = m + log(s);  loss = lse - z_label;  p_a = exp(z_a - lse)
 *       correct = (the first index of the largest logit) == label
 *     loss of the minibatch = the mean of the row losses (Keras SparseCategoricalCrossentropy(from_logits=True) with
 *       its default sum-over-batch-size reduction);  its gradients by back-propagation:
 *       dz_a = (p_a - [a == label]) / n;  d_L = (W_out^T dz) * [a_L > 0];  d_l = (W_l^T d_{l+1}) * [a_l > 0]
 *       g(W_out) = sum over rows of dz a_L^T;  g(b_out) = sum over rows of dz;  likewise g(W_l) = d_{l+1} a_l^T, g(b_l)
 *       (every gradient taken at the minibatch's parameters, before any of them is updated)
 *     then Keras' Adam (beta1 = 0.9, beta2 = 0.999, epsilon = 1e-7), in this order:
 *       t = t + 1
 *       alpha = lr * sqrt(1 - beta2^t) / (1 - beta1^t)          (evaluated in float64, rounded to float32 once)
 *       per parameter:  m = m + (g - m) * (1 - beta1);  v = v + (g*g - v) * (1 - beta2);  p = p - alpha * m / (sqrt(v) + epsilon)
 *         ((1 - beta1) and (1 - beta2) as the float32 constants 0.1f and 0.001f)
 *
 * Outputs: stats float64 [n_models][4] =
 *     (sum of the training rows' losses, each taken before its minibatch's update; the number of correct training rows;
 *      sum of the validation rows' losses after the epoch's last update; the number of correct validation rows)
 *   so the epoch's mean loss is stats[0] / n_train and its accuracy stats[1] / n_train, as Keras logs them.  The row
 *   losses of each minibatch are summed in float64 in a fixed order.
 *
 * A model's results depend only on its own inputs: training it alone or among others gives the same bits.  Any
 * n_models >= 0 (the grid may exceed one wave); n_models = 0 does nothing.  n_rows and row_stride in [0, 2^31).
 */
int ovc_bc_train_epoch(const float *features, const int32_t *labels, int64_t n_rows, const int32_t *train_rows,
                       const int32_t *n_train, const int32_t *val_rows, const int32_t *n_val, int64_t row_stride, float *params,
                       float *adam_m, float *adam_v, int32_t *step, const float *lr, const uint8_t *active, double *stats,
                       int n_models, int n_features, int hidden, int num_hidden_layers, int num_actions, int batch, void *stream);

#ifdef __cplusplus
}
#endif
#endif /* OVC_BC_H */
