"""Self-play rollout collection with a torch policy on top of the batched engine (BASELINE config 5).

The reference collects PPO rollouts with Ray workers that each run one Python env and a TF copy of
the policy (human_aware_rl/rllib/rllib.py:293-342, ppo/ppo_rllib.py:7-80).  Here one process per GPU
keeps N environments on the device and runs, per transition,

    lossless_state_encoding (K2, [N,2,W,H,26])  ->  policy CNN (torch)  ->  sampling
    ->  ovc_step (K1)  ->  reward accumulation

or, with the dense bf16 policy, K7 in place of K2 + the first layer: encoding, first layer and its leaky ReLU evaluated
from the packed records (``ovc_encode_linear``), the observation tensor never written

with no host round trip; the whole transition can be captured in one CUDA graph.  The observation
tensor is consumed zero-copy: ``[N,2,W,H,26]`` viewed as ``(2N, 26, W, H)`` is exactly torch's
channels-last memory format.

The policy is shaped like the reference's ``RllibPPOModel`` defaults (ppo_rllib.py:43-79 with
ppo_rllib_client.py:85-88: conv 5x5x25 'same', conv 3x3x25 'same', conv 3x3x25 'valid', 3 dense layers
of 64, leaky ReLU, heads 6 + 1), random init, shared by both agents.  ``RllibShapedCNN`` is that model in torch
(the consumer a user brings: cuDNN / cuBLAS); ``DenseGridPolicy`` is the same function as one matrix per layer, and
on a 5x4 grid ``SelfPlayRollout`` evaluates it entirely with this library's kernels: K7 (encoding + first layer from
the packed records), K9 (the two wide layers, wgmma), K8 (dense tail + heads + action draw).
"""
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _native


class RllibShapedCNN(nn.Module):
    def __init__(self, width, height, in_planes=26, num_filters=25, hidden=64, num_hidden_layers=3, num_actions=6):
        super().__init__()
        self.conv_initial = nn.Conv2d(in_planes, num_filters, 5, padding=2)
        self.conv_0 = nn.Conv2d(num_filters, num_filters, 3, padding=1)
        self.conv_1 = nn.Conv2d(num_filters, num_filters, 3, padding=0)
        flat = num_filters * (width - 2) * (height - 2)
        dims = [flat] + [hidden] * num_hidden_layers
        self.dense = nn.ModuleList([nn.Linear(dims[i], dims[i + 1]) for i in range(num_hidden_layers)])
        self.logits = nn.Linear(hidden, num_actions)
        self.value = nn.Linear(hidden, 1)

    def load_keras_weights(self, conv, dense, logits, value):
        """Weights of the reference's ``RllibPPOModel`` (ppo_rllib.py:43-79, a Keras model) into this module: ``conv`` =
        [(kernel, bias)] of conv_initial, conv_0, conv_1 with Keras kernels ``(kh, kw, in, out)`` over an observation of shape
        ``(W, H, 26)``; ``dense`` = [(kernel, bias)] of the hidden layers with Keras kernels ``(in, out)``, the first one over
        Keras' flatten order ``(x, y, channel)``; ``logits`` / ``value`` = (kernel, bias) of the two heads.  Arrays or
        tensors.  The function computed is the Keras model's (tests/test_host_cpu.py restates it in numpy)."""
        t = lambda a: torch.as_tensor(a, dtype=torch.float32)
        with torch.no_grad():
            for mod, (k, b) in zip((self.conv_initial, self.conv_0, self.conv_1), conv):
                mod.weight.copy_(t(k).permute(3, 2, 0, 1))  # (kh, kw, in, out) -> (out, in, kh, kw): the grid's x is the kernel's first axis in both
                mod.bias.copy_(t(b))
            co = self.conv_1.out_channels
            k0, b0 = dense[0]
            k0 = t(k0)  # rows in (x, y, c) order; torch flattens (c, x, y)
            wo_ho = k0.shape[0] // co
            self.dense[0].weight.copy_(k0.view(wo_ho, co, -1).permute(2, 1, 0).reshape(k0.shape[1], -1))
            self.dense[0].bias.copy_(t(b0))
            for mod, (k, b) in zip(list(self.dense)[1:], dense[1:]):
                mod.weight.copy_(t(k).t()), mod.bias.copy_(t(b))
            self.logits.weight.copy_(t(logits[0]).t()), self.logits.bias.copy_(t(logits[1]))
            self.value.weight.copy_(t(value[0]).t()), self.value.bias.copy_(t(value[1]))
        return self

    def forward(self, obs_nchw):
        x = F.leaky_relu(self.conv_initial(obs_nchw), 0.2)
        x = F.leaky_relu(self.conv_0(x), 0.2)
        x = F.leaky_relu(self.conv_1(x), 0.2)
        x = x.flatten(1)
        for d in self.dense:
            x = F.leaky_relu(d(x), 0.3)
        return self.logits(x), self.value(x).squeeze(-1)


class DenseGridPolicy(nn.Module):
    """The same network as ``RllibShapedCNN`` with every convolution folded into ONE matrix per layer.

    On a 5x4 (or 9x5) grid a 'same' convolution spends most of its taps on padding: conv 5x5x26->25 over 20 cells is
    325 k MACs per observation, while the linear map it IS — 520 inputs -> 500 outputs — is 260 k.  cuDNN also runs
    25/26-channel convolutions far below the tensor-core peak, whereas ``[2N, 520] x [520, 500]`` is a plain library
    GEMM.  The matrices are built once by pushing the identity through each convolution (exact: same weights, same
    function, only the summation order differs), in the observation kernel's own element order ``[x][y][channel]``, so
    K2's output is consumed as ``[2N, W*H*26]`` without any permute.

    ``pad_to``: every layer's width is rounded up to a multiple of it with zero weights and zero biases (leaky ReLU of 0
    is 0, the next layer's extra input columns are zero too: the function is unchanged).  Widths of 500 / 150 bf16
    elements give rows that are not 16-byte multiples, which sends the library to its Ampere-era ``align2`` mma.sync
    kernels; 512 / 160 reach its tensor-core kernels for the GPU.  The two heads are one matrix (6 logits + 1 value, padded to 8).  ``forward`` / ``forward_from`` / ``trunk`` run
    it as library GEMMs; ``first_layer_table`` / ``wide_tables`` / ``tail_tables`` hand the same weights to K7 / K9 / K8."""

    def __init__(self, cnn, width, height, pad_to=1):
        super().__init__()
        self.W, self.H = width, height
        up = lambda n: -(-n // pad_to) * pad_to
        with torch.no_grad():
            mats = []
            shape = (26, width, height)  # (channels, x, y) as the conv sees it
            for conv in (cnn.conv_initial, cnn.conv_0, cnn.conv_1):
                c, w, h = shape
                n_in = c * w * h
                # basis vector k of the flat [x][y][c] input -> NCHW image with a single one
                eye = torch.eye(n_in, dtype=conv.weight.dtype, device=conv.weight.device).view(n_in, w, h, c).permute(0, 3, 1, 2)
                out = F.conv2d(eye, conv.weight, None, padding=conv.padding)  # (n_in, c_out, w', h'), bias added separately
                co, wo, ho = out.shape[1:]
                mats.append((out.permute(0, 2, 3, 1).reshape(n_in, wo * ho * co).t().contiguous(),   # [n_out, n_in], [x][y][c] order
                             conv.bias.view(1, 1, co).expand(wo, ho, co).reshape(-1).clone()))
                shape = (co, wo, ho)
            # the first dense layer consumed conv_1's NCHW flatten (c, x, y): re-order its inputs to [x][y][c]
            co, wo, ho = shape
            first = cnn.dense[0]
            mats.append((first.weight.view(-1, co, wo, ho).permute(0, 2, 3, 1).reshape(first.out_features, -1), first.bias))
            mats += [(d.weight, d.bias) for d in cnn.dense[1:]]
            mats.append((torch.cat([cnn.logits.weight, cnn.value.weight]), torch.cat([cnn.logits.bias, cnn.value.bias])))
            self.n_actions = cnn.logits.out_features
            layers, n_in = [], mats[0][0].shape[1]  # the input width is K2's row: never padded
            for m, bias in mats:
                lin = nn.Linear(n_in, up(m.shape[0]))
                lin.weight.zero_(), lin.bias.zero_()
                lin.weight[:m.shape[0], :m.shape[1]].copy_(m), lin.bias[:m.shape[0]].copy_(bias)
                layers.append(lin)
                n_in = lin.out_features
            self.conv_as_linear = nn.ModuleList(layers[:3])
            self.dense = nn.ModuleList(layers[3:-1])
            self.heads = layers[-1]

    def forward(self, obs_flat):
        """obs_flat: [2N, W*H*26] in K2's element order.  Returns (logits [2N, 6], value [2N]) as views of one matrix."""
        return self.forward_from(obs_flat, 0)

    def first_layer_table(self):
        """(wt bfloat16 [W*H*26, n_out], bias float32 [n_out]) of the first layer in the form ``ovc_encode_linear`` (K7)
        takes: the matrix transposed, rows in the observation's element order."""
        lin = self.conv_as_linear[0]
        return lin.weight.detach().t().contiguous().to(torch.bfloat16), lin.bias.detach().float().contiguous()

    def tail_tables(self):
        """The dense tail in the form ``ovc_policy_tail`` (K8) takes: (w_first bf16 [64, k0], b_first f32 [64], w_hidden bf16
        [n_hidden, 64, 64], b_hidden f32 [n_hidden, 64], w_heads bf16 [8, 64], b_heads f32 [8]).  Its input is the LAST
        convolution's pre-activation (``trunk``)."""
        d = list(self.dense)
        assert all(l.out_features == 64 for l in d) and d[0].in_features % 32 == 0 and d[0].in_features <= 256 and self.n_actions <= 7
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().float().contiguous()
        return (bf(d[0].weight), f32(d[0].bias), bf(torch.stack([l.weight for l in d[1:]])), f32(torch.stack([l.bias for l in d[1:]])),
                bf(self.heads.weight[:8]), f32(self.heads.bias[:8]))

    def wide_tables(self):
        """The two wide layers in the form ``ovc_wide_layers`` (K9) takes: (w1 bf16 [n1, k0], b1 f32, w2 bf16 [n2, n1], b2 f32)."""
        l1, l2 = self.conv_as_linear[1], self.conv_as_linear[2]
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()
        return bf(l1.weight), l1.bias.detach().float().contiguous(), bf(l2.weight), l2.bias.detach().float().contiguous()

    def trunk(self, x, first, out=None):
        """The wide layers from index ``first`` on, up to the last convolution's PRE-activation ``[rows, k0]`` (its leaky ReLU
        is applied by K8 on load)."""
        convs = list(self.conv_as_linear)
        for lin in convs[first:-1]:
            x = F.leaky_relu(lin(x), 0.2, inplace=True)
        last = convs[-1]
        return torch.addmm(last.bias, x, last.weight.t(), out=out)

    def forward_from(self, x, first):
        """The layers from index ``first`` on (0: the whole network from the observation; 1: from the first layer's
        activations, e.g. K7's output)."""
        for lin in self.conv_as_linear[first:]:
            x = F.leaky_relu(lin(x), 0.2, inplace=True)
        for d in self.dense:
            x = F.leaky_relu(d(x), 0.3, inplace=True)
        hv = self.heads(x)
        return hv[:, :self.n_actions], hv[:, self.n_actions]


def fused_kernel_support(dense_model, width, height):
    """(K7, K9, K8) usable for this network on this grid: K7 needs the first layer's width to be a multiple of 64 and its
    narrowest column slice (64 columns of the 19 dynamic planes) to fit shared memory; K9 is built for 512 -> 512 -> 160 (5x4
    grids); K8 for a tail of 64-wide layers behind an input of a multiple of 32 (<= 256) and at most 7 actions.  Whatever is
    not supported runs as library GEMMs / the separate draw kernel."""
    l0, l1, l2 = dense_model.conv_as_linear
    d = list(dense_model.dense)
    k7 = l0.out_features % 64 == 0 and width * height * 19 * 64 * 2 + 4096 <= 227 * 1024
    k9 = (l1.in_features, l1.out_features, l2.out_features) == (512, 512, 160)
    k8 = all(l.out_features == 64 for l in d) and d[0].in_features % 32 == 0 and d[0].in_features <= 256 and dense_model.n_actions <= 7
    return k7, k9, k8


def sample_categorical(logits, noise):
    """One draw per row from softmax(logits) by the Gumbel-max rule: argmax_i (logit_i - log E_i) with E_i ~ Exp(1) picks i
    with probability softmax(logits)_i — four small kernels where softmax + ``torch.multinomial`` launch about twenty.
    ``logits`` (float32) is overwritten with the perturbed scores, ``noise`` is scratch of
    the same shape."""
    logits.sub_(noise.exponential_().log_())
    return torch.argmax(logits, dim=-1)


class SelfPlayRollout(object):
    """Policy-in-the-loop rollout: both agents of every environment act from the same network."""

    def __init__(self, env, model=None, autocast_dtype=torch.bfloat16, use_graph=True, reward_shaping_factor=1.0,
                 obs_dtype=None, dense=True, sub_batches=1, fused_first_layer=None, native_glue=True, seed=0, fused_tail=None, fused_wide=None):
        """obs_dtype: element type K2 writes (default: bfloat16 when the policy runs in bf16 — the plane values are exact
        in bf16 and the conversion pass disappears — else float32).
        dense: evaluate the network through ``DenseGridPolicy`` (one library GEMM per layer, widths padded to 16-byte rows,
        weights held in ``autocast_dtype``: what autocast computes, without its per-call weight casts) instead of cuDNN
        convolutions under autocast.
        sub_batches: the policy runs over this many row blocks one after the other, so that a block's activations
        (rows x 512 bf16) are still in L2 when the activation pass and the next layer read them.
        fused_first_layer (default: on for the dense bf16 policy): the observation is never materialised — kernel K7
        (``env.encoded_linear``) evaluates encoding + first layer + leaky ReLU from the packed records, and the library
        GEMMs start at the second layer.
        native_glue: the joint action is drawn by ``ovc_sample_actions`` (Gumbel-max on Philox draws keyed by ``seed``,
        one kernel) and the rewards are folded into the returns by ``ovc_accumulate_returns`` (one kernel) instead of five
        and four tensor-library kernels.
        fused_tail (default: with native_glue on the dense bf16 policy): the dense layers of 64, the heads and the draw run as
        ONE kernel (``ovc_policy_tail``, K8) on the last convolution's pre-activation; the library GEMMs are then only the
        two wide layers.
        fused_wide (default: with K7 and K8 when the wide layers are 512 -> 512 -> 160, i.e. on 5x4 grids): those two layers
        run as ONE wgmma kernel (``ovc_wide_layers``, K9: the 512-wide activation stays in registers) — the
        whole policy is then K7 -> K9 -> K8, no library call."""
        assert len({(l.width, l.height) for l in env.layouts}) == 1, "one grid shape per rollout (group envs by layout)"
        self.env = env
        l = env.layouts[0]
        self.W, self.H = l.width, l.height
        dev = env.device
        self.model = (model or RllibShapedCNN(self.W, self.H)).to(dev).to(memory_format=torch.channels_last).eval()
        self.autocast_dtype = autocast_dtype
        self.dense_model = None
        if dense:
            self.dense_model = DenseGridPolicy(self.model, self.W, self.H, pad_to=16).to(dev).eval()
            if autocast_dtype is not None:
                self.dense_model = self.dense_model.to(autocast_dtype)
        k7_ok, k9_ok, k8_ok = fused_kernel_support(self.dense_model, self.W, self.H) if dense else (False, False, False)
        if fused_first_layer is None:
            fused_first_layer = dense and autocast_dtype == torch.bfloat16 and k7_ok
        assert not fused_first_layer or (dense and autocast_dtype == torch.bfloat16 and k7_ok), \
            "K7 feeds the dense bf16 policy (first layer width a multiple of 64, table within shared memory)"
        self.fused_first_layer = bool(fused_first_layer)
        self.factor = float(reward_shaping_factor)
        N = env.n_envs
        if obs_dtype is None:
            obs_dtype = torch.bfloat16 if autocast_dtype == torch.bfloat16 else torch.float32
        if dense and autocast_dtype is not None:
            assert obs_dtype == autocast_dtype, "the dense policy consumes K2's rows as they are"
        self.obs = None if self.fused_first_layer else torch.empty((N, 2, self.W, self.H, 26), dtype=obs_dtype, device=dev)
        if self.fused_first_layer:
            self._wt0, self._b0 = self.dense_model.first_layer_table()
            self._act0 = torch.empty((2 * N, self._wt0.shape[1]), dtype=torch.bfloat16, device=dev)
        self.actions = torch.zeros((N, 2), dtype=torch.int32, device=dev)
        self.ret_sparse = torch.zeros(N, dtype=torch.int64, device=dev)      # running episode return (sparse)
        self.ret_mixed = torch.zeros(N, dtype=torch.float32, device=dev)    # sparse + factor * shaped (rllib.py:328-329)
        self.values = torch.zeros((N, 2), dtype=torch.float32, device=dev)
        self.native_glue = bool(native_glue)
        if fused_tail is None:
            fused_tail = self.native_glue and dense and autocast_dtype == torch.bfloat16 and k8_ok
        assert not fused_tail or (self.native_glue and dense and autocast_dtype == torch.bfloat16 and k8_ok), \
            "K8 ends the dense bf16 policy (64-wide tail behind an input of a multiple of 32, <= 256)"
        self.fused_tail = bool(fused_tail)
        if self.fused_tail:
            self._tail = self.dense_model.tail_tables()
            self._z = torch.empty((2 * N, self._tail[0].shape[1]), dtype=torch.bfloat16, device=dev)  # last convolution, pre-activation
        if fused_wide is None:
            fused_wide = self.fused_tail and self.fused_first_layer and k9_ok
        assert not fused_wide or (self.fused_tail and self.fused_first_layer and k9_ok), \
            "K9 sits between K7 and K8 and is built for 512 -> 512 -> 160"
        self.fused_wide = bool(fused_wide)
        if self.fused_wide:
            self._wide = self.dense_model.wide_tables()
        self.seed = int(seed)
        self._draw_counter = torch.zeros(2, dtype=torch.int64, device=dev)  # [step, scratch] of ovc_sample_actions
        self._scores8 = None  # set to a float32 [2N, 8] tensor to make K8 also write the heads (tests)
        self._noise = torch.empty((2 * N, 6), dtype=torch.float32, device=dev)
        self._scores = torch.empty((2 * N, 6), dtype=torch.float32, device=dev)
        self.sub_batches = int(sub_batches)
        assert (2 * N) % self.sub_batches == 0
        self.graph = None
        self.use_graph = use_graph

    def _policy(self):
        """(scores float32 [2N, 6] = logits, values written to self.values) for the observations in self.obs."""
        env = self.env
        rows = 2 * env.n_envs
        with torch.no_grad():
            if self.dense_model is not None:
                if self.fused_first_layer:
                    flat, first = env.encoded_linear(self._wt0, self._b0, out=self._act0, neg_slope=0.2), 1  # K7
                else:
                    flat, first = self.obs.view(rows, self.W * self.H * 26), 0
                vals = self.values.view(rows)
                step = rows // self.sub_batches
                if self.fused_tail:  # K8 draws the actions itself: nothing to return
                    if self.fused_wide:
                        w1, b1, w2, b2 = self._wide
                        _native.check(_native.lib().ovc_wide_layers(flat.data_ptr(), rows, flat.shape[1], w1.data_ptr(), b1.data_ptr(), w1.shape[0],
                                                                    w2.data_ptr(), b2.data_ptr(), w2.shape[0], 0.2, self._z.data_ptr(), env._stream()))
                    else:
                        for b in range(0, rows, step):
                            self.dense_model.trunk(flat[b:b + step], first, out=self._z[b:b + step])
                    w1, b1, wh, bh, wo, bo = self._tail
                    _native.check(_native.lib().ovc_policy_tail(
                        self._z.data_ptr(), rows, self._z.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(),
                        wh.shape[0], wo.data_ptr(), bo.data_ptr(), 0.3, self.dense_model.n_actions, self.seed & (2**64 - 1),
                        self._draw_counter.data_ptr(), self.actions.data_ptr(), vals.data_ptr(),
                        self._scores8.data_ptr() if self._scores8 is not None else 0, env._stream()))
                    return None
                for b in range(0, rows, step):
                    logits, value = self.dense_model.forward_from(flat[b:b + step], first)
                    self._scores[b:b + step].copy_(logits)
                    vals[b:b + step].copy_(value)
            else:
                with torch.autocast("cuda", dtype=self.autocast_dtype, enabled=self.autocast_dtype is not None):
                    x = self.obs.view(rows, self.W, self.H, 26).permute(0, 3, 1, 2)  # (2N,26,W,H), channels-last strides
                    logits, value = self.model(x)
                self._scores.copy_(logits)
                self.values.view(rows).copy_(value)
        return self._scores

    def _transition(self):
        env = self.env
        if not self.fused_first_layer:
            env.lossless_state_encoding(out=self.obs)  # K2
        scores = self._policy()
        if self.native_glue:
            if not self.fused_tail:
                env.sample_actions(scores, self._draw_counter, seed=self.seed, out=self.actions)
            env.step(self.actions)  # K1 (auto-reset inside)
            env.accumulate_returns(self.ret_sparse, self.ret_mixed, self.factor)
            return
        self.actions.copy_(sample_categorical(scores, self._noise).view(env.n_envs, 2))
        sparse, shaped, done, events = env.step(self.actions)  # K1 (auto-reset inside)
        self.ret_sparse.add_(sparse)
        self.ret_mixed.add_(sparse).add_(shaped[:, 0], alpha=self.factor).add_(shaped[:, 1], alpha=self.factor)

    def run(self, n_steps):
        """Advance every environment n_steps transitions; returns the number of env-steps done."""
        if self.use_graph and self.graph is None:
            # warm-up + capture must not advance the environments: snapshot, then restore
            saved = (self.env.state.clone(), self.ret_sparse.clone(), self.ret_mixed.clone(), self._draw_counter.clone())
            s = torch.cuda.Stream(self.env.device)
            s.wait_stream(torch.cuda.current_stream(self.env.device))
            with torch.cuda.stream(s):
                for _ in range(3):
                    self._transition()
            torch.cuda.current_stream(self.env.device).wait_stream(s)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph):
                self._transition()
            self.env.state.copy_(saved[0]), self.ret_sparse.copy_(saved[1]), self.ret_mixed.copy_(saved[2]), self._draw_counter.copy_(saved[3])
        for _ in range(n_steps):
            if self.graph is not None:
                self.graph.replay()
            else:
                self._transition()
        return n_steps * self.env.n_envs

    def env_only(self, n_steps):
        """The same transitions without the policy: encode + step with the last sampled actions
        (used to report the env-only share of the pipeline)."""
        for _ in range(n_steps):
            if self.fused_first_layer:
                self.env.encoded_linear(self._wt0, self._b0, out=self._act0, neg_slope=0.2)
            else:
                self.env.lossless_state_encoding(out=self.obs)
            self.env.step(self.actions)
        return n_steps * self.env.n_envs
