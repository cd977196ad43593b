"""Self-play rollout collection with the PPO policy in the loop on top of the batched engine (BASELINE config 5).

The reference collects PPO rollouts with Ray workers that each run one Python env and a TF copy of
the policy (human_aware_rl/rllib/rllib.py:293-342, ppo/ppo_rllib.py:7-80).  Here one process per GPU
keeps N environments on the device and runs, per transition,

    K7 (encoding + first layer + leaky ReLU from the packed records)  ->  K9 (the two wide layers)
    ->  K8 (dense tail + heads + action draw)  ->  ovc_step (K1)  ->  reward accumulation

with no host round trip; the whole transition can be captured in one CUDA graph.  Where a grid or a dtype does not suit
a fused kernel, its layers run as library GEMMs instead: K2 then writes the observation ``[N,2,W,H,26]`` (consumed
zero-copy as ``[2N, W*H*26]``), and without K8 the draw is its own kernel (``ovc_sample_actions``).

The policy is shaped like the reference's ``RllibPPOModel`` defaults (ppo_rllib.py:43-79 with
ppo_rllib_client.py:85-88: conv 5x5x25 'same', conv 3x3x25 'same', conv 3x3x25 'valid', 3 dense layers
of 64, leaky ReLU, heads 6 + 1), random init, shared by both agents.  ``RllibShapedCNN`` is that model in torch
(the module a user trains and loads weights into); ``DenseGridPolicy`` is the same function as one matrix per layer,
the network ``SelfPlayRollout`` evaluates: on a 5x4 grid entirely with this library's kernels K7, K9 and K8.
"""
import copy
import functools
from types import SimpleNamespace

import numpy as np
import torch
import torch.nn as nn
import torch.nn.functional as F

from . import _native
from .batched import EpisodeRecords, EpisodeStats
from .greedy import GREEDY_DRAW_SALT, GreedyHumanModel


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

    dense_slope = 0.3  # RllibPPOModel's LeakyReLU() layers (Keras' default alpha)

    def trunk(self, obs_nchw):
        """The convolutions and the dense layers: the last dense layer's activation [B, hidden]."""
        x = F.leaky_relu(self.conv_initial(obs_nchw), 0.2)
        x = F.leaky_relu(self.conv_0(x), 0.2)
        x = F.leaky_relu(self.conv_1(x), 0.2)
        x = x.flatten(1)
        for d in self.dense:
            x = F.leaky_relu(d(x), self.dense_slope)
        return x

    def forward(self, obs_nchw):
        x = self.trunk(obs_nchw)
        return self.logits(x), self.value(x).squeeze(-1)


class RllibLSTMShapedCNN(RllibShapedCNN):
    """The reference's ``RllibLSTMPPOModel`` (ppo_rllib.py:89-238, ``use_lstm``): ``RllibShapedCNN``'s convolutions and dense
    layers, then an LSTM of ``cell_size`` (256, ``CELL_SIZE``) and the logits / value heads on its output.  The gates follow
    ``tf.keras.layers.LSTM``'s defaults (order i, f, c, o; sigmoid recurrent activation, tanh activation, one bias), which is
    torch's ``LSTMCell`` with Keras' bias in ``bias_ih`` and ``bias_hh`` zero.

    dense_slope: the negative slope of the dense layers' leaky ReLU.  The default 0.2 is ``tf.nn.leaky_relu``'s alpha, the
    activation the reference's LSTM model is recalled to give its ``TimeDistributed(Dense)`` layers (the CNN model's
    ``LeakyReLU()`` layers use 0.3); this is not pinned against the reference's source, so set it when loading weights
    from a model whose slope is known."""

    def __init__(self, width, height, in_planes=26, num_filters=25, hidden=64, num_hidden_layers=3, num_actions=6,
                 cell_size=256, dense_slope=0.2):
        super().__init__(width, height, in_planes, num_filters, hidden, num_hidden_layers, num_actions)
        self.dense_slope = float(dense_slope)
        self.lstm = nn.LSTMCell(hidden, cell_size)
        with torch.no_grad():
            self.lstm.bias_hh.zero_()
        self.logits = nn.Linear(cell_size, num_actions)
        self.value = nn.Linear(cell_size, 1)

    def load_keras_weights(self, conv, dense, lstm, logits, value):
        """As ``RllibShapedCNN.load_keras_weights``, and ``lstm`` = (kernel [in, 4 cell], recurrent_kernel [cell, 4 cell],
        bias [4 cell]) of the Keras LSTM layer, gate order i, f, c, o.  ``logits`` / ``value`` read the LSTM's output."""
        super().load_keras_weights(conv, dense, logits, value)
        t = lambda a: torch.as_tensor(a, dtype=torch.float32)
        k, rk, b = lstm
        with torch.no_grad():
            self.lstm.weight_ih.copy_(t(k).t()), self.lstm.weight_hh.copy_(t(rk).t())
            self.lstm.bias_ih.copy_(t(b)), self.lstm.bias_hh.zero_()
        return self

    def initial_state(self, batch):
        """(h, c) of zeros [batch, cell]: RLlib's ``get_initial_state``."""
        z = self.lstm.weight_hh.new_zeros((batch, self.lstm.hidden_size))
        return z, z.clone()

    def forward(self, obs_nchw, state):
        """One step: (logits, value, (h, c)) from observations [B, 26, W, H] and the state (h, c) [B, cell]."""
        h, c = self.lstm(self.trunk(obs_nchw), state)
        return self.logits(h), self.value(h).squeeze(-1), (h, c)

    def forward_sequence(self, obs, h0, c0, reset=None):
        """obs [L, B, 26, W, H] from the state (h0, c0) [B, cell]; the state is zeroed before step t wherever reset[t]
        ([L, B], nullable).  Returns logits [L, B, n_actions], values [L, B] and the final (h, c)."""
        L, B = obs.shape[:2]
        x = self.trunk(obs.flatten(0, 1)).view(L, B, -1)
        h, c, out = h0, c0, []
        for t in range(L):
            if reset is not None:
                keep = (reset[t] == 0).unsqueeze(-1)
                h, c = torch.where(keep, h, torch.zeros_like(h)), torch.where(keep, c, torch.zeros_like(c))
            h, c = self.lstm(x[t], (h, c))
            out.append(h)
        y = torch.stack(out)
        return self.logits(y), self.value(y).squeeze(-1), (h, c)


def lstm_gate_permutation(cell):
    """The order in which ``ovc_lstm_head`` (K11) takes the 4 cell gate rows of an LSTM (torch's / Keras' blocks i, f, g, o
    of ``cell`` rows): row 64 j + 8 (4 half + gate) + n is gate ``gate`` of hidden unit 16 j + 8 half + n, so that one lane
    of the kernel holds all four gates of its units."""
    p = torch.arange(4 * cell)
    j, q, n = p // 64, (p % 64) // 8, p % 8
    return (q % 4) * cell + 16 * j + 8 * (q // 4) + n


def _conv_matrix(conv, c, w, h, grad=False):
    """(matrix [n_out, n_in], (c_out, w', h')) of a convolution over a (c, x = w, y = h) image, inputs and outputs flat in
    [x][y][channel] order.  Each tap's weights are placed by index, with no arithmetic, so the matrix holds the convolution's
    own weights on any device (a convolution of the identity would be rounded to TF32 by cuDNN's default on the GPU).
    ``grad``: the placement stays in autograd, so a gradient on the matrix reaches ``conv.weight``."""
    if grad:  # one gather of the weights through the placement of their indices (_tap_index), one scatter in backward
        idx = _tap_index(tuple(conv.weight.shape), tuple(conv.padding), tuple(conv.stride), tuple(conv.dilation), w, h,
                         conv.weight.device)
        co, _, kx, ky = conv.weight.shape
        return torch.cat([conv.weight.new_zeros(1), conv.weight.reshape(-1)])[idx], \
            (co, w + 2 * conv.padding[0] - kx + 1, h + 2 * conv.padding[1] - ky + 1)
    k = conv.weight.detach()
    co, ci, kx, ky = k.shape
    px, py = conv.padding
    assert ci == c and conv.stride == (1, 1) and conv.dilation == (1, 1)
    wo, ho = w + 2 * px - kx + 1, h + 2 * py - ky + 1
    m = k.new_zeros((w, h, c, wo, ho, co))
    for dx in range(kx):
        for dy in range(ky):
            # out[xo][yo][o] += k[o, :, dx, dy] . in[xo + dx - px][yo + dy - py][:]   (torch's conv2d is a cross-correlation)
            xo = torch.arange(max(0, px - dx), min(wo, w + px - dx), device=k.device)
            yo = torch.arange(max(0, py - dy), min(ho, h + py - dy), device=k.device)
            m[(xo + dx - px)[:, None], (yo + dy - py)[None, :], :, xo[:, None], yo[None, :], :] = k[:, :, dx, dy].t()
    return m.reshape(w * h * c, wo * ho * co).t().contiguous(), (co, wo, ho)


@functools.lru_cache(maxsize=None)
def _tap_index(shape, padding, stride, dilation, w, h, device):
    """int64 [n_out, n_in]: 1 + the flat index into a weight of ``shape`` that ``_conv_matrix`` places at each matrix
    element, 0 where it places nothing (the placement of the weights 1, 2, ... in float64, exact far beyond these sizes)."""
    n = int(np.prod(shape))
    stand_in = SimpleNamespace(weight=torch.arange(1, n + 1, dtype=torch.float64, device=device).view(shape), padding=padding,
                               stride=stride, dilation=dilation)
    return _conv_matrix(stand_in, shape[1], w, h)[0].long()


def _folded_mats(cnn, width, height, grad=False):
    """The layers of ``cnn`` (``RllibShapedCNN``) as [(matrix [n_out, n_in], bias [n_out])], unpadded: the three
    convolutions (``_conv_matrix``), the dense layers (the first one's inputs re-ordered from torch's (c, x, y) flatten to
    [x][y][c]) and the heads (logits rows, then the value row).  ``grad``: every step stays in autograd."""
    mats = []
    shape = (26, width, height)  # (channels, x, y) as the conv sees it
    for conv in (cnn.conv_initial, cnn.conv_0, cnn.conv_1):
        m, shape = _conv_matrix(conv, *shape, grad=grad)
        co, wo, ho = shape
        mats.append((m, conv.bias.view(1, 1, co).expand(wo, ho, co).reshape(-1).clone()))
    # the first dense layer consumed conv_1's NCHW flatten (c, x, y): re-order its inputs to [x][y][c]
    co, wo, ho = shape
    first = cnn.dense[0]
    mats.append((first.weight.view(-1, co, wo, ho).permute(0, 2, 3, 1).reshape(first.out_features, -1), first.bias))
    mats += [(d.weight, d.bias) for d in cnn.dense[1:]]
    mats.append((torch.cat([cnn.logits.weight, cnn.value.weight]), torch.cat([cnn.logits.bias, cnn.value.bias])))
    return mats


def folded_layers(cnn, width, height, pad_to=16):
    """``DenseGridPolicy(cnn, width, height, pad_to)``'s layers as [(weight, bias)] float tensors that stay in autograd:
    a gradient on a folded (padded, tap-placed, re-ordered) matrix reaches ``cnn``'s parameters.  Same values, same
    padding as the module: conv_initial, conv_0, conv_1, the dense layers, the heads."""
    assert not hasattr(cnn, "lstm"), "the LSTM model is not folded here"
    up = lambda n: -(-n // pad_to) * pad_to
    out, n_in = [], None
    for m, bias in _folded_mats(cnn, width, height, grad=True):
        n_in = m.shape[1] if n_in is None else n_in  # the input width is K2's row: never padded
        n_out = up(m.shape[0])
        out.append((F.pad(m, (0, n_in - m.shape[1], 0, n_out - m.shape[0])), F.pad(bias, (0, n_out - bias.shape[0]))))
        n_in = n_out
    return out


class DenseGridPolicy(nn.Module):
    """The same network as ``RllibShapedCNN`` with every convolution folded into ONE matrix per layer.

    On a 5x4 (or 9x5) grid a 'same' convolution spends most of its taps on padding: conv 5x5x26->25 over 20 cells is
    325 k MACs per observation, while the linear map it IS — 520 inputs -> 500 outputs — is 260 k.  cuDNN also runs
    25/26-channel convolutions far below the tensor-core peak, whereas ``[2N, 520] x [520, 500]`` is a plain library
    GEMM.  The matrices are built once by placing each convolution's weights at the positions of its taps (exact on any
    device: the same weights, the same function, only the summation order differs), in the observation kernel's own
    element order ``[x][y][channel]``, so K2's output is consumed as ``[2N, W*H*26]`` without any permute.

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
            mats = _folded_mats(cnn, width, height)
            self.n_actions = cnn.logits.out_features
            self.dense_slope = cnn.dense_slope
            # RllibLSTMShapedCNN: the LSTM between the dense layers and the heads, kept as it is (lstm_tables folds it for K11)
            self.lstm = copy.deepcopy(cnn.lstm) if hasattr(cnn, "lstm") else None
            layers, n_in = [], mats[0][0].shape[1]  # the input width is K2's row: never padded
            for i, (m, bias) in enumerate(mats):
                if i == len(mats) - 1 and self.lstm is not None:
                    n_in = self.lstm.hidden_size  # the heads read the LSTM's output
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

    def hidden_tables(self):
        """The dense layers in the form ``ovc_policy_tail`` (K8) and ``ovc_policy_hidden`` take: (w_first bf16 [64, k0],
        b_first f32 [64], w_hidden bf16 [n_hidden, 64, 64], b_hidden f32 [n_hidden, 64]).  Their input is the LAST
        convolution's pre-activation (``trunk``)."""
        d = list(self.dense)
        assert all(l.out_features == 64 for l in d) and d[0].in_features % 32 == 0 and d[0].in_features <= 256
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().float().contiguous()
        return bf(d[0].weight), f32(d[0].bias), bf(torch.stack([l.weight for l in d[1:]])), f32(torch.stack([l.bias for l in d[1:]]))

    def tail_tables(self):
        """The dense tail in the form ``ovc_policy_tail`` (K8) takes: ``hidden_tables()`` and (w_heads bf16 [8, 64], b_heads
        f32 [8])."""
        assert self.lstm is None and self.n_actions <= 7
        return self.hidden_tables() + (self.heads.weight[:8].detach().to(torch.bfloat16).contiguous(),
                                       self.heads.bias[:8].detach().float().contiguous())

    def lstm_tables(self):
        """The LSTM and the heads in the form ``ovc_lstm_head`` (K11) takes: (w bf16 [4 cell, in + cell] = [W_ih | W_hh], b f32
        [4 cell] = b_ih + b_hh (one float32 sum), both with the gate rows in ``lstm_gate_permutation`` order; w_heads bf16
        [8, cell], b_heads f32 [8]).  Read from the parameters as they are: fold before casting this module to bfloat16
        (``SelfPlayRollout`` does), or the biases are rounded to bfloat16 first."""
        l = self.lstm
        assert l is not None and (l.input_size, l.hidden_size) == (64, 256) and self.n_actions <= 7, \
            "K11 is built for an LSTM of 256 on 64 inputs and at most 7 actions"
        perm = lstm_gate_permutation(l.hidden_size).to(l.weight_ih.device)
        w = torch.cat([l.weight_ih, l.weight_hh], 1).detach()[perm]
        b = (l.bias_ih.detach().float() + l.bias_hh.detach().float())[perm]
        return (w.to(torch.bfloat16).contiguous(), b.contiguous(), self.heads.weight[:8].detach().to(torch.bfloat16).contiguous(),
                self.heads.bias[:8].detach().float().contiguous())

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

    def hidden_from(self, x, first):
        """The layers from index ``first`` up to the last dense layer's activation (what ``ovc_policy_hidden`` writes)."""
        for lin in self.conv_as_linear[first:]:
            x = F.leaky_relu(lin(x), 0.2, inplace=True)
        for d in self.dense:
            x = F.leaky_relu(d(x), self.dense_slope, inplace=True)
        return x

    def forward_from(self, x, first):
        """The layers from index ``first`` on (0: the whole network from the observation; 1: from the first layer's
        activations, e.g. K7's output).  Not for the LSTM policy (its heads read the LSTM)."""
        assert self.lstm is None
        hv = self.heads(self.hidden_from(x, first))
        return hv[:, :self.n_actions], hv[:, self.n_actions]


K7_MAX_LAYOUTS = 8  # EL_MAX_LAYOUTS of ovc_encode_linear: its prologue folds the terrain sums of at most 8 layouts per call


def fused_kernel_support(dense_model, width, height, n_layouts=1):
    """(K7, K9, K8) usable for this network on this grid with ``n_layouts`` layouts in the batch: K7 needs the first layer's
    width to be a multiple of 64, its narrowest column slice (64 columns of the 19 dynamic planes) to fit shared memory, and
    at most ``K7_MAX_LAYOUTS`` (8) layouts; K9 is built for 512 -> 512 -> 160 (5x4 grids); K8 for a tail of 64-wide layers
    behind an input of a multiple of 32 (<= 256) and at most 7 actions.  Whatever is not supported runs as library GEMMs /
    the separate draw kernel.  ``SelfPlayRollout`` uses K9 only behind K7, so a pool of more than 8 5x4 layouts runs K2, the
    wide layers as library GEMMs, then K8."""
    l0, l1, l2 = dense_model.conv_as_linear
    d = list(dense_model.dense)
    k7 = _k7_fits(l0.out_features, width, height, n_layouts)
    k9 = (l1.in_features, l1.out_features, l2.out_features) == (512, 512, 160)
    k8 = all(l.out_features == 64 for l in d) and d[0].in_features % 32 == 0 and d[0].in_features <= 256 and dense_model.n_actions <= 7
    return k7, k9, k8


def _k7_fits(n_out, width, height, n_layouts):
    """K7 (and K12, whose narrowest table takes the same bytes) on a first layer of width ``n_out``: see ``fused_kernel_support``."""
    return n_out % 64 == 0 and width * height * 19 * 64 * 2 + 4096 <= 227 * 1024 and n_layouts <= K7_MAX_LAYOUTS


class _RecordsFirstLayer(torch.autograd.Function):
    """The first layer of the folded network on packed records: forward K7 (bf16 out, exactly what the behaviour policy's
    K7 computed from the same weights), backward K12 for the weight gradient.  The records have no gradient."""

    @staticmethod
    def forward(ctx, w0, b0, env, recs, seat, swap):
        wt = w0.detach().t().to(torch.bfloat16).contiguous()
        bias = b0.detach().to(torch.bfloat16).float()  # the rollout folds into a bf16 module: its K7 bias is bf16-rounded
        if seat is None:
            y = env.encoded_linear(wt, bias, neg_slope=0.2, states=recs)
        else:
            y = env.encoded_linear_view(wt, bias, seat, swap, neg_slope=0.2, states=recs)
        ctx.save_for_backward(y)
        ctx.env, ctx.recs, ctx.seat, ctx.swap, ctx.n_in = env, recs, seat, swap, w0.shape[1]
        return y

    @staticmethod
    def backward(ctx, grad):
        y, = ctx.saved_tensors
        # bf16 keeps float32's exponent range, so y's sign is the pre-activation's: the leaky ReLU's derivative from y
        dz = (grad.float() * torch.where(y > 0, 1.0, 0.2)).contiguous()
        dwt = torch.zeros((ctx.n_in, dz.shape[1]), dtype=torch.float32, device=dz.device)
        ctx.env.encoded_linear_wgrad(ctx.recs, dz, dwt, seat=ctx.seat, swap=ctx.swap)
        return dwt.t(), dz.sum(0), None, None, None, None


def records_forward(model, env, recs, seat=None, swap=None, fused_first_layer=None):
    """(logits float32 [rows, n_actions], values float32 [rows]) of ``model`` (``RllibShapedCNN``) on the packed records
    ``recs`` (int32 CUDA [M, S]), differentiable with respect to ``model``'s parameters.  Rows as K7's: ``seat`` None, both
    views (row 2 m + v); 0 / 1, one view (row m: player ``seat ^ (swap[m] != 0)``).

    The network is ``DenseGridPolicy``'s fold (``folded_layers``, pad 16) at the rollout's precision: bf16 operands, float32
    accumulation, float32 master weights and gradients.  The first layer runs as K7 / K12 (``_RecordsFirstLayer``) where
    K7 takes the grid and the layout count (``fused_first_layer`` None), else as K2's bf16 observation times the same
    matrix; the wide and dense layers are library GEMMs with bf16 outputs, and the heads are computed in float32 from the
    bf16 activations and weights (K8 writes float32 heads too)."""
    assert not isinstance(model, RllibLSTMShapedCNN), \
        "the LSTM model is trained on sequences: use RllibLSTMShapedCNN.forward_sequence on batch.observations"
    assert len({(l.width, l.height) for l in env.layouts}) == 1, "one grid shape per call (group envs by layout)"
    W, H = env.layouts[0].width, env.layouts[0].height
    layers = folded_layers(model, W, H, pad_to=16)
    bf = lambda t: t.to(torch.bfloat16)
    w0, b0 = layers[0]
    k7 = _k7_fits(w0.shape[0], W, H, env.n_layouts)
    if fused_first_layer is None:
        fused_first_layer = k7
    assert not fused_first_layer or k7, "K7 / K12 do not take this grid, layout count or first-layer width"
    if fused_first_layer:
        x = _RecordsFirstLayer.apply(w0, b0, env, recs, seat, swap)
    else:
        if seat is None:
            obs = env.lossless_state_encoding(dtype=torch.bfloat16, states=recs)
        else:
            vs = torch.full((recs.shape[0],), int(seat), dtype=torch.int32, device=recs.device)
            if swap is not None:
                vs ^= (swap != 0).to(torch.int32)
            obs = env.lossless_state_encoding(dtype=torch.bfloat16, states=recs, view_swap=vs.contiguous())[:, 0]
        x = F.leaky_relu(F.linear(obs.reshape(-1, w0.shape[1]), bf(w0), bf(b0)), 0.2)
    n_conv = 3
    for i, (w, b) in enumerate(layers[1:-1], 1):
        x = F.leaky_relu(F.linear(x, bf(w), bf(b)), 0.2 if i < n_conv else model.dense_slope)
    wh, bh = layers[-1]
    hv = F.linear(x.float(), bf(wh).float(), bf(bh).float())
    n_act = model.logits.out_features
    return hv[:, :n_act], hv[:, n_act]


class BCPolicy(nn.Module):
    """The behaviour-cloning partner of PPO_BC (human_aware_rl/imitation/behavior_cloning_tf2.py, the default MLP):
    featurize_state (96 features at num_pots = 2) -> Dense 64 ReLU (x ``num_hidden_layers``) -> ``num_actions`` logits, the
    action sampled from the softmax.  ``tables()`` hands it to K10 (``BatchedOvercookedEnv.partner_actions``)."""

    def __init__(self, n_features=96, hidden=64, num_hidden_layers=2, num_actions=6):
        super().__init__()
        dims = [n_features] + [hidden] * num_hidden_layers
        self.dense = nn.ModuleList([nn.Linear(dims[i], dims[i + 1]) for i in range(num_hidden_layers)])
        self.logits = nn.Linear(dims[-1], num_actions)

    def load_keras_weights(self, dense, logits):
        """The reference's Keras weights: ``dense`` = [(kernel, bias)] of the hidden layers, ``logits`` = (kernel, bias), Keras
        kernels ``(in, out)``.  Arrays or tensors."""
        t = lambda a: torch.as_tensor(a, dtype=torch.float32)
        with torch.no_grad():
            for mod, (k, b) in zip(self.dense, dense):
                mod.weight.copy_(t(k).t()), mod.bias.copy_(t(b))
            self.logits.weight.copy_(t(logits[0]).t()), self.logits.bias.copy_(t(logits[1]))
        return self

    def forward(self, features):
        x = features
        for d in self.dense:
            x = F.relu(d(x))
        return self.logits(x)

    def tables(self):
        """The network in the form ``ovc_partner_policy`` (K10) takes: (w_first bf16 [64, 96], b_first f32 [64], w_hidden bf16
        [n_hidden, 64, 64], b_hidden f32 [n_hidden, 64], w_heads bf16 [8, 64], b_heads f32 [8]) with n_hidden = the hidden
        layers after the first; the heads are the logits padded to 8 rows with zeros (row ``num_actions`` is the value row
        K8 reads; a BC policy has none)."""
        d = list(self.dense)
        assert len(d) >= 1 and all(l.out_features == 64 for l in d) and d[0].in_features == 96 and self.logits.out_features <= 7, \
            "K10 is built for 96 features, 64-wide layers and at most 7 actions"
        bf = lambda t: t.detach().to(torch.bfloat16).contiguous()
        f32 = lambda t: t.detach().float().contiguous()
        dev = self.logits.weight.device
        wh = torch.stack([l.weight for l in d[1:]]) if len(d) > 1 else torch.zeros((0, 64, 64), device=dev)
        bh = torch.stack([l.bias for l in d[1:]]) if len(d) > 1 else torch.zeros((0, 64), device=dev)
        wo, bo = torch.zeros((8, 64), device=dev), torch.zeros(8, device=dev)
        wo[:self.logits.out_features], bo[:self.logits.out_features] = self.logits.weight.detach(), self.logits.bias.detach()
        return bf(d[0].weight), f32(d[0].bias), bf(wh), f32(bh), bf(wo), f32(bo)


class SampleBatch(object):
    """One window of T self-play transitions as a PPO learner consumes it (RLlib's per-agent ``SampleBatch``), on the device.
    Agent rows are ``2 env + agent``, so ``actions[t].view(N, 2)`` is the joint action ``ovc_step`` took.

    states        int32 [T, N, S]    the records the actions were drawn from (observations are re-encoded on demand)
    actions       int32 [T, 2N]
    logp          float32 [T, 2N]    log-probability of each action under the behaviour policy
    values        float32 [T, 2N]    value head on states[t]
    rewards       float32 [T, 2N]    sparse + reward_shaping_factor * shaped_i (rllib.py:328-329)
    dones         uint8 [T, N]       the episode ended with transition t (the environment auto-reset)
    last_values   float32 [2N]       value head on the state after the window (bootstrap)
    advantages, value_targets  float32 [T, 2N]   GAE (ovc_gae; with ``bootstrap_horizon``, ovc_gae_horizon)
    terminal_values float32 [T, 2N]  only with collect()'s ``bootstrap_horizon``, else None: the learner's value of the
                                     terminal state (the record before the reset) where ``dones[t]`` on a learner row, 0
                                     elsewhere (partner rows included); GAE bootstraps from it at the horizon cut
    logits        float32 [T, 2N, 8] the policy's heads (columns 0..5 the logits), only with ``keep_logits``
    partner_seat  int8 [T, N]        with a partner: its player index at transition t (-1: self-play), else None
                                     (``one_view``: agent 1's player)
    partner_member int8 [T, N]       with a population of partners: each environment's member at transition t (in a
                                     two-view batch meaningful where partner_seat >= 0), else None
    pair          int8 [T, N, 2]     population play: the members on players 0 / 1 of each environment at transition t, so
                                     ``pair.view(T, 2N)[t, r]`` is the member that acted on row r; else None
    learner_mask  uint8 [T, 2N]      (property) the rows the learner trains on: all rows but the partner's
    episodes      EpisodeRecords     the episodes that ended in the window (``episodes.finished()``), capacity
                                     ceil(T / horizon): an environment cannot end more episodes in T transitions

    With the LSTM policy (``RllibLSTMShapedCNN``) the window is cut into chunks of ``seq_len`` = L transitions (RLlib's
    ``max_seq_len``), and the batch holds the recurrent state each chunk starts from:

    seq_len       int                L (None without the LSTM policy)
    state_h       bfloat16 [ceil(T/L), 2N, 256]   the LSTM state h / c the policy used at t = k L (zero where an episode
    state_c       float32 [ceil(T/L), 2N, 256]    started there)

    A learner replays chunk k from (state_h[k], state_c[k]) and zeroes the state before step t > k L wherever
    dones[t - 1] (the environment auto-reset: a new episode starts at t), as ``RllibLSTMShapedCNN.forward_sequence`` does
    with ``reset[t] = dones[t - 1]`` (``reset[k L]`` = 0: the stored state already follows the rule).

    ``one_view`` (``AgentPairRollout.collect``: a learner next to a different agent): ONE row per environment, the learner's.
    Every [T, 2N] / [2N] field above is then [T, N] / [N] (row e: the learner of environment e, at player
    ``1 - partner_seat[t, e]``), ``state_h`` / ``state_c`` are [ceil(T/L), N, 256], ``partner_seat`` is agent 1's player and
    ``learner_mask`` is all ones.  Next to a population of partners (``members``) ``partner_member`` int8 [T, N] is the member
    agent 1 was at transition t, and ``episodes.finished()`` has ``partner_member``; both are None / absent otherwise.
    """

    def __init__(self, env, n_steps, keep_logits=False, partner=False, seq_len=None, one_view=False, members=False, pairs=False):
        N, T, dev = env.n_envs, int(n_steps), env.device
        R = N if one_view else 2 * N
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
        self.env = env
        self.one_view = bool(one_view)
        self.states = z((T, N, env.state_words), torch.int32)
        self.actions = z((T, R), torch.int32)
        self.logp, self.values, self.rewards, self.advantages, self.value_targets = (z((T, R), torch.float32) for _ in range(5))
        self.dones = z((T, N), torch.uint8)
        self.last_values = z(R, torch.float32)
        self.logits = z((T, R, 8), torch.float32) if keep_logits else None
        self.terminal_values = None  # set by collect(bootstrap_horizon=True)
        self.partner_seat = z((T, N), torch.int8) if partner or one_view else None
        self.partner_member = z((T, N), torch.int8) if members else None
        self.pair = z((T, N, 2), torch.int8) if pairs else None
        self.episodes = EpisodeRecords(env, -(-T // env.horizon) if env.horizon > 0 else 0, members=members, pairs=pairs)
        self.seq_len = seq_len
        self.state_h = z((-(-T // seq_len), R, 256), torch.bfloat16) if seq_len else None
        self.state_c = z((-(-T // seq_len), R, 256), torch.float32) if seq_len else None

    @property
    def learner_mask(self):
        """uint8 [T, 2N] (``one_view``: [T, N]): 1 on the rows the PPO agent acted on — both rows of a self-play environment,
        the non-partner row otherwise, every row of a one-view batch.  Computed from ``partner_seat``."""
        T, N = self.dones.shape
        if self.one_view:
            return torch.ones((T, N), dtype=torch.uint8, device=self.dones.device)
        if self.partner_seat is None:
            return torch.ones((T, 2 * N), dtype=torch.uint8, device=self.dones.device)
        agent = torch.arange(2, dtype=torch.int8, device=self.dones.device)
        return (self.partner_seat.unsqueeze(-1) != agent).to(torch.uint8).view(T, 2 * N)

    def observations(self, env_steps, dtype=torch.float32):
        """lossless_state_encoding ``[M, 2, W, H, 26]`` of the env-steps ``env_steps`` (CUDA int64 [M], flat indices
        ``t * N + env``), both agents' views in [env][agent] order: rows ``2 m + i`` of the flattened per-agent tensors
        (``actions.view(-1, 2)[env_steps]`` etc.) belong to view ``i`` of entry ``m``.  Encoded from the stored records by K2.
        ``one_view``: the learner's view only, ``[M, W, H, 26]`` (row m belongs to ``actions.view(-1)[env_steps[m]]``)."""
        recs = self.states.view(-1, self.states.shape[-1]).index_select(0, env_steps)
        if not self.one_view:
            return self.env.lossless_state_encoding(dtype=dtype, states=recs)
        learner = (1 - self.partner_seat.view(-1).index_select(0, env_steps)).to(torch.int32).contiguous()  # view_swap: this view first
        return self.env.lossless_state_encoding(dtype=dtype, states=recs, view_swap=learner)[:, 0]

    def forward(self, model, env_steps, fused_first_layer=None):
        """(logits float32 [rows, 6], values float32 [rows]) of ``model`` (``RllibShapedCNN``, e.g. the learner after some
        updates) on the env-steps ``env_steps``, with autograd to ``model``'s parameters, in the row order of
        ``observations(env_steps)``: both views (rows ``2 m + i``), or the learner's view in a ``one_view`` batch.

        The network is the fold the rollout runs, at its precision (``records_forward``), evaluated from the stored records:
        where K7 takes the grid and the layout count, the first layer is K7 on the records (its output bit for bit what the
        behaviour policy's K7 computed from the same weights) and its weight gradient is K12; no observation is written.
        Else the first layer reads K2's bf16 observation.  Not for ``RllibLSTMShapedCNN`` (use ``forward_sequence``)."""
        recs = self.states.view(-1, self.states.shape[-1]).index_select(0, env_steps)
        if not self.one_view:
            return records_forward(model, self.env, recs, fused_first_layer=fused_first_layer)
        # the learner is player 1 - partner_seat = 1 ^ partner_seat
        swap = self.partner_seat.view(-1).index_select(0, env_steps).to(torch.int32).contiguous()
        return records_forward(model, self.env, recs, seat=1, swap=swap, fused_first_layer=fused_first_layer)


# The BC partner's draws use their own Philox keys: seed ^ PARTNER_DRAW_SALT for K10's action draw, seed ^ PARTNER_SEAT_SALT
# for the seat draw.  A partner action is then never drawn from the noise the PPO draw (key = seed) used on the same row and
# step, and the seat draw's counters (env, step) cannot meet the action draws' (row, step, block).
PARTNER_DRAW_SALT = 0x9E3779B97F4A7C15
PARTNER_SEAT_SALT = 0xD1B54A32D192ED03


class _FoldedPolicy(object):
    """A PPO network in the form the policy kernels take: ``model`` (``RllibShapedCNN`` or ``RllibLSTMShapedCNN``), its
    ``DenseGridPolicy`` and the K7 / K9 / K8 / K11 tables, with the kernels ``fused_kernel_support`` allows on ``env``'s grid.
    ``SelfPlayRollout`` evaluates it on both views of every environment, an ``AgentPairRollout`` agent on one."""

    def _fold(self, env, model, autocast_dtype, fused_first_layer, fused_tail, fused_wide):
        """See ``SelfPlayRollout.__init__`` for the arguments; ``self.env`` is ``env``."""
        assert len({(l.width, l.height) for l in env.layouts}) == 1, "one grid shape per rollout (group envs by layout)"
        assert autocast_dtype in (torch.bfloat16, None), "the dense model runs in bfloat16, or in float32 with None"
        l = env.layouts[0]
        self.W, self.H = l.width, l.height
        dev = env.device
        self.model = (model or RllibShapedCNN(self.W, self.H)).to(dev).eval()
        self.lstm = isinstance(self.model, RllibLSTMShapedCNN)
        assert not self.lstm or autocast_dtype == torch.bfloat16, \
            "the LSTM policy runs as ovc_lstm_head (K11), which takes bfloat16 operands: autocast_dtype=None is not supported"
        self.autocast_dtype = autocast_dtype
        self.dense_model = DenseGridPolicy(self.model, self.W, self.H, pad_to=16).to(dev).eval()
        if self.lstm:  # folded before the cast: K11's gate bias is the float32 sum of the model's float32 biases
            self._lstm_tables = self.dense_model.lstm_tables()
        if autocast_dtype is not None:
            self.dense_model = self.dense_model.to(autocast_dtype)
        bf16 = autocast_dtype == torch.bfloat16
        k7_ok, k9_ok, k8_ok = fused_kernel_support(self.dense_model, self.W, self.H, env.n_layouts)
        if fused_first_layer is None:
            fused_first_layer = bf16 and k7_ok
        assert not fused_first_layer or (bf16 and k7_ok), \
            "K7 feeds the bf16 policy (first layer width a multiple of 64, table within shared memory, at most %d layouts; " \
            "this environment has %d)" % (K7_MAX_LAYOUTS, env.n_layouts)
        self.fused_first_layer = bool(fused_first_layer)
        if self.fused_first_layer:
            self._wt0, self._b0 = self.dense_model.first_layer_table()
        if fused_tail is None:
            fused_tail = bf16 and k8_ok
        assert not fused_tail or (bf16 and k8_ok), \
            "K8 ends the bf16 policy (64-wide tail behind an input of a multiple of 32, <= 256)"
        self.fused_tail = bool(fused_tail)
        if self.fused_tail:
            self._tail = self.dense_model.hidden_tables() if self.lstm else self.dense_model.tail_tables()
        if fused_wide is None:
            fused_wide = self.fused_tail and self.fused_first_layer and k9_ok
        assert not fused_wide or (self.fused_tail and self.fused_first_layer and k9_ok), \
            "K9 sits between K7 and K8 and is built for 512 -> 512 -> 160"
        self.fused_wide = bool(fused_wide)
        if self.fused_wide:
            self._wide = self.dense_model.wide_tables()

    def sync_weights(self):
        """Re-fold ``self.model`` (e.g. after a learner's update) into the policy the kernels evaluate, in place: the dense
        model's parameters and the K7 / K9 / K8 tables keep their storage, so the captured graphs of run() and collect()
        use the new weights without a re-capture."""
        with torch.no_grad():
            new = DenseGridPolicy(self.model, self.W, self.H, pad_to=16).to(self.env.device)
            pairs = list(zip(self._lstm_tables, new.lstm_tables())) if self.lstm else []  # from the float32 fold, as in __init__
            if self.autocast_dtype is not None:
                new = new.to(self.autocast_dtype)
            for dst, src in zip(self.dense_model.parameters(), new.parameters()):
                dst.copy_(src)
            if self.fused_first_layer:
                pairs += zip((self._wt0, self._b0), self.dense_model.first_layer_table())
            if self.fused_wide:
                pairs += zip(self._wide, self.dense_model.wide_tables())
            if self.fused_tail:
                pairs += zip(self._tail, self.dense_model.hidden_tables() if self.lstm else self.dense_model.tail_tables())
            for dst, src in pairs:
                dst.copy_(src)

    def _chain_buffers(self, rows):
        """The buffers of ``_chain`` on ``rows`` rows: K7's output, K8's input (the last convolution's pre-activation), the
        library layers' logits, and the LSTM's input and live state (zero at every episode start)."""
        dev = self.env.device
        if self.fused_first_layer:
            self._act0 = torch.empty((rows, self._wt0.shape[1]), dtype=torch.bfloat16, device=dev)
        if self.fused_tail:
            self._z = torch.empty((rows, self._tail[0].shape[1]), dtype=torch.bfloat16, device=dev)
        self._scores = torch.empty((rows, 6), dtype=torch.float32, device=dev)
        if self.lstm:
            cell = self.model.lstm.hidden_size
            self._x = torch.empty((rows, self.model.lstm.input_size), dtype=torch.bfloat16, device=dev)
            self.h = torch.zeros((rows, cell), dtype=torch.bfloat16, device=dev)
            self.c = torch.zeros((rows, cell), dtype=torch.float32, device=dev)

    def _horizon_values_rows(self, h, partner_seat, one_view, out, counter, actions):
        """The horizon bootstrap's value pass on K7 -> K9 -> K8: ``ovc_horizon_rows`` compacts the learner rows of the
        environments that just ended (their terminal records, views and output rows) and zeroes ``out``; K7's rows form
        on those records, K9 and K8's joint form on the compact range then write each row's value at its output row of
        ``out``.  With no environment done every launch finds an empty range.  K8's draws go to the scratch ``counter`` and
        ``actions``.  ``h``: the buffers of ``_Rollout._horizon_buffers``."""
        env, lib, st = self.env, _native.lib(), self.env._stream()
        rows = self._act0.shape[0]
        env.horizon_rows(partner_seat, one_view, h.records, h.view, h.jrow, h.range, out)
        _native.check(lib.ovc_encode_linear_rows(
            env.tables.data_ptr(), env.n_layouts, h.records.data_ptr(), h.view.data_ptr(), 0, h.ident.data_ptr(), h.range.data_ptr(),
            self._wt0.data_ptr(), self._b0.data_ptr(), self._act0.data_ptr(), rows, env.state_words, self.W, self.H,
            env.horizon if env.horizon > 0 else 2**31 - 1, self._wt0.shape[1], 0.2, st))
        _native.check(lib.ovc_wide_layers_range(*self._k9_args(self._act0), h.range.data_ptr(), self._z.data_ptr(), st))
        _native.check(lib.ovc_policy_tail_joint(*self._k8_args(self._z), counter.data_ptr(), h.jrow.data_ptr(), h.range.data_ptr(),
                                                actions.data_ptr(), out.data_ptr(), 0, h.logp.data_ptr(), st))

    def _k9_args(self, x, tables=None):
        """``ovc_wide_layers``' arguments (and its range and grouped forms') up to the slope, on the rows of ``x``
        [rows, k0]: ``tables`` (default this policy's) may be a member stack."""
        w1, b1, w2, b2 = self._wide if tables is None else tables
        return (x.data_ptr(), x.shape[0], x.shape[1], w1.data_ptr(), b1.data_ptr(), w1.shape[-2], w2.data_ptr(), b2.data_ptr(),
                w2.shape[-2], 0.2)

    def _k8_args(self, x, tables=None):
        """K8's arguments on the rows of ``x`` [rows, k0]: up to the seed for the drawing forms (``ovc_policy_tail`` and its
        view, rows, joint and grouped forms), up to the dense slope for ``ovc_policy_hidden`` (LSTM policy).  ``tables``
        (default this policy's) may be a member stack."""
        w1, b1, wh, bh = (self._tail if tables is None else tables)[:4]
        args = (x.data_ptr(), x.shape[0], x.shape[1], 0.2, w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(), wh.shape[-3])
        if self.lstm:
            return args + (self.dense_model.dense_slope,)
        wo, bo = (self._tail if tables is None else tables)[4:]
        return args + (wo.data_ptr(), bo.data_ptr(), 0.3, self.dense_model.n_actions, self.seed & (2**64 - 1))

    def _chain(self, flat, actions, values, logp, scores8, counter, view=None, state_out=None, snap=None):
        """The policy after its first layer, on the rows of ``flat`` (K7's output, else the observation's rows): K9 or the
        library trunk, then K8's draw; or K8's hidden output (or the library layers) and K11 on the live state, which it
        writes to ``state_out`` (h, c) (default in place) and, as it used it, to ``snap``; or the library layers to
        ``self._scores`` and ``values``.  ``view`` None: both views of every environment (the two-view entry points), and
        the library path returns the logits for the caller to draw from.  ``view`` (seat, swap): one view per environment
        (the ``_view`` entry points, ``sample_actions_view``).  Returns None once the actions are drawn."""
        env, lib, stream = self.env, _native.lib(), self.env._stream()
        ptr = lambda t: 0 if t is None else t.data_ptr()
        first = 1 if self.fused_first_layer else 0
        with torch.no_grad():
            if self.fused_wide:
                _native.check(lib.ovc_wide_layers(*self._k9_args(flat), self._z.data_ptr(), stream))
            elif self.fused_tail:
                self.dense_model.trunk(flat, first, out=self._z)
            if self.lstm:
                if self.fused_tail:
                    _native.check(lib.ovc_policy_hidden(*self._k8_args(self._z), self._x.data_ptr(), stream))
                else:
                    self._x.copy_(self.dense_model.hidden_from(flat, first))
                w, b, wo, bo = self._lstm_tables
                h_out, c_out = state_out or (self.h, self.c)
                snap_h, snap_c = snap or (None, None)
                head = (self._x.data_ptr(), self.h.data_ptr(), self.c.data_ptr(), env.done.data_ptr(), self._x.shape[0], w.data_ptr(),
                        b.data_ptr(), wo.data_ptr(), bo.data_ptr(), self.dense_model.n_actions, self.seed & (2**64 - 1),
                        counter.data_ptr()) + (() if view is None else (ptr(view[1]), view[0]))
                out = (h_out.data_ptr(), c_out.data_ptr(), ptr(snap_h), ptr(snap_c), actions.data_ptr(), ptr(values), ptr(logp),
                       ptr(scores8), stream)
                _native.check((lib.ovc_lstm_head if view is None else lib.ovc_lstm_head_view)(*head, *out))
                return None
            if self.fused_tail:
                args = self._k8_args(self._z) + (counter.data_ptr(),)
                if view is not None:
                    _native.check(lib.ovc_policy_tail_view(*args, ptr(view[1]), view[0], actions.data_ptr(), values.data_ptr(),
                                                           ptr(scores8), ptr(logp), stream))
                elif logp is None:
                    _native.check(lib.ovc_policy_tail(*args, actions.data_ptr(), values.data_ptr(), ptr(scores8), stream))
                else:
                    _native.check(lib.ovc_policy_tail_logp(*args, actions.data_ptr(), values.data_ptr(), ptr(scores8), logp.data_ptr(),
                                                           stream))
                return None
            logits, value = self.dense_model.forward_from(flat, first)
            self._scores.copy_(logits)
            values.copy_(value)
            if view is None:
                return self._scores
            env.sample_actions_view(self._scores, counter, view[0], view[1], seed=self.seed, out=actions, logp_out=logp)
            if scores8 is not None:
                scores8[:, :self._scores.shape[1]].copy_(self._scores)
        return None


PHI_GAMMA = 0.99  # the gamma of the reference's use_phi reward (get_state_transition(display_phi=True), MDP:1422-1429)


class _PhiReward(object):
    """use_phi's scratch: phi(s) (float64 [N]) and the dense reward (float32 [N]), both rewritten every transition, so
    neither is state a captured graph has to restore.  The 0.99 potential tables are built here, never inside a capture."""

    def __init__(self, env):
        assert env.auto_reset, "use_phi needs an auto_reset environment: ovc_potential_shaping resets every episode that ends"
        env.potential_tables(PHI_GAMMA)
        self.phi_s = torch.empty(env.n_envs, dtype=torch.float64, device=env.device)
        self.dense = torch.empty(env.n_envs, dtype=torch.float32, device=env.device)


def _env_step(env, actions, phi, terminal=None):
    """K1 with its auto-reset; with ``phi`` (a ``_PhiReward``), K6 on s, K1 without the reset, then
    ovc_potential_shaping (phi(s') on the terminal records, the dense reward, the reset).  ``terminal`` (a callable, the
    horizon bootstrap's value pass) runs between K1 without the reset and the reset (``env.reset_ended()``, or inside
    ovc_potential_shaping with ``phi``), while the ended environments still hold their terminal records.  Returns the
    dense reward for the record (None without ``phi``)."""
    if phi is None and terminal is None:
        env.step(actions)  # K1 (auto-reset inside)
        return None
    if phi is not None:
        env.potential(PHI_GAMMA, out=phi.phi_s)  # K6
    env.step(actions, auto_reset=False)
    if terminal is not None:
        terminal()
    if phi is None:
        env.reset_ended()
        return None
    return env.potential_shaping(phi.phi_s, phi.dense)


def _capture_graph(env, live, warm_up, body):
    """A CUDA graph of ``body``, captured after ``warm_up`` (on a side stream).  The tensors ``live`` (what warm-up and
    capture advance: the state, returns, statistics, counters...) are restored after them."""
    saved = [t.clone() for t in live]
    dev = env.device
    s = torch.cuda.Stream(dev)
    s.wait_stream(torch.cuda.current_stream(dev))
    with torch.cuda.stream(s):
        warm_up()
    torch.cuda.current_stream(dev).wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        body()
    for t, v in zip(live, saved):
        t.copy_(v)
    return graph


# A population of learners runs grouped K9 from this many members on; below it, K9 per member on its block is faster
# (cramped_room, 32 768 envs, inside a CUDA graph on an H100 80GB HBM3 at 700 W: 103.1 / 109.3 us grouped against
# 89.9 / 101.1 us for K = 1 / 2, 110.1 against 116.3 us for K = 4; tools/prof_selfplay_population.py).
GROUPED_K9_MIN_MEMBERS = 4


def _check_members(members, most, kinds, count_msg, kind_msg):
    """The checks on a population of models: 1..``most`` members, each an instance of ``kinds`` and none an
    ``RllibLSTMShapedCNN`` (K11 has no rows or grouped form)."""
    assert 1 <= len(members) <= most, count_msg
    for m in members:
        assert isinstance(m, kinds) and not isinstance(m, RllibLSTMShapedCNN), kind_msg


class _Rollout(object):
    """The rollout driver of ``SelfPlayRollout`` and ``AgentPairRollout``: run() and collect() over the subclass's
    ``_transition(b, t)``, their CUDA graphs, the bootstrap step's scratch and GAE, the returns, the episode statistics and
    records, the shaping factor, the seat draw and the population's members.  A subclass provides ``_transition``,
    ``_live()`` (the tensors a transition advances besides the state, the returns, the statistics and the records),
    ``_bootstrap(b)`` (the learner's value of the state after a window into ``b.last_values``), ``_new_batch(n_steps,
    keep_logits)`` and ``_agents()`` (its policies); it sets ``population``, ``_pop`` (the population, or None) and
    ``_member``."""

    def _init_rollout(self, env, learner, use_graph, reward_shaping_factor, episode_capacity, max_seq_len, pairs=False):
        """The shared state; ``learner`` is the policy whose LSTM state (if any) the bootstrap step leaves alone, ``pairs``
        (population play) makes the episode records hold each episode's pair."""
        N, dev = env.n_envs, env.device
        self.use_graph = use_graph
        self.actions = torch.zeros((N, 2), dtype=torch.int32, device=dev)
        self.ret_sparse = torch.zeros(N, dtype=torch.int64, device=dev)  # running episode return (sparse)
        self.factor = float(reward_shaping_factor)
        self._factor = torch.full((1,), self.factor, dtype=torch.float32, device=dev)  # read by the captured graphs
        self.stats = EpisodeStats(env)
        self.episodes = EpisodeRecords(env, episode_capacity, members=self.population, pairs=pairs)
        self.max_seq_len = int(max_seq_len)
        assert self.max_seq_len >= 1
        self.graph = None          # run()'s CUDA graph of one transition
        # (n_steps, keep_logits), and "bootstrap_horizon" after them with the flag -> ((gamma, lam), CUDA graph of the window)
        self._collect_graphs = {}
        self._batches = {}         # the same keys -> SampleBatch the window writes
        self._horizon = None       # the horizon bootstrap's buffers (_horizon_buffers), made at its first collect()
        self._boot_counter = torch.zeros(2, dtype=torch.int64, device=dev)  # the bootstrap's draws leave the learner's counter alone
        self._boot_actions = torch.zeros((N, 2), dtype=torch.int32, device=dev)
        if learner.lstm:  # the bootstrap's (discarded) LSTM state: the next window continues from the live state
            self._h_boot, self._c_boot = torch.empty_like(learner.h), torch.empty_like(learner.c)

    @property
    def reward_shaping_factor(self):
        """The factor of the shaped rewards (rllib.py:328-329) in the rewards, the returns and the episode records'
        ``ep_reward_by_agent``.  Setting it takes effect in run() and collect() alike, without a re-capture (their graphs
        read a device scalar)."""
        return self.factor

    @reward_shaping_factor.setter
    def reward_shaping_factor(self, value):
        self.factor = float(value)
        self._factor.fill_(self.factor)

    @property
    def member_weights(self):
        """The population's draw weights (K non-negative floats with a positive sum).  Setting them writes the device
        table the draw reads, so run() and collect() follow a new distribution at the next episode ends without a re-capture
        (prioritised sampling of the population between windows)."""
        assert self._pop is not None and self._pop._thresholds is not None, "member_weights: a population drawn per episode"
        return self._pop.weights

    @member_weights.setter
    def member_weights(self, value):
        assert self._pop is not None and self._pop._thresholds is not None, "member_weights: a population drawn per episode"
        self._pop.weights = value

    @property
    def member(self):
        """int32 [N]: with a population of partners, each environment's member in its running episode (in a self-play
        mixture it plays only where ``partner_seat >= 0``); with a population of learners, the member that plays environment
        e (fixed); else None."""
        return self._member if self._pop is None else self._pop.member

    def _assign_seats(self, done):
        """The seat draw (``env.assign_partners``): ``partner_seat`` for every environment whose episode ended (done None:
        every environment), paired with probability ``_bc_factor``."""
        self.env.assign_partners(self.partner_seat, self._bc_factor, self._seat_counter, seed=self.seed ^ PARTNER_SEAT_SALT, done=done)

    def _capture(self, warm_up, body):
        """A CUDA graph of ``body``, captured after ``warm_up`` (on a side stream).  Warm-up and capture must not advance
        the environments: the state, the returns, the episode statistics and records, the draw counters and the seats are
        restored after them."""
        live = [self.env.state, self.ret_sparse] + self.stats.state_tensors() + self.episodes.tensors() + self._live()
        return _capture_graph(self.env, live, warm_up, body)

    def run(self, n_steps):
        """Advance every environment n_steps transitions (one CUDA graph per transition with use_graph); returns the number
        of env-steps done."""
        if self.use_graph and self.graph is None:
            def warm_up():
                for _ in range(3):
                    self._transition()
            self.graph = self._capture(warm_up, self._transition)
        step = self._transition if self.graph is None else self.graph.replay
        for _ in range(n_steps):
            step()
        return n_steps * self.env.n_envs

    def _collect_window(self, b, n_steps, gamma, lam):
        """n_steps transitions into slots 0.. of ``b``, then the bootstrap value of the state after them and GAE over the
        whole batch."""
        b.episodes.clear()
        for t in range(n_steps):
            self._transition(b, t)
        self._bootstrap(b)
        if b.terminal_values is not None:
            self.env.gae_horizon(b.rewards, b.values, b.dones, b.terminal_values, b.last_values, gamma, lam, b.advantages,
                                 b.value_targets, one_view=b.one_view)
            return
        gae = self.env.gae_view if b.one_view else self.env.gae
        gae(b.rewards, b.values, b.dones, b.last_values, gamma, lam, b.advantages, b.value_targets)

    def collect(self, n_steps, gamma, lam, keep_logits=False, bootstrap_horizon=False):
        """Advance every environment n_steps transitions, as run() does (the same kernels and the same draws from the same
        seed and counters), and return them as a ``SampleBatch`` with GAE(gamma, lam) advantages.  The batch's tensors are
        reused: the next collect() with the same n_steps / keep_logits / bootstrap_horizon overwrites them.  With use_graph
        the whole window is one CUDA graph (captured once per n_steps / keep_logits / bootstrap_horizon; a new gamma or lam
        re-captures it); no host synchronisation otherwise.  With a population, the batch's ``partner_member`` is each
        transition's member.

        bootstrap_horizon: every episode ends at the horizon, a time limit, and no state of the MDP is terminal; by default
        (RLlib's GAE, which the reference trains with) the state after the last step still counts as terminal.  With
        bootstrap_horizon the learner's value head is evaluated on the terminal record of every environment that ends
        (between K1, run without its auto-reset, and the reset; only the ended environments' learner rows are evaluated),
        stored in the batch's ``terminal_values``, and GAE bootstraps from it (``ovc_gae_horizon``): delta = r + gamma *
        V(s_T) - V(s).  Every other field of the batch, the environments, the counters, the episode records and the
        statistics are bit for bit those of the same collect() without it.  Not for an LSTM learner, a population of
        learners or an environment without auto_reset."""
        if bootstrap_horizon:
            self._check_bootstrap_horizon()
        assert self.env.auto_reset, "collect() needs an auto_reset environment: a window runs across episode ends"
        key = (int(n_steps), bool(keep_logits)) + ("bootstrap_horizon",) * bool(bootstrap_horizon)
        b = self._batches.get(key)
        if b is None:
            b = self._new_batch(n_steps, keep_logits)
            if bootstrap_horizon:
                b.terminal_values = torch.zeros_like(b.values)
                self._horizon_buffers()
            self._batches[key] = b
        if not self.use_graph:
            self._collect_window(b, n_steps, gamma, lam)
            return b
        g = self._collect_graphs.get(key)
        if g is None or g[0] != (gamma, lam):
            g = self._collect_graphs[key] = ((gamma, lam), self._capture(lambda: self._collect_window(b, 1, gamma, lam),
                                                                         lambda: self._collect_window(b, n_steps, gamma, lam)))
        g[1].replay()
        return b

    def _check_bootstrap_horizon(self):
        """The configurations collect(bootstrap_horizon=True) refuses."""
        assert self.env.auto_reset, "bootstrap_horizon needs an auto_reset environment: the terminal states are evaluated " \
            "between the step and the reset of the episodes that end"
        assert getattr(self, "_learners", None) is None, \
            "bootstrap_horizon is not supported for a population of learners (blocks or population play)"
        assert not self._agents()[0].lstm, "bootstrap_horizon is not supported for an LSTM learner: the value of the terminal " \
            "state needs one more ovc_lstm_head step on a scratch copy of the recurrent state"

    def _horizon_buffers(self):
        """The horizon bootstrap's scratch on the learner's rows (2N, or N for one view): the compaction's records, views,
        output rows, identity rows map, range and K8's logp where the learner runs K7 -> K9 -> K8, else the full value
        pass's values."""
        if self._horizon is not None:
            return
        learner, env = self._agents()[0], self.env
        rows = 2 * env.n_envs if learner is self else env.n_envs
        i32 = lambda *shape: torch.zeros(shape, dtype=torch.int32, device=env.device)
        h = SimpleNamespace(fused=learner.fused_first_layer and learner.fused_wide and learner.fused_tail)
        if h.fused:
            h.records, h.view, h.jrow, h.range = i32(rows, env.state_words), i32(rows), i32(rows), i32(2)
            h.ident = torch.arange(rows, dtype=torch.int32, device=env.device)
            h.logp = torch.zeros(rows, dtype=torch.float32, device=env.device)
        else:
            h.values = torch.zeros(rows, dtype=torch.float32, device=env.device)
            h.zero = torch.zeros((), dtype=torch.float32, device=env.device)
        self._horizon = h

    def reset_state(self):
        """Zero the LSTM policies' live state and forget the greedy agents' previous states.  run() and collect() do both at
        every auto-reset (through ``env.done``); call this after resetting the environments directly (``env.reset()``), so
        that the new episodes start from zero state."""
        for a in self._agents():
            if a.lstm:
                a.h.zero_(), a.c.zero_()
        for a in self._agents() + [getattr(self, "_partner", None)]:
            if isinstance(a, _GreedyAgent):  # no previous state for the stuck rule, as Agent.reset()
                a.prev.zero_()


class SelfPlayRollout(_FoldedPolicy, _Rollout):
    """Policy-in-the-loop rollout: both agents of every environment act from the same network, or, with a ``partner``,
    one seat of an environment is the partner's in the episodes the seat draw gives it (PPO_BC, or a self-play mixture with
    a frozen network or a population).  The network evaluated is
    ``DenseGridPolicy`` of ``model``: K7 / K9 / K8 where they fit (``fused_kernel_support``; K7, and K9 behind it, only with
    at most 8 layouts in ``env``), library GEMMs and the draw kernel elsewhere."""

    def __init__(self, env, model=None, autocast_dtype=torch.bfloat16, use_graph=True, reward_shaping_factor=1.0,
                 fused_first_layer=None, seed=0, fused_tail=None, fused_wide=None, partner=None, bc_factor=0.0, episode_capacity=1,
                 max_seq_len=20, member=None, member_weights=None, use_phi=False, blocks=None, pairs=None, pair_weights=None):
        """autocast_dtype: the dtype of the dense model (``DenseGridPolicy``, widths padded to 16-byte rows) and of the
        observation K2 writes for it: bfloat16 (the plane values are exact in bf16), or None for float32 throughout.
        fused_first_layer (default: on for the bf16 policy where ``fused_kernel_support`` allows K7): the observation is
        never materialised — kernel K7 (``env.encoded_linear``) evaluates encoding + first layer + leaky ReLU from the
        packed records, and the library GEMMs start at the second layer.  K7 takes at most 8 layouts per call: on a larger
        layout pool the default is off (K2 writes the observation) and an explicit True is refused here.
        fused_tail (default: on for the bf16 policy): the dense layers of 64, the heads and the draw run as ONE kernel
        (``ovc_policy_tail``, K8) on the last convolution's pre-activation; the library GEMMs are then only the two wide
        layers.  Without it the joint action is drawn by ``ovc_sample_actions`` (Gumbel-max on Philox draws keyed by
        ``seed``, one kernel).
        fused_wide (default: with K7 and K8 when the wide layers are 512 -> 512 -> 160, i.e. on 5x4 grids): those two layers
        run as ONE wgmma kernel (``ovc_wide_layers``, K9: the 512-wide activation stays in registers) — the
        whole policy is then K7 -> K9 -> K8, no library call.
        partner: a ``BCPolicy`` that plays next to the PPO agent (PPO_BC, human_aware_rl's OvercookedMultiAgent): at every
        episode start (and for every environment at construction) an environment gets the partner with probability
        ``bc_factor``, in seat 0 or 1 with equal probability (``env.assign_partners``); per transition K10
        (``env.partner_actions``) overwrites that seat's action after the PPO policy drew both.  partner may also be a
        ``GreedyHumanModel`` (the reference's scripted partner, no weights needed), in the same seats and episodes:
        ``env.greedy_actions`` then overwrites the seat's action.
        partner may instead be a frozen ``RllibShapedCNN`` or a population: a list of 1..63 members, each an ``RllibShapedCNN``
        or a ``BCPolicy`` (a self-play mixture: each episode is self-play with probability ``1 - bc_factor``, else played
        next to the partner, or next to the population member the environment holds).  The partner, or member k, then
        evaluates only the seat it holds in the paired environments that play it (``ovc_group_members`` over the paired
        environments; a network member runs the rows forms of K7 / K9 / K8, a BC member K10), and never writes a self-play
        row.  A network partner draws with key ``seed`` on a counter of its own, a BC member with ``seed ^
        PARTNER_DRAW_SALT``: ``partner=copy.deepcopy(model)`` draws exactly what self-play draws.  Where the learner runs K7,
        K9 and K8, it evaluates only its own rows (``ovc_learner_rows``, ``ovc_encode_linear_masked``, K9 on the compact
        rows, ``ovc_policy_tail_joint``); the partner rows' values, logp and advantages are then not written.  Other learners
        run on all 2N rows, as without a partner.  LSTM partners and members are refused (K11 has no rows form).
        member, member_weights: with a population only, as ``AgentPairRollout``'s: a fixed member per environment, or one
        drawn at construction and at every episode end (uniform by default), whether or not the next episode is paired.
        ``episodes.finished()`` and collect()'s batches then report ``partner_member``, meaningful where ``partner_seat >= 0``.
        bc_factor: see the property.
        episode_capacity: episodes per environment that ``self.episodes`` holds (an ``EpisodeRecords``): every episode that
        ends in run() is written there, up to this many per environment since ``self.episodes.clear()`` (the rest are
        counted in ``episodes.dropped``).  ``self.stats`` (an ``EpisodeStats``) is the running state of the episodes in
        progress, shared by run() and collect(): an episode may span windows and both calls.
        model: an ``RllibShapedCNN`` (default, random init) or an ``RllibLSTMShapedCNN`` (``use_lstm``).  The LSTM policy runs
        the same trunk, then the dense layers (K8's hidden output, ``ovc_policy_hidden``, where K8 fits, else library GEMMs),
        then K11 (``ovc_lstm_head``: the LSTM cell, the heads and the draw) on the live state ``self.h`` (bf16 [2N, 256]) /
        ``self.c`` (float32 [2N, 256]), zeroed at every auto-reset (K11 is passed the previous transition's ``env.done``); after
        an ``env.reset()`` outside run() / collect(), call ``reset_state()``.  It needs the bf16 policy.  The LSTM's tables
        are folded from the float32 model (the gate bias is one float32 sum of its two biases).
        max_seq_len: RLlib's model-config key for the LSTM policy: collect() records the state every ``max_seq_len``
        transitions (``SampleBatch.state_h`` / ``state_c``).
        use_phi: the reference's potential-based dense reward (rllib.py:314-329): both agents get ``sparse +
        reward_shaping_factor * (phi(s') - phi(s))``, phi at gamma 0.99 with s' taken before an ending episode's reset,
        instead of ``sparse + reward_shaping_factor * shaped_i``.  Only the rewards, the returns, the advantages, the value
        targets and the episodes' reward sums change; the draws, the states and the game statistics are those without it.
        Needs an ``auto_reset`` env.
        model may instead be a population of self-play learners: a list of 1..64 ``RllibShapedCNN`` members of one
        architecture, each playing both views of its block of environments (``blocks``), or paired per environment
        (population play: ``pairs`` or ``pair_weights``).  See ``_Learners`` for both forms; ``self.blocks``, ``self.member``,
        ``self.pair`` and ``self.pair_weights`` describe the population, and ``sync_weights()`` refolds every member.  Not
        with a ``partner`` or an ``RllibLSTMShapedCNN`` member."""
        assert not isinstance(model, GreedyHumanModel), "a GreedyHumanModel does not learn: pass it as the partner"
        self.env = env
        self.seed = int(seed)
        models = list(model) if isinstance(model, (list, tuple)) else None
        self._phi = _PhiReward(env) if use_phi else None
        if models is None:
            assert pairs is None and pair_weights is None, "pairs / pair_weights go with a population of learners (a list model)"
            assert blocks is None, "blocks go with a population of learners (a list model)"
            self._fold(env, model, autocast_dtype, fused_first_layer, fused_tail, fused_wide)
            self._learners = None
        else:
            assert partner is None, "population play has no partner: every row is a learner's" \
                if pairs is not None or pair_weights is not None else "a population of learners plays self-play only: no partner with a list model"
            self._learners = _Learners(self, models, blocks, pairs, pair_weights, autocast_dtype, fused_first_layer, fused_tail, fused_wide)
        L = self._learners  # the block offsets and each environment's member (blocks), the live pairing (population play)
        self.blocks, self._member, self.pair = (None, None, None) if L is None else (L.blocks, L.member, L.pair)
        dev = env.device
        N = env.n_envs
        self.partner = partner
        self.bc = float(bc_factor)
        self.population = isinstance(partner, (list, tuple))
        if partner is not None and not isinstance(partner, GreedyHumanModel):
            _check_members(partner if self.population else [partner], MAX_MEMBERS - 1, (RllibShapedCNN, BCPolicy),
                           "a mixture's population has 1..%d members (one of ovc_group_members' %d groups holds the self-play "
                           "environments)" % (MAX_MEMBERS - 1, MAX_MEMBERS),
                           "a partner is a BCPolicy, an RllibShapedCNN or a list of them (an LSTM partner or member is not "
                           "supported in a self-play mixture: ovc_lstm_head has no rows form)")
        if not self.population:
            assert member is None and member_weights is None, "member / member_weights go with a population in partner"
        self._partner = None  # the partner's agent: a _BCAgent, or a _Population (of one for a network partner)
        self._pop = None      # the population of partners
        if partner is not None:
            self._bc_factor = torch.full((1,), self.bc, dtype=torch.float32, device=dev)  # read by the seat draw
            self.partner_seat = torch.full((N,), -1, dtype=torch.int32, device=dev)
            self._seat_counter = torch.zeros(2, dtype=torch.int64, device=dev)     # [step, scratch] of the seat draw
        if isinstance(partner, BCPolicy):
            self._partner = _BCAgent(env, partner, self.partner_seat, seed)
            self._partner_counter = self._partner._counter  # [step, scratch] of K10's draw
        elif isinstance(partner, GreedyHumanModel):
            self._partner = _GreedyAgent(env, self.partner_seat, seed)
            self._partner_counter = self._partner._counter  # [step, scratch] of the stuck draws
        elif partner is not None:
            members = list(partner) if self.population else [partner]
            if not self.population:  # one network partner: a population of one, its member fixed
                member = torch.zeros(N, dtype=torch.int32, device=dev)
            self._partner = _Population(env, members, self.partner_seat, seed, autocast_dtype, member, member_weights, mixture=True)
            self._pop = self._partner if self.population else None
        self._learner_rows = False
        self.obs = None if self.fused_first_layer else torch.empty((N, 2, self.W, self.H, 26), dtype=autocast_dtype or torch.float32, device=dev)
        self._chain_buffers(2 * N)
        self.ret_mixed = torch.zeros(N, dtype=torch.float32, device=dev)    # sparse + factor * shaped (rllib.py:328-329)
        self.values = torch.zeros((N, 2), dtype=torch.float32, device=dev)
        self.native_glue = True  # the draw and the returns are always native kernels; bench.py's launch count reads this
        self._init_rollout(env, self, use_graph, reward_shaping_factor, episode_capacity, max_seq_len, pairs=self.pair is not None)
        self._draw_counter = torch.zeros(2, dtype=torch.int64, device=dev)  # [step, scratch] of ovc_sample_actions
        self._scores8 = None  # set to a float32 [2N, 8] tensor to make K8 also write the heads (tests)
        if partner is not None:
            self._assign_seats(None)
        if isinstance(self._partner, _Population):
            if self._partner.needs_obs and self.obs is None:
                self.obs = torch.empty((N, 2, self.W, self.H, 26), dtype=autocast_dtype or torch.float32, device=dev)
            self._partner.obs = self.obs
            # the learner on its own rows only, where it runs K7 -> K9 -> K8
            self._learner_rows = self.fused_first_layer and self.fused_wide and self.fused_tail and not self.lstm
            if self._learner_rows:
                self._lst = torch.empty(N, dtype=torch.int32, device=dev)
                self._first = torch.empty(N, dtype=torch.int32, device=dev)
                self._jrow = torch.empty(2 * N, dtype=torch.int32, device=dev)
                self._lrange = torch.zeros(2, dtype=torch.int32, device=dev)
                self._logp = torch.empty(2 * N, dtype=torch.float32, device=dev)  # run()'s logp: the joint K8 always writes it

    @property
    def bc_factor(self):
        """The probability that an episode is played with the partner (human_aware_rl's ``bc_factor``, annealed by its
        ``bc_schedule``).  Setting it takes effect at the next episode starts, in run() and collect() alike, without a
        re-capture (the seat draw reads a device scalar)."""
        return self.bc

    @bc_factor.setter
    def bc_factor(self, value):
        assert self.partner is not None, "bc_factor needs a partner"
        self.bc = float(value)
        self._bc_factor.fill_(self.bc)

    @property
    def pair_weights(self):
        """Population play's pair weights (K x K non-negative floats with a positive sum; entry [i][j] weighs member i on
        player 0 next to member j on player 1).  Setting them rewrites the device thresholds the pair draw reads, so run() and
        collect() follow the new weights at the next episode ends without a re-capture."""
        assert self.pair is not None and self._learners._thresholds is not None, "pair_weights: population play with drawn pairs"
        return self._learners.pair_weights

    @pair_weights.setter
    def pair_weights(self, value):
        assert self.pair is not None and self._learners._thresholds is not None, "pair_weights: population play with drawn pairs"
        self._learners.pair_weights = value

    def sync_weights(self):
        """Re-fold the learner (``_FoldedPolicy.sync_weights``), the partner (a network partner, every population member, or
        a BC partner's K10 tables) and every member of a population of learners, in place: the captured graphs use the new
        weights without a re-capture."""
        _FoldedPolicy.sync_weights(self)
        if self._partner is not None:
            self._partner.sync_weights()
        if self._learners is not None:
            self._learners.sync_weights()

    def _agents(self):
        return [self]

    def _live(self):
        live = [self.ret_mixed, self._draw_counter]
        if self.lstm:
            live += [self.h, self.c, self.env.done]  # env.done: the next transition's LSTM reset
        if self.partner is not None:
            live += [self.partner_seat, self._seat_counter] + self._partner.live()
        if self._learners is not None:
            live += self._learners.live()
        return live

    def _policy(self, actions=None, values=None, logp=None, scores8=None, counter=None, state_out=None, snap=None):
        """(scores float32 [2N, 6] = logits, values written to ``values``) for the observations in self.obs, or None when
        K8 or K11 has also drawn the actions (into ``actions``, with ``logp`` when given).  The outputs default to
        self.actions, self.values, self._scores8 and self._draw_counter.  LSTM policy: K11 reads the live state and writes
        the new one to ``state_out`` (h, c) (default: in place), the state it used to ``snap`` (h, c) when given."""
        env = self.env
        rows = 2 * env.n_envs
        actions = self.actions if actions is None else actions
        vals = self.values.view(rows) if values is None else values
        scores8 = self._scores8 if scores8 is None else scores8
        counter = self._draw_counter if counter is None else counter
        if self._learners is not None:
            return self._learners.act(self, actions, vals, logp, scores8, counter)
        with torch.no_grad():
            if self.fused_first_layer:
                flat = env.encoded_linear(self._wt0, self._b0, out=self._act0, neg_slope=0.2)  # K7
            else:
                flat = self.obs.view(rows, self.W * self.H * 26)
        return self._chain(flat, actions, vals, logp, scores8, counter, state_out=state_out, snap=snap)

    def _policy_learner_rows(self, actions, values, logp, scores8):
        """K7 -> K9 -> K8 on the learner's rows only: both views of a self-play environment, view 1 - partner_seat[e] of a
        paired one.  Each row is drawn and written at its joint row, bit for bit what ``_policy`` writes there."""
        env, lib = self.env, _native.lib()
        env.learner_rows(self.partner_seat, self._lst, self._first, self._jrow, self._lrange)
        env.encoded_linear_masked(self._wt0, self._b0, self._lst, self._first, self._act0, neg_slope=0.2)  # K7
        _native.check(lib.ovc_wide_layers_range(*self._k9_args(self._act0), self._lrange.data_ptr(), self._z.data_ptr(), env._stream()))
        _native.check(lib.ovc_policy_tail_joint(
            *self._k8_args(self._z), self._draw_counter.data_ptr(), self._jrow.data_ptr(), self._lrange.data_ptr(), actions.data_ptr(),
            values.data_ptr(), 0 if scores8 is None else scores8.data_ptr(), (self._logp if logp is None else logp).data_ptr(),
            env._stream()))

    def _transition(self, b=None, t=0):
        """One transition: K2 or K7, the policy, the draw, K10 for the partner, K1 (auto-reset inside), the returns and the
        episode statistics, the seat draw.  Without ``b`` (run()) the actions and values go to self.actions / self.values and
        finished episodes to self.episodes; with a ``SampleBatch`` ``b`` (collect()) the transition is recorded in its slot
        ``t``: state, actions, values, logp, logits, rewards, dones and partner seats, and finished episodes in b.episodes."""
        env = self.env
        if b is None:
            actions, values, logp, logits, rewards, dones = self.actions, None, None, None, None, None
        else:
            b.states[t].copy_(env.state)
            actions, values, logp, rewards, dones = b.actions[t], b.values[t], b.logp[t], b.rewards[t], b.dones[t]
            logits = None if b.logits is None else b.logits[t]
            if b.pair is not None:
                b.pair[t].copy_(self.pair)
        if self.obs is not None:
            env.lossless_state_encoding(out=self.obs)  # K2
        snap = None
        if self.lstm and b is not None and t % b.seq_len == 0:
            snap = (b.state_h[t // b.seq_len], b.state_c[t // b.seq_len])
        if self._learner_rows:
            scores = self._policy_learner_rows(actions, self.values.view(-1) if values is None else values, logp,
                                               self._scores8 if logits is None else logits)
        else:
            scores = self._policy(actions=actions, values=values, logp=logp, scores8=logits, snap=snap)
        if scores is not None:  # library layers: the separate draw kernel
            env.sample_actions(scores, self._draw_counter, seed=self.seed, out=actions, logp_out=logp)
            if logits is not None:
                logits[:, :scores.shape[1]].copy_(scores)
        if self.partner is not None:
            if b is not None:
                b.partner_seat[t].copy_(self.partner_seat)
                if self.population:
                    b.partner_member[t].copy_(self._pop.member)
            self._partner.act(actions)  # K10, or the network partner / the population
        terminal = None
        if b is not None and b.terminal_values is not None:
            terminal = lambda: self._terminal_values(b.terminal_values[t])
        dense = _env_step(env, actions.view(env.n_envs, 2), self._phi, terminal)
        if self.population:  # before the record: both use the slot count[e] the ending episode goes to
            self._pop.assign(env.done, self.episodes if b is None else b.episodes)
        if self._learners is not None:  # before the record, likewise
            self._learners.assign(env.done, self.episodes if b is None else b.episodes)
        # the seat draw below runs after this kernel, so partner_seat is still the ending episode's
        env.record_transition(self._factor, rewards=rewards, dones=dones, ret_sparse=self.ret_sparse, ret_mixed=self.ret_mixed,
                              stats=self.stats, records=self.episodes if b is None else b.episodes,
                              partner_seat=None if self.partner is None else self.partner_seat, dense=dense)
        if self.partner is not None:
            self._assign_seats(env.done)

    def _bootstrap(self, b):
        if not self.fused_first_layer:
            self.env.lossless_state_encoding(out=self.obs)
        # the LSTM's bootstrap step writes its state to scratch: the next window continues from the live state
        self._policy(actions=self._boot_actions, values=b.last_values, counter=self._boot_counter,
                     state_out=(self._h_boot, self._c_boot) if self.lstm else None)

    def _terminal_values(self, out):
        """The horizon bootstrap's value pass into ``out`` (float32 [2N]): the learner's value on its rows of the ended
        environments, 0 elsewhere.  On K7 -> K9 -> K8 only those rows are evaluated (``_horizon_values_rows``); otherwise
        the policy runs on all 2N rows (library layers take their row count from the host) and the rows are selected."""
        h, env, N = self._horizon, self.env, self.env.n_envs
        seats = self.partner_seat if self.partner is not None else None
        if h.fused:
            self._horizon_values_rows(h, seats, False, out, self._boot_counter, self._boot_actions)
            return
        if not self.fused_first_layer:
            env.lossless_state_encoding(out=self.obs)
        self._policy(actions=self._boot_actions, values=h.values, counter=self._boot_counter)
        mine = (env.done != 0).view(N, 1)
        if seats is not None:
            mine = mine & (seats.view(N, 1) != torch.arange(2, dtype=torch.int32, device=env.device))
        torch.where(mine.expand(N, 2).reshape(-1), h.values, h.zero, out=out)

    def _new_batch(self, n_steps, keep_logits):
        """collect()'s two-view batch.  With a partner, its ``partner_seat`` / ``learner_mask`` say which rows were the
        partner's; their actions are the partner's, their logp / values / advantages are meaningless (the PPO network's, or,
        where the learner runs on its own rows only, not written); ``partner_member`` is meaningful where ``partner_seat >=
        0``.  A seat changes hands only at a done, where GAE cuts, so a learner row's advantages never read a partner step."""
        return SampleBatch(self.env, n_steps, keep_logits, partner=self.partner is not None,
                           seq_len=self.max_seq_len if self.lstm else None, members=self.population, pairs=self.pair is not None)

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


class _NetworkAgent(_FoldedPolicy):
    """One network agent of an ``AgentPairRollout``: its policy on ONE view per environment, the view of player
    ``p(e) = seat ^ swap[e]``, written to ``actions[e, p(e)]`` of the joint action.  Where K7 fits: K7's one-view form
    (``encoded_linear_view``) -> K9 on N rows -> K8's one-view draw (``ovc_policy_tail_view``), or K8's hidden output -> K11's
    one-view form (``ovc_lstm_head_view``) for the LSTM model; elsewhere rows 2 e + p(e) of the observation ``self.obs``
    (K2's output, which the pair writes once per transition for all its agents: set it before act()), the dense model on N
    rows (K7 -> library layers where K7 fits but K8 does not) and the one-view draw (``sample_actions_view``, or K11).  Its
    draws use key ``seed`` and a counter of its own, on the joint row 2 e + p(e): the numbers a self-play rollout with the
    same seed draws for that row.  ``live_seats``: ``swap`` (0 / 1 only) changes between transitions; ``follow_seats()``
    recomputes the joint rows from it."""

    def __init__(self, env, model, seat, swap, seed, autocast_dtype, live_seats=False):
        self.env = env
        self._fold(env, model, autocast_dtype, None, None, None)
        N, dev = env.n_envs, env.device
        self.seat, self.swap, self.seed, self.live_seats = int(seat), swap, int(seed), live_seats
        self._counter = torch.zeros(2, dtype=torch.int64, device=dev)  # [step, scratch] of this agent's draws
        self._scores8 = None  # set to a float32 [N, 8] tensor to make K8 / K11 also write the heads (tests)
        self.values = torch.zeros(N, dtype=torch.float32, device=dev)
        self.obs = None  # [N, 2, W, H, 26] without K7, shared with the other agent of the pair
        self._base = 2 * torch.arange(N, device=dev) + self.seat
        self._rows = 2 * torch.arange(N, device=dev) + (self.seat if swap is None else self.seat ^ (swap != 0).long())  # 2 e + p(e)
        self._chain_buffers(N)
        if not self.fused_first_layer:
            self._flat = torch.empty((N, self.W * self.H * 26), dtype=autocast_dtype or torch.float32, device=dev)

    def live(self):
        """The tensors a transition advances (restored around graph capture)."""
        return [self._counter] + ([self.h, self.c] if self.lstm else []) + ([self._rows] if self.live_seats else [])

    def follow_seats(self):
        """The joint rows 2 e + (seat ^ swap[e]) after the seats changed (swap 0 / 1)."""
        torch.add(self._base, self.swap, alpha=1 - 2 * self.seat, out=self._rows)

    def act(self, actions, values=None, logp=None, scores8=None, counter=None, state_out=None, snap=None):
        """This agent's entries of ``actions`` (int32 [N, 2]) from the current state (without K7: from ``self.obs``, K2's
        encoding of it); values into ``values`` (default ``self.values``), and, each optional, the log-probability of the
        draw into ``logp`` and the heads into ``scores8`` (float32 [N, 8]).  ``counter``: the draw's counter (default this
        agent's).  The LSTM state is zeroed where the previous transition ended an episode (``env.done``); K11 writes the new
        state to ``state_out`` (h, c) (default: in place) and the state it used to ``snap`` (h, c) when given."""
        env, N = self.env, self.env.n_envs
        values = self.values if values is None else values
        scores8 = self._scores8 if scores8 is None else scores8
        counter = self._counter if counter is None else counter
        with torch.no_grad():
            if self.fused_first_layer:
                flat = env.encoded_linear_view(self._wt0, self._b0, self.seat, self.swap, out=self._act0, neg_slope=0.2)  # K7
            else:
                flat = torch.index_select(self.obs.view(2 * N, -1), 0, self._rows, out=self._flat)
        self._chain(flat, actions, values, logp, scores8, counter, view=(self.seat, self.swap), state_out=state_out, snap=snap)


class _BCAgent(object):
    """A ``BCPolicy`` agent: K10 with ``partner_seat`` (int32 [N]: the player it plays in environment e, -1 where it does
    not play), its draws keyed by ``seed ^ PARTNER_DRAW_SALT`` on a counter of its own (the draws of PPO_BC's partner).
    ``complement_of``: seats (0 / 1 only) that change between transitions; ``follow_seats()`` then sets ``partner_seat``
    to their complement."""

    lstm = False

    def __init__(self, env, policy, partner_seat, seed, complement_of=None):
        self.env, self.policy = env, policy.to(env.device).eval()
        self.partner_seat, self.seed, self._complement_of = partner_seat, int(seed), complement_of
        self._tables = self.policy.tables()
        self._n_actions = self.policy.logits.out_features
        self._counter = torch.zeros(2, dtype=torch.int64, device=env.device)

    def live(self):
        return [self._counter] + ([self.partner_seat] if self._complement_of is not None else [])

    def follow_seats(self):
        if self._complement_of is not None:
            torch.bitwise_xor(self._complement_of, 1, out=self.partner_seat)

    def act(self, actions):
        self.env.partner_actions(self._tables, self.partner_seat, self._counter, seed=self.seed ^ PARTNER_DRAW_SALT,
                                 n_actions=self._n_actions, out=actions)

    def sync_weights(self):
        for dst, src in zip(self._tables, self.policy.tables()):
            dst.copy_(src)


class _GreedyAgent(object):
    """A ``GreedyHumanModel`` agent: ``env.greedy_actions`` (include/ovc_greedy.h) with ``partner_seat`` (int32 [N]: the
    player it plays in environment e, -1 where it does not play), its previous states for the stuck rule in ``prev``
    (forgotten where the previous transition ended an episode, through ``env.done``, as ``Agent.reset()``), its stuck draws
    keyed by ``seed ^ GREEDY_DRAW_SALT`` on a counter of its own.  ``complement_of`` as ``_BCAgent``'s.  The plan tables
    are built here, never inside a graph capture."""

    lstm = False

    def __init__(self, env, partner_seat, seed, complement_of=None):
        self.env, self.partner_seat, self.seed, self._complement_of = env, partner_seat, int(seed), complement_of
        env.greedy_tables()
        self._counter = torch.zeros(2, dtype=torch.int64, device=env.device)
        self.prev = torch.zeros(env.n_envs, dtype=torch.int32, device=env.device)

    def live(self):
        return [self._counter, self.prev, self.env.done] + ([self.partner_seat] if self._complement_of is not None else [])

    def follow_seats(self):
        if self._complement_of is not None:
            torch.bitwise_xor(self._complement_of, 1, out=self.partner_seat)

    def act(self, actions):
        self.env.greedy_actions(self.partner_seat, self.prev, self._counter, seed=self.seed ^ GREEDY_DRAW_SALT, done=self.env.done,
                                out=actions)

    def sync_weights(self):
        pass


# The population draw's key is seed ^ PARTNER_MEMBER_SALT: its counters (env, step) are the seat draw's, so it needs a key of
# its own to draw numbers independent of the seats.
PARTNER_MEMBER_SALT = 0x94D049BB133111EB
MAX_MEMBERS = 64  # ovc_group_members / ovc_assign_members


def member_thresholds(weights):
    """The table ``ovc_assign_members`` draws a member from: int64 [K - 1] with entry k = floor(cdf[k] * 2^32), cdf[k] the
    float64 share of members 0..k in ``weights`` (K non-negative floats with a positive sum).  A member of weight 0 is never
    drawn: its entry equals the one before (or is 0 for member 0, 2^32 after the last positive weight).  K is not bounded
    here (``pair_thresholds`` passes K^2 pair weights): a population's size is checked where it is built."""
    w = np.asarray(weights, dtype=np.float64)
    assert w.ndim == 1, "member weights: one flat list, one weight per member"
    assert np.all(np.isfinite(w)) and np.all(w >= 0) and w.sum() > 0, "member weights: finite, non-negative, a positive sum"
    c = np.cumsum(w)
    return np.floor(c[:-1] / c[-1] * 2.0**32).astype(np.int64)


# The pair draw's key is seed ^ PAIR_SALT: its counters (env, step) are those of the other per-episode draws
PAIR_SALT = 0xBF58476D1CE4E5B9


def pair_thresholds(weights, n_members):
    """The table ``ovc_assign_pairs`` draws an ordered pair from: ``member_thresholds``' rule on the row-major flattened
    ``n_members`` x ``n_members`` weights (int64 [K^2 - 1]); entry [i][j] weighs member i on player 0 next to member j on
    player 1, and a pair of weight 0 is never drawn."""
    w = np.asarray(weights, dtype=np.float64)
    K = int(n_members)
    assert w.shape == (K, K), "pair_weights: a %d x %d array (one weight per ordered pair of members), got shape %s" % (K, K, w.shape)
    return member_thresholds(w.ravel())


class _Population(object):
    """Agent 1 of an ``AgentPairRollout`` drawn from a population: member k (an ``RllibShapedCNN`` or a ``BCPolicy``) plays
    player ``partner_seat[e]`` in the environments e with ``member[e] == k``.  Per transition ``ovc_group_members`` sorts
    the environments by member (``order``, ``offsets``), then each network member runs its kernels on its own range of
    compact rows only: the rows forms of K7 / K9 / K8 (one shared set of compact buffers), or, off the fused path, the
    library layers over all N compact rows of the observation (gathered once for all members) and the rows form of the
    draw.  A BC member is K10 with ``partner_seat`` where ``member == k`` and -1 elsewhere.  Every member keeps its own
    counter, advanced by one per transition whatever its share, so member k draws in environment e what the pair
    ``(learner, m_k)`` draws there.  ``member``: fixed, or drawn per episode from ``weights`` (``ovc_assign_members``).
    ``mixture`` (``SelfPlayRollout``'s partner): ``partner_seat[e]`` is -1 in self-play environments, which no member may
    write; the grouping key is then ``member[e]`` where ``partner_seat[e] >= 0`` and K elsewhere, and group K never runs."""

    lstm = False

    def __init__(self, env, members, partner_seat, seed, autocast_dtype, member=None, weights=None, mixture=False):
        N, dev = env.n_envs, env.device
        self.env, self.K, self.seed, self.partner_seat = env, len(members), int(seed), partner_seat
        # a BC member plays partner_seat where member == k, -1 elsewhere (rebuilt every transition)
        self.agents = [_BCAgent(env, m, torch.full((N,), -1, dtype=torch.int32, device=dev), seed) if isinstance(m, BCPolicy)
                       else _NetworkAgent(env, m, 0, partner_seat, seed, autocast_dtype) for m in members]
        shared = {}

        def buf(shape, dt):
            key = (tuple(shape), dt)
            if key not in shared:
                shared[key] = torch.empty(key[0], dtype=dt, device=dev)
            return shared[key]

        self.obs = None  # K2's observation, set by the pair when a member runs without K7
        nets = [a for a in self.agents if isinstance(a, _NetworkAgent)]
        for a in nets:  # one set of compact buffers for all members: each writes its own rows only
            a.values = buf((N,), torch.float32)
            a._flat = None
            if a.fused_first_layer:
                a._act0 = buf(a._act0.shape, torch.bfloat16)
            if a.fused_tail:
                a._z = buf(a._z.shape, torch.bfloat16)
            else:
                a._scores = buf((N, 6), torch.float32)
        self._unpaired = torch.full((N,), -1, dtype=torch.int32, device=dev)
        self.needs_obs = any(not a.fused_first_layer for a in nets)
        l = env.layouts[0]
        self._cobs = torch.empty((N, l.width * l.height * 26), dtype=autocast_dtype or torch.float32, device=dev) if self.needs_obs else None
        self._jrows = torch.empty(N, dtype=torch.int32, device=dev)
        self.order = torch.empty(N, dtype=torch.int32, device=dev)
        self.offsets = torch.zeros(self.K + 1 + bool(mixture), dtype=torch.int32, device=dev)
        self._key = torch.empty(N, dtype=torch.int32, device=dev) if mixture else None  # the grouping key of a mixture
        self._self_play_key = torch.full((N,), self.K, dtype=torch.int32, device=dev) if mixture else None
        self._counter = torch.zeros(2, dtype=torch.int64, device=dev)  # [step, scratch] of the population draw
        if member is not None:
            assert weights is None, "member fixes each environment's member, member_weights draws it: pass one of them"
            assert member.dtype == torch.int32 and member.is_contiguous() and member.numel() == N, "member: int32 [N]"
            lo, hi = int(member.min()), int(member.max())
            assert 0 <= lo and hi < self.K, "member values must lie in [0, %d): found %d..%d" % (self.K, lo, hi)
            assert member.device == dev, "member: on the environments' device"
            self.member, self._thresholds = member, None
        else:
            self.member = torch.zeros(N, dtype=torch.int32, device=dev)
            self._thresholds = torch.zeros(max(self.K - 1, 1), dtype=torch.int64, device=dev)  # never NULL: NULL skips the draw
            self.weights = [1.0] * self.K if weights is None else weights
            self.assign(None, None)

    @property
    def weights(self):
        return list(self._weights)

    @weights.setter
    def weights(self, value):
        assert self._thresholds is not None, "member_weights: the population was built with a fixed member tensor"
        w = [float(x) for x in value]
        assert len(w) == self.K, "one weight per member (%d)" % self.K
        thr = member_thresholds(w)
        self._weights = w
        self._thresholds[:self.K - 1].copy_(torch.from_numpy(thr))

    def assign(self, done, records):
        """After K1: the ending episodes' member into ``records``, then (drawn members) a new member; done None: every
        environment, no record (construction)."""
        drawn = self._thresholds is not None
        self.env.assign_members(self.member, self.K, self._thresholds, self._counter if drawn else None,
                                seed=self.seed ^ PARTNER_MEMBER_SALT, done=done, records=records)

    def live(self):
        out = [self.member, self._counter]
        for a in self.agents:
            out += a.live()
        return out

    def follow_seats(self):
        pass  # every member reads partner_seat itself

    def sync_weights(self):
        for a in self.agents:
            a.sync_weights()

    def act(self, actions):
        env, N = self.env, self.env.n_envs
        lib, stream = _native.lib(), env._stream()
        if self._key is None:
            env.group_members(self.member, self.K, self.order, self.offsets)
        else:
            torch.where(self.partner_seat >= 0, self.member, self._self_play_key, out=self._key)
            env.group_members(self._key, self.K + 1, self.order, self.offsets)
        if self._cobs is not None:  # the members' observation rows 2 e + p(e), in compact order, once for all members
            torch.index_select(self.partner_seat, 0, self.order, out=self._jrows)
            self._jrows.add_(self.order, alpha=2)
            if self._key is not None:  # group K's rows (2 e - 1 at seat -1) are gathered but never read: keep them in bounds
                self._jrows.clamp_(min=0)
            torch.index_select(self.obs.view(2 * N, -1), 0, self._jrows, out=self._cobs)
        for k, a in enumerate(self.agents):
            rng = self.offsets[k:k + 2]
            if isinstance(a, _BCAgent):
                torch.where(self.member == k, self.partner_seat, self._unpaired, out=a.partner_seat)
                a.act(actions)
                continue
            with torch.no_grad():
                if a.fused_first_layer:
                    flat, first = env.encoded_linear_rows(a._wt0, a._b0, 0, self.partner_seat, self.order, rng, a._act0), 1  # K7
                else:
                    flat, first = self._cobs, 0
                if a.fused_wide:
                    _native.check(lib.ovc_wide_layers_range(*a._k9_args(flat), rng.data_ptr(), a._z.data_ptr(), stream))
                elif a.fused_tail:
                    a.dense_model.trunk(flat, first, out=a._z)
                if a.fused_tail:
                    _native.check(lib.ovc_policy_tail_rows(
                        *a._k8_args(a._z), a._counter.data_ptr(), self.partner_seat.data_ptr(), 0, self.order.data_ptr(), rng.data_ptr(),
                        actions.data_ptr(), 0, 0, 0, stream))
                else:
                    logits, _ = a.dense_model.forward_from(flat, first)
                    a._scores.copy_(logits)
                    env.sample_actions_rows(a._scores, a._counter, 0, self.partner_seat, self.order, rng, seed=a.seed, out=actions)


class _Learners(object):
    """A population of self-play learners in one ``SelfPlayRollout`` (a list ``model``): K members (1..64
    ``RllibShapedCNN``s of one architecture), every row a learner's, drawn with key ``seed`` on the rollout's one counter.
    Member 0 is the rollout itself, passed in as ``first`` and never stored: a rollout that held itself would be a reference
    cycle, freed by the garbage collector at any later point, possibly inside another rollout's graph capture, which its
    graphs' destruction would then invalidate.  ``others`` are members 1.. folded like it, with the same kernels; their
    K7 / K9 / K8 tables are views of the stacks the grouped kernels read, so ``sync_weights()`` refreshes the stacks in place.
    Per transition ``act`` runs K9 on each member's rows as one grouped launch from ``GROUPED_K9_MIN_MEMBERS`` members on,
    one launch per member below that.  The population takes one of two forms.

    Blocks (fictitious co-play's first stage): member k plays both views of the environments of its block ``[blocks[k],
    blocks[k + 1])``; blocks (argument): K positive environment counts summing to N, default equal blocks (``blocks[k] = k N
    // K``).  ``blocks`` is then the offsets (int32 [K + 1]) and ``member`` the member of each environment (int32 [N]).  The
    fused layers run as one grouped launch each for all members (``ovc_encode_linear_grouped``, K9, ``ovc_policy_tail_grouped``),
    library layers per member on its block's rows; every row is drawn with the one counter (grouped K8, or, without K8, one
    ``ovc_sample_actions`` over all rows): block k is bit for bit what ``SelfPlayRollout(env, model[k], seed=seed)`` does on
    those environments.

    Population play (``pairs`` or ``pair_weights``): member ``pair[e, 0]`` plays player 0 of environment e and member ``pair[e,
    1]`` player 1.  ``pairs`` (int32 [N, 2] on the environments' device) fixes the pairing (the evaluation form: a cross-play
    matrix through run()); ``pair_weights`` (K x K non-negative floats with a positive sum) draws the ordered pair (i, j) with
    probability proportional to ``pair_weights[i][j]`` at construction and at every episode end (the training form: uniform
    weights are PBT-style population play, a zero diagonal excludes self-play).  ``pair`` (int32 [N, 2]) is the live
    pairing.  Per transition ``ovc_group_pairs`` groups the entries by member on the device, then
    ``ovc_encode_linear_grouped_masked`` (the object part once per environment), K9 on each member's compact rows (off K9
    each member's library layers on all compact rows, its own rows selected on the device) and
    ``ovc_policy_tail_grouped_joint`` (off K8: the library heads and one ``ovc_sample_actions`` over the joint rows).  Every
    row is drawn at its joint row ``2 e + v``, so copies of one model draw exactly what ``SelfPlayRollout(env, model)``
    draws; the pair draw uses key ``seed ^ PAIR_SALT`` and a counter of its own.  collect()'s batches carry ``pair`` and
    ``episodes.finished()`` reports each episode's ``pair``.  Needs K7 (at most 8 layouts, a grid within its shared memory)
    and the bf16 policy; not with ``blocks``."""

    def __init__(self, first, models, blocks, pairs, pair_weights, autocast_dtype, fused_first_layer, fused_tail, fused_wide):
        """Check the arguments (see ``SelfPlayRollout.__init__``), fold member 0 into ``first`` (the rollout, with its
        ``env`` and ``seed`` set) and the others alike, and stack their tables."""
        env = self.env = first.env
        K, N, dev = len(models), env.n_envs, env.device
        self.K, self.seed = K, first.seed
        pair_play = pairs is not None or pair_weights is not None
        if pair_play:
            assert pairs is None or pair_weights is None, "pairs fixes each environment's pair, pair_weights draws it: pass one of them"
            assert blocks is None, "population play pairs the members per environment: pass no blocks with pairs / pair_weights"
            assert autocast_dtype == torch.bfloat16, "population play runs K7 and K8 on the bf16 policy: autocast_dtype=None is not supported"
        _check_members(models, MAX_MEMBERS, RllibShapedCNN, "a population of learners has 1..%d members" % MAX_MEMBERS,
                       "a population learner is an RllibShapedCNN (an LSTM member is not supported)")
        arch = lambda m: (m.dense_slope,) + tuple((n, tuple(p.shape)) for n, p in m.named_parameters())
        assert len({arch(m) for m in models}) == 1, "the members of a population of learners must share one architecture"
        if pairs is not None:
            assert isinstance(pairs, torch.Tensor) and pairs.dtype == torch.int32 and tuple(pairs.shape) == (N, 2) and \
                pairs.is_contiguous(), "pairs: a contiguous int32 tensor [N, 2] (N = %d environments)" % N
            assert pairs.device == dev, "pairs: on the environments' device (%s), got %s" % (dev, pairs.device)
            lo, hi = int(pairs.min()), int(pairs.max())
            assert 0 <= lo and hi < K, "pairs values must lie in [0, %d): found %d..%d" % (K, lo, hi)
        elif pair_play:
            pair_thresholds(pair_weights, K)
        elif blocks is None:
            assert N >= K, "equal blocks need at least one environment per member (%d members, %d environments)" % (K, N)
            counts = [(k + 1) * N // K - k * N // K for k in range(K)]
        else:
            counts = [int(b) for b in blocks]
            assert len(counts) == K, "blocks: one environment count per member (%d)" % K
            assert all(c > 0 for c in counts) and sum(counts) == N, \
                "blocks: positive environment counts summing to the %d environments, got %s" % (N, counts)
        first._fold(env, models[0], autocast_dtype, fused_first_layer, fused_tail, fused_wide)
        assert not pair_play or first.fused_first_layer, \
            "population play needs K7: a first layer width a multiple of 64, a grid whose table fits shared memory, and at " \
            "most %d layouts (this environment has %d layouts on a %dx%d grid)" % (K7_MAX_LAYOUTS, env.n_layouts, first.W, first.H)
        self.others = []
        for m in models[1:]:
            f = _FoldedPolicy()
            f.env = env
            f._fold(env, m, autocast_dtype, first.fused_first_layer, first.fused_tail, first.fused_wide)
            self.others.append(f)
        members = [first] + self.others

        def stack(attr):  # the grouped kernels' stacked tables; each member's tables become views of them
            st = tuple(torch.stack(ts) for ts in zip(*(getattr(f, attr) for f in members)))
            for k, f in enumerate(members):
                setattr(f, attr, tuple(t[k] for t in st))
            return st
        if first.fused_first_layer:
            self._k7_stack = (torch.stack([f._wt0 for f in members]), torch.stack([f._b0 for f in members]))
            for k, f in enumerate(members):
                f._wt0, f._b0 = self._k7_stack[0][k], self._k7_stack[1][k]
        if first.fused_wide:
            self._wide_stack = stack("_wide")
        if first.fused_tail:
            self._tail_stack = stack("_tail")
        self.blocks = self.member = self.pair = self._thresholds = None
        if not pair_play:
            self._offs = [0] + np.cumsum(counts).tolist()
            self.blocks = torch.tensor(self._offs, dtype=torch.int32, device=dev)
            self._row_offsets = 2 * self.blocks  # K9's and K8's offsets are joint rows
            self.member = torch.repeat_interleave(torch.arange(K, dtype=torch.int32, device=dev),
                                                  torch.tensor(counts, device=dev)).to(torch.int32)
            return
        # population play: the live pairing, its draw, and the compact layout ovc_group_pairs writes
        i32 = lambda n: torch.zeros(n, dtype=torch.int32, device=dev)
        self._counter = torch.zeros(2, dtype=torch.int64, device=dev)  # [step, scratch] of the pair draw
        if pairs is not None:
            self.pair = pairs
        else:
            self.pair = torch.zeros((N, 2), dtype=torch.int32, device=dev)
            self._thresholds = torch.zeros(max(K * K - 1, 1), dtype=torch.int64, device=dev)  # never NULL: NULL skips the draw
            self.pair_weights = pair_weights
        self._plist, self._pfirst, self._pjrow = i32(2 * N), i32(2 * N), i32(2 * N)
        self._entry_offsets, self._row_offsets = i32(K + 1), i32(K + 1)
        self._logp = torch.empty(2 * N, dtype=torch.float32, device=dev)  # run()'s logp: the joint K8 always writes it
        if not first.fused_wide:  # the member of each compact row, for the library layers' selection
            self._rmember = torch.empty(2 * N, dtype=torch.int64, device=dev)
            self._rindex = torch.arange(2 * N, device=dev)
        if not first.fused_tail:  # the library heads on compact rows, scattered to the joint rows for the draw kernel
            self._jrow64 = torch.empty(2 * N, dtype=torch.int64, device=dev)
            self._cscores = torch.zeros((2 * N, first.dense_model.n_actions), dtype=torch.float32, device=dev)
            self._cvalues = torch.zeros(2 * N, dtype=torch.float32, device=dev)
        if pairs is None:
            self.assign(None, None)

    @property
    def pair_weights(self):
        return [list(r) for r in self._pair_weights]

    @pair_weights.setter
    def pair_weights(self, value):
        thr = pair_thresholds(value, self.K)
        self._pair_weights = np.asarray(value, dtype=np.float64).tolist()
        self._thresholds[:self.K * self.K - 1].copy_(torch.from_numpy(thr))

    def assign(self, done, records):
        """After K1, in population play: the ending episodes' pair into ``records``, then (drawn pairs) a new pair; done
        None: every environment, no record (construction).  Nothing for blocks."""
        if self.pair is not None:
            drawn = self._thresholds is not None
            self.env.assign_pairs(self.pair, self.K, self._thresholds, self._counter if drawn else None, seed=self.seed ^ PAIR_SALT,
                                  done=done, records=records)

    def live(self):
        """The tensors a transition advances (restored around graph capture)."""
        return [] if self.pair is None else [self.pair, self._counter]

    def sync_weights(self):
        """Re-fold members 1.. in place (the rollout re-folds member 0)."""
        for f in self.others:
            f.sync_weights()

    def act(self, first, actions, values, logp, scores8, counter):
        """``SelfPlayRollout._policy`` for the population, in ``first``'s buffers: grouped K7 (blocks), or ``ovc_group_pairs``
        then the grouped masked K7 into compact rows; K9 on each member's rows; grouped K8 (blocks) or grouped joint K8 (None
        returned).  Off K7 (blocks only) the layers start from K2's observation ``first.obs``; off K9 the library layers run
        per member on its block's rows, or on every compact row with its own rows selected on the device (no host
        synchronisation); off K8 the logits go to the joint rows of ``first._scores``, returned for the one draw kernel over
        all rows."""
        env, lib, st, K, rows = self.env, _native.lib(), self.env._stream(), self.K, 2 * self.env.n_envs
        members = [first] + self.others
        block = lambda k: slice(2 * self._offs[k], 2 * self._offs[k + 1])  # member k's rows [2 o_k, 2 o_{k+1}) (blocks)
        ptr = lambda t: 0 if t is None else t.data_ptr()
        horizon = env.horizon if env.horizon > 0 else 2**31 - 1
        with torch.no_grad():
            if self.pair is not None:
                env.group_pairs(self.pair, K, self._plist, self._pfirst, self._pjrow, self._entry_offsets, self._row_offsets)
            if first.fused_first_layer:
                wt, b0 = self._k7_stack
                if self.pair is None:
                    _native.check(lib.ovc_encode_linear_grouped(
                        env.tables.data_ptr(), env.n_layouts, env.state.data_ptr(), wt.data_ptr(), b0.data_ptr(), self.blocks.data_ptr(),
                        K, first._act0.data_ptr(), env.n_envs, env.state_words, first.W, first.H, horizon, wt.shape[2], 0.2, st))
                else:
                    _native.check(lib.ovc_encode_linear_grouped_masked(
                        env.tables.data_ptr(), env.n_layouts, env.state.data_ptr(), self._plist.data_ptr(), self._pfirst.data_ptr(),
                        wt.data_ptr(), b0.data_ptr(), self._entry_offsets.data_ptr(), K, first._act0.data_ptr(), rows, env.state_words,
                        first.W, first.H, horizon, wt.shape[2], 0.2, st))
                flat, lib_first = first._act0, 1
            else:
                flat, lib_first = first.obs.view(rows, first.W * first.H * 26), 0
            if first.fused_wide and K >= GROUPED_K9_MIN_MEMBERS:
                _native.check(lib.ovc_wide_layers_grouped(*first._k9_args(flat, self._wide_stack), self._row_offsets.data_ptr(), K,
                                                          first._z.data_ptr(), st))
            elif first.fused_wide:  # K9 per member: on its block, or on its range of compact rows
                for k, f in enumerate(members):
                    if self.pair is None:
                        _native.check(lib.ovc_wide_layers(*f._k9_args(flat[block(k)]), first._z[block(k)].data_ptr(), st))
                    else:
                        _native.check(lib.ovc_wide_layers_range(*f._k9_args(flat), self._row_offsets[k:k + 2].data_ptr(),
                                                                first._z.data_ptr(), st))
            elif self.pair is None:  # library layers per member on its block's rows; bit for bit the member's own rollout only
                # where cuBLAS computes a row independently of the row count (tested at up to 2 x 300 rows per call)
                for k, f in enumerate(members):
                    if first.fused_tail:
                        f.dense_model.trunk(flat[block(k)], lib_first, out=first._z[block(k)])
                    else:
                        logits, value = f.dense_model.forward_from(flat[block(k)], lib_first)
                        first._scores[block(k)].copy_(logits)
                        values[block(k)].copy_(value)
            else:  # library layers per member on every compact row; bit for bit the member's own rollout only where cuBLAS
                # computes a row independently of the other rows
                torch.searchsorted(self._row_offsets[1:], self._rindex, right=True, out=self._rmember)
                for k, f in enumerate(members):
                    mine = (self._rmember == k).unsqueeze(1)
                    if first.fused_tail:
                        torch.where(mine, f.dense_model.trunk(flat, 1), first._z, out=first._z)
                    else:
                        logits, value = f.dense_model.forward_from(flat, 1)
                        torch.where(mine, logits.float(), self._cscores, out=self._cscores)
                        torch.where(mine[:, 0], value.float(), self._cvalues, out=self._cvalues)
            if not first.fused_tail:
                if self.pair is not None:
                    self._jrow64.copy_(self._pjrow)
                    first._scores.index_copy_(0, self._jrow64, self._cscores)
                    values.index_copy_(0, self._jrow64, self._cvalues)
                return first._scores
            args = first._k8_args(first._z, self._tail_stack) + (counter.data_ptr(),)
            if self.pair is None:
                _native.check(lib.ovc_policy_tail_grouped(*args, self._row_offsets.data_ptr(), K, actions.data_ptr(), values.data_ptr(),
                                                          ptr(scores8), ptr(logp), st))
            else:
                _native.check(lib.ovc_policy_tail_grouped_joint(*args, self._pjrow.data_ptr(), self._row_offsets.data_ptr(), K,
                                                                actions.data_ptr(), values.data_ptr(), ptr(scores8),
                                                                (self._logp if logp is None else logp).data_ptr(), st))
        return None


class AgentPairRollout(_Rollout):
    """Two different agents, each evaluated on its own seat's view only: the reference's evaluation of an agent pair
    (rllib.py ``evaluate``: ``AgentEvaluator.evaluate_agent_pair(AgentPair(agent_0_policy, agent_1_policy))``) with N
    environments on the device — PPO against a held-out BC human proxy, cross-play of two PPO agents, BC against BC, PPO against the reference's scripted GreedyHumanModel — and,
    with ``collect()``, PPO training of agent 0 next to a fixed agent 1 (a best response, the second stage of fictitious
    co-play, training against a held-out PPO, LSTM or BC partner).

    agents: (agent0, agent1), each an ``RllibShapedCNN``, an ``RllibLSTMShapedCNN``, a ``BCPolicy`` or a ``GreedyHumanModel``
    (the same object twice is allowed).  agent1 may instead be a population: a list of 1..64 members, each an ``RllibShapedCNN`` or a ``BCPolicy``
    (fictitious co-play's second stage, training against a set of checkpoints, PPO_BC with several BC human proxies).  Agent 0 plays player ``swap[e]`` of environment e, agent 1 the other one.  A network agent runs its own
    policy on N rows (the one-view forms of K7 / K8 / K11 and the draw, with K9 on N rows, where ``fused_kernel_support``
    allows them; K2, the dense model on the agent's rows and the one-view draw elsewhere); a BC agent is K10.
    swap: int32 CUDA tensor [N] or None (no swap): both seat orders in one batch; fixed for the rollout's lifetime.
    random_seats: instead of ``swap``, agent 1's player ``partner_seat[e]`` is drawn at construction and again for every
    environment whose episode ended (the reference's gym ``Overcooked`` wrapper and ``OvercookedMultiAgent`` redraw the
    agents' players at every reset): PPO_BC's seat draw (``env.assign_partners``) at a ``bc_factor`` of 1, key ``seed ^
    PARTNER_SEAT_SALT``, with a counter of its own, so that ``(learner, bc)`` plays exactly the seats of
    ``SelfPlayRollout(learner, partner=bc, bc_factor=1)``.  Not together with ``swap``.
    seed: the draws' key.  Each agent has its own counter; network agents use ``seed``, BC agents ``seed ^
    PARTNER_DRAW_SALT`` (K10's key in PPO_BC), greedy agents ``seed ^ GREEDY_DRAW_SALT`` for their stuck steps.  A pair therefore draws what ``SelfPlayRollout`` (both agents one network) or
    PPO_BC (``SelfPlayRollout(partner=..., bc_factor=1)``) draw on the same rows and steps.
    autocast_dtype: as ``SelfPlayRollout``'s, for every network agent (an LSTM agent needs bfloat16).
    episode_capacity: as ``SelfPlayRollout``'s.  Every finished episode's ``partner_seat`` is agent 1's player.
    max_seq_len: as ``SelfPlayRollout``'s, for an LSTM learner's ``collect()``.
    member (population only): int32 CUDA tensor [N] with values in [0, K): environment e plays member member[e] for the
    rollout's lifetime (checked once here).
    member_weights (population only; see the property): instead of ``member``, each environment's member is drawn at
    construction and again at every episode end (``env.assign_members``, key ``seed ^ PARTNER_MEMBER_SALT``), member k with
    probability ``member_weights[k] / sum``; default uniform.  The seats follow ``swap`` / ``random_seats`` as for a pair, so
    a population of one draws what the pair draws.  Member k's actions in environment e are those ``AgentPairRollout(env,
    (agent0, m_k))`` draws there.  ``episodes.finished()`` and collect()'s batches then report ``partner_member``.

    A transition is K2 (once, when a network agent runs without K7), agent 0's policy, agent 1's policy, K1 (auto-reset
    inside), ``record_transition`` with the episode statistics (``record_transition_view`` of agent 0's row in collect()),
    then, with random_seats, the seat draw.  With a population, agent 1's step is ``ovc_group_members`` and each member's
    kernels on its own environments, and ``ovc_assign_members`` (the ending episodes' member, the new draw) runs between
    K1 and the record.  ``ret_sparse`` is the running sparse return of every environment.
    use_phi: as ``SelfPlayRollout``'s: both agents' rewards are the potential-based dense reward (K6 before K1, K1 without
    the reset, ovc_potential_shaping after it)."""

    def __init__(self, env, agents, swap=None, seed=0, use_graph=True, episode_capacity=1, autocast_dtype=torch.bfloat16,
                 random_seats=False, max_seq_len=20, member=None, member_weights=None, use_phi=False):
        assert len({(l.width, l.height) for l in env.layouts}) == 1, "one grid shape per rollout (group envs by layout)"
        self._phi = _PhiReward(env) if use_phi else None
        assert len(agents) == 2, "agents: (agent0, agent1)"
        assert not (random_seats and swap is not None), "random_seats draws the seats: pass no swap tensor with it"
        assert not isinstance(agents[0], (list, tuple)), "a population plays agent 1 only: agents = (agent0, [m_0, ..., m_K-1])"
        self.population = isinstance(agents[1], (list, tuple))
        if self.population:
            _check_members(agents[1], MAX_MEMBERS, (RllibShapedCNN, BCPolicy), "a population has 1..%d members" % MAX_MEMBERS,
                           "a population member is an RllibShapedCNN or a BCPolicy (an LSTM member is not supported)")
        else:
            assert member is None and member_weights is None, "member / member_weights go with a population in agents[1]"
        for a in agents[:1] if self.population else agents:
            assert isinstance(a, (RllibShapedCNN, BCPolicy, GreedyHumanModel)), \
                "an agent is an RllibShapedCNN, an RllibLSTMShapedCNN, a BCPolicy or a GreedyHumanModel"
        if swap is not None:
            assert swap.dtype == torch.int32 and swap.is_cuda and swap.is_contiguous() and swap.numel() == env.n_envs, \
                "swap: int32 CUDA [N]"
        self.env, self.swap, self.seed = env, swap, int(seed)
        self.random_seats = bool(random_seats)
        if self.random_seats:
            # agent 1's player, drawn for every environment now and at every episode end; agent k then sits at player
            # (1 - k) ^ partner_seat[e], i.e. it is passed seat 1 - k and swap = partner_seat
            self.partner_seat = torch.full((env.n_envs,), -1, dtype=torch.int32, device=env.device)
            self._bc_factor = torch.ones(1, dtype=torch.float32, device=env.device)  # every episode is paired
            self._seat_counter = torch.zeros(2, dtype=torch.int64, device=env.device)  # [step, scratch] of the seat draw
            self._assign_seats(None)
            seats, swap = (1, 0), self.partner_seat
        else:
            seats = (0, 1)

        def player(seat):  # int32 [N]: seat ^ (swap[e] != 0), the player of the agent passed seat
            if swap is None:
                return torch.full((env.n_envs,), seat, dtype=torch.int32, device=env.device)
            return (seat ^ (swap != 0).int()).to(torch.int32).contiguous()
        def scripted(a, players, complement_of=None):  # a BC or greedy agent on the players ``players``
            if isinstance(a, GreedyHumanModel):
                return _GreedyAgent(env, players, seed, complement_of)
            return _BCAgent(env, a, players, seed, complement_of)
        # with fixed seats partner_seat is made after the agents: a network agent's fold checks its model first
        self.agents = []
        for seat, a in zip(seats, agents[:1] if self.population else agents):
            if isinstance(a, RllibShapedCNN):
                self.agents.append(_NetworkAgent(env, a, seat, swap, seed, autocast_dtype, self.random_seats))
            elif self.random_seats and seat == 0:  # agent 1 plays the drawn seats themselves
                self.agents.append(scripted(a, self.partner_seat))
            else:  # under random_seats, agent 0 plays their complement
                self.agents.append(scripted(a, player(seat), self.partner_seat if self.random_seats else None))
        if not self.random_seats:
            self.partner_seat = player(1)  # agent 1's player
        if self.population:
            self.agents.append(_Population(env, list(agents[1]), self.partner_seat, seed, autocast_dtype, member, member_weights))
        self._pop = self.agents[1] if self.population else None
        self._member = None
        # network agents without K7 read K2's observation, written once per transition for all of them
        library = [a for a in self.agents if (isinstance(a, _NetworkAgent) and not a.fused_first_layer) or getattr(a, "needs_obs", False)]
        l = env.layouts[0]
        self.obs = torch.empty((env.n_envs, 2, l.width, l.height, 26), dtype=autocast_dtype or torch.float32, device=env.device) \
            if library else None
        for a in library:
            a.obs = self.obs
        self._init_rollout(env, self.agents[0], use_graph, 1.0, episode_capacity, max_seq_len)

    def _agents(self):
        return self.agents

    def _live(self):
        live = [self.env.done]
        if self.random_seats:
            live += [self.partner_seat, self._seat_counter]
        for a in self.agents:
            live += a.live()
        return live

    def _transition(self, b=None, t=0):
        """One transition.  Without ``b`` (run()) finished episodes go to self.episodes; with a one-view ``SampleBatch`` ``b``
        (collect()) agent 0's row is recorded in its slot ``t``: state, action, value, logp, logits, reward, done, agent 1's
        player, the LSTM state every seq_len transitions, and finished episodes in b.episodes."""
        env = self.env
        learner, partner = self.agents
        if self.obs is not None:
            env.lossless_state_encoding(out=self.obs)  # K2
        if b is None:
            learner.act(self.actions)
        else:
            b.states[t].copy_(env.state)
            snap = None
            if b.seq_len and t % b.seq_len == 0:
                snap = (b.state_h[t // b.seq_len], b.state_c[t // b.seq_len])
            learner.act(self.actions, values=b.values[t], logp=b.logp[t], scores8=None if b.logits is None else b.logits[t], snap=snap)
            torch.index_select(self.actions.view(-1), 0, learner._rows, out=b.actions[t])
            b.partner_seat[t].copy_(self.partner_seat)
            if self.population:
                b.partner_member[t].copy_(partner.member)
        partner.act(self.actions)
        terminal = None
        if b is not None and b.terminal_values is not None:
            terminal = lambda: self._terminal_values(b.terminal_values[t])
        dense = _env_step(env, self.actions, self._phi, terminal)
        if self.population:  # before the record: both use the slot count[e] the ending episode goes to
            partner.assign(env.done, self.episodes if b is None else b.episodes)
        if b is None:
            env.record_transition(self._factor, ret_sparse=self.ret_sparse, stats=self.stats, records=self.episodes,
                                  partner_seat=self.partner_seat, dense=dense)
        else:
            env.record_transition_view(self._factor, learner.seat, learner.swap, b.rewards[t], dones=b.dones[t], ret_sparse=self.ret_sparse,
                                       stats=self.stats, records=b.episodes, partner_seat=self.partner_seat, dense=dense)
        if self.random_seats:  # after the record: the ending episode's seats went into it
            self._assign_seats(env.done)
            for a in self.agents:
                a.follow_seats()

    def _bootstrap(self, b):
        if self.obs is not None:
            self.env.lossless_state_encoding(out=self.obs)
        # the learner's bootstrap value at the seats after the window; its LSTM state goes to scratch
        learner = self.agents[0]
        learner.act(self._boot_actions, values=b.last_values, counter=self._boot_counter,
                    state_out=(self._h_boot, self._c_boot) if learner.lstm else None)

    def _terminal_values(self, out):
        """The horizon bootstrap's value pass into ``out`` (float32 [N]): agent 0's value on the terminal record of each
        ended environment, at the seat it played, 0 elsewhere; as ``SelfPlayRollout._terminal_values``."""
        h, env, learner = self._horizon, self.env, self.agents[0]
        if h.fused:
            learner._horizon_values_rows(h, self.partner_seat, True, out, self._boot_counter, self._boot_actions)
            return
        if self.obs is not None:
            env.lossless_state_encoding(out=self.obs)
        learner.act(self._boot_actions, values=h.values, counter=self._boot_counter)
        torch.where(env.done != 0, h.values, h.zero, out=out)

    def _new_batch(self, n_steps, keep_logits):
        """collect()'s batch: agent 0's side of the transitions as a one-view ``SampleBatch`` (one row per environment:
        agent 0's action, logp, value, reward and GAE advantages; ``partner_seat`` is agent 1's player), for a PPO update of
        agent 0 next to the fixed agent 1.  After an update, call ``sync_weights()`` (it refolds every population member
        too)."""
        assert isinstance(self.agents[0], _NetworkAgent), \
            "collect() trains agents[0]: an RllibShapedCNN or RllibLSTMShapedCNN, not a BCPolicy or a GreedyHumanModel"
        return SampleBatch(self.env, n_steps, keep_logits, seq_len=self.max_seq_len if self.agents[0].lstm else None,
                           one_view=True, members=self.population)

    def sync_weights(self):
        """Re-fold every agent's network (e.g. a learner's after an update) in place: the captured graphs use the new weights
        without a re-capture."""
        for a in self.agents:
            a.sync_weights()
