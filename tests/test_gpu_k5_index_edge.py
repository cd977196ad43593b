"""K5 at its 32-bit index edge.  The fused rollout kernel addresses a thread's action and output rows with one 32-bit
unsigned element index per stream, and ovc_rollout cuts a rollout into launches of at most 0xFFFFFFFF / n_envs - 1
transitions so that no launch reaches 2^32 env-steps.  At 100 003 environments that is 42 947 transitions: one launch of
that length addresses elements up to about 2^32 - 1.4e5, one transition more is cut for real into 42 947 + 1, and
2 x 42 947 + 5 into three launches.  The sparse event stream is never cut: its dense backup is checked at the largest
length it takes, and one transition more must be refused.

The formats are the compact host ones (one-byte joint actions, one 16-bit code word per env-step: 3 B per env-step, up to
26 GB for the longest case), and each case skips when the card has less free memory than it needs plus a margin.  Ground
truth is the same start records run through consecutive rollouts of at most 4096 transitions (indices below 2^31),
compared slice by slice on the device, and the final records; 256 sampled environments, env 0 and env N - 1 among them,
are also replayed through the CPU oracle over every transition."""
import numpy as np
import pytest
import torch

from oracle import cpu
from overcooked_ai_b200 import wire
from overcooked_ai_b200.batched import BatchedOvercookedEnv

pytestmark = pytest.mark.gpu

N = 100003  # a multiple of neither 32 nor the CTA tile
MAX_STEPS = 0xFFFFFFFF // N - 1  # the longest launch ovc_rollout makes at this size
NAMES = ["cramped_room", "counter_circuit"]
HORIZON = 400
CHUNK = 4096  # reference launches: below 2^31 element indices
MARGIN = 2 << 30


def _need(nbytes):
    """Skips unless the card has nbytes free besides the action draw's transients and a margin.  Blocks this process
    keeps cached from earlier cases are returned first, so that they do not count as used."""
    nbytes += 1024 * N * 2 * 6  # _packed_actions: one block of 1024 transitions as uint8, float32 and bool
    torch.cuda.empty_cache()
    free, _ = torch.cuda.mem_get_info()
    if free < nbytes + MARGIN:
        pytest.skip("needs %.1f GB of free device memory, %.1f GB free (the card is shared)" % ((nbytes + MARGIN) / 1e9, free / 1e9))


def _env():
    return BatchedOvercookedEnv(NAMES, N, horizon=HORIZON, auto_reset=True)


def _packed_actions(T, seed):
    """uint8 [T, N] one-byte joint actions (wire.pack_actions), interact-biased, drawn on the device."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    out = torch.empty((T, N), dtype=torch.uint8, device="cuda")
    for t0 in range(0, T, 1024):
        t1 = min(T, t0 + 1024)
        a = torch.randint(0, 6, (t1 - t0, N, 2), generator=g, device="cuda", dtype=torch.uint8)
        a[torch.rand((t1 - t0, N, 2), generator=g, device="cuda") < 0.4] = 5
        out[t0:t1] = a[..., 0] | (a[..., 1] << 4)
    return out


def _check_against_chunks(start, acts, words, final):
    """The same start records through rollouts of at most CHUNK transitions must give words [T, N] and the final records."""
    ref = _env()
    ref.state.copy_(start)
    buf = torch.empty((CHUNK, N), dtype=torch.int16, device="cuda")
    T = acts.shape[0]
    for t0 in range(0, T, CHUNK):
        t1 = min(T, t0 + CHUNK)
        ref.rollout(acts[t0:t1], out=(None, None, None, buf[:t1 - t0]))
        if not torch.equal(buf[:t1 - t0], words[t0:t1]):
            bad = (buf[:t1 - t0] != words[t0:t1]).nonzero()[:5].tolist()
            raise AssertionError("transitions %d..%d differ from the reference launches, first at (t, env) %s" % (t0, t1, [(t0 + t, e) for t, e in bad]))
    assert torch.equal(ref.state, final), "final records differ from the reference launches"


def _check_against_oracle(env, start, acts, words):
    """256 sampled environments, env 0 and env N - 1 among them, through the oracle over every transition."""
    rng = np.random.RandomState(7)
    idx = np.unique(np.concatenate([[0, N - 1], rng.choice(N, 254, replace=False)]))
    d_idx = torch.from_numpy(idx).cuda()
    a = acts.index_select(1, d_idx).cpu().numpy()
    a = np.stack([a & 15, a >> 4], -1).astype(np.int32)
    state = start.index_select(0, d_idx).cpu().numpy()
    want = cpu.rollout(env._tab_host, env._starts_host, state, a, horizon=HORIZON, flags=1)
    got = wire.decode_codes(words.index_select(1, d_idx).cpu().numpy(), env.code_reward_table(), env.env_layout_host[idx])
    for k, g, w in zip(("sparse", "shaped", "done", "events"), got, want):
        assert np.array_equal(g.astype(np.int64), w.astype(np.int64)), k
    assert np.array_equal(env.state.index_select(0, d_idx).cpu().numpy(), state), "final records of the sampled environments"
    assert want[0].any() and want[2].any(), "premise: soups are delivered and episodes end"


@pytest.mark.parametrize("T", [MAX_STEPS, MAX_STEPS + 1, 2 * MAX_STEPS + 5], ids=["one_launch", "cut_1", "cut_2"])
def test_k5_past_2_to_the_31_element_indices(T):
    assert T * N > 2**31 and MAX_STEPS * N < 2**32
    _need(3 * T * N + CHUNK * N * 2)
    env = _env()
    start = env.state.clone()
    acts = _packed_actions(T, seed=T)
    words = torch.empty((T, N), dtype=torch.int16, device="cuda")
    env.rollout(acts, out=(None, None, None, words))
    final = env.state.clone()
    _check_against_chunks(start, acts, words, final)
    _check_against_oracle(env, start, acts, words)


def test_k5_stream_at_its_longest_launch_and_refused_one_transition_above():
    T = MAX_STEPS
    cap = 16
    G = (N + 31) // 32
    _need(3 * (T + 1) * N + 4 * (T + 1) * G + CHUNK * N * 2)
    env = _env()
    start = env.state.clone()
    acts = _packed_actions(T + 1, seed=5)
    masks = torch.zeros((T + 1, G), dtype=torch.int32, device="cuda")
    values = torch.zeros((1, G, cap), dtype=torch.int16, device="cuda")
    dense = torch.zeros((T + 1, N), dtype=torch.int16, device="cuda")
    with pytest.raises(RuntimeError, match=r"\(-3\)"):  # OVC_E_UNSUPPORTED: the stream is never cut
        env.rollout_stream(acts, cap, out=(masks, values, dense))
    assert torch.equal(env.state, start) and not dense.any(), "a refused call touched the records or the outputs"
    env.rollout_stream(acts[:T], cap, out=(masks[:T], values, dense[:T]))
    final = env.state.clone()
    _check_against_chunks(start, acts[:T], dense[:T], final)
    # the lane masks of the last transitions name exactly the non-zero words
    nz = torch.nn.functional.pad((dense[T - 64:T] != 0).to(torch.int64), (0, 32 * G - N)).view(64, G, 32)
    want = (nz << torch.arange(32, device="cuda")).sum(-1)
    assert torch.equal(masks[T - 64:T].to(torch.int64) & 0xFFFFFFFF, want)
    _check_against_oracle(env, start, acts[:T], dense[:T])
