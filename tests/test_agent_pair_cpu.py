"""The agent-pair entry points without a GPU: the one-view symbols are declared and exported, malformed calls are refused at
n = 0 (nothing is launched), and AgentPairRollout refuses what SelfPlayRollout refuses."""
import os
import re
from types import SimpleNamespace

import pytest
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200.selfplay import AgentPairRollout, BCPolicy, RllibLSTMShapedCNN, RllibShapedCNN

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
VIEW_SYMBOLS = ("ovc_encode_linear_view", "ovc_sample_actions_view", "ovc_policy_tail_view", "ovc_lstm_head_view")


def test_view_entry_points_are_declared_and_exported():
    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    declared = set(re.findall(r"\b(ovc_[a-z_0-9]+)\s*\(", hdr))
    lib = _native.lib()
    for sym in VIEW_SYMBOLS:
        assert sym in declared and sym in _native.EXPORTED_SYMBOLS and hasattr(lib, sym), sym
    assert lib.ovc_abi_version() == 5


A = 4096  # an aligned stand-in address: with n = 0 nothing is dereferenced


def _calls(lib, swap=A, seat=0, actions=A, ptr=A):
    """Each one-view entry point at n = 0, with ``ptr`` for its 4-byte-aligned outputs."""
    return {
        "encode_linear_view": lambda: lib.ovc_encode_linear_view(A, 1, A, swap, seat, A, A, A, 0, 16, 5, 4, 400, 64, 0.2, None),
        "sample_actions_view": lambda: lib.ovc_sample_actions_view(A, 8, 6, 0, 0, A, swap, seat, actions, ptr, None),
        "policy_tail_view": lambda: lib.ovc_policy_tail_view(A, 0, 160, 0.2, A, A, A, A, 2, A, A, 0.3, 6, 0, A, swap, seat, actions, ptr,
                                                             A, ptr, None),
        "lstm_head_view": lambda: lib.ovc_lstm_head_view(A, A, A, A, 0, A, A, A, A, 6, 0, A, swap, seat, A, A, 0, 0, actions, ptr, ptr,
                                                         A, None),
    }


def test_view_entry_points_accept_a_well_formed_empty_call_and_refuse_malformed_ones():
    lib = _native.lib()
    for name, call in _calls(lib).items():
        assert call() == 0, (name, lib.ovc_last_error())
    for name, call in _calls(lib, swap=0).items():
        assert call() == 0, (name, lib.ovc_last_error())
    for name, call in _calls(lib, seat=2).items():
        assert call() != 0 and b"seat" in lib.ovc_last_error(), name
    for name, call in _calls(lib, seat=-1).items():
        assert call() != 0, name
    for name, call in _calls(lib, swap=A + 2).items():
        assert call() != 0 and b"aligned" in lib.ovc_last_error(), name
    for name, call in _calls(lib, actions=0).items():
        if name != "encode_linear_view":
            assert call() != 0 and b"null" in lib.ovc_last_error(), name
    for name, call in _calls(lib, ptr=A + 2).items():
        if name != "encode_linear_view":
            assert call() != 0 and b"aligned" in lib.ovc_last_error(), name


def _env(shapes):
    return SimpleNamespace(layouts=[SimpleNamespace(width=w, height=h) for w, h in shapes], device=torch.device("cpu"), n_layouts=len(shapes))


def test_agent_pair_refuses_mixed_grids_and_a_float32_lstm_agent():
    with pytest.raises(AssertionError, match="one grid shape"):
        AgentPairRollout(_env([(5, 4), (9, 5)]), (RllibShapedCNN(5, 4), BCPolicy()))
    with pytest.raises(AssertionError, match="K11"):
        AgentPairRollout(_env([(5, 4)]), (RllibLSTMShapedCNN(5, 4), BCPolicy()), autocast_dtype=None)
    with pytest.raises(AssertionError, match="agent"):
        AgentPairRollout(_env([(5, 4)]), (RllibShapedCNN(5, 4), object()))


def test_agent_with_k7_but_not_k8_gets_the_library_layers_buffers():
    """Dense layers of 128 on 5x4: K7 fits, K8 does not; the agent keeps the logits buffer the draw reads."""
    from overcooked_ai_b200.selfplay import _NetworkAgent

    env = SimpleNamespace(layouts=[SimpleNamespace(width=5, height=4)], device=torch.device("cpu"), n_layouts=1, n_envs=3)
    a = _NetworkAgent(env, RllibShapedCNN(5, 4, hidden=128), 0, None, 0, torch.bfloat16)
    assert a.fused_first_layer and not a.fused_tail and a._scores.shape == (3, 6)
