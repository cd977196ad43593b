"""overcooked_ai_b200 — H100-native batched Overcooked MDP step engine.

Only the data-parallel hot path of HumanCompatibleAI/overcooked_ai lives here (SURVEY.md §8):
``OvercookedGridworld.get_state_transition`` / ``lossless_state_encoding`` / ``featurize_state``
and ``OvercookedEnv.step`` / ``reset``, behind the reference's own call surface, executed by
hand-written sm_90a CUDA kernels through the C ABI of include/ovc_b200.h.
"""
from overcooked_ai_b200.actions import Action, Direction  # noqa: F401
from overcooked_ai_b200.state import (  # noqa: F401
    ObjectState,
    OvercookedState,
    PlayerState,
    Recipe,
    SoupState,
)

__version__ = "0.1.0"
