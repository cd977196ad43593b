"""ctypes binding of the C ABI in include/ovc_b200.h (csrc/libovc_b200.so).

There is no CPU fallback anywhere in this package: if the CUDA library is missing or a CUDA
device is not available, the calls below raise.  Build it with ``python -m overcooked_ai_b200.build``
(or ``__graft_entry__.build()``).
"""
import ctypes
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.environ.get("OVC_B200_LIB") or os.path.join(_HERE, "csrc", "libovc_b200.so")  # OVC_B200_LIB: an experiment build (build.py)

ABI_VERSION = 5
F_AUTO_RESET = 1
F_PDL = 2
F_ACT_U8 = 4
F_OUT_NARROW = 8
F_OUT_PACKED = 16
F_OUT_CODES = 32
F_ACT_PACKED = 64
F_OUT_STREAM = 128
F_STREAM_CAP_SHIFT = 16
STREAM_CAP_MAX = 0xFFFF
F_IO_SHIFT = 8
IO_DEFAULT, IO_TMA_TENSOR, IO_TMA_BULK, IO_DIRECT = 0, 1, 2, 3
DT_F32, DT_U8, DT_I32, DT_BF16 = 0, 1, 2, 3



class RandomStart(ctypes.Structure):
    """ovc_random_start_t (include/ovc_b200.h): random start states, passed by host pointer."""
    _fields_ = [("seed", ctypes.c_uint64), ("obj_threshold", ctypes.c_uint32), ("random_start_pos", ctypes.c_int32),
                ("random_layout", ctypes.c_int32), ("reserved", ctypes.c_int32)]


class EpisodeStatsDesc(ctypes.Structure):
    """ovc_episode_stats_t (include/ovc_b200.h): device pointers of the episode statistics, passed by host pointer."""
    _fields_ = [(k, ctypes.c_void_p) for k in (
        "layouts", "state", "events", "partner_seat", "event_counts", "sparse_by_agent", "shaped_by_agent", "reward_by_agent",
        "ep_length", "layout_id", "count", "dropped", "rec_length", "rec_layout", "rec_partner_seat", "rec_sparse_by_agent",
        "rec_shaped_by_agent", "rec_event_counts", "rec_reward_by_agent")] + [("capacity", ctypes.c_int32), ("state_words", ctypes.c_int32)]


class PipelineDesc(ctypes.Structure):
    """ovc_pipeline_desc_t (include/ovc_b200.h)"""
    _fields_ = [("layouts", ctypes.c_void_p), ("n_layouts", ctypes.c_int32), ("state_words", ctypes.c_int32),
                ("start_records", ctypes.c_void_p), ("state", ctypes.c_void_p), ("n_envs", ctypes.c_int64),
                ("horizon", ctypes.c_int32), ("flags", ctypes.c_int32), ("chunk", ctypes.c_int32),
                ("has_random_start", ctypes.c_int32), ("random_start", RandomStart),
                ("d_actions", ctypes.c_void_p * 2), ("d_sparse", ctypes.c_void_p * 2), ("d_shaped", ctypes.c_void_p * 2),
                ("d_done", ctypes.c_void_p * 2), ("d_events", ctypes.c_void_p * 2),
                ("stream_cap", ctypes.c_int32), ("reserved", ctypes.c_int32), ("d_codes_full", ctypes.c_void_p * 2)]


_lib = None


class NativeLibraryError(RuntimeError):
    pass


def lib():
    """Load (once) and return the CUDA library; raises NativeLibraryError if it is not built."""
    global _lib
    if _lib is not None:
        return _lib
    if not os.path.exists(LIB_PATH):
        raise NativeLibraryError(
            "%s not found: the CUDA extension is not built (python -m overcooked_ai_b200.build). "
            "This engine has no CPU fallback." % LIB_PATH
        )
    L = ctypes.CDLL(LIB_PATH)
    vp, i32, i64 = ctypes.c_void_p, ctypes.c_int, ctypes.c_int64
    L.ovc_abi_version.restype = i32
    L.ovc_layout_table_size.restype = ctypes.c_size_t
    L.ovc_feat_lut_entry_size.restype = ctypes.c_size_t
    L.ovc_last_error.restype = ctypes.c_char_p
    L.ovc_step.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, vp, vp]
    L.ovc_rollout.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, i32, vp, vp]
    L.ovc_reset.argtypes = [vp, i32, vp, vp, vp, vp, i64, i32, vp, vp]
    L.ovc_encode_lossless.argtypes = [vp, i32, vp, vp, vp, i32, i64, i32, i32, i32, i32, vp]
    L.ovc_encode_linear.argtypes = [vp, i32, vp, vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, ctypes.c_float, vp]
    L.ovc_sample_actions.argtypes = [vp, i32, i32, i64, ctypes.c_uint64, vp, vp, vp]
    L.ovc_accumulate_returns.argtypes = [vp, vp, ctypes.c_float, i64, vp, vp, vp]
    L.ovc_policy_tail.argtypes = [vp, i64, i32, ctypes.c_float, vp, vp, vp, vp, i32, vp, vp, ctypes.c_float, i32, ctypes.c_uint64, vp, vp, vp, vp, vp]
    L.ovc_policy_tail_logp.argtypes = L.ovc_policy_tail.argtypes[:-1] + [vp, vp]
    L.ovc_policy_hidden.argtypes = [vp, i64, i32, ctypes.c_float, vp, vp, vp, vp, i32, ctypes.c_float, vp, vp]
    L.ovc_lstm_head.argtypes = [vp, vp, vp, vp, i64, vp, vp, vp, vp, i32, ctypes.c_uint64, vp, vp, vp, vp, vp, vp, vp, vp, vp, vp]
    L.ovc_sample_actions_logp.argtypes = [vp, i32, i32, i64, ctypes.c_uint64, vp, vp, vp, vp]
    L.ovc_encode_linear_view.argtypes = [vp, i32, vp, vp, i32, vp, vp, vp, i64, i32, i32, i32, i32, i32, ctypes.c_float, vp]
    L.ovc_sample_actions_view.argtypes = [vp, i32, i32, i64, ctypes.c_uint64, vp, vp, i32, vp, vp, vp]
    L.ovc_policy_tail_view.argtypes = L.ovc_policy_tail.argtypes[:15] + [vp, i32, vp, vp, vp, vp, vp]
    L.ovc_lstm_head_view.argtypes = L.ovc_lstm_head.argtypes[:12] + [vp, i32] + L.ovc_lstm_head.argtypes[12:]
    L.ovc_record_transition.argtypes = [vp, vp, vp, vp, i64, vp, vp, vp, vp, vp]
    L.ovc_record_transition_stats.argtypes = [vp, vp, vp, vp, i64, vp, vp, vp, vp, ctypes.POINTER(EpisodeStatsDesc), vp]
    L.ovc_gae.argtypes = [vp, vp, vp, vp, i64, i64, ctypes.c_float, ctypes.c_float, vp, vp, vp]
    L.ovc_record_transition_view.argtypes = [vp, vp, vp, vp, i64, vp, i32, vp, vp, vp, vp, ctypes.POINTER(EpisodeStatsDesc), vp]
    L.ovc_gae_view.argtypes = L.ovc_gae.argtypes
    L.ovc_wide_layers.argtypes = [vp, i64, i32, vp, vp, i32, vp, vp, i32, ctypes.c_float, vp, vp]
    L.ovc_featurize.argtypes = [vp, i32, vp, vp, vp, vp, i64, i32, i32, vp]
    L.ovc_partner_policy.argtypes = [vp, i32, vp, vp, vp, i64, i32, i32, i32, vp, vp, vp, vp, i32, vp, vp, i32, ctypes.c_uint64, vp, vp, vp, vp]
    L.ovc_assign_partners.argtypes = [vp, vp, i64, ctypes.c_uint64, vp, vp, vp]
    L.ovc_group_members.argtypes = [vp, i32, i64, vp, vp, vp]
    L.ovc_assign_members.argtypes = [vp, vp, i32, i64, ctypes.c_uint64, vp, vp, vp, vp, i32, vp]
    L.ovc_encode_linear_rows.argtypes = L.ovc_encode_linear_view.argtypes[:5] + [vp, vp] + L.ovc_encode_linear_view.argtypes[5:]
    L.ovc_wide_layers_range.argtypes = L.ovc_wide_layers.argtypes[:10] + [vp, vp, vp]
    L.ovc_policy_tail_rows.argtypes = L.ovc_policy_tail.argtypes[:15] + [vp, i32, vp, vp, vp, vp, vp, vp, vp]
    L.ovc_sample_actions_rows.argtypes = [vp, i32, i32, i64, ctypes.c_uint64, vp, vp, i32, vp, vp, vp, vp, vp]
    L.ovc_learner_rows.argtypes = [vp, i64, vp, vp, vp, vp, vp]
    L.ovc_encode_linear_masked.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, i64, i32, i32, i32, i32, i32, ctypes.c_float, vp]
    L.ovc_policy_tail_joint.argtypes = L.ovc_policy_tail.argtypes[:15] + [vp, vp, vp, vp, vp, vp, vp]
    L.ovc_encode_linear_wgrad.argtypes = [vp, i32, vp, vp, i32, vp, vp, i64, i32, i32, i32, i32, i32, vp]
    L.ovc_policy_tail_grouped.argtypes = L.ovc_policy_tail.argtypes[:15] + [vp, i32, vp, vp, vp, vp, vp]
    L.ovc_encode_linear_grouped.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp, i64, i32, i32, i32, i32, i32, ctypes.c_float, vp]
    L.ovc_wide_layers_grouped.argtypes = L.ovc_wide_layers.argtypes[:10] + [vp, i32, vp, vp]
    L.ovc_assign_pairs.argtypes = L.ovc_assign_members.argtypes
    L.ovc_group_pairs.argtypes = [vp, i32, i64, vp, vp, vp, vp, vp, vp]
    L.ovc_encode_linear_grouped_masked.argtypes = [vp, i32, vp, vp, vp, vp, vp, vp, i32, vp, i64, i32, i32, i32, i32, i32, ctypes.c_float, vp]
    L.ovc_policy_tail_grouped_joint.argtypes = L.ovc_policy_tail.argtypes[:15] + [vp, vp, i32, vp, vp, vp, vp, vp]
    L.ovc_potential.argtypes = [vp, i32, vp, vp, vp, i32, vp, vp, i64, i32, vp]
    L.ovc_potential_table_size.restype = ctypes.c_size_t
    L.ovc_potential_shaping.argtypes = [vp, i32, vp, vp, vp, vp, i32, vp, vp, vp, vp, i64, i32, vp, vp]
    L.ovc_record_transition_dense.argtypes = [vp, vp, vp, vp, vp, i64, i32, vp, vp, vp, vp, ctypes.POINTER(EpisodeStatsDesc), vp]
    L.ovc_expand_codes_host.argtypes = [vp, i64, i64, vp, vp, i32, vp, vp, vp, vp, i32]
    L.ovc_expand_stream_host.argtypes = [vp, vp, i64, i64, i64, i64, vp, vp, i32, vp, vp, vp, vp, i32, ctypes.POINTER(i64)]
    L.ovc_pipeline_create.argtypes = [ctypes.POINTER(PipelineDesc), ctypes.POINTER(vp)]
    L.ovc_pipeline_run.argtypes = [vp, vp, vp, vp, vp, vp, i32, vp, i32, ctypes.POINTER(i64)]
    L.ovc_pipeline_wait.argtypes = [vp, i64]
    L.ovc_pipeline_join.argtypes = [vp, vp]
    L.ovc_pipeline_destroy.argtypes = [vp]
    L.ovc_pipeline_destroy.restype = None
    for f in (L.ovc_step, L.ovc_rollout, L.ovc_reset, L.ovc_encode_lossless, L.ovc_encode_linear, L.ovc_sample_actions, L.ovc_accumulate_returns, L.ovc_policy_tail, L.ovc_wide_layers, L.ovc_featurize, L.ovc_potential,
              L.ovc_policy_tail_logp, L.ovc_policy_hidden, L.ovc_lstm_head,
              L.ovc_encode_linear_view, L.ovc_sample_actions_view, L.ovc_policy_tail_view, L.ovc_lstm_head_view, L.ovc_sample_actions_logp, L.ovc_record_transition, L.ovc_record_transition_stats, L.ovc_gae, L.ovc_record_transition_view, L.ovc_gae_view, L.ovc_partner_policy, L.ovc_assign_partners,
              L.ovc_group_members, L.ovc_assign_members, L.ovc_encode_linear_rows, L.ovc_wide_layers_range, L.ovc_policy_tail_rows, L.ovc_sample_actions_rows,
              L.ovc_learner_rows, L.ovc_encode_linear_masked, L.ovc_policy_tail_joint, L.ovc_potential_shaping, L.ovc_record_transition_dense, L.ovc_encode_linear_wgrad, L.ovc_policy_tail_grouped, L.ovc_encode_linear_grouped, L.ovc_wide_layers_grouped, L.ovc_assign_pairs, L.ovc_group_pairs, L.ovc_encode_linear_grouped_masked, L.ovc_policy_tail_grouped_joint, L.ovc_expand_codes_host, L.ovc_expand_stream_host, L.ovc_pipeline_create, L.ovc_pipeline_run, L.ovc_pipeline_wait, L.ovc_pipeline_join):
        f.restype = i32
    if L.ovc_abi_version() != ABI_VERSION:
        raise NativeLibraryError("ABI version mismatch: library %d, binding %d" % (L.ovc_abi_version(), ABI_VERSION))
    _lib = L
    return L


EXPORTED_SYMBOLS = (
    "ovc_abi_version", "ovc_layout_table_size", "ovc_feat_lut_entry_size", "ovc_last_error",
    "ovc_step", "ovc_rollout", "ovc_reset", "ovc_encode_lossless", "ovc_encode_linear", "ovc_sample_actions", "ovc_accumulate_returns", "ovc_policy_tail", "ovc_wide_layers", "ovc_featurize", "ovc_potential",
    "ovc_potential_table_size", "ovc_expand_codes_host", "ovc_expand_stream_host",
    "ovc_policy_tail_logp", "ovc_sample_actions_logp", "ovc_record_transition", "ovc_record_transition_stats", "ovc_gae",
    "ovc_partner_policy", "ovc_assign_partners", "ovc_policy_hidden", "ovc_lstm_head",
    "ovc_encode_linear_view", "ovc_sample_actions_view", "ovc_policy_tail_view", "ovc_lstm_head_view",
    "ovc_record_transition_view", "ovc_gae_view",
    "ovc_group_members", "ovc_assign_members", "ovc_encode_linear_rows", "ovc_wide_layers_range", "ovc_policy_tail_rows",
    "ovc_sample_actions_rows", "ovc_learner_rows", "ovc_encode_linear_masked", "ovc_policy_tail_joint",
    "ovc_potential_shaping", "ovc_record_transition_dense", "ovc_encode_linear_wgrad", "ovc_policy_tail_grouped",
    "ovc_encode_linear_grouped", "ovc_wide_layers_grouped", "ovc_assign_pairs", "ovc_group_pairs", "ovc_encode_linear_grouped_masked",
    "ovc_policy_tail_grouped_joint",
    "ovc_pipeline_create", "ovc_pipeline_run", "ovc_pipeline_wait", "ovc_pipeline_join", "ovc_pipeline_destroy",
)


def check(rc):
    if rc != 0:
        raise RuntimeError("ovc native call failed (%d): %s" % (rc, lib().ovc_last_error().decode()))
