"""Wire / on-disk formats <-> packed tensors, in bulk (SURVEY.md §8f row 4).

The reference speaks three formats around the hot path:
  * ``OvercookedState.to_dict()`` JSON (overcooked_mdp.py:998-1015; soups :615-663) — the demo server, the
    human-trial CSVs (``state`` column) and ``AgentEvaluator.save_traj_as_json`` (benchmarking.py:431-502);
  * joint actions as direction lists / ``"interact"`` (``joint_action`` column, actions.py:47-52);
  * trajectory dicts (overcooked_trajectory.py:14-44): ``ep_states / ep_actions / ep_rewards / ep_dones /
    ep_infos / ep_returns / ep_lengths / mdp_params / env_params / metadatas``.
These helpers move whole batches between those and the engine's ``state[N, S]`` / ``actions[T, N, 2]``
tensors, so recorded games can be replayed on the device and device rollouts can be handed to tools that
expect the reference's files.  Host side only; nothing here is on the per-step path.
"""
import json

import numpy as np

from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.actions import Action
from overcooked_ai_b200.state import OvercookedState


def records_from_dicts(layout, state_dicts, layout_id=0, state_words=None):
    """List of ``to_dict()`` dicts (or JSON strings) -> int32 [N, S] records."""
    S = layout.state_words if state_words is None else state_words
    out = np.zeros((len(state_dicts), S), np.int32)
    for i, d in enumerate(state_dicts):
        if isinstance(d, str):
            d = json.loads(d)
        out[i] = L.pack_state(layout, OvercookedState.from_dict(d), layout_id, S)
    return out


def dicts_from_records(layout, records):
    """int32 [N, S] records -> list of ``to_dict()`` dicts (JSON-ready: tuples become lists)."""
    return [json.loads(json.dumps(L.unpack_state(layout, r).to_dict())) for r in np.asarray(records)]


def action_indices(joint_actions):
    """Reference joint actions (tuples / lists of direction pairs, "interact", any capitalisation; or their JSON
    strings) -> int32 [N, 2] action indices."""
    out = np.zeros((len(joint_actions), 2), np.int32)
    for i, ja in enumerate(joint_actions):
        if isinstance(ja, str):
            ja = json.loads(ja)
        for p in range(2):
            a = ja[p]
            a = a.lower() if isinstance(a, str) else tuple(a)
            out[i, p] = Action.to_index(a)
    return out


def joint_actions_from_indices(idx):
    """int [N, 2] -> list of reference joint-action tuples."""
    return [tuple(Action.INDEX_TO_ACTION[int(a)] for a in row) for row in np.asarray(idx)]


def trajectories_from_rollout(layout, states, actions, sparse, done, mdp_params=None, env_params=None):
    """Device rollout outputs -> the reference's trajectory dict (overcooked_trajectory.py:14-44).

    states   int32 [T+1, N, S] (state before each transition, plus the final one) or [T, N, S]
    actions  int   [T, N, 2];  sparse int [T, N];  done int [T, N]
    One trajectory per environment, cut at its first ``done`` (or T).  ``ep_states`` holds OvercookedState
    objects like the reference's (``to_dict`` them for JSON); ``ep_infos`` carries empty dicts.
    """
    states, actions, sparse, done = (np.asarray(x) for x in (states, actions, sparse, done))
    T, N = actions.shape[:2]
    traj = {k: [] for k in ("ep_states", "ep_actions", "ep_rewards", "ep_dones", "ep_infos", "ep_returns", "ep_lengths",
                            "mdp_params", "env_params")}
    traj["metadatas"] = {}
    for e in range(N):
        ends = np.nonzero(done[:, e])[0]
        length = int(ends[0]) + 1 if len(ends) else T
        traj["ep_states"].append([L.unpack_state(layout, states[t, e]) for t in range(length)])
        traj["ep_actions"].append(joint_actions_from_indices(actions[:length, e]))
        traj["ep_rewards"].append([int(r) for r in sparse[:length, e]])
        traj["ep_dones"].append([bool(d) for d in done[:length, e]])
        traj["ep_infos"].append([{} for _ in range(length)])
        traj["ep_returns"].append(int(sparse[:length, e].sum()))
        traj["ep_lengths"].append(length)
        traj["mdp_params"].append(mdp_params if mdp_params is not None else {"layout_name": layout.layout_name})
        traj["env_params"].append(env_params if env_params is not None else {"horizon": length})
    for k in ("ep_returns", "ep_lengths"):
        traj[k] = np.array(traj[k])
    return traj


def replay_table(layout, state_dicts, joint_actions, rewards=None):
    """A recorded game (rows of state JSON + joint action, e.g. a human-trial CSV) as tensors ready for the
    engine: (records int32 [N, S], actions int32 [N, 2], rewards int64 [N] or None)."""
    rec = records_from_dicts(layout, state_dicts)
    act = action_indices(joint_actions)
    rew = None if rewards is None else np.asarray(rewards).astype(np.int64)
    return rec, act, rew


_DELIVERY_ROWS = [r for r in range(1, 16) if (r >> 2) + (r & 3) <= 3]  # n_onion*4 + n_tomato: 1,2,3,4,5,6,8,9,12 (code 23 + rank)


def _event_code_table():
    """32 event codes (include/ovc_b200.h, OVC_F_OUT_PACKED) -> int32 event mask incl. the delivered-recipe bits."""
    E = {n: i for i, n in enumerate(L.EVENT_TYPES)}
    t = np.zeros(32, np.int64)
    for k, obj in enumerate(("onion", "tomato", "dish")):
        for useful in (0, 1):
            t[1 + 2 * k + useful] = (1 << E[obj + "_pickup"]) | (useful << E["useful_" + obj + "_pickup"])
            t[8 + 2 * k + useful] = (1 << E[obj + "_drop"]) | (useful << E["useful_" + obj + "_drop"])
    t[7], t[14] = 1 << E["soup_pickup"], 1 << E["soup_drop"]
    for k, obj in enumerate(("onion", "tomato")):
        base = 1 << E["potting_" + obj]
        combos = (("optimal", "viable"), ("viable",), ("catastrophic",), ("optimal", "useless"))
        for c, names in enumerate(combos):
            t[15 + 4 * k + c] = base | sum(1 << E["%s_%s_potting" % (nm, obj)] for nm in names)
    for rank, row in enumerate(_DELIVERY_ROWS):
        t[23 + rank] = (1 << E["soup_delivery"]) | (row << L.EV_RECIPE_SHIFT)
    return t.astype(np.int32)


EVENT_CODE_TABLE = _event_code_table()


def pack_actions(actions):
    """int array [..., 2] of action indices -> uint8 [...]: agent 0 in bits 0-3, agent 1 in bits 4-7 (OVC_F_ACT_PACKED)."""
    a = np.asarray(actions)
    assert a.shape[-1] == 2 and a.min() >= 0 and a.max() < 6
    return (a[..., 0] | (a[..., 1] << 4)).astype(np.uint8)


def code_reward_table(layouts):
    """int32 [n_layouts, 2, 32]: [l][0][code] = delivery reward of the code's recipe on layout l, [l][1][code] = the
    shaped reward an agent gets WITH that code when its grant bit is set (include/ovc_b200.h, OVC_F_OUT_CODES)."""
    t = np.zeros((len(layouts), 2, 32), np.int32)
    for i, l in enumerate(layouts):
        for rank, row in enumerate(_DELIVERY_ROWS):
            t[i, 0, 23 + rank] = int(l.deliver_value[row])
        t[i, 1, 15:23] = int(l.reward_shaping_params["PLACEMENT_IN_POT_REW"])
        t[i, 1, 6] = int(l.reward_shaping_params["DISH_PICKUP_REWARD"])
        t[i, 1, 7] = int(l.reward_shaping_params["SOUP_PICKUP_REWARD"])
    return t


def decode_codes(evcode, reward_tbl, env_layout=None):
    """numpy reference of ovc_expand_codes_host: int16 [..., N] OVC_F_OUT_CODES words ->
    (sparse int64 [..., N], shaped int64 [..., N, 2], done bool, events int32 [..., N, 2])."""
    w = np.asarray(evcode).astype(np.int32) & 0xFFFF
    c = np.stack([w & 31, (w >> 5) & 31], -1)
    lay = np.zeros(w.shape[-1], np.int64) if env_layout is None else np.asarray(env_layout).astype(np.int64)
    lay = np.broadcast_to(lay, w.shape)[..., None]
    grant = np.stack([(w >> 12) & 1, (w >> 13) & 1], -1)
    sparse = reward_tbl[lay, 0, c].sum(-1).astype(np.int64)
    shaped = (reward_tbl[lay, 1, c] * grant).astype(np.int64)
    events, done = decode_event_codes(w & 0xFFF)
    return sparse, shaped, done, events


def decode_event_codes(evcode):
    """int16 [...] packed event codes -> (events int32 [..., 2], done bool [...]) exactly as the int32 formats."""
    ev = np.asarray(evcode).astype(np.int32)
    events = np.stack([EVENT_CODE_TABLE[ev & 31], EVENT_CODE_TABLE[(ev >> 5) & 31]], -1)
    stepped = ((ev >> 11) & 1).astype(bool)
    events[stepped] = L.EVF_STEPPED_DONE
    return events, ((ev >> 10) & 1).astype(bool)
