"""CPU tests of the host logic: layout compiler, value types, the C-ABI library's exports,
and the multi-process sharding helpers (gloo, world_size 2)."""
import ctypes
import os
import subprocess
import sys

import numpy as np
import pytest

from overcooked_ai_b200 import _native
from overcooked_ai_b200 import layout as L
from overcooked_ai_b200.actions import Action, Direction
from overcooked_ai_b200.state import ObjectState, OvercookedState, PlayerState, Recipe, SoupState

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_native_library_loads_and_exports_every_declared_symbol():
    """Every function include/ovc_b200.h declares is exported by the built library (no compute calls)."""
    import re

    hdr = open(os.path.join(ROOT, "include", "ovc_b200.h")).read()
    declared = set(re.findall(r"\b(ovc_[a-z_0-9]+)\s*\(", hdr)) - {"ovc_layout", "ovc_feat_lut_entry"}
    assert declared == set(_native.EXPORTED_SYMBOLS)
    lib = _native.lib()
    for sym in declared:
        assert hasattr(lib, sym), sym
    assert lib.ovc_abi_version() == _native.ABI_VERSION == 5
    assert lib.ovc_layout_table_size() == L.LAYOUT_DTYPE.itemsize == 1024
    assert lib.ovc_feat_lut_entry_size() == L.FEAT_LUT_DTYPE.itemsize == 12


def test_product_package_never_touches_the_oracle():
    """The product path must not import / link / execute anything under oracle/."""
    pkg = os.path.join(ROOT, "overcooked_ai_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in src.replace("# no oracle", ""), f


def test_missing_cuda_device_fails_loudly():
    import torch

    if torch.cuda.is_available():
        pytest.skip("a GPU is present")
    from overcooked_ai_b200.batched import BatchedOvercookedEnv

    with pytest.raises(RuntimeError, match="no CPU fallback"):
        BatchedOvercookedEnv("cramped_room", 4)


def test_recipe_tables_of_the_five_classic_layouts():
    """SURVEY.md §8a table (probed from the reference)."""
    for name in ("cramped_room", "asymmetric_advantages", "coordination_ring", "forced_coordination"):
        l = L.compile_layout(name)
        assert set(l.cook_time[[4, 1, 8, 5, 2, 12, 9, 6, 3]]) == {20}
        assert l.deliver_value[12] == 20 and l.deliver_value.sum() == 20
        assert l.best_value[[0, 4, 8, 12]].tolist() == [20] * 4 and l.best_value[[1, 5, 2, 9, 6, 3]].sum() == 0
    cc = L.compile_layout("counter_circuit")
    assert cc.cook_time[12] == 45 and cc.base_value[12] == 63
    assert (cc.deliver_value[5], cc.deliver_value[9], cc.deliver_value[6]) == (68, 55, 47)
    assert cc.best_value[[0, 4, 1, 8, 5, 2, 12, 9, 6, 3]].tolist() == [68, 68, 68, 55, 68, 47, 0, 55, 47, 0]
    t = L.compile_layout("mdp_test")
    assert (t.deliver_value[4], t.deliver_value[12], t.deliver_value[9]) == (10, 30, 50)
    assert t.cook_time[9] == 6


def test_layouts_are_independent_no_global_recipe_state():
    """Quirk Q1 does not exist here: compiling counter_circuit does not change cramped_room."""
    a = L.compile_layout("cramped_room")
    L.compile_layout("counter_circuit")
    b = L.compile_layout("cramped_room")
    assert np.array_equal(a.cook_time, b.cook_time) and np.array_equal(a.deliver_value, b.deliver_value)


def test_state_words_and_slots():
    exp = {"cramped_room": (16, 10, 1), "asymmetric_advantages": (32, 25, 2), "coordination_ring": (32, 13, 2),
           "forced_coordination": (32, 15, 2), "counter_circuit": (32, 25, 2), "corridor": (128, 63, 2)}
    for name, (S, slots, pots) in exp.items():
        l = L.compile_layout(name)
        assert (l.state_words, l.n_slots, l.n_pots) == (S, slots, pots)
        assert l.slot_positions[:pots] == l.pot_locations
    with pytest.raises(ValueError):
        L.compile_layout("cramped_room_single")  # 1 player
    with pytest.raises(ValueError):
        L.compile_layout("tutorial_3")  # order_bonus = inf: rewards are not integers


def test_start_records():
    tab, starts, S = L.build_tables([L.compile_layout(n) for n in ("cramped_room", "counter_circuit")])
    assert S == 32 and tab.shape == (2, 1024) and starts.shape == (2, 32)
    # cramped_room: P0 (1,2) P1 (3,1) facing north, nothing held, t = 0 (SURVEY §8a)
    assert starts[0, :4].tolist() == [0, (2 << 4) | 1, (1 << 4) | 3, 0] and not starts[0, 4:].any()
    assert starts[1, 3] == 1


def test_pack_unpack_objects_and_soups():
    l = L.compile_layout("mdp_test")
    soup = SoupState((2, 0), [ObjectState("onion", (2, 0)), ObjectState("tomato", (2, 0))], cooking_tick=3)
    held = SoupState.get_soup((1, 1), 2, 1, cooking_tick=6, cook_time=6)
    st = OvercookedState(
        [PlayerState((1, 1), Direction.EAST, held), PlayerState((3, 1), Direction.WEST, ObjectState("dish", (3, 1)))],
        {(2, 0): soup, (0, 0): ObjectState("dish", (0, 0)), (4, 0): ObjectState("tomato", (4, 0))},
        bonus_orders=l.start_bonus_orders, all_orders=l.start_all_orders, timestep=17)
    rec = L.pack_state(l, st)
    assert rec[0] == 17 and (rec[3] >> 8) & 0xFF == 1  # one loose dish
    back = L.unpack_state(l, rec)
    assert back == st and back.get_object((2, 0)).ingredients == ["onion", "tomato"]
    assert back.get_object((2, 0)).cook_time == 4 and back.players[0].held_object.is_ready
    # ordered ingredients survive (quirk Q6)
    soup2 = SoupState((2, 0), [ObjectState("tomato", (2, 0)), ObjectState("onion", (2, 0))], cooking_tick=3)
    assert L.pack_object(soup) != L.pack_object(soup2)
    # a tick with bit 13 set lands in the sign bit of the player word and still round-trips
    big = SoupState.get_soup((1, 1), 3, 0, cooking_tick=9000, cook_time=6)
    st2 = OvercookedState([PlayerState((1, 1), Direction.EAST, big), PlayerState((3, 1), Direction.WEST)], {},
                          bonus_orders=l.start_bonus_orders, all_orders=l.start_all_orders)
    rec2 = L.pack_state(l, st2)
    assert rec2[1] < 0 and L.unpack_state(l, rec2).players[0].held_object._cooking_tick == 9000


def test_value_types_wire_format():
    d = {"players": [{"position": [1, 2], "orientation": [0, -1], "held_object": {"name": "onion", "position": [1, 2]}},
                     {"position": [3, 1], "orientation": [1, 0], "held_object": None}],
         "objects": [{"name": "soup", "position": [2, 0], "_ingredients": [{"name": "onion", "position": [2, 0]}],
                      "cooking_tick": -1, "is_cooking": False, "is_ready": False, "is_idle": True, "cook_time": -1,
                      "_cooking_tick": -1}],
         "bonus_orders": [], "all_orders": [{"ingredients": ["onion", "onion", "onion"]}], "timestep": 3}
    st = OvercookedState.from_dict(d)
    assert st.players[0].held_object == ObjectState("onion", (1, 2)) and st.timestep == 3
    out = st.to_dict()
    assert out["objects"][0]["cook_time"] == -1 and out["objects"][0]["is_idle"] is True
    assert OvercookedState.from_dict(out) == st and st.deepcopy() == st
    assert Recipe(["onion", "tomato"]) == Recipe(["tomato", "onion"]) and len(Recipe.all_recipes()) == 9
    assert Action.to_index("interact") == 5 and Action.to_index((0, 0)) == 4 and Action.to_index([0, -1]) == 0
    with pytest.raises(ValueError):
        Action.to_index((1, 1))


def test_soups_without_an_explicit_cook_time_behave_like_the_reference():
    """Legacy (2019) soup dicts and get_soup(finished=True) carry no cook time: the reference falls back to Recipe.time
    (20 with nothing configured, overcooked_mdp.py:523-530,565-569,638-656); so do these."""
    legacy = SoupState.from_dict({"name": "soup", "position": (1, 0), "state": ("onion", 3, 20)})
    assert legacy.ingredients == ["onion"] * 3 and legacy._cooking_tick == 20 and legacy.is_ready and not legacy.is_cooking
    assert legacy.to_dict()["cook_time"] == 20 and legacy.cook_time_remaining == 0
    cooking = SoupState.from_dict({"name": "soup", "position": (1, 0), "state": ("onion", 2, 5)})
    assert cooking.is_cooking and cooking.to_dict()["is_cooking"] and cooking.cook_time == 20 and cooking.cook_time_remaining == 15
    idle = SoupState.from_dict({"name": "soup", "position": (1, 0), "state": ("onion", 1, 0)})
    assert idle.is_idle and idle.to_dict()["cook_time"] == -1
    tom = SoupState.from_dict({"name": "soup", "position": (1, 0), "state": ("tomato", 2, 7)})
    assert tom.ingredients == ["onion", "tomato", "tomato"], "the reference's tomato branch keeps get_soup's default onion"
    with pytest.raises(ValueError):
        SoupState.from_dict({"name": "soup", "position": (1, 0), "state": ("tomato", 3, 7)})
    done = SoupState.get_soup((2, 0), 3, 0, finished=True)
    assert done._cooking_tick == 20 and done.is_ready and done.recipe == Recipe(["onion"] * 3)
    assert SoupState.get_soup((2, 0), 1, 1, finished=True, cook_time=9)._cooking_tick == 9
    # a layout's own cook time replaces the fallback once the soup meets its layout
    cc = L.compile_layout("counter_circuit")
    rec = L.pack_state(cc, OvercookedState.from_dict({
        "players": [{"position": p, "orientation": (0, -1), "held_object": None} for p in cc.start_player_positions],
        "objects": [SoupState.get_soup(cc.slot_positions[0], 1, 1, cooking_tick=3).to_dict()],
        "bonus_orders": cc.start_bonus_orders, "all_orders": cc.start_all_orders, "timestep": 0}))
    soup = L.unpack_state(cc, rec).objects[cc.slot_positions[0]]
    assert soup.cook_time == 15 + 7 and soup.is_cooking and soup.to_dict()["cook_time"] == 22


def test_layout_file_in_reference_format(tmp_path):
    p = tmp_path / "tiny.layout"
    p.write_text('{"grid": """XPDX\n             O12S\n             XXXX""", "start_all_orders": [{"ingredients": ["onion"]}], "cook_time": 5, "delivery_reward": 7}')
    l = L.compile_layout(str(p))
    assert (l.width, l.height, l.n_pots) == (4, 3, 1) and l.cook_time[4] == 5 and l.deliver_value[4] == 7
    assert l.deliver_value[8] == 0 and l.best_value[0] == 7


def test_sharding_world_size_2_gloo():
    """Env-index sharding + seed broadcast + throughput all-reduce over gloo, 2 processes (the N>1 path
    of bench.py without a GPU)."""
    script = os.path.join(ROOT, "tests", "_dist_worker.py")
    port = 29500 + os.getpid() % 2000
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", str(port), script]
    env = dict(os.environ, PYTHONPATH=ROOT, OMP_NUM_THREADS="1")
    out = subprocess.run(cmd, capture_output=True, text=True, timeout=300, env=env)
    assert out.returncode == 0, out.stdout + out.stderr
    assert "DIST_OK" in out.stdout


def test_wire_formats_round_trip_with_reference_dicts():
    """to_dict JSON / joint-action lists / trajectory dicts <-> packed tensors (wire.py), on the reference's own
    dict samples stored in the fixtures (incl. real human-trial rows)."""
    import glob
    import json

    from overcooked_ai_b200 import wire

    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "trace_human2020_*.npz"))):
        d = np.load(path)
        cl = L.compile_layout(str(d["layout"]))
        sample = json.loads(str(d["to_dict_sample"]))
        dicts = [sample[k] for k in sorted(sample)]
        rec = wire.records_from_dicts(cl, [json.dumps(x) for x in dicts])
        assert rec.shape == (len(dicts), cl.state_words)
        assert np.array_equal(rec[0], d["states"][0, 0])
        back = wire.dicts_from_records(cl, rec)
        for a, b in zip(back, dicts):
            a["objects"].sort(key=lambda o: o["position"]), b["objects"].sort(key=lambda o: o["position"])
            assert a == b
    acts = wire.action_indices(['[[0, 0], "INTERACT"]', [[0, -1], [1, 0]], ("interact", (0, 1))])
    assert acts.tolist() == [[4, 5], [0, 2], [5, 1]]
    assert wire.joint_actions_from_indices(acts)[1] == ((0, -1), (1, 0))
    # trajectory dict of a recorded game: keys and shapes of overcooked_trajectory.py
    d = np.load(os.path.join(ROOT, "tests", "golden", "greedy_cramped_room.npz"))
    cl = L.compile_layout("cramped_room")
    states = d["states"].transpose(1, 0, 2)  # [T, E, S]
    actions = d["actions"].transpose(1, 0, 2)
    sparse = d["sparse"].sum(-1).T
    done = np.zeros_like(sparse)
    done[-1] = 1
    tr = wire.trajectories_from_rollout(cl, states, actions, sparse, done)
    assert set(tr) == {"ep_states", "ep_actions", "ep_rewards", "ep_dones", "ep_infos", "ep_returns", "ep_lengths",
                       "mdp_params", "env_params", "metadatas"}
    assert tr["ep_returns"].tolist() == [180] * 5 and tr["ep_lengths"].tolist() == [400] * 5
    assert tr["ep_states"][0][0] == cl.get_standard_start_state() and tr["ep_dones"][2][-1] is True
    assert tr["ep_actions"][0][0] == tuple(Action.INDEX_TO_ACTION[a] for a in d["actions"][0, 0])


def test_event_code_table_covers_every_mask_the_engine_can_produce():
    """wire.EVENT_CODE_TABLE (32 codes of the packed result format) contains every per-agent event mask that
    occurs in the reference-generated fixtures, once each — so decoding the 5-bit codes is lossless."""
    import glob

    from oracle import cpu
    from overcooked_ai_b200 import wire

    table = wire.EVENT_CODE_TABLE.astype(np.int64)
    assert len(set(table.tolist())) == 32 and table[0] == 0
    seen = set()
    for path in sorted(glob.glob(os.path.join(ROOT, "tests", "golden", "trace_*.npz"))):
        d = np.load(path)
        import json as _json

        cl = L.compile_layout(str(d["layout"]), **(_json.loads(str(d["params"])) if "params" in d else {}))
        tab, starts, S = L.build_tables([cl])
        st = np.ascontiguousarray(d["states"][:, :-1].reshape(-1, S)).copy()
        a = np.ascontiguousarray(d["actions"].reshape(-1, 2))
        _, _, _, ev = cpu.step(tab, starts, st, a, horizon=0)
        seen |= set(np.unique(ev.astype(np.int64) & 0x1FFFFFFF).tolist())
    assert seen <= set(table.tolist()), sorted(seen - set(table.tolist()))
    assert len(seen) >= 26


def test_host_expander_of_code_words_matches_the_numpy_decoder():
    """ovc_expand_codes_host (host code of the library, no GPU involved) against wire.decode_codes on random valid
    words, several layouts, threaded and not."""
    import torch

    from overcooked_ai_b200 import _native, wire

    lib = _native.lib()
    layouts = [L.compile_layout(n) for n in ("cramped_room", "counter_circuit", "asymmetric_advantages")]
    tbl = wire.code_reward_table(layouts)
    assert tbl[0, 0, 31] == 20 and tbl[1, 0].max() == 68 and tbl[0, 1, 15] == 3 and tbl[0, 1, 7] == 5 and tbl[0, 1, 5] == 0
    rng = np.random.RandomState(0)
    T, N = 37, 1501
    w = (rng.randint(0, 32, (T, N)) | (rng.randint(0, 32, (T, N)) << 5) | (rng.randint(0, 2, (T, N)) << 10)
         | ((rng.rand(T, N) < 0.05).astype(np.int64) << 11) | (rng.randint(0, 4, (T, N)) << 12)).astype(np.uint16).view(np.int16)
    lay = rng.randint(0, 3, N).astype(np.int32)
    want = wire.decode_codes(w, tbl, lay)
    for threads in (1, 5):
        sp, sh = np.zeros((T, N), np.int16), np.zeros((T, N, 2), np.int8)
        dn, ev = np.zeros((T, N), np.uint8), np.zeros((T, N, 2), np.int32)
        rc = lib.ovc_expand_codes_host(w.ctypes.data, T, N, lay.ctypes.data, tbl.ctypes.data, 3, sp.ctypes.data, sh.ctypes.data,
                                       dn.ctypes.data, ev.ctypes.data, threads)
        assert rc == 0
        assert np.array_equal(sp, want[0]) and np.array_equal(sh, want[1]) and np.array_equal(dn != 0, want[2])
        assert np.array_equal(ev, want[3])
    assert lib.ovc_expand_codes_host(w.ctypes.data, T, N, (lay + 5).ctypes.data, tbl.ctypes.data, 3, 0, 0, 0, 0, 1) != 0
    assert np.array_equal(wire.pack_actions(np.array([[5, 3], [0, 4]])), np.array([0x35, 0x40], np.uint8))


@pytest.mark.parametrize("N", [1000, 1024], ids=["ragged_rows", "cache_line_aligned_rows"])
def test_host_expander_of_the_sparse_event_stream(N):
    """ovc_expand_stream_host (host code of the library, no GPU involved): lane masks + compacted non-zero words built
    here with numpy from random code words, chunked as the pipeline chunks them; the expansion must equal the expansion
    of the dense words, count overflowing (chunk, group) slices, and read dropped words as zero."""
    from overcooked_ai_b200 import _native, wire

    lib = _native.lib()
    layouts = [L.compile_layout(n) for n in ("cramped_room", "counter_circuit")]
    tbl = wire.code_reward_table(layouts)
    rng = np.random.RandomState(3)
    T, chunk = 23, 8  # N = 1000: the last group is partial and rows are unaligned (memcpy path); 1024: streaming stores
    G, n_chunks = (N + 31) // 32, -(-T // chunk)
    w = (rng.randint(0, 32, (T, N)) | (rng.randint(0, 32, (T, N)) << 5) | (rng.randint(0, 2, (T, N)) << 10)
         | (rng.randint(0, 4, (T, N)) << 12)).astype(np.uint16)
    w[rng.rand(T, N) < 0.85] = 0
    lay = rng.randint(0, 2, N).astype(np.int32)

    def build(cap):
        masks, vals = np.zeros((T, G), np.uint32), np.zeros((n_chunks, G, cap), np.uint16)
        over = 0
        for c in range(n_chunks):
            for g in range(G):
                k = 0
                for t in range(c * chunk, min(T, (c + 1) * chunk)):
                    for l in range(32):
                        e = g * 32 + l
                        if e < N and w[t, e]:
                            masks[t, g] |= np.uint32(1) << np.uint32(l)
                            if k < cap:
                                vals[c, g, k] = w[t, e]
                            k += 1
                over += k > cap
        return masks, vals, over

    def expand(words):
        sp, sh = np.full((T, N), -1, np.int16), np.full((T, N, 2), -1, np.int8)
        dn, ev = np.full((T, N), 7, np.uint8), np.full((T, N, 2), -1, np.int32)
        assert lib.ovc_expand_codes_host(words.ctypes.data, T, N, lay.ctypes.data, tbl.ctypes.data, 2, sp.ctypes.data, sh.ctypes.data,
                                         dn.ctypes.data, ev.ctypes.data, 1) == 0
        return sp, sh, dn, ev

    want = expand(w)
    for cap, threads in ((chunk * 32, 1), (chunk * 32, 4), (40, 3)):
        masks, vals, n_over = build(cap)
        sp, sh = np.full((T, N), -1, np.int16), np.full((T, N, 2), -1, np.int8)
        dn, ev = np.full((T, N), 7, np.uint8), np.full((T, N, 2), -1, np.int32)
        over = ctypes.c_int64(-1)
        rc = lib.ovc_expand_stream_host(masks.ctypes.data, vals.ctypes.data, T, chunk, cap, N, lay.ctypes.data, tbl.ctypes.data, 2,
                                        sp.ctypes.data, sh.ctypes.data, dn.ctypes.data, ev.ctypes.data, threads, ctypes.byref(over))
        assert rc == 0 and over.value == n_over
        if n_over == 0:
            for got, wnt in zip((sp, sh, dn, ev), want):
                assert np.array_equal(got, wnt)
        else:  # dropped words read as zero: rebuild the dense words the stream still holds and compare with their expansion
            assert n_over > 0
            kept = w.copy()
            for c in range(n_chunks):
                for g in range(G):
                    k = 0
                    for t in range(c * chunk, min(T, (c + 1) * chunk)):
                        for l in range(32):
                            e = g * 32 + l
                            if e < N and w[t, e]:
                                if k >= cap:
                                    kept[t, e] = 0
                                k += 1
            for got, wnt in zip((sp, sh, dn, ev), expand(kept)):
                assert np.array_equal(got, wnt)
    assert lib.ovc_expand_stream_host(None, None, T, chunk, 8, N, 0, tbl.ctypes.data, 1, 0, 0, 0, 0, 1, None) != 0


def test_host_expander_pool_survives_concurrent_and_repeated_regions():
    """The persistent worker pool behind ovc_expand_codes_host: many regions with changing thread counts, issued
    from two host threads at once, all produce the right arrays and none hangs."""
    import threading

    from overcooked_ai_b200 import _native, wire

    lib = _native.lib()
    tbl = wire.code_reward_table([L.compile_layout("cramped_room")])
    rng = np.random.RandomState(1)
    T, N = 16, 20011
    w = (rng.randint(0, 32, (T, N)) | (rng.randint(0, 32, (T, N)) << 5) | (rng.randint(0, 4, (T, N)) << 12)).astype(np.uint16).view(np.int16)
    want = wire.decode_codes(w, tbl)
    errors = []

    def worker(seed):
        r = np.random.RandomState(seed)
        sp, sh = np.zeros((T, N), np.int16), np.zeros((T, N, 2), np.int8)
        for _ in range(60):
            sp[:] = -1
            thr = int(r.choice([1, 2, 3, 5, 8, 16]))
            if lib.ovc_expand_codes_host(w.ctypes.data, T, N, 0, tbl.ctypes.data, 1, sp.ctypes.data, sh.ctypes.data, 0, 0, thr) != 0:
                errors.append("rc")
            if not (np.array_equal(sp, want[0]) and np.array_equal(sh, want[1])):
                errors.append("mismatch with %d threads" % thr)

    ts = [threading.Thread(target=worker, args=(k,)) for k in range(2)]
    for t in ts:
        t.start()
    for t in ts:
        t.join(timeout=120)
    assert not any(t.is_alive() for t in ts), "expander pool deadlocked"
    assert not errors, errors[:3]


def test_pipeline_descriptor_layout_matches_the_c_struct():
    """ovc_pipeline_create validates its descriptor before it touches CUDA, so the argument checks double as a
    field-offset check of the ctypes mirror (no GPU needed): each error below is reached only if the fields before
    it were read where the C struct has them."""
    import ctypes

    from overcooked_ai_b200 import _native

    lib = _native.lib()
    assert ctypes.sizeof(_native.PipelineDesc) == 184 and _native.PipelineDesc.random_start.offset == 56
    assert _native.PipelineDesc.stream_cap.offset == 160 and _native.PipelineDesc.d_codes_full.offset == 168
    buf = (ctypes.c_char * 4096)()
    base = ctypes.addressof(buf) & ~15 | 16  # any non-null, 16-byte aligned address: nothing is dereferenced

    def create(**kw):
        d = _native.PipelineDesc()
        d.layouts, d.n_layouts, d.state_words, d.start_records, d.state = base, 1, 16, base, base
        d.n_envs, d.horizon, d.flags, d.chunk = 128, 400, _native.F_OUT_CODES | _native.F_ACT_PACKED, 8
        for b in range(2):
            d.d_actions[b], d.d_events[b] = base, base
        for k, v in kw.items():
            if isinstance(v, tuple):
                getattr(d, k)[v[0]] = v[1]
            else:
                setattr(d, k, v)
        h = ctypes.c_void_p()
        rc = lib.ovc_pipeline_create(ctypes.byref(d), ctypes.byref(h))
        return rc, lib.ovc_last_error().decode(), h

    for kw, msg in (({"chunk": 0}, "chunk must be >= 1"), ({"state_words": 24}, "state_words"), ({"n_layouts": 0}, "n_layouts"),
                    ({"n_envs": -1}, "negative n_envs"), ({"state": base + 4}, "16-byte aligned"),
                    ({"d_events": (1, None)}, "missing device staging buffer"), ({"d_actions": (0, None)}, "missing device staging buffer"),
                    ({"flags": _native.F_OUT_PACKED}, "missing device staging buffer"),  # packed also needs sparse / shaped
                    ({"flags": _native.F_OUT_STREAM | _native.F_ACT_PACKED}, "missing device staging buffer"),  # stream needs the value slots
                    ({"flags": _native.F_OUT_STREAM | _native.F_ACT_PACKED, "d_sparse": (0, base)}, "missing device staging buffer"),
                    ):
        rc, err, h = create(**kw)
        assert rc != 0 and msg in err and not h.value, (kw, rc, err)
    d = _native.PipelineDesc()  # stream format: the capacity field is read where the C struct has it
    d.layouts, d.n_layouts, d.state_words, d.start_records, d.state = base, 1, 16, base, base
    d.n_envs, d.horizon, d.flags, d.chunk = 128, 400, _native.F_OUT_STREAM | _native.F_ACT_PACKED, 8
    for b in range(2):
        d.d_actions[b], d.d_events[b], d.d_sparse[b] = base, base, base
    for cap in (0, 70000):
        d.stream_cap = cap
        h = ctypes.c_void_p()
        assert lib.ovc_pipeline_create(ctypes.byref(d), ctypes.byref(h)) != 0 and "stream_cap" in lib.ovc_last_error().decode()
    assert lib.ovc_pipeline_run(None, base, None, None, None, base, 1, None, 1, None) != 0
    assert lib.ovc_pipeline_wait(None, 0) != 0 and lib.ovc_pipeline_join(None, None) != 0
    lib.ovc_pipeline_destroy(None)


@pytest.mark.parametrize("fmt", ["int32", "narrow", "packed", "codes", "stream"])
def test_rollout_refuses_arrays_that_break_their_alignment(fmt):
    """ovc_rollout and ovc_step refuse an action or output array that is not aligned to the element size its transfer
    format stores it with (OVC_E_BADARG), and accept the same call with aligned arrays.  Every call has n_envs = 0 and is
    refused or accepted before anything is launched: no GPU is needed and no kernel runs."""
    lib = _native.lib()
    buf = (ctypes.c_char * 4096)()
    base = ctypes.addressof(buf) + (-ctypes.addressof(buf)) % 64  # 64-byte aligned; nothing is dereferenced
    stream = _native.F_OUT_STREAM | (8 << _native.F_STREAM_CAP_SHIFT)
    # output flag, and the alignment of sparse / shaped / done / events (0: the format does not use the array)
    out_flag, out_align = {"int32": (0, (4, 8, 4, 8)), "narrow": (_native.F_OUT_NARROW, (2, 2, 1, 8)),
                           "packed": (_native.F_OUT_PACKED, (2, 2, 0, 2)), "codes": (_native.F_OUT_CODES, (0, 0, 0, 2)),
                           "stream": (stream, (2, 0, 2, 4))}[fmt]
    for act_flag, act_align in ((0, 8), (_native.F_ACT_U8, 2), (_native.F_ACT_PACKED, 1)):
        flags = out_flag | act_flag
        calls = [lambda p: lib.ovc_rollout(base, 1, base, base, *p, 0, 3, 16, 400, flags, None, None)]
        if fmt != "stream":
            calls.append(lambda p: lib.ovc_step(base, 1, base, base, *p, 0, 16, 400, flags, None, None))
        for call in calls:
            ptrs = [base + 512 * k for k in range(5)]  # actions, sparse, shaped, done, events
            assert call(ptrs) == 0, lib.ovc_last_error().decode()
            for k, align in enumerate((act_align,) + out_align):
                if align > 1:
                    bad = list(ptrs)
                    bad[k] += align // 2
                    rc = call(bad)
                    assert rc == -1 and "aligned" in lib.ovc_last_error().decode(), (fmt, act_flag, k, rc)


def test_recipe_config_validity_rules():
    """Recipe.configure's rules (overcooked_mdp.py:236-300) as restated in layout._check_recipe_config; the verdicts
    below are the reference's (tests/test_oracle_live_reference.py checks them live where the reference is present)."""
    orders = [{"ingredients": ["onion", "onion", "onion"]}]
    bad = [
        {"onion_value": 3}, {"tomato_time": 4}, {"onion_value": 3, "tomato_value": 2, "delivery_reward": 9},
        {"onion_value": 3, "tomato_value": 2, "recipe_values": [5], "start_all_orders": orders},
        {"recipe_values": [5], "delivery_reward": 9, "start_all_orders": orders},
        {"onion_time": 3, "tomato_time": 2, "cook_time": 9},
        {"onion_time": 3, "tomato_time": 2, "recipe_times": [5], "start_all_orders": orders},
        {"recipe_times": [5], "cook_time": 9, "start_all_orders": orders},
        {"recipe_values": [5, 6]}, {"recipe_times": [5, 6], "start_all_orders": orders},
    ]
    for kw in bad:
        with pytest.raises(ValueError):
            L.compile_layout("cramped_room", **kw)
    assert L.compile_layout("cramped_room", recipe_values=[5]).deliver_value[12] == 5  # the layout file's one order
    ok = L.compile_layout("cramped_room", recipe_values=[5], recipe_times=[7], start_all_orders=orders)
    assert ok.deliver_value[12] == 5 and ok.cook_time[12] == 7
    ok = L.compile_layout("cramped_room", onion_value=3, tomato_value=2, onion_time=4, tomato_time=5)
    assert ok.base_value[12] == 9 and ok.cook_time[6] == 14  # 3 onions: 3 * 3; 1 onion + 2 tomatoes: 4 + 2 * 5


def test_grid_validity_rules():
    """OvercookedGridworld._assert_valid_grid (overcooked_mdp.py:2064-2115): AssertionError, the reference's messages."""
    from overcooked_ai_b200.mdp import OvercookedGridworld

    ok = ["XXPXX", "O  2O", "X1  X", "XDXSX"]
    OvercookedGridworld.from_grid(ok)
    cases = [
        (["XXPXX", "O  2", "X1  X", "XDXSX"], "Ragged grid"),
        (["XXPXX", "   2O", "X1  X", "XDXSX"], "Left border must not be free"),
        (["XXPXX", "O  2 ", "X1  X", "XDXSX"], "Right border must not be free"),
        (["XX XX", "O  2O", "X1  X", "XDXSX"], "Top border must not be free"),
        (["XXPXX", "O  2O", "X1  X", "XD1SX"], "Bottom border must not be free"),
        (["XXPXX", "O   O", "X   X", "XDXSX"], "No players (digits) in grid"),
        (["XXPXX", "O  3O", "X1  X", "XDXSX"], "Some players were missing"),
        (["XXPXX", "O ?2O", "X1  X", "XDXSX"], "Invalid character in grid"),
        (["XXPXX", "O  2O", "X1  X", "XXXSX"], "'D' must be present at least once"),
        (["XXPXX", "O  2O", "X1  X", "XDXXX"], "'S' must be present at least once"),
        (["XXXXX", "O  2O", "X1  X", "XDXSX"], "'P' must be present at least once"),
        (["XXPXX", "X  2X", "X1  X", "XDXSX"], "'O' or 'T' must be present at least once"),
    ]
    for grid, msg in cases:
        with pytest.raises(AssertionError, match=msg.replace("(", r"\(").replace(")", r"\)")):
            OvercookedGridworld.from_grid(grid)
    with pytest.raises(ValueError):  # valid for the reference, outside this engine: the batched game is the 2-player game
        OvercookedGridworld.from_grid(["XXPXX", "O   O", "X1  X", "XDXSX"])


def test_dense_grid_policy_is_the_same_network_as_the_cnn():
    """selfplay.DenseGridPolicy folds every convolution of RllibShapedCNN into one matrix per layer (library GEMMs on the
    observation kernel's own element order): same function, to float32 round-off, on every grid shape of the layouts."""
    import torch

    from overcooked_ai_b200.selfplay import DenseGridPolicy, RllibShapedCNN

    torch.manual_seed(0)
    for W, H in ((5, 4), (9, 5), (5, 5), (13, 4)):
        cnn = RllibShapedCNN(W, H).eval()
        dense = DenseGridPolicy(cnn, W, H).eval()
        obs = torch.rand(9, W, H, 26)  # [n][x][y][channel], what lossless_state_encoding writes
        with torch.no_grad():
            l1, v1 = cnn(obs.permute(0, 3, 1, 2))
            l2, v2 = dense(obs.reshape(9, -1))
        assert torch.allclose(l1, l2, atol=1e-6) and torch.allclose(v1, v2, atol=1e-6)


def test_dense_grid_policy_padding_keeps_the_function():
    """Width padding (16-byte rows for the library's tensor-core GEMM kernels) adds zero weights only; merged heads."""
    import torch

    from overcooked_ai_b200.selfplay import DenseGridPolicy, RllibShapedCNN

    torch.manual_seed(2)
    cnn = RllibShapedCNN(5, 4).eval()
    plain, padded = DenseGridPolicy(cnn, 5, 4).eval(), DenseGridPolicy(cnn, 5, 4, pad_to=16).eval()
    assert [l.out_features for l in plain.conv_as_linear] == [500, 500, 150] and plain.heads.out_features == 7
    assert [l.out_features for l in padded.conv_as_linear] == [512, 512, 160] and padded.heads.out_features == 16
    obs = torch.rand(11, 520)
    with torch.no_grad():
        (l1, v1), (l2, v2) = plain(obs), padded(obs)
    assert l2.shape == (11, 6) and torch.allclose(l1, l2, atol=1e-6) and torch.allclose(v1, v2, atol=1e-6)


def test_dense_grid_policy_kernel_tables_are_the_policy():
    """first_layer_table / wide_tables / tail_tables (what K7 / K9 / K8 are given) evaluated with plain float matmuls equal
    DenseGridPolicy.forward: the three kernels together are the whole network, nothing is left to a library call."""
    import torch
    import torch.nn.functional as F

    from overcooked_ai_b200.selfplay import DenseGridPolicy, RllibShapedCNN

    torch.manual_seed(4)
    cnn = RllibShapedCNN(5, 4).eval()
    d = DenseGridPolicy(cnn, 5, 4, pad_to=16).eval()
    wt0, b0 = d.first_layer_table()
    w1, b1, w2, b2 = d.wide_tables()
    wf, bf, wh, bh, wo, bo = d.tail_tables()
    assert wt0.shape == (520, 512) and w1.shape == (512, 512) and w2.shape == (160, 512) and wf.shape == (64, 160)
    assert wh.shape == (2, 64, 64) and wo.shape == (8, 64) and all(t.dtype == torch.bfloat16 for t in (wt0, w1, w2, wf, wh, wo))
    obs = (torch.rand(9, 520) < 0.1).float()
    with torch.no_grad():
        want_logits, want_value = d(obs)
        a = F.leaky_relu(obs @ wt0.float() + b0, 0.2)                                   # K7
        z = F.leaky_relu(a @ w1.float().t() + b1, 0.2) @ w2.float().t() + b2               # K9 (pre-activation out)
        a = F.leaky_relu(F.leaky_relu(z, 0.2) @ wf.float().t() + bf, 0.3)                  # K8: activation on load, first dense layer
        for l in range(wh.shape[0]):
            a = F.leaky_relu(a @ wh[l].float().t() + bh[l], 0.3)
        heads = a @ wo.float().t() + bo
    # the tables hold the weights rounded to bf16: agreement to bf16 accuracy of the weights
    assert torch.allclose(heads[:, :6], want_logits, atol=3e-3) and torch.allclose(heads[:, 6], want_value, atol=3e-3)


def test_policy_loads_the_reference_keras_model_weights():
    """RllibShapedCNN.load_keras_weights: weights in the reference PPO model's own (Keras) layouts give the Keras model's
    function — restated here in numpy from ppo_rllib.py:43-79 (Conv2D 5x5 'same', 3x3 'same', 3x3 'valid' with
    tf.nn.leaky_relu = 0.2, Flatten over (x, y, channel), Dense + LeakyReLU() = 0.3, two linear heads) — and so does the
    dense-matrix form the kernels consume."""
    import torch

    from overcooked_ai_b200.selfplay import DenseGridPolicy, RllibShapedCNN

    rng = np.random.RandomState(11)
    W, H, C, NF, HID = 5, 4, 26, 25, 64
    conv = [(rng.normal(size=(5, 5, C, NF)) * 0.1, rng.normal(size=NF) * 0.1), (rng.normal(size=(3, 3, NF, NF)) * 0.1, rng.normal(size=NF) * 0.1),
            (rng.normal(size=(3, 3, NF, NF)) * 0.1, rng.normal(size=NF) * 0.1)]
    flat = (W - 2) * (H - 2) * NF
    dense = [(rng.normal(size=(flat, HID)) * 0.1, rng.normal(size=HID) * 0.1)] + [(rng.normal(size=(HID, HID)) * 0.1, rng.normal(size=HID) * 0.1) for _ in range(2)]
    logits, value = (rng.normal(size=(HID, 6)) * 0.1, rng.normal(size=6) * 0.1), (rng.normal(size=(HID, 1)) * 0.1, rng.normal(size=1) * 0.1)

    def conv2d(x, k, b, same):  # x (n, W, H, cin) channels last, k (kh, kw, cin, cout): Keras Conv2D, stride 1
        kh, kw = k.shape[:2]
        if same:
            x = np.pad(x, ((0, 0), (kh // 2, kh // 2), (kw // 2, kw // 2), (0, 0)))
        wo, ho = x.shape[1] - kh + 1, x.shape[2] - kw + 1
        out = np.zeros((x.shape[0], wo, ho, k.shape[3]))
        for i in range(kh):
            for j in range(kw):
                out += x[:, i:i + wo, j:j + ho, :] @ k[i, j]
        return out + b

    lrelu = lambda z, a: np.where(z > 0, z, a * z)
    obs = (rng.rand(7, W, H, C) < 0.1).astype(np.float64) * rng.randint(1, 4, size=(7, W, H, C))
    x = lrelu(conv2d(obs, *conv[0], True), 0.2)
    x = lrelu(conv2d(x, *conv[1], True), 0.2)
    x = lrelu(conv2d(x, *conv[2], False), 0.2).reshape(7, -1)
    for k, b in dense:
        x = lrelu(x @ k + b, 0.3)
    want_logits, want_value = x @ logits[0] + logits[1], (x @ value[0] + value[1])[:, 0]

    cnn = RllibShapedCNN(W, H).eval().load_keras_weights(conv, dense, logits, value)
    t_obs = torch.from_numpy(obs).float()
    with torch.no_grad():
        l1, v1 = cnn(t_obs.permute(0, 3, 1, 2))
        l2, v2 = DenseGridPolicy(cnn, W, H, pad_to=16).eval()(t_obs.reshape(7, -1))
    for l, v in ((l1, v1), (l2, v2)):
        assert np.allclose(l.numpy(), want_logits, atol=2e-4) and np.allclose(v.numpy(), want_value, atol=2e-4)


def test_fused_kernel_support_by_grid():
    """Which of K7 / K9 / K8 a grid's policy can use (the rest runs as library GEMMs): all three on 5x4, K7 only on 5x5
    (tail input 240 is not a multiple of 32), none on 9x5 (first layer 1136 wide: not a multiple of 64; tail input 528)."""
    import torch

    from overcooked_ai_b200.selfplay import DenseGridPolicy, RllibShapedCNN, fused_kernel_support

    for (W, H), want in (((5, 4), (True, True, True)), ((5, 5), (True, False, False)), ((9, 5), (False, False, False))):
        d = DenseGridPolicy(RllibShapedCNN(W, H), W, H, pad_to=16)
        assert fused_kernel_support(d, W, H) == want, (W, H, fused_kernel_support(d, W, H))


def test_fused_kernel_support_bounds_the_layout_count():
    """K7 takes at most 8 layouts per call (EL_MAX_LAYOUTS): above that fused_kernel_support turns K7 off on every grid it
    would otherwise allow, and leaves K9 and K8 as they are."""
    from types import SimpleNamespace

    from overcooked_ai_b200.selfplay import K7_MAX_LAYOUTS, fused_kernel_support

    lin = lambda i, o: SimpleNamespace(in_features=i, out_features=o)
    net = SimpleNamespace(conv_as_linear=[lin(520, 512), lin(512, 512), lin(512, 160)], dense=[lin(160, 64)] * 3, n_actions=6)
    assert K7_MAX_LAYOUTS == 8
    assert fused_kernel_support(net, 5, 4) == (True, True, True)
    for n_layouts, k7 in ((1, True), (2, True), (8, True), (9, False), (12, False), (255, False)):
        assert fused_kernel_support(net, 5, 4, n_layouts) == (k7, True, True), n_layouts
        assert fused_kernel_support(net, 13, 7, n_layouts)[0] == k7, n_layouts  # the largest grids K7's table fits
        assert not fused_kernel_support(net, 12, 8, n_layouts)[0], n_layouts     # refused by shared memory alone
