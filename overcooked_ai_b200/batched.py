"""BatchedOvercookedEnv — N independent Overcooked environments advanced by one CUDA launch.

The tensor-level API of the engine (SURVEY.md §8b).  State lives in ONE int32 tensor
``state[N, S]`` (record layout in include/ovc_b200.h); ``step`` / ``rollout`` / ``reset`` /
``lossless_state_encoding`` / ``featurize_state`` are thin calls into the C ABI on torch's current
CUDA stream, so they compose with CUDA graphs and user streams.  torch owns every buffer; the
native library allocates nothing.

Semantics follow the reference per environment:
  step     OvercookedEnv.step      (src/overcooked_ai_py/mdp/overcooked_env.py:244-274) on top of
           OvercookedGridworld.get_state_transition (overcooked_mdp.py:1375-1430)
  reset    OvercookedEnv.reset     (overcooked_env.py:288-319), standard start state
  done     OvercookedEnv.is_done   (overcooked_env.py:321-325): timestep >= horizon
Stepping an environment that is already done leaves it untouched and sets EVF_STEPPED_DONE in its
event words (the reference raises AssertionError, overcooked_env.py:255); with ``auto_reset=True``
an environment that reaches the horizon is put back to its start state in the same launch (its
``done`` output is still 1 for that transition), which is what rollout collection wants.
"""
import ctypes

import numpy as np
import torch

from overcooked_ai_b200 import _native
from overcooked_ai_b200 import layout as L

_TORCH_DT = {torch.float32: _native.DT_F32, torch.uint8: _native.DT_U8, torch.int32: _native.DT_I32,
             torch.bfloat16: _native.DT_BF16}


def _as_layouts(layouts, mdp_params):
    if isinstance(layouts, (str, L.CompiledLayout)) or hasattr(layouts, "compiled"):
        layouts = [layouts]
    out = []
    for l in layouts:
        if isinstance(l, str):
            l = L.compile_layout(l, **(mdp_params or {}))
        elif hasattr(l, "compiled"):  # an overcooked_ai_b200.mdp.OvercookedGridworld
            l = l.compiled
        out.append(l)
    return out


class BatchedOvercookedEnv(object):
    def __init__(self, layouts, n_envs, horizon=400, device="cuda", auto_reset=False, state_words=None,
                 io=_native.IO_DEFAULT, env_layout=None, mdp_params=None, pdl=True,
                 random_start_pos=False, rnd_obj_prob_thresh=0.0, seed=0, random_layout=False):
        """
        layouts      layout name / CompiledLayout / OvercookedGridworld, or a list of them (mixed batch)
        n_envs       number of environments on THIS device
        horizon      episode length (OvercookedEnv's ``horizon``); <= 0 means no horizon
        env_layout   optional int array [n_envs] of layout indices; default: contiguous, near-equal
                     segments, one per layout (a warp then sees one layout; SURVEY.md §7)
        io           record I/O strategy of the step kernel (_native.IO_*); 0 = library default
        pdl          launch the step kernel with programmatic dependent launch: back-to-back transitions overlap
                     the next launch's prologue with the current kernel (3.58 -> 3.20 us per launch at 65 536 envs)
        random_start_pos, rnd_obj_prob_thresh, seed
                     start every episode from the reference's randomised start states
                     (get_random_start_state_fn, overcooked_mdp.py:1307-1369) instead of the standard one;
                     drawn on the device with a counter-based generator (see ovc_random_start_t)
        random_layout
                     variable MDP — OvercookedEnv(mdp_generator_fn, num_mdp > 1) whose reset draws a new MDP
                     (overcooked_env.py:288-302): every (auto-)reset redraws the environment's layout uniformly
                     from ``layouts`` (e.g. a pool from layout_generator.generate_layout_pool); ``layout_ids()``
                     gives the current assignment, ``env_layout`` only the initial one
        """
        self._lib = _native.lib()
        if not torch.cuda.is_available():
            raise RuntimeError("BatchedOvercookedEnv needs a CUDA device: this engine has no CPU fallback")
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise ValueError("device must be a CUDA device")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.layouts = _as_layouts(layouts, mdp_params)
        self.n_layouts = len(self.layouts)
        self._longest_cook = max(int(l.cook_time.max()) for l in self.layouts)  # bounds the cook-time-remaining plane
        self.n_envs = int(n_envs)
        self.horizon = int(horizon) if horizon < 2**31 else 0
        self.auto_reset = bool(auto_reset)
        self.io = int(io)
        self.pdl = bool(pdl)  # programmatic dependent launch for back-to-back step() calls / graphs
        tab, starts, S = L.build_tables(self.layouts, state_words)
        assert tab.shape[1] == self._lib.ovc_layout_table_size(), "layout table size mismatch with the native library"
        self.state_words = S
        self._tab_host, self._starts_host = tab, starts
        with torch.cuda.device(self.device):
            self.tables = torch.from_numpy(tab).to(self.device)
            self.start_records = torch.from_numpy(starts).to(self.device)
            if env_layout is None:
                bounds = [self.n_envs * i // self.n_layouts for i in range(self.n_layouts + 1)]
                env_layout = np.zeros(self.n_envs, np.int32)
                for i in range(self.n_layouts):
                    env_layout[bounds[i]:bounds[i + 1]] = i
            env_layout = np.ascontiguousarray(env_layout, dtype=np.int32)
            assert env_layout.shape == (self.n_envs,) and (env_layout >= 0).all() and (env_layout < self.n_layouts).all()
            self.env_layout_host = env_layout
            self.env_layout = torch.from_numpy(env_layout).to(self.device)
            self.state = torch.zeros((self.n_envs, S), dtype=torch.int32, device=self.device)
            self.sparse = torch.zeros(self.n_envs, dtype=torch.int32, device=self.device)
            self.shaped = torch.zeros((self.n_envs, 2), dtype=torch.int32, device=self.device)
            self.done = torch.zeros(self.n_envs, dtype=torch.int32, device=self.device)
            self.events = torch.zeros((self.n_envs, 2), dtype=torch.int32, device=self.device)
        self._rs = None
        self.random_layout = bool(random_layout)
        if random_start_pos or rnd_obj_prob_thresh > 0 or random_layout:
            thr = min(int(float(rnd_obj_prob_thresh) * 4294967296.0), 0xFFFFFFFF)  # 0xFFFFFFFF = always (ovc_rng.cuh)
            self._rs = _native.RandomStart(int(seed) & 0xFFFFFFFFFFFFFFFF, thr, int(bool(random_start_pos)),
                                           int(self.random_layout), 0)
        self._lut = None
        self._greedy = None
        self._segments = None
        self._pot = {}  # gamma -> potential tables; never dropped, so a captured graph's tables stay alive
        with torch.cuda.device(self.device):
            self.reset()

    # ---------------------------------------------------------------------------------------------
    def _flags(self, auto_reset=None):
        return ((_native.F_AUTO_RESET if (self.auto_reset if auto_reset is None else auto_reset) else 0) | (_native.F_PDL if self.pdl else 0)
                | (self.io << _native.F_IO_SHIFT))

    def _rs_ptr(self):
        return ctypes.byref(self._rs) if self._rs is not None else None

    def _stream(self):
        # the C ABI launches on the calling thread's current device: make a mismatch loud instead of a fault
        if torch.cuda.current_device() != self.device.index:
            raise RuntimeError("this environment lives on %s but the current CUDA device is cuda:%d; wrap the call in "
                               "torch.cuda.device(env.device) (one process per GPU sets it once)" % (self.device, torch.cuda.current_device()))
        return torch.cuda.current_stream(self.device).cuda_stream

    def reset(self, mask=None):
        """Put all environments (or those with mask != 0; int32 tensor [N]) back to their layout's
        standard start state (overcooked_mdp.py:1297-1305)."""
        if mask is not None:
            assert mask.dtype == torch.int32 and mask.is_cuda and mask.is_contiguous() and mask.numel() == self.n_envs
        _native.check(self._lib.ovc_reset(
            self.tables.data_ptr(), self.n_layouts, self.start_records.data_ptr(), self.state.data_ptr(),
            self.env_layout.data_ptr(), 0 if mask is None else mask.data_ptr(), self.n_envs, self.state_words,
            self._rs_ptr(), self._stream()))

    def reset_ended(self):
        """Reset every environment whose episode ended with the last ``step(..., auto_reset=False)`` (``self.done``) to
        exactly the record ``step``'s auto-reset would have written: the start record of the record's own layout, or the
        next episode's random start (and, with ``random_layout``, its drawn layout).  ``reset(mask)`` takes the layout from
        the initial assignment ``env_layout``; this reset reads it from the record, as the step kernel does."""
        _native.check(self._lib.ovc_reset(
            self.tables.data_ptr(), self.n_layouts, self.start_records.data_ptr(), self.state.data_ptr(), 0, self.done.data_ptr(),
            self.n_envs, self.state_words, self._rs_ptr(), self._stream()))

    def step(self, actions, out=None, auto_reset=None):
        """One joint transition of every environment.

        actions  int32 CUDA tensor [N, 2], action indices 0..5 (Action.INDEX_TO_ACTION order)
        out      optional (sparse[N], shaped[N,2], done[N], events[N,2]) int32 CUDA tensors to write
        auto_reset  None: the env's own setting; False: finished episodes keep their terminal record (for
                 ``potential_shaping``, which takes phi on it and then resets them)
        returns  (sparse, shaped, done, events); without ``out`` these are buffers owned by the env and
                 overwritten by the next call.  ``sparse`` is the summed delivery reward
                 (what OvercookedEnv.step returns), ``shaped`` is shaped_reward_by_agent,
                 ``events`` holds one bit per EVENT_TYPES entry per agent (layout.EVENT_TYPES).
        """
        assert actions.dtype == torch.int32 and actions.is_cuda and actions.is_contiguous()
        assert actions.numel() == 2 * self.n_envs
        sparse, shaped, done, events = (self.sparse, self.shaped, self.done, self.events) if out is None else out
        if out is not None:
            for o, n in zip(out, (1, 2, 1, 2)):
                assert o.dtype == torch.int32 and o.is_cuda and o.is_contiguous() and o.numel() == n * self.n_envs, \
                    "step(out=...) takes int32 CUDA tensors (sparse[N], shaped[N,2], done[N], events[N,2])"
        _native.check(self._lib.ovc_step(
            self.tables.data_ptr(), self.n_layouts, self.start_records.data_ptr(), self.state.data_ptr(),
            actions.data_ptr(), sparse.data_ptr(), shaped.data_ptr(), done.data_ptr(),
            events.data_ptr(), self.n_envs, self.state_words, self.horizon, self._flags(auto_reset), self._rs_ptr(), self._stream()))
        return sparse, shaped, done, events

    def narrow_ok(self):
        """True if every layout's rewards fit the narrow transfer formats (int16 sparse, int8 shaped)."""
        return all(int(l.deliver_value.max()) * 2 <= 32767 and max(
            int(l.reward_shaping_params[k]) for k in ("PLACEMENT_IN_POT_REW", "DISH_PICKUP_REWARD", "SOUP_PICKUP_REWARD")) <= 127
            for l in self.layouts)

    def n_groups(self):
        """Groups of 32 consecutive environments (one warp each) — the unit of the sparse event stream."""
        return (self.n_envs + 31) // 32

    def alloc_stream_out(self, T, cap, n_chunks=1, pin=False, dense_backup=False):
        """Buffers of the sparse event stream (OVC_F_OUT_STREAM): (masks uint32 as int32 [T, G], values int16 [n_chunks, G, cap],
        dense code words int16 [T, N] or None)."""
        G = self.n_groups()
        mk = (lambda sh, dt: torch.zeros(sh, dtype=dt, pin_memory=True)) if pin else (lambda sh, dt: torch.zeros(sh, dtype=dt, device=self.device))
        return (mk((T, G), torch.int32), mk((n_chunks, G, cap), torch.int16), mk((T, self.n_envs), torch.int16) if dense_backup else None)

    def rollout_stream(self, actions, cap, out=None, dense_backup=False):
        """T transitions in one launch with the result as a sparse event stream (include/ovc_b200.h OVC_F_OUT_STREAM):
        per transition and group of 32 environments one lane mask of the non-zero code words, plus each group's
        non-zero words compacted in (transition, lane) order, at most ``cap`` per group (the masks count the rest).
        actions: int32 / uint8 [T, N, 2] or one-byte joint actions uint8 [T, N].  Returns (masks, values, dense or None);
        expand with ``expand_stream``."""
        act_flag = self._action_flag(actions)
        T = actions.shape[0]
        assert 1 <= cap <= _native.STREAM_CAP_MAX
        if out is None:
            out = self.alloc_stream_out(T, cap, dense_backup=dense_backup)
        masks, values, dense = out
        assert masks.dtype == torch.int32 and tuple(masks.shape) == (T, self.n_groups()) and masks.is_cuda and masks.is_contiguous()
        assert values.dtype == torch.int16 and values.numel() == self.n_groups() * cap and values.is_cuda and values.is_contiguous()
        flags = self._flags() | act_flag | _native.F_OUT_STREAM | (int(cap) << _native.F_STREAM_CAP_SHIFT)
        if flags >= 2**31:  # the C int carries the capacity in its upper half
            flags -= 2**32
        _native.check(self._lib.ovc_rollout(
            self.tables.data_ptr(), self.n_layouts, self.start_records.data_ptr(), self.state.data_ptr(),
            actions.data_ptr(), values.data_ptr(), 0, 0 if dense is None else dense.data_ptr(), masks.data_ptr(),
            self.n_envs, T, self.state_words, self.horizon, flags, self._rs_ptr(), self._stream()))
        return out

    def expand_stream(self, masks, values, chunk=None, sparse=True, shaped=True, done=True, events=False, n_threads=0, out=None):
        """Dense host arrays from a HOST sparse event stream (ovc_expand_stream_host): masks int32 [T, G], values int16
        [n_chunks, G, cap] with ``chunk`` transitions per launch (default: all T in one).  Returns (dict of arrays as
        expand_codes, number of (chunk, group) slices that overflowed their capacity)."""
        assert masks.dtype == torch.int32 and not masks.is_cuda and masks.is_contiguous() and masks.dim() == 2
        assert values.dtype == torch.int16 and not values.is_cuda and values.is_contiguous() and values.dim() == 3
        T, G = masks.shape
        assert G == self.n_groups() and values.shape[1] == G
        chunk = T if chunk is None else int(chunk)
        assert values.shape[0] == -(-T // chunk)
        out, tbl, lay, ptrs = self._dense_host_out(T, out, sparse, shaped, done, events)
        over = ctypes.c_int64(0)
        _native.check(self._lib.ovc_expand_stream_host(
            masks.data_ptr(), values.data_ptr(), T, chunk, values.shape[2], self.n_envs, lay, tbl.ctypes.data, self.n_layouts, *ptrs,
            int(n_threads), ctypes.byref(over)))
        return out, int(over.value)

    def _dense_host_out(self, T, out, sparse, shaped, done, events):
        """What the host expanders take besides the words: the dense arrays (``out``, or new ones for the requested keys), the
        reward table, the layout ids (a pointer; 0 = one table for all) and the four output pointers (0 = not requested)."""
        tbl = np.ascontiguousarray(self.code_reward_table(), dtype=np.int32)
        lay = self.env_layout_host.ctypes.data
        if self.random_layout:
            assert (tbl == tbl[:1]).all(), "random_layout with different reward tables: the codes alone do not name the layout"
            lay = 0
        if out is None:
            N = self.n_envs
            want = (("sparse", sparse, (T, N), torch.int16), ("shaped", shaped, (T, N, 2), torch.int8),
                    ("done", done, (T, N), torch.uint8), ("events", events, (T, N, 2), torch.int32))
            out = {k: torch.empty(shape, dtype=dt) for k, on, shape, dt in want if on}
        ptrs = [out[k].data_ptr() if k in out else 0 for k in ("sparse", "shaped", "done", "events")]
        return out, tbl, lay, ptrs

    def alloc_rollout_out(self, T, narrow=False, pin=False, packed=False, codes=False):
        """Output tensors for rollout(): (sparse[T,N], shaped[T,N,2], done[T,N], events[T,N,2]); int32, or with
        ``narrow`` int16 / int8 / uint8 / int32 (13 bytes per env-step), or with ``packed`` (6 bytes per env-step)
        (sparse int16 [T,N], shaped int8 [T,N,2], None, evcode int16 [T,N]) where evcode carries both agents' 5-bit
        event codes + done (include/ovc_b200.h OVC_F_OUT_PACKED; expand with wire.decode_event_codes), or with
        ``codes`` (2 bytes per env-step) (None, None, None, evcode int16 [T,N]): the same word plus one
        "shaped reward granted" bit per agent, from which rewards follow by table (OVC_F_OUT_CODES; expand_codes)."""
        N = self.n_envs
        mk = (lambda sh, dt: torch.empty(sh, dtype=dt, pin_memory=True)) if pin else (lambda sh, dt: torch.empty(sh, dtype=dt, device=self.device))
        if codes:
            return (None, None, None, mk((T, N), torch.int16))
        if packed:
            return (mk((T, N), torch.int16), mk((T, N, 2), torch.int8), None, mk((T, N), torch.int16))
        dts = (torch.int16, torch.int8, torch.uint8, torch.int32) if narrow else (torch.int32,) * 4
        shapes = ((T, N), (T, N, 2), (T, N), (T, N, 2))
        return tuple(mk(sh, dt) for sh, dt in zip(shapes, dts))

    def _action_flag(self, actions):
        """Checks an action trace (int32 / uint8 CUDA [T, N, 2], or one-byte joint actions uint8 [T, N]) and returns its
        OVC_F_ACT_* flag."""
        assert actions.dtype in (torch.int32, torch.uint8) and actions.is_cuda and actions.is_contiguous() and actions.dim() in (2, 3)
        assert actions.shape[1] == self.n_envs
        if actions.dim() == 2:
            assert actions.dtype == torch.uint8, "one-byte joint actions are uint8 [T, N]"
            return _native.F_ACT_PACKED
        assert actions.shape[2] == 2
        return _native.F_ACT_U8 if actions.dtype == torch.uint8 else 0

    def rollout(self, actions, out=None):
        """T transitions in one launch (state stays on chip between them).

        actions  int32 or uint8 CUDA tensor [T, N, 2], or uint8 [T, N] with both agents' indices in one byte
                 (agent 0 in bits 0-3, agent 1 in bits 4-7; wire.pack_actions)
        out      optional (sparse[T,N], shaped[T,N,2], done[T,N], events[T,N,2]): all int32, or one of the narrower
                 sets of alloc_rollout_out(narrow= / packed= / codes=).
        Equivalent to T calls of step() with the same actions.
        """
        flags = self._flags() | self._action_flag(actions)
        T = actions.shape[0]
        if out is None:
            out = self.alloc_rollout_out(T)
        sparse, shaped, done, events = out
        if sparse is None:  # codes: 2 bytes per env-step
            assert shaped is None and done is None and events.dtype == torch.int16 and events.dim() == 2
            assert tuple(events.shape) == (T, self.n_envs) and events.is_cuda and events.is_contiguous()
            flags |= _native.F_OUT_CODES
            _native.check(self._lib.ovc_rollout(
                self.tables.data_ptr(), self.n_layouts, self.start_records.data_ptr(), self.state.data_ptr(),
                actions.data_ptr(), 0, 0, 0, events.data_ptr(), self.n_envs, T, self.state_words, self.horizon, flags,
                self._rs_ptr(), self._stream()))
            return out
        if done is None:  # packed: 6 bytes per env-step
            assert sparse.dtype == torch.int16 and shaped.dtype == torch.int8 and events.dtype == torch.int16 and events.dim() == 2
            assert self.narrow_ok(), "rewards of these layouts do not fit the narrow formats"
            flags |= _native.F_OUT_PACKED
        elif sparse.dtype == torch.int16:
            assert shaped.dtype == torch.int8 and done.dtype == torch.uint8 and events.dtype == torch.int32
            assert self.narrow_ok(), "rewards of these layouts do not fit the narrow formats"
            flags |= _native.F_OUT_NARROW
        else:
            assert sparse.dtype == shaped.dtype == done.dtype == events.dtype == torch.int32
        _native.check(self._lib.ovc_rollout(
            self.tables.data_ptr(), self.n_layouts, self.start_records.data_ptr(), self.state.data_ptr(),
            actions.data_ptr(), sparse.data_ptr(), shaped.data_ptr(), 0 if done is None else done.data_ptr(), events.data_ptr(),
            self.n_envs, T, self.state_words, self.horizon, flags, self._rs_ptr(), self._stream()))
        return out

    def code_reward_table(self):
        """int32 numpy [n_layouts, 2, 32]: delivery reward and shaped reward of each event code (OVC_F_OUT_CODES)."""
        from overcooked_ai_b200 import wire

        return wire.code_reward_table(self.layouts)

    def expand_codes(self, evcode, sparse=True, shaped=True, done=True, events=False, n_threads=0, out=None):
        """Dense host arrays from a HOST int16 [T, N] tensor of OVC_F_OUT_CODES words, on the host cores
        (ovc_expand_codes_host): dict with the requested int16 sparse [T,N], int8 shaped [T,N,2], uint8 done [T,N],
        int32 events [T,N,2].  With ``random_layout`` every layout of the pool must share one reward table."""
        assert evcode.dtype == torch.int16 and not evcode.is_cuda and evcode.is_contiguous() and evcode.dim() == 2
        T, N = evcode.shape
        assert N == self.n_envs
        out, tbl, lay, ptrs = self._dense_host_out(T, out, sparse, shaped, done, events)
        _native.check(self._lib.ovc_expand_codes_host(evcode.data_ptr(), T, N, lay, tbl.ctypes.data, self.n_layouts, *ptrs, int(n_threads)))
        return out

    # ---------------------------------------------------------------------------------------------
    def segments(self):
        """[(begin, end, layout index)] maximal runs of equal layout in env order."""
        if self._segments is None:
            el = self.env_layout_host
            cuts = [0] + (np.nonzero(np.diff(el))[0] + 1).tolist() + [self.n_envs]
            self._segments = [(cuts[i], cuts[i + 1], int(el[cuts[i]])) for i in range(len(cuts) - 1) if cuts[i] < cuts[i + 1]]
        return self._segments

    def layout_ids(self):
        """int32 [N]: the layout each environment is on NOW (the id lives in word 3 of its record)."""
        return (self.state[:, 3] & 0xFF).to(torch.int32)

    def _layout_ids_host(self):
        return self.layout_ids().cpu().numpy() if self.random_layout else self.env_layout_host

    def obs_shape(self, layout_index=0):
        l = self.layouts[layout_index]
        return (l.width, l.height, 26)

    def lossless_state_encoding(self, out=None, dtype=torch.float32, view_swap=None, states=None):
        """lossless_state_encoding (overcooked_mdp.py:2385-2561) of every environment, both players:
        tensor [N, 2, W, H, 26] (index order [x][y][channel], as the reference) when all layouts share
        one grid shape, else a list of such tensors, one per layout segment.  dtype float32 (what the
        reference's RLlib consumer casts to), bfloat16, uint8 or int32.  ``view_swap`` (int32 CUDA tensor [N]):
        where non-zero, ``out[env, 0]`` is player 1's view (primary-agent-first order of the gym wrapper).
        ``states``: encode these records (int32 CUDA tensor [M, S], e.g. gathered from a ``selfplay.SampleBatch``)
        instead of ``self.state``; the result is then [M, 2, W, H, 26] and every layout must share one grid shape.
        uint8 holds every value reachable play produces when no cook time exceeds 255 (the cook-time-remaining plane is
        the only one above 3), and is refused (ValueError) for a batch with a longer cook time.  A hand-built over-cooked
        soup (tick > cook time) has a negative cook time remaining (``MDP:2498-2513``), which uint8 cannot hold: its
        plane value is stored modulo 256."""
        out_dtypes = {o.dtype for o in (out if isinstance(out, (list, tuple)) else [out]) if o is not None}
        if torch.uint8 in out_dtypes or (out is None and dtype == torch.uint8):
            if self._longest_cook > 255:
                raise ValueError("lossless_state_encoding: a cook time of %d does not fit uint8 (at most 255); use int32, "
                                 "float32 or bfloat16" % self._longest_cook)
        rows = self.n_envs if states is None else states.shape[0]
        if states is not None:
            assert states.dtype == torch.int32 and states.is_cuda and states.is_contiguous() and states.dim() == 2 and \
                states.shape[1] == self.state_words, "states: int32 CUDA records [M, %d]" % self.state_words
        if view_swap is not None:
            assert view_swap.dtype == torch.int32 and view_swap.is_cuda and view_swap.is_contiguous() and view_swap.numel() == rows
        shapes = {(l.width, l.height) for l in self.layouts}
        if len(shapes) == 1:
            runs = [(0, rows, 0)]
        else:
            assert states is None, "states= needs layouts of one grid shape"
            assert not self.random_layout, "random_layout needs layouts of one grid shape (pad them, LayoutGenerator does)"
            runs = self.segments()
        outs = []
        for k, (b, e, li) in enumerate(runs):
            W, H = self.layouts[li].width, self.layouts[li].height
            o = out[k] if isinstance(out, (list, tuple)) else out
            if o is None:
                o = torch.empty((e - b, 2, W, H, 26), dtype=dtype, device=self.device)
            assert o.is_cuda and o.is_contiguous() and o.numel() == (e - b) * 2 * W * H * 26
            assert o.dtype in _TORCH_DT, "lossless_state_encoding writes float32, bfloat16, uint8 or int32, not %s" % o.dtype
            _native.check(self._lib.ovc_encode_lossless(
                self.tables.data_ptr(), self.n_layouts, (self.state if states is None else states).data_ptr() + 4 * self.state_words * b,
                0 if view_swap is None else view_swap.data_ptr() + 4 * b, o.data_ptr(),
                _TORCH_DT[o.dtype], e - b, self.state_words, W, H, self.horizon if self.horizon > 0 else 2**31 - 1,
                self._stream()))
            outs.append(o)
        return outs[0] if len(shapes) == 1 else outs

    def _records(self, states):
        """(records, count): ``self.state`` or the int32 CUDA records ``states`` [M, S] (e.g. gathered from a sample batch)."""
        if states is None:
            return self.state, self.n_envs
        assert states.dtype == torch.int32 and states.is_cuda and states.is_contiguous() and states.dim() == 2 and \
            states.shape[1] == self.state_words, "states: int32 CUDA records [M, %d]" % self.state_words
        return states, states.shape[0]

    def encoded_linear(self, wt, bias, out=None, neg_slope=0.2, view_swap=None, states=None):
        """First policy layer on ``lossless_state_encoding`` without the observation tensor (kernel K7, ovc_encode_linear):
        ``out[2 env + view] = leaky_relu(obs[env, view].flatten() @ wt + bias, neg_slope)`` as bfloat16 ``[2N, n_out]``.
        ``wt``: bfloat16 CUDA tensor ``[W*H*26, n_out]`` (the layer's matrix TRANSPOSED, rows in the observation's own
        element order ``[x][y][plane]`` — for a convolution, the matrix ``selfplay.DenseGridPolicy`` builds), ``bias``
        float32 ``[n_out]``, ``n_out`` a multiple of 64.  All environments must share one grid shape.  ``states``: these
        records (int32 CUDA [M, S]) instead of ``self.state``; N is then M."""
        assert len({(l.width, l.height) for l in self.layouts}) == 1, "one grid shape per call (group envs by layout)"
        W, H = self.layouts[0].width, self.layouts[0].height
        recs, n = self._records(states)
        assert wt.is_cuda and wt.dtype == torch.bfloat16 and wt.is_contiguous() and wt.shape[0] == W * H * 26, wt.shape
        n_out = wt.shape[1]
        assert bias.is_cuda and bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == n_out
        if view_swap is not None:
            assert view_swap.dtype == torch.int32 and view_swap.is_cuda and view_swap.is_contiguous() and view_swap.numel() == n
        if out is None:
            out = torch.empty((2 * n, n_out), dtype=torch.bfloat16, device=self.device)
        assert out.is_cuda and out.dtype == torch.bfloat16 and out.is_contiguous() and out.numel() == 2 * n * n_out
        _native.check(self._lib.ovc_encode_linear(
            self.tables.data_ptr(), self.n_layouts, recs.data_ptr(), 0 if view_swap is None else view_swap.data_ptr(),
            wt.data_ptr(), bias.data_ptr(), out.data_ptr(), n, self.state_words, W, H,
            self.horizon if self.horizon > 0 else 2**31 - 1, n_out, float(neg_slope), self._stream()))
        return out

    def encoded_linear_view(self, wt, bias, seat, swap=None, out=None, neg_slope=0.2, states=None):
        """``encoded_linear`` for one view per environment (ovc_encode_linear_view): ``out[e]`` (bfloat16 ``[N, n_out]``) is
        the view of player ``seat ^ (swap[e] != 0)``, bit for bit the row ``encoded_linear`` writes for that view.  ``swap``:
        int32 CUDA tensor [N] or None.  ``states``: as in ``encoded_linear``."""
        assert len({(l.width, l.height) for l in self.layouts}) == 1, "one grid shape per call (group envs by layout)"
        W, H = self.layouts[0].width, self.layouts[0].height
        recs, n = self._records(states)
        assert wt.is_cuda and wt.dtype == torch.bfloat16 and wt.is_contiguous() and wt.shape[0] == W * H * 26, wt.shape
        n_out = wt.shape[1]
        assert bias.is_cuda and bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == n_out
        if swap is not None:
            assert swap.dtype == torch.int32 and swap.is_cuda and swap.is_contiguous() and swap.numel() == n
        if out is None:
            out = torch.empty((n, n_out), dtype=torch.bfloat16, device=self.device)
        assert out.is_cuda and out.dtype == torch.bfloat16 and out.is_contiguous() and out.numel() == n * n_out
        _native.check(self._lib.ovc_encode_linear_view(
            self.tables.data_ptr(), self.n_layouts, recs.data_ptr(), 0 if swap is None else swap.data_ptr(), int(seat),
            wt.data_ptr(), bias.data_ptr(), out.data_ptr(), n, self.state_words, W, H,
            self.horizon if self.horizon > 0 else 2**31 - 1, n_out, float(neg_slope), self._stream()))
        return out

    def encoded_linear_wgrad(self, states, dz, dwt, seat=None, swap=None):
        """The weight gradient of ``encoded_linear``'s layer from the records (kernel K12, ovc_encode_linear_wgrad):
        ``dwt[f] += sum over rows r of enc(r)[f] * dz[r]``, with ``dwt`` float32 ``[W*H*26, n_out]`` in ``wt``'s layout and
        ``dz`` float32 ``[rows, n_out]`` the gradient at the layer's pre-activation.  ``states`` int32 CUDA records [M, S].
        ``seat`` None: both views, rows ``2 m + v`` (``encoded_linear``'s rows); 0 / 1: one view, row m is player
        ``seat ^ (swap[m] != 0)`` (``encoded_linear_view``'s rows).  Summation order is unspecified.  Returns ``dwt``."""
        assert len({(l.width, l.height) for l in self.layouts}) == 1, "one grid shape per call (group envs by layout)"
        W, H = self.layouts[0].width, self.layouts[0].height
        recs, n = self._records(states)
        rows = n if seat is not None else 2 * n
        assert dwt.is_cuda and dwt.dtype == torch.float32 and dwt.is_contiguous() and dwt.dim() == 2 and dwt.shape[0] == W * H * 26, dwt.shape
        n_out = dwt.shape[1]
        assert dz.is_cuda and dz.dtype == torch.float32 and dz.is_contiguous() and dz.dim() == 2 and dz.shape[1] == n_out and \
            dz.shape[0] >= rows, (dz.shape, rows)
        assert swap is None or seat is not None, "swap goes with a seat (one view)"
        if swap is not None:
            assert swap.dtype == torch.int32 and swap.is_cuda and swap.is_contiguous() and swap.numel() == n
        if n == 0:  # nothing to add (an empty tensor's data pointer is null)
            return dwt
        _native.check(self._lib.ovc_encode_linear_wgrad(
            self.tables.data_ptr(), self.n_layouts, recs.data_ptr(), 0 if swap is None else swap.data_ptr(),
            -1 if seat is None else int(seat), dz.data_ptr(), dwt.data_ptr(), n, self.state_words, W, H,
            self.horizon if self.horizon > 0 else 2**31 - 1, n_out, self._stream()))
        return dwt

    def sample_actions_view(self, scores, counter, seat, swap=None, seed=0, out=None, logp_out=None):
        """``sample_actions`` for one agent per environment (ovc_sample_actions_view): ``scores`` float32 ``[N, ld]`` (row e:
        the agent at player ``p = seat ^ (swap[e] != 0)``) is drawn with the Philox counter of joint row ``2 e + p`` into
        ``out[e, p]`` (int32 [N, 2]; the other seat is left alone).  ``logp_out`` float32 [N] optional.  Returns ``out``."""
        assert scores.is_cuda and scores.dtype == torch.float32 and scores.dim() == 2 and scores.stride(1) == 1 and scores.shape[0] == self.n_envs
        assert counter.is_cuda and counter.dtype == torch.int64 and counter.numel() == 2 and counter.is_contiguous()
        if swap is not None:
            assert swap.dtype == torch.int32 and swap.is_cuda and swap.is_contiguous() and swap.numel() == self.n_envs
        if out is None:
            out = torch.zeros((self.n_envs, 2), dtype=torch.int32, device=self.device)
        assert out.is_cuda and out.dtype == torch.int32 and out.is_contiguous() and out.numel() == 2 * self.n_envs
        if logp_out is not None:
            assert logp_out.is_cuda and logp_out.dtype == torch.float32 and logp_out.is_contiguous() and logp_out.numel() == self.n_envs
        _native.check(self._lib.ovc_sample_actions_view(
            scores.data_ptr(), scores.stride(0), 6, self.n_envs, int(seed) & (2**64 - 1), counter.data_ptr(),
            0 if swap is None else swap.data_ptr(), int(seat), out.data_ptr(), 0 if logp_out is None else logp_out.data_ptr(),
            self._stream()))
        return out

    def encoded_linear_rows(self, wt, bias, seat, swap, rows, rng, out, neg_slope=0.2):
        """``encoded_linear_view`` on the rows map (ovc_encode_linear_rows): ``out[r]`` (bfloat16 ``[N, n_out]``) for the
        compact rows ``r`` in ``[rng[0], rng[1])`` only, the row ``encoded_linear_view`` writes for environment ``rows[r]``.
        ``rows`` int32 CUDA [N] (e.g. ``group_members``' order), ``rng`` two int32 in device memory (e.g. ``offsets[k:k + 2]``)."""
        assert len({(l.width, l.height) for l in self.layouts}) == 1, "one grid shape per call (group envs by layout)"
        W, H = self.layouts[0].width, self.layouts[0].height
        assert wt.is_cuda and wt.dtype == torch.bfloat16 and wt.is_contiguous() and wt.shape[0] == W * H * 26, wt.shape
        n_out = wt.shape[1]
        assert bias.is_cuda and bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == n_out
        for t, n in ((swap, self.n_envs), (rows, self.n_envs), (rng, 2)):
            assert t is None or (t.dtype == torch.int32 and t.is_cuda and t.is_contiguous() and t.numel() == n)
        assert out.is_cuda and out.dtype == torch.bfloat16 and out.is_contiguous() and out.numel() == self.n_envs * n_out
        _native.check(self._lib.ovc_encode_linear_rows(
            self.tables.data_ptr(), self.n_layouts, self.state.data_ptr(), 0 if swap is None else swap.data_ptr(), int(seat),
            rows.data_ptr(), rng.data_ptr(), wt.data_ptr(), bias.data_ptr(), out.data_ptr(), self.n_envs, self.state_words, W, H,
            self.horizon if self.horizon > 0 else 2**31 - 1, n_out, float(neg_slope), self._stream()))
        return out

    def sample_actions_rows(self, scores, counter, seat, swap, rows, rng, seed=0, out=None, logp_out=None):
        """``sample_actions_view`` on the rows map (ovc_sample_actions_rows): ``scores`` float32 ``[N, ld]`` row r (for r in
        ``[rng[0], rng[1])``) is environment ``rows[r]``'s agent, drawn with the Philox counter of its joint row into
        ``out`` (int32 [N, 2]); ``logp_out[r]`` optional.  The counter advances by one whatever the range holds."""
        assert scores.is_cuda and scores.dtype == torch.float32 and scores.dim() == 2 and scores.stride(1) == 1 and scores.shape[0] == self.n_envs
        assert counter.is_cuda and counter.dtype == torch.int64 and counter.numel() == 2 and counter.is_contiguous()
        for t, n in ((swap, self.n_envs), (rows, self.n_envs), (rng, 2)):
            assert t is None or (t.dtype == torch.int32 and t.is_cuda and t.is_contiguous() and t.numel() == n)
        assert out.is_cuda and out.dtype == torch.int32 and out.is_contiguous() and out.numel() == 2 * self.n_envs
        if logp_out is not None:
            assert logp_out.is_cuda and logp_out.dtype == torch.float32 and logp_out.is_contiguous() and logp_out.numel() == self.n_envs
        _native.check(self._lib.ovc_sample_actions_rows(
            scores.data_ptr(), scores.stride(0), 6, self.n_envs, int(seed) & (2**64 - 1), counter.data_ptr(),
            0 if swap is None else swap.data_ptr(), int(seat), rows.data_ptr(), rng.data_ptr(), out.data_ptr(),
            0 if logp_out is None else logp_out.data_ptr(), self._stream()))
        return out

    def learner_rows(self, partner_seat, lst, first, jrow, rng):
        """A self-play mixture's learner rows (ovc_learner_rows, one CTA on the device): from ``partner_seat`` int32 [N]
        (-1: self-play, else the partner's player) writes ``lst`` int32 [N] (``e << 2 | mask``, bit v of the mask: the learner
        plays view v), ``first`` int32 [N] (the compact row of e's first view), ``jrow`` int32 [2N] (compact row -> joint row)
        and ``rng`` int32 [2] = (0, the row count)."""
        for t, n in ((partner_seat, self.n_envs), (lst, self.n_envs), (first, self.n_envs), (jrow, 2 * self.n_envs), (rng, 2)):
            assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n
        _native.check(self._lib.ovc_learner_rows(partner_seat.data_ptr(), self.n_envs, lst.data_ptr(), first.data_ptr(), jrow.data_ptr(),
                                                 rng.data_ptr(), self._stream()))

    def encoded_linear_masked(self, wt, bias, lst, first, out, neg_slope=0.2):
        """``encoded_linear`` on the views of a list (ovc_encode_linear_masked): entry r of ``lst`` (int32, ``e << 2 | mask``)
        writes the views of its mask to rows ``first[r], first[r] + 1, ...`` of ``out`` (bfloat16 ``[rows, n_out]``), each bit
        for bit row ``2 e + v`` of ``encoded_linear``; the object part is computed once per entry."""
        assert len({(l.width, l.height) for l in self.layouts}) == 1, "one grid shape per call (group envs by layout)"
        W, H = self.layouts[0].width, self.layouts[0].height
        assert wt.is_cuda and wt.dtype == torch.bfloat16 and wt.is_contiguous() and wt.shape[0] == W * H * 26, wt.shape
        n_out = wt.shape[1]
        assert bias.is_cuda and bias.dtype == torch.float32 and bias.is_contiguous() and bias.numel() == n_out
        for t in (lst, first):
            assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == lst.numel()
        assert out.is_cuda and out.dtype == torch.bfloat16 and out.is_contiguous() and out.shape[-1] == n_out
        _native.check(self._lib.ovc_encode_linear_masked(
            self.tables.data_ptr(), self.n_layouts, self.state.data_ptr(), lst.data_ptr(), first.data_ptr(), wt.data_ptr(),
            bias.data_ptr(), out.data_ptr(), lst.numel(), self.state_words, W, H, self.horizon if self.horizon > 0 else 2**31 - 1,
            n_out, float(neg_slope), self._stream()))
        return out

    def group_members(self, member, n_members, order, offsets):
        """The environments grouped by population member (ovc_group_members, a stable counting sort on the device):
        ``member`` int32 [N] with values in [0, n_members); writes ``order`` int32 [N] (environment indices by member,
        ascending within a member) and ``offsets`` int32 [n_members + 1] (member k's environments are
        ``order[offsets[k]:offsets[k + 1]]``)."""
        assert 1 <= n_members <= 64
        for t, n in ((member, self.n_envs), (order, self.n_envs), (offsets, n_members + 1)):
            assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n
        _native.check(self._lib.ovc_group_members(member.data_ptr(), int(n_members), self.n_envs, order.data_ptr(), offsets.data_ptr(),
                                                  self._stream()))
        return order, offsets

    def assign_members(self, member, n_members, thresholds=None, counter=None, seed=0, done=None, records=None):
        """The per-episode population draw (ovc_assign_members): for every environment whose episode ended with the last
        ``step`` (``done`` int32 [N], e.g. ``self.done``; None = every environment), first the ending episode's member into
        ``records.partner_member`` (an ``EpisodeRecords`` built with ``members=True``, before ``record_transition`` writes
        the episode to the same slot), then, with ``thresholds`` (int64 CUDA [n_members - 1], ``member_thresholds``), a new
        member drawn from them.  ``counter`` as ``partner_actions``'."""
        assert member.is_cuda and member.dtype == torch.int32 and member.is_contiguous() and member.numel() == self.n_envs
        if thresholds is not None:
            assert thresholds.is_cuda and thresholds.dtype == torch.int64 and thresholds.is_contiguous() and thresholds.numel() >= n_members - 1
            assert counter.is_cuda and counter.dtype == torch.int64 and counter.numel() == 2 and counter.is_contiguous()
        if done is not None:
            assert done.is_cuda and done.dtype == torch.int32 and done.is_contiguous() and done.numel() == self.n_envs
        rec = None
        if records is not None:
            assert records.env is self and records.partner_member is not None, "records built with members=True"
            rec = records
        ptr = lambda t: 0 if t is None else t.data_ptr()
        _native.check(self._lib.ovc_assign_members(
            ptr(done), ptr(thresholds), int(n_members), self.n_envs, int(seed) & (2**64 - 1), ptr(counter), member.data_ptr(),
            0 if rec is None or rec.capacity == 0 else rec.partner_member.data_ptr(), 0 if rec is None else rec.count.data_ptr(),
            0 if rec is None else rec.capacity, self._stream()))
        return member

    def group_pairs(self, pair, n_members, lst, first, jrow, entry_offsets, row_offsets):
        """Population play's compact layout (ovc_group_pairs, one CTA on the device): from ``pair`` int32 [N, 2] (values in
        [0, n_members)) writes ``lst`` int32 [2N] (entries ``e << 2 | mask`` grouped by member, ascending in e: mask 3 for a
        self-play pair, 1 / 2 for view 0 / 1 of a cross pair), ``first`` int32 [2N] (each entry's first compact row), ``jrow``
        int32 [2N] (compact row -> joint row ``2 e + v``), ``entry_offsets`` and ``row_offsets`` int32 [n_members + 1]."""
        assert 1 <= n_members <= 64
        assert pair.is_cuda and pair.dtype == torch.int32 and pair.is_contiguous() and pair.shape == (self.n_envs, 2)
        for t, n in ((lst, 2 * self.n_envs), (first, 2 * self.n_envs), (jrow, 2 * self.n_envs), (entry_offsets, n_members + 1),
                     (row_offsets, n_members + 1)):
            assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n
        _native.check(self._lib.ovc_group_pairs(pair.data_ptr(), int(n_members), self.n_envs, lst.data_ptr(), first.data_ptr(),
                                                jrow.data_ptr(), entry_offsets.data_ptr(), row_offsets.data_ptr(), self._stream()))

    def assign_pairs(self, pair, n_members, thresholds=None, counter=None, seed=0, done=None, records=None):
        """``assign_members`` for population play's ordered pairs (ovc_assign_pairs): for every environment whose episode
        ended (``done`` int32 [N]; None = every environment), the ending pair into ``records.pair`` (an ``EpisodeRecords``
        built with ``pairs=True``), then, with ``thresholds`` (int64 CUDA [n_members^2 - 1], ``member_thresholds`` of the
        row-major flattened pair weights), a new pair ``(p // n_members, p % n_members)`` into ``pair`` int32 [N, 2]."""
        assert pair.is_cuda and pair.dtype == torch.int32 and pair.is_contiguous() and pair.shape == (self.n_envs, 2)
        if thresholds is not None:
            assert thresholds.is_cuda and thresholds.dtype == torch.int64 and thresholds.is_contiguous()
            assert thresholds.numel() >= n_members * n_members - 1
            assert counter.is_cuda and counter.dtype == torch.int64 and counter.numel() == 2 and counter.is_contiguous()
        if done is not None:
            assert done.is_cuda and done.dtype == torch.int32 and done.is_contiguous() and done.numel() == self.n_envs
        if records is not None:
            assert records.env is self and records.pair is not None, "records built with pairs=True"
        ptr = lambda t: 0 if t is None else t.data_ptr()
        _native.check(self._lib.ovc_assign_pairs(
            ptr(done), ptr(thresholds), int(n_members), self.n_envs, int(seed) & (2**64 - 1), ptr(counter), pair.data_ptr(),
            0 if records is None or records.capacity == 0 else records.pair.data_ptr(), 0 if records is None else records.count.data_ptr(),
            0 if records is None else records.capacity, self._stream()))
        return pair

    def sample_actions(self, scores, counter, seed=0, out=None, logp_out=None):
        """Joint actions drawn from the policy's logits (ovc_sample_actions: Gumbel-max on Philox draws, one kernel).
        ``scores`` float32 ``[2N, ld]`` (rows ordered [env][agent], the first 6 columns are the logits), ``counter`` an
        int64 CUDA tensor of 2 zeros that the kernel advances (one step per call; graph-replay safe).  Returns int32 [N, 2].
        ``logp_out`` (float32 [2N]): also the log-probability of each drawn action (ovc_sample_actions_logp)."""
        assert scores.is_cuda and scores.dtype == torch.float32 and scores.dim() == 2 and scores.stride(1) == 1 and scores.shape[0] == 2 * self.n_envs
        assert counter.is_cuda and counter.dtype == torch.int64 and counter.numel() == 2 and counter.is_contiguous()
        if out is None:
            out = torch.empty((self.n_envs, 2), dtype=torch.int32, device=self.device)
        assert out.is_cuda and out.dtype == torch.int32 and out.is_contiguous() and out.numel() == 2 * self.n_envs
        if logp_out is None:
            _native.check(self._lib.ovc_sample_actions(scores.data_ptr(), scores.stride(0), 6, 2 * self.n_envs, int(seed) & (2**64 - 1),
                                                       counter.data_ptr(), out.data_ptr(), self._stream()))
            return out
        assert logp_out.is_cuda and logp_out.dtype == torch.float32 and logp_out.is_contiguous() and logp_out.numel() == 2 * self.n_envs
        _native.check(self._lib.ovc_sample_actions_logp(scores.data_ptr(), scores.stride(0), 6, 2 * self.n_envs, int(seed) & (2**64 - 1),
                                                        counter.data_ptr(), out.data_ptr(), logp_out.data_ptr(), self._stream()))
        return out

    def accumulate_returns(self, ret_sparse, ret_mixed, factor=1.0):
        """``ret_sparse += sparse`` (int64 [N]) and ``ret_mixed += sparse + factor * (shaped[:, 0] + shaped[:, 1])`` (float32 [N])
        from the last ``step``'s outputs, in one kernel (ovc_accumulate_returns; rllib.py:328-329)."""
        for t, dt in ((ret_sparse, torch.int64), (ret_mixed, torch.float32)):
            assert t is None or (t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == self.n_envs)
        _native.check(self._lib.ovc_accumulate_returns(self.sparse.data_ptr(), self.shaped.data_ptr(), float(factor), self.n_envs,
                                                       0 if ret_sparse is None else ret_sparse.data_ptr(),
                                                       0 if ret_mixed is None else ret_mixed.data_ptr(), self._stream()))

    def record_transition(self, factor, rewards=None, dones=None, ret_sparse=None, ret_mixed=None, stats=None, records=None,
                          partner_seat=None, dense=None):
        """What a sample batch keeps of the last ``step`` (ovc_record_transition, one kernel): ``rewards`` float32 [N, 2] =
        sparse + factor * shaped[:, i] per agent (rllib.py:328-329), ``dones`` uint8 [N], and the running returns as
        ``accumulate_returns`` keeps them; each output optional.  ``factor``: float32 CUDA scalar tensor, read by the
        kernel (a captured graph follows its current value).
        ``stats`` (an ``EpisodeStats``) with ``records`` (an ``EpisodeRecords``): in the same kernel
        (ovc_record_transition_stats), fold the step into the running episode statistics and write every episode that
        ended with it into ``records``; ``partner_seat`` (int32 [N], nullable): the partner's seat each episode was played
        with, -1 = self-play.
        ``dense`` (float32 [N], ``potential_shaping``'s output): both agents' reward is ``sparse + factor * dense`` instead
        (use_phi; ovc_record_transition_dense); the shaped rewards still go into the statistics."""
        self._record(self.sparse, self.shaped, self.done, self.events, factor, rewards, dones, ret_sparse, ret_mixed, stats, records,
                     partner_seat, dense=dense)

    def record_transition_view(self, factor, seat, swap, rewards, dones=None, ret_sparse=None, ret_mixed=None, stats=None, records=None,
                               partner_seat=None, dense=None):
        """``record_transition`` for ONE agent per environment (ovc_record_transition_view): ``rewards`` float32 [N] is the
        reward of the agent at player ``seat ^ (swap[e] != 0)`` (``swap`` int32 CUDA [N] or None), bit for bit the entry
        ``record_transition`` writes for that player; everything else as ``record_transition``.  With ``dense`` both agents'
        rewards are equal, so the one-view form of ovc_record_transition_dense needs no seat."""
        if swap is not None:
            assert swap.dtype == torch.int32 and swap.is_cuda and swap.is_contiguous() and swap.numel() == self.n_envs
        self._record(self.sparse, self.shaped, self.done, self.events, factor, rewards, dones, ret_sparse, ret_mixed, stats, records,
                     partner_seat, view=(int(seat), swap), dense=dense)

    def _record(self, sparse, shaped, done, events, factor, rewards=None, dones=None, ret_sparse=None, ret_mixed=None, stats=None,
                records=None, partner_seat=None, view=None, dense=None):
        assert factor.is_cuda and factor.dtype == torch.float32 and factor.numel() == 1
        assert dense is None or (dense.is_cuda and dense.dtype == torch.float32 and dense.is_contiguous() and dense.numel() == self.n_envs)
        for t, dt, n in ((rewards, torch.float32, 1 if view else 2), (dones, torch.uint8, 1), (ret_sparse, torch.int64, 1),
                         (ret_mixed, torch.float32, 1)):
            assert t is None or (t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == n * self.n_envs)
        ptr = lambda t: 0 if t is None else t.data_ptr()
        d = None
        if stats is None:
            assert records is None and partner_seat is None, "records and partner_seat go with stats"
        else:
            assert stats.env is self and records is not None and records.env is self, "stats and records of this environment"
            for t, n in ((sparse, 1), (shaped, 2), (done, 1), (events, 2), (partner_seat, 1)):
                assert t is None or (t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n * self.n_envs)
            d = _native.EpisodeStatsDesc()
            d.layouts, d.state, d.events, d.partner_seat = self.tables.data_ptr(), self.state.data_ptr(), events.data_ptr(), ptr(partner_seat)
            d.event_counts, d.sparse_by_agent = stats.event_counts.data_ptr(), stats.cumulative_sparse_rewards_by_agent.data_ptr()
            d.shaped_by_agent, d.reward_by_agent = stats.cumulative_shaped_rewards_by_agent.data_ptr(), stats.ep_reward_by_agent.data_ptr()
            d.ep_length, d.layout_id = stats.ep_length.data_ptr(), stats.layout_id.data_ptr()
            d.count, d.dropped, d.capacity, d.state_words = records.count.data_ptr(), records.dropped.data_ptr(), records.capacity, self.state_words
            if records.capacity:
                d.rec_length, d.rec_layout, d.rec_partner_seat = records.length.data_ptr(), records.layout.data_ptr(), records.partner_seat.data_ptr()
                d.rec_sparse_by_agent, d.rec_shaped_by_agent = records.sparse_r_by_agent.data_ptr(), records.shaped_r_by_agent.data_ptr()
                d.rec_event_counts, d.rec_reward_by_agent = records.game_stats.data_ptr(), records.reward_by_agent.data_ptr()
        args = (sparse.data_ptr(), shaped.data_ptr(), done.data_ptr(), factor.data_ptr(), self.n_envs)
        outs = (ptr(rewards), ptr(dones), ptr(ret_sparse), ptr(ret_mixed))
        if dense is not None:
            _native.check(self._lib.ovc_record_transition_dense(sparse.data_ptr(), shaped.data_ptr(), dense.data_ptr(), done.data_ptr(),
                                                                factor.data_ptr(), self.n_envs, int(view is not None), *outs,
                                                                None if d is None else ctypes.byref(d), self._stream()))
        elif view is not None:
            seat, swap = view
            _native.check(self._lib.ovc_record_transition_view(*args, ptr(swap), seat, *outs, None if d is None else ctypes.byref(d),
                                                               self._stream()))
        elif d is None:
            _native.check(self._lib.ovc_record_transition(*args, *outs, self._stream()))
        else:
            _native.check(self._lib.ovc_record_transition_stats(*args, *outs, ctypes.byref(d), self._stream()))

    def gae(self, rewards, values, dones, last_values, gamma, lam, advantages=None, value_targets=None):
        """Generalized advantage estimation over a window (ovc_gae; include/ovc_b200.h gives the recurrence): rewards /
        values float32 [T, 2N] (rows [env][agent]), dones uint8 [T, N] (terminal), last_values float32 [2N].  Returns
        (advantages, value_targets) float32 [T, 2N]."""
        T = rewards.shape[0]
        R = 2 * self.n_envs
        if advantages is None:
            advantages = torch.empty((T, R), dtype=torch.float32, device=self.device)
        if value_targets is None:
            value_targets = torch.empty((T, R), dtype=torch.float32, device=self.device)
        for t, dt, n in ((rewards, torch.float32, T * R), (values, torch.float32, T * R), (dones, torch.uint8, T * self.n_envs),
                         (last_values, torch.float32, R), (advantages, torch.float32, T * R), (value_targets, torch.float32, T * R)):
            assert t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == n, (t.dtype, tuple(t.shape))
        _native.check(self._lib.ovc_gae(rewards.data_ptr(), values.data_ptr(), dones.data_ptr(), last_values.data_ptr(), T, R,
                                        float(gamma), float(lam), advantages.data_ptr(), value_targets.data_ptr(), self._stream()))
        return advantages, value_targets

    def gae_view(self, rewards, values, dones, last_values, gamma, lam, advantages, value_targets):
        """``gae`` over ONE row per environment (ovc_gae_view): rewards / values / advantages / value_targets float32 [T, N],
        dones uint8 [T, N], last_values float32 [N]; bit for bit ``gae`` on those rows of a two-row layout."""
        T, N = rewards.shape[0], self.n_envs
        for t, dt, n in ((rewards, torch.float32, T * N), (values, torch.float32, T * N), (dones, torch.uint8, T * N),
                         (last_values, torch.float32, N), (advantages, torch.float32, T * N), (value_targets, torch.float32, T * N)):
            assert t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == n, (t.dtype, tuple(t.shape))
        _native.check(self._lib.ovc_gae_view(rewards.data_ptr(), values.data_ptr(), dones.data_ptr(), last_values.data_ptr(), T, N,
                                             float(gamma), float(lam), advantages.data_ptr(), value_targets.data_ptr(), self._stream()))
        return advantages, value_targets

    def gae_horizon(self, rewards, values, dones, terminal_values, last_values, gamma, lam, advantages, value_targets, one_view=False):
        """``gae`` (``one_view``: ``gae_view``) that bootstraps from ``terminal_values`` (float32, the shape of ``values``) at
        every episode end instead of counting the state after it terminal (ovc_gae_horizon / ovc_gae_horizon_view,
        include/ovc_horizon.h gives the recurrence).  Returns (advantages, value_targets)."""
        from . import _horizon_native

        T, N = rewards.shape[0], self.n_envs
        R = N if one_view else 2 * N
        for t, dt, n in ((rewards, torch.float32, T * R), (values, torch.float32, T * R), (dones, torch.uint8, T * N),
                         (terminal_values, torch.float32, T * R), (last_values, torch.float32, R), (advantages, torch.float32, T * R),
                         (value_targets, torch.float32, T * R)):
            assert t.is_cuda and t.dtype == dt and t.is_contiguous() and t.numel() == n, (t.dtype, tuple(t.shape))
        L = _horizon_native.lib()
        _horizon_native.check((L.ovc_gae_horizon_view if one_view else L.ovc_gae_horizon)(
            rewards.data_ptr(), values.data_ptr(), dones.data_ptr(), terminal_values.data_ptr(), last_values.data_ptr(), T, R,
            float(gamma), float(lam), advantages.data_ptr(), value_targets.data_ptr(), self._stream()))
        return advantages, value_targets

    def horizon_rows(self, partner_seat, one_view, records, view, jrow, rng, values=None):
        """The learner rows of the environments whose episode ended with the last ``step`` (``self.done``), compacted on the
        device (ovc_horizon_rows, include/ovc_horizon.h): both views of a self-play environment (``partner_seat`` None or
        -1), view ``1 - partner_seat[e]`` of a paired one, and with ``one_view`` that view at row e.  Writes ``records``
        int32 [rows, S] (the terminal records), ``view`` and ``jrow`` int32 [rows] (each compact row's view and output row)
        and ``rng`` int32 [2] = (0, the row count), rows = 2N (N with ``one_view``); ``values`` (float32 [rows], optional)
        is zeroed."""
        from . import _horizon_native

        R = self.n_envs if one_view else 2 * self.n_envs
        assert partner_seat is not None or not one_view, "one_view needs partner_seat (agent 1's player)"
        for t, n in ((partner_seat, self.n_envs), (view, R), (jrow, R), (rng, 2)):
            assert t is None or (t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n)
        assert records.is_cuda and records.dtype == torch.int32 and records.is_contiguous() and records.shape == (R, self.state_words)
        assert values is None or (values.is_cuda and values.dtype == torch.float32 and values.is_contiguous() and values.numel() == R)
        ptr = lambda t: 0 if t is None else t.data_ptr()
        _horizon_native.check(_horizon_native.lib().ovc_horizon_rows(
            self.state.data_ptr(), self.state_words, self.done.data_ptr(), ptr(partner_seat), int(bool(one_view)), self.n_envs,
            records.data_ptr(), view.data_ptr(), jrow.data_ptr(), rng.data_ptr(), ptr(values), self._stream()))

    def partner_actions(self, tables, partner_seat, counter, seed=0, n_actions=6, out=None, scores=None):
        """The behaviour-cloned partner's actions (ovc_partner_policy, K10: featurize_state of the partner's view -> the BC
        MLP -> the ovc_sample_actions draw, one kernel, the features never materialised).  ``tables``: the six tensors of
        ``selfplay.BCPolicy.tables()``; ``partner_seat`` int32 [N] (-1: no partner, 0 / 1: the partner's player index);
        ``counter`` int64 CUDA tensor of 2 zeros that the kernel advances.  Writes ``out[e, seat]`` (int32 [N, 2], e.g. the
        joint action the PPO policy drew) for partnered environments only, and their heads into ``scores`` (float32 [N, 8])
        when given.  Returns ``out``."""
        w1, b1, wh, bh, wo, bo = tables
        for t, dt in ((w1, torch.bfloat16), (b1, torch.float32), (wh, torch.bfloat16), (bh, torch.float32), (wo, torch.bfloat16), (bo, torch.float32)):
            assert t.is_cuda and t.dtype == dt and t.is_contiguous(), "partner tables: bf16 weights, float32 biases, contiguous CUDA tensors"
        assert partner_seat.is_cuda and partner_seat.dtype == torch.int32 and partner_seat.is_contiguous() and partner_seat.numel() == self.n_envs
        assert counter.is_cuda and counter.dtype == torch.int64 and counter.numel() == 2 and counter.is_contiguous()
        if out is None:
            out = torch.zeros((self.n_envs, 2), dtype=torch.int32, device=self.device)
        assert out.is_cuda and out.dtype == torch.int32 and out.is_contiguous() and out.numel() == 2 * self.n_envs
        if scores is not None:
            assert scores.is_cuda and scores.dtype == torch.float32 and scores.is_contiguous() and scores.numel() == 8 * self.n_envs
        _native.check(self._lib.ovc_partner_policy(
            self.tables.data_ptr(), self.n_layouts, self.feature_lut().data_ptr(), self.state.data_ptr(), partner_seat.data_ptr(),
            self.n_envs, self.state_words, w1.shape[1], w1.shape[0], w1.data_ptr(), b1.data_ptr(), wh.data_ptr(), bh.data_ptr(),
            wh.shape[0], wo.data_ptr(), bo.data_ptr(), int(n_actions), int(seed) & (2**64 - 1), counter.data_ptr(), out.data_ptr(),
            0 if scores is None else scores.data_ptr(), self._stream()))
        return out

    def assign_partners(self, partner_seat, bc_factor, counter, seed=0, done=None):
        """The per-episode seat draw of PPO_BC (ovc_assign_partners): for every environment whose episode ended with the last
        ``step`` (``done``: int32 [N], e.g. ``self.done``; None = every environment) ``partner_seat[e]`` becomes 0 or 1 (the
        partner's player index, equally likely) with probability ``bc_factor``, else -1 (self-play).  ``bc_factor``:
        float32 CUDA scalar tensor, read by the kernel (a captured graph follows its current value); ``counter`` as
        ``partner_actions``'."""
        assert partner_seat.is_cuda and partner_seat.dtype == torch.int32 and partner_seat.is_contiguous() and partner_seat.numel() == self.n_envs
        assert bc_factor.is_cuda and bc_factor.dtype == torch.float32 and bc_factor.numel() == 1
        assert counter.is_cuda and counter.dtype == torch.int64 and counter.numel() == 2 and counter.is_contiguous()
        if done is not None:
            assert done.is_cuda and done.dtype == torch.int32 and done.is_contiguous() and done.numel() == self.n_envs
        _native.check(self._lib.ovc_assign_partners(0 if done is None else done.data_ptr(), bc_factor.data_ptr(), self.n_envs,
                                                    int(seed) & (2**64 - 1), counter.data_ptr(), partner_seat.data_ptr(), self._stream()))
        return partner_seat

    def greedy_tables(self):
        """(tables uint8 [n_layouts, 2660], plans uint16): every layout's greedy partner tables on the device
        (``greedy.build_greedy_tables``), built at the first call and kept, so a captured graph's tables stay alive.
        Raises ValueError for a layout whose orders are not one 3-onion order."""
        if self._greedy is None:
            from . import _greedy_native, greedy

            tab, plans = greedy.build_greedy_tables(self.layouts)
            assert tab.shape[1] == _greedy_native.lib().ovc_greedy_layout_table_size(), "greedy table size mismatch with the native library"
            self._greedy = (torch.from_numpy(tab).to(self.device), torch.from_numpy(plans.view(np.int16)).to(self.device))
        return self._greedy

    def greedy_actions(self, player, prev, counter, seed=0, done=None, out=None):
        """The greedy partner's actions (ovc_greedy_actions, include/ovc_greedy.h): GreedyHumanModel.action of player
        ``player[e]`` (int32 [N]; -1: the agent does not play e) on every environment, written to ``out[e, player[e]]``
        (int32 [N, 2]; default a new zero tensor).  ``prev`` (int32 [N]) holds each environment's previous players' key for
        the stuck rule and is updated; ``done`` (int32 [N], e.g. ``self.done`` from the previous ``step``) invalidates it;
        ``counter`` int64 CUDA tensor of 2 zeros that the kernel advances; stuck draws use key ``seed``.  Returns ``out``."""
        from . import _greedy_native

        tables, plans = self.greedy_tables()
        for t, n in ((player, self.n_envs), (prev, self.n_envs)) + (() if done is None else ((done, self.n_envs),)):
            assert t.is_cuda and t.dtype == torch.int32 and t.is_contiguous() and t.numel() == n, "player / prev / done: int32 CUDA [N]"
        assert counter.is_cuda and counter.dtype == torch.int64 and counter.numel() == 2 and counter.is_contiguous()
        if out is None:
            out = torch.zeros((self.n_envs, 2), dtype=torch.int32, device=self.device)
        assert out.is_cuda and out.dtype == torch.int32 and out.is_contiguous() and out.numel() == 2 * self.n_envs
        _greedy_native.check(_greedy_native.lib().ovc_greedy_actions(
            self.tables.data_ptr(), tables.data_ptr(), plans.data_ptr(), self.n_layouts, self.state.data_ptr(), player.data_ptr(),
            0 if done is None else done.data_ptr(), prev.data_ptr(), self.n_envs, self.state_words, int(seed) & (2**64 - 1),
            counter.data_ptr(), out.data_ptr(), self._stream()))
        return out

    def feature_lut(self):
        if self._lut is None:
            lut = np.stack([l.feature_lut() for l in self.layouts]).view(np.uint8).reshape(self.n_layouts, -1)
            assert lut.shape[1] == 1024 * self._lib.ovc_feat_lut_entry_size()
            self._lut = torch.from_numpy(lut).to(self.device)
        return self._lut

    def featurize_state(self, num_pots=2, out=None, view_swap=None, states=None):
        """featurize_state (overcooked_mdp.py:2579-2898; default NO_COUNTERS_PARAMS planner):
        float32 [N, 2, 2*(10*num_pots+28)].  ``states``: featurize these records (int32 CUDA tensor [M, S], e.g. stored
        games) instead of ``self.state``; N is then M."""
        F = 2 * (10 * num_pots + 28)
        recs, n = self._records(states)
        if view_swap is not None:
            assert view_swap.dtype == torch.int32 and view_swap.is_cuda and view_swap.is_contiguous() and view_swap.numel() == n
        if out is None:
            out = torch.empty((n, 2, F), dtype=torch.float32, device=self.device)
        assert out.dtype == torch.float32 and out.is_cuda and out.is_contiguous() and out.numel() == n * 2 * F
        _native.check(self._lib.ovc_featurize(
            self.tables.data_ptr(), self.n_layouts, self.feature_lut().data_ptr(), recs.data_ptr(),
            0 if view_swap is None else view_swap.data_ptr(), out.data_ptr(), n, self.state_words, num_pots,
            self._stream()))
        return out

    def potential_tables(self, gamma=0.99):
        """The device tables ``potential`` evaluates phi with at ``gamma`` (potential tables, cost LUT, gamma powers): built
        on first use and kept for the env's lifetime, so a CUDA graph that captured them never reads freed memory.  Build
        them before a capture: building copies host data to the device."""
        if gamma not in self._pot:
            pt, cl, gpow = L.build_potential_tables(self.layouts, gamma)
            assert pt.shape[1] == self._lib.ovc_potential_table_size()
            self._pot[gamma] = (torch.from_numpy(pt).to(self.device), torch.from_numpy(cl).to(self.device),
                                torch.from_numpy(gpow).to(self.device))
        return self._pot[gamma]

    def potential(self, gamma=0.99, out=None):
        """potential_function (overcooked_mdp.py:2920-3250) of every environment: float64 [N], bit-identical
        to the reference's Python floats (planner costs from the default NO_COUNTERS_PARAMS planner)."""
        pt, cl, gpow = self.potential_tables(gamma)
        if out is None:
            out = torch.empty(self.n_envs, dtype=torch.float64, device=self.device)
        assert out.dtype == torch.float64 and out.is_cuda and out.is_contiguous() and out.numel() == self.n_envs
        _native.check(self._lib.ovc_potential(
            self.tables.data_ptr(), self.n_layouts, pt.data_ptr(), cl.data_ptr(), gpow.data_ptr(), gpow.numel(),
            self.state.data_ptr(), out.data_ptr(), self.n_envs, self.state_words, self._stream()))
        return out

    def potential_shaping(self, phi_s, dense):
        """The dense reward of the last ``step(..., auto_reset=False)`` (ovc_potential_shaping, one kernel):
        ``dense[e] = float32(phi(s') - phi_s[e])`` with phi at gamma 0.99 on the record the step left (the terminal one where
        an episode ended), then every environment with ``done`` is reset as ``auto_reset`` would have reset it.
        ``phi_s``: float64 [N], ``potential(0.99)`` taken before the step; ``dense``: float32 [N], written."""
        assert phi_s.is_cuda and phi_s.dtype == torch.float64 and phi_s.is_contiguous() and phi_s.numel() == self.n_envs
        assert dense.is_cuda and dense.dtype == torch.float32 and dense.is_contiguous() and dense.numel() == self.n_envs
        pt, cl, gpow = self.potential_tables(0.99)
        _native.check(self._lib.ovc_potential_shaping(
            self.tables.data_ptr(), self.n_layouts, self.start_records.data_ptr(), pt.data_ptr(), cl.data_ptr(), gpow.data_ptr(),
            gpow.numel(), self.state.data_ptr(), self.done.data_ptr(), phi_s.data_ptr(), dense.data_ptr(), self.n_envs,
            self.state_words, self._rs_ptr(), self._stream()))
        return dense

    # ---------------------------------------------------------------------------------------------
    def sparse_by_agent(self, events, layout_ids=None):
        """Per-agent delivery reward int32 [..., N, 2] from the event words (bits 25-28 carry the delivered recipe).
        ``layout_ids`` (int [N]): the layouts the events were produced on; default the initial assignment — with
        ``random_layout`` pass ``layout_ids()`` taken BEFORE the step (a finished environment has moved on)."""
        val = torch.from_numpy(np.stack([l.deliver_value for l in self.layouts]).astype(np.int32)).to(events.device)
        rec = (events >> L.EV_RECIPE_SHIFT) & 15
        ids = self.env_layout if layout_ids is None else layout_ids
        lid = ids.long().view(*([1] * (events.dim() - 2)), -1, 1).expand_as(rec)
        return val[lid, rec.long()] * ((events >> 15) & 1)

    def get_states(self, indices=None):
        """Unpack records into OvercookedState objects (host; for debugging / the drop-in adapters)."""
        recs = self.state.cpu().numpy()
        idx = range(self.n_envs) if indices is None else indices
        return [L.unpack_state(self.layouts[int(recs[i][3]) & 0xFF], recs[i]) for i in idx]

    def set_states(self, states, indices=None):
        idx = list(range(self.n_envs)) if indices is None else list(indices)
        lids = self._layout_ids_host()
        recs = np.stack([L.pack_state(self.layouts[lids[i]], s, int(lids[i]), self.state_words) for i, s in zip(idx, states)])
        self.state[torch.as_tensor(idx, device=self.device)] = torch.from_numpy(recs).to(self.device)


class PassTicket(object):
    """Completion handle of one HostRolloutPipeline pass submitted with wait=False."""

    def __init__(self, pipe, ticket):
        self._pipe, self.ticket = pipe, ticket

    def synchronize(self):
        """Block the host until the pass's last device->host copy has landed."""
        _native.check(self._pipe._lib.ovc_pipeline_wait(self._pipe._handle, self.ticket))


class HostRolloutPipeline(object):
    """Rollout collection with HOST buffers: the end-to-end path a host-side policy / learner sees.

    ``run(actions_host[T,N,2])`` hands pinned host buffers to the native driver (``ovc_pipeline_run``), which
    copies the action trace host->device in chunks of ``chunk`` steps (copy stream), advances the environments with
    the fused rollout kernel (compute stream) and copies sparse / shaped / done / events device->host (second copy
    stream), the three stages overlapped across chunks with double buffering — and across successive passes with
    ``wait=False``.  Returns pinned host tensors (sparse[T,N], shaped[T,N,2], done[T,N], events[T,N,2]).  Per
    environment-step this moves 8 bytes host->device and 24 bytes device->host (2 + 13 with ``narrow``, 2 + 6 with
    ``packed``, 1 + 2 with ``codes``).
    ``run`` is stream ordered like every other call here: the returned tensors are complete once the current
    stream has been synchronised (``torch.cuda.current_stream().synchronize()``), not when ``run`` returns.
    """

    def __init__(self, env, n_steps, chunk=50, narrow=False, packed=False, codes=False, host_buffers=1, stream=False,
                 stream_fill=0.25, packed_actions=True):
        """narrow=True: uint8 actions in, int16 sparse / int8 shaped / uint8 done / int32 events out — the same
        values in 2 + 13 instead of 8 + 24 bytes per env-step.  packed=True: uint8 actions in, int16 sparse / int8
        shaped / int16 event codes (+done) out — 2 + 6 bytes per env-step, lossless (wire.decode_event_codes).
        codes=True: one byte of joint action in (wire.pack_actions, actions_host uint8 [T,N]), one int16 word of
        event codes + done + reward-grant bits out — 1 + 2 bytes per env-step, lossless (env.expand_codes).
        host_buffers: number of pinned output sets, used round robin by successive run() calls (2 lets a consumer
        read pass i while pass i+1 is in flight, see run(wait=False)).
        stream=True: the result as a sparse event stream (OVC_F_OUT_STREAM): per transition one lane mask per 32
        environments + the non-zero code words, ``stream_fill`` x 32 x chunk value slots per group and chunk (0.125 + 2 x
        stream_fill bytes per env-step device->host instead of 2); run() returns (masks, values) host tensors and
        ``expand(result)`` rebuilds dense arrays, falling back to the dense code words kept on the device for any chunk
        whose group overflowed.  packed_actions=False (with codes / stream): uint8 [T, N, 2] actions instead of one byte
        per joint action."""
        codes = codes or stream
        narrow = narrow or packed or codes
        self.env, self.T, self.chunk, self.narrow, self.packed = env, int(n_steps), int(chunk), bool(narrow), bool(packed)
        self.codes, self.stream = bool(codes), bool(stream)
        self.packed_actions = bool(packed_actions) and self.codes
        if narrow:
            assert env.narrow_ok(), "rewards of these layouts do not fit the narrow formats"
        N, dev = env.n_envs, env.device
        self._lib = env._lib
        self.act_dtype = torch.uint8 if narrow else torch.int32
        self.act_shape = (N,) if self.packed_actions else (N, 2)
        self.n_chunks = -(-self.T // self.chunk)
        self.stream_cap = max(1, min(_native.STREAM_CAP_MAX, int(round(self.chunk * 32 * float(stream_fill))))) if stream else 0
        with torch.cuda.device(dev):
            self.d_act = [torch.empty((self.chunk,) + self.act_shape, dtype=self.act_dtype, device=dev) for _ in range(2)]
            if stream:
                G = env.n_groups()
                self.d_out = [(torch.empty((G, self.stream_cap), dtype=torch.int16, device=dev), None, None,
                               torch.empty((self.chunk, G), dtype=torch.int32, device=dev)) for _ in range(2)]
                # dense code words of a whole pass stay on the device (two sets: pass k uses set k & 1): overflow backup
                self.d_codes_full = [torch.empty((self.T, N), dtype=torch.int16, device=dev) for _ in range(2)]
                self.h_outs = [(torch.zeros((self.n_chunks, G, self.stream_cap), dtype=torch.int16, pin_memory=True), None, None,
                                torch.zeros((self.T, G), dtype=torch.int32, pin_memory=True)) for _ in range(max(1, int(host_buffers)))]
            else:
                self.d_out = [env.alloc_rollout_out(self.chunk, narrow=narrow, packed=packed, codes=codes) for _ in range(2)]
                self.h_outs = [env.alloc_rollout_out(self.T, narrow=narrow, pin=True, packed=packed, codes=codes)
                               for _ in range(max(1, int(host_buffers)))]
        self.h_out = self.h_outs[0]
        self._runs = 0
        self.h2d_bytes_per_step = N * (1 if self.packed_actions else 2) * self.d_act[0].element_size()
        if stream:
            self.d2h_bytes_per_step = (self.h_out[3].numel() * 4 + self.h_out[0].numel() * 2) / float(self.T)
        else:
            self.d2h_bytes_per_step = sum(N * (2 if o.dim() == 3 else 1) * o.element_size() for o in self.h_out if o is not None)
        flags = env._flags() | (_native.F_ACT_PACKED if self.packed_actions else _native.F_ACT_U8 if narrow else 0)
        flags |= (_native.F_OUT_STREAM if stream else _native.F_OUT_CODES if codes else _native.F_OUT_PACKED if packed
                  else _native.F_OUT_NARROW if narrow else 0)
        d = _native.PipelineDesc()
        d.layouts, d.n_layouts, d.state_words = env.tables.data_ptr(), env.n_layouts, env.state_words
        d.start_records, d.state, d.n_envs = env.start_records.data_ptr(), env.state.data_ptr(), N
        d.horizon, d.flags, d.chunk = env.horizon, flags, self.chunk
        d.has_random_start = int(env._rs is not None)
        if env._rs is not None:
            d.random_start = env._rs
        ptr = lambda t: 0 if t is None else t.data_ptr()
        for b in range(2):
            d.d_actions[b] = self.d_act[b].data_ptr()
            d.d_sparse[b], d.d_shaped[b], d.d_done[b], d.d_events[b] = (ptr(t) for t in self.d_out[b])
            d.d_codes_full[b] = self.d_codes_full[b].data_ptr() if stream else 0
        d.stream_cap = self.stream_cap
        h = ctypes.c_void_p()
        with torch.cuda.device(dev):
            _native.check(self._lib.ovc_pipeline_create(ctypes.byref(d), ctypes.byref(h)))
        self._handle = h

    def run(self, actions_host, wait=True):
        """wait=True: the current stream waits for the pass (stream-ordered like every other call); returns the
        host tensors.  wait=False: returns (host tensors, PassTicket) without joining the current stream, so the
        next run() starts its copies while this pass is still draining — the steady state of a collection
        loop; ``ticket.synchronize()`` before reading, and ``join()`` before touching the env from the current
        stream again."""
        assert actions_host.dtype == self.act_dtype and actions_host.is_pinned() and actions_host.is_contiguous()
        assert tuple(actions_host.shape) == (self.T,) + self.act_shape
        h_out = self.h_outs[self._runs % len(self.h_outs)]
        self._last_set = self._runs & 1  # which dense-backup set this pass writes (the native side counts the same way)
        self._runs += 1
        ptr = lambda t: 0 if t is None else t.data_ptr()
        ticket = ctypes.c_int64(-1)
        _native.check(self._lib.ovc_pipeline_run(
            self._handle, actions_host.data_ptr(), ptr(h_out[0]), ptr(h_out[1]), ptr(h_out[2]), ptr(h_out[3]), self.T,
            self.env._stream(), int(bool(wait)), ctypes.byref(ticket)))
        self._last_actions = actions_host  # keep the source alive until the copies have run
        if wait:
            return h_out
        return h_out, PassTicket(self, ticket.value)

    def expand(self, h_out, codes_set=None, out=None, n_threads=0, **which):
        """stream=True: dense host arrays (dict, as env.expand_codes) from one pass's (values, -, -, masks) host tensors,
        AFTER the pass has landed.  ``codes_set``: the dense-backup set that pass wrote (``self._last_set`` right after
        its run()); if a group overflowed its value slots the dense words are fetched from that set and expanded instead
        (correct as long as no later pass has reused the set: passes k and k + 2 share one)."""
        assert self.stream
        dense, over = self.env.expand_stream(h_out[3], h_out[0], chunk=self.chunk, out=out, n_threads=n_threads, **which)
        self.last_overflow = over
        if over:
            cs = self._last_set if codes_set is None else codes_set
            words = self.d_codes_full[cs].cpu()  # synchronising copy: the rare slow path
            dense = self.env.expand_codes(words, out=dense, n_threads=n_threads)
        return dense

    def join(self):
        """Make the current stream wait for everything the pipeline has in flight."""
        _native.check(self._lib.ovc_pipeline_join(self._handle, self.env._stream()))

    def close(self):
        if getattr(self, "_handle", None) is not None and self._handle.value:
            self._lib.ovc_pipeline_destroy(self._handle)
            self._handle = ctypes.c_void_p()

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


class EpisodeStats(object):
    """Running per-environment episode statistics on the device — the batched form of OvercookedEnv.game_stats
    (overcooked_env.py:308-319, 382-401) and of the ``episode`` entry of the info dict (:363-380).

    The reference keeps, per event and agent, the LIST of timesteps at which it fired; its consumers only ever
    take ``len()`` of those lists (rllib.py:480-483), so counts are kept: ``event_counts[N, 2, 25]``, plus
    ``cumulative_sparse_rewards_by_agent[N, 2]``, ``cumulative_shaped_rewards_by_agent[N, 2]`` and ``ep_length[N]``.
    ``update`` returns the finished environments' statistics (a dict of tensors, rows selected by ``done``) and
    clears them for the next episode.

    The running state is kept by the kernel of ``env.record_transition(..., stats=, records=)``
    (ovc_record_transition_stats), which also sums ``ep_reward_by_agent[N, 2]`` (float32, the per-agent rewards
    ``sparse + factor * shaped_i`` of that call; ``update`` uses factor 1) and keeps ``layout_id[N]``, the layout each
    running episode is played on (it changes at resets with random_layout).
    """

    def __init__(self, env):
        self.env = env
        N, dev = env.n_envs, env.device
        self.event_counts = torch.zeros((N, 2, 25), dtype=torch.int32, device=dev)
        self.cumulative_sparse_rewards_by_agent = torch.zeros((N, 2), dtype=torch.int64, device=dev)
        self.cumulative_shaped_rewards_by_agent = torch.zeros((N, 2), dtype=torch.int64, device=dev)
        self.ep_reward_by_agent = torch.zeros((N, 2), dtype=torch.float32, device=dev)
        self.ep_length = torch.zeros(N, dtype=torch.int32, device=dev)
        self.layout_id = env.layout_ids()
        self._records = None  # update()'s one-slot record buffer
        self._one = None

    def state_tensors(self):
        """The running state, every tensor the kernel writes."""
        return [self.event_counts, self.cumulative_sparse_rewards_by_agent, self.cumulative_shaped_rewards_by_agent, self.ep_reward_by_agent,
                self.ep_length, self.layout_id]

    def update(self, sparse, shaped, done, events):
        """Feed the outputs of one step() (tensors [N], [N,2], [N], [N,2]); call it after EVERY step."""
        if self._records is None:
            self._records = EpisodeRecords(self.env, 1)
            self._one = torch.ones(1, dtype=torch.float32, device=self.env.device)
        r = self._records
        r.clear()
        self.env._record(sparse, shaped, done, events, self._one, stats=self, records=r)
        d = done != 0
        finished = None
        if bool(d.any()):
            idx = torch.nonzero(d).squeeze(1)
            finished = {
                "env_index": idx,
                "ep_game_stats": r.game_stats[0, idx],
                "ep_sparse_r_by_agent": r.sparse_r_by_agent[0, idx],
                "ep_shaped_r_by_agent": r.shaped_r_by_agent[0, idx],
                "ep_sparse_r": r.sparse_r_by_agent[0, idx].sum(1),
                "ep_shaped_r": r.shaped_r_by_agent[0, idx].sum(1),
                "ep_length": r.length[0, idx],
            }
        return finished


class EpisodeRecords(object):
    """The episodes that finished, kept on the device by ``env.record_transition(..., stats=, records=)``: struct-of-arrays
    tensors ``[capacity, N, ...]`` where slot ``k`` of environment ``e`` is its ``k``-th episode to end since ``clear()``.

    length int32, layout int32 (the layout id the episode was played on), partner_seat int32 (-1: self-play),
    sparse_r_by_agent / shaped_r_by_agent int64 [.., 2], game_stats int32 [.., 2, 25] (event counts, the ``len()`` of the
    reference's game_stats lists), reward_by_agent float32 [.., 2] (the sum of the per-agent rewards of the episode);
    count int32 [N] (episodes written per environment), dropped int32 [N] (episodes that ended with the buffer full,
    not written).  ``members=True`` (a population of partners): also partner_member int32 [capacity, N], the member each
    episode was played with (written by ``env.assign_members``); None otherwise.  ``pairs=True`` (population play): also
    pair int32 [capacity, N, 2], the members on players 0 / 1 of each episode (written by ``env.assign_pairs``); None
    otherwise."""

    def __init__(self, env, capacity, members=False, pairs=False):
        self.env = env
        self.capacity = int(capacity)
        assert self.capacity >= 0
        C, N, dev = self.capacity, env.n_envs, env.device
        z = lambda shape, dt: torch.zeros(shape, dtype=dt, device=dev)
        self.length, self.layout, self.partner_seat = (z((C, N), torch.int32) for _ in range(3))
        self.sparse_r_by_agent, self.shaped_r_by_agent = z((C, N, 2), torch.int64), z((C, N, 2), torch.int64)
        self.game_stats = z((C, N, 2, 25), torch.int32)
        self.reward_by_agent = z((C, N, 2), torch.float32)
        self._counters = z((2, N), torch.int32)  # count and dropped: one memset clears both
        self.count, self.dropped = self._counters[0], self._counters[1]
        self.partner_member = z((C, N), torch.int32) if members else None
        self.pair = z((C, N, 2), torch.int32) if pairs else None

    def tensors(self):
        return [self.length, self.layout, self.partner_seat, self.sparse_r_by_agent, self.shaped_r_by_agent, self.game_stats,
                self.reward_by_agent, self._counters] + [t for t in (self.partner_member, self.pair) if t is not None]

    def clear(self):
        """Forget every record (stream ordered, one memset: capturable in a CUDA graph)."""
        self._counters.zero_()

    def finished(self):
        """The records as a dict of tensors in the keys of the reference's episode info (overcooked_env.py:363-401) and of
        ``EpisodeStats.update``: env_index, ep_game_stats, ep_sparse_r(_by_agent), ep_shaped_r(_by_agent), ep_length, plus
        ep_reward_by_agent, layout and partner_seat (and partner_member with ``members=True``, pair with ``pairs=True``).  Rows are ordered by (slot,
        env).  Synchronises with the host."""
        k, e = torch.nonzero(torch.arange(self.capacity, device=self.env.device)[:, None] < self.count[None, :], as_tuple=True)
        sp, sh = self.sparse_r_by_agent[k, e], self.shaped_r_by_agent[k, e]
        out = {"env_index": e, "ep_game_stats": self.game_stats[k, e], "ep_sparse_r_by_agent": sp, "ep_shaped_r_by_agent": sh,
               "ep_sparse_r": sp.sum(1), "ep_shaped_r": sh.sum(1), "ep_length": self.length[k, e],
               "ep_reward_by_agent": self.reward_by_agent[k, e], "layout": self.layout[k, e], "partner_seat": self.partner_seat[k, e]}
        if self.partner_member is not None:
            out["partner_member"] = self.partner_member[k, e]
        if self.pair is not None:
            out["pair"] = self.pair[k, e]
        return out
