"""Every compiled form of the policy kernels against the float64 restatement of tests/policy_reference.py.

``INSTANTIATIONS`` names each device instantiation of the policy-kernel templates as ``cuobjdump -symbols | cu++filt``
prints it (tests/test_policy_forms_cpu.py checks that the table is exactly what the built library holds) and says which
test compares it with float64: a case of this file, or another test that already does.  A case reaches its instantiation
through the public entry point, by k0 = 32 KS2 (K8) or by an (n_out, grid) pair that encode_linear_impl maps to the CPL
(K7), and compares with the restatement at the rows the form's map names, never with another kernel form: scores, values
and activations bit for bit at their output index, the action at its joint row against the Philox + Gumbel-max
definition at that row id, logp within 1e-5 plus the float32 rounding of the formula at the row's largest score.  Every
element outside the map and past the end keeps its sentinel, input rows outside the map hold NaN, and the draw counter
advances once per launch."""
import numpy as np
import pytest
import torch

import policy_reference as P
from oracle import cpu
from overcooked_ai_b200 import _native
from overcooked_ai_b200.batched import BatchedOvercookedEnv

GUARD = 64  # sentinel rows past each output's end
ROWMAP = {"identity": 0, "view": 1, "rows": 2, "joint": 3}
K7_NOUT = {8: 512, 4: 384, 2: 192}  # on 5x4 grids encode_linear_impl picks CPL 8 / 4 / 2 for these; on 13x7 always CPL 2


def _instantiations():
    t = {}
    for ks2 in range(1, 9):
        for form, logps in (("identity", (0, 1)), ("view", (0, 1)), ("rows", (0, 1)), ("joint", (1,))):
            for lp in logps:
                t["ovc::policy_tail_kernel<(int)%d, (ovc::RowMap)%d, (bool)%d, (bool)0>" % (ks2, ROWMAP[form], lp)] = ("k8", form, ks2, lp)
        t["ovc::policy_tail_kernel<(int)%d, (ovc::RowMap)0, (bool)0, (bool)1>" % ks2] = "test_gpu_lstm_policy.py::test_k8_hidden_output_exact"
        for lp in (0, 1):
            t["ovc::policy_tail_grouped_kernel<(int)%d, (bool)%d, (ovc::RowMap)0>" % (ks2, lp)] = ("k8", "grouped", ks2, lp)
        t["ovc::policy_tail_grouped_kernel<(int)%d, (bool)1, (ovc::RowMap)3>" % ks2] = ("k8", "grouped_joint", ks2, 1)
    for cpl in (2, 4, 8):
        t["ovc::encode_linear_kernel<(int)%d, (bool)0, (bool)0>" % cpl] = ("k7", "two_view", cpl)
        t["ovc::encode_linear_kernel<(int)%d, (bool)1, (bool)0>" % cpl] = ("k7", "view", cpl)
        t["ovc::encode_linear_kernel<(int)%d, (bool)1, (bool)1>" % cpl] = ("k7", "rows", cpl)
        for form in ("masked", "grouped", "grouped_masked"):
            t["ovc::encode_linear_%s_kernel<(int)%d>" % (form, cpl)] = ("k7", form, cpl)
    for cpl in (1, 2, 4):  # CPL 1 on long_cook_time's 13x7 grid, 2 and 4 on cramped_room
        t["ovc::encode_linear_wgrad_kernel<(int)%d>" % cpl] = "test_gpu_records_learner.py::test_k12_exact_on_random_play"
    for lp in (0, 1):
        t["ovc::sample_actions_kernel<(bool)%d, (ovc::RowMap)0>" % lp] = "test_gpu_policy_exact.py::test_draw_counter_past_2_to_the_32"
        for form in ("view", "rows"):
            t["ovc::sample_actions_kernel<(bool)%d, (ovc::RowMap)%d>" % (lp, ROWMAP[form])] = ("draw", form, lp)
    t["ovc::wide_layers_kernel<(bool)0, (bool)0>"] = "test_gpu_policy_exact.py::test_k9_exact"
    t["ovc::wide_layers_kernel<(bool)1, (bool)0>"] = ("k9", "range")
    t["ovc::wide_layers_kernel<(bool)0, (bool)1>"] = ("k9", "grouped")
    t["ovc::lstm_head_kernel<(bool)0>"] = "test_gpu_lstm_policy.py::test_k11_exact"
    t["ovc::lstm_head_kernel<(bool)1>"] = "test_gpu_lstm_policy.py::test_k11_view_exact"
    return t


INSTANTIATIONS = _instantiations()


def _cases(kind):
    return [v[1:] for v in INSTANTIATIONS.values() if isinstance(v, tuple) and v[0] == kind]


def _np(t):
    return t.cpu().numpy()


def _dev(v, dt):
    return torch.from_numpy(np.ascontiguousarray(v)).cuda().to(dt)


def _ptr(t):
    return 0 if t is None else t.data_ptr()


def _full(n, dt, fill, inner=()):
    return torch.full((n + GUARD,) + tuple(inner), fill, dtype=dt, device="cuda")


def _untouched(got, idx, fill):
    """Every row of ``got`` (numpy, the whole guarded allocation) outside ``idx`` holds ``fill``."""
    rest = np.ones(len(got), bool)
    rest[idx] = False
    return bool(np.isnan(got[rest]).all()) if isinstance(fill, float) and np.isnan(fill) else bool((got[rest] == fill).all())


def _range(n, i):
    """[lo, hi) for a Rows / Joint case, never empty: a start that is not 16-row aligned, an end past n_rows (clipped) or
    before it.  The empty range is an extra launch of the case."""
    lo = min(n // 4, 1 + i % 13)
    return lo, (n + 3 if i % 2 else max(lo + 1, n - i % 3))


def _swap(rng, n, i):
    return None if i % 3 == 0 else rng.randint(0, 3, size=n).astype(np.int32)  # 2: any non-zero value swaps


def _player(seat, swap, e):
    e = np.asarray(e)
    return seat ^ (np.zeros(e.shape, np.int64) if swap is None else (swap[e] != 0).astype(np.int64))


# ------------------------------------------------------------------------------------------------------------------ K8
SLOPES = [(0.0, 0.25), (0.25, 0.5), (0.5, 1.0), (1.0, 0.0)]
SIZES = [15, 16, 17, 33, 257, 4099]
HEAD_MAX = 8.0  # heads scaled into [-8, 8]: the Gumbel noise moves the draw, so the row id it is drawn on matters
K8_CASES = _cases("k8")


def _k8_members(form, ks2, logp, i, rng):
    """(n_rows, member row lists, swap, seat, rows map, range, offsets) of the case: grouped members of 0, 1 and 17 rows,
    64 members at KS2 2, and one large case per template."""
    n = SIZES[i % len(SIZES)]
    if form in ("grouped", "grouped_joint"):
        if (ks2, form, logp) == (2, "grouped", 0):
            sizes = rng.randint(0, 40, size=64)
            sizes[[3, 10, 40]] = (0, 1, 17)
        elif (ks2, form, logp) == (6, "grouped", 1):
            sizes = np.array([17, 0, 1, 20000, 15003])
        else:
            sizes = np.array([17, 0, 1, n])[np.roll(np.arange(4), i)]
        start = i % 3
        offsets = start + np.concatenate([[0], np.cumsum(sizes)])
        n_rows = int(offsets[-1]) + 2  # rows before the first member and after the last belong to none
        return n_rows, [np.arange(offsets[k], offsets[k + 1]) for k in range(len(sizes))], None, 0, None, None, offsets.astype(np.int32)
    if form == "rows" and ks2 == 7 and logp:
        n = 34011  # some warps of the 132 x 16 walk three tiles
    swap, seat = _swap(rng, n, i), i % 2
    if form in ("identity", "view"):
        return n, [np.arange(n)], swap, seat, None, None, None
    lo, hi = _range(n, i)
    rows = rng.permutation(2 * n)[:n] if form == "joint" else rng.permutation(n)
    return n, [np.arange(lo, min(hi, n))], swap, seat, rows.astype(np.int32), np.array([lo, hi], np.int32), None


def _k8_case(form, ks2, logp):
    """The operands and the float64 restatement of a K8 case.  Each member's heads layer is scaled by a power of two
    (exact) so that its heads lie in [-HEAD_MAX, HEAD_MAX]."""
    c = dict(form=form, ks2=ks2, logp=logp)
    i = c["i"] = K8_CASES.index((form, ks2, logp))
    k0 = c["k0"] = 32 * ks2
    n_hidden = c["n_hidden"] = (0, 2, 8)[i % 3]
    c["n_actions"] = 2 + i % 6
    c["in_slope"], c["slope"] = SLOPES[i % 4]
    rng = np.random.RandomState(1000 + i)
    n, members, c["swap"], c["seat"], rows, c["range"], c["offsets"] = _k8_members(form, ks2, logp, i, rng)
    x = np.full((n, k0), np.nan)
    heads = np.full((n, 8), np.nan)
    ops = []
    for R in members:
        w = P.k8_operands(rng, 1, k0, n_hidden)[1:]
        if len(R):
            x[R], heads[R], certs = P.certified_rows(rng, P.k8_rows(rng, len(R), k0), lambda r, m: P.k8_rows(r, m, k0),
                                                     lambda x, w=w: P.k8_reference(x, *w, c["in_slope"], c["slope"]))
            assert all(cert.holds() for cert in certs), "premise"
            scale = 2.0 ** -max(0, int(np.ceil(np.log2(np.abs(heads[R]).max() / HEAD_MAX))))
            w = w[:4] + (w[4] * scale, w[5] * scale)
            heads[R] *= scale
        ops.append(w)
    R = np.concatenate(members).astype(np.int64)
    # the output index o of each row, the joint row d it is drawn on (which indexes actions), and the buffers' sizes
    o = R if rows is None or form == "rows" else rows[R].astype(np.int64)
    if form == "view":
        d = 2 * R + _player(c["seat"], c["swap"], R)
    elif form == "rows":
        d = 2 * rows[R].astype(np.int64) + _player(c["seat"], c["swap"], rows[R])
    else:
        d = o
    if form == "grouped_joint":
        rows = rng.permutation(2 * n)[:n].astype(np.int32)
        o = d = rows[R].astype(np.int64)
    c["n_out"] = 2 * n if form in ("joint", "grouped_joint") else n
    c["n_act"] = 2 * n if form in ("view", "rows", "joint", "grouped_joint") else n
    c.update(n=n, members=members, rows=rows, x=x, heads=heads, ops=ops, R=R, o=o, d=d, seed=0xF0F0 + 7919 * i,
             step0=2 ** 32 - 1 if i % 5 == 0 else i)
    return c


@pytest.mark.parametrize("form,ks2,logp", K8_CASES, ids=["%s-k0_%d-%s" % (f, 32 * k, "logp" if l else "plain") for f, k, l in K8_CASES])
@pytest.mark.gpu
def test_k8_form_exact(form, ks2, logp):
    """Two launches over the case's rows (at least 8, at least two actions, the draw on them depending on the row id);
    the Rows and Joint forms also launch once over an empty range, which writes nothing and still advances the counter."""
    c = _k8_case(form, ks2, logp)
    n, k0, n_hidden, n_actions, heads, ops, seed, step0 = (c[k] for k in ("n", "k0", "n_hidden", "n_actions", "heads", "ops", "seed", "step0"))
    assert len(c["R"]) >= 8 and n_actions >= 2
    nh = max(n_hidden, 1)
    dw = (_dev(np.stack([w[0] for w in ops]), torch.bfloat16), _dev(np.stack([w[1] for w in ops]), torch.float32),
          _dev(np.stack([w[2] if n_hidden else np.zeros((nh, 64, 64)) for w in ops]), torch.bfloat16),
          _dev(np.stack([w[3] if n_hidden else np.zeros((nh, 64)) for w in ops]), torch.float32),
          _dev(np.stack([w[4] for w in ops]), torch.bfloat16), _dev(np.stack([w[5] for w in ops]), torch.float32))
    tx = _full(n, torch.bfloat16, float("nan"), (k0,))
    tx[:n] = _dev(c["x"], torch.bfloat16)
    tswap, trows, toff = (None if a is None else _dev(a, torch.int32) for a in (c["swap"], c["rows"], c["offsets"]))
    ranged = form in ("rows", "joint")
    trange = _dev(c["range"], torch.int32) if ranged else None
    empty = _dev(np.array([n // 2, n // 2], np.int32), torch.int32) if ranged else None
    counter = torch.tensor([step0, 0], dtype=torch.int64, device="cuda")
    lib = _native.lib()
    for launch in range(3 if ranged else 2):
        R, o, d = (c[k][:0] if launch == 2 else c[k] for k in ("R", "o", "d"))
        rg = empty if launch == 2 else trange
        acts, vals = _full(c["n_act"], torch.int32, -7), _full(c["n_out"], torch.float32, float("nan"))
        sc, lp = _full(c["n_out"], torch.float32, float("nan"), (8,)), _full(c["n_out"], torch.float32, float("nan"))
        args = (tx.data_ptr(), n, k0, c["in_slope"], *(t.data_ptr() for t in dw[:4]), n_hidden, dw[4].data_ptr(), dw[5].data_ptr(), c["slope"],
                n_actions, seed, counter.data_ptr())
        outs = (acts.data_ptr(), vals.data_ptr(), sc.data_ptr(), lp.data_ptr() if logp else 0, None)
        if form == "identity":
            rc = lib.ovc_policy_tail_logp(*args, *outs) if logp else lib.ovc_policy_tail(*args, *outs[:3], None)
        elif form == "view":
            rc = lib.ovc_policy_tail_view(*args, _ptr(tswap), c["seat"], *outs)
        elif form == "rows":
            rc = lib.ovc_policy_tail_rows(*args, _ptr(tswap), c["seat"], trows.data_ptr(), rg.data_ptr(), *outs)
        elif form == "joint":
            rc = lib.ovc_policy_tail_joint(*args, trows.data_ptr(), rg.data_ptr(), *outs)
        elif form == "grouped":
            rc = lib.ovc_policy_tail_grouped(*args, toff.data_ptr(), len(c["members"]), *outs)
        else:
            rc = lib.ovc_policy_tail_grouped_joint(*args, trows.data_ptr(), toff.data_ptr(), len(c["members"]), *outs)
        _native.check(rc)
        a, v, s, l = _np(acts), _np(vals), _np(sc), _np(lp)
        assert np.array_equal(s[o], heads[R]), ((s[o] != heads[R]).sum(), form, ks2)
        assert np.array_equal(v[o], heads[R, n_actions])
        if len(R):
            P.check_draw(a[d], heads[R], seed, step0 + launch, n_actions, rows=d, row_sensitive=True)
            if logp:
                P.check_logp(l[o], heads[R], a[d], n_actions)
        assert _untouched(a, d, -7) and _untouched(v, o, float("nan")) and _untouched(s, o, float("nan"))
        assert _untouched(l, o if logp else [], float("nan"))
        assert _np(counter).tolist() == [step0 + launch + 1, 0]


# ------------------------------------------------------------------------------------------------------------------ K7
_ENVS = {}


def _k7_env(kind):
    """(env, float64 encoding [N, 2, W*H*26]) after random play: 1 or 8 layouts of the 5x4 shape, or 13x7."""
    if kind not in _ENVS:
        from overcooked_ai_b200 import layout as L

        if kind == "13x7":
            names, n = ["long_cook_time"], 150
        else:
            names = []
            for name in L.layout_names():
                try:
                    l = L.compile_layout(name)
                except ValueError:
                    continue
                if (l.width, l.height) == (5, 4):
                    names.append(name)
            names, n = names[:kind], (301 if kind == 1 else 8 * 37 + 3)
        env = BatchedOvercookedEnv(names, n, horizon=50, auto_reset=True, random_start_pos=True, rnd_obj_prob_thresh=0.5, seed=n)
        rng = np.random.RandomState(n)
        acts = rng.randint(0, 6, size=(14, n, 2)).astype(np.int32)
        acts[rng.rand(14, n, 2) < 0.3] = 5
        env.rollout(torch.from_numpy(acts).cuda())
        assert len(np.unique(env.env_layout_host)) == len(names)
        l = env.layouts[0]
        obs = cpu.encode_lossless(env._tab_host, _np(env.state), l.width, l.height, env.horizon).astype(np.float64)
        _ENVS[kind] = env, obs.reshape(n, 2, -1)
    return _ENVS[kind]


def _k7_variants(form, rng, n):
    """[(call arguments, output rows, expected (member, env, view) per written row)] of the form's map."""
    e = np.arange(n)
    out = []
    if form == "two_view":
        for swap in (None, rng.randint(0, 3, size=n).astype(np.int32)):
            p = _player(0, swap, e)
            out.append((dict(swap=swap), 2 * n, np.concatenate([2 * e + p, 2 * e + 1 - p]), 0, np.concatenate([e, e]),
                        np.concatenate([np.zeros(n, np.int64), np.ones(n, np.int64)])))
    elif form == "view":
        for seat, swap in ((0, None), (1, None), (0, rng.randint(0, 2, size=n).astype(np.int32)), (1, rng.randint(0, 2, size=n).astype(np.int32))):
            out.append((dict(swap=swap, seat=seat), n, e, 0, e, _player(seat, swap, e)))
    elif form == "rows":
        for seat, lo, hi in ((0, 37, n - 5), (1, 1, n + 9), (1, n // 3, n // 3)):
            swap, rows = rng.randint(0, 2, size=n).astype(np.int32), rng.permutation(n).astype(np.int32)
            r = np.arange(lo, min(hi, n))
            out.append((dict(swap=swap, seat=seat, rows=rows, range=np.array([lo, hi], np.int32)), n, r, 0, rows[r], _player(seat, swap, rows[r])))
    else:
        grouped_offsets = np.array([0, 5, 5, n - 40, n - 3], np.int32)  # uneven, an empty member, the last 3 in none
        if form == "grouped":
            k = np.repeat(np.arange(4), np.diff(grouped_offsets))
            m = np.arange(grouped_offsets[-1])
            out.append((dict(offsets=grouped_offsets), 2 * n, np.concatenate([2 * m, 2 * m + 1]), np.concatenate([k, k]),
                        np.concatenate([m, m]), np.concatenate([np.zeros(len(m), np.int64), np.ones(len(m), np.int64)])))
        else:
            env, vmask = rng.permutation(n), rng.randint(0, 4, size=n)
            vmask[:4] = (0, 1, 2, 3)
            cnt = (vmask & 1) + (vmask >> 1)
            first = np.concatenate([[0], np.cumsum(cnt)[:-1]]).astype(np.int32)
            lst = (env << 2 | vmask).astype(np.int32)
            k = np.repeat(np.arange(4), np.diff(grouped_offsets)) if form == "grouped_masked" else np.zeros(n, np.int64)
            listed = np.arange(grouped_offsets[-1] if form == "grouped_masked" else n)
            rows_, mem, envs, views = [], [], [], []
            for r in listed:
                j = first[r]
                for v in (0, 1):
                    if vmask[r] >> v & 1:
                        rows_.append(j), mem.append(k[r]), envs.append(env[r]), views.append(v)
                        j += 1
            kw = dict(list=lst, first=first)
            if form == "grouped_masked":
                kw["offsets"] = grouped_offsets
            out.append((kw, int(cnt.sum()), np.array(rows_), np.array(mem), np.array(envs), np.array(views)))
    return out


K7_CASES = _cases("k7")


@pytest.mark.parametrize("form,cpl", K7_CASES, ids=["%s-cpl%d" % c for c in K7_CASES])
@pytest.mark.gpu
def test_k7_form_exact(form, cpl):
    """One layout and eight per call on 5x4 grids (and 13x7 at CPL 2); two-view with and without view_swap, both seats,
    rows with a non-zero range start (and an empty range), list entries of every view mask, uneven member offsets with an
    empty member."""
    lib = _native.lib()
    i = K7_CASES.index((form, cpl))
    grouped = form.startswith("grouped")
    computed = 0
    for kind in (1, 8) + (("13x7",) if cpl == 2 else ()):
        env, obs = _k7_env(kind)
        n, W, H = env.n_envs, env.layouts[0].width, env.layouts[0].height
        n_out = K7_NOUT[cpl] if kind != "13x7" else 64
        slope = SLOPES[i % 4][1]
        rng = np.random.RandomState(i)
        tables = [P.k7_operands(rng, obs.shape[2], n_out) for _ in range(4 if grouped else 1)]
        want = []
        for wt, b in tables:
            z, certs = P.k7_reference(obs.reshape(2 * n, -1), wt, b, slope)
            assert certs[0].holds(), "premise"
            want.append(z.reshape(n, 2, n_out))
        wt = _dev(np.stack([t[0] for t in tables]), torch.bfloat16)
        bias = _dev(np.stack([t[1] for t in tables]), torch.float32)
        hz = env.horizon if env.horizon > 0 else 2 ** 31 - 1
        for kw, n_rows, idx, mem, envs, views in _k7_variants(form, rng, n):
            t = {k: _dev(v, torch.int32) for k, v in kw.items() if isinstance(v, np.ndarray)}
            out = _full(n_rows, torch.bfloat16, float("nan"), (n_out,))
            head = (env.tables.data_ptr(), env.n_layouts, env.state.data_ptr())
            tail = (env.state_words, W, H, hz, n_out, slope, None)
            if form == "two_view":
                rc = lib.ovc_encode_linear(*head, _ptr(t.get("swap")), wt.data_ptr(), bias.data_ptr(), out.data_ptr(), n, *tail)
            elif form == "view":
                rc = lib.ovc_encode_linear_view(*head, _ptr(t.get("swap")), kw["seat"], wt.data_ptr(), bias.data_ptr(), out.data_ptr(), n, *tail)
            elif form == "rows":
                rc = lib.ovc_encode_linear_rows(*head, t["swap"].data_ptr(), kw["seat"], t["rows"].data_ptr(), t["range"].data_ptr(),
                                                wt.data_ptr(), bias.data_ptr(), out.data_ptr(), n, *tail)
            elif form == "masked":
                rc = lib.ovc_encode_linear_masked(*head, t["list"].data_ptr(), t["first"].data_ptr(), wt.data_ptr(), bias.data_ptr(),
                                                  out.data_ptr(), n, *tail)
            elif form == "grouped":
                rc = lib.ovc_encode_linear_grouped(*head, wt.data_ptr(), bias.data_ptr(), t["offsets"].data_ptr(), 4, out.data_ptr(), n, *tail)
            else:
                rc = lib.ovc_encode_linear_grouped_masked(*head, t["list"].data_ptr(), t["first"].data_ptr(), wt.data_ptr(), bias.data_ptr(),
                                                          t["offsets"].data_ptr(), 4, out.data_ptr(), n, *tail)
            _native.check(rc)
            got = _np(out.float()).astype(np.float64)
            expect = np.stack([want[k][e, v] for k, e, v in zip(np.broadcast_to(mem, idx.shape), envs, views)]) if len(idx) else np.zeros((0, n_out))
            assert np.array_equal(got[idx], expect), (kind, kw.keys(), (got[idx] != expect).sum())
            assert _untouched(got, idx, float("nan")), (kind, kw.keys())
            computed += len(idx)
    assert computed > 0


# ------------------------------------------------------------------------------------------------------------ the draw
DRAW_CASES = _cases("draw")


@pytest.mark.parametrize("form,logp", DRAW_CASES, ids=["%s-%s" % (f, "logp" if l else "plain") for f, l in DRAW_CASES])
@pytest.mark.gpu
def test_draw_form_exact(form, logp):
    """ovc_sample_actions_view / _rows: the action of row r at its joint row, from the Philox counter of that row id; the
    other seat, rows outside the range and everything past the end untouched; one large launch; the Rows form also
    launches once over an empty range."""
    lib = _native.lib()
    i = DRAW_CASES.index((form, logp))
    for n, n_actions in ((1, 3), (257, 8), (3001, 5), (100003, 7)):
        rng = np.random.RandomState(n + i)
        scores = rng.normal(size=(n, 8)).astype(np.float32).astype(np.float64) * 2
        swap, seat = _swap(rng, n, i + n), (i + n) % 2
        r = np.arange(n)
        rows, rng_ = None, None
        if form == "rows":
            rows = rng.permutation(n).astype(np.int32)
            lo, hi = _range(n, i + n)
            r = np.arange(lo, min(hi, n))
            rng_ = np.array([lo, hi], np.int32)
            d = 2 * rows[r].astype(np.int64) + _player(seat, swap, rows[r])
        else:
            d = 2 * r + _player(seat, swap, r)
        tsc = _dev(scores, torch.float32)
        tswap, trows, trange = (None if a is None else _dev(a, torch.int32) for a in (swap, rows, rng_))
        step0 = 2 ** 32 - 1 if n == 257 else n
        counter = torch.tensor([step0, 0], dtype=torch.int64, device="cuda")
        assert len(r) > 0
        empty = _dev(np.array([n // 2, n // 2], np.int32), torch.int32)
        for launch in range(3 if form == "rows" else 2):
            if launch == 2:
                r, d, trange = r[:0], d[:0], empty
            acts, lp = _full(2 * n, torch.int32, -7), _full(n, torch.float32, float("nan"))
            lpp = lp.data_ptr() if logp else 0
            if form == "view":
                rc = lib.ovc_sample_actions_view(tsc.data_ptr(), 8, n_actions, n, 99, counter.data_ptr(), _ptr(tswap), seat, acts.data_ptr(), lpp, None)
            else:
                rc = lib.ovc_sample_actions_rows(tsc.data_ptr(), 8, n_actions, n, 99, counter.data_ptr(), _ptr(tswap), seat, trows.data_ptr(),
                                                 trange.data_ptr(), acts.data_ptr(), lpp, None)
            _native.check(rc)
            a, l = _np(acts), _np(lp)
            if len(r):
                P.check_draw(a[d], scores[r], 99, step0 + launch, n_actions, rows=d, row_sensitive=len(r) >= 16)
                if logp:
                    P.check_logp(l[r], scores[r], a[d], n_actions)
            assert _untouched(a, d, -7) and _untouched(l, r if logp else [], float("nan"))
            assert _np(counter).tolist() == [step0 + launch + 1, 0]


# ------------------------------------------------------------------------------------------------------------------ K9
K9_CASES = _cases("k9")


def _k9_run(lib, form, a0, m, ops, slope, sel, n_members=1):
    """K9 over a0 (rows outside the map NaN) into a guarded z2; returns the whole z2 allocation."""
    w1, b1, w2, b2 = ops
    ta0 = _full(m, torch.bfloat16, float("nan"), (512,))
    ta0[:m] = _dev(a0, torch.bfloat16)
    z2 = _full(m, torch.bfloat16, float("nan"), (160,))
    tsel = _dev(sel, torch.int32)
    args = (ta0.data_ptr(), m, 512, w1.data_ptr(), b1.data_ptr(), 512, w2.data_ptr(), b2.data_ptr(), 160, slope)
    if form == "range":
        _native.check(lib.ovc_wide_layers_range(*args, tsel.data_ptr(), z2.data_ptr(), None))
    else:
        _native.check(lib.ovc_wide_layers_grouped(*args, tsel.data_ptr(), n_members, z2.data_ptr(), None))
    return _np(z2.float()).astype(np.float64)


@pytest.mark.parametrize("form", [c[0] for c in K9_CASES])
@pytest.mark.gpu
def test_k9_form_exact(form):
    """ovc_wide_layers_range at starts that are not 128-row aligned, tile edges +- 1, an empty range and one past m;
    ovc_wide_layers_grouped over uneven members (0, 1, 127 - 129 rows) from an unaligned start, each with its own weights;
    one large launch each (persistent CTAs walk two tiles)."""
    lib = _native.lib()
    rng = np.random.RandomState(9 if form == "range" else 10)
    if form == "range":
        _, w1, b1, w2, b2 = P.k9_operands(rng, 1)
        ops = tuple(_dev(v, dt) for v, dt in ((w1, torch.bfloat16), (b1, torch.float32), (w2, torch.bfloat16), (b2, torch.float32)))
        layouts = [(1000, lo, hi, 0.25) for lo, hi in ((5, 132), (5, 133), (5, 134), (128, 256), (300, 300), (7, 1000), (990, 1100), (0, 1))]
        layouts.append((132 * 128 + 77, 3, 132 * 128 + 72, 1.0))
        for m, lo, hi, slope in layouts:
            r = np.arange(lo, min(hi, m))
            a0 = np.full((m, 512), np.nan)
            want = np.zeros((len(r), 160))
            if len(r):
                a0[r], want, certs = P.certified_rows(rng, P.k9_rows(rng, len(r)), P.k9_rows, lambda x: P.k9_reference(x, w1, b1, w2, b2, slope))
                assert all(c.holds() for c in certs), "premise"
            got = _k9_run(lib, form, a0, m, ops, slope, np.array([lo, hi], np.int32))
            assert np.array_equal(got[r], want), (m, lo, hi, (got[r] != want).sum())
            assert _untouched(got, r, float("nan")), (m, lo, hi)
        return
    for sizes, slope in (([127, 0, 129, 1, 128, 300], 0.5), ([16000, 1, 0, 129], 0.0)):
        offsets = 5 + np.concatenate([[0], np.cumsum(sizes)]).astype(np.int32)
        m = int(offsets[-1]) + 3
        a0 = np.full((m, 512), np.nan)
        want = np.full((m, 160), np.nan)
        ops = []
        for k in range(len(sizes)):
            _, w1, b1, w2, b2 = P.k9_operands(rng, 1)
            ops.append((w1, b1, w2, b2))
            r = np.arange(offsets[k], offsets[k + 1])
            if len(r):
                a0[r], want[r], certs = P.certified_rows(rng, P.k9_rows(rng, len(r)), P.k9_rows,
                                                         lambda x, w=ops[-1]: P.k9_reference(x, *w, slope))
                assert all(c.holds() for c in certs), "premise"
        dops = (_dev(np.concatenate([o[0] for o in ops]), torch.bfloat16), _dev(np.stack([o[1] for o in ops]), torch.float32),
                _dev(np.concatenate([o[2] for o in ops]), torch.bfloat16), _dev(np.stack([o[3] for o in ops]), torch.float32))
        got = _k9_run(lib, form, a0, m, dops, slope, offsets, len(sizes))
        r = np.arange(offsets[0], offsets[-1])
        assert np.array_equal(got[r], want[r]), (sizes, (got[r] != want[r]).sum())
        assert _untouched(got, r, float("nan")), sizes
