"""numpy restatements of the sample-batch kernels (include/ovc_b200.h: ovc_gae, ovc_record_transition, the logp outputs),
shared by the CPU and GPU tests."""
import numpy as np


def gae_f32(rewards, values, dones, last_values, gamma, lam):
    """ovc_gae in float32, every operation rounded on its own in the documented order.  rewards / values [T, 2N],
    dones [T, N] (terminal), last_values [2N] -> (advantages, value_targets) [T, 2N]."""
    f = np.float32
    r, v = np.asarray(rewards, f), np.asarray(values, f)
    nt = (1 - (np.asarray(dones) != 0)).astype(f).repeat(2, axis=1)
    g, gl = f(gamma), f(f(gamma) * f(lam))
    T = r.shape[0]
    adv = np.zeros_like(r)
    a = np.zeros(r.shape[1], f)
    nv = np.asarray(last_values, f)
    for t in range(T - 1, -1, -1):
        delta = (r[t] + (g * nv) * nt[t]) - v[t]
        a = delta + (gl * nt[t]) * a
        adv[t] = a
        nv = v[t]
    return adv, adv + v


def gae_horizon_f32(r, v, d, tv, last, gamma, lam):
    """include/ovc_horizon.h's recurrence in numpy float32 (every operation rounded on its own): r, v, tv [T, R], d [T, R]
    or [T, R / 2] (one flag per environment of two rows), last [R]."""
    T, R = r.shape
    dd = np.repeat(d, R // d.shape[1], axis=1) != 0
    g, gl = np.float32(gamma), np.float32(np.float32(gamma) * np.float32(lam))
    A, nv = np.zeros(R, np.float32), last.astype(np.float32)
    adv, tgt = np.empty_like(r), np.empty_like(r)
    for t in reversed(range(T)):
        nxt = np.where(dd[t], tv[t], nv).astype(np.float32)
        delta = (r[t] + g * nxt) - v[t]
        A = delta + (gl * np.where(dd[t], np.float32(0), np.float32(1))) * A
        adv[t], tgt[t], nv = A, A + v[t], v[t]
    return adv, tgt


def gae_f64(rewards, values, dones, last_values, gamma, lam):
    """The same recurrence in float64."""
    r, v = np.asarray(rewards, np.float64), np.asarray(values, np.float64)
    nt = 1.0 - (np.asarray(dones) != 0).repeat(2, axis=1)
    adv = np.zeros_like(r)
    a = np.zeros(r.shape[1])
    nv = np.asarray(last_values, np.float64)
    for t in range(r.shape[0] - 1, -1, -1):
        a = r[t] + gamma * nv * nt[t] - v[t] + gamma * lam * nt[t] * a
        adv[t] = a
        nv = v[t]
    return adv, adv + v


def log_softmax_at(scores, actions, n_actions):
    """float64 log-softmax of scores[:, :n_actions] at the given actions."""
    s = np.asarray(scores, np.float64)[:, :n_actions]
    m = s.max(1, keepdims=True)
    lse = m[:, 0] + np.log(np.exp(s - m).sum(1))
    return s[np.arange(len(s)), np.asarray(actions)] - lse
