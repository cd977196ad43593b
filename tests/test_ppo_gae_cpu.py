"""The GAE restatement the GPU tests hold ovc_gae to, checked against an independent formulation: RLlib's per-episode
postprocessing (compute_advantages: discounted cumulative sums by scipy.signal.lfilter, bootstrapped with the last value
only where the window cuts an episode)."""
import numpy as np
import pytest
from scipy.signal import lfilter

from ppo_reference import gae_f32, gae_f64


def _discount_cumsum(x, gamma):
    return lfilter([1], [1, -gamma], x[::-1])[::-1]


def _gae_per_episode(rewards, values, dones, last_values, gamma, lam):
    T, R = rewards.shape
    adv = np.zeros((T, R))
    for r in range(R):
        d = dones[:, r // 2] != 0
        start = 0
        for end in list(np.nonzero(d)[0] + 1) + [T]:
            if end <= start:
                continue
            rw, vp = rewards[start:end, r].astype(np.float64), values[start:end, r].astype(np.float64)
            boot = 0.0 if d[end - 1] else float(last_values[r])  # terminal: no bootstrap
            vn = np.append(vp[1:], boot)
            adv[start:end, r] = _discount_cumsum(rw + gamma * vn - vp, gamma * lam)
            start = end
    return adv, adv + values


@pytest.mark.parametrize("T,R", [(1, 2), (7, 6), (60, 40)])
@pytest.mark.parametrize("gamma,lam", [(0.99, 0.95), (0.99, 1.0), (0.0, 0.95)])
def test_gae_restatement_matches_per_episode_discounted_cumsum(T, R, gamma, lam):
    rng = np.random.RandomState(T * 100 + R)
    rewards = rng.normal(size=(T, R)).astype(np.float32)
    values = rng.normal(size=(T, R)).astype(np.float32)
    last = rng.normal(size=R).astype(np.float32)
    dones = (rng.rand(T, R // 2) < 0.15).astype(np.uint8)
    dones[0, 0] = 1
    dones[-1, -1] = 1
    want_adv, want_tgt = _gae_per_episode(rewards, values, dones, last, gamma, lam)
    adv, tgt = gae_f32(rewards, values, dones, last, gamma, lam)
    assert adv.dtype == np.float32 and tgt.dtype == np.float32
    tol = 1e-5 * (1 + np.abs(want_adv))
    assert (np.abs(adv - want_adv) <= tol).all() and (np.abs(tgt - want_tgt) <= tol + 1e-5 * np.abs(values)).all()
    adv64, tgt64 = gae_f64(rewards, values, dones, last, gamma, lam)
    assert np.allclose(adv64, want_adv, rtol=1e-12, atol=1e-12) and np.allclose(tgt64, want_tgt, rtol=1e-12, atol=1e-12)
