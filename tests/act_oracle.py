"""NumPy restatement of DDPG.act's exploration (DESIGN.md §3 "Exploration"): the Philox draws, the Box-Muller z in fp64,
the Gaussian and Ornstein-Uhlenbeck noise in the reference's operation order (random_process.py), and the fp64 clip."""
import numpy as np

from tests.helpers import philox_uniform53

COUNTER_BASE = 1 << 63          # exploring act() call k draws with counter 2^63 + k


def standard_normal(seed, k, n):
    """z of draw indices 0..n-1 of exploring call k: z = sqrt(-2 log(1 - u1)) * cos(2 pi u2),
    u1 / u2 = uniform53(seed, 2^63 + k, 2i / 2i + 1)."""
    ctr = COUNTER_BASE + k
    u1 = np.array([philox_uniform53(seed, ctr, 2 * i) for i in range(n)], dtype=np.float64)
    u2 = np.array([philox_uniform53(seed, ctr, 2 * i + 1) for i in range(n)], dtype=np.float64)
    return np.sqrt(-2.0 * np.log(1.0 - u1)) * np.cos(2.0 * np.pi * u2)


def gaussian_noise(z, eps, mu, var):
    """GaussianNoise.sample(): eps * np.random.normal(mu, var) = eps * (mu + var * z)."""
    return eps * (mu + var * z)


def ou_step(x, z, theta, mu, sigma, dt, reset=None):
    """OrnsteinUhlenbeckProcess: rows with reset start from 0 (reset()), then sample()'s update.  Returns the new x."""
    x = np.array(x, dtype=np.float64, copy=True)
    if reset is not None:
        x[np.asarray(reset, dtype=bool)] = 0.0
    return x + theta * (mu - x) * dt + sigma * np.sqrt(dt) * z


def action(a, n):
    """np.clip(action + noise, -1, 1) in fp64, rounded once to fp32."""
    return np.clip(np.asarray(a, dtype=np.float32).astype(np.float64) + n, -1.0, 1.0).astype(np.float32)


def check_actions(got, want, min_equal=0.99):
    """Every action within 1 fp32 ulp of the oracle, at least `min_equal` of them bit-equal.  The only allowed
    difference is the device's fp64 log / cos against the host libm (like the tree-leaf rule of tests/helpers.py)."""
    got, want = np.asarray(got, np.float32), np.asarray(want, np.float32)
    assert got.shape == want.shape, (got.shape, want.shape)
    ulp = np.spacing(np.abs(want))
    err = np.abs(got.astype(np.float64) - want.astype(np.float64))
    assert (err <= ulp).all(), "max error %.3e ulp" % float((err / ulp).max())
    eq = float((got == want).mean())
    assert eq >= min_equal, "only %.4f of the actions are bit-equal" % eq
    return eq
