"""CPU-only checks of the streaming n-step insert (add_steps): the oracle against a hand-worked stream, the host mirror's
row counts against the oracle over random end patterns, argument validation before any device work, and the ctypes
prototypes and C-side argument checks."""
import ctypes as C

import numpy as np
import pytest

from oracle import d4pg_oracle as O
from tests import nstep_stream_oracle as SO


def test_oracle_hand_worked_stream():
    """E = 2, n = 2, gamma = 0.5.  Env 0: an episode of 3 steps ending in a termination, then 1 step.  Env 1: a
    truncation after 1 step (a window that never fills), then 3 steps."""
    S, A = 1, 1
    term = [[0, 0], [0, 0], [1, 0], [0, 0]]
    trunc = [[0, 1], [0, 0], [0, 0], [0, 0]]
    calls = []
    for k in range(4):
        obs = np.array([[10 * k], [100 + 10 * k]], np.float32)
        calls.append((obs, obs.copy() + 1, np.array([k + 1.0, -(k + 1.0)]), obs + 5, np.array(term[k], bool),
                      np.array(trunc[k], bool)))
    rows = SO.stream_rows(calls, 2, 0.5)
    got = [(k, e, float(r[0][0]), float(r[2]), float(r[3][0]), bool(r[4])) for k, e, r in rows]
    assert got == [(1, 0, 0.0, 1.0 + 0.5 * 2.0, 15.0, False),
                   (2, 0, 10.0, 2.0 + 0.5 * 3.0, 25.0, True),
                   (2, 1, 110.0, -2.0 - 0.5 * 3.0, 125.0, False),
                   (3, 1, 120.0, -3.0 - 0.5 * 4.0, 135.0, False)]
    assert float(rows[0][2][1][0]) == 1.0          # the window's oldest action (replay_memory.py:44)
    assert SO.rows_per_call(np.array(term, bool) | np.array(trunc, bool), 2) == [0, 1, 2, 1]


def test_oracle_single_environment_equals_episodes():
    """With E = 1 the stream is the episodes one after the other: the rows are O.nstep_transitions of each."""
    rng = np.random.RandomState(3)
    calls = SO.random_calls(rng, 60, 1, 3, 2, 3)
    rows = [r for _, _, r in SO.stream_rows(calls, 3, 0.9)]
    want, ep = [], []
    for k, c in enumerate(calls):
        ep.append(c)
        if c[4][0] or c[5][0] or k == len(calls) - 1:
            want += O.nstep_transitions([x[0][0] for x in ep], [x[1][0] for x in ep], [float(x[2][0]) for x in ep],
                                        [x[3][0] for x in ep], [bool(x[4][0]) for x in ep], 3, 0.9)
            ep = []
    assert len(rows) == len(want) > 0
    for r, w in zip(rows, want):
        assert all(np.array_equal(np.asarray(x), np.asarray(y)) for x, y in zip(r, w))


@pytest.mark.parametrize("n_steps", [1, 2, 5, 7])
@pytest.mark.parametrize("E", [1, 31, 33])
def test_host_mirror_counts_vs_oracle(n_steps, E):
    from d4pg_b200.prioritized_replay_memory import StepsMirror
    rng = np.random.RandomState(n_steps * 1000 + E)
    K = 120
    term, trunc = SO.random_ends(rng, K, E, n_steps)
    want = SO.rows_per_call(term | trunc, n_steps)
    calls = [(np.zeros((E, 1), np.float32), np.zeros((E, 1), np.float32), np.zeros(E), np.zeros((E, 1), np.float32),
              term[k], trunc[k]) for k in range(K)]
    per_call = np.bincount([k for k, _, _ in SO.stream_rows(calls, n_steps, 0.9)], minlength=K).tolist()
    assert per_call == want
    m = StepsMirror(E, n_steps, 0.9)
    got, late = [], None
    for k in range(K):
        if late is not None:                          # CUDA flags: applied at the start of the next call
            m.end(late)
            late = None
        got.append(m.rows())
        m.advance()
        if k % 3:                                     # host flags: applied right away
            m.end(term[k] | trunc[k])
        else:
            late = term[k] | trunc[k]
    assert got == want
    assert sum(want) > 0 or n_steps > 1


def _buf(size=16, **kw):
    import d4pg_b200 as d4pg
    return d4pg.ReplayBuffer(size, **kw)


def _args(E=4, S=3, A=2):
    return (np.zeros((E, S), np.float32), np.zeros((E, A), np.float32), np.zeros(E), np.zeros((E, S), np.float32),
            np.zeros(E, bool))


def test_add_steps_validation_before_device_work():
    from d4pg_b200.prioritized_replay_memory import StepsMirror
    b = _buf(16)
    s, a, r, s2, d = _args()
    for n in (0, 65, 2.5, True, -1):
        with pytest.raises(ValueError, match="n_steps"):
            b.add_steps(s, a, r, s2, d, n_steps=n)
    with pytest.raises(ValueError, match="exceed"):
        b.add_steps(*_args(E=17), n_steps=2)
    bad = [(s[:, :2], a, r, s2, d), (s, a[:3], r, s2, d), (s, a, r[:3], s2, d), (s, a, r, s2[:, :2], d),
           (s, a, r, s2, d[:3]), (s[0], a, r, s2, d), (s, a, r.reshape(4, 1), s2, d)]
    for args in bad:
        with pytest.raises(ValueError, match="shape|must be"):
            b.add_steps(*args, n_steps=2)
    with pytest.raises(ValueError, match="shape"):
        b.add_steps(s, a, r, s2, d, truncated=np.zeros(5, bool), n_steps=2)
    # the fixed (E, n_steps, gamma) of pending windows
    b._store._steps = StepsMirror(4, 3, 0.9)
    for kw in (dict(n_steps=2, gamma=0.9), dict(n_steps=3, gamma=0.99)):
        with pytest.raises(ValueError, match="drop_steps"):
            b.add_steps(s, a, r, s2, d, **kw)
    with pytest.raises(ValueError, match="drop_steps"):
        b.add_steps(*_args(E=5), n_steps=3, gamma=0.9)
    b.drop_steps()
    assert b._store._steps is None
    assert len(b) == 0


def test_add_steps_dims_must_match_the_buffer():
    import d4pg_b200 as d4pg
    b = d4pg.PrioritizedReplayBuffer(16, 0.6, obs_dim=5, act_dim=2)
    with pytest.raises(ValueError, match="rows of"):
        b.add_steps(*_args(), n_steps=1)
    rp = d4pg.Replay(16, None, n_steps=3, gamma=0.9, obs_dim=3, act_dim=2)
    with pytest.raises(ValueError, match="Replay"):
        rp.add_steps(*_args(), n_steps=2)
    with pytest.raises(ValueError, match="Replay"):
        rp.add_steps(*_args(), gamma=0.99)
    rp.drop_steps()


def test_observe_validates_before_device_work():
    import d4pg_b200 as d4pg
    dd = d4pg.DDPG(3, 2, memory_size=8, batch_size=4, n_steps=5,
                   critic_dist_info={"type": "categorical", "v_min": -1.0, "v_max": 0.0, "n_atoms": 11})
    with pytest.raises(ValueError, match="exceed"):
        dd.observe(*_args(E=9))
    with pytest.raises(ValueError, match="shape"):
        dd.observe(*_args()[:4], np.zeros(3, bool))


def test_prototypes_and_c_validation():
    from d4pg_b200 import _lib
    L = _lib.lib()
    P = C.c_void_p
    assert L.d4pg_replay_steps_window_bytes.restype is C.c_int64
    assert L.d4pg_replay_steps_window_bytes.argtypes == [C.c_int64, C.c_int32, C.c_int32, C.c_int32]
    assert L.d4pg_replay_add_steps.restype is C.c_int32
    assert L.d4pg_replay_add_steps.argtypes == [P, C.c_int64, P, P, P, P, P, P, C.c_int32, C.c_double, P, C.c_int64,
                                                C.c_int32, P]
    assert L.d4pg_version() >= 1000
    up = lambda b: (b + 15) & ~15

    def want(E, S, A, n):
        return up(up(up(up(E * 8) + E * 2 * n * 8) + E * n * S * 4) + E * n * A * 4)
    for E, S, A, n in [(1, 3, 2, 1), (33, 17, 6, 5), (4096, 376, 17, 7), (5, 1, 1, 64)]:
        assert L.d4pg_replay_steps_window_bytes(E, S, A, n) == want(E, S, A, n)
    for bad in [(0, 3, 2, 1), (1, 0, 2, 1), (1, 3, 0, 1), (1, 3, 2, 0), (1, 3, 2, 65)]:
        assert L.d4pg_replay_steps_window_bytes(*bad) == -1
    x = P(0x10000)
    assert L.d4pg_replay_add_steps(None, 4, x, x, x, x, x, None, 2, 0.9, x, 0, 0, None) == _lib.EINVAL
    assert "null" in L.d4pg_last_error().decode()
