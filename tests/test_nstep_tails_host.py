"""Episode tails of the streaming insert on the host (DESIGN.md §3 "Episode tails"): the oracle's rows against its own
row counts, the host mirror's count per call against the oracle over random streams, and the argument checks that run
before any device work."""
import ctypes as C

import numpy as np
import pytest

from tests import nstep_stream_oracle as SO
from tests import nstep_tails_oracle as TO


@pytest.mark.parametrize("n_steps", [1, 2, 5, 7, 64])
@pytest.mark.parametrize("E", [1, 3, 33])
def test_mirror_counts_vs_oracle(n_steps, E):
    """StepsMirror with tails counts, before each call, exactly the rows the oracle inserts at that call -- episodes
    shorter than, equal to and longer than n, ended by termination or truncation -- with the ends applied after the call
    (host flags) or at the start of the next one (CUDA flags)."""
    from d4pg_b200.prioritized_replay_memory import StepsMirror
    rng = np.random.RandomState(n_steps * 101 + E)
    K = 3 * n_steps + 40
    calls = SO.random_calls(rng, K, E, 2, 1, n_steps)
    rows = TO.tail_rows(calls, n_steps, 0.9)
    want = np.bincount([r[0] for r in rows], minlength=K).tolist()
    ends = np.array([c[4] | c[5] for c in calls])
    assert TO.rows_per_call(ends, n_steps) == want
    if n_steps == 1:
        assert want == SO.rows_per_call(ends, 1)
    if n_steps == 1:
        assert not any(r[3] for r in rows)
    for late in (False, True):
        m = StepsMirror(E, n_steps, 0.9, tails=True)
        got = []
        for k in range(K):
            if late and k:
                m.end(ends[k - 1])
            got.append(m.rows())
            m.advance()
            if not late:
                m.end(ends[k])
        assert got == want


def test_tail_rows_shape():
    """One environment, n = 4: an episode of 6 steps ending by truncation gives full rows u = 0..2 and tails u = 3, 4, 5
    (horizons 3, 2, 1) at the next call, not done; a terminated episode of 2 steps gives tails u = 0, 1 (horizons 2, 1),
    done; a third episode that is still running at the end of the stream gives no tails."""
    K, n = 11, 4
    term = np.zeros((K, 1), bool)
    trunc = np.zeros((K, 1), bool)
    trunc[5, 0] = True
    term[7, 0] = True
    calls = [(np.full((1, 2), k, np.float32), np.full((1, 1), k, np.float32), np.array([float(k + 1)]),
              np.full((1, 2), 100 + k, np.float32), term[k], trunc[k]) for k in range(K)]
    rows = TO.tail_rows(calls, n, 0.5)
    got = [(c, u, h, float(r[0][0]), r[2], float(r[3][0]), r[4]) for c, e, u, h, r in rows]
    assert got == [(3, 0, 0, 0.0, 1 + 0.5 * 2 + 0.25 * 3 + 0.125 * 4, 103.0, False),
                   (4, 1, 0, 1.0, 2 + 0.5 * 3 + 0.25 * 4 + 0.125 * 5, 104.0, False),
                   (5, 2, 0, 2.0, 3 + 0.5 * 4 + 0.25 * 5 + 0.125 * 6, 105.0, False),
                   (6, 3, 3, 3.0, 4 + 0.5 * 5 + 0.25 * 6, 105.0, False),
                   (6, 4, 2, 4.0, 5 + 0.5 * 6, 105.0, False),
                   (6, 5, 1, 5.0, 6.0, 105.0, False),
                   (8, 0, 2, 6.0, 7 + 0.5 * 8, 107.0, True),
                   (8, 1, 1, 7.0, 8.0, 107.0, True)]


def test_validation_before_device_work():
    """projection="reference" with n_steps > 1 and tails raises ValueError in DDPG's constructor, before any network
    is built; E * (n - 1) > size raises ValueError from add_steps before the buffer allocates anything."""
    import d4pg_b200 as d4pg
    info = {"type": "categorical", "v_min": -10.0, "v_max": 0.0, "n_atoms": 51}
    with pytest.raises(ValueError, match="projection"):
        d4pg.DDPG(5, 2, critic_dist_info=info, n_steps=3, nstep_tails=True)
    buf = d4pg.ReplayBuffer(20, nstep_tails=True)
    E, S, A = 6, 3, 2
    args = (np.zeros((E, S), np.float32), np.zeros((E, A), np.float32), np.zeros(E), np.zeros((E, S), np.float32),
            np.zeros(E, bool))
    with pytest.raises(ValueError, match="E \\* \\(n_steps - 1\\)"):
        buf.add_steps(*args, n_steps=5)
    assert buf._store.handle is None and len(buf) == 0
    with pytest.raises(ValueError, match="E \\* \\(n_steps - 1\\)"):
        d4pg.Replay(20, None, n_steps=5, nstep_tails=True).add_steps(*args)


def test_abi():
    """The new entry points are bound, the config mirror has the library's size, and the C side rejects a tails call
    without a horizon column or with too many rows before any device work."""
    from d4pg_b200 import _lib
    L = _lib.lib()
    assert L.d4pg_version() >= 1100
    assert L.d4pg_struct_size(0) == C.sizeof(_lib.LearnerConfig)
    assert "nstep_tails" in [f[0] for f in _lib.LearnerConfig._fields_][-1:]
    base = L.d4pg_replay_steps_window_bytes_ex(64, 17, 6, 5, 0)
    assert base == L.d4pg_replay_steps_window_bytes(64, 17, 6, 5)
    assert L.d4pg_replay_steps_window_bytes_ex(64, 17, 6, 5, 1) == base + 64 * 17 * 4
    assert L.d4pg_replay_steps_window_bytes_ex(64, 17, 6, 5, 2) == -1
    assert L.d4pg_replay_set_horizons(None, None, None) == _lib.EINVAL
    assert L.d4pg_replay_add_steps_ex(None, 4, None, None, None, None, None, None, 5, 0.9, None, 0, 1, 0, None) == _lib.EINVAL
