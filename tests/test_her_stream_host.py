"""Streaming hindsight relabelling on the host (DESIGN.md §3 "Streaming hindsight relabelling"): the vectorized oracle
against O.her_relabel, the host mirror's row counts, plan and generator state against the oracle over random streams,
and every argument check, raised before any device work."""
import numpy as np
import pytest

from tests import her_stream_oracle as HO


def _bits(x):
    return x if x.dtype == bool else x.view(np.uint8)


@pytest.mark.parametrize("her_action", ["reference", "own"])
@pytest.mark.parametrize("E,M", [(1, 1), (1, 9), (7, 6), (30, 4)])
def test_vectorized_oracle_is_her_relabel(E, M, her_action):
    """The vectorized oracle's rows are bit-identical to O.her_relabel called once per episode with the same draws,
    with flushes in the stream and her_ratio 0, 0.5 and 1."""
    rng = np.random.RandomState(E * 100 + M)
    calls = HO.random_calls(rng, 5 * M + 6, E, 5, 3, 2, M, flush_at=(2, 3 * M))
    for ratio in (0.0, 0.5, 1.0):
        a = HO.stream_rows(calls, ratio, 0.05, her_action, 11, vectorized=True)
        b = HO.stream_rows(calls, ratio, 0.05, her_action, 11, vectorized=False)
        assert len(a) == len(b) == len(calls)
        for x, y in zip(a, b):
            for k in x:
                assert x[k].dtype == y[k].dtype and np.array_equal(_bits(x[k]), _bits(y[k])), k
        n = sum(len(x["r"]) for x in a)
        assert n > 0


def test_oracle_rows_by_hand():
    """E = 2, max 3 steps: env 0 ends a 2-step episode at call 1 (terminated), env 1 a 3-step one at call 2
    (truncated); both are emitted one call later, and a flush emits env 0's second episode (calls 2 and 3)."""
    So, G, A = 1, 1, 1
    term = [[0, 0], [1, 0], [0, 0], [0, 0]]
    trunc = [[0, 0], [0, 0], [0, 1], [0, 0]]
    calls = []
    for k in range(4):
        calls.append((np.array([[10. * k], [20. * k]], np.float32), np.array([[0.5], [0.7]]),
                      np.array([[k], [-k]], np.float32), np.array([-1., -1.]), np.array([[10. * k + 1], [20. * k + 1]], np.float32),
                      np.array([[0.5 + k], [0.7]]), np.array(term[k], bool), np.array(trunc[k], bool)))
    calls[3] = calls[3][:6] + (np.array([True, False]), calls[3][7])
    calls.append(None)
    rows = HO.stream_rows(calls, 1.0, 0.05, "reference", 0)
    assert [len(r["r"]) for r in rows] == [0, 0, 4, 6, 4]
    r2 = rows[2]                                   # env 0, steps 0 and 1, both relabelled
    rng = np.random.default_rng(0)
    rng.random(2)
    f0 = rng.integers(np.array([0, 1]), np.array([2, 2]))
    assert np.array_equal(r2["s"][:, 1], [0.5, 0.5 + f0[0], 0.5, 0.5 + f0[1]])
    assert np.array_equal(r2["a"][:, 0], [0., 1., 1., 1.])        # copies carry the episode's last action
    assert list(r2["d"]) == [False, f0[0] == 0, True, True]
    assert rows[3]["s"][0, 1] == 0.7 and all(rows[3]["r"][1::2] == 0) and rows[3]["d"][1::2].all()
    assert np.array_equal(rows[4]["s"][:, 0], [20., 20., 30., 30.])


@pytest.mark.parametrize("late", [False, True])
@pytest.mark.parametrize("E,M", [(1, 5), (13, 7), (64, 50)])
def test_mirror_counts_draws_and_generator(E, M, late):
    """GoalStepsMirror: before every call (and flush) its row count equals the oracle's, its plan decodes to the
    oracle's draws (select = future >= 0, the future steps, the ranks), and its generator's state equals an oracle
    generator advanced by the same draws -- with the ends applied after the call (host flags) or at the start of the
    next one (CUDA flags)."""
    import d4pg_b200 as d4pg
    GoalStepsMirror = d4pg.prioritized_replay_memory.GoalStepsMirror
    rng = np.random.RandomState(E + M)
    calls = HO.random_calls(rng, 3 * M + 5, E, 2, 3, 1, M, flush_at=(M,))
    want = [len(r["r"]) for r in HO.stream_rows(calls, 0.8, 0.05, "reference", 5)]
    m = GoalStepsMirror(E, 2, 3, 1, 0.8, 0.05, "reference", M, 5)
    orng = np.random.default_rng(5)
    cur = np.zeros(E, np.int64)
    ended = np.zeros(E, np.int64)
    last_end = None
    got = []
    for c in calls:
        if late and last_end is not None:
            m.end(last_end)
            last_end = None
        if c is not None:
            m.check_step()
        plan, n_draws, n_rows = m.draw()
        got.append(n_rows)
        em = np.flatnonzero(ended)
        if em.size:
            sel, fut = HO.draws(orng, ended[em], 0.8)
            assert n_draws == sel.size and n_rows == sel.size + sel.sum()
            assert np.array_equal(plan[:E][em], np.cumsum(ended[em]) - ended[em])
            future, dst = plan[E:E + n_draws], plan[E + n_draws:]
            assert np.array_equal(future >= 0, sel) and np.array_equal(future[sel], fut[sel])
            assert np.array_equal(dst, np.cumsum(1 + sel) - (1 + sel))
        else:
            assert plan is None and n_draws == 0
        assert m.rng.bit_generator.state == orng.bit_generator.state
        ended[:] = 0
        m.advance(c is not None)
        if c is None:
            continue
        cur += 1
        end = c[6] | c[7]
        ended[end] = cur[end]
        cur[end] = 0
        assert (m.fill[~end] == cur[~end]).all() if late else True
        if late:
            last_end = end
        else:
            m.end(end)
    assert got == want and sum(got) > 0


def _args(E, So=4, G=3, A=2):
    return (np.zeros((E, So), np.float32), np.zeros((E, G)), np.zeros((E, A), np.float32), np.zeros(E),
            np.zeros((E, So), np.float32), np.zeros((E, G)), np.zeros(E, bool))


def test_validation_before_device_work():
    """Every ValueError of add_goal_steps is raised before the buffer allocates anything: the parameters, the shapes,
    E * 2 * max_episode_steps > size, a change of a fixed parameter, an episode past max_episode_steps, and add_steps /
    add_goal_steps while the other has pending state.  DDPG validates her= at construction, before any network."""
    import d4pg_b200 as d4pg
    GoalStepsMirror = d4pg.prioritized_replay_memory.GoalStepsMirror
    StepsMirror = d4pg.prioritized_replay_memory.StepsMirror
    info = {"type": "categorical", "v_min": -10.0, "v_max": 0.0, "n_atoms": 51}
    for cls in (lambda: d4pg.ReplayBuffer(400), lambda: d4pg.PrioritizedReplayBuffer(400, 0.6),
                lambda: d4pg.Replay(400, None)):
        buf = cls()
        a = _args(4)
        for kw, msg in ((dict(her_ratio=1.5), "her_ratio"), (dict(her_ratio=float("nan")), "her_ratio"),
                        (dict(threshold=-0.1), "threshold"), (dict(threshold=float("inf")), "threshold"),
                        (dict(her_action="last"), "her_action"), (dict(max_episode_steps=0), "max_episode_steps"),
                        (dict(max_episode_steps=2.5), "max_episode_steps"), (dict(seed=-1), "seed"),
                        (dict(max_episode_steps=51), "E \\* 2 \\* max_episode_steps")):
            with pytest.raises(ValueError, match=msg):
                buf.add_goal_steps(*a, **kw)
        bad = list(a)
        bad[5] = np.zeros((4, 2))
        with pytest.raises(ValueError, match="shapes"):
            buf.add_goal_steps(*bad)
        with pytest.raises(ValueError, match="shapes"):
            buf.add_goal_steps(*a, truncated=np.zeros(3, bool))
        with pytest.raises(ValueError, match="obs, desired_goal and action"):
            buf.add_goal_steps(np.zeros(4, np.float32), *a[1:])
        st = buf._store
        # pending state, as a first call leaves it
        st._goals = GoalStepsMirror(4, 4, 3, 2, 0.8, 0.05, "reference", 50, 0)
        for kw in (dict(her_ratio=0.5), dict(threshold=0.1), dict(her_action="own"), dict(max_episode_steps=40),
                   dict(seed=1)):
            with pytest.raises(ValueError, match="drop_goal_steps"):
                buf.add_goal_steps(*a, **kw)
        with pytest.raises(ValueError, match="drop_goal_steps"):
            buf.add_goal_steps(*_args(5))
        with pytest.raises(ValueError, match="drop_goal_steps"):
            buf.add_goal_steps(*_args(4, So=5, G=2))
        with pytest.raises(ValueError, match="add_goal_steps has pending"):
            buf.add_steps(*(a[i] for i in (0, 2, 3, 4, 6)))
        st._goals.fill[2] = 50
        with pytest.raises(ValueError, match="environment 2 already has max_episode_steps = 50"):
            buf.add_goal_steps(*a)
        buf.drop_goal_steps()
        assert st._goals is None
        st._steps = StepsMirror(4, 1, 0.99)
        with pytest.raises(ValueError, match="add_steps has pending"):
            buf.add_goal_steps(*a)
        buf.drop_steps()
        assert st.handle is None and len(buf) == 0 and buf.flush_goal_steps() == 0
    for her, msg in (({"her_ratio": 2.0}, "her_ratio"), ({"ratio": 0.5}, "her must be"), ("yes", "her must be")):
        with pytest.raises(ValueError, match=msg):
            d4pg.DDPG(7, 2, critic_dist_info=info, her=her)
    with pytest.raises(ValueError, match="n_steps"):
        d4pg.DDPG(7, 2, critic_dist_info=info, n_steps=3, her=True)
    _her_params = d4pg.ddpg._her_params
    assert _her_params(True) == {"her_ratio": 0.8, "threshold": 0.05, "her_action": "reference",
                                 "max_episode_steps": 50, "seed": 0}
    assert _her_params({"her_action": "own", "seed": 3})["seed"] == 3 and _her_params(None) is None


def test_abi():
    """The new entry points are bound; the window size follows the documented layout; the C side rejects bad calls."""
    from d4pg_b200 import _lib
    L = _lib.lib()
    assert L.d4pg_version() >= 1200
    up = lambda b: (b + 15) & ~15
    E, So, G, A, M = 64, 25, 3, 4, 50
    want = up(E * 4) + 2 * up(E * M * So * 4) + up(E * M * A * 4) + 2 * up(E * M * G * 8) + up(E * M * 8) + up(E * M)
    assert L.d4pg_replay_goal_window_bytes(E, So, G, A, M) == want
    assert L.d4pg_replay_goal_window_bytes(E, So, G, A, 0) == -1
    assert L.d4pg_replay_goal_window_bytes(E, So, 0, A, M) == -1
    assert L.d4pg_replay_goal_window_bytes(E, So, G, A, _lib.GOAL_MAX_STEPS + 1) == -1
    assert L.d4pg_replay_add_goal_steps(None, 4, 3, 2, *([None] * 8), 5, None, None, 0, 0, 0.05, 0, 0, 0, None) == _lib.EINVAL
