"""Oracle of the streaming hindsight relabelling (ReplayBuffer.add_goal_steps, DESIGN.md §3 "Streaming hindsight
relabelling"), derived from O.her_relabel (main.py:154-184, "future" strategy).  Environment e's episode runs from the
step after its last end to the next terminated or truncated step; an episode that ends at call k is emitted at call
k + 1 (or at a flush), before that call's step.  The episodes a call emits, in ascending e, draw from one
numpy.random.default_rng(seed): rng.random(sum L) < her_ratio selects, then one rng.integers(t, L) over the selected
(e, t) gives their future steps.  Each episode's rows are O.her_relabel's rows for those draws, with the step's own
action on the copies for her_action="own".

`calls` is a list whose items are one vector step (obs [E, So], goal [E, G], act [E, A], rew [E], obs_next [E, So],
ag_next [E, G], terminated [E], truncated [E] or None), or None for flush_goal_steps().  `stream_rows` gives, per call,
the rows it inserts as arrays {s, a, r, s2, d}; `vectorized=True` computes the same bits with whole-array numpy
operations (fast enough for E = 4096), `vectorized=False` calls O.her_relabel once per episode."""
import numpy as np

from oracle import d4pg_oracle as O

F64 = np.float64


def draws(rng, lengths, her_ratio):
    """One call's draws for ended episodes of `lengths` (ascending e) -> (select bool [n], future int64 [n]), n = sum L;
    future[i] = t where not selected."""
    L = np.asarray(lengths, dtype=np.int64)
    n = int(L.sum())
    starts = np.cumsum(L) - L
    t = np.arange(n, dtype=np.int64) - np.repeat(starts, L)
    sel = rng.random(n) < her_ratio
    fut = t.copy()
    if sel.any():
        fut[sel] = rng.integers(t[sel], np.repeat(L, L)[sel])
    return sel, fut


def _empty(S, A):
    return dict(s=np.zeros((0, S), F64), a=np.zeros((0, A), np.float32), r=np.zeros(0, F64), s2=np.zeros((0, S), F64),
                d=np.zeros(0, bool))


def _episode_loop(X, ks, e, sel, fut, threshold, her_action):
    """O.her_relabel over the steps (ks[t], e) of one episode."""
    obs, goal, act, rew, obs2, ag2, term = (np.stack([np.asarray(X[i][k][e]) for k in ks]) for i in range(7))
    rows = O.her_relabel(obs, obs2, goal, ag2, act, rew, term, sel, fut, threshold, act[-1])
    if her_action == "own":                       # the copy of step t carries a_t
        i = 0
        for t in range(len(ks)):
            i += 1
            if sel[t]:
                rows[i] = (rows[i][0], act[t]) + tuple(rows[i][2:])
                i += 1
    return dict(s=np.stack([np.asarray(r[0], F64) for r in rows]), a=np.stack([np.asarray(r[1], np.float32) for r in rows]),
                r=np.array([r[2] for r in rows], F64), s2=np.stack([np.asarray(r[3], F64) for r in rows]),
                d=np.array([bool(r[4]) for r in rows]))


def _call_vectorized(X, eps, sel, fut, threshold, her_action):
    """All rows of one call: eps = [(e, [call of step t])] in ascending e, draws over their concatenated steps."""
    L = np.array([len(ks) for _, ks in eps], dtype=np.int64)
    kk = np.concatenate([np.asarray(ks, np.int64) for _, ks in eps])
    ee = np.repeat(np.array([e for e, _ in eps], np.int64), L)
    starts = np.repeat(np.cumsum(L) - L, L)
    last = starts + np.repeat(L, L) - 1
    obs, goal, act, rew, obs2, ag2, term = (X[i][kk, ee] for i in range(7))
    g = starts + fut                              # flat index of each step's future step
    n = kk.size
    counts = 1 + sel.astype(np.int64)
    dst = np.cumsum(counts) - counts
    m = int(counts.sum())
    S = obs.shape[1] + goal.shape[1]
    out = dict(s=np.zeros((m, S), F64), a=np.zeros((m, act.shape[1]), np.float32), r=np.zeros(m, F64),
               s2=np.zeros((m, S), F64), d=np.zeros(m, bool))
    So = obs.shape[1]
    out["s"][dst, :So], out["s"][dst, So:] = obs, goal
    out["s2"][dst, :So], out["s2"][dst, So:] = obs2, goal
    out["a"][dst], out["r"][dst], out["d"][dst] = act, rew, term.astype(bool)
    c = dst[sel] + 1
    gp = ag2[g[sel]]
    out["s"][c, :So], out["s"][c, So:] = obs[sel], gp
    out["s2"][c, :So], out["s2"][c, So:] = obs2[sel], gp
    out["a"][c] = act[sel] if her_action == "own" else act[last[sel]]
    dist = np.linalg.norm(ag2[sel] - gp, axis=-1)  # the same reduction as O.her_relabel's per-row norm
    r = -(dist > threshold).astype(F64)
    out["r"][c], out["d"][c] = r, r == 0.0
    assert n == L.sum()
    return out


def stream_rows(calls, her_ratio=0.8, threshold=0.05, her_action="reference", seed=0, vectorized=True):
    """-> [rows of call k as {s, a, r, s2, d}] (s / s2 f64, before the ring's f32 cast)."""
    first = next(c for c in calls if c is not None)
    E, So, G, A = first[0].shape[0], first[0].shape[1], first[1].shape[1], first[2].shape[1]
    steps = [c for c in calls if c is not None]
    X = [np.stack([np.asarray(c[i]) for c in steps]) for i in range(7)]   # [K', E, ...]; X[i][j] = step j
    rng = np.random.default_rng(seed)
    cur = [[] for _ in range(E)]
    ended = [None] * E
    out = []
    j = 0
    for c in calls:
        eps = [(e, ended[e]) for e in range(E) if ended[e] is not None]
        rows = _empty(So + G, A)
        if eps:
            sel, fut = draws(rng, [len(ks) for _, ks in eps], her_ratio)
            if vectorized:
                rows = _call_vectorized(X, eps, sel, fut, threshold, her_action)
            else:
                parts, o = [], 0
                for e, ks in eps:
                    parts.append(_episode_loop(X, ks, e, sel[o:o + len(ks)], fut[o:o + len(ks)], threshold, her_action))
                    o += len(ks)
                rows = {k: np.concatenate([p[k] for p in parts]) for k in parts[0]}
            ended = [None] * E
        out.append(rows)
        if c is None:
            continue
        end = np.asarray(c[6], bool) | (np.zeros(E, bool) if c[7] is None else np.asarray(c[7], bool))
        for e in range(E):
            cur[e].append(j)
            if end[e]:
                ended[e], cur[e] = cur[e], []
        j += 1
    return out


def random_calls(rng, K, E, So, G, A, M, p_trunc=0.5, flush_at=(), with_trunc=True):
    """K vector steps of episodes whose lengths are uniform in [1, M] (so 1 and M both occur), each ended by
    termination or truncation, with None inserted after the calls in `flush_at`.  Achieved goals lie on a 0.02 grid
    near each other, so the relabelled distances fall on both sides of a 0.05 threshold and are often exactly 0."""
    left = rng.randint(1, M + 1, E)
    calls = []
    for k in range(K):
        left -= 1
        end = left == 0
        trunc = end & (rng.rand(E) < p_trunc) if with_trunc else np.zeros(E, bool)
        term = end & ~trunc
        left[end] = rng.randint(1, M + 1, int(end.sum()))
        calls.append((rng.randn(E, So).astype(np.float32), rng.randn(E, G), rng.uniform(-1, 1, (E, A)).astype(np.float32),
                      -rng.randint(0, 2, E).astype(F64), rng.randn(E, So).astype(np.float32),
                      rng.randint(0, 4, (E, G)) * 0.02, term, trunc if with_trunc else None))
        if k in flush_at:
            calls.append(None)
    return calls


def concat(rows):
    """The rows of several calls, in insertion order."""
    return {k: np.concatenate([r[k] for r in rows]) for k in rows[0]}
