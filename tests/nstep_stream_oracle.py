"""Oracle of the streaming n-step insert (ReplayBuffer.add_steps, DESIGN.md §3 "Streaming n-step insert"), built on
the episode restatement O.nstep_transitions (pinned to the reference's Replay.initialize by tests/golden/nstep_init.npz):
each environment's stream of steps is cut into episodes at terminated | truncated, every episode goes through
O.nstep_transitions, and a row is inserted at the call of its last step.  Rows are ordered by (emitting call, e)."""
import numpy as np

from oracle import d4pg_oracle as O


def stream_rows(calls, n_steps, gamma):
    """calls: list of (obs [E,S], act [E,A], rew [E], obs2 [E,S], terminated [E], truncated [E] or None), one per
    vector step.  Returns [(call, e, (s, a, R, s2, done))] in insertion order."""
    E = np.shape(calls[0][0])[0]
    out = []
    for e in range(E):
        ep = []
        for k, c in enumerate(calls):
            ep.append(k)
            ended = bool(c[4][e]) or (c[5] is not None and bool(c[5][e]))
            if ended or k == len(calls) - 1:
                rows = O.nstep_transitions([calls[j][0][e] for j in ep], [calls[j][1][e] for j in ep],
                                           [float(calls[j][2][e]) for j in ep], [calls[j][3][e] for j in ep],
                                           [bool(calls[j][4][e]) for j in ep], n_steps, gamma)
                for i, row in enumerate(rows):
                    out.append((ep[n_steps - 1 + i], e, row))
                ep = []
    out.sort(key=lambda x: (x[0], x[1]))
    return out


def rows_per_call(ends, n_steps):
    """Rows each call inserts, from the episode ends alone (bool [K, E]): e emits at call k when its current episode
    has reached n_steps steps by then."""
    ends = np.asarray(ends, dtype=bool)
    K, E = ends.shape
    steps = np.zeros(E, dtype=np.int64)
    out = []
    for k in range(K):
        steps += 1
        out.append(int(np.count_nonzero(steps >= n_steps)))
        steps[ends[k]] = 0
    return out


def random_ends(rng, K, E, n_steps, p_term=0.08, p_trunc=0.04):
    """Per-environment terminations and truncations at different steps: episode lengths < n, == n and >> n."""
    term = rng.rand(K, E) < p_term
    trunc = (rng.rand(K, E) < p_trunc) & ~term
    for e in range(1, min(E, 3)):                  # environment 1 ends every n_steps steps, environment 2 every n_steps - 1
        term[:, e] = trunc[:, e] = False
        L = max(1, n_steps + 1 - e)
        term[L - 1::L, e] = True
    return term, trunc


def random_calls(rng, K, E, S, A, n_steps, with_trunc=True):
    term, trunc = random_ends(rng, K, E, n_steps)
    calls = []
    for k in range(K):
        calls.append((rng.randn(E, S).astype(np.float32), rng.uniform(-1, 1, (E, A)).astype(np.float32), rng.randn(E),
                      rng.randn(E, S).astype(np.float32), term[k].copy(), trunc[k].copy() if with_trunc else None))
    return calls
