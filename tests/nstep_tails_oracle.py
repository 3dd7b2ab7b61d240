"""Oracle of the streaming insert with episode tails (ReplayBuffer.add_steps(..., nstep_tails=True), DESIGN.md §3
"Episode tails"), derived from the stream oracle.  Full rows come from O.nstep_transitions (pinned to the reference's
Replay.initialize by tests/golden/nstep_init.npz), with horizon 0.  An episode of L steps that ends (terminated or
truncated) at call k also gives, at call k + 1 -- if there is one -- a tail row for every start u in
[max(0, L-n+1), L-1]: (s_u, a_u, R over the k = L - u remaining rewards, obs_next_{L-1}, terminated_{L-1}) with horizon k,
R the same left-to-right Python float loop.  Rows are ordered by (emitting call, e, u).

Also the per-row-discount restatement of the mode-1 projection (O.project_nstep with `disc` a [B, 1] array of gamma ** k,
the same association as the kernel's (disc * (1 - d)) * z_j)."""
import numpy as np

from oracle import d4pg_oracle as O

F64 = np.float64


def _ret(rewards, gamma):
    cum, eg = 0., 1
    for r in rewards:
        cum += eg * r
        eg *= gamma
    return cum


def tail_rows(calls, n_steps, gamma):
    """calls as for nstep_stream_oracle.stream_rows.  Returns [(call, e, u, horizon, (s, a, R, s2, done))] in insertion
    order: the full rows (horizon 0, u their start) and the tail rows."""
    K = len(calls)
    E = np.shape(calls[0][0])[0]
    out = []
    for e in range(E):
        ep = []
        for k, c in enumerate(calls):
            ep.append(k)
            ended = bool(c[4][e]) or (c[5] is not None and bool(c[5][e]))
            if ended or k == K - 1:
                S = [calls[j][0][e] for j in ep]
                A = [calls[j][1][e] for j in ep]
                R = [float(calls[j][2][e]) for j in ep]
                rows = O.nstep_transitions(S, A, R, [calls[j][3][e] for j in ep], [bool(calls[j][4][e]) for j in ep],
                                           n_steps, gamma)
                for i, row in enumerate(rows):
                    out.append((ep[n_steps - 1 + i], e, i, 0, row))
                L = len(ep)
                if ended and k + 1 < K:
                    for u in range(max(0, L - n_steps + 1), L):
                        out.append((k + 1, e, u, L - u, (np.asarray(S[u]).reshape(-1), A[u], _ret(R[u:], gamma),
                                                         calls[k][3][e], bool(calls[k][4][e]))))
                ep = []
    out.sort(key=lambda x: (x[0], x[1], x[2]))
    return out


def rows_per_call(ends, n_steps):
    """Rows each call inserts with tails, from the episode ends alone (bool [K, E])."""
    ends = np.asarray(ends, dtype=bool)
    K, E = ends.shape
    steps = np.zeros(E, dtype=np.int64)
    pending = np.zeros(E, dtype=np.int64)
    out = []
    for k in range(K):
        steps += 1
        out.append(int(np.count_nonzero(steps >= n_steps) + pending.sum()))
        pending[:] = 0
        pending[ends[k]] = np.minimum(steps[ends[k]], n_steps - 1)
        steps[ends[k]] = 0
    return out


def row_discounts(horizons, gamma, n_steps):
    """[B, 1] f64: gamma ** k for a tail row, gamma ** n_steps for a full row (horizon 0)."""
    h = np.asarray(horizons).reshape(-1)
    return np.array([gamma ** int(k) if k else gamma ** n_steps for k in h], dtype=F64).reshape(-1, 1)


def project_disc(target_probs, rewards, dones, v_min, v_max, n_atoms, disc):
    """O.project_nstep with a per-row discount `disc` [B, 1]."""
    p = np.asarray(target_probs)
    r = np.asarray(rewards, dtype=F64).reshape(-1, 1)
    d = np.asarray(dones, dtype=F64).reshape(-1, 1)
    B = r.shape[0]
    delta, centers = O.atom_support(v_min, v_max, n_atoms)
    tz = r + disc * (1 - d) * centers.reshape(1, -1)
    tz = np.minimum(O.atom_clip_top(v_min, v_max, n_atoms), np.maximum(v_min, tz))
    b = (tz - v_min) / delta
    l = np.floor(b).astype(np.int64)
    u = np.ceil(b).astype(np.int64)
    l[(u > 0) & (l == u)] -= 1
    u[(l < (n_atoms - 1)) & (l == u)] += 1
    m = np.zeros(B * n_atoms, dtype=F64)
    off = (np.arange(B, dtype=np.int64) * n_atoms).reshape(-1, 1)
    np.add.at(m, (l + off).reshape(-1), (p * (u.astype(F64) - b)).reshape(-1))
    np.add.at(m, (u + off).reshape(-1), (p * (b - l.astype(F64))).reshape(-1))
    return m.reshape(B, n_atoms), l, u


class TailsLearnerOracle(O.LearnerOracle):
    """O.LearnerOracle (projection "nstep") whose next train_step projects with the per-row discounts set in `disc`."""
    disc = None

    def project(self, target_probs, r, done):
        return project_disc(target_probs, r, done, self.v_min, self.v_max, self.n_atoms, self.disc)[0].astype(O.F32)
