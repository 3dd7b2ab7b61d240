"""Numpy restatement of the observation normalizer (DERIVED: the reference has no normalization; the definition is
DESIGN.md section 3 "Observation normalization" and include/d4pg_b200.h d4pg_replay_set_obs_norm).

float64 elementwise numpy operations are correctly rounded and never fused, so the Welford fold below (a loop over
rows, vectorised over features) gives the device's bits; the apply is float32 numpy, also rounded per operation.
"""
import numpy as np

CLIP, EPS = 5.0, 1e-8


class Stats(object):
    """n, mean[S], M2[S] in fp64, folded one row at a time in insertion order."""

    def __init__(self, obs_dim):
        self.n = 0.0
        self.mean = np.zeros(obs_dim, dtype=np.float64)
        self.m2 = np.zeros(obs_dim, dtype=np.float64)

    def fold(self, rows):
        rows = np.asarray(rows, dtype=np.float32).reshape(-1, self.mean.size)
        for row in rows:
            x = row.astype(np.float64)
            self.n = self.n + 1.0
            d = x - self.mean
            self.mean = self.mean + d / self.n
            self.m2 = self.m2 + d * (x - self.mean)
        return self

    def packed(self):
        """The device layout {n, mean[S], M2[S]}."""
        return np.concatenate([[self.n], self.mean, self.m2])

    def affine(self, eps=EPS):
        """(shift, scale) float32 [S] each."""
        S = self.mean.size
        if self.n == 0:
            return np.zeros(S, np.float32), np.ones(S, np.float32)
        var = self.m2 / self.n
        return self.mean.astype(np.float32), (1.0 / np.sqrt(var + eps)).astype(np.float32)


def pre_clip(x, shift, scale):
    x = np.asarray(x, dtype=np.float32)
    return (x - shift.astype(np.float32)) * scale.astype(np.float32)


def apply(x, shift, scale, clip=CLIP):
    c = np.float32(clip)
    return np.minimum(np.maximum(pre_clip(x, shift, scale), -c), c)


def dydx(x, shift, scale, clip=CLIP):
    v, c = pre_clip(x, shift, scale), np.float32(clip)
    return np.where((v >= -c) & (v <= c), np.broadcast_to(scale.astype(np.float32), v.shape), np.float32(0)).astype(np.float32)


def train_step_normalized(lo, stats, rows, idx, clip=CLIP, eps=EPS, **kw):
    """LearnerOracle.train_step on the batch rows[idx] with s and s2 normalized by `stats` (the oracle statistics of
    every row added before the step)."""
    S, A, R, S2, D = rows
    shift, scale = stats.affine(eps)
    return lo.train_step(apply(S[idx], shift, scale, clip), A[idx], R[idx], apply(S2[idx], shift, scale, clip), D[idx],
                         **kw)
