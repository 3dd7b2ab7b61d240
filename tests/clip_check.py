"""Global-norm gradient clipping and Adam weight decay of the learner step, restated in numpy on the device's own values
and held to bit-exactness on top of tests/update_check.py.

Per network, on the step's complete flat gradient g (padding included, as flat_grads() shows it: the buffer keeps the
UNCLIPPED gradient) and the pre-step parameters p, the Adam kernel (csrc/adam_dev.cuh clip_coef / adam_segment<true>)
forms

    norm = sqrt(sum g_i^2)                                  float64, fixed order (csrc/adam.cu grad_sqnorm_kernel)
    coef = float32(min(1, max_norm / (norm + 1e-6)))        float64, cast once; exactly 1 when nothing is clipped
    ge   = (g * coef) + (wd * p)                            float32, each operation rounded; the decay term only when wd != 0

and runs the plain update on ge.  `check_step` forms ge from the device's g and p and hands update_check.check_arrays a
step whose gradient is ge, so m, v, p, t, the padding and the step clock are checked exactly as they are without
clipping.  The device's float64 sum and the host's differ in their last bits: where the float64 coefficient lies that
close to a float32 rounding midpoint both neighbours are accepted (`coef_candidates`).

Power: the update restated without the clipping coefficient (on steps that clip) and without the decay term must each
disagree with the device's first moment in at least one element of each network.

`clip_hook` gives oracle.d4pg_oracle.LearnerOracle the same two options through its grad_hook: DERIVED (the reference has
neither feature), torch.nn.utils.clip_grad_norm_ per network, then the `grad.add(param, alpha=weight_decay)` of torch
2.11's _single_tensor_adam.
"""
import itertools
import math

import numpy as np
import torch

from tests import update_check as UC

F32 = np.float32
EPS = 1e-6
# float64 ulps the device's fixed-order sum of squares (3 sequential adds per thread, a 5-level warp tree, 8 warps, then
# 64 partials as a 6-level tree) may lie from the exactly rounded sum, as a multiple of update_check.POW_ULP
NORM_AMP = 16.0


def norm(g):
    """sqrt of the exactly rounded float64 sum of squares of the float32 array g (each square is exact in float64)."""
    g64 = np.asarray(g, dtype=F32).astype(np.float64)
    return math.sqrt(math.fsum(g64 * g64))


def coef_candidates(nrm, max_norm):
    """([float32 coefficients the device may hold], near_midpoint) for gradient norm `nrm` and threshold `max_norm`
    (0 / None: no clipping, the coefficient is exactly 1)."""
    if not max_norm:
        return [F32(1.0)], False
    return UC.scalar_candidates(min(1.0, max_norm / (nrm + EPS)), NORM_AMP)


def effective_gradient(g, p, coef, wd):
    ge = (np.asarray(g, dtype=F32) * F32(coef)).astype(F32)
    if F32(wd) != 0:
        ge = (ge + (F32(wd) * np.asarray(p, dtype=F32)).astype(F32)).astype(F32)
    return ge


class ClipStats(object):
    def __init__(self):
        self.update = UC.Stats()
        self.steps, self.midpoints, self.worst_norm_ulp = 0, 0, 0
        self.clipped = {"actor": 0, "critic": 0}
        self.unclipped = {"actor": 0, "critic": 0}
        self.power_min = None

    def power(self, n):
        self.power_min = n if self.power_min is None else min(self.power_min, n)

    def line(self):
        return ("%d clipped-update steps bit-exact; clipped steps %s, unclipped %s; %d coefficient-midpoint exceptions; "
                "reported norms worst %d ulp; fewest elements a no-clip / no-decay restatement got wrong: %s; %s"
                % (self.steps, self.clipped, self.unclipped, self.midpoints, self.worst_norm_ulp, self.power_min,
                   self.update.line()))


def check_step(before, after, pads, h, k, max_norm, wd, dev_norms=None, stats=None, label=""):
    """The update of step k from `before` to `after` (dicts of update_check.read) under thresholds `max_norm` and decays
    `wd` ((actor, critic) pairs; 0 = off).  dev_norms: the (actor, critic) norms the device reported, held to one float32
    ulp of the restated norm.  Returns {net: coefficient} (the first candidate)."""
    stats = stats if stats is not None else ClipStats()
    bad, cands, coefs = [], [], {}
    for i, (name, _) in enumerate(UC.NETS):
        g, pad = after[name]["g"], pads[name]
        n = int(np.count_nonzero(g[pad]))
        if n:
            bad.append("%s.g: %d nonzero padding elements in the unclipped gradient" % (name, n))
        nrm = norm(g)
        cs, mid = coef_candidates(nrm, max_norm[i])
        stats.midpoints += int(mid)
        cands.append(cs)
        coefs[name] = cs[0]
        if max_norm[i]:
            (stats.clipped if cs[0] < 1 else stats.unclipped)[name] += 1
            if dev_norms is not None:
                u = int(UC.ulps(np.asarray([F32(nrm)]), np.asarray([F32(dev_norms[i])]))[0])
                stats.worst_norm_ulp = max(stats.worst_norm_ulp, u)
                if u > 1:
                    bad.append("%s: reported norm %r is %d ulp from the restated %r" % (name, dev_norms[i], u, F32(nrm)))
    err = None
    for combo in itertools.product(*cands):
        forced = {name: dict(after[name], g=effective_gradient(after[name]["g"], before[name]["p"], combo[i], wd[i]))
                  for i, (name, _) in enumerate(UC.NETS)}
        try:
            UC.check_arrays(before, forced, pads, h, k, stats.update, label)
            err = None
            break
        except AssertionError as e:
            err = e
    if err is not None:
        bad.append(str(err))
    # power: without the coefficient, and without the decay term, the first moment must come out different
    for i, (name, _) in enumerate(UC.NETS):
        g, p, m0, m1 = after[name]["g"], before[name]["p"], before[name]["m"], after[name]["m"]
        if cands[i][0] < 1:
            n = int(np.count_nonzero(UC.differ(UC.restate_m(h, effective_gradient(g, p, 1.0, wd[i]), m0), m1)))
            stats.power(n)
            if n == 0:
                bad.append("%s: the restatement without clipping matches the device too" % name)
        if F32(wd[i]) != 0:
            n = int(np.count_nonzero(UC.differ(UC.restate_m(h, effective_gradient(g, p, cands[i][0], 0.0), m0), m1)))
            stats.power(n)
            if n == 0:
                bad.append("%s: the restatement without weight decay matches the device too" % name)
    stats.steps += 1
    assert not bad, "%s step %d: %s" % (label, k, "; ".join(bad))
    return coefs


def clip_hook(oracle, max_grad_norm=None, weight_decay=(0.0, 0.0), log=None):
    """grad_hook for LearnerOracle.train_step: clip each network's gradients to max_grad_norm (None, a number or an
    (actor, critic) pair) with torch.nn.utils.clip_grad_norm_, then add weight_decay * parameter as torch 2.11's
    _single_tensor_adam does.  log: a list that receives (actor_norm, critic_norm, actor_coef, critic_coef) per step."""
    pair = max_grad_norm if isinstance(max_grad_norm, (tuple, list)) else (max_grad_norm, max_grad_norm)

    def hook(g_a, g_c):
        rec = []
        for grads, weights, mx, wd in ((g_a, oracle.actor, pair[0], weight_decay[0]),
                                       (g_c, oracle.critic, pair[1], weight_decay[1])):
            if mx is not None:
                params = []
                for key in grads:
                    prm = torch.nn.Parameter(weights[key].clone(), requires_grad=True)
                    prm.grad = grads[key]                       # clipped in place
                    params.append(prm)
                total = float(torch.nn.utils.clip_grad_norm_(params, mx))
                rec.append((total, min(1.0, mx / (total + EPS))))
            else:
                rec.append((0.0, 1.0))
            if wd != 0:
                for key in grads:
                    grads[key].add_(weights[key], alpha=wd)
        if log is not None:
            log.append((rec[0][0], rec[1][0], rec[0][1], rec[1][1]))
    return hook
