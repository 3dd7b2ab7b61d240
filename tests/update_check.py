"""The optimizer update of one learner step -- Adam, Polyak and the step clock that feeds them -- restated in numpy float32
on the device's own values, and held to bit-exactness.

Snapshot, then check.  Before the step: the four networks' flat parameters and both optimizers' flat moments.  After
it: the same buffers and the learner's flat gradient buffer, all including padding.  The fused kernel
(csrc/adam_dev.cuh adam_segment) computes, per element, with explicitly round-to-nearest operations (the build has no
-ftz and no fast-math):

    m' = fma(w1, g - m, m)            v' = (v * b2) + ((w2 * g) * g)
    denom = sqrt(v') / bc2s + eps     p' = p + nss * (m' / denom)      t' = (1 - tau) * t + tau * p'

w1, w2, b2, eps, tau and 1 - tau are float32 casts of the learner's double expressions; nss = float(-(lr / (1 - b1^k)))
and bc2s = float(sqrt(1 - b2^k)) come from the device clock (csrc/adam.cuh clock_derive), k is the step's 1-based
count.  Teacher forcing: m' from the device's g and m, v' from its g and v, p' from its p, m' and v', t' from its t and
p'.  Each must match on every element bit for bit; every padding element of p, g, m, v and t must be exactly zero.

The device's double `pow` may differ from the host's in the last bit.  Where a scalar's float64 value lies that close
to a float32 rounding midpoint (`scalar_candidates`), both float32 neighbours are accepted and the case is counted.

Power: the restatement at step k - 1 and at k + 1 must each disagree with the device in at least one element of each
network, and so must a target left one step stale (tau = 0).

IS weights (`is_weight_check`): the sampler's formula (csrc/replay_dev.cuh sample_body) on the trees as they were when
the batch was sampled, with beta from the Python LinearSchedule at that step, to one float32 ulp.  Power: beta at the
neighbouring steps must move some row's weight by more than IS_POWER_ULP ulp wherever the sampled priorities differ.
"""
import math

import numpy as np
import torch

F32 = np.float32
IS_POWER_ULP = 4
# the device's and the host's float64 pow may differ by this many ulp (CUDA documents 2 for pow)
POW_ULP = 4


def fma32(a, b, c):
    """float32 a * b + c with a single round-to-nearest-even, exactly.  The product of two float32 values is exact in
    float64, so only the float64 sum s can be inexact; it changes the float32 result only where s lies exactly on a
    float32 rounding midpoint, and there the TwoSum residual r (a * b + c = s + r) decides the direction."""
    a64, b64, c64 = (np.asarray(x, dtype=F32).astype(np.float64) for x in (a, b, c))
    p = a64 * b64
    s = p + c64
    bp = s - c64                          # TwoSum (Knuth): the part of s that came from p
    r = (c64 - (s - bp)) + (p - bp)
    f = s.astype(F32)
    f64 = f.astype(np.float64)
    other = np.nextafter(f, np.where(s > f64, F32(np.inf), F32(-np.inf)).astype(F32))
    o64 = other.astype(np.float64)
    on_mid = (s != f64) & (s == (f64 + o64) * 0.5)
    up = on_mid & (r != 0) & ((r > 0) == (o64 > f64))
    return np.where(up, other, f).astype(F32)


def scalar_candidates(x, amp=1.0):
    """([float32 values], near_midpoint) the device may hold for the float64 value x that it computed through pow:
    both neighbours when x is within POW_ULP * amp float64 ulp of a float32 rounding midpoint (amp: how much the
    expression amplifies a relative error of its pow), else float32(x) alone."""
    f = F32(x)
    if float(f) == x:
        return [f], False
    other = np.nextafter(f, F32(math.inf if x > float(f) else -math.inf))
    mid = (float(f) + float(other)) / 2
    if abs(x - mid) <= POW_ULP * amp * math.ulp(x):
        return [f, other], True
    return [f], False


class Hyper(object):
    """The update's float32 scalars, cast from the double expressions the learner uses (csrc/learner.cu, step 7)."""

    def __init__(self, lr, b1, b2, eps, tau):
        self.lr, self.b1, self.b2 = tuple(lr), b1, b2
        self.w1, self.w2, self.b2f, self.eps = F32(1.0 - b1), F32(1.0 - b2), F32(b2), F32(eps)
        self.tau, self.omt = F32(tau), F32(1.0 - tau)

    @classmethod
    def of(cls, dd):
        lr_a, b1, b2, eps = dd.optimizer_global_actor.hyper()
        lr_c = dd.optimizer_global_critic.hyper()[0]
        return cls((lr_a, lr_c), b1, b2, eps, float(dd.tau))

    def scalars(self, k, net):
        """[(nss, bc2s)] the device may use at step k for network `net` (0 actor, 1 critic), and how many of the two
        scalars lay near a float32 midpoint."""
        p1, p2 = self.b1 ** k, self.b2 ** k
        nss, e1 = scalar_candidates(-(self.lr[net] / (1.0 - p1)), max(1.0, p1 / (1.0 - p1)))
        bc2s, e2 = scalar_candidates(math.sqrt(1.0 - p2), max(1.0, p2 / (1.0 - p2)))
        return [(a, b) for a in nss for b in bc2s], int(e1) + int(e2)


def _bits(x):
    return np.ascontiguousarray(x, dtype=F32).view(np.uint32)


def differ(a, b):
    """Elements whose float32 bit patterns differ."""
    return _bits(a) != _bits(b)


def restate_m(h, g, m):
    return fma32(h.w1, g - m, m)


def restate_v(h, g, v):
    return (v * h.b2f) + ((h.w2 * g) * g)


def restate_p(h, p, m1, v1, nss, bc2s):
    denom = np.sqrt(v1) / bc2s + h.eps
    return p + nss * (m1 / denom)


def restate_t(h, t, p1, stale=False):
    if stale:
        return t.copy()
    return (h.omt * t) + (h.tau * p1)


NETS = (("actor", "actor_target"), ("critic", "critic_target"))


def pad_mask(net):
    """True on the padding elements of `net`'s flat layout (pitch columns and the gaps between tensors)."""
    m = torch.ones(net._total, dtype=torch.bool)
    for w, b in net._views(m):
        w.fill_(False)
        b.fill_(False)
    return m.numpy()


def read(dd, grads):
    """{net: {"p", "t", "m", "v"[, "g"]}} as float32 numpy copies of the flat device buffers."""
    torch.cuda.synchronize()
    g = dd._learner.global_model if dd._learner is not None else dd
    opts = (dd.optimizer_global_actor, dd.optimizer_global_critic)
    out = {}
    for i, (name, tname) in enumerate(NETS):
        net = getattr(g, name)
        m, v = opts[i].moments(net)
        d = {"p": net.flat_params(), "t": getattr(dd, tname).flat_params(), "m": m, "v": v}
        if grads:
            d["g"] = getattr(dd, name).flat_grads()
        out[name] = {k: x.detach().cpu().numpy().astype(F32, copy=True) for k, x in d.items()}
    return out


class Stats(object):
    """Counted over every checked step: scalar-midpoint exceptions and the smallest number of elements the k-1 / k+1 /
    stale-target restatements got wrong (the margin of the power check)."""

    def __init__(self):
        self.steps, self.midpoints, self.power_min = 0, 0, None
        self.is_steps, self.is_power_steps, self.is_worst_ulp, self.is_midpoints = 0, 0, 0, 0

    def power(self, n):
        self.power_min = n if self.power_min is None else min(self.power_min, n)

    def line(self):
        return ("%d update steps bit-exact, %d scalar-midpoint exceptions, fewest elements a k-1/k+1/stale restatement "
                "got wrong: %s; %d IS-weight steps, worst %d ulp, %d pow-midpoint exceptions, %d steps with power"
                % (self.steps, self.midpoints, self.power_min, self.is_steps, self.is_worst_ulp, self.is_midpoints,
                   self.is_power_steps))


def check_arrays(before, after, pads, h, k, stats=None, label=""):
    """The update of step k (1-based) from `before` to `after` (dicts of `read`; `pads` {net: pad_mask}).  Raises
    AssertionError naming every failed part."""
    stats = stats if stats is not None else Stats()
    bad = []
    for i, (name, _) in enumerate(NETS):
        b, a, pad = before[name], after[name], pads[name]
        for key in ("p", "g", "m", "v", "t"):
            n = int(np.count_nonzero(a[key][pad]))
            if n:
                bad.append("%s.%s: %d nonzero padding elements" % (name, key, n))
        with np.errstate(all="ignore"):
            for key, ref in (("m", restate_m(h, a["g"], b["m"])), ("v", restate_v(h, a["g"], b["v"]))):
                n = int(np.count_nonzero(differ(ref, a[key])))
                if n:
                    bad.append("%s.%s: %d elements differ from the restatement" % (name, key, n))
            cands, mids = h.scalars(k, i)
            stats.midpoints += mids
            if mids:
                print("%s step %d %s: a bias-correction scalar lies near a float32 midpoint; both neighbours accepted"
                      % (label, k, name))
            errs = [int(np.count_nonzero(differ(restate_p(h, b["p"], a["m"], a["v"], nss, bc2s), a["p"])))
                    for nss, bc2s in cands]
            if min(errs):
                bad.append("%s.p: %d elements differ from the restatement at step %d" % (name, min(errs), k))
            n = int(np.count_nonzero(differ(restate_t(h, b["t"], a["p"]), a["t"])))
            if n:
                bad.append("%s.t: %d elements differ from the restatement" % (name, n))
            # power: the neighbouring clocks and a stale target must be told apart from the device
            for kk in (k - 1, k + 1):
                if kk < 1:
                    continue
                nss, bc2s = h.scalars(kk, i)[0][0]
                n = int(np.count_nonzero(differ(restate_p(h, b["p"], a["m"], a["v"], nss, bc2s), a["p"])))
                stats.power(n)
                if n == 0:
                    bad.append("%s: the restatement at step %d (not %d) matches the device too" % (name, kk, k))
            n = int(np.count_nonzero(differ(restate_t(h, b["t"], a["p"], stale=True), a["t"])))
            stats.power(n)
            if n == 0:
                bad.append("%s: a stale target matches the device too" % name)
    stats.steps += 1
    assert not bad, "%s step %d: %s" % (label, k, "; ".join(bad))
    return stats


class UpdateCheck(object):
    """`UpdateCheck(dd)` before a step, `.check(dd, k)` after it."""

    def __init__(self, dd):
        self.h = Hyper.of(dd)
        self.before = read(dd, grads=False)
        g = dd._learner.global_model if dd._learner is not None else dd
        self.pads = {name: pad_mask(getattr(g, name)) for name, _ in NETS}

    def check(self, dd, k, stats=None, label=""):
        return check_arrays(self.before, read(dd, grads=True), self.pads, self.h, k, stats, label)


# ---- importance-sampling weights ---------------------------------------------------------------------------------------
def trees(dd):
    """(sum tree, min tree, len, capacity) of the replay as the next sample sees them (float32 numpy copies)."""
    torch.cuda.synchronize()
    st = dd.replayBuffer._store
    return st.sum_tree.cpu().numpy().copy(), st.min_tree.cpu().numpy().copy(), len(st), st.capacity


def schedule_beta(sch, t):
    """LinearSchedule.value() at clock t, without advancing it; as the device's clock_beta casts it."""
    return F32(sch.initial_p + min(float(t) / sch.schedule_timesteps, 1.0) * (sch.final_p - sch.initial_p))


def _pow_candidates(x, beta):
    """float32 of x ** -beta for a float32 array x, with both neighbours where the float64 pow lies near a midpoint."""
    y = np.power(x.astype(np.float64), -float(beta))
    f = y.astype(F32)
    f64 = f.astype(np.float64)
    other = np.nextafter(f, np.where(y > f64, F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (f64 + other.astype(np.float64)) * 0.5
    near = (y != f64) & (np.abs(y - mid) <= POW_ULP * np.spacing(np.abs(y)))
    return f, np.where(near, other, f), near


def restate_weights(tr, idx, beta):
    """The device's IS weights of leaves `idx` (csrc/replay_dev.cuh sample_body): [(weights, midpoint count)] for every
    combination of the pow neighbours."""
    s, mn, n_len, cap = tr
    tot = s[1]
    pmin = F32(mn[1] / tot)
    n = F32(n_len)
    ps = (s[cap + idx] / tot).astype(F32)
    mw0, mw1, mnear = _pow_candidates(np.asarray([pmin * n], dtype=F32), beta)
    w0, w1, near = _pow_candidates((ps * n).astype(F32), beta)
    out = []
    for mw in {float(mw0[0]), float(mw1[0])}:
        for w in (w0, w1):
            out.append((w / F32(mw)).astype(F32))
    return out, int(mnear.sum()) + int(near.sum())


def ulps(a, b):
    """|a - b| in float32 ulps (positive operands)."""
    return np.abs(_bits(a).astype(np.int64) - _bits(b).astype(np.int64))


def is_weight_check(tr, idx, weights, sch, t, stats=None, label=""):
    """The IS weights the device gave batch `idx` (sampled from trees `tr` at schedule clock t) to one ulp; returns
    whether beta at t - 1 / t + 1 is visible (only asked where the sampled priorities differ)."""
    stats = stats if stats is not None else Stats()
    idx = np.asarray(idx, dtype=np.int64)
    dev = np.asarray(weights, dtype=F32)
    with np.errstate(all="ignore"):
        cands, mids = restate_weights(tr, idx, schedule_beta(sch, t))
        err = np.min(np.stack([ulps(c, dev) for c in cands]), axis=0)
        stats.is_midpoints += mids
        worst = int(err.max())
        stats.is_worst_ulp = max(stats.is_worst_ulp, worst)
        stats.is_steps += 1
        assert worst <= 1, "%s clock %d: IS weights %d ulp from the restatement" % (label, t, worst)
        if bool(np.all(cands[0] == 1)):            # every sampled leaf at the minimum priority: beta is invisible
            return False
        for tt in (t - 1, t + 1):
            if tt < 0:
                continue
            off = int(ulps(restate_weights(tr, idx, schedule_beta(sch, tt))[0][0], dev).max())
            if off <= IS_POWER_ULP:
                return False
    stats.is_power_steps += 1
    return True
