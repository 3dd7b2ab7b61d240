"""The GPU-resident prioritized replay (csrc/replay.cu, csrc/replay_dev.cuh) restated on the device's own inputs and held
to bit-exactness: the sum/min trees after update_priorities and add, the sampler's indices, IS weights and gathers.

Snapshot, then check.  A `Snapshot` holds both trees (every node) and the device state record (`ReplayState`: f32
max_priority, i32 pristine, i64 len, i64 next_idx, u64 reserved -- the fast update's CTA ticket).

- Tree invariant, on every node of both trees: sum[i] == f32(sum[2i] + sum[2i+1]), min[i] == fmin(min[2i], min[2i+1]);
  the sum and min leaves are equal where written, and past the written leaves they are 0 and inf.
- update(idx, prio): every leaf not named in idx is bitwise unchanged; a named leaf holds
  f32(pow(f64(p_w), f64(f32(alpha)))) with w the LARGEST batch position naming it (the reference's sequential loop);
  max_priority = max(old, max(prio)), pristine = 0, the ticket back at 0.
- add(n): the ring positions (next_idx + i) % size hold one common leaf, pow_alpha(max_priority); every other leaf is
  unchanged; len and next_idx advance like the reference's.
- sample: indices bit-exact against the oracle's _sample_proportional on the same trees, IS weights within one float32
  ulp of the device formula (update_check.restate_weights).

Together with "unchanged elsewhere", the invariant on every node pins the whole tree: a wrong ancestor, a lost level
or a wrong duplicate winner all show.  Where the float64 pow lies within POW_ULP float64 ulp of a float32 midpoint the
device's pow and the host's may round apart; there both neighbours are accepted and the case is counted.
"""
import numpy as np

from tests import update_check as UC

F32 = np.float32
POW_ULP = UC.POW_ULP


def _bits(x):
    return np.ascontiguousarray(x, dtype=F32).view(np.uint32)


class Snapshot(object):
    """Both trees and the state record of one replay at one moment (host copies)."""

    def __init__(self, s, mn, max_priority, pristine, length, next_idx, reserved, size):
        self.s, self.mn = np.asarray(s, dtype=F32), np.asarray(mn, dtype=F32)
        self.cap = self.s.size // 2
        self.max_priority, self.pristine = F32(max_priority), int(pristine)
        self.len, self.next_idx, self.reserved, self.size = int(length), int(next_idx), int(reserved), int(size)

    def copy(self, **kw):
        d = dict(s=self.s.copy(), mn=self.mn.copy(), max_priority=self.max_priority, pristine=self.pristine,
                 length=self.len, next_idx=self.next_idx, reserved=self.reserved, size=self.size)
        d.update(kw)
        return Snapshot(**d)

    def trees(self):
        """(sum, min, len, capacity), as update_check.restate_weights takes them."""
        return self.s, self.mn, self.len, self.cap


def parse_state(raw):
    """The 32-byte ReplayState record (uint8 array) -> (max_priority, pristine, len, next_idx, reserved)."""
    raw = np.ascontiguousarray(raw, dtype=np.uint8)
    return (raw[0:4].view(F32)[0], int(raw[4:8].view(np.int32)[0]), int(raw[8:16].view(np.int64)[0]),
            int(raw[16:24].view(np.int64)[0]), int(raw[24:32].view(np.uint64)[0]))


def snapshot(store):
    """Snapshot of a _DeviceReplay after everything queued on it has finished."""
    import torch
    store.flush()
    torch.cuda.synchronize()
    mp, pr, ln, nx, rs = parse_state(store.state.view(torch.uint8).cpu().numpy())
    return Snapshot(store.sum_tree.cpu().numpy(), store.min_tree.cpu().numpy(), mp, pr, ln, nx, rs, store.size)


# ---- the device's arithmetic ---------------------------------------------------------------------------------------------
def pow_alpha(p, alpha):
    """(value, alternative, near) of the device's leaf pow_alpha(p, f32(alpha)) = f32(pow(f64(p), f64(f32(alpha)))) for a
    float32 array p: `alternative` is the other float32 neighbour where the float64 pow lies within POW_ULP float64 ulp
    of a rounding midpoint (`near`), else the value itself.  p == 1 gives exactly 1 either way."""
    p64 = np.asarray(p, dtype=F32).astype(np.float64)
    y = np.power(p64, float(F32(alpha)))
    f = y.astype(F32)
    f64 = f.astype(np.float64)
    other = np.nextafter(f, np.where(y > f64, F32(np.inf), F32(-np.inf)).astype(F32))
    mid = (f64 + other.astype(np.float64)) * 0.5
    near = (y != f64) & (np.abs(y - mid) <= POW_ULP * np.spacing(np.abs(y)))
    return f, np.where(near, other, f).astype(F32), near


def rebuild(s, mn):
    """Every internal node recomputed bottom-up from the leaves, in place (f32 add, fmin)."""
    c = s.size // 2
    while c > 1:
        h = c // 2
        s[h:c] = s[c:2 * c:2] + s[c + 1:2 * c:2]
        mn[h:c] = np.fmin(mn[c:2 * c:2], mn[c + 1:2 * c:2])
        c = h


def winners(idx):
    """(distinct leaves, batch position of each one's LAST writer)."""
    idx = np.asarray(idx, dtype=np.int64)
    u, first_rev = np.unique(idx[::-1], return_index=True)
    return u, idx.size - 1 - first_rev


def restate_update(before, idx, prio, alpha):
    """What update_priorities(idx, prio) leaves behind, as the device computes it (no midpoint alternatives)."""
    prio = np.asarray(prio, dtype=F32)
    a = before.copy(pristine=0, reserved=0, max_priority=F32(max(before.max_priority, prio.max())))
    u, w = winners(idx)
    leaf = pow_alpha(prio[w], alpha)[0]
    a.s[a.cap + u] = leaf
    a.mn[a.cap + u] = leaf
    rebuild(a.s, a.mn)
    return a


def add_positions(before, n):
    return (before.next_idx + np.arange(n, dtype=np.int64)) % before.size


def restate_add(before, n, alpha):
    """What an add of n rows leaves in the trees and the state record."""
    a = before.copy(length=min(before.size, max(before.len, before.next_idx + n)), next_idx=(before.next_idx + n) % before.size)
    pos = add_positions(before, n)
    leaf = pow_alpha(np.asarray([before.max_priority]), alpha)[0][0]
    a.s[a.cap + pos] = leaf
    a.mn[a.cap + pos] = leaf
    rebuild(a.s, a.mn)
    return a


# ---- checks --------------------------------------------------------------------------------------------------------------
class Stats(object):
    """Counted over every check: pow-midpoint exceptions, updates, adds and samples checked."""

    def __init__(self):
        self.midpoints = self.updates = self.adds = self.samples = 0

    def line(self):
        return ("%d updates, %d adds, %d samples bit-exact; %d pow-midpoint exceptions"
                % (self.updates, self.adds, self.samples, self.midpoints))


def invariant_problems(snap, written=None):
    """Every node of both trees against its children; leaves [0, written) equal in both trees, the rest 0 / inf."""
    s, mn, cap = snap.s, snap.mn, snap.cap
    written = snap.len if written is None else written
    bad = []
    c = cap
    while c > 1:
        h = c // 2
        ds = np.nonzero(_bits(s[h:c]) != _bits(s[c:2 * c:2] + s[c + 1:2 * c:2]))[0]
        dm = np.nonzero(_bits(mn[h:c]) != _bits(np.fmin(mn[c:2 * c:2], mn[c + 1:2 * c:2])))[0]
        for name, d in (("sum", ds), ("min", dm)):
            if d.size:
                bad.append("%s tree: %d nodes of level [%d, %d) are not op(children), first node %d"
                           % (name, d.size, h, c, h + int(d[0])))
        c = h
    if _bits(s[0:1])[0] != _bits(F32(0))[0] or mn[0] != np.inf:
        bad.append("node 0 (unused) was written")
    n = int(np.count_nonzero(_bits(s[cap:cap + written]) != _bits(mn[cap:cap + written])))
    if n:
        bad.append("%d written leaves differ between the sum and the min tree" % n)
    n = int(np.count_nonzero(_bits(s[cap + written:]) != 0) + np.count_nonzero(mn[cap + written:] != np.inf))
    if n:
        bad.append("%d leaves past the %d written ones are not 0 / inf" % (n, written))
    return bad


def check_invariant(snap, written=None, label=""):
    bad = invariant_problems(snap, written)
    assert not bad, "%s: %s" % (label, "; ".join(bad))


def _unchanged(before, after, keep, bad):
    """Leaves outside the named positions bitwise unchanged in both trees."""
    cap = before.cap
    for name, b, a in (("sum", before.s, after.s), ("min", before.mn, after.mn)):
        x = a[cap:].copy()
        x[keep] = b[cap:][keep]
        n = int(np.count_nonzero(_bits(x) != _bits(b[cap:])))
        if n:
            bad.append("%s tree: %d leaves that were not written changed" % (name, n))


def check_update(before, after, idx, prio, alpha, stats=None, label=""):
    """update_priorities(idx, prio) took the replay from `before` to `after`.  Raises AssertionError naming every failed
    part; returns the stats with the pow-midpoint exceptions counted."""
    stats = stats if stats is not None else Stats()
    idx = np.asarray(idx, dtype=np.int64)
    prio = np.asarray(prio, dtype=F32)
    cap = before.cap
    bad = []
    u, w = winners(idx)
    f, alt, near = pow_alpha(prio[w], alpha)
    stats.midpoints += int(near.sum())
    if near.any():
        print("%s: %d leaves lie within %d ulp of a float32 midpoint; both neighbours accepted" % (label, int(near.sum()), POW_ULP))
    got = after.s[cap + u]
    ok = (_bits(got) == _bits(f)) | (near & (_bits(got) == _bits(alt)))
    if not ok.all():
        k = int(np.nonzero(~ok)[0][0])
        bad.append("%d written leaves are not pow(p_w, alpha) of their last writer (leaf %d: %r, want %r)"
                   % (int((~ok).sum()), int(u[k]), float(got[k]), float(f[k])))
    _unchanged(before, after, u, bad)
    bad += invariant_problems(after, after.len)
    want_max = F32(max(before.max_priority, prio.max()))
    if _bits(after.max_priority) != _bits(want_max):
        bad.append("max_priority %r, want max(old, max(prio)) = %r" % (float(after.max_priority), float(want_max)))
    if after.pristine != 0:
        bad.append("pristine is %d after an update" % after.pristine)
    if after.reserved != 0:
        bad.append("the CTA ticket is %d, not back at 0" % after.reserved)
    if (after.len, after.next_idx) != (before.len, before.next_idx):
        bad.append("len / next_idx moved: (%d, %d) -> (%d, %d)" % (before.len, before.next_idx, after.len, after.next_idx))
    stats.updates += 1
    assert not bad, "%s: %s" % (label, "; ".join(bad))
    return stats


def check_add(before, after, n, alpha, stats=None, label=""):
    """An add of n rows took the replay from `before` to `after` (trees and state record)."""
    stats = stats if stats is not None else Stats()
    cap = before.cap
    bad = []
    pos = add_positions(before, n)
    f, alt, near = pow_alpha(np.asarray([before.max_priority]), alpha)
    stats.midpoints += int(near.sum())
    got = after.s[cap + pos]
    first = got[:1]
    if np.count_nonzero(_bits(got) != _bits(first[0])):
        bad.append("the %d new leaves are not one common value" % n)
    elif not (_bits(first)[0] == _bits(f)[0] or (near[0] and _bits(first)[0] == _bits(alt)[0])):
        bad.append("new leaf %r, want pow_alpha(max_priority %r) = %r" % (float(first[0]), float(before.max_priority), float(f[0])))
    _unchanged(before, after, pos, bad)
    want_len, want_next = min(before.size, max(before.len, before.next_idx + n)), (before.next_idx + n) % before.size
    if (after.len, after.next_idx) != (want_len, want_next):
        bad.append("device len / next_idx (%d, %d), want (%d, %d)" % (after.len, after.next_idx, want_len, want_next))
    bad += invariant_problems(after, after.len)
    if _bits(after.max_priority) != _bits(before.max_priority) or after.pristine != before.pristine:
        bad.append("add changed max_priority or pristine")
    if after.reserved != 0:
        bad.append("the CTA ticket is %d" % after.reserved)
    stats.adds += 1
    assert not bad, "%s: %s" % (label, "; ".join(bad))
    return stats


def _oracle(snap):
    """A PrioritizedReplayOracle whose sum tree, pristine flag and length are the snapshot's own."""
    from oracle import d4pg_oracle as O
    ob = O.PrioritizedReplayOracle.__new__(O.PrioritizedReplayOracle)
    ob.capacity, ob.length, ob.pristine = snap.cap, snap.len, bool(snap.pristine)
    ob.sum = O.SegmentTree32.__new__(O.SegmentTree32)
    ob.sum.capacity, ob.sum.kind, ob.sum.value = snap.cap, "sum", snap.s
    return ob


def oracle_indices(snap, uniforms):
    """PrioritizedReplayOracle.sample_indices on the snapshot's own trees."""
    return _oracle(snap).sample_indices(uniforms)


def sampling_total(snap):
    """sum(0, len - 1), the mass the sampler scales its uniforms by (float32)."""
    return _oracle(snap).sum.reduce_prefix(snap.len - 2)


def check_sample(snap, uniforms, idx, weights=None, beta=None, stats=None, label=""):
    """The sampler's indices (bit-exact) and IS weights (one ulp) for `uniforms` on the trees of `snap`."""
    stats = stats if stats is not None else Stats()
    idx = np.asarray(idx, dtype=np.int64)
    want = oracle_indices(snap, uniforms)
    d = np.nonzero(idx != want)[0]
    assert d.size == 0, "%s: %d of %d indices differ from the oracle (row %d: u=%r -> %d, want %d)" % (
        label, d.size, idx.size, int(d[0]) if d.size else -1, float(uniforms[d[0]]) if d.size else 0.0,
        int(idx[d[0]]) if d.size else -1, int(want[d[0]]) if d.size else -1)
    if weights is not None:
        with np.errstate(all="ignore"):
            cands, mids = UC.restate_weights(snap.trees(), want, F32(beta))
            err = np.min(np.stack([UC.ulps(c, np.asarray(weights, dtype=F32)) for c in cands]), axis=0)
        stats.midpoints += mids
        assert int(err.max()) <= 1, "%s: IS weights %d ulp from the restatement" % (label, int(err.max()))
    stats.samples += 1
    return stats


# ---- SegmentTree.reduce ----------------------------------------------------------------------------------------------
def reduce_helper(values, cap, start, end, op):
    """SegmentTree._reduce_helper (prioritized_replay_memory.py:61-96) over leaves [start, end] (inclusive), evaluated in
    float32 on a node array."""
    def rec(s, e, node, ns, ne):
        if s == ns and e == ne:
            return F32(values[node])
        mid = (ns + ne) // 2
        if e <= mid:
            return rec(s, e, 2 * node, ns, mid)
        if mid + 1 <= s:
            return rec(s, e, 2 * node + 1, mid + 1, ne)
        return op(rec(s, mid, 2 * node, ns, mid), rec(mid + 1, e, 2 * node + 1, mid + 1, ne))
    return rec(start, end, 1, 0, cap - 1)


def f32_add(a, b):
    return F32(F32(a) + F32(b))


def f32_min(a, b):
    return F32(np.fmin(F32(a), F32(b)))


def reduce_range(values, cap, start=0, end=None, op=f32_add):
    """SegmentTree.reduce(start, end): end None = capacity, a negative end counts from the capacity (:91-94)."""
    if end is None:
        end = cap
    if end < 0:
        end += cap
    return reduce_helper(values, cap, start, end - 1, op)
