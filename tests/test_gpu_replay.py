"""The GPU-resident prioritized replay held bit-exactly to tests/replay_check.py at every launch path: tree updates
(the one-thread-per-leaf fast kernel at every subtree split, the level-synchronous CTA), adds (the one-round-trip fast
range, the block-level range, the bulk fill + level rebuild; split at the ring end or not), the sampler's descent
(shared-memory top levels, three levels per L2 round trip, single levels; pristine fp64 and fp32 masses, edge
uniforms), the SegmentTree API, and the priority write-back of real learner steps.

Which kernel runs (csrc/replay.cu): update_priorities of n <= 512 leaves below capacity 2^24 runs
tree_update_fast_kernel on 2^D CTAs (D = min(4, log2 capacity)), otherwise tree_write_kernel<TREE_UPDATE>; an add
of <= 2048 contiguous rows runs tree_add_range_fast_kernel, up to 65536 rows tree_add_range_kernel (a wrapping add is
split in two), more rows leaf_fill_kernel + level_rebuild_kernel.  Every buffer stores the insertion number of a row in
obs[:, 0], so each gather is checked by identity.
"""
import random

import numpy as np
import pytest
import torch

from oracle import d4pg_oracle as O
from tests import helpers as H
from tests import replay_check as RC
from tests import update_check as UC

F32 = np.float32


# ---- CPU: the checker itself --------------------------------------------------------------------------------------------
def _fresh(cap, size):
    s = np.zeros(2 * cap, dtype=F32)
    mn = np.full(2 * cap, np.inf, dtype=F32)
    return RC.Snapshot(s, mn, 1.0, 1, 0, 0, 0, size)


def _filled(rng, cap=64, size=60, mp=1.5):
    """A replay of `size` rows with random leaves and a float32 max_priority, as an update leaves it."""
    b = _fresh(cap, size)
    leaves = rng.uniform(0.1, 2.0, size).astype(F32)
    b.s[cap:cap + size] = leaves
    b.mn[cap:cap + size] = leaves
    RC.rebuild(b.s, b.mn)
    return b.copy(max_priority=F32(mp), pristine=0, length=size, next_idx=size - 3)


def _rejects(fn, *args, **kw):
    with pytest.raises(AssertionError):
        fn(*args, **kw)


def test_update_check_passes_the_restatement_and_rejects_each_mutant():
    rng = np.random.RandomState(1)
    before = _filled(rng)
    cap = before.cap
    # a duplicated leaf (7) with different priorities, a sibling pair (10, 11), a priority above the max, exactly 1
    idx = np.array([7, 10, 11, 30, 7, 41, 7, 52], dtype=np.int64)
    prio = np.array([0.3, 0.9, 1.7, 1.0, 2.5, 0.05, 0.8, 3.0], dtype=F32)
    after = RC.restate_update(before, idx, prio, 0.6)
    st = RC.check_update(before, after, idx, prio, 0.6)
    assert st.midpoints == 0
    assert after.s[cap + 30] == 1.0 and after.max_priority == F32(3.0)

    first = before.copy()                                   # the first writer of leaf 7 wins
    first.s[cap:], first.mn[cap:] = after.s[cap:], after.mn[cap:]
    first.s[cap + 7] = first.mn[cap + 7] = RC.pow_alpha(prio[:1], 0.6)[0][0]
    RC.rebuild(first.s, first.mn)
    first = first.copy(max_priority=after.max_priority, pristine=0)
    assert first.s[cap + 7] != after.s[cap + 7]
    _rejects(RC.check_update, before, first, idx, prio, 0.6)

    for node in ((cap + 41) >> 1, 1):                       # one stale ancestor: the deepest level, the root
        stale = after.copy()
        assert stale.s[node] != before.s[node]
        stale.s[node] = before.s[node]
        _rejects(RC.check_update, before, stale, idx, prio, 0.6)
        stale = after.copy()
        stale.mn[1] = F32(before.mn[1] * 2)
        _rejects(RC.check_update, before, stale, idx, prio, 0.6)

    off = idx.copy()                                        # leaf 41 written at 42
    off[5] = 42
    _rejects(RC.check_update, before, RC.restate_update(before, off, prio, 0.6), idx, prio, 0.6)
    _rejects(RC.check_update, before, after.copy(max_priority=before.max_priority), idx, prio, 0.6)
    _rejects(RC.check_update, before, after.copy(pristine=1), idx, prio, 0.6)
    _rejects(RC.check_update, before, after.copy(reserved=15), idx, prio, 0.6)
    bump = after.copy()                                     # a leaf past len written
    bump.s[cap + 62] = bump.mn[cap + 62] = F32(1)
    RC.rebuild(bump.s, bump.mn)
    _rejects(RC.check_update, before, bump, idx, prio, 0.6)


def test_add_check_passes_the_restatement_and_rejects_unequal_new_leaves():
    rng = np.random.RandomState(2)
    before = _filled(rng)                                   # next_idx = size - 3: an add of 7 wraps
    after = RC.restate_add(before, 7, 0.6)
    RC.check_add(before, after, 7, 0.6)
    assert (after.len, after.next_idx) == (60, 4)
    cap = before.cap
    odd = after.copy()
    odd.s[cap + 2] = odd.mn[cap + 2] = np.nextafter(odd.s[cap + 2], F32(9))
    RC.rebuild(odd.s, odd.mn)
    _rejects(RC.check_add, before, odd, 7, 0.6)
    _rejects(RC.check_add, before, RC.restate_add(before, 6, 0.6), 7, 0.6)
    _rejects(RC.check_add, before, after.copy(next_idx=5), 7, 0.6)
    _rejects(RC.check_add, before, RC.restate_add(before.copy(max_priority=F32(1.25)), 7, 0.6), 7, 0.6)


def _descend_ge(snap, u):
    """A descent that goes left on `left >= mass`: off by one exactly where the mass lands on a left-subtree sum."""
    total = RC.sampling_total(snap)
    mass = F32(F32(u) * total)
    i = 1
    while i < snap.cap:
        left = snap.s[2 * i]
        if left >= mass:
            i = 2 * i
        else:
            mass = F32(mass - left)
            i = 2 * i + 1
    return i - snap.cap


def test_sample_check_rejects_an_index_off_by_one_at_a_tie():
    """Integer leaves with a power-of-two total: masses on left-subtree sums are exact, and a descent with the wrong
    comparison is caught there; IS weights two ulp off are caught too."""
    cap, n = 32, 29
    b = _fresh(cap, cap)
    leaves = np.array([1, 3, 2, 2, 4, 1, 1, 2] * 4, dtype=F32)[:n]
    leaves[n - 2] += F32(64 - leaves[:n - 1].sum())        # sum(0, len - 1) = 64
    b.s[cap:cap + n] = b.mn[cap:cap + n] = leaves
    RC.rebuild(b.s, b.mn)
    b = b.copy(length=n, pristine=0)
    assert RC.sampling_total(b) == 64
    us = np.array([4 / 64, 8 / 64, 16 / 64, 32 / 64, 0.0, 0.3, 1 - 2 ** -53], dtype=np.float64)
    want = RC.oracle_indices(b, us)
    w = UC.restate_weights(b.trees(), want, F32(0.4))[0][0]
    RC.check_sample(b, us, want, w, 0.4)
    wrong = np.array([_descend_ge(b, u) for u in us])
    assert np.count_nonzero(wrong != want) >= 3
    _rejects(RC.check_sample, b, us, wrong)
    w2 = w.copy()
    w2[1] = np.nextafter(np.nextafter(w2[1], F32(9)), F32(9))
    _rejects(RC.check_sample, b, us, want, w2, 0.4)


def _segment_leaves(cap, seed):
    """Non-integer leaves over 16 binades: the association of a range sum decides its last bits."""
    rng = np.random.RandomState(seed)
    return (rng.uniform(1, 2, cap) * 2.0 ** rng.randint(-8, 8, cap)).astype(F32)


def _cover_reduce(values, cap, s, e, right_left_nested):
    """SegmentTree.reduce over leaves [s, e] as a node cover; the reference nests the right part to the right."""
    node, lo, hi = 1, 0, cap - 1
    while True:
        if s == lo and e == hi:
            return F32(values[node])
        mid = (lo + hi) // 2
        if e <= mid:
            node, hi = 2 * node, mid
        elif s > mid:
            node, lo = 2 * node + 1, mid + 1
        else:
            break
    left = RC.reduce_helper(values, cap, s, mid, RC.f32_add)
    terms, nd, l2, h2 = [], 2 * node + 1, mid + 1, hi
    while e != h2:
        m2 = (l2 + h2) // 2
        if e <= m2:
            nd, h2 = 2 * nd, m2
        else:
            terms.append(values[2 * nd])
            nd, l2 = 2 * nd + 1, m2 + 1
    terms.append(values[nd])
    if right_left_nested:
        right = F32(terms[0])
        for t in terms[1:]:
            right = RC.f32_add(right, t)
    else:
        right = F32(terms[-1])
        for t in reversed(terms[:-1]):
            right = RC.f32_add(t, right)
    return RC.f32_add(left, right)


def test_reduce_restatement_is_the_reference_association():
    """reduce_helper equals the oracle's prefix reduction and the node-cover form of _reduce_helper on every range of
    the capacity-32 leaves the GPU test uses; a left-nested right part differs on some of them."""
    cap = 32
    t = O.SegmentTree32(cap, "sum")
    t.value[cap:] = _segment_leaves(cap, 0)
    t.rebuild()
    v = t.value
    nested = 0
    for s in range(cap):
        for e in range(s + 1, cap + 1):
            r = RC.reduce_range(v, cap, s, e)
            assert r == _cover_reduce(v, cap, s, e - 1, False), (s, e)
            if s == 0:
                assert r == t.reduce_prefix(e - 1), e
            nested += int(r != _cover_reduce(v, cap, s, e - 1, True))
    assert nested >= 10, nested
    assert RC.reduce_range(v, cap, 3, None) == RC.reduce_range(v, cap, 3, cap)
    assert RC.reduce_range(v, cap, 3, -2) == RC.reduce_range(v, cap, 3, cap - 2)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def d4pg():
    import d4pg_b200
    return d4pg_b200


def _id_rows(rng, n, first, S, A):
    """n transitions whose obs[:, 0] is their insertion number."""
    s = rng.randn(n, S).astype(F32)
    s[:, 0] = np.arange(first, first + n, dtype=np.float64)
    return (s, rng.uniform(-1, 1, (n, A)).astype(F32), rng.randn(n), rng.randn(n, S).astype(F32), rng.rand(n) < 0.3)


class Ring(object):
    """A PrioritizedReplayBuffer driven through its public API, every operation checked against the snapshot before it."""

    def __init__(self, d4pg, size, alpha, S=2, A=1, seed=0, stats=None):
        self.buf = d4pg.PrioritizedReplayBuffer(size, alpha=alpha, obs_dim=S, act_dim=A)
        self.st = self.buf._store
        self.size, self.alpha, self.S, self.A = size, alpha, S, A
        self.rng = np.random.RandomState(seed)
        self.stats = stats if stats is not None else RC.Stats()
        self.ids = np.full(size, -1, dtype=np.int64)           # insertion number of the row at each position
        self.n_added = 0
        self.snap = RC.snapshot(self.st)
        RC.check_invariant(self.snap, 0, "fresh buffer")
        assert self.snap.pristine == 1 and self.snap.max_priority == 1 and self.snap.len == 0

    def add(self, n, how="device", label=""):
        before = self.snap
        rows = _id_rows(self.rng, n, self.n_added, self.S, self.A)
        if how == "host":                                     # numpy: the packed single-copy path up to 4096 rows
            self.buf.add_batch(*rows)
        elif how == "device":
            self.buf.add_batch(*[torch.from_numpy(np.ascontiguousarray(x)).cuda() for x in rows])
        else:                                                 # add(): staged rows, flushed 4096 at a time
            for i in range(n):
                self.buf.add(rows[0][i], rows[1][i], float(rows[2][i]), rows[3][i], bool(rows[4][i]))
        after = RC.snapshot(self.st)
        label = "%s add %d at %d via %s" % (label, n, before.next_idx, how)
        RC.check_add(before, after, n, self.alpha, self.stats, label)
        pos = RC.add_positions(before, n)
        p = torch.from_numpy(pos).cuda()
        for name, dev, want in zip(("obs", "act", "rew", "obs2", "done"),
                                   (self.st.obs, self.st.act, self.st.rew, self.st.obs2, self.st.done), rows):
            got = dev[p].cpu().numpy()
            assert np.array_equal(got, np.asarray(want).astype(got.dtype).reshape(got.shape)), "%s: stored %s" % (label, name)
        self.ids[pos] = np.arange(self.n_added, self.n_added + n)
        self.n_added += n
        from d4pg_b200 import _lib
        lib = _lib.lib()
        host = (len(self.buf), self.buf._next_idx)
        abi = (int(lib.d4pg_replay_len(self.st.handle)), int(lib.d4pg_replay_next_idx(self.st.handle)))
        assert host == abi == (after.len, after.next_idx), "%s: len / next_idx host %s, library %s, device %s" % (
            label, host, abi, (after.len, after.next_idx))
        self.snap = after

    def seek(self, target, label=""):
        """Add rows until the next add starts at ring position `target`."""
        k = (target - self.snap.next_idx) % self.size
        if k:
            self.add(k, "device", label)

    def update(self, idx, prio, label=""):
        before = self.snap
        self.buf.update_priorities(np.asarray(idx, dtype=np.int64), np.asarray(prio, dtype=F32))
        after = RC.snapshot(self.st)
        RC.check_update(before, after, idx, prio, self.alpha, self.stats, "%s update n=%d" % (label, len(idx)))
        self.snap = after

    def sample(self, B, uniforms=None, philox=None, beta=0.4, label=""):
        o = self.st.sample_proportional(B, beta, uniforms=uniforms, philox=philox)
        if philox is not None:
            uniforms = [H.philox_uniform53(philox[0], philox[1], i) for i in range(B)]
        idx = o["idx"].cpu().numpy().astype(np.int64)
        RC.check_sample(self.snap, np.asarray(uniforms, dtype=np.float64), idx, o["w"].cpu().numpy(), beta, self.stats,
                        "%s sample B=%d len=%d" % (label, B, self.snap.len))
        s = o["s"].cpu().numpy()
        # a position never written holds a zero row: its id column reads 0
        assert np.array_equal(s[:, 0].astype(np.int64), np.maximum(self.ids[idx], 0)), label
        p = torch.from_numpy(idx).cuda()
        for key, dev in (("s", self.st.obs), ("a", self.st.act), ("r", self.st.rew), ("s2", self.st.obs2), ("d", self.st.done)):
            assert torch.equal(o[key].reshape(dev[p].shape), dev[p]), "%s: gathered %s" % (label, key)


def _prio(rng, n, mp):
    """Random priorities, every 7th exactly 1, one above the current max_priority."""
    p = rng.uniform(0.05, 2.0, n).astype(F32)
    p[::7] = 1.0
    p[rng.randint(n)] = F32(float(mp) + 0.25)
    return p


def _patterns(rng, L, n, log2cap):
    """(name, indices) of n updated leaves among the L stored ones."""
    D = min(4, log2cap)
    sub = 1 << (log2cap - D)                                   # leaves per top-level subtree of the fast kernel
    subs = [c for c in range(1 << D) if c * sub < L]
    yield "distinct", rng.choice(L, n, replace=n > L)
    yield "equal", np.full(n, rng.randint(L))
    if L >= 2:
        ev = 2 * rng.randint(0, L // 2, (n + 1) // 2)
        yield "siblings", np.stack([ev, ev + 1], 1).reshape(-1)[:n]
    c = subs[rng.randint(len(subs))]
    yield "one subtree", rng.randint(c * sub, min(L, (c + 1) * sub), n)
    yield "every subtree", np.resize(np.array([rng.randint(c * sub, min(L, (c + 1) * sub)) for c in subs]), n)
    yield "duplicates", rng.randint(0, max(1, min(L, n // 4)), n)


ALL_N = (1, 31, 32, 33, 511, 512, 513, 1024, 4096)
UPDATE_CASES = [(cap, cap, alpha, ALL_N) for cap in (1, 2, 4, 8, 16, 1 << 11, 1 << 20) for alpha in (0.6, 1.0, 0.0)]
UPDATE_CASES += [(1 << 23, 1 << 23, 0.6, (1, 33, 512, 4096)),          # the deepest tree of the fast kernel
                 (1 << 24, (1 << 23) + 1, 0.6, (1, 512))]               # log2 capacity 24: the CTA kernel at any n


@pytest.mark.gpu
@pytest.mark.parametrize("cap,size,alpha,ns", UPDATE_CASES,
                         ids=["cap%d-size%d-alpha%g" % c[:3] for c in UPDATE_CASES])
def test_update_priorities_every_launch_path(d4pg, cap, size, alpha, ns):
    """update_priorities at n on both sides of the fast kernel's 512, at capacities with D < 4 top-level subtrees, 16,
    and the deepest fast and the first CTA-kernel tree; indices distinct, all equal, sibling pairs, inside one subtree,
    one per subtree and heavy duplicates with different priorities: every node of both trees, max_priority, pristine
    and the CTA ticket after each."""
    S = A = 1 if cap > (1 << 20) else 2
    ring = Ring(d4pg, size, alpha, S, A, seed=cap + int(10 * alpha))
    ring.add(size, "device", "fill")
    rng = np.random.RandomState(cap)
    log2cap = cap.bit_length() - 1
    for n in ns:
        for name, idx in _patterns(rng, size, n, log2cap):
            ring.update(idx, _prio(rng, n, ring.snap.max_priority), "cap %d %s" % (cap, name))
    print(ring.stats.line())
    assert ring.stats.midpoints == 0


ADD_SIZES = (5, 3000, 100003)
ADD_N = (1, 2, 33, 2047, 2048, 2049, 65536, 65537)


@pytest.mark.gpu
@pytest.mark.parametrize("how", ["host", "device", "add"])
def test_add_every_path_start_and_size(d4pg, how):
    """Adds of every size class (fast range, block range, bulk fill) and n = size, starting at 0, at odd and even
    positions and just before the ring end (split in two), into buffers whose size is not a power of two; before any
    update (new leaf 1) and after one (new leaf pow(max_priority, alpha) of a float32 max_priority)."""
    stats = RC.Stats()
    for size in ADD_SIZES:
        ring = Ring(d4pg, size, 0.6, seed=size, stats=stats)
        rng = np.random.RandomState(size)
        ns = sorted({n for n in ADD_N if n <= size} | {size})
        if how == "add":                                       # row by row: keep it to what one staging flush holds
            ns = [n for n in ns if n <= 2049 or n == size <= 4096]
        for phase in ("pristine", "updated"):
            if phase == "updated":
                L = ring.snap.len
                ring.update(rng.choice(L, min(L, 64), replace=False), _prio(rng, min(L, 64), ring.snap.max_priority))
                assert ring.snap.max_priority > 1
            for k, n in enumerate(ns):
                first = (0, 2 * rng.randint(1, max(2, size // 2)), 2 * rng.randint(0, max(1, size // 2)) + 1)[k % 3]
                starts = [first % size]
                if n > 1:
                    starts.append(size - (n + 1) // 2)           # just before the ring end: split in two
                for start in starts:
                    ring.seek(start % size, "size %d" % size)
                    ring.add(n, how, "size %d %s" % (size, phase))
    print(stats.line())
    assert stats.midpoints == 0


SAMPLE_CAPS = (2, 4, 1 << 10, 1 << 11, 1 << 12, 1 << 13, 1 << 14, 1 << 20)
EDGE_U = [0.0, 1 - 2.0 ** -53, 1 - 2.0 ** -25, 1 - 2.0 ** -26, 1 - 2.0 ** -30, 1 - 2.0 ** -24, 0.5, 2.0 ** -40]


def _int_prio(rng, L):
    """Integer priorities whose sum over leaves [0, L - 1) -- the sampled mass -- is a power of two."""
    p = rng.randint(1, 5, L).astype(np.int64)
    if L > 1:
        head = p[:L - 1]
        diff = (1 << int(np.ceil(np.log2(head.sum())))) - int(head.sum())
        head += diff // (L - 1)
        head[:diff % (L - 1)] += 1
    return p.astype(F32)


def _uniforms(rng, snap, B, k):
    """B uniforms: the edges, masses exactly on left-subtree sums (exact when the total is a power of two), random."""
    total = float(RC.sampling_total(snap))
    L, cap = snap.len, snap.cap
    leaves = snap.s[cap:cap + L].astype(np.float64)
    pre = np.concatenate([[0.0], np.cumsum(leaves)])
    bounds = []
    for m in range(int(np.log2(cap)) + 1):
        j = (rng.randint(0, max(1, (L - 1) >> m) + 1, 4) << m)
        bounds += [pre[x] / total for x in j if 0 < x < L - 1]
    pool = EDGE_U + bounds
    if B >= len(pool):
        return np.concatenate([pool, rng.rand(B - len(pool))])
    return np.array([pool[(k * B + i) % len(pool)] for i in range(B)])


@pytest.mark.gpu
@pytest.mark.parametrize("cap", SAMPLE_CAPS)
def test_sample_descent_edges(d4pg, cap):
    """Proportional sampling at capacities on both sides of the 11 shared-memory levels and every remainder of the
    three-level unroll; len 2, a partial fill with a power-of-two mass, full; B 1, 31, 32, 33, 4096 and Philox draws
    at a nonzero counter; pristine trees (fp64 descent), integer priorities at alpha 1 (masses exactly on left-subtree
    sums) and real ones (fp32 descent).  Indices bit-exact, IS weights within one ulp, gathers by identity."""
    stats = RC.Stats()
    for L in sorted({2, cap // 2 + 1, cap}):
        ring = Ring(d4pg, cap, 1.0, seed=cap + L, stats=stats)
        ring.add(L, "device")
        rng = np.random.RandomState(L)
        for k, tree in enumerate(("pristine", "integer", "real")):
            if tree == "integer":
                ring.update(np.arange(L), _int_prio(rng, L), "integer")
                tot = float(RC.sampling_total(ring.snap))
                assert tot == 2.0 ** round(np.log2(tot)), tot
            elif tree == "real":
                ring.update(np.arange(L), rng.uniform(0.01, 3.0, L).astype(F32), "real")
            label = "cap %d len %d %s" % (cap, L, tree)
            for B in (1, 31, 32, 33, 4096):
                ring.sample(B, _uniforms(rng, ring.snap, B, k), label=label)
            ring.sample(257, philox=(0x5EED + cap, 11 + k), beta=0.7, label=label + " philox")
        del ring
    print(stats.line())
    assert stats.midpoints == 0


def _set_leaves(d4pg, tree, vals):
    from d4pg_b200 import _lib
    st = tree._store
    v = torch.from_numpy(vals).cuda()
    i = torch.arange(vals.size, dtype=torch.int32, device="cuda")
    _lib.check(_lib.lib().d4pg_replay_set_leaves(st.handle, vals.size, _lib.ptr(i), _lib.ptr(v), _lib.ptr(v),
                                                 _lib.stream_ptr()), "d4pg_replay_set_leaves")


@pytest.mark.gpu
def test_segment_tree_reduce_every_range(d4pg):
    """SumSegmentTree / MinSegmentTree at capacity 32: reduce, sum and min over every (start, end), end = None and
    negative ends, against _reduce_helper restated on the device's own nodes (non-integer leaves: the association shows)."""
    cap = 32
    leaves = _segment_leaves(cap, 0)
    t, mt = d4pg.SumSegmentTree(cap), d4pg.MinSegmentTree(cap)
    for i, x in enumerate(leaves):
        t[i] = float(x)
        mt[i] = float(x)
    for tree in (t, mt):
        snap = RC.snapshot(tree._store)
        RC.check_invariant(snap, cap, "SegmentTree")
        assert np.array_equal(snap.s[cap:], leaves)
    v, vm = RC.snapshot(t._store).s, RC.snapshot(mt._store).mn
    for s in range(cap):
        for e in list(range(s + 1, cap + 1)) + [None] + [x for x in (-1, -5, -16) if s < cap + x]:
            want, want_m = RC.reduce_range(v, cap, s, e), RC.reduce_range(vm, cap, s, e, RC.f32_min)
            assert t.sum(s, e) == want and t.reduce(s, e) == want, (s, e)
            assert mt.min(s, e) == want_m and mt.reduce(s, e) == want_m, (s, e)


@pytest.mark.gpu
def test_segment_tree_large_ranges_and_prefix_search(d4pg):
    """Capacity 2^20: reduce over random ranges and the edges (start = end - 1, end = None, negative end), and
    find_prefixsum_idx at 0, the total, exact left-subtree sums and random masses, on the device's own nodes."""
    cap = 1 << 20
    rng = np.random.RandomState(6)
    leaves = _segment_leaves(cap, 7)
    t = d4pg.SumSegmentTree(cap)
    _set_leaves(d4pg, t, leaves)
    snap = RC.snapshot(t._store)
    RC.check_invariant(snap, cap, "SegmentTree 2^20")
    v = snap.s
    ranges = [(int(a), int(b)) for a, b in np.sort(rng.randint(0, cap + 1, (120, 2)), axis=1) if a < b]
    ends = rng.randint(1, cap + 1, 40)
    ranges += [(int(e) - 1, int(e)) for e in ends] + [(int(s), None) for s in rng.randint(0, cap, 20)]
    ranges += [(int(s), -int(k)) for s, k in zip(rng.randint(0, cap // 2, 20), rng.randint(1, cap // 2, 20))]
    ranges += [(0, None), (0, cap), (cap - 1, None), (0, -1), (cap // 2, cap // 2 + 1)]
    for s, e in ranges:
        assert t.sum(s, e) == RC.reduce_range(v, cap, s, e), (s, e)
    total = float(v[1])
    pre = np.cumsum(leaves.astype(np.float64))
    masses = [0.0, total, float(v[2]), float(v[2] + v[6])] + list(rng.rand(30) * total)
    masses += [float(pre[(int(j) << m) - 1]) for m, j in zip(rng.randint(4, 19, 30), rng.randint(1, 8, 30))
               if (int(j) << m) <= cap // 2]
    for mass in masses:
        assert t.find_prefixsum_idx(mass) == O.find_prefixsum_idx(v, cap, F32(mass)), mass


# ---- the learner step's priority write-back ------------------------------------------------------------------------------
def _cat(N, v=(-50.0, 0.0)):
    return {"type": "categorical", "v_min": v[0], "v_max": v[1], "n_atoms": N}


def _learner(d4pg, B, mem, info, fill=None, S=17, A=6, seed=5, **kw):
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    dd = d4pg.DDPG(S, A, memory_size=mem, batch_size=B, critic_dist_info=info, precision="tf32x3", **kw)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    dd.replayBuffer.add_batch(*_id_rows(np.random.RandomState(seed + 1), fill or mem, 0, S, A))
    return dd


LEARNER_CASES = {
    "bench_c2": None,                                                          # fast kernel, D = 4, prefetch, graph
    "b512_m4096": (512, 4096, _cat(51), dict(sampling="device", philox_seed=3)),
    "b513_m4096": (513, 4096, _cat(51), dict(sampling="device", philox_seed=3)),     # the CTA kernel
    "b4096_m1024_c5": (4096, 1024, _cat(101, (-150.0, 150.0)),                       # ~4 writers per leaf
                       dict(sampling="device", philox_seed=4, projection="nstep", n_steps=5)),
    "m6_b32": (32, 6, _cat(51), dict(sampling="device", philox_seed=5)),              # capacity 8: D = 3
    "host_pipeline": (64, 1024, _cat(51), dict(sampling="reference", prefetch=True, use_graph=True)),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(LEARNER_CASES))
def test_learner_step_priority_write_back(d4pg, name):
    """Each train() writes |td| + eps back into the trees: from a snapshot taken before the step, the checker's update
    with the step's own idx and prio must give every node of both trees.  The host pipeline also adds pinned rows
    between steps (its ingest gate is opened by the write-back)."""
    stats = RC.Stats()
    if LEARNER_CASES[name] is None:
        from tests import test_gpu_update as TU
        dd = TU._bench_c2(d4pg)
    else:
        B, mem, info, kw = LEARNER_CASES[name]
        dd = _learner(d4pg, B, mem, info, **kw)
    st = dd.replayBuffer._store
    rng = np.random.RandomState(9)
    for t in range(3):
        if name == "host_pipeline":
            before = RC.snapshot(st)
            rows = _id_rows(rng, 96, 1024 + 96 * t, 17, 6)
            dd.replayBuffer.add_batch(*[torch.from_numpy(np.ascontiguousarray(x)).pin_memory() for x in rows])
            RC.check_add(before, RC.snapshot(st), 96, 0.6, stats, "%s add before step %d" % (name, t))
        before = RC.snapshot(st)
        random.seed(40 + t)
        dd.train()
        info = dd.last_batch_info()
        idx, prio = info["idx"].cpu().numpy(), info["prio"].cpu().numpy()
        RC.check_update(before, RC.snapshot(st), idx, prio, 0.6, stats, "%s step %d" % (name, t))
    print(name, stats.line())
    assert stats.midpoints == 0


@pytest.mark.gpu
def test_learner_uniform_device_sampling(d4pg):
    """A non-prioritized learner with sampling="device" draws row min(floor(u * len), len - 1), u = Philox(seed, step,
    row): the gathered batch must be those rows (checked by the insertion number in obs[:, 0]) on a partial fill."""
    seed, B, mem, L = 0xABCDEF, 256, 4096, 3001
    dd = _learner(d4pg, B, mem, _cat(51), fill=L, sampling="device", philox_seed=seed, prioritized_replay=False)
    assert len(dd.replayBuffer) == L
    for t in range(3):
        dd.train()
        us = [H.philox_uniform53(seed, t, i) for i in range(B)]
        want = np.array([min(int(u * L), L - 1) for u in us])
        s = dd.debug_tensor("s", (B, 17)).cpu().numpy()
        assert np.array_equal(s[:, 0].astype(np.int64), want), "step %d: gathered rows are not floor(u * len)" % t
        assert np.array_equal(dd.last_batch_info()["idx"].cpu().numpy(), want)
