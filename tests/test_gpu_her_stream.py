"""Streaming hindsight relabelling on the device (ReplayBuffer / PrioritizedReplayBuffer / Replay.add_goal_steps and
DDPG.observe_goals, DESIGN.md §3 "Streaming hindsight relabelling"): every ring row bit-exact against the oracle
(tests/her_stream_oracle.py) over environment counts, both her_action values, host and CUDA end flags, all three buffer
classes, flushes and ring wraps inside one call; len() / _next_idx against the device state after every call; the PER
trees and the normalizer's statistics against add_batch of the oracle's rows and tests/obs_norm_oracle.py; E = 1
against add_her_episode; horizons cleared; drop_goal_steps(); a learner fed by observe_goals against one fed the
oracle's rows; the launches per call; and the widest launch, E = 4096 at Fetch shapes with every episode ending at once."""
import numpy as np
import pytest
import torch

from tests import her_stream_oracle as HO
from tests import obs_norm_oracle as NO

pytestmark = pytest.mark.gpu

INFO = {"type": "categorical", "v_min": -10.0, "v_max": 0.0, "n_atoms": 51}


def _make(kind, size, S, A, **kw):
    import d4pg_b200 as d4pg
    if kind == "per":
        return d4pg.PrioritizedReplayBuffer(size, 0.6, obs_dim=S, act_dim=A, **kw)
    if kind == "uniform":
        return d4pg.ReplayBuffer(size, obs_dim=S, act_dim=A, **kw)
    return d4pg.Replay(size, None, obs_dim=S, act_dim=A, **kw)


def _cuda(c):
    return None if c is None else tuple(None if x is None else torch.as_tensor(x).cuda() for x in c)


def _device_len(store):
    torch.cuda.synchronize()
    st = store.state.view(torch.int64).cpu().numpy()
    return int(st[1]), int(st[2])


def _feed(buf, calls, on_dev, **her):
    """Every call (None: flush_goal_steps()) -> rows returned; len() and _next_idx checked against the device."""
    out = []
    store = buf._store
    for c in calls:
        if c is None:
            got = buf.flush_goal_steps()
        else:
            got = buf.add_goal_steps(*(_cuda(c) if on_dev else c), **her)
        out.append(got)
        if store.handle is not None:
            assert (len(buf), store._next_idx) == _device_len(store)
    return out


def _ring(rows, size):
    """The ring after inserting the rows {s, a, r, s2, d} in order: row i at i % size (s / s2 cast to f32)."""
    m = len(rows["r"])
    lo = max(0, m - size)
    pos = np.arange(lo, m) % size
    order = np.argsort(pos)
    return {k: (v[lo:].astype(np.float32) if k in ("s", "s2") else v[lo:])[order] for k, v in rows.items()}


def _check_ring(store, want, n):
    torch.cuda.synchronize()
    got = dict(s=store.obs[:n].cpu().numpy(), a=store.act[:n].cpu().numpy(), r=store.rew[:n].cpu().numpy(),
               s2=store.obs2[:n].cpu().numpy(), d=store.done[:n].cpu().numpy().astype(bool))
    for k in ("s", "a", "s2", "d"):
        assert np.array_equal(got[k], want[k]), k
    assert np.array_equal(got["r"].view(np.int64), want["r"].view(np.int64)), "r"      # -0.0 included


def _pick_size(counts, floor):
    """A ring size >= floor that one call's rows straddle (rows before it + half of its own)."""
    cum = 0
    for c in counts:
        if c >= 2 and cum + c // 2 >= floor:
            return cum + c // 2
        cum += c
    return None


CASES = [(E, act, flags, kind) for E in (1, 7, 300) for act in ("reference", "own") for flags in ("host", "cuda")
         for kind in ("uniform", "per", "replay")]


@pytest.mark.parametrize("E,her_action,flags,kind", CASES, ids=["E%d-%s-%s-%s" % c for c in CASES])
def test_vs_oracle(E, her_action, flags, kind):
    """Every ring row bit-exact (s, a, f64 r with its sign, s2, done) against the oracle; episodes of 1 to exactly
    max_episode_steps steps, terminated and truncated; two flushes; one call's rows straddle the ring's end.  The
    return values equal the oracle's row counts; with PER the trees and max_priority equal a buffer fed the oracle's
    rows by add_batch at the same points.  At E = 7 the normalizer's statistics equal the oracle's fold."""
    So, G, A = 5, 3, 2
    M = {1: 9, 7: 6, 300: 6}[E]
    rng = np.random.RandomState(E * 13 + len(her_action) + len(kind))
    K = {1: 80, 7: 40, 300: 24}[E]
    calls = HO.random_calls(rng, K, E, So, G, A, M, flush_at=(K // 3, K // 3 + 1, 2 * K // 3))
    her = dict(her_ratio=0.8, threshold=0.05, her_action=her_action, max_episode_steps=M, seed=E + 1)
    rows = HO.stream_rows(calls, her["her_ratio"], her["threshold"], her_action, her["seed"])
    counts = [len(r["r"]) for r in rows]
    size = _pick_size(counts, E * 2 * M)
    assert size is not None and sum(counts) > size
    norm = E == 7
    buf = _make(kind, size, So + G, A, obs_norm=norm)
    assert _feed(buf, calls, flags == "cuda", **her) == counts
    allrows = HO.concat(rows)
    _check_ring(buf._store, _ring(allrows, size), size)
    if kind == "per":
        ref = _make(kind, size, So + G, A)
        for r in rows:
            if len(r["r"]):
                ref.add_batch(*(torch.as_tensor(r[k].astype(np.float32) if k in ("s", "s2") else r[k]).cuda()
                                for k in ("s", "a", "r", "s2", "d")))
        torch.cuda.synchronize()
        for name in ("sum_tree", "min_tree", "state"):
            assert torch.equal(getattr(buf._store, name), getattr(ref._store, name)), name
    if norm:
        st = NO.Stats(So + G).fold(allrows["s"].astype(np.float32))
        on = buf._store.obs_norm
        assert np.array_equal(on.stats.cpu().numpy(), st.packed())
        shift, scale = st.affine()
        assert np.array_equal(on.affine.cpu().numpy(), np.concatenate([shift, scale]))


def test_e1_equals_add_her_episode():
    """One environment, one episode: the rows add_goal_steps stores equal add_her_episode's for the same select /
    future draws (fed to add_her_episode through a stand-in for np.random), for both her_action values."""
    So, G, A, M = 6, 3, 2, 12
    rng = np.random.RandomState(5)
    for her_action in ("reference", "own"):
        for T in (1, 7, M):
            calls = HO.random_calls(rng, T, 1, So, G, A, M)
            term = np.zeros((T, 1), bool)
            term[-1] = True
            calls = [c[:6] + (term[k], None) for k, c in enumerate(calls)] + [None]
            a = _make("per", 64, So + G, A)
            got = _feed(a, calls, False, her_action=her_action, max_episode_steps=M, seed=3)
            sel, fut = HO.draws(np.random.default_rng(3), [T], 0.8)

            class Draws:
                i = j = 0

                def uniform(self):
                    self.i += 1
                    return 0.0 if sel[self.i - 1] else 1.0

                def randint(self, lo, hi):
                    assert sel[lo] and hi == T
                    return int(fut[lo])
            b = _make("per", 64, So + G, A)
            X = [np.stack([c[i][0] for c in calls[:-1]]) for i in range(7)]
            n = b.add_her_episode(X[0], X[4], X[1], X[5], X[2], X[3], X[6], her_ratio=0.8, threshold=0.05,
                                  her_action=her_action, rng=Draws())
            assert sum(got) == n == len(a) == len(b)
            torch.cuda.synchronize()
            for name in ("obs", "act", "rew", "obs2", "done", "sum_tree", "min_tree", "state"):
                assert torch.equal(getattr(a._store, name), getattr(b._store, name)), (her_action, T, name)


def test_horizons_cleared_and_drop():
    """In an nstep_tails buffer the slots add_goal_steps writes get horizon 0 and no other slot changes.
    drop_goal_steps() discards the pending episodes: a restarted stream with other parameters stores what a fresh
    buffer stores for it."""
    So, G, A, M, E = 4, 2, 3, 5, 9
    rng = np.random.RandomState(8)
    calls = HO.random_calls(rng, 20, E, So, G, A, M)
    buf = _make("per", 2000, So + G, A, nstep_tails=True)
    hz = buf._store.horizon
    buf.add_batch(*(np.zeros((1, d), np.float32) for d in (So + G, A)), np.zeros(1), np.zeros((1, So + G), np.float32),
                  np.zeros(1, bool))
    hz.fill_(7)
    n = sum(_feed(buf, calls, True, max_episode_steps=M))
    assert n > 0 and len(buf) == 1 + n
    h = hz.cpu().numpy()
    assert not h[1:1 + n].any() and (h[1 + n:] == 7).all() and h[0] == 7
    # restart with other parameters after a drop: nothing of the first stream's pending episodes is emitted
    buf.drop_goal_steps()
    calls2 = HO.random_calls(rng, 15, 4, So, G, A, 3)
    fresh = _make("per", 2000, So + G, A)
    her = dict(her_ratio=0.3, threshold=0.01, her_action="own", max_episode_steps=3, seed=9)
    got = _feed(buf, calls2, False, **her)
    assert got == _feed(fresh, calls2, False, **her)
    m = sum(got)
    torch.cuda.synchronize()
    for name in ("obs", "act", "rew", "obs2", "done"):
        assert torch.equal(getattr(buf._store, name)[1 + n:1 + n + m], getattr(fresh._store, name)[:m]), name


def test_learner_observe_goals_vs_oracle_rows():
    """DDPG(her=..., sampling="device") fed by observe_goals on CUDA tensors against one fed the oracle's rows through
    add_batch at the same points, train_n() between calls: actor, critic and both targets bit-identical."""
    import d4pg_b200 as d4pg
    So, G, A, E, M, K = 10, 3, 4, 16, 8, 40
    rng = np.random.RandomState(2)
    calls = HO.random_calls(rng, K, E, So, G, A, M)
    her = dict(her_ratio=0.8, threshold=0.05, her_action="reference", max_episode_steps=M, seed=4)
    rows = HO.stream_rows(calls, her["her_ratio"], her["threshold"], her["her_action"], her["seed"])
    runs = []
    for feed in ("observe", "oracle"):
        torch.manual_seed(0)
        dd = d4pg.DDPG(So + G, A, memory_size=4096, batch_size=32, critic_dist_info=INFO, sampling="device", her=her,
                       obs_norm=True)
        dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
        out = []
        for k, c in enumerate(calls):
            if feed == "observe":
                got = dd.observe_goals(*_cuda(c))
            else:
                r = rows[k]
                got = len(r["r"])
                if got:
                    dd.replayBuffer.add_batch(*(torch.as_tensor(r[x].astype(np.float32) if x in ("s", "s2") else r[x]).cuda()
                                                for x in ("s", "a", "r", "s2", "d")))
            out.append(got)
            if len(dd.replayBuffer) >= 64 and k % 3 == 0:
                dd.train_n(4)
        torch.cuda.synchronize()
        out += [dd.actor.flat_params().clone(), dd.critic.flat_params().clone(),
                dd.actor_target.flat_params().clone(), dd.critic_target.flat_params().clone()]
        runs.append(out)
    assert sum(x for x in runs[0] if not torch.is_tensor(x)) > 200
    for x, y in zip(*runs):
        assert torch.equal(x, y) if torch.is_tensor(x) else x == y


def test_widest_launch():
    """E = 4096 environments at Fetch shapes (So = 25, G = 3, A = 4, 50-step episodes) all ending at the same call: the
    next call emits about 370 k rows in one launch, every one bit-exact against the oracle; the ring holds exactly
    E * 2 * max_episode_steps rows."""
    E, So, G, A, M = 4096, 25, 3, 4, 50
    rng = np.random.RandomState(1)
    calls = []
    for k in range(M + 1):
        end = np.full(E, k == M - 1)
        calls.append((rng.randn(E, So).astype(np.float32), rng.randn(E, G), rng.uniform(-1, 1, (E, A)).astype(np.float32),
                      -rng.randint(0, 2, E).astype(np.float64), rng.randn(E, So).astype(np.float32),
                      rng.randint(0, 4, (E, G)) * 0.02, end & (np.arange(E) % 2 == 0), end & (np.arange(E) % 2 == 1)))
    rows = HO.stream_rows(calls, 0.8, 0.05, "reference", 0)
    counts = [len(r["r"]) for r in rows]
    assert counts[:M] == [0] * M and 360000 < counts[M] <= E * 2 * M
    size = E * 2 * M
    buf = _make("per", size, So + G, A)
    assert _feed(buf, calls, True, max_episode_steps=M) == counts
    _check_ring(buf._store, _ring(HO.concat(rows), size), counts[M])


_LAUNCH_COUNT_SCRIPT = r"""
import json
import numpy as np, torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
import d4pg_b200 as d4pg
So, G, A, E, M = 9, 3, 2, 64, 4
rng = np.random.RandomState(1)

def step(end):
    c = lambda *s: torch.as_tensor(rng.randn(*s)).cuda()
    return (c(E, So).float(), c(E, G), c(E, A).float(), c(E), c(E, So).float(), c(E, G),
            torch.full((E,), end, dtype=torch.bool, device="cuda"), torch.zeros(E, dtype=torch.bool, device="cuda"))

def kernels(fn):
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rows = fn()
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA
                 and not e.name.startswith(("Memcpy", "Memset"))), key=lambda e: e.time_range.start)
    return dict(rows=rows, kernels=[e.name for e in ev])

out = {}
for name, per, norm in [("plain", False, False), ("per", True, False), ("per_norm", True, True)]:
    buf = d4pg.PrioritizedReplayBuffer(1000, 0.6, obs_dim=So + G, act_dim=A, obs_norm=norm) if per else \
        d4pg.ReplayBuffer(1000, obs_dim=So + G, act_dim=A, obs_norm=norm)
    for k in range(M):
        buf.add_goal_steps(*step(k == M - 1), max_episode_steps=M)
    s = step(False)
    out[name] = kernels(lambda: buf.add_goal_steps(*s, max_episode_steps=M))        # emits every episode
    s = step(True)
    out[name + "_none"] = kernels(lambda: buf.add_goal_steps(*s, max_episode_steps=M))  # emits nothing
    out[name + "_flush"] = kernels(lambda: buf.flush_goal_steps())                   # emits the one-step episodes
print(json.dumps(out))
"""


def test_launch_counts():
    """Per call: one kernel; with rows, the insert tail too (the tree add with PER, the normalizer's fold with
    obs_norm); a call that emits nothing launches the kernel alone whatever the buffer.  A flush launches what an
    emitting call launches.  One profiler session per call, in a fresh process."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _LAUNCH_COUNT_SCRIPT], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    tails = {"plain": [], "per": ["tree_add_range_fast"], "per_norm": ["obs_stats", "tree_add_range_fast"]}
    for name, tail in tails.items():
        for suffix, rows, names in (("", lambda n: n > 64 * 4, ["replay_add_goal_steps"] + tail),
                                    ("_none", lambda n: n == 0, ["replay_add_goal_steps"]),
                                    ("_flush", lambda n: n >= 64, ["replay_add_goal_steps"] + tail)):
            g = got[name + suffix]
            assert rows(g["rows"]), (name + suffix, g)
            ks = g["kernels"]
            assert len(ks) == len(names) and all(w + "_kernel" in k for k, w in zip(ks, names)), (name + suffix, ks)
