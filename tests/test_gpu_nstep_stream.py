"""The streaming n-step insert on the device (ReplayBuffer.add_steps / Replay.add_steps / DDPG.observe, DESIGN.md §3
"Streaming n-step insert"): pinned to the reference's Replay.initialize, bit-exact against the oracle
(tests/nstep_stream_oracle.py) over environment counts, window lengths, shapes and ring wraps, identical to add_batch at
n_steps = 1 (storage, both trees, max_priority, normalizer statistics), device and host end flags alike, the learner fed
by observe() identical to the learner fed the oracle's rows, the launches per call, and the argument checks."""
import random

import numpy as np
import pytest
import torch

from tests import helpers as H
from tests import nstep_stream_oracle as SO

pytestmark = pytest.mark.gpu


def _stored(store, n):
    torch.cuda.synchronize()
    return (store.obs[:n].cpu().numpy(), store.act[:n].cpu().numpy(), store.rew[:n].cpu().numpy(),
            store.obs2[:n].cpu().numpy(), store.done[:n].cpu().numpy().astype(bool))


def _on_device(c):
    cu = lambda x: None if x is None else torch.as_tensor(x).cuda()
    return tuple(cu(x) for x in c)


def test_pinned_to_reference_initialize():
    """The episodes the reference's Replay.initialize ran (tests/golden/nstep_init.npz), fed one step per call with
    E = 1 through Replay.add_steps, give the reference's buffer bit for bit."""
    import d4pg_b200 as d4pg
    g = H.load("nstep_init.npz")
    n_steps, _, n_buf, n_eps = [int(x) for x in g["meta"]]
    rp = d4pg.Replay(64, None, n_steps=n_steps, gamma=float(g["gamma"]), obs_dim=3, act_dim=2)
    total = 0
    for i in range(n_eps):
        s, a, r, s2, d = [g["ep%d_%s" % (i, k)] for k in ("s", "a", "r", "s2", "d")]
        T = len(r)
        for t in range(T):
            # the last episode may stop mid-way (initialize stops at init_length): end every episode's window
            got = rp.add_steps(s[t:t + 1], a[t:t + 1], r[t:t + 1], s2[t:t + 1], d[t:t + 1], truncated=[t == T - 1])
            assert got == int(t >= n_steps - 1)
            total += got
            assert len(rp) == total
    assert total == n_buf
    s, a, r, s2, d = _stored(rp._store, n_buf)
    assert np.array_equal(s, g["buf_s"].astype(np.float32)) and np.array_equal(a, g["buf_a"].astype(np.float32))
    assert np.array_equal(r, g["buf_r"]), "n-step returns are not bit-identical to the reference's f64 loop"
    assert np.array_equal(s2, g["buf_s2"].astype(np.float32)) and np.array_equal(d, g["buf_d"])


def _pick_size(counts, E):
    """A ring size >= E that one call's rows straddle (rows before it + half of its own), or None."""
    cum = 0
    for c in counts:
        if c >= 2 and cum + c // 2 >= E:
            return cum + c // 2
        cum += c
    return None


def _expected_ring(rows, size):
    """The ring after inserting `rows` in order: row i at i % size, later rows overwrite earlier ones."""
    m = len(rows)
    keep = rows[max(0, m - size):]
    pos = [(max(0, m - size) + j) % size for j in range(len(keep))]
    order = np.argsort(pos)
    cols = [np.stack([np.asarray(r[i]) for r in keep]) for i in range(5)]
    return [c[order] for c in cols]


@pytest.mark.parametrize("dims", [(3, 2), (17, 6), (376, 17)])
@pytest.mark.parametrize("E", [1, 31, 32, 33, 1024, 4096])
@pytest.mark.parametrize("n_steps", [1, 2, 5, 7])
def test_vs_oracle(n_steps, E, dims):
    """Random episode lengths (< n, == n, >> n) with terminations and truncations at different steps per environment:
    every stored row bit-exact (f64 reward, s, a, s2, done), len() and the return value after every call, the ring
    wrapped with one call's rows straddling its end (E > 1).  Host inputs for n in (1, 5), CUDA tensors for (2, 7)."""
    import d4pg_b200 as d4pg
    S, A = dims
    rng = np.random.RandomState(n_steps * 7919 + E * 31 + S)
    K = 120 if E == 1 else 2 * n_steps + 10
    calls = SO.random_calls(rng, K, E, S, A, n_steps)
    gamma = 0.97
    rows = SO.stream_rows(calls, n_steps, gamma)
    counts = np.bincount([k for k, _, _ in rows], minlength=K).tolist()
    size = _pick_size(counts, E) if E > 1 else 7
    assert size is not None and len(rows) > size, (counts, size)
    prio = n_steps % 2 == 1
    buf = d4pg.PrioritizedReplayBuffer(size, 0.6, obs_dim=S, act_dim=A) if prio else \
        d4pg.ReplayBuffer(size, obs_dim=S, act_dim=A)
    on_dev = n_steps in (2, 7)
    total = 0
    for k, c in enumerate(calls):
        got = buf.add_steps(*(_on_device(c) if on_dev else c), n_steps=n_steps, gamma=gamma)
        assert got == counts[k], k
        total += got
        assert len(buf) == min(total, size) and buf._next_idx == total % size
    want = _expected_ring([r for _, _, r in rows], size)
    mine = _stored(buf._store, size)
    for name, x, y in zip(("s", "a", "r", "s2", "done"), mine, want):
        assert np.array_equal(x, y.astype(x.dtype)), name
    if prio:
        assert float(buf._it_sum.sum(0, size)) == size and float(buf._it_min.min(0, size)) == 1.0


def _pair(kind, size, S, A, obs_norm):
    import d4pg_b200 as d4pg
    mk = (lambda: d4pg.PrioritizedReplayBuffer(size, 0.6, obs_dim=S, act_dim=A, obs_norm=obs_norm)) if kind == "per" \
        else (lambda: d4pg.ReplayBuffer(size, obs_dim=S, act_dim=A, obs_norm=obs_norm))
    return mk(), mk()


@pytest.mark.parametrize("obs_norm", [False, True])
@pytest.mark.parametrize("kind", ["uniform", "per"])
def test_n1_is_add_batch(kind, obs_norm):
    """n_steps = 1: one add_steps call stores what add_batch stores for the same E rows -- storage, every node of both
    trees, max_priority and the normalizer's statistics -- across ring wraps (one call straddling the end) and after
    update_priorities raised max_priority."""
    S, A, E, size = 11, 4, 37, 100
    a_buf, b_buf = _pair(kind, size, S, A, obs_norm)
    rng = np.random.RandomState(5)
    calls = SO.random_calls(rng, 9, E, S, A, 1)
    for k, c in enumerate(calls):
        if k == 5 and kind == "per":
            idx = rng.randint(0, size, 16).astype(np.int32)
            pr = (rng.rand(16) * 4 + 2).astype(np.float32)
            a_buf.update_priorities(idx, pr)
            b_buf.update_priorities(idx, pr)
        assert a_buf.add_steps(*(_on_device(c) if k % 2 else c), n_steps=1, gamma=0.5) == E
        b_buf.add_batch(*(torch.as_tensor(x).cuda() for x in c[:5]))
        assert len(a_buf) == len(b_buf) and a_buf._next_idx == b_buf._next_idx
    sa, sb = a_buf._store, b_buf._store
    torch.cuda.synchronize()
    for name in ("obs", "act", "rew", "obs2", "done", "sum_tree", "min_tree", "state"):
        assert torch.equal(getattr(sa, name), getattr(sb, name)), name
    if kind == "per":
        assert a_buf._max_priority == b_buf._max_priority > 1.0
    if obs_norm:
        assert torch.equal(sa.obs_norm.stats, sb.obs_norm.stats) and torch.equal(sa.obs_norm.affine, sb.obs_norm.affine)
        assert sa.obs_norm.count == 9 * E


def test_device_flags_equal_host_flags():
    """CUDA terminated / truncated (read back asynchronously, applied at the next call) and host flags give identical
    buffers, return values and lengths after every call; so do CUDA flags with truncated=None."""
    import d4pg_b200 as d4pg
    S, A, E, n = 9, 3, 33, 5
    rng = np.random.RandomState(11)
    calls = SO.random_calls(rng, 30, E, S, A, n)
    for trunc in (True, False):
        cs = calls if trunc else [c[:5] + (None,) for c in calls]
        counts = np.bincount([k for k, _, _ in SO.stream_rows(cs, n, 0.9)], minlength=len(cs)).tolist()
        bufs = [d4pg.PrioritizedReplayBuffer(300, 0.6, obs_dim=S, act_dim=A) for _ in range(3)]
        for k, c in enumerate(cs):
            host = bufs[0].add_steps(*c, n_steps=n, gamma=0.9)
            dev = bufs[1].add_steps(*_on_device(c), n_steps=n, gamma=0.9)
            flags_only = bufs[2].add_steps(*c[:4], *_on_device(c)[4:], n_steps=n, gamma=0.9)
            assert host == dev == flags_only == counts[k] and len(bufs[0]) == len(bufs[1]) == len(bufs[2])
        assert sum(counts) > 300
        torch.cuda.synchronize()
        for name in ("obs", "act", "rew", "obs2", "done", "sum_tree", "min_tree"):
            x = getattr(bufs[0]._store, name)
            assert torch.equal(x, getattr(bufs[1]._store, name)) and torch.equal(x, getattr(bufs[2]._store, name)), name


INFO = {"type": "categorical", "v_min": -10.0, "v_max": 0.0, "n_atoms": 51}
LEARNER_CASES = [dict(sampling="reference"), dict(sampling="device", prefetch=True),
                 dict(sampling="device", n_steps=5, projection="nstep"), dict(sampling="reference", prioritized_replay=False)]


@pytest.mark.parametrize("case", LEARNER_CASES, ids=["host_pipeline", "device_prefetch", "nstep5", "uniform_replay"])
def test_learner_observe_vs_oracle_rows(case):
    """DDPG.observe() fed by act() on device tensors against a DDPG fed the oracle's rows through add_batch at the same
    points, train() interleaved: parameters and sampled indices bit-identical after every step."""
    import d4pg_b200 as d4pg
    S, A, E, K = 17, 6, 16, 30
    kw = dict(memory_size=256, batch_size=32, critic_dist_info=INFO, **case)
    n = case.get("n_steps", 1) if "n_steps" in case else 3
    kw["n_steps"] = n
    rng = np.random.RandomState(2)
    term, trunc = SO.random_ends(rng, K, E, n)
    S_all = [rng.randn(E, S).astype(np.float32) for _ in range(K + 1)]
    R_all = [rng.randn(E) for _ in range(K)]
    runs = []
    actions = []
    for feed in ("observe", "oracle"):
        torch.manual_seed(0)
        random.seed(4)
        dd = d4pg.DDPG(S, A, **kw)
        dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                                   d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
        if feed == "oracle":
            calls = [(S_all[k], actions[k], R_all[k], S_all[k + 1], term[k], trunc[k]) for k in range(K)]
            rows = SO.stream_rows(calls, n, dd.gamma)
        out = []
        for k in range(K):
            if feed == "observe":
                s = torch.as_tensor(S_all[k]).cuda()
                a = dd.act(s)
                actions.append(a.cpu().numpy())
                got = dd.observe(s, a, torch.as_tensor(R_all[k]).cuda(), torch.as_tensor(S_all[k + 1]).cuda(),
                                 torch.as_tensor(term[k]).cuda(), torch.as_tensor(trunc[k]).cuda())
            else:
                rk = [r for c, _, r in rows if c == k]
                if rk:
                    dd.replayBuffer.add_batch(*[np.stack([np.asarray(r[i]) for r in rk]) for i in range(5)])
                got = len(rk)
            out.append(got)
            if len(dd.replayBuffer) >= 64:
                dd.train()
                out.append(dd.last_batch_info()["idx"].clone())
        torch.cuda.synchronize()
        out += [dd.actor.flat_params().clone(), dd.critic.flat_params().clone(),
                dd.actor_target.flat_params().clone(), dd.critic_target.flat_params().clone()]
        runs.append(out)
    assert len(runs[0]) == len(runs[1]) and sum(1 for x in runs[0] if torch.is_tensor(x)) > 10
    for x, y in zip(*runs):
        assert torch.equal(x, y) if torch.is_tensor(x) else x == y


_LAUNCH_COUNT_SCRIPT = r"""
import json
import numpy as np, torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
import d4pg_b200 as d4pg
S, A, E, n = 17, 6, 64, 3
rng = np.random.RandomState(1)

def args():
    return (torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda(), torch.rand(E, A, device="cuda"),
            torch.rand(E, dtype=torch.float64, device="cuda"), torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda(),
            torch.zeros(E, dtype=torch.bool, device="cuda"), torch.zeros(E, dtype=torch.bool, device="cuda"))

out = {}
for name, per, norm, size in [("plain", False, False, 1000), ("per", True, False, 1000), ("per_wrap", True, False, 150),
                              ("norm", False, True, 1000), ("per_norm", True, True, 1000)]:
    buf = d4pg.PrioritizedReplayBuffer(size, 0.6, obs_dim=S, act_dim=A, obs_norm=norm) if per else \
        d4pg.ReplayBuffer(size, obs_dim=S, act_dim=A, obs_norm=norm)
    for _ in range(n + 1):                 # windows full: every call inserts E rows; per_wrap's next one wraps at 150
        buf.add_steps(*args(), n_steps=n, gamma=0.9)
    a = args()
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rows = buf.add_steps(*a, n_steps=n, gamma=0.9)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA
                 and not e.name.startswith(("Memcpy", "Memset"))), key=lambda e: e.time_range.start)
    out[name] = dict(rows=rows, kernels=[e.name for e in ev])
print(json.dumps(out))
"""


def test_launch_counts():
    """Per call: one kernel without PER or obs_norm; the tree add with PER (two when the rows wrap the ring); the
    normalizer's fold with obs_norm.  One profiler session per call, in a fresh process."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _LAUNCH_COUNT_SCRIPT], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    want = {"plain": ["replay_add_steps"], "per": ["replay_add_steps", "tree_add_range_fast"],
            "per_wrap": ["replay_add_steps", "tree_add_range_fast", "tree_add_range_fast"],
            "norm": ["replay_add_steps", "obs_stats"], "per_norm": ["replay_add_steps", "obs_stats", "tree_add_range_fast"]}
    for name, names in want.items():
        assert got[name]["rows"] == 64, got
        ks = got[name]["kernels"]
        assert len(ks) == len(names) and all(w + "_kernel" in k for k, w in zip(ks, names)), (name, ks)


def test_validation_and_restart():
    """The first call fixes E, n_steps and gamma; changing any raises before device work and leaves the buffer as it
    was; drop_steps() allows a restart with new values, whose windows start empty.  E > size and n_steps > 64 raise."""
    import d4pg_b200 as d4pg
    S, A = 5, 2
    rng = np.random.RandomState(0)
    calls = SO.random_calls(rng, 6, 8, S, A, 3, with_trunc=False)
    buf = d4pg.PrioritizedReplayBuffer(64, 0.6, obs_dim=S, act_dim=A)
    for c in calls[:4]:
        buf.add_steps(*c, n_steps=3, gamma=0.9)
    before = len(buf), buf._next_idx
    small = SO.random_calls(rng, 1, 4, S, A, 3)[0]
    for args, kw in ((small, dict(n_steps=3, gamma=0.9)), (calls[4], dict(n_steps=2, gamma=0.9)),
                     (calls[4], dict(n_steps=3, gamma=0.95))):
        with pytest.raises(ValueError, match="drop_steps"):
            buf.add_steps(*args, **kw)
    assert (len(buf), buf._next_idx) == before
    with pytest.raises(ValueError, match="exceed"):
        buf.add_steps(*SO.random_calls(rng, 1, 65, S, A, 1)[0], n_steps=1)
    with pytest.raises(ValueError, match="n_steps"):
        buf.add_steps(*small, n_steps=65)
    buf.drop_steps()
    assert [buf.add_steps(*small, n_steps=2, gamma=0.5) for _ in range(3)] == [0, 4, 4]
    assert len(buf) == before[0] + 8
