"""Stream order between the replay's writers and the learner's sampler, in a rollout loop that never waits on the host.

With the host pipeline (the default: sampling="reference", prefetch=True, use_graph=True) DDPG.train() samples batch k
on the learner's ingest stream, and that stream does not wait for the caller's stream (DESIGN.md §2.3).  A replay write
issued on the caller's stream -- add_batch of CUDA tensors, observe(), observe_goals(), add_episode(),
update_priorities() ... -- must therefore be followed by an ordering edge before the next step
(`_DeviceReplay.before_step`).  Without it batch k may be drawn from the rows, trees and normalizer statistics of
before insert k.  No fault shows this; the learner just trains on other numbers.

- `test_async_loop_equals_synchronized_twin`: two learners with the same seeds, options and inserts.  The async one
  never waits on the host inside the loop: every input is a CUDA tensor made before it, and every per-step result
  (indices, IS weights, the sampled s / s2, the losses) is kept with device-side clones.  The sync twin runs
  torch.cuda.synchronize() after every call, so it reads in the reference's order update(k-1) -> add(k) -> sample(k).
  To make any missing edge show, the async loop puts a delay kernel on the writing stream right before each write: the
  caller's stream before a caller-stream insert, the ingest stream before add_batch_host, and the learner stream before
  each step, which delays its priority write-back.  A correct order waits the delay out; a missing edge reads the old
  data, the same way on every run.  After the loop both learners must be bit-identical (parameters, Adam moments,
  targets, every step's indices, IS weights, batches and losses, trees, ring, horizons, normalizer statistics, len and
  next_idx).  Each step's batch must equal the ring rows at its indices, normalized with the statistics of every row
  inserted before it (tests/obs_norm_oracle.py; the ring never wraps), and the trees must pass tests/replay_check.py.
- `test_reads_after_delayed_host_add`: the reverse direction.  A delayed add_batch_host on the ingest stream, then reads
  on the caller's stream (sample, gather, max_priority, act() through the normalizer, the normalizer's state_dict),
  equal to the synchronized twin's.
- `test_caller_writes_are_ordered_before_the_next_step`: the protocol, with no timing involved.  A recording proxy
  around the library sees every call; each caller-stream replay write must be followed by
  d4pg_replay_order_after(replay, caller, ingest) before the next d4pg_learner_step_host*.
- `test_host_add_loop_issues_no_ordering`: a loop that adds only through add_batch_host (the `e2e` benchmark's loop)
  issues no such edge once the learner is attached, so its adds and samples keep overlapping the running step.

Writers that wait on the host before their launch hide a race behind that wait, so they are left to the protocol test:
flush() (its staged rows go up from pageable memory, and it synchronizes), add_batch_host of more than 4096 rows (a
pageable copy), flush_goal_steps() (it waits for the end flags of the call before it), add_her_episode() (host arrays)
and update_priorities() (it checks its arguments with bool(...)).  set_leaves is reached only through the standalone
SegmentTree, which has no learner.

Every case runs the fp32 chain plan, whose step waits for the ingest stream's sample on a stream event.  The wgmma
plans' forward chains poll epochs the sample publishes instead, and a sample drawn before step k-1 has advanced the
step clock publishes a stale epoch: there a missing edge does not read stale data, the step never starts.  The first
async case hung that way on the commit before the ordering was added; on the fp32 plan the same slip fails the
comparison instead of hanging the suite.

DELAY_CYCLES = 4e7 SM cycles, about 20 ms at the H100's 1.98 GHz boost clock (24 ms at 1.65 GHz).  One iteration of the
async loop (an insert, train(), four clones) is guessed at well under 2 ms of host time, so the delay is at least 10x
that; that host time has not been measured.  Each case runs once.
"""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from tests import obs_norm_oracle as ON
from tests import replay_check as RC

S, A, SO, G = 17, 6, 11, 6          # goal cases: obs 11 + goal 6 = the same 17 columns
B, MEM, FILL, K = 64, 4096, 256, 6
DELAY_CYCLES = 40_000_000
INFO = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}

EXECUTION = {
    "host": {},                                            # the host pipeline: the defaults
    "prefetch": dict(sampling="device"),                   # device prefetch, one step per train()
    "train_n": dict(sampling="device"),                    # device prefetch, train_n(2) between inserts
    "graph": dict(prefetch=False),                         # host-drawn uniforms, one CUDA graph per step, no pipeline
    "eager": dict(use_graph=False),                        # host-drawn uniforms, eager launches
}
DISCOUNT = {"1": {}, "5": dict(n_steps=5, projection="nstep"), "tails": dict(n_steps=5, projection="nstep", nstep_tails=True)}

# (writer, replay, obs_norm, discount, execution): a covering set -- every writer under the host pipeline, each on both
# replays and with the normalizer on and off somewhere; every other execution mode at least once, with caller writers
CASES = [
    ("add_batch_cuda", "prioritized", "off", "1", "host"),
    ("add_batch_cuda", "uniform", "on", "1", "host"),
    ("observe", "prioritized", "on", "1", "host"),
    ("observe", "uniform", "off", "5", "host"),
    ("observe", "prioritized", "off", "tails", "host"),
    ("observe_goals", "prioritized", "on", "1", "host"),
    ("observe_goals", "uniform", "off", "1", "host"),
    ("add_episode", "uniform", "on", "5", "host"),
    ("add_episode", "prioritized", "off", "5", "host"),
    ("add_batch_host", "prioritized", "on", "1", "host"),
    ("add_batch_host", "uniform", "off", "5", "host"),
    ("observe", "prioritized", "on", "tails", "prefetch"),
    ("add_batch_cuda", "uniform", "off", "1", "prefetch"),
    ("add_episode", "prioritized", "on", "5", "graph"),
    ("observe", "uniform", "on", "1", "eager"),
    ("add_batch_cuda", "prioritized", "on", "5", "train_n"),
    ("observe_goals", "prioritized", "off", "1", "train_n"),
]


def _id(case):
    return "-".join(case)


def _rows(rng, n):
    s = (rng.randn(n, S) * np.logspace(-2, 2, S) + np.linspace(-30.0, 30.0, S)).astype(np.float32)
    s2 = (rng.randn(n, S) * np.logspace(-2, 2, S) + np.linspace(-30.0, 30.0, S)).astype(np.float32)
    return s, rng.uniform(-1, 1, (n, A)).astype(np.float32), (-3 * rng.rand(n)).astype(np.float64), s2, rng.rand(n) < 0.05


def _make(d4pg, replay, obs_norm, discount, execution, her=False):
    torch.manual_seed(5); np.random.seed(5); random.seed(5)
    kw = dict(DISCOUNT[discount], **EXECUTION[execution])
    dd = d4pg.DDPG(S, A, memory_size=MEM, batch_size=B, critic_dist_info=INFO, precision="fp32", philox_seed=3,
                   gamma=0.95, prioritized_replay=replay == "prioritized", obs_norm=True if obs_norm == "on" else None,
                   her=True if her else None, **kw)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    dd.replayBuffer.add_batch(*_rows(np.random.RandomState(1), FILL))
    return dd


class Inputs(object):
    """The K inserts of one writer, drawn once: CUDA tensors for the caller-stream writers, host arrays for
    add_batch_host."""

    def __init__(self, writer, dev):
        rng = np.random.RandomState(7)
        cuda = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(dev)
        self.writer, self.steps = writer, []
        for k in range(K):
            if writer in ("add_batch_cuda", "add_batch_host"):
                rows = _rows(rng, 48)
                self.steps.append(rows if writer == "add_batch_host" else [cuda(x) for x in rows])
            elif writer == "add_episode":
                s, a, r, s2, d = _rows(rng, 12)
                d[:] = False
                d[-1] = k % 2 == 0
                self.steps.append([cuda(x) for x in (s, a, r, s2, d)])
            elif writer == "observe":
                s, a, r, s2, _ = _rows(rng, 8)
                self.steps.append([cuda(x) for x in (s, a, r, s2, rng.rand(8) < 0.2, rng.rand(8) < 0.1)])
            else:                                              # observe_goals: E = 4 episodes of a few steps each
                s, a, r, s2, _ = _rows(rng, 4)
                g, ag = rng.randn(4, G), rng.randn(4, G)
                self.steps.append([cuda(x) for x in (s[:, :SO], g, a, r, s2[:, :SO], ag, rng.rand(4) < 0.35, rng.rand(4) < 0.1)])
        torch.cuda.synchronize()

    def put(self, dd, k):
        x, rb = self.steps[k], dd.replayBuffer
        if self.writer in ("add_batch_cuda", "add_batch_host"):
            rb.add_batch(*x)
        elif self.writer == "add_episode":
            if dd.prioritized_replay:
                rb.add_episode(*x, n_steps=dd.n_steps, gamma=dd.gamma)
            else:
                rb.add_episode(*x)
        elif self.writer == "observe":
            dd.observe(*x)
        else:
            dd.observe_goals(*x)


def _sleep_on(stream):
    with torch.cuda.stream(stream):
        torch.cuda._sleep(DELAY_CYCLES)


def _run(case, sync):
    """K inserts and steps of one learner -> (per-step records, lens after each insert, final state, DDPG)."""
    import d4pg_b200 as d4pg
    writer, replay, obs_norm, discount, execution = case
    dd = _make(d4pg, replay, obs_norm, discount, execution, her=writer == "observe_goals")
    feed = Inputs(writer, dd.device)
    step = (lambda: dd.train_n(2)) if execution == "train_n" else dd.train
    rng = np.random.RandomState(2)
    for _ in range(4):                     # create the learner and capture its graph variants before the loop
        dd.replayBuffer.add_batch(*_rows(rng, 8))
        step()
    torch.cuda.synchronize()
    L, store = dd._learner, dd.replayBuffer._store
    assert (store._ingest_stream is not None) == (execution == "host")
    ingest = torch.cuda.ExternalStream(store._ingest_stream) if store._ingest_stream else None
    wait = torch.cuda.synchronize if sync else (lambda: None)
    recs, lens = [], []
    for k in range(K):
        if not sync:
            _sleep_on(ingest if writer == "add_batch_host" else torch.cuda.current_stream())
        feed.put(dd, k)
        wait()
        lens.append(len(dd.replayBuffer))
        if not sync:
            _sleep_on(L.stream)
        step()
        wait()
        info = dd.last_batch_info()        # the caller's stream waits for the step; the host does not
        recs.append([info["idx"].clone(), info["weights"].clone(), L.tensor("s"), L.tensor("s2"), L.losses.clone()])
        wait()
    torch.cuda.synchronize()
    return [[t.cpu() for t in r] for r in recs], lens, _final(dd), dd


def _final(dd):
    """Everything the loop leaves behind, as named CPU tensors."""
    store = dd.replayBuffer._store
    out = {n: getattr(dd, n).flat_params() for n in ("actor", "actor_target", "critic", "critic_target")}
    for name, opt, net in (("actor", dd.optimizer_global_actor, dd.actor), ("critic", dd.optimizer_global_critic, dd.critic)):
        out[name + " exp_avg"], out[name + " exp_avg_sq"] = opt.moments(net)
    for n in ("obs", "act", "rew", "obs2", "done", "horizon", "state"):
        if getattr(store, n) is not None:
            out["ring " + n] = getattr(store, n)
    if dd.prioritized_replay:
        out["sum tree"], out["min tree"] = store.sum_tree, store.min_tree
    if dd.obs_normalizer is not None:
        out["normalizer stats"], out["normalizer affine"] = dd.obs_normalizer.stats, dd.obs_normalizer.affine
    out = {k: v.detach().cpu().clone() for k, v in out.items()}
    out["len / next_idx"] = torch.tensor([len(store), store._next_idx])
    return out


def _same(a, b):
    a, b = a.contiguous(), b.contiguous()
    return a.shape == b.shape and a.dtype == b.dtype and torch.equal(a.view(torch.uint8), b.view(torch.uint8))


def _check_batches(dd, recs, lens, final, label):
    """Each step's s / s2 are the ring rows at its indices, normalized with the statistics of the rows inserted before."""
    obs, obs2 = final["ring obs"].numpy(), final["ring obs2"].numpy()
    assert final["len / next_idx"][0].item() < dd.replayBuffer._store.size, "%s: the ring wrapped" % label
    for k, (idx, _, s, s2, _) in enumerate(recs):
        idx = idx.numpy().astype(np.int64)
        assert (idx >= 0).all() and (idx < lens[k]).all(), "%s step %d: an index past the rows inserted" % (label, k)
        if dd.obs_normalizer is not None:
            shift, scale = ON.Stats(S).fold(obs[:lens[k]]).affine()
            want_s, want_s2 = ON.apply(obs[idx], shift, scale), ON.apply(obs2[idx], shift, scale)
        else:
            want_s, want_s2 = obs[idx], obs2[idx]
        for name, got, want in (("s", s, want_s), ("s2", s2, want_s2)):
            got = got.numpy()[:, :S]
            assert np.array_equal(got.view(np.uint32), np.ascontiguousarray(want, np.float32).view(np.uint32)), (
                "%s step %d: the sampled %s is not the ring rows at its indices (%d rows differ)"
                % (label, k, name, int((got != want).any(1).sum())))


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_async_loop_equals_synchronized_twin(case):
    label = _id(case)
    recs_s, lens_s, fin_s, dd_s = _run(case, sync=True)
    del dd_s
    recs_a, lens_a, fin_a, dd_a = _run(case, sync=False)
    assert lens_a == lens_s
    names = ("indices", "IS weights", "batch s", "batch s2", "losses")
    bad = ["step %d %s" % (k, names[i]) for k in range(K) for i in range(5) if not _same(recs_a[k][i], recs_s[k][i])]
    bad += [n for n in fin_s if not _same(fin_a[n], fin_s[n])]
    assert not bad, "%s: the unsynchronized loop differs from its synchronized twin in %s" % (label, ", ".join(bad))
    _check_batches(dd_a, recs_a, lens_a, fin_a, label)
    if dd_a.prioritized_replay:
        RC.check_invariant(RC.snapshot(dd_a.replayBuffer._store), label=label)


# ---- reverse direction: ingest-stream adds, then caller-stream reads -----------------------------------------------
def _reads_run(sync):
    import d4pg_b200 as d4pg
    dd = _make(d4pg, "prioritized", "on", "1", "host")
    feed = Inputs("add_batch_host", dd.device)
    rng = np.random.RandomState(11)
    uniforms = [list(rng.rand(B)) for _ in range(K)]
    positions = [rng.randint(0, FILL, B) for _ in range(K)]
    states = torch.as_tensor(_rows(rng, 32)[0]).to(dd.device)
    for _ in range(3):
        dd.train()
    torch.cuda.synchronize()
    store = dd.replayBuffer._store
    ingest = torch.cuda.ExternalStream(store._ingest_stream)
    wait = torch.cuda.synchronize if sync else (lambda: None)
    out = []
    for k in range(K):
        if not sync:
            _sleep_on(ingest)
        feed.put(dd, k)
        wait()
        o = store.sample_proportional(B, 0.5, uniforms=uniforms[k])
        g = store.gather(positions[k])
        got = [o[n].clone() for n in ("idx", "w", "s", "a", "r", "s2", "d")] + [g[n].clone() for n in ("s", "a", "r", "s2", "d")]
        got.append(dd.act(states, explore=False).clone())
        wait()
        got.append(torch.tensor([store.max_priority]))
        got.append(dd.obs_normalizer.state_dict()["stats"])
        wait()
        dd.train()
        wait()
        out.append([t.cpu() for t in got])
    torch.cuda.synchronize()
    return out, _final(dd)


@pytest.mark.gpu
def test_reads_after_delayed_host_add():
    out_s, fin_s = _reads_run(sync=True)
    out_a, fin_a = _reads_run(sync=False)
    names = ["sample " + n for n in ("idx", "w", "s", "a", "r", "s2", "d")] + ["gather " + n for n in ("s", "a", "r", "s2", "d")]
    names += ["act", "max_priority", "normalizer state_dict"]
    bad = ["step %d %s" % (k, names[i]) for k in range(K) for i in range(len(names)) if not _same(out_a[k][i], out_s[k][i])]
    bad += [n for n in fin_s if not _same(fin_a[n], fin_s[n])]
    assert not bad, "reads after a delayed ingest-stream add differ from the synchronized twin in %s" % ", ".join(bad)


# ---- the protocol, independent of timing ------------------------------------------------------------------------------
WRITES = ("d4pg_replay_add", "d4pg_replay_add_host", "d4pg_replay_add_steps_ex", "d4pg_replay_add_goal_steps",
          "d4pg_replay_add_nstep", "d4pg_replay_update_priorities", "d4pg_replay_set_leaves", "d4pg_replay_obs_norm_refresh")


class Recorder(object):
    """Delegates to the real library and records (name, args) of every d4pg_* call."""

    def __init__(self, real):
        self._real, self.calls = real, []

    def __getattr__(self, name):
        fn = getattr(self._real, name)
        if not name.startswith("d4pg_"):
            return fn

        def call(*args):
            self.calls.append((name, args))
            return fn(*args)
        return call


def _stream(x):
    """A stream argument as an int (ctypes gives None for a NULL c_void_p: the legacy default stream is 0)."""
    return (x.value if isinstance(x, C.c_void_p) else x) or 0


def _unordered_writes(calls, caller, ingest):
    """The caller-stream writes not followed by order_after(caller -> ingest) before the next host-pipeline step."""
    pending, bad = [], []
    for name, args in calls:
        if name in WRITES and _stream(args[-1]) == caller:
            pending.append(name)
        elif name == "d4pg_replay_order_after" and _stream(args[1]) == caller and _stream(args[2]) == ingest:
            pending = []
        elif name.startswith("d4pg_learner_step_host"):
            bad += pending
            pending = []
    return bad


def _protocol_writer(dd, writer, rng):
    rb, dev = dd.replayBuffer, dd.device
    cuda = lambda x: torch.as_tensor(np.ascontiguousarray(x)).to(dev)
    if writer == "add_batch_cuda":
        rb.add_batch(*[cuda(x) for x in _rows(rng, 48)])
    elif writer == "flush":
        s, a, r, s2, d = _rows(rng, 3)
        for i in range(3):                       # staged in pinned memory; train() flushes them on the caller's stream
            rb.add(s[i], a[i], r[i], s2[i], d[i])
    elif writer == "add_batch_host_large":
        rb.add_batch(*_rows(rng, rb._store.STAGE_ROWS + 4))
    elif writer in ("observe", "observe_tails"):
        s, a, r, s2, _ = _rows(rng, 8)
        for _ in range(5):
            dd.observe(*[cuda(x) for x in (s, a, r, s2, rng.rand(8) < 0.3)])
    elif writer in ("observe_goals", "flush_goal_steps"):
        s, a, r, s2, _ = _rows(rng, 4)
        for _ in range(2 if writer == "observe_goals" else 1):       # the second call inserts the ended episodes
            dd.observe_goals(s[:, :SO], rng.randn(4, G), a, r, s2[:, :SO], rng.randn(4, G), np.ones(4, bool))
        if writer == "flush_goal_steps":
            dd.train()
            assert rb.flush_goal_steps() > 0
    elif writer == "add_episode":
        s, a, r, s2, d = _rows(rng, 12)
        rb.add_episode(*[cuda(x) for x in (s, a, r, s2, d)], n_steps=dd.n_steps, gamma=dd.gamma)
    elif writer == "add_her_episode":
        s, a, r, s2, d = _rows(rng, 10)
        rb.add_her_episode(s[:, :SO], s2[:, :SO], rng.randn(10, G), rng.randn(10, G), a, r, d,
                           rng=np.random.RandomState(3))
    elif writer == "update_priorities":
        rb.update_priorities(torch.arange(0, 64, 2, device=dev, dtype=torch.int32),
                             torch.rand(32, device=dev) + 0.5)
    elif writer == "obs_norm_load":
        dd.obs_normalizer.load_state_dict(dd.obs_normalizer.state_dict())


PROTOCOL_WRITERS = ("add_batch_cuda", "flush", "add_batch_host_large", "observe", "observe_tails", "observe_goals",
                    "flush_goal_steps", "add_episode", "add_her_episode", "update_priorities", "obs_norm_load")


@pytest.mark.gpu
@pytest.mark.parametrize("writer", PROTOCOL_WRITERS)
def test_caller_writes_are_ordered_before_the_next_step(writer, monkeypatch):
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib
    rec = Recorder(_lib.lib())
    monkeypatch.setattr(_lib, "_lib", rec)      # before the learner exists: _Learner binds step_host* at creation
    discount = "tails" if writer == "observe_tails" else "1"
    dd = _make(d4pg, "prioritized", "on", discount, "host", her=writer in ("observe_goals", "flush_goal_steps"))
    dd.train()
    store = dd.replayBuffer._store
    caller, ingest = _stream(_lib.raw_stream()), store._ingest_stream
    assert ingest is not None
    start = len(rec.calls)
    _protocol_writer(dd, writer, np.random.RandomState(4))
    dd.train()
    torch.cuda.synchronize()
    calls = rec.calls[start:]
    assert any(n in WRITES and _stream(a[-1]) == caller for n, a in calls), "%s wrote nothing on the caller's stream" % writer
    bad = _unordered_writes(calls, caller, ingest)
    assert not bad, "%s: caller-stream writes %s reach a host-pipeline step with no order_after(caller, ingest)" % (
        writer, sorted(set(bad)))


@pytest.mark.gpu
def test_host_add_loop_issues_no_ordering(monkeypatch):
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib
    rec = Recorder(_lib.lib())
    monkeypatch.setattr(_lib, "_lib", rec)
    dd = _make(d4pg, "prioritized", "on", "1", "host")
    rows = _rows(np.random.RandomState(9), 8 * B)
    pinned = [torch.from_numpy(np.ascontiguousarray(x)).pin_memory() for x in rows]
    dd.replayBuffer.add_batch(*[x[:B] for x in rows])          # numpy: sets up the packed staging buffers
    dd.train()
    dd.replayBuffer.add_batch(*[p[B:2 * B] for p in pinned])
    dd.train()
    caller, ingest = _stream(_lib.raw_stream()), dd.replayBuffer._store._ingest_stream
    start = len(rec.calls)
    for i in range(2, 8):
        dd.replayBuffer.add_batch(*[p[i * B:(i + 1) * B] for p in pinned])
        dd.train()
        if i > 2:
            dd.last_losses(lag=1)
    dd.last_losses()
    calls = rec.calls[start:]
    assert sum(n == "d4pg_replay_add_host" and _stream(a[-1]) == ingest for n, a in calls) == 6
    edges = [a for n, a in calls if n == "d4pg_replay_order_after" and _stream(a[1]) == caller and _stream(a[2]) == ingest]
    assert not edges, "%d order_after(caller, ingest) edges in a loop of add_batch_host + train()" % len(edges)
