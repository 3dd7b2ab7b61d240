"""The learner's options in combination: every allowed pair of step plan, critic head, discount, observation
normalizer, clipping, actor-critic semantics, priorities, replay and execution mode is one of CASES, and every case runs
every checker the options have, at every step.

csrc/learner.cu chooses its launches, workspace offsets, batch halves and kernel variants from these options together,
so a slip in that composition (a horizon plane read from the other prefetch half, a normalizer affine missing at one
sample call site, a clip coefficient missing from the post-update critic's Adam launch) shows only when they meet.

- `test_cases_cover_every_allowed_pair` (CPU): each pair of levels of two factors that `excluded` allows appears in some
  case, no case holds an excluded pair, and each case's shapes force the plan it names.
- `test_excluded_pairs_are_rejected`: the library refuses every pair excluded as "rejected".
- `test_case_every_step_checked`: eager steps, each followed by the Adam / Polyak / clock update bit-exact
  (tests/update_check.py, tests/clip_check.py when clipping), the IS weights (prioritized), the loss head
  (tests/heads_check.py, per-row horizons and IS weights included), the batch against the ring (normalized with the
  statistics of every row inserted so far, tests/obs_norm_oracle.py), the priority write-back (tests/replay_check.py),
  and the layers of the first and the last step (tests/step_check.py); plus that each option really took effect.
- `test_case_pipeline_equals_eager`: the case's execution mode (CUDA graph per step, the 8-step graph, device prefetch,
  the host pipeline) against eager steps with the same seeds and inserts, bit for bit after every step or train_n call.

Batches stay below 1024 rows: from there the level plan's dW sums split-K slices with fp32 atomics, which is not
bit-reproducible from run to run.
"""
import itertools
import math
import random

import numpy as np
import pytest
import torch

from tests import clip_check as CC
from tests import heads_check as HC
from tests import obs_norm_oracle as ON
from tests import replay_check as RC
from tests import step_check as SC
from tests.test_gpu_heads import _cat, _mog, _qr
from tests.test_gpu_obs_norm import _check_batch, _check_stats, _rows
from tests.test_gpu_update import STATE_ITEMS, Checked, _id, _state

# ---- factors, constraints, cases ----------------------------------------------------------------------------------
FACTORS = {
    "plan": ["%s/%s" % k for k in SC.MODES],
    "head": ["categorical", "mixture", "quantile"],
    "discount": ["gamma", "gamma_n", "tails"],               # n = 1; n = 5 with projection="nstep"; the same + tails
    "obs_norm": ["off", "on"],
    "gradient": ["plain", "clip"],                           # clip: max_grad_norm and weight decay on both networks
    "actor_critic": ["reference", "post_update"],
    "priorities": ["plain", "iw", "iw_ce"],                  # importance_weighted; + priority="ce"
    "replay": ["prioritized", "uniform"],
    "execution": ["eager", "graph", "train_n", "prefetch", "host"],
}


def excluded(a, x, b, y):
    """(kind, reason) when level x of factor a and level y of factor b cannot meet, else None.  rejected: the library
    raises; impossible: the plan rule cannot produce the pair."""
    p = {a: x, b: y}
    if p.get("actor_critic") == "post_update" and "plan" in p and not p["plan"].startswith("tc_chain/"):
        return ("rejected", "the post-update critic runs on the tensor-core chain plan only")
    if p.get("head") == "mixture" and p.get("priorities") == "iw_ce":
        return ("rejected", "the cross-entropy of a density can be negative: no CE priority for a mixture critic")
    return None


NSTEP = dict(projection="nstep", n_steps=5)
TAILS = dict(NSTEP, nstep_tails=True)
LEVELS, NORM, CLIP = {"chain": "levels"}, {"obs_norm": True}, {"clip": True}
POST, IW, UNI = {"actor_critic": "post_update"}, {"importance_weighted": True}, {"replay": "uniform"}
CE = dict(IW, priority="ce")


def _o(*parts, **kw):
    """Case options: DDPG keywords, plus clip=True (thresholds and decays on both networks), replay="uniform" and
    run= (the execution mode; eager when absent)."""
    out = {}
    for p in parts + (kw,):
        out.update(p)
    return out


# (plan, precision, B, |s|, |a|, critic head, options).  tc_chain: |s|, |a| <= 32; chain at tf32x3 / tf32: |s| or
# |a| = 33; levels: chain="levels" (bf16 runs the level plan whatever chain says).  Odd batches leave partial CTAs.
CASES = [
    ("tc_chain", "tf32x3", 64, 17, 6, _qr(33), _o(TAILS, CLIP, POST, CE)),
    ("tc_chain", "tf32x3", 33, 17, 6, _cat(51), _o(NORM, IW, UNI, run="graph")),
    ("tc_chain", "tf32x3", 130, 17, 6, _mog(5), _o(NSTEP, run="train_n")),
    ("tc_chain", "tf32x3", 257, 17, 6, _qr(65), _o(NSTEP, NORM, CLIP, POST, UNI, run="prefetch")),
    ("tc_chain", "tf32x3", 65, 17, 6, _mog(11), _o(CLIP, POST, IW, UNI, run="host")),
    ("tc_chain", "tf32", 511, 17, 6, _cat(97), _o(TAILS, NORM, CE)),
    ("tc_chain", "tf32", 97, 17, 6, _cat(33), _o(NSTEP, CLIP, POST, run="graph")),
    ("tc_chain", "tf32", 64, 17, 6, _qr(51), _o(TAILS, NORM, POST, IW, UNI, run="train_n")),
    ("tc_chain", "tf32", 33, 17, 6, _qr(33), _o(IW, run="prefetch")),
    ("tc_chain", "tf32", 130, 17, 6, _mog(4), _o(TAILS, NORM, CLIP, UNI, run="host")),
    ("chain", "fp32", 257, 17, 6, _mog(17), _o(NORM, UNI)),
    ("chain", "fp32", 65, 17, 6, _qr(65), _o(NSTEP, CLIP, CE, UNI, run="graph")),
    ("chain", "fp32", 511, 17, 6, _cat(51), _o(CLIP, CE, run="train_n")),
    ("chain", "fp32", 96, 17, 6, _mog(5), _o(TAILS, CLIP, IW, run="prefetch")),
    ("chain", "fp32", 64, 17, 6, _cat(97), _o(NSTEP, IW, run="host")),
    ("chain", "tf32x3", 130, 33, 6, _qr(51), _o(NSTEP, IW)),
    ("chain", "tf32x3", 65, 33, 6, _mog(11), _o(TAILS, NORM, CLIP, UNI, run="graph")),
    ("chain", "tf32x3", 96, 33, 6, _cat(33), _o(NORM, CE, run="train_n")),
    ("chain", "tf32x3", 33, 17, 33, _cat(51), _o(NSTEP, NORM, CE, UNI, run="prefetch")),
    ("chain", "tf32x3", 257, 17, 33, _qr(33), _o(NSTEP, NORM, CE, run="host")),
    ("chain", "tf32", 511, 33, 6, _mog(4), _o(NORM, CLIP, IW, UNI)),
    ("chain", "tf32", 64, 17, 33, _cat(97), _o(TAILS, CE, run="graph")),
    ("chain", "tf32", 130, 33, 6, _qr(65), _o(NSTEP, CLIP, UNI, run="train_n")),
    ("chain", "tf32", 65, 33, 6, _qr(51), _o(NSTEP, run="prefetch")),
    ("chain", "tf32", 96, 33, 6, _qr(33), _o(NSTEP, CLIP, run="host")),
    ("levels", "fp32", 64, 17, 6, _qr(65), _o(LEVELS, IW, UNI)),
    ("levels", "fp32", 33, 17, 6, _cat(33), _o(TAILS, LEVELS, NORM, CLIP, run="graph")),
    ("levels", "fp32", 130, 17, 6, _qr(51), _o(NSTEP, LEVELS, NORM, CE, run="train_n")),
    ("levels", "fp32", 257, 17, 6, _mog(17), _o(LEVELS, CLIP, run="prefetch")),
    ("levels", "fp32", 65, 17, 6, _mog(5), _o(NSTEP, LEVELS, NORM, UNI, run="host")),
    ("levels", "tf32x3", 511, 17, 6, _cat(51), _o(LEVELS, NORM, UNI)),
    ("levels", "tf32x3", 96, 17, 6, _qr(33), _o(TAILS, LEVELS, CLIP, CE, run="graph")),
    ("levels", "tf32x3", 64, 17, 6, _mog(11), _o(NSTEP, LEVELS, NORM, CLIP, IW, UNI, run="train_n")),
    ("levels", "tf32x3", 33, 17, 6, _mog(4), _o(TAILS, LEVELS, NORM, IW, run="prefetch")),
    ("levels", "tf32x3", 130, 17, 6, _mog(17), _o(NSTEP, LEVELS, run="host")),
    ("levels", "tf32", 257, 17, 6, _mog(5), _o(NSTEP, LEVELS)),
    ("levels", "tf32", 65, 17, 6, _qr(65), _o(TAILS, LEVELS, NORM, CLIP, CE, UNI, run="graph")),
    ("levels", "tf32", 511, 17, 6, _cat(97), _o(LEVELS, CLIP, IW, UNI, run="train_n")),
    ("levels", "tf32", 96, 17, 6, _cat(33), _o(NSTEP, LEVELS, NORM, IW, UNI, run="prefetch")),
    ("levels", "tf32", 64, 17, 6, _mog(11), _o(TAILS, LEVELS, NORM, CLIP, UNI, run="host")),
    ("levels", "bf16", 33, 17, 6, _qr(51), _o(NORM, CE)),
    ("levels", "bf16", 130, 17, 6, _cat(51), _o(NSTEP, CLIP, UNI, run="graph")),
    ("levels", "bf16", 257, 17, 6, _mog(4), _o(TAILS, NORM, IW, run="train_n")),
    ("levels", "bf16", 65, 17, 6, _cat(97), _o(TAILS, run="prefetch")),
    ("levels", "bf16", 511, 17, 6, _cat(33), _o(IW, UNI, run="host")),
]
STEPS = 6
MEM = 4096
E = 32                    # environments per observe() call
WD = (1e-4, 3e-4)
ALPHA = 0.6


def levels(case):
    """{factor: level} of a case."""
    plan, precision, B, S, A, info, opt = case
    head = {"categorical": "categorical", "mixture_of_gaussian": "mixture", "quantile": "quantile"}[info["type"]]
    return {"plan": "%s/%s" % (plan, precision), "head": head,
            "discount": "tails" if opt.get("nstep_tails") else "gamma_n" if opt.get("n_steps", 1) > 1 else "gamma",
            "obs_norm": "on" if opt.get("obs_norm") else "off", "gradient": "clip" if opt.get("clip") else "plain",
            "actor_critic": opt.get("actor_critic", "reference"),
            "priorities": "iw_ce" if opt.get("priority") == "ce" else "iw" if opt.get("importance_weighted") else "plain",
            "replay": opt.get("replay", "prioritized"), "execution": opt.get("run", "eager")}


def _step_plan(case):
    """csrc/learner.cu step_plan for the case's shapes (DESIGN.md §2.4)."""
    plan, precision, B, S, A, info, opt = case
    width = 3 * info["n_components"] if info["type"] == "mixture_of_gaussian" else \
        info.get("n_atoms") or info.get("n_quantiles")
    if B > 512 or opt.get("chain") == "levels" or precision == "bf16":
        return "levels"
    if precision != "fp32" and S <= 32 and A <= 32 and width <= 256:
        return "tc_chain"
    return "chain"


def _pairs(lv):
    return {(a, lv[a], b, lv[b]) for a, b in itertools.combinations(FACTORS, 2)}


def _allowed_and_barred():
    allowed, barred = set(), set()
    for a, b in itertools.combinations(FACTORS, 2):
        for x in FACTORS[a]:
            for y in FACTORS[b]:
                (barred if excluded(a, x, b, y) else allowed).add((a, x, b, y))
    return allowed, barred


def test_cases_cover_every_allowed_pair():
    """Every pair of levels of two factors that `excluded` allows is in some case; no case holds an excluded pair; each
    case's shapes force its plan; batches stay below 1024 rows; ids are unique."""
    allowed, barred = _allowed_and_barred()
    seen = set()
    for case in CASES:
        lv = levels(case)
        assert all(lv[f] in FACTORS[f] for f in FACTORS), _id(case)
        bad = _pairs(lv) & barred
        assert not bad, "%s holds excluded pairs %s" % (_id(case), sorted(bad))
        seen |= _pairs(lv)
        assert _step_plan(case) == case[0], "%s: the shapes select the %s plan" % (_id(case), _step_plan(case))
        assert case[2] < 1024
    missing = sorted(allowed - seen)
    assert not missing, "%d allowed pairs in no case, e.g. %s" % (len(missing), missing[:5])
    assert len({_id(c) for c in CASES}) == len(CASES)
    assert all(excluded(*p)[0] in ("rejected", "impossible") for p in barred)
    print("%d cases cover %d allowed pairs; %d pairs excluded" % (len(CASES), len(allowed), len(barred)))


# ---- the excluded pairs --------------------------------------------------------------------------------------------
# the DDPG keywords of the levels a rejected pair names
LEVEL_KW = {("head", "mixture"): {"critic_dist_info": _mog(5)},
            ("priorities", "iw_ce"): dict(importance_weighted=True, priority="ce"),
            ("actor_critic", "post_update"): {"actor_critic": "post_update"}}


@pytest.mark.gpu
def test_excluded_pairs_are_rejected():
    """Every pair excluded as rejected raises ValueError or D4PGError, at DDPG() or when the first train() creates the
    learner, before the step runs."""
    import d4pg_b200 as d4pg
    rejected = sorted(p for p in _allowed_and_barred()[1] if excluded(*p)[0] == "rejected")
    assert rejected
    for a, x, b, y in rejected:
        kw = dict(critic_dist_info=_cat(51), sampling="device", use_graph=False, prefetch=False)
        S, A = 17, 6
        for f, lvl in ((a, x), (b, y)):
            if f == "plan":
                plan, precision = lvl.split("/")
                S = 33 if plan == "chain" and precision != "fp32" else 17
                kw.update({"chain": "levels"} if plan == "levels" else {}, precision=precision)
            else:
                kw.update(LEVEL_KW[f, lvl])
        with pytest.raises((ValueError, d4pg.D4PGError)):
            dd = d4pg.DDPG(S, A, memory_size=256, batch_size=32, **kw)
            dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
            dd.replayBuffer.add_batch(*_rows(np.random.RandomState(0), 64, S, A))
            dd.train()
        print("rejected:", (a, x, b, y), excluded(a, x, b, y)[1])


# ---- building and feeding a learner --------------------------------------------------------------------------------
def _kwargs(case, eager):
    """DDPG keywords of the case; eager: the same learner with use_graph=False, prefetch=False."""
    opt = case[6]
    kw = {k: v for k, v in opt.items() if k not in ("clip", "replay", "run")}
    run = opt.get("run", "eager")
    kw.update(prioritized_replay=opt.get("replay") != "uniform", sampling="reference" if run == "host" else "device")
    if eager:
        kw.update(use_graph=False, prefetch=False)
    else:
        kw.update(use_graph=run != "eager", prefetch=run in ("train_n", "prefetch", "host"))
    return kw


def _make(d4pg, case, eager, max_norm=None):
    plan, precision, B, S, A, info, opt = case
    torch.manual_seed(12); np.random.seed(12); random.seed(12)
    dd = d4pg.DDPG(S, A, memory_size=MEM, batch_size=B, critic_dist_info=info, precision=precision, philox_seed=3,
                   gamma=0.95, max_grad_norm=max_norm, **_kwargs(case, eager))
    wd = WD if opt.get("clip") else (0.0, 0.0)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3, weight_decay=wd[0]),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3, weight_decay=wd[1]))
    with torch.no_grad():                     # the target networks differ from the online ones
        dd.actor_target.flat_params().mul_(1.01)
        dd.critic_target.flat_params().mul_(0.99)
    return dd


def _ring_pos(store):
    return (store._next_idx + store._n_staged) % store.size


class Feed(object):
    """The rows a case inserts, drawn once so that two learners receive the same ones: a fill, then `inserts[k]` before
    step (or train_n call) k + 1.  Tails cases insert through observe() with many truncations and precomputed random
    actions; the others through add_batch (pinned tensors for the host pipeline).  A prioritized fill gets unequal
    priorities, so that the IS weights differ."""

    def __init__(self, case, n_inserts, seed=0):
        plan, precision, B, S, A, info, opt = case
        rng = np.random.RandomState(seed + B * 7 + S)
        self.tails, self.pinned = bool(opt.get("nstep_tails")), opt.get("run") == "host"
        if self.tails:
            calls = lambda K: [self._observe_call(rng, S, A) for _ in range(K)]
            self.fill, self.inserts = calls(B // E + 10), [calls(2) for _ in range(n_inserts)]
        else:
            self.fill = [_rows(rng, max(2 * B, 256), S, A)]
            self.inserts = [[_rows(rng, 48, S, A)] for _ in range(n_inserts)]

    @staticmethod
    def _observe_call(rng, S, A):
        term = rng.rand(E) < 0.05
        trunc = (rng.rand(E) < 0.3) & ~term
        return (rng.randn(E, S).astype(np.float32) * 3, rng.uniform(-1, 1, (E, A)).astype(np.float32), -rng.rand(E),
                rng.randn(E, S).astype(np.float32) * 3, term, trunc)

    def _put(self, dd, calls, stats):
        store = dd.replayBuffer._store
        for c in calls:
            if self.tails:
                pos = _ring_pos(store)
                n = dd.observe(*(torch.as_tensor(x).cuda() for x in c))
                if stats is not None:             # the rows observe() stored, in insertion order
                    torch.cuda.synchronize()
                    at = torch.arange(pos, pos + n, device=store.obs.device) % store.size
                    stats.fold(store.obs[at].cpu().numpy())
            else:
                rows = [torch.from_numpy(np.ascontiguousarray(x)).pin_memory() for x in c] if self.pinned else c
                dd.replayBuffer.add_batch(*rows)
                if stats is not None:
                    stats.fold(c[0])

    def put_fill(self, dd, stats=None):
        self._put(dd, self.fill, stats)
        if dd.prioritized_replay:
            n = len(dd.replayBuffer)
            dd.replayBuffer.update_priorities(np.arange(n), np.random.RandomState(5).uniform(0.1, 2.0, n))

    def put(self, dd, k, stats=None):
        self._put(dd, self.inserts[k], stats)


def _thresholds(d4pg, case, feed):
    """Clipping thresholds: the median gradient norms of a report-only run of the same eager learner with the same
    inserts, so that clipped and unclipped steps both occur."""
    dd = _make(d4pg, case, eager=True, max_norm=math.inf)
    feed.put_fill(dd)
    seen = []
    for i in range(STEPS):
        if i:
            feed.put(dd, i - 1)
        random.seed(100 + i)
        dd.train()
        seen.append(dd.last_grad_norms())
    del dd
    torch.cuda.empty_cache()
    out = tuple(float(sorted(n[j] for n in seen)[STEPS // 2]) for j in range(2))
    assert all(math.isfinite(x) and x > 0 for x in out), seen
    return out


# ---- the checks after one eager step -------------------------------------------------------------------------------
def _check_rows(dd, stats, label):
    """The step's batch against the ring at its indices: s / s2 (normalized with `stats` when the learner normalizes),
    a, r, done and the horizons bit for bit.  Returns (idx, horizons, done)."""
    B, S, A = dd.batch_size, dd.obs_dim, dd.act_dim
    store = dd.replayBuffer._store
    idx = dd.last_batch_info()["idx"].cpu().numpy().astype(np.int64)
    torch.cuda.synchronize()
    at = lambda t: t[torch.as_tensor(idx, device=t.device)].cpu().numpy()
    ring = {"s": at(store.obs), "a": at(store.act), "r": at(store.rew), "s2": at(store.obs2), "done": at(store.done)}
    if stats is not None:
        rows = (np.zeros((store.size, S), np.float32), None, None, np.zeros((store.size, S), np.float32))
        rows[0][idx], rows[3][idx] = ring["s"], ring["s2"]
        _check_batch(dd, stats, rows, label)
    else:
        for name in ("s", "s2"):
            got = dd.debug_tensor(name, shape=(B, S)).cpu().numpy()
            assert np.array_equal(got.view(np.uint32), ring[name].view(np.uint32)), "%s: %s differs from the ring" % (
                label, name)
    got = {"a": dd.debug_tensor("a", shape=(B, A)).cpu().numpy(),
           "r": dd.debug_tensor("r", dtype=torch.float64).cpu().numpy()[:B],
           "done": dd.debug_tensor("done", dtype=torch.uint8).cpu().numpy()[:B]}
    for name, x in got.items():
        assert np.array_equal(x, ring[name].astype(x.dtype)), "%s: %s differs from the ring" % (label, name)
    h = np.zeros(B, np.uint8)
    if dd.nstep_tails:
        h = dd.debug_tensor("h", dtype=torch.uint8).cpu().numpy()[:B]
        assert np.array_equal(h, at(store.horizon)), "%s: the batch horizons differ from the ring" % label
    return idx, h, got["done"].astype(bool)


WORST = {}


def _record(name, value):
    WORST[name] = max(WORST.get(name, 0.0), value)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_case_every_step_checked(case):
    import d4pg_b200 as d4pg
    plan, precision, B, S, A, info, opt = case
    label = _id(case)
    lv = levels(case)
    post, clip = lv["actor_critic"] == "post_update", lv["gradient"] == "clip"
    feed = Feed(case, STEPS - 1)
    max_norm = _thresholds(d4pg, case, feed) if clip else None
    dd = _make(d4pg, case, eager=True, max_norm=max_norm)
    stats = ON.Stats(S) if dd.obs_normalizer is not None else None
    feed.put_fill(dd, stats)
    cstats = CC.ClipStats() if clip else None
    run = Checked(dd, plan, precision, label, post_update=post, stats=cstats.update if clip else None,
                  clip=(max_norm, WD, cstats) if clip else None)
    rstats = RC.Stats()
    store = dd.replayBuffer._store
    tail_rows, affines = 0, []
    for i in range(STEPS):
        if i:
            feed.put(dd, i - 1, stats)
        before = RC.snapshot(store) if dd.prioritized_replay else None
        W = SC.snapshot(dd) if i in (0, STEPS - 1) else None
        run.step(seed=100 + i)
        step = "%s k=%d" % (label, dd.optimizer_global_actor.step_count)
        torch.cuda.synchronize()
        if i == 0 and not post:       # a post-update learner is created on the tensor-core chain plan only
            # clipping adds the sum-of-squares launch; a uniform eager step has no priority write-back
            want = SC.KERNELS[plan] + (1 if clip else 0) - (0 if dd.prioritized_replay else 1)
            assert dd.kernels_per_step() == want, (plan, dd.kernels_per_step(), want)
        # the loss head, with each row's discount and IS weight
        P, cfg = HC.step_planes(dd), HC.step_config(dd)
        if dd.importance_weighted and dd.prioritized_replay:
            assert float(P["isw"].min()) < 0.99 * float(P["isw"].max()), "%s: IS weights all equal" % step
        rep = HC.Report(step + " heads")
        HC.check_planes(rep, P, cfg)
        _record("heads", rep.finish()[0])
        # the batch against the ring
        if stats is not None:
            _check_stats(dd.obs_normalizer, stats, step)
            affines.append(dd.obs_normalizer.affine.cpu().clone())
        idx, h, done = _check_rows(dd, stats, step)
        assert np.array_equal(h, P["h"])
        tail_rows += int(((h > 0) & ~done).sum())
        # the priority write-back
        if before is not None:
            prio = dd.last_batch_info()["prio"].cpu().numpy()
            RC.check_update(before, RC.snapshot(store), idx, prio, ALPHA, rstats, step)
        if W is not None:
            _record("layers", SC.check_step(dd, W, plan, precision, post_update=post, label=step)[0])
    ustats = cstats.update if clip else run.stats
    print(label, (cstats or ustats).line())
    _record("IS weight ulp", ustats.is_worst_ulp)
    assert ustats.steps == STEPS and ustats.power_min >= 1
    if dd.prioritized_replay:
        assert ustats.is_steps == STEPS and rstats.updates == STEPS
    if clip:
        _record("clip norm ulp", cstats.worst_norm_ulp)
        for name in ("actor", "critic"):
            assert cstats.clipped[name] >= 1 and cstats.unclipped[name] >= 1, (cstats.clipped, cstats.unclipped)
    if dd.nstep_tails:
        assert tail_rows > 0, "%s: no tail row (h > 0, done = 0) was sampled" % label
    if stats is not None:
        assert any(not torch.equal(x, y) for x, y in zip(affines, affines[1:])), "%s: the affine never changed" % label
    print("worst ratios so far:", WORST)


# ---- execution modes against eager steps ---------------------------------------------------------------------------
def _everything(dd):
    """(name, tensor) of STATE_ITEMS, the gradient norms, the normalizer's statistics and affine, the horizon column and
    the ring's length and position."""
    names = [n for n in STATE_ITEMS if dd.prioritized_replay or n not in ("sum tree", "min tree")]
    out = list(zip(names, _state(dd)))
    if any(dd.max_grad_norm):
        out.append(("gradient norms", torch.tensor(dd.last_grad_norms())))
    store = dd.replayBuffer._store
    if dd.obs_normalizer is not None:
        out += [("normalizer stats", dd.obs_normalizer.stats.cpu().clone()),
                ("normalizer affine", dd.obs_normalizer.affine.cpu().clone())]
    if dd.nstep_tails:
        out.append(("horizons", store.horizon.cpu().clone()))
    out.append(("len / position", torch.tensor([len(dd.replayBuffer), _ring_pos(store)])))
    return out


PIPE_CASES = [c for c in CASES if c[6].get("run", "eager") != "eager"]


@pytest.mark.gpu
@pytest.mark.parametrize("case", PIPE_CASES, ids=[_id(c) for c in PIPE_CASES])
def test_case_pipeline_equals_eager(case):
    """The case's execution mode and eager steps of the same learner, with the same seeds and the same inserts at the
    same points (train_n: between calls only), leave identical state after every step or train_n call (DESIGN.md
    §2.3-2.4: prefetch and the host pipeline give what sampling at the start of each step gives)."""
    import d4pg_b200 as d4pg
    run = case[6]["run"]
    calls = (1, 8, 8) if run == "train_n" else (1,) * 8
    feed = Feed(case, max(len(calls), STEPS) - 1)            # the threshold probe takes STEPS steps
    max_norm = _thresholds(d4pg, case, feed) if case[6].get("clip") else None
    piped, eager = _make(d4pg, case, eager=False, max_norm=max_norm), _make(d4pg, case, eager=True, max_norm=max_norm)
    for dd in (piped, eager):
        feed.put_fill(dd)
    steps = 0
    for j, n in enumerate(calls):
        if j:
            for dd in (piped, eager):
                feed.put(dd, j - 1)
        if run == "train_n":
            piped.train_n(n)
        else:
            random.seed(700 + steps)
            piped.train()
        for q in range(n):
            random.seed(700 + steps + q)
            eager.train()
        steps += n
        got, want = _everything(piped), _everything(eager)
        assert [k for k, _ in got] == [k for k, _ in want]
        for (item, x), (_, y) in zip(got, want):
            assert torch.equal(x, y), "%s after %d steps: %s differs from eager steps" % (_id(case), steps, item)
    assert piped.optimizer_global_actor.step_count == steps
