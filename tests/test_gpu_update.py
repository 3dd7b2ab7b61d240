"""The optimizer update of the learner step, bit for bit, on every step plan, clock and pipeline -- and the benchmarked
8-step graph, the host pipeline and profile_step against plain single steps.

tests/update_check.py restates Adam, Polyak and the device step clock in float32 on the device's own gradients and
moments (teacher-forced, bit-exact, with the power to tell step k from k - 1 / k + 1 and a stale target), and the IS
weights from the trees each batch was sampled from.  tests/step_check.py checks the layers of the step that produced
those gradients.

Which graph runs which step (csrc/learner.cu): d4pg_learner_run replays warm prefetch steps RUN_UNROLL = 8 at a time
from one graph, of which only the first step re-packs the wgmma weight images; steps 2-8 run on the images the Adam
kernel wrote.  The host pipeline (reference sampling with a CUDA graph) never re-packs unless the caller wrote the
parameters.  A learner re-created after steps were taken resumes its clock through d4pg_learner_set_counters.
"""
import random
from fractions import Fraction

import numpy as np
import pytest
import torch

from tests import clip_check as CC
from tests import step_check as SC
from tests import update_check as UC

F32 = np.float32


# ---- CPU: the restatement itself ----------------------------------------------------------------------------------------
def _round_f32(q):
    """Fraction -> the nearest float32, ties to even (the float32 neighbours of float(q) compared exactly)."""
    c = F32(float(q))
    cands = (np.nextafter(c, F32(-np.inf)), c, np.nextafter(c, F32(np.inf)))
    return min(cands, key=lambda x: (abs(Fraction(float(x)) - q), int(UC._bits(x).reshape(-1)[0]) & 1))


def _midpoint_cases(rng, n):
    """(a, b, c) with a * b + c within 2^-70 relative of a float32 rounding midpoint, on both sides of it and next to
    odd and even c: the float64 sum rounds onto the midpoint, and only its residual tells the direction."""
    cs = (rng.uniform(1.1, 1.9, n) * 2.0 ** rng.randint(-30, 30, n)).astype(F32)
    half = (np.spacing(cs).astype(np.float64) / 2)
    scale = 2.0 ** rng.randint(-3, 4, n)
    a = ((1 + 2.0 ** -23) * scale).astype(F32)
    sign = np.where(rng.rand(n) < 0.5, -1.0, 1.0)
    b = (sign * half * (1 - 2.0 ** -23) / scale).astype(F32)
    return a, b, cs


def test_fma32_equals_exact_rounding():
    """The float32 fma emulation equals the exactly rounded a * b + c (Fraction arithmetic) on random operands of wide
    range and on constructed midpoint cases, where a float64 sum rounded once more to float32 is wrong."""
    rng = np.random.RandomState(5)
    n = 1500
    a = (rng.uniform(0.01, 1, n) * 2.0 ** rng.randint(-8, 2, n)).astype(F32)
    b = (rng.randn(n) * 2.0 ** rng.randint(-40, 10, n)).astype(F32)
    c = (rng.randn(n) * 2.0 ** rng.randint(-40, 10, n)).astype(F32)
    ma, mb, mc = _midpoint_cases(rng, 500)
    a, b, c = np.concatenate([a, ma]), np.concatenate([b, mb]), np.concatenate([c, mc])
    got = UC.fma32(a, b, c)
    want = np.array([_round_f32(Fraction(float(x)) * Fraction(float(y)) + Fraction(float(z))) for x, y, z in zip(a, b, c)],
                    dtype=F32)
    assert not np.any(UC.differ(got, want))
    naive = (a.astype(np.float64) * b.astype(np.float64) + c.astype(np.float64)).astype(F32)
    wrong = int(np.count_nonzero(UC.differ(naive[n:], want[n:])))
    print("double rounding wrong on %d of 500 midpoint cases" % wrong)
    assert wrong >= 100


def _fake_net(rng, n=96):
    """Flat buffers of one network with padding at every 6th group of 4 and a few tail elements: before the step, and
    the gradient the step produced."""
    pad = np.zeros(n, dtype=bool)
    pad[(np.arange(n) // 4) % 6 == 5] = True
    pad[n - 8:n - 5] = True
    z = lambda x: np.where(pad, F32(0), x).astype(F32)
    g = z(rng.randn(n) * 1e-3)
    before = {"p": z(rng.randn(n) * 0.1), "t": z(rng.randn(n) * 0.1), "m": z(rng.randn(n) * 1e-4),
              "v": z(rng.rand(n) * 1e-7)}
    return before, g, pad


def _device(h, before, g, k, net):
    """What the kernel writes at step k: the same float32 operations in the same order."""
    nss, bc2s = h.scalars(k, net)[0][0]
    m1, v1 = UC.restate_m(h, g, before["m"]), UC.restate_v(h, g, before["v"])
    p1 = UC.restate_p(h, before["p"], m1, v1, nss, bc2s)
    return {"p": p1, "t": UC.restate_t(h, before["t"], p1), "m": m1, "v": v1, "g": g.copy()}


def _synthetic(k):
    rng = np.random.RandomState(17)
    h = UC.Hyper((1e-3, 2e-3), 0.9, 0.9, 1e-8, 0.001)
    before, after, pads = {}, {}, {}
    for i, (name, _) in enumerate(UC.NETS):
        b, g, pad = _fake_net(rng)
        before[name], pads[name] = b, pad
        after[name] = _device(h, b, g, k, i)
    return h, before, after, pads


@pytest.mark.parametrize("k", [1, 2, 7, 50])
def test_update_check_passes_the_kernel_and_rejects_a_wrong_update(k):
    """The check passes the kernel's own arithmetic and fails: a clock one step early or late, a stale target, the last
    float4 group of a network left un-updated, and a nonzero padding element."""
    h, before, after, pads = _synthetic(k)
    stats = UC.check_arrays(before, after, pads, h, k)
    assert stats.power_min >= 1

    def fails(after_, kk=k):
        with pytest.raises(AssertionError):
            UC.check_arrays(before, after_, pads, h, kk)

    for kk in (k - 1, k + 1):
        if kk >= 1:
            fails({name: _device(h, before[name], after[name]["g"], kk, i) for i, (name, _) in enumerate(UC.NETS)})
    fails(after, k + 1)
    stale = {name: dict(d, t=before[name]["t"].copy()) for name, d in after.items()}
    fails(stale)
    for name in ("actor", "critic"):
        short = {n_: dict(d) for n_, d in after.items()}
        e = np.nonzero(~pads[name])[0][-1] // 4 * 4          # the last float4 group that holds a parameter
        for key in ("p", "t", "m", "v"):
            x = short[name][key].copy()
            x[e:e + 4] = before[name][key][e:e + 4]
            short[name][key] = x
        fails(short)
    for key in ("p", "g", "m", "v", "t"):
        padded = {n_: dict(d) for n_, d in after.items()}
        x = padded["critic"][key].copy()
        x[np.nonzero(pads["critic"])[0][3]] = F32(1e-30)
        padded["critic"][key] = x
        fails(padded)


def test_scalar_candidates_only_near_a_midpoint():
    f = F32(0.1)
    lo, hi = float(f), float(np.nextafter(f, F32(1)))
    mid = (lo + hi) / 2
    assert len(UC.scalar_candidates(mid)[0]) == 2
    assert len(UC.scalar_candidates(np.nextafter(mid, 1.0))[0]) == 2
    assert UC.scalar_candidates(lo + (hi - lo) / 4) == ([f], False)
    assert UC.scalar_candidates(lo) == ([f], False)


def test_is_weight_check_passes_the_formula_and_rejects_a_neighbouring_beta():
    """A sampler that used beta at clock t passes; beta at t + 1 is off by more than the power margin."""
    from importlib import import_module
    sch = import_module("d4pg-pytorch_b200.prioritized_replay_memory").LinearSchedule(100000, final_p=1.0, initial_p=0.4)
    rng = np.random.RandomState(3)
    cap, n_len = 64, 50
    leaves = np.zeros(cap, dtype=F32)
    leaves[:n_len] = (rng.rand(n_len) * 3 + 0.01).astype(F32)
    s = np.zeros(2 * cap, dtype=F32); mn = np.full(2 * cap, np.inf, dtype=F32)
    s[cap:], mn[cap:cap + n_len] = leaves, leaves[:n_len]
    for i in range(cap - 1, 0, -1):
        s[i] = s[2 * i] + s[2 * i + 1]
        mn[i] = min(mn[2 * i], mn[2 * i + 1])
    tr = (s, mn, n_len, cap)
    idx = rng.randint(0, n_len, 32)
    t = 40
    w = UC.restate_weights(tr, idx, UC.schedule_beta(sch, t))[0][0]
    assert UC.is_weight_check(tr, idx, w, sch, t)
    with pytest.raises(AssertionError):
        UC.is_weight_check(tr, idx, UC.restate_weights(tr, idx, UC.schedule_beta(sch, t + 1))[0][0], sch, t)


# ---- GPU ---------------------------------------------------------------------------------------------------------------
def _cat(N, v=(-50.0, 0.0)):
    return {"type": "categorical", "v_min": v[0], "v_max": v[1], "n_atoms": N}


C5 = dict(projection="nstep", n_steps=5)


def _ddpg(d4pg, B, S, A, info, precision, seed=12, n=None, **kw):
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    n = n or max(2048, 2 * B)
    opts = dict(use_graph=False, chain="cluster", sampling="device", philox_seed=3, prefetch=False)
    opts.update(kw)
    dd = d4pg.DDPG(S, A, memory_size=n, batch_size=B, critic_dist_info=info, precision=precision, **opts)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(seed + 1)
    dd.replayBuffer.add_batch(*_rows(rng, n, S, A))
    with torch.no_grad():                     # the target networks differ from the online ones
        dd.actor_target.flat_params().mul_(1.01)
        dd.critic_target.flat_params().mul_(0.99)
    return dd


def _rows(rng, n, S, A):
    return (rng.randn(n, S).astype(np.float32), rng.uniform(-1, 1, (n, A)).astype(np.float32),
            (-3 * rng.rand(n)).astype(np.float32).astype(np.float64), rng.randn(n, S).astype(np.float32),
            rng.rand(n) < 0.05)


class Checked(object):
    """Steps of one learner, each followed by the update check at the step count the host has taken, the IS-weight
    check when prioritized, and the teacher-forced layer check when asked.  clip: (max_norm, weight_decay, ClipStats)
    of a learner that clips or decays; its update is then held to tests/clip_check.py."""

    def __init__(self, dd, plan, precision, label, post_update=False, stats=None, clip=None):
        self.dd, self.plan, self.precision, self.label, self.post_update = dd, plan, precision, label, post_update
        self.stats = stats if stats is not None else UC.Stats()
        self.clip = clip

    def step(self, how="train", layers=False, seed=None):
        dd = self.dd
        uc = UC.UpdateCheck(dd)
        W = SC.snapshot(dd) if layers else None
        tr = UC.trees(dd) if dd.prioritized_replay else None
        t = dd.beta_schedule.t if dd.prioritized_replay else None
        if seed is not None:
            random.seed(seed)
        dd.profile_step() if how == "profile" else dd.train()
        k = dd.optimizer_global_actor.step_count
        if self.clip is None:
            uc.check(dd, k, self.stats, self.label)
        else:
            max_norm, wd, cstats = self.clip
            CC.check_step(uc.before, UC.read(dd, grads=True), uc.pads, uc.h, k, max_norm, wd, dd.last_grad_norms(), cstats,
                          self.label)
        power = None
        if tr is not None:
            info = dd.last_batch_info()
            power = UC.is_weight_check(tr, info["idx"].cpu().numpy(), info["weights"].cpu().numpy(), dd.beta_schedule, t,
                                       self.stats, self.label)
        if layers:
            SC.check_step(dd, W, self.plan, self.precision, post_update=self.post_update, label="%s k=%d" % (self.label, k))
        return power


# (plan, precision, B, |s|, |a|, critic head, DDPG options): every (plan, precision) pair of step_check.MODES, both clock
# variants (prefetch / host pipeline: per-parity slots; otherwise the plain clock) and both sampling modes
UPDATE_CASES = [
    ("tc_chain", "tf32x3", 256, 17, 6, _cat(51), {"prefetch": True, "use_graph": True}),          # config 2 as benchmarked
    ("tc_chain", "tf32", 64, 17, 6, _cat(51), {"sampling": "reference", "prefetch": True, "use_graph": True}),  # host pipeline
    ("tc_chain", "tf32x3", 64, 17, 6, _cat(51), {"actor_critic": "post_update"}),                # two Adam launches
    ("tc_chain", "tf32x3", 256, 17, 6, _cat(51), {"importance_weighted": True, "priority": "ce", "sampling": "reference"}),
    ("tc_chain", "tf32x3", 64, 17, 6, {"type": "mixture_of_gaussian", "n_components": 5}, {"prefetch": True}),
    ("chain", "fp32", 64, 17, 6, _cat(51), {}),
    ("chain", "tf32x3", 64, 33, 6, _cat(51), {"prefetch": True}),
    ("chain", "tf32", 64, 33, 6, _cat(51), {"sampling": "reference"}),
    ("levels", "fp32", 1025, 17, 6, {"type": "quantile", "n_quantiles": 51}, {}),                # split-K dW, quantile head
    ("levels", "tf32x3", 4096, 17, 6, _cat(101, (-150.0, 150.0)), dict(C5, prefetch=True)),     # config 5 shapes
    ("levels", "tf32", 1025, 17, 6, _cat(51), {"prefetch": True, "chain": "levels"}),
    ("levels", "bf16", 256, 17, 6, _cat(51), {}),
    ("levels", "fp32", 64, 17, 6, _cat(51), {"chain": "levels", "sampling": "reference", "prefetch": True, "use_graph": True}),
]
STEPS = 20


def _id(case):
    plan, prec, B, S, A, info, kw = case
    head = {"categorical": "N", "quantile": "qr", "mixture_of_gaussian": "mogK"}[info["type"]]
    width = info.get("n_atoms") or info.get("n_quantiles") or info.get("n_components")
    return "%s-%s-B%d-s%d-a%d-%s%d%s" % (plan, prec, B, S, A, head, width,
                                         "".join("-%s" % (k if v is True else v) for k, v in sorted(kw.items())))


@pytest.mark.gpu
@pytest.mark.parametrize("case", UPDATE_CASES, ids=[_id(c) for c in UPDATE_CASES])
def test_update_bit_exact_every_step(case):
    """20 steps of every plan: the update bit-exact at the right step count on each, the IS weights within one ulp,
    every layer of the first and the last step within its bound."""
    import d4pg_b200 as d4pg
    plan, precision, B, S, A, info, kw = case
    dd = _ddpg(d4pg, B, S, A, info, precision, **kw)
    run = Checked(dd, plan, precision, _id(case), post_update=kw.get("actor_critic") == "post_update")
    powered = [run.step(layers=(i in (0, STEPS - 1)), seed=100 + i) for i in range(STEPS)]
    print(run.stats.line())
    assert sum(bool(p) for p in powered) >= STEPS // 2, powered


# ---- the 8-step graph ----------------------------------------------------------------------------------------------------
def _bench_c2(d4pg):
    """The device-sampled learner of bench.py's c2 workload, built as bench.py builds it."""
    import bench
    cfg = bench.CFG["c2"]
    info = {"type": "categorical", "v_min": cfg["v_min"], "v_max": cfg["v_max"], "n_atoms": cfg["atoms"]}
    torch.manual_seed(0); random.seed(0)
    dd = d4pg.DDPG(cfg["obs"], cfg["act"], memory_size=cfg["cap"], batch_size=cfg["batch"], critic_dist_info=info,
                   n_steps=cfg["n_steps"], projection=cfg["proj"], sampling="device", philox_seed=1234,
                   precision="tf32x3", chain="cluster")
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    dd.replayBuffer.add_batch(*bench.synth(cfg, cfg["cap"], seed=0))
    return dd


GRAPH_CASES = {
    "bench_c2": ("tc_chain", "tf32x3", None),
    "tc_chain_tf32": ("tc_chain", "tf32", (256, 17, 6, _cat(51), {})),
    "post_update": ("tc_chain", "tf32x3", (64, 17, 6, _cat(51), {"actor_critic": "post_update"})),
    "iw_ce": ("tc_chain", "tf32x3", (256, 17, 6, _cat(51), {"importance_weighted": True, "priority": "ce"})),
    "quantile": ("tc_chain", "tf32x3", (256, 17, 6, {"type": "quantile", "n_quantiles": 51}, {})),
    "c5": ("levels", "tf32x3", (4096, 17, 6, _cat(101, (-150.0, 150.0)), C5)),
}


STATE_ITEMS = ("actor", "actor_target", "critic", "critic_target", "actor exp_avg", "actor exp_avg_sq", "critic exp_avg",
               "critic exp_avg_sq", "actor gradient", "critic gradient", "sum tree", "min tree", "idx", "weights", "prio",
               "losses")


def _state(dd):
    """Everything a step of a prioritized learner leaves behind (STATE_ITEMS), as CPU tensors."""
    torch.cuda.synchronize()
    out = [getattr(dd, n).flat_params().cpu().clone() for n in ("actor", "actor_target", "critic", "critic_target")]
    for opt, net in ((dd.optimizer_global_actor, dd.actor), (dd.optimizer_global_critic, dd.critic)):
        out += [x.cpu().clone() for x in opt.moments(net)]
    out += [dd.actor.flat_grads().cpu().clone(), dd.critic.flat_grads().cpu().clone()]
    if dd.prioritized_replay:
        st = dd.replayBuffer._store
        out += [st.sum_tree.cpu().clone(), st.min_tree.cpu().clone()]
    info = dd.last_batch_info()
    out += [info[k].cpu().clone() for k in ("idx", "weights", "prio")]
    out.append(torch.tensor(dd.last_losses()))
    return out


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(GRAPH_CASES))
def test_eight_step_graph_equals_single_steps(name):
    """train_n replays warm steps 8 at a time from one graph (steps 2-8 on the weight images the Adam kernel wrote):
    it must leave exactly what single train() steps (CUDA graph per step) and eager steps leave.  A runs train_n(1, 8,
    1, 8), an add_batch, train_n(9): both parities of the 8-step graph and a cold step before a graph in one call; one
    more checked step then holds its clocks to step 28.  The config-5 learner (levels, B 4096) sums split-K dW slices
    with atomics, which is not bit-reproducible run to run: there only the clocks are checked."""
    import d4pg_b200 as d4pg
    plan, precision, shape = GRAPH_CASES[name]
    add_rng = np.random.RandomState(77)
    extra = _rows(add_rng, 37, 17, 6)

    def make(use_graph):
        if shape is None:
            dd = _bench_c2(d4pg)
            dd.use_graph = use_graph
            return dd
        B, S, A, info, kw = shape
        return _ddpg(d4pg, B, S, A, info, precision, prefetch=True, use_graph=use_graph, **kw)

    stats = UC.Stats()
    a = make(True)
    for n in (1, 8, 1, 8):
        a.train_n(n)
    a.replayBuffer.add_batch(*extra)
    a.train_n(9)
    assert a.optimizer_global_actor.step_count == 27
    ref = _state(a)
    # the clocks the graphs left behind: the next step's update and IS weights at step 28
    Checked(a, plan, precision, "%s after train_n" % name, post_update="post_update" in name, stats=stats).step()
    del a
    torch.cuda.empty_cache()
    if plan == "levels":          # split-K dW sums its slices with fp32 atomics: not bit-reproducible, only the clock is
        print(name, stats.line())
        return
    for use_graph in (True, False):
        dd = make(use_graph)
        run = Checked(dd, plan, precision, "%s graph=%s" % (name, use_graph), post_update="post_update" in name, stats=stats)
        for i in range(27):
            if i == 18:
                dd.replayBuffer.add_batch(*extra)
            run.step()
        got = _state(dd)
        for item, x, y in zip(STATE_ITEMS, ref, got):
            assert torch.equal(x, y), "%s: %s after train_n differs from single steps (graph=%s)" % (name, item, use_graph)
        del dd, run
        torch.cuda.empty_cache()
    print(name, stats.line())


# ---- the host pipeline ---------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["tf32x3", "tf32"])
def test_host_pipeline_equals_eager(precision):
    """bench.py's end-to-end loop -- pinned add_batch, train() with host-drawn uniforms through the host pipeline, which
    re-packs the wgmma weight images only after a parameter write -- against eager steps: losses, indices and parameters
    bit-identical after every step, across a load_state_dict and a .data write reported with weights_changed()."""
    import d4pg_b200 as d4pg
    B, S, A = 64, 17, 6
    runs = [_ddpg(d4pg, B, S, A, _cat(51), precision, n=1024, sampling="reference", prefetch=True, use_graph=g)
            for g in (True, False)]
    eager = Checked(runs[1], "tc_chain", precision, "eager %s" % precision)
    rng = np.random.RandomState(12)
    for t in range(10):
        pin = [torch.from_numpy(np.ascontiguousarray(x)).pin_memory() for x in _rows(rng, 96, S, A)]
        for dd in runs:
            dd.replayBuffer.add_batch(*pin)
        if t == 5:
            for dd in runs:
                dd.actor.load_state_dict({k: v * 0.9 for k, v in dd.actor.state_dict().items()})
        if t == 6:
            for dd in runs:
                for prm in dd.critic.parameters():
                    prm.data.mul_(0.95)
                dd.weights_changed()
        random.seed(700 + t)
        runs[0].train()
        eager.step(seed=700 + t)
        for item, x, y in zip(STATE_ITEMS, _state(runs[0]), _state(runs[1])):
            assert torch.equal(x, y), "step %d: %s of the host pipeline differs from eager steps" % (t, item)
    print(eager.stats.line())


# ---- the clock across a re-created learner ---------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("sampling", ["device", "reference"])
def test_clock_continues_across_a_recreated_learner(sampling):
    """assign_global_optimizer with the same optimizers mid-run re-creates the learner, which resumes the Adam and PER
    beta clocks through d4pg_learner_set_counters: with train(), train_n() and profile_step() mixed, the run must be
    bit-identical to one that keeps its learner, and the update must hold at the right step count throughout."""
    import d4pg_b200 as d4pg
    B, S, A = 64, 17, 6
    plan = [("train", 3), ("n", 9), ("profile", 1), ("recreate", 0), ("train", 2), ("n", 8), ("profile", 1),
            ("recreate", 0), ("profile", 1), ("train", 2)]
    if sampling == "reference":                       # train_n needs device sampling
        plan = [(h, n) if h != "n" else ("train", 2) for h, n in plan]
    finals = []
    for recreate in (True, False):
        dd = _ddpg(d4pg, B, S, A, _cat(51), "tf32x3", sampling=sampling, prefetch=True, use_graph=True)
        run = Checked(dd, "tc_chain", "tf32x3", "%s recreate=%s" % (sampling, recreate))
        seed = 0
        for how, n in plan:
            if how == "recreate":
                if recreate:
                    dd.assign_global_optimizer(dd.optimizer_global_actor, dd.optimizer_global_critic)
                continue
            if how == "n":
                dd.train_n(n)
                continue
            for _ in range(n):
                run.step(how, seed=seed)
                seed += 1
        finals.append(_state(dd))
        print(run.stats.line())
    for item, x, y in zip(STATE_ITEMS, *finals):
        assert torch.equal(x, y), "%s differs after re-creating the learner" % item


# ---- profile_step --------------------------------------------------------------------------------------------------------
PROFILE_CASES = [("tc_chain", "tf32x3", 256), ("levels", "fp32", 1025), ("levels", "tf32x3", 1025),
                 ("levels", "fp32", 4096), ("levels", "tf32x3", 4096)]


@pytest.mark.gpu
@pytest.mark.parametrize("plan,precision,B", PROFILE_CASES)
def test_profile_step_is_a_real_step(plan, precision, B):
    """profile_step times every launch of an eager step (repeating the idempotent ones) and counts as a training step:
    its gradients, update and clock must be those of an ordinary step, also where the level plan's dW runs split-K."""
    import d4pg_b200 as d4pg
    dd = _ddpg(d4pg, B, 17, 6, _cat(51), precision)
    run = Checked(dd, plan, precision, "profile %s/%s B%d" % (plan, precision, B))
    run.step()
    run.step("profile", layers=True)
    print(run.stats.line())
