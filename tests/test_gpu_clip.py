"""Global-norm gradient clipping, Adam weight decay and the reported gradient norms of the fused learner step.

tests/clip_check.py restates the clipping coefficient and the effective gradient on the device's own gradient and
parameters and hands the rest of the update to tests/update_check.py (bit-exact, teacher-forced).  Here: that check on
every step plan, precision, critic head and pipeline; "report only" (max_grad_norm=inf) against a learner without the
option; the 8-step graph, single-step graphs, eager steps and the host pipeline against each other; the oracle with
torch's clip_grad_norm_ and Adam(weight_decay=); SharedAdam.step() against torch.optim.Adam; the rejected configs.
"""
import ctypes as C
import math
import random

import numpy as np
import pytest
import torch

from tests import clip_check as CC
from tests import step_check as SC
from tests import update_check as UC
from tests.test_gpu_update import STATE_ITEMS, UPDATE_CASES, _cat, _ddpg, _id, _rows, _state

F32 = np.float32
WD = (1e-4, 3e-4)


# ---- CPU: the restatement itself ----------------------------------------------------------------------------------------
def _fake_net(rng, n=96):
    pad = np.zeros(n, dtype=bool)
    pad[(np.arange(n) // 4) % 6 == 5] = True
    z = lambda x: np.where(pad, F32(0), x).astype(F32)
    g = z(rng.randn(n) * 1e-2)
    before = {"p": z(rng.randn(n) * 0.1), "t": z(rng.randn(n) * 0.1), "m": z(rng.randn(n) * 1e-4), "v": z(rng.rand(n) * 1e-7)}
    return before, g, pad


def _device(h, before, g, k, net, coef, wd):
    """What the kernel writes at step k: the plain update on the effective gradient; the buffer keeps g."""
    nss, bc2s = h.scalars(k, net)[0][0]
    ge = CC.effective_gradient(g, before["p"], coef, wd)
    m1, v1 = UC.restate_m(h, ge, before["m"]), UC.restate_v(h, ge, before["v"])
    p1 = UC.restate_p(h, before["p"], m1, v1, nss, bc2s)
    return {"p": p1, "t": UC.restate_t(h, before["t"], p1), "m": m1, "v": v1, "g": g.copy()}


def _synthetic(k, max_norm, wd, coef_shift=0, drop_decay=False):
    rng = np.random.RandomState(23)
    h = UC.Hyper((1e-3, 2e-3), 0.9, 0.9, 1e-8, 0.001)
    before, after, pads, norms = {}, {}, {}, []
    for i, (name, _) in enumerate(UC.NETS):
        b, g, pad = _fake_net(rng)
        coef = CC.coef_candidates(CC.norm(g), max_norm[i])[0][0]
        for _ in range(coef_shift):
            coef = np.nextafter(coef, F32(0))
        before[name], pads[name] = b, pad
        after[name] = _device(h, b, g, k, i, coef, 0.0 if drop_decay else wd[i])
        norms.append(F32(CC.norm(g)))
    return h, before, after, pads, norms


@pytest.mark.parametrize("k", [1, 7])
def test_clip_check_passes_the_kernel_and_rejects_a_wrong_coefficient_or_decay(k):
    """The check accepts the kernel's own arithmetic -- clipping, not clipping, decay or not -- and fails a coefficient
    one ulp off, a missing decay term, a norm two ulp off and a gradient buffer that holds the clipped gradient."""
    na, nc = (float(x) for x in _synthetic(k, (0.0, 0.0), (0.0, 0.0))[4])
    for max_norm, wd, clips in (((na / 3, nc / 5), WD, (True, True)), ((na * 4, nc / 2), (0.0, 1e-3), (False, True)),
                                ((math.inf, 0.0), (0.0, 0.0), (False, False))):
        h, before, after, pads, norms = _synthetic(k, max_norm, wd)
        coefs = CC.check_step(before, after, pads, h, k, max_norm, wd, norms)
        assert tuple(c < 1 for c in coefs.values()) == clips
    max_norm = (na / 3, nc / 5)
    h, before, after, pads, norms = _synthetic(k, max_norm, WD, coef_shift=1)
    with pytest.raises(AssertionError, match="differ from the restatement"):
        CC.check_step(before, after, pads, h, k, max_norm, WD, norms)
    h, before, after, pads, norms = _synthetic(k, max_norm, WD, drop_decay=True)
    with pytest.raises(AssertionError, match="differ from the restatement"):
        CC.check_step(before, after, pads, h, k, max_norm, WD, norms)
    h, before, after, pads, norms = _synthetic(k, max_norm, WD)
    off = [np.nextafter(np.nextafter(norms[0], F32(np.inf)), F32(np.inf)), norms[1]]
    with pytest.raises(AssertionError, match="reported norm"):
        CC.check_step(before, after, pads, h, k, max_norm, WD, off)
    clipped = {n_: dict(d) for n_, d in after.items()}
    clipped["actor"]["g"] = CC.effective_gradient(after["actor"]["g"], before["actor"]["p"], F32(0.5), 0.0)
    with pytest.raises(AssertionError):
        CC.check_step(before, clipped, pads, h, k, max_norm, WD, norms)


def test_coef_candidates():
    assert CC.coef_candidates(3.0, None) == ([F32(1.0)], False)
    assert CC.coef_candidates(3.0, math.inf) == ([F32(1.0)], False)
    assert CC.coef_candidates(0.5, 40.0) == ([F32(1.0)], False)
    c, mid = CC.coef_candidates(80.0, 40.0)
    assert c == [F32(40.0 / (80.0 + 1e-6))] and not mid
    f = F32(0.3)
    midpoint = (float(f) + float(np.nextafter(f, F32(1)))) / 2
    both, mid = CC.coef_candidates(1.0 / midpoint - 1e-6, 1.0)
    assert mid and len(both) == 2


def test_options_are_validated_on_the_host():
    """(DDPG on its default device: with a GPU present its replay store is allocated, and initialised, at once.)"""
    import d4pg_b200 as d4pg
    info = _cat(51)
    a = d4pg.actor(5, 2, device="cpu")
    opt = d4pg.SharedAdam(a.parameters(), weight_decay=1e-4)
    assert opt.weight_decay() == 1e-4 and opt.hyper() == (1e-3, 0.9, 0.9, 1e-8)
    assert d4pg.SharedAdam(a.parameters()).weight_decay() == 0.0
    assert d4pg.SharedAdam(a.parameters(), max_grad_norm=math.inf).max_grad_norm == math.inf
    for bad in (-1e-4, math.nan, math.inf):
        with pytest.raises(ValueError):
            d4pg.SharedAdam(a.parameters(), weight_decay=bad)
    for bad in (0.0, -1.0, math.nan):
        with pytest.raises(ValueError):
            d4pg.SharedAdam(a.parameters(), max_grad_norm=bad)
        with pytest.raises(ValueError):
            d4pg.DDPG(5, 2, memory_size=8, batch_size=4, critic_dist_info=info, max_grad_norm=bad)
        with pytest.raises(ValueError):
            d4pg.DDPG(5, 2, memory_size=8, batch_size=4, critic_dist_info=info, max_grad_norm=(1.0, bad))
    dd = d4pg.DDPG(5, 2, memory_size=8, batch_size=4, critic_dist_info=info, max_grad_norm=(40.0, None))
    assert dd.max_grad_norm == (40.0, 0.0)
    assert d4pg.DDPG(5, 2, memory_size=8, batch_size=4, critic_dist_info=info).max_grad_norm == (0.0, 0.0)
    with pytest.raises(d4pg.D4PGError, match="max_grad_norm"):
        d4pg.DDPG(5, 2, memory_size=8, batch_size=4, critic_dist_info=info).last_grad_norms()


def test_oracle_hook_with_the_options_off_changes_nothing():
    """clip_hook(None, (0, 0)) leaves LearnerOracle.train_step bit for bit what it is without a hook."""
    from oracle import d4pg_oracle as O
    from tests import helpers as H
    g = H.load("train_per_part.npz")
    S, A, R, S2, D = H.train_data(g)
    obs_dim, act_dim, n_atoms = [int(x) for x in g["meta"][:3]]
    info = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": n_atoms}
    outs = []
    for hooked in (False, True):
        a, c = H.regen_init(int(g["seed"]), obs_dim, act_dim, n_atoms)
        lo = O.LearnerOracle(obs_dim, act_dim, info, actor_w=a, critic_w=c)
        log = []
        for t in range(2):
            rows = slice(16 * t, 16 * t + 16)
            lo.train_step(S[rows], A[rows], R[rows], S2[rows], D[rows],
                          grad_hook=CC.clip_hook(lo, None, (0.0, 0.0), log) if hooked else None)
        outs.append([O.flatten(w) for w in (lo.actor, lo.critic, lo.actor_target, lo.critic_target, lo.m_a, lo.v_c)])
    for x, y in zip(*outs):
        assert np.array_equal(x, y)
    a, c = H.regen_init(int(g["seed"]), obs_dim, act_dim, n_atoms)
    lo = O.LearnerOracle(obs_dim, act_dim, info, actor_w=a, critic_w=c)
    log = []
    lo.train_step(S[:16], A[:16], R[:16], S2[:16], D[:16], grad_hook=CC.clip_hook(lo, 1e-4, WD, log))
    assert log[0][2] < 1 and log[0][3] < 1
    assert not np.array_equal(O.flatten(lo.m_a), outs[0][4])


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _learner(d4pg, case, max_grad_norm, wd=WD, **more):
    plan, precision, B, S, A, info, kw = case
    dd = _ddpg(d4pg, B, S, A, info, precision, max_grad_norm=max_grad_norm, **dict(kw, **more))
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3, weight_decay=wd[0]),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3, weight_decay=wd[1]))
    return dd


STEPS = 20


@pytest.mark.gpu
@pytest.mark.parametrize("case", UPDATE_CASES, ids=[_id(c) for c in UPDATE_CASES])
def test_clipped_update_bit_exact_every_step(case):
    """20 steps of every plan with a threshold and a decay on both networks: m, v, p, t bit-equal to the restatement on
    the effective gradient, padding zero, the gradient buffer unclipped, the reported norms within one ulp.  The
    thresholds are the lower-quartile norms of a report-only run of the same learner, so both branches are taken."""
    import d4pg_b200 as d4pg
    plan, precision = case[0], case[1]
    probe = _learner(d4pg, case, math.inf)
    seen = []
    for i in range(STEPS):
        random.seed(100 + i)
        probe.train()
        seen.append(probe.last_grad_norms())
    del probe
    torch.cuda.empty_cache()
    max_norm = tuple(float(sorted(n[i] for n in seen)[STEPS // 4]) for i in range(2))
    assert all(math.isfinite(x) and x > 0 for x in max_norm), seen

    dd = _learner(d4pg, case, max_norm)
    post = case[6].get("actor_critic") == "post_update"
    stats = CC.ClipStats()
    pads = None
    # The layers of the first step, whose weights and batch the seeds fix, and of the last one where the run repeats
    # bit for bit.  Split-K dW (the level plan from batch 1024) adds its slices with fp32 atomics in any order, and
    # Adam turns those last-bit differences into different weights: the last step's planes, and the power of the bound
    # on them, then change from run to run.
    layer_steps = (0,) if plan == "levels" and case[2] >= 1024 else (0, STEPS - 1)
    for i in range(STEPS):
        before = UC.read(dd, grads=False)
        W = SC.snapshot(dd) if i in layer_steps else None
        random.seed(100 + i)
        dd.train()
        if pads is None:
            pads = {name: UC.pad_mask(getattr(dd._learner.global_model, name)) for name, _ in UC.NETS}
        k = dd.optimizer_global_actor.step_count
        CC.check_step(before, UC.read(dd, grads=True), pads, UC.Hyper.of(dd), k, max_norm, WD, dd.last_grad_norms(),
                      stats, _id(case))
        if W is not None:             # the layers that produced the gradient are those of an unclipped step
            SC.check_step(dd, W, plan, precision, post_update=post, label="%s k=%d" % (_id(case), k))
    print(stats.line(), "thresholds", max_norm)
    assert dd.kernels_per_step() > 0
    for name in ("actor", "critic"):
        assert stats.clipped[name] >= STEPS // 2 and stats.unclipped[name] >= 1, (stats.clipped, stats.unclipped)
    assert stats.power_min >= 1


DET_CASES = {
    "bench_like": ("tc_chain", "tf32x3", 256, 17, 6, _cat(51), {"prefetch": True, "use_graph": True}),
    "post_update": ("tc_chain", "tf32x3", 64, 17, 6, _cat(51), {"prefetch": True, "use_graph": True, "actor_critic": "post_update"}),
    "chain_fp32": ("chain", "fp32", 64, 17, 6, {"type": "quantile", "n_quantiles": 51}, {"prefetch": True, "use_graph": True}),
}


@pytest.mark.gpu
@pytest.mark.parametrize("name", sorted(DET_CASES))
def test_report_only_changes_nothing_but_the_launch_count(name):
    """max_grad_norm=inf measures and reports: after train_n(1, 8, 1, 8) the learner's whole state is bit for bit that of
    a learner without the option, with one more launch per Adam launch; weight decay alone adds no launch."""
    import d4pg_b200 as d4pg
    case = DET_CASES[name]
    adams = 2 if name == "post_update" else 1
    states, counts = [], []
    for max_norm, wd in ((None, (0.0, 0.0)), (math.inf, (0.0, 0.0)), (None, WD)):
        dd = _learner(d4pg, case, max_norm, wd)
        for n in (1, 8, 1, 8):
            dd.train_n(n)
        states.append(_state(dd))
        counts.append(dd.kernels_per_step())
        if max_norm:
            na, nc = dd.last_grad_norms()
            assert abs(na - float(dd.actor.flat_grads().double().norm())) <= 1e-6 * na
            assert abs(nc - float(dd.critic.flat_grads().double().norm())) <= 1e-6 * nc
        del dd
        torch.cuda.empty_cache()
    assert counts[1] == counts[0] + adams and counts[2] == counts[0], counts
    for item, x, y in zip(STATE_ITEMS, states[0], states[1]):
        assert torch.equal(x, y), "%s: %s differs with max_grad_norm=inf" % (name, item)
    assert not torch.equal(states[0][0], states[2][0]), "weight decay left the actor unchanged"


def _full_state(dd):
    return _state(dd) + [torch.tensor(dd.last_grad_norms())]


@pytest.mark.gpu
@pytest.mark.parametrize("name", ["bench_like", "post_update"])
def test_clipped_graphs_equal_eager_steps(name):
    """Clipping and decay on: the 8-step graph, single-step graphs and eager profile_step steps leave identical state
    and report identical norms."""
    import d4pg_b200 as d4pg
    case = DET_CASES[name]
    max_norm = (0.02, 0.05)

    def make(use_graph):
        return _learner(d4pg, case, max_norm, use_graph=use_graph)

    a = make(True)
    for n in (1, 8, 1, 8):
        a.train_n(n)
    ref = _full_state(a)
    del a
    for use_graph, how in ((True, "train"), (False, "profile")):
        dd = make(use_graph)
        for i in range(18):
            names = dd.profile_step() if how == "profile" else dd.train()
        if how == "profile":
            assert [n for n, _ in names].count("launch_grad_sqnorm") == (2 if name == "post_update" else 1), names
        for item, x, y in zip(STATE_ITEMS + ("gradient norms",), ref, _full_state(dd)):
            assert torch.equal(x, y), "%s: %s after train_n differs from %s steps" % (name, item, how)
        del dd
        torch.cuda.empty_cache()


@pytest.mark.gpu
def test_clipped_host_pipeline_equals_eager():
    import d4pg_b200 as d4pg
    case = ("tc_chain", "tf32x3", 64, 17, 6, _cat(51), {"sampling": "reference", "prefetch": True})
    runs = [_learner(d4pg, case, (0.02, 0.05), use_graph=g, n=1024) for g in (True, False)]
    rng = np.random.RandomState(12)
    for t in range(8):
        pin = [torch.from_numpy(np.ascontiguousarray(x)).pin_memory() for x in _rows(rng, 96, 17, 6)]
        for dd in runs:
            dd.replayBuffer.add_batch(*pin)
            random.seed(700 + t)
            dd.train()
        for item, x, y in zip(STATE_ITEMS + ("gradient norms",), _full_state(runs[0]), _full_state(runs[1])):
            assert torch.equal(x, y), "step %d: %s of the host pipeline differs from eager steps" % (t, item)
        assert runs[0].last_grad_norms(lag=1 if t else 0) is not None


@pytest.mark.gpu
@pytest.mark.parametrize("plan,precision,chain", [("tc_chain", "tf32x3", "cluster"), ("chain", "fp32", "cluster"),
                                                  ("levels", "fp32", "levels")])
def test_clipped_steps_vs_oracle(plan, precision, chain):
    """Five steps at config-2 shapes against the oracle with clip_grad_norm_ and Adam's weight decay, clipping active."""
    import d4pg_b200 as d4pg
    from oracle import d4pg_oracle as O
    from tests import helpers as H
    TOL = 1e-5
    B, n = 256, 4096
    info = _cat(51)
    wd = (1e-4, 1e-4)
    rows = _rows(np.random.RandomState(4), n, 17, 6)

    def make(max_norm):
        torch.manual_seed(3); np.random.seed(3); random.seed(3)
        dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=info, precision=precision, chain=chain,
                       sampling="device", philox_seed=5, max_grad_norm=max_norm)
        dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3, weight_decay=wd[0]),
                                   d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3, weight_decay=wd[1]))
        dd.replayBuffer.add_batch(*rows)
        return dd

    probe = make(math.inf)                     # thresholds: a quarter of the first step's norms, so every step clips
    probe.train()
    max_norm = tuple(0.25 * x for x in probe.last_grad_norms())
    del probe
    dd = make(max_norm)
    lo = O.LearnerOracle(17, 6, info, actor_w={k: v.cpu().clone() for k, v in dd.actor.state_dict().items()},
                         critic_w={k: v.cpu().clone() for k, v in dd.critic.state_dict().items()})
    log = []
    for t in range(5):
        dd.train()
        idx = dd.last_batch_info()["idx"].cpu().numpy()
        lo.train_step(*[x[idx] for x in rows], grad_hook=CC.clip_hook(lo, max_norm, wd, log))
        assert log[-1][2] < 1 and log[-1][3] < 1, log[-1]
        for mine, ref in zip(dd.last_grad_norms(), log[-1][:2]):
            assert abs(mine - ref) <= 1e-5 * ref + 1e-4 * TOL, (t, mine, ref)
        opts = (dd.optimizer_global_actor, dd.optimizer_global_critic)
        for k in H.NAMES:
            pairs = [(dd.actor.state_dict()[k], lo.actor[k]), (dd.critic.state_dict()[k], lo.critic[k]),
                     (dd.actor_target.state_dict()[k], lo.actor_target[k]), (dd.critic_target.state_dict()[k], lo.critic_target[k])]
            for mine, ref in pairs:
                err = (mine.cpu() - ref).abs()
                assert err.max().item() <= 2.5e-4 and (err > TOL).float().mean().item() <= 0.1, (t, k)
        for opt, net, m_ref, v_ref in ((opts[0], dd.actor, lo.m_a, lo.v_a), (opts[1], dd.critic, lo.m_c, lo.v_c)):
            m, v = opt.moments(net)
            for (mw, mb), (vw, vb), name in zip(net._views(m), net._views(v), ("fc1", "fc2", "fc2_2", "fc3")):
                for mine, ref in ((mw, m_ref[name + ".weight"]), (mb, m_ref[name + ".bias"]),
                                  (vw, v_ref[name + ".weight"]), (vb, v_ref[name + ".bias"])):
                    assert (mine.cpu().reshape(ref.shape) - ref).abs().max().item() <= TOL, (t, name)


@pytest.mark.gpu
@pytest.mark.parametrize("max_norm,wd", [(None, 1e-2), (0.05, 0.0), (0.05, 1e-2), (math.inf, 0.0)])
def test_shared_adam_step_vs_torch(max_norm, wd):
    """SharedAdam.step() on a differentiable critic against clip_grad_norm_ + torch.optim.Adam(weight_decay=) on a CPU
    copy fed the same gradients."""
    import d4pg_b200 as d4pg
    torch.manual_seed(2)
    c = d4pg.critic(17, 6, _cat(51), device="cuda", differentiable=True)
    opt = d4pg.SharedAdam(c.parameters(), lr=1e-3, weight_decay=wd, max_grad_norm=max_norm)
    ref = [torch.nn.Parameter(p.detach().cpu().clone()) for p in c.parameters()]
    topt = torch.optim.Adam(ref, lr=1e-3, betas=(0.9, 0.9), eps=1e-8, weight_decay=wd)
    s, a = torch.randn(32, 17, device="cuda"), torch.rand(32, 6, device="cuda") * 2 - 1
    w = torch.randn(32, 51, device="cuda")
    for t in range(3):
        c.zero_grad()
        (c(s, a) * w).sum().backward()
        c.flat_grads()
        for r, p in zip(ref, c.parameters()):
            r.grad = p.grad.detach().cpu().clone()
        if max_norm is not None:
            total = float(torch.nn.utils.clip_grad_norm_(ref, max_norm))
        topt.step()
        opt.step()
        if max_norm is not None:
            assert abs(opt.last_grad_norm() - total) <= 1e-5 * total
            if max_norm == 0.05:
                assert total > max_norm            # the threshold does clip
        for r, p in zip(ref, c.parameters()):
            assert (p.detach().cpu() - r.detach()).abs().max().item() <= 1e-6, t
    assert float(c.flat_params().cpu()[torch.from_numpy(UC.pad_mask(c))].abs().max()) == 0.0


@pytest.mark.gpu
def test_rejected_configurations():
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib
    dd = _ddpg(d4pg, 64, 17, 6, _cat(51), "fp32")
    dd.train()
    with pytest.raises(d4pg.D4PGError, match="max_grad_norm"):
        dd.last_grad_norms()
    # the C entry: the learner's own (valid) config with one field changed at a time
    L = _lib.lib()
    cfg = _lib.LearnerConfig.from_buffer_copy(dd._learner.cfg)
    buf = _lib.LearnerBuffers()
    h = C.c_void_p()

    def create(**fields):
        c = _lib.LearnerConfig.from_buffer_copy(cfg)
        for k, v in fields.items():
            setattr(c, k, v)
        rc = L.d4pg_learner_create(C.byref(c), C.byref(buf), dd.replayBuffer._store.handle, None, C.byref(h))
        return rc, L.d4pg_last_error().decode()

    for fields, text in (({"max_grad_norm_actor": -1.0}, "max_grad_norm must be"),
                         ({"max_grad_norm_critic": math.nan}, "max_grad_norm must be"),
                         ({"weight_decay_actor": -1e-4}, "weight_decay must be"),
                         ({"weight_decay_critic": math.inf}, "weight_decay must be")):
        rc, msg = create(**fields)
        assert rc == _lib.EINVAL and text in msg, (fields, rc, msg)
    # data parallel: the library rejects the threshold before it looks at the communicator, and so does DDPG
    rc, msg = create(world_size=2, max_grad_norm_critic=40.0)
    assert rc == _lib.EINVAL and "world_size > 1" in msg and "summed inside the Adam kernel" in msg, (rc, msg)
    rc, msg = create(world_size=2, weight_decay_critic=1e-4)
    assert rc == _lib.EINVAL and "needs a communicator" in msg, (rc, msg)      # decay alone gets as far as an unclipped config

    class _Comm(object):
        world_size, handle = 2, None
    dd2 = _ddpg(d4pg, 64, 17, 6, _cat(51), "fp32", max_grad_norm=1.0)
    dd2.comm = _Comm()
    with pytest.raises(d4pg.D4PGError, match="world size > 1"):
        dd2.train()
    z = torch.zeros(8, device="cuda")
    args = [_lib.ptr(z)] * 4 + [None, 8, 1e-3, 0.9, 0.9, 1e-8, 1, 0.0, 1.0, None]
    assert L.d4pg_adam_polyak_ex(*args, -1.0, 0.0, None, None) == _lib.EINVAL
    assert L.d4pg_adam_polyak_ex(*args, 0.0, -2.0, None, None) == _lib.EINVAL
    assert L.d4pg_adam_polyak_ex(*args, 0.0, 1.0, None, None) == _lib.EINVAL          # clipping without a workspace
    assert L.d4pg_adam_polyak_ex(*args, 0.0, 0.0, None, None) == _lib.OK
