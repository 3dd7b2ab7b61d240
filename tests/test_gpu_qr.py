"""Quantile-regression critic (critic_dist_info {"type": "quantile", "n_quantiles": N, "kappa": kappa}).

The reference has no quantile code, so the yardstick is the derived oracle tests/qr_oracle.py: the quantile-Huber head in
float64 from the fp32 quantile rows, the pinned init / Adam / Polyak / PER of oracle/d4pg_oracle.py around it.  CPU tests
pin the oracle itself (gradcheck, the order-statistic minimiser) and the Python-side checks; GPU tests hold the kernel
(d4pg_qr_loss), the module (d4pg_critic_forward / d4pg_critic_backward without the softmax) and the learner step on
every plan to it.
"""
import os
import random
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import d4pg_oracle as O
from tests import bf16_oracle as BO
from tests import helpers as H
from tests import qr_oracle as QO
from tests import step_check as SC
from tests import tf32_oracle as TO

H_ = 256
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _info(N, kappa=None):
    d = {"type": "quantile", "n_quantiles": N}
    if kappa is not None:
        d["kappa"] = kappa
    return d


def _close(name, mine, ref, tol=1e-5):
    mine, ref = torch.as_tensor(mine).double().cpu(), torch.as_tensor(ref).double().cpu()
    assert mine.shape == ref.shape, (name, mine.shape, ref.shape)
    scale = max(1.0, float(ref.abs().max()))
    err = float((mine - ref).abs().max())
    assert err <= tol * scale, "%s: max abs err %.3e (scale %.3g)" % (name, err, scale)


def _rel(x, ref):
    x, ref = torch.as_tensor(x).double().cpu(), torch.as_tensor(ref).double().cpu()
    return float((x - ref).norm() / max(float(ref.norm()), 1e-30))


# ---- CPU ----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("kappa", [0.5, 1.0, 2.0])
def test_oracle_gradient_passes_gradcheck(kappa):
    N, B = 7, 4
    g = torch.Generator().manual_seed(0)
    tq = 2.0 * torch.randn(B, N, generator=g, dtype=torch.float64)
    q = (2.0 * torch.randn(B, N, generator=g, dtype=torch.float64)).requires_grad_(True)
    r, done = [-1.0, 0.5, 2.0, -0.25], [False, True, False, False]
    assert torch.autograd.gradcheck(lambda x: QO.loss_rows(tq, x, r, done, 0.99, kappa), (q,))
    assert torch.autograd.gradcheck(lambda x: QO.policy_rows(x), (q,))
    # the header's closed-form gradient is the autograd gradient
    QO.loss_rows(tq, q, r, done, 0.99, kappa).sum().backward()
    assert torch.allclose(q.grad, QO.grad_closed_form(tq, q, r, done, 0.99, kappa), rtol=0, atol=1e-14)


@pytest.mark.parametrize("N", [2, 5, 11])
def test_quantile_loss_minimiser_is_the_order_statistic(N):
    """Semantics pin: with kappa -> 0, theta_k minimises sum_j rho_tau_k(y_j - theta) at the (k+1)-th order statistic of
    the targets (tau_k N = k + 1/2 is never an integer, so the minimiser is unique)."""
    from scipy.optimize import minimize_scalar
    kappa = 1e-6
    y = torch.from_numpy(np.random.RandomState(N).randn(N) * 3.0).double()
    ys = np.sort(y.numpy())
    tau = QO.taus(N)
    for k in range(N):
        def f(th):
            u = y - th
            w = (tau[k] - (u < 0).double()).abs()
            return float((w * QO.huber(u, kappa)).sum() / kappa)
        res = minimize_scalar(f, bounds=(ys[0] - 1.0, ys[-1] + 1.0), method="bounded", options={"xatol": 1e-10})
        assert abs(res.x - ys[k]) <= 1e-5, (k, res.x, ys[k])


def test_cpu_quantile_critic_shapes_and_seeded_weights():
    import d4pg_b200 as d4pg
    N = 51
    torch.manual_seed(3)
    m = d4pg.models.critic(17, 6, _info(N), device="cpu")
    torch.manual_seed(3)
    c = d4pg.models.critic(17, 6, {"type": "categorical", "v_min": -1.0, "v_max": 1.0, "n_atoms": N}, device="cpu")
    sm, sc = m.state_dict(), c.state_dict()
    assert list(sm) == list(sc) == H.NAMES
    assert sm["fc3.weight"].shape == (N, 256) and sm["fc3.bias"].shape == (N,)
    for k in H.NAMES:
        assert torch.equal(sm[k], sc[k]), k
    assert m.n_atoms == N and m.kappa == 1.0


@pytest.mark.parametrize("info", [_info(1), _info(129), _info(51, 0.0), _info(51, -1.0), _info(51, float("nan")),
                                  _info(51, float("inf"))])
def test_quantile_critic_rejects_bad_n_and_kappa(info):
    import d4pg_b200 as d4pg
    with pytest.raises(d4pg._lib.D4PGError):
        d4pg.models.critic(17, 6, info, device="cpu")
    with pytest.raises(d4pg._lib.D4PGError):
        d4pg.DDPG(17, 6, memory_size=64, batch_size=8, critic_dist_info=info)


def test_quantile_ddpg_rejects_categorical_projection():
    import d4pg_b200 as d4pg
    dd = d4pg.DDPG(17, 6, memory_size=64, batch_size=8, critic_dist_info=_info(11, 2.0), priority="ce")
    assert dd.critic.state_dict()["fc3.weight"].shape == (11, 256)
    assert dd.n_atoms == 11 and dd.qr_kappa == 2.0
    assert dd.bin_centers is None and dd.v_min is None and dd.v_max is None
    with pytest.raises(d4pg._lib.D4PGError):
        dd.reproject2(np.zeros((2, 11), np.float32), [0.0, 0.0], [False, False])
    with pytest.raises(d4pg._lib.D4PGError):
        dd.reproj_categorical_dist(np.zeros((2, 11), np.float32), [0.0, 0.0], [False, False])
    with pytest.raises(NotImplementedError, match="quantile"):
        d4pg.DDPG(17, 6, memory_size=64, batch_size=8, critic_dist_info={"type": "iqn"})


# ---- GPU: the head kernel alone -----------------------------------------------------------------------------------
def _qr_loss(L, _lib, t_, q_, p_, r_, d_, B, N, disc, kappa, ce):
    outs = {k: torch.empty(B, device="cuda") for k in ("loss_rows", "td", "prio", "pi_rows")}
    dq, dpi = torch.empty(B, N, device="cuda"), torch.empty(B, N, device="cuda")
    _lib.check(L.d4pg_qr_loss(_lib.ptr(t_), _lib.ptr(q_), _lib.ptr(p_), _lib.ptr(r_), _lib.ptr(d_), B, N, disc, kappa,
                              1e-6, 1.0 / B, 1 if ce else 0, _lib.ptr(outs["loss_rows"]), _lib.ptr(outs["td"]),
                              _lib.ptr(outs["prio"]), _lib.ptr(dq), _lib.ptr(outs["pi_rows"]), _lib.ptr(dpi),
                              _lib.stream_ptr()), "d4pg_qr_loss")
    outs.update(dq=dq, dpi=dpi)
    torch.cuda.synchronize()
    return outs


@pytest.mark.gpu
@pytest.mark.parametrize("kappa", [0.5, 1.0, 2.0])
@pytest.mark.parametrize("N", [2, 51, 128])
@pytest.mark.parametrize("B", [1, 256, 4096])
def test_qr_loss_kernel_vs_oracle(B, N, kappa):
    """Raw quantiles at scale 1.5 and rewards in [-2, 1]: |u| falls on both sides of kappa.  Both priority modes, both
    discounts; every output within 1e-5 of the oracle (scaled by max(1, |ref|)), two launches bit-identical."""
    from d4pg_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(1000 * N + B + int(10 * kappa))
    tq, q, pq = (1.5 * torch.randn(B, N, generator=g) for _ in range(3))
    r = -3.0 * torch.rand(B, generator=g, dtype=torch.float64) + 1.0
    done = torch.rand(B, generator=g) < 0.05
    if B > 1:
        done[0] = True
    dev = lambda t: t.cuda().contiguous()
    t_, q_, p_, r_, d_ = dev(tq), dev(q), dev(pq), dev(r), dev(done.to(torch.uint8))
    u = (r.view(-1, 1, 1) + 0.99 * tq.double().unsqueeze(2)) - q.double().unsqueeze(1)
    if B > 1:                           # a single row of 2 quantiles has only 4 pairs
        assert bool((u.abs() > kappa).any()) and bool((u.abs() < kappa).any())
    for disc in (0.99, 0.99 ** 5):
        for ce in (False, True):
            outs = _qr_loss(L, _lib, t_, q_, p_, r_, d_, B, N, disc, kappa, ce)
            ref = QO.heads(tq, q, pq, r.numpy(), done.numpy(), disc, kappa, 1.0 / B, ce_priority=ce)
            for k in ("loss_rows", "td", "prio", "pi_rows", "dq", "dpi"):
                _close("%s disc=%g ce=%d" % (k, disc, ce), outs[k], ref[k])
            again = _qr_loss(L, _lib, t_, q_, p_, r_, d_, B, N, disc, kappa, ce)
            for k in outs:
                assert torch.equal(outs[k], again[k]), k


@pytest.mark.gpu
def test_qr_loss_kernel_rejects_bad_arguments():
    from d4pg_b200 import _lib
    L = _lib.lib()
    x = torch.zeros(4, 8, device="cuda")
    r = torch.zeros(4, dtype=torch.float64, device="cuda")
    d = torch.zeros(4, dtype=torch.uint8, device="cuda")
    for N, kappa in ((1, 1.0), (129, 1.0), (8, 0.0), (8, -1.0), (8, float("nan")), (8, float("inf"))):
        rc = L.d4pg_qr_loss(_lib.ptr(x), _lib.ptr(x), None, _lib.ptr(r), _lib.ptr(d), 4, N, 0.99, kappa, 1e-6, 0.25, 0,
                            None, None, None, None, None, None, _lib.stream_ptr())
        assert rc == _lib.EINVAL, (N, kappa, rc)


# ---- GPU: the module ------------------------------------------------------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1, 2, 3])
@pytest.mark.parametrize("N,B", [(51, 256), (101, 1024)])
def test_qr_module_forward_and_gradients(precision, N, B):
    """Forward: theta equals the logits of d4pg_critic_forward bit for bit (plain and differentiable forward).
    Gradients of a quantile-Huber loss written in torch on the module's output (kappa 1): precisions 0 / 1 within 1e-5
    of float64 autograd (device ReLU masks), precision 3 within relative L2 1e-3 of the bf16 linear."""
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib
    S, A = 17, 6
    torch.manual_seed(60 + N)
    cri = d4pg.models.critic(S, A, _info(N), device="cuda")
    with torch.no_grad():
        cri.fc3.weight.normal_(0.0, 0.1)
    cri.precision = precision
    g = torch.Generator().manual_seed(61)
    s0 = torch.randn(B, S, generator=g); a0 = torch.rand(B, A, generator=g) * 2 - 1
    sd, ad = s0.cuda(), a0.cuda()
    theta = cri(sd, ad)
    torch.cuda.synchronize()
    ws = cri._ws[:3 * B * H_].view(3, B, H_).cpu().double()
    probs, logits = torch.empty(B, N, device="cuda"), torch.empty(B, N, device="cuda")
    wsp = torch.empty(3 * B * H_, device="cuda")
    _lib.check(_lib.lib().d4pg_critic_forward(_lib.ptr(cri.flat_params()), S, A, N, _lib.ptr(sd), _lib.ptr(ad), B,
                                              _lib.ptr(probs), _lib.ptr(logits), _lib.ptr(wsp), precision,
                                              _lib.stream_ptr()), "d4pg_critic_forward")
    torch.cuda.synchronize()
    assert theta.shape == (B, N) and torch.equal(theta, logits)
    if precision == 2:
        return                          # TF32 gradients are held to their oracle by test_gpu_tf32 / test_gpu_autograd

    cri.differentiable = True
    s = s0.cuda().requires_grad_(True); a = a0.cuda().requires_grad_(True)
    for p in cri.parameters():
        p.grad = None
    out = cri(s, a)
    assert out.grad_fn is not None and torch.equal(out.detach(), theta)
    y = (1.5 * torch.randn(B, N, generator=g)).double()
    (QO.pair_loss(y.cuda(), out, 1.0).sum() / B).backward()
    dt = torch.float64 if precision in (0, 1) else torch.float32
    lin = BO.linear("bf16") if precision == 3 else F.linear
    W = {k: v.detach().cpu() for k, v in cri.state_dict().items()}
    Wl = {k: v.to(dt).requires_grad_(True) for k, v in W.items()}
    sl, al = s0.to(dt).requires_grad_(True), a0.to(dt).requires_grad_(True)
    m1, m2, m3 = (ws[i] > 0 for i in range(3))
    h = lin(sl, Wl["fc1.weight"], Wl["fc1.bias"]) * m1
    h = lin(torch.cat([h, al], 1), Wl["fc2.weight"], Wl["fc2.bias"]) * m2
    h = lin(h, Wl["fc2_2.weight"], Wl["fc2_2.bias"]) * m3
    o = lin(h, Wl["fc3.weight"], Wl["fc3.bias"])
    (QO.pair_loss(y, o, 1.0).sum() / B).backward()
    views = cri.named_grad_views()
    checks = [(k, views[k].cpu(), Wl[k].grad) for k in H.NAMES] + [("d state", s.grad.cpu(), sl.grad),
                                                                   ("d action", a.grad.cpu(), al.grad)]
    for name, mine, ref in checks:
        if precision in (0, 1):
            err = float((mine.double() - ref.double()).abs().max())
            assert err <= 1e-5 * max(1.0, float(ref.abs().max())), (name, err)
        else:
            assert _rel(mine, ref) <= 1e-3, (name, _rel(mine, ref))


# ---- GPU: the learner -------------------------------------------------------------------------------------------------
def _qr_ddpg(d4pg, N, B, precision, chain="cluster", n=None, seed=12, kappa=1.0, **kw):
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    n = n or max(2048, 2 * B)
    dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=_info(N, kappa), precision=precision,
                   chain=chain, **kw)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(seed + 1)
    data = (rng.randn(n, 17).astype(np.float32), rng.uniform(-1, 1, (n, 6)).astype(np.float32),
            (-3 * rng.rand(n)).astype(np.float32).astype(np.float64), rng.randn(n, 17).astype(np.float32), rng.rand(n) < 0.05)
    dd.replayBuffer.add_batch(*data)
    with torch.no_grad():            # targets differ from the online networks; quantiles at a visible scale
        for net in (dd.critic, dd.critic_target):
            net.fc3.weight.normal_(0.0, 0.05)
        dd.actor_target.flat_params().mul_(1.01)
        dd.critic_target.flat_params().mul_(0.99)
    return dd, data


def _snapshot(dd):
    return {k: {n_: v.detach().cpu().clone() for n_, v in net.state_dict().items()}
            for k, net in (("a", dd.actor), ("at", dd.actor_target), ("c", dd.critic), ("ct", dd.critic_target))}


PLANS = {"wgmma": ("tf32x3", 256, "cluster"), "mma_ffma": ("fp32", 256, "cluster"), "levels_b1024": ("fp32", 1024, "cluster"),
         "levels": ("tf32x3", 256, "levels")}
STEP_PLANS = {"wgmma": ("tc_chain", "tf32x3"), "mma_ffma": ("chain", "fp32"), "levels_b1024": ("levels", "fp32"),
              "levels": ("levels", "tf32x3")}       # (step plan, precision) of tests/step_check.py


@pytest.mark.gpu
@pytest.mark.parametrize("variant", ["plain", "nstep", "is_weights", "post_update", "ce_priority"])
@pytest.mark.parametrize("plan", list(PLANS))
@pytest.mark.parametrize("N", [51, 101])
def test_qr_learner_step_vs_oracle(N, plan, variant):
    """One eager DDPG.train() against QrLearnerOracle.train_step on the sampled batch: quantile planes, loss rows, td,
    priorities, both losses, quantile gradients and every parameter gradient."""
    import d4pg_b200 as d4pg
    precision, B, chain = PLANS[plan]
    if variant == "post_update" and plan != "wgmma":
        pytest.skip("the post-update critic runs on the tensor-core chain plan only")
    kw = dict(use_graph=False, sampling="device", philox_seed=5, prefetch=False)
    if variant == "nstep":
        kw.update(projection="nstep", n_steps=5)
    if variant == "is_weights":
        kw.update(importance_weighted=True)
    if variant == "post_update":
        kw.update(actor_critic="post_update")
    if variant == "ce_priority":
        kw.update(priority="ce")
    dd, (S, A, R, S2, D) = _qr_ddpg(d4pg, N, B, precision, chain=chain, **kw)
    if variant == "is_weights":                       # a non-uniform tree so the IS weights are not all 1
        pr = (np.random.RandomState(3).rand(len(S)).astype(np.float32) + np.float32(1e-3))
        dd.replayBuffer.update_priorities(np.arange(len(S)), pr)
    W = _snapshot(dd)
    W_step = SC.snapshot(dd)                          # the oracle's Adam and Polyak update W in place
    lo = QO.QrLearnerOracle(17, 6, N, n_steps=kw.get("n_steps", 1), projection="nstep" if variant == "nstep" else "live",
                            actor_w=W["a"], critic_w=W["c"])
    lo.actor_target, lo.critic_target = W["at"], W["ct"]
    dd.train()
    info = dd.last_batch_info()
    idx = info["idx"].cpu().numpy()
    isw = info["weights"].cpu().numpy() if variant == "is_weights" else None
    if isw is not None:
        assert isw.min() < 0.999
    out = lo.train_step(S[idx], A[idx], R[idx], S2[idx], D[idx], is_weights=isw,
                        post_update_critic=variant == "post_update", ce_priority=variant == "ce_priority")
    t = lambda name, w=None: dd.debug_tensor(name, (B, w) if w else None).cpu()
    _close("target_q", t("target_logits", N), out["target_q"])
    _close("q", t("q_logits", N), out["q"])
    _close("pi_q", t("pi_logits", N), out["pi_q"])
    _close("loss_rows", t("loss_rows"), out["loss_rows"])
    _close("pi_rows", t("pi_rows"), out["pi_rows"])
    _close("td", info["td"], out["td"])
    _close("prio", info["prio"], out["prio"])
    lc, la = dd.last_losses()
    _close("loss_critic", torch.tensor(lc), torch.tensor(out["loss_critic"]))
    _close("loss_actor", torch.tensor(la), torch.tensor(out["loss_actor"]))
    gs = max(float(out["dq"].abs().max()), float(out["dpi"].abs().max()))
    for name, ref in (("dlogits_q", out["dq"]), ("dlogits_pi", out["dpi"])):
        err = float((t(name, N).double() - ref.double()).abs().max())
        assert err <= 1e-5 * gs, (name, err, gs)
    # every layer and parameter gradient from the device's own quantile gradients (held to the oracle above)
    SC.check_step(dd, W_step, *STEP_PLANS[plan], post_update=variant == "post_update", label="qr %s/%s N=%d" % (plan, variant, N))


@pytest.mark.gpu
def test_config5_bf16_and_tf32_quantile_vs_oracle():
    """Config-5 shapes (batch 4096, n-step 5) with N=101 at bf16: gradients within relative L2 1e-3 of the oracle on the
    bf16 linear.  At tf32 (plan 0 truncates every operand to TF32): within relative L2 5e-3 of the oracle on the rz TF32
    linear of tests/tf32_oracle.py."""
    import d4pg_b200 as d4pg
    B, N = 4096, 101
    for precision, lin, bound in (("bf16", BO.linear("bf16"), 1e-3), ("tf32", TO.linear("rz"), 5e-3)):
        dd, (S, A, R, S2, D) = _qr_ddpg(d4pg, N, B, precision, n=16384, seed=21, use_graph=False, sampling="device",
                                        prefetch=False, projection="nstep", n_steps=5)
        W = _snapshot(dd)
        lo = QO.QrLearnerOracle(17, 6, N, n_steps=5, projection="nstep", actor_w=W["a"], critic_w=W["c"], linear=lin)
        lo.actor_target, lo.critic_target = W["at"], W["ct"]
        dd.train()
        idx = dd.last_batch_info()["idx"].cpu().numpy()
        out = lo.train_step(S[idx], A[idx], R[idx], S2[idx], D[idx])
        worst = 0.0
        for net, grads in ((dd.critic, out["grads_critic"]), (dd.actor, out["grads_actor"])):
            for k in H.NAMES:
                worst = max(worst, _rel(net.named_grad_views()[k].cpu(), grads[k]))
        assert worst <= bound, (precision, worst)
        print("config 5 quantile %s: worst gradient rel L2 %.2e" % (precision, worst))
        del dd


@pytest.mark.gpu
def test_qr_graph_steps_with_reference_sampling_and_adds():
    """Three CUDA-graph steps (host pipeline) with reference sampling and adds between them: sampled indices bit-exact
    against the PER oracle, losses and priorities within 1e-5 of the quantile oracle."""
    import d4pg_b200 as d4pg
    N, B, n = 51, 64, 1024
    torch.manual_seed(7); random.seed(7)
    dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=_info(N), precision="tf32x3")
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
    rng = np.random.RandomState(8)
    mk = lambda m: (rng.randn(m, 17).astype(np.float32), rng.uniform(-1, 1, (m, 6)).astype(np.float32),
                    (-3 * rng.rand(m)).astype(np.float32).astype(np.float64), rng.randn(m, 17).astype(np.float32),
                    rng.rand(m) < 0.05)
    ob = O.PrioritizedReplayOracle(n, 0.6, 17, 6)
    batch0 = mk(512)
    dd.replayBuffer.add_batch(*batch0)
    ob.add_batch(*batch0)
    lo = QO.QrLearnerOracle(17, 6, N, actor_w={k: v.cpu().clone() for k, v in dd.actor.state_dict().items()},
                            critic_w={k: v.cpu().clone() for k, v in dd.critic.state_dict().items()})
    sched = O.LinearScheduleOracle(100000, 1.0, 0.4)
    for step in range(3):
        random.seed(90 + step)
        st = random.getstate(); us = [random.random() for _ in range(B)]; random.setstate(st)
        dd.train()
        batch = ob.sample(B, sched.value(), us)
        assert np.array_equal(dd.last_batch_info()["idx"].cpu().numpy(), batch[6])
        out = lo.train_step(*batch[:5])
        lc, la = dd.last_losses()
        assert abs(lc - out["loss_critic"]) <= 1e-5 * max(1.0, abs(out["loss_critic"]))
        prio = dd.last_batch_info()["prio"].cpu().numpy()
        assert np.abs(prio - out["prio"]).max() <= 1e-5 * max(1.0, float(np.abs(out["prio"]).max()))
        ob.update_priorities(batch[6], prio)          # follow the device's priorities: indices stay comparable
        add = mk(16)
        dd.replayBuffer.add_batch(*add)
        ob.add_batch(*add)


@pytest.mark.gpu
def test_qr_train_n_equals_single_steps():
    """One cold step, then train_n(8) with device sampling (one 8-step graph, prefetch pipeline) is bit-identical to 9
    single steps: the quantile head kernel advances the sampler clock."""
    import d4pg_b200 as d4pg
    res = []
    for multi in (True, False):
        dd, _ = _qr_ddpg(d4pg, 51, 256, "tf32x3", sampling="device", philox_seed=9)
        dd.train()                      # the prefetched batch makes the next step warm: train_n(8) replays the graph
        if multi:
            dd.train_n(8)
        else:
            for _ in range(8):
                dd.train()
        torch.cuda.synchronize()
        res.append((dd.critic.flat_params().cpu().clone(), dd.actor.flat_params().cpu().clone(),
                    dd.last_batch_info()["idx"].cpu().clone(), dd.last_batch_info()["prio"].cpu().clone()))
        del dd
    for x, y in zip(*res):
        assert torch.equal(x, y)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_qr_data_parallel_matches_single_big_batch_oracle(precision):
    """Two ranks with the quantile critic (tests/qr_dp_worker.py): replicas stay identical after every step, and the
    summed gradients equal ONE QrLearnerOracle on the concatenated batches within 1e-5 -- the check of the head's
    1/(B_local * world) gradient fold."""
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    env = dict(os.environ, D4PG_PRECISION=precision)
    cmd = [sys.executable, "-m", "torch.distributed.run", "--nnodes=1", "--nproc-per-node=2", "--master-addr", "127.0.0.1",
           "--master-port", "29611", os.path.join(ROOT, "tests", "qr_dp_worker.py")]
    r = subprocess.run(cmd, env=env, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True, timeout=600)
    assert r.returncode == 0 and "QR_DP_OK" in r.stdout, r.stdout[-3000:]
