"""The learner step with the mixture-of-Gaussians and the quantile critics against their derived oracles.

Both heads run the same checks: one eager step on every plan and semantics variant, config-5 shapes at bf16 and tf32,
CUDA-graph steps with reference sampling and adds, and train_n against single steps.  The oracles are
tests/mog_oracle.py's MogLearnerOracle and tests/qr_oracle.py's QrLearnerOracle: oracle/d4pg_oracle.py's LearnerOracle
with the head replaced.  The head kernels, modules and data-parallel runs are tested in test_gpu_mog.py and
test_gpu_qr.py.
"""
import random

import numpy as np
import pytest
import torch

from oracle import d4pg_oracle as O
from tests import bf16_oracle as BO
from tests import helpers as H
from tests import mog_oracle as MO
from tests import qr_oracle as QO
from tests import step_check as SC
from tests import tf32_oracle as TO

# head -> (critic_dist_info for a size, the oracle, the oracle's names for target, q, pi, dq and dpi)
HEADS = {"mixture": (lambda K: {"type": "mixture_of_gaussian", "n_components": K}, MO.MogLearnerOracle,
                     ("target_raw", "q_raw", "pi_raw", "dq_raw", "dpi_raw")),
         "quantile": (lambda N: {"type": "quantile", "n_quantiles": N, "kappa": 1.0}, QO.QrLearnerOracle,
                      ("target_q", "q", "pi_q", "dq", "dpi"))}


def _close(name, mine, ref, tol=1e-5):
    mine, ref = torch.as_tensor(mine).double().cpu(), torch.as_tensor(ref).double().cpu()
    assert mine.shape == ref.shape, (name, mine.shape, ref.shape)
    scale = max(1.0, float(ref.abs().max()))
    err = float((mine - ref).abs().max())
    assert err <= tol * scale, "%s: max abs err %.3e (scale %.3g)" % (name, err, scale)


def _rel(x, ref):
    x, ref = torch.as_tensor(x).double().cpu(), torch.as_tensor(ref).double().cpu()
    return float((x - ref).norm() / max(float(ref.norm()), 1e-30))


def _ddpg(info, B, precision, chain="cluster", n=None, seed=12, **kw):
    import d4pg_b200 as d4pg
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    n = n or max(2048, 2 * B)
    dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=info, precision=precision, chain=chain, **kw)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(seed + 1)
    data = (rng.randn(n, 17).astype(np.float32), rng.uniform(-1, 1, (n, 6)).astype(np.float32),
            (-3 * rng.rand(n)).astype(np.float32).astype(np.float64), rng.randn(n, 17).astype(np.float32), rng.rand(n) < 0.05)
    dd.replayBuffer.add_batch(*data)
    with torch.no_grad():            # targets differ from the online networks; a critic head at a visible scale
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
VARIANTS = ["plain", "nstep", "is_weights", "post_update"]
STEP_CASES = ([("mixture", K, plan, v) for K in (5, 11) for plan in PLANS for v in VARIANTS]
              + [("quantile", N, plan, v) for N in (51, 101) for plan in PLANS for v in VARIANTS + ["ce_priority"]])


@pytest.mark.gpu
@pytest.mark.parametrize("head,size,plan,variant", STEP_CASES)
def test_learner_step_vs_oracle(head, size, plan, variant):
    """One eager DDPG.train() against the head's oracle train_step on the sampled batch: the critic's raw fc3 rows, loss
    rows, td, priorities, both losses, the raw-row gradients and every parameter gradient."""
    dist, oracle, names = HEADS[head]
    precision, B, chain = PLANS[plan]
    if variant == "post_update" and plan != "wgmma":
        pytest.skip("the post-update critic runs on the tensor-core chain plan only")
    if head == "mixture" and variant != "plain" and plan == "levels":
        pytest.skip("variants are covered on the three automatic plans")
    kw = dict(use_graph=False, sampling="device", philox_seed=5, prefetch=False)
    if variant == "nstep":
        kw.update(projection="nstep", n_steps=5)
    if variant == "is_weights":
        kw.update(importance_weighted=True)
    if variant == "post_update":
        kw.update(actor_critic="post_update")
    if variant == "ce_priority":
        kw.update(priority="ce")
    dd, (S, A, R, S2, D) = _ddpg(dist(size), B, precision, chain=chain, **kw)
    if variant == "is_weights":                       # a non-uniform tree so the IS weights are not all 1
        pr = (np.random.RandomState(3).rand(len(S)).astype(np.float32) + np.float32(1e-3))
        dd.replayBuffer.update_priorities(np.arange(len(S)), pr)
    W = _snapshot(dd)
    W_step = SC.snapshot(dd)                          # the oracle's Adam and Polyak update W in place
    lo = oracle(17, 6, size, n_steps=kw.get("n_steps", 1), projection="nstep" if variant == "nstep" else "live",
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
    target, q, pi, dq, dpi = (torch.as_tensor(out[k]) for k in names)
    N = q.shape[1]
    t = lambda name, w=None: dd.debug_tensor(name, (B, w) if w else None).cpu()
    _close(names[0], t("target_logits", N), target)
    _close(names[1], t("q_logits", N), q)
    _close(names[2], t("pi_logits", N), pi)
    _close("loss_rows", t("loss_rows"), out["loss_rows"])
    _close("pi_rows", t("pi_rows"), out["pi_rows"])
    _close("td", info["td"], out["td"])
    _close("prio", info["prio"], out["prio"])
    lc, la = dd.last_losses()
    _close("loss_critic", torch.tensor(lc), torch.tensor(out["loss_critic"]))
    _close("loss_actor", torch.tensor(la), torch.tensor(out["loss_actor"]))
    gs = max(float(dq.abs().max()), float(dpi.abs().max()))
    for name, ref in (("dlogits_q", dq), ("dlogits_pi", dpi)):
        err = float((t(name, N).double() - ref.double()).abs().max())
        assert err <= 1e-5 * gs, (name, err, gs)
    # every layer and parameter gradient from the device's own raw-row gradients (held to the oracle above)
    SC.check_step(dd, W_step, *STEP_PLANS[plan], post_update=variant == "post_update",
                  label="%s %s/%s %d" % (head, plan, variant, size))


def _config5_bf16_and_tf32(head, size):
    """Config-5 shapes (batch 4096, n-step 5) at bf16: gradients within relative L2 1e-3 of the oracle on the bf16
    linear.  At tf32 (plan 0 truncates every operand to TF32): within relative L2 5e-3 of the oracle on the rz TF32
    linear of tests/tf32_oracle.py."""
    dist, oracle, _ = HEADS[head]
    B = 4096
    for precision, lin, bound in (("bf16", BO.linear("bf16"), 1e-3), ("tf32", TO.linear("rz"), 5e-3)):
        dd, (S, A, R, S2, D) = _ddpg(dist(size), B, precision, n=16384, seed=21, use_graph=False, sampling="device",
                                     prefetch=False, projection="nstep", n_steps=5)
        W = _snapshot(dd)
        lo = oracle(17, 6, size, n_steps=5, projection="nstep", actor_w=W["a"], critic_w=W["c"], linear=lin)
        lo.actor_target, lo.critic_target = W["at"], W["ct"]
        dd.train()
        idx = dd.last_batch_info()["idx"].cpu().numpy()
        out = lo.train_step(S[idx], A[idx], R[idx], S2[idx], D[idx])
        worst = 0.0
        for net, grads in ((dd.critic, out["grads_critic"]), (dd.actor, out["grads_actor"])):
            for k in H.NAMES:
                worst = max(worst, _rel(net.named_grad_views()[k].cpu(), grads[k]))
        assert worst <= bound, (precision, worst)
        print("config 5 %s %s: worst gradient rel L2 %.2e" % (head, precision, worst))
        del dd


def _graph_steps_with_reference_sampling_and_adds(head, size):
    """Three CUDA-graph steps (host pipeline) with reference sampling and adds between them: sampled indices bit-exact
    against the PER oracle, losses and priorities within 1e-5 of the head's oracle."""
    import d4pg_b200 as d4pg
    dist, oracle, _ = HEADS[head]
    B, n = 64, 1024
    torch.manual_seed(7); random.seed(7)
    dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=dist(size), precision="tf32x3")
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
    rng = np.random.RandomState(8)
    mk = lambda m: (rng.randn(m, 17).astype(np.float32), rng.uniform(-1, 1, (m, 6)).astype(np.float32),
                    (-3 * rng.rand(m)).astype(np.float32).astype(np.float64), rng.randn(m, 17).astype(np.float32),
                    rng.rand(m) < 0.05)
    ob = O.PrioritizedReplayOracle(n, 0.6, 17, 6)
    batch0 = mk(512)
    dd.replayBuffer.add_batch(*batch0)
    ob.add_batch(*batch0)
    lo = oracle(17, 6, size, actor_w={k: v.cpu().clone() for k, v in dd.actor.state_dict().items()},
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


def _train_n_equals_single_steps(head, size):
    """One cold step, then train_n(8) with device sampling (one 8-step graph, prefetch pipeline) is bit-identical to 9
    single steps: the head kernel advances the sampler clock."""
    res = []
    for multi in (True, False):
        dd, _ = _ddpg(HEADS[head][0](size), 256, "tf32x3", sampling="device", philox_seed=9)
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
def test_config5_bf16_and_tf32_mixture_vs_oracle():
    _config5_bf16_and_tf32("mixture", 5)


@pytest.mark.gpu
def test_config5_bf16_and_tf32_quantile_vs_oracle():
    _config5_bf16_and_tf32("quantile", 101)


@pytest.mark.gpu
def test_mog_graph_steps_with_reference_sampling_and_adds():
    _graph_steps_with_reference_sampling_and_adds("mixture", 5)


@pytest.mark.gpu
def test_qr_graph_steps_with_reference_sampling_and_adds():
    _graph_steps_with_reference_sampling_and_adds("quantile", 51)


@pytest.mark.gpu
def test_mog_train_n_equals_single_steps():
    _train_n_equals_single_steps("mixture", 5)


@pytest.mark.gpu
def test_qr_train_n_equals_single_steps():
    _train_n_equals_single_steps("quantile", 51)
