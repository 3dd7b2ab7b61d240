"""precision="bf16" (libd4pg precision 3): one bf16 wgmma pass per MLP GEMM (csrc/gemm_bf16.cu).

Every GEMM operand is rounded fp32 -> bf16 (nearest even) when the kernel stages it -- X and W forward, dZ and W for
dX, dZ and X for dW -- and products accumulate in fp32; activations, deltas, bias terms, bias gradients, the loss heads
and Adam stay fp32.  So the yardstick is a float64 restatement on the same ROUNDED operands (tests/bf16_oracle.py, a
derived oracle: the reference has no bf16 mode), not the fp32 oracle: against that, bf16 differs by ~1e-2 relative.
Config 5 (BASELINE.json configs[4]: n-step 5, 101 atoms, batch 4096, bf16 MLPs) runs here as specified.
"""
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import d4pg_oracle as O
from tests import bf16_oracle as BO
from tests import helpers as H
from tests import step_check as SC

H_ = 256
rb = BO.rb


def _close(name, mine, ref, tol=1e-5):
    mine, ref = mine.double().cpu(), ref.double().cpu()
    assert mine.shape == ref.shape, (name, mine.shape, ref.shape)
    scale = max(1.0, float(ref.abs().max()))
    err = float((mine - ref).abs().max())
    assert err <= tol * scale, "%s: max abs err %.3e (scale %.3g)" % (name, err, scale)
    return err


# ---- CPU: the derived oracle itself ---------------------------------------------------------------------------------
def test_bf16_oracle_linear_rounds_operands_and_keeps_fp32_bias_grad():
    torch.manual_seed(3)
    x = torch.randn(37, 19, requires_grad=True); w = torch.randn(11, 19, requires_grad=True); b = torch.randn(11, requires_grad=True)
    y = BO.linear("bf16")(x, w, b)
    assert torch.equal(y, (rb(x.detach()) @ rb(w.detach()).T).float() + b.detach())
    g = torch.randn(37, 11)
    y.backward(g)
    assert torch.equal(x.grad, (rb(g) @ rb(w.detach())).float())
    assert torch.equal(w.grad, (rb(g).T @ rb(x.detach())).float())
    assert torch.equal(b.grad, g.sum(0))
    assert (y - torch.nn.functional.linear(x, w, b)).abs().max() > 1e-3     # the rounding is visible


# ---- GPU --------------------------------------------------------------------------------------------------------------
def _lin(x, w, b=None, bf16=True):
    """One layer in float64 on (optionally) bf16-rounded operands; the bias is added to the fp64 sum."""
    y = (rb(x) @ rb(w).T) if bf16 else (x.double() @ w.double().T)
    return y if b is None else y + b.double()


def _ddpg(d4pg, B, S, A, N, n=None, graph=False, chain="cluster", projection="reference", n_steps=1, seed=12, **kw):
    info = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": N}
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    n = n or max(2048, 2 * B)
    dd = d4pg.DDPG(S, A, memory_size=n, batch_size=B, critic_dist_info=info, precision="bf16", use_graph=graph,
                   sampling="device", philox_seed=3, prefetch=False, chain=chain, projection=projection, n_steps=n_steps, **kw)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(1)
    dd.replayBuffer.add_batch(rng.randn(n, S).astype(np.float32), rng.uniform(-1, 1, (n, A)).astype(np.float32),
                              (-3 * rng.rand(n)), rng.randn(n, S).astype(np.float32), rng.rand(n) < 0.05)
    return dd


@pytest.mark.gpu
@pytest.mark.parametrize("B,S,A,N,graph,chain,projection", [
    (4096, 17, 6, 101, False, "cluster", "nstep"),      # config 5 shapes: split-K dW
    (1024, 376, 17, 51, False, "cluster", "reference"),  # config 3 shapes: split-K dW, ragged fc2 concat tail
    (200, 3, 1, 101, True, "cluster", "reference"),      # ragged M (200 rows), CUDA graph
    (256, 17, 6, 51, False, "cluster", "reference")])    # chain="cluster" at 256 rows still runs the level plan
def test_bf16_every_intermediate_vs_rounded_restatement(B, S, A, N, graph, chain, projection):
    """Every activation, logit, delta and parameter gradient of one eager DDPG.train() at precision="bf16" against the
    float64 restatement on bf16-rounded operands.  Each layer is fed the device's own inputs and ReLU masks (the same
    fp32 value rounds to the same bf16 on both sides); bound 1e-5 x max(1, |ref|max), for the parameter gradients (~1e-6)
    the componentwise bound of tests/step_check.py."""
    import d4pg_b200 as d4pg
    dd = _ddpg(d4pg, B, S, A, N, graph=graph, chain=chain, projection=projection, n_steps=5 if projection == "nstep" else 1)
    with torch.no_grad():
        dd.actor_target.flat_params().mul_(1.01)
        dd.critic_target.flat_params().mul_(0.99)
    W = {k: {n_: v.detach().cpu() for n_, v in net.state_dict().items()}
         for k, net in (("a", dd.actor), ("at", dd.actor_target), ("c", dd.critic), ("ct", dd.critic_target))}
    dd.train()
    torch.cuda.synchronize()
    if chain == "cluster" and B <= 512:      # bf16 has no chain kernels: the same launches as chain="levels"
        ref_dd = _ddpg(d4pg, B, S, A, N, graph=graph, chain="levels")
        ref_dd.train()
        torch.cuda.synchronize()
        assert dd.kernels_per_step() == ref_dd.kernels_per_step()
        del ref_dd
    t = lambda name, w=None: dd.debug_tensor(name, (B, w) if w else None).cpu()
    s, a, s2 = t("s", S), t("a", A), t("s2", S)
    relu = torch.relu
    Wa, Wat, Wc, Wct = W["a"], W["at"], W["c"], W["ct"]
    L = lambda x, w, l: _lin(x, w[l + ".weight"], w[l + ".bias"])

    # forward: every layer from the device's own input to it
    ah1, ah2, ah3, aout = t("h1_a", H_), t("h2_a", H_), t("h3_a", H_), t("actor_out", A)
    _close("h1_a", ah1, relu(L(s, Wa, "fc1")))
    _close("h2_a", ah2, L(ah1, Wa, "fc2"))
    _close("h3_a", ah3, relu(L(ah2, Wa, "fc2_2")))
    _close("actor_out", aout, torch.tanh(L(ah3, Wa, "fc3")))
    ch1, ch2, ch3 = t("h1_c", H_), t("h2_c", H_), t("h3_c", H_)
    _close("h1_c", ch1, relu(L(s, Wc, "fc1")))
    _close("h2_c", ch2, relu(L(torch.cat([ch1, a], 1), Wc, "fc2")))
    _close("h3_c", ch3, relu(L(ch2, Wc, "fc2_2")))
    _close("q_logits", t("q_logits", N), L(ch3, Wc, "fc3"))
    ph2, ph3 = t("h2_p", H_), t("h3_p", H_)
    _close("h2_p", ph2, relu(L(torch.cat([ch1, aout], 1), Wc, "fc2")))
    _close("h3_p", ph3, relu(L(ph2, Wc, "fc2_2")))
    _close("pi_logits", t("pi_logits", N), L(ph3, Wc, "fc3"))
    th1, th2, th3, at_out = t("h1_at", H_), t("h2_at", H_), t("h3_at", H_), t("actor_target_out", A)
    _close("h1_at", th1, relu(L(s2, Wat, "fc1")))
    _close("h2_at", th2, L(th1, Wat, "fc2"))
    _close("h3_at", th3, relu(L(th2, Wat, "fc2_2")))
    _close("actor_target_out", at_out, torch.tanh(L(th3, Wat, "fc3")))
    ct1, ct2, ct3 = t("h1_ct", H_), t("h2_ct", H_), t("h3_ct", H_)
    _close("h1_ct", ct1, relu(L(s2, Wct, "fc1")))
    _close("h2_ct", ct2, relu(L(torch.cat([ct1, at_out], 1), Wct, "fc2")))
    _close("h3_ct", ct3, relu(L(ct2, Wct, "fc2_2")))
    _close("target_logits", t("target_logits", N), L(ct3, Wct, "fc3"))

    # backward: deltas from the device's own upstream delta and masks
    dq, dpi = t("dlogits_q", N), t("dlogits_pi", N)
    dm = {k: v > 0 for k, v in (("h1_c", ch1), ("h2_c", ch2), ("h3_c", ch3), ("h1_a", ah1), ("h3_a", ah3), ("h2_p", ph2), ("h3_p", ph3))}
    dev = {k: t(k, A if k == "a_dz3" else H_) for k in ("c_dz22", "c_dz2", "c_dz1", "p_dz22", "p_dz2", "a_dz3", "a_dz22", "a_dh2", "a_dz1")}
    dx = lambda g, w: rb(g) @ rb(w)
    gs = max(float(dq.abs().max()), float(dpi.abs().max()), 1e-30)      # deltas are O(1/B): relative to the input scale
    refs = {"c_dz22": dx(dq, Wc["fc3.weight"]) * dm["h3_c"],
            "c_dz2": dx(dev["c_dz22"], Wc["fc2_2.weight"]) * dm["h2_c"],
            "c_dz1": dx(dev["c_dz2"], Wc["fc2.weight"][:, :H_]) * dm["h1_c"],
            "p_dz22": dx(dpi, Wc["fc3.weight"]) * dm["h3_p"],
            "p_dz2": dx(dev["p_dz22"], Wc["fc2_2.weight"]) * dm["h2_p"],
            "a_dz3": dx(dev["p_dz2"], Wc["fc2.weight"][:, H_:]) * (1 - aout.double() ** 2),
            "a_dz22": dx(dev["a_dz3"], Wa["fc3.weight"]) * dm["h3_a"],
            "a_dh2": dx(dev["a_dz22"], Wa["fc2_2.weight"]),
            "a_dz1": dx(dev["a_dh2"], Wa["fc2.weight"]) * dm["h1_a"]}
    for name, ref in refs.items():
        _close(name, dev[name], ref)
        err = float((dev[name].double() - ref).abs().max())
        assert err <= 1e-5 * max(gs, float(ref.abs().max())), "%s: %.3e vs scale %.3e" % (name, err, gs)

    # dW from the device's deltas and activations on bf16-rounded operands, bias gradients as sums of the unrounded
    # fp32 deltas: against the componentwise bound of tests/step_check.py, with its power check
    sc = SC.StepCheck(dd, W, "levels", "bf16", label="bf16(%d,%d,%d,%d)" % (B, S, A, N))
    sc.grads({"c": {"fc3": (dq, ch3), "fc2_2": (dev["c_dz22"], ch2), "fc2": (dev["c_dz2"], torch.cat([ch1, a], 1)),
                    "fc1": (dev["c_dz1"], s)},
              "a": {"fc3": (dev["a_dz3"], ah3), "fc2_2": (dev["a_dz22"], ah2), "fc2": (dev["a_dh2"], ah1), "fc1": (dev["a_dz1"], s)}})
    sc.rep.finish()


def _rel(x, ref):
    x, ref = x.double(), ref.double()
    return float((x - ref).norm() / max(float(ref.norm()), 1e-30))


@pytest.mark.gpu
def test_config5_bf16_vs_derived_oracle():
    """Config 5 as specified (BASELINE.json configs[4]): n-step 5 projection, 101 atoms, batch 4096, bf16 Actor/Critic
    MLPs.  One DDPG.train() against the derived bf16 oracle on the same batch: m within 1e-5, losses within
    1e-5 x max(1, |loss|), every gradient within relative L2 1e-3; and the worst tensor at least 10x farther from the
    fp32 oracle than from the bf16 one.  One step only: Adam turns last-bit gradient differences on near-zero elements
    into lr-sized steps, so later steps drift apart for reasons unrelated to the GEMMs."""
    import d4pg_b200 as d4pg
    info = {"type": "categorical", "v_min": -150.0, "v_max": 150.0, "n_atoms": 101}
    torch.manual_seed(21); random.seed(21)
    B, n, S, A = 4096, 16384, 17, 6
    dd = d4pg.DDPG(S, A, memory_size=n, batch_size=B, critic_dist_info=info, n_steps=5, projection="nstep", precision="bf16")
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
    rng = np.random.RandomState(22)
    Sx = rng.randn(n, S).astype(np.float32); Ax = rng.uniform(-1, 1, (n, A)).astype(np.float32)
    R = (40 * (rng.rand(n) - 0.5)).astype(np.float32).astype(np.float64); S2 = rng.randn(n, S).astype(np.float32)
    D = rng.rand(n) < 0.05
    dd.replayBuffer.add_batch(Sx, Ax, R, S2, D)
    oracle = lambda linear: O.LearnerOracle(S, A, info, n_steps=5, projection="nstep", linear=linear,
                                            actor_w={k: v.cpu().clone() for k, v in dd.actor.state_dict().items()},
                                            critic_w={k: v.cpu().clone() for k, v in dd.critic.state_dict().items()})
    lo_b, lo_f = oracle(BO.linear("bf16")), oracle(F.linear)
    dd.train()
    idx = dd.last_batch_info()["idx"].cpu().numpy()
    batch = (Sx[idx], Ax[idx], R[idx], S2[idx], D[idx])
    ob, of = lo_b.train_step(*batch), lo_f.train_step(*batch)
    m = dd.debug_tensor("m", (B, 101)).cpu().numpy()
    assert np.abs(m - ob["m"]).max() <= 1e-5
    lc, la = dd.last_losses()
    assert abs(lc - float(ob["loss_critic"])) <= 1e-5 * max(1.0, abs(lc))
    assert abs(la - float(ob["loss_actor"])) <= 1e-5 * max(1.0, abs(la))
    rel_b, rel_f = {}, {}
    for tag, net, gb, gf in (("actor", dd.actor, ob["grads_actor"], of["grads_actor"]),
                             ("critic", dd.critic, ob["grads_critic"], of["grads_critic"])):
        for k in H.NAMES:
            gk = net.named_grad_views()[k].cpu()
            rel_b[tag, k], rel_f[tag, k] = _rel(gk, gb[k]), _rel(gk, gf[k])
    worst_b = max(rel_b, key=rel_b.get)
    assert rel_b[worst_b] <= 1e-3, ("vs bf16 oracle", worst_b, rel_b[worst_b])
    worst_f = max(rel_f, key=rel_f.get)
    assert rel_f[worst_f] >= 10 * rel_b[worst_f], ("vs fp32 oracle", worst_f, rel_f[worst_f], rel_b[worst_f])
    print("config 5 bf16: worst rel L2 vs bf16 oracle %.2e %s, vs fp32 oracle %.2e %s" % (rel_b[worst_b], worst_b, rel_f[worst_f], worst_f))


@pytest.mark.gpu
def test_bf16_rejections():
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib
    info = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}
    dd = _ddpg(d4pg, 64, 17, 6, 51, n=1024, actor_critic="post_update")
    with pytest.raises(_lib.D4PGError):
        dd.train()                                  # post-update critic needs the tensor-core chain plan (precision 1/2)
    torch.manual_seed(0)
    act = d4pg.models.actor(17, 6, device="cuda")
    cri = d4pg.models.critic(17, 6, info, device="cuda")
    act.precision = 4; cri.precision = 4
    s = torch.zeros(8, 17, device="cuda"); a = torch.zeros(8, 6, device="cuda")
    with pytest.raises(_lib.D4PGError):
        act(s)
    with pytest.raises(_lib.D4PGError):
        cri(s, a)
