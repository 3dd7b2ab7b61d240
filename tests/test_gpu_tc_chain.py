"""The cluster chains at precision="tf32x3" against a plain PyTorch float64 restatement of the same layers
(models.py:32-41,76-88 forward, autograd of ddpg.py:230,242 backward): every hidden activation, logit, delta and
parameter gradient of one eager DDPG.train() step.  Shapes with |s|, |a| <= 32 run the wgmma chains
(d4pg-pytorch_b200/csrc/mlp_tc_chain.cu); wider ones run the mma.sync 3xTF32 tiles of mlp_chain.cu.
Tolerance: 1e-5 absolute scaled by max(1, |ref|max) -- the 3xTF32 split is ~2^-21 relative per layer."""
import random

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu


def _ref(x):
    return x.double().cpu()


def _close(name, mine, ref, tol=1e-5):
    mine, ref = mine.double().cpu(), ref.double().cpu()
    assert mine.shape == ref.shape, (name, mine.shape, ref.shape)
    scale = max(1.0, float(ref.abs().max()))
    err = float((mine - ref).abs().max())
    assert err <= tol * scale, "%s: max abs err %.3e (scale %.3g)" % (name, err, scale)
    return err


@pytest.mark.parametrize("B,S,A,N,graph", [(256, 17, 6, 51, False), (256, 17, 6, 51, True), (64, 17, 6, 51, False), (200, 3, 1, 101, False),
                                           (512, 32, 8, 64, False), (40, 17, 6, 51, True),
                                           (96, 376, 17, 51, False)])
def test_tc_chain_every_intermediate_vs_torch(B, S, A, N, graph):
    import d4pg_b200 as d4pg
    info = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": N}
    torch.manual_seed(12); np.random.seed(12); random.seed(12)
    n = 2048
    dd = d4pg.DDPG(S, A, memory_size=n, batch_size=B, critic_dist_info=info, precision="tf32x3", use_graph=graph,
                   sampling="device", philox_seed=3, prefetch=False)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(1)
    dd.replayBuffer.add_batch(rng.randn(n, S).astype(np.float32), rng.uniform(-1, 1, (n, A)).astype(np.float32),
                              (-3 * rng.rand(n)), rng.randn(n, S).astype(np.float32), rng.rand(n) < 0.05)
    # make the target networks differ from the online ones
    with torch.no_grad():
        dd.actor_target.flat_params().mul_(1.01)
        dd.critic_target.flat_params().mul_(0.99)
    W = {k: {n_: _ref(v) for n_, v in net.state_dict().items()}
         for k, net in (("a", dd.actor), ("at", dd.actor_target), ("c", dd.critic), ("ct", dd.critic_target))}
    dd.train()
    torch.cuda.synchronize()
    # wgmma chains: sample, pack fwd, pack dX (side branch), fwd chains, loss, tree update, dX chains, dW, Adam;
    # the mma.sync chains read the weights directly and launch the same minus the two packs
    assert dd.kernels_per_step() == (9 if S <= 32 and A <= 32 and N <= 256 else 7)
    t = lambda name, w=None: dd.debug_tensor(name, (B, w) if w else None)
    s, a, s2 = _ref(t("s", S)), _ref(t("a", A)), _ref(t("s2", S))
    relu = torch.relu

    def actor_fwd(w, x):
        h1 = relu(x @ w["fc1.weight"].T + w["fc1.bias"])
        h2 = h1 @ w["fc2.weight"].T + w["fc2.bias"]                      # no ReLU here (models.py:36-37, SURVEY H9)
        h3 = relu(h2 @ w["fc2_2.weight"].T + w["fc2_2.bias"])
        return h1, h2, h3, torch.tanh(h3 @ w["fc3.weight"].T + w["fc3.bias"])

    def critic_fwd(w, x, act):
        h1 = relu(x @ w["fc1.weight"].T + w["fc1.bias"])
        h2 = relu(torch.cat([h1, act], 1) @ w["fc2.weight"].T + w["fc2.bias"])
        h3 = relu(h2 @ w["fc2_2.weight"].T + w["fc2_2.bias"])
        return h1, h2, h3, h3 @ w["fc3.weight"].T + w["fc3.bias"]

    _, _, _, at_out = actor_fwd(W["at"], s2)
    _, _, _, t_logits = critic_fwd(W["ct"], s2, at_out)
    ch1, ch2, ch3, q_logits = critic_fwd(W["c"], s, a)
    ah1, ah2, ah3, a_out = actor_fwd(W["a"], s)
    _, ph2, ph3, pi_logits = critic_fwd(W["c"], s, a_out)
    _close("target_logits", t("target_logits", N), t_logits)
    _close("q_logits", t("q_logits", N), q_logits)
    _close("pi_logits", t("pi_logits", N), pi_logits)
    _close("actor_out", t("actor_out", A), a_out)
    _close("actor_target_out", t("actor_target_out", A), at_out)
    for name, ref in (("h1_c", ch1), ("h2_c", ch2), ("h3_c", ch3), ("h1_a", ah1), ("h2_a", ah2), ("h3_a", ah3),
                      ("h2_p", ph2), ("h3_p", ph3)):
        _close(name, t(name, 256), ref)
    # backward: the logit gradients come from the loss kernel (tested elsewhere); the chains propagate them
    dq, dpi = _ref(t("dlogits_q", N)), _ref(t("dlogits_pi", N))
    Wc, Wa = W["c"], W["a"]
    # ReLU masks come from the DEVICE's forward activations (validated above to 1e-5): an element whose pre-activation is
    # ~0 may round to the other side of zero than the float64 restatement, which would flip a whole delta element
    dm = {k: _ref(t(k, 256)) > 0 for k in ("h1_c", "h2_c", "h3_c", "h1_a", "h3_a", "h2_p", "h3_p")}
    d_aout = _ref(t("actor_out", A))
    c_dz22 = (dq @ Wc["fc3.weight"]) * dm["h3_c"]
    c_dz2 = (c_dz22 @ Wc["fc2_2.weight"]) * dm["h2_c"]
    c_dz1 = (c_dz2 @ Wc["fc2.weight"][:, :256]) * dm["h1_c"]
    p_dz22 = (dpi @ Wc["fc3.weight"]) * dm["h3_p"]
    p_dz2 = (p_dz22 @ Wc["fc2_2.weight"]) * dm["h2_p"]
    a_dz3 = (p_dz2 @ Wc["fc2.weight"][:, 256:]) * (1 - d_aout * d_aout)
    a_dz22 = (a_dz3 @ Wa["fc3.weight"]) * dm["h3_a"]
    a_dh2 = a_dz22 @ Wa["fc2_2.weight"]
    a_dz1 = (a_dh2 @ Wa["fc2.weight"]) * dm["h1_a"]
    gs = max(float(dq.abs().max()), float(dpi.abs().max()), 1e-30)      # deltas are O(1/B): compare relative to the input scale
    for name, ref, w in (("c_dz22", c_dz22, 256), ("c_dz2", c_dz2, 256), ("c_dz1", c_dz1, 256), ("a_dz3", a_dz3, A),
                         ("a_dz22", a_dz22, 256), ("a_dh2", a_dh2, 256), ("a_dz1", a_dz1, 256)):
        mine = _ref(t(name, w))
        err = float((mine - ref).abs().max())
        assert err <= 1e-5 * max(gs, float(ref.abs().max())), "%s: %.3e vs scale %.3e" % (name, err, gs)
    grads = {"c": {"fc3.weight": dq.T @ ch3, "fc3.bias": dq.sum(0), "fc2_2.weight": c_dz22.T @ ch2, "fc2_2.bias": c_dz22.sum(0),
                   "fc2.weight": c_dz2.T @ torch.cat([ch1, a], 1), "fc2.bias": c_dz2.sum(0), "fc1.weight": c_dz1.T @ s, "fc1.bias": c_dz1.sum(0)},
             "a": {"fc3.weight": a_dz3.T @ ah3, "fc3.bias": a_dz3.sum(0), "fc2_2.weight": a_dz22.T @ ah2, "fc2_2.bias": a_dz22.sum(0),
                   "fc2.weight": a_dh2.T @ ah1, "fc2.bias": a_dh2.sum(0), "fc1.weight": a_dz1.T @ s, "fc1.bias": a_dz1.sum(0)}}
    for key, net in (("c", dd.critic), ("a", dd.actor)):
        views = net.named_grad_views()
        for k, ref in grads[key].items():
            mine = _ref(views[k]).reshape(ref.shape)
            assert float((mine - ref).abs().max()) <= 1e-5, (key, k, float((mine - ref).abs().max()))
            rel = float((mine - ref).norm() / max(float(ref.norm()), 1e-30))
            assert rel <= 1e-4, (key, k, rel)
