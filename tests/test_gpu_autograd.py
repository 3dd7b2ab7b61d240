"""`actor(..., differentiable=True)` / `critic(..., differentiable=True)`: an opt-in autograd path whose backward runs
d4pg_actor_backward / d4pg_critic_backward (csrc/mlp_backward.cu: an output-head kernel, then the level GEMMs).

Yardsticks: a float64 torch autograd restatement of models.py:32-41,76-88 (precisions 0-1), the TF32 linear of
tests/tf32_oracle.py with truncated operands (precision 2: the level GEMMs' rounding), the bf16 linear of
tests/bf16_oracle.py (precision 3: that oracle already defines the bf16 backward), and the learner's own gradient
buffer after one DDPG.train() step, recomputed here through the reference's learner body (ddpg.py:229-244)."""
import ctypes as C
import random

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import d4pg_oracle as O
from tests import bf16_oracle as BO
from tests import tf32_oracle as TO

NAMES = ("fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc2_2.weight", "fc2_2.bias", "fc3.weight", "fc3.bias")
# (S, A, N, B); A = 300 makes the actor's head plane wider than the 256-wide delta planes
SHAPES = [(17, 6, 51, 256), (3, 1, 51, 64), (5, 2, 7, 37), (17, 6, 51, 1), (376, 17, 51, 1024), (17, 6, 101, 4096),
          (5, 300, 7, 33)]
# precision 2 against the rz linear of tests/tf32_oracle.py: the reference chain computes its own forward, and an
# activation whose fp32 value differs in the last bit from the device's may truncate to the neighbouring TF32 value.
# Worst measured on one H100: 1.3e-4 (actor fc3.weight); against the unrounded float64 chain this bound was 5e-3.
TF32_REL_L2 = 3e-4


def _info(N):
    return {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": N}


def _close(name, mine, ref, tol=1e-5):
    """max abs error <= tol * max(1, |ref|max): a whole-tensor bound (tests/step_check.py, run by
    tests/test_gpu_step_edges.py, holds the learner step's layers to componentwise ones)"""
    mine, ref = mine.double().cpu(), ref.double().cpu()
    assert mine.shape == ref.shape, (name, mine.shape, ref.shape)
    scale = max(1.0, float(ref.abs().max()))
    err = float((mine - ref).abs().max())
    assert err <= tol * scale, "%s: max abs err %.3e (scale %.3g)" % (name, err, scale)


def _rel_l2(name, mine, ref, tol):
    mine, ref = mine.double().cpu(), ref.double().cpu()
    assert mine.shape == ref.shape, (name, mine.shape, ref.shape)
    rel = float((mine - ref).norm() / max(float(ref.norm()), 1e-30))
    assert rel <= tol, "%s: relative L2 %.3e > %.1e" % (name, rel, tol)


def _grads(net):
    return {k: p.grad for k, p in net.named_parameters()}


# ---- float64 / bf16 restatements of the two networks ------------------------------------------------------------------
# Each ReLU takes the device's branch: relu(x) = x * mask with mask = (device's h > 0).  A pre-activation within the
# forward's rounding error of zero may take either branch, and a flipped branch moves a whole delta (at TF32, a few in a
# thousand entries, ~3e-2 relative L2 on fc1); with the device's masks the comparison measures the backward alone.
def _ref_actor(w, s, lin, masks):
    h = lin(s, w["fc1.weight"], w["fc1.bias"]) * masks[0]
    h = lin(h, w["fc2.weight"], w["fc2.bias"])                       # no ReLU (H9)
    h = lin(h, w["fc2_2.weight"], w["fc2_2.bias"]) * masks[2]
    return torch.tanh(lin(h, w["fc3.weight"], w["fc3.bias"]))


def _ref_critic(w, s, a, lin, masks):
    h = lin(s, w["fc1.weight"], w["fc1.bias"]) * masks[0]
    h = lin(torch.cat([h, a], 1), w["fc2.weight"], w["fc2.bias"]) * masks[1]
    h = lin(h, w["fc2_2.weight"], w["fc2_2.bias"]) * masks[2]
    z = lin(h, w["fc3.weight"], w["fc3.bias"])
    return F.softmax(z, dim=1), z


def _device_masks(net, inputs, dtype):
    """ReLU masks of the device's forward (h1..h3 of the no-grad path, bit-identical to the differentiable one).  The
    critic is given a logits buffer: without one its forward reuses h1 as logits scratch."""
    with torch.no_grad():
        net(*inputs, **({"return_logits": True} if len(inputs) == 2 else {}))
    B = inputs[0].shape[0]
    ws = net._ws[:3 * B * 256].view(3, B, 256)
    return [(ws[i] > 0).cpu().to(dtype) for i in range(3)]


def _leaf(t, dtype):
    return t.detach().cpu().to(dtype).requires_grad_(True)


# ---- CPU ----------------------------------------------------------------------------------------------------------------
def test_differentiable_is_off_by_default():
    import d4pg_b200 as d4pg
    assert d4pg.models._FlatNet.differentiable is False
    assert d4pg.actor(5, 2, device="cpu").differentiable is False
    assert d4pg.critic(5, 2, _info(7), device="cpu").differentiable is False
    assert d4pg.actor(5, 2, device="cpu", differentiable=True).differentiable is True
    assert d4pg.critic(5, 2, _info(7), device="cpu", differentiable=True).differentiable is True


def test_differentiable_forward_on_cpu_module_raises():
    import d4pg_b200 as d4pg
    a = d4pg.actor(5, 2, device="cpu", differentiable=True)
    c = d4pg.critic(5, 2, _info(7), device="cpu", differentiable=True)
    s = torch.zeros(3, 5, requires_grad=True)
    with pytest.raises(d4pg.D4PGError):
        a(s)
    with pytest.raises(d4pg.D4PGError):
        c(s, torch.zeros(3, 2))


def test_zero_grad_and_flat_grads_handle_grads_outside_the_flat_buffer():
    """A .grad that autograd put outside the flat gradient buffer: zero_grad() clears it, flat_grads() takes its values
    over (so SharedAdam.step(), which reads flat_grads(), sees them) and rebinds .grad to the buffer."""
    import d4pg_b200 as d4pg
    a = d4pg.actor(5, 2, device="cpu")
    a.fc1.weight.grad = torch.ones(256, 5)
    a.zero_grad()
    assert float(a.fc1.weight.grad.abs().max()) == 0.0
    a.zero_grad(set_to_none=True)
    assert a.fc1.weight.grad is None

    b = d4pg.actor(5, 2, device="cpu")
    b.fc2.bias.grad = torch.full((256,), 2.0)
    b.fc3.weight.grad = torch.full((2, 256), 3.0)
    flat = b.flat_grads()
    views = b.named_grad_views()
    assert torch.equal(views["fc2.bias"], torch.full((256,), 2.0)) and torch.equal(views["fc3.weight"], torch.full((2, 256), 3.0))
    assert float(flat.abs().sum()) == 256 * 2.0 + 2 * 256 * 3.0          # everything else (pad columns too) is zero
    for k, p in b.named_parameters():
        assert torch.equal(p.grad, views[k]) and b._grad_in_flat(p.grad), k
    b.fc2.bias.grad = None                                               # None counts as zero
    b.flat_grads()
    assert float(b.named_grad_views()["fc2.bias"].abs().max()) == 0.0 and b._grad_in_flat(b.fc2.bias.grad)
    b.zero_grad()
    assert float(flat.abs().max()) == 0.0


def test_backward_entry_points_reject_bad_arguments():
    """Argument checks come before any device work: the dummy non-NULL pointers below are never dereferenced."""
    from d4pg_b200 import _lib
    L = _lib.lib()
    p = C.c_void_p(256)
    assert L.d4pg_actor_backward(p, 17, 6, p, 8, p, p, p, p, p, p, 7, None) == _lib.ENOTSUP
    assert L.d4pg_actor_backward(p, 17, 6, p, 0, p, p, p, p, p, p, 0, None) == _lib.EINVAL
    assert L.d4pg_actor_backward(p, 17, 6, p, 8, p, p, None, p, p, p, 0, None) == _lib.EINVAL
    assert L.d4pg_critic_backward(p, 17, 6, 51, p, p, 8, p, p, None, None, p, p, p, p, 0, None) == _lib.EINVAL
    assert L.d4pg_critic_backward(p, 17, 6, 51, p, p, 8, None, p, p, None, p, p, p, p, 0, None) == _lib.EINVAL
    assert L.d4pg_critic_backward(p, 17, 6, 500, p, p, 8, p, p, p, None, p, p, p, p, 0, None) == _lib.EINVAL
    assert L.d4pg_critic_backward(p, 17, 6, 51, p, p, 8, p, p, p, None, p, p, p, p, 4, None) == _lib.ENOTSUP


# ---- GPU ----------------------------------------------------------------------------------------------------------------
def _nets(d4pg, S, A, N, precision, seed=31):
    torch.manual_seed(seed)
    a = d4pg.actor(S, A, device="cuda", differentiable=True)
    c = d4pg.critic(S, A, _info(N), device="cuda", differentiable=True)
    # the weights are the constructors' own initialisation (the reference's, models.py:25-30,66-71), on purpose: with
    # output weights at the hidden layers' scale the tanh saturates, and 1 - y^2 turns the forward's own 3xTF32 error
    # (~1e-6 relative in the pre-activation) into a ~1e-5 relative error of every actor gradient, which would measure
    # the forward, not this backward.
    a.precision = c.precision = precision
    return a, c


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1, 2, 3])
def test_differentiable_forward_is_the_no_grad_forward(precision):
    import d4pg_b200 as d4pg
    for (S, A, N, B) in ((17, 6, 51, 256), (5, 2, 7, 37), (376, 17, 101, 200)):
        a, c = _nets(d4pg, S, A, N, precision)
        g = torch.Generator().manual_seed(5)
        s = torch.randn(B, S, generator=g).cuda(); act = (torch.rand(B, A, generator=g) * 2 - 1).cuda()
        with torch.no_grad():
            ref_a = a(s); ref_q, ref_z = c(s, act, return_logits=True)
        out_a = a(s)
        q, z = c(s, act, return_logits=True)
        q_only = c(s, act)
        assert out_a.grad_fn is not None and q.grad_fn is not None and z.grad_fn is not None and q_only.grad_fn is not None
        assert torch.equal(out_a, ref_a) and torch.equal(q, ref_q) and torch.equal(z, ref_z) and torch.equal(q_only, ref_q)
        a.differentiable = c.differentiable = False
        plain_a, plain_q = a(s), c(s, act)
        assert plain_a.grad_fn is None and not plain_a.requires_grad and plain_q.grad_fn is None
        assert torch.equal(plain_a, ref_a) and torch.equal(plain_q, ref_q)


def _check(name, mine, ref, precision):
    if precision in (0, 1):
        _close(name, mine, ref, 1e-5)
    elif precision == 2:
        _rel_l2(name, mine, ref, TF32_REL_L2)
    else:
        _rel_l2(name, mine, ref, 1e-3)


@pytest.mark.gpu
@pytest.mark.parametrize("S,A,N,B", SHAPES)
@pytest.mark.parametrize("precision", [0, 1, 2, 3])
def test_gradients_vs_float64_autograd(precision, S, A, N, B):
    """Random upstream gradients on the output; every parameter gradient, d state and d action against torch autograd on
    the float64 restatement (precision 2: the rz TF32 linear of tests/tf32_oracle.py; precision 3: the bf16 linear of
    tests/bf16_oracle.py).  B >= 1024 runs split-K dW.  The
    upstream gradients are N(0, 1) / B, what a batch-mean loss (ddpg.py:217,238) hands the output layer."""
    import d4pg_b200 as d4pg
    a, c = _nets(d4pg, S, A, N, precision)
    g = torch.Generator().manual_seed(7)
    s0 = torch.randn(B, S, generator=g); act0 = torch.rand(B, A, generator=g) * 2 - 1
    ga, gp, gz = (torch.randn(B, n, generator=g) / B for n in (A, N, N))
    dt = torch.float32 if precision in (2, 3) else torch.float64
    lin = {2: TO.linear("rz"), 3: BO.linear("bf16")}.get(precision, F.linear)

    # actor
    s = s0.cuda().requires_grad_(True)
    a(s).backward(ga.cuda())
    w = {k: _leaf(v, dt) for k, v in a.state_dict().items()}
    s_ref = _leaf(s0, dt)
    _ref_actor(w, s_ref, lin, _device_masks(a, (s0.cuda(),), dt)).backward(ga.to(dt))
    for k in NAMES:
        _check("actor " + k, _grads(a)[k], w[k].grad, precision)
    _check("actor d state", s.grad, s_ref.grad, precision)

    # critic: upstream gradient on probs, on logits, on both
    for mode in ("probs", "logits", "both"):
        for p in c.parameters():
            p.grad = None
        s = s0.cuda().requires_grad_(True); act = act0.cuda().requires_grad_(True)
        q, z = c(s, act, return_logits=True) if mode != "probs" else (c(s, act), None)
        outs, grads = {"probs": ([q], [gp]), "logits": ([z], [gz]), "both": ([q, z], [gp, gz])}[mode]
        torch.autograd.backward(outs, [x.cuda() for x in grads])
        w = {k: _leaf(v, dt) for k, v in c.state_dict().items()}
        s_ref, a_ref = _leaf(s0, dt), _leaf(act0, dt)
        q_ref, z_ref = _ref_critic(w, s_ref, a_ref, lin, _device_masks(c, (s0.cuda(), act0.cuda()), dt))
        ref_outs = {"probs": [q_ref], "logits": [z_ref], "both": [q_ref, z_ref]}[mode]
        torch.autograd.backward(ref_outs, [x.to(dt) for x in grads])
        for k in NAMES:
            _check("critic(%s) %s" % (mode, k), _grads(c)[k], w[k].grad, precision)
        _check("critic(%s) d state" % mode, s.grad, s_ref.grad, precision)
        _check("critic(%s) d action" % mode, act.grad, a_ref.grad, precision)


@pytest.mark.gpu
@pytest.mark.parametrize("B", [256, 1024])
@pytest.mark.parametrize("precision", ["fp32", "tf32x3"])
def test_reference_learner_body_through_autograd(precision, B):
    """One eager DDPG.train() step; then ddpg.py:229-244 written against differentiable modules holding the pre-step
    weights: loss_c from the learner's projected target m and sampled batch, .backward(); the policy loss through the
    pre-update critic (H7), .backward().  Both .grads must equal the learner's gradient buffer."""
    import d4pg_b200 as d4pg
    S, A, N, n = 17, 6, 51, 4096
    torch.manual_seed(8); random.seed(8); np.random.seed(8)
    dd = d4pg.DDPG(S, A, memory_size=n, batch_size=B, critic_dist_info=_info(N), precision=precision,
                   sampling="device", prefetch=False, use_graph=False, philox_seed=11)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
    rng = np.random.RandomState(9)
    dd.replayBuffer.add_batch(rng.randn(n, S).astype(np.float32), rng.uniform(-1, 1, (n, A)).astype(np.float32),
                              -3 * rng.rand(n), rng.randn(n, S).astype(np.float32), rng.rand(n) < 0.05)
    wa = {k: v.detach().clone() for k, v in dd.actor.state_dict().items()}
    wc = {k: v.detach().clone() for k, v in dd.critic.state_dict().items()}
    dd.train()
    s, a, m = dd.debug_tensor("s", (B, S)), dd.debug_tensor("a", (B, A)), dd.debug_tensor("m", (B, N))
    g_actor = {k: v.clone() for k, v in dd.actor.named_grad_views().items()}
    g_critic = {k: v.clone() for k, v in dd.critic.named_grad_views().items()}

    prec = {"fp32": 0, "tf32x3": 1}[precision]
    actor = d4pg.actor(S, A, device="cuda", differentiable=True)
    critic = d4pg.critic(S, A, _info(N), device="cuda", differentiable=True)
    actor.load_state_dict(wa); critic.load_state_dict(wc)
    actor.precision = critic.precision = prec
    z = torch.from_numpy(O.atom_support(-50.0, 0.0, N)[1].reshape(-1, 1)).float().cuda()

    critic.zero_grad()                                                   # ddpg.py:229-230
    q = critic(s, a)
    loss_c = (-(m * torch.log(q + 1e-10)).sum(dim=1)).mean()
    loss_c.backward()
    for k in NAMES:
        _close("critic " + k, _grads(critic)[k], g_critic[k])
    actor.zero_grad()                                                    # ddpg.py:236-242
    loss_a = -critic(s, actor(s)).matmul(z).mean()
    loss_a.backward()
    for k in NAMES:
        _close("actor " + k, _grads(actor)[k], g_actor[k])


@pytest.mark.gpu
def test_reference_training_loop_with_zero_grad_and_shared_adam():
    """Two iterations of the loop of ddpg.py:229-244 on fresh modules, with nothing called beforehand:
    critic.zero_grad(); loss_c.backward(); step(); actor.zero_grad(); loss_a.backward(); step().  Every .grad must be
    that iteration's gradient alone (not a sum with earlier losses), and SharedAdam must step on it: the same update
    as twin modules whose flat gradient buffer is filled by hand."""
    import d4pg_b200 as d4pg
    S, A, N, B = 17, 6, 51, 64
    torch.manual_seed(4)
    actor = d4pg.actor(S, A, device="cuda", differentiable=True)
    critic = d4pg.critic(S, A, _info(N), device="cuda", differentiable=True)
    twin_a, twin_c = d4pg.actor(S, A, device="cuda"), d4pg.critic(S, A, _info(N), device="cuda")
    twin_a.load_state_dict(actor.state_dict()); twin_c.load_state_dict(critic.state_dict())
    opts = {net: d4pg.SharedAdam(net.parameters(), lr=1e-3) for net in (actor, critic, twin_a, twin_c)}
    z = torch.from_numpy(O.atom_support(-50.0, 0.0, N)[1].reshape(-1, 1)).float().cuda()
    g = torch.Generator().manual_seed(6)

    def check_and_step(net, twin, loss):
        names = [k for k, _ in net.named_parameters()]
        alone = torch.autograd.grad(loss, [p for _, p in net.named_parameters()], retain_graph=True)
        loss.backward()
        for k, p, e in zip(names, net.parameters(), alone):
            _close(k, p.grad, e, 1e-6)
        before = net.flat_params().clone()
        opts[net].step()
        views = twin.named_grad_views()
        for k, e in zip(names, alone):
            views[k].copy_(e)
        opts[twin].step()
        assert not torch.equal(net.flat_params(), before)
        assert torch.equal(net.flat_params(), twin.flat_params())

    for _ in range(2):
        s = torch.randn(B, S, generator=g).cuda(); a = (torch.rand(B, A, generator=g) * 2 - 1).cuda()
        m = torch.softmax(torch.randn(B, N, generator=g), 1).cuda()
        critic.zero_grad()
        check_and_step(critic, twin_c, (-(m * torch.log(critic(s, a) + 1e-10)).sum(dim=1)).mean())
        actor.zero_grad()
        check_and_step(actor, twin_a, -critic(s, actor(s)).matmul(z).mean())


@pytest.mark.gpu
def test_autograd_semantics():
    import d4pg_b200 as d4pg
    S, A, N, B = 17, 6, 51, 64
    a, c = _nets(d4pg, S, A, N, 0)
    g = torch.Generator().manual_seed(3)
    s = torch.randn(B, S, generator=g).cuda()
    a1 = (torch.rand(B, A, generator=g) * 2 - 1).cuda(); a2 = (torch.rand(B, A, generator=g) * 2 - 1).cuda()
    g1 = torch.randn(B, N, generator=g).cuda(); g2 = torch.randn(B, N, generator=g).cuda()

    def grads(net):
        return {k: v.clone() for k, v in _grads(net).items()}

    def clear(net):
        for p in net.parameters():
            p.grad = None

    # two critic forwards before one backward (the reference's critic(s, a) and critic(s, actor(s))) = sum of the two
    (c(s, a1) * g1).sum().backward(); G1 = grads(c); clear(c)
    (c(s, a2) * g2).sum().backward(); G2 = grads(c); clear(c)
    ((c(s, a1) * g1).sum() + (c(s, a2) * g2).sum()).backward(); G12 = grads(c)
    for k in NAMES:
        _close("sum " + k, G12[k], G1[k] + G2[k], 1e-6)
    # a second .backward() accumulates
    (c(s, a1) * g1).sum().backward()
    for k in NAMES:
        _close("accumulate " + k, _grads(c)[k], G12[k] + G1[k], 1e-6)

    # torch.autograd.grad w.r.t. the input leaves every .grad untouched
    before = grads(c)
    sg = s.clone().requires_grad_(True)
    ds, = torch.autograd.grad((c(sg, a1) * g1).sum(), [sg])
    assert ds.shape == (B, S) and float(ds.abs().max()) > 0
    after = grads(c)
    assert all(torch.equal(before[k], after[k]) for k in NAMES)

    # frozen parameters: only d state is computed (no dW problems), and it equals the full path's
    clear(a)
    sg = s.clone().requires_grad_(True)
    ga = torch.randn(B, A, generator=g).cuda()
    a(sg).backward(ga)
    full = sg.grad.clone()
    for p in a.parameters():
        p.requires_grad_(False)
    sg = s.clone().requires_grad_(True)
    a(sg).backward(ga)
    assert torch.equal(sg.grad, full)
    for p in a.parameters():
        p.requires_grad_(True)
    clear(a)

    # .grad bound to the flat gradient buffer: autograd accumulates into it, zero_grad() clears it
    flat = a.flat_grads()
    a(s).backward(ga)
    views = a.named_grad_views()
    for k, p in a.named_parameters():
        assert torch.equal(views[k], p.grad)
        assert p.grad.data_ptr() >= flat.data_ptr() and p.grad.data_ptr() < flat.data_ptr() + flat.numel() * 4
    assert float(flat.abs().max()) > 0
    a.zero_grad()
    assert float(flat.abs().max()) == 0.0 and all(float(p.grad.abs().max()) == 0.0 for p in a.parameters())

    # an in-place parameter write between forward and backward is caught by the version counters
    out = a(s)
    with torch.no_grad():
        a.fc2.weight.mul_(1.0)
    with pytest.raises(RuntimeError, match="modified by an inplace operation"):
        out.backward(ga)

    # double backward is not supported
    sg = s.clone().requires_grad_(True)
    ds, = torch.autograd.grad((c(sg, a1) * g1).sum(), [sg], create_graph=True)
    with pytest.raises(RuntimeError):
        ds.sum().backward()
