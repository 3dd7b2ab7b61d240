"""Mixture-of-Gaussians critic (critic_dist_info {"type": "mixture_of_gaussian", "n_components": K}).

The reference stubs this branch, so the yardstick is the derived oracle tests/mog_oracle.py: the head in float64 from
the fp32 raw head (quadrature cross-entropy, td, policy loss), the pinned init / Adam / Polyak / PER of
oracle/d4pg_oracle.py around it.  CPU tests pin the oracle itself; GPU tests hold the kernel (d4pg_mog_loss) and the module
(d4pg_critic_forward_mog / d4pg_critic_backward_mog) to it; tests/test_gpu_mog_qr_learner.py holds the learner step.
"""
import math

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import bf16_oracle as BO
from tests import helpers as H
from tests import mog_oracle as MO
from tests import tf32_oracle as TO

H_ = 256


def _info(K):
    return {"type": "mixture_of_gaussian", "n_components": K}


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
def test_library_quadrature_is_hermgauss8():
    from d4pg_b200 import _lib
    x, h = _lib.mog_quadrature()
    xr, hr = np.polynomial.hermite.hermgauss(8)
    assert np.all(np.abs(np.array(x) - xr) <= 1e-15 * np.abs(xr))
    assert np.all(np.abs(np.array(h) - hr) <= 1e-15 * np.abs(hr))


def test_oracle_quadrature_integrates_polynomials_exactly():
    """8 Gauss-Hermite nodes integrate polynomials of degree <= 15 exactly: E[y^n] under every target component
    N(r + c mu', (c sigma')^2) equals the closed-form Gaussian moment."""
    K = 3
    raw = torch.tensor([[0.3, -1.0, 0.7, 0.4, -0.8, 1.2, -0.5, 0.2, 1.5]], dtype=torch.float64)
    r, done, disc = [-1.25], [False], 0.97
    y, om = MO.target_points(raw, r, done, disc, K)
    tw, tmu, tsig = MO.head(raw, K)
    for k in range(K):
        m, s = r[0] + disc * float(tmu[0, k]), disc * float(tsig[0, k])
        yk, wk = y[0, k * 8:(k + 1) * 8], om[0, k * 8:(k + 1) * 8] / float(tw[0, k])
        for n in range(16):
            exact = sum(math.comb(n, j) * m ** (n - j) * s ** j * (0 if j % 2 else math.prod(range(j - 1, 0, -2)))
                        for j in range(n + 1))
            got = float((wk * yk ** n).sum())
            assert abs(got - exact) <= 1e-12 * max(1.0, abs(exact)), (k, n, got, exact)
    # a terminal row collapses to a Dirac at r
    y, om = MO.target_points(raw, r, [True], disc, K)
    assert torch.all(y == r[0]) and abs(float(om.sum()) - 1.0) < 1e-14


def test_oracle_head_gradient_passes_gradcheck():
    K, B = 4, 3
    g = torch.Generator().manual_seed(0)
    traw = torch.randn(B, 3 * K, generator=g, dtype=torch.float64)
    qraw = torch.randn(B, 3 * K, generator=g, dtype=torch.float64).requires_grad_(True)
    r, done = [-1.0, 0.5, 2.0], [False, True, False]
    assert torch.autograd.gradcheck(lambda q: MO.loss_rows(traw, q, r, done, 0.99, K), (qraw,))
    assert torch.autograd.gradcheck(lambda q: MO.policy_rows(q, K), (qraw,))


def test_cpu_mixture_critic_shapes_and_seeded_weights():
    import d4pg_b200 as d4pg
    K = 5
    torch.manual_seed(3)
    m = d4pg.models.critic(17, 6, _info(K), device="cpu")
    torch.manual_seed(3)
    c = d4pg.models.critic(17, 6, {"type": "categorical", "v_min": -1.0, "v_max": 1.0, "n_atoms": 3 * K}, device="cpu")
    sm, sc = m.state_dict(), c.state_dict()
    assert list(sm) == list(sc) == H.NAMES
    assert sm["fc3.weight"].shape == (3 * K, 256) and sm["fc3.bias"].shape == (3 * K,)
    for k in H.NAMES:
        assert torch.equal(sm[k], sc[k]), k
    with pytest.raises(d4pg._lib.D4PGError):
        d4pg.models.critic(17, 6, _info(33), device="cpu")


def test_mixture_ddpg_rejects_ce_priority_and_categorical_projection():
    import d4pg_b200 as d4pg
    with pytest.raises(d4pg._lib.D4PGError):
        d4pg.DDPG(17, 6, memory_size=64, batch_size=8, critic_dist_info=_info(5), priority="ce")
    dd = d4pg.DDPG(17, 6, memory_size=64, batch_size=8, critic_dist_info=_info(5))
    assert dd.critic.state_dict()["fc3.weight"].shape == (15, 256)
    with pytest.raises(d4pg._lib.D4PGError):
        dd.reproject2(np.zeros((2, 15), np.float32), [0.0, 0.0], [False, False])


# ---- GPU: the head kernel alone -----------------------------------------------------------------------------------
def _raw(B, K, g):
    o = torch.empty(B, 3 * K)
    o[:, :K] = 2.0 * torch.randn(B, K, generator=g)
    o[:, K:2 * K] = 5.0 * torch.randn(B, K, generator=g)
    o[:, 2 * K:] = torch.rand(B, K, generator=g) * 60.0 - 30.0       # softplus threshold and the 1e-3 floor
    return o


@pytest.mark.gpu
@pytest.mark.parametrize("K", [1, 5, 32])
@pytest.mark.parametrize("B", [1, 256, 4096])
def test_mog_loss_kernel_vs_oracle(K, B):
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib
    L = _lib.lib()
    g = torch.Generator().manual_seed(100 * K + B)
    traw, qraw, praw = _raw(B, K, g), _raw(B, K, g), _raw(B, K, g)
    r = (-3.0 * torch.rand(B, generator=g, dtype=torch.float64) + 1.0)
    done = torch.rand(B, generator=g) < 0.05
    if B > 1:
        done[0] = True
    for disc in (0.99, 0.99 ** 5):
        dev = lambda t: t.cuda().contiguous()
        outs = {k: torch.empty(B, device="cuda") for k in ("loss_rows", "td", "prio", "pi_rows")}
        dq, dpi = torch.empty(B, 3 * K, device="cuda"), torch.empty(B, 3 * K, device="cuda")
        t_, q_, p_, r_, d_ = dev(traw), dev(qraw), dev(praw), dev(r), dev(done.to(torch.uint8))
        _lib.check(L.d4pg_mog_loss(_lib.ptr(t_), _lib.ptr(q_), _lib.ptr(p_), _lib.ptr(r_), _lib.ptr(d_), B, K, disc, 1e-6,
                                   1.0 / B, _lib.ptr(outs["loss_rows"]), _lib.ptr(outs["td"]), _lib.ptr(outs["prio"]),
                                   _lib.ptr(dq), _lib.ptr(outs["pi_rows"]), _lib.ptr(dpi), _lib.stream_ptr()),
                   "d4pg_mog_loss")
        torch.cuda.synchronize()
        ref = MO.heads(traw, qraw, praw, r.numpy(), done.numpy(), disc, K, 1.0 / B)
        for k in ("loss_rows", "td", "prio", "pi_rows"):
            mine, want = outs[k].double().cpu(), ref[k]
            err = (mine - want).abs() / want.abs().clamp(min=1.0)
            assert float(err.max()) <= 1e-5, (k, disc, float(err.max()))
        for k, mine in (("dq_raw", dq), ("dpi_raw", dpi)):
            want = ref[k]
            scale = want.abs().amax(1, keepdim=True).clamp(min=1e-30)
            err = ((mine.double().cpu() - want).abs() / scale).max()
            assert float(err) <= 1e-5, (k, disc, float(err))


# ---- GPU: the module ------------------------------------------------------------------------------------------------
def _lin_for(precision):
    return {2: TO.linear("rz"), 3: BO.linear("bf16")}.get(precision, F.linear)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [0, 1, 2, 3])
@pytest.mark.parametrize("K,B", [(5, 256), (11, 1024)])
def test_mog_module_forward_and_gradients(precision, K, B):
    """Forward: each layer fed the device's own input, against the restatement at that precision.  The differentiable
    forward is bit-identical to the no-grad one.  Gradients (random upstream gradients on w, mu and sigma): precisions
    0 / 1 against float64 autograd within 1e-5 (device ReLU masks), precision 3 against the bf16 linear at relative L2
    1e-3, precision 2 against the rz TF32 linear at relative L2 3e-4."""
    import d4pg_b200 as d4pg
    S, A = 17, 6
    torch.manual_seed(40 + K)
    cri = d4pg.models.critic(S, A, _info(K), device="cuda")
    with torch.no_grad():
        cri.fc3.weight.normal_(0.0, 0.1)
    cri.precision = precision
    g = torch.Generator().manual_seed(41)
    s0 = torch.randn(B, S, generator=g); a0 = torch.rand(B, A, generator=g) * 2 - 1
    w_, mu_, sig_, raw = cri(s0.cuda(), a0.cuda(), return_logits=True)
    torch.cuda.synchronize()
    ws = cri._ws[:3 * B * H_].view(3, B, H_).cpu().double()
    W = {k: v.detach().cpu() for k, v in cri.state_dict().items()}
    tol = {0: 1e-5, 1: 1e-5, 2: 1e-5, 3: 1e-4}[precision]
    if precision == 2:
        lin64 = lambda x, w, b: TO.linear("rz")(x.float(), w, b).double()
    elif precision == 3:
        lin64 = lambda x, w, b: BO.rb(x.float()) @ BO.rb(w).T + b.double()
    else:
        lin64 = lambda x, w, b: F.linear(x.double(), w.double(), b.double())
    L = lambda x, l: lin64(x, W[l + ".weight"], W[l + ".bias"])
    _close("h1", ws[0], torch.relu(L(s0, "fc1")), tol)
    _close("h2", ws[1], torch.relu(L(torch.cat([ws[0], a0.double()], 1), "fc2")), tol)
    _close("h3", ws[2], torch.relu(L(ws[1], "fc2_2")), tol)
    ref_raw = L(ws[2], "fc3")
    _close("raw", raw.cpu(), ref_raw, tol)
    rw, rmu, rsig = MO.head(raw.cpu().double(), K)
    for name, mine, ref in (("w", w_, rw), ("mu", mu_, rmu), ("sigma", sig_, rsig)):
        _close(name, mine.cpu(), ref, 1e-6)

    # differentiable forward: bit-identical outputs, gradients through d4pg_critic_backward_mog
    cri.differentiable = True
    s = s0.cuda().requires_grad_(True); a = a0.cuda().requires_grad_(True)
    for p in cri.parameters():
        p.grad = None
    out = cri(s, a)
    for x, y in zip(out, (w_, mu_, sig_)):
        assert torch.equal(x.detach(), y)
    gw, gm, gs = (torch.randn(B, K, generator=g) / B for _ in range(3))
    torch.autograd.backward(list(out), [t.cuda() for t in (gw, gm, gs)])
    dt = torch.float64 if precision in (0, 1) else torch.float32
    lin = _lin_for(precision)
    Wl = {k: v.to(dt).requires_grad_(True) for k, v in W.items()}
    sl, al = s0.to(dt).requires_grad_(True), a0.to(dt).requires_grad_(True)
    m1, m2, m3 = (ws[i] > 0 for i in range(3))
    h = lin(sl, Wl["fc1.weight"], Wl["fc1.bias"]) * m1
    h = lin(torch.cat([h, al], 1), Wl["fc2.weight"], Wl["fc2.bias"]) * m2
    h = lin(h, Wl["fc2_2.weight"], Wl["fc2_2.bias"]) * m3
    o = lin(h, Wl["fc3.weight"], Wl["fc3.bias"]).double()
    torch.autograd.backward(list(MO.head(o, K)), [t.double() for t in (gw, gm, gs)])
    views = cri.named_grad_views()
    checks = [(k, views[k].cpu(), Wl[k].grad) for k in H.NAMES] + [("d state", s.grad.cpu(), sl.grad), ("d action", a.grad.cpu(), al.grad)]
    for name, mine, ref in checks:
        if precision in (0, 1):
            err = float((mine.double() - ref.double()).abs().max())
            assert err <= 1e-5 * max(1.0, float(ref.abs().max())), (name, err)
        else:
            assert _rel(mine, ref) <= (1e-3 if precision == 3 else 3e-4), (name, _rel(mine, ref))
