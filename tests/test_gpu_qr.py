"""Quantile-regression critic (critic_dist_info {"type": "quantile", "n_quantiles": N, "kappa": kappa}).

The reference has no quantile code, so the yardstick is the derived oracle tests/qr_oracle.py: the quantile-Huber head in
float64 from the fp32 quantile rows, the pinned init / Adam / Polyak / PER of oracle/d4pg_oracle.py around it.  CPU tests
pin the oracle itself (gradcheck, the order-statistic minimiser) and the Python-side checks; GPU tests hold the kernel
(d4pg_qr_loss), the module (d4pg_critic_forward / d4pg_critic_backward without the softmax) and the data-parallel step
to it; tests/test_gpu_mog_qr_learner.py holds the single-GPU learner step.
"""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests import bf16_oracle as BO
from tests import helpers as H
from tests import qr_oracle as QO

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


# ---- GPU: data parallel ---------------------------------------------------------------------------------------------
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
