"""The categorical, mixture and quantile loss heads at every per-lane template and width edge, alone (the C ABI) and
inside the learner step, against the float64 restatements and per-output bounds of tests/heads_check.py.

Instantiations (the launchers' dispatch): heads_kernel<MODE, NT> with NT = 2 for N <= 64, 4 above (csrc/proj_loss.cu);
mog_heads_kernel<NT, HZ> with NT = 1 / 2 / 4 / 8 for K <= 4 / 8 / 16 / 32 and HZ when the batch carries per-row horizons
(csrc/mog_heads.cu); qr_heads_kernel<NT> with NT = ceil(N / 32) (csrc/qr_heads.cu).  The grid is cdiv(2B, 4) warps,
critic rows then policy rows, so an odd B puts a critic row and a policy row in one CTA.

CPU tests hold the bounds to a correct restatement rounded to fp32 and show that each one rejects a wrong head at the
same fixtures the GPU tests use.
"""
import math
import random

import numpy as np
import pytest
import torch

from oracle import d4pg_oracle as O
from tests import heads_check as HC
from tests import mog_oracle as MO
from tests import qr_oracle as QO
from tests import step_check as SC

F32, F64 = np.float32, np.float64
CAT_N = (2, 3, 31, 32, 33, 63, 64, 65, 96, 97, 127, 128)
MOG_K = (1, 2, 4, 5, 8, 9, 16, 17, 31, 32)
QR_N = (2, 31, 32, 33, 64, 65, 96, 97, 128)
BATCHES = (1, 2, 3, 5, 4097)
KAPPAS = (1e-3, 1.0, 1e3)

WORST = {}          # (head, template) -> worst ratio to the bound over the cases run


def _record(head, nt, worst):
    WORST[head, nt] = max(WORST.get((head, nt), 0.0), worst)
    print("%s<%s> worst so far %.3f of bound" % (head, nt, WORST[head, nt]))


def _f32(x):
    return torch.as_tensor(x).float()


# ---- CPU: a correct head rounded to fp32 passes, each wrong head fails ------------------------------------------------
def _cat_emulate(inp, v_min, v_max, disc, mode, flags=0, isw=None, gs=1.0, ce=False, eps=HC.EPS10, drop_integral=False,
                 proj_disc=None):
    """A categorical head that does the right thing up to one fp32 rounding per output (mode 0: project_live itself);
    eps / drop_integral / proj_disc give the mutants."""
    tl, ql, pl, r, d = inp["tl"], inp["ql"], inp["pl"], inp["r"], inp["d"]
    B, N = tl.shape
    NT = HC.cat_nt(N)
    tp = _f32(HC.softmax_bound(tl, NT, bool(flags & 1))[0])
    qp = _f32(HC.softmax_bound(ql, NT, bool(flags & 2))[0])
    pd = disc if proj_disc is None else proj_disc
    if mode == 0 and not drop_integral:
        m = torch.from_numpy(O.project_live(tp.numpy(), r, d, v_min, v_max, N, float(np.asarray(pd).reshape(-1)[0])))
    else:
        m = _f32(HC.project(tp.numpy(), r, d, v_min, v_max, N, pd, mode, drop_integral)[0])
    isw = np.ones(B) if isw is None else isw
    out = {k: _f32(v[0]) for k, v in HC.cat_loss(m, qp, isw, gs, NT, ce_priority=ce, eps=eps).items()}
    z32 = O.atom_support(v_min, v_max, N)[1].astype(F32)
    out.update({k: _f32(v[0]) for k, v in HC.policy_bound(pl, z32, gs, NT).items()})
    out.update(m=m.float(), tp=tp, qp=qp)
    return out


def _cat_ratios(inp, dev, v_min, v_max, disc, mode, flags=0, isw=None, gs=1.0, ce=False):
    rep = HC.Report("cpu")
    HC.cat_check(rep, inp, dev, v_min, v_max, disc, mode, flags, isw, gs, 1e-6, ce)
    return dict(rep.rows)


def _fails(rows, *names):
    """Every named check (a prefix matches all its stages) lands POWER_MIN x outside its bound, or is NaN."""
    for name in names:
        hits = [r for n, r in rows.items() if n == name or n.startswith(name + " ")]
        assert hits, name
        assert any(not r < HC.POWER_MIN for r in hits), (name, hits)


@pytest.mark.parametrize("N", [33, 97, 128])
@pytest.mark.parametrize("mode", [0, 1])
def test_categorical_bound_passes_the_head_and_rejects_each_mutant(N, mode):
    B = 4097
    for s, variant in enumerate(HC.CAT_VARIANTS):
        inp, v_min, v_max, disc, flags = HC.cat_fixture(N, B, variant, seed=s)
        disc_n = disc ** 5 if mode else disc                    # the standalone call takes gamma (mode 0) or gamma^n
        gs = float(F32(1.0 / B))
        good = _cat_emulate(inp, v_min, v_max, disc_n, mode, flags, gs=gs)
        rows = _cat_ratios(inp, good, v_min, v_max, disc_n, mode, flags, gs=gs)
        assert max(rows.values()) <= 1.0, (variant, {k: v for k, v in rows.items() if not v <= 1.0})
        if variant == "wide":                                   # logits over +-80: some q are exactly 0
            assert bool((good["qp"] == 0).any())
            bad = _cat_emulate(inp, v_min, v_max, disc_n, mode, flags, gs=gs, eps=0.0)
            _fails(_cat_ratios(inp, bad, v_min, v_max, disc_n, mode, flags, gs=gs), "loss_rows", "dq")
        if variant == "exact" and mode == 1:                    # b_j on atoms: the l -= 1 / u += 1 adjustment
            bad = _cat_emulate(inp, v_min, v_max, disc_n, mode, flags, gs=gs, drop_integral=True)
            _fails(_cat_ratios(inp, bad, v_min, v_max, disc_n, mode, flags, gs=gs), "m", "td")


def test_mixture_bound_passes_the_head_and_rejects_the_softplus_threshold_at_20():
    """sigma raw exactly 20 takes log1p(exp(20)) (torch: linear only for x > 20); a head taking x >= 20 moves the
    target points of the `points` rows by ~1e-9, which the online mean gradients at the 1e-3 sigma floor resolve."""
    for K, B in ((8, 4097), (9, 4097), (16, 5), (17, 5), (32, 5)):
        inp, disc = HC.mog_fixture(K, B, "plain")
        ref = HC.mog_refs(inp["tr"], inp["q"], inp["pi"], inp["r"], inp["d"], K, disc, np.ones(B), 1.0 / B)
        good = {k: _f32(v[0]) for k, v in ref.items()}
        rows = {k: HC.ratio(good[k], *v) for k, v in ref.items()}
        assert max(rows.values()) <= 1.0, rows
        real = MO.head

        def head_ge(o, K):
            w, mu, _ = real(o, K)
            x = o[:, 2 * K:3 * K]
            return w, mu, torch.where(x >= 20, x, torch.log1p(torch.exp(x))) + 1e-3
        MO.head = head_ge
        try:
            bad = HC.mog_refs(inp["tr"], inp["q"], inp["pi"], inp["r"], inp["d"], K, disc, np.ones(B), 1.0 / B)
        finally:
            MO.head = real
        rows = {k: HC.ratio(_f32(bad[k][0]), *v) for k, v in ref.items()}
        assert rows["dq"] >= HC.POWER_MIN, (K, rows)


def _qr_le(tq, q, r, d, disc, kappa):
    """Loss rows and dL/dtheta with the indicator 1{u <= 0} in place of 1{u < 0}."""
    y = QO.targets(tq, r, d, disc)
    th = q.double()
    N = th.shape[1]
    u = y.unsqueeze(2) - th.unsqueeze(1)
    w = (QO.taus(N).view(1, 1, N) - (u <= 0).double()).abs()
    return (w * QO.huber(u, kappa)).sum((1, 2)) / (kappa * N), -(w * u.clamp(-kappa, kappa)).sum(1) / (kappa * N)


@pytest.mark.parametrize("kappa", KAPPAS)
def test_quantile_bound_passes_the_head_and_rejects_a_shifted_tau(kappa):
    """One quantile's tau taken from the next index fails the gradient bound.  The indicator tie is harmless: where
    u = 0, both H(u) and clamp(u) vanish, so 1{u <= 0} computes the same head at the fixtures' exact ties (and the
    Huber pieces meet at |u| = kappa): no bound can reject it, and the check below pins that it does not matter."""
    for N in (33, 65, 97):
        inp, disc = HC.qr_fixture(N, 4097, kappa, seed=KAPPAS.index(kappa))
        B = 4097
        ref = HC.qr_refs(inp["tq"], inp["q"], inp["pi"], inp["r"], inp["d"], disc, kappa, np.ones(B), 1.0 / B)
        rows = {k: HC.ratio(_f32(v[0]), *v) for k, v in ref.items()}
        assert max(rows.values()) <= 1.0, rows
        y = QO.targets(inp["tq"], inp["r"], inp["d"], disc)
        u = y.unsqueeze(2) - inp["q"].unsqueeze(1)
        assert bool((u == 0).any()) and bool((u == kappa).any()) and bool((u == -kappa).any())
        real = QO.taus
        k0 = N // 2
        QO.taus = lambda n: torch.cat([real(n)[:k0], real(n)[k0 + 1:k0 + 2], real(n)[k0 + 1:]])
        try:
            bad = HC.qr_refs(inp["tq"], inp["q"], inp["pi"], inp["r"], inp["d"], disc, kappa, np.ones(B), 1.0 / B)
        finally:
            QO.taus = real
        assert HC.ratio(_f32(bad["dq"][0]), *ref["dq"]) >= HC.POWER_MIN
        lo, go = _qr_le(inp["tq"], inp["q"], inp["r"], inp["d"], disc, kappa)
        assert torch.equal(lo, QO.loss_rows(inp["tq"], inp["q"], inp["r"], inp["d"], disc, kappa))
        assert torch.equal(go, QO.grad_closed_form(inp["tq"], inp["q"], inp["r"], inp["d"], disc, kappa))


# in-step fixtures on the CPU: planes at pitch Np > N with zero pads, IS weights, per-row horizons
def _planes(kind, N, B=64, seed=3, mode=1, tails=True, gamma=0.95, n=5, ce=False, emulate=None):
    rng = np.random.RandomState(seed)
    Np = -(-N // 4) * 4 + (4 if N % 4 == 0 else 0)             # a pad of at least one column
    K = N // 3 if kind == "mog" else None
    planes = {}
    for k in ("target_logits", "q_logits", "pi_logits"):
        x = np.zeros((B, Np), F32)
        x[:, :N] = rng.randn(B, N) * 2
        planes[k] = torch.from_numpy(x)
    h = rng.randint(0, n, B).astype(np.uint8) if tails else np.zeros(B, np.uint8)
    cfg = dict(kind=kind, N=N, K=K, v_min=-10.0, v_max=0.0, gamma=gamma, n_steps=n, mode=mode, tails=tails, kappa=1.0,
               B=B, gs=float(F32(1.0) / F32(B)), prio_eps=1e-6, ce=ce)
    planes.update(r=-3 * rng.rand(B), d=rng.rand(B) < 0.1, h=h, isw=rng.uniform(0.3, 1.0, B).astype(F32).astype(F64))
    return planes, cfg


def _emulate_step(P, cfg, disc=None, isw=None, stride=False):
    """Device planes of a head that does the right thing up to one fp32 rounding per output -- or, through the
    arguments, reads rows with stride N instead of the pitch, drops the IS weight, or uses another discount."""
    N, B = cfg["N"], cfg["B"]
    Np = P["q_logits"].shape[1]
    disc = HC.step_discounts(cfg, P["h"]) if disc is None else disc
    isw = P["isw"] if isw is None else isw
    rd = (lambda k: P[k].reshape(-1)[:B * N].reshape(B, N).double()) if stride else (lambda k: P[k][:, :N].double())
    tl, ql, pl = rd("target_logits"), rd("q_logits"), rd("pi_logits")
    if cfg["kind"] == "cat":
        inp = dict(tl=tl, ql=ql, pl=pl, r=P["r"], d=P["d"])
        out = _cat_emulate(inp, cfg["v_min"], cfg["v_max"], disc if cfg["mode"] else float(disc[0]), cfg["mode"], 0, isw,
                           cfg["gs"], cfg["ce"])
    elif cfg["kind"] == "mog":
        out = {k: _f32(v[0]) for k, v in HC.mog_refs(tl, ql, pl, P["r"], P["d"], cfg["K"], disc, isw, cfg["gs"]).items()}
    else:
        out = {k: _f32(v[0]) for k, v in HC.qr_refs(tl, ql, pl, P["r"], P["d"], disc, cfg["kappa"], isw, cfg["gs"],
                                                    1e-6, cfg["ce"]).items()}
    Q = dict(P)
    for k, src in (("m", "m"), ("target_probs", "tp"), ("q_probs", "qp"), ("dlogits_q", "dq"), ("dlogits_pi", "dpi")):
        x = torch.zeros(B, Np)
        if src in out:
            x[:, :N] = out[src]
        Q[k] = x
    for k in ("loss_rows", "td", "prio", "pi_rows"):
        Q[k] = out[k]
    Q["losses"] = torch.tensor([float(out["loss_rows"].double().mean()), float(out["pi_rows"].double().mean()), 0, 0])
    return Q


def _step_rows(P, cfg):
    rep = HC.Report("cpu")
    HC.check_planes(rep, P, cfg)
    return dict(rep.rows)


@pytest.mark.parametrize("kind,N", [("cat", 51), ("cat", 97), ("mog", 15), ("mog", 27), ("qr", 33), ("qr", 65)])
@pytest.mark.parametrize("mode", [0, 1])
def test_step_check_passes_the_head_and_rejects_stride_weight_and_discount_mutants(kind, N, mode):
    """At pitch Np > N with IS weights and (mode 1) per-row horizons: rows read with stride N, the IS weight left out of
    the loss row and of dq, and gamma where gamma^n / gamma^h is due (gamma^n where gamma is due in mode 0) all fail."""
    for ce in ((False, True) if kind != "mog" else (False,)):
        P, cfg = _planes(kind, N, mode=mode, tails=bool(mode), ce=ce)
        good = _emulate_step(P, cfg)
        rows = _step_rows(good, cfg)
        assert max(rows.values()) <= 1.0, {k: v for k, v in rows.items() if not v <= 1.0}
        _fails(_step_rows(_emulate_step(P, cfg, stride=True), cfg), "dq", "loss_rows")
        _fails(_step_rows(_emulate_step(P, cfg, isw=np.ones(cfg["B"])), cfg), "loss_rows", "dq")
        g = cfg["gamma"]
        wrong = np.full(cfg["B"], g if mode else g ** cfg["n_steps"])
        _fails(_step_rows(_emulate_step(P, cfg, disc=wrong), cfg), "td")
        # a dropped pad guard: a head writing its last row past N
        bad = dict(good)
        bad["dlogits_q"] = good["dlogits_q"].clone()
        bad["dlogits_q"][:, N] = 1e-3
        _fails(_step_rows(bad, cfg), "pad dlogits_q")


@pytest.mark.parametrize("v_min,v_max", [(-50.0, 0.0), (-150.0, 150.0), (-10.0, 0.0), (0.1, 0.7), (-1e-3, 3.0)])
def test_clip_top_keeps_every_bin_inside_the_row(v_min, v_max):
    """The return clip's top (O.atom_clip_top, restating csrc/proj_loss.cu proj_clip_top): v_max wherever b(v_max) is at
    most N - 1, else the largest double whose b is -- one double above it, b passes N - 1.  On [-50, 0] that is 30, 32,
    59, 63, 98, 117 and 125 atoms, where a return at v_max used to give u = N."""
    moved = []
    for N in range(2, 129):
        delta, _ = O.atom_support(v_min, v_max, N)
        b = lambda t: (t - v_min) / delta
        top = O.atom_clip_top(v_min, v_max, N)
        assert top <= v_max and b(top) <= N - 1
        if top != v_max:
            assert b(v_max) > N - 1 and b(float(np.nextafter(top, np.inf))) > N - 1
            moved.append(N)
        m, l, u = O.project_live(np.full((1, N), 1.0 / N, F32), [v_max + 1.0], [False], v_min, v_max, N, 0.99,
                                 return_bins=True)
        assert u.max() <= N - 1
    print("clip top below v_max at N =", moved)
    assert v_min != -50.0 or moved == [30, 32, 59, 63, 98, 117, 125]


def test_fixtures_reach_every_instantiation():
    assert {HC.cat_nt(n) for n in CAT_N} == {2, 4}
    assert {HC.mog_nt(k) for k in MOG_K} == {1, 2, 4, 8}
    assert {HC.qr_nt(n) for n in QR_N} == {1, 2, 3, 4}
    for nt in (1, 2, 4, 8):                                     # both sides of every boundary
        assert nt == 8 or any(HC.mog_nt(k) == nt and HC.mog_nt(k + 1) != nt for k in MOG_K)
    heads = [c[5]["type"] for c in STEP_CASES]
    mog = {(HC.mog_nt(c[5]["n_components"]), bool(c[6].get("nstep_tails"))) for c in STEP_CASES
           if c[5]["type"] == "mixture_of_gaussian"}
    assert {(nt, True) for nt in (1, 2, 4, 8)} <= mog          # HZ = true runs only inside the step
    tails = [c[5]["type"] for c in STEP_CASES if c[6].get("nstep_tails")]
    assert set(tails) == set(heads)


# ---- GPU: the C ABI at every width, batch and input edge --------------------------------------------------------------
def _nan(*shape):
    return torch.full(shape, math.nan, dtype=torch.float32, device="cuda")


def _dev(x, dt=torch.float32):
    return torch.as_tensor(np.ascontiguousarray(x)).to(dt).cuda()


def _run_cat(inp, v_min, v_max, disc, mode, flags, only_dq=False):
    from d4pg_b200 import _lib
    B, N = inp["tl"].shape
    tl, ql, pl = _dev(inp["tl"].numpy()), _dev(inp["ql"].numpy()), _dev(inp["pl"].numpy())
    r, d = _dev(inp["r"], torch.float64), _dev(np.asarray(inp["d"]).astype(np.uint8), torch.uint8)
    o = {k: _nan(B, N) for k in ("m", "tp", "qp", "dq", "dpi")}
    o.update({k: _nan(B) for k in ("loss_rows", "td", "prio", "pi_rows")})
    bl, bu = torch.full((B, N), -1, dtype=torch.int32, device="cuda"), torch.full((B, N), -1, dtype=torch.int32, device="cuda")
    P = _lib.ptr
    opt = (lambda k: None) if only_dq else (lambda k: P(o[k]))
    _lib.check(_lib.lib().d4pg_proj_loss(P(tl), P(ql), P(pl), P(r), P(d), B, N, v_min, v_max, disc, mode, flags, 1e-6,
                                         1.0 / B, opt("m"), None if only_dq else P(bl), None if only_dq else P(bu),
                                         opt("tp"), opt("qp"), opt("loss_rows"), opt("td"), opt("prio"), P(o["dq"]),
                                         opt("pi_rows"), opt("dpi"), _lib.stream_ptr()), "d4pg_proj_loss")
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}, (bl.cpu().numpy(), bu.cpu().numpy())


@pytest.mark.gpu
@pytest.mark.parametrize("mode", [0, 1])
@pytest.mark.parametrize("N", CAT_N)
def test_categorical_head_every_width_batch_and_input_edge(N, mode):
    NT = HC.cat_nt(N)
    worst = 0.0
    for B in BATCHES:
        for s, variant in enumerate(HC.CAT_VARIANTS):
            inp, v_min, v_max, disc, flags = HC.cat_fixture(N, B, variant, seed=s)
            disc = disc ** 5 if mode else disc
            dev, bins = _run_cat(inp, v_min, v_max, disc, mode, flags)
            rep = HC.Report("cat<%d,%d> N=%d B=%d %s" % (mode, NT, N, B, variant))
            HC.cat_check(rep, inp, dev, v_min, v_max, disc, mode, flags, None, 1.0 / B, 1e-6, False, bins)
            worst = max(worst, rep.finish()[0])
            if B == 4097 and s == 0:                           # only dq requested: the same dq bit for bit
                only, _ = _run_cat(inp, v_min, v_max, disc, mode, flags, only_dq=True)
                assert torch.equal(only["dq"], dev["dq"])
                assert bool(torch.isnan(only["m"]).all() and torch.isnan(only["loss_rows"]).all())
    _record("heads_kernel<%d,%d>" % (mode, NT), NT, worst)


def _run_mog(inp, K, disc, only_dq=False):
    from d4pg_b200 import _lib
    B = inp["tr"].shape[0]
    t, q, pi = (_dev(inp[k].numpy()) for k in ("tr", "q", "pi"))
    r, d = _dev(inp["r"], torch.float64), _dev(np.asarray(inp["d"]).astype(np.uint8), torch.uint8)
    o = {"dq": _nan(B, 3 * K), "dpi": _nan(B, 3 * K)}
    o.update({k: _nan(B) for k in ("loss_rows", "td", "prio", "pi_rows")})
    P = _lib.ptr
    opt = (lambda k: None) if only_dq else (lambda k: P(o[k]))
    _lib.check(_lib.lib().d4pg_mog_loss(P(t), P(q), P(pi), P(r), P(d), B, K, disc, 1e-6, 1.0 / B, opt("loss_rows"),
                                        opt("td"), opt("prio"), P(o["dq"]), opt("pi_rows"), opt("dpi"),
                                        _lib.stream_ptr()), "d4pg_mog_loss")
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("K", MOG_K)
def test_mixture_head_every_width_batch_and_input_edge(K):
    worst = 0.0
    for B in BATCHES:
        for s, variant in enumerate(HC.MOG_VARIANTS):
            inp, disc = HC.mog_fixture(K, B, variant, seed=s)
            dev = _run_mog(inp, K, disc)
            rep = HC.Report("mog<%d> K=%d B=%d %s" % (HC.mog_nt(K), K, B, variant))
            HC.check_refs(rep, HC.mog_refs(inp["tr"], inp["q"], inp["pi"], inp["r"], inp["d"], K, disc, np.ones(B),
                                           1.0 / B), dev)
            worst = max(worst, rep.finish()[0])
            if B == 4097 and s == 0:
                assert torch.equal(_run_mog(inp, K, disc, only_dq=True)["dq"], dev["dq"])
    _record("mog_heads_kernel<%d,false>" % HC.mog_nt(K), HC.mog_nt(K), worst)


def _run_qr(inp, disc, kappa, ce, only_dq=False):
    from d4pg_b200 import _lib
    B, N = inp["tq"].shape
    t, q, pi = (_dev(inp[k].numpy()) for k in ("tq", "q", "pi"))
    r, d = _dev(inp["r"], torch.float64), _dev(np.asarray(inp["d"]).astype(np.uint8), torch.uint8)
    o = {"dq": _nan(B, N), "dpi": _nan(B, N)}
    o.update({k: _nan(B) for k in ("loss_rows", "td", "prio", "pi_rows")})
    P = _lib.ptr
    opt = (lambda k: None) if only_dq else (lambda k: P(o[k]))
    _lib.check(_lib.lib().d4pg_qr_loss(P(t), P(q), P(pi), P(r), P(d), B, N, disc, kappa, 1e-6, 1.0 / B, int(ce),
                                       opt("loss_rows"), opt("td"), opt("prio"), P(o["dq"]), opt("pi_rows"), opt("dpi"),
                                       _lib.stream_ptr()), "d4pg_qr_loss")
    torch.cuda.synchronize()
    return {k: v.cpu() for k, v in o.items()}


@pytest.mark.gpu
@pytest.mark.parametrize("N", QR_N)
def test_quantile_head_every_width_batch_and_input_edge(N):
    worst = 0.0
    for B in BATCHES:
        for s, kappa in enumerate(KAPPAS):
            for ce in ((False, True) if B < 4097 else (s == 1,)):
                inp, disc = HC.qr_fixture(N, B, kappa, seed=s + 2 * ce)
                dev = _run_qr(inp, disc, kappa, ce)
                rep = HC.Report("qr<%d> N=%d B=%d kappa=%g ce=%d" % (HC.qr_nt(N), N, B, kappa, ce))
                HC.check_refs(rep, HC.qr_refs(inp["tq"], inp["q"], inp["pi"], inp["r"], inp["d"], disc, kappa, np.ones(B),
                                              1.0 / B, 1e-6, ce), dev)
                worst = max(worst, rep.finish()[0])
                if B == 4097 and s == 0:
                    assert torch.equal(_run_qr(inp, disc, kappa, ce, only_dq=True)["dq"], dev["dq"])
    _record("qr_heads_kernel<%d>" % HC.qr_nt(N), HC.qr_nt(N), worst)


# ---- GPU: the heads inside one eager learner step ----------------------------------------------------------------------
def _cat(N, v=(-50.0, 0.0)):
    return {"type": "categorical", "v_min": v[0], "v_max": v[1], "n_atoms": N}


def _qr(N):
    return {"type": "quantile", "n_quantiles": N}


def _mog(K):
    return {"type": "mixture_of_gaussian", "n_components": K}


IW, CE = {"importance_weighted": True}, {"priority": "ce"}
TAILS = dict(projection="nstep", n_steps=5, nstep_tails=True, gamma=0.95)
C5 = dict(projection="nstep", n_steps=5)
# (plan, precision, B, |s|, |a|, critic head, DDPG options); each comment names the edge.  Planes are at pitch
# Np = pitch4(N): 51 -> 52, 97 -> 100, 2 -> 4, 33 -> 36, 65 -> 68, a K = 5 mixture's 15 -> 16, K = 9's 27 -> 28
STEP_CASES = [
    ("tc_chain", "tf32x3", 64, 17, 6, _cat(51), {}),                    # config 2 head, N = 51 at pitch 52
    ("tc_chain", "tf32", 65, 17, 6, _cat(97), {}),                      # NT = 4 at pitch 100, odd B: mixed CTA
    ("tc_chain", "tf32x3", 64, 17, 6, _cat(51), {"actor_critic": "post_update"}),   # the only_policy launch
    ("tc_chain", "tf32", 33, 17, 6, _mog(5), {}),                       # K = 5: NT = 2, 15 at pitch 16
    ("tc_chain", "tf32x3", 64, 17, 6, _cat(51), dict(IW, **CE)),        # IS weights and CE priorities
    ("tc_chain", "tf32x3", 64, 17, 6, _mog(5), TAILS),                  # mog_heads_kernel<2, true>
    ("chain", "fp32", 3, 1, 1, _cat(2), {}),                            # N = 2 at pitch 4, three rows
    ("chain", "tf32x3", 130, 17, 33, _cat(128), {}),                    # N = 128: no pad
    ("chain", "tf32", 65, 33, 6, _qr(33), {}),                          # qr NT = 2, 33 at pitch 36
    ("chain", "fp32", 64, 17, 6, _mog(9), IW),                          # K = 9: NT = 4, 27 at pitch 28, IS weights
    ("chain", "tf32", 64, 33, 6, _qr(65), TAILS),                       # per-row horizons, qr NT = 3
    ("chain", "fp32", 64, 17, 6, _mog(16), TAILS),                      # mog_heads_kernel<4, true>
    ("levels", "fp32", 65, 17, 6, _qr(65), {}),                         # qr NT = 3, 65 at pitch 68
    ("levels", "tf32x3", 64, 17, 6, _qr(97), {}),                       # qr NT = 4, 97 at pitch 100
    ("levels", "tf32", 64, 17, 6, _mog(16), {}),                        # K = 16: the last of NT = 4
    ("levels", "bf16", 65, 17, 6, _cat(97), {}),                        # bf16 planes into the fp32 head
    ("levels", "fp32", 64, 17, 6, _cat(51), IW),                        # IS weights
    ("levels", "fp32", 64, 17, 6, _qr(33), dict(IW, **CE)),             # quantile CE priorities
    ("levels", "bf16", 64, 17, 6, _cat(128), CE),
    ("levels", "fp32", 64, 17, 6, _cat(51), TAILS),                     # heads_kernel<1, 2> with gamma^h rows
    ("levels", "tf32x3", 64, 17, 6, _cat(97), TAILS),                   # heads_kernel<1, 4> with gamma^h rows
    ("levels", "tf32", 64, 17, 6, _qr(97), TAILS),
    ("levels", "fp32", 4096, 17, 6, _cat(101, (-150.0, 150.0)), C5),    # config 5: gamma^n, 4096 rows
    ("levels", "tf32x3", 1025, 17, 6, _mog(5), C5),                     # mixture with gamma^n
    ("levels", "bf16", 64, 17, 6, _mog(17), {}),                        # K = 17: NT = 8
    ("levels", "fp32", 64, 17, 6, _mog(4), TAILS),                      # mog_heads_kernel<1, true>
    ("levels", "tf32x3", 64, 17, 6, _mog(17), TAILS),                   # mog_heads_kernel<8, true>
]


def _id(case):
    plan, prec, B, S, A, info, kw = case
    head = {"categorical": "N", "quantile": "qr", "mixture_of_gaussian": "mogK"}[info["type"]]
    width = info.get("n_atoms") or info.get("n_quantiles") or info.get("n_components")
    tags = "".join("-" + ("tails" if k == "nstep_tails" else k if v is True else str(v)) for k, v in kw.items()
                   if k not in ("n_steps", "gamma") and not (k == "projection" and kw.get("nstep_tails")))
    return "%s-%s-B%d-%s%d%s" % (plan, prec, B, head, width, tags)


def _stream(dd, rng, K, E=32):
    """Vectorized-environment steps through observe() with many truncations: tail rows of every horizon."""
    S = dd.obs_dim
    for _ in range(K):
        s = torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda()
        a = dd.act(s)
        term = rng.rand(E) < 0.05
        trunc = (rng.rand(E) < 0.4) & ~term
        dd.observe(s, a, torch.as_tensor(-rng.rand(E)).cuda(), torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda(),
                   torch.as_tensor(term).cuda(), torch.as_tensor(trunc).cuda())


@pytest.mark.gpu
@pytest.mark.parametrize("case", STEP_CASES, ids=[_id(c) for c in STEP_CASES])
def test_heads_inside_the_learner_step(case):
    import d4pg_b200 as d4pg
    from tests.test_gpu_step_edges import _ddpg
    plan, precision, B, S, A, info, kw = case
    kw = dict(kw)
    if kw.get("nstep_tails"):
        torch.manual_seed(0); np.random.seed(0); random.seed(0)
        dd = d4pg.DDPG(S, A, memory_size=4096, batch_size=B, critic_dist_info=info, precision=precision,
                       sampling="device", prefetch=False, philox_seed=3, use_graph=False,
                       chain="levels" if plan == "levels" else "cluster", **kw)
        dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                                   d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
        _stream(dd, np.random.RandomState(8), 13)
    else:
        if plan == "levels":
            kw.setdefault("chain", "levels")
        dd = _ddpg(d4pg, B, S, A, info, precision, **kw)
    if dd.importance_weighted:                 # unequal priorities, so that the rows' IS weights differ
        n = len(dd.replayBuffer)
        dd.replayBuffer.update_priorities(np.arange(n), np.random.RandomState(5).uniform(0.1, 2.0, n))
    dd.train()
    torch.cuda.synchronize()
    if kw.get("actor_critic") != "post_update":                  # the plan the case names
        assert dd.kernels_per_step() == SC.KERNELS[plan], (plan, dd.kernels_per_step())
    P, cfg = HC.step_planes(dd), HC.step_config(dd)
    if cfg["tails"]:
        assert ((P["h"] > 0) & ~P["d"]).any(), "no tail rows in the batch"
    if dd.importance_weighted:
        assert float(P["isw"].min()) < 0.99 * float(P["isw"].max()), "IS weights all equal"
    rep = HC.Report(_id(case))
    HC.check_planes(rep, P, cfg)
    worst = rep.finish()[0]
    if cfg["kind"] == "cat":
        name, nt = "heads_kernel<%d,%d> in step" % (cfg["mode"], HC.cat_nt(cfg["N"])), HC.cat_nt(cfg["N"])
    elif cfg["kind"] == "mog":
        nt = HC.mog_nt(cfg["K"])
        name = "mog_heads_kernel<%d,%s> in step" % (nt, "true" if cfg["tails"] else "false")
    else:
        name, nt = "qr_heads_kernel<%d> in step" % HC.qr_nt(cfg["N"]), HC.qr_nt(cfg["N"])
    _record(name, nt, worst)
