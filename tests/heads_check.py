"""The three loss heads (categorical, mixture, quantile) against float64 restatements computed from the DEVICE's own fp32
inputs, each output held to a componentwise bound justified by the arithmetic the kernel does.

Categorical head (csrc/heads_dev.cuh).  One warp per row; lane owns atoms k = lane + 32 t, t < NT (NT = 2 for N <= 64,
4 above).  U = 2^-24 (half an fp32 ulp, relative); TREE = log2(32) = 5 levels of the warp_sum butterfly; every lane
also adds its NT terms in sequence (NT - 1 rounded adds).  A sum of terms t_i computed so is within
U (NT - 1 + TREE) sum |t_i| of the sum of the rounded terms.  The bounds below state, per output, the few ulps each term
picks up before the sum (the `c` of c U sum |terms|):

  probabilities  p_k = expf(x_k - mx) / s: the difference x_k - mx is rounded (|x_k - mx| U of e_k, the derivative of
                 exp), expf is within 2 ulp (4 U), s is a warp sum of the e_k, and the divide rounds (U):
                 |p - p64| <= U p_k (4 + |d_k| + sum_j e_j (4 + |d_j|) / s + NT - 1 + TREE + 1) + 4 2^-149
                 (the last term: an e_k in the subnormal range, where expf's 2 ulp are absolute)
  projection     mode 0: bit-exact against oracle/d4pg_oracle.py project_live (the same fp64 bins, the same ordered fp32
                 adds); mode 1: the kernel sums in fp64 and rounds once, so at most 1 ulp of the float64 sum
                 (tests/nstep_tails_oracle.py project_disc, whose adds go in another order)
  CE loss row    -isw sum m_k log(q_k + 1e-10f): the add rounds (U m_k after log), logf is within 1 ulp (2 U |log|), the
                 product rounds (U): c = 3 + NT - 1 + TREE per term |m_k log q_k|, plus U sum m_k and the final * isw
  td             -sum m_k q_k: c = 1 + NT - 1 + TREE
  priority       |td| + eps or (ce_priority) -ce + eps: the bound of td or ce plus one rounded add
  logit grad     gq_k = -(m_k / (q_k + 1e-10f)) * f32(grad_scale * isw): four roundings (4 U); sq = sum q_k gq_k:
                 c = 4 + 1 + NT - 1 + TREE; dq_k = q_k (gq_k - sq): two more roundings.  So
                 |dq - ref| <= U |q_k| (6 |gq_k| + (NT + 11) sum_j |q_j gq_j|)
  policy         E_q[z] over the fp32 atoms z_k = f32(v_min + k delta): c = 1 + NT - 1 + TREE, and the gradient
                 -(gs q_k) (z_k - E) three roundings; both carry the error of the policy softmax they start from.

Where an fp32 product or partial sum falls in the subnormal range its rounding is absolute, up to 2^-150: every sum
bound also carries (N + 8) 2^-149 (and the policy gradient, whose subnormal product is scaled by |z - E|, 2^-149 (|z - E|
+ 2)).  Rewards at or past v_max put b = (v_max - v_min) / delta, which may round past N - 1 (e.g. [-50, 0] with 32 or
63 atoms): kernel and oracles clip returns at the largest double whose b is at most N - 1 there
(oracle/d4pg_oracle.py atom_clip_top).

Each stage is checked twice: from the device's own softmax outputs and projected row (`iso`, isolating the stage, as
the bound is stated) and end to end from the logits (`e2e`: the float64 softmax and projection, with the probability
bounds carried through the stage to first order, x 1.01).

Mixture and quantile heads (csrc/mog_heads.cu, csrc/qr_heads.cu) evaluate the whole row in fp64 from the fp32 inputs
and round each output once; fp64 evaluation error is ~1e-16 relative.  The bound is C_FP64 = 4 U (two fp32 ulps) of
the row's scale: sum |omega log p| for a mixture loss row, the loss row itself for a quantile row (its terms are all
>= 0), |E[Q]| + |r| + c |E[Q']| in absolute terms for td, and the row's largest |g| for a gradient row.  The references
are tests/mog_oracle.py heads and tests/qr_oracle.py heads.
"""
import math

import numpy as np
import torch

from oracle import d4pg_oracle as O
from tests import mog_oracle as MO
from tests import nstep_tails_oracle as NTO
from tests import qr_oracle as QO
from tests.step_check import POWER_MIN, Report, ratio  # noqa: F401  (re-exported for the tests)

F32, F64 = np.float32, np.float64
U = 2.0 ** -24
TREE = 5
C_EXP = 4.0
C_FP64 = 4.0
EPS10 = float(F32(1e-10))             # the kernel's 1e-10f, as the reference's fp32 q + 1e-10 rounds it
TINY = 4 * 2.0 ** -149
SUB = 2.0 ** -149                     # an fp32 result in the subnormal range: each rounding is absolute, <= SUB / 2
PROP = 1.01                           # first-order propagation of the probability bounds: second-order margin


# ---- which instantiation a width selects (the launchers' dispatch) -----------------------------------------------------
def cat_nt(N):
    return 2 if N <= 64 else 4


def mog_nt(K):
    return 1 if K <= 4 else 2 if K <= 8 else 4 if K <= 16 else 8


def qr_nt(N):
    return -(-N // 32)


def t64(x):
    return torch.as_tensor(np.asarray(x)).double()


def ulp_ratio(dev, ref):
    """max |dev - ref| in fp32 ulps of the reference's fp32 rounding (mode-1 projection: at most 1)."""
    ref = np.asarray(ref, dtype=F64)
    sp = np.spacing(np.abs(ref).astype(F32)).astype(F64)
    err = np.abs(np.asarray(dev, dtype=F64) - ref)
    return float(np.max(err / sp)) if err.size else 0.0


# ---- categorical ---------------------------------------------------------------------------------------------------------
def softmax_bound(x, NT, is_probs=False):
    """fp32 row x [B, N] (float64 tensor) -> (float64 softmax, bound of the kernel's fp32 softmax); probs: x itself."""
    x = x.double()
    if is_probs:
        return x, torch.zeros_like(x)
    mx = x.max(1, keepdim=True).values
    d = x - mx
    e = torch.exp(d)
    s = e.sum(1, keepdim=True)
    p = e / s
    rel = C_EXP + d.abs()
    srel = (e * rel).sum(1, keepdim=True) / s + (NT - 1) + TREE
    return p, (U * p * (rel + srel + 1) + TINY) * (1 + 1e-6)


def _b(r, d, v_min, v_max, N, disc):
    delta, centers = O.atom_support(v_min, v_max, N)
    tz = np.minimum(O.atom_clip_top(v_min, v_max, N),
                    np.maximum(v_min, np.asarray(r, F64).reshape(-1, 1) + disc * (1 - np.asarray(d, F64).reshape(-1, 1))
                               * centers.reshape(1, -1)))
    return (tz - v_min) / delta


def project(p, r, d, v_min, v_max, N, disc, mode, drop_integral=False):
    """The projection in float64 of the fp32 (or float64) probabilities p: mode 0 is project_live's arithmetic on
    float64 masses (non-terminal rows: the same bins and weights as the per-row-discount mode-1 projection; terminal
    rows: the Dirac at clip(r), independent of p); mode 1 is project_disc.  drop_integral: the mode-1 mutant without the
    l -= 1 / u += 1 adjustment (an atom whose b_j is an integer gets weight u - b = b - l = 0)."""
    p = np.asarray(p, F64)
    d = np.asarray(d).astype(bool)
    disc = np.broadcast_to(np.asarray(disc, F64).reshape(-1, 1), (p.shape[0], 1))
    if drop_integral:
        b = _b(r, d, v_min, v_max, N, disc)
        p = np.where(np.floor(b) == np.ceil(b), 0.0, p)
    if mode == 1:
        return NTO.project_disc(p, r, d, v_min, v_max, N, disc)
    m, l, u = NTO.project_disc(p, r, np.zeros_like(d), v_min, v_max, N, disc)
    if d.any():
        live = O.project_live(np.zeros((int(d.sum()), N), F32), np.asarray(r, F64)[d], d[d], v_min, v_max, N,
                              float(disc[0, 0]))
        m[d] = live
    return m, l, u


def project_bound(p, tolp, r, d, v_min, v_max, N, disc, mode):
    """(float64 projection of p, bound of the device's projection of its own softmax whose error is within tolp)."""
    m, l, u = project(p, r, d, v_min, v_max, N, disc, mode)
    tm = project(tolp, r, d, v_min, v_max, N, disc, mode)[0]
    dd = np.asarray(d).astype(bool)
    if mode == 0:
        tm[dd] = 0.0                                   # the Dirac of a terminal row does not depend on p
        cnt = np.zeros(m.size)
        off = (np.arange(m.shape[0]) * N).reshape(-1, 1)
        np.add.at(cnt, (l + off).reshape(-1), 1.0)
        np.add.at(cnt, (u + off).reshape(-1), 1.0)
        tm = tm * PROP + cnt.reshape(m.shape) * (U * m + SUB)  # one rounded fp32 add per contribution
    else:
        tm = tm * PROP + 2 * U * m + SUB
    return t64(m), t64(tm)


def cat_loss(m, q, isw, gs, NT, prio_eps=1e-6, ce_priority=False, tolm=None, tolq=None, eps=EPS10):
    """{output: (float64 reference, bound)} of the CE / td / priority / logit-gradient stage from m and q [B, N]
    (the device's own, or float64 ones whose error is within tolm / tolq).  isw [B] (ones without IS weights)."""
    m, q = m.double(), q.double()
    floor = (q.shape[1] + 8) * SUB                   # products and partial sums that underflow fp32
    isw = t64(isw).reshape(-1)
    gsc = float(F32(gs)) * isw                       # f32 grad_scale times the f32 weight, in float64
    qe = q + eps
    lq = torch.log(qe)
    t = m * lq
    ce = t.sum(1)
    tol_ce = U * ((3 + NT - 1 + TREE) * t.abs().sum(1) + m.abs().sum(1)) + floor
    mq = m * q
    td = -mq.sum(1)
    tol_td = U * (NT + TREE) * mq.abs().sum(1) + floor
    gq = -(m / qe) * gsc.view(-1, 1)
    qg = q * gq
    sq = qg.sum(1, keepdim=True)
    dq = q * (gq - sq)
    tol_dq = U * q.abs() * (6 * gq.abs() + (NT + 11) * qg.abs().sum(1, keepdim=True)) + floor
    if tolm is not None:                             # first-order propagation of the input errors
        tolm, tolq = tolm.double(), tolq.double()
        tol_ce = tol_ce + PROP * (lq.abs() * tolm + m.abs() * tolq / qe).sum(1)
        tol_td = tol_td + PROP * (q.abs() * tolm + m.abs() * tolq).sum(1)
        dgq = gsc.view(-1, 1).abs() * (tolm / qe + m.abs() * tolq / qe ** 2)
        dsq = (gq.abs() * tolq + q.abs() * dgq).sum(1, keepdim=True)
        tol_dq = tol_dq + PROP * (tolq * (gq - sq).abs() + q.abs() * (dgq + dsq))
    pe = float(F32(prio_eps))
    rows = -ce * isw
    prio = (-ce if ce_priority else td.abs()) + pe
    tol_prio = (tol_ce if ce_priority else tol_td) + U * prio.abs()
    return {"loss_rows": (rows, tol_ce * isw + U * rows.abs()), "td": (td, tol_td), "prio": (prio, tol_prio),
            "dq": (dq, tol_dq)}


def policy_bound(pl, z32, gs, NT):
    """{pi_rows, dpi: (float64 reference, bound)} of the categorical policy head from the fp32 logits pl."""
    qp, tq = softmax_bound(pl, NT)
    z = t64(z32).view(1, -1)
    ez = (qp * z).sum(1)
    tol_ez = PROP * (tq * z.abs()).sum(1) + U * (NT + TREE) * (qp * z).abs().sum(1) + (z.shape[1] + 8) * SUB
    g = float(F32(gs))
    dz = z - ez.view(-1, 1)
    dpi = -g * qp * dz
    tol_dpi = g * (PROP * (tq * dz.abs() + qp * tol_ez.view(-1, 1))) + 3 * U * dpi.abs() + SUB * (dz.abs() + 2)
    return {"pi_rows": (-ez, tol_ez), "dpi": (dpi, tol_dpi)}


def cat_refs(tl, ql, pl, r, d, v_min, v_max, disc, mode, flags=0, isw=None, gs=1.0, prio_eps=1e-6, ce_priority=False,
             tp=None, qp=None, m=None, eps=EPS10):
    """Every (name, reference, bound) of the categorical head.  tp / qp / m: the device's softmax outputs and projected
    row (the `iso` stage); without them only the end-to-end checks."""
    B, N = tl.shape
    NT = cat_nt(N)
    isw = np.ones(B) if isw is None else isw
    disc = np.broadcast_to(np.asarray(disc, F64).reshape(-1, 1), (B, 1))
    p64, tolp = softmax_bound(tl, NT, bool(flags & 1))
    q64, tolq = softmax_bound(ql, NT, bool(flags & 2))
    out = [("tp", p64, tolp), ("qp", q64, tolq)]
    m64, tolm = project_bound(p64.numpy(), tolp.numpy(), r, d, v_min, v_max, N, disc, mode)
    out.append(("m e2e", m64, tolm))
    kw = dict(prio_eps=prio_eps, ce_priority=ce_priority, eps=eps)
    for k, (ref, tol) in cat_loss(m64, q64, isw, gs, NT, tolm=tolm, tolq=tolq, **kw).items():
        out.append((k + " e2e", ref, tol))
    if tp is not None:
        for k, (ref, tol) in cat_loss(m, qp, isw, gs, NT, **kw).items():
            out.append((k, ref, tol))
    if pl is not None:
        z32 = O.atom_support(v_min, v_max, N)[1].astype(F32)
        for k, (ref, tol) in policy_bound(pl, z32, gs, NT).items():
            out.append((k, ref, tol))
    return out


def cat_check(rep, inp, dev, v_min, v_max, disc, mode, flags=0, isw=None, gs=1.0, prio_eps=1e-6, ce_priority=False,
              bins=None, eps=EPS10):
    """Every output of the categorical head in `dev` ({name: fp32 tensor [B, N] / [B]}) against its bound; inp: tl, ql,
    pl (None: no policy head), r, d.  The projection checks: mode 0 bit-exact against project_live of the device's own
    target probabilities (and its bins), mode 1 within 1 ulp of project_disc of them (and its bins)."""
    tl, ql, pl, r, d = inp["tl"], inp["ql"], inp.get("pl"), inp["r"], inp["d"]
    B, N = tl.shape
    disc = np.broadcast_to(np.asarray(disc, F64).reshape(-1, 1), (B, 1))
    tp = dev["tp"].double() if "tp" in dev else None
    qp = dev["qp"].double() if "qp" in dev else None
    m = dev["m"].double() if "m" in dev else None
    if "tp" in dev and "m" in dev:
        tp32 = dev["tp"].numpy().astype(F32)
        if mode == 0:
            mo, bl, bu = O.project_live(tp32, r, d, v_min, v_max, N, float(disc[0, 0]), return_bins=True)
            rep.add("m", 0.0 if np.array_equal(dev["m"].numpy(), mo) else math.inf)
        else:
            mo, bl, bu = NTO.project_disc(tp32, r, d, v_min, v_max, N, disc)
            rep.add("m (ulps)", ulp_ratio(dev["m"].numpy(), mo))
        if bins is not None:
            rep.add("bins", 0.0 if np.array_equal(bins[0], bl) and np.array_equal(bins[1], bu) else math.inf)
    for name, ref, tol in cat_refs(tl, ql, pl, r, d, v_min, v_max, disc, mode, flags, isw, gs, prio_eps, ce_priority,
                                   tp, qp, m if (tp is not None and qp is not None and m is not None) else None, eps):
        key = name.split(" ")[0]
        if key not in dev or (name in ("loss_rows", "td", "prio", "dq") and (qp is None or m is None)):
            continue
        rep.add(name, ratio(dev[key], ref, tol))


# ---- mixture -------------------------------------------------------------------------------------------------------------
def _groups(disc, chunk=512):
    """(discount, rows) of every group of rows that share a discount, at most `chunk` rows at a time (the oracles'
    per-row autograd graphs stay small at 4097 rows)."""
    disc = np.asarray(disc, F64).reshape(-1)
    for c in np.unique(disc):
        sel = np.nonzero(disc == c)[0]
        for i in range(0, len(sel), chunk):
            yield float(c), sel[i:i + chunk]


def mog_refs(tr, q, pi, r, d, K, disc, isw, gs, prio_eps=1e-6):
    """{output: (float64 reference, bound)} of the mixture head from the fp32 raw rows tr, q, pi [B, 3K] (pi None: no
    policy part); disc [B] the discount of each row (gamma, gamma^n or gamma^h)."""
    B = tr.shape[0]
    isw = t64(isw).reshape(-1)
    g = float(F32(gs))
    ref = {k: torch.zeros(B, dtype=torch.float64) for k in ("loss_rows", "td", "prio", "pi_rows", "loss_scale", "td_scale")}
    ref.update(dq=torch.zeros(B, 3 * K, dtype=torch.float64), dpi=torch.zeros(B, 3 * K, dtype=torch.float64))
    r, d = np.asarray(r, F64).reshape(-1), np.asarray(d).astype(bool).reshape(-1)
    for c, sel in _groups(np.broadcast_to(np.asarray(disc, F64).reshape(-1), (B,))):
        o = MO.heads(tr[sel], q[sel], None if pi is None else pi[sel], r[sel], d[sel], c, K, g, prio_eps)
        for k, k2 in (("loss_rows", "loss_rows"), ("td", "td"), ("dq", "dq_raw"), ("pi_rows", "pi_rows"), ("dpi", "dpi_raw")):
            if k2 in o:
                ref[k][sel] = o[k2]
        y, om = MO.target_points(tr[sel], r[sel], d[sel], c, K)
        ref["loss_scale"][sel] = (om * MO.log_density(y, *MO.head(q[sel].double(), K))).abs().sum(1)
        w, mu, _ = MO.head(q[sel].double(), K)
        tw, tmu, _ = MO.head(tr[sel].double(), K)
        cc = c * (1.0 - torch.as_tensor(d[sel], dtype=torch.float64))
        ref["td_scale"][sel] = (w * mu).abs().sum(1) + torch.as_tensor(np.abs(r[sel])) + cc * (tw * tmu).abs().sum(1)
    pe = float(F32(prio_eps))
    out = {"loss_rows": (ref["loss_rows"] * isw, C_FP64 * U * ref["loss_scale"] * isw),
           "td": (ref["td"], C_FP64 * U * ref["td_scale"]),
           "prio": (ref["td"].abs() + pe, C_FP64 * U * ref["td_scale"] + U * (ref["td"].abs() + pe)),
           "dq": (ref["dq"] * isw.view(-1, 1), C_FP64 * U * (ref["dq"] * isw.view(-1, 1)).abs().amax(1, keepdim=True)
                  .expand(B, 3 * K))}
    if pi is not None:
        w, mu, _ = MO.head(pi.double(), K)
        out["pi_rows"] = (ref["pi_rows"], C_FP64 * U * (w * mu).abs().sum(1))
        out["dpi"] = (ref["dpi"], C_FP64 * U * ref["dpi"].abs().amax(1, keepdim=True).expand(B, 3 * K))
    return out


# ---- quantile ------------------------------------------------------------------------------------------------------------
def qr_refs(tq, q, pi, r, d, disc, kappa, isw, gs, prio_eps=1e-6, ce_priority=False):
    """{output: (float64 reference, bound)} of the quantile head from the fp32 rows tq, q, pi [B, N]."""
    B, N = tq.shape
    isw = t64(isw).reshape(-1)
    g = float(F32(gs))
    ref = {k: torch.zeros(B, dtype=torch.float64) for k in ("loss_rows", "td", "prio", "pi_rows")}
    ref.update(dq=torch.zeros(B, N, dtype=torch.float64), dpi=torch.zeros(B, N, dtype=torch.float64))
    r, d = np.asarray(r, F64).reshape(-1), np.asarray(d).astype(bool).reshape(-1)
    cs = torch.zeros(B, dtype=torch.float64)
    for c, sel in _groups(np.broadcast_to(np.asarray(disc, F64).reshape(-1), (B,))):
        o = QO.heads(tq[sel], q[sel], None if pi is None else pi[sel], r[sel], d[sel], c, kappa, g, prio_eps, ce_priority)
        for k in ("loss_rows", "td", "prio", "dq", "pi_rows", "dpi"):
            if k in o:
                ref[k][sel] = o[k]
        cs[sel] = c * (1.0 - torch.as_tensor(d[sel], dtype=torch.float64))
    td_scale = q.double().abs().mean(1) + torch.as_tensor(np.abs(r)) + cs * tq.double().abs().mean(1)
    loss = ref["loss_rows"]
    out = {"loss_rows": (loss * isw, C_FP64 * U * loss * isw),
           "td": (ref["td"], C_FP64 * U * td_scale),
           "prio": (ref["prio"], (C_FP64 * U * (loss if ce_priority else td_scale)) + U * ref["prio"].abs()),
           "dq": (ref["dq"] * isw.view(-1, 1), C_FP64 * U * (ref["dq"] * isw.view(-1, 1)).abs().amax(1, keepdim=True)
                  .expand(B, N))}
    if pi is not None:
        out["pi_rows"] = (ref["pi_rows"], C_FP64 * U * pi.double().abs().mean(1))
        out["dpi"] = (ref["dpi"], C_FP64 * U * ref["dpi"].abs())
    return out


def check_refs(rep, refs, dev, prefix=""):
    for k, (ref, tol) in refs.items():
        if k in dev:
            rep.add(prefix + k, ratio(dev[k], ref, tol))


# ---- fixtures (shared by the GPU sweeps and the CPU mutant tests) ------------------------------------------------------
def cat_fixture(N, B, variant, seed=0):
    """Inputs of one d4pg_proj_loss call: (inp, v_min, v_max, discount, flags).  Rows cycle through patterns, so that
    B = 1..5 each start on a different one and 4097 has them all:
      variant "wide": support [-50, 0], logits N(0, 3^2) / spread over +-80 (some q underflow to 0: the 1e-10 decides
                      dq) / all equal; rewards inside, beyond v_max, below v_min; terminals with non-integral b
      variant "exact": delta = 1 on [-(N-1), 0], gamma 0.5, integer rewards: b_j lands on atoms; integral terminals
      variant "gamma0": every atom of a row maps to one bin;  variant "probs": both inputs already probabilities."""
    rng = np.random.RandomState(seed * 1009 + N * 7 + B)
    i = np.arange(B) + seed
    if variant == "exact":
        v_min, v_max, disc = -float(N - 1), 0.0, 0.5
    else:
        v_min, v_max, disc = -50.0, 0.0, (0.0 if variant == "gamma0" else 0.99)

    def logits():
        x = rng.randn(B, N) * 3
        x[i % 4 == 1] = rng.uniform(-80, 80, (int((i % 4 == 1).sum()), N))
        x[i % 4 == 2] = 0.7
        return x.astype(F32)
    tl, ql, pl = logits(), logits(), logits()
    pat = i % 5
    if variant == "exact":
        r = -rng.randint(0, N + 3, B).astype(F64)
        r[pat == 3] = 4.0                                              # beyond v_max
    else:
        r = rng.uniform(v_min, v_max, B)
        r[pat == 3] = v_max + 5.0
        r[pat == 4] = v_min - 30.0
    d = (i % 3 == 2)
    flags = 3 if variant == "probs" else 0
    if flags:
        tl = torch.softmax(torch.from_numpy(tl), 1).numpy()
        ql = torch.softmax(torch.from_numpy(ql), 1).numpy()
    return dict(tl=t64(tl), ql=t64(ql), pl=t64(pl), r=r, d=d), v_min, v_max, disc, flags


CAT_VARIANTS = ("wide", "exact", "gamma0", "probs")


def mog_fixture(K, B, variant, seed=0):
    """Inputs of one d4pg_mog_loss call: (inp, discount).  Row patterns: random mixtures; sigma raw exactly 20, the next
    float above 20 and -30 (the 1e-3 floor); targets ~1e6 online sigmas from every online component (the logsumexp
    path); and `points`: a target component with sigma raw exactly 20 whose 8 quadrature points each carry an online
    component of floor sigma placed on it (to fp32), so that the online mean gradients see y to ~1e-9 and the softplus
    branch at 20 is visible.  variant "disc0": discount 0; every third row is terminal."""
    rng = np.random.RandomState(seed * 1013 + K * 11 + B)
    i = np.arange(B) + seed
    disc = 0.0 if variant == "disc0" else 0.99
    tr = np.concatenate([rng.randn(B, K), rng.randn(B, K) * 3, rng.randn(B, K)], 1)
    q = np.concatenate([rng.randn(B, K), rng.randn(B, K) * 3, rng.randn(B, K)], 1)
    pi = np.concatenate([rng.randn(B, K), rng.randn(B, K) * 3, rng.randn(B, K)], 1)
    r = -3 * rng.rand(B)
    d = (i % 3 == 2)
    pat = i % 5
    s20, s20n = 20.0, float(np.nextafter(F32(20), F32(np.inf)))
    for row in np.nonzero(pat == 1)[0]:
        tr[row, 2 * K:] = np.resize([s20, s20n, -30.0], K)
        q[row, 2 * K:] = np.resize([-30.0, s20, s20n], K)
    for row in np.nonzero(pat == 2)[0]:                                # far targets, online sigmas at the floor
        tr[row, K:2 * K] = 1e3
        q[row, 2 * K:] = -30.0
    for row in np.nonzero(pat == 3)[0]:
        tr[row, :K] = -200.0
        tr[row, 0], tr[row, K], tr[row, 2 * K] = 0.0, 0.0, s20
        c = 0.0 if d[row] else disc
        sig = math.log1p(math.exp(20.0)) + 1e-3
        for j in range(K):
            if j < MO.Q:
                q[row, j] = math.log(MO.HW[j])
                q[row, K + j] = F32(r[row] + c * (math.sqrt(2.0) * sig * MO.X[j]))
            else:
                q[row, j], q[row, K + j] = -5.0, 1e3
            q[row, 2 * K + j] = -30.0
    return dict(tr=t64(tr.astype(F32)), q=t64(q.astype(F32)), pi=t64(pi.astype(F32)), r=r, d=d), disc


MOG_VARIANTS = ("plain", "disc0")


def qr_fixture(N, B, kappa, seed=0):
    """Inputs of one d4pg_qr_loss call: (inp, discount).  Row patterns: random quantiles; ties: target quantiles 0 and
    r in {0, kappa, -kappa} against online quantiles half of them 0, so that some u = y - theta are exactly 0 and exactly
    +-kappa (whatever the discount); terminal rows; discount 0.99, or 0 on every fourth call (seed)."""
    rng = np.random.RandomState(seed * 1019 + N * 13 + B)
    i = np.arange(B) + seed
    disc = 0.0 if seed % 4 == 3 else 0.99
    tq = rng.randn(B, N) * 2
    q = rng.randn(B, N) * 2
    pi = rng.randn(B, N) * 2
    r = -3 * rng.rand(B)
    d = (i % 3 == 2)
    pat = i % 4
    for row in np.nonzero(pat == 1)[0]:
        tq[row] = 0.0
        q[row, ::2] = 0.0
        r[row] = [0.0, kappa, -kappa][row % 3]
        d[row] = False
    return dict(tq=t64(tq.astype(F32)), q=t64(q.astype(F32)), pi=t64(pi.astype(F32)), r=r, d=d), disc


# ---- the heads inside the learner step ----------------------------------------------------------------------------------
def step_planes(dd):
    """The heads' inputs and outputs of the step `dd` just ran, read through the learner's tensors: planes at pitch Np.
    The IS weights are `dd._learner.weights`: without a pipeline (prefetch=False) the learner samples straight into the
    caller's buffers (csrc/learner.cu, d4pg_learner_create: batch[0].wts = buf->weights), and head_common hands that
    plane to the loss kernel when importance_weighted is set on a prioritized replay (a uniform replay's rows all weigh
    1; the sampler writes no weights there)."""
    L = dd._learner
    B = dd.batch_size
    T = lambda n, dt=torch.float32: L.tensor(n, dt).cpu()
    P = {k: T(k) for k in ("target_logits", "q_logits", "pi_logits", "m", "target_probs", "q_probs", "dlogits_q",
                           "dlogits_pi")}
    P.update(r=T("r", torch.float64).numpy()[:B], d=T("done", torch.uint8).numpy()[:B].astype(bool),
             h=T("h", torch.uint8).numpy()[:B] if dd.nstep_tails else np.zeros(B, np.uint8),
             loss_rows=T("loss_rows")[:B], pi_rows=T("pi_rows")[:B], td=L.td.cpu(), prio=L.prio.cpu(),
             losses=L.losses.cpu(),
             isw=L.weights.cpu().numpy() if dd.importance_weighted and dd.prioritized_replay else np.ones(B))
    return P


def step_config(dd):
    kind = {"categorical": "cat", "mixture_of_gaussian": "mog", "quantile": "qr"}[dd.dist_type]
    mode = 1 if dd.projection == "nstep" else 0
    return dict(kind=kind, N=dd.n_atoms, K=dd.n_components, v_min=dd.v_min, v_max=dd.v_max, gamma=dd.gamma,
                n_steps=dd.n_steps, mode=mode, tails=bool(dd.nstep_tails), kappa=dd.qr_kappa, B=dd.batch_size,
                gs=float(F32(1.0) / F32(dd.batch_size)), ce=dd.priority == "ce",
                # a uniform replay's learner computes its (unused) priorities with eps 1e-6
                prio_eps=dd.prioritized_replay_eps if dd.prioritized_replay else 1e-6)


def step_discounts(cfg, h):
    """The learner's discount of each row: gamma (live projection), gamma^n, or gamma^h for a tail row (the gtab)."""
    B = len(h)
    if cfg["mode"] == 0:
        return np.full(B, cfg["gamma"])
    if cfg["tails"]:
        return NTO.row_discounts(h, cfg["gamma"], cfg["n_steps"]).reshape(-1)
    return np.full(B, cfg["gamma"] ** cfg["n_steps"])


def check_planes(rep, P, cfg, disc=None):
    """Every output of the step's loss head in P (step_planes) against its bound, restated with the learner's own
    discount of each row; the pad columns [N, Np) of every head plane exactly zero; the two reported batch-mean losses
    against the device's own rows (a fixed-order fp32 sum of at most ceil(B / 256) + 5 + 8 adds, times 1/B)."""
    N, B = cfg["N"], cfg["B"]
    disc = step_discounts(cfg, P["h"]) if disc is None else disc
    sl = lambda k: P[k][:B, :N].double()
    inp = dict(tl=sl("target_logits"), ql=sl("q_logits"), pl=sl("pi_logits"), r=P["r"], d=P["d"])
    dev = dict(loss_rows=P["loss_rows"], td=P["td"], prio=P["prio"], dq=P["dlogits_q"][:B, :N], pi_rows=P["pi_rows"],
               dpi=P["dlogits_pi"][:B, :N])
    if cfg["kind"] == "cat":
        dev.update(m=P["m"][:B, :N], tp=P["target_probs"][:B, :N], qp=P["q_probs"][:B, :N])
        assert cfg["mode"] == 1 or len(np.unique(disc)) == 1
        cat_check(rep, inp, dev, cfg["v_min"], cfg["v_max"], disc if cfg["mode"] else float(disc[0]), cfg["mode"], 0,
                  P["isw"], cfg["gs"], cfg["prio_eps"], cfg["ce"])
        pads = ("m", "target_probs", "q_probs", "dlogits_q", "dlogits_pi")
    elif cfg["kind"] == "mog":
        check_refs(rep, mog_refs(inp["tl"], inp["ql"], inp["pl"], P["r"], P["d"], cfg["K"], disc, P["isw"], cfg["gs"],
                                 cfg["prio_eps"]), dev)
        pads = ("dlogits_q", "dlogits_pi")
    else:
        check_refs(rep, qr_refs(inp["tl"], inp["ql"], inp["pl"], P["r"], P["d"], disc, cfg["kappa"], P["isw"], cfg["gs"],
                                cfg["prio_eps"], cfg["ce"]), dev)
        pads = ("dlogits_q", "dlogits_pi")
    for k in pads:
        rep.add("pad " + k, 0.0 if bool((P[k][:B, N:] == 0).all()) else math.inf)
    n = -(-B // 256) + TREE + 8 + 2
    for i, k in enumerate(("loss_rows", "pi_rows")):
        x = P[k].double()
        rep.add("losses[%d]" % i, ratio(P["losses"][i:i + 1], x.mean().view(1), (n * U * x.abs().sum() / B).view(1)))
