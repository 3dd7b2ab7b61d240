"""The actor and critic forward and backward entry points at every precision, layer by layer, against the teacher-forced
float64 restatement and componentwise bound of tests/step_check.py (`LayerCheck` on the level plan's `MODES` rows:
these entry points run the level GEMMs), at the level kernels' tile, split-K and unpadded-operand edges.

The entry points take the caller's rows at pitch |s| / |a| from wherever they start, so they reach staging paths the
learner's 16-B pitched planes never do: the scalar staging of gemm_ffma_dev.cuh, gemm_tc's thread-staged A operand
(no TMA) and gemm_bf16's scalar staging of the dW X operand.  The backward composes its own problems
(csrc/mlp_backward.cu): the critic's fc2 level is four of them, the head plane is pitch4(out) wide, the gradient buffer
is cleared first and split-K dW adds into it from batch 1024 on.

Each case calls the C ABI directly with its own buffers, every one of them filled with NaN first: an element a ragged
tile skips, or a gradient buffer the call did not clear, fails its check.  After the backward the scratch holds the
head's dZ plane, p1 = dz2 and p0 = dz1; dz22 is overwritten, so it is chained from the device's head plane and ReLU
mask (`chained_layer`, `stored`), as step_check chains p_dz22.  Then the same inputs go through the differentiable
modules and autograd, whose gradients must be the direct call's.

Tiles: gemm_ffma_dev.cuh BM = 32; gemm_tc.cu TC_BM = 128, TC_KC = 32; gemm_bf16.cu BF_BM = 128.  Split-K slices:
step_check.kslice (1024 rows: two of 512; 1025: three, the last of 257; 3585: eight, the last of one row).
"""
import itertools
import math
import time

import pytest
import torch

from tests import mog_oracle as MO
from tests import step_check as SC

H_ = 256
U = SC.U
PRECISIONS = {0: "fp32", 1: "tf32x3", 2: "tf32", 3: "bf16"}
# softmax_rows_kernel (csrc/abi.cu) against softmax of the device's own logits, relative to each probability, in units
# of 2^-24: expf is within 2 ulp (4 units) in the numerator and in every summand, the row sum of at most 128 positive
# terms takes at most 9 fp32 adds per term (4 per lane, then 5 butterfly levels), the division 1; and the fp32
# subtraction z - max z moves each exponent by |z - max z| units (added per element, below)
PROBS_UNITS = 18
# one fp32 rounding of a float64 value (half an ulp: at most 2^-24 of it), with room for the few float64 ulps by which
# the kernel's fp64 arithmetic and torch's may differ
ONE_ROUNDING = U * (1 + 2.0 ** -20)


def _cat(N):
    return {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": N}


def _mog(K):
    return {"type": "mixture_of_gaussian", "n_components": K}


def _qr(N):
    return {"type": "quantile", "n_quantiles": N}


# (|s|, |a|, critic head, B, s and a 4 B past a 16-B boundary); each comment names the edge
CASES = [
    (1, 1, _cat(2), 1, False),              # a single row, minimal widths
    (17, 6, _cat(51), 33, False),           # FFMA: 1-row last 32-row tile
    (17, 6, _cat(51), 129, False),          # wgmma / bf16: 1-row last 128-row tile
    (33, 6, _cat(7), 128, False),           # fc1 K one column into a second TC K chunk; N = 7 (pitch 8)
    (376, 17, _cat(101), 1023, False),      # the largest unsplit dW; s rows 16-B pitched (vector / TMA staging)
    (376, 16, _cat(101), 1023, True),       # the same widths on the scalar / thread-staged path
    (376, 16, _cat(101), 1025, True),       # scalar staging inside split-K
    (17, 6, _cat(51), 1024, False),         # the first split-K batch: two even slices
    (17, 6, _cat(128), 1025, False),        # three slices, the last of 257 rows; max atoms
    (17, 33, _cat(101), 3585, False),       # eight slices, the last of one row
    (2053, 6, _cat(51), 1025, False),       # fc1 dW 2053 wide, K_in not a multiple of 4, split-K
    (17, 257, _cat(51), 64, False),         # actor head plane wider than 256 (pitch 260)
    (576, 256, _cat(64), 512, False),       # the widest action: vector staging of a
    (17, 6, _mog(1), 129, False),           # mixture, 3-column raw head
    (17, 6, _mog(32), 1025, False),         # mixture, 96-column raw head, split-K
    (17, 6, _qr(2), 33, False),             # the narrowest theta
    (376, 17, _qr(128), 1025, False),       # the widest theta, split-K
    (17, 6, _cat(51), 256, False),          # config 2 widths
    (376, 17, _cat(101), 200, False),       # ragged 128-row tile, |s| not a multiple of 32
    (3, 1, _cat(51), 64, False),
    (17, 6, _cat(101), 4096, False),        # config 5 widths, eight slices of 512
]


def _id(case):
    S, A, info, B, mis = case
    head = {"categorical": "N%d" % info.get("n_atoms", 0), "mixture_of_gaussian": "mogK%d" % info.get("n_components", 0),
            "quantile": "qr%d" % info.get("n_quantiles", 0)}[info["type"]]
    return "s%d-a%d-%s-B%d%s" % (S, A, head, B, "-misaligned" if mis else "")


def _pitch4(x):
    return (x + 3) & ~3


def _nan(*shape):
    return torch.full(shape, math.nan, dtype=torch.float32, device="cuda")


def _place(x, misaligned, grad=False):
    """x copied into a flat device buffer at float offset 1 (4 B past a 16-B boundary) or 0: (the [B, w] view, the flat
    buffer, a leaf when grad)."""
    off = 1 if misaligned else 0
    flat = torch.zeros(off + x.numel() + 3, device="cuda")
    flat[off:off + x.numel()] = x.flatten().cuda()
    if grad:
        flat.requires_grad_(True)
    view = flat[off:off + x.numel()].view(x.shape)
    assert view.data_ptr() % 16 == 4 * off
    return view, flat


class _Ctx:
    """One case: the two modules (the constructors' seeded initialisation), the inputs and the upstream gradients."""

    def __init__(self, d4pg, S, A, info, B, misaligned, precision, seed=31):
        self.d4pg, self.S, self.A, self.info, self.B, self.mis, self.precision = d4pg, S, A, info, B, misaligned, precision
        torch.manual_seed(seed)
        self.actor = d4pg.actor(S, A, device="cuda")
        self.critic = d4pg.critic(S, A, info, device="cuda")
        self.kind = info["type"]
        self.N = self.critic.n_atoms                                    # the raw head's width (3K for the mixture)
        g = torch.Generator().manual_seed(seed + B)
        self.s0, self.a0 = torch.randn(B, S, generator=g), torch.rand(B, A, generator=g) * 2 - 1
        self.s, _ = _place(self.s0, misaligned)
        self.a, _ = _place(self.a0, misaligned)
        # upstream gradients N(0, 1) / B, what a batch-mean loss hands the outputs
        up = lambda n: (torch.randn(B, n, generator=g) / B).cuda()
        self.g_action = up(A)
        K = self.N // 3
        self.g_head = {"categorical": (up(self.N), up(self.N)), "mixture_of_gaussian": (up(K), up(K), up(K)),
                       "quantile": (up(self.N),)}[self.kind]


def _lib():
    from d4pg_b200 import _lib
    return _lib


def _views(net, flat):
    return {n + k: v for n, wb in zip(("fc1", "fc2", "fc2_2", "fc3"), net._views(flat)) for k, v in zip((".weight", ".bias"), wb)}


def _pads_zero(net, G):
    """Every float of the flat gradient buffer outside the parameter views (row-pitch columns, alignment gaps) is 0."""
    pad = torch.ones(G.numel(), dtype=torch.bool, device=G.device)
    for v in _views(net, pad).values():
        v.fill_(False)
    return 0.0 if bool((G[pad] == 0).all()) else math.inf


def _weights(net):
    return {k: v.detach().clone() for k, v in net.state_dict().items()}


# ---- direct calls ------------------------------------------------------------------------------------------------------
def _actor_forward(c):
    L = _lib()
    B = c.B
    out, ws = _nan(B, c.A), _nan(3 * B * H_)
    L.check(L.lib().d4pg_actor_forward(L.ptr(c.actor.flat_params()), c.S, c.A, L.ptr(c.s), B, L.ptr(out), L.ptr(ws),
                                       c.precision, L.stream_ptr()), "d4pg_actor_forward")
    return out, ws


def _actor_backward(c, out, ws):
    L = _lib()
    B = c.B
    G, gs = _nan(c.actor._total), _nan(B, c.S)
    scratch = _nan(B * (2 * H_ + max(H_, _pitch4(c.A))))
    L.check(L.lib().d4pg_actor_backward(L.ptr(c.actor.flat_params()), c.S, c.A, L.ptr(c.s), B, L.ptr(out), L.ptr(ws),
                                        L.ptr(c.g_action), L.ptr(G), L.ptr(gs), L.ptr(scratch), c.precision,
                                        L.stream_ptr()), "d4pg_actor_backward")
    return G, gs, scratch


def _critic_forward(c, logits=True):
    """-> (outputs by name, workspace); the categorical critic without a logits buffer when not `logits`."""
    L = _lib()
    B, net, P = c.B, c.critic, L.ptr
    ws = _nan(3 * B * H_)
    st = L.stream_ptr()
    if c.kind == "mixture_of_gaussian":
        K = net.n_components
        out = {"w": _nan(B, K), "mu": _nan(B, K), "sigma": _nan(B, K), "raw": _nan(B, c.N)}
        L.check(L.lib().d4pg_critic_forward_mog(P(net.flat_params()), c.S, c.A, K, P(c.s), P(c.a), B, P(out["w"]),
                                                P(out["mu"]), P(out["sigma"]), P(out["raw"]), P(ws), c.precision, st),
                "d4pg_critic_forward_mog")
    elif c.kind == "quantile":
        out = {"theta": _nan(B, c.N)}
        L.check(L.lib().d4pg_critic_forward(P(net.flat_params()), c.S, c.A, c.N, P(c.s), P(c.a), B, None,
                                            P(out["theta"]), P(ws), c.precision, st), "d4pg_critic_forward")
    else:
        out = {"probs": _nan(B, c.N), "logits": _nan(B, c.N) if logits else None}
        L.check(L.lib().d4pg_critic_forward(P(net.flat_params()), c.S, c.A, c.N, P(c.s), P(c.a), B, P(out["probs"]),
                                            P(out["logits"]), P(ws), c.precision, st), "d4pg_critic_forward")
    return out, ws


def _critic_backward(c, out, ws):
    L = _lib()
    B, net, P = c.B, c.critic, L.ptr
    G, gs, ga = _nan(net._total), _nan(B, c.S), _nan(B, c.A)
    scratch = _nan(B * (2 * H_ + max(H_, _pitch4(c.N))))
    st = L.stream_ptr()
    if c.kind == "mixture_of_gaussian":
        gw, gmu, gsig = c.g_head
        rc = L.lib().d4pg_critic_backward_mog(P(net.flat_params()), c.S, c.A, net.n_components, P(c.s), P(c.a), B,
                                              P(out["raw"]), P(ws), P(gw), P(gmu), P(gsig), P(G), P(gs), P(ga),
                                              P(scratch), c.precision, st)
    elif c.kind == "quantile":
        rc = L.lib().d4pg_critic_backward(P(net.flat_params()), c.S, c.A, c.N, P(c.s), P(c.a), B, None, P(ws), None,
                                          P(c.g_head[0]), P(G), P(gs), P(ga), P(scratch), c.precision, st)
    else:
        gp, gz = c.g_head
        rc = L.lib().d4pg_critic_backward(P(net.flat_params()), c.S, c.A, c.N, P(c.s), P(c.a), B, P(out["probs"]),
                                          P(ws), P(gp), P(gz), P(G), P(gs), P(ga), P(scratch), c.precision, st)
    L.check(rc, "critic backward")
    return G, gs, ga, scratch


def _planes(scratch, B, out_dim):
    """The backward scratch after the call: (p0, p1, the head's dZ plane [B, pitch4(out)])."""
    p0, p1 = scratch[:B * H_].view(B, H_), scratch[B * H_:2 * B * H_].view(B, H_)
    return p0, p1, scratch[2 * B * H_:2 * B * H_ + B * _pitch4(out_dim)].view(B, _pitch4(out_dim))


def _exact(rep, name, ok):
    rep.add(name, 0.0 if ok else math.inf)


# ---- teacher-forced checks ---------------------------------------------------------------------------------------------
def _chained(chk, x, e, wt, mask=None):
    """One dX layer of the plan from an input that may differ from the device's by e: (reference, bound)."""
    return SC.chained_layer(x, e, wt, None, chk.rho, chk.beta, x.shape[1] if chk.tc_fwd else 0, mask=mask)


def _check_actor(chk, c, out, ws, G, gs, scratch):
    B, A, rep = c.B, c.A, chk.rep
    w = _weights(c.actor)
    h1, h2, h3 = ws.view(3, B, H_)
    s = c.s
    chk.layer("a.h1", "fwd", h1, s, w["fc1.weight"].T, w["fc1.bias"], "relu")
    chk.layer("a.h2", "fwd", h2, h1, w["fc2.weight"].T, w["fc2.bias"])
    chk.layer("a.h3", "fwd", h3, h2, w["fc2_2.weight"].T, w["fc2_2.bias"], "relu")
    chk.layer("a.action", "fwd", out, h3, w["fc3.weight"].T, w["fc3.bias"], "tanh")

    # head: dz3 = g (1 - y^2) in fp32 from the saved tanh output (t*t, 1 - t^2 and the product each round once)
    p0, p1, dz = _planes(scratch, B, A)
    y, g = out.double(), c.g_action.double()
    rep.add("a.dz3", SC.ratio(dz[:, :A], g * (1 - y * y), U * g.abs() * (y * y + 2 * (1 - y * y)) * (1 + 4 * U)))
    _exact(rep, "a.dz3 pads", bool((dz[:, A:] == 0).all()))
    dz3 = dz[:, :A]
    m1, m3 = (h1 > 0).double(), (h3 > 0).double()
    zero = lambda x: torch.zeros(x.shape, dtype=torch.float64, device=x.device)
    dz22, e22 = SC.stored(*_chained(chk, dz3, zero(dz3), w["fc3.weight"], m3))
    rep.add("a.dh2 (p1)", SC.ratio(p1, *_chained(chk, dz22, e22, w["fc2_2.weight"])))      # no ReLU after fc2 (H9)
    chk.layer("a.dz1 (p0)", "dX", p0, p1, w["fc2.weight"], mask=m1)
    chk.layer("a.grad_s", "dX", gs, p0, w["fc1.weight"])
    views = _views(c.actor, G)
    refs = {}
    for layer, delta, x, e in (("fc3", dz3, h3, None), ("fc2_2", dz22, h2, e22), ("fc2", p1, h1, None), ("fc1", p0, s, None)):
        refs[layer + ".weight"] = chk.grad("a.%s.weight" % layer, views[layer + ".weight"], delta, x, e=e, sep=True)
        refs[layer + ".bias"] = chk.grad("a.%s.bias" % layer, views[layer + ".bias"], delta, None, e=e)
    rep.add("a.grad_params pads", _pads_zero(c.actor, G))
    return refs


def _check_critic(chk, c, out, ws, G, gs, ga, scratch):
    B, N, A, rep = c.B, c.N, c.A, chk.rep
    w = _weights(c.critic)
    h1, h2, h3 = ws.view(3, B, H_)
    s, a = c.s, c.a
    chk.layer("c.h1", "fwd", h1, s, w["fc1.weight"].T, w["fc1.bias"], "relu")
    chk.layer("c.h2", "fwd", h2, torch.cat([h1, a], 1), w["fc2.weight"].T, w["fc2.bias"], "relu")
    chk.layer("c.h3", "fwd", h3, h2, w["fc2_2.weight"].T, w["fc2_2.bias"], "relu")
    z = out.get("logits", out.get("raw", out.get("theta")))
    chk.layer("c.fc3", "fwd", z, h3, w["fc3.weight"].T, w["fc3.bias"])
    if c.kind == "categorical":
        zd = z.double()
        d = (zd - zd.max(1, keepdim=True).values).abs()
        ref = torch.softmax(zd, 1)
        rep.add("c.probs", SC.ratio(out["probs"], ref, U * ref * (PROBS_UNITS + d + d.max(1, keepdim=True).values)))
    elif c.kind == "mixture_of_gaussian":
        for name, ref in zip(("w", "mu", "sigma"), MO.head(z.double(), c.critic.n_components)):
            rep.add("c." + name, SC.ratio(out[name], ref, ONE_ROUNDING * ref.abs()))

    # the head's dZ plane
    p0, p1, dz = _planes(scratch, B, N)
    if c.kind == "categorical":
        # dz = y (gy - sum_j gy_j y_j) + gz from the saved probabilities y, the dot in fp32 over N (SC.bound)
        y, (gy, gz) = out["probs"].double(), (t.double() for t in c.g_head)
        dot = (gy * y).sum(1, keepdim=True)
        t1 = gy - dot
        ref = y * t1 + gz
        e_dot = SC.bound((gy * y).abs().sum(1, keepdim=True), N)
        tol = (y.abs() * (e_dot + U * t1.abs()) + U * (y * t1).abs() + U * ref.abs()) * (1 + 4 * U)
        rep.add("c.dz", SC.ratio(dz[:, :N], ref, tol))
    elif c.kind == "mixture_of_gaussian":
        # mog_head_backward_kernel runs in fp64: within one fp32 rounding of the fp64 autograd of the head
        raw = z.double().requires_grad_(True)
        torch.autograd.backward(MO.head(raw, c.critic.n_components), [t.double() for t in c.g_head])
        rep.add("c.dz", SC.ratio(dz[:, :N], raw.grad, ONE_ROUNDING * raw.grad.abs()))
    else:
        _exact(rep, "c.dz", torch.equal(dz[:, :N], c.g_head[0]))                 # theta is the raw head
    _exact(rep, "c.dz pads", bool((dz[:, N:] == 0).all()))

    dzN = dz[:, :N]
    m1, m2, m3 = (h1 > 0).double(), (h2 > 0).double(), (h3 > 0).double()
    zero = lambda x: torch.zeros(x.shape, dtype=torch.float64, device=x.device)
    dz22, e22 = SC.stored(*_chained(chk, dzN, zero(dzN), w["fc3.weight"], m3))
    rep.add("c.dz2 (p1)", SC.ratio(p1, *_chained(chk, dz22, e22, w["fc2_2.weight"], m2)))
    chk.layer("c.dz1 (p0)", "dX", p0, p1, w["fc2.weight"][:, :H_], mask=m1)
    chk.layer("c.grad_a", "dX", ga, p1, w["fc2.weight"][:, H_:])
    chk.layer("c.grad_s", "dX", gs, p0, w["fc1.weight"])
    views = _views(c.critic, G)
    refs = {}
    for layer, delta, x, e in (("fc3", dzN, h3, None), ("fc2_2", dz22, h2, e22), ("fc2", p1, torch.cat([h1, a], 1), None),
                               ("fc1", p0, s, None)):
        refs[layer + ".weight"] = chk.grad("c.%s.weight" % layer, views[layer + ".weight"], delta, x, e=e, sep=True)
        refs[layer + ".bias"] = chk.grad("c.%s.bias" % layer, views[layer + ".bias"], delta, None, e=e)
    rep.add("c.grad_params pads", _pads_zero(c.critic, G))
    return refs


# ---- the same inputs through the differentiable modules ---------------------------------------------------------------
def _module_outputs(c, net, s, a):
    if net is c.actor:
        return [net(s)]
    if c.kind == "categorical":
        return list(net(s, a, return_logits=True))
    if c.kind == "mixture_of_gaussian":
        return list(net(s, a))
    return [net(s, a)]


def _through_autograd(c, net, grads):
    """(parameter .grads, d state, d action) of the module's autograd backward on the case's inputs, placed at the
    same alignment as the direct call's."""
    net.differentiable, net.precision = True, c.precision
    for p in net.parameters():
        p.grad = None
    s, s_flat = _place(c.s0, c.mis, grad=True)
    a, a_flat = _place(c.a0, c.mis, grad=True)
    torch.autograd.backward(_module_outputs(c, net, s, a), grads)
    off = 1 if c.mis else 0
    ds = s_flat.grad[off:off + c.s0.numel()].view(c.s0.shape)
    da = a_flat.grad[off:off + c.a0.numel()].view(c.a0.shape) if a_flat.grad is not None else None
    return {k: p.grad for k, p in net.named_parameters()}, ds, da


def _link(rep, tag, B, got, direct, refs):
    """Module gradients against the direct call's: bit for bit below batch 1024, within the direct check's bound from
    1024 on (split-K slices add into the buffer with atomics, in any order)."""
    for k, g in got.items():
        if B < 1024:
            _exact(rep, "%s module %s" % (tag, k), torch.equal(g, direct[k]))
        else:
            rep.add("%s module %s" % (tag, k), SC.ratio(g, *refs[k]))


# precision -> {forward output name, "dX", "dW": the largest ratio of its checks to the bound of the UNROUNDED layer},
# over the cases run so far
_SEPARATION = {}
FORWARD_OUTPUTS = ("a.h1", "a.h2", "a.h3", "a.action", "c.h1", "c.h2", "c.h3", "c.fc3")


def _run_case(case, precision):
    import d4pg_b200 as d4pg
    S, A, info, B, mis = case
    t0 = time.perf_counter()
    c = _Ctx(d4pg, S, A, info, B, mis, precision)
    chk = SC.LayerCheck("levels", PRECISIONS[precision], "%s/%s" % (PRECISIONS[precision], _id(case)))
    rep = chk.rep

    out, ws = _actor_forward(c)
    G, gs, scratch = _actor_backward(c, out, ws)
    refs = _check_actor(chk, c, out, ws, G, gs, scratch)
    got, ds, _ = _through_autograd(c, c.actor, [c.g_action])
    _link(rep, "a", B, got, _views(c.actor, G), refs)
    _exact(rep, "a module d state", torch.equal(ds, gs))

    cout, cws = _critic_forward(c)
    if c.kind == "categorical":                 # without a logits buffer (h1 is the logits scratch): the same probs
        probs_only = _critic_forward(c, logits=False)[0]["probs"]
        _exact(rep, "c.probs (logits NULL)", torch.equal(probs_only, cout["probs"]))
    G, gs, ga, scratch = _critic_backward(c, cout, cws)
    refs = _check_critic(chk, c, cout, cws, G, gs, ga, scratch)
    got, ds, da = _through_autograd(c, c.critic, list(c.g_head))
    _link(rep, "c", B, got, _views(c.critic, G), refs)
    _exact(rep, "c module d state", torch.equal(ds, gs))
    _exact(rep, "c module d action", torch.equal(da, ga))
    torch.cuda.synchronize()
    print("%s: %.2f s" % (rep.label, time.perf_counter() - t0))
    rep.finish()
    if rep.sep:
        sep = _SEPARATION.setdefault(precision, {})
        for kind, name, r in rep.sep:
            key = name if kind == "fwd" else kind
            sep[key] = max(sep.get(key, 0.0), r)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
@pytest.mark.parametrize("precision", [0, 1, 2, 3])
def test_module_entry_points_every_layer_at_tile_and_split_k_edges(precision, case):
    _run_case(case, precision)


@pytest.mark.gpu
@pytest.mark.parametrize("precision", [2, 3])
def test_one_pass_rounding_is_present_and_applied_once(precision):
    """Across the cases of a one-pass precision, every forward layer output of both networks, at least one dX layer
    and at least one weight gradient land more than 10x the bound of the unrounded layer away from it: the operands
    are rounded, and only once (a kernel that quietly ran 3xTF32 or fp32 would be within that bound).  The witnesses
    come from the small batches, where the weight gradients' rounding errors do not average out.  Where no case of
    the precision ran in this session, they all run here."""
    if precision not in _SEPARATION:
        for case in CASES:
            _run_case(case, precision)
    sep = _SEPARATION[precision]
    print("%s: %s x the unrounded bound" % (PRECISIONS[precision], ", ".join("%s %.3g" % kv for kv in sorted(sep.items()))))
    for key in FORWARD_OUTPUTS + ("dX", "dW"):
        assert sep.get(key, 0.0) > 10, (precision, key, sep)


SUBSETS = {"actor": ("params", "s"), "categorical": ("params", "s", "a"), "mixture_of_gaussian": ("params", "s", "a"),
           "quantile": ("params", "s", "a")}


@pytest.mark.gpu
@pytest.mark.parametrize("net", list(SUBSETS))
@pytest.mark.parametrize("precision", [0, 1, 2, 3])
def test_every_gradient_subset_is_the_full_calls(precision, net):
    """Every non-empty subset of {parameters, state, action} (the actor: {parameters, state}) marked as requiring grad,
    at B = 129: each requested gradient is bit-identical to the call that requests all of them, and each one not
    requested is None.  The frozen critic with a differentiable action is the policy loss written against the modules
    (ddpg.py:236-238): d action alone, the fc1 level skipped."""
    import d4pg_b200 as d4pg
    S, A, B = 17, 6, 129
    info = {"actor": _cat(51), "categorical": _cat(51), "mixture_of_gaussian": _mog(4), "quantile": _qr(32)}[net]
    c = _Ctx(d4pg, S, A, info, B, False, precision)
    module = c.actor if net == "actor" else c.critic
    module.differentiable, module.precision = True, precision
    grads = [c.g_action] if net == "actor" else list(c.g_head)
    names = SUBSETS[net]

    def run(want):
        for p in module.parameters():
            p.grad = None
            p.requires_grad_("params" in want)
        s = c.s0.cuda().requires_grad_("s" in want)
        a = c.a0.cuda().requires_grad_("a" in want)
        torch.autograd.backward(_module_outputs(c, module, s, a), grads)
        out = {"params": [None if p.grad is None else p.grad.clone() for p in module.parameters()], "s": s.grad, "a": a.grad}
        for p in module.parameters():
            p.requires_grad_(True)
        return out

    full = run(names)
    assert all(g is not None for g in full["params"]) and full["s"] is not None
    for r in range(1, len(names) + 1):
        for want in itertools.combinations(names, r):
            got = run(want)
            for k in names:
                if k not in want:
                    assert (all(g is None for g in got[k]) if k == "params" else got[k] is None), (want, k)
                elif k == "params":
                    assert all(torch.equal(g, f) for g, f in zip(got[k], full[k])), (want, k)
                else:
                    assert torch.equal(got[k], full[k]), (want, k)
