"""precision="tf32" (libd4pg precision 2): one TF32 tensor-core pass per MLP GEMM, against a float64 restatement on the
same TF32-ROUNDED operands (tests/tf32_oracle.py, a derived oracle: the reference has no TF32 mode).

How an fp32 operand becomes TF32 depends on the kernel that runs the layer, so the oracle follows the step plan:

  plan            kernel                          forward / dX operands            dW
  PLAN_TC_CHAIN   mlp_tc_chain.cu (wgmma)         truncated (tf32_hi, "rz")        exact fp32 FFMA (gemm_wide_kernel)
  PLAN_CHAIN      mlp_chain.cu (mma.sync tiles)   cvt.rna.tf32.f32 ("rna")         exact fp32 FFMA (gemm_wide_kernel)
  PLAN_LEVELS     gemm_tc.cu (wgmma, one pass)    truncated ("rz")                 truncated ("rz")

Bias gradients are column sums of the unrounded fp32 deltas on every plan.  Against the unrounded float64 layer a
one-pass TF32 result differs by ~2^-11 relative; every test also checks that it does (a kernel that quietly ran 3xTF32,
or skipped the rounding, would be closer to the unrounded layer than to this oracle).
"""
import random

import numpy as np
import pytest
import torch

from tests import step_check as SC
from tests import tf32_oracle as TO

H_ = 256
rt = TO.rt
TOL = 1e-5                   # one layer on the device's own input: operands round identically on both sides


def _lin(x, w, b=None, mode="rz"):
    """One layer in float64 on TF32-rounded operands (mode None: unrounded); the bias is added to the fp64 sum."""
    y = (rt(x, mode) @ rt(w, mode).T) if mode else (x.double() @ w.double().T)
    return y if b is None else y + b.double()


class _Report:
    """Collects (name, error, bound) so that every measurement is printed before the first failing one is reported."""

    def __init__(self, label):
        self.label, self.rows, self.sep = label, [], []

    def check(self, name, mine, ref, tol=TOL, scale=None, unrounded=None, kind=None, l2=False):
        """max abs error <= tol * scale (default max(1, |ref|max)); l2: relative L2 error <= tol"""
        mine, ref = mine.double().cpu(), ref.double().cpu()
        assert mine.shape == ref.shape, (name, mine.shape, ref.shape)
        if l2:
            dist = lambda x: float((mine - x).norm()) / max(float(ref.norm()), 1e-30)
            bound = tol
        else:
            dist = lambda x: float((mine - x).abs().max())
            bound = tol * (max(1.0, float(ref.abs().max())) if scale is None else scale)
        err = dist(ref)
        self.rows.append((name, err, bound))
        if unrounded is not None:      # distance from the unrounded float64 result, in units of this check's bound
            self.sep.append((kind, name, dist(unrounded.double().cpu()) / bound))
        return err

    def finish(self):
        for name, err, bound in self.rows:
            print("%s %-22s err %.3e  bound %.3e  (%.3f of bound)" % (self.label, name, err, bound, err / bound))
        for kind, name, s in self.sep:
            print("%s %-22s %s: %.1f x bound from the unrounded layer" % (self.label, name, kind, s))
        bad = [r for r in self.rows if not r[1] <= r[2]]
        assert not bad, "%s: %s" % (self.label, ", ".join("%s err %.3e > %.3e" % r for r in bad))


def _seps(rep, kind):
    return [s for k, _, s in rep.sep if k == kind]


# ---- CPU: the derived oracle itself ---------------------------------------------------------------------------------
def test_tf32_oracle_rounding_is_bit_exact():
    one = 1.0
    cases = [(one + 2 ** -11, one + 2 ** -10, one),          # a tie: away from zero under rna, dropped under rz
             (one + 2 ** -11 - 2 ** -23, one, one),           # just below the tie: down under both
             (one + 2 ** -10, one + 2 ** -10, one + 2 ** -10),  # already TF32
             (3.0 + 3 * 2 ** -11, 3.0 + 2 ** -9, 3.0)]            # TF32 ulp 2^-9 in [2, 4): 3/4 ulp up / down
    for sign in (1.0, -1.0):
        for x, rna, rz in cases:
            t = torch.tensor([sign * x], dtype=torch.float32)
            assert float(t) == sign * x                       # every case is an exact fp32 value
            assert float(rt(t, "rna")) == sign * rna, (sign * x, float(rt(t, "rna")))
            assert float(rt(t, "rz")) == sign * rz, (sign * x, float(rt(t, "rz")))
    with pytest.raises(ValueError):
        rt(torch.ones(1), "rn")


def test_tf32_oracle_rounders_are_idempotent_and_drop_13_bits():
    torch.manual_seed(4)
    x = torch.randn(4096) * torch.logspace(-20, 20, 4096)
    for mode in ("rz", "rna"):
        y = rt(x, mode)
        assert y.dtype == torch.float64
        assert torch.equal(rt(y.float(), mode), y), mode
        assert int((y.float().view(torch.int32) & 0x1FFF).abs().max()) == 0, mode
        assert float(((y - x.double()).abs() / x.double().abs()).max()) <= (2 ** -10 if mode == "rz" else 2 ** -11)
    assert float((rt(x, "rz").abs() - x.double().abs()).max()) <= 0.0      # rz never grows a magnitude


@pytest.mark.parametrize("mode", ["rz", "rna"])
def test_tf32_oracle_linear_rounds_operands_and_keeps_fp32_bias_grad(mode):
    torch.manual_seed(3)
    x = torch.randn(37, 19, requires_grad=True); w = torch.randn(11, 19, requires_grad=True); b = torch.randn(11, requires_grad=True)
    g = torch.randn(37, 11)
    for round_dw in (True, False):
        for p in (x, w, b):
            p.grad = None
        y = TO.linear(mode, round_dw)(x, w, b)
        assert torch.equal(y, (rt(x, mode) @ rt(w, mode).T).float() + b.detach())
        y.backward(g)
        assert torch.equal(x.grad, (rt(g, mode) @ rt(w, mode)).float())
        dw = (rt(g, mode).T @ rt(x, mode)) if round_dw else (g.double().T @ x.detach().double())
        assert torch.equal(w.grad, dw.float())
        assert torch.equal(b.grad, g.sum(0))
        assert (y - torch.nn.functional.linear(x, w, b)).abs().max() > 1e-4     # the rounding is visible
    assert not torch.equal(TO.linear("rz")(x, w, b), TO.linear("rna")(x, w, b))


# ---- GPU: every intermediate of one learner step ----------------------------------------------------------------------
def _ddpg(d4pg, B, S, A, N, graph=False, chain="cluster", projection="reference", n_steps=1, seed=12):
    info = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": N}
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    n = max(2048, 2 * B)
    dd = d4pg.DDPG(S, A, memory_size=n, batch_size=B, critic_dist_info=info, precision="tf32", use_graph=graph,
                   sampling="device", philox_seed=3, prefetch=False, chain=chain, projection=projection, n_steps=n_steps)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(1)
    dd.replayBuffer.add_batch(rng.randn(n, S).astype(np.float32), rng.uniform(-1, 1, (n, A)).astype(np.float32),
                              (-3 * rng.rand(n)), rng.randn(n, S).astype(np.float32), rng.rand(n) < 0.05)
    return dd


# plan -> (forward / dX rounding, dW rounded, kernels per eager step)
PLANS = {"tc_chain": ("rz", False, 9), "chain": ("rna", False, 7), "levels": ("rz", True, 18)}
# The wgmma chains do not write the target chain's hidden planes, p_dz22 / p_dz2 or the policy chain's critic h1 row-major
# (they travel as TF32 images between the CTAs), so actor_target_out, target_logits and a_dz3 are checked against the
# oracle CHAINED through those layers (tests/step_check.py: a componentwise bound carried through each chained layer,
# and relative L2 at `CHAINED_TOL`).  A chained operand whose fp32 value differs in the last bit from the device's may
# truncate to the neighbouring TF32 value, 2^-10 relative: a few sparse elements per layer.  Their largest effect on one
# output is within ~10x of the one-pass error itself, so a max-abs bound cannot separate one pass from three; relative
# L2 can (the sparse flips barely move it, the dense one-pass error does).  Worst measured on one H100 over the three
# wgmma-chain cases: actor_target_out 1.7e-5, target_logits 9.7e-7, a_dz3 4.2e-5; the same outputs were 2.1e-4 - 7.7e-4,
# 3.5e-5 - 5.6e-5 and 1.9e-3 - 2.2e-3 from the unrounded chain.


@pytest.mark.gpu
@pytest.mark.parametrize("plan,B,S,A,N,graph,chain,projection", [
    ("tc_chain", 256, 17, 6, 51, False, "cluster", "reference"),
    ("tc_chain", 200, 3, 1, 101, True, "cluster", "reference"),      # ragged M (200 rows), CUDA graph
    ("tc_chain", 512, 32, 8, 64, False, "cluster", "reference"),     # the limits of the wgmma chain plan
    ("chain", 96, 376, 17, 51, False, "cluster", "reference"),       # |s| > 32: mma.sync tiles
    ("chain", 64, 17, 40, 51, False, "cluster", "reference"),        # |a| > 32: mma.sync tiles
    ("levels", 256, 17, 6, 51, False, "levels", "reference"),
    ("levels", 1024, 376, 17, 51, False, "cluster", "reference"),    # split-K dW, ragged fc2 concat tail
    ("levels", 4096, 17, 6, 101, False, "cluster", "nstep")])        # config 5 shapes: split-K dW, n-step projection
def test_tf32_every_intermediate_vs_rounded_restatement(plan, B, S, A, N, graph, chain, projection):
    """Every activation, logit, delta and parameter gradient of one eager DDPG.train() at precision="tf32" against the
    float64 restatement on operands rounded the way the plan's kernels round them.  Each layer is fed the device's own
    inputs, ReLU masks and upstream deltas; bound 1e-5 x max(1, |ref|max), for the deltas (O(1/B)) 1e-5 x |ref|max, for
    the parameter gradients (~1e-6) the componentwise bound of tests/step_check.py."""
    import d4pg_b200 as d4pg
    mode, round_dw, nk = PLANS[plan]
    tc = plan == "tc_chain"
    dd = _ddpg(d4pg, B, S, A, N, graph=graph, chain=chain, projection=projection, n_steps=5 if projection == "nstep" else 1)
    with torch.no_grad():
        dd.actor_target.flat_params().mul_(1.01)
        dd.critic_target.flat_params().mul_(0.99)
    W = {k: {n_: v.detach().cpu() for n_, v in net.state_dict().items()}
         for k, net in (("a", dd.actor), ("at", dd.actor_target), ("c", dd.critic), ("ct", dd.critic_target))}
    dd.train()
    torch.cuda.synchronize()
    assert dd.kernels_per_step() == nk
    t = lambda name, w=None: dd.debug_tensor(name, (B, w) if w else None).cpu()
    s, a, s2 = t("s", S), t("a", A), t("s2", S)
    relu, ident = torch.relu, (lambda x: x)
    Wa, Wat, Wc, Wct = W["a"], W["at"], W["c"], W["ct"]
    rep = _Report("%s(%d,%d,%d,%d)" % (plan, B, S, A, N))

    def check_fwd(name, x, w, l, act_fn):
        ref = act_fn(_lin(x, w[l + ".weight"], w[l + ".bias"], mode=mode))
        unr = act_fn(_lin(x, w[l + ".weight"], w[l + ".bias"], mode=None))
        rep.check(name, t(name, A if name.startswith("actor") else (N if name.endswith("logits") else H_)), ref,
                  unrounded=unr, kind="fwd")

    # forward: every layer from the device's own input to it
    check_fwd("h1_a", s, Wa, "fc1", relu)
    check_fwd("h2_a", t("h1_a", H_), Wa, "fc2", ident)
    check_fwd("h3_a", t("h2_a", H_), Wa, "fc2_2", relu)
    check_fwd("actor_out", t("h3_a", H_), Wa, "fc3", torch.tanh)
    ch1, ch2, ch3, aout = t("h1_c", H_), t("h2_c", H_), t("h3_c", H_), t("actor_out", A)
    check_fwd("h1_c", s, Wc, "fc1", relu)
    check_fwd("h2_c", torch.cat([ch1, a], 1), Wc, "fc2", relu)
    check_fwd("h3_c", ch2, Wc, "fc2_2", relu)
    check_fwd("q_logits", ch3, Wc, "fc3", ident)
    ph2, ph3 = t("h2_p", H_), t("h3_p", H_)
    check_fwd("h2_p", torch.cat([ch1, aout], 1), Wc, "fc2", relu)      # the policy pass's critic h1 is h1_c
    check_fwd("h3_p", ph2, Wc, "fc2_2", relu)
    check_fwd("pi_logits", ph3, Wc, "fc3", ident)
    at_out = t("actor_target_out", A)
    if not tc:
        check_fwd("h1_at", s2, Wat, "fc1", relu)
        check_fwd("h2_at", t("h1_at", H_), Wat, "fc2", ident)
        check_fwd("h3_at", t("h2_at", H_), Wat, "fc2_2", relu)
        check_fwd("actor_target_out", t("h3_at", H_), Wat, "fc3", torch.tanh)
        check_fwd("h1_ct", s2, Wct, "fc1", relu)
        check_fwd("h2_ct", torch.cat([t("h1_ct", H_), at_out], 1), Wct, "fc2", relu)
        check_fwd("h3_ct", t("h2_ct", H_), Wct, "fc2_2", relu)
        check_fwd("target_logits", t("h3_ct", H_), Wct, "fc3", ident)

    # backward: deltas from the device's own upstream delta and masks
    dq, dpi = t("dlogits_q", N), t("dlogits_pi", N)
    dm = {k: v > 0 for k, v in (("h1_c", ch1), ("h2_c", ch2), ("h3_c", ch3), ("h1_a", t("h1_a", H_)), ("h3_a", t("h3_a", H_)),
                                ("h2_p", ph2), ("h3_p", ph3))}
    names = ["c_dz22", "c_dz2", "c_dz1", "a_dz3", "a_dz22", "a_dh2", "a_dz1"] + ([] if tc else ["p_dz22", "p_dz2"])
    dev = {k: t(k, A if k == "a_dz3" else H_) for k in names}
    dx = lambda g, w, m=mode: (rt(g, m) @ rt(w, m)) if m else (g.double() @ w.double())
    tanh_d = 1 - aout.double() ** 2
    upstream = {"c_dz22": (dq, Wc["fc3.weight"], dm["h3_c"]),
                "c_dz2": (dev["c_dz22"], Wc["fc2_2.weight"], dm["h2_c"]),
                "c_dz1": (dev["c_dz2"], Wc["fc2.weight"][:, :H_], dm["h1_c"]),
                "a_dz22": (dev["a_dz3"], Wa["fc3.weight"], dm["h3_a"]),
                "a_dh2": (dev["a_dz22"], Wa["fc2_2.weight"], None),
                "a_dz1": (dev["a_dh2"], Wa["fc2.weight"], dm["h1_a"])}
    if not tc:
        upstream.update({"p_dz22": (dpi, Wc["fc3.weight"], dm["h3_p"]),
                         "p_dz2": (dev["p_dz22"], Wc["fc2_2.weight"], dm["h2_p"]),
                         "a_dz3": (dev["p_dz2"], Wc["fc2.weight"][:, H_:], tanh_d)})
    for name, (g, w, msk) in upstream.items():
        ref, unr = dx(g, w), dx(g, w, None)
        if msk is not None:
            ref, unr = ref * msk, unr * msk
        rep.check(name, dev[name], ref, scale=max(float(ref.abs().max()), 1e-30), unrounded=unr, kind="dX")

    # dW from the device's deltas and activations (rounded on the level plan only), bias gradients as sums of the
    # unrounded fp32 deltas: against the componentwise bound of tests/step_check.py, with its power check
    ah1, ah2, ah3 = t("h1_a", H_), t("h2_a", H_), t("h3_a", H_)
    sc = SC.StepCheck(dd, W, plan, "tf32", label=rep.label)
    if tc:
        # the chained outputs against the rz chain (bound, power, relative L2), and how far they land from the
        # unrounded chain, in units of CHAINED_TOL
        refs, unrounded = sc.chained_refs(), sc.chained_refs(rho=None)
        sc.chained(refs)
        for name, (ref, _, _) in unrounded.items():
            rep.sep.append(("chained", name, SC.rel_l2(sc.dev(name[:-1]), ref) / SC.CHAINED_TOL["rz"][name]))
    sc.grads({"c": {"fc3": (dq, ch3), "fc2_2": (dev["c_dz22"], ch2), "fc2": (dev["c_dz2"], torch.cat([ch1, a], 1)),
                    "fc1": (dev["c_dz1"], s)},
              "a": {"fc3": (dev["a_dz3"], ah3), "fc2_2": (dev["a_dz22"], ah2), "fc2": (dev["a_dh2"], ah1), "fc1": (dev["a_dz1"], s)}})
    rep.finish()
    sc.rep.finish()

    # the rounding is there, once: one forward layer and one dX layer land far outside the bound of the unrounded layer
    assert max(_seps(rep, "fwd")) > 10, ("forward", rep.sep)
    assert max(_seps(rep, "dX")) > 10, ("dX", rep.sep)
    if tc:
        # the chained bounds stay far below how far one pass lands from the unrounded chain: a_dz3 (measured ~20x) at
        # least 10x, and every chained output at least 2x
        assert max(_seps(rep, "chained")) >= 10 and min(_seps(rep, "chained")) >= 2, ("chained", rep.sep)
