"""One learner step, layer by layer: every forward layer, dX layer, weight gradient and bias gradient of one eager
DDPG.train() recomputed in float64 from the DEVICE's own input to that layer (teacher forcing), and held to a
componentwise bound.

`LayerCheck` holds the per-layer part (the `MODES` row, one layer, one weight or bias gradient, chained layers and the
`Report`) and checks whatever device tensor it is handed (tests/test_gpu_module_edges.py: the actor and critic entry
points); `StepCheck` reads the step's planes through `dd.debug_tensor`.

Teacher forcing.  Each layer is fed the device's input plane, the device's ReLU mask (h > 0) and the device's upstream
delta, and the tanh' factor is 1 - y^2 of the device's own actor output.  A pre-activation within rounding of zero then
masks the same element on both sides, so no delta element can flip and a tight bound survives any batch size.

Rounding.  `rho` is the operand rounding the plan's kernels apply before the products: None for fp32 and 3xTF32
(tf32x3), "rz" / "rna" for one TF32 pass (tests/tf32_oracle.py), "bf16" for the bf16 kernels (tests/bf16_oracle.py).
Which kernel computes dW, and so whether dW is rounded, follows the plan table of test_gpu_tf32.py (`MODES` below).

Bound.  An element computed as sum_k a_k b_k (+ bias) from K products, with S = |rho(A)| |rho(B)|^T (+ |bias|):

    |dev - ref| <= (ALPHA * 2^-24 * sqrt(K) + beta + TRUNC * Kc * 2^-24) * S

Kc is the number of rows one tensor-core accumulator sums (0 for the FFMA kernels; see TRUNC).  beta = 0 where the oracle reproduces the operand rounding (fp32, tf32, bf16), BETA_3XTF32 for the 3xTF32 split, which
the oracle does not reproduce (it takes the fp32 operands as exact).  A bias gradient is sum_k delta_k: S = sum |delta|.
ReLU and tanh are monotone: the bound maps through them as max(f(z + e) - f(z), f(z) - f(z - e)), at most the
pre-activation bound e and zero where the unit is off by more than e; tanh adds 4 ulp of its output, and the tanh' factor of
d action (computed in fp32 from y) adds 4 ulp of its input sum.  On the CPU (test_gpu_step_edges.py), fp32 matmul,
8-way split-K and sequential fp32 accumulation reach at most 0.99 x 2^-24 sqrt(K) S (at K = 1), the 3xTF32 split
with rz hi/lo 1.23 x 2^-20 S; dropping one row's contribution exceeds the bound by > 100x.

Power.  A bound is only worth what it rejects: for every weight and bias gradient, the reference with the contribution
of the last batch row that contributes anything removed must be at least POWER_MIN x the bound away from the device.

Chained layers.  Layers the wgmma chains keep inside the cluster (the target chains' hidden planes, p_dz22 and p_dz2)
are not written row-major, and actor_critic="post_update" sends the policy pass through the critic AFTER its Adam step,
whose h1 the device recomputes without storing.  So actor_target_out, target_logits, a_dz3 and (post_update) h2_p are
checked through a chain: each chained layer's reference input x_ref is the previous layer's reference cast to fp32, and
the device's unobserved input x differs from it by at most e componentwise (e = 0 for a plane read back from the
device).  A layer y = f(rho(x) W^T + b) then carries the bound forward (`chained_layer`):

    d   = max |rho(x) - rho(x_ref)| over |x - x_ref| <= e           (`operand_error`: rho is monotone, so the ends of
                                                                     the interval, rounded outward to fp32, give it)
    e_y = |rho(W)| d + bound(|rho(W)| (|rho(x_ref)| + d) + |b|, K)   (the operand error, then the accumulation of the
                                                                     device's own operands, whose |.| sum is at most S)

mapped through f as above (monotone and 1-Lipschitz, so no mask flip needs a case of its own, and a unit that is off by
more than e_y passes no error on), plus 4 ulp for tanh, and, where the next layer consumes it, |y_ref - fp32(y_ref)|
for the fp32 store of the reference.  Mapping through the ReLUs, rather than carrying e_y past them, keeps the bound
~5x tighter over three chained layers, where |W| d grows it by up to ~sqrt(256) per layer against W x.  This holds
row by row, so it is valid at every batch size.
Under one TF32 pass an e of one fp32 ulp may move an operand to the neighbouring TF32 value (2^-10 relative), so the
bound grows toward the one-pass error itself over three chained layers: it cannot separate one pass from three
(test_gpu_tf32.py), which the teacher-forced planes already do.  Power: the reference without the last chained layer's
bias (a_dz3, which has none: without the ReLU mask of p_dz2, the last layer the cluster keeps) must land POWER_MIN x
outside the bound.  From batch 200 on, where it was measured, the relative L2 error of the same outputs is also held to
`CHAINED_TOL`, as a separation statistic.
"""
import math

import torch

from tests import bf16_oracle as BO
from tests import tf32_oracle as TO

H_ = 256
U = 2.0 ** -24                     # unit roundoff of fp32
ALPHA = 4.0
BETA_3XTF32 = 4 * 2.0 ** -20
# The tensor cores' fp32 accumulator rounds its adds toward zero, so over a sum whose terms share a sign the errors do
# not cancel: each add loses up to 2^-23 of a partial sum that grows toward S, ~2^-24 S per row on average.  Sequential
# round-toward-zero accumulation of same-sign terms reaches 0.35-0.46 x K 2^-24 S on the CPU (test_gpu_step_edges.py),
# and 3xTF32 dW on wgmma reached 1.9x the sqrt(K) bound alone at 1023 unsplit rows (~2.1e-5 S, the same as that
# emulation's 2.3e-5 S).
TRUNC = 1.0
POWER_MIN = 10.0

# (plan, precision) -> (rho, beta, tensor-core accumulation) of forward / dX, then the same of dW
#   tc_chain  mlp_tc_chain.cu wgmma chains; dW with exact fp32 FFMA (gemm_wide_kernel)
#   chain     mlp_chain.cu cluster chains: FFMA tiles at fp32, mma.sync tiles otherwise; dW as above
#   levels    one launch per level: gemm_ffma (fp32), gemm_tc (wgmma tf32x3 / tf32), gemm_bf16 -- dW included
MODES = {("tc_chain", "tf32x3"): (None, BETA_3XTF32, True, None, 0.0, False),
         ("tc_chain", "tf32"): ("rz", 0.0, True, None, 0.0, False),
         ("chain", "fp32"): (None, 0.0, False, None, 0.0, False),
         ("chain", "tf32x3"): (None, BETA_3XTF32, True, None, 0.0, False),
         ("chain", "tf32"): ("rna", 0.0, True, None, 0.0, False),
         ("levels", "fp32"): (None, 0.0, False, None, 0.0, False),
         ("levels", "tf32x3"): (None, BETA_3XTF32, True, None, BETA_3XTF32, True),
         ("levels", "tf32"): ("rz", 0.0, True, "rz", 0.0, True),
         ("levels", "bf16"): ("bf16", 0.0, True, "bf16", 0.0, True)}


def kslice(K):
    """Rows one dW accumulator sums on the level plan: split-K from 1024 rows (csrc/gemm_ffma.cu prepare_problem)."""
    if K < 1024:
        return K
    ksplit = min(8, -(-K // 512))
    return -(-(-(-K // ksplit)) // 64) * 64
# kernels of one eager step, by plan (no post-update critic)
KERNELS = {"tc_chain": 9, "chain": 7, "levels": 18}
# relative L2 of the chained outputs, a separation statistic from CHAINED_L2_MIN_B rows on (a batch statistic: nothing
# averages it over a few rows).  A one-pass TF32 chain may truncate a chained operand whose fp32 value differs in the
# last bit to the neighbouring TF32 value (test_gpu_tf32.py); an unrounded chain differs by fp32 casts only
CHAINED_TOL = {None: {"actor_target_out*": 1e-5, "target_logits*": 1e-5, "a_dz3*": 1e-5, "h2_p*": 1e-5},
               "rz": {"actor_target_out*": 5e-5, "target_logits*": 5e-6, "a_dz3*": 1e-4, "h2_p*": 5e-5}}
CHAINED_L2_MIN_B = 200


def rnd(t, rho):
    """The operand a kernel with rounding `rho` multiplies, held exactly in float64."""
    if rho is None:
        return t.double()
    if rho == "bf16":
        return BO.rb(t)
    return TO.rt(t, rho)


def bound(S, K, beta=0.0, alpha=ALPHA, kc=0):
    """kc: rows summed by one tensor-core accumulator (0: none), whose fp32 adds truncate (TRUNC below)."""
    return (alpha * U * math.sqrt(K) + beta + TRUNC * kc * U) * S


def ratio(dev, ref, tol):
    """max |dev - ref| / tol; an element with tol == 0 (every product zero) must match exactly."""
    err = (dev.double() - ref).abs()
    zero = tol == 0
    r = torch.where(zero, torch.zeros_like(err), err / torch.where(zero, torch.ones_like(tol), tol))
    if bool((zero & (err != 0)).any()):
        return math.inf
    return float(r.max()) if r.numel() else 0.0


def matmul_bound(a, b, rho, beta=0.0, kc=0):
    """a [M, K] @ b [K, N] on rho-rounded operands: (float64 reference, componentwise bound)."""
    ra, rb_ = rnd(a, rho), rnd(b, rho)
    return ra @ rb_, bound(ra.abs() @ rb_.abs(), a.shape[1], beta, kc=kc)


def drop_row_ratio(dev, ref, tol, a, b, rho):
    """For ref = a^T b (a [K, M], b [K, N] or None for a column sum): the ratio to the bound of the reference with the
    contribution of the last row k whose contribution is nonzero removed; None when no row contributes."""
    ra = rnd(a, rho)
    rb_ = rnd(b, rho) if b is not None else None
    nz = (ra != 0).any(1) if rb_ is None else ((ra != 0).any(1) & (rb_ != 0).any(1))
    rows = torch.nonzero(nz).flatten()
    if rows.numel() == 0:
        return None
    k = int(rows[-1])
    contrib = ra[k] if rb_ is None else torch.outer(ra[k], rb_[k])
    return ratio(dev, ref - contrib.reshape(ref.shape), tol)


def rel_l2(dev, ref):
    return float((dev.double() - ref.double()).norm()) / max(float(ref.norm()), 1e-30)


def _fp32_outward(v, up):
    """The nearest fp32 value >= v (up) or <= v of a float64 tensor."""
    f = v.float()
    past = f.double() < v if up else f.double() > v
    return torch.where(past, torch.nextafter(f, torch.full_like(f, math.inf if up else -math.inf)), f)


def operand_error(x, e, rho):
    """The largest |rho(x') - rho(x)| over fp32 x' with |x' - x| <= e, componentwise: rho is monotone, so it is
    reached at an end of [x - e, x + e] rounded outward to fp32 (rho None: e itself)."""
    e = e.double()
    if rho is None:
        return e
    xd = x.float().double()
    r0 = rnd(x.float(), rho)
    hi, lo = rnd(_fp32_outward(xd + e, True), rho), rnd(_fp32_outward(xd - e, False), rho)
    return torch.maximum((hi - r0).abs(), (r0 - lo).abs())


def chained_layer(x, e, wt, b, rho, beta=0.0, kc=0, act=None, mask=None, tanh_y=None):
    """One layer act(rho(x) @ rho(wt) + b) (b None: no bias), then * mask or * (1 - tanh_y^2), on the fp32 input x whose
    device value may differ from it by up to e componentwise (e = 0: the device's own plane).  Returns the float64
    reference and the componentwise bound of |device - reference| (module docstring)."""
    d = operand_error(x, e, rho)
    rx, aw = rnd(x, rho), rnd(wt, rho)
    ref = rx @ aw
    aw = aw.abs()
    S = (rx.abs() + d) @ aw
    if b is not None:
        ref, S = ref + b.double(), S + b.double().abs()
    tol = d @ aw + bound(S, x.shape[1], beta, kc=kc)
    if act is not None:            # monotone: the device's z within [ref - tol, ref + tol] maps into [f(.), f(.)]
        f = torch.relu if act == "relu" else torch.tanh
        y = f(ref)
        tol, ref = torch.maximum(f(ref + tol) - y, y - f(ref - tol)), y
        if act == "tanh":
            tol = tol + 4 * 2.0 ** -23 * ref.abs()
    if mask is not None:
        ref, tol = ref * mask, tol * mask
    if tanh_y is not None:         # the tanh' factor, computed in fp32 from y, adds 4 ulp of its input sum
        f = 1 - tanh_y.double() ** 2
        ref, tol = ref * f, tol * f.abs() + 4 * U * S
    return ref, tol


def stored(ref, tol):
    """A chained layer's output as the next layer's input: the reference cast to fp32 and the bound widened by that
    cast, so that it bounds |device fp32 value - fp32 reference|."""
    x = ref.float()
    return x, tol + (ref - x.double()).abs()


class Report:
    """(name, ratio to the bound) of every check and the power ratios; all printed before the first failure.  `chained`
    holds (name, relative L2, its tolerance or None where the batch is too small to hold it to one)."""

    def __init__(self, label):
        self.label, self.rows, self.power, self.chained, self.sep = label, [], [], [], []

    def add(self, name, r):
        self.rows.append((name, r))

    def finish(self):
        for name, r in self.rows:
            print("%s %-20s %.3f of bound" % (self.label, name, r))
        for name, r, tol in self.chained:
            print("%s %-20s rel L2 %.3e (%s)" % (self.label, name, r, "bound %.1e" % tol if tol else "not held"))
        for name, r in self.power:
            print("%s %-20s power: %.3g x bound" % (self.label, name, r if r is not None else math.nan))
        for kind, name, r in self.sep:
            print("%s %-20s %s: %.3g x bound from the unrounded layer" % (self.label, name, kind, r))
        worst = max((r for _, r in self.rows), default=0.0)
        pmin = min((r for _, r in self.power if r is not None), default=math.inf)
        print("%s worst %.3f of bound, smallest power ratio %.3g" % (self.label, worst, pmin))
        bad = ["%s %.3g" % (n, r) for n, r in self.rows if not r <= 1.0]
        bad += ["%s rel L2 %.3e > %.1e" % (n, r, tol) for n, r, tol in self.chained if tol and not r <= tol]
        bad += ["%s power %s" % (n, r) for n, r in self.power if r is None or not r >= POWER_MIN]
        assert not bad, "%s: %s" % (self.label, ", ".join(bad))
        return worst, pmin


def snapshot(dd):
    """The four networks' weights before a step (float32, on the CPU)."""
    return {k: {n_: v.detach().cpu().clone() for n_, v in net.state_dict().items()}
            for k, net in (("a", dd.actor), ("at", dd.actor_target), ("c", dd.critic), ("ct", dd.critic_target))}


class LayerCheck:
    """Teacher-forced checks of single layers computed by the kernels of (plan, precision) (`MODES`), each against the
    device tensor it is handed; every result goes to `rep`."""

    def __init__(self, plan, precision, label):
        self.rho, self.beta, self.tc_fwd, self.rho_dw, self.beta_dw, self.tc_dw = MODES[plan, precision]
        self.rep = Report(label)

    def layer(self, name, kind, dev, x, wt, b=None, act=None, mask=None, tanh_y=None):
        """act(x @ wt + b) (* mask, or * (1 - tanh_y^2)) on the device's own input x against the device tensor `dev`.
        A one-pass precision also records in `rep.sep` how far the device lands from the UNROUNDED layer, in units of
        that layer's bound: far outside it where the operands really are rounded."""
        kc = x.shape[1] if self.tc_fwd else 0
        e = torch.zeros(x.shape, dtype=torch.float64, device=x.device)
        self.rep.add(name, ratio(dev, *chained_layer(x, e, wt, b, self.rho, self.beta, kc, act, mask, tanh_y)))
        if self.rho is not None:
            self.rep.sep.append((kind, name, ratio(dev, *chained_layer(x, e, wt, b, None, 0.0, kc, act, mask, tanh_y))))

    def grad(self, name, dev, delta, x, e=None, sep=False):
        """dW = delta^T x (x None: the bias gradient, sum of the fp32 delta) against the device gradient `dev`, and the
        power of the bound against a dropped row.  e: the componentwise bound of |device delta - delta| where the
        device's delta is not observed (a chained layer's `stored` output), carried through the sum as `chained_layer`
        carries an input error.  sep: record in `rep.sep` (kind "dW") how far the device lands from the unrounded dW.
        Returns (reference, bound)."""
        rho = None if x is None else self.rho_dw
        if x is None:
            err = 0.0 if e is None else e.sum(0)
            ref, tol = delta.double().sum(0), err + bound(delta.double().abs().sum(0) + err, delta.shape[0])
        else:
            kc = kslice(delta.shape[0]) if self.tc_dw else 0
            dw = lambda rho, beta: (matmul_bound(delta.T, x, rho, beta, kc) if e is None
                                    else chained_layer(delta.T, e.T, x, None, rho, beta, kc))
            ref, tol = dw(rho, self.beta_dw)
        dev = dev.to(ref.device).reshape(ref.shape)
        self.rep.add(name, ratio(dev, ref, tol))
        self.rep.power.append((name, drop_row_ratio(dev, ref, tol, delta, x, rho)))
        if sep and rho is not None:
            self.rep.sep.append(("dW", name, ratio(dev, *dw(None, 0.0))))
        return ref, tol

    def chain(self, x, e, w, layers, rho):
        """Forward layers [(layer, act)] of `w` from the fp32 input x (device error e): (reference, bound, reference
        without the last layer's bias) of the last layer, each earlier one `stored` as the next one's input."""
        kc = lambda x: x.shape[1] if self.tc_fwd else 0
        for i, (l, act) in enumerate(layers):
            if i:
                x, e = stored(ref, tol)
            ref, tol = chained_layer(x, e, w[l + ".weight"].T, w[l + ".bias"], rho, self.beta, kc(x), act)
        return ref, tol, chained_layer(x, e, w[l + ".weight"].T, None, rho, self.beta, kc(x), act)[0]


class StepCheck(LayerCheck):
    """The teacher-forced restatement of the step `dd` just ran from the weights `W` (a `snapshot` taken before it)."""

    def __init__(self, dd, W, plan, precision, post_update=False, label=None):
        self.tc, self.post_update = plan == "tc_chain", post_update
        dev = dd.critic.fc3.weight.device
        self.W = {k: {n_: v.to(dev) for n_, v in w.items()} for k, w in W.items()}
        # the policy pass's critic: the critic after its Adam step under actor_critic="post_update"
        self.W["p"] = ({n_: v.detach().clone() for n_, v in dd.critic.state_dict().items()} if post_update
                       else self.W["c"])
        self.N = W["c"]["fc3.weight"].shape[0]
        self.S, self.A = W["a"]["fc1.weight"].shape[1], W["a"]["fc3.weight"].shape[0]
        self.dd = dd
        B = dd.batch_size
        self.B = B
        self.t = lambda name, w=None: dd.debug_tensor(name, (B, w) if w else None)
        super().__init__(plan, precision, label or "%s/%s(%d,%d,%d,%d)" % (plan, precision, B, self.S, self.A, self.N))

    def _width(self, name):
        if name in ("actor_out", "actor_target_out", "a_dz3"):
            return self.A
        if "logits" in name:
            return self.N
        return H_

    def dev(self, name):
        return self.t(name, self._width(name))

    # ---- one layer ------------------------------------------------------------------------------------------------
    def forward(self, name, x, w, layer, act):
        """y = act(x @ W^T + b) against the device plane `name`."""
        self.layer(name, "fwd", self.dev(name), x, w[layer + ".weight"].T, w[layer + ".bias"], act)

    def backward(self, name, g, w, mask=None, tanh_y=None):
        """dX = (g @ W) * mask (or * (1 - y^2)) against the device plane `name`."""
        self.layer(name, "dX", self.dev(name), g, w, mask=mask, tanh_y=tanh_y)

    # ---- chained layers ---------------------------------------------------------------------------------------------
    def chained_refs(self, rho="plan"):
        """{output: (reference, bound, power reference)} of every output this plan computes through layers it does
        not write row-major (module docstring), from the device's planes; rho=None gives the unrounded chains."""
        rho = self.rho if rho == "plan" else rho
        t, dev, W = self.t, self.dev, self.W
        zero = lambda x: torch.zeros(x.shape, dtype=torch.float64, device=x.device)
        out = {}
        if self.post_update:      # h1 of the updated critic is recomputed on the device, not stored
            s, aout = t("s", self.S), dev("actor_out")
            h1, e1 = stored(*self.chain(s, zero(s), W["p"], (("fc1", "relu"),), rho)[:2])
            out["h2_p*"] = self.chain(torch.cat([h1, aout], 1), torch.cat([e1, zero(aout)], 1), W["p"], (("fc2", "relu"),), rho)
        if not self.tc:
            return out
        s2, at_out = t("s2", self.S), dev("actor_target_out")
        out["actor_target_out*"] = self.chain(s2, zero(s2), W["at"], (("fc1", "relu"), ("fc2", None), ("fc2_2", "relu"),
                                                                      ("fc3", "tanh")), rho)
        h1, e1 = stored(*self.chain(s2, zero(s2), W["ct"], (("fc1", "relu"),), rho)[:2])
        out["target_logits*"] = self.chain(torch.cat([h1, at_out], 1), torch.cat([e1, zero(at_out)], 1), W["ct"],
                                           (("fc2", "relu"), ("fc2_2", "relu"), ("fc3", None)), rho)
        # the dX chain p_dz22 -> p_dz2 -> a_dz3 from the device's dlogits_pi, masks and actor output
        Wp, dpi, aout = W["p"], dev("dlogits_pi"), dev("actor_out")
        m2, m3 = (dev("h2_p") > 0).double(), (dev("h3_p") > 0).double()
        kc = lambda x: x.shape[1] if self.tc_fwd else 0
        p22, e22 = stored(*chained_layer(dpi, zero(dpi), Wp["fc3.weight"], None, rho, self.beta, kc(dpi), mask=m3))
        p2 = chained_layer(p22, e22, Wp["fc2_2.weight"], None, rho, self.beta, kc(p22), mask=m2)
        p2, e2 = stored(*p2)
        w3 = Wp["fc2.weight"][:, H_:]
        ref, tol = chained_layer(p2, e2, w3, None, rho, self.beta, kc(p2), tanh_y=aout)
        # power: a_dz3 has no bias; drop the ReLU mask of p_dz2, the last layer the cluster keeps
        p2_unmasked = stored(*chained_layer(p22, e22, Wp["fc2_2.weight"], None, rho, self.beta, kc(p22)))[0]
        out["a_dz3*"] = (ref, tol, chained_layer(p2_unmasked, zero(p2), w3, None, rho, self.beta, kc(p2), tanh_y=aout)[0])
        return out

    def chained(self, refs):
        """Every output of `refs` (chained_refs) against its device plane: the propagated bound and its power at every
        batch size, the relative L2 error from CHAINED_L2_MIN_B rows on."""
        for name, (ref, tol, ref_power) in refs.items():
            dev = self.dev(name[:-1])
            self.rep.add(name, ratio(dev, ref, tol))
            self.rep.power.append((name, ratio(dev, ref_power, tol)))
            held = self.B >= CHAINED_L2_MIN_B
            self.rep.chained.append((name, rel_l2(dev, ref), CHAINED_TOL["rz" if self.rho else None][name] if held else None))

    # ---- the step ---------------------------------------------------------------------------------------------------
    def run(self):
        t, dev, W = self.t, self.dev, self.W
        S, A, N = self.S, self.A, self.N
        Wa, Wat, Wc, Wct, Wp = W["a"], W["at"], W["c"], W["ct"], W["p"]
        s, a, s2 = t("s", S), t("a", A), t("s2", S)
        f = self.forward
        ah1, ah2, ah3, aout = dev("h1_a"), dev("h2_a"), dev("h3_a"), dev("actor_out")
        f("h1_a", s, Wa, "fc1", "relu")
        f("h2_a", ah1, Wa, "fc2", None)
        f("h3_a", ah2, Wa, "fc2_2", "relu")
        f("actor_out", ah3, Wa, "fc3", "tanh")
        ch1, ch2, ch3 = dev("h1_c"), dev("h2_c"), dev("h3_c")
        f("h1_c", s, Wc, "fc1", "relu")
        f("h2_c", torch.cat([ch1, a], 1), Wc, "fc2", "relu")
        f("h3_c", ch2, Wc, "fc2_2", "relu")
        f("q_logits", ch3, Wc, "fc3", None)
        ph2, ph3 = dev("h2_p"), dev("h3_p")
        if not self.post_update:  # the policy pass's critic h1 is h1_c (post_update: chained_refs)
            f("h2_p", torch.cat([ch1, aout], 1), Wp, "fc2", "relu")
        f("h3_p", ph2, Wp, "fc2_2", "relu")
        f("pi_logits", ph3, Wp, "fc3", None)
        at_out = dev("actor_target_out")
        if not self.tc:
            th1, th2, th3 = dev("h1_at"), dev("h2_at"), dev("h3_at")
            f("h1_at", s2, Wat, "fc1", "relu")
            f("h2_at", th1, Wat, "fc2", None)
            f("h3_at", th2, Wat, "fc2_2", "relu")
            f("actor_target_out", th3, Wat, "fc3", "tanh")
            ct1, ct2, ct3 = dev("h1_ct"), dev("h2_ct"), dev("h3_ct")
            f("h1_ct", s2, Wct, "fc1", "relu")
            f("h2_ct", torch.cat([ct1, at_out], 1), Wct, "fc2", "relu")
            f("h3_ct", ct2, Wct, "fc2_2", "relu")
            f("target_logits", ct3, Wct, "fc3", None)
        self.chained(self.chained_refs())

        # backward: from the device's logit gradients, deltas and masks
        dq, dpi = dev("dlogits_q"), dev("dlogits_pi")
        m = lambda h: (h > 0).double()
        bw = self.backward
        c_dz22, c_dz2, c_dz1 = dev("c_dz22"), dev("c_dz2"), dev("c_dz1")
        bw("c_dz22", dq, Wc["fc3.weight"], m(ch3))
        bw("c_dz2", c_dz22, Wc["fc2_2.weight"], m(ch2))
        bw("c_dz1", c_dz2, Wc["fc2.weight"][:, :H_], m(ch1))
        a_dz3 = dev("a_dz3")
        if not self.tc:           # tc: p_dz22 / p_dz2 stay in the cluster (chained_refs)
            p_dz22, p_dz2 = dev("p_dz22"), dev("p_dz2")
            bw("p_dz22", dpi, Wp["fc3.weight"], m(ph3))
            bw("p_dz2", p_dz22, Wp["fc2_2.weight"], m(ph2))
            bw("a_dz3", p_dz2, Wp["fc2.weight"][:, H_:], tanh_y=aout)
        a_dz22, a_dh2, a_dz1 = dev("a_dz22"), dev("a_dh2"), dev("a_dz1")
        bw("a_dz22", a_dz3, Wa["fc3.weight"], m(ah3))
        bw("a_dh2", a_dz22, Wa["fc2_2.weight"])
        bw("a_dz1", a_dh2, Wa["fc2.weight"], m(ah1))

        # weight and bias gradients from the device's deltas and activations
        deltas = {"c": {"fc3": (dq, ch3), "fc2_2": (c_dz22, ch2), "fc2": (c_dz2, torch.cat([ch1, a], 1)), "fc1": (c_dz1, s)},
                  "a": {"fc3": (a_dz3, ah3), "fc2_2": (a_dz22, ah2), "fc2": (a_dh2, ah1), "fc1": (a_dz1, s)}}
        self.grads(deltas)
        return self.rep.finish()

    def grads(self, deltas):
        """deltas: {"c" / "a": {layer: (delta, input)}} -> every weight and bias gradient of both networks."""
        for key, net in (("c", self.dd.critic), ("a", self.dd.actor)):
            views = net.named_grad_views()
            for layer, (g, x) in deltas[key].items():
                self.grad("%s.%s.weight" % (key, layer), views[layer + ".weight"], g, x)
                self.grad("%s.%s.bias" % (key, layer), views[layer + ".bias"], g, None)


def check_step(dd, W, plan, precision, post_update=False, label=None):
    """Every layer of the step `dd` just ran (from the weights `W`) against its bound; returns (worst ratio to the
    bound, smallest power ratio) after printing one line per check."""
    return StepCheck(dd, W, plan, precision, post_update=post_update, label=label).run()
