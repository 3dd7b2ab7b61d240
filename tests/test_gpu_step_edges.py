"""Every layer of one learner step at the shapes where the step's kernels branch, against the teacher-forced float64
restatement and componentwise bound of tests/step_check.py.

The edges: the step plan (csrc/learner.cu step_plan) switches at batch 512 / 513, |s| or |a| 32 / 33, precision, and
where the cluster chain no longer fits one CTA (|s| 576 / 577, |a| 256 / 257, at every chain precision); the fp32
cluster chain folds the actor's fc3 into the next slot for |a| <= 8; the level plan's dW runs split-K from batch
1024 (csrc/gemm_ffma.cu prepare_problem: 1025 rows give three slices, the last of 257 rows; 3585 rows eight slices, the
last of ONE row); chain clusters own 64 rows and level tiles 128, so 65 and 513 rows leave a 1-row cluster / tile.
Every precision runs here: fp32, 3xTF32, one TF32 pass (each plan) and bf16 (the level plan).
"""
import math
import random

import numpy as np
import pytest
import torch

from tests import bf16_oracle as BO
from tests import step_check as SC
from tests import tf32_oracle as TO

KS = (1, 65, 513, 1025, 3585, 4096)


# ---- CPU: the bound itself --------------------------------------------------------------------------------------------
def _operands(K, seed=7):
    """G [K, 256] with half its entries masked to zero (a ReLU-masked delta) and X [K, 17]: dW = G^T X."""
    g = torch.Generator().manual_seed(seed + K)
    G = torch.randn(K, 256, generator=g) * (torch.rand(K, 256, generator=g) < 0.5)
    X = torch.randn(K, 17, generator=g)
    return G, X


def _split_k(G, X, ksplit, kslice):
    acc = torch.zeros(G.shape[1], X.shape[1])
    for i in range(ksplit):
        acc = acc + G[i * kslice:(i + 1) * kslice].T @ X[i * kslice:(i + 1) * kslice]
    return acc


def _emulations(G, X):
    """fp32 results of G^T X as the kernels may accumulate them, and the 3xTF32 split (rz hi / lo) of the wgmma kernels."""
    K = G.shape[0]
    out = {"fp32 matmul": G.T @ X}
    out["8-way split-K"] = _split_k(G, X, 8, -(-K // 8))
    kslice = SC.kslice(K)                                 # the level kernels' split (gemm_ffma.cu prepare_problem)
    out["level split-K"] = _split_k(G, X, -(-K // kslice), kslice)
    acc = torch.zeros(G.shape[1], X.shape[1])
    for k in range(K):                                    # one fp32 rounding per product and per sum, in row order
        acc = acc + torch.outer(G[k], X[k])
    out["sequential"] = acc
    split = lambda t: (TO.rt(t, "rz"), TO.rt((t.double() - TO.rt(t, "rz")).float(), "rz"))
    (gh, gl), (xh, xl) = split(G), split(X)
    out["3xtf32 rz"] = (gh.T @ xh + gh.T @ xl + gl.T @ xh).float()
    return out


@pytest.mark.parametrize("K", KS)
def test_bound_holds_for_fp32_split_k_sequential_and_3xtf32(K):
    """Every accumulation order a kernel may use lands within the bound (3xTF32 with beta); a result that drops the
    last row, or is all zero, lands at least 100x outside it."""
    G, X = _operands(K)
    ref, tol = SC.matmul_bound(G.T, X, None)
    tol3 = SC.matmul_bound(G.T, X, None, SC.BETA_3XTF32)[1]
    for name, dev in _emulations(G, X).items():
        r = SC.ratio(dev, ref, tol3 if "3xtf32" in name else tol)
        print("K=%d %-14s %.3f of bound" % (K, name, r))
        assert r <= 1.0, (K, name, r)
        assert SC.drop_row_ratio(dev, ref, tol3, G, X, None) >= 100, (K, name)
    dropped = G[:-1].T @ X[:-1]
    for t in (tol, tol3):
        assert SC.ratio(dropped, ref, t) >= 100, K
        assert SC.ratio(torch.zeros_like(dropped), ref, t) >= 100, K


def _truncating_sum(P):
    """Sequential fp32 sums of the rows of P with every add rounded toward zero, like the tensor cores' accumulator."""
    acc = torch.zeros(P.shape[1:], dtype=torch.float32)
    for k in range(P.shape[0]):
        x = acc.double() + P[k]
        y = x.float()
        acc = torch.where(y.double().abs() > x.abs(), torch.nextafter(y, torch.zeros_like(y)), y)
    return acc


@pytest.mark.parametrize("K", KS)
def test_truncated_accumulation_needs_and_meets_the_tensor_core_term(K):
    """Same-sign products (a ReLU activation times a delta column of one sign) summed with truncating adds: the
    truncation errors add up linearly in K, past the sqrt(K) bound from a few hundred rows, and stay within it once
    the Kc term of one accumulator is added."""
    G, X = _operands(K)
    G, X = G.abs(), X.abs()
    P = (G.double()[:, :, None] * X.double()[:, None, :]).float().double()     # exact fp32 products
    dev = _truncating_sum(P)
    ref, tol = SC.matmul_bound(G.T, X, None, kc=K)
    r = SC.ratio(dev, ref, tol)
    r_sqrt = SC.ratio(dev, ref, SC.matmul_bound(G.T, X, None)[1])
    print("K=%d truncating: %.3f of bound, %.3f of the sqrt(K) term alone" % (K, r, r_sqrt))
    assert r <= 1.0, (K, r)
    assert K < 1023 or r_sqrt > 1.0, (K, r_sqrt)
    assert SC.drop_row_ratio(dev, ref, tol, G, X, None) >= 10, K


@pytest.mark.parametrize("K", KS)
def test_bias_bound_holds_for_fp32_sums(K):
    """A bias gradient is a column sum of the fp32 delta: pairwise and sequential fp32 sums pass, a sum without the
    last row fails by at least 100x."""
    G, _ = _operands(K)
    ref, tol = G.double().sum(0), SC.bound(G.double().abs().sum(0), K)
    seq = torch.zeros(G.shape[1])
    for k in range(K):
        seq = seq + G[k]
    for dev in (G.sum(0), seq):
        assert SC.ratio(dev, ref, tol) <= 1.0
    assert SC.ratio(G[:-1].sum(0), ref, tol) >= 100
    assert SC.drop_row_ratio(G.sum(0), ref, tol, G, None, None) >= 100


@pytest.mark.parametrize("rho", ["rz", "rna", "bf16"])
def test_bound_holds_for_rounded_operands(rho):
    """One TF32 / bf16 pass: fp32 accumulation of the rounded operands' products passes the bound with beta 0 (the
    oracle reproduces the rounding), and at 65 rows the unrounded product does not (the rounding is visible; over
    thousands of rows the independent rounding errors average out toward the bound)."""
    for K in (65, 4096):
        G, X = _operands(K, seed=11)
        ref, tol = SC.matmul_bound(G.T, X, rho)
        dev = SC.rnd(G, rho).float().T @ SC.rnd(X, rho).float()
        assert SC.ratio(dev, ref, tol) <= 1.0, (rho, K)
        assert K > 65 or SC.ratio(G.T @ X, ref, tol) >= 10, (rho, K)


@pytest.mark.parametrize("rho", [None, "rz", "rna", "bf16"])
def test_operand_error_is_the_largest_rounding_change_within_e(rho):
    """operand_error against brute force: every fp32 value within e of x (e = 0 to 3 fp32 ulps), rounded, including x
    on a TF32 / bf16 rounding boundary and one ulp either side of it."""
    g = torch.Generator().manual_seed(5)
    x = torch.randn(512, generator=g)
    edge = TO.rt(x[:128], "rz").float()                        # low 13 bits zero: a TF32 boundary
    x = torch.cat([x[128:], edge, torch.nextafter(edge, torch.zeros_like(edge)), BO.rb(x[:128]).float()])
    ulp = (torch.nextafter(x, torch.full_like(x, math.inf)) - x).double()
    for k in range(4):
        e = k * ulp
        d = SC.operand_error(x, e, rho)
        want = torch.zeros_like(e)
        for s in range(-k, k + 1):                              # x + s ulp: every fp32 value within e
            y = x.clone()
            for _ in range(abs(s)):
                y = torch.nextafter(y, torch.full_like(y, math.inf if s > 0 else -math.inf))
            want = torch.maximum(want, (SC.rnd(y, rho) - SC.rnd(x, rho)).abs())
        assert torch.equal(d, want) if rho else torch.equal(d, e), (rho, k)
        if rho in ("rz", "bf16") and k:
            assert bool((d > 0).any()), (rho, k)                # the boundaries are crossed


def _mlp(S, A, gen):
    """Actor-shaped weights as models.py draws them: fan-in normal hidden layers, a narrow fc3, uniform biases."""
    w = {}
    for l, (k, n) in zip(("fc1", "fc2", "fc2_2", "fc3"), ((S, 256), (256, 256), (256, 256), (256, A))):
        w[l + ".weight"] = torch.randn(n, k, generator=gen) * (3e-3 if l == "fc3" else n ** -0.5)
        w[l + ".bias"] = (torch.rand(n, generator=gen) * 2 - 1) * k ** -0.5
    return w


ACTOR_LAYERS = (("fc1", "relu"), ("fc2", None), ("fc2_2", "relu"), ("fc3", "tanh"))


def _nudge(y, gen):
    """y moved by one fp32 ulp: toward zero where its low 13 bits are zero (on a TF32 truncation boundary, so that rz
    drops a whole TF32 ulp), away from zero where they are all ones (so that rz gains one), either way elsewhere."""
    low = y.view(torch.int32) & 0x1FFF
    up = torch.rand(y.shape, generator=gen) < 0.5
    away = torch.where(low == 0, torch.zeros_like(up), torch.where(low == 0x1FFF, torch.ones_like(up), up))
    target = torch.where(away == (y >= 0), torch.full_like(y, math.inf), torch.full_like(y, -math.inf))
    return torch.nextafter(y, target), int(((low == 0) & (y != 0)).sum() + (low == 0x1FFF).sum())


def _one_pass_chain(s, w, gen, drop_bias=None):
    """The actor chain as a one-pass rz wgmma chain computes it: fp32 products of the truncated operands and an fp32
    output, each hidden pre-activation nudged by one fp32 ulp (another accumulation order) before its activation and
    the next layer's read.  Returns (output, [hidden layers], boundary elements nudged)."""
    x, hidden, edges = s, [], 0
    for i, (l, act) in enumerate(ACTOR_LAYERS):
        b = torch.zeros_like(w[l + ".bias"]) if l == drop_bias else w[l + ".bias"]
        y = TO.rt(x, "rz").float() @ TO.rt(w[l + ".weight"], "rz").float().T + b
        if i + 1 < len(ACTOR_LAYERS):
            y, n = _nudge(y, gen)
            edges += n
        x = torch.relu(y) if act == "relu" else torch.tanh(y) if act == "tanh" else y
        hidden.append(x)
    return x, hidden[:-1], edges


def _chain_bound(s, w):
    """(reference, bound) of every layer of the actor chain from the device plane s, as step_check chains them."""
    x, e, out = s, torch.zeros(s.shape, dtype=torch.float64), []
    for i, (l, act) in enumerate(ACTOR_LAYERS):
        if i:
            x, e = SC.stored(*out[-1])
        out.append(SC.chained_layer(x, e, w[l + ".weight"].T, w[l + ".bias"], "rz", 0.0, x.shape[1], act))
    return out


@pytest.mark.parametrize("B", [1, 65, 512])
def test_chained_bound_holds_for_a_nudged_one_pass_chain(B):
    """A one-pass rz chain whose hidden pre-activations are each one fp32 ulp off, many of them across a TF32 truncation
    boundary, stays within the propagated bound at every layer, one row as well as 512."""
    gen = torch.Generator().manual_seed(B)
    S, A = 17, 6
    w, s = _mlp(S, A, gen), torch.randn(B, S, generator=gen)
    bounds = _chain_bound(s, w)
    out, hidden, edges = _one_pass_chain(s, w, gen)
    for i, (dev, (ref, tol)) in enumerate(zip(hidden + [out], bounds)):
        r = SC.ratio(dev, ref, tol)
        print("B=%d layer %d: %.3f of bound" % (B, i + 1, r))
        assert r <= 1.0, (B, i, r)
    assert B < 512 or edges >= 10, edges


@pytest.mark.parametrize("B", [1, 65, 512])
def test_chained_bound_rejects_a_dropped_last_bias(B):
    """The same chain without its last layer's bias lands at least POWER_MIN x outside the bound of its output.  An
    earlier layer's bias is no such witness: the propagated bound grows by up to ~sqrt(256) per chained layer (|W| d
    against W x)."""
    gen = torch.Generator().manual_seed(B)
    S, A = 17, 6
    w, s = _mlp(S, A, gen), torch.randn(B, S, generator=gen)
    ref, tol = _chain_bound(s, w)[-1]
    out = _one_pass_chain(s, w, gen, drop_bias="fc3")[0]
    r = SC.ratio(out, ref, tol)
    print("B=%d without fc3.bias: %.3g x bound" % (B, r))
    assert r >= SC.POWER_MIN, (B, r)


def test_ratio_demands_exact_zero_where_every_product_is_zero():
    ref, tol = torch.zeros(3, dtype=torch.float64), torch.zeros(3, dtype=torch.float64)
    assert SC.ratio(torch.zeros(3), ref, tol) == 0.0
    assert SC.ratio(torch.tensor([0.0, 1e-30, 0.0]), ref, tol) == float("inf")


# ---- GPU: one eager step per edge --------------------------------------------------------------------------------------
def _cat(N, v=(-50.0, 0.0)):
    return {"type": "categorical", "v_min": v[0], "v_max": v[1], "n_atoms": N}


def _qr(N):
    return {"type": "quantile", "n_quantiles": N}


def _mog(K):
    return {"type": "mixture_of_gaussian", "n_components": K}


C5 = dict(projection="nstep", n_steps=5)
# (plan, precision, B, |s|, |a|, critic head, DDPG options); each comment names the edge
CASES = [
    # wgmma chains, 3xTF32
    ("tc_chain", "tf32x3", 1, 1, 1, _cat(2), {}),                       # a single row, minimal widths
    ("tc_chain", "tf32x3", 65, 32, 32, _cat(128), {}),                  # 1-row second cluster, wgmma width limits, max atoms
    ("tc_chain", "tf32x3", 511, 17, 6, _cat(51), {"use_graph": True}),  # CUDA graph, one row short of the chain limit
    ("tc_chain", "tf32x3", 64, 17, 6, _cat(51), {"actor_critic": "post_update"}),   # policy pass through the updated critic
    ("tc_chain", "tf32x3", 65, 17, 6, _mog(32), {}),                    # mixture head, K = 32: 96 columns
    ("tc_chain", "tf32x3", 256, 17, 6, _cat(51), {}),                   # config 2
    ("tc_chain", "tf32x3", 256, 17, 6, _cat(51), {"use_graph": True}),
    ("tc_chain", "tf32x3", 64, 17, 6, _cat(51), {}),
    ("tc_chain", "tf32x3", 200, 3, 1, _cat(101), {}),                   # ragged last cluster
    ("tc_chain", "tf32x3", 512, 32, 8, _cat(64), {}),                   # the chain plan's batch limit
    ("tc_chain", "tf32x3", 40, 17, 6, _cat(51), {"use_graph": True}),
    # mma.sync chains, 3xTF32
    ("chain", "tf32x3", 96, 376, 17, _cat(51), {}),                     # config 3 widths
    ("chain", "tf32x3", 65, 33, 6, _cat(51), {}),                       # |s| = 33: one past the wgmma chain
    ("chain", "tf32x3", 130, 17, 33, _cat(128), {}),                    # |a| = 33, max atoms, 2-row last cluster
    # FFMA chains, fp32
    ("chain", "fp32", 1, 1, 1, _cat(2), {}),                            # a single row, minimal widths
    ("chain", "fp32", 65, 17, 8, _cat(51), {}),                         # |a| = 8: actor fc3 as a pre-layer
    ("chain", "fp32", 65, 17, 9, _cat(51), {}),                         # |a| = 9: actor fc3 as a slot of its own
    ("chain", "fp32", 512, 376, 17, _cat(128), {}),                     # batch limit, config 3 widths, max atoms
    # the chain's shared-memory and width limits (csrc/mlp_chain.cu chain_fits): fc1 holds all |s| columns, 222,208 B
    # at |s| = 576; a layer is at most 256 wide
    ("chain", "fp32", 512, 576, 6, _cat(51), {}),                       # the largest fc1 slot, pre-layer fc3
    ("chain", "tf32x3", 256, 576, 17, _cat(101), {}),
    ("chain", "fp32", 128, 17, 256, _cat(51), {}),                      # |a| = 256: actor fc3 on all 8 cluster ranks
    # one past them: the level plan
    ("levels", "fp32", 256, 577, 6, _cat(51), {}),                      # 230,528 B
    ("levels", "tf32x3", 256, 577, 17, _cat(51), {}),
    ("levels", "fp32", 64, 17, 257, _cat(51), {}),                      # actor fc3 257 wide
    ("levels", "tf32x3", 512, 700, 6, _qr(51), {}),                     # quantile head
    ("levels", "fp32", 1025, 2053, 6, _cat(51), {}),                    # split-K dW with fc1 K = 2053, not a multiple of 4
]
for _p in ("fp32", "tf32x3"):
    CASES += [
        ("levels", _p, 513, 17, 6, _cat(51), {}),                       # 1-row last level tile
        ("levels", _p, 1023, 376, 17, _cat(51), {}),                    # the largest unsplit dW
        ("levels", _p, 1025, 17, 6, _cat(101), {}),                     # split-K: 3 slices, the last of 257 rows
        ("levels", _p, 4096, 17, 6, _cat(101, (-150.0, 150.0)), C5),    # config 5: n-step projection, 8 slices
        ("levels", _p, 1, 1, 1, _cat(2), {"chain": "levels"}),          # a single row through the level kernels
        ("levels", _p, 1025, 17, 6, _qr(128), {}),                      # quantile head, N = 128, split-K
    ]
CASES += [("levels", "fp32", 3585, 17, 6, _cat(101), {}),               # split-K: 8 slices, the last of ONE row
          ("levels", "tf32x3", 3585, 33, 33, _cat(128), {})]
# One TF32 pass (precision 2).  The chain limits are those of fp32 and 3xTF32: chain_fits (csrc/mlp_chain.cu) holds
# one A plane and two weight slices of the widest slot in 220 KiB, and a layer to 256 columns.  At precision 2 the A
# plane's floor is the 9,216-float reduce buffer (8 warps x 32 rows x pitch 36), below fc1's 32 |s| floats from
# |s| = 288 on, so fc1 still sets it: 222,208 B at |s| = 576, 230,528 B at 577.  Actor fc3 and the d-action layer are
# |a| wide: 256 fits, 257 does not.  The wgmma chain (tc_chain) takes |s|, |a| <= 32 first (step_plan).
CASES += [
    # wgmma chains, one pass (rz operands)
    ("tc_chain", "tf32", 1, 1, 1, _cat(2), {}),                         # a single row, minimal widths
    ("tc_chain", "tf32", 65, 32, 32, _cat(128), {}),                    # 1-row second cluster, wgmma width limits, max atoms
    ("tc_chain", "tf32", 511, 17, 6, _cat(51), {"use_graph": True}),    # CUDA graph, one row short of the chain limit
    ("tc_chain", "tf32", 64, 17, 6, _cat(51), {"actor_critic": "post_update"}),     # policy pass through the updated critic
    ("tc_chain", "tf32", 65, 17, 6, _mog(32), {}),                      # mixture head, K = 32: 96 columns
    ("tc_chain", "tf32", 200, 3, 1, _cat(101), {}),                     # ragged last cluster
    ("tc_chain", "tf32", 512, 32, 8, _cat(64), {}),                     # the chain plan's batch limit
    # mma.sync chains, one pass (rna operands)
    ("chain", "tf32", 65, 33, 6, _cat(51), {}),                         # |s| = 33: one past the wgmma chain
    ("chain", "tf32", 130, 17, 33, _cat(128), {}),                      # |a| = 33, max atoms, 2-row last cluster
    ("chain", "tf32", 512, 376, 17, _cat(128), {}),                     # batch limit, config 3 widths, max atoms
    ("chain", "tf32", 256, 576, 17, _cat(101), {}),                     # the largest fc1 slot at precision 2
    ("chain", "tf32", 128, 17, 256, _cat(51), {}),                      # the widest actor fc3 at precision 2
    # level kernels, one pass (rz operands, dW included)
    ("levels", "tf32", 256, 577, 6, _cat(51), {}),                      # one past the chain's fc1 slot
    ("levels", "tf32", 64, 17, 257, _cat(51), {}),                      # one past the chain's layer width
    ("levels", "tf32", 512, 700, 6, _qr(51), {}),                       # quantile head
    ("levels", "tf32", 1025, 2053, 6, _cat(51), {}),                    # split-K dW with fc1 K = 2053, not a multiple of 4
    ("levels", "tf32", 513, 17, 6, _cat(51), {}),                       # 1-row last level tile
    ("levels", "tf32", 1023, 376, 17, _cat(51), {}),                    # the largest unsplit dW
    ("levels", "tf32", 1025, 17, 6, _cat(101), {}),                     # split-K: 3 slices, the last of 257 rows
    ("levels", "tf32", 3585, 17, 6, _cat(101), {}),                     # split-K: 8 slices, the last of ONE row
    ("levels", "tf32", 4096, 17, 6, _cat(101, (-150.0, 150.0)), C5),    # config 5 shapes
    ("levels", "tf32", 1, 1, 1, _cat(2), {"chain": "levels"}),          # a single row through the level kernels
    ("levels", "tf32", 1025, 17, 6, _qr(128), {}),                      # quantile head, N = 128, split-K
    # bf16: the level kernels only (step_plan), gemm_bf16.cu.  Its operand staging is float4 where K % 4 == 0
    # (forward) or N % 4 == 0 (transposed stage), scalar otherwise: |s| 576 / 577 and |a| 256 / 257 take both
    ("levels", "bf16", 1, 1, 1, _cat(2), {}),                           # a single row, minimal widths
    ("levels", "bf16", 65, 17, 6, _cat(51), {}),                        # dW: the last 64-deep K chunk holds one row
    ("levels", "bf16", 511, 17, 6, _cat(51), {"use_graph": True}),      # CUDA graph
    ("levels", "bf16", 513, 17, 6, _cat(51), {}),                       # 1-row last level tile
    ("levels", "bf16", 1023, 376, 17, _cat(51), {}),                    # the largest unsplit dW, scalar concat tail (|a| 17)
    ("levels", "bf16", 1025, 17, 6, _cat(101), {}),                     # split-K: 3 slices, the last of 257 rows (odd)
    ("levels", "bf16", 3585, 33, 33, _cat(128), {}),                    # split-K: 8 slices, the last of ONE row
    ("levels", "bf16", 4096, 17, 6, _cat(101, (-150.0, 150.0)), C5),    # config 5
    ("levels", "bf16", 256, 576, 6, _cat(51), {}),                      # fc1 K = 576: float4 staging
    ("levels", "bf16", 256, 577, 6, _cat(51), {}),                      # fc1 K = 577: scalar staging
    ("levels", "bf16", 128, 17, 256, _cat(51), {}),                     # actor fc3 N = 256: float4 transposed stage
    ("levels", "bf16", 64, 17, 257, _cat(51), {}),                      # actor fc3 N = 257: scalar transposed stage
    ("levels", "bf16", 1025, 2053, 6, _cat(51), {}),                    # split-K dW with fc1 K = 2053
    ("levels", "bf16", 1025, 17, 6, _qr(128), {}),                      # quantile head, N = 128, split-K
    ("levels", "bf16", 65, 17, 6, _mog(32), {}),                        # mixture head, K = 32: 96 columns
]
ONE_PASS = [("tc_chain", "tf32"), ("chain", "tf32"), ("levels", "tf32"), ("levels", "bf16")]


def _id(case):
    plan, prec, B, S, A, info, kw = case
    head = {"categorical": "N", "quantile": "qr", "mixture_of_gaussian": "mogK"}[info["type"]]
    width = info.get("n_atoms") or info.get("n_quantiles") or info.get("n_components")
    return "%s-%s-B%d-s%d-a%d-%s%d%s" % (plan, prec, B, S, A, head, width, "".join("-%s" % (k if v is True else v) for k, v in kw.items()))


def _ddpg(d4pg, B, S, A, info, precision, seed=12, **kw):
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    n = max(2048, 2 * B)
    opts = dict(use_graph=False, chain="cluster")
    opts.update(kw)
    dd = d4pg.DDPG(S, A, memory_size=n, batch_size=B, critic_dist_info=info, precision=precision, sampling="device",
                   philox_seed=3, prefetch=False, **opts)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(seed + 1)
    dd.replayBuffer.add_batch(rng.randn(n, S).astype(np.float32), rng.uniform(-1, 1, (n, A)).astype(np.float32),
                              (-3 * rng.rand(n)).astype(np.float32).astype(np.float64), rng.randn(n, S).astype(np.float32),
                              rng.rand(n) < 0.05)
    with torch.no_grad():                     # the target networks differ from the online ones
        dd.actor_target.flat_params().mul_(1.01)
        dd.critic_target.flat_params().mul_(0.99)
    return dd


# (plan, precision) -> the largest ratio of any forward / dX layer to the bound of the UNROUNDED layer, over the one-pass
# cases run so far
_SEPARATION = {}


def _run_case(case):
    import d4pg_b200 as d4pg
    plan, precision, B, S, A, info, kw = case
    post_update = kw.get("actor_critic") == "post_update"
    dd = _ddpg(d4pg, B, S, A, info, precision, **kw)
    W = SC.snapshot(dd)
    dd.train()
    torch.cuda.synchronize()
    if not post_update:                       # the post-update critic adds its own launches
        assert dd.kernels_per_step() == SC.KERNELS[plan], (plan, dd.kernels_per_step())
    sc = SC.StepCheck(dd, W, plan, precision, post_update=post_update, label=_id(case))
    sc.run()
    if sc.rep.sep:
        sep = _SEPARATION.setdefault((plan, precision), {"fwd": 0.0, "dX": 0.0})
        for kind, _, r in sc.rep.sep:
            sep[kind] = max(sep[kind], r)


@pytest.mark.gpu
@pytest.mark.parametrize("case", CASES, ids=[_id(c) for c in CASES])
def test_step_every_layer_at_plan_tile_and_split_k_edges(case):
    _run_case(case)


@pytest.mark.gpu
@pytest.mark.parametrize("plan,precision", ONE_PASS, ids=["%s-%s" % p for p in ONE_PASS])
def test_one_pass_rounding_is_present_and_applied_once(plan, precision):
    """Across the cases of a one-pass (plan, precision), at least one forward and one dX layer land more than 10x the
    bound of the unrounded layer away from it: the operands are rounded, and only once (a kernel that quietly ran
    3xTF32 or fp32 would be within that bound).  Where none of its cases ran in this session, the first one runs here.
    Not every case is a witness: over a deep fc1 (|s| >= 376) the independent round-to-nearest errors of the mma.sync
    chain average out to within ~10x of the bound."""
    if (plan, precision) not in _SEPARATION:
        _run_case(next(c for c in CASES if c[:2] == (plan, precision)))
    sep = _SEPARATION[plan, precision]
    print("%s/%s: forward %.3g x, dX %.3g x the unrounded bound" % (plan, precision, sep["fwd"], sep["dX"]))
    assert sep["fwd"] > 10 and sep["dX"] > 10, (plan, precision, sep)
