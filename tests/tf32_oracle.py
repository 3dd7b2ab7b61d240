"""CPU restatement of precision="tf32" (libd4pg precision 2) for the GPU tests.

DERIVED oracle: the reference has no TF32 mode (like tests/bf16_oracle.py, it restates a variant the reference does
not implement).  Only the linear layer changes:

  forward   y  = fp32(rt(x) @ rt(W)^T) + b          products and sums in fp64, one cast to fp32, then the fp32 bias
  backward  dX = fp32(rt(g) @ rt(W)),  dW = fp32(rt(g)^T @ rt(x)),  db = sum(g)   (the unrounded fp32 delta)

where rt(t, mode) takes each fp32 operand to TF32 (10 explicit mantissa bits) the way the kernel that runs the layer
does it:

  "rz"   bits & ~0x1FFF               round toward zero: tf32_hi of the wgmma kernels (gemm_tc.cu, mlp_tc_chain.cu)
  "rna"  (bits + 0x1000) & ~0x1FFF    round to nearest, ties away from zero: PTX cvt.rna.tf32.f32 (mlp_chain.cu)

Both work on the magnitude bits, so they are symmetric in the sign.  The chain plans compute dW with exact fp32 FFMA
(gemm_wide_kernel), so `linear(mode, round_dw=False)` keeps dW unrounded.
"""
import torch

_LOW13 = -8192                                   # ~0x1FFF as an int32 mask


def rt(t, mode="rz"):
    """fp32 -> TF32 by `mode` ("rz" or "rna") -> fp64: the operand the TF32 tensor cores see, held exactly."""
    bits = t.detach().float().contiguous().view(torch.int32)
    if mode == "rz":
        bits = bits & _LOW13
    elif mode == "rna":
        bits = (bits + 0x1000) & _LOW13
    else:
        raise ValueError("rt: unknown rounding %r" % (mode,))
    return bits.view(torch.float32).double()


def _make_linear(mode, round_dw):
    class _LinearTf32(torch.autograd.Function):
        @staticmethod
        def forward(ctx, x, w, b):
            ctx.save_for_backward(x, w)
            return (rt(x, mode) @ rt(w, mode).T).float() + b

        @staticmethod
        def backward(ctx, g):
            x, w = ctx.saved_tensors
            dw = (rt(g, mode).T @ rt(x, mode)) if round_dw else (g.double().T @ x.double())
            return (rt(g, mode) @ rt(w, mode)).float(), dw.float(), g.sum(0)

    return _LinearTf32.apply


_LINEARS = {(m, r): _make_linear(m, r) for m in ("rz", "rna") for r in (True, False)}


def linear(mode="rz", round_dw=True):
    """The TF32 linear layer as an autograd function of (x, W, b); round_dw=False keeps dW unrounded (chain plans)."""
    return _LINEARS[mode, round_dw]
