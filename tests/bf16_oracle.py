"""CPU restatement of precision="bf16" (libd4pg precision 3) for the GPU tests.

DERIVED oracle: the reference has no bf16 mode (like `her_relabel` and `post_update_critic` in oracle/d4pg_oracle.py,
it restates a variant the reference does not implement).  It is oracle/d4pg_oracle.py's networks and LearnerOracle
with only the linear layer changed (`linear("bf16")` passed as their `linear`):

  forward   y  = fp32(rb(x) @ rb(W)^T)  + b          products and sums in fp64, one cast to fp32, then the fp32 bias
  backward  dX = fp32(rb(g) @ rb(W)),  dW = fp32(rb(g)^T @ rb(x)),  db = sum(g)   (the unrounded fp32 delta)

where rb(t) = t.to(torch.bfloat16) rounds to nearest even, exactly what the kernel's cvt.rn.bf16x2.f32 does when it
stages an operand.  Everything around the GEMMs (activations, softmax, projection, loss) stays fp32 as in the oracle.
It lives beside the tests so that oracle/ keeps only code pinned to, or derived next to, the reference's own lines.
"""
import torch
import torch.nn.functional as F


def rb(t):
    """fp32 -> bf16 (round to nearest even) -> fp64: the operand the bf16 tensor cores see, held exactly."""
    return t.to(torch.bfloat16).double()


class _LinearBf16(torch.autograd.Function):
    @staticmethod
    def forward(ctx, x, w, b):
        ctx.save_for_backward(x, w)
        return (rb(x) @ rb(w).T).float() + b

    @staticmethod
    def backward(ctx, g):
        x, w = ctx.saved_tensors
        return (rb(g) @ rb(w)).float(), (rb(g).T @ rb(x)).float(), g.sum(0)


def linear(gemm):
    return _LinearBf16.apply if gemm == "bf16" else F.linear
