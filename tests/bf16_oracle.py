"""CPU restatement of precision="bf16" (libd4pg precision 3) for the GPU tests.

DERIVED oracle: the reference has no bf16 mode (like `her_relabel` and `post_update_critic` in oracle/d4pg_oracle.py,
it restates a variant the reference does not implement).  It reuses the reference-pinned pieces of
oracle/d4pg_oracle.py (projection, loss, atom support, the learner's weights) and changes only the linear layer:

  forward   y  = fp32(rb(x) @ rb(W)^T)  + b          products and sums in fp64, one cast to fp32, then the fp32 bias
  backward  dX = fp32(rb(g) @ rb(W)),  dW = fp32(rb(g)^T @ rb(x)),  db = sum(g)   (the unrounded fp32 delta)

where rb(t) = t.to(torch.bfloat16) rounds to nearest even, exactly what the kernel's cvt.rn.bf16x2.f32 does when it
stages an operand.  Everything around the GEMMs (activations, softmax, projection, loss) stays fp32 as in the oracle.
It lives beside the tests so that oracle/ keeps only code pinned to, or derived next to, the reference's own lines.
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import d4pg_oracle as O


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


def actor_forward(w, s, gemm="bf16"):
    """oracle.actor_forward with the given GEMM arithmetic (models.py:32-41)."""
    lin = linear(gemm)
    h = F.relu(lin(s, w["fc1.weight"], w["fc1.bias"]))
    h = lin(h, w["fc2.weight"], w["fc2.bias"])                       # no ReLU (H9)
    h = F.relu(lin(h, w["fc2_2.weight"], w["fc2_2.bias"]))
    return torch.tanh(lin(h, w["fc3.weight"], w["fc3.bias"]))


def critic_forward(w, s, a, logits=False, gemm="bf16"):
    """oracle.critic_forward with the given GEMM arithmetic (models.py:76-88)."""
    lin = linear(gemm)
    h = F.relu(lin(s, w["fc1.weight"], w["fc1.bias"]))
    h = F.relu(lin(torch.cat([h, a], 1), w["fc2.weight"], w["fc2.bias"]))
    h = F.relu(lin(h, w["fc2_2.weight"], w["fc2_2.bias"]))
    z = lin(h, w["fc3.weight"], w["fc3.bias"])
    return z if logits else F.softmax(z, dim=1)


def learner_gradients(lo, s, a, r, s2, done, gemm="bf16"):
    """The gradient half of `LearnerOracle.train_step` (ddpg.py:200-242) on `lo`'s current weights, with the given GEMM
    arithmetic: projection target m, both losses and both gradients.  Adam is not applied (`lo` is left unchanged)."""
    s_t = torch.from_numpy(np.asarray(s, dtype=O.F32))
    a_t = torch.from_numpy(np.asarray(a, dtype=O.F32))
    s2_t = torch.from_numpy(np.asarray(s2, dtype=O.F32))
    with torch.no_grad():
        tz = critic_forward(lo.critic_target, s2_t, actor_forward(lo.actor_target, s2_t, gemm), gemm=gemm)
    cw = {k: v.clone().requires_grad_(True) for k, v in lo.critic.items()}
    q = critic_forward(cw, s_t, a_t, gemm=gemm)
    m = lo.project(tz.numpy(), np.asarray(r, dtype=O.F64), np.asarray(done))
    m_t = torch.from_numpy(m)
    loss_c = (-(m_t * torch.log(q + 1e-10)).sum(dim=1)).mean()
    loss_c.backward()
    aw = {k: v.clone().requires_grad_(True) for k, v in lo.actor.items()}
    qp = critic_forward(lo.critic, s_t, actor_forward(aw, s_t, gemm), gemm=gemm)
    loss_a = -qp.matmul(lo.z).mean()
    loss_a.backward()
    return dict(m=m, loss_critic=loss_c.detach().numpy(), loss_actor=loss_a.detach().numpy(),
                grads_actor={k: aw[k].grad.detach().clone() for k in O.PARAM_ORDER},
                grads_critic={k: cw[k].grad.detach().clone() for k in O.PARAM_ORDER})
