"""CPU restatement of the quantile-regression critic (critic_dist_info type "quantile") for the tests.

DERIVED oracle: the reference has no quantile code, so this module restates the library's own definition
(include/d4pg_b200.h, d4pg_qr_loss; QR-DQN, Dabney et al. 2018) rather than reference lines.  Its learner is
oracle/d4pg_oracle.py's LearnerOracle -- the pinned networks, initialisation, Adam, Polyak and step order -- with the head
replaced, and takes the linear layer as a parameter (fp32 `F.linear`, `bf16_oracle.linear("bf16")` or
`tf32_oracle.linear("rz")`).  The head is evaluated in float64 from the fp32 quantile rows, as the kernel does:

  tau_k = (2k+1) / (2N),  y_j = r_i + c theta'_j,  u_jk = y_j - theta_k,  c = discount * (1 - done_i)
  H(u) = u^2/2 if |u| <= kappa else kappa (|u| - kappa/2),  rho_jk = |tau_k - 1{u_jk < 0}| H(u_jk) / kappa
  L_i = (1/N) sum_j sum_k rho_jk,  td_i = mean_k theta_k - (r_i + c mean_j theta'_j),  policy row = -mean_k theta_k
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import d4pg_oracle as O

CHUNK = 512          # rows per pairwise block: [CHUNK, N, N] float64 stays small at B = 4096, N = 128


def taus(N):
    return (2.0 * torch.arange(N, dtype=torch.float64) + 1.0) / (2.0 * N)


def huber(u, kappa):
    a = u.abs()
    return torch.where(a <= kappa, 0.5 * u * u, kappa * (a - 0.5 * kappa))


def targets(target_q, r, done, discount):
    """y [B, N] = r + c theta' in float64 (constant: no gradient)."""
    r = torch.as_tensor(np.asarray(r, dtype=np.float64)).view(-1, 1)
    c = discount * (1.0 - torch.as_tensor(np.asarray(done, dtype=np.float64)).view(-1, 1))
    return r + c * target_q.detach().double()


def pair_loss(y, theta, kappa):
    """L [B] = (1/N) sum_j sum_k |tau_k - 1{y_j - theta_k < 0}| H(y_j - theta_k) / kappa, differentiable in theta."""
    N = theta.shape[1]
    tau = taus(N).view(1, 1, N).to(theta.device)
    out = []
    for i in range(0, theta.shape[0], CHUNK):
        u = y[i:i + CHUNK].unsqueeze(2) - theta[i:i + CHUNK].unsqueeze(1)        # [b, j, k]
        w = (tau - (u < 0).double()).abs()
        out.append((w * huber(u, kappa)).sum((1, 2)) / (kappa * N))
    return torch.cat(out)


def loss_rows(target_q, q, r, done, discount, kappa):
    """Per-row quantile-Huber loss [B], float64, differentiable in q."""
    return pair_loss(targets(target_q, r, done, discount), q.double(), kappa)


def grad_closed_form(target_q, q, r, done, discount, kappa):
    """dL_i/dtheta_k = -(1/N) sum_j |tau_k - 1{u_jk < 0}| clamp(u_jk, -kappa, kappa) / kappa  [B, N] (the header's formula)."""
    y = targets(target_q, r, done, discount)
    th = q.detach().double()
    N = th.shape[1]
    u = y.unsqueeze(2) - th.unsqueeze(1)
    w = (taus(N).view(1, 1, N) - (u < 0).double()).abs()
    return -(w * u.clamp(-kappa, kappa)).sum(1) / (kappa * N)


def td(target_q, q, r, done, discount):
    r = torch.as_tensor(np.asarray(r, dtype=np.float64))
    c = discount * (1.0 - torch.as_tensor(np.asarray(done, dtype=np.float64)))
    return q.detach().double().mean(1) - (r + c * target_q.detach().double().mean(1))


def policy_rows(pi_q):
    return -pi_q.double().mean(1)


def heads(target_q, q, pi_q, r, done, discount, kappa, grad_scale, prio_eps=1e-6, ce_priority=False):
    """What d4pg_qr_loss computes, in float64: loss rows, td, priorities and both quantile gradients."""
    qq = q.detach().double().requires_grad_(True)
    rows = loss_rows(target_q, qq, r, done, discount, kappa)
    (rows.sum() * grad_scale).backward()
    t = td(target_q, q, r, done, discount)
    prio = (rows.detach() if ce_priority else t.abs()) + prio_eps
    out = dict(loss_rows=rows.detach(), td=t, prio=prio, dq=qq.grad)
    if pi_q is not None:
        p = pi_q.detach().double().requires_grad_(True)
        pr = policy_rows(p)
        (pr.sum() * grad_scale).backward()
        out.update(pi_rows=pr.detach(), dpi=p.grad)
    return out


class QrLearnerOracle(O.LearnerOracle):
    """O.LearnerOracle.train_step with the quantile head: the critic's raw N-wide fc3 row, the quantile-Huber loss rows,
    td and the policy rows above.  `projection` picks the discount (gamma, or gamma ** n_steps for "nstep")."""

    logits = True
    names = {"target": "target_q", "pi": "pi_q"}

    def __init__(self, obs_dim, act_dim, N, kappa=1.0, gamma=0.99, tau=0.001, n_steps=1, lr=1e-3, betas=(0.9, 0.9),
                 eps=1e-8, actor_w=None, critic_w=None, projection="live", linear=F.linear):
        self.kappa = kappa
        super().__init__(obs_dim, act_dim, N, gamma, tau, n_steps, lr, betas, eps, actor_w, critic_w, projection, linear)

    def init_head(self, N):
        self.N = N
        self.discount = self.gamma if self.projection == "live" else self.gamma ** self.n_steps
        return N

    def critic_head(self, target, q, r, done):
        return (loss_rows(target, q, r, done, self.discount, self.kappa), td(target, q, r, done, self.discount), {})

    def policy_head(self, pi):
        return policy_rows(pi)
