"""CPU restatement of the mixture-of-Gaussians critic (critic_dist_info type "mixture_of_gaussian") for the tests.

DERIVED oracle: the reference stubs its mixture branch (`TODO: pass`, ddpg.py:48-50, models.py:63-65), so this module
restates the library's own definition (include/d4pg_b200.h, d4pg_mog_loss) rather than reference lines.  Its learner
is oracle/d4pg_oracle.py's LearnerOracle -- the pinned networks, initialisation, Adam, Polyak and step order -- with the
head replaced, and takes the linear layer as a parameter (fp32 `F.linear`, or `bf16_oracle.linear("bf16")`).  The head
itself is evaluated in float64 from the fp32 raw head, as the kernel does:

  w = softmax(o[:, :K]),  mu = o[:, K:2K],  sigma = softplus(o[:, 2K:]) + 1e-3
  L_i = -sum_{k,q} w'_k h_q / sqrt(pi) * log p(r_i + c (mu'_k + sqrt(2) sigma'_k x_q)),   c = discount * (1 - done_i)
  td_i = sum_j w_j mu_j - (r_i + c sum_k w'_k mu'_k),  policy row = -sum_j w_j mu_j
with (x_q, h_q) = numpy.polynomial.hermite.hermgauss(8).
"""
import math

import numpy as np
import torch
import torch.nn.functional as F

from oracle import d4pg_oracle as O

Q = 8
X, HW = np.polynomial.hermite.hermgauss(Q)


def head(o, K):
    """raw [B, 3K] -> (w, mu, sigma), each [B, K], in o's dtype."""
    return F.softmax(o[:, :K], dim=1), o[:, K:2 * K], F.softplus(o[:, 2 * K:3 * K]) + 1e-3


def target_points(target_raw, r, done, discount, K):
    """Quadrature points y [B, K*Q] and weights omega [B, K*Q] of the target mixture (constant: no gradient)."""
    tw, tmu, tsig = head(target_raw.detach().double(), K)
    r = torch.as_tensor(np.asarray(r, dtype=np.float64)).view(-1, 1, 1)
    c = discount * (1.0 - torch.as_tensor(np.asarray(done, dtype=np.float64)).view(-1, 1, 1))
    x = torch.from_numpy(X).view(1, 1, Q)
    h = torch.from_numpy(HW).view(1, 1, Q)
    y = r + c * (tmu.unsqueeze(2) + math.sqrt(2.0) * tsig.unsqueeze(2) * x)
    om = tw.unsqueeze(2) * h / math.sqrt(math.pi)
    B = y.shape[0]
    return y.reshape(B, -1), om.reshape(B, -1)


def log_density(y, w, mu, sigma):
    """log p(y) of the mixture (w, mu, sigma) [B, K] at points y [B, P] -> [B, P]."""
    z = (y.unsqueeze(2) - mu.unsqueeze(1)) / sigma.unsqueeze(1)
    l = torch.log(w).unsqueeze(1) - torch.log(sigma).unsqueeze(1) - 0.5 * math.log(2 * math.pi) - 0.5 * z * z
    return torch.logsumexp(l, dim=2)


def loss_rows(target_raw, q_raw, r, done, discount, K):
    """Per-row quadrature cross-entropy [B], float64, differentiable in q_raw."""
    y, om = target_points(target_raw, r, done, discount, K)
    return -(om * log_density(y, *head(q_raw.double(), K))).sum(1)


def td(target_raw, q_raw, r, done, discount, K):
    w, mu, _ = head(q_raw.detach().double(), K)
    tw, tmu, _ = head(target_raw.detach().double(), K)
    r = torch.as_tensor(np.asarray(r, dtype=np.float64))
    c = discount * (1.0 - torch.as_tensor(np.asarray(done, dtype=np.float64)))
    return (w * mu).sum(1) - (r + c * (tw * tmu).sum(1))


def policy_rows(pi_raw, K):
    w, mu, _ = head(pi_raw.double(), K)
    return -(w * mu).sum(1)


def heads(target_raw, q_raw, pi_raw, r, done, discount, K, grad_scale, prio_eps=1e-6):
    """What d4pg_mog_loss computes, in float64: loss rows, td, priorities and both raw-head gradients."""
    q = q_raw.detach().double().requires_grad_(True)
    rows = loss_rows(target_raw, q, r, done, discount, K)
    (rows.sum() * grad_scale).backward()
    t = td(target_raw, q_raw, r, done, discount, K)
    out = dict(loss_rows=rows.detach(), td=t, prio=t.abs() + prio_eps, dq_raw=q.grad)
    if pi_raw is not None:
        p = pi_raw.detach().double().requires_grad_(True)
        pr = policy_rows(p, K)
        (pr.sum() * grad_scale).backward()
        out.update(pi_rows=pr.detach(), dpi_raw=p.grad)
    return out


class MogLearnerOracle(O.LearnerOracle):
    """O.LearnerOracle.train_step with the mixture head: the critic's raw 3K-wide fc3 row, the quadrature loss rows,
    td and the policy rows above.  `projection` picks the discount (gamma, or gamma ** n_steps for "nstep")."""

    logits = True
    names = {"target": "target_raw", "q": "q_raw", "pi": "pi_raw", "dq": "dq_raw", "dpi": "dpi_raw"}

    def __init__(self, obs_dim, act_dim, K, gamma=0.99, tau=0.001, n_steps=1, lr=1e-3, betas=(0.9, 0.9), eps=1e-8,
                 actor_w=None, critic_w=None, projection="live", linear=F.linear):
        super().__init__(obs_dim, act_dim, K, gamma, tau, n_steps, lr, betas, eps, actor_w, critic_w, projection, linear)

    def init_head(self, K):
        self.K = K
        self.discount = self.gamma if self.projection == "live" else self.gamma ** self.n_steps
        return 3 * K

    def critic_head(self, target, q, r, done):
        return (loss_rows(target, q, r, done, self.discount, self.K), td(target, q, r, done, self.discount, self.K),
                {})

    def policy_head(self, pi):
        return policy_rows(pi, self.K)

    def priority(self, rows, td, ce_priority):
        if ce_priority:
            raise ValueError("the mixture critic has no cross-entropy priority (DDPG rejects priority=\"ce\" with it)")
        return super().priority(rows, td, False)
