"""CPU restatement of the mixture-of-Gaussians critic (critic_dist_info type "mixture_of_gaussian") for the tests.

DERIVED oracle: the reference stubs its mixture branch (`TODO: pass`, ddpg.py:48-50, models.py:63-65), so this module
restates the library's own definition (include/d4pg_b200.h, d4pg_mog_loss) rather than reference lines.  It reuses the
reference-pinned pieces of oracle/d4pg_oracle.py -- the initialisation, Adam, Polyak and the PER oracle -- and takes
the linear layer as a parameter (fp32 `F.linear`, or `bf16_oracle.linear("bf16")`).  The head itself is evaluated in
float64 from the fp32 raw head, as the kernel does:

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


def actor_forward(w, s, lin=F.linear):
    h = F.relu(lin(s, w["fc1.weight"], w["fc1.bias"]))
    h = lin(h, w["fc2.weight"], w["fc2.bias"])                       # no ReLU (H9)
    h = F.relu(lin(h, w["fc2_2.weight"], w["fc2_2.bias"]))
    return torch.tanh(lin(h, w["fc3.weight"], w["fc3.bias"]))


def critic_raw(w, s, a, lin=F.linear):
    """The critic MLP up to its 3K-wide fc3 output (no head transform)."""
    h = F.relu(lin(s, w["fc1.weight"], w["fc1.bias"]))
    h = F.relu(lin(torch.cat([h, a], 1), w["fc2.weight"], w["fc2.bias"]))
    h = F.relu(lin(h, w["fc2_2.weight"], w["fc2_2.bias"]))
    return lin(h, w["fc3.weight"], w["fc3.bias"])


class MogLearnerOracle:
    """One DDPG.train() body with the mixture critic, mirroring `LearnerOracle.train_step` (same Adam, Polyak,
    pre-update critic for the policy loss unless `post_update_critic`)."""

    def __init__(self, obs_dim, act_dim, K, gamma=0.99, tau=0.001, n_steps=1, lr=1e-3, betas=(0.9, 0.9), eps=1e-8,
                 actor_w=None, critic_w=None, projection="live", linear=F.linear):
        self.K, self.gamma, self.tau, self.n_steps = K, gamma, tau, n_steps
        self.lr, self.betas, self.eps, self.lin = lr, betas, eps, linear
        self.discount = gamma if projection == "live" else gamma ** n_steps
        self.actor = actor_w if actor_w is not None else O.init_actor(obs_dim, act_dim)
        self.actor_target = {k: v.clone() for k, v in self.actor.items()}
        self.critic = critic_w if critic_w is not None else O.init_critic(obs_dim, act_dim, 3 * K)
        self.critic_target = {k: v.clone() for k, v in self.critic.items()}
        z = lambda d: {k: torch.zeros_like(v) for k, v in d.items()}
        self.m_a, self.v_a, self.m_c, self.v_c = z(self.actor), z(self.actor), z(self.critic), z(self.critic)
        self.step_a = self.step_c = 0

    def _adam(self, which, g):
        p, m, v = (self.critic, self.m_c, self.v_c) if which == "c" else (self.actor, self.m_a, self.v_a)
        if which == "c":
            self.step_c += 1
        else:
            self.step_a += 1
        for k in O.PARAM_ORDER:
            O.adam_step(p[k], g[k], m[k], v[k], self.step_c if which == "c" else self.step_a, self.lr,
                        self.betas[0], self.betas[1], self.eps)

    def train_step(self, s, a, r, s2, done, is_weights=None, post_update_critic=False):
        lin, K = self.lin, self.K
        s_t = torch.from_numpy(np.asarray(s, dtype=O.F32))
        a_t = torch.from_numpy(np.asarray(a, dtype=O.F32))
        s2_t = torch.from_numpy(np.asarray(s2, dtype=O.F32))
        with torch.no_grad():
            traw = critic_raw(self.critic_target, s2_t, actor_forward(self.actor_target, s2_t, lin), lin)
        cw = {k: v.clone().requires_grad_(True) for k, v in self.critic.items()}
        qraw = critic_raw(cw, s_t, a_t, lin)
        qraw.retain_grad()
        rows = loss_rows(traw, qraw, r, done, self.discount, K)
        if is_weights is not None:
            rows = rows * torch.from_numpy(np.asarray(is_weights, dtype=O.F32)).double()
        loss_c = rows.mean()
        loss_c.backward()
        g_c = {k: cw[k].grad.detach().clone() for k in O.PARAM_ORDER}
        t = td(traw, qraw, r, done, self.discount, K)
        if post_update_critic:
            self._adam("c", g_c)
        aw = {k: v.clone().requires_grad_(True) for k, v in self.actor.items()}
        act = actor_forward(aw, s_t, lin)
        praw = critic_raw(self.critic, s_t, act, lin)
        praw.retain_grad()
        prow = policy_rows(praw, K)
        loss_a = prow.mean()
        loss_a.backward()
        g_a = {k: aw[k].grad.detach().clone() for k in O.PARAM_ORDER}
        if not post_update_critic:
            self._adam("c", g_c)
        self._adam("a", g_a)
        for k in O.PARAM_ORDER:
            O.polyak(self.actor_target[k], self.actor[k], self.tau)
            O.polyak(self.critic_target[k], self.critic[k], self.tau)
        prio = (np.abs(t.numpy()).astype(O.F32) + O.F32(1e-6)).astype(O.F32)
        return dict(target_raw=traw, q_raw=qraw.detach(), pi_raw=praw.detach(), actor_out=act.detach(),
                    loss_rows=rows.detach(), pi_rows=prow.detach(), loss_critic=float(loss_c.detach()), loss_actor=float(loss_a.detach()),
                    td=t, prio=prio, dq_raw=qraw.grad.detach(), dpi_raw=praw.grad.detach(),
                    grads_actor=g_a, grads_critic=g_c)
