"""CPU restatement of the quantile-regression critic (critic_dist_info type "quantile") for the tests.

DERIVED oracle: the reference has no quantile code, so this module restates the library's own definition
(include/d4pg_b200.h, d4pg_qr_loss; QR-DQN, Dabney et al. 2018) rather than reference lines.  It reuses the MLP
restatements of tests/mog_oracle.py and the reference-pinned pieces of oracle/d4pg_oracle.py -- the initialisation, Adam,
Polyak and the PER oracle -- and takes the linear layer as a parameter (fp32 `F.linear`, `bf16_oracle.linear("bf16")`
or `tf32_oracle.linear("rz")`).  The head is evaluated in float64 from the fp32 quantile rows, as the kernel does:

  tau_k = (2k+1) / (2N),  y_j = r_i + c theta'_j,  u_jk = y_j - theta_k,  c = discount * (1 - done_i)
  H(u) = u^2/2 if |u| <= kappa else kappa (|u| - kappa/2),  rho_jk = |tau_k - 1{u_jk < 0}| H(u_jk) / kappa
  L_i = (1/N) sum_j sum_k rho_jk,  td_i = mean_k theta_k - (r_i + c mean_j theta'_j),  policy row = -mean_k theta_k
"""
import numpy as np
import torch
import torch.nn.functional as F

from oracle import d4pg_oracle as O
from tests.mog_oracle import actor_forward, critic_raw

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


class QrLearnerOracle:
    """One DDPG.train() body with the quantile critic, mirroring `MogLearnerOracle.train_step` (same Adam, Polyak,
    pre-update critic for the policy loss unless `post_update_critic`)."""

    def __init__(self, obs_dim, act_dim, N, kappa=1.0, gamma=0.99, tau=0.001, n_steps=1, lr=1e-3, betas=(0.9, 0.9),
                 eps=1e-8, actor_w=None, critic_w=None, projection="live", linear=F.linear):
        self.N, self.kappa, self.gamma, self.tau, self.n_steps = N, kappa, gamma, tau, n_steps
        self.lr, self.betas, self.eps, self.lin = lr, betas, eps, linear
        self.discount = gamma if projection == "live" else gamma ** n_steps
        self.actor = actor_w if actor_w is not None else O.init_actor(obs_dim, act_dim)
        self.actor_target = {k: v.clone() for k, v in self.actor.items()}
        self.critic = critic_w if critic_w is not None else O.init_critic(obs_dim, act_dim, N)
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

    def train_step(self, s, a, r, s2, done, is_weights=None, post_update_critic=False, ce_priority=False):
        lin = self.lin
        s_t = torch.from_numpy(np.asarray(s, dtype=O.F32))
        a_t = torch.from_numpy(np.asarray(a, dtype=O.F32))
        s2_t = torch.from_numpy(np.asarray(s2, dtype=O.F32))
        with torch.no_grad():
            tq = critic_raw(self.critic_target, s2_t, actor_forward(self.actor_target, s2_t, lin), lin)
        cw = {k: v.clone().requires_grad_(True) for k, v in self.critic.items()}
        q = critic_raw(cw, s_t, a_t, lin)
        q.retain_grad()
        raw_rows = loss_rows(tq, q, r, done, self.discount, self.kappa)
        rows = raw_rows
        if is_weights is not None:
            rows = rows * torch.from_numpy(np.asarray(is_weights, dtype=O.F32)).double()
        loss_c = rows.mean()
        loss_c.backward()
        g_c = {k: cw[k].grad.detach().clone() for k in O.PARAM_ORDER}
        t = td(tq, q, r, done, self.discount)
        if post_update_critic:
            self._adam("c", g_c)
        aw = {k: v.clone().requires_grad_(True) for k, v in self.actor.items()}
        act = actor_forward(aw, s_t, lin)
        pq = critic_raw(self.critic, s_t, act, lin)
        pq.retain_grad()
        prow = policy_rows(pq)
        loss_a = prow.mean()
        loss_a.backward()
        g_a = {k: aw[k].grad.detach().clone() for k in O.PARAM_ORDER}
        if not post_update_critic:
            self._adam("c", g_c)
        self._adam("a", g_a)
        for k in O.PARAM_ORDER:
            O.polyak(self.actor_target[k], self.actor[k], self.tau)
            O.polyak(self.critic_target[k], self.critic[k], self.tau)
        base = raw_rows.detach().numpy() if ce_priority else np.abs(t.numpy())
        prio = (base.astype(O.F32) + O.F32(1e-6)).astype(O.F32)
        return dict(target_q=tq, q=q.detach(), pi_q=pq.detach(), actor_out=act.detach(),
                    loss_rows=rows.detach(), pi_rows=prow.detach(), loss_critic=float(loss_c.detach()),
                    loss_actor=float(loss_a.detach()), td=t, prio=prio, dq=q.grad.detach(), dpi=pq.grad.detach(),
                    grads_actor=g_a, grads_critic=g_c)
