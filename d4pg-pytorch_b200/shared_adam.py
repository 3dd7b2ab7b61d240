"""`SharedAdam` with the reference signature (shared_adam.py:3-17): Adam with betas=(0.9, 0.9)
and pre-allocated moments.  The moments are ONE flat fp32 device buffer per network (matching
the flat parameter buffer of `models._FlatNet`); `DDPG.train` hands them to the fused
Adam+Polyak kernel, and `step()` itself runs the same kernel (no target update) for callers
that drive the optimiser directly.  `weight_decay` is torch.optim.Adam's (L2: `wd * p` added to the
gradient); `max_grad_norm` clips this optimiser's gradient to a global norm first, as
`torch.nn.utils.clip_grad_norm_` before `step()` would.  The reference's `share_memory_()` of the moments
(cross-process Hogwild) has no device equivalent and is a no-op here.
"""
import math

import torch

from . import _lib


def check_max_grad_norm(x):
    """A clipping threshold as float: None -> 0.0 (off); otherwise > 0, where inf measures and reports without clipping."""
    if x is None:
        return 0.0
    x = float(x)
    if not x > 0.0:
        raise ValueError("max_grad_norm must be None, a positive number or inf, got %r" % (x,))
    return x


class SharedAdam(torch.optim.Optimizer):
    def __init__(self, params, lr=1e-3, betas=(0.9, 0.9), eps=1e-8, weight_decay=0, max_grad_norm=None):
        if not (math.isfinite(weight_decay) and weight_decay >= 0):
            raise ValueError("weight_decay must be finite and >= 0, got %r" % (weight_decay,))
        self.max_grad_norm = check_max_grad_norm(max_grad_norm)       # of step(); DDPG.train() takes DDPG's own
        self._clip_ws = {}                                            # per owner: (64 fp64 partial sums, the norm)
        defaults = dict(lr=lr, betas=betas, eps=eps, weight_decay=weight_decay)
        super(SharedAdam, self).__init__(list(params), defaults)
        self._owners = []
        self._moments = {}
        self.step_count = 0
        for group in self.param_groups:
            for p in group["params"]:
                owner = getattr(p, "_d4pg_owner", None)
                if owner is None:
                    raise TypeError("SharedAdam expects parameters of d4pg `actor`/`critic` modules")
                if not any(owner is o for o in self._owners):
                    self._owners.append(owner)
        for owner in self._owners:
            self._alloc(owner)

    def _alloc(self, owner):
        flat = owner.flat_params()
        m, v = torch.zeros_like(flat), torch.zeros_like(flat)
        self._moments[id(owner)] = (m, v)
        for (mw, mb), (vw, vb), name in zip(owner._views(m), owner._views(v), ("fc1", "fc2", "fc2_2", "fc3")):
            layer = getattr(owner, name)
            self.state[layer.weight] = {"step": 0, "exp_avg": mw, "exp_avg_sq": vw}
            self.state[layer.bias] = {"step": 0, "exp_avg": mb, "exp_avg_sq": vb}

    def moments(self, owner):
        """(exp_avg, exp_avg_sq) flat buffers for `owner`, re-allocated if it moved device."""
        m, v = self._moments[id(owner)]
        if m.device != owner.flat_params().device:
            self._alloc(owner)
            m, v = self._moments[id(owner)]
        return m, v

    @property
    def owners(self):
        return list(self._owners)

    def hyper(self):
        g = self.param_groups[0]
        return float(g["lr"]), float(g["betas"][0]), float(g["betas"][1]), float(g["eps"])

    def weight_decay(self):
        return float(self.param_groups[0]["weight_decay"])

    def last_grad_norm(self, owner=None):
        """Gradient norm (before clipping) the last step() measured for `owner` (default: the first module); needs
        max_grad_norm."""
        if not self.max_grad_norm:
            raise _lib.D4PGError("last_grad_norm needs SharedAdam(max_grad_norm=...)")
        return float(self._clip_ws[id(owner if owner is not None else self._owners[0])][1].item())

    @torch.no_grad()
    def step(self, closure=None):
        _lib.require_cuda()
        lr, b1, b2, eps = self.hyper()
        wd = self.weight_decay()
        self.step_count += 1
        for owner in self._owners:
            m, v = self.moments(owner)
            p, g = owner.flat_params(), owner.flat_grads()
            if wd or self.max_grad_norm:
                part, norm = None, None
                if self.max_grad_norm:
                    ws = self._clip_ws.get(id(owner))
                    if ws is None or ws[0].device != p.device:
                        ws = self._clip_ws[id(owner)] = (torch.zeros(64, dtype=torch.float64, device=p.device),
                                                         torch.zeros(1, dtype=torch.float32, device=p.device))
                    part, norm = ws
                _lib.check(_lib.lib().d4pg_adam_polyak_ex(_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(v), None,
                                                          p.numel(), lr, b1, b2, eps, self.step_count, 0.0, 1.0,
                                                          _lib.stream_ptr(), wd, self.max_grad_norm, _lib.ptr(part),
                                                          _lib.ptr(norm)), "d4pg_adam_polyak_ex")
            else:
                _lib.check(_lib.lib().d4pg_adam_polyak(_lib.ptr(p), _lib.ptr(g), _lib.ptr(m), _lib.ptr(v), None,
                                                       p.numel(), lr, b1, b2, eps, self.step_count, 0.0, 1.0,
                                                       _lib.stream_ptr()), "d4pg_adam_polyak")
            torch.autograd.graph.increment_version(p)      # written through a raw pointer: let version watchers see it
        for st in self.state.values():
            st["step"] = self.step_count
