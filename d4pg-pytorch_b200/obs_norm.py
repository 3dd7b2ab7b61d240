"""Running per-feature observation normalizer (the `normalize_observations` of DDPG implementations, with clipping).

    norm = ObsNormalizer(clip=5.0, eps=1e-8)
    buf = PrioritizedReplayBuffer(size, alpha, obs_norm=norm)     # every insert updates the statistics on the device
    y = norm.normalize(x)                                          # clamp((x - shift) * scale, -clip, clip)

The statistics (n, mean, M2 in fp64) fold in every row the replay stores, in insertion order, with Welford's update;
the fp32 affine (shift = mean, scale = 1 / sqrt(M2 / n + eps)) is recomputed on the device after every insert.  The
replay keeps raw rows: sample() / gather return them unchanged.  A `DDPG(obs_norm=...)` learner reads the affine inside
its batch sampler, and the actor / critic modules of that DDPG normalize their `state` input.  The exact arithmetic is
in include/d4pg_b200.h (d4pg_replay_set_obs_norm).
"""
import math

import numpy as np
import torch

from . import _lib

DEFAULT_CLIP = 5.0
DEFAULT_EPS = 1e-8


def _check_param(name, v):
    try:
        v = float(v)
    except (TypeError, ValueError):
        raise ValueError("obs_norm %s must be a number, got %r" % (name, v))
    if not (math.isfinite(v) and v > 0.0):
        raise ValueError("obs_norm %s must be finite and > 0, got %r" % (name, v))
    return v


def make_obs_normalizer(spec, obs_dim=None, device=None):
    """None / False -> None; True -> defaults; {"clip": c, "eps": e} (either key optional) -> validated; an
    ObsNormalizer is used as it is."""
    if spec is None or spec is False:
        return None
    if isinstance(spec, ObsNormalizer):
        return spec
    if spec is True:
        return ObsNormalizer(obs_dim=obs_dim, device=device)
    if isinstance(spec, dict):
        unknown = set(spec) - {"clip", "eps"}
        if unknown:
            raise ValueError("obs_norm accepts the keys 'clip' and 'eps', got %s" % sorted(unknown))
        return ObsNormalizer(clip=spec.get("clip", DEFAULT_CLIP), eps=spec.get("eps", DEFAULT_EPS), obs_dim=obs_dim,
                             device=device)
    raise ValueError("obs_norm must be None, False, True or a dict {'clip': c, 'eps': e}, got %r" % (spec,))


class ObsNormalizer(object):
    """Owns the device buffers stats f64 [1 + 2S] = {n, mean[S], M2[S]} and affine f32 [2S] = {shift[S], scale[S]}.

    Registered with one replay buffer (`obs_norm=` of PrioritizedReplayBuffer / Replay / DDPG), whose inserts update it
    on the device.  Without a replay, `update(rows)` folds caller rows in.  `count`, `mean` and `var` are read after the
    replay's pending inserts (staged rows included)."""

    def __init__(self, clip=DEFAULT_CLIP, eps=DEFAULT_EPS, obs_dim=None, device=None):
        self.clip = _check_param("clip", clip)
        self.eps = _check_param("eps", eps)
        self.obs_dim = None
        self.device = torch.device(device) if device is not None else None
        self.stats = self.affine = None
        self._store = None
        if obs_dim is not None and torch.cuda.is_available():
            self._allocate(int(obs_dim), self.device)

    # -- buffers -----------------------------------------------------------------------
    def _allocate(self, obs_dim, device):
        _lib.require_cuda()
        if self.stats is not None:
            if obs_dim != self.obs_dim:
                raise _lib.D4PGError("ObsNormalizer has obs_dim %d, the replay stores rows of %d" % (self.obs_dim, obs_dim))
            return
        dev = device if device is not None else torch.device("cuda", torch.cuda.current_device())
        self.obs_dim, self.device = obs_dim, dev
        self.stats = torch.zeros(1 + 2 * obs_dim, dtype=torch.float64, device=dev)
        self.affine = torch.cat([torch.zeros(obs_dim), torch.ones(obs_dim)]).to(device=dev, dtype=torch.float32)

    def _bind(self, store):
        """Register with a replay store (called by _DeviceReplay._allocate).  The library resets the statistics to
        n = 0; statistics loaded before the store existed are written back."""
        if self._store is not None and self._store is not store:
            raise _lib.D4PGError("an ObsNormalizer can be registered with one replay buffer only")
        had = self.stats is not None and bool(self.stats[0].item() > 0)
        keep = self.stats.clone() if had else None
        self._allocate(store.obs_dim, store.device)
        _lib.check(_lib.lib().d4pg_replay_set_obs_norm(store.handle, _lib.ptr(self.stats), _lib.ptr(self.affine),
                                                       self.clip, self.eps, _lib.stream_ptr()), "d4pg_replay_set_obs_norm")
        self._store = store
        if keep is not None:
            self._write_stats(keep)

    def _require(self):
        if self.stats is None:
            raise _lib.D4PGError("ObsNormalizer has no buffers yet: give obs_dim or register it with a replay buffer")

    def _sync_reads(self):
        """Order the caller's stream after every insert issued so far (the ingest stream included)."""
        if self._store is not None and self._store.handle is not None:
            self._store.flush()

    # -- statistics --------------------------------------------------------------------
    @property
    def count(self):
        self._require()
        self._sync_reads()
        return int(self.stats[0].item())

    @property
    def mean(self):
        self._require()
        self._sync_reads()
        return self.stats[1:1 + self.obs_dim].clone()

    @property
    def var(self):
        """M2 / n (population variance); zeros while n == 0."""
        self._require()
        self._sync_reads()
        n = self.stats[0]
        m2 = self.stats[1 + self.obs_dim:].clone()
        return torch.where(n > 0, m2 / torch.clamp(n, min=1.0), torch.zeros_like(m2))

    @property
    def shift(self):
        self._require()
        self._sync_reads()
        return self.affine[:self.obs_dim].clone()

    @property
    def scale(self):
        self._require()
        self._sync_reads()
        return self.affine[self.obs_dim:].clone()

    def update(self, rows):
        """Fold caller rows [n, obs_dim] in (standalone use; a registered normalizer is updated by its replay)."""
        if self._store is not None:
            raise _lib.D4PGError("this ObsNormalizer is updated by its replay buffer's inserts")
        x = torch.as_tensor(rows, dtype=torch.float32)
        if x.dim() == 1:
            x = x.view(1, -1)
        if self.stats is None:
            self._allocate(int(x.shape[1]), self.device)
        if x.shape[1] != self.obs_dim:
            raise ValueError("expected rows of width %d, got %s" % (self.obs_dim, tuple(x.shape)))
        x = x.to(self.device).contiguous()
        _lib.check(_lib.lib().d4pg_obs_norm_update(_lib.ptr(self.stats), _lib.ptr(self.affine), self.obs_dim,
                                                   _lib.ptr(x), x.shape[0], self.obs_dim, self.eps, _lib.stream_ptr()),
                   "d4pg_obs_norm_update")

    # -- apply -------------------------------------------------------------------------
    def _join(self):
        """A forward that reads the affine: order the caller's stream after the inserts issued on a learner's ingest
        stream (rows staged by single add() calls count once they are flushed)."""
        if self._store is not None:
            self._store._join_ingest()

    def _apply(self, x, want_grad):
        self._require()
        self._join()
        x = x.to(device=self.affine.device, dtype=torch.float32)
        if x.dim() == 1:
            x = x.view(1, -1)
        if x.shape[1] != self.obs_dim:
            raise ValueError("expected observations of width %d, got %s" % (self.obs_dim, tuple(x.shape)))
        x = x.contiguous()
        y = torch.empty_like(x)
        dydx = torch.empty_like(x) if want_grad else None
        if x.shape[0]:
            _lib.check(_lib.lib().d4pg_obs_normalize(_lib.ptr(self.affine), self.obs_dim, self.clip, _lib.ptr(x),
                                                     x.shape[0], _lib.ptr(y), _lib.ptr(dydx), _lib.stream_ptr()),
                       "d4pg_obs_normalize")
        return y, dydx

    def normalize(self, x):
        """clamp((x - shift) * scale, -clip, clip) on the device (no autograd)."""
        if not torch.is_tensor(x):
            x = torch.as_tensor(np.asarray(x))
        return self._apply(x.detach(), False)[0]

    def apply(self, x):
        """normalize() on the autograd graph: d y / d x = scale inside the clip range (both ends included), else 0."""
        return _ObsNormFn.apply(self, x)

    # -- checkpointing -----------------------------------------------------------------
    def state_dict(self):
        self._require()
        self._sync_reads()
        return {"stats": self.stats.detach().cpu().clone(), "clip": self.clip, "eps": self.eps}

    def _write_stats(self, stats):
        self.stats.copy_(stats.to(device=self.stats.device, dtype=torch.float64))
        if self._store is not None and self._store.handle is not None:
            store = self._store
            _lib.check(_lib.lib().d4pg_replay_obs_norm_refresh(store.handle, _lib.stream_ptr()),
                       "d4pg_replay_obs_norm_refresh")
            store._order_ingest_after_caller()
        else:
            _lib.check(_lib.lib().d4pg_obs_norm_update(_lib.ptr(self.stats), _lib.ptr(self.affine), self.obs_dim, None,
                                                       0, self.obs_dim, self.eps, _lib.stream_ptr()),
                       "d4pg_obs_norm_update")

    def load_state_dict(self, state):
        """Write saved statistics and recompute the affine from them (a learner's prefetched batch is re-sampled)."""
        stats = torch.as_tensor(state["stats"], dtype=torch.float64).reshape(-1)
        if float(state.get("clip", self.clip)) != self.clip or float(state.get("eps", self.eps)) != self.eps:
            raise ValueError("ObsNormalizer state has clip=%r, eps=%r; this normalizer has clip=%r, eps=%r"
                             % (state.get("clip"), state.get("eps"), self.clip, self.eps))
        if (stats.numel() - 1) % 2 or stats.numel() < 3:
            raise ValueError("ObsNormalizer state: stats must hold 1 + 2 * obs_dim values")
        S = (stats.numel() - 1) // 2
        if self.stats is None:
            self._allocate(S, self.device)
        if S != self.obs_dim:
            raise ValueError("ObsNormalizer state is for obs_dim %d, this normalizer has %d" % (S, self.obs_dim))
        if self._store is not None and self._store.handle is not None:
            self._store.flush()          # pending inserts (ingest stream included) land before the overwrite
        self._write_stats(stats)


class _ObsNormFn(torch.autograd.Function):
    @staticmethod
    def forward(ctx, norm, x):
        y, dydx = norm._apply(x.detach(), True)
        ctx.save_for_backward(dydx)
        return y

    @staticmethod
    def backward(ctx, g):
        (dydx,) = ctx.saved_tensors
        return None, (g * dydx) if ctx.needs_input_grad[1] else None
