"""Prioritized replay with the reference's class names and method signatures
(prioritized_replay_memory.py), backed by GPU-resident storage + segment trees.

  LinearSchedule(schedule_timesteps, final_p, initial_p).value()            :5-29
  SegmentTree / SumSegmentTree / MinSegmentTree(capacity)                    :33-162
  ReplayBuffer(size).add/.sample/__len__                                     :164-222
  PrioritizedReplayBuffer(size, alpha).add/.sample(B, beta)/.update_priorities/__len__   :224-335

Transitions live in SoA device arrays (obs/obs2 f32, act f32, reward f64, done u8) and the
sum/min trees are fp32 device arrays; every operation is a call into libd4pg_sm90.so.
`add()` stages rows in pinned host memory and flushes them with one H2D copy + one kernel
before anything reads the buffer, so the observable behaviour is the reference's.
Seeded-index parity: `sample()` draws its B uniforms from Python's global `random`
exactly as `_sample_proportional` does (:262), so `random.seed(k)` reproduces the
reference's indices.
"""
import ctypes as C
import random

import numpy as np
import torch

from . import _lib
from .obs_norm import make_obs_normalizer
from .utils import default_device


class LinearSchedule(object):
    """Linear interpolation initial_p -> final_p over `schedule_timesteps` calls; `value()`
    post-increments its clock (:25-29)."""

    def __init__(self, schedule_timesteps, final_p, initial_p=1.0):
        self.schedule_timesteps = schedule_timesteps
        self.final_p = final_p
        self.initial_p = initial_p
        self.t = 0

    def value(self):
        fraction = min(float(self.t) / self.schedule_timesteps, 1.0)
        self.t += 1
        return self.initial_p + fraction * (self.final_p - self.initial_p)


def dev_flags(x, E, device):
    """terminated / truncated flags (numpy, CPU or CUDA) -> u8 [E] on `device`."""
    x = torch.as_tensor(x, device=device).reshape(E)
    return (x if x.dtype == torch.bool else x != 0).contiguous().view(torch.uint8)


def _shape(x):
    return tuple(x.shape) if hasattr(x, "shape") else np.shape(x)


def _step_vectors_ok(E, reward, terminated, truncated):
    """reward, terminated and (unless None) truncated of a vector step are [E]."""
    return _shape(reward) == (E,) and _shape(terminated) == (E,) and (truncated is None or _shape(truncated) == (E,))


class _StreamMirror(object):
    """The device state of a streaming insert (add_steps, add_goal_steps) and its end-flag protocol.  The window bytes
    live on the device; the episode ends of a call with CUDA flags are copied back into a pinned slot and applied, by
    the subclass's end(), at the next call, so no call waits for its own flags."""

    def __init__(self):
        self.window = self.ends = self.event = None
        self.pending = False

    def ensure_window(self, nbytes, device):
        """On first use: the zero-filled window of nbytes() bytes, the pinned end-flag slot and its event."""
        if self.window is None:
            self.window = torch.zeros(int(nbytes()), dtype=torch.uint8, device=device)
            self.ends = torch.zeros(2, self.E, dtype=torch.uint8, pin_memory=True)
            self.event = torch.cuda.Event()

    def resolve(self):
        """Apply the end flags of the previous call when they were CUDA tensors (copied back asynchronously)."""
        if self.pending:
            self.event.synchronize()
            e = self.ends.numpy()
            self.end((e[0] | e[1]) != 0)
            self.pending = False

    def record_ends(self, term, trunc, terminated, truncated):
        """Close a call: its episode ends (term / trunc: the u8 device flags the launch read, terminated / truncated: the
        caller's) are applied now when they are host flags, else copied back and applied at the next call."""
        if (torch.is_tensor(terminated) and terminated.is_cuda) or (torch.is_tensor(truncated) and truncated.is_cuda):
            self.ends[0].copy_(term, non_blocking=True)
            if trunc is not None:
                self.ends[1].copy_(trunc, non_blocking=True)
            else:
                self.ends[1].zero_()                 # host memory: no copy into it is in flight (resolved before)
            self.event.record()
            self.pending = True
        else:
            ended = np.asarray(terminated).reshape(self.E).astype(bool)
            if truncated is not None:
                ended = ended | np.asarray(truncated).reshape(self.E).astype(bool)
            self.end(ended)


class StepsMirror(_StreamMirror):
    """add_steps' pending n-step windows: the fixed (E, n, gamma) and the host mirror of each window's fill (steps of
    the current episode, capped at n - 1, which is all the emit decision needs).  Environment e emits a row at a call
    iff fill[e] == n - 1 before it, so the count is exact before the call without a device read.  With episode tails
    (`tails`), an episode that ended also leaves tails[e] = min(its length, n - 1) rows, which e emits at its next
    call."""

    def __init__(self, E, n, gamma, tails=False):
        super(StepsMirror, self).__init__()
        self.E, self.n, self.gamma = int(E), int(n), float(gamma)
        self.fill = np.zeros(self.E, dtype=np.int64)
        self.tails = np.zeros(self.E, dtype=np.int64) if tails else None

    def rows(self):
        """Rows the next call inserts."""
        full = int(np.count_nonzero(self.fill >= self.n - 1))
        return full if self.tails is None else full + int(self.tails.sum())

    def advance(self):
        """Every environment took one step (and emitted its pending tails first)."""
        np.minimum(self.fill + 1, self.n - 1, out=self.fill)
        if self.tails is not None:
            self.tails[:] = 0

    def end(self, ended):
        """Clear the windows of the environments whose episode ended (bool [E]); with tails, their last
        min(length, n - 1) starts become pending."""
        ended = np.asarray(ended, dtype=bool)
        if self.tails is not None:
            self.tails[ended] = self.fill[ended]          # fill = min(length, n - 1) after advance()
        self.fill[ended] = 0


HER_ACTIONS = ("reference", "own")


def check_her_params(her_ratio, threshold, her_action, max_episode_steps, seed):
    """The parameters of add_goal_steps, validated -> (her_ratio, threshold, her_action, max_episode_steps, seed)."""
    try:
        ratio, thr = float(her_ratio), float(threshold)
    except (TypeError, ValueError):
        raise ValueError("add_goal_steps: her_ratio and threshold must be numbers, got %r / %r" % (her_ratio, threshold))
    if not 0.0 <= ratio <= 1.0:
        raise ValueError("add_goal_steps: her_ratio must be in [0, 1], got %r" % (her_ratio,))
    if not (np.isfinite(thr) and thr >= 0.0):
        raise ValueError("add_goal_steps: threshold must be finite and >= 0, got %r" % (threshold,))
    if her_action not in HER_ACTIONS:
        raise ValueError("add_goal_steps: her_action must be 'reference' (the episode's last action, main.py:184) or "
                         "'own' (the step's action), got %r" % (her_action,))
    if isinstance(max_episode_steps, bool) or int(max_episode_steps) != max_episode_steps \
            or not 1 <= int(max_episode_steps) <= _lib.GOAL_MAX_STEPS:
        raise ValueError("add_goal_steps: max_episode_steps must be an integer in [1, %d], got %r"
                         % (_lib.GOAL_MAX_STEPS, max_episode_steps))
    if isinstance(seed, bool) or int(seed) != seed or int(seed) < 0:
        raise ValueError("add_goal_steps: seed must be a non-negative integer, got %r" % (seed,))
    return ratio, thr, her_action, int(max_episode_steps), int(seed)


class GoalStepsMirror(_StreamMirror):
    """add_goal_steps' pending episodes on the host: the fixed parameters, each environment's fill (steps of its current
    episode), the length of the episode it ended at the last call (0: none) and the generator of the relabelling draws.
    An ended episode is emitted at the next call, so the rows of a call, and the draws that make them, are known before
    it without a device read."""

    def __init__(self, E, So, G, A, her_ratio, threshold, her_action, max_episode_steps, seed):
        super(GoalStepsMirror, self).__init__()
        self.E, self.So, self.G, self.A = int(E), int(So), int(G), int(A)
        self.her_ratio, self.threshold, self.her_action = float(her_ratio), float(threshold), her_action
        self.M, self.seed = int(max_episode_steps), int(seed)
        self.key = (self.E, self.So, self.G, self.A, self.her_ratio, self.threshold, self.her_action, self.M, self.seed)
        self.fill = np.zeros(self.E, dtype=np.int64)
        self.ended = np.zeros(self.E, dtype=np.int64)
        self.rng = np.random.default_rng(self.seed)

    def check_step(self):
        """ValueError if this call's step would take an episode past max_episode_steps."""
        over = np.flatnonzero(self.fill >= self.M)
        if over.size:
            raise ValueError("add_goal_steps: the episode of environment %d already has max_episode_steps = %d steps and "
                             "did not end" % (int(over[0]), self.M))

    def draw(self):
        """The relabelling draws of the episodes that ended at the last call -> (plan i32 or None, n_draws, n_rows).
        Ended episodes in ascending e; one rng.random(sum L) gives select = u < her_ratio, then one rng.integers(t, L)
        over the selected (e, t) in that order gives their future steps.  plan = {step_off [E], future [n_draws] (-1: no
        copy), dst [n_draws] (rank of the original row in this call)}, the layout of d4pg_replay_add_goal_steps."""
        em = np.flatnonzero(self.ended)
        if em.size == 0:
            return None, 0, 0
        L = self.ended[em]
        n = int(L.sum())
        starts = np.cumsum(L) - L
        sel = self.rng.random(n) < self.her_ratio
        future = np.full(n, -1, dtype=np.int64)
        if sel.any():
            t = np.arange(n, dtype=np.int64) - np.repeat(starts, L)
            future[sel] = self.rng.integers(t[sel], np.repeat(L, L)[sel])
        counts = 1 + sel.astype(np.int64)
        dst = np.cumsum(counts) - counts
        step_off = np.zeros(self.E, dtype=np.int64)
        step_off[em] = starts
        return np.concatenate([step_off, future, dst]).astype(np.int32), n, int(counts.sum())

    def advance(self, step=True):
        """The ended episodes were emitted; with `step`, every environment took one step."""
        self.ended[:] = 0
        if step:
            self.fill += 1

    def end(self, ended):
        """The episodes of the environments in `ended` (bool [E]) ended at this call: emitted at the next."""
        ended = np.asarray(ended, dtype=bool)
        self.ended[ended] = self.fill[ended]
        self.fill[ended] = 0


class _DeviceReplay(object):
    """Device storage + trees + the C handle.  Allocated lazily on the first add (the
    reference constructors do not know obs/act dims)."""

    STAGE_ROWS = 4096

    def __init__(self, size, alpha, prioritized, obs_dim=None, act_dim=None, device=None, obs_norm=None,
                 nstep_tails=False):
        self.size = int(size)
        # episode tails of add_steps (DESIGN.md §3 "Episode tails"): a u8 horizon column beside `done`, fixed at construction
        self.nstep_tails = bool(nstep_tails)
        self.horizon = None
        self.obs_norm = obs_norm         # ObsNormalizer (obs_norm.py): registered when the store is allocated
        self.alpha = float(alpha)
        self.prioritized = bool(prioritized)
        self.device = torch.device(device) if device is not None else None
        self.obs_dim, self.act_dim = obs_dim, act_dim
        self.handle = None
        self._n_staged = 0
        self._len = 0
        self._next_idx = 0
        self._steps = None               # add_steps: the device windows and the host mirror of their fills
        self._goals = None               # add_goal_steps: the device episode windows and their GoalStepsMirror
        # host pipeline (a learner's ingest stream, ddpg.py): add_batch_host is issued there; every other device
        # operation runs on the caller's stream -- the two are kept in program order by events, only when they interleave.
        # _cs_dirty: the caller's stream touched the buffer (the next host add waits for it); _cs_wrote: it wrote the
        # buffer (the next step's sample on the ingest stream waits for it, before_step)
        self._ingest_stream = None
        self._ing_dirty = False
        self._cs_dirty = False
        self._cs_wrote = False
        if obs_dim is not None and act_dim is not None and torch.cuda.is_available():
            self._allocate(obs_dim, act_dim)

    # -- allocation --------------------------------------------------------------------
    def _allocate(self, obs_dim, act_dim):
        _lib.require_cuda()
        self.obs_dim, self.act_dim = int(obs_dim), int(act_dim)
        dev = self.device or default_device()
        self.device = dev
        cap = C.c_int64()
        _lib.check(_lib.lib().d4pg_replay_capacity(self.size, C.byref(cap)), "d4pg_replay_capacity")
        self.capacity = int(cap.value)
        f32, n = torch.float32, self.size
        self.sum_tree = torch.empty(2 * self.capacity, dtype=f32, device=dev)
        self.min_tree = torch.empty(2 * self.capacity, dtype=f32, device=dev)
        self.obs = torch.zeros(n, self.obs_dim, dtype=f32, device=dev)
        self.obs2 = torch.zeros(n, self.obs_dim, dtype=f32, device=dev)
        self.act = torch.zeros(n, self.act_dim, dtype=f32, device=dev)
        self.rew = torch.zeros(n, dtype=torch.float64, device=dev)
        self.done = torch.zeros(n, dtype=torch.uint8, device=dev)
        self.scratch = torch.empty(self.capacity, dtype=torch.int32, device=dev)
        self.state = torch.zeros(8, dtype=f32, device=dev)
        h = C.c_void_p()
        _lib.check(_lib.lib().d4pg_replay_create(self.size, self.obs_dim, self.act_dim, self.alpha,
                                                 _lib.ptr(self.sum_tree), _lib.ptr(self.min_tree),
                                                 _lib.ptr(self.obs), _lib.ptr(self.act), _lib.ptr(self.rew),
                                                 _lib.ptr(self.obs2), _lib.ptr(self.done), _lib.ptr(self.scratch),
                                                 _lib.ptr(self.state), _lib.stream_ptr(), C.byref(h)),
                   "d4pg_replay_create")
        self.handle = h
        if self.nstep_tails:
            self.horizon = torch.zeros(n, dtype=torch.uint8, device=dev)
            _lib.check(_lib.lib().d4pg_replay_set_horizons(h, _lib.ptr(self.horizon), _lib.stream_ptr()),
                       "d4pg_replay_set_horizons")
        if self.obs_norm is not None:
            self.obs_norm._bind(self)
        R = self.STAGE_ROWS
        pin = dict(pin_memory=True)
        self._st_obs = torch.empty(R, self.obs_dim, dtype=f32, **pin)
        self._st_obs2 = torch.empty(R, self.obs_dim, dtype=f32, **pin)
        self._st_act = torch.empty(R, self.act_dim, dtype=f32, **pin)
        self._st_rew = torch.empty(R, dtype=torch.float64, **pin)
        self._st_done = torch.empty(R, dtype=torch.uint8, **pin)
        self._np = [t.numpy() for t in (self._st_obs, self._st_act, self._st_rew, self._st_obs2, self._st_done)]
        self._dev_stage = [torch.empty_like(t, device=dev) for t in
                           (self._st_obs, self._st_act, self._st_rew, self._st_obs2, self._st_done)]

    def __del__(self):
        try:
            if self.handle is not None:
                h, self.handle = self.handle, None       # a learner collected later (reference cycles) must not touch it
                self._ingest_stream = None
                _lib.lib().d4pg_replay_destroy(h)
        except Exception:
            pass

    # -- streams -----------------------------------------------------------------------
    def attach_ingest_stream(self, raw_stream):
        """raw cudaStream_t (int) of the learner's ingest stream, or None to detach (joins it first)."""
        if self._ingest_stream is not None and self.handle is not None:
            self._join_ingest()
        self._ingest_stream = raw_stream
        self._ing_dirty = False
        self._cs_dirty = self._cs_wrote = raw_stream is not None     # whatever the caller's stream did so far comes first

    def _caller_wrote(self):
        """A write to the ring, trees, horizons or normalizer statistics was issued on the caller's stream."""
        self._cs_dirty = self._cs_wrote = True

    def before_step(self):
        """A host-pipeline step is about to sample on the ingest stream, which does not wait for the caller's stream:
        order it after the caller's writes since the last ordering.  Reads on the caller's stream need no edge."""
        if self._cs_wrote:
            self._order_ingest_after_caller()

    def _join_ingest(self):
        """The caller's stream is about to touch the buffer: order it after the ingest stream's adds."""
        if self._ingest_stream is not None and self.handle is not None:
            if self._ing_dirty:
                _lib.check(_lib.lib().d4pg_replay_order_after(self.handle, C.c_void_p(self._ingest_stream), _lib.stream_ptr()),
                           "d4pg_replay_order_after")
                self._ing_dirty = False
            self._cs_dirty = True

    def _order_ingest_after_caller(self):
        """Order the ingest stream after everything issued so far on the caller's stream."""
        if self._ingest_stream is not None and self.handle is not None:
            _lib.check(_lib.lib().d4pg_replay_order_after(self.handle, _lib.stream_ptr(), C.c_void_p(self._ingest_stream)),
                       "d4pg_replay_order_after")
        self._cs_dirty = self._cs_wrote = False

    def _ingest_ptr(self):
        """Stream of a host add: the ingest stream when attached (ordered after the caller's earlier buffer operations)."""
        ing = self._ingest_stream
        if ing is None:
            return _lib.raw_stream()
        if self._cs_dirty:
            self._order_ingest_after_caller()
        self._ing_dirty = True
        return ing

    # -- ingest ------------------------------------------------------------------------
    def add(self, s, a, r, s2, done):
        s = np.asarray(s, dtype=np.float32).reshape(-1)
        a = np.asarray(a, dtype=np.float32).reshape(-1)
        if self.handle is None:
            self._allocate(s.shape[0], a.shape[0])
        i = self._n_staged
        o, ac, rw, o2, dn = self._np
        o[i] = s
        ac[i] = a
        rw[i] = float(r)
        o2[i] = np.asarray(s2, dtype=np.float32).reshape(-1)
        dn[i] = 1 if done else 0
        self._n_staged = i + 1
        self._len = min(self.size, self._len + 1)
        if self._n_staged == self.STAGE_ROWS or self._n_staged == self.size:
            self.flush()

    def add_batch_host(self, s, a, r, s2, done):
        """Fast ingest of n <= STAGE_ROWS host transitions through ONE library call
        (`d4pg_replay_add_host`): packed into a pinned staging buffer, one async H2D copy, ring +
        tree kernels."""
        if (torch.is_tensor(s) and self.handle is not None and getattr(self, "_pack_host", None) is not None
                and s.dtype == torch.float32 and s.dim() == 2 and 0 < s.shape[0] <= min(self.STAGE_ROWS, self.size)
                and not self._n_staged and torch.is_tensor(a) and torch.is_tensor(r) and torch.is_tensor(s2)
                and torch.is_tensor(done) and a.dtype == torch.float32 and r.dtype == torch.float64
                and s2.dtype == torch.float32 and done.dtype in (torch.bool, torch.uint8)
                and s.is_contiguous() and a.is_contiguous() and r.is_contiguous() and s2.is_contiguous()
                and done.is_contiguous()):
            # host tensors of the right types (e.g. slices of a pinned rollout buffer): no numpy round trip
            n = s.shape[0]
            ptrs = [t.data_ptr() for t in (s, a, r, s2, done)]
        else:
            s = np.ascontiguousarray(s, dtype=np.float32)
            n = s.shape[0] if s.ndim == 2 else 1
            a = np.ascontiguousarray(a, dtype=np.float32)
            if self.handle is None:
                self._allocate(s.reshape(n, -1).shape[1], a.reshape(n, -1).shape[1])
            if n > self.STAGE_ROWS or n > self.size:
                return self.add_batch(s, a, r, s2, done)
            if self._n_staged:
                self.flush()
            if getattr(self, "_pack_host", None) is None:
                L = _lib.lib()
                nbytes = int(L.d4pg_replay_staging_bytes(self.handle, self.STAGE_ROWS))
                self._pack_host = torch.empty(nbytes, dtype=torch.uint8, pin_memory=True)
                self._pack_dev = torch.empty(nbytes, dtype=torch.uint8, device=self.device)
                _lib.check(L.d4pg_replay_set_staging(self.handle, _lib.ptr(self._pack_host), _lib.ptr(self._pack_dev),
                                                     nbytes), "d4pg_replay_set_staging")
            r = np.ascontiguousarray(r, dtype=np.float64)
            s2 = np.ascontiguousarray(s2, dtype=np.float32)
            done = np.ascontiguousarray(done)
            if done.dtype != np.uint8:
                done = done.astype(np.uint8)
            ptrs = [x.ctypes.data for x in (s, a, r, s2, done)]
        rc = _lib.lib().d4pg_replay_add_host(self.handle, n, *ptrs, 1 if self.prioritized else 0, self._ingest_ptr())
        if rc:
            _lib.check(rc, "d4pg_replay_add_host")
        self._next_idx = (self._next_idx + n) % self.size
        self._len = min(self.size, self._len + n)

    def _rows_to_device(self, s, a, r, s2, done, non_blocking):
        """n rows (host numpy / CPU or CUDA tensors) -> (n, contiguous device tensors s, a, r f64, s2, done u8); the
        copies from host memory are asynchronous with `non_blocking`."""
        self.flush()
        s = torch.as_tensor(s, dtype=torch.float32)
        if s.dim() == 1:
            s = s.view(1, -1)
        n = s.shape[0]
        a = torch.as_tensor(a, dtype=torch.float32).reshape(n, -1)
        if self.handle is None:
            self._allocate(s.shape[1], a.shape[1])
        dev, nb = self.device, non_blocking and not s.is_cuda
        return n, [s.to(dev, non_blocking=nb).contiguous(), a.to(dev, non_blocking=nb).contiguous(),
                   torch.as_tensor(r, dtype=torch.float64).reshape(n).to(dev, non_blocking=nb).contiguous(),
                   torch.as_tensor(s2, dtype=torch.float32).reshape(n, -1).to(dev, non_blocking=nb).contiguous(),
                   torch.as_tensor(done).reshape(n).to(torch.uint8).to(dev, non_blocking=nb).contiguous()]

    def add_batch(self, s, a, r, s2, done):
        """Vectorised ingest of n transitions (host numpy / CPU or CUDA tensors)."""
        n, args = self._rows_to_device(s, a, r, s2, done, non_blocking=True)
        for lo in range(0, n, self.size):
            hi = min(n, lo + self.size)
            self._add_device(hi - lo, [t[lo:hi] for t in args])

    def add_episode_nstep(self, s, a, r, s2, done, n_steps, gamma):
        """One episode of T consecutive steps with the n-step return accumulated ON THE DEVICE at insert
        (replay_memory.py:38-45): transition i = (s_i, a_i, sum_k gamma^k r_{i+k}, s'_{i+n-1}, done_{i+n-1})."""
        T, args = self._rows_to_device(s, a, r, s2, done, non_blocking=False)
        n_steps = int(n_steps)
        if T < n_steps:
            return 0
        m = T - n_steps + 1
        if m > self.size:
            raise _lib.D4PGError("add_episode_nstep: episode longer than the buffer")
        scratch = torch.empty(T, dtype=torch.float64, device=self.device)
        _lib.check(_lib.lib().d4pg_replay_add_nstep(self.handle, T, *[_lib.ptr(t) for t in args], n_steps, float(gamma),
                                                    _lib.ptr(scratch), 1 if self.prioritized else 0, _lib.stream_ptr()),
                   "d4pg_replay_add_nstep")
        self._caller_wrote()
        self._sync_ring()
        return m

    def add_her_episode(self, obs, obs_next, goal, ag_next, act, rew, done, her_ratio=0.8, threshold=0.05,
                        her_action="reference", rng=None):
        """Hindsight relabelling of one goal-conditioned episode on the device (main.py:154-184): every transition is
        stored, and with probability `her_ratio` also a copy whose goal is the achieved goal of a uniformly chosen
        FUTURE step (reward recomputed as the sparse -(distance > threshold), done = reward == 0).  The random draws
        are made on the host in the reference's order (np.random.uniform() then np.random.randint(t, T) per step)."""
        rng = np.random if rng is None else rng
        obs = np.ascontiguousarray(obs, dtype=np.float32)
        T, So = obs.shape
        goal = np.ascontiguousarray(goal, dtype=np.float64).reshape(T, -1)
        G = goal.shape[1]
        act = np.ascontiguousarray(act, dtype=np.float32).reshape(T, -1)
        A = act.shape[1]
        select = np.zeros(T, dtype=np.uint8)
        future = np.arange(T, dtype=np.int32)
        for t in range(T):
            if rng.uniform() < her_ratio:                                                   # main.py:166
                select[t] = 1
                future[t] = rng.randint(t, T)                                               # main.py:170
        counts = 1 + select.astype(np.int64)
        dst = (np.cumsum(counts) - counts).astype(np.int32)
        n_out = int(counts.sum())
        if self.handle is None:
            self._allocate(So + G, A)
        if n_out > self.size:
            raise _lib.D4PGError("add_her_episode: episode longer than the buffer")
        self.flush()
        dev = self.device
        up = lambda x, dt: torch.as_tensor(np.ascontiguousarray(x, dtype=dt)).to(dev)
        ins = [up(obs, np.float32), up(np.asarray(obs_next).reshape(T, So), np.float32), up(goal, np.float64),
               up(np.asarray(ag_next).reshape(T, G), np.float64), up(act, np.float32), up(np.asarray(rew).reshape(T), np.float64),
               up(np.asarray(done).reshape(T).astype(np.uint8), np.uint8), up(select, np.uint8), up(future, np.int32),
               up(dst, np.int32)]
        outs = [torch.empty(n_out, So + G, dtype=torch.float32, device=dev), torch.empty(n_out, A, dtype=torch.float32, device=dev),
                torch.empty(n_out, dtype=torch.float64, device=dev), torch.empty(n_out, So + G, dtype=torch.float32, device=dev),
                torch.empty(n_out, dtype=torch.uint8, device=dev)]
        _lib.check(_lib.lib().d4pg_her_relabel(T, So, G, A, *[_lib.ptr(t) for t in ins], float(threshold),
                                               0 if her_action == "reference" else 1, *[_lib.ptr(t) for t in outs],
                                               _lib.stream_ptr()), "d4pg_her_relabel")
        self._add_device(n_out, outs)
        return n_out

    # -- streaming n-step insert (DESIGN.md §3 "Streaming n-step insert") ------------------------------------------
    def _check_steps(self, obs, action, reward, obs_next, terminated, truncated, n_steps, gamma):
        """Shapes and the fixed (E, n_steps, gamma) of the pending windows, before any device work -> (E, S, A)."""
        if isinstance(n_steps, bool) or int(n_steps) != n_steps or not 1 <= int(n_steps) <= _lib.STEPS_MAX_N:
            raise ValueError("add_steps: n_steps must be an integer in [1, %d], got %r" % (_lib.STEPS_MAX_N, n_steps))
        so, sa = _shape(obs), _shape(action)
        if len(so) != 2 or len(sa) != 2 or so[0] < 1:
            raise ValueError("add_steps: obs and action must be [E, obs_dim] / [E, act_dim], got %s / %s" % (so, sa))
        E, S, A = so[0], so[1], sa[1]
        if sa[0] != E or _shape(obs_next) != (E, S) or not _step_vectors_ok(E, reward, terminated, truncated):
            raise ValueError("add_steps: shapes must be obs / obs_next [E, obs_dim], action [E, act_dim], reward / "
                             "terminated / truncated [E]; got %s %s %s %s %s %s" % (so, sa, _shape(reward), _shape(obs_next),
                                                                                 _shape(terminated), _shape(truncated)))
        if self._goals is not None:
            raise ValueError("add_steps: add_goal_steps has pending episodes (drop_goal_steps() discards them)")
        if self.obs_dim is not None and (S, A) != (self.obs_dim, self.act_dim):
            raise ValueError("add_steps: rows of (%d, %d) into a buffer of (%d, %d)" % (S, A, self.obs_dim, self.act_dim))
        if E > self.size:
            raise ValueError("add_steps: E = %d environments exceed the buffer size %d" % (E, self.size))
        if self.nstep_tails and E * max(1, int(n_steps) - 1) > self.size:
            raise ValueError("add_steps: with nstep_tails one call can insert E * (n_steps - 1) = %d rows, more than the "
                             "buffer size %d" % (E * (int(n_steps) - 1), self.size))
        w = self._steps
        if w is not None and (w.E, w.n, w.gamma) != (E, int(n_steps), float(gamma)):
            raise ValueError("add_steps: the pending windows hold E=%d, n_steps=%d, gamma=%r; this call has E=%d, "
                             "n_steps=%d, gamma=%r (drop_steps() discards them)" % (w.E, w.n, w.gamma, E,
                                                                                    int(n_steps), float(gamma)))
        return E, S, A

    def add_steps(self, obs, action, reward, obs_next, terminated, truncated=None, n_steps=1, gamma=0.99):
        """One vector step of E environments into per-environment n-step windows on the device; the rows of the windows
        that are full go straight into the ring in one launch.  Returns the number of rows inserted, known on the host
        without a device read (a mirror of the window fills).  See ReplayBuffer.add_steps."""
        E, S, A = self._check_steps(obs, action, reward, obs_next, terminated, truncated, n_steps, gamma)
        n, gamma, tails = int(n_steps), float(gamma), 1 if self.nstep_tails else 0
        w = self._steps
        if w is not None:                         # the fills are exact once the previous call's flags are in
            w.resolve()
        if self.handle is None:
            self._allocate(S, A)
        self.flush()
        dev = self.device
        if w is None:
            w = self._steps = StepsMirror(E, n, gamma, self.nstep_tails)
        w.ensure_window(lambda: _lib.lib().d4pg_replay_steps_window_bytes_ex(E, S, A, n, tails), dev)
        n_rows = w.rows()
        term = dev_flags(terminated, E, dev)
        trunc = dev_flags(truncated, E, dev) if truncated is not None else None
        args = [torch.as_tensor(obs, dtype=torch.float32).to(dev).contiguous(),
                torch.as_tensor(action, dtype=torch.float32).to(dev).contiguous(),
                torch.as_tensor(reward, dtype=torch.float64).to(dev).contiguous(),
                torch.as_tensor(obs_next, dtype=torch.float32).to(dev).contiguous(), term, trunc]
        _lib.check(_lib.lib().d4pg_replay_add_steps_ex(self.handle, E, *[_lib.ptr(t) for t in args], n, gamma,
                                                       _lib.ptr(w.window), n_rows, tails, 1 if self.prioritized else 0,
                                                       _lib.stream_ptr()), "d4pg_replay_add_steps_ex")
        self._caller_wrote()
        self._sync_ring()
        w.advance()
        w.record_ends(term, trunc, terminated, truncated)
        return n_rows

    def drop_steps(self):
        """Discard the pending n-step windows (and pending episode tails); the next add_steps may use another E, n_steps
        or gamma."""
        self._steps = None

    # -- streaming hindsight relabelling (DESIGN.md §3 "Streaming hindsight relabelling") ------------------------------
    def _check_goal_steps(self, obs, desired_goal, action, reward, obs_next, achieved_goal_next, terminated, truncated,
                          params):
        """Shapes, parameters and the fixed key of the pending episodes, before any device work -> (E, So, G, A)."""
        params = check_her_params(*params)
        so, sg, sa = _shape(obs), _shape(desired_goal), _shape(action)
        if len(so) != 2 or len(sg) != 2 or len(sa) != 2 or so[0] < 1:
            raise ValueError("add_goal_steps: obs, desired_goal and action must be [E, obs_dim] / [E, goal_dim] / "
                             "[E, act_dim], got %s / %s / %s" % (so, sg, sa))
        E, So, G, A = so[0], so[1], sg[1], sa[1]
        if sg[0] != E or sa[0] != E or _shape(obs_next) != (E, So) or _shape(achieved_goal_next) != (E, G) \
                or not _step_vectors_ok(E, reward, terminated, truncated):
            raise ValueError("add_goal_steps: shapes must be obs / obs_next [E, obs_dim], desired_goal / "
                             "achieved_goal_next [E, goal_dim], action [E, act_dim], reward / terminated / truncated [E]; "
                             "got %s %s %s %s %s %s %s %s" % (so, sg, sa, _shape(reward), _shape(obs_next),
                                                              _shape(achieved_goal_next), _shape(terminated),
                                                              _shape(truncated)))
        if self._steps is not None:
            raise ValueError("add_goal_steps: add_steps has pending windows (drop_steps() discards them)")
        if self.obs_dim is not None and (So + G, A) != (self.obs_dim, self.act_dim):
            raise ValueError("add_goal_steps: rows of (%d + %d, %d) into a buffer of (%d, %d)"
                             % (So, G, A, self.obs_dim, self.act_dim))
        w = self._goals
        key = (E, So, G, A) + params
        if w is None and E * 2 * params[3] > self.size:
            raise ValueError("add_goal_steps: one call can insert E * 2 * max_episode_steps = %d rows, more than the "
                             "buffer size %d" % (E * 2 * params[3], self.size))
        if w is not None and w.key != key:
            names = ("E", "obs_dim", "goal_dim", "act_dim", "her_ratio", "threshold", "her_action", "max_episode_steps",
                     "seed")
            diff = ", ".join("%s %r -> %r" % (k, x, y) for k, x, y in zip(names, w.key, key) if x != y)
            raise ValueError("add_goal_steps: the pending episodes were started with other parameters (%s); "
                             "drop_goal_steps() discards them" % diff)
        return key

    def _goal_launch(self, w, inputs, plan, n_draws, n_rows, no_step):
        plan_dev = None
        if plan is not None:                      # the draws and row offsets: one host-to-device copy
            plan_dev = torch.from_numpy(plan).pin_memory().to(self.device, non_blocking=True)
        _lib.check(_lib.lib().d4pg_replay_add_goal_steps(
            self.handle, w.E, w.So, w.G, *[_lib.ptr(t) for t in inputs], w.M, _lib.ptr(w.window), _lib.ptr(plan_dev),
            n_draws, n_rows, w.threshold, 0 if w.her_action == "reference" else 1, 1 if no_step else 0,
            1 if self.prioritized else 0, _lib.stream_ptr()), "d4pg_replay_add_goal_steps")
        self._caller_wrote()
        self._sync_ring()

    def add_goal_steps(self, obs, desired_goal, action, reward, obs_next, achieved_goal_next, terminated, truncated=None,
                       her_ratio=0.8, threshold=0.05, her_action="reference", max_episode_steps=50, seed=0):
        """One vector step of E goal-conditioned environments into per-environment episode windows on the device;
        episodes that ended at the previous call are relabelled and inserted first, in one launch.  Returns the number
        of rows inserted, known on the host without a device read.  See ReplayBuffer.add_goal_steps."""
        key = self._check_goal_steps(obs, desired_goal, action, reward, obs_next, achieved_goal_next, terminated,
                                     truncated, (her_ratio, threshold, her_action, max_episode_steps, seed))
        E, So, G, A = key[:4]
        w = self._goals
        if w is not None:                         # the fills are exact once the previous call's flags are in
            w.resolve()
            w.check_step()
        if self.handle is None:
            self._allocate(So + G, A)
        self.flush()
        dev = self.device
        if w is None:
            w = self._goals = GoalStepsMirror(*key)
        w.ensure_window(lambda: _lib.lib().d4pg_replay_goal_window_bytes(E, So, G, A, w.M), dev)
        plan, n_draws, n_rows = w.draw()
        term = dev_flags(terminated, E, dev)
        trunc = dev_flags(truncated, E, dev) if truncated is not None else None
        f32 = lambda x: torch.as_tensor(x, dtype=torch.float32).to(dev).contiguous()
        f64 = lambda x: torch.as_tensor(x, dtype=torch.float64).to(dev).contiguous()       # widened exactly
        inputs = [f32(obs), f64(desired_goal), f32(action), f64(reward).reshape(E), f32(obs_next),
                  f64(achieved_goal_next), term, trunc]
        self._goal_launch(w, inputs, plan, n_draws, n_rows, False)
        w.advance(True)
        w.record_ends(term, trunc, terminated, truncated)
        return n_rows

    def flush_goal_steps(self):
        """Insert the episodes that have ended without taking a step; running episodes stay pending.  Returns the
        number of rows inserted."""
        w = self._goals
        if w is None:
            return 0
        self.flush()
        w.resolve()
        plan, n_draws, n_rows = w.draw()
        if n_rows:
            self._goal_launch(w, [None] * 8, plan, n_draws, n_rows, True)
        w.advance(False)
        return n_rows

    def drop_goal_steps(self):
        """Discard the pending episodes of add_goal_steps; the next call may use other shapes or parameters."""
        self._goals = None

    def _add_device(self, n, tensors):
        _lib.check(_lib.lib().d4pg_replay_add(self.handle, n, *[_lib.ptr(t) for t in tensors],
                                              1 if self.prioritized else 0, _lib.stream_ptr()), "d4pg_replay_add")
        self._caller_wrote()
        self._sync_ring()

    def _sync_ring(self):
        """len / next_idx after a device insert, read from the handle's host mirror (no device read)."""
        L = _lib.lib()
        self._len = int(L.d4pg_replay_len(self.handle))
        self._next_idx = int(L.d4pg_replay_next_idx(self.handle))

    def flush(self):
        self._join_ingest()
        n = self._n_staged
        if n == 0:
            return
        host = (self._st_obs, self._st_act, self._st_rew, self._st_obs2, self._st_done)
        for d, h in zip(self._dev_stage, host):
            d[:n].copy_(h[:n], non_blocking=True)
        self._add_device(n, [d[:n] for d in self._dev_stage])
        # the pinned staging rows may be overwritten by the next add(): wait for the copies
        torch.cuda.current_stream().synchronize()
        self._n_staged = 0

    def __len__(self):
        return self._len

    # -- read paths -------------------------------------------------------------------
    def _batch_buffers(self, B):
        dev, f32 = self.device, torch.float32
        return dict(idx=torch.empty(B, dtype=torch.int32, device=dev),
                    w=torch.empty(B, dtype=f32, device=dev),
                    s=torch.empty(B, self.obs_dim, dtype=f32, device=dev),
                    a=torch.empty(B, self.act_dim, dtype=f32, device=dev),
                    r=torch.empty(B, dtype=torch.float64, device=dev),
                    s2=torch.empty(B, self.obs_dim, dtype=f32, device=dev),
                    d=torch.empty(B, dtype=torch.uint8, device=dev))

    def sample_proportional(self, B, beta, uniforms=None, philox=None):
        """Device tensors (idx i32, weights f32, s, a, r f64, s2, done u8)."""
        self.flush()
        if self.handle is None:
            raise _lib.D4PGError("sample() on an empty replay buffer")
        o = self._batch_buffers(B)
        u_dev = None
        seed, ctr = 0, 0
        if philox is not None:
            seed, ctr = philox
        else:
            if uniforms is None:
                uniforms = [random.random() for _ in range(B)]          # :262, global `random`
            u_dev = torch.tensor(np.asarray(uniforms, dtype=np.float64)).to(self.device)
        _lib.check(_lib.lib().d4pg_replay_sample(self.handle, B, _lib.ptr(u_dev), seed, ctr, float(beta),
                                                 _lib.ptr(o["idx"]), _lib.ptr(o["w"]), _lib.ptr(o["s"]), _lib.ptr(o["a"]),
                                                 _lib.ptr(o["r"]), _lib.ptr(o["s2"]), _lib.ptr(o["d"]), _lib.stream_ptr()),
                   "d4pg_replay_sample")
        return o

    def gather(self, positions):
        self.flush()
        pos = torch.as_tensor(np.asarray(positions, dtype=np.int32)).to(self.device)
        B = pos.numel()
        o = self._batch_buffers(B)
        o["idx"] = pos
        _lib.check(_lib.lib().d4pg_replay_gather(self.handle, B, _lib.ptr(pos), _lib.ptr(o["s"]), _lib.ptr(o["a"]),
                                                 _lib.ptr(o["r"]), _lib.ptr(o["s2"]), _lib.ptr(o["d"]), _lib.stream_ptr()),
                   "d4pg_replay_gather")
        return o

    def update_priorities(self, idxes, priorities):
        self.flush()
        idx = torch.as_tensor(np.asarray(idxes, dtype=np.int32)).to(self.device) if not torch.is_tensor(idxes) \
            else idxes.to(device=self.device, dtype=torch.int32)
        pr = torch.as_tensor(np.asarray(priorities, dtype=np.float32)).to(self.device) if not torch.is_tensor(priorities) \
            else priorities.to(device=self.device, dtype=torch.float32)
        assert idx.numel() == pr.numel()                                                   # :328
        if idx.numel():
            # the reference's per-element asserts (:330-331); an unchecked index would be a stray device write into the trees
            assert bool((pr > 0).all()), "priorities must be > 0"
            assert bool(((idx >= 0) & (idx < len(self))).all()), "index out of range"
        _lib.check(_lib.lib().d4pg_replay_update_priorities(self.handle, idx.numel(), _lib.ptr(idx), _lib.ptr(pr),
                                                            _lib.stream_ptr()), "d4pg_replay_update_priorities")
        self._caller_wrote()

    def reduce(self, start=0, end=None):
        self.flush()
        out = torch.empty(2, dtype=torch.float32, device=self.device)
        e = 0 if end is None else int(end)
        _lib.check(_lib.lib().d4pg_replay_reduce(self.handle, int(start), e, _lib.ptr(out), _lib.stream_ptr()),
                   "d4pg_replay_reduce")
        return out.cpu().numpy()

    @property
    def max_priority(self):
        self.flush()
        return float(self.state[0].item())


class _TreeView(object):
    """`_it_sum` / `_it_min` facade: the reference's SegmentTree read API over the device tree."""

    def __init__(self, store, which):
        self._store, self._which = store, which

    def _tree(self):
        self._store.flush()
        return self._store.sum_tree if self._which == 0 else self._store.min_tree

    def __getitem__(self, idx):
        assert 0 <= idx < self._store.capacity                                              # :111
        return np.float32(self._tree()[self._store.capacity + idx].item())

    def reduce(self, start=0, end=None):
        return np.float32(self._store.reduce(start, end)[self._which])

    def sum(self, start=0, end=None):
        return self.reduce(start, end)

    def min(self, start=0, end=None):
        return self.reduce(start, end)

    def values(self):
        """All 2*capacity node values (host copy)."""
        return self._tree().cpu().numpy()


class SegmentTree(object):
    """Standalone device segment tree with the reference constructor (:34-58).  `operation`
    must be addition or min (the only two the reference instantiates)."""

    def __init__(self, capacity, operation=None, neutral_element=None, _which=0):
        assert capacity > 0 and capacity & (capacity - 1) == 0, "capacity must be positive and a power of 2."
        self._capacity = capacity
        self._which = _which
        self._store = _DeviceReplay(capacity, 1.0, True, obs_dim=1, act_dim=1)
        if self._store.handle is None:
            _lib.require_cuda()

    def __setitem__(self, idx, val):
        st = self._store
        i = torch.tensor([idx], dtype=torch.int32, device=st.device)
        v = torch.tensor([val], dtype=torch.float32, device=st.device)
        _lib.check(_lib.lib().d4pg_replay_set_leaves(st.handle, 1, _lib.ptr(i), _lib.ptr(v), _lib.ptr(v),
                                                     _lib.stream_ptr()), "d4pg_replay_set_leaves")
        st._caller_wrote()

    def __getitem__(self, idx):
        assert 0 <= idx < self._capacity
        tree = self._store.sum_tree if self._which == 0 else self._store.min_tree
        return np.float32(tree[self._capacity + idx].item())

    def reduce(self, start=0, end=None):
        return np.float32(self._store.reduce(start, end)[self._which])


class SumSegmentTree(SegmentTree):
    def __init__(self, capacity):
        super(SumSegmentTree, self).__init__(capacity, _which=0)

    def sum(self, start=0, end=None):
        return self.reduce(start, end)

    def find_prefixsum_idx(self, prefixsum):
        st = self._store
        assert 0 <= prefixsum <= self.sum() + 1e-5                                          # :141
        m = torch.tensor([float(prefixsum)], dtype=torch.float64, device=st.device)
        out = torch.empty(1, dtype=torch.int32, device=st.device)
        _lib.check(_lib.lib().d4pg_replay_find_prefixsum(st.handle, 1, _lib.ptr(m), _lib.ptr(out), _lib.stream_ptr()),
                   "d4pg_replay_find_prefixsum")
        return int(out.item())


class MinSegmentTree(SegmentTree):
    def __init__(self, capacity):
        super(MinSegmentTree, self).__init__(capacity, _which=1)

    def min(self, start=0, end=None):
        return self.reduce(start, end)


def _to_host_batch(o):
    return (o["s"].cpu().numpy(), o["a"].cpu().numpy(), o["r"].cpu().numpy(), o["s2"].cpu().numpy(),
            o["d"].cpu().numpy().astype(bool))


class ReplayBuffer(object):
    """Uniform-sampling ring buffer (:164-222)."""

    _prioritized = False

    def __init__(self, size, obs_dim=None, act_dim=None, device=None, _alpha=1.0, obs_norm=None, nstep_tails=False):
        self._maxsize = size
        self._store = _DeviceReplay(size, _alpha, self._prioritized, obs_dim, act_dim, device,
                                    make_obs_normalizer(obs_norm, obs_dim, device), nstep_tails)

    @property
    def obs_normalizer(self):
        """The ObsNormalizer every insert updates (None without obs_norm=)."""
        return self._store.obs_norm

    def __len__(self):
        return len(self._store)

    @property
    def _next_idx(self):
        return (self._store._next_idx + self._store._n_staged) % self._store.size

    def add(self, obs_t, action, reward, obs_tp1, done):
        self._store.add(obs_t, action, reward, obs_tp1, done)

    def add_batch(self, obs_t, action, reward, obs_tp1, done):
        """n transitions at once.  Host arrays of up to 4096 rows take the packed single-copy path."""
        if isinstance(obs_t, np.ndarray) or (torch.is_tensor(obs_t) and not obs_t.is_cuda):
            self._store.add_batch_host(obs_t, action, reward, obs_tp1, done)
        else:
            self._store.add_batch(obs_t, action, reward, obs_tp1, done)

    def add_episode(self, obs, action, reward, obs_next, done, n_steps=1, gamma=0.99):
        """One episode of consecutive steps; the n-step return is accumulated on the device at insert
        (the arithmetic of replay_memory.py:38-45).  Returns the number of transitions inserted."""
        return self._store.add_episode_nstep(obs, action, reward, obs_next, done, n_steps, gamma)

    def add_her_episode(self, obs, obs_next, goal, achieved_goal_next, action, reward, done, **kw):
        """Hindsight relabelling on the device (main.py:154-184); see _DeviceReplay.add_her_episode."""
        return self._store.add_her_episode(obs, obs_next, goal, achieved_goal_next, action, reward, done, **kw)

    def add_steps(self, obs, action, reward, obs_next, terminated, truncated=None, n_steps=1, gamma=0.99):
        """One vector step of E environments, with the n-step windows kept on the device (DESIGN.md §3 "Streaming
        n-step insert").  obs / obs_next [E, obs_dim] (obs_next: the true next or final observation, not an auto-reset
        one), action [E, act_dim], reward [E], terminated / truncated bool [E] (truncated=None: no truncation); numpy,
        CPU or CUDA tensors.  Returns the number of rows inserted.

        Environment e appends (s, a, r) to its window; once the window holds n_steps steps of the current episode, the
        row (s_{t-n+1}, a_{t-n+1}, R, obs_next_t, terminated_t) is inserted with R the reference's left-to-right f64
        return (replay_memory.py:38-45, as add_episode); then terminated or truncated clears the window.  Windows that
        never fill are dropped.  The stored action is the window's oldest, as replay_memory.py:44 stores it, not the
        episode's last action that main.py:233 stores.  The rows of one call go in ascending e, which fixes their ring
        positions, their leaves and the normalizer's fold; with n_steps=1 a call stores what add_batch stores (a reward
        of -0.0 becomes +0.0, as in the reference's loop).

        The first call fixes E, n_steps and gamma; a call that changes one raises ValueError until drop_steps().  CUDA
        terminated / truncated are read back asynchronously and waited for at the next call.  The pending windows are
        not part of any checkpoint.

        With nstep_tails=True (DESIGN.md §3 "Episode tails") an episode of L steps that ends -- terminated or
        truncated -- also stores its last min(L, n_steps - 1) starts u as shorter rows (s_u, a_u, R over the k = L - u
        remaining rewards, the final obs_next, terminated) with horizon k in `_store.horizon` (0 for every full row), so
        a learner bootstraps them with gamma^k.  They are inserted by the NEXT call, ahead of that call's own rows, and
        are lost by drop_steps(); nothing flushes them when the stream stops.  One call may then insert up to
        E * (n_steps - 1) rows, which must not exceed the buffer size."""
        return self._store.add_steps(obs, action, reward, obs_next, terminated, truncated, n_steps, gamma)

    def drop_steps(self):
        """Discard the pending n-step windows of add_steps."""
        self._store.drop_steps()

    def add_goal_steps(self, obs, desired_goal, action, reward, obs_next, achieved_goal_next, terminated, truncated=None,
                       her_ratio=0.8, threshold=0.05, her_action="reference", max_episode_steps=50, seed=0):
        """One vector step of E goal-conditioned environments, with hindsight relabelling on the device (DESIGN.md §3
        "Streaming hindsight relabelling").  obs / obs_next [E, So], desired_goal / achieved_goal_next [E, G] (the goal
        achieved after the step), action [E, A], reward [E], terminated / truncated bool [E] (truncated=None: no
        truncation); numpy, CPU or CUDA tensors.  The buffer's obs_dim is So + G.  Returns the number of rows inserted.

        Environment e appends the step to its current episode, which ends on terminated or truncated.  An episode of L
        steps that ends at one call is inserted at the next (or by flush_goal_steps()), before that call's step: for
        every t the row (obs_t || goal_t, a_t, r_t, obs_next_t || goal_t, terminated_t), and, with probability
        her_ratio, directly after it the copy whose goal is the achieved goal after a uniformly drawn future step
        f in [t, L), with reward -(||achieved_t - goal'|| > threshold) and done = (reward == 0) -- main.py:154-184, the
        rows add_her_episode stores.  The copy's action is the episode's last action (her_action="reference", as
        main.py:184 stores it) or a_t ("own").  Unlike main.py, an episode that ends in success is stored too.  Rows go
        in ascending e, then t; goals and rewards are stored widened to f64 exactly.

        The draws come from numpy.random.default_rng(seed), per call over the ended episodes in ascending e: one
        random(sum L) for the selection, then one integers(t, L) over the selected steps.  A vectorized stream cannot
        keep the interleaved np.random order of main.py; add_her_episode keeps it for one episode.

        The first call fixes E, the dims, her_ratio, threshold, her_action, max_episode_steps and seed; a call that
        changes one raises ValueError until drop_goal_steps().  So do an episode longer than max_episode_steps,
        E * 2 * max_episode_steps > size, and add_steps while these episodes are pending (or the reverse).  CUDA
        terminated / truncated are read back asynchronously and waited for at the next call.  The pending episodes
        are not part of any checkpoint."""
        return self._store.add_goal_steps(obs, desired_goal, action, reward, obs_next, achieved_goal_next, terminated,
                                          truncated, her_ratio, threshold, her_action, max_episode_steps, seed)

    def flush_goal_steps(self):
        """Insert the episodes of add_goal_steps that have ended, without taking a step (e.g. before training on them).
        Returns the number of rows inserted."""
        return self._store.flush_goal_steps()

    def drop_goal_steps(self):
        """Discard the pending episodes of add_goal_steps."""
        self._store.drop_goal_steps()

    def _encode_sample(self, idxes):
        return _to_host_batch(self._store.gather(idxes))

    def sample(self, batch_size):
        idxes = [random.randint(0, len(self) - 1) for _ in range(batch_size)]              # :221
        return self._encode_sample(idxes)


class PrioritizedReplayBuffer(ReplayBuffer):
    """Proportional prioritized replay (:224-335) on GPU-resident fp32 sum/min trees."""

    _prioritized = True

    def __init__(self, size, alpha, obs_dim=None, act_dim=None, device=None, obs_norm=None, nstep_tails=False):
        assert alpha >= 0                                                                    # :240
        self._alpha = alpha
        super(PrioritizedReplayBuffer, self).__init__(size, obs_dim, act_dim, device, _alpha=alpha, obs_norm=obs_norm,
                                                      nstep_tails=nstep_tails)
        self._it_sum = _TreeView(self._store, 0)
        self._it_min = _TreeView(self._store, 1)

    @property
    def _max_priority(self):
        return self._store.max_priority

    def sample(self, batch_size, beta, uniforms=None):
        """-> (obs, act, rew, obs2, done, weights, idxes) as the reference returns them:
        host numpy arrays, `idxes` a list of ints.  `uniforms` (optional) overrides the
        `random.random()` draws."""
        assert beta > 0                                                                      # :299
        o = self._store.sample_proportional(batch_size, beta, uniforms)
        idxes = [int(i) for i in o["idx"].cpu().numpy()]
        return tuple(list(_to_host_batch(o)) + [o["w"].cpu().numpy(), idxes])

    def update_priorities(self, idxes, priorities):
        self._store.update_priorities(idxes, priorities)
