"""`DDPG` with the reference's constructor and method names (ddpg.py:15-255); the body of
`train()` is one `d4pg_learner_step` call into libd4pg_sm90.so (a CUDA graph of hand-written
sm_90a kernels), not Python/NumPy/ATen.

Reference behaviours kept on purpose (SURVEY.md H3-H9), each switchable only explicitly:
  * importance weights are sampled but NOT used by the loss                (ddpg.py:217)
  * priority = |sum_j m_ij q_ij| + 1e-6, not a KL/CE                       (ddpg.py:221-222,253)
  * the live projection discounts with gamma even when n_steps > 1         (ddpg.py:155);
    `projection="nstep"` selects the gamma**n variant (ddpg.py:122-140)
  * the actor gradient uses the critic weights from BEFORE this step's critic update
  * Adam betas (0.9, 0.9) come from SharedAdam; DDPG's own lr_actor/lr_critic optimisers are
    constructed but never stepped (ddpg.py:67-68)
"""
import ctypes as C
import random

import numpy as np
import torch

from . import _lib
from .models import CriticHead, actor, critic
from .obs_norm import make_obs_normalizer
from .prioritized_replay_memory import LinearSchedule, PrioritizedReplayBuffer, check_her_params
from .random_process import AdaptiveParamNoiseSpec, GaussianNoise, OrnsteinUhlenbeckProcess
from .replay_memory import Replay
from .shared_adam import SharedAdam, check_max_grad_norm
from .utils import default_device

# Philox counter of perturbation j (DDPG.perturb_actor / adapt_param_noise): 2^63 + 2^62 + j, apart from act()'s
# 2^63 + k (k < 2^62) and from the learner sampler's step counter
PERTURB_COUNTER_BASE = (1 << 63) + (1 << 62)


class _Learner(object):
    """Owns the C learner handle and the device buffers handed to it."""

    def __init__(self, ddpg, global_model):
        _lib.require_cuda()
        L = _lib.lib()
        dev = ddpg.device
        g = global_model
        opt_a, opt_c = ddpg.optimizer_global_actor, ddpg.optimizer_global_critic
        lr_a, b1, b2, eps = opt_a.hyper()
        lr_c, b1c, b2c, epsc = opt_c.hyper()
        if (b1, b2, eps) != (b1c, b2c, epsc):
            raise _lib.D4PGError("actor and critic SharedAdam must share betas/eps")
        # local networks alias the global storage (what ddpg.py:104-108,118-120 converge to)
        if g is not ddpg:
            ddpg.actor.adopt_flat(g.actor.flat_params())
            ddpg.critic.adopt_flat(g.critic.flat_params())
        Pa, Pc = ddpg.actor._total, ddpg.critic._total
        self.grads = torch.zeros(Pa + Pc, dtype=torch.float32, device=dev)
        for net, view in ((ddpg.actor, self.grads[:Pa]), (ddpg.critic, self.grads[Pa:])):
            net._flat_grad = view
            net._bind_grads()
        ma, va = opt_a.moments(g.actor)
        mc, vc = opt_c.moments(g.critic)
        B = ddpg.batch_size
        cfg = _lib.LearnerConfig()
        cfg.obs_dim, cfg.act_dim, cfg.n_atoms, cfg.batch = ddpg.obs_dim, ddpg.act_dim, ddpg.n_atoms, B
        # n_atoms is the head width (3K for a mixture); the library reads v_min / v_max only for a categorical head
        head = ddpg.critic_head
        cfg.dist_type, cfg.n_components, cfg.qr_kappa = head.code, head.n_components or 0, head.kappa or 0.0
        cfg.v_min, cfg.v_max = (float(head.v_min), float(head.v_max)) if head.kind == "categorical" else (0.0, 0.0)
        cfg.gamma = float(ddpg.gamma)
        cfg.n_steps = int(ddpg.n_steps)
        cfg.proj_mode = 1 if ddpg.projection == "nstep" else 0
        cfg.tau = float(ddpg.tau)
        cfg.lr_actor, cfg.lr_critic, cfg.beta1, cfg.beta2, cfg.adam_eps = lr_a, lr_c, b1, b2, eps
        cfg.prioritized = 1 if ddpg.prioritized_replay else 0
        if ddpg.prioritized_replay:
            sch = ddpg.beta_schedule
            cfg.per_beta0, cfg.per_beta_final, cfg.per_beta_iters = sch.initial_p, sch.final_p, sch.schedule_timesteps
            cfg.prio_eps = ddpg.prioritized_replay_eps
        else:
            cfg.per_beta0, cfg.per_beta_final, cfg.per_beta_iters, cfg.prio_eps = 1.0, 1.0, 1, 1e-6
        cfg.precision = {"fp32": 0, "tf32x3": 1, "tf32": 2, "bf16": 3}[ddpg.precision]
        cfg.sample_mode = 0 if ddpg.sampling == "reference" else 1
        cfg.philox_seed = int(ddpg.philox_seed)
        cfg.world_size = ddpg.comm.world_size if ddpg.comm is not None else 1
        cfg.use_graph = 1 if ddpg.use_graph else 0
        cfg.loss_flags = ((1 if ddpg.importance_weighted else 0) | (2 if ddpg.priority == "ce" else 0) |
                          (4 if ddpg.actor_critic == "post_update" else 0))
        # plan 1: fp32 = FFMA chain tiles; tf32x3 / tf32 = wgmma chain tiles (mlp_tc_chain.cu); plan 0: one launch per level
        # (bf16 always runs plan 0)
        cfg.chain = {"levels": 0, "cluster": 1, False: 0, True: 1, 0: 0, 1: 1}[ddpg.chain]
        # device sampling: step t samples batch t+1 on a side branch; reference sampling (host-drawn uniforms): the host
        # pipeline -- train() samples batch k on the learner's ingest stream, behind the add()s issued there, while step
        # k-1 still runs (needs the CUDA-graph step)
        cfg.prefetch = 1 if (ddpg.prefetch and (cfg.sample_mode == 1 or ddpg.use_graph)) else 0
        # per-network clipping thresholds from DDPG, decay from the two global optimisers (which may differ)
        cfg.max_grad_norm_actor, cfg.max_grad_norm_critic = ddpg.max_grad_norm
        cfg.weight_decay_actor, cfg.weight_decay_critic = opt_a.weight_decay(), opt_c.weight_decay()
        cfg.obs_norm = 1 if ddpg.obs_normalizer is not None else 0
        cfg.nstep_tails = 1 if ddpg.nstep_tails else 0
        if cfg.obs_norm and cfg.world_size > 1:
            raise _lib.D4PGError("obs_norm is not supported with a communicator of world size > 1")
        if any(ddpg.max_grad_norm) and cfg.world_size > 1:
            raise _lib.D4PGError("max_grad_norm is not supported with a communicator of world size > 1: the ranks' "
                                 "gradients are summed inside the Adam kernel, so the norm of the summed gradient does "
                                 "not exist before the update")
        self.cfg = cfg
        nws = L.d4pg_learner_workspace_floats(C.byref(cfg))
        f32 = torch.float32
        self.workspace = torch.zeros(nws, dtype=f32, device=dev)
        self.uniforms = torch.zeros(B, dtype=torch.float64, device=dev)
        self.positions = torch.zeros(B, dtype=torch.int32, device=dev)
        self.idx = torch.zeros(B, dtype=torch.int32, device=dev)
        self.weights = torch.zeros(B, dtype=f32, device=dev)
        self.prio = torch.zeros(B, dtype=f32, device=dev)
        self.td = torch.zeros(B, dtype=f32, device=dev)
        self.losses = torch.zeros(4, dtype=f32, device=dev)
        buf = _lib.LearnerBuffers()
        buf.actor, buf.actor_target = g.actor.flat_params().data_ptr(), ddpg.actor_target.flat_params().data_ptr()
        buf.critic, buf.critic_target = g.critic.flat_params().data_ptr(), ddpg.critic_target.flat_params().data_ptr()
        buf.grad_actor = self.grads.data_ptr()
        buf.grad_critic = self.grads.data_ptr() + 4 * Pa
        buf.adam_m_actor, buf.adam_v_actor = ma.data_ptr(), va.data_ptr()
        buf.adam_m_critic, buf.adam_v_critic = mc.data_ptr(), vc.data_ptr()
        buf.uniforms, buf.positions = self.uniforms.data_ptr(), self.positions.data_ptr()
        buf.idx, buf.weights = self.idx.data_ptr(), self.weights.data_ptr()
        buf.prio, buf.td, buf.losses = self.prio.data_ptr(), self.td.data_ptr(), self.losses.data_ptr()
        buf.workspace = self.workspace.data_ptr()
        self._keep = (ma, va, mc, vc, g.actor.flat_params(), g.critic.flat_params(),
                      ddpg.actor_target.flat_params(), ddpg.critic_target.flat_params())
        store = ddpg.replayBuffer._store
        if store.handle is None:
            raise _lib.D4PGError("train() called before any transition was added to the replay buffer")
        store.flush()
        h = C.c_void_p()
        if ddpg.comm is not None and cfg.world_size > 1:
            ddpg.comm.setup_peers(Pa + Pc)            # fused all-reduce over peer memory (collective call)
        comm = ddpg.comm.handle if ddpg.comm is not None else None
        _lib.check(L.d4pg_learner_create(C.byref(cfg), C.byref(buf), store.handle, comm, C.byref(h)), "d4pg_learner_create")
        self.handle = h
        self.global_model = g
        self.stream = torch.cuda.Stream(device=dev)      # graph capture needs a non-default stream
        self.dev_index = dev.index if dev.index is not None else torch.cuda.current_device()
        self.stream_ptr = C.c_void_p(self.stream.cuda_stream)
        self.step_host = L.d4pg_learner_step_host
        self.step_host_mt = L.d4pg_learner_step_host_mt
        self.read_losses = L.d4pg_learner_read_losses
        self.losses_out = (C.c_float * 4)()
        self.fresh_host_step = False          # the most recent step was a train() (its losses are in the pinned ring)
        self._store = store
        # parameter writes that advance a flat buffer's version counter (in-place ops on the flat buffer, load_state_dict,
        # hard_update, SharedAdam.step) are reported to the library by train(); see DDPG.weights_changed
        self._flats = (g.actor.flat_params(), g.critic.flat_params(), ddpg.actor_target.flat_params(), ddpg.critic_target.flat_params())
        self.seen_versions = None
        self.weights_changed = L.d4pg_learner_weights_changed
        ing = L.d4pg_learner_ingest_stream(h)
        store.attach_ingest_stream(int(ing) if ing else None)   # host pipeline: add_batch_host goes to the ingest stream
        if opt_a.step_count or (ddpg.prioritized_replay and ddpg.beta_schedule.t):
            _lib.check(L.d4pg_learner_set_counters(h, opt_a.step_count,
                                                   ddpg.beta_schedule.t if ddpg.prioritized_replay else 0,
                                                   _lib.stream_ptr()), "d4pg_learner_set_counters")

    def tensor(self, name, dtype=torch.float32):
        """Copy of a named intermediate.  2-D planes come back as [rows, pitch] (pitch >= width)."""
        p, n, ld = C.c_void_p(), C.c_int64(), C.c_int32()
        _lib.check(_lib.lib().d4pg_learner_tensor(self.handle, name.encode(), C.byref(p), C.byref(n), C.byref(ld)),
                   "d4pg_learner_tensor")
        esize = {torch.float32: 4, torch.float64: 8, torch.uint8: 1}[dtype]
        typestr = {torch.float32: "<f4", torch.float64: "<f8", torch.uint8: "|u1"}[dtype]

        class _Arr(object):
            __cuda_array_interface__ = {"shape": (int(n.value),), "typestr": typestr, "data": (int(p.value), False),
                                        "version": 2, "strides": (esize,)}
        t = torch.as_tensor(_Arr(), device=self.workspace.device).clone()
        return t.view(-1, ld.value) if ld.value > 1 else t

    def close(self):
        if self.handle is not None:
            if getattr(self, "_store", None) is not None:
                self._store.attach_ingest_stream(None)            # joins the ingest stream first
                self._store = None
            _lib.lib().d4pg_learner_destroy(self.handle)
            self.handle = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


HER_DEFAULTS = {"her_ratio": 0.8, "threshold": 0.05, "her_action": "reference", "max_episode_steps": 50, "seed": 0}


def _her_params(her):
    """DDPG(her=...): None / False -> None, True -> the defaults, a dict -> the defaults updated with it, validated."""
    if her is None or her is False:
        return None
    if her is True:
        her = {}
    if not isinstance(her, dict) or set(her) - set(HER_DEFAULTS):
        raise ValueError("her must be None, True or a dict with keys from %s, got %r" % (sorted(HER_DEFAULTS), her))
    p = dict(HER_DEFAULTS, **her)
    return dict(zip(("her_ratio", "threshold", "her_action", "max_episode_steps", "seed"),
                    check_her_params(p["her_ratio"], p["threshold"], p["her_action"], p["max_episode_steps"], p["seed"])))


class DDPG:
    replayBuffer = None

    def __init__(self, obs_dim, act_dim, env=None, memory_size=50000, batch_size=64,
                 lr_critic=1e-4, lr_actor=1e-4, gamma=0.99, tau=0.001, prioritized_replay=True,
                 critic_dist_info=None, n_steps=1,
                 # ---- GPU build extensions (keyword-only in spirit; reference callers never pass them)
                 device=None, sampling="reference", projection="reference", precision="fp32",
                 use_graph=True, philox_seed=0, comm=None, chain="cluster", prefetch=True, track_weights=True,
                 importance_weighted=False, priority="reference", actor_critic="reference", max_grad_norm=None,
                 obs_norm=None, param_noise=None, nstep_tails=False, her=None):
        # adaptive parameter-space exploration noise (random_process.AdaptiveParamNoiseSpec, DESIGN §3): None = off
        if param_noise is not None and not isinstance(param_noise, AdaptiveParamNoiseSpec):
            raise ValueError("param_noise must be None or an AdaptiveParamNoiseSpec, got %r" % (param_noise,))
        self.param_noise = param_noise
        self.gamma = gamma
        self.n_steps = n_steps
        self.n_step_gamma = self.gamma ** self.n_steps
        self.batch_size = batch_size
        self.obs_dim, self.act_dim = obs_dim, act_dim
        self.memory_size = memory_size
        self.tau = tau
        self.env = env
        self.device = torch.device(device) if device is not None else default_device()
        assert sampling in ("reference", "device") and projection in ("reference", "nstep")
        # "bf16": every MLP GEMM operand rounded to bf16, fp32 accumulate; runs the "levels" plan whatever `chain` says
        assert precision in ("fp32", "tf32x3", "tf32", "bf16")
        self.sampling, self.projection, self.precision = sampling, projection, precision
        # episode tails (DESIGN.md §3 "Episode tails"): observe() also stores the last n_steps - 1 starts of every episode
        # as shorter rows, each bootstrapped with gamma^k of its own horizon k.  Fixed here: the buffer and the learner
        # both depend on it.  The reference projection discounts every row with gamma, so a horizon means nothing there
        self.nstep_tails = bool(nstep_tails)
        if self.nstep_tails and projection == "reference" and n_steps > 1:
            raise ValueError('nstep_tails=True with n_steps > 1 needs projection="nstep": the reference projection '
                             'discounts every row with gamma (no per-row horizon)')
        # streaming hindsight relabelling (DESIGN.md §3 "Streaming hindsight relabelling"): observe_goals() stores goal-
        # conditioned steps with these parameters.  None = off, True = the defaults, or a dict of some of them.  One-step
        # rows only, as main.py stores them: n-step returns over relabelled rewards are not defined here
        self.her = _her_params(her)
        if self.her is not None and n_steps > 1:
            raise ValueError("her= stores one-step transitions (main.py:154-184); it cannot be combined with n_steps = %r"
                             % (n_steps,))
        self.use_graph, self.philox_seed, self.comm = use_graph, philox_seed, comm
        # step plan of the MLP passes: "cluster" (default) cluster-fused layer chains (exact FFMA tiles for fp32,
        # wgmma tiles for tf32x3 / tf32), "levels" one launch per dependency level
        self.chain = chain
        # device-side sampling only: step t already samples batch t+1 behind its own backward pass (identical results)
        self.prefetch = prefetch
        self.track_weights = track_weights
        # corrected-semantics switches (default = the reference's behaviour, SURVEY.md H3 / H4)
        assert priority in ("reference", "ce") and actor_critic in ("reference", "post_update")
        self.importance_weighted, self.priority = bool(importance_weighted), priority
        # "post_update": the actor gradient flows through the critic AFTER this step's critic update (corrected SURVEY.md
        # H7); "reference": through the stale pre-update copy, as ddpg.py:229-247 does.  Tensor-core chain plan, one GPU.
        self.actor_critic = actor_critic
        # clip each network's gradient to a global norm before its Adam update (torch.nn.utils.clip_grad_norm_): None =
        # off, a positive float for both networks, float("inf") = measure and report only, or an (actor, critic) pair.
        # The norms of every step are then read with last_grad_norms(); .grad keeps the unclipped gradient.  One GPU.
        pair = max_grad_norm if isinstance(max_grad_norm, (tuple, list)) else (max_grad_norm, max_grad_norm)
        if len(pair) != 2:
            raise ValueError("max_grad_norm must be None, a number or an (actor, critic) pair")
        self.max_grad_norm = tuple(check_max_grad_norm(x) for x in pair)
        # running per-feature observation normalization (obs_norm.py): None / False = off, True = clip 5, eps 1e-8, or
        # {"clip": c, "eps": e}.  Every replay insert updates the statistics; the learner's s / s2 and the `state` input
        # of the four networks below are normalized with them.  One GPU.
        self.obs_normalizer = make_obs_normalizer(obs_norm, obs_dim, self.device)
        if self.obs_normalizer is not None and comm is not None and comm.world_size > 1:
            raise _lib.D4PGError("obs_norm is not supported with a communicator of world size > 1: each rank would "
                                 "normalize with the statistics of its own replay shard")

        # the critic head (models.CriticHead); the critic built below checks its ranges
        if priority == "ce" and critic_dist_info["type"] == "mixture_of_gaussian":
            raise _lib.D4PGError('priority="ce" is not supported with a mixture_of_gaussian critic: the '
                                 'cross-entropy of a density can be negative')
        head = self.critic_head = CriticHead(critic_dist_info, learner=True)
        self.dist_type, self.n_atoms, self.n_components = head.kind, head.width, head.n_components
        self.n_quantiles, self.qr_kappa = head.n_quantiles, head.kappa
        self.v_min, self.v_max, self.delta, self.bin_centers = head.v_min, head.v_max, head.delta, head.bin_centers

        # networks, built in the reference's order so a seeded RNG yields the same weights (ddpg.py:56-64)
        self.actor = actor(input_size=obs_dim, output_size=act_dim, device=self.device)
        self.actor_target = actor(input_size=obs_dim, output_size=act_dim, device=self.device)
        self.actor_target.load_state_dict(self.actor.state_dict())
        self.critic = critic(state_size=obs_dim, action_size=act_dim, dist_info=critic_dist_info, device=self.device)
        self.critic_target = critic(state_size=obs_dim, action_size=act_dim, dist_info=critic_dist_info, device=self.device)
        self.critic_target.load_state_dict(self.critic.state_dict())
        if self.obs_normalizer is not None:
            for net in (self.actor, self.actor_target, self.critic, self.critic_target):
                net.obs_normalizer = self.obs_normalizer

        # constructed for attribute compatibility; like the reference's, never stepped by train()
        self.optimizer_actor = SharedAdam(self.actor.parameters(), lr=lr_actor, betas=(0.9, 0.999))
        self.optimizer_critic = SharedAdam(self.critic.parameters(), lr=lr_critic, betas=(0.9, 0.999))
        self.optimizer_global_actor = None
        self.optimizer_global_critic = None

        self.noise = GaussianNoise(dimension=act_dim, num_epochs=5000)                       # ddpg.py:75
        # act(): exploring calls so far (the Philox counter of the next one is 2^63 + this), the device OU state and the
        # per-E workspace / pitch-4 input buffers
        self._act_calls = 0
        self._exploration_state = None
        self._act_buffers = {}
        # parameter noise: perturbations drawn so far (the Philox counter of the next is PERTURB_COUNTER_BASE + this),
        # the device {sigma, last distance}, the rollout's perturbed actor and adapt_param_noise's own perturbed copy
        self._perturbations = 0
        self._param_noise_state = None
        self._perturbed_actor = None
        self._adaptive_flat = None

        self.prioritized_replay = prioritized_replay
        if self.prioritized_replay:                                                          # ddpg.py:78-87
            self.replayBuffer = PrioritizedReplayBuffer(self.memory_size, alpha=0.6, obs_dim=obs_dim,
                                                        act_dim=act_dim, device=self.device, obs_norm=self.obs_normalizer,
                                                        nstep_tails=self.nstep_tails)
            self.beta_schedule = LinearSchedule(100000, initial_p=0.4, final_p=1.0)
            self.prioritized_replay_eps = 1e-6
        else:
            self.replayBuffer = Replay(self.memory_size, self.env, n_steps=self.n_steps, gamma=self.gamma,
                                       obs_dim=obs_dim, act_dim=act_dim, device=self.device, obs_norm=self.obs_normalizer,
                                       nstep_tails=self.nstep_tails)
        self._learner = None

    # ---- reference plumbing methods ------------------------------------------------------
    def hard_update(self):                                                                   # ddpg.py:92-94
        self.actor_target.load_state_dict(self.actor.state_dict())
        self.critic_target.load_state_dict(self.critic.state_dict())

    def share_memory(self):                                                                  # ddpg.py:96-98
        self.actor.share_memory()
        self.critic.share_memory()

    def assign_global_optimizer(self, optimizer_global_actor, optimizer_global_critic):      # ddpg.py:100-102
        self.optimizer_global_actor = optimizer_global_actor
        self.optimizer_global_critic = optimizer_global_critic
        self._drop_learner()

    def copy_gradients(self, model_local, model_global):                                     # ddpg.py:104-108
        if model_global.flat_params().data_ptr() == model_local.flat_params().data_ptr():
            return                                    # shared storage: gradients are already "global"
        model_global._flat_grad = model_local.flat_grads()
        model_global._bind_grads()

    def weights_changed(self):
        """Report a parameter write the learner cannot see.  train() notices writes that advance the version counter of
        an actor / critic / target flat buffer: in-place torch operations on `flat_params()`, load_state_dict (so
        hard_update and sync_local_global) and SharedAdam.step.  A parameter's own version counter is not the flat
        buffer's, so in-place writes to single parameters (`with torch.no_grad(): p.copy_(..)`, `p.data`) and writes
        through raw pointers bypass it -- call this after them (or construct with track_weights=False: the weight images
        are then rebuilt on every step)."""
        if self._learner is not None and self._learner.handle is not None:
            self._learner.seen_versions = None

    def update_target_parameters(self):                                                      # ddpg.py:110-116
        _lib.require_cuda()
        self.weights_changed()
        for tgt, src in ((self.actor_target, self.actor), (self.critic_target, self.critic)):
            _lib.check(_lib.lib().d4pg_polyak(_lib.ptr(tgt.flat_params()), _lib.ptr(src.flat_params()),
                                              tgt._total, float(self.tau), _lib.stream_ptr()), "d4pg_polyak")

    def sync_local_global(self, global_model):                                               # ddpg.py:118-120
        self.actor.load_state_dict(global_model.actor.state_dict())
        self.critic.load_state_dict(global_model.critic.state_dict())

    # ---- projections as standalone methods (numpy in / numpy out, computed on the GPU) --------
    def _project(self, target_z_dist, rewards, terminates, mode):
        if self.dist_type != "categorical":
            raise _lib.D4PGError("reproject2 / reproj_categorical_dist project onto the categorical atoms; this DDPG has "
                                 "a %s critic" % self.dist_type)
        _lib.require_cuda()
        p = torch.as_tensor(np.ascontiguousarray(target_z_dist, dtype=np.float32)).to(self.device)
        B, N = p.shape
        r = torch.as_tensor(np.asarray(rewards, dtype=np.float64).reshape(-1)).to(self.device)
        d = torch.as_tensor(np.asarray(terminates).reshape(-1).astype(bool).astype(np.uint8)).to(self.device)
        m = torch.empty(B, N, dtype=torch.float32, device=self.device)
        disc = self.n_step_gamma if mode == 1 else self.gamma
        _lib.check(_lib.lib().d4pg_proj_loss(_lib.ptr(p), _lib.ptr(p), None, _lib.ptr(r), _lib.ptr(d), B, N,
                                             float(self.v_min), float(self.v_max), float(disc), mode,
                                             _lib.PROJ_TARGET_IS_PROBS | _lib.PROJ_Q_IS_PROBS, 1e-6, 1.0 / B,
                                             _lib.ptr(m), None, None, None, None, None, None, None, None, None, None,
                                             _lib.stream_ptr()), "d4pg_proj_loss")
        return m.cpu().numpy()

    def reproject2(self, target_z_dist, rewards, terminates):                                # ddpg.py:142-185
        return self._project(target_z_dist, rewards, terminates, 0)

    def reproj_categorical_dist(self, target_z_dist, rewards, terminates):                   # ddpg.py:122-140
        return self._project(target_z_dist, rewards, terminates, 1).astype(np.float64)

    # ---- sampling -------------------------------------------------------------------------
    def sample(self, batch_size=None):                                                       # ddpg.py:187-197
        weights = None
        batch_idxes = None
        if self.prioritized_replay:
            experience = self.replayBuffer.sample(batch_size, beta=self.beta_schedule.value())
            (states, actions, rewards, next_states, terminates, weights, batch_idxes) = experience
        else:
            states, actions, rewards, next_states, terminates = self.replayBuffer.sample(self.batch_size)
        return states, actions, rewards, next_states, terminates, weights, batch_idxes

    # ---- storing transitions -----------------------------------------------------------------
    def observe(self, s, a, r, s2, terminated, truncated=None):
        """Store one vector step of E environments: `replayBuffer.add_steps(..., n_steps=self.n_steps, gamma=self.gamma)`,
        the n-step windows kept on the device (DESIGN.md §3 "Streaming n-step insert").  s / s2 [E, obs_dim] (s2 the
        true next or final observation), a [E, act_dim] (e.g. what act() returned), r [E], terminated / truncated bool
        [E]; numpy, CPU or CUDA tensors.  With `a = ddpg.act(s)` and device-resident environments the rollout step
        stays on the device.  Returns the number of rows inserted.  With DDPG(nstep_tails=True) the last n_steps - 1
        starts of every episode are stored too, at the next call (DESIGN.md §3 "Episode tails")."""
        return self.replayBuffer.add_steps(s, a, r, s2, terminated, truncated, n_steps=self.n_steps, gamma=self.gamma)

    def observe_goals(self, obs, desired_goal, a, r, obs_next, achieved_goal_next, terminated, truncated=None):
        """Store one vector step of E goal-conditioned environments with hindsight relabelling on the device:
        `replayBuffer.add_goal_steps(..., **her)` with the parameters of DDPG(her=...) (DESIGN.md §3 "Streaming
        hindsight relabelling").  obs / obs_next [E, So], desired_goal / achieved_goal_next [E, G], a [E, act_dim],
        r [E], terminated / truncated bool [E]; numpy, CPU or CUDA tensors; this DDPG's obs_dim is So + G.  An episode
        that ends is inserted, with its relabelled copies, at the next call (or replayBuffer.flush_goal_steps()).
        Returns the number of rows inserted."""
        if self.her is None:
            raise ValueError("observe_goals needs DDPG(her=True or a dict of HER parameters)")
        return self.replayBuffer.add_goal_steps(obs, desired_goal, a, r, obs_next, achieved_goal_next, terminated,
                                                truncated, **self.her)

    # ---- action selection -------------------------------------------------------------------
    def act(self, state, explore=True, reset=None):
        """The rollout's action, `np.clip(actor(s) + noise.sample(), -1, 1)` (main.py:145-146, 216-217, 279), for E
        environments in one launch on the caller's stream.  `state`: numpy or tensor, host or device, [obs_dim] or
        [E, obs_dim].  Returns an fp32 device tensor [E, act_dim] ([1, act_dim] for one row).

        The actor runs at fp32 (precision 0) with this DDPG's observation normalizer, if any.  explore=False returns
        actor(state) bit for bit.  explore=True adds the noise of `self.noise` -- GaussianNoise or
        OrnsteinUhlenbeckProcess, whose epsilon / mu / var (theta / sigma / dt) are read at each call -- drawn on the
        device from Philox (key philox_seed, counter 2^63 + the number of earlier exploring calls), and clips to
        [-1, 1] in fp64.  OU noise keeps one state row per environment in `exploration_state`; `reset` (bool [E]) restarts
        the rows of environments that began a new episode.  The arithmetic is in DESIGN.md §3 "Exploration".

        With DDPG(param_noise=...), explore=True runs `perturbed_actor` instead of the actor (drawing perturbation 0
        first if none was drawn yet) and adds the noise of `self.noise` to it; self.noise = None is parameter noise
        alone.  explore=False still runs the actor itself.  `reset` never re-perturbs (DESIGN.md §3 "Parameter-space
        noise")."""
        mode, params = self._act_noise(explore)
        x, E = self._act_rows(state)
        if mode == 2:
            st = self._exploration_state
            if st is not None and st.shape[0] != E:
                raise _lib.D4PGError("act: the Ornstein-Uhlenbeck state holds %d environments, this call has %d (assign "
                                     "exploration_state = None to start over)" % (st.shape[0], E))
            if reset is not None and tuple(np.shape(reset)) != (E,):
                raise ValueError("act: reset must be a bool mask of shape (%d,), got %s" % (E, tuple(np.shape(reset))))
        _lib.require_cuda()
        L = _lib.lib()
        S, A = self.obs_dim, self.act_dim
        flat = self.actor.flat_params()
        dev = flat.device
        if explore and self.param_noise is not None:
            pa = self._perturbed_actor
            if pa is None or pa.flat_params().device != dev:
                pa = self.perturb_actor()
            flat = pa.flat_params()
        bufs = self._act_workspace(E, dev)
        rows, lds = self._act_input(x, E, dev, bufs)
        st = rmask = None
        if mode == 2:
            st = self._exploration_state
            if st is None:
                st = torch.from_numpy(np.zeros((E, A))).to(dev)          # a copy, not a fill kernel
            rmask = self._act_reset(reset, dev) if reset is not None else None
        affine, clip = self._act_affine()
        out = torch.empty(E, A, dtype=torch.float32, device=dev)
        p = (C.c_double * 5)(*params)
        counter = (1 << 63) + self._act_calls
        _lib.check(L.d4pg_act(_lib.ptr(flat), S, A, _lib.ptr(rows), lds, E, affine, clip, mode, p,
                              int(self.philox_seed) & 0xFFFFFFFFFFFFFFFF, counter, _lib.ptr(st), _lib.ptr(rmask),
                              _lib.ptr(out), _lib.ptr(bufs[0]), _lib.stream_ptr()), "d4pg_act")
        if mode:
            self._act_calls += 1
        if mode == 2:
            self._exploration_state = st
        return out

    @property
    def exploration_state(self):
        """The device Ornstein-Uhlenbeck state of act(): None until the first exploring call with OU noise, then fp64
        [E, act_dim].  That call fixes E.  Assign None to drop it: the next call starts from zeros, with any E."""
        return self._exploration_state

    @exploration_state.setter
    def exploration_state(self, value):
        if value is not None:
            raise ValueError("exploration_state can only be set to None")
        self._exploration_state = None

    def _act_noise(self, explore):
        """(noise mode of d4pg_act, its parameters) for the current `self.noise`."""
        if not explore:
            return 0, ()
        nz = self.noise
        if self._param_noise_args() is not None and nz is None:
            return 0, ()                                  # parameter noise alone
        if isinstance(nz, GaussianNoise):
            return 1, tuple(float(v) for v in (nz.epsilon, nz.mu, nz.var))
        if isinstance(nz, OrnsteinUhlenbeckProcess):
            return 2, tuple(float(v) for v in (nz.epsilon, nz.theta, nz.mu, nz.sigma, nz.dt))
        raise _lib.D4PGError("act(explore=True) draws GaussianNoise or OrnsteinUhlenbeckProcess noise on the device; "
                             "self.noise is a %s" % type(nz).__name__)

    def _act_workspace(self, E, dev):
        """[d4pg_act workspace, pitch-4 input buffer or None] cached per E."""
        bufs = self._act_buffers.get(E)
        if bufs is None or bufs[0].device != dev:
            ws = torch.empty(_lib.lib().d4pg_act_workspace_floats(E, self.obs_dim), dtype=torch.float32, device=dev)
            bufs = self._act_buffers[E] = [ws, None]
        return bufs

    def _act_affine(self):
        """(affine pointer, clip) of the observation normalizer for d4pg_act, (None, 0.0) without one."""
        norm = self.obs_normalizer
        if norm is None:
            return None, 0.0
        norm._require()
        norm._join()
        return _lib.ptr(norm.affine), norm.clip

    def _act_rows(self, state):
        """(rows, E): `state` as [E, obs_dim], a tensor where it lives, anything else as float32 numpy."""
        x = state.detach() if torch.is_tensor(state) else np.asarray(state, dtype=np.float32)
        if x.ndim == 1:
            x = x.reshape(1, -1)
        if x.ndim != 2 or x.shape[1] != self.obs_dim:
            raise ValueError("act: expected states of shape (%d,) or (E, %d), got %s"
                             % (self.obs_dim, self.obs_dim, tuple(x.shape)))
        E = int(x.shape[0])
        if E < 1:
            raise ValueError("act: no states (E = 0)")
        if 2 * E * self.act_dim >= 2 ** 31:
            raise ValueError("act: E = %d rows of %d actions exceed the noise draw index (2 * E * act_dim < 2^31)"
                             % (E, self.act_dim))
        return x, E

    def _act_input(self, x, E, dev, bufs):
        """(rows, pitch) as d4pg_act reads them.  A float32 tensor on `dev` with 16-B aligned rows is read in place;
        anything else lands in the cached [E, pitch4(obs_dim)] buffer with one 2-D copy."""
        S = self.obs_dim
        if torch.is_tensor(x):
            if x.device.type == "cpu":
                x = x.to(torch.float32).contiguous().numpy()
            elif x.device != dev or x.dtype != torch.float32 or x.stride(1) != 1 or x.stride(0) < S:
                x = x.to(device=dev, dtype=torch.float32).contiguous()
        if torch.is_tensor(x) and x.stride(0) % 4 == 0 and x.data_ptr() % 16 == 0:
            return x, x.stride(0)
        if bufs[1] is None:
            bufs[1] = torch.empty(E, (S + 3) & ~3, dtype=torch.float32, device=dev)
        buf = bufs[1]
        if torch.is_tensor(x):
            src, lds = _lib.ptr(x), x.stride(0)
        else:
            x = np.ascontiguousarray(x, dtype=np.float32)
            src, lds = C.c_void_p(x.ctypes.data), S
        _lib.check(_lib.lib().d4pg_copy_rows_f32(_lib.ptr(buf), buf.stride(0), src, lds, E, S, _lib.stream_ptr()),
                   "d4pg_copy_rows_f32")
        return buf, buf.stride(0)

    @staticmethod
    def _act_reset(reset, dev):
        """The reset mask as a u8 device tensor (a bool / u8 device tensor is read in place)."""
        if torch.is_tensor(reset):
            r = reset.detach()
            if r.device == dev and r.dtype in (torch.bool, torch.uint8) and r.is_contiguous():
                return r.view(torch.uint8)
            reset = r.cpu().numpy()
        return torch.from_numpy(np.asarray(reset).astype(bool).astype(np.uint8)).to(dev)

    # ---- parameter-space noise ----------------------------------------------------------------
    def _param_noise_args(self):
        """`self.param_noise.check()` -- (initial_stddev, desired_action_stddev, adoption_coefficient) -- or None when
        parameter noise is off.  Raises ValueError for anything else, before any device work."""
        spec = self.param_noise
        if spec is None:
            return None
        if not isinstance(spec, AdaptiveParamNoiseSpec):
            raise ValueError("param_noise must be None or an AdaptiveParamNoiseSpec, got %r" % (spec,))
        return spec.check()

    def _require_param_noise(self, what):
        args = self._param_noise_args()
        if args is None:
            raise _lib.D4PGError("%s needs DDPG(param_noise=AdaptiveParamNoiseSpec(...))" % what)
        return args

    def _noise_state(self, dev, initial_stddev):
        st = self._param_noise_state
        if st is None or st.device != dev:
            st = torch.tensor([initial_stddev, float("nan")], dtype=torch.float64).to(dev)     # a copy, not a fill kernel
            self._param_noise_state = st
        return st

    def _perturb(self, src, dst, initial_stddev):
        """dst = src + sigma * N(0, 1) per logical parameter: perturbation j = self._perturbations (one launch)."""
        st = self._noise_state(src.device, initial_stddev)
        _lib.check(_lib.lib().d4pg_actor_perturb(_lib.ptr(src), self.obs_dim, self.act_dim, _lib.ptr(st),
                                                 int(self.philox_seed) & 0xFFFFFFFFFFFFFFFF,
                                                 PERTURB_COUNTER_BASE + self._perturbations, _lib.ptr(dst),
                                                 _lib.stream_ptr()), "d4pg_actor_perturb")
        self._perturbations += 1

    def perturb_actor(self):
        """Draw the next parameter perturbation of the actor into `perturbed_actor` (one launch on the caller's stream)
        and return that module.  Baselines' perturb_policy: call it at the start of every episode.  Reads the actor's
        current parameters and the device sigma of `param_noise_state`; the result is a snapshot that later train()
        steps do not change.  Perturbation j (j counts this DDPG's perturbations, including adapt_param_noise's, from 0)
        adds sigma * z to logical parameter i, z from Philox (key philox_seed, counter 2^63 + 2^62 + j, lanes 2i / 2i + 1);
        DESIGN.md §3 "Parameter-space noise"."""
        initial, _, _ = self._require_param_noise("perturb_actor")
        _lib.require_cuda()
        src = self.actor.flat_params()
        pa = self._perturbed_actor
        if pa is None or pa.flat_params().device != src.device:
            pa = actor.unfilled(self.obs_dim, self.act_dim, device=src.device)
            if self.obs_normalizer is not None:
                pa.obs_normalizer = self.obs_normalizer
            self._perturbed_actor = pa
        self._perturb(src, pa.flat_params(), initial)
        return pa

    def adapt_param_noise(self, states):
        """Adapt sigma to the policy distance on `states` ([B, obs_dim] raw observations, host or device; act()'s limits
        on B): perturb an adaptive copy of the actor with the current sigma (perturbation j), run the actor and the copy
        on the states without action noise, d = sqrt(mean((a_perturbed - a)^2)) in fp64, then sigma = sigma /
        adoption_coefficient if d > desired_action_stddev else sigma * adoption_coefficient.  Four launches on the
        caller's stream; returns d as a 0-d fp64 device tensor (a view of param_noise_state), without synchronising.
        `perturbed_actor` is not touched.  Baselines calls this every ~50 training steps on a replay batch."""
        initial, desired, coef = self._require_param_noise("adapt_param_noise")
        x, E = self._act_rows(states)
        _lib.require_cuda()
        L = _lib.lib()
        S, A = self.obs_dim, self.act_dim
        src = self.actor.flat_params()
        dev = src.device
        ad = self._adaptive_flat
        if ad is None or ad.device != dev:
            ad = self._adaptive_flat = torch.empty(self.actor._total, dtype=torch.float32, device=dev)
        bufs = self._act_workspace(E, dev)
        rows, lds = self._act_input(x, E, dev, bufs)
        affine, clip = self._act_affine()
        self._perturb(src, ad, initial)
        out = torch.empty(2, E, A, dtype=torch.float32, device=dev)
        for k, flat in enumerate((src, ad)):
            _lib.check(L.d4pg_act(_lib.ptr(flat), S, A, _lib.ptr(rows), lds, E, affine, clip, 0, None, 0, 0, None, None,
                                  _lib.ptr(out[k]), _lib.ptr(bufs[0]), _lib.stream_ptr()), "d4pg_act")
        st = self._param_noise_state
        _lib.check(L.d4pg_param_noise_adapt(_lib.ptr(out[0]), _lib.ptr(out[1]), E * A, desired, coef, _lib.ptr(st),
                                            _lib.stream_ptr()), "d4pg_param_noise_adapt")
        return st[1]

    @property
    def perturbed_actor(self):
        """The actor with the most recent perturb_actor() draw (an `actor` module: same dimensions and device, this
        DDPG's observation normalizer, precision 0), or None before the first.  Never part of the learner."""
        return self._perturbed_actor

    @property
    def param_noise_state(self):
        """fp64 [2] device tensor {sigma, last distance}: None until the first perturbation or adaptation, which
        creates it as {initial_stddev, NaN}.  Assign None to drop it: the next use starts again from initial_stddev."""
        return self._param_noise_state

    @param_noise_state.setter
    def param_noise_state(self, value):
        if value is not None:
            raise ValueError("param_noise_state can only be set to None")
        self._param_noise_state = None

    # ---- the hot path ----------------------------------------------------------------------
    def _drop_learner(self):
        if self._learner is not None:
            self._learner.close()
            self._learner = None

    def _get_learner(self, global_model):
        if self._learner is None or self._learner.global_model is not global_model:
            self._drop_learner()
            if self.optimizer_global_actor is None or self.optimizer_global_critic is None:
                raise _lib.D4PGError("call assign_global_optimizer(SharedAdam, SharedAdam) before train() "
                                     "(main.py:194)")
            self._learner = _Learner(self, global_model)
        return self._learner

    def train(self, global_model=None):
        """One learner gradient step (ddpg.py:200-255), asynchronous on the learner's stream.
        Results (losses, td, priorities, sampled indices) stay on the device; read them with
        `last_losses()` / `last_batch_info()`."""
        g = global_model if global_model is not None else self
        L = self._learner
        if L is None or L.global_model is not g:
            L = self._get_learner(g)
        store = self.replayBuffer._store
        if store._n_staged:
            store.flush()
        store.before_step()                   # the ingest stream's sample waits for the caller's replay writes
        f = L._flats
        v = (f[0]._version, f[1]._version, f[2]._version, f[3]._version) if self.track_weights else None
        if v != L.seen_versions or v is None:
            L.weights_changed(L.handle)
            L.seen_versions = v
        B = self.batch_size
        # one library call: order after the caller's stream, H2D of this step's host inputs, the step's
        # CUDA graph on the learner stream, order the caller's stream after it
        if self.sampling == "reference" and self.prioritized_replay:
            # B x random.random() in order (prioritized_replay_memory.py:262): the 2*B raw MT19937 words are drawn in
            # one call -- same generator state afterwards -- and turned into the doubles by the library
            rc = L.step_host_mt(L.handle, random.randbytes(8 * B), _lib.raw_stream(L.dev_index), L.stream_ptr)
        elif self.sampling == "reference":
            pos = np.ascontiguousarray(self.replayBuffer.sample_positions(B), dtype=np.int32)
            rc = L.step_host(L.handle, None, pos.ctypes.data, _lib.raw_stream(L.dev_index), L.stream_ptr)
        else:
            rc = L.step_host(L.handle, None, None, _lib.raw_stream(L.dev_index), L.stream_ptr)
        if rc:
            _lib.check(rc, "d4pg_learner_step_host")
        L.fresh_host_step = True
        if self.prioritized_replay:
            self.beta_schedule.t += 1
        for opt in (self.optimizer_global_actor, self.optimizer_global_critic):
            opt.step_count += 1

    def train_n(self, n, global_model=None):
        """`n` gradient steps in one C call (device-side sampling only): the learner's CUDA graph is
        replayed back to back with no Python in between."""
        if self.sampling != "device":
            raise _lib.D4PGError("train_n needs sampling='device' (host-drawn uniforms are per-step inputs)")
        g = global_model if global_model is not None else self
        L = self._get_learner(g)
        self.replayBuffer._store.flush()
        L.stream.wait_stream(torch.cuda.current_stream())
        _lib.check(_lib.lib().d4pg_learner_run(L.handle, int(n), C.c_void_p(L.stream.cuda_stream)), "d4pg_learner_run")
        L.fresh_host_step = False
        torch.cuda.current_stream().wait_stream(L.stream)
        if self.prioritized_replay:
            self.beta_schedule.t += n
        for opt in (self.optimizer_global_actor, self.optimizer_global_critic):
            opt.step_count += n

    def last_losses(self, lag=0):
        """(critic_loss, actor_loss) of the most recent train() -- waits for that step's result (a 16-byte D2H copy every
        train() queues).  `lag=1` returns the result of the train() call BEFORE the most recent one instead, which lets a
        training loop read every step's losses without draining the GPU: `train(); losses = last_losses(lag=1)`.
        After train_n / profile_step (no per-step copy queued) the result is read synchronously."""
        L = self._learner
        if L.fresh_host_step:
            rc = _lib.lib().d4pg_learner_fetch_losses(L.handle, int(lag), L.losses_out)
            if rc:
                _lib.check(rc, "d4pg_learner_fetch_losses")
            return L.losses_out[0], L.losses_out[1]
        rc = L.read_losses(L.handle, L.losses_out, L.stream_ptr)       # D2H + wait: the step's result
        if rc:
            _lib.check(rc, "d4pg_learner_read_losses")
        return L.losses_out[0], L.losses_out[1]

    def last_grad_norms(self, lag=0):
        """(actor_norm, critic_norm): the global gradient norms, before clipping, of the step `last_losses(lag)` reports,
        read the same way.  A network without a threshold reports 0.0.  Needs DDPG(max_grad_norm=...)."""
        if not any(self.max_grad_norm):
            raise _lib.D4PGError("last_grad_norms needs DDPG(max_grad_norm=...): the norm is only measured when a "
                                 "threshold (or float('inf')) is set")
        self.last_losses(lag)
        out = self._learner.losses_out
        return out[2], out[3]

    def last_batch_info(self):
        """Device tensors of the most recent step: sampled idx, IS weights, td, new priorities."""
        L = self._learner
        torch.cuda.current_stream().wait_stream(L.stream)
        return dict(idx=L.idx, weights=L.weights, td=L.td, prio=L.prio)

    def debug_tensor(self, name, shape=None, dtype=torch.float32):
        L = self._learner
        L.stream.synchronize()
        t = L.tensor(name, dtype)
        if shape is not None and t.dim() == 2:
            return t[:, :shape[1]].contiguous()          # drop the pad columns of the row pitch
        return t.view(*shape) if shape is not None else t

    def profile_step(self, global_model=None):
        """One eager step with CUDA events around every launch -> [(launcher, ms), ...].
        Counts as a real training step (device-side sampling state advances)."""
        g = global_model if global_model is not None else self
        L = self._get_learner(g)
        self.replayBuffer._store.flush()
        L.stream.wait_stream(torch.cuda.current_stream())
        n, cap, stride = C.c_int32(), 64, 48
        ms = (C.c_float * cap)()
        names = C.create_string_buffer(cap * stride)
        with torch.cuda.stream(L.stream):
            if self.sampling == "reference":
                if self.prioritized_replay:
                    L.uniforms.copy_(torch.tensor([random.random() for _ in range(self.batch_size)], dtype=torch.float64))
                else:
                    L.positions.copy_(torch.as_tensor(np.asarray(self.replayBuffer.sample_positions(self.batch_size), dtype=np.int32)))
            _lib.check(_lib.lib().d4pg_learner_profile_step(L.handle, C.c_void_p(L.stream.cuda_stream), cap, ms, names,
                                                            stride, C.byref(n)), "d4pg_learner_profile_step")
        L.fresh_host_step = False
        if self.prioritized_replay:
            self.beta_schedule.t += 1
        for opt in (self.optimizer_global_actor, self.optimizer_global_critic):
            opt.step_count += 1
        raw = names.raw
        return [(raw[i * stride:(i + 1) * stride].split(b"\0")[0].decode(), float(ms[i])) for i in range(n.value)]

    def kernels_per_step(self):
        return int(_lib.lib().d4pg_learner_kernels_per_step(self._learner.handle)) if self._learner else 0
