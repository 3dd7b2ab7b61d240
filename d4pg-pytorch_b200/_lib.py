"""ctypes binding of libd4pg_sm90.so (the C ABI declared in include/d4pg_b200.h).

There is NO CPU fallback: if the shared library is missing or no sm_90 device is
present, every compute entry point raises.  (Host-only bookkeeping -- layouts,
state_dict plumbing -- works without a GPU so the CPU test-suite can exercise it.)
"""
import ctypes as C
import os

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libd4pg_sm90.so")

OK, EINVAL, ECUDA, ENOTSUP, ENCCL, ESTATE = 0, -1, -2, -3, -4, -5
PROJ_TARGET_IS_PROBS, PROJ_Q_IS_PROBS = 1, 2
HIDDEN = 256
MAX_ATOMS = 128
MAX_COMPONENTS = 32
STEPS_MAX_N = 64          # D4PG_STEPS_MAX_N: the longest n-step window of d4pg_replay_add_steps
GOAL_MAX_STEPS = 65536    # D4PG_GOAL_MAX_STEPS: the longest episode window of d4pg_replay_add_goal_steps

c_float_p = C.POINTER(C.c_float)
c_double_p = C.POINTER(C.c_double)
c_int32_p = C.POINTER(C.c_int32)
c_uint8_p = C.POINTER(C.c_uint8)


class D4PGError(RuntimeError):
    pass


class NetLayout(C.Structure):
    _fields_ = [("offsets", C.c_int64 * 8), ("sizes", C.c_int64 * 8), ("pitch", C.c_int64 * 4), ("total", C.c_int64)]


class LearnerConfig(C.Structure):
    _fields_ = [
        ("obs_dim", C.c_int32), ("act_dim", C.c_int32), ("n_atoms", C.c_int32), ("batch", C.c_int32),
        ("v_min", C.c_double), ("v_max", C.c_double), ("gamma", C.c_double),
        ("n_steps", C.c_int32), ("proj_mode", C.c_int32),
        ("tau", C.c_double),
        ("lr_actor", C.c_double), ("lr_critic", C.c_double), ("beta1", C.c_double), ("beta2", C.c_double),
        ("adam_eps", C.c_double),
        ("prioritized", C.c_int32),
        ("per_beta0", C.c_double), ("per_beta_final", C.c_double), ("per_beta_iters", C.c_int64),
        ("prio_eps", C.c_double),
        ("precision", C.c_int32), ("sample_mode", C.c_int32),
        ("philox_seed", C.c_uint64),
        ("world_size", C.c_int32), ("use_graph", C.c_int32),
        ("loss_flags", C.c_int32), ("chain", C.c_int32), ("prefetch", C.c_int32),
        ("dist_type", C.c_int32), ("n_components", C.c_int32),
        ("qr_kappa", C.c_double),
        ("max_grad_norm_actor", C.c_double), ("max_grad_norm_critic", C.c_double),
        ("weight_decay_actor", C.c_double), ("weight_decay_critic", C.c_double),
        ("obs_norm", C.c_int32),
        ("nstep_tails", C.c_int32),
    ]


class LearnerBuffers(C.Structure):
    _fields_ = [
        ("actor", C.c_void_p), ("actor_target", C.c_void_p), ("critic", C.c_void_p), ("critic_target", C.c_void_p),
        ("grad_actor", C.c_void_p), ("grad_critic", C.c_void_p),
        ("adam_m_actor", C.c_void_p), ("adam_v_actor", C.c_void_p),
        ("adam_m_critic", C.c_void_p), ("adam_v_critic", C.c_void_p),
        ("uniforms", C.c_void_p), ("positions", C.c_void_p), ("idx", C.c_void_p), ("weights", C.c_void_p),
        ("prio", C.c_void_p), ("td", C.c_void_p), ("losses", C.c_void_p), ("workspace", C.c_void_p),
    ]


_P = C.c_void_p
_PROTOS = {
    "d4pg_last_error": (C.c_char_p, []),
    "d4pg_version": (C.c_int32, []),
    "d4pg_struct_size": (C.c_int32, [C.c_int32]),
    "d4pg_device_sm": (C.c_int32, []),
    "d4pg_actor_layout": (C.c_int32, [C.c_int32, C.c_int32, C.POINTER(NetLayout)]),
    "d4pg_critic_layout": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.POINTER(NetLayout)]),
    "d4pg_proj_loss": (C.c_int32, [_P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double,
                                   C.c_int32, C.c_int32, C.c_double, C.c_float,
                                   _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P]),
    "d4pg_mog_loss": (C.c_int32, [_P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_float,
                                  _P, _P, _P, _P, _P, _P, _P]),
    "d4pg_mog_quadrature": (C.c_int32, [_P, _P]),
    "d4pg_qr_loss": (C.c_int32, [_P, _P, _P, _P, _P, C.c_int32, C.c_int32, C.c_double, C.c_double, C.c_double, C.c_float,
                                 C.c_int32, _P, _P, _P, _P, _P, _P, _P]),
    "d4pg_replay_capacity": (C.c_int32, [C.c_int64, C.POINTER(C.c_int64)]),
    "d4pg_replay_create": (C.c_int32, [C.c_int64, C.c_int32, C.c_int32, C.c_double, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                       _P, C.POINTER(_P)]),
    "d4pg_replay_destroy": (C.c_int32, [_P]),
    "d4pg_replay_len": (C.c_int64, [_P]),
    "d4pg_replay_next_idx": (C.c_int64, [_P]),
    "d4pg_replay_add": (C.c_int32, [_P, C.c_int64, _P, _P, _P, _P, _P, C.c_int32, _P]),
    "d4pg_replay_staging_bytes": (C.c_int64, [_P, C.c_int64]),
    "d4pg_replay_set_staging": (C.c_int32, [_P, _P, _P, C.c_int64]),
    "d4pg_replay_add_host": (C.c_int32, [_P, C.c_int64, _P, _P, _P, _P, _P, C.c_int32, _P]),
    "d4pg_replay_sample": (C.c_int32, [_P, C.c_int32, _P, C.c_uint64, C.c_uint64, C.c_double, _P, _P, _P, _P, _P, _P, _P, _P]),
    "d4pg_replay_gather": (C.c_int32, [_P, C.c_int32, _P, _P, _P, _P, _P, _P, _P]),
    "d4pg_replay_update_priorities": (C.c_int32, [_P, C.c_int32, _P, _P, _P]),
    "d4pg_replay_reduce": (C.c_int32, [_P, C.c_int64, C.c_int64, _P, _P]),
    "d4pg_replay_find_prefixsum": (C.c_int32, [_P, C.c_int32, _P, _P, _P]),
    "d4pg_replay_set_leaves": (C.c_int32, [_P, C.c_int32, _P, _P, _P, _P]),
    "d4pg_nstep_returns": (C.c_int32, [_P, C.c_int64, C.c_int32, C.c_double, _P, _P]),
    "d4pg_replay_add_nstep": (C.c_int32, [_P, C.c_int64, _P, _P, _P, _P, _P, C.c_int32, C.c_double, _P, C.c_int32, _P]),
    "d4pg_replay_steps_window_bytes": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32, C.c_int32]),
    "d4pg_replay_add_steps": (C.c_int32, [_P, C.c_int64, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_double, _P, C.c_int64,
                                          C.c_int32, _P]),
    "d4pg_replay_set_horizons": (C.c_int32, [_P, _P, _P]),
    "d4pg_replay_steps_window_bytes_ex": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "d4pg_replay_add_steps_ex": (C.c_int32, [_P, C.c_int64, _P, _P, _P, _P, _P, _P, C.c_int32, C.c_double, _P, C.c_int64,
                                             C.c_int32, C.c_int32, _P]),
    "d4pg_replay_goal_window_bytes": (C.c_int64, [C.c_int64, C.c_int32, C.c_int32, C.c_int32, C.c_int32]),
    "d4pg_replay_add_goal_steps": (C.c_int32, [_P, C.c_int64, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P,
                                               C.c_int32, _P, _P, C.c_int64, C.c_int64, C.c_double, C.c_int32, C.c_int32,
                                               C.c_int32, _P]),
    "d4pg_her_relabel": (C.c_int32, [C.c_int32, C.c_int32, C.c_int32, C.c_int32, _P, _P, _P, _P, _P, _P, _P, _P, _P, _P,
                                     C.c_double, C.c_int32, _P, _P, _P, _P, _P, _P]),
    "d4pg_replay_set_len": (C.c_int32, [_P, C.c_int64, C.c_int64, C.c_int32, _P]),
    "d4pg_replay_set_obs_norm": (C.c_int32, [_P, _P, _P, C.c_double, C.c_double, _P]),
    "d4pg_replay_obs_norm_refresh": (C.c_int32, [_P, _P]),
    "d4pg_obs_norm_update": (C.c_int32, [_P, _P, C.c_int32, _P, C.c_int64, C.c_int64, C.c_double, _P]),
    "d4pg_obs_normalize": (C.c_int32, [_P, C.c_int32, C.c_double, _P, C.c_int64, _P, _P, _P]),
    "d4pg_actor_forward": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, C.c_int32, _P]),
    "d4pg_critic_forward": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, _P, _P, C.c_int32, _P]),
    "d4pg_act_workspace_floats": (C.c_int64, [C.c_int32, C.c_int32]),
    "d4pg_act": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int64, C.c_int32, _P, C.c_double, C.c_int32, _P,
                             C.c_uint64, C.c_uint64, _P, _P, _P, _P, _P]),
    "d4pg_copy_rows_f32": (C.c_int32, [_P, C.c_int64, _P, C.c_int64, C.c_int64, C.c_int64, _P]),
    "d4pg_actor_perturb": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_uint64, C.c_uint64, _P, _P]),
    "d4pg_param_noise_adapt": (C.c_int32, [_P, _P, C.c_int64, C.c_double, C.c_double, _P, _P]),
    "d4pg_actor_backward": (C.c_int32, [_P, C.c_int32, C.c_int32, _P, C.c_int32, _P, _P, _P, _P, _P, _P, C.c_int32, _P]),
    "d4pg_critic_backward": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, _P, _P, _P,
                                         _P, _P, _P, _P, C.c_int32, _P]),
    "d4pg_critic_forward_mog": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, _P, _P, _P, _P,
                                            C.c_int32, _P]),
    "d4pg_critic_backward_mog": (C.c_int32, [_P, C.c_int32, C.c_int32, C.c_int32, _P, _P, C.c_int32, _P, _P, _P, _P, _P,
                                             _P, _P, _P, _P, C.c_int32, _P]),
    "d4pg_adam_polyak": (C.c_int32, [_P, _P, _P, _P, _P, C.c_int64, C.c_double, C.c_double, C.c_double, C.c_double,
                                     C.c_int64, C.c_double, C.c_float, _P]),
    "d4pg_adam_polyak_ex": (C.c_int32, [_P, _P, _P, _P, _P, C.c_int64, C.c_double, C.c_double, C.c_double, C.c_double,
                                        C.c_int64, C.c_double, C.c_float, _P, C.c_double, C.c_double, _P, _P]),
    "d4pg_polyak": (C.c_int32, [_P, _P, C.c_int64, C.c_double, _P]),
    "d4pg_copy_f32": (C.c_int32, [_P, _P, C.c_int64, _P]),
    "d4pg_learner_workspace_floats": (C.c_int64, [C.POINTER(LearnerConfig)]),
    "d4pg_learner_create": (C.c_int32, [C.POINTER(LearnerConfig), C.POINTER(LearnerBuffers), _P, _P, C.POINTER(_P)]),
    "d4pg_learner_destroy": (C.c_int32, [_P]),
    "d4pg_learner_step": (C.c_int32, [_P, _P]),
    "d4pg_learner_run": (C.c_int32, [_P, C.c_int32, _P]),
    "d4pg_learner_step_host_mt": (C.c_int32, [_P, _P, _P, _P]),
    "d4pg_learner_step_host": (C.c_int32, [_P, _P, _P, _P, _P]),
    "d4pg_learner_read_losses": (C.c_int32, [_P, _P, _P]),
    "d4pg_learner_fetch_losses": (C.c_int32, [_P, C.c_int32, _P]),
    "d4pg_learner_tensor": (C.c_int32, [_P, C.c_char_p, C.POINTER(_P), C.POINTER(C.c_int64), C.POINTER(C.c_int32)]),
    "d4pg_learner_profile_step": (C.c_int32, [_P, _P, C.c_int32, _P, _P, C.c_int32, C.POINTER(C.c_int32)]),
    "d4pg_learner_steps_done": (C.c_int64, [_P]),
    "d4pg_learner_ingest_stream": (_P, [_P]),
    "d4pg_learner_weights_changed": (C.c_int32, [_P]),
    "d4pg_replay_order_after": (C.c_int32, [_P, _P, _P]),
    "d4pg_learner_kernels_per_step": (C.c_int32, [_P]),
    "d4pg_learner_set_counters": (C.c_int32, [_P, C.c_int64, C.c_int64, _P]),
    "d4pg_debug_tc_trace": (C.c_int32, [_P]),
    "d4pg_debug_trace_read": (C.c_int32, [_P, C.c_int32]),
    "d4pg_debug_watchdog": (C.c_int32, [_P]),
    "d4pg_comm_unique_id": (C.c_int32, [_P]),
    "d4pg_comm_create": (C.c_int32, [_P, C.c_int32, C.c_int32, C.POINTER(_P)]),
    "d4pg_comm_destroy": (C.c_int32, [_P]),
    "d4pg_comm_peer_alloc": (C.c_int32, [_P, C.c_int64, _P]),
    "d4pg_comm_peer_open": (C.c_int32, [_P, _P]),
    "d4pg_comm_peer_ready": (C.c_int32, [_P]),
    "d4pg_comm_peer_disable": (C.c_int32, [_P]),
    "d4pg_comm_allreduce_sum": (C.c_int32, [_P, _P, C.c_int64, _P]),
    "d4pg_comm_mc_supported": (C.c_int32, [_P]),
    "d4pg_comm_mc_create": (C.c_int32, [_P, C.POINTER(C.c_int32)]),
    "d4pg_comm_mc_import": (C.c_int32, [_P, C.c_int32]),
    "d4pg_comm_mc_add_device": (C.c_int32, [_P]),
    "d4pg_comm_mc_bind": (C.c_int32, [_P]),
    "d4pg_comm_mc_ready": (C.c_int32, [_P]),
    "d4pg_comm_mc_disable": (C.c_int32, [_P]),
    "d4pg_comm_mc_selftest": (C.c_int32, [_P, _P, _P, C.c_int64, _P]),
}
EXPORTED_SYMBOLS = sorted(_PROTOS)

_lib = None


def lib():
    """The loaded shared library (built on demand by `build.py` is NOT done here: a missing
    .so is an error the caller must see)."""
    global _lib
    if _lib is None:
        if not os.path.exists(LIB_PATH):
            raise D4PGError("CUDA extension missing: %s (run `python d4pg-pytorch_b200/build.py`); "
                            "there is no CPU fallback" % LIB_PATH)
        try:
            import torch  # noqa: F401  (makes libcudart / libnccl resolvable in-process)
        except Exception:
            pass
        L = C.CDLL(LIB_PATH, mode=C.RTLD_GLOBAL)
        for name, (res, args) in _PROTOS.items():
            fn = getattr(L, name)
            fn.restype = res
            fn.argtypes = args
        _lib = L
    return _lib


def check(rc, what=""):
    if rc != 0:
        msg = lib().d4pg_last_error()
        raise D4PGError("%s failed (code %d): %s" % (what or "libd4pg call", rc, (msg or b"").decode()))


def require_cuda():
    """Every compute path calls this first: fail loudly, never fall back."""
    import torch
    if not torch.cuda.is_available():
        raise D4PGError("no CUDA device: the D4PG hot path runs only on sm_90a (H100); there is no CPU fallback")
    lib()


def ptr(t):
    """Raw device/host pointer of a torch tensor (None -> NULL)."""
    if t is None:
        return None
    return C.c_void_p(t.data_ptr())


def raw_stream(device_index=None):
    """cudaStream_t of torch's current stream as an int.  torch.cuda.current_stream() builds a Stream object through
    several Python layers, twice per training step; the raw getter skips them."""
    import torch
    if device_index is None:
        device_index = torch.cuda.current_device()
    return torch._C._cuda_getCurrentRawStream(device_index)


def stream_ptr():
    return C.c_void_p(raw_stream())


def actor_layout(obs_dim, act_dim):
    out = NetLayout()
    check(lib().d4pg_actor_layout(obs_dim, act_dim, C.byref(out)), "d4pg_actor_layout")
    return list(out.offsets), list(out.sizes), int(out.total), list(out.pitch)


def mog_quadrature():
    """The library's 8-node Gauss-Hermite table (x, h) of the mixture critic's loss (host only, no GPU needed)."""
    x, h = (C.c_double * 8)(), (C.c_double * 8)()
    check(lib().d4pg_mog_quadrature(x, h), "d4pg_mog_quadrature")
    return list(x), list(h)


def critic_layout(obs_dim, act_dim, n_atoms):
    out = NetLayout()
    check(lib().d4pg_critic_layout(obs_dim, act_dim, n_atoms, C.byref(out)), "d4pg_critic_layout")
    return list(out.offsets), list(out.sizes), int(out.total), list(out.pitch)
