"""Import the UNMODIFIED reference behind the compat shim: from a reference checkout (D4PG_REFERENCE_PATH) where it
exists, else from `oracle/_ref/` -- the same modules byte-compiled by oracle/build_ref.py (bench.py's CPU arm and
tests/golden/make_golden.py; no test needs them).

TEST INFRASTRUCTURE ONLY (see oracle/__init__.py).

Shim items (SURVEY.md section 8c, each verified by running the reference here):
  1. SharedAdam `state['step']` must be a 0-d tensor for torch>=2 (shared_adam.py:11).
  2. `nn.Module.zero_grad` forced to `set_to_none=False`, otherwise the gradient
     aliasing of ddpg.py:104-108 silently freezes the global model's grads.
  3. `np.float = float` for replay_memory.py:75-79 on numpy>=1.24.
  4. `ddpg.bp` (pdb) replaced by a raising stub so ddpg.py:182-184 surfaces errors.
"""
import os
import sys

REFERENCE_PATH = os.environ.get("D4PG_REFERENCE_PATH", "/root/reference")
COMPILED_PATH = os.path.join(os.path.dirname(os.path.abspath(__file__)), "_ref")


class ReferenceBreakpoint(RuntimeError):
    """Raised where the reference would have dropped into pdb."""


def source_available():
    return os.path.isfile(os.path.join(REFERENCE_PATH, "ddpg.py"))


def compiled_available():
    return os.path.isfile(os.path.join(COMPILED_PATH, "ddpg.pyc"))


def available():
    return source_available() or compiled_available()


def import_path():
    return REFERENCE_PATH if source_available() else COMPILED_PATH


_cached = None


def load():
    """Returns a namespace with the reference modules (ddpg, models, ...)."""
    global _cached
    if _cached is not None:
        return _cached
    if not available():
        raise RuntimeError("reference not present at %s nor compiled under %s" % (REFERENCE_PATH, COMPILED_PATH))
    ref_path = import_path()
    import types
    import numpy as np
    import torch
    import torch.nn as nn

    sys.dont_write_bytecode = True          # the mount is read-only
    if not hasattr(np, "float"):
        np.float = float                     # shim 3
    if not getattr(nn.Module.zero_grad, "_d4pg_shim", False):
        _orig = nn.Module.zero_grad

        def zero_grad(self, set_to_none=False):   # shim 2
            return _orig(self, set_to_none=False)
        zero_grad._d4pg_shim = True
        nn.Module.zero_grad = zero_grad

    # The reference's module names (utils, models, ...) are generic: import them
    # with the reference first on sys.path, then restore sys.path and move the
    # modules out of sys.modules' generic names so they cannot shadow anything.
    names = ["utils", "models", "random_process", "replay_memory",
             "prioritized_replay_memory", "shared_adam", "ddpg"]
    saved = {n: sys.modules.pop(n) for n in names if n in sys.modules}
    sys.path.insert(0, ref_path)
    try:
        mods = {}
        import importlib
        for n in names:
            mods[n] = importlib.import_module(n)
    finally:
        sys.path.remove(ref_path)
        for n in names:
            m = sys.modules.pop(n, None)
            if m is not None:
                sys.modules["_d4pg_reference." + n] = m
        sys.modules.update(saved)

    def _bp():                               # shim 4
        raise ReferenceBreakpoint("reference called pdb.set_trace()")
    mods["ddpg"].bp = _bp

    def make_shared_adam(params, lr=1e-3, **kw):   # shim 1
        opt = mods["shared_adam"].SharedAdam(params, lr=lr, **kw)
        for group in opt.param_groups:
            for p in group["params"]:
                opt.state[p]["step"] = torch.zeros((), dtype=torch.float32)
        return opt

    ns = types.SimpleNamespace(**mods)
    ns.make_shared_adam = make_shared_adam
    ns.ReferenceBreakpoint = ReferenceBreakpoint
    _cached = ns
    return ns


def make_learner_pair(obs_dim, act_dim, dist_info, batch_size, memory_size,
                      prioritized_replay=True, gamma=0.99, tau=0.001, n_steps=1,
                      lr=1e-3, seed=0):
    """Wire global + local DDPG and the two SharedAdam objects as main.py:382-392
    / main.py:187-195,248-249 do (single worker)."""
    import random
    import numpy as np
    import torch
    ref = load()
    torch.manual_seed(seed)
    np.random.seed(seed)
    random.seed(seed)
    kw = dict(memory_size=memory_size, batch_size=batch_size, tau=tau, gamma=gamma,
              critic_dist_info=dist_info, prioritized_replay=prioritized_replay,
              n_steps=n_steps)
    g = ref.ddpg.DDPG(obs_dim, act_dim, **kw)
    opt_a = ref.make_shared_adam(g.actor.parameters(), lr=lr)
    opt_c = ref.make_shared_adam(g.critic.parameters(), lr=lr)
    l = ref.ddpg.DDPG(obs_dim, act_dim, **kw)
    l.assign_global_optimizer(opt_a, opt_c)
    l.sync_local_global(g)
    l.hard_update()
    return g, l, opt_a, opt_c
