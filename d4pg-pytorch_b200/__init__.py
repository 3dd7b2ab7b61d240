"""d4pg-pytorch_b200 -- H100-native (sm_90a) D4PG learner hot path behind the reference's
Python API (ajgupta93/d4pg-pytorch: ddpg.py, models.py, prioritized_replay_memory.py,
replay_memory.py, shared_adam.py).

    import d4pg_b200 as d4pg            # alias module at the repo root
    ddpg = d4pg.DDPG(obs_dim, act_dim, critic_dist_info={...})

or, to run the reference's own `main.py` unmodified against this build:

    import d4pg_b200; d4pg_b200.install_reference_aliases()   # `from ddpg import DDPG` now binds here

The directory name contains a hyphen (it is the name the build contract prescribes), so it is
imported through `importlib`; `d4pg_b200.py` at the repo root does that.
"""
import sys as _sys

from . import _lib
from ._lib import D4PGError, LIB_PATH
from . import utils, random_process, models, obs_norm, prioritized_replay_memory, replay_memory, shared_adam, ddpg, dist
from .ddpg import DDPG
from .models import actor, critic, fanin_init
from .obs_norm import ObsNormalizer
from .random_process import AdaptiveParamNoiseSpec
from .prioritized_replay_memory import (LinearSchedule, SegmentTree, SumSegmentTree, MinSegmentTree,
                                        ReplayBuffer, PrioritizedReplayBuffer)
from .replay_memory import Replay
from .shared_adam import SharedAdam
from .utils import to_tensor, to_numpy

# the north-star paraphrases the class names; keep aliases (SURVEY.md H12)
Actor, Critic = actor, critic
ReplayMemory = Replay
PrioritizedReplayMemory = PrioritizedReplayBuffer

__version__ = "0.5.0"


def install_reference_aliases():
    """Register this package's modules under the reference's top-level module names so that
    `from ddpg import DDPG`, `from shared_adam import SharedAdam`, ... (main.py:6-9) bind here."""
    for name, mod in (("ddpg", ddpg), ("models", models), ("shared_adam", shared_adam),
                      ("prioritized_replay_memory", prioritized_replay_memory),
                      ("replay_memory", replay_memory), ("utils", utils), ("random_process", random_process)):
        _sys.modules[name] = mod


def build(force=False, verbose=False):
    from . import build as _b
    return _b.build(force=force, verbose=verbose)
