"""CPU-only checks of adaptive parameter-space noise: AdaptiveParamNoiseSpec and DDPG(param_noise=) validation before any
device work, the ctypes prototypes and the C-side argument checks of d4pg_actor_perturb / d4pg_param_noise_adapt, and
the oracle's vectorised Philox against the scalar restatement."""
import ctypes as C
import math
import random

import numpy as np
import pytest
import torch

from tests import param_noise_oracle as PO
from tests.helpers import philox_uniform53

INFO = {"type": "categorical", "v_min": -10.0, "v_max": 0.0, "n_atoms": 51}


def _ddpg(**kw):
    import d4pg_b200 as d4pg
    return d4pg.DDPG(17, 6, memory_size=64, batch_size=8, critic_dist_info=INFO, **kw)


def test_spec_defaults_and_validation():
    import d4pg_b200 as d4pg
    from d4pg_b200 import AdaptiveParamNoiseSpec
    assert AdaptiveParamNoiseSpec is d4pg.random_process.AdaptiveParamNoiseSpec
    sp = AdaptiveParamNoiseSpec()
    assert (sp.initial_stddev, sp.desired_action_stddev, sp.adoption_coefficient) == (0.1, 0.1, 1.01)
    assert sp.check() == (0.1, 0.1, 1.01)
    assert AdaptiveParamNoiseSpec(initial_stddev=0.0).check()[0] == 0.0
    bad = [dict(initial_stddev=-1e-3), dict(initial_stddev=math.inf), dict(initial_stddev=math.nan),
           dict(desired_action_stddev=0.0), dict(desired_action_stddev=-0.1), dict(desired_action_stddev=math.inf),
           dict(adoption_coefficient=1.0), dict(adoption_coefficient=0.5), dict(adoption_coefficient=math.inf),
           dict(adoption_coefficient=math.nan), dict(initial_stddev="x"), dict(desired_action_stddev=None)]
    for kw in bad:
        with pytest.raises(ValueError):
            AdaptiveParamNoiseSpec(**kw)
    sp.adoption_coefficient = 1.0                   # read and checked again at every use
    with pytest.raises(ValueError, match="adoption_coefficient"):
        sp.check()
    assert "desired_action_stddev=0.1" in repr(AdaptiveParamNoiseSpec())


def test_ddpg_param_noise_validation_before_device_work():
    import d4pg_b200 as d4pg
    for bad in (0.1, True, "adaptive", {"initial_stddev": 0.1}, d4pg.random_process.GaussianNoise(6, 10)):
        with pytest.raises(ValueError, match="param_noise"):
            _ddpg(param_noise=bad)
    dd = _ddpg()
    assert dd.param_noise is None and dd.perturbed_actor is None and dd.param_noise_state is None
    with pytest.raises(d4pg.D4PGError, match="param_noise"):
        dd.perturb_actor()
    with pytest.raises(d4pg.D4PGError, match="param_noise"):
        dd.adapt_param_noise(np.zeros((4, 17), np.float32))

    spec = d4pg.AdaptiveParamNoiseSpec()
    dd = _ddpg(param_noise=spec)
    assert dd.param_noise is spec
    # an attribute gone bad is a ValueError on every path, before any device work (on a GPU-less host the device work
    # would raise D4PGError)
    spec.desired_action_stddev = 0.0
    for call in (dd.perturb_actor, lambda: dd.adapt_param_noise(np.zeros((4, 17), np.float32)),
                 lambda: dd.act(np.zeros((4, 17), np.float32))):
        with pytest.raises(ValueError, match="desired_action_stddev"):
            call()
    spec.desired_action_stddev = 0.1
    dd.param_noise = "other"
    with pytest.raises(ValueError, match="param_noise"):
        dd.perturb_actor()
    dd.param_noise = spec
    with pytest.raises(ValueError, match="expected states"):
        dd.adapt_param_noise(np.zeros((4, 16), np.float32))
    with pytest.raises(ValueError, match="E = 0"):
        dd.adapt_param_noise(np.zeros((0, 17), np.float32))
    with pytest.raises(ValueError):
        dd.param_noise_state = torch.zeros(2, dtype=torch.float64)
    dd.param_noise_state = None
    assert dd.param_noise_state is None
    with pytest.raises(AttributeError):
        dd.perturbed_actor = dd.actor


def test_noise_none_without_param_noise_still_raises():
    import d4pg_b200 as d4pg
    dd = _ddpg()
    dd.noise = None
    with pytest.raises(d4pg.D4PGError, match="NoneType"):
        dd.act(np.zeros((4, 17), np.float32))


def test_param_noise_draws_nothing_at_construction():
    """A DDPG with param_noise gets the weights of one without it and leaves every RNG where that one leaves it."""
    import d4pg_b200 as d4pg
    out = []
    for pn in (None, d4pg.AdaptiveParamNoiseSpec()):
        torch.manual_seed(3); np.random.seed(3); random.seed(3)
        dd = _ddpg(param_noise=pn)
        out.append(([t.clone() for t in dd.actor.state_dict().values()], torch.rand(4), np.random.rand(4), random.random()))
    (wa, ta, na, ra), (wb, tb, nb, rb) = out
    assert all(torch.equal(x, y) for x, y in zip(wa, wb))
    assert torch.equal(ta, tb) and np.array_equal(na, nb) and ra == rb


def test_unfilled_actor_draws_nothing():
    import d4pg_b200 as d4pg
    torch.manual_seed(5)
    st = torch.get_rng_state()
    net = d4pg.actor.unfilled(17, 6, device="cpu")
    assert torch.equal(torch.get_rng_state(), st)
    assert net.flat_params().numel() == d4pg.actor(17, 6, device="cpu").flat_params().numel()
    assert [tuple(p.shape) for p in net.parameters()] == [(256, 17), (256,), (256, 256), (256,), (256, 256), (256,),
                                                          (6, 256), (6,)]
    assert net.precision == 0 and not net.differentiable and net.obs_normalizer is None


def test_prototypes_and_c_validation():
    from d4pg_b200 import _lib
    L = _lib.lib()
    P = C.c_void_p
    assert L.d4pg_actor_perturb.restype is C.c_int32
    assert L.d4pg_actor_perturb.argtypes == [P, C.c_int32, C.c_int32, P, C.c_uint64, C.c_uint64, P, P]
    assert L.d4pg_param_noise_adapt.restype is C.c_int32
    assert L.d4pg_param_noise_adapt.argtypes == [P, P, C.c_int64, C.c_double, C.c_double, P, P]
    assert L.d4pg_version() >= 900

    def err():
        return L.d4pg_last_error().decode()
    # argument checks run before any device work: aligned dummy addresses are never dereferenced
    prm, st, out, a, ap = P(0x10000), P(0x20000), P(0x30000), P(0x40000), P(0x50000)

    def perturb(p=prm, S=17, A=6, s=st, o=out):
        return L.d4pg_actor_perturb(p, S, A, s, 0, PO.PERTURB_COUNTER_BASE, o, None)
    assert perturb(p=None) == _lib.EINVAL and "null" in err()
    assert perturb(s=None) == _lib.EINVAL and perturb(o=None) == _lib.EINVAL
    assert perturb(p=P(0x10004)) == _lib.EINVAL and "aligned" in err()
    assert perturb(o=P(0x30008)) == _lib.EINVAL
    assert perturb(s=P(0x20004)) == _lib.EINVAL
    assert perturb(S=0) == _lib.EINVAL and perturb(A=0) == _lib.EINVAL and perturb(S=-3) == _lib.EINVAL
    # 256 * obs_dim + 131584 + 257 * act_dim + 256 logical parameters; the draw lane 2i is 32-bit
    assert perturb(S=(1 << 23)) == _lib.EINVAL and "2^32" in err()

    def adapt(x=a, y=ap, n=24, desired=0.1, coef=1.01, s=st):
        return L.d4pg_param_noise_adapt(x, y, n, desired, coef, s, None)
    assert adapt(x=None) == _lib.EINVAL and adapt(y=None) == _lib.EINVAL and adapt(s=None) == _lib.EINVAL
    assert adapt(x=P(0x40002)) == _lib.EINVAL and adapt(s=P(0x20004)) == _lib.EINVAL
    assert adapt(n=0) == _lib.EINVAL and "n >= 1" in err()
    assert adapt(n=-5) == _lib.EINVAL
    for d in (0.0, -0.1, math.inf, math.nan):
        assert adapt(desired=d) == _lib.EINVAL and "desired_stddev" in err()
    for c in (1.0, 0.9, math.inf, math.nan):
        assert adapt(coef=c) == _lib.EINVAL and "coefficient" in err()


def test_vectorised_philox_matches_the_scalar_restatement():
    rng = np.random.RandomState(0)
    for seed, ctr in ((0, PO.PERTURB_COUNTER_BASE), (0x5EED, PO.PERTURB_COUNTER_BASE + 7),
                      ((1 << 64) - 1, (1 << 63) + 3), (12345, 17)):
        lanes = np.concatenate([np.arange(8), rng.randint(0, 1 << 32, 56, dtype=np.uint64), [(1 << 32) - 1]])
        got = PO.uniform53(seed, ctr, lanes)
        want = np.array([philox_uniform53(seed, ctr, int(l)) for l in lanes])
        assert np.array_equal(got, want)
        assert ((got >= 0.0) & (got < 1.0)).all()


def test_oracle_rule_and_distance():
    assert PO.adapt(0.2, 0.3, 0.1, 1.01) == 0.2 / 1.01
    assert PO.adapt(0.2, 0.05, 0.1, 1.01) == 0.2 * 1.01
    assert PO.adapt(0.2, 0.1, 0.1, 1.01) == 0.2 * 1.01              # a tie grows sigma, as in baselines
    a = np.array([[0.5, -0.25], [1.0, 0.0]], np.float32)
    assert PO.distance(a, a) == 0.0
    assert PO.distance(a, a + np.float32(0.5)) == 0.5
    p = np.linspace(-1, 1, 50).astype(np.float32)
    assert np.array_equal(PO.perturb(p, 0.0, 1, 0), p)
    q0, q1 = PO.perturb(p, 0.1, 1, 0), PO.perturb(p, 0.1, 1, 1)
    assert not np.array_equal(q0, q1) and 0.03 < float(np.std(q0 - p)) < 0.3
