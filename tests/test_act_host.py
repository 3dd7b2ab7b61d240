"""CPU-only checks of DDPG.act: argument validation before any device work, the ctypes prototypes and the C-side
validation of d4pg_act, and the oracle's noise formulas against the unmodified reference's random_process.py."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import ref_shim
from tests import act_oracle as AO

INFO = {"type": "categorical", "v_min": -10.0, "v_max": 0.0, "n_atoms": 51}


def _ddpg(obs_dim=17, act_dim=6):
    import d4pg_b200 as d4pg
    return d4pg.DDPG(obs_dim, act_dim, memory_size=64, batch_size=8, critic_dist_info=INFO)


def test_act_rejects_bad_arguments_before_device_work():
    import d4pg_b200 as d4pg
    dd = _ddpg()
    with pytest.raises(ValueError, match="expected states"):
        dd.act(np.zeros((4, 16), np.float32))
    with pytest.raises(ValueError, match="expected states"):
        dd.act(np.zeros((2, 3, 17), np.float32))
    with pytest.raises(ValueError, match="expected states"):
        dd.act(torch.zeros(18))
    with pytest.raises(ValueError, match="E = 0"):
        dd.act(np.zeros((0, 17), np.float32))
    big = np.broadcast_to(np.zeros(17, np.float32), ((1 << 30) // 6 + 1, 17))     # no memory behind the rows
    with pytest.raises(ValueError, match="2\\^31"):
        dd.act(big, explore=False)
    dd.noise = d4pg.random_process.OrnsteinUhlenbeckProcess(dimension=6, num_steps=100)
    for bad in (np.zeros(3, bool), np.zeros((4, 1), bool), [True] * 5):
        with pytest.raises(ValueError, match="reset"):
            dd.act(np.zeros((4, 17), np.float32), reset=bad)

    class OtherNoise(object):
        epsilon = 0.3

        def sample(self):
            return np.zeros(6)
    dd.noise = OtherNoise()
    with pytest.raises(d4pg.D4PGError, match="OtherNoise"):
        dd.act(np.zeros((4, 17), np.float32))
    with pytest.raises(ValueError):
        dd.exploration_state = torch.zeros(4, 6, dtype=torch.float64)
    dd.exploration_state = None
    assert dd.exploration_state is None


def test_act_without_gpu_fails_loudly():
    import d4pg_b200 as d4pg
    if torch.cuda.is_available():
        pytest.skip("GPU present")
    with pytest.raises(d4pg.D4PGError):
        _ddpg().act(np.zeros((4, 17), np.float32))


def test_act_prototypes_and_c_validation():
    from d4pg_b200 import _lib
    L = _lib.lib()
    P = C.c_void_p
    assert L.d4pg_act.restype is C.c_int32
    assert L.d4pg_act.argtypes == [P, C.c_int32, C.c_int32, P, C.c_int64, C.c_int32, P, C.c_double, C.c_int32, P,
                                   C.c_uint64, C.c_uint64, P, P, P, P, P]
    assert L.d4pg_act_workspace_floats.restype is C.c_int64
    assert L.d4pg_act_workspace_floats.argtypes == [C.c_int32, C.c_int32]
    assert L.d4pg_copy_rows_f32.argtypes == [P, C.c_int64, P, C.c_int64, C.c_int64, C.c_int64, P]
    # three published planes of 256 x 32 floats per 32-row cluster
    assert L.d4pg_act_workspace_floats(1, 17) == 3 * 256 * 32
    assert L.d4pg_act_workspace_floats(33, 376) == 2 * 3 * 256 * 32
    assert L.d4pg_act_workspace_floats(0, 17) == -1 and L.d4pg_act_workspace_floats(4, 0) == -1

    # argument checks run before any device work: 16-B aligned dummy addresses are never dereferenced
    prm, s, out, ws, st = P(0x10000), P(0x20000), P(0x30000), P(0x40000), P(0x50000)
    gp = (C.c_double * 5)(0.3, 0.0, 1.0, 0.0, 0.0)

    def act(obs=17, A=6, s_=s, lds=20, E=4, aff=None, clip=5.0, noise=1, params=gp, ou=None):
        return L.d4pg_act(prm, obs, A, s_, lds, E, aff, clip, noise, params, 0, 1 << 63, ou, None, out, ws, None)

    def err():
        return L.d4pg_last_error().decode()
    assert act(s_=None) == _lib.EINVAL
    assert act(lds=17) == _lib.EINVAL and "row pitch" in err()             # not a multiple of 4
    assert act(lds=16) == _lib.EINVAL                                       # narrower than a row
    assert act(s_=P(0x20004)) == _lib.EINVAL                                # unaligned base
    assert act(E=0) == _lib.EINVAL and "E = 0" in err()
    assert act(E=(1 << 30) // 6 + 1) == _lib.EINVAL
    assert act(A=0) == _lib.EINVAL and act(A=257) == _lib.EINVAL
    assert act(noise=3) == _lib.EINVAL
    assert act(params=None) == _lib.EINVAL
    assert act(noise=2, params=(C.c_double * 5)(1.0, 0.25, 0.0, 0.05, 0.01)) == _lib.EINVAL      # no OU state
    assert act(params=(C.c_double * 5)(float("nan"), 0.0, 1.0, 0, 0)) == _lib.EINVAL
    assert act(aff=st, clip=0.0) == _lib.EINVAL
    # fc1 of obs_dim 577 does not fit one chain slot: refused, no fallback
    assert act(obs=577, lds=580) == _lib.ENOTSUP and "576" in err()
    assert L.d4pg_copy_rows_f32(out, 4, s, 20, 0, 17, None) == _lib.EINVAL


def _reference_random_process():
    if not ref_shim.available():
        pytest.skip("reference not present")
    return ref_shim.load().random_process


def test_oracle_noise_equals_reference_sample(monkeypatch):
    """With np.random.normal patched to hand out given standard normals z (loc + scale * z, what numpy's normal
    computes from its standard normal), the reference's sample() is the oracle's formula bit for bit, in fp64."""
    rp = _reference_random_process()
    A = 6
    zs = [AO.standard_normal(1234, k, A) for k in range(6)]
    it = iter(zs)

    def normal(loc=0.0, scale=1.0, size=None):
        z = next(it)
        assert size == A
        return loc + scale * z
    monkeypatch.setattr(np.random, "normal", normal)

    g = rp.GaussianNoise(dimension=A, num_epochs=100, mu=0.125, var=0.7)
    for k in range(3):
        g.iter = 10 * k
        g.reset()                                     # epsilon decays between calls
        want = AO.gaussian_noise(zs[k], g.epsilon, g.mu, g.var)
        assert np.array_equal(g.sample(), want)

    ou = rp.OrnsteinUhlenbeckProcess(dimension=A, num_steps=50, theta=0.25, mu=0.1, sigma=0.5, dt=0.01)
    x = np.zeros(A)
    for k in range(3, 6):
        reset = k == 5
        if reset:
            ou.reset()
        got = ou.sample()
        x = AO.ou_step(x, zs[k], ou.theta, ou.mu, ou.sigma, ou.dt, reset=np.full(A, reset))
        assert np.array_equal(ou.x, x)
        assert np.array_equal(got, ou.epsilon * x)
