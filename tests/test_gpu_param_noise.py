"""Adaptive parameter-space noise on the H100: the perturbation against tests/param_noise_oracle.py (padding written as
zeros, the source untouched), its Philox stream, act() through the perturbed actor, the snapshot semantics, the
adaptation kernel and adapt_param_noise against fp64, isolation from the learner and the launch counts."""
import random

import numpy as np
import pytest
import torch

from tests import act_oracle as AO
from tests import param_noise_oracle as PO

pytestmark = pytest.mark.gpu

INFO = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}
NAMES = ["fc1.weight", "fc1.bias", "fc2.weight", "fc2.bias", "fc2_2.weight", "fc2_2.bias", "fc3.weight", "fc3.bias"]


def _spec(**kw):
    import d4pg_b200 as d4pg
    return d4pg.AdaptiveParamNoiseSpec(**kw)


def _ddpg(obs_dim, act_dim, seed=0, memory_size=4096, batch_size=64, **kw):
    import d4pg_b200 as d4pg
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    return d4pg.DDPG(obs_dim, act_dim, memory_size=memory_size, batch_size=batch_size, critic_dist_info=INFO, **kw)


def _fill(dd, n, rng):
    S, A = dd.obs_dim, dd.act_dim
    loc, scl = rng.uniform(-2, 2, S), rng.uniform(0.5, 3, S)
    st = (rng.randn(n, S) * scl + loc).astype(np.float32)
    s2 = (rng.randn(n, S) * scl + loc).astype(np.float32)
    a = rng.uniform(-1, 1, (n, A)).astype(np.float32)
    r = (-3 * rng.rand(n)).astype(np.float32).astype(np.float64)
    dd.replayBuffer.add_batch(st, a, r, s2, rng.rand(n) < 0.05)
    return loc, scl


def _states(rng, E, S, loc=0.0, scl=1.0):
    return (rng.randn(E, S) * 4 * scl + loc).astype(np.float32)


def _logical(net):
    """torch.cat([p.flatten() for p in net.parameters()]) as numpy."""
    return torch.cat([p.detach().flatten() for p in net.parameters()]).cpu().numpy()


def _unflatten(net, vec):
    out, k = {}, 0
    for name, p in zip(NAMES, net.parameters()):
        out[name] = vec[k:k + p.numel()].reshape(tuple(p.shape))
        k += p.numel()
    return out


def _pad_mask(net):
    """True at every float of the flat buffer that is not a parameter element."""
    pad = np.ones(net._total, bool)
    for i, (fin, fout) in enumerate(net._dims):
        ow, ob, pitch = net._offsets[2 * i], net._offsets[2 * i + 1], net._pitch[i]
        pad[ow:ow + pitch * fout].reshape(fout, pitch)[:, :fin] = False
        pad[ob:ob + fout] = False
    return pad


def _check_perturbation(dd, src, sigma, seed, j):
    pa = dd.perturbed_actor
    want = PO.perturb(src, sigma, seed, j)
    got = _logical(pa)
    AO.check_actions(got, want)                           # 1 fp32 ulp, >= 99 % bit-equal (device log / cos vs libm)
    bits = pa.flat_params().view(torch.int32).cpu().numpy()
    assert (bits[_pad_mask(pa)] == 0).all(), "padding is not +0.0"


@pytest.mark.parametrize("dims", [(3, 1), (17, 6), (376, 17), (1000, 4)], ids=["3x1", "17x6", "376x17", "1000x4"])
def test_perturbation_matches_oracle(dims):
    S, A = dims
    seed = 0x1234 + S
    dd = _ddpg(S, A, philox_seed=seed, param_noise=_spec(initial_stddev=0.2))
    assert dd.perturbed_actor is None and dd.param_noise_state is None
    before = dd.actor.flat_params().clone()
    src = _logical(dd.actor)
    pa = dd.perturb_actor()
    assert pa is dd.perturbed_actor and type(pa) is type(dd.actor)
    assert (pa.input_size, pa.output_size, pa.precision) == (S, A, 0)
    assert pa.flat_params().device == dd.actor.flat_params().device
    assert pa.flat_params().data_ptr() != dd.actor.flat_params().data_ptr()
    st = dd.param_noise_state
    assert st.dtype == torch.float64 and tuple(st.shape) == (2,)
    st = st.cpu().numpy()
    assert st[0] == 0.2 and np.isnan(st[1])
    _check_perturbation(dd, src, 0.2, seed, 0)
    pa.flat_params().fill_(float("nan"))                  # every float is rewritten, pads as 0
    assert dd.perturb_actor() is pa
    _check_perturbation(dd, src, 0.2, seed, 1)
    assert torch.equal(dd.actor.flat_params(), before)

    dz = _ddpg(S, A, philox_seed=seed, param_noise=_spec(initial_stddev=0.0))
    dz.perturb_actor()
    dz.perturbed_actor.flat_params().fill_(float("nan"))
    dz.perturb_actor()
    assert torch.equal(dz.perturbed_actor.flat_params(), dz.actor.flat_params())


def test_perturbation_stream_is_reproducible():
    runs = []
    for seed, philox in ((0, 42), (9, 42), (0, 43)):      # the second DDPG has other weights, then loads the first's
        dd = _ddpg(17, 6, seed=seed, philox_seed=philox, param_noise=_spec())
        if runs:
            dd.actor.load_state_dict(first.actor.state_dict())
        else:
            first = dd
        runs.append([dd.perturb_actor().flat_params().clone() for _ in range(2)])
    (a0, a1), (b0, b1), (c0, c1) = runs
    assert torch.equal(a0, b0) and torch.equal(a1, b1)
    assert not torch.equal(a0, a1) and not torch.equal(a0, c0) and not torch.equal(a1, c1)


def test_creating_the_perturbed_actor_draws_no_rng():
    dd = _ddpg(17, 6, param_noise=_spec())
    st = (torch.get_rng_state(), torch.cuda.get_rng_state(), np.random.get_state()[1].copy(), random.getstate())
    dd.perturb_actor()
    dd.adapt_param_noise(_states(np.random.RandomState(1), 8, 17))
    assert torch.equal(torch.get_rng_state(), st[0]) and torch.equal(torch.cuda.get_rng_state(), st[1])
    assert np.array_equal(np.random.get_state()[1], st[2]) and random.getstate() == st[3]


@pytest.mark.parametrize("E", [1, 33, 1024])
@pytest.mark.parametrize("obs_norm", [False, True], ids=["raw", "obs_norm"])
def test_act_runs_the_perturbed_actor(obs_norm, E):
    import d4pg_b200 as d4pg
    seed, S, A = 0x77 + E, 17, 6
    dd = _ddpg(S, A, philox_seed=seed, obs_norm=obs_norm or None, param_noise=_spec(initial_stddev=0.3))
    rng = np.random.RandomState(E)
    loc, scl = _fill(dd, 2000, rng) if obs_norm else (0.0, 1.0)
    s = _states(rng, E, S, loc, scl)
    sd = torch.from_numpy(s).cuda()
    assert torch.equal(dd.act(s, explore=False), dd.actor(sd))
    assert dd.perturbed_actor is None                     # explore=False draws no perturbation

    dd.noise = None                                       # parameter noise alone
    got = dd.act(s)
    pa = dd.perturbed_actor
    assert dd._perturbations == 1 and pa.obs_normalizer is dd.obs_normalizer
    assert torch.equal(got, pa(sd))
    _check_perturbation(dd, _logical(dd.actor), 0.3, seed, 0)
    assert dd._act_calls == 0

    # action noise on top: act's own stream counts exploring calls with action noise, whatever the perturbations did
    k = 0
    dd.noise = d4pg.random_process.GaussianNoise(dimension=A, num_epochs=100, mu=0.05, var=0.8)
    ap = pa(sd).cpu().numpy()
    for call, eps in enumerate((0.3, 1.5, 0.05)):
        if call == 1:
            dd.perturb_actor()
            ap = pa(sd).cpu().numpy()
        dd.noise.epsilon = eps
        got = dd.act(s).cpu().numpy()
        n = AO.gaussian_noise(PO.standard_normal(seed, AO.COUNTER_BASE + k, E * A).reshape(E, A), eps, 0.05, 0.8)
        AO.check_actions(got, AO.action(ap, n))
        k += 1
    nz = dd.noise = d4pg.random_process.OrnsteinUhlenbeckProcess(dimension=A, num_steps=1000, theta=0.25, mu=0.1,
                                                                sigma=0.5, dt=0.01)
    x = np.zeros((E, A))
    for call in range(4):
        reset = None if call == 0 else rng.rand(E) < 0.3
        if call == 2:
            dd.perturb_actor()
            ap = pa(sd).cpu().numpy()
        j = dd._perturbations
        got = dd.act(s, reset=reset).cpu().numpy()
        assert dd._perturbations == j                     # reset never re-perturbs
        z = PO.standard_normal(seed, AO.COUNTER_BASE + k, E * A).reshape(E, A)
        x = AO.ou_step(x, z, nz.theta, nz.mu, nz.sigma, nz.dt, reset=reset)
        AO.check_actions(got, AO.action(ap, nz.epsilon * x))
        k += 1
    assert dd._act_calls == k and dd._perturbations == 3
    assert torch.equal(dd.act(s, explore=False), dd.actor(sd))


def test_perturbation_is_a_snapshot():
    import d4pg_b200 as d4pg
    seed = 31
    dd = _ddpg(17, 6, seed=7, memory_size=2048, batch_size=64, sampling="device", philox_seed=seed,
               param_noise=_spec(initial_stddev=0.1))
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-2),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-2))
    _fill(dd, 1024, np.random.RandomState(8))
    s = _states(np.random.RandomState(9), 33, 17)
    dd.noise = None
    first = dd.act(s)
    snap = dd.perturbed_actor.flat_params().clone()
    before = dd.actor.flat_params().clone()
    dd.train_n(3)
    assert not torch.equal(dd.actor.flat_params(), before)
    assert torch.equal(dd.act(s), first) and torch.equal(dd.perturbed_actor.flat_params(), snap)
    dd.perturb_actor()                                    # perturbation 1, of the trained actor
    _check_perturbation(dd, _logical(dd.actor), 0.1, seed, 1)
    assert torch.equal(dd.act(s), dd.perturbed_actor(s))


def test_adapt_kernel_against_fp64():
    from d4pg_b200 import _lib
    L = _lib.lib()
    rng = np.random.RandomState(12)

    def run(a, ap, desired, coef, sigma=0.3):
        st = torch.tensor([sigma, 0.0], dtype=torch.float64).cuda()
        _lib.check(L.d4pg_param_noise_adapt(_lib.ptr(a), _lib.ptr(ap), a.numel(), desired, coef, _lib.ptr(st),
                                            _lib.stream_ptr()), "d4pg_param_noise_adapt")
        out = st.cpu().numpy()
        return float(out[0]), float(out[1])
    for n in (1, 7, 256, 1000, 6144, 100003):
        a = torch.from_numpy((rng.randn(n) * 0.5).astype(np.float32)).cuda()
        ap = torch.from_numpy((a.cpu().numpy() + rng.randn(n) * 0.1).astype(np.float32)).cuda()
        want = PO.distance(a.cpu().numpy(), ap.cpu().numpy())
        for coef in (1.01, 1.5):
            sig, d = run(a, ap, 0.5 * want, coef)                 # d > desired: shrink
            assert abs(d - want) <= 1e-13 * want, (n, d, want)
            assert sig == PO.adapt(0.3, d, 0.5 * want, coef) == 0.3 / coef
            sig, d2 = run(a, ap, 2.0 * want, coef)                # d < desired: grow
            assert d2 == d and sig == 0.3 * coef
            sig, d3 = run(a, ap, d, coef)                         # the tie grows
            assert d3 == d and sig == 0.3 * coef
    a = torch.full((5,), 0.25, device="cuda")
    assert run(a, a, 1e-9, 1.01) == (0.3 * 1.01, 0.0)


def test_adapt_param_noise_against_oracle():
    seed, S, A, B = 5150, 17, 6, 256
    spec = _spec(initial_stddev=0.05, desired_action_stddev=1e-6, adoption_coefficient=1.05)
    dd = _ddpg(S, A, philox_seed=seed, param_noise=spec)
    s = _states(np.random.RandomState(13), B, S)
    src = _logical(dd.actor)
    a_or = PO.actor_forward(_unflatten(dd.actor, src), s)
    assert dd.param_noise_state is None
    sigma, seq = 0.05, []
    for call in range(10):
        if call == 5:
            spec.desired_action_stddev = 1e3                      # read at every call
        desired = spec.desired_action_stddev
        d = dd.adapt_param_noise(s if call % 2 else torch.from_numpy(s).cuda())
        st = dd.param_noise_state
        assert d.dim() == 0 and d.dtype == torch.float64 and d.data_ptr() == st.data_ptr() + 8
        ap_or = PO.actor_forward(_unflatten(dd.actor, PO.perturb(src, sigma, seed, call)), s)
        want = float(np.sqrt(np.mean((ap_or - a_or) ** 2)))
        got = d.item()
        assert abs(got - want) <= 1e-5 * want, (call, got, want)
        assert (got > desired) == (call < 5)
        sigma = PO.adapt(sigma, got, desired, 1.05)
        seq.append(sigma)
        assert st[0].item() == sigma, call
    assert seq[4] < seq[3] and seq[5] > seq[4]
    assert dd._perturbations == 10 and dd.perturbed_actor is None and dd._act_calls == 0
    dd.param_noise_state = None                                   # restart from initial_stddev
    spec.desired_action_stddev = 1e-6
    dd.adapt_param_noise(s)
    assert dd.param_noise_state[0].item() == 0.05 / 1.05
    dd.param_noise_state = None
    dd.perturb_actor()
    st = dd.param_noise_state.cpu().numpy()
    assert st[0] == 0.05 and np.isnan(st[1])


def test_param_noise_does_not_touch_the_learner():
    """train_n with device sampling leaves bit-identical parameters and sampled indices whether or not perturbations,
    adaptations and exploring act() calls are interleaved."""
    import d4pg_b200 as d4pg
    s = _states(np.random.RandomState(4), 100, 17)
    runs = []
    for interleave in (False, True):
        dd = _ddpg(17, 6, seed=5, memory_size=4096, batch_size=64, sampling="device", philox_seed=9,
                   param_noise=_spec())
        dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                                   d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
        _fill(dd, 2048, np.random.RandomState(6))
        idx = []
        for t in range(4):
            dd.train_n(3)
            idx.append(dd.last_batch_info()["idx"].clone())
            if interleave:
                dd.perturb_actor()
                dd.act(s)
                dd.adapt_param_noise(s[:64])
                dd.act(s, explore=False)
        torch.cuda.synchronize()
        runs.append([dd.actor.flat_params().clone(), dd.critic.flat_params().clone(), dd.actor_target.flat_params().clone(),
                     dd.critic_target.flat_params().clone(), torch.stack(idx)])
    for p, q in zip(*runs):
        assert torch.equal(p, q)


_LAUNCH_COUNT_SCRIPT = r"""
import json, sys
import numpy as np, torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
from tests import test_gpu_param_noise as T
rng = np.random.RandomState(10)
dd = T._ddpg(17, 6, obs_norm=True, param_noise=T._spec())
loc, scl = T._fill(dd, 1000, rng)
s = T._states(rng, 100, 17, loc, scl)
fresh = T._ddpg(17, 6, param_noise=T._spec())
dd.perturb_actor()

def no_noise_act():
    dd.noise = None
    dd.act(s)
calls = [dd.perturb_actor, lambda: dd.adapt_param_noise(s), lambda: dd.adapt_param_noise(s),
         lambda: fresh.adapt_param_noise(s), lambda: dd.act(s), no_noise_act]
torch.cuda.synchronize()
with profile(activities=[ProfilerActivity.CUDA]) as prof:
    for f in calls:
        f()
    torch.cuda.synchronize()
ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA
             and not e.name.startswith(("Memcpy", "Memset"))), key=lambda e: e.time_range.start)
print(json.dumps([e.name for e in ev]))
"""


def test_launch_counts():
    """perturb_actor(): 1 kernel; adapt_param_noise: 4 (the first adaptation of a DDPG included); act() after the
    first perturbation: 1.  One profiler session in a fresh process (kernel records of an earlier session in the same
    process can spill into a later one), the kernels in launch order."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _LAUNCH_COUNT_SCRIPT], cwd=root, capture_output=True, text=True,
                       timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    names = json.loads(r.stdout.strip().splitlines()[-1])
    adapt = ["actor_perturb", "act_chain", "act_chain", "param_noise_adapt"]
    want = ["actor_perturb"] + adapt * 3 + ["act_chain", "act_chain"]
    assert len(names) == len(want), names
    for n, w in zip(names, want):
        assert w + "_kernel" in n, (names, want)
