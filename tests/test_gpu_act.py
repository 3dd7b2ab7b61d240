"""DDPG.act on the H100: without exploration bit-identical to the actor module, with Gaussian / Ornstein-Uhlenbeck
noise against tests/act_oracle.py, its Philox stream apart from the learner's, and one kernel per call."""
import random

import numpy as np
import pytest
import torch

from tests import act_oracle as AO

pytestmark = pytest.mark.gpu

INFO = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}
# (17, 33) / (17, 256): actor fc3 has output tiles on 2 / all 8 cluster ranks; (545, 6): chain_wpitch steps to the next
# 32 floats; (576, 17): the largest fc1 slot that fits the chain's shared memory
DIMS = [(1, 1), (3, 1), (17, 6), (17, 9), (376, 17), (17, 33), (17, 256), (545, 6), (576, 17)]
ES = (1, 31, 32, 33, 256, 4097)


def _ddpg(obs_dim, act_dim, seed=0, memory_size=8192, batch_size=64, **kw):
    import d4pg_b200 as d4pg
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    return d4pg.DDPG(obs_dim, act_dim, memory_size=memory_size, batch_size=batch_size, critic_dist_info=INFO, **kw)


def _fill(dd, n, rng):
    """n real replay inserts; the observations are shifted and scaled per feature so that the normalizer's affine is
    not the identity."""
    S, A = dd.obs_dim, dd.act_dim
    loc, scl = rng.uniform(-2, 2, S), rng.uniform(0.5, 3, S)
    st = (rng.randn(n, S) * scl + loc).astype(np.float32)
    s2 = (rng.randn(n, S) * scl + loc).astype(np.float32)
    a = rng.uniform(-1, 1, (n, A)).astype(np.float32)
    r = (-3 * rng.rand(n)).astype(np.float32).astype(np.float64)
    dd.replayBuffer.add_batch(st, a, r, s2, rng.rand(n) < 0.05)
    return loc, scl


def _states(rng, E, S, loc=0.0, scl=1.0):
    # 4 sigma wide: with the normalizer on, a share of the features lands beyond the clip of 5
    return (rng.randn(E, S) * 4 * scl + loc).astype(np.float32)


def _ou(dd, **kw):
    import d4pg_b200 as d4pg
    p = dict(theta=0.25, mu=0.1, sigma=0.5, dt=0.01)
    p.update(kw)
    dd.noise = d4pg.random_process.OrnsteinUhlenbeckProcess(dimension=dd.act_dim, num_steps=1000, **p)
    return dd.noise


@pytest.mark.parametrize("obs_norm", [False, True], ids=["raw", "obs_norm"])
@pytest.mark.parametrize("dims", DIMS, ids=["%dx%d" % d for d in DIMS])
def test_act_without_exploration_is_the_actor(dims, obs_norm):
    S, A = dims
    dd = _ddpg(S, A, obs_norm=obs_norm or None)
    rng = np.random.RandomState(100 * S + A)
    loc, scl = _fill(dd, 3000, rng) if obs_norm else (0.0, 1.0)
    if obs_norm:
        assert dd.obs_normalizer.count == 3000
    P = (S + 3) & ~3
    for E in ES:
        s = _states(rng, E, S, loc, scl)
        sd = torch.from_numpy(s).cuda()
        want = dd.actor(sd)
        pitched = torch.full((E, P + 4), float("nan"), device="cuda")      # rows read in place; pad columns never used
        pitched[:, :S] = sd
        for x in (s, sd, pitched[:, :S]):
            got = dd.act(x, explore=False)
            assert got.shape == (E, A) and got.dtype == torch.float32 and got.device == want.device
            assert torch.equal(got, want), "E=%d input %s" % (E, type(x).__name__)
        for row in (s[E - 1], sd[E - 1]):
            got = dd.act(row, explore=False)
            assert got.shape == (1, A) and torch.equal(got, want[E - 1:E])
    assert dd._act_calls == 0 and dd.exploration_state is None


def test_gaussian_exploration_matches_oracle():
    seed, E, A = 0x5EED, 4096, 6
    dd = _ddpg(17, A, obs_norm=True, philox_seed=seed)
    rng = np.random.RandomState(1)
    loc, scl = _fill(dd, 2000, rng)
    s = _states(rng, E, 17, loc, scl)
    a = dd.actor(torch.from_numpy(s).cuda()).cpu().numpy()
    dd.noise.mu, dd.noise.var = 0.05, 0.8
    for k, eps in enumerate((0.3, 1.5, 0.05)):          # epsilon is read at every call
        dd.noise.epsilon = eps
        got = dd.act(s).cpu().numpy()
        n = AO.gaussian_noise(AO.standard_normal(seed, k, E * A).reshape(E, A), eps, 0.05, 0.8)
        AO.check_actions(got, AO.action(a, n))
        v = a.astype(np.float64) + n
        clipped = np.abs(v) > 1.0 + 1e-9
        if eps > 1:
            assert clipped.mean() > 0.1
        assert np.array_equal(got[clipped], np.sign(v[clipped]).astype(np.float32))
    assert dd._act_calls == 3


def test_ou_exploration_matches_oracle():
    import d4pg_b200 as d4pg
    seed, E, A = 77, 300, 6
    dd = _ddpg(17, A, philox_seed=seed)
    nz = _ou(dd)
    rng = np.random.RandomState(2)
    s = _states(rng, E, 17)
    a = dd.actor(torch.from_numpy(s).cuda()).cpu().numpy()
    x = np.zeros((E, A))
    step = nz.sigma * np.sqrt(nz.dt)
    for k in range(20):
        reset = None if k == 0 else rng.rand(E) < 0.2
        if k % 4 == 3:
            nz.reset()                                    # the host object's epsilon decay is read by act
        arg = reset
        if reset is not None and k % 3 == 1:
            arg = torch.from_numpy(reset).cuda()          # device bool mask, read in place
        elif reset is not None and k % 3 == 2:
            arg = list(reset)
        got = dd.act(s, reset=arg).cpu().numpy()
        z = AO.standard_normal(seed, k, E * A).reshape(E, A)
        carried = AO.ou_step(x, z, nz.theta, nz.mu, nz.sigma, nz.dt)
        x = AO.ou_step(x, z, nz.theta, nz.mu, nz.sigma, nz.dt, reset=reset)
        st = dd.exploration_state
        assert st.dtype == torch.float64 and tuple(st.shape) == (E, A)
        st = st.cpu().numpy()
        assert (np.abs(st - x) <= 1e-14 * np.maximum(np.abs(x), step)).all(), "call %d" % k
        if reset is not None and reset.any():
            fresh = AO.ou_step(np.zeros((E, A)), z, nz.theta, nz.mu, nz.sigma, nz.dt)
            assert np.array_equal(x[reset], fresh[reset]) and not np.allclose(st[reset], carried[reset])
        AO.check_actions(got, AO.action(a, nz.epsilon * x))
    with pytest.raises(d4pg.D4PGError, match="300 environments"):
        dd.act(s[:10])
    dd.exploration_state = None
    dd.act(s[:10])
    assert tuple(dd.exploration_state.shape) == (10, A)


def test_exploration_stream_is_fresh_and_reproducible():
    rng = np.random.RandomState(3)
    s = _states(rng, 64, 17)
    seqs = []
    for seed in (0, 9):                                   # the second DDPG gets other weights, then loads the first's
        dd = _ddpg(17, 6, seed=seed, philox_seed=42)
        if seqs:
            dd.actor.load_state_dict(first.actor.state_dict())
        else:
            first = dd
        out = [dd.act(s) for _ in range(3)]
        _ou(dd)
        out += [dd.act(s, reset=(np.arange(64) % (2 + k)) == 0) for k in range(3)]
        seqs.append([t.clone() for t in out])
    y = seqs[0]
    assert not torch.equal(y[0], y[1]) and not torch.equal(y[3], y[4])
    for p, q in zip(*seqs):
        assert torch.equal(p, q)


def test_act_does_not_touch_the_learner():
    """train_n with device sampling leaves bit-identical parameters and sampled indices whether or not act() calls
    are interleaved (act's counter has the top bit set; the sampler's counter is the step index)."""
    import d4pg_b200 as d4pg
    rng0 = np.random.RandomState(4)
    s = _states(rng0, 100, 17)
    runs = []
    for interleave in (False, True):
        dd = _ddpg(17, 6, seed=5, memory_size=4096, batch_size=64, sampling="device", philox_seed=9)
        dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                                   d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
        _fill(dd, 2048, np.random.RandomState(6))
        idx = []
        for t in range(4):
            dd.train_n(3)
            idx.append(dd.last_batch_info()["idx"].clone())
            if interleave:
                dd.act(s)
                dd.act(s, explore=False)
        torch.cuda.synchronize()
        runs.append([dd.actor.flat_params().clone(), dd.critic.flat_params().clone(), dd.actor_target.flat_params().clone(),
                     dd.critic_target.flat_params().clone(), torch.stack(idx)])
    for p, q in zip(*runs):
        assert torch.equal(p, q)


def test_act_after_train_sees_the_updated_actor():
    import d4pg_b200 as d4pg
    dd = _ddpg(17, 6, seed=7, memory_size=2048, batch_size=64)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-2),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-2))
    _fill(dd, 1024, np.random.RandomState(8))
    s = _states(np.random.RandomState(9), 33, 17)
    before = dd.act(s, explore=False)
    for _ in range(3):
        dd.train()
        got = dd.act(s, explore=False)               # same stream as train() hands back to: no synchronize
        assert torch.equal(got, dd.actor(s))
    assert not torch.equal(got, before)


def _kernels(prof):
    from torch.autograd import DeviceType
    return [e.name for e in prof.events() if e.device_type == DeviceType.CUDA
            and not e.name.startswith(("Memcpy", "Memset"))]


def test_one_kernel_per_act_call():
    from torch.profiler import ProfilerActivity, profile
    dd = _ddpg(17, 6, obs_norm=True)
    rng = np.random.RandomState(10)
    loc, scl = _fill(dd, 1000, rng)
    s = _states(rng, 100, 17, loc, scl)
    sd = torch.from_numpy(s).cuda()                      # 17-wide rows: one 2-D device copy into the pitch-4 buffer
    sp = torch.zeros(100, 20, device="cuda")[:, :17]     # 16-B pitched: read in place
    sp.copy_(sd)
    dd_ou = _ddpg(17, 6, obs_norm=True)
    _fill(dd_ou, 1000, rng)
    _ou(dd_ou)
    mask_d = torch.from_numpy(np.arange(100) % 3 == 0).cuda()
    calls = [lambda: dd.act(s, explore=False), lambda: dd.act(sd, explore=False), lambda: dd.act(sp),
             lambda: dd.act(s), lambda: dd.act(s[0]),
             lambda: dd_ou.act(s),                                    # first OU call: the state is allocated
             lambda: dd_ou.act(sd, reset=np.arange(100) % 2 == 0), lambda: dd_ou.act(sp, reset=mask_d)]
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for f in calls:
            f()
        torch.cuda.synchronize()
    names = _kernels(prof)
    assert len(names) == len(calls) and all("act_chain_kernel" in n for n in names), names
