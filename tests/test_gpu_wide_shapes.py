"""The widest shapes and largest launches of the learner's plan choice, act(), the actor perturbation, the streaming
n-step insert and the observation normalizer: the code that only runs past one cluster rank, one grid-stride pass, one
environment per warp, one tile per CTA or one feature per thread, against the oracles the narrow shapes use.

Launch geometry follows the SM count, so every geometry case derives its threshold from the device it runs on and
asserts that its shape crosses it:
  actor_perturb_kernel      at most 8 * SMs CTAs of 256 threads, 4 floats each   (csrc/param_noise.cu)
  replay_add_steps_kernel   min(ceil(E / 8), 4 * SMs) CTAs of 8 warps; chunk = ceil(E / CTAs) environments per CTA,
                            256 per tile (csrc/replay.cu d4pg_replay_add_steps)
  obs_stats_kernel          one CTA of at most 1024 threads, thread j owns features j, j + 1024, ...
  obs_normalize_kernel      at most 4 * SMs CTAs of 256 threads, grid-strided over n * S elements (csrc/obs_norm.cu)
"""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from tests import act_oracle as AO
from tests import nstep_stream_oracle as SO
from tests import obs_norm_oracle as ON
from tests import param_noise_oracle as PO

INFO = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _ddpg(obs_dim, act_dim, seed=0, memory_size=4096, batch_size=64, **kw):
    import d4pg_b200 as d4pg
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    return d4pg.DDPG(obs_dim, act_dim, memory_size=memory_size, batch_size=batch_size, critic_dist_info=INFO, **kw)


def _states(rng, E, S):
    return (rng.randn(E, S) * 4).astype(np.float32)


# ---- 1. the step plan where the cluster chain stops fitting (CPU: the workspace carries the plan) --------------------
def _workspace_floats(S, A, B, precision, chain):
    from d4pg_b200 import _lib
    c = _lib.LearnerConfig(obs_dim=S, act_dim=A, n_atoms=51, batch=B, precision=precision, chain=chain)
    return _lib.lib().d4pg_learner_workspace_floats(C.byref(c))


@pytest.mark.parametrize("S, A, B, precision, fits", [
    (576, 6, 512, 0, True), (577, 6, 256, 0, False), (576, 17, 256, 1, True), (577, 17, 256, 1, False),
    (17, 256, 128, 0, True), (17, 257, 64, 0, False), (17, 257, 64, 1, False), (700, 6, 512, 1, False)])
def test_chain_plan_only_where_its_slots_fit(S, A, B, precision, fits):
    """A chain plan's workspace holds the cluster exchange planes, the level plan's does not: with chain=1 the learner
    sizes the chain's workspace exactly up to |s| = 576 and |a| = 256, the level plan's one past them."""
    chain, levels = _workspace_floats(S, A, B, precision, 1), _workspace_floats(S, A, B, precision, 0)
    assert levels > 0 and (chain > levels) == fits, (chain, levels)


# ---- 2. act() with fc3 on every cluster rank -------------------------------------------------------------------------
@pytest.mark.gpu
def test_gaussian_and_ou_exploration_at_256_actions():
    """(17, 256), E = 4097: fc3's output tiles sit on all 8 cluster ranks, so the epilogue's Philox draw index and OU
    state index run past column 32; Gaussian noise over two calls, then OU over three with rows restarted."""
    import d4pg_b200 as d4pg
    seed, E, S, A = 0xACE, 4097, 17, 256
    dd = _ddpg(S, A, philox_seed=seed)
    rng = np.random.RandomState(21)
    s = _states(rng, E, S)
    a = dd.actor(torch.from_numpy(s).cuda()).cpu().numpy()
    dd.noise.mu, dd.noise.var = 0.05, 0.8
    k = 0
    for eps in (0.3, 1.5):
        dd.noise.epsilon = eps
        got = dd.act(s).cpu().numpy()
        n = AO.gaussian_noise(PO.standard_normal(seed, AO.COUNTER_BASE + k, E * A).reshape(E, A), eps, 0.05, 0.8)
        AO.check_actions(got, AO.action(a, n))
        k += 1
    nz = dd.noise = d4pg.random_process.OrnsteinUhlenbeckProcess(dimension=A, num_steps=1000, theta=0.25, mu=0.1,
                                                                sigma=0.5, dt=0.01)
    x = np.zeros((E, A))
    step = nz.sigma * np.sqrt(nz.dt)
    for call in range(3):
        reset = None if call == 0 else rng.rand(E) < 0.3
        got = dd.act(s, reset=reset).cpu().numpy()
        z = PO.standard_normal(seed, AO.COUNTER_BASE + k, E * A).reshape(E, A)
        carried = AO.ou_step(x, z, nz.theta, nz.mu, nz.sigma, nz.dt)
        x = AO.ou_step(x, z, nz.theta, nz.mu, nz.sigma, nz.dt, reset=reset)
        st = dd.exploration_state.cpu().numpy()
        assert (np.abs(st - x) <= 1e-14 * np.maximum(np.abs(x), step)).all(), "call %d" % call
        if reset is not None:
            assert reset.any() and not np.allclose(st[reset], carried[reset])
        AO.check_actions(got, AO.action(a, nz.epsilon * x))
        k += 1
    assert dd._act_calls == k


# ---- 3. the actor perturbation over more than one grid-stride pass --------------------------------------------------
@pytest.mark.gpu
def test_perturbation_beyond_one_grid_pass():
    """act_dim 256 and an obs_dim = 1 (mod 4) whose padded actor is about 1.125 passes of the capped grid (obs_dim 3981
    on 132 SMs): fc1 rows carry 3 pad columns, fc3 has 256 rows, and the grid-stride loop runs a second time.  The
    existing oracle comparison, pads and sigma = 0 included."""
    import d4pg_b200 as d4pg
    from tests import test_gpu_param_noise as TP
    one_pass = 8 * _sms() * 256 * 4
    A = 256
    rest = 2 * (256 * 256 + 256) + A * 256 + A + 256     # fc2, fc2_2, fc3 and the fc1 bias, all 4-float aligned
    S = -(-(one_pass * 9 // 8 - rest) // 256)
    S += (1 - S) % 4                                     # 3 pad columns per fc1 row
    total = d4pg.actor(S, A)._total
    assert S % 4 == 1 and one_pass < total < 2 * one_pass, (S, total, one_pass)
    TP.test_perturbation_matches_oracle((S, A))


@pytest.mark.gpu
def test_act_through_perturbed_actor_at_576x256():
    """act() through the perturbed actor at the largest act() shape with fc3 on every cluster rank: parameter noise
    alone equals the perturbed actor module bit for bit, then Gaussian action noise on top."""
    import d4pg_b200 as d4pg
    from tests import test_gpu_param_noise as TP
    seed, S, A, E = 0x5176, 576, 256, 33
    dd = _ddpg(S, A, philox_seed=seed, param_noise=d4pg.AdaptiveParamNoiseSpec(initial_stddev=0.2))
    s = _states(np.random.RandomState(22), E, S)
    sd = torch.from_numpy(s).cuda()
    src = TP._logical(dd.actor)
    dd.noise = None
    got = dd.act(s)
    pa = dd.perturbed_actor
    assert torch.equal(got, pa(sd)) and not torch.equal(got, dd.actor(sd))
    TP._check_perturbation(dd, src, 0.2, seed, 0)
    dd.noise = d4pg.random_process.GaussianNoise(dimension=A, num_epochs=100, mu=0.05, var=0.8)
    dd.noise.epsilon = 0.7
    got = dd.act(s).cpu().numpy()
    n = AO.gaussian_noise(PO.standard_normal(seed, AO.COUNTER_BASE, E * A).reshape(E, A), 0.7, 0.05, 0.8)
    AO.check_actions(got, AO.action(pa(sd).cpu().numpy(), n))


# ---- 4. the streaming n-step insert at many environments per CTA ----------------------------------------------------
def stream_columns(calls, n_steps, gamma):
    """tests/nstep_stream_oracle.stream_rows restated on arrays: every environment's window held at once, one vector
    step at a time.  A window appends (s, a, r) at slot fill % n; once its episode has n steps it emits (s, a of the
    oldest step, R, s', terminated), R = sum_i gamma^i r_i accumulated oldest first in float64 as the reference's loop
    does; an episode end clears it.  Returns (call, s, a, R, s2, done) column arrays in insertion order (call, then e)."""
    s0, a0 = np.asarray(calls[0][0]), np.asarray(calls[0][1])
    E, n = s0.shape[0], n_steps
    ws = np.zeros((E, n, s0.shape[1]), np.float32)
    wa = np.zeros((E, n, a0.shape[1]), np.float32)
    wr = np.zeros((E, n))
    fill = np.zeros(E, np.int64)
    eg = [1.0]
    for _ in range(n - 1):
        eg.append(eg[-1] * gamma)
    env = np.arange(E)
    cols = [[] for _ in range(6)]
    for k, (s, a, r, s2, term, trunc) in enumerate(calls):
        slot = fill % n
        ws[env, slot], wa[env, slot], wr[env, slot] = s, a, r
        fill += 1
        em = np.nonzero(fill >= n)[0]
        old = fill[em] % n
        R = np.zeros(em.size)
        for i in range(n):
            R = R + eg[i] * wr[em, (old + i) % n]
        for c, v in zip(cols, (np.full(em.size, k), ws[em, old], wa[em, old], R, np.asarray(s2)[em],
                               np.asarray(term, bool)[em])):
            c.append(v)
        ended = np.asarray(term, bool) | (np.asarray(trunc, bool) if trunc is not None else False)
        fill[ended] = 0
    return tuple(np.concatenate(c) for c in cols)


def _ring(cols, size):
    """The ring after inserting the rows in order: row j at j % size, later rows overwrite earlier ones."""
    m = cols[0].shape[0]
    j = np.arange(max(0, m - size), m)
    out = []
    for c in cols:
        r = np.zeros((size,) + c.shape[1:], c.dtype)
        r[j % size] = c[j]
        out.append(r)
    return out


def _long_calls(rng, K, E, S, A, n):
    """Episodes of every length: environment 0 never ends, 1 ends every n steps, 2 every n - 1, the rest rarely, so
    windows run past 2n steps."""
    term = rng.rand(K, E) < 0.004
    trunc = (rng.rand(K, E) < 0.002) & ~term
    term[:, 0] = trunc[:, 0] = False
    for e in range(1, min(E, 3)):
        term[:, e] = trunc[:, e] = False
        L = max(1, n + 1 - e)
        term[L - 1::L, e] = True
    return [(rng.randn(E, S).astype(np.float32), rng.uniform(-1, 1, (E, A)).astype(np.float32), rng.randn(E),
             rng.randn(E, S).astype(np.float32), term[k].copy(), trunc[k].copy()) for k in range(K)]


def _bits(x):
    x = np.ascontiguousarray(x)
    return x.view(np.uint8)


@pytest.mark.parametrize("E, n, long", [(1, 1, False), (5, 3, False), (33, 7, False), (40, 2, False), (3, 64, True),
                                        (5, 63, True), (7, 5, True)])
def test_vectorized_oracle_equals_stream_rows(E, n, long):
    rng = np.random.RandomState(E * 100 + n)
    K = 3 * n + 20 if long else 2 * n + 10
    calls = _long_calls(rng, K, E, 3, 2, n) if long else SO.random_calls(rng, K, E, 3, 2, n)
    if E > 3:
        calls[4] = calls[4][:5] + (None,)                # a call without truncation flags
    rows = SO.stream_rows(calls, n, 0.97)
    cols = stream_columns(calls, n, 0.97)
    assert len(rows) == cols[0].size > 0
    assert np.array_equal(cols[0], [k for k, _, _ in rows])
    for i in range(5):
        want = np.stack([np.asarray(r[i]) for _, _, r in rows]).astype(cols[i + 1].dtype)
        assert np.array_equal(_bits(cols[i + 1]), _bits(want)), i


def _steps_geometry(E):
    """(CTAs, environments per CTA, tiles per CTA) of one add_steps launch."""
    ctas = min(-(-E // 8), 4 * _sms())
    chunk = -(-E // ctas)
    return ctas, chunk, -(-chunk // 256)


def _run_stream(E, n, calls, size, obs_norm=False, prio=True, on_dev=False):
    import d4pg_b200 as d4pg
    from tests.test_gpu_nstep_stream import _on_device, _stored
    S, A = np.shape(calls[0][0])[1], np.shape(calls[0][1])[1]
    cols = stream_columns(calls, n, 0.97)
    counts = np.bincount(cols[0], minlength=len(calls))
    buf = d4pg.PrioritizedReplayBuffer(size, 0.6, obs_dim=S, act_dim=A, obs_norm=obs_norm or None) if prio else \
        d4pg.ReplayBuffer(size, obs_dim=S, act_dim=A, obs_norm=obs_norm or None)
    total = 0
    for k, c in enumerate(calls):
        got = buf.add_steps(*(_on_device(c) if on_dev else c), n_steps=n, gamma=0.97)
        assert got == counts[k], k
        total += got
        assert len(buf) == min(total, size) and buf._next_idx == total % size
    assert total > size
    want = _ring(cols[1:], size)
    mine = _stored(buf._store, size)
    for name, x, y in zip(("s", "a", "r", "s2", "done"), mine, want):
        assert np.array_equal(_bits(x), _bits(y.astype(x.dtype))), name
    if prio:
        assert float(buf._it_sum.sum(0, size)) == size and float(buf._it_min.min(0, size)) == 1.0
    if obs_norm:
        st = ON.Stats(S).fold(cols[1])
        stats = buf.obs_normalizer.stats.cpu().numpy()
        assert buf.obs_normalizer.count == total and np.array_equal(_bits(stats), _bits(st.packed()))
        shift, scale = st.affine(buf.obs_normalizer.eps)
        aff = buf.obs_normalizer.affine.cpu().numpy()
        assert np.array_equal(_bits(aff[:S]), _bits(shift)) and np.array_equal(_bits(aff[S:]), _bits(scale))
    return counts


# E as a function of the SM count: one past a warp per environment, exactly one full tile, one environment on a second
# tile, three tiles
STEPS_ES = ["warps+1", "tile", "tile+1", "2tiles+37"]


def _steps_E(which):
    w = 4 * _sms()
    return {"warps+1": 8 * w + 1, "tile": 256 * w, "tile+1": 256 * w + 1, "2tiles+37": 2 * 256 * w + 37}[which]


@pytest.mark.gpu
@pytest.mark.parametrize("n", [1, 3])
@pytest.mark.parametrize("which", STEPS_ES)
def test_add_steps_many_environments_per_warp_and_tiles_per_cta(which, n):
    """Bit-exact rows against the vectorized oracle, with a ring one call's rows straddle.  E = 8 * 4 * SMs + 1 gives a
    warp a second environment; E > 256 * 4 * SMs gives a CTA a second tile (red[] reused).  The first E runs with the
    normalizer on, which folds the rows read back across the wrap."""
    E = _steps_E(which)
    ctas, chunk, tiles = _steps_geometry(E)
    assert ctas == 4 * _sms() and chunk > 8
    assert tiles == {"warps+1": 1, "tile": 1, "tile+1": 2, "2tiles+37": 3}[which] and (which != "tile" or chunk == 256)
    rng = np.random.RandomState(E % 1000 + n)
    K = 2 * n + 6
    calls = SO.random_calls(rng, K, E, 3, 2, n)
    counts = np.bincount(stream_columns(calls, n, 0.97)[0], minlength=K).tolist()
    from tests.test_gpu_nstep_stream import _pick_size
    size = _pick_size(counts, E)
    assert size is not None
    _run_stream(E, n, calls, size, obs_norm=which == "warps+1", prio=n == 3, on_dev=which in ("tile", "2tiles+37"))


@pytest.mark.gpu
@pytest.mark.parametrize("n", [63, 64])
@pytest.mark.parametrize("E", [1, 33, 4097])
def test_add_steps_longest_windows(E, n):
    """n_steps 63 and 64 (the maximum) with episodes longer than 2n: a window's fill reaches 2n - 1 = 127 in the
    record's 8-bit fields and wraps by subtracting n."""
    rng = np.random.RandomState(E + n)
    K = 3 * n + 20
    calls = _long_calls(rng, K, E, 3, 2, n)
    ends = np.stack([c[4] | c[5] for c in calls])
    assert not ends[:, 0].any() and K > 2 * n + 1               # environment 0's window passes 2n steps
    counts = np.bincount(stream_columns(calls, n, 0.97)[0], minlength=K).tolist()
    if E == 1:
        size = 7
    else:
        from tests.test_gpu_nstep_stream import _pick_size
        size = _pick_size(counts, E)
    _run_stream(E, n, calls, size, prio=n == 63, on_dev=E == 33)


# ---- 5. the observation normalizer wider than one CTA's threads -----------------------------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("S", [1024, 1025, 2049])
def test_statistics_wider_than_one_cta(S):
    """obs_dim 1024 / 1025 / 2049: one, two and three features per thread of the 1024-thread statistics CTA, through
    ObsNormalizer.update (in two parts) and through a replay add_batch."""
    import d4pg_b200 as d4pg
    from tests.test_gpu_obs_norm import _check_stats, _rows
    assert -(-S // 1024) == {1024: 1, 1025: 2, 2049: 3}[S]
    rng = np.random.RandomState(S)
    rows = _rows(rng, 300, S=S)
    norm = d4pg.ObsNormalizer(obs_dim=S)
    norm.update(rows[0][:101])
    norm.update(rows[0][101:])
    st = ON.Stats(S).fold(rows[0])
    _check_stats(norm, st, "update S=%d" % S)
    buf = d4pg.PrioritizedReplayBuffer(1024, 0.6, obs_norm=True)
    buf.add_batch(*rows)
    more = _rows(rng, 77, S=S)
    buf.add_batch(*[torch.as_tensor(x).cuda() for x in more])
    _check_stats(buf.obs_normalizer, st.fold(more[0]), "add_batch S=%d" % S)


@pytest.mark.gpu
def test_apply_and_derivative_beyond_one_grid_pass():
    """n * S past two passes of the capped normalize grid, S = 1025 so a pass ends mid-row."""
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib
    from tests.test_gpu_obs_norm import _bits_equal, _rows
    S = 1025
    one_pass = 4 * _sms() * 256
    n = 2 * one_pass // S + 7
    assert n * S > 2 * one_pass and one_pass % S != 0
    rng = np.random.RandomState(9)
    norm = d4pg.ObsNormalizer(clip=3.0, obs_dim=S)
    rows = _rows(rng, 200, S=S)[0]
    norm.update(rows)
    shift, scale = ON.Stats(S).fold(rows).affine()
    x = _rows(rng, n, S=S)[0]
    xt = torch.from_numpy(x).cuda()
    y, g = torch.full_like(xt, float("nan")), torch.full_like(xt, float("nan"))
    _lib.check(_lib.lib().d4pg_obs_normalize(_lib.ptr(norm.affine), S, 3.0, _lib.ptr(xt), n, _lib.ptr(y), _lib.ptr(g),
                                             _lib.stream_ptr()), "d4pg_obs_normalize")
    assert _bits_equal(y.cpu().numpy(), ON.apply(x, shift, scale, 3.0))
    assert _bits_equal(g.cpu().numpy(), ON.dydx(x, shift, scale, 3.0))
    pre = ON.pre_clip(x, shift, scale)
    assert (np.abs(pre) > 3).any() and (np.abs(pre) < 3).any()


@pytest.mark.gpu
def test_learner_normalized_batch_at_1025_features():
    """|s| = 1025, B = 256 at fp32 with the cluster chain requested: the level plan runs (fc1 does not fit a chain
    CTA), and the step's s / s2 equal the oracle normalization of the sampled raw rows bit for bit."""
    import d4pg_b200 as d4pg
    from tests.test_gpu_obs_norm import _bits_equal, _rows
    S, A, B = 1025, 6, 256
    torch.manual_seed(3); np.random.seed(3); random.seed(3)
    dd = d4pg.DDPG(S, A, memory_size=4096, batch_size=B, critic_dist_info=INFO, precision="fp32", chain="cluster",
                   sampling="device", philox_seed=5, obs_norm=True, use_graph=False, prefetch=False)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rows = _rows(np.random.RandomState(11), 3000, S=S, A=A)
    dd.replayBuffer.add_batch(*rows)
    dd.train()
    torch.cuda.synchronize()
    assert dd.kernels_per_step() == 18                    # the level plan (the chain plan launches 7)
    shift, scale = ON.Stats(S).fold(rows[0]).affine()
    idx = dd.last_batch_info()["idx"].cpu().numpy()
    for name, src in (("s", rows[0]), ("s2", rows[3])):
        got = dd.debug_tensor(name, shape=(B, S)).cpu().numpy()
        assert _bits_equal(got, ON.apply(src[idx], shift, scale)), name
