"""Observation normalization: the device statistics at every insert path, the apply, the learner's normalized batch on
every plan / pipeline / head, the modules, checkpointing and the rejected configurations, against the numpy
restatement in tests/obs_norm_oracle.py (bit for bit where the definition is exact)."""
import ctypes as C
import math
import random

import numpy as np
import pytest
import torch

from tests import obs_norm_oracle as ON

S_DIM, A_DIM = 17, 6


def _cat(N=51):
    return {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": N}


def _rows(rng, n, S=S_DIM, A=A_DIM, const_col=None):
    """Features of very different scales and offsets (some rows far out, so the clip is hit)."""
    scales = np.logspace(-2, 2, S)
    offs = np.linspace(-30.0, 30.0, S)
    s = (rng.randn(n, S) * scales + offs).astype(np.float32)
    s2 = (rng.randn(n, S) * scales + offs).astype(np.float32)
    if const_col is not None:
        s[:, const_col] = 2.5
    return (s, rng.uniform(-1, 1, (n, A)).astype(np.float32), (-3 * rng.rand(n)).astype(np.float64), s2,
            rng.rand(n) < 0.05)


def _bits_equal(a, b):
    a, b = np.ascontiguousarray(a), np.ascontiguousarray(b)
    return a.shape == b.shape and a.dtype == b.dtype and np.array_equal(a.view(np.uint8), b.view(np.uint8))


def _check_stats(norm, st, what=""):
    torch.cuda.synchronize()
    assert norm.count == int(st.n), what
    stats = norm.stats.cpu().numpy()
    assert _bits_equal(stats, st.packed()), "%s: stats differ (max |d| %.3g)" % (what, np.abs(stats - st.packed()).max())
    shift, scale = st.affine(norm.eps)
    aff = norm.affine.cpu().numpy()
    assert _bits_equal(aff[:norm.obs_dim], shift), what
    assert _bits_equal(aff[norm.obs_dim:], scale), what


# ---- host-only ---------------------------------------------------------------------------------------------------
def test_oracle_matches_numpy_moments():
    rng = np.random.RandomState(0)
    x = _rows(rng, 500)[0]
    st = ON.Stats(S_DIM).fold(x[:123]).fold(x[123:])
    assert np.allclose(st.mean, x.astype(np.float64).mean(0), rtol=1e-12, atol=1e-12)
    assert np.allclose(st.m2 / st.n, x.astype(np.float64).var(0), rtol=1e-9)
    shift, scale = ON.Stats(S_DIM).affine()
    assert (shift == 0).all() and (scale == 1).all()
    y = ON.apply(np.array([[-6.0, -5.0, 0.5, 5.0, 7.0]], np.float32), np.zeros(5, np.float32), np.ones(5, np.float32))
    assert y.tolist() == [[-5.0, -5.0, 0.5, 5.0, 5.0]]
    g = ON.dydx(np.array([[-6.0, -5.0, 0.5, 5.0, 7.0]], np.float32), np.zeros(5, np.float32), np.ones(5, np.float32))
    assert g.tolist() == [[0.0, 1.0, 1.0, 1.0, 0.0]]


@pytest.mark.parametrize("spec", [{"clip": 0.0}, {"clip": -1.0}, {"clip": math.inf}, {"eps": 0.0}, {"eps": math.nan},
                                  {"clip": "x"}, {"scale": 2.0}, 5, "on"])
def test_invalid_options_are_rejected(spec):
    from d4pg_b200.obs_norm import make_obs_normalizer
    with pytest.raises(ValueError):
        make_obs_normalizer(spec)


def test_option_forms():
    from d4pg_b200.obs_norm import ObsNormalizer, make_obs_normalizer
    assert make_obs_normalizer(None) is None and make_obs_normalizer(False) is None
    n = make_obs_normalizer(True)
    assert (n.clip, n.eps) == (5.0, 1e-8)
    n = make_obs_normalizer({"clip": 3})
    assert (n.clip, n.eps) == (3.0, 1e-8)
    m = ObsNormalizer(clip=2.0, eps=1e-6)
    assert make_obs_normalizer(m) is m


# ---- statistics at every insert path -------------------------------------------------------------------------------
INSERT_PATHS = ["add_single", "add_batch_host", "add_batch_device", "add_episode_nstep", "add_her_episode", "ring_wrap",
                "one_and_4097_rows", "constant_feature", "uniform_replay"]


@pytest.mark.gpu
@pytest.mark.parametrize("path", INSERT_PATHS)
def test_statistics_bit_exact_at_every_insert_path(path):
    import d4pg_b200 as d4pg
    rng = np.random.RandomState(7)
    size = 1000 if path == "ring_wrap" else 16384
    if path == "uniform_replay":
        buf = d4pg.Replay(size, None, n_steps=3, gamma=0.9, obs_norm=True)
    else:
        buf = d4pg.PrioritizedReplayBuffer(size, 0.6, obs_norm=True)
    norm = buf.obs_normalizer
    st = ON.Stats(S_DIM)
    if path == "add_single":
        s, a, r, s2, d = _rows(rng, 4100)
        for i in range(4100):                                     # the staging flush at 4096 rows, then 4 more
            buf.add(s[i], a[i], r[i], s2[i], d[i])
        st.fold(s)
        _check_stats(norm, st, path)
    elif path == "add_batch_host":
        for k in range(3):                                        # both staging slots, then the first again
            rows = _rows(rng, 300)
            buf.add_batch(*rows)
            st.fold(rows[0])
            _check_stats(norm, st, "%s %d" % (path, k))
    elif path == "add_batch_device":
        rows = _rows(rng, 777)
        buf.add_batch(*[torch.as_tensor(x).cuda() for x in rows])
        st.fold(rows[0])
        _check_stats(norm, st, path)
    elif path in ("add_episode_nstep", "uniform_replay"):
        for T in (10, 2, 25):                                     # T = 2 < n = 3 inserts nothing
            s, a, r, s2, d = _rows(rng, T)
            got = buf.add_episode(s, a, r, s2, d, n_steps=3, gamma=0.9) if path == "add_episode_nstep" \
                else buf.add_episode(s, a, r, s2, d)
            assert got == max(0, T - 2)
            st.fold(s[:max(0, T - 2)])
            _check_stats(norm, st, "%s T=%d" % (path, T))
    elif path == "add_her_episode":
        buf = d4pg.PrioritizedReplayBuffer(size, 0.6, obs_norm=True)
        norm = buf.obs_normalizer
        T, So, G = 30, S_DIM - 3, 3
        obs = (rng.randn(T, So) * 10).astype(np.float32)
        goal = rng.randn(T, G)
        n_out = buf.add_her_episode(obs, obs + 1, goal, rng.randn(T, G), rng.uniform(-1, 1, (T, A_DIM)),
                                    -np.ones(T), np.zeros(T, bool), rng=np.random.RandomState(3))
        assert n_out > T                                          # relabelled copies were stored, and count
        torch.cuda.synchronize()
        st.fold(buf._store.obs[:n_out].cpu().numpy())             # the stored rows, in insertion order
        _check_stats(norm, st, path)
    elif path == "ring_wrap":
        for k in range(3):                                        # 2100 rows through a ring of 1000
            rows = _rows(rng, 700)
            buf.add_batch(*[torch.as_tensor(x).cuda() for x in rows])
            st.fold(rows[0])
        assert len(buf) == 1000
        _check_stats(norm, st, path)
    elif path == "one_and_4097_rows":
        rows = _rows(rng, 1)
        buf.add_batch(*rows)
        st.fold(rows[0])
        _check_stats(norm, st, "1 row")
        rows = _rows(rng, 4097)
        buf.add_batch(*rows)                                      # above the packed path's 4096 rows
        st.fold(rows[0])
        _check_stats(norm, st, "4097 rows")
    elif path == "constant_feature":
        rows = _rows(rng, 500, const_col=4)
        buf.add_batch(*rows)
        st.fold(rows[0])
        _check_stats(norm, st, path)
        assert st.m2[4] == 0.0 and norm.scale[4].item() == np.float32(1.0 / math.sqrt(1e-8))


@pytest.mark.gpu
def test_empty_statistics_and_standalone_update_split_invariance():
    import d4pg_b200 as d4pg
    norm = d4pg.ObsNormalizer(obs_dim=S_DIM)
    assert norm.count == 0 and (norm.shift.cpu() == 0).all() and (norm.scale.cpu() == 1).all()
    x = torch.tensor([[-7.0, -5.0, 5.0, 6.0] + [0.25] * (S_DIM - 4)], device="cuda")
    assert norm.normalize(x).cpu().tolist() == [[-5.0, -5.0, 5.0, 5.0] + [0.25] * (S_DIM - 4)]
    rows = _rows(np.random.RandomState(2), 1500)[0]
    st = ON.Stats(S_DIM).fold(rows)
    for cuts in ((1500,), (1, 999, 1500), (700, 701, 1500)):
        n = d4pg.ObsNormalizer(obs_dim=S_DIM)
        lo = 0
        for hi in cuts:
            n.update(rows[lo:hi])
            lo = hi
        _check_stats(n, st, str(cuts))


@pytest.mark.gpu
def test_apply_and_derivative_bit_exact():
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib
    rng = np.random.RandomState(5)
    norm = d4pg.ObsNormalizer(clip=3.0, obs_dim=S_DIM)
    rows = _rows(rng, 400)[0]
    norm.update(rows)
    st = ON.Stats(S_DIM).fold(rows)
    shift, scale = st.affine()
    x = _rows(rng, 333)[0]
    x[0] = shift + np.float32(3.0) / scale                      # near +clip and exactly at it where it rounds so
    x[1] = shift - np.float32(3.0) / scale
    x[2] = shift
    xt = torch.from_numpy(x).cuda()
    y = torch.empty_like(xt)
    g = torch.empty_like(xt)
    _lib.check(_lib.lib().d4pg_obs_normalize(_lib.ptr(norm.affine), S_DIM, 3.0, _lib.ptr(xt), x.shape[0], _lib.ptr(y),
                                             _lib.ptr(g), _lib.stream_ptr()), "d4pg_obs_normalize")
    assert _bits_equal(y.cpu().numpy(), ON.apply(x, shift, scale, 3.0))
    assert _bits_equal(g.cpu().numpy(), ON.dydx(x, shift, scale, 3.0))
    pre = ON.pre_clip(x, shift, scale)
    assert (np.abs(pre) > 3).any() and (np.abs(pre) < 3).any()
    # the identity affine: +-clip exactly is inside (derivative = scale), the next float is outside
    ident = d4pg.ObsNormalizer(clip=5.0, obs_dim=4)
    v = torch.tensor([[5.0, -5.0, np.nextafter(np.float32(5), np.float32(6)), -6.0]], device="cuda")
    yy, gg = ident._apply(v, True)
    assert yy.cpu().tolist() == [[5.0, -5.0, 5.0, -5.0]] and gg.cpu().tolist() == [[1.0, 1.0, 0.0, 0.0]]


# ---- the learner's normalized batch --------------------------------------------------------------------------------
def _make(d4pg, B=256, info=None, precision="tf32x3", chain="cluster", sampling="device", n=8192, seed=3, **kw):
    torch.manual_seed(seed); np.random.seed(seed); random.seed(seed)
    dd = d4pg.DDPG(S_DIM, A_DIM, memory_size=n, batch_size=B, critic_dist_info=info or _cat(), precision=precision,
                   chain=chain, sampling=sampling, philox_seed=5, obs_norm=True, **kw)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    return dd


def _check_batch(dd, st, all_rows, what):
    B = dd.batch_size
    idx = dd.last_batch_info()["idx"].cpu().numpy()
    shift, scale = st.affine()
    for name, src in (("s", all_rows[0]), ("s2", all_rows[3])):
        got = dd.debug_tensor(name, shape=(B, dd.obs_dim)).cpu().numpy()
        want = ON.apply(src[idx], shift, scale)
        assert _bits_equal(got, want), "%s: %s differs from the oracle-normalized rows (max |d| %.3g)" % (
            what, name, np.abs(got - want).max())
    return idx


def _cat_rows(parts):
    return tuple(np.concatenate([p[i] for p in parts]) for i in range(5))


LEARNER_CASES = {
    "tc_chain_train_n": dict(precision="tf32x3", chain="cluster"),
    "tc_chain_host_pipeline": dict(precision="tf32x3", chain="cluster", sampling="reference"),
    "chain_fp32": dict(precision="fp32", chain="cluster"),
    "levels_b1024": dict(precision="fp32", chain="levels", B=1024),
    "bf16": dict(precision="bf16", chain="levels"),
    "eager": dict(precision="tf32x3", chain="cluster", use_graph=False),
    "uniform_replay": dict(precision="tf32x3", chain="cluster", prioritized_replay=False),
    "mixture_head": dict(precision="tf32x3", chain="cluster", info={"type": "mixture_of_gaussian", "n_components": 5}),
    "quantile_head": dict(precision="tf32x3", chain="cluster", info={"type": "quantile", "n_quantiles": 32}),
}
ORACLE_CASES = ("tc_chain_host_pipeline", "chain_fp32", "levels_b1024")


@pytest.mark.gpu
@pytest.mark.parametrize("case", list(LEARNER_CASES))
def test_learner_batch_is_normalized_bit_exact(case):
    """After every step, debug_tensor("s"/"s2") equals the oracle normalization of the raw rows at the step's indices
    with the statistics of every row added before it; adds between steps change the statistics.  For three cases the
    parameters after five steps are held to the oracle step on the normalized batch."""
    import d4pg_b200 as d4pg
    from oracle import d4pg_oracle as O
    from tests import helpers as H
    kw = dict(LEARNER_CASES[case])
    B = kw.pop("B", 256)
    dd = _make(d4pg, B=B, **kw)
    rng = np.random.RandomState(11)
    parts = [_rows(rng, 3000)]
    dd.replayBuffer.add_batch(*parts[0])
    st = ON.Stats(S_DIM).fold(parts[0][0])
    lo = None
    if case in ORACLE_CASES:
        lo = O.LearnerOracle(S_DIM, A_DIM, _cat(), actor_w={k: v.cpu().clone() for k, v in dd.actor.state_dict().items()},
                             critic_w={k: v.cpu().clone() for k, v in dd.critic.state_dict().items()})
    steps = 5 if lo is not None else 4
    for t in range(steps):
        if t and (case != "tc_chain_train_n" or t % 2 == 0):
            new = _rows(rng, 256)                                 # host rows: the ingest stream under the host pipeline
            dd.replayBuffer.add_batch(*new)
            parts.append(new)
            st.fold(new[0])
        all_rows = _cat_rows(parts)
        if case == "tc_chain_train_n":
            dd.train_n(8)                                         # the 8-step graph; no adds inside it
        else:
            dd.train()
        idx = _check_batch(dd, st, all_rows, "%s step %d" % (case, t))
        if lo is not None:
            ON.train_step_normalized(lo, st, all_rows, idx)
    if lo is not None:
        for k in H.NAMES:
            for mine, ref in ((dd.actor.state_dict()[k], lo.actor[k]), (dd.critic.state_dict()[k], lo.critic[k]),
                              (dd.actor_target.state_dict()[k], lo.actor_target[k]),
                              (dd.critic_target.state_dict()[k], lo.critic_target[k])):
                err = (mine.cpu() - ref).abs()
                assert err.max().item() <= 2.5e-4 and (err > 1e-5).float().mean().item() <= 0.1, (case, k)


@pytest.mark.gpu
def test_option_adds_no_launch_and_leaves_raw_paths_raw():
    import d4pg_b200 as d4pg
    on = _make(d4pg)
    torch.manual_seed(3); np.random.seed(3); random.seed(3)
    off = d4pg.DDPG(S_DIM, A_DIM, memory_size=8192, batch_size=256, critic_dist_info=_cat(), precision="tf32x3",
                    sampling="device", philox_seed=5)
    off.assign_global_optimizer(d4pg.SharedAdam(off.actor.parameters(), lr=1e-3), d4pg.SharedAdam(off.critic.parameters(), lr=1e-3))
    rows = _rows(np.random.RandomState(1), 3000)
    for dd in (on, off):
        dd.replayBuffer.add_batch(*rows)
        dd.train()
    assert on.kernels_per_step() == off.kernels_per_step()
    # the stored rows and the replay's own sample / gather paths stay raw
    random.seed(9)
    s_on = on.replayBuffer.sample(64, beta=0.4)[0]
    random.seed(9)
    s_off = off.replayBuffer.sample(64, beta=0.4)[0]
    assert np.array_equal(s_on, s_off)
    idx = on.replayBuffer.sample(8, beta=0.4)[-1]
    assert np.array_equal(on.replayBuffer._encode_sample(idx)[0], rows[0][idx])


# ---- modules -------------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_modules_normalize_their_state_input():
    import d4pg_b200 as d4pg
    dd = _make(d4pg, sampling="reference")
    rng = np.random.RandomState(4)
    rows = _rows(rng, 2000)
    dd.replayBuffer.add_batch(*rows)
    st = ON.Stats(S_DIM).fold(rows[0])
    dd.train()                                                    # attaches the learner's ingest stream
    new = _rows(rng, 256)
    dd.replayBuffer.add_batch(*new)                               # issued on the ingest stream
    st.fold(new[0])
    shift, scale = st.affine()
    s = _rows(rng, 64)[0]
    a = rng.uniform(-1, 1, (64, A_DIM)).astype(np.float32)
    sn = torch.from_numpy(ON.apply(s, shift, scale)).cuda()
    out = {}
    for name in ("actor", "actor_target", "critic", "critic_target"):
        net = getattr(dd, name)
        assert net.obs_normalizer is dd.obs_normalizer
        x = torch.from_numpy(s).cuda()
        out[name] = net(x) if name.startswith("actor") else net(x, torch.from_numpy(a).cuda())
    for name in out:
        net = getattr(dd, name)
        net.obs_normalizer = None
        ref = net(sn) if name.startswith("actor") else net(sn, torch.from_numpy(a).cuda())
        net.obs_normalizer = dd.obs_normalizer
        assert torch.equal(out[name], ref), name
    # standalone modules have no normalizer
    assert d4pg.actor(S_DIM, A_DIM).obs_normalizer is None


@pytest.mark.gpu
@pytest.mark.parametrize("net_name", ["actor", "critic"])
def test_differentiable_state_gradient(net_name):
    import d4pg_b200 as d4pg
    dd = _make(d4pg)
    rng = np.random.RandomState(6)
    rows = _rows(rng, 1000)
    dd.replayBuffer.add_batch(*rows)
    shift, scale = ON.Stats(S_DIM).fold(rows[0]).affine()
    net = getattr(dd, net_name)
    net.differentiable = True
    s = torch.from_numpy(_rows(rng, 48)[0] * np.float32(1.5)).cuda().requires_grad_(True)
    a = torch.from_numpy(rng.uniform(-1, 1, (48, A_DIM)).astype(np.float32)).cuda()
    call = (lambda x: net(x)) if net_name == "actor" else (lambda x: net(x, a))
    w = torch.randn_like(call(s.detach()))
    (call(s) * w).sum().backward()
    # d loss / d normalized input from the same module without the normalizer, then float64 autograd through the clamp
    y = torch.from_numpy(ON.apply(s.detach().cpu().numpy(), shift, scale)).cuda().requires_grad_(True)
    net.obs_normalizer = None
    (call(y) * w).sum().backward()
    x64 = s.detach().double().cpu().requires_grad_(True)
    z = torch.clamp((x64 - torch.from_numpy(shift).double()) * torch.from_numpy(scale).double(), -5.0, 5.0)
    z.backward(y.grad.double().cpu())
    clipped = (ON.dydx(s.detach().cpu().numpy(), shift, scale) == 0)
    assert clipped.any() and not clipped.all()
    err = (s.grad.double().cpu() - x64.grad).abs()
    assert err.max().item() <= 1e-6 * max(1.0, x64.grad.abs().max().item()), err.max().item()


# ---- checkpointing and rejections ----------------------------------------------------------------------------------
@pytest.mark.gpu
def test_state_dict_round_trip_and_prefetched_batch_resampled():
    import d4pg_b200 as d4pg
    rng = np.random.RandomState(8)
    rows_a, rows_b = _rows(rng, 3000), _rows(rng, 3000)
    src = _make(d4pg)
    src.replayBuffer.add_batch(*rows_b)
    saved = src.obs_normalizer.state_dict()
    fresh = _make(d4pg)
    fresh.replayBuffer.add_batch(*rows_a)
    fresh.obs_normalizer.load_state_dict(saved)
    assert _bits_equal(fresh.obs_normalizer.affine.cpu().numpy(), src.obs_normalizer.affine.cpu().numpy())
    assert _bits_equal(fresh.obs_normalizer.stats.cpu().numpy(), src.obs_normalizer.stats.cpu().numpy())
    # a learner with a prefetched batch: the load makes it stale, the next step re-samples with the loaded affine
    dd = _make(d4pg)
    dd.replayBuffer.add_batch(*rows_a)
    dd.train()
    dd.train()                                                    # batch 3 is now prefetched with rows_a's statistics
    dd.obs_normalizer.load_state_dict(saved)
    dd.train()
    st_b = ON.Stats(S_DIM).fold(rows_b[0])
    _check_batch(dd, st_b, rows_a, "after load")
    with pytest.raises(ValueError):
        d4pg.ObsNormalizer(clip=4.0, obs_dim=S_DIM).load_state_dict(saved)


@pytest.mark.gpu
def test_rejected_configurations():
    import d4pg_b200 as d4pg
    from d4pg_b200 import _lib

    class _Comm(object):
        world_size, handle = 2, None
    with pytest.raises(d4pg.D4PGError, match="world size > 1"):
        d4pg.DDPG(S_DIM, A_DIM, critic_dist_info=_cat(), obs_norm=True, comm=_Comm())
    with pytest.raises(ValueError):
        d4pg.DDPG(S_DIM, A_DIM, critic_dist_info=_cat(), obs_norm={"clip": -1.0})
    with pytest.raises(ValueError):
        d4pg.DDPG(S_DIM, A_DIM, critic_dist_info=_cat(), obs_norm={"eps": math.inf})
    # the C entry: a valid config of a learner without the option, then obs_norm = 1 on its normalizer-less replay
    torch.manual_seed(0)
    dd = d4pg.DDPG(S_DIM, A_DIM, memory_size=4096, batch_size=64, critic_dist_info=_cat(), sampling="device")
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters()), d4pg.SharedAdam(dd.critic.parameters()))
    dd.replayBuffer.add_batch(*_rows(np.random.RandomState(0), 1000))
    dd.train()
    assert dd._learner.cfg.obs_norm == 0
    L = _lib.lib()
    h = C.c_void_p()
    buf = _lib.LearnerBuffers()

    def create(**fields):
        c = _lib.LearnerConfig.from_buffer_copy(dd._learner.cfg)
        for k, v in fields.items():
            setattr(c, k, v)
        return L.d4pg_learner_create(C.byref(c), C.byref(buf), dd.replayBuffer._store.handle, None, C.byref(h)), \
            L.d4pg_last_error().decode()
    rc, msg = create(obs_norm=1)
    assert rc == _lib.EINVAL and "observation normalizer" in msg, (rc, msg)
    rc, msg = create(obs_norm=1, world_size=2)
    assert rc == _lib.EINVAL and "world_size > 1" in msg, (rc, msg)
    rc, msg = create(obs_norm=2)
    assert rc == _lib.EINVAL and "obs_norm must be" in msg, (rc, msg)
    st = dd.replayBuffer._store
    z = torch.zeros(1 + 2 * S_DIM, dtype=torch.float64, device="cuda")
    f = torch.zeros(2 * S_DIM, device="cuda")
    assert L.d4pg_replay_set_obs_norm(st.handle, _lib.ptr(z), _lib.ptr(f), 0.0, 1e-8, None) == _lib.EINVAL
    assert L.d4pg_replay_set_obs_norm(st.handle, _lib.ptr(z), _lib.ptr(f), 5.0, -1.0, None) == _lib.EINVAL
    assert L.d4pg_replay_obs_norm_refresh(st.handle, None) == _lib.ESTATE
