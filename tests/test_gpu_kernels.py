"""CUDA kernels vs oracle / golden fixtures, called through the C ABI (libd4pg_sm90.so).
Run on an H100: `pytest -m gpu`."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from oracle import d4pg_oracle as O
from tests import helpers as H

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def d4pg():
    import d4pg_b200
    return d4pg_b200


def _proj(d4pg, probs, r, done, v_min, v_max, N, disc, mode, want_bins=True):
    from d4pg_b200 import _lib
    dev = "cuda"
    p = torch.from_numpy(np.ascontiguousarray(probs, dtype=np.float32)).to(dev)
    B = p.shape[0]
    rr = torch.from_numpy(np.asarray(r, dtype=np.float64)).to(dev)
    dd = torch.from_numpy(np.asarray(done).astype(np.uint8)).to(dev)
    m = torch.empty(B, N, dtype=torch.float32, device=dev)
    bl = torch.empty(B, N, dtype=torch.int32, device=dev)
    bu = torch.empty(B, N, dtype=torch.int32, device=dev)
    _lib.check(_lib.lib().d4pg_proj_loss(_lib.ptr(p), _lib.ptr(p), None, _lib.ptr(rr), _lib.ptr(dd), B, N,
                                         v_min, v_max, disc, mode, 3, 1e-6, 1.0 / B,
                                         _lib.ptr(m), _lib.ptr(bl), _lib.ptr(bu), None, None, None, None, None, None,
                                         None, None, _lib.stream_ptr()), "proj")
    torch.cuda.synchronize()
    return m.cpu().numpy(), bl.cpu().numpy(), bu.cpu().numpy()


def test_extension_is_loaded_not_a_fallback(d4pg):
    from d4pg_b200 import _lib
    assert _lib.lib().d4pg_version() >= 100
    assert _lib.lib().d4pg_device_sm() == 90, "expected an sm_90 (H100) device"
    maps = open("/proc/self/maps").read()
    assert "libd4pg_sm90.so" in maps


def test_projection_bit_exact_vs_golden_and_oracle(d4pg):
    g = H.load("projection.npz")
    for k in ("kat_nt", "kat_t", "kat_ti"):
        m, bl, bu = _proj(d4pg, g[k + "_probs"], g[k + "_r"], g[k + "_done"], -50.0, 0.0, 51, 0.99, 0)
        assert np.array_equal(m, g[k + "_m"]), k
    for c in range(int(g["n_rand"])):
        k = "rand%d" % c
        v_min, v_max, N, gamma = g[k + "_meta"]
        m, bl, bu = _proj(d4pg, g[k + "_probs"], g[k + "_r"], g[k + "_done"], float(v_min), float(v_max), int(N),
                          float(gamma), 0)
        assert np.array_equal(m, g[k + "_m"]), k
        _, ol, ou = O.project_live(g[k + "_probs"], g[k + "_r"], g[k + "_done"], float(v_min), float(v_max), int(N),
                                   float(gamma), return_bins=True)
        assert np.array_equal(bl, ol) and np.array_equal(bu, ou), k


def test_projection_mixed_terminal_rows_per_row_semantics(d4pg):
    """Batches the reference crashes on (SURVEY H6): integer and non-integer terminal b_j mixed."""
    rng = np.random.RandomState(8)
    B, N = 300, 51
    p = torch.softmax(torch.from_numpy(rng.randn(B, N).astype(np.float32) * 2), 1).numpy()
    r = np.where(rng.rand(B) < 0.5, -rng.randint(0, 60, B).astype(np.float64), -60 * rng.rand(B))
    done = rng.rand(B) < 0.5
    m, bl, bu = _proj(d4pg, p, r, done, -50.0, 0.0, N, 0.99, 0)
    mo, ol, ou = O.project_live(p, r, done, -50.0, 0.0, N, 0.99, return_bins=True)
    assert np.array_equal(m, mo) and np.array_equal(bl, ol) and np.array_equal(bu, ou)


def test_projection_nstep_vs_golden(d4pg):
    g = H.load("projection.npz")
    for i in range(2):
        k = "nstep%d" % i
        m, bl, bu = _proj(d4pg, g[k + "_probs"], g[k + "_r"], g[k + "_done"], -150.0, 150.0, 101, 0.99 ** 5, 1)
        _, ol, ou = O.project_nstep(g[k + "_probs"], g[k + "_r"], g[k + "_done"], -150.0, 150.0, 101, 0.99, 5,
                                    return_bins=True)
        assert np.array_equal(bl, ol) and np.array_equal(bu, ou)
        assert np.abs(m.astype(np.float64) - g[k + "_m"]).max() <= 1e-6     # tolerance: 1e-5 allowed, 1e-6 asserted


def test_projection_nstep_config5_size_vs_golden(d4pg):
    """B=4096, 101 atoms, n_steps=5: the reference's reproj_categorical_dist (ddpg.py:122-140) run at the BASELINE size."""
    g, p, r, done = H.projection_c5_inputs()
    m, bl, bu = _proj(d4pg, p, r, done, -150.0, 150.0, 101, 0.99 ** 5, 1)
    _, ol, ou = O.project_nstep(p, r, done, -150.0, 150.0, 101, 0.99, 5, return_bins=True)
    assert np.array_equal(bl, ol) and np.array_equal(bu, ou)
    H.check_compact(g, "m", m.astype(np.float64), 1e-6)


def test_projection_full_size_properties(d4pg):
    """Config-5 size (B=4096, N=101): rows sum to sum(p) (mass conservation), non-negative."""
    rng = np.random.RandomState(9)
    B, N = 4096, 101
    p = torch.softmax(torch.from_numpy(rng.randn(B, N).astype(np.float32) * 2), 1).numpy()
    r = 300 * (rng.rand(B) - 0.5)
    done = rng.rand(B) < 0.05
    for mode, disc in ((0, 0.99), (1, 0.99 ** 5)):
        m, bl, bu = _proj(d4pg, p, r, done, -150.0, 150.0, N, disc, mode)
        assert (m >= 0).all() and (bl >= 0).all() and (bu <= N - 1).all()
        tgt = np.where(done & (mode == 0), 1.0, p.astype(np.float64).sum(1))
        assert np.abs(m.astype(np.float64).sum(1) - tgt).max() < 5e-6


def test_heads_losses_and_gradients(d4pg):
    from d4pg_b200 import _lib
    rng = np.random.RandomState(10)
    for B, N in ((256, 51), (64, 101), (33, 7)):
        tl = (rng.randn(B, N) * 2).astype(np.float32)
        ql = (rng.randn(B, N) * 2).astype(np.float32)
        pl = (rng.randn(B, N) * 2).astype(np.float32)
        r = -3 * rng.rand(B)
        done = rng.rand(B) < 0.1
        v_min, v_max = (-50.0, 0.0)
        dev = "cuda"
        keep = []

        def t(x):
            keep.append(torch.from_numpy(np.ascontiguousarray(x)).to(dev))
            return keep[-1]
        outs = {k: torch.empty(B, N, dtype=torch.float32, device=dev) for k in ("m", "tp", "qp", "dq", "dpi")}
        rows = {k: torch.empty(B, dtype=torch.float32, device=dev) for k in ("loss", "td", "prio", "pi")}
        _lib.check(_lib.lib().d4pg_proj_loss(_lib.ptr(t(tl)), _lib.ptr(t(ql)), _lib.ptr(t(pl)), _lib.ptr(t(r)),
                                             _lib.ptr(t(done.astype(np.uint8))), B, N, v_min, v_max, 0.99, 0, 0, 1e-6,
                                             1.0 / B, _lib.ptr(outs["m"]), None, None, _lib.ptr(outs["tp"]),
                                             _lib.ptr(outs["qp"]), _lib.ptr(rows["loss"]), _lib.ptr(rows["td"]),
                                             _lib.ptr(rows["prio"]), _lib.ptr(outs["dq"]), _lib.ptr(rows["pi"]),
                                             _lib.ptr(outs["dpi"]), _lib.stream_ptr()), "heads")
        torch.cuda.synchronize()
        tp = torch.softmax(torch.from_numpy(tl), 1).numpy()
        q = torch.softmax(torch.from_numpy(ql), 1).numpy()
        np.testing.assert_allclose(outs["tp"].cpu().numpy(), tp, atol=2e-7)
        np.testing.assert_allclose(outs["qp"].cpu().numpy(), q, atol=2e-7)
        # oracle on the GPU's own softmax outputs isolates the projection/loss arithmetic
        m_o = O.project_live(outs["tp"].cpu().numpy(), r, done, v_min, v_max, N, 0.99)
        assert np.array_equal(outs["m"].cpu().numpy(), m_o)
        terms = O.critic_loss_terms(m_o, outs["qp"].cpu().numpy())
        np.testing.assert_allclose(rows["loss"].cpu().numpy(), terms["loss_rows"], atol=1e-5, rtol=1e-6)
        np.testing.assert_allclose(rows["td"].cpu().numpy(), terms["td"], atol=1e-6)
        np.testing.assert_allclose(rows["prio"].cpu().numpy(), terms["prio"], atol=1e-6)
        np.testing.assert_allclose(outs["dq"].cpu().numpy(), terms["dlogits"], atol=1e-6)
        # policy head vs autograd
        z = torch.from_numpy(O.atom_support(v_min, v_max, N)[1].reshape(-1, 1)).float()
        plt = torch.from_numpy(pl).requires_grad_(True)
        la = -torch.softmax(plt, 1).matmul(z).mean()
        la.backward()
        np.testing.assert_allclose(outs["dpi"].cpu().numpy(), plt.grad.numpy(), atol=1e-6)
        np.testing.assert_allclose(rows["pi"].cpu().numpy().mean(), la.item(), atol=1e-4, rtol=1e-6)


@pytest.mark.parametrize("name", ["full", "part", "wrap"])
def test_tree_golden_indices_bit_exact(d4pg, name):
    g = H.load("tree.npz")
    size, n_fill, B, rounds = [int(x) for x in g[name + "_meta"]]
    buf = d4pg.PrioritizedReplayBuffer(size, alpha=0.6)
    for i in range(n_fill):
        buf.add(np.full(2, i, np.float32), np.zeros(1, np.float32), -1.0, np.zeros(2, np.float32), False)
    assert len(buf) == min(size, n_fill)
    assert np.array_equal(buf._it_sum.values().astype(np.float64), g[name + "_sum_r0"])
    assert np.array_equal(buf._it_min.values().astype(np.float64), g[name + "_min_r0"])
    for k in range(rounds):
        out = buf.sample(B, float(g[name + "_beta"][k]), uniforms=g[name + "_u"][k])
        assert np.array_equal(np.array(out[6]), g[name + "_idx"][k]), (name, k)
        np.testing.assert_allclose(out[5], g[name + "_w"][k], rtol=1e-5)
        # gathered rows are the stored rows
        if k <= 3:      # (after round 3 seven zero rows are added, see below)
            assert np.array_equal(out[0][:, 0].astype(np.int64) % size, np.array(out[6]))
        buf.update_priorities(g[name + "_upd_idx"][k], g[name + "_upd_prio"][k])
        H.assert_tree_close_and_sync(buf, g["%s_sum_r%d" % (name, k + 1)], g["%s_min_r%d" % (name, k + 1)])
        if k == 3:
            for j in range(7):
                buf.add(np.zeros(2, np.float32), np.zeros(1, np.float32), -1.0, np.zeros(2, np.float32), False)
            assert np.array_equal(buf._it_sum.values().astype(np.float64), g[name + "_sum_after_add"])
            assert np.array_equal(buf._it_min.values().astype(np.float64), g[name + "_min_after_add"])
    assert np.float32(buf._max_priority) == np.float32(float(g[name + "_max_priority"]))


def test_tree_seeded_random_matches_oracle_default_uniforms(d4pg):
    """sample() without explicit uniforms draws random.random() like the reference (:262)."""
    size = 500
    buf = d4pg.PrioritizedReplayBuffer(size, alpha=0.6)
    ob = O.PrioritizedReplayOracle(size, 0.6, 3, 2)
    rng = np.random.RandomState(0)
    for i in range(size):
        row = (rng.randn(3).astype(np.float32), rng.rand(2).astype(np.float32), float(rng.rand()), rng.randn(3).astype(np.float32), bool(i % 7 == 0))
        buf.add(*row)
        ob.add(*row)
    for rnd in range(4):
        random.seed(77 + rnd)
        st = random.getstate()
        us = [random.random() for _ in range(32)]
        random.setstate(st)
        out = buf.sample(32, 0.5)
        exp = ob.sample(32, 0.5, us)
        assert out[6] == list(exp[6])
        for a, b in zip(out[:5], exp[:5]):
            assert np.array_equal(a, b)
        pr = (rng.rand(32).astype(np.float32) + np.float32(1e-6))
        buf.update_priorities(out[6], pr)
        ob.update_priorities(exp[6], pr)
        H.assert_tree_close_and_sync(buf, ob.sum.value, ob.min.value)


def test_tree_full_size_capacity_1m(d4pg):
    """Config 3 AS CONFIGURED (BASELINE.json configs[2]): capacity 10^6 (tree 2^20), |s| = 376, |a| = 17 (3 GB of rows),
    batch 1024: tree invariants, oracle indices, and the gathered 3-KB rows."""
    size, B, S, A = 1_000_000, 1024, 376, 17
    buf = d4pg.PrioritizedReplayBuffer(size, alpha=0.6, obs_dim=S, act_dim=A)
    dev = torch.device("cuda")
    step = 125_000                                     # filled from device tensors in chunks; row i carries i in column 0
    for lo in range(0, size, step):
        ids = torch.arange(lo, lo + step, device=dev, dtype=torch.float32)
        obs = torch.zeros(step, S, device=dev); obs[:, 0] = ids; obs[:, S - 1] = -ids
        obs2 = torch.zeros(step, S, device=dev); obs2[:, 1] = ids
        act = torch.zeros(step, A, device=dev); act[:, A - 1] = ids
        buf.add_batch(obs, act, ids.double() * 0.5, obs2, torch.zeros(step, dtype=torch.bool, device=dev))
    assert len(buf) == size
    ob = O.PrioritizedReplayOracle(size, 0.6, 1, 1)    # the oracle's trees only (its row storage is not needed)
    ob.length, ob.next_idx = size, 0
    ob.sum.value[ob.capacity:ob.capacity + size] = 1.0
    ob.min.value[ob.capacity:ob.capacity + size] = 1.0
    ob.sum.rebuild(); ob.min.rebuild()
    assert np.array_equal(buf._it_sum.values(), ob.sum.value)
    rng = np.random.RandomState(1)
    for rnd in range(3):
        us = rng.rand(B)
        out = buf.sample(B, 0.4, uniforms=us)
        idx = ob.sample_indices(us)
        assert np.array_equal(np.array(out[6]), idx)
        fi = idx.astype(np.float32)
        assert np.array_equal(out[0][:, 0], fi) and np.array_equal(out[0][:, S - 1], -fi) and np.array_equal(out[3][:, 1], fi)
        assert np.array_equal(out[1][:, A - 1], fi) and np.array_equal(np.asarray(out[2]).reshape(-1), idx * 0.5)
        pr = (rng.rand(B).astype(np.float32) + np.float32(1e-6))
        buf.update_priorities(out[6], pr)
        ob.update_priorities(idx, pr)
        H.assert_tree_close_and_sync(buf, ob.sum.value, ob.min.value)
    got = buf._it_sum.values()
    root = float(buf._it_sum.sum())
    assert abs(root - float(got[ob.capacity:].astype(np.float64).sum())) < 1.0      # checksum of leaves


def test_segment_tree_api(d4pg):
    t = d4pg.SumSegmentTree(16)
    o = O.SegmentTree32(16, "sum")
    om = O.SegmentTree32(16, "min")
    mt = d4pg.MinSegmentTree(16)
    rng = np.random.RandomState(2)
    for i in range(13):
        v = float(np.float32(rng.rand()))
        t[i] = v; mt[i] = v; o.set(i, v); om.set(i, v)
    assert t[5] == o.get(5)
    assert np.float32(t.sum()) == o.root()
    for s, e in ((0, 13), (0, 12), (3, 11), (7, 8), (5, 16), (1, 2)):
        ref_tree = [float(x) for x in o.value]
        # reference _reduce_helper evaluated on the oracle's node array
        def helper(start, end, node, ns, ne):
            if start == ns and end == ne:
                return np.float32(ref_tree[node])
            mid = (ns + ne) // 2
            if end <= mid:
                return helper(start, end, 2 * node, ns, mid)
            if mid + 1 <= start:
                return helper(start, end, 2 * node + 1, mid + 1, ne)
            return np.float32(helper(start, mid, 2 * node, ns, mid) + helper(mid + 1, end, 2 * node + 1, mid + 1, ne))
        assert np.float32(t.sum(s, e)) == helper(s, e - 1, 1, 0, 15), (s, e)
        assert np.float32(mt.min(s, e)) == np.float32(om.value[16 + s:16 + e].min())
    total = float(t.sum())
    for frac in (0.0, 0.3, 0.77, 0.999):
        assert t.find_prefixsum_idx(frac * total) == O.find_prefixsum_idx(o.value, 16, np.float32(frac * total))


def test_adam_polyak_kernel_vs_torch_formula(d4pg):
    from d4pg_b200 import _lib
    rng = np.random.RandomState(3)
    n = 4096 + 8
    p0, g0 = rng.randn(n).astype(np.float32), (rng.randn(n) * 1e-3).astype(np.float32)
    g0[::17] = 0.0
    t0 = rng.randn(n).astype(np.float32)
    p, m, v, tg = (torch.from_numpy(x.copy()).cuda() for x in (p0, np.zeros(n, np.float32), np.zeros(n, np.float32), t0))
    pt, mt, vt, tt = torch.from_numpy(p0.copy()), torch.zeros(n), torch.zeros(n), torch.from_numpy(t0.copy())
    for step in range(1, 6):
        g = torch.from_numpy(g0 * step)
        _lib.check(_lib.lib().d4pg_adam_polyak(_lib.ptr(p), _lib.ptr(g.cuda()), _lib.ptr(m), _lib.ptr(v), _lib.ptr(tg), n,
                                               1e-3, 0.9, 0.9, 1e-8, step, 0.001, 1.0, _lib.stream_ptr()), "adam")
        O.adam_step(pt, g, mt, vt, step, 1e-3)
        O.polyak(tt, pt, 0.001)
    torch.cuda.synchronize()
    np.testing.assert_allclose(p.cpu().numpy(), pt.numpy(), atol=1e-6)
    np.testing.assert_allclose(m.cpu().numpy(), mt.numpy(), atol=1e-8)
    np.testing.assert_allclose(v.cpu().numpy(), vt.numpy(), atol=1e-10)
    np.testing.assert_allclose(tg.cpu().numpy(), tt.numpy(), atol=1e-6)


def test_models_seeded_init_and_forward_vs_golden(d4pg):
    g = H.load("init.npz")
    torch.manual_seed(5)
    a = d4pg.actor(17, 6)
    c = d4pg.critic(17, 6, {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51})
    for k in H.NAMES:
        H.check_compact(g, "actor_" + k, a.state_dict()[k].cpu().numpy(), 0.0)
        H.check_compact(g, "critic_" + k, c.state_dict()[k].cpu().numpy(), 0.0)
    out = a(torch.from_numpy(g["x"])).cpu().numpy()
    np.testing.assert_allclose(out, g["actor_out"], atol=1e-6)
    q = c(torch.from_numpy(g["x"]), torch.from_numpy(g["act"])).cpu().numpy()
    np.testing.assert_allclose(q, g["critic_out"], atol=1e-6)
    # state_dict round trip through torch.save-compatible dicts (main.py:367-368)
    sd = {k: v.cpu() for k, v in a.state_dict().items()}
    a2 = d4pg.actor(17, 6)
    a2.load_state_dict(sd)
    assert torch.equal(a2.flat_params(), a.flat_params())
