"""Episode tails of the streaming insert on the device (DESIGN.md §3 "Episode tails"): every stored row and horizon
bit-exact against the oracle (tests/nstep_tails_oracle.py) over window lengths, environment counts, shapes, ring wraps
and both kinds of end flags, with the trees, max_priority and the normalizer equal to add_batch of the oracle's rows;
n = 1 and the full rows equal to a tails-off buffer; other insert paths clearing horizons; the learner's per-row
discounts in the categorical, mixture and quantile heads against their oracles; every layer of one-pass TF32 and bf16
learner steps over tail rows; a tails-on learner over all-zero
horizons bit-identical to a tails-off one; and the launches per call."""
import random

import numpy as np
import pytest
import torch

from tests import mog_oracle as MO
from tests import nstep_stream_oracle as SO
from tests import nstep_tails_oracle as TO
from tests import qr_oracle as QO
from tests import step_check as SC

pytestmark = pytest.mark.gpu

INFO = {"type": "categorical", "v_min": -10.0, "v_max": 0.0, "n_atoms": 51}


def _on_device(c):
    cu = lambda x: None if x is None else torch.as_tensor(x).cuda()
    return tuple(cu(x) for x in c)


def _stored(store, n):
    torch.cuda.synchronize()
    return (store.obs[:n].cpu().numpy(), store.act[:n].cpu().numpy(), store.rew[:n].cpu().numpy(),
            store.obs2[:n].cpu().numpy(), store.done[:n].cpu().numpy().astype(bool),
            None if store.horizon is None else store.horizon[:n].cpu().numpy())


def _expected_ring(rows, size):
    """The ring after inserting `rows` ((s, a, R, s2, done), horizon) in order: row i at i % size."""
    m = len(rows)
    keep = rows[max(0, m - size):]
    pos = [(max(0, m - size) + j) % size for j in range(len(keep))]
    order = np.argsort(pos)
    cols = [np.stack([np.asarray(r[i]) for r, _ in keep]) for i in range(5)] + [np.array([h for _, h in keep])]
    return [c[order] for c in cols]


def _pick_size(counts, floor):
    """A ring size >= floor that one call's rows straddle (rows before it + half of its own), or None."""
    cum = 0
    for c in counts:
        if c >= 2 and cum + c // 2 >= floor:
            return cum + c // 2
        cum += c
    return None


def _many_ends(rng, K, E, n):
    """Ends often enough that many calls carry tail rows; every environment ends in the first n calls."""
    term, trunc = SO.random_ends(rng, K, E, n, p_term=0.1, p_trunc=0.1)
    first = rng.randint(0, n, E)
    trunc[first, np.arange(E)] |= ~term[first, np.arange(E)]
    return term, trunc


def _calls(rng, K, E, S, A, n):
    term, trunc = _many_ends(rng, K, E, n)
    return [(rng.randn(E, S).astype(np.float32), rng.uniform(-1, 1, (E, A)).astype(np.float32), rng.randn(E),
             rng.randn(E, S).astype(np.float32), term[k].copy(), trunc[k].copy()) for k in range(K)]


CASES = [(n, E, d) for n in (2, 5, 7) for E in (1, 31, 32, 33, 1024, 4096) for d in ((3, 2), (17, 6), (376, 17))] + \
        [(64, E, d) for E in (1, 33) for d in ((3, 2), (17, 6))]


@pytest.mark.parametrize("n_steps,E,dims", CASES, ids=["n%d-E%d-%dx%d" % (n, E, *d) for n, E, d in CASES])
def test_vs_oracle(n_steps, E, dims):
    """Every stored row bit-exact (s, a, f64 R, s2, done, horizon), len() and the return value after every call, the
    ring wrapped with one call's rows straddling its end.  Host flags for n in (5, 64), CUDA tensors otherwise; PER for
    odd n, whose trees and max_priority must equal a buffer fed the oracle's rows by add_batch, as must the normalizer's
    statistics."""
    import d4pg_b200 as d4pg
    S, A = dims
    rng = np.random.RandomState(n_steps * 7919 + E * 31 + S)
    K = 3 * n_steps + 12
    calls = _calls(rng, K, E, S, A, n_steps)
    gamma = 0.97
    rows = TO.tail_rows(calls, n_steps, gamma)
    counts = np.bincount([r[0] for r in rows], minlength=K).tolist()
    assert any(r[3] for r in rows)
    size = _pick_size(counts, E * max(1, n_steps - 1)) if E > 1 else max(7, n_steps - 1)
    assert size is not None and len(rows) > size, (counts, size)
    prio = n_steps % 2 == 1
    mk = (lambda: d4pg.PrioritizedReplayBuffer(size, 0.6, obs_dim=S, act_dim=A, obs_norm=True, nstep_tails=True)) if prio \
        else (lambda: d4pg.ReplayBuffer(size, obs_dim=S, act_dim=A, obs_norm=True, nstep_tails=True))
    buf = mk()
    on_dev = n_steps not in (5, 64)
    total = 0
    for k, c in enumerate(calls):
        got = buf.add_steps(*(_on_device(c) if on_dev else c), n_steps=n_steps, gamma=gamma)
        assert got == counts[k], k
        total += got
        assert len(buf) == min(total, size) and buf._next_idx == total % size
    want = _expected_ring([(r[4], r[3]) for r in rows], size)
    mine = _stored(buf._store, size)
    for name, x, y in zip(("s", "a", "r", "s2", "done", "horizon"), mine, want):
        assert np.array_equal(x, y.astype(x.dtype)), name
    ref = mk()
    for k in range(K):
        rk = [r[4] for r in rows if r[0] == k]
        if rk:
            ref.add_batch(*(torch.as_tensor(np.stack([np.asarray(r[i]) for r in rk])).cuda() for i in range(5)))
    torch.cuda.synchronize()
    sa, sb = buf._store, ref._store
    names = ("sum_tree", "min_tree", "state") if prio else ("state",)
    for name in names:
        assert torch.equal(getattr(sa, name), getattr(sb, name)), name
    assert torch.equal(sa.obs_norm.stats, sb.obs_norm.stats) and torch.equal(sa.obs_norm.affine, sb.obs_norm.affine)


def test_n1_and_full_rows_equal_tails_off():
    """n = 1 with tails stores exactly what it stores without (every horizon 0); at n = 5 the rows of horizon 0 of a
    tails-on buffer are, in order, the rows of a tails-off buffer fed the same stream."""
    import d4pg_b200 as d4pg
    S, A, E = 9, 3, 37
    rng = np.random.RandomState(3)
    for n in (1, 5):
        calls = _calls(rng, 25, E, S, A, n)
        on = d4pg.PrioritizedReplayBuffer(4000, 0.6, obs_dim=S, act_dim=A, nstep_tails=True)
        off = d4pg.PrioritizedReplayBuffer(4000, 0.6, obs_dim=S, act_dim=A)
        for k, c in enumerate(calls):
            x = c if k % 2 else _on_device(c)
            on.add_steps(*x, n_steps=n, gamma=0.9)
            off.add_steps(*x, n_steps=n, gamma=0.9)
        a, b = _stored(on._store, len(on)), _stored(off._store, len(off))[:5]
        if n == 1:
            assert len(on) == len(off) and not a[5].any()
            for x, y in zip(a[:5], b):
                assert np.array_equal(x, y)
            for name in ("sum_tree", "min_tree", "state"):
                assert torch.equal(getattr(on._store, name), getattr(off._store, name))
        else:
            full = a[5] == 0
            assert len(on) > len(off) == int(full.sum())
            for x, y in zip(a[:5], b):
                assert np.array_equal(x[full], y)


def test_other_inserts_clear_horizons():
    """add_batch (device and host rows), add and add_episode over ring slots that held tail rows store horizon 0 there;
    every other slot keeps its horizon."""
    import d4pg_b200 as d4pg
    S, A, E, n, size, m = 5, 2, 8, 4, 64, 9
    rng = np.random.RandomState(9)
    buf = d4pg.ReplayBuffer(size, obs_dim=S, act_dim=A, nstep_tails=True)
    calls = _calls(rng, 200, E, S, A, n)
    for c in calls:                              # stop where the next m slots hold at least two tail rows
        buf.add_steps(*c, n_steps=n, gamma=0.9)
        torch.cuda.synchronize()
        h0 = buf._store.horizon.cpu().numpy().copy()
        touched = [(buf._next_idx + i) % size for i in range(m)]
        if len(buf) == size and (h0[touched] > 0).sum() >= 2:
            break
    assert (h0[touched] > 0).sum() >= 2
    rows = [rng.randn(3, S).astype(np.float32), rng.randn(3, A).astype(np.float32), rng.randn(3),
            rng.randn(3, S).astype(np.float32), np.zeros(3, bool)]
    buf.add_batch(*(torch.as_tensor(x).cuda() for x in rows))
    buf.add_batch(*rows)
    buf.add(rows[0][0], rows[1][0], 1.0, rows[3][0], False)
    buf._store.flush()
    buf.add_episode(*[x[:2] for x in rows])
    torch.cuda.synchronize()
    h = buf._store.horizon.cpu().numpy()
    assert not h[touched].any()
    rest = np.setdiff1d(np.arange(size), touched)
    assert np.array_equal(h[rest], h0[rest])


def _learner_stream(dd, rng, K, E, trunc_p=0.3):
    S = dd.obs_dim
    steps = []
    for k in range(K):
        s = torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda()
        a = dd.act(s)
        term = rng.rand(E) < 0.05
        trunc = (rng.rand(E) < trunc_p) & ~term
        steps.append(dd.observe(s, a, torch.as_tensor(-rng.rand(E)).cuda(), torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda(),
                                torch.as_tensor(term).cuda(), torch.as_tensor(trunc).cuda()))
    return steps


def _batch(dd):
    B = dd.batch_size
    idx = dd.last_batch_info()["idx"].cpu().numpy()
    st = dd.replayBuffer._store
    torch.cuda.synchronize()
    h = dd.debug_tensor("h", dtype=torch.uint8).cpu().numpy()[:B]
    assert np.array_equal(h, st.horizon[torch.as_tensor(idx).long().cuda()].cpu().numpy()), "batch horizons"
    s = st.obs[idx].cpu().numpy(); a = st.act[idx].cpu().numpy(); r = st.rew[idx].cpu().numpy()
    s2 = st.obs2[idx].cpu().numpy(); d = st.done[idx].cpu().numpy().astype(bool)
    assert np.array_equal(dd.debug_tensor("r", dtype=torch.float64).cpu().numpy()[:B], r)
    return s, a, r, s2, d, h


PLANS = [dict(precision="fp32", chain="levels"), dict(precision="fp32", chain="cluster"),
         dict(precision="tf32x3", chain="cluster")]
PIPES = [dict(sampling="reference", prefetch=True), dict(sampling="device", prefetch=True)]


@pytest.mark.parametrize("pipe", PIPES, ids=["host_pipeline", "device_prefetch"])
@pytest.mark.parametrize("plan", PLANS, ids=["levels_fp32", "ffma_chain_fp32", "tc_chain_tf32x3"])
def test_learner_categorical_vs_oracle(plan, pipe):
    """A DDPG(nstep_tails=True, n_steps=5, projection="nstep") fed by observe() with many truncations: each step's
    batch (indices, rows, the `h` plane) is the ring's rows at the sampled indices, the projection's bins equal the
    per-row-discount oracle's, and the oracle learner trained on the same batch with discounts gamma ** h, from the
    learner's parameters before the step, gives the projected rows and the losses within 1e-5 and the gradients within
    1e-6 + 1e-4 of their largest entry.  The parameters after Adam are held to 1e-4 only: Adam divides a near-zero
    gradient by its own magnitude, so fp32 summation order alone moves such an entry by more than 1e-5."""
    import d4pg_b200 as d4pg
    from oracle import d4pg_oracle as O
    S, A, E, n, B = 17, 6, 32, 5, 64
    torch.manual_seed(0)
    random.seed(1)
    dd = d4pg.DDPG(S, A, memory_size=4096, batch_size=B, critic_dist_info=INFO, n_steps=n, projection="nstep",
                   nstep_tails=True, gamma=0.95, **plan, **pipe)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    lo = TO.TailsLearnerOracle(S, A, INFO, gamma=0.95, n_steps=n, projection="nstep",
                               actor_w={k: v.cpu().clone() for k, v in dd.actor.state_dict().items()},
                               critic_w={k: v.cpu().clone() for k, v in dd.critic.state_dict().items()})
    rng = np.random.RandomState(4)
    _learner_stream(dd, rng, 12, E)
    seen_tail = 0
    for step in range(6):
        _learner_stream(dd, rng, 1, E)
        dd.train()
        s, a, r, s2, d, h = _batch(dd)
        seen_tail += int(((h > 0) & ~d).sum())
        lo.disc = TO.row_discounts(h, 0.95, n)
        out = lo.train_step(s, a, r, s2, d)
        prev = [dd.actor.state_dict(), dd.critic.state_dict(), dd.actor_target.state_dict(), dd.critic_target.state_dict()]
        m_dev = dd.debug_tensor("m", shape=(B, 51)).cpu().numpy()
        assert np.abs(m_dev - out["m"]).max() <= 1e-5
        lc, la = dd.last_losses()
        assert abs(lc - float(out["loss_critic"])) <= 1e-5 and abs(la - float(out["loss_actor"])) <= 1e-4
        torch.cuda.synchronize()
        for net, mine, want, params in ((dd.critic, out["grads_critic"], lo.critic, dd.critic.state_dict()),
                                        (dd.actor, out["grads_actor"], lo.actor, dd.actor.state_dict())):
            grads = dict(net.named_parameters())
            for k in O.PARAM_ORDER:
                g = grads[k].grad.detach().cpu()
                assert (g - mine[k]).abs().max().item() <= 1e-6 + 1e-4 * mine[k].abs().max().item(), k
                assert (params[k].cpu() - want[k]).abs().max().item() <= 1e-4, k
        # the next step starts from the learner's parameters: the per-step check does not compound earlier rounding
        for dst, src in zip((lo.actor, lo.critic, lo.actor_target, lo.critic_target), prev):
            for k in O.PARAM_ORDER:
                dst[k].copy_(src[k].cpu())
    assert seen_tail > 10


def test_categorical_projection_per_row():
    """The learner's projected target rows of a batch with many tail rows equal the f64 per-row-discount projection
    of its own target probabilities to within one f32 rounding, bin for bin (fp32 levels plan, n = 7)."""
    import d4pg_b200 as d4pg
    S, A, E, n, B = 17, 6, 32, 7, 128
    torch.manual_seed(0)
    dd = d4pg.DDPG(S, A, memory_size=4096, batch_size=B, critic_dist_info=INFO, n_steps=n, projection="nstep",
                   nstep_tails=True, sampling="device", chain="levels")
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(5)
    _learner_stream(dd, rng, 20, E, trunc_p=0.4)
    dd.train()
    s, a, r, s2, d, h = _batch(dd)
    assert ((h > 0) & ~d).sum() > 10
    tp = dd.debug_tensor("target_probs", shape=(B, 51)).cpu().numpy()
    m, _, _ = TO.project_disc(tp, r, d, INFO["v_min"], INFO["v_max"], 51, TO.row_discounts(h, dd.gamma, n))
    assert np.abs(dd.debug_tensor("m", shape=(B, 51)).cpu().numpy() - m).max() <= 2e-7


# (plan, precision, |s|, |a|, DDPG options): the one-pass precisions on each plan they run (csrc/learner.cu step_plan)
ONE_PASS = [("tc_chain", "tf32", 17, 6, {}), ("chain", "tf32", 33, 6, {}),
            ("levels", "tf32", 17, 6, {"chain": "levels"}), ("levels", "bf16", 17, 6, {})]


@pytest.mark.parametrize("plan,precision,S,A,opts", ONE_PASS, ids=["%s_%s" % c[:2] for c in ONE_PASS])
def test_one_pass_learner_tails(plan, precision, S, A, opts):
    """One TF32 pass and bf16 with tails, fed by observe() with many truncations: after each step the projected rows
    equal the f64 per-row-discount projection of the learner's own target probabilities to within one f32 rounding,
    every layer of the step passes tests/step_check.py for its plan and precision, and the batch holds tail rows."""
    import d4pg_b200 as d4pg
    E, n, B = 32, 5, 64
    torch.manual_seed(0)
    dd = d4pg.DDPG(S, A, memory_size=4096, batch_size=B, critic_dist_info=INFO, n_steps=n, projection="nstep",
                   nstep_tails=True, gamma=0.95, precision=precision, sampling="device", prefetch=False, **opts)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(8)
    _learner_stream(dd, rng, 12, E, trunc_p=0.4)
    for step in range(3):
        _learner_stream(dd, rng, 1, E, trunc_p=0.4)
        W = SC.snapshot(dd)
        dd.train()
        torch.cuda.synchronize()
        assert dd.kernels_per_step() == SC.KERNELS[plan], (plan, dd.kernels_per_step())
        s, a, r, s2, d, h = _batch(dd)
        assert ((h > 0) & ~d).any(), step
        tp = dd.debug_tensor("target_probs", shape=(B, 51)).cpu().numpy()
        m, _, _ = TO.project_disc(tp, r, d, INFO["v_min"], INFO["v_max"], 51, TO.row_discounts(h, dd.gamma, n))
        assert np.abs(dd.debug_tensor("m", shape=(B, 51)).cpu().numpy() - m).max() <= 2e-7, step
        SC.check_step(dd, W, plan, precision, label="tails %s/%s step %d" % (plan, precision, step))


@pytest.mark.parametrize("kind", ["mixture", "quantile"])
@pytest.mark.parametrize("pipe", PIPES, ids=["host_pipeline", "device_prefetch"])
def test_learner_mog_qr_heads_vs_oracle(kind, pipe):
    """Mixture (K = 5) and quantile (N = 51) critics with tails: each step's loss rows, td and priorities equal the f64
    head oracle evaluated on the learner's own raw planes with each row's discount gamma ** h (gamma ** n for h = 0)."""
    import d4pg_b200 as d4pg
    S, A, E, n, B = 17, 6, 32, 5, 64
    info = {"type": "mixture_of_gaussian", "n_components": 5} if kind == "mixture" else \
        {"type": "quantile", "n_quantiles": 51, "kappa": 1.0}
    W = 15 if kind == "mixture" else 51
    torch.manual_seed(0)
    random.seed(2)
    dd = d4pg.DDPG(S, A, memory_size=4096, batch_size=B, critic_dist_info=info, n_steps=n, projection="nstep",
                   nstep_tails=True, chain="levels", gamma=0.95, **pipe)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                               d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    rng = np.random.RandomState(6)
    _learner_stream(dd, rng, 12, E)
    seen = 0
    for step in range(4):
        _learner_stream(dd, rng, 1, E)
        dd.train()
        s, a, r, s2, d, h = _batch(dd)
        seen += int(((h > 0) & ~d).sum())
        tr = dd.debug_tensor("target_logits", shape=(B, W)).cpu().double()
        q = dd.debug_tensor("q_logits", shape=(B, W)).cpu().double()
        rows = dd.debug_tensor("loss_rows").cpu().numpy()[:B]
        td = dd.last_batch_info()["td"].cpu().numpy()
        for k in np.unique(h):
            sel = np.nonzero(h == k)[0]
            disc = 0.95 ** int(k) if k else 0.95 ** n
            if kind == "mixture":
                o = MO.heads(tr[sel], q[sel], None, r[sel], d[sel], disc, 5, 1.0 / B)
            else:
                o = QO.heads(tr[sel], q[sel], None, r[sel], d[sel], disc, 1.0, 1.0 / B)
            for name, got in (("loss_rows", rows[sel]), ("td", td[sel])):
                want = o[name].numpy()
                assert np.abs(got - want).max() <= 1e-4 * max(1.0, np.abs(want).max()), (name, k)
    assert seen > 10


@pytest.mark.parametrize("kind", ["categorical", "mixture", "quantile"])
def test_zero_horizons_bit_identical(kind):
    """A tails-on learner over a buffer with no tail rows (every horizon 0) is bit-identical to a tails-off learner:
    parameters, losses and priorities over 20 steps."""
    import d4pg_b200 as d4pg
    info = {"categorical": INFO, "mixture": {"type": "mixture_of_gaussian", "n_components": 5},
            "quantile": {"type": "quantile", "n_quantiles": 51}}[kind]
    S, A, N = 17, 6, 1024
    rng = np.random.RandomState(7)
    data = [rng.randn(N, S).astype(np.float32), rng.uniform(-1, 1, (N, A)).astype(np.float32), -rng.rand(N),
            rng.randn(N, S).astype(np.float32), rng.rand(N) < 0.1]
    runs = []
    for tails in (False, True):
        torch.manual_seed(0)
        dd = d4pg.DDPG(S, A, memory_size=N, batch_size=64, critic_dist_info=info, n_steps=5, projection="nstep",
                       sampling="device", nstep_tails=tails)
        dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                                   d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
        dd.replayBuffer.add_batch(*data)
        out = []
        for _ in range(20):
            dd.train()
            out += [torch.tensor(dd.last_losses()), dd.last_batch_info()["prio"].cpu().clone()]
        torch.cuda.synchronize()
        out += [dd.actor.flat_params().cpu().clone(), dd.critic.flat_params().cpu().clone()]
        runs.append(out)
    for x, y in zip(*runs):
        assert torch.equal(x, y)


_LAUNCH_COUNT_SCRIPT = r"""
import json
import numpy as np, torch
from torch.autograd import DeviceType
from torch.profiler import ProfilerActivity, profile
import d4pg_b200 as d4pg
S, A, E, n = 17, 6, 64, 3
rng = np.random.RandomState(1)

def args(ended):
    end = torch.zeros(E, dtype=torch.bool)
    end[::2] = ended
    return (torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda(), torch.rand(E, A, device="cuda"),
            torch.rand(E, dtype=torch.float64, device="cuda"), torch.as_tensor(rng.randn(E, S).astype(np.float32)).cuda(),
            torch.zeros(E, dtype=torch.bool, device="cuda"), end.cuda())

out = {}
for name, per, tails in [("plain", False, False), ("plain_tails", False, True), ("per", True, False), ("per_tails", True, True)]:
    buf = d4pg.PrioritizedReplayBuffer(1000, 0.6, obs_dim=S, act_dim=A, nstep_tails=tails) if per else \
        d4pg.ReplayBuffer(1000, obs_dim=S, act_dim=A, nstep_tails=tails)
    for k in range(n + 1):
        buf.add_steps(*args(k == n), n_steps=n, gamma=0.9)      # the last one ends half the episodes
    a = args(False)
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        rows = buf.add_steps(*a, n_steps=n, gamma=0.9)
        torch.cuda.synchronize()
    ev = sorted((e for e in prof.events() if e.device_type == DeviceType.CUDA and not e.name.startswith("Memcpy")),
                key=lambda e: e.time_range.start)
    out[name] = dict(rows=rows, kernels=[e.name for e in ev])
print(json.dumps(out))
"""


def test_launch_counts():
    """A call that emits tail rows launches what a tails-off call launches: the insert kernel, and the tree add with
    PER; no memset."""
    import json
    import os
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, "-c", _LAUNCH_COUNT_SCRIPT], cwd=root, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    got = json.loads(r.stdout.strip().splitlines()[-1])
    assert got["plain"]["rows"] == 32 and got["plain_tails"]["rows"] == 32 + 32 * 2, got
    for name, names in {"plain": ["replay_add_steps"], "per": ["replay_add_steps", "tree_add_range_fast"]}.items():
        for g in (got[name], got[name + "_tails"]):
            ks = g["kernels"]
            assert len(ks) == len(names) and all(w + "_kernel" in k for k, w in zip(ks, names)), (name, ks)
