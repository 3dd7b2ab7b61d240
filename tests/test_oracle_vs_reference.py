"""oracle/ vs the unmodified reference, on inputs beyond the other fixtures.  What the reference computed on these
inputs is stored in tests/golden/reference_live.npz (tests/golden/make_golden.py `live`); large weight tensors are
pinned bit-for-bit by their SHA-256 digests."""
import hashlib
import random

import numpy as np
import torch

from oracle import d4pg_oracle as O
from tests import helpers as H

INFO = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}


def _digest(arr):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(arr).tobytes()).digest(), dtype=np.uint8)


def test_projection_random_vs_reproject2():
    g = H.load("reference_live.npz")
    rng = np.random.RandomState(5)
    for trial in range(6):
        B = 97
        p = torch.softmax(torch.from_numpy(rng.randn(B, 51).astype(np.float32) * 3), 1).numpy()
        r = (-60 * rng.rand(B)) if trial % 2 else -rng.randint(0, 3, B).astype(np.float64)
        done = np.zeros(B, bool) if trial < 4 else (rng.rand(B) < 0.3)
        if trial == 5:
            r = -40 * rng.rand(B)      # terminal rows all non-integer, unclamped (no H6 mix)
        m = O.project_live(p, r, done, -50.0, 0.0, 51, 0.99)
        assert np.array_equal(m, g["proj%d_m" % trial])


def test_h5_live_projection_ignores_n_steps():
    """SURVEY H5: reproject2 discounts with gamma, reproj_categorical_dist with gamma**n."""
    g = H.load("reference_live.npz")
    rng = np.random.RandomState(6)
    B = 32
    p = torch.softmax(torch.from_numpy(rng.randn(B, 51).astype(np.float32)), 1).numpy()
    r = -3 * rng.rand(B)
    done = np.zeros(B, bool)
    assert np.array_equal(g["h5_live_m"], O.project_live(p, r, done, -50.0, 0.0, 51, 0.99))
    m5 = g["h5_nstep_m"]
    assert np.array_equal(m5, O.project_nstep(p, r, done, -50.0, 0.0, 51, 0.99, 5))
    assert np.abs(m5 - g["h5_live_m"]).max() > 0.05


def test_five_train_steps_vs_live_reference():
    """The stored reference run used one torch thread: the oracle does too, so that its sums are ordered alike."""
    threads = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        _five_train_steps()
    finally:
        torch.set_num_threads(threads)


def _five_train_steps():
    g = H.load("reference_live.npz")
    B, mem = 48, 700
    rng = np.random.RandomState(22)
    buf = O.PrioritizedReplayOracle(mem, 0.6, 17, 6)
    for i in range(650):
        s = rng.randn(17).astype(np.float32)
        a = rng.uniform(-1, 1, 6).astype(np.float32)
        r = float(np.float32(-3 * rng.rand()))
        s2 = rng.randn(17).astype(np.float32)
        buf.add(s, a, r, s2, False)
    a0, c0 = H.regen_init(21, 17, 6, 51)
    for net, w in (("actor", a0), ("critic", c0)):
        for k, v in w.items():
            assert np.array_equal(_digest(v.numpy()), g["train_init_%s_%s" % (net, k)]), (net, k)
    lo = O.LearnerOracle(17, 6, INFO, actor_w={k: v.clone() for k, v in a0.items()},
                         critic_w={k: v.clone() for k, v in c0.items()})
    sched = O.LinearScheduleOracle(100000, 1.0, 0.4)
    for t in range(5):
        random.seed(300 + t)
        us = [random.random() for _ in range(B)]
        batch = buf.sample(B, sched.value(), us)
        out = lo.train_step(*batch[:5])
        buf.update_priorities(batch[6], out["prio"])
        assert np.array_equal(g["train_tree_sum_%d" % t], buf.sum.value.astype(np.float64))
        for name, mine in (("actor", lo.actor), ("critic", lo.critic), ("actor_target", lo.actor_target),
                           ("critic_target", lo.critic_target)):
            for k, v in mine.items():
                assert np.array_equal(_digest(v.numpy()), g["train_%s_%s_%d" % (name, k, t)]), (t, name, k)


def test_pristine_tree_sampling_is_f64_at_scale():
    """Before any update_priorities the reference tree holds Python floats: mass = u*sum and the
    descent run in f64.  Needs a buffer large enough that f32 rounding of the mass would matter."""
    g = H.load("reference_live.npz")
    size = 1 << 16
    ob = O.PrioritizedReplayOracle(size, 0.6, 1, 1)
    ob.add_batch(np.zeros((size - 3, 1), np.float32), np.zeros((size - 3, 1), np.float32), np.zeros(size - 3),
                 np.zeros((size - 3, 1), np.float32), np.zeros(size - 3, bool))
    random.seed(5)
    us = [random.random() for _ in range(2000)]
    idx_ref = [int(i) for i in g["pristine_idx"]]
    idx = ob.sample_indices(us)
    assert list(idx) == idx_ref
    f32_idx = [O.find_prefixsum_idx(ob.sum.value, ob.capacity, np.float32(np.float32(u) * ob.sum.reduce_prefix(ob.length - 2)))
               for u in us]
    assert f32_idx != idx_ref          # the f32 rule really is different at this size
