#!/usr/bin/env python
"""nstep_stream_bench.py -- what storing one vector step of E environments with n-step returns (n = 5) costs.

    python tools/nstep_stream_bench.py [--es 1,64,1024,4096] [--iters 100] [--regions 5] [--profile]

Three ways, each into its own PrioritizedReplayBuffer, for the c2 (|s|=17, |a|=6) and c3 (|s|=376, |a|=17) shapes, with
host (numpy) and with device (CUDA tensor) inputs:
  host_deques  per-environment deques in Python form the rows (replay_memory.py:21-59 for E environments), add_batch
  torch_eager  the windows as CUDA tensors restated with torch index ops (a nonzero() per step), add_batch
  add_steps    ReplayBuffer.add_steps: the windows and the row forming in one sm_90a launch (+ the tree add)
Timed regions of --iters calls alternate between the three; each region's wall time runs to a synchronise and its device
time is the span between CUDA events recorded around it.  Prints the median per call with the spread of the regions
((max - min) / median), and one JSON line with the GPU name and power limit.  --profile instead runs each variant under
torch.profiler (a separate run) and reports the CUDA kernel time per call.  Needs a GPU.
"""
import argparse
import collections
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from mog_bench import gpu_info    # noqa: E402

SHAPES = {"c2": (17, 6), "c3": (376, 17)}
N, GAMMA, POOL, SIZE = 5, 0.99, 8, 1 << 18


def make_pool(rng, E, S, A, device):
    """POOL vector steps of data, cycled through: (s, a, r, s2, terminated, truncated)."""
    out = []
    for _ in range(POOL):
        c = (rng.randn(E, S).astype(np.float32), rng.uniform(-1, 1, (E, A)).astype(np.float32), rng.randn(E),
             rng.randn(E, S).astype(np.float32), rng.rand(E) < 0.01, rng.rand(E) < 0.005)
        out.append(tuple(torch.as_tensor(x).cuda() for x in c) if device else c)
    return out


class HostDeques(object):
    def __init__(self, buf, E):
        self.buf, self.q = buf, [collections.deque(maxlen=N) for _ in range(E)]

    def __call__(self, s, a, r, s2, term, trunc):
        if torch.is_tensor(s):
            s, a, r, s2, term, trunc = (x.cpu().numpy() for x in (s, a, r, s2, term, trunc))
        rows = []
        for e, q in enumerate(self.q):
            q.append((s[e], a[e], float(r[e])))
            if len(q) == N:
                cum, eg = 0.0, 1.0
                for _, _, rk in q:
                    cum += eg * rk
                    eg *= GAMMA
                rows.append((q[0][0], q[0][1], cum, s2[e], term[e]))
            if term[e] or trunc[e]:
                q.clear()
        if rows:
            self.buf.add_batch(*[np.stack([row[i] for row in rows]) for i in range(5)])


class TorchEager(object):
    def __init__(self, buf, E, S, A):
        dev = "cuda"
        self.buf, self.E = buf, E
        self.ws = torch.zeros(E, N, S, device=dev)
        self.wa = torch.zeros(E, N, A, device=dev)
        self.wr = torch.zeros(E, N, dtype=torch.float64, device=dev)
        self.fill = torch.zeros(E, dtype=torch.int64, device=dev)
        self.ar = torch.arange(E, device=dev)

    def __call__(self, s, a, r, s2, term, trunc):
        s, a, r, s2, term, trunc = (torch.as_tensor(x).cuda() for x in (s, a, r, s2, term, trunc))
        slot = self.fill % N
        self.ws[self.ar, slot] = s
        self.wa[self.ar, slot] = a
        self.wr[self.ar, slot] = r.double()
        idx = (self.fill >= N - 1).nonzero().squeeze(1)
        if idx.numel():
            old = (self.fill[idx] + 1) % N
            cum = torch.zeros(idx.numel(), dtype=torch.float64, device="cuda")
            eg = 1.0
            for k in range(N):
                cum = cum + eg * self.wr[idx, (old + k) % N]
                eg *= GAMMA
            self.buf.add_batch(self.ws[idx, old], self.wa[idx, old], cum, s2[idx], term[idx])
        self.fill = torch.where(term | trunc, torch.zeros_like(self.fill), torch.clamp(self.fill + 1, max=N - 1))


class AddSteps(object):
    def __init__(self, buf):
        self.buf = buf

    def __call__(self, s, a, r, s2, term, trunc):
        self.buf.add_steps(s, a, r, s2, term, trunc, n_steps=N, gamma=GAMMA)


def region(fn, pool, iters):
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    e0.record()
    for i in range(iters):
        fn(*pool[i % POOL])
    e1.record()
    torch.cuda.synchronize()
    return 1e6 * (time.perf_counter() - t0) / iters, 1000.0 * e0.elapsed_time(e1) / iters


def kernel_us(fn, pool, iters):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(iters):
            fn(*pool[i % POOL])
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    kern = sum(e.time_range.elapsed_us() for e in ev if not e.name.startswith(("Memcpy", "Memset")))
    copy = sum(e.time_range.elapsed_us() for e in ev if e.name.startswith(("Memcpy", "Memset")))
    return kern / iters, copy / iters


def main():
    global torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--es", default="1,64,1024,4096")
    ap.add_argument("--iters", type=int, default=100, help="calls per timed region")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--profile", action="store_true", help="kernel time per call under torch.profiler instead")
    args = ap.parse_args()
    import torch
    import d4pg_b200 as d4pg
    d4pg._lib.require_cuda()
    result = {"gpu": gpu_info(torch.cuda.current_device()), "n_steps": N, "iters": args.iters, "regions": args.regions,
              "mode": "profile" if args.profile else "timing"}
    rng = np.random.RandomState(0)
    for name, (S, A) in SHAPES.items():
        for E in [int(e) for e in args.es.split(",")]:
            for inputs in ("host", "device"):
                pool = make_pool(rng, E, S, A, inputs == "device")
                mk = lambda: d4pg.PrioritizedReplayBuffer(SIZE, 0.6, obs_dim=S, act_dim=A)
                variants = {"host_deques": HostDeques(mk(), E), "torch_eager": TorchEager(mk(), E, S, A),
                            "add_steps": AddSteps(mk())}
                for fn in variants.values():
                    region(fn, pool, max(2 * N, args.iters // 5))           # warm-up: windows full, buffers, modules
                key = "%s_E%d_%s" % (name, E, inputs)
                if args.profile:
                    res = {k: kernel_us(fn, pool, args.iters) for k, fn in variants.items()}
                    result[key] = {k: {"kernel_us": v[0], "copy_us": v[1]} for k, v in res.items()}
                    print("%s  kernel us/call: %s" % (key, "  ".join("%s %.1f (+copies %.1f)" % (k, v[0], v[1])
                                                                      for k, v in res.items())))
                    continue
                wall, devt = {k: [] for k in variants}, {k: [] for k in variants}
                for _ in range(args.regions):
                    for k, fn in variants.items():
                        w, d = region(fn, pool, args.iters)
                        wall[k].append(w)
                        devt[k].append(d)
                med = {k: float(np.median(v)) for k, v in wall.items()}
                dmed = {k: float(np.median(v)) for k, v in devt.items()}
                spread = {k: (max(v) - min(v)) / med[k] for k, v in wall.items()}
                result[key] = {"wall_us": med, "event_us": dmed, "wall_spread": spread, "wall_regions_us": wall}
                print("%s  wall us/call: %s" % (key, "  ".join("%s %.1f (+-%.0f%%, events %.1f)" % (k, med[k], 50 * spread[k],
                                                                                                  dmed[k]) for k in variants)))
    print(json.dumps(result))


if __name__ == "__main__":
    main()
