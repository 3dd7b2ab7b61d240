#!/usr/bin/env python
"""her_stream_bench.py -- what storing goal-conditioned vector steps of E environments with hindsight relabelling costs,
at Fetch shapes (obs 25, goal 3, action 4, 50-step episodes, her_ratio 0.8, threshold 0.05).

    python tools/her_stream_bench.py [--es 1,64,1024,4096] [--regions 5] [--profile]

Three ways, each into its own PrioritizedReplayBuffer, with host (numpy) and with device (CUDA tensor) inputs, and
with every episode ending at the same call ("simultaneous") or environment e ending at call e % 50 ("staggered"):
  host_idiom     per-environment Python episode lists; each ended episode goes through add_her_episode (draws in a
                 Python loop, ten uploads, one relabel launch, one add) -- main.py:137-184 for E environments
  torch_eager    the episode windows as CUDA tensors, restated with torch index ops; the draws from the same generator
                 as add_goal_steps, the rows built with torch ops and stored with add_batch (a timing restatement:
                 its rewards use torch.linalg.vector_norm and are not checked bit for bit)
  add_goal_steps ReplayBuffer.add_goal_steps: the windows and the relabelled rows in one sm_90a launch (+ the tree add)
A timed region is one 50-call cycle, so every environment ends one episode in it; regions alternate between the three
and each runs to a synchronise.  Prints the median per call with the spread of the regions ((max - min) / median), and
one JSON line with the GPU name and power limit.  --profile instead runs each variant under torch.profiler (a separate
run) and reports the CUDA kernel time per call.  Needs a GPU.
"""
import argparse
import json
import os
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tools"))
from mog_bench import gpu_info    # noqa: E402

So, G, A, M = 25, 3, 4, 50
RATIO, THR = 0.8, 0.05
SIZE = 1 << 19


def make_cycle(rng, E, device, staggered):
    """M vector steps (obs, goal, act, rew, obs_next, ag_next, terminated, truncated): one episode end per environment."""
    out = []
    for k in range(M):
        end = (np.arange(E) % M == k) if staggered else np.full(E, k == M - 1)
        c = (rng.randn(E, So).astype(np.float32), rng.randn(E, G), rng.uniform(-1, 1, (E, A)).astype(np.float32),
             -rng.randint(0, 2, E).astype(np.float64), rng.randn(E, So).astype(np.float32), rng.randn(E, G) * 0.05,
             end & (rng.rand(E) < 0.3), end)
        out.append(tuple(torch.as_tensor(x).cuda() for x in c) if device else c)
    return out


class HostIdiom(object):
    def __init__(self, buf, E):
        self.buf, self.ep = buf, [[] for _ in range(E)]

    def __call__(self, obs, goal, act, rew, obs2, ag2, term, trunc):
        if torch.is_tensor(obs):
            obs, goal, act, rew, obs2, ag2, term, trunc = (x.cpu().numpy() for x in (obs, goal, act, rew, obs2, ag2, term,
                                                                                      trunc))
        for e, ep in enumerate(self.ep):
            ep.append((obs[e], obs2[e], goal[e], ag2[e], act[e], rew[e], term[e]))
            if term[e] or trunc[e]:
                cols = [np.stack([s[i] for s in ep]) for i in range(7)]
                self.buf.add_her_episode(*cols, her_ratio=RATIO, threshold=THR)
                ep.clear()


class TorchEager(object):
    def __init__(self, buf, E):
        dev, f64 = "cuda", torch.float64
        self.buf, self.E = buf, E
        self.w = dict(obs=torch.zeros(E, M, So, device=dev), goal=torch.zeros(E, M, G, dtype=f64, device=dev),
                      act=torch.zeros(E, M, A, device=dev), rew=torch.zeros(E, M, dtype=f64, device=dev),
                      obs2=torch.zeros(E, M, So, device=dev), ag=torch.zeros(E, M, G, dtype=f64, device=dev),
                      term=torch.zeros(E, M, dtype=torch.bool, device=dev))
        self.fill = np.zeros(E, np.int64)
        self.ended = np.zeros(E, np.int64)
        self.rng = np.random.default_rng(0)
        self.ar = torch.arange(E, device=dev)

    def _emit(self):
        em = np.flatnonzero(self.ended)
        if not em.size:
            return
        L = self.ended[em]
        n = int(L.sum())
        starts = np.repeat(np.cumsum(L) - L, L)
        t = np.arange(n) - starts
        sel = self.rng.random(n) < RATIO
        fut = t.copy()
        if sel.any():
            fut[sel] = self.rng.integers(t[sel], np.repeat(L, L)[sel])
        counts = 1 + sel
        dst = np.cumsum(counts) - counts
        up = lambda x: torch.as_tensor(x).cuda()
        ee, tt, ff, ll, d0, s1 = up(np.repeat(em, L)), up(t), up(fut[sel]), up(np.repeat(L, L)[sel] - 1), up(dst), up(sel)
        m = int(counts.sum())
        w = self.w
        s = torch.empty(m, So + G, device="cuda")
        s2 = torch.empty(m, So + G, device="cuda")
        a = torch.empty(m, A, device="cuda")
        r = torch.empty(m, dtype=torch.float64, device="cuda")
        d = torch.empty(m, dtype=torch.bool, device="cuda")
        o, o2, g = w["obs"][ee, tt], w["obs2"][ee, tt], w["goal"][ee, tt].float()
        s[d0] = torch.cat([o, g], 1)
        s2[d0] = torch.cat([o2, g], 1)
        a[d0], r[d0], d[d0] = w["act"][ee, tt], w["rew"][ee, tt], w["term"][ee, tt]
        c = d0[s1] + 1
        es, ts = ee[s1], tt[s1]
        gp = w["ag"][es, ff]
        s[c] = torch.cat([o[s1], gp.float()], 1)
        s2[c] = torch.cat([o2[s1], gp.float()], 1)
        a[c] = w["act"][es, ll]
        rc = -(torch.linalg.vector_norm(w["ag"][es, ts] - gp, dim=1) > THR).double()
        r[c], d[c] = rc, rc == 0
        self.buf.add_batch(s, a, r, s2, d)
        self.ended[:] = 0

    def __call__(self, obs, goal, act, rew, obs2, ag2, term, trunc):
        obs, goal, act, rew, obs2, ag2, term, trunc = (torch.as_tensor(x).cuda() for x in (obs, goal, act, rew, obs2, ag2,
                                                                                            term, trunc))
        self._emit()
        slot = torch.as_tensor(self.fill).cuda()
        w = self.w
        for k, x in (("obs", obs), ("goal", goal), ("act", act), ("rew", rew), ("obs2", obs2), ("ag", ag2), ("term", term)):
            w[k][self.ar, slot] = x
        self.fill += 1
        end = (term | trunc).cpu().numpy()
        self.ended[end] = self.fill[end]
        self.fill[end] = 0


class AddGoalSteps(object):
    def __init__(self, buf):
        self.buf = buf

    def __call__(self, *c):
        self.buf.add_goal_steps(*c, her_ratio=RATIO, threshold=THR, max_episode_steps=M)


def region(fn, cycle):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    for c in cycle:
        fn(*c)
    torch.cuda.synchronize()
    return 1e6 * (time.perf_counter() - t0) / len(cycle)


def kernel_us(fn, cycle):
    from torch.autograd import DeviceType
    from torch.profiler import ProfilerActivity, profile
    torch.cuda.synchronize()
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for c in cycle:
            fn(*c)
        torch.cuda.synchronize()
    ev = [e for e in prof.events() if e.device_type == DeviceType.CUDA]
    kern = sum(e.time_range.elapsed_us() for e in ev if not e.name.startswith(("Memcpy", "Memset")))
    copy = sum(e.time_range.elapsed_us() for e in ev if e.name.startswith(("Memcpy", "Memset")))
    goal = sum(e.time_range.elapsed_us() for e in ev if "replay_add_goal_steps" in e.name)
    return kern / len(cycle), copy / len(cycle), goal / len(cycle)


def main():
    global torch
    ap = argparse.ArgumentParser()
    ap.add_argument("--es", default="1,64,1024,4096")
    ap.add_argument("--regions", type=int, default=5, help="timed 50-call cycles per variant")
    ap.add_argument("--profile", action="store_true", help="kernel time per call under torch.profiler instead")
    args = ap.parse_args()
    import torch
    import d4pg_b200 as d4pg
    d4pg._lib.require_cuda()
    result = {"gpu": gpu_info(torch.cuda.current_device()), "shape": [So, G, A, M], "regions": args.regions,
              "mode": "profile" if args.profile else "timing"}
    rng = np.random.RandomState(0)
    for E in [int(e) for e in args.es.split(",")]:
        for inputs in ("host", "device"):
            for ends in ("simultaneous", "staggered"):
                cycle = make_cycle(rng, E, inputs == "device", ends == "staggered")
                mk = lambda: d4pg.PrioritizedReplayBuffer(SIZE, 0.6, obs_dim=So + G, act_dim=A)
                variants = {"host_idiom": HostIdiom(mk(), E), "torch_eager": TorchEager(mk(), E),
                            "add_goal_steps": AddGoalSteps(mk())}
                for fn in variants.values():
                    region(fn, cycle)                          # warm-up: windows full, buffers, modules
                key = "E%d_%s_%s" % (E, inputs, ends)
                if args.profile:
                    res = {k: kernel_us(fn, cycle) for k, fn in variants.items()}
                    result[key] = {k: {"kernel_us": v[0], "copy_us": v[1], "goal_kernel_us": v[2]} for k, v in res.items()}
                    print("%s  kernel us/call: %s" % (key, "  ".join("%s %.1f (+copies %.1f)" % (k, v[0], v[1])
                                                                      for k, v in res.items())), flush=True)
                    continue
                wall = {k: [] for k in variants}
                for _ in range(args.regions):
                    for k, fn in variants.items():
                        wall[k].append(region(fn, cycle))
                med = {k: float(np.median(v)) for k, v in wall.items()}
                spread = {k: (max(v) - min(v)) / med[k] for k, v in wall.items()}
                result[key] = {"wall_us": med, "wall_spread": spread, "wall_regions_us": wall}
                print("%s  wall us/call: %s" % (key, "  ".join("%s %.1f (+-%.0f%%)" % (k, med[k], 50 * spread[k])
                                                                for k in variants)), flush=True)
    print(json.dumps(result))


if __name__ == "__main__":
    main()
