#!/usr/bin/env python
"""autograd_bench.py -- forward + backward of the differentiable actor / critic modules against torch eager.

    python tools/autograd_bench.py [--iters 200] [--regions 5] [--warmup 20]

For configs c2 (batch 256) and c5 (batch 4096) and precisions 0 (fp32 FFMA), 1 (3xTF32 wgmma) and 3 (bf16 wgmma), one
iteration is `loss = (net(inputs) * g).sum(); loss.backward()` on `actor(..., differentiable=True)` and on
`critic(..., differentiable=True)` (parameters require grad, inputs do not; .grad views a flat buffer, as in training).
Beside them the same layers restated as an eager `F.linear` stack (cuBLAS): TF32 off for the fp32 rows, bf16 autocast
for the bf16 rows.  Each region times `--iters` iterations between CUDA events on the current stream; the variants'
regions alternate, and the median region is reported in microseconds per iteration.  GPU name, power limit and max SM
clock are read in the same run.  Prints one JSON line.  Needs a GPU: there is no CPU fallback.
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CFG  # noqa: E402


def gpu_info(index):
    out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    f = [x.strip() for x in out.stdout.strip().split(",")]
    if out.returncode != 0 or len(f) < 3:
        return {"name": None, "power_limit_w": None, "max_sm_mhz": None, "error": out.stderr.strip()[:200]}
    return {"name": f[0], "power_limit_w": float(f[1]), "max_sm_mhz": float(f[2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--configs", default="c2,c5")
    ap.add_argument("--iters", type=int, default=200, help="iterations per timed region")
    ap.add_argument("--regions", type=int, default=5)
    ap.add_argument("--warmup", type=int, default=20)
    args = ap.parse_args()
    import torch
    import torch.nn.functional as F
    if not torch.cuda.is_available():
        raise SystemExit("autograd_bench.py needs a CUDA GPU (no CPU fallback)")
    import d4pg_b200 as d4pg
    dev = torch.cuda.current_device()
    torch.backends.cuda.matmul.allow_tf32 = False

    def eager_actor(w, s):
        h = F.relu(F.linear(s, w["fc1.weight"], w["fc1.bias"]))
        h = F.linear(h, w["fc2.weight"], w["fc2.bias"])
        h = F.relu(F.linear(h, w["fc2_2.weight"], w["fc2_2.bias"]))
        return torch.tanh(F.linear(h, w["fc3.weight"], w["fc3.bias"]))

    def eager_critic(w, s, a):
        h = F.relu(F.linear(s, w["fc1.weight"], w["fc1.bias"]))
        h = F.relu(F.linear(torch.cat([h, a], 1), w["fc2.weight"], w["fc2.bias"]))
        h = F.relu(F.linear(h, w["fc2_2.weight"], w["fc2_2.bias"]))
        return F.softmax(F.linear(h, w["fc3.weight"], w["fc3.bias"]).float(), dim=1)

    results = {}
    for cname in args.configs.split(","):
        cfg = CFG[cname]
        S, A, N, B = cfg["obs"], cfg["act"], cfg["atoms"], cfg["batch"]
        info = {"type": "categorical", "v_min": cfg["v_min"], "v_max": cfg["v_max"], "n_atoms": N}
        torch.manual_seed(0)
        actor = d4pg.actor(S, A, device="cuda", differentiable=True)
        critic = d4pg.critic(S, A, info, device="cuda", differentiable=True)
        actor.flat_grads(); critic.flat_grads()
        wa = {k: v.detach().clone().requires_grad_(True) for k, v in actor.state_dict().items()}
        wc = {k: v.detach().clone().requires_grad_(True) for k, v in critic.state_dict().items()}
        s = torch.randn(B, S, device="cuda"); act = torch.rand(B, A, device="cuda") * 2 - 1
        ga = torch.randn(B, A, device="cuda"); gq = torch.randn(B, N, device="cuda")

        def ours(net, precision):
            def run():
                net.precision = precision
                out = net(s) if net is actor else net(s, act)
                (out * (ga if net is actor else gq)).sum().backward()
            return run

        def eager(which, bf16):
            def run():
                with torch.autocast("cuda", dtype=torch.bfloat16, enabled=bf16):
                    out = eager_actor(wa, s) if which == "actor" else eager_critic(wc, s, act)
                    loss = (out.float() * (ga if which == "actor" else gq)).sum()
                loss.backward()
            return run

        variants = {}
        for net_name, net in (("actor", actor), ("critic", critic)):
            for p in (0, 1, 3):
                variants["%s/precision%d" % (net_name, p)] = ours(net, p)
            variants["%s/eager_fp32" % net_name] = eager(net_name, False)
            variants["%s/eager_bf16_autocast" % net_name] = eager(net_name, True)
        for run in variants.values():
            for _ in range(args.warmup):
                run()
        torch.cuda.synchronize()
        regions = {k: [] for k in variants}
        for _ in range(args.regions):
            for k, run in variants.items():
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for _ in range(args.iters):
                    run()
                e1.record()
                torch.cuda.synchronize()
                regions[k].append(e0.elapsed_time(e1) * 1e3 / args.iters)
        results[cname] = {"shape": {"obs": S, "act": A, "atoms": N, "batch": B},
                          "us_per_fwd_bwd": {k: round(float(np.median(v)), 2) for k, v in regions.items()},
                          "regions_us": {k: [round(x, 2) for x in v] for k, v in regions.items()}}
    line = {"tool": "autograd_bench", "iters_per_region": args.iters, "regions": args.regions,
            "timing": "CUDA events around each region on the current stream, host launch overhead included",
            "results": results, "gpu": gpu_info(dev)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
