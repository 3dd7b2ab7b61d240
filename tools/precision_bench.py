#!/usr/bin/env python
"""precision_bench.py -- config 5 (n-step 5, 101 atoms, batch 4096) step time at precision tf32x3 vs bf16.

    python tools/precision_bench.py [--steps 300] [--regions 3] [--warmup 20]

Both learners live in one process and their timed regions alternate (tf32x3, bf16, tf32x3, ...), so clock and
co-tenant drift hit both alike.  A region is `--steps` device-sampled DDPG.train_n steps (CUDA-graph replays) between
CUDA events on the learner stream, after a warm-up that captures every graph variant.  Batch 4096 runs the level plan:
one grouped GEMM launch per dependency level, whose per-launch device times come from DDPG.profile_step() (CUDA events
around each launch).  The bf16 GEMM rate = the step's algorithmic MLP FLOPs (bench.algorithmic) / the summed level-GEMM
time, against the H100 SXM data sheet's 989 TFLOP/s dense BF16.  Prints one JSON line; GPU name, power limit and max
SM clock are read in the same run.  Needs a GPU: there is no CPU fallback.
"""
import argparse
import json
import os
import random
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from bench import CFG, algorithmic, synth  # noqa: E402

PEAK_BF16_TFLOPS = 989.0                      # H100 SXM data sheet, dense BF16 (700 W card)


def gpu_info(index):
    out = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm",
                          "--format=csv,noheader,nounits"], capture_output=True, text=True, timeout=30)
    f = [x.strip() for x in out.stdout.strip().split(",")]
    if out.returncode != 0 or len(f) < 3:
        return {"name": None, "power_limit_w": None, "max_sm_mhz": None, "error": out.stderr.strip()[:200]}
    return {"name": f[0], "power_limit_w": float(f[1]), "max_sm_mhz": float(f[2])}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--config", default="c5", choices=sorted(CFG))
    ap.add_argument("--steps", type=int, default=300, help="train_n steps per timed region (>= 300)")
    ap.add_argument("--regions", type=int, default=3, help="timed regions per precision (alternating)")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--profile-steps", type=int, default=5)
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        raise SystemExit("precision_bench.py needs a CUDA GPU (no CPU fallback)")
    import d4pg_b200 as d4pg
    dev = torch.cuda.current_device()
    cfg = CFG[args.config]
    info = {"type": "categorical", "v_min": cfg["v_min"], "v_max": cfg["v_max"], "n_atoms": cfg["atoms"]}
    B, cap = cfg["batch"], cfg["cap"]
    precisions = ("tf32x3", "bf16")

    def make(precision):
        torch.manual_seed(0); random.seed(0)
        dd = d4pg.DDPG(cfg["obs"], cfg["act"], memory_size=cap, batch_size=B, critic_dist_info=info,
                       n_steps=cfg["n_steps"], projection=cfg["proj"], sampling="device", philox_seed=1234,
                       precision=precision, chain="cluster")
        dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3),
                                   d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
        dd.replayBuffer.add_batch(*synth(cfg, cap, seed=0))
        for n in (1, 4, 1, 4, 1):                      # capture every graph variant before timing
            dd.train_n(n)
        dd.train_n(max(args.warmup, 3))
        torch.cuda.synchronize()
        return dd

    nets = {p: make(p) for p in precisions}
    regions = {p: [] for p in precisions}
    for _ in range(args.regions):
        for p in precisions:
            dd = nets[p]
            stream = dd._learner.stream
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            dd.train_n(args.steps)
            e1.record(stream)
            torch.cuda.synchronize()
            regions[p].append(e0.elapsed_time(e1) / args.steps)
    for p in precisions:
        lc, la = nets[p].last_losses()
        assert np.isfinite(lc) and np.isfinite(la), (p, lc, la)

    alg = algorithmic(cfg)
    gemm = {}
    for p in precisions:
        sums = []
        for _ in range(args.profile_steps):
            prof = nets[p].profile_step()
            sums.append(sum(ms for name, ms in prof if name == "gemm_launch"))
            launches = [round(ms * 1e3, 2) for name, ms in prof if name == "gemm_launch"]
        gemm[p] = {"level_gemm_ms_per_step": float(np.median(sums)), "level_gemm_launches": len(launches),
                   "last_profile_us_per_launch": launches}
    g = gemm["bf16"]["level_gemm_ms_per_step"]
    tflops = alg["flops"] / (g * 1e-3) / 1e12
    line = {"tool": "precision_bench", "config": args.config, "batch": B, "steps_per_region": args.steps,
            "regions": args.regions, "order": "alternating " + ", ".join(precisions),
            "ms_per_step": {p: float(np.median(regions[p])) for p in precisions},
            "regions_ms_per_step": {p: [round(x, 5) for x in regions[p]] for p in precisions},
            "level_gemm": gemm, "kernels_per_step": {p: nets[p].kernels_per_step() for p in precisions},
            "bf16_gemm": {"algorithmic_flops_per_step": alg["flops"], "achieved_tflops": tflops,
                          "peak_tflops": PEAK_BF16_TFLOPS, "peak_source": "H100 SXM data sheet, dense BF16",
                          "frac_of_peak": tflops / PEAK_BF16_TFLOPS},
            "gpu": gpu_info(dev)}
    print(json.dumps(line))


if __name__ == "__main__":
    main()
