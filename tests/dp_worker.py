"""torchrun worker for the multi-GPU data-parallel parity test (tests/test_gpu_multi.py).

Each rank: own replay shard + trees, B_local rows per step, ONE NCCL all-reduce of the flat gradient
inside the learner's CUDA graph.  Checks: (1) replicas stay bit-identical across ranks; (2) the
result equals ONE oracle learner trained on the concatenation of the ranks' batches (SURVEY 8e)."""
import os
import random
import sys

import numpy as np
import torch
import torch.distributed as dist

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import d4pg_b200 as d4pg                      # noqa: E402
from oracle import d4pg_oracle as O           # noqa: E402


def main():
    rank, world, local = int(os.environ["RANK"]), int(os.environ["WORLD_SIZE"]), int(os.environ["LOCAL_RANK"])
    torch.cuda.set_device(local)
    dist.init_process_group("nccl", device_id=torch.device("cuda", local))
    comm = d4pg.dist.Comm()
    precision = os.environ.get("D4PG_PRECISION", "fp32")
    info = {"type": "categorical", "v_min": -50.0, "v_max": 0.0, "n_atoms": 51}
    B, n = 64, 2048
    torch.manual_seed(0)                       # identical initial replicas
    dd = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=info, comm=comm, precision=precision)
    dd.assign_global_optimizer(d4pg.SharedAdam(dd.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dd.critic.parameters(), lr=1e-3))
    a0 = {k: v.cpu().clone() for k, v in dd.actor.state_dict().items()}
    c0 = {k: v.cpu().clone() for k, v in dd.critic.state_dict().items()}

    def shard(r):
        rng = np.random.RandomState(1000 + r)
        return (rng.randn(n, 17).astype(np.float32), rng.uniform(-1, 1, (n, 6)).astype(np.float32),
                (-3 * rng.rand(n)).astype(np.float32).astype(np.float64), rng.randn(n, 17).astype(np.float32),
                rng.rand(n) < 0.05)
    dd.replayBuffer.add_batch(*shard(rank))

    if os.environ.get("D4PG_DP_MODE") == "device":
        # the benchmark's configuration: device-side sampling, prefetch pipeline, 8-step graphs, gradient exchange fused
        # into the dW / Adam kernels.  Replicas must stay bit-identical through replays, adds and single steps.
        torch.manual_seed(0)
        dv = d4pg.DDPG(17, 6, memory_size=n, batch_size=B, critic_dist_info=info, comm=comm, precision=precision,
                       sampling="device", philox_seed=100 + rank)
        dv.assign_global_optimizer(d4pg.SharedAdam(dv.actor.parameters(), lr=1e-3), d4pg.SharedAdam(dv.critic.parameters(), lr=1e-3))
        dv.replayBuffer.add_batch(*shard(rank))
        for phase in range(3):
            dv.train_n(11)
            dv.train()
            dv.replayBuffer.add_batch(*[x[:37] for x in shard(rank + 10 * (phase + 1))])     # invalidates the prefetched batch
            dv.train()
            lc, la = dv.last_losses()
            assert np.isfinite(lc) and np.isfinite(la)
            flat = torch.cat([dv.actor.flat_params(), dv.critic.flat_params(), dv.actor_target.flat_params(),
                              dv.critic_target.flat_params()])
            ref = flat.clone()
            dist.broadcast(ref, src=0)
            assert torch.equal(flat, ref), "device-sampling replicas diverged in phase %d on rank %d" % (phase, rank)
        dist.barrier()
        if rank == 0:
            print("DP_OK world=%d precision=%s mode=device kernels/step=%d" % (world, precision, dv.kernels_per_step()))
        dist.destroy_process_group()
        return

    oracle_bufs, lo = None, None
    if rank == 0:
        oracle_bufs = []
        for r in range(world):
            ob = O.PrioritizedReplayOracle(n, 0.6, 17, 6)
            ob.add_batch(*shard(r))
            oracle_bufs.append(ob)
        lo = O.LearnerOracle(17, 6, info, actor_w=a0, critic_w=c0)
    steps = 3
    for t in range(steps):
        random.seed(500 + 10 * t + rank)       # each rank draws its own uniforms
        dd.train()
        idx = dd.last_batch_info()["idx"].clone()
        prio = dd.last_batch_info()["prio"].clone()
        lc, la = dd.last_losses()
        all_idx = [torch.zeros_like(idx) for _ in range(world)]
        all_prio = [torch.zeros_like(prio) for _ in range(world)]
        dist.all_gather(all_idx, idx)
        dist.all_gather(all_prio, prio)
        losses = torch.tensor([lc, la], dtype=torch.float64, device="cuda")
        dist.all_reduce(losses)
        flat = torch.cat([dd.actor.flat_params(), dd.critic.flat_params(), dd.actor_target.flat_params()])
        ref = flat.clone()
        dist.broadcast(ref, src=0)
        assert torch.equal(flat, ref), "replicas diverged at step %d on rank %d" % (t, rank)
        if rank == 0:
            batches = []
            for r in range(world):
                random.seed(500 + 10 * t + r)
                us = [random.random() for _ in range(B)]
                b = oracle_bufs[r].sample(B, 0.4, us)
                assert np.array_equal(b[6], all_idx[r].cpu().numpy()), "rank %d indices differ from its oracle shard" % r
                batches.append(b)
            cat = [np.concatenate([b[i] for b in batches]) for i in range(5)]
            out = lo.train_step(*cat)                                   # ONE learner, batch = world*B
            for r in range(world):                                     # priorities are shard-local
                p = out["prio"][r * B:(r + 1) * B]
                assert np.abs(p - all_prio[r].cpu().numpy()).max() <= 1e-5
                oracle_bufs[r].update_priorities(batches[r][6], all_prio[r].cpu().numpy())
            assert abs(losses[0].item() / world - float(out["loss_critic"])) <= 1e-5
            for net, grads in ((dd.actor, out["grads_actor"]), (dd.critic, out["grads_critic"])):      # the rank-order SUM of the shards' gradients
                for k in O.PARAM_ORDER:
                    gk = net.named_grad_views()[k].cpu()
                    assert (gk - grads[k]).abs().max().item() <= 1e-5, (t, k, (gk - grads[k]).abs().max().item())
            for k in O.PARAM_ORDER:
                for mine, refw in ((dd.actor.state_dict()[k], lo.actor[k]), (dd.critic.state_dict()[k], lo.critic[k])):
                    err = (mine.cpu() - refw).abs()
                    assert err.max().item() <= 2.5e-4 and (err > 1e-5).float().mean().item() <= 0.1, (t, k, err.max().item())
        # keep the GPU trees equal to the oracle's for the next step's index parity
        dist.barrier()
    if rank == 0:
        print("DP_OK world=%d precision=%s kernels/step=%d" % (world, precision, dd.kernels_per_step()))
    dist.destroy_process_group()


if __name__ == "__main__":
    main()
