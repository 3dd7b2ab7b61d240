"""Data-parallel plumbing: one process per GPU, torch.distributed for rendezvous, ONE NCCL
all-reduce of the flat gradient buffer per learner step (inside the CUDA graph).

The reference has no collective (its multi-worker mode is Hogwild over shared CPU memory,
main.py:394-405); this is the synchronous-DP layout of SURVEY.md section 8e: replay storage and
trees are sharded by rank (each rank owns its own ring / trees / max_priority), every rank
samples B_local rows from its shard, gradients are summed over ranks with 1/(B_local*world)
folded into the loss-gradient kernel, and the identical fused Adam runs on every rank so the
replicas stay bit-identical.
"""
import ctypes as C
import os

import torch


def shard_range(n, rank, world):
    """Contiguous [lo, hi) slice of n items owned by `rank` (sizes differ by at most 1)."""
    base, rem = divmod(n, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def env_rank_world():
    return int(os.environ.get("RANK", "0")), int(os.environ.get("WORLD_SIZE", "1")), int(os.environ.get("LOCAL_RANK", "0"))


def broadcast_bytes(payload, nbytes, src=0, device="cpu"):
    """Broadcast a fixed-size byte string from `src` over the default process group
    (works on gloo with CPU tensors and on NCCL with CUDA tensors)."""
    import torch.distributed as dist
    t = torch.zeros(nbytes, dtype=torch.uint8, device=device)
    if dist.get_rank() == src:
        t.copy_(torch.tensor(list(payload), dtype=torch.uint8))
    dist.broadcast(t, src=src)
    return bytes(t.cpu().tolist())


class Comm(object):
    """NCCL communicator owned by libd4pg_sm90.so (d4pg_comm_*), bootstrapped through the
    torch.distributed default group."""

    def __init__(self, rank=None, world_size=None, device=None):
        import torch.distributed as dist
        from . import _lib
        _lib.require_cuda()
        self.rank = dist.get_rank() if rank is None else rank
        self.world_size = dist.get_world_size() if world_size is None else world_size
        uid = (C.c_uint8 * 128)()
        if self.rank == 0:
            _lib.check(_lib.lib().d4pg_comm_unique_id(uid), "d4pg_comm_unique_id")
        dev = device if device is not None else ("cuda" if dist.get_backend() == "nccl" else "cpu")
        raw = broadcast_bytes(bytes(uid), 128, src=0, device=dev)
        uid2 = (C.c_uint8 * 128).from_buffer_copy(raw)
        h = C.c_void_p()
        _lib.check(_lib.lib().d4pg_comm_create(uid2, self.rank, self.world_size, C.byref(h)), "d4pg_comm_create")
        self.handle = h

    def setup_peers(self, n_floats):
        """Fused all-reduce over peer memory (one node): allocate this rank's exchange block, gather the CUDA IPC
        handles of all ranks, map them.  Collective (every rank must call it); falls back to the NCCL all-reduce --
        on every rank -- if any rank cannot export or map (D4PG_COMM_PEER=0 disables it)."""
        import torch.distributed as dist
        from . import _lib
        L = _lib.lib()
        if self.world_size <= 1 or self.world_size > 8 or L.d4pg_comm_peer_ready(self.handle):
            return bool(L.d4pg_comm_peer_ready(self.handle))
        dev = "cuda" if dist.get_backend() == "nccl" else "cpu"
        ok = os.environ.get("D4PG_COMM_PEER", "1") != "0"
        mine = (C.c_uint8 * 64)()
        if ok and L.d4pg_comm_peer_alloc(self.handle, int(n_floats), mine) != 0:
            ok = False
        flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:
            return False
        t = torch.tensor(list(bytes(mine)), dtype=torch.uint8, device=dev)
        parts = [torch.zeros(64, dtype=torch.uint8, device=dev) for _ in range(self.world_size)]
        dist.all_gather(parts, t)
        blob = b"".join(bytes(p.cpu().tolist()) for p in parts)
        arr = (C.c_uint8 * len(blob)).from_buffer_copy(blob)
        ok = L.d4pg_comm_peer_open(self.handle, arr) == 0
        flag = torch.tensor([1 if ok else 0], dtype=torch.int32, device=dev)
        dist.all_reduce(flag, op=dist.ReduceOp.MIN)
        if int(flag.item()) == 0:                  # e.g. no CUDA IPC between the ranks' containers: NCCL path on every rank
            L.d4pg_comm_peer_disable(self.handle)
            return False
        self.multicast = bool(self.setup_multicast())
        return True

    def exchange_mode(self):
        """How the learner sums the gradient over the ranks: "nccl" (all-reduce fallback), or over peer memory "mc"
        (in-switch reduction, multimem.ld_reduce; "mc2" = its two-phase form: reduce 1/N, multimem.st broadcast), "pull" (every rank sums all halves) / "rs" (reduce-scatter + all-gather)."""
        from . import _lib
        L = _lib.lib()
        if self.world_size <= 1:
            return "single"
        if not L.d4pg_comm_peer_ready(self.handle):
            return "nccl"
        env = os.environ.get("D4PG_COMM_MODE", "")
        if L.d4pg_comm_mc_ready(self.handle) and env[:1] in ("", "m"):       # same selection as learner.cu
            if env[:3] == "mc2" or (env == "" and self.world_size >= int(os.environ.get("D4PG_COMM_MC2_FROM", "1000"))):
                return "mc2"
            if env[:1] == "m" or self.world_size >= int(os.environ.get("D4PG_COMM_MC_FROM", "3")):
                return "mc"
        return "rs" if env[:1] == "r" else "pull"

    def setup_multicast(self):
        """In-switch reduction (NVLS): one multicast object over every rank's gradient buffer, so that the fused Adam
        kernel reads the sum over all ranks with `multimem.ld_reduce` (one NVLink hop, the NVSwitch adds).  Collective;
        every failure mode (no NVSwitch multicast support, descriptor passing refused, sums not bit-identical across
        ranks) leaves every rank on the peer-memory pull.  D4PG_COMM_MC=0 skips it."""
        import socket
        import torch.distributed as dist
        from . import _lib
        L = _lib.lib()
        dev = "cuda" if dist.get_backend() == "nccl" else "cpu"

        def all_ok(ok):
            t = torch.tensor([1 if ok else 0], dtype=torch.int32, device=dev)
            dist.all_reduce(t, op=dist.ReduceOp.MIN)
            return int(t.item()) == 1
        if not all_ok(os.environ.get("D4PG_COMM_MC", "1") != "0" and L.d4pg_comm_mc_supported(self.handle) == 1):
            return False
        # rank 0 creates + exports the object; the file descriptor travels over an abstract-namespace Unix socket
        name = "\0d4pg_mc_%s_%s" % (os.environ.get("MASTER_PORT", "0"), os.environ.get("TORCHELASTIC_RUN_ID", "0"))
        ok, srv, fd = True, None, C.c_int32(-1)
        if self.rank == 0:
            ok = L.d4pg_comm_mc_create(self.handle, C.byref(fd)) == 0
            if ok:
                try:
                    srv = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
                    srv.bind(name)
                    srv.listen(self.world_size)
                except OSError:
                    ok = False
        if not all_ok(ok):                         # (also the rendezvous: the socket is listening from here on)
            if srv is not None:
                srv.close()
            return False
        try:
            if self.rank == 0:
                srv.settimeout(60)
                for _ in range(self.world_size - 1):
                    conn, _ = srv.accept()
                    socket.send_fds(conn, [b"x"], [fd.value])
                    conn.close()
                srv.close()
                os.close(fd.value)
            else:
                cli = socket.socket(socket.AF_UNIX, socket.SOCK_STREAM)
                cli.settimeout(60)
                cli.connect(name)
                _, fds, _, _ = socket.recv_fds(cli, 16, 1)
                cli.close()
                ok = len(fds) == 1 and L.d4pg_comm_mc_import(self.handle, fds[0]) == 0
        except OSError:
            ok = False
        if not all_ok(ok):
            return False
        if not all_ok(L.d4pg_comm_mc_add_device(self.handle) == 0):      # everyone joined the team ...
            return False
        if not all_ok(L.d4pg_comm_mc_bind(self.handle) == 0):            # ... before anyone binds memory
            L.d4pg_comm_mc_disable(self.handle)
            return False
        # self-test: every rank must read the SAME bits (replicas have to stay identical) and the right sum
        n = 4096
        g = torch.Generator(device="cpu").manual_seed(1234 + self.rank)
        mine = torch.randn(n, generator=g).cuda()
        out = torch.empty(n, dtype=torch.float32, device="cuda")
        ok = L.d4pg_comm_mc_selftest(self.handle, _lib.ptr(mine), None, n, _lib.stream_ptr()) == 0
        torch.cuda.synchronize()
        dist.barrier()
        ok = ok and L.d4pg_comm_mc_selftest(self.handle, None, _lib.ptr(out), n, _lib.stream_ptr()) == 0
        torch.cuda.synchronize()
        if ok:
            parts = [torch.empty_like(out) for _ in range(self.world_size)]
            dist.all_gather(parts, out)
            vals = [torch.empty_like(mine) for _ in range(self.world_size)]
            dist.all_gather(vals, mine)
            want = torch.stack(vals).double().sum(0)
            ok = all(torch.equal(parts[0], p) for p in parts) and float((out.double() - want).abs().max()) < 1e-4
        if not all_ok(ok):
            L.d4pg_comm_mc_disable(self.handle)
            return False
        return True

    def allreduce_sum_(self, flat):
        from . import _lib
        _lib.check(_lib.lib().d4pg_comm_allreduce_sum(self.handle, _lib.ptr(flat), flat.numel(), _lib.stream_ptr()),
                   "d4pg_comm_allreduce_sum")
        return flat

    def close(self):
        from . import _lib
        if self.handle is not None:
            _lib.lib().d4pg_comm_destroy(self.handle)
            self.handle = None
