"""Row sharding of a batch of independent queries over the GPUs of one box.

Evidence rows are independent (each is one `BayesNet.query` call in the reference,
/root/reference/sorobn/bayes_net.py:796), so the hot path has no data-path collective:
rank r answers a contiguous slice of the rows on its own GPU.  The only exchange is the
final gather of the posteriors on the destination rank (NCCL on GPUs; the CPU tests run
the same code over gloo with world_size 2).
"""
from __future__ import annotations

import numpy as np

__all__ = ["row_shard", "gather_rows", "run_sharded", "ShardedProgram", "query_many_sharded"]


def row_shard(n_rows: int, rank: int, world: int) -> slice:
    """Contiguous, balanced slice of `n_rows` for `rank` (sizes differ by at most one;
    ranks beyond n_rows get empty slices)."""
    if world < 1 or not 0 <= rank < world:
        raise ValueError(f"bad rank {rank} / world {world}")
    base, extra = divmod(int(n_rows), world)
    lo = rank * base + min(rank, extra)
    return slice(lo, lo + base + (1 if rank < extra else 0))


def gather_rows(local, n_rows: int, group=None, dst: int = 0, device=None):
    """Gather per-rank posteriors [Q, n_local] (row slices in rank order) into
    [Q, n_rows] on `dst` (a global rank, which must belong to `group`); other ranks get None.  `local` is a numpy array or a torch
    tensor; the collective runs on whatever backend `group` uses."""
    import torch
    import torch.distributed as dist

    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    t = torch.as_tensor(local)
    if device is not None:
        t = t.to(device)
    Q = t.shape[0]
    widest = row_shard(n_rows, 0, world)
    width = widest.stop - widest.start
    padded = torch.zeros((Q, width), dtype=t.dtype, device=t.device)
    padded[:, : t.shape[1]] = t
    # `dst` is a GLOBAL rank (what dist.gather takes); inside a sub-group the group-local rank differs
    is_dst = dist.get_rank() == dst
    bufs = [torch.empty_like(padded) for _ in range(world)] if is_dst else None
    dist.gather(padded, bufs, dst=dst, group=group)
    if not is_dst:
        return None
    parts = []
    for r in range(world):
        sl = row_shard(n_rows, r, world)
        parts.append(bufs[r][:, : sl.stop - sl.start])
    return torch.cat(parts, dim=1)


def run_sharded(codes: np.ndarray, n_rows: int, run_fn, group=None, dst: int = 0, device=None):
    """Answer `n_rows` queries across the ranks of `group`.

    codes  : uint8 [n_ev, n_rows] evidence codes, identical on every rank (each rank only
             reads its slice).
    run_fn : (codes_slice [n_ev, n_local], n_local) -> posterior [Q, n_local]; in
             production `engine.Program.run` / `run_device`, in the CPU tests a stand-in.
    Returns [Q, n_rows] on `dst`, None elsewhere.
    """
    import torch.distributed as dist

    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    sl = row_shard(n_rows, rank, world)
    n_local = sl.stop - sl.start
    local_codes = np.ascontiguousarray(codes[:, sl])
    if n_local > 0:
        local = run_fn(local_codes, n_local)
    else:
        local = None
    # every rank needs Q to build its (possibly empty) contribution
    import torch

    q = torch.tensor([0 if local is None else int(local.shape[0])], dtype=torch.int64,
                     device=device if device is not None else "cpu")
    dist.all_reduce(q, op=dist.ReduceOp.MAX, group=group)
    Q = int(q.item())
    if local is None:
        local = np.zeros((Q, 0), dtype=np.float32)
    return gather_rows(local, n_rows, group=group, dst=dst, device=device)


class ShardedProgram:
    """One device program per rank of a torch.distributed group (torchrun: one process per GPU).

    Every rank answers ITS evidence rows; the posteriors are gathered on `dst`.  With an NCCL
    group the data path stays on the device -- H2D of the rank's codes, `Program.run_device`,
    NCCL gather of the [Q, rows] blocks, one D2H on `dst` -- with a gloo group (CPU tests) the
    host path `Program.run` is used and CPU tensors are gathered.  This is what
    `query_many_sharded` and `bench.py --gpus N` run.

    program  : engine.Program (or any object with run(codes, n) -> [Q, n]; run_device for NCCL)
    rows_max : the largest per-rank batch; every rank passes the same value (buffers and the
               gather are sized by it, ragged tails are padded)
    """

    def __init__(self, program, Q: int, n_ev: int, rows_max: int, group=None, dst: int = 0, device=None):
        import torch
        import torch.distributed as dist

        self.program, self.Q, self.n_ev, self.rows_max = program, int(Q), int(n_ev), int(rows_max)
        self.group, self.dst = group, int(dst)
        self.world = dist.get_world_size(group)
        self.is_dst = dist.get_rank() == self.dst
        self.on_device = device is not None and str(device).startswith("cuda")
        self.device = torch.device(device) if device is not None else torch.device("cpu")
        self.d_ev = torch.zeros((max(self.n_ev, 1), self.rows_max), dtype=torch.uint8, device=self.device)
        self.d_out = torch.zeros((self.Q, self.rows_max), dtype=torch.float32, device=self.device)
        self.gathered = (torch.empty((self.world, self.Q, self.rows_max), dtype=torch.float32, device=self.device)
                         if self.is_dst else None)
        self.host = None
        if self.is_dst:
            self.host = torch.empty((self.world, self.Q, self.rows_max), dtype=torch.float32,
                                    pin_memory=self.on_device)

    def upload(self, codes):
        """Host codes uint8 [n_ev, n_local] (ideally pinned) -> this rank's device buffer."""
        import torch

        n = codes.shape[1] if self.n_ev else 0
        if self.n_ev:
            self.d_ev[: self.n_ev, :n].copy_(torch.from_numpy(codes), non_blocking=True)
        return n

    def run_resident(self, n_local: int):
        """Codes already in `d_ev`: run this rank's rows and gather the posteriors on `dst`
        (device-resident result `gathered[world, Q, rows_max]`; rows >= a rank's count are padding)."""
        import torch
        import torch.distributed as dist

        if self.on_device:
            stream = torch.cuda.current_stream(self.device).cuda_stream
            if n_local > 0:
                self.program.run_device(self.d_ev.data_ptr(), self.rows_max, n_local, self.d_out.data_ptr(),
                                        self.rows_max, stream)
        elif n_local > 0:
            post = self.program.run(self.d_ev[: self.n_ev, :n_local].numpy(), n_local)
            self.d_out[:, :n_local] = torch.as_tensor(np.asarray(post, dtype=np.float32))
        dist.gather(self.d_out, list(self.gathered.unbind(0)) if self.is_dst else None, dst=self.dst, group=self.group)
        return self.gathered

    def run_host(self, codes, n_local: int, counts=None, blocks: bool = False):
        """End to end with host buffers: H2D, run, gather, D2H.  Returns [Q, sum(counts)] float32
        on `dst` (rank order; `counts` = rows per rank, default `rows_max` each), None elsewhere.
        blocks=True returns the per-rank blocks instead -- a list of [Q, counts[r]] views of the
        pinned staging buffer, valid until the next call -- and skips the host-side concatenation
        (16 MB and ~1.2 ms for 8 ranks x 100k rows of the benchmark grid)."""
        import torch

        self.upload(codes)
        self.run_resident(n_local)
        if not self.is_dst:
            return None
        self.host.copy_(self.gathered, non_blocking=self.on_device)
        if self.on_device:
            torch.cuda.current_stream(self.device).synchronize()
        counts = [self.rows_max] * self.world if counts is None else list(counts)
        parts = [self.host[r, :, : counts[r]].numpy() for r in range(self.world)]
        return parts if blocks else np.concatenate(parts, axis=1)


def query_many_sharded(bn, *query, events, group=None, dst: int = 0):
    """`BayesNet.query_many` with the rows of `events` sharded over the ranks of `group`
    (torchrun, one process per GPU; `bn.device` is this rank's GPU).  Every rank passes the same
    `events`; rank r answers `row_shard(len(events), r, world)`.  Returns the DataFrame on the
    global rank `dst`, None elsewhere.  Rows flagged by the float32 program are settled in
    float64 on the rank that owns them, before the gather."""
    import torch
    import torch.distributed as dist

    ev_vars = tuple(events.columns)
    plan, _ = bn._plan(query, ev_vars, 1)
    n = len(events.index)
    world, rank = dist.get_world_size(group), dist.get_rank(group)
    codes, bad = bn._encode_events(events, ev_vars)
    backend = dist.get_backend(group)
    device = f"cuda:{torch.cuda.current_device()}" if backend == "nccl" else None

    def run_fn(local_codes, n_local):
        sl = row_shard(n, rank, world)
        return bn._posterior_codes(query, ev_vars, local_codes, bad[sl]).astype(np.float32)

    post = run_sharded(codes, n, run_fn, group=group, dst=dst, device=device)
    if post is None:
        return None
    return bn._answer_frame(post.cpu().numpy().astype(np.float64), events.index, bn._answer_index(plan), bad)
