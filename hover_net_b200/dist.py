"""Multi-GPU plumbing: tiles shard by index across ranks (one process per GPU, weights replicated
once), and the only exchange is the end-of-batch gather of the variable-length instance tables to
every rank -- the multi-GPU replacement for the reference's single-process `torch.nn.DataParallel`
scatter/gather (reference infer/base.py:69, run_infer.py:139).  Works on any torch.distributed
backend (NCCL on the GPUs; gloo in the CPU tests)."""
try:  # torch is only needed for the multi-rank paths; single-GPU tile / WSI runs work without it
    import torch
    import torch.distributed as dist
except ImportError:  # pragma: no cover
    torch = dist = None


def dist_info():
    """(torch.distributed module or None, rank, world): world == 1 when torch is missing or no group is initialised."""
    if dist is not None and dist.is_available() and dist.is_initialized():
        return dist, dist.get_rank(), dist.get_world_size()
    return None, 0, 1


def shard_range(n_items, rank, world):
    """Contiguous [lo, hi) slice of n_items owned by `rank` (first ranks take the remainder)."""
    base, rem = divmod(int(n_items), int(world))
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_tables(table, nrows, group=None):
    """table [B,max_rows,10] int64, nrows [B] int32 (same B and max_rows on every rank) ->
    (table_all [world*B,max_rows,10], nrows_all [world*B]) on every rank, rank-major order."""
    world = dist.get_world_size(group) if (dist is not None and dist.is_initialized()) else 1
    if world == 1:
        return table, nrows
    t_all = torch.empty((world * table.shape[0],) + tuple(table.shape[1:]), dtype=table.dtype, device=table.device)
    n_all = torch.empty((world * nrows.shape[0],), dtype=nrows.dtype, device=nrows.device)
    dist.all_gather_into_tensor(n_all, nrows.contiguous(), group=group)
    dist.all_gather_into_tensor(t_all, table.contiguous(), group=group)
    return t_all, n_all


class PackedGather(object):
    """End-of-batch gather of the instance tables without padding and without a host synchronisation
    (SURVEY.md 8e): the library compacts a batch's tables into `cap_rows` x 10 int64 rows on its own stream
    (`hvn_pack_tables_dev`), the collective is ordered after that stream through a CUDA event (the stream is
    wrapped as a torch ExternalStream) and runs on NCCL's stream while the next batch computes; `wait()`
    joins it.  Two payload slots alternate, so batch i's gather overlaps batch i+1's kernels."""

    def __init__(self, ctx, batch, max_rows, cap_rows, world, device):
        self.ctx, self.B, self.max_rows, self.cap, self.world = ctx, int(batch), int(max_rows), int(cap_rows), int(world)
        self.stream = torch.cuda.ExternalStream(ctx.stream_handle(), device=device)
        n = self.cap * 10 + self.B + 1
        # payload = [packed rows (cap*10 int64) | offs (B+1, stored as int64 pairs of int32)]
        self.send = [torch.zeros(n, dtype=torch.int64, device=device) for _ in range(2)]
        self.recv = [torch.zeros(n * self.world, dtype=torch.int64, device=device) for _ in range(2)]
        self.work = [None, None]
        self.i = 0

    def launch(self, d_table, d_nrows):
        """Pack on the library stream and start the all_gather; returns the slot index."""
        k = self.i & 1
        self.i += 1
        if self.work[k] is not None:  # slot reuse: the library stream waits for the gather that last read it
            with torch.cuda.stream(self.stream):
                self.work[k].wait()
            self.work[k] = None
        send = self.send[k]
        offs_ptr = send.data_ptr() + self.cap * 80
        self.ctx.pack_tables_dev(d_table.data_ptr(), d_nrows.data_ptr(), self.B, self.max_rows, send.data_ptr(), self.cap, offs_ptr)
        if self.world > 1:
            with torch.cuda.stream(self.stream):
                self.work[k] = dist.all_gather_into_tensor(self.recv[k], send, async_op=True)
        else:
            self.recv[k] = send
        return k

    def wait(self, k=None):
        for j in ([k] if k is not None else [0, 1]):
            if self.work[j] is not None:
                with torch.cuda.stream(self.stream):
                    self.work[j].wait()
                self.work[j] = None

    def rows(self, k):
        """Host view of slot k after wait(): list over ranks of (offs [B+1], packed [total,10])."""
        n = self.cap * 10 + self.B + 1
        flat = self.recv[k].cpu().numpy().reshape(-1, n)
        out = []
        for r in range(flat.shape[0]):
            offs = flat[r, self.cap * 10:].view("int32")[: self.B + 1]
            out.append((offs.copy(), flat[r, : int(min(offs[-1], self.cap)) * 10].reshape(-1, 10).copy()))
        return out


def compact_rows(table_all, nrows_all):
    """Drop the padding: list of [n_i,10] arrays, one per tile, in global tile order."""
    t = table_all.cpu().numpy()
    n = nrows_all.cpu().numpy()
    return [t[i, : int(n[i])] for i in range(t.shape[0])]
