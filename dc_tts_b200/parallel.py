"""Utterance sharding across GPUs (SURVEY.md 8e).

Utterances never interact on the synthesis path (every op is per batch row,
/root/reference/networks.py:140-153, synthesize.py:54), so the batch is split into
contiguous shards, one per rank, with weights replicated.  The only communication is
ONE gather of the finished spectrograms; the reference has no counterpart (it is a
single-process program).  Backend: NCCL over NVLink on GPUs, gloo in the CPU tests.

Training (BASELINE config 5) is plain data parallelism: every rank runs `Engine.train_step(..., apply=False)`
on its own 32 utterances, the flat gradient arena (`Engine.train_grads()`) is averaged over the ranks
(`allreduce_mean_`), then every rank applies the identical Adam update (`Engine.train_apply`).
"""
import torch
import torch.distributed as dist


def shard_bounds(total, rank, world):
    """Contiguous split of `total` utterances: rank g gets [lo, hi); sizes differ by <= 1."""
    if not (0 <= rank < world):
        raise ValueError("rank %d outside world %d" % (rank, world))
    base, rem = divmod(total, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def gather_spectrograms(local, total, dst=0, group=None):
    """Gather per-rank (b_g, T, F) tensors into the (total, T, F) tensor on `dst`
    (None elsewhere).  Shards may be ragged by one utterance; rows keep global order."""
    world = dist.get_world_size(group)
    rank = dist.get_rank(group)
    if world == 1:
        return local
    out = None
    if rank == dst:
        out = torch.empty((total,) + tuple(local.shape[1:]), dtype=local.dtype, device=local.device)
    ops = []
    if rank == dst:
        for g in range(world):
            lo, hi = shard_bounds(total, g, world)
            if g == dst:
                out[lo:hi].copy_(local)
            elif hi > lo:
                ops.append(dist.P2POp(dist.irecv, out[lo:hi], g, group))
    else:
        lo, hi = shard_bounds(total, rank, world)
        if hi > lo:
            ops.append(dist.P2POp(dist.isend, local.contiguous(), dst, group))
    if ops:
        for w in dist.batch_isend_irecv(ops):
            w.wait()
    return out


class OverlappedGather:
    """The same single gather, hidden under the SSRN (VERDICT r1 item 5): SSRN runs in utterance chunks and every finished
    chunk leaves at once on a side stream into a receive buffer that is allocated ONCE, so only the last chunk's transfer
    is exposed.  Round 1 gathered after the whole SSRN, allocating the receive tensor every step: a fixed ~2.4 ms at every
    N > 1.  Rows keep global order and are bit-identical to the per-rank results (no arithmetic here).

        og = OverlappedGather(total, shape_tail, dtype, device, chunks=4)
        for step:  og.begin(); for c in og.chunks(): z = produce(c.lo, c.hi); og.send(c, z);  Z = og.finish()
    """

    class Chunk:
        __slots__ = ("index", "lo", "hi")

        def __init__(self, index, lo, hi):
            self.index, self.lo, self.hi = index, lo, hi

    def __init__(self, total, shape_tail, dtype, device, chunks=4, dst=0, group=None):
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.total, self.dst, self.group, self.device = total, dst, group, device
        self.lo, self.hi = shard_bounds(total, self.rank, self.world)
        n = self.hi - self.lo
        self.nchunks = max(1, min(chunks, n)) if n > 0 else 1
        base, rem = divmod(total, self.world)
        self.nchunks_max = max(1, min(chunks, base + (1 if rem else 0)))
        self.cuda = torch.device(device).type == "cuda"
        self.side = torch.cuda.Stream(device=device) if self.cuda else None
        self.out = torch.empty((total,) + tuple(shape_tail), dtype=dtype, device=device) if self.rank == dst else None
        self._pending = []

    def _bounds(self, rank, c, nchunks):
        lo, hi = shard_bounds(self.total, rank, self.world)
        n = hi - lo
        return lo + (n * c) // nchunks, lo + (n * (c + 1)) // nchunks

    def chunks(self):
        """This rank's chunks as LOCAL row ranges [lo, hi) of its shard."""
        n = self.hi - self.lo
        return [self.Chunk(c, (n * c) // self.nchunks, (n * (c + 1)) // self.nchunks) for c in range(self.nchunks)]

    def begin(self):
        """Destination: post the receives, one NCCL group per chunk index holding that chunk of EVERY other rank, so that the
        peers' chunk c arrive concurrently while chunk c+1 is still being computed (receives posted one by one would serialise
        the peers on the destination's communication stream)."""
        self._pending = []
        if self.world == 1 or self.rank != self.dst:
            return
        ctx = torch.cuda.stream(self.side) if self.cuda else _Null()
        if self.cuda:
            self.side.wait_stream(torch.cuda.current_stream(self.device))      # the buffer's previous consumer is done
        with ctx:
            for c in range(self.nchunks_max):
                ops = []
                for g in range(self.world):
                    if g == self.dst:
                        continue
                    glo, ghi = shard_bounds(self.total, g, self.world)
                    nch = max(1, min(self.nchunks, ghi - glo))
                    if c < nch:
                        a, b = self._bounds(g, c, nch)
                        if b > a:
                            ops.append(dist.P2POp(dist.irecv, self.out[a:b], g, self.group))
                if ops:
                    self._pending.extend(dist.batch_isend_irecv(ops))

    def send(self, chunk, z):
        """Hand over the finished local rows [chunk.lo, chunk.hi) (a tensor of exactly those rows)."""
        a, b = self.lo + chunk.lo, self.lo + chunk.hi
        if b <= a:
            return
        if self.world == 1 or self.rank == self.dst:
            if self.out is not None and z.data_ptr() != self.out[a:b].data_ptr():
                self.out[a:b].copy_(z)
            return
        if self.cuda:
            self.side.wait_stream(torch.cuda.current_stream(self.device))      # chunk is complete on the compute stream
            with torch.cuda.stream(self.side):
                z.record_stream(self.side)
                self._pending.extend(dist.batch_isend_irecv([dist.P2POp(dist.isend, z.contiguous(), self.dst, self.group)]))
        else:
            self._pending.extend(dist.batch_isend_irecv([dist.P2POp(dist.isend, z.contiguous(), self.dst, self.group)]))

    def local_view(self, chunk):
        """Destination rank: the slice of the receive buffer its own chunk belongs in (produce straight into it)."""
        if self.out is None:
            return None
        return self.out[self.lo + chunk.lo:self.lo + chunk.hi]

    def finish(self):
        for w in self._pending:
            w.wait()
        self._pending = []
        if self.cuda and self.side is not None:
            torch.cuda.current_stream(self.device).wait_stream(self.side)
        return self.out


class _Null:
    def __enter__(self):
        return self

    def __exit__(self, *a):
        return False


def allreduce_mean_(flat, group=None):
    """In-place average of a flat gradient buffer over the ranks (sum all-reduce, then 1/world): the gradient of the mean
    loss over the global batch when every rank holds the same number of utterances.  Returns `flat`."""
    world = dist.get_world_size(group)
    if world > 1:
        dist.all_reduce(flat, op=dist.ReduceOp.SUM, group=group)
        flat.mul_(1.0 / world)
    return flat
