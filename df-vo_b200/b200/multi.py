"""Multi-GPU plumbing of the tracking path: one process per GPU, one image sequence per process.

DF-VO's per-frame path has no cross-sequence data dependency (dfvo.py:358-403 walks one sequence), so the path
shards over *sequences*: rank r owns sequences r, r+world, ... and runs them with the weights every rank
received once at start-up.  That broadcast is the only collective; there is no data-path exchange, hence no
fused compute+collective kernel to write (DESIGN.md section 7).  Timing is the max over ranks.

Works on any torch.distributed backend: NCCL on GPUs, gloo in the CPU test-suite
(tests/test_multi_gloo.py).
"""
import numpy as np


def weight_layout(dicts):
    """Deterministic (dict index, key, shape, offset) table over the array-valued entries of the state dicts."""
    table, off = [], 0
    for di, d in enumerate(dicts):
        for k in sorted(d):
            v = d[k]
            if hasattr(v, "shape") and getattr(v, "dtype", None) is not None:
                n = int(np.prod(v.shape)) if len(v.shape) else 1
                table.append((di, k, tuple(v.shape), off, n))
                off += n
    return table, off


def pack_weights(dicts):
    table, total = weight_layout(dicts)
    flat = np.empty(total, np.float32)
    for di, k, shape, off, n in table:
        flat[off:off + n] = np.asarray(dicts[di][k], np.float32).reshape(-1)
    return flat, table


def unpack_weights(flat, table, dicts):
    for di, k, shape, off, n in table:
        dicts[di][k] = np.array(flat[off:off + n], np.float32).reshape(shape)
    return dicts


def broadcast_weights(dicts, src=0, device=None):
    """Every rank passes state dicts of identical structure (keys + shapes); on return all hold rank `src`'s
    values.  One flat fp32 buffer, one collective."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return dicts
    flat, table = pack_weights(dicts)
    t = torch.from_numpy(flat)
    if device is not None:
        t = t.to(device)
    if dist.get_rank() != src:
        t.zero_()
    dist.broadcast(t, src=src)
    return unpack_weights(t.cpu().numpy(), table, dicts)


def rank_sequences(n_sequences, rank, world):
    """Round-robin ownership of sequences (stripes of the dataset); every sequence has exactly one owner."""
    return list(range(rank, n_sequences, world))


def max_over_ranks(ms, device=None):
    """A timed region's duration is the slowest rank's."""
    import torch
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return float(ms)
    t = torch.tensor([float(ms)], dtype=torch.float64, device=device or "cpu")
    dist.all_reduce(t, op=dist.ReduceOp.MAX)
    return float(t.item())


def gather_trajectories(poses, dst=0):
    """Collect each rank's {sequence: {frame: 4x4}} on `dst` (evaluation / saving happens on one rank)."""
    import torch.distributed as dist
    if not (dist.is_available() and dist.is_initialized()) or dist.get_world_size() == 1:
        return [poses]
    out = [None] * dist.get_world_size() if dist.get_rank() == dst else None
    dist.gather_object(poses, out, dst=dst)
    return out


# ---------------------------------------------------------------------------------------------
# pair-level sharding: the "batched many-frames mode" (independent image pairs split over the GPUs)
# ---------------------------------------------------------------------------------------------
class PairShard:
    """Contiguous block of the `total` independent image pairs owned by `rank` (SURVEY 8e: "contiguous block of 64/G pairs per
    GPU").  The first `total % world` ranks take one extra pair, so every pair has exactly one owner for any world size."""

    def __init__(self, total, rank, world):
        base, rem = divmod(int(total), int(world))
        self.total, self.rank, self.world = int(total), int(rank), int(world)
        self.count = base + (1 if rank < rem else 0)
        self.first = rank * base + min(rank, rem)

    def owner_table(self):
        """[(first, count)] for every rank."""
        return [(PairShard(self.total, r, self.world).first, PairShard(self.total, r, self.world).count) for r in range(self.world)]


class PairBatchRunner:
    """LiteFlowNet forward+backward flow and the consistency map for a rank's block of pairs in ONE batched forward
    (``dfvo_liteflow_build(pairs=count)``; the reference itself is hard-wired to one pair per call, deep_flow.py:34).  Frames
    and outputs stay on the device; per pair only the mean inconsistency and the fraction of consistent pixels leave it."""

    def __init__(self, rt, height, width, pairs, flow_weights, precision=1, thre=0.1):
        from . import tracking
        self.rt, self.pairs, self.thre = rt, int(pairs), float(thre)
        self.eng = tracking.Engine(height, width, rt)
        self.eng.build_flow(flow_weights, pairs=self.pairs, precision=precision)

    def forward(self, img_bufs):
        """img_bufs: 2*pairs uint8 HWC device buffers [ref0, cur0, ref1, cur1, ...] -> float64 [pairs, 2] =
        (mean flow_diff, fraction of pixels with flow_diff < thre)."""
        assert len(img_bufs) == 2 * self.pairs
        fwd, bwd, diff = self.eng.flow(img_bufs)
        d = diff.t.reshape(self.pairs, -1) if hasattr(diff.t, "reshape") else diff.t
        if hasattr(d, "mean") and not isinstance(d, np.ndarray):          # torch tensor on the device: two tiny reductions
            stats = self.rt.torch.stack([d.double().mean(1), (d < self.thre).double().mean(1)], 1)
            return stats.cpu().numpy()
        d = np.asarray(d)
        return np.stack([d.astype(np.float64).mean(1), (d < self.thre).mean(1)], 1)


def gather_pair_stats(stats, shard, world, device=None):
    """all_gather of the per-pair statistics ([count, 2] per rank, ragged blocks padded to the largest) -> [total, 2] in
    global pair order on every rank."""
    import torch
    import torch.distributed as dist
    stats = np.asarray(stats, np.float64).reshape(-1, 2)
    if not (dist.is_available() and dist.is_initialized()) or world == 1:
        return stats
    table = shard.owner_table()
    cap = max(c for _, c in table)
    mine = torch.zeros((cap, 2), dtype=torch.float64, device=device or "cpu")
    mine[:stats.shape[0]] = torch.from_numpy(stats).to(mine.device)
    parts = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(parts, mine)
    return np.concatenate([parts[r][:table[r][1]].cpu().numpy() for r in range(world)], 0)
