"""Row-sharded prototype search across GPUs (SURVEY.md section 8(e)); one process per GPU, torch.distributed (NCCL).

    E   data-parallel: every rank encodes its own B queries (replicated encoder weights, no communication)
    K   P is row-sharded (N/G contiguous rows per rank, global id = local + offset):
          1. all-gather of the unit embeddings        -> every rank holds all G*B queries   (G*B*D*4 bytes)
          2. local top-k over the shard for all G*B queries (ac_knn_l2_topk, row_offset = shard start)
          3. ONE all-to-all of the packed candidates  -> rank r receives the G lists of ITS B queries
                                                         (chunk = distances fp32 | global ids int64, B*k*12 bytes per peer)
          4. merge by (d, global id)                  -> bit-identical to a single-shard search
    H   data-parallel on the rank's own queries, on a side stream concurrently with K; blend as in predict_batch.

`ShardedPipeline` is the product path (bench.py at N > 1): it drives the SAME C pipeline as N = 1 phase by phase
(`ac_pipeline_encode` / `_search_shard` / `_finish_sharded`) with the two collectives in between on the same stream; nothing
synchronises with the host.  The two collectives are plain NCCL: the messages are small (1.5 MB and 30 KB per peer at 512
queries), so the cost is expected to be launch latency, not NVLink bandwidth (not measured on H100).

`ShardedIndex` is the same exchange at the index level (any k, used by tests and by callers that only need the search); its
search / pack / merge callables are injectable so that the host logic (sharding arithmetic, collectives, chunk layout, merge
order) is covered by world_size-2 gloo tests on CPU with the oracle standing in for the kernels (tests only); the default
callables are the CUDA kernels and raise without a GPU.
"""
from __future__ import annotations

from typing import Callable, Tuple

import torch
import torch.distributed as dist


def shard_bounds(N: int, rank: int, world: int) -> Tuple[int, int]:
    """contiguous row range [lo, hi) of `rank`; the first N % world ranks get one extra row"""
    base, rem = divmod(N, world)
    lo = rank * base + min(rank, rem)
    return lo, lo + base + (1 if rank < rem else 0)


def pack_candidates(d: torch.Tensor, i: torch.Tensor, G: int) -> torch.Tensor:
    """d [G*B, k] fp32, i [G*B, k] int64 (block g = queries of rank g) -> uint8 [G, B*k*12]: chunk g = d bytes | id bytes.
    Same layout as csrc/predict.cu::pack_candidates_kernel."""
    bk = d.numel() // G
    return torch.cat([d.contiguous().view(G, bk).view(torch.uint8), i.contiguous().view(G, bk).view(torch.uint8)], dim=1).contiguous()


def unpack_candidates(buf: torch.Tensor, G: int, B: int, k: int):
    """inverse of pack_candidates on the received buffer: -> (d [G, B, k], i [G, B, k]); chunk g = shard g's list of MY queries"""
    bk = B * k
    d = buf[:, : bk * 4].contiguous().view(torch.float32).view(G, B, k)
    i = buf[:, bk * 4 :].contiguous().view(torch.int64).view(G, B, k)
    return d, i


def _cuda_search(Q, P, k, row_offset):
    from . import _cabi
    return _cabi.knn_l2_topk(Q, P, k, row_offset=row_offset)


def _cuda_merge(d, i):
    from . import _cabi
    return _cabi.topk_merge(d, i)


class ShardedIndex:
    """This rank's shard of the prototype matrix plus the collective search."""

    def __init__(self, P_local: torch.Tensor, row_offset: int, *, group=None,
                 search: Callable = _cuda_search, merge: Callable = _cuda_merge):
        self.P = P_local
        self.row_offset = int(row_offset)
        self.group = group
        self.search = search
        self.merge = merge
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0

    def search_local_queries(self, q_local: torch.Tensor, k: int):
        """q_local [B, D] (this rank's queries) -> (d [B,k], global ids [B,k]) over the WHOLE index."""
        G = self.world
        B, D = q_local.shape
        if G == 1:
            return self.search(q_local, self.P, k, self.row_offset)
        q_all = torch.empty((G * B, D), dtype=q_local.dtype, device=q_local.device)
        dist.all_gather_into_tensor(q_all, q_local.contiguous(), group=self.group)
        d_loc, i_loc = self.search(q_all, self.P, k, self.row_offset)         # [G*B, k]
        send = pack_candidates(d_loc, i_loc, G)
        recv = torch.empty_like(send)
        # chunk g of the send buffer (queries of rank g) goes to rank g; received chunk g = shard g's list of MY queries
        dist.all_to_all_single(recv, send, group=self.group)
        d_recv, i_recv = unpack_candidates(recv, G, B, k)
        return self.merge(d_recv, i_recv)


class ShardedPipeline:
    """One predict step (E -> K over row shards -> H -> blend) of a rank: the C pipeline's phases with the two NCCL
    collectives between them.  `pipe` is a _cabi.Pipeline created with shards = world size over this rank's row shard."""

    def __init__(self, pipe, group=None):
        self.pipe = pipe
        self.group = group
        self.G = dist.get_world_size(group)
        self.rank = dist.get_rank(group)
        dev = pipe.P.device
        B, D, k = pipe.max_B, pipe.P.shape[1], pipe.k
        self.q_all = torch.empty((self.G * B, D), dtype=torch.float32, device=dev)
        self.send = torch.empty((self.G, B * k * 12), dtype=torch.uint8, device=dev)
        self.recv = torch.empty_like(self.send)

    def predict_device(self, ids_dev: torch.Tensor):
        p, G = self.pipe, self.G
        B = ids_dev.shape[0]
        assert B == p.max_B, "the sharded step runs full batches (every rank contributes the same number of queries)"
        emb = p.encode(ids_dev)                                                       # [B, D] view of the pipeline's buffer
        dist.all_gather_into_tensor(self.q_all, emb, group=self.group)
        p.search_shard(self.q_all, G, B, self.send)
        dist.all_to_all_single(self.recv, self.send, group=self.group)
        return p.finish_sharded(self.recv, G, B)
