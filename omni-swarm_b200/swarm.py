"""Swarm-wide keyframe exchange: ONE all-gather of the fixed-size keyframe record per keyframe round.

Replaces LoopNet::broadcast_fisheye_desc / image_desc_callback (/root/reference/swarm_loop/src/loop_net.cpp:20-120,
142-172): the reference multicasts one LCM header message (global descriptor) plus one message per landmark over UDP
and reassembles them with timeouts; on the 8-GPU box the 8 drones are 8 ranks and the same information moves as one
`all_gather_into_tensor` of `lib.RECORD_BYTES` bytes per rank over NVLink (NCCL).  The reference's "skip my own
messages" rule (loop_net.cpp:133-136) becomes "my own slot goes to the local database" -- handled by
osb_frontend_ingest, which routes each record by its drone_id.
"""
from __future__ import annotations

import torch
import torch.distributed as dist

from . import lib as _l


def exchange_records(record: torch.Tensor, gathered: torch.Tensor | None = None, group=None) -> torch.Tensor:
    """record: uint8 tensor [RECORD_BYTES] (this rank's osb_keyframe_record, device memory under NCCL, host memory
    under gloo) -> uint8 tensor [world * RECORD_BYTES] holding every rank's record in rank order."""
    assert record.dtype == torch.uint8 and record.numel() == _l.RECORD_BYTES
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if gathered is None:
        gathered = torch.empty(world * _l.RECORD_BYTES, dtype=torch.uint8, device=record.device)
    if world == 1:
        gathered.copy_(record)
        return gathered
    dist.all_gather_into_tensor(gathered, record, group=group)
    return gathered


def exchange_metas(meta: torch.Tensor, gathered: torch.Tensor | None = None, group=None) -> torch.Tensor:
    """meta: uint8 tensor [META_BYTES] (this rank's osb_keyframe_meta, the one beside its record) -> uint8 tensor
    [world * META_BYTES] in rank order, so that gathered metas and records share their index."""
    assert meta.dtype == torch.uint8 and meta.numel() == _l.META_BYTES
    world = dist.get_world_size(group) if dist.is_initialized() else 1
    if gathered is None:
        gathered = torch.empty(world * _l.META_BYTES, dtype=torch.uint8, device=meta.device)
    if world == 1:
        gathered.copy_(meta)
        return gathered
    dist.all_gather_into_tensor(gathered, meta, group=group)
    return gathered


def record_view(gathered: torch.Tensor, rank: int) -> torch.Tensor:
    return gathered[rank * _l.RECORD_BYTES:(rank + 1) * _l.RECORD_BYTES]


def routing(gathered_host: torch.Tensor, self_id: int):
    """Host-side statement of what osb_frontend_ingest does with a gathered buffer (used by the CPU tests):
    -> list of (slot, drone_id, msg_id, 'local' | 'remote', [directions with landmark_num > 0])."""
    out = []
    n = gathered_host.numel() // _l.RECORD_BYTES
    raw = gathered_host.cpu().numpy().tobytes()
    for r in range(n):
        rec = _l.KeyframeRecord.from_buffer_copy(raw[r * _l.RECORD_BYTES:(r + 1) * _l.RECORD_BYTES])
        dirs = [d for d in range(min(rec.n_dirs, _l.MAX_DIRS)) if rec.n_kpts[d] > 0]      # loop_detector.cpp:153
        out.append((r, rec.drone_id, rec.msg_id, "local" if rec.drone_id == self_id else "remote", dirs))
    return out


# ---------------------------------------------------------------------------------------------------------------
# Row-sharded keyframe database (SURVEY.md section 8e, the alternative layout for the 50 k-row sweep)
# ---------------------------------------------------------------------------------------------------------------
def shard_rows(n_rows: int, rank: int, world: int) -> tuple[int, int]:
    """contiguous balanced split of the database rows: the first n_rows % world ranks hold one extra row."""
    base, extra = divmod(n_rows, world)
    start = rank * base + min(rank, extra)
    return start, start + base + (1 if rank < extra else 0)


class RowShardedIndex:
    """faiss::IndexFlatIP semantics (loop_detector.h:27-29, loop_detector.cpp:213) over a database whose ROWS are split
    across the ranks: two collectives per search -- all-gather the queries (world x dim floats), every rank scans its
    own shard for all of them (one pass over the shard, up to 8 queries per pass), ONE all-gather of the k candidates per
    (shard, query) with score and row id packed together, and each rank merges world x k candidates for its own query.  Global row ids = shard-local row +
    the shard's first row; order = score descending, ties by ascending global id, -1 / -inf padding.

    `shard` is this rank's rows [n_local, dim] (float32 numpy, or a CUDA tensor); `n_rows_total` fixes every rank's
    row range.
    """

    def __init__(self, shard, n_rows_total: int, dim: int = 4096, group=None, device=None):
        self.group = group
        self.world = dist.get_world_size(group) if dist.is_initialized() else 1
        self.rank = dist.get_rank(group) if dist.is_initialized() else 0
        self.dim, self.n_total = dim, n_rows_total
        self.starts = [shard_rows(n_rows_total, r, self.world)[0] for r in range(self.world)]
        a, b = shard_rows(n_rows_total, self.rank, self.world)
        assert tuple(shard.shape) == (b - a, dim), (shard.shape, a, b)
        self.device = device
        self._open(shard)

    # -- the three device steps (overridden by the CPU/gloo test with host stand-ins) --
    def _open(self, shard):
        from . import host
        self._index = host.IndexFlatIP(self.dim, capacity=max(1, shard.shape[0]))
        if shard.shape[0]:
            if isinstance(shard, torch.Tensor):                      # rows already in HBM
                assert shard.is_cuda and shard.dtype == torch.float32 and shard.is_contiguous()
                self._index.add_dev(shard.data_ptr(), shard.shape[0], torch.cuda.current_stream().cuda_stream)
                torch.cuda.current_stream().synchronize()
            else:
                self._index.add(shard)
        self._lib = _l.load()
        self._offs = torch.tensor(self.starts, dtype=torch.int64, device=self.device)

    def _local_search(self, queries: torch.Tensor, k: int):
        nq = queries.shape[0]
        sc = torch.empty(nq, k, dtype=torch.float32, device=queries.device)
        ids = torch.empty(nq, k, dtype=torch.int64, device=queries.device)
        st = torch.cuda.current_stream().cuda_stream
        self._index.search_dev(queries.data_ptr(), nq, k, sc.data_ptr(), ids.data_ptr(), st)
        return sc, ids

    def _merge(self, cand_scores: torch.Tensor, cand_ids: torch.Tensor, k: int):
        """cand_* [n_lists, k] (ids shard-local) -> global top-k of ONE query"""
        import ctypes as C
        out_s = torch.empty(k, dtype=torch.float32, device=cand_scores.device)
        out_i = torch.empty(k, dtype=torch.int64, device=cand_scores.device)
        st = torch.cuda.current_stream().cuda_stream
        _l.check(self._lib.osb_topk_merge_dev(1, cand_scores.shape[0], k, C.c_void_p(cand_scores.data_ptr()),
                                              C.c_void_p(cand_ids.data_ptr()), C.c_void_p(self._offs.data_ptr()),
                                              C.c_void_p(out_s.data_ptr()), C.c_void_p(out_i.data_ptr()), C.c_void_p(st)))
        return out_s, out_i

    def search(self, query: torch.Tensor, k: int):
        """query: this rank's [dim] float32 tensor -> (scores [k], global ids [k]) for THIS rank's query."""
        w = self.world
        q_all = torch.empty(w, self.dim, dtype=torch.float32, device=query.device)
        if w > 1:
            dist.all_gather_into_tensor(q_all, query.reshape(1, self.dim).contiguous(), group=self.group)
        else:
            q_all.copy_(query.reshape(1, self.dim))
        sc, ids = self._local_search(q_all, k)                       # [w queries, k] over my shard
        if w > 1:
            # ONE exchange back: (score bits, shard-local row id) packed as three int32 words per candidate
            mine = torch.cat([sc.contiguous().view(torch.int32).unsqueeze(-1),
                              ids.contiguous().view(torch.int32).view(w, k, 2)], dim=-1).contiguous()   # [query, k, 3]
            packed = torch.empty(w, w, k, 3, dtype=torch.int32, device=query.device)                    # [shard, query, k, 3]
            dist.all_gather_into_tensor(packed.view(w * w, k * 3), mine.view(w, k * 3), group=self.group)
            got = packed[:, self.rank]                                                                   # [shard, k, 3]
            sc = got[..., 0].contiguous().view(torch.float32)
            ids = got[..., 1:].contiguous().view(torch.int64).view(w, k)
        return self._merge(sc, ids, k)

    def close(self):
        if getattr(self, "_index", None) is not None:
            self._index.close()
            self._index = None
