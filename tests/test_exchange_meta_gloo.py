"""CPU, world_size 2 (gloo): the keyframe-meta all-gather beside the record all-gather -- every rank's meta lands at its
record's index, so a received keyframe's pose and stamp are known on every rank."""
import os
import socket

import numpy as np
import torch
import torch.distributed as dist
import torch.multiprocessing as mp

from omniswarm_b200 import lib, swarm


def _free_port():
    s = socket.socket(); s.bind(("127.0.0.1", 0)); p = s.getsockname()[1]; s.close()
    return p


def _worker(rank, world, port, q):
    os.environ.update(MASTER_ADDR="127.0.0.1", MASTER_PORT=str(port), RANK=str(rank), WORLD_SIZE=str(world))
    dist.init_process_group("gloo", rank=rank, world_size=world)
    rec = lib.KeyframeRecord()
    rec.drone_id, rec.msg_id, rec.n_dirs = rank + 1, 100 + rank, 4
    meta = lib.KeyframeMeta(drone_id=rank + 1, msg_id=100 + rank, stamp_ns=10**18 + 7 * rank)
    meta.pose_drone[:] = [rank + 0.5, -1.0, 2.0, 1.0, 0.0, 0.0, 0.0]
    recs = swarm.exchange_records(torch.frombuffer(bytearray(bytes(rec)), dtype=torch.uint8))
    metas = swarm.exchange_metas(torch.frombuffer(bytearray(bytes(meta)), dtype=torch.uint8))
    raw_r, raw_m = recs.numpy().tobytes(), metas.numpy().tobytes()
    pairs = []
    for r in range(world):
        rr = lib.KeyframeRecord.from_buffer_copy(raw_r[r * lib.RECORD_BYTES:(r + 1) * lib.RECORD_BYTES])
        mm = lib.KeyframeMeta.from_buffer_copy(raw_m[r * lib.META_BYTES:(r + 1) * lib.META_BYTES])
        pairs.append((rr.drone_id, rr.msg_id, mm.drone_id, mm.msg_id, mm.stamp_ns, list(mm.pose_drone)))
    q.put((rank, pairs, metas.numel()))
    dist.destroy_process_group()


def test_meta_all_gather_shares_the_record_index():
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = _free_port()
    ps = [ctx.Process(target=_worker, args=(r, 2, port, q)) for r in range(2)]
    [p.start() for p in ps]
    res = sorted([q.get(timeout=120) for _ in range(2)])
    [p.join(timeout=60) for p in ps]
    assert res[0][1] == res[1][1]
    for rank, pairs, n in res:
        assert n == 2 * lib.META_BYTES == 144
        for r, (rd, rm, md, mm, stamp, pose) in enumerate(pairs):
            assert (rd, rm) == (md, mm) == (r + 1, 100 + r)
            assert stamp == 10**18 + 7 * r and pose == [r + 0.5, -1.0, 2.0, 1.0, 0.0, 0.0, 0.0]


def test_single_rank_meta_exchange_is_identity():
    m = torch.arange(lib.META_BYTES, dtype=torch.int64).to(torch.uint8)
    assert torch.equal(swarm.exchange_metas(m), m)
    assert np.dtype([("a", "<i4"), ("b", "<i4"), ("t", "<i8"), ("p", "<f8", 7)]).itemsize == lib.META_BYTES
