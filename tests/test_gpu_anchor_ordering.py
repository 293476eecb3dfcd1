"""The anchor handle's ordering across streams: a call that touches a part of the handle's state (the store, the observe
record, the sync's paths, the keyframe store, the loop map, the data association result) waits for the last call that
touched it on any stream.  In each case the first call goes on stream A behind a bounded sleep, so it has not run when
the second call is made on stream B; the outputs must equal, byte for byte, those of a second handle fed the same inputs
that makes the same calls on one stream.  The one-stream handle goes first, so every kernel has been loaded before the
two-stream calls (a kernel's first launch can wait for the device, and the sleep with it)."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l, synth
import keyframe_ref as kr
import test_gpu_anchor_data_association as dat
import test_gpu_anchor_init_by_loops as ibl
import test_gpu_anchor_keyframe as kft
from backend_harness import feed, make_anchor
from test_publish_ref import flight, frames_of

pytestmark = pytest.mark.gpu
SLEEP = 500_000_000                              # cycles: the first call waits this long behind its stream's sleep
ROW = _l.ANCHOR_RESULT_DTYPE.itemsize


def streams():
    """stream A, already sleeping, and stream B; both after the current stream's work"""
    a, b = torch.cuda.Stream(), torch.cuda.Stream()
    for s in (a, b):
        s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(a):
        torch.cuda._sleep(SLEEP)
    return a, b


def rows_buf(n):
    return torch.zeros(max(n, 1) * ROW, dtype=torch.uint8, device="cuda")


def host_bytes(t):
    torch.cuda.synchronize()
    return t.cpu().numpy().tobytes()


def test_runs_on_two_streams_then_set_window(gpu):
    """a run on B comes after an earlier run on A, and set_window after both: A's rows are the old window's"""
    g = synth.anchor_swarm(4, 20, 200, seed=5)
    stamps, first, ents = g["window"]
    later = frames_of(g["window"], 1, len(stamps))
    out = []
    for two in (False, True):
        a = make_anchor(g)
        feed(a, g)
        n = sum(a.size())
        ra, rb = rows_buf(n), rows_buf(n)
        sa, sb = streams()
        if not two:
            sb = sa
        a.run_dev(ra.data_ptr(), sa.cuda_stream)
        a.run_dev(rb.data_ptr(), sb.cuda_stream)
        if two:
            assert not sa.query()
        a.set_window(*later)
        out.append((host_bytes(ra), host_bytes(rb), a.run().tobytes()))
        a.close()
    assert out[0] == out[1]
    assert out[0][0] == out[0][1] and out[0][0] != out[0][2]       # the old window's rows, not the new one's


def test_data_association_then_run_on_another_stream(gpu):
    """a run_dev on B after data_association_dev on A re-anchors the renamed rows"""
    trajs, dets = dat.flight(5, 3, 1)
    win = dat.window(trajs, range(5))
    out = []
    for two in (False, True):
        a = dat.anchor(trajs, dets, 5)
        c = host.AnchoredChain(512)
        n = dat.front(a, c, win, 1)
        r0, rb = rows_buf(n), rows_buf(n)
        assert a.run_dev(r0.data_ptr(), c.stream.cuda_stream) == n     # the rows before the renaming
        c.stream.synchronize()
        before = host_bytes(r0)
        sa, sb = streams()
        if not two:
            sb = sa
        a.data_association_dev(1, sa.cuda_stream)
        assert a.run_dev(rb.data_ptr(), sb.cuda_stream) == n
        if two:
            assert not sa.query()
        assert a.data_association_result()[:2] == (True, _l.OK)
        out.append(host_bytes(rb))
        a.close()
    assert out[0] == out[1] and out[0] != before


def test_observe_then_init_mask(gpu):
    g = synth.anchor_swarm(4, 20, 200, seed=6)
    n_nodes = int(g["window"][2]["block"].max()) + 1
    out = []
    for two in (False, True):
        a = make_anchor(g)
        feed(a, g)
        c = host.AnchoredChain(sum(a.size()))
        c.observe(a, 0, 0, 1e6, 1e6)                                # no motion, no rows: to_init holds self only
        c.init_mask(a, 0, n_nodes)                                  # the first call acquires the block table
        c.stream.synchronize()
        sa, sb = streams()
        if not two:
            sb = sa
        a.observe_dev(c.rows.data_ptr(), 0, sa.cuda_stream, 0, -1.0, -1.0)   # motion: every node without pos
        a.init_mask_dev(0, n_nodes, c.mask.data_ptr(), c.yaw.data_ptr(), sb.cuda_stream)
        if two:
            assert not sa.query()
        out.append((host_bytes(c.mask), host_bytes(c.yaw)))
        a.close()
    assert out[0] == out[1] and any(out[0][0])


def init_by_loops_rigs():
    """two rigs of the pre-motion scenario, each after its first round's run, observe, reject and compact"""
    g, base = ibl.scenario()
    win = frames_of(flight(g["window"]), 0, 8)
    rigs = []
    for _ in range(2):
        r = ibl.Rig(g, base)
        r.a.set_window(*win)
        c = r.chain
        n = c.run(r.a)
        c.observe(r.a, n, ibl.SELF, ibl.XY, ibl.Z)
        c.reject(r.pcm, n)
        c.compact(n)
        rigs.append((r, n))
    return rigs


def test_sync_then_init_by_loops(gpu):
    out = []
    for two, (r, n) in zip((False, True), init_by_loops_rigs()):
        c = r.chain
        c.record_loops(r.a, n)
        c.init_by_loops(r.a, r.pcm, r.dev, ibl.SELF, r.n_nodes)    # nothing estimated yet
        c.init_solve(r.dev, 4096, 1, 7, ibl.WIN, np.inf, options=r.o)
        c.stream.synchronize()
        sa, sb = streams()
        if not two:
            sb = sa
        r.a.sync_dev(r.dev, sa.cuda_stream, ibl.SELF, np.inf, ibl.WIN, True, False)
        r.a.init_by_loops_dev(r.pcm, r.dev, ibl.SELF, sb.cuda_stream)   # the sync's paths and estimated drones
        if two:
            assert not sa.query()
        assert r.a.sync_result() == (True, _l.OK) and r.a.init_by_loops_result() == _l.OK
        out.append(r.dev.graph_get_poses().tobytes())
        r.close()
    assert out[0] == out[1]


def test_record_loops_then_init_by_loops(gpu):
    out = []
    for two, (r, n) in zip((False, True), init_by_loops_rigs()):
        c = r.chain
        c.stream.synchronize()
        sa, sb = streams()
        if not two:
            sb = sa
        r.a.record_loops_dev(c.rows.data_ptr(), n, sa.cuda_stream)
        r.a.init_by_loops_dev(r.pcm, r.dev, ibl.SELF, sb.cuda_stream)   # the map holds every set's smallest id
        if two:
            assert not sa.query()
        assert r.a.init_by_loops_result() == _l.OK
        m = r.a.loop_map()
        out.append((r.dev.graph_get_poses().tobytes(), m["records"].tobytes(), m["pair_min"].tobytes()))
        r.close()
    assert out[0] == out[1] and len(out[0][1]) > 0


K, KF0, WIN_KF = 6, 10, 4                       # ring slots; keyframes stored before the case; stored window frames


def keyframe_flight():
    """keyframes 0..KF0-1 stored in a ring of K slots, and the next one's records: the window holds the last WIN_KF
    stored frames and the next one, whose keyframe takes the slot of one that left the window"""
    f = kft.Flight(KF0 + 1)
    f.a.close()
    f.a = host.LoopAnchor(8, 64, 64, 4096, 1.0, 0.01, 0.01, max_keyframes=K)
    for k in range(KF0):
        f.keyframe(k, finish_init=k >= 5, check=False)
    kf = f.kfs[KF0]
    nodes, dists = kr.keyframe_records(kf, f.asg, kft.SELF, True)
    if f.asg.next > f.n_blocks:
        f.s.graph_add_nodes(np.zeros((f.asg.next - f.n_blocks, 4)))
    fr = f.frames[-WIN_KF:] + [(kf["stamp"], nodes)]
    first = np.concatenate([[0], np.cumsum([len(x) for _, x in fr])]).astype(np.int32)
    f.a.set_window([ts for ts, _ in fr], first, np.concatenate([kft.entries(x, ts) for ts, x in fr]))
    c = f.chain
    c.observe(f.a, 0, kft.SELF, -1.0, -1.0)                       # motion: every node enabled
    c.compact(0, keep=False)
    c.stream.synchronize()

    def add(stream):
        f.a.add_keyframe_dev(f.s, kf["stamp"], nodes, dists, stream, kft.SELF, True, seed=kft.SEED)

    def distances(stream):
        f.a.distance_factors_dev(c.factors, c.factors.type.numel(), stream, kft.SELF)

    def result(stream):
        rows = c.factors.on_host(stream)
        return (b"".join(np.asarray(rows[k]).tobytes() for k in host.FACTOR_KEYS), f.s.graph_get_poses().tobytes(),
                f.a.keyframe_flags(kf["stamp"]).tobytes())

    return f, add, distances, result


@pytest.mark.parametrize("first", ["add_keyframe", "distance_factors"])
def test_keyframe_store_between_add_and_distances(gpu, first):
    """add_keyframe_dev -> distance_factors_dev reads the new keyframe; distance_factors_dev -> an add_keyframe_dev that
    takes a slot of the ring it reads does not"""
    out = []
    for two in (False, True):
        f, add, distances, result = keyframe_flight()
        calls = (add, distances) if first == "add_keyframe" else (distances, add)
        sa, sb = streams()
        if not two:
            sb = sa
        calls[0](sa.cuda_stream)
        calls[1](sb.cuda_stream)
        if two:
            assert not sa.query()
        sa.synchronize()
        out.append(result(sb))
        f.a.close()
        f.s.close()
    assert out[0] == out[1] and len(out[0][0]) > 0
