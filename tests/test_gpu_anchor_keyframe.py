"""osb_anchor_add_keyframe_dev / osb_anchor_distance_factors_dev: add_as_keyframe's initial poses and outlier flags and
setup_problem_with_sferror's rows on the device, against tests/keyframe_ref.py keyframe by keyframe over a flight with a
late drone, a static node, merged blocks, self before and after finish_init, a sliding window and enable flipping
between solves; the solve that follows against the same tail built on the host; max_tail overflow; refusals; CUDA
graph capture; and that add_keyframe_dev does not synchronise."""
import ctypes

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l
import keyframe_ref as kr

pytestmark = pytest.mark.gpu
SELF, N_DRONES, WIN, SEED = 0, 6, 50, 11
PRM = dict(outlier_threshold=0.3, elevation_threshold=0.5, minimum_distance=0.2, enable_distance=True,
           debug_no_rejection=False, distance_measurement_cov=0.2, self_id=SELF)


def close(got, want):
    """1e-12 relative: only libm-vs-CUDA transcendental ulps (atan2, sin, cos of the yaw algebra) may differ"""
    scale = np.maximum(1.0, np.abs(want))
    assert np.all(np.abs(got - want) <= 1e-12 * scale), float(np.max(np.abs(got - want) / scale))


def entries(nodes, stamp):
    e = np.zeros(len(nodes), _l.WINDOW_ENTRY_DTYPE)
    e["drone_id"], e["block"], e["vo_available"], e["stamp"] = nodes["drone_id"], nodes["block"], nodes["vo_available"], stamp
    e["self_pose"] = nodes["pose"]
    return e


class Flight:
    """a LoopAnchor, a solver whose resident graph gains one node per new block, a chain, and the oracle's record"""

    def __init__(self, n_kf, max_tail=8192, **kw):
        self.kfs = kr.random_keyframes(N_DRONES, n_kf, SEED, self_id=SELF, late=(4,), static=(5,), **kw)
        self.a = host.LoopAnchor(8, 64, 64, 4096, 1.0, 0.01, 0.01, max_keyframes=128)
        self.s = host.PoseGraphSolver(4096, 32768)
        self.chain = host.AnchoredChain(max_tail)
        self.asg = kr.BlockAssigner()
        self.frames, self.last, self.n_blocks = [], None, 0
        self.store = {}

    def keyframe(self, k, finish_init, check=True):
        kf = self.kfs[k]
        nodes, dists = kr.keyframe_records(kf, self.asg, SELF, finish_init)
        grow = self.asg.next - self.n_blocks
        if grow:
            first = self.s.graph_add_nodes(np.zeros((grow, 4)))
            if first == 0:                                              # the base graph: block 0 held, one factor
                self.s.graph_set_fixed(0, True)
            self.n_blocks = self.asg.next
        before = self.s.graph_get_poses()
        self.a.add_keyframe_dev(self.s, kf["stamp"], nodes, dists, self.chain.stream.cuda_stream, SELF, finish_init,
                                seed=SEED, **{k2: PRM[k2] for k2 in ("outlier_threshold", "elevation_threshold",
                                                                     "minimum_distance")})
        after = self.s.graph_get_poses()                                # the host mirror follows the device write
        want = kr.init_poses(nodes, before, kf["stamp"], SELF, finish_init, SEED)
        if check:
            close(after, want)
            noisy = nodes[(nodes["new_block"] != 0) & ((nodes["prev_block"] < 0) | (nodes["is_static"] != 0))]
            if not finish_init:
                noisy = noisy[noisy["drone_id"] != SELF]
            assert after[noisy["block"], :3].tobytes() == want[noisy["block"], :3].tobytes()
        flags = kr.outlier_flags(nodes, dists, after, self.last, dict(PRM, finish_init=finish_init))
        got = self.a.keyframe_flags(kf["stamp"])
        if check:
            assert np.array_equal(got, flags), k
        self.store[kf["stamp"]] = (nodes, dists, got)
        self.last = nodes
        self.frames.append((kf["stamp"], nodes))

    def window(self):
        fr = self.frames[-WIN:]
        first = np.concatenate([[0], np.cumsum([len(n) for _, n in fr])]).astype(np.int32)
        ent = np.concatenate([entries(n, ts) for ts, n in fr])
        self.a.set_window([ts for ts, _ in fr], first, ent)
        return [(ts, {int(x["drone_id"]): int(x["block"]) for x in n}) for ts, n in fr]

    def rows(self, xy, z, max_tail=None):
        """observe (no loop rows) -> compact -> distance_factors_dev -> (device rows, oracle rows)"""
        win = self.window()
        c = self.chain
        c.observe(self.a, 0, SELF, xy, z)
        c.compact(0, keep=False)
        cap = max_tail if max_tail is not None else c.factors.type.numel()
        c.distances(self.a, cap, SELF, distance_measurement_cov=PRM["distance_measurement_cov"])
        got = c.factors.on_host(c.stream)
        want = kr.distance_rows(win, self.store, self.a.observability()["enable"].tolist() + [False] * 248, PRM)
        return got, want


def same_rows(got, want):
    for k in host.FACTOR_KEYS:
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k


def test_keyframes_and_rows_against_the_oracle():
    """>= 100 keyframes, the window sliding at 50 frames, finish_init from keyframe 10, enable off then on"""
    f = Flight(110)
    n_rows = []
    for k in range(110):
        f.keyframe(k, finish_init=k >= 10)
        if k % 10 == 9:
            xy = 1e6 if k < 40 else 0.0                                 # self's box: no motion, then motion enables all
            got, want = f.rows(xy, xy)
            same_rows(got, want)
            n_rows.append(len(got["ia"]))
    assert n_rows[:4] == [0] * 4 and min(n_rows[4:]) > 0               # only self_id (drone 0) enabled: no b < a;
                                                                        # then enable flips: rows on frames already there
    assert set(f.a.observability()["enable"][:N_DRONES]) == {True}


def test_solve_starts_from_the_device_poses_and_matches_the_host_tail():
    f = Flight(30)
    for k in range(30):
        f.keyframe(k, finish_init=k >= 5)
    f.s.graph_add_factors(np.array([0], np.int32), np.array([0], np.int32), np.array([1], np.int32),
                          np.zeros((1, _l.PAYLOAD_LEN)), np.array([0], np.uint8))
    got, want = f.rows(0.0, 0.0)
    same_rows(got, want)
    start = f.s.graph_get_poses()
    o = f.s.default_options()
    f.chain.solve(f.s, f.chain.factors.type.numel(), o)
    dev = f.s.graph_get_poses()
    assert f.s.last_summary() is not None
    f.s.graph_set_poses(0, start)                                       # the host form: same poses, same tail
    rows = host.FactorRows(f.chain.factors.type.numel())
    rows.set(want)
    rows.solve(f.s, f.chain.factors.type.numel(), o)
    torch.cuda.synchronize()
    assert f.s.graph_get_poses().tobytes() == dev.tobytes()
    assert not np.array_equal(dev, start)


def test_max_tail_overflow_refuses_the_solve():
    f = Flight(12)
    for k in range(12):
        f.keyframe(k, finish_init=k >= 3)
    f.s.graph_add_factors(np.array([0], np.int32), np.array([0], np.int32), np.array([1], np.int32),
                          np.zeros((1, _l.PAYLOAD_LEN)), np.array([0], np.uint8))
    got, want = f.rows(0.0, 0.0)
    n = len(want["ia"])
    assert n > 2
    f.window()
    c = f.chain
    c.compact(0, keep=False)
    c.distances(f.a, n - 1, SELF, distance_measurement_cov=PRM["distance_measurement_cov"])
    with torch.cuda.stream(c.stream):
        assert int(c.factors.count.cpu()[0]) == -1
    before = f.s.graph_get_poses()
    c.solve(f.s, n - 1, f.s.default_options())
    with pytest.raises(_l.OsbError):
        f.s.last_summary()
    assert f.s.graph_get_poses().tobytes() == before.tobytes()


def test_refusals_launches_and_no_synchronisation():
    f = Flight(4)
    st = f.chain.stream.cuda_stream
    kf = f.kfs[0]
    nodes, dists = kr.keyframe_records(kf, f.asg, SELF, False)
    f.s.graph_add_nodes(np.zeros((f.asg.next, 4)))
    bad = nodes.copy(); bad["drone_id"][0] = 99
    for args in ((bad, dists), (nodes[::-1].copy(), dists)):
        with pytest.raises(_l.OsbError):
            f.a.add_keyframe_dev(f.s, kf["stamp"], *args, st, SELF, False)
    bad = nodes.copy(); bad["block"][0] = 10_000
    with pytest.raises(_l.OsbError):
        f.a.add_keyframe_dev(f.s, kf["stamp"], bad, dists, st, SELF, False)
    with pytest.raises(_l.OsbError):                                    # no observe since create
        f.a.distance_factors_dev(f.chain.factors, 16, st, SELF)
    L = _l.load()
    assert L.osb_anchor_distance_factors_dev(None, None, None, None, None, None, None, None, 0, None) == _l.ERR_INVALID
    n0 = host.launch_count()
    s = torch.cuda.Stream()
    with torch.cuda.stream(s):
        torch.cuda._sleep(200_000_000)                                  # a bounded delay ahead of the call
        f.a.add_keyframe_dev(f.s, kf["stamp"], nodes, dists, s.cuda_stream, SELF, False, seed=SEED)
        ev = torch.cuda.Event()
        ev.record(s)
    assert not ev.query()                                               # the call returned before the sleep ended
    s.synchronize()
    assert host.launch_count() - n0 == 1
    with pytest.raises(_l.OsbError):                                    # the stamp is stored now
        f.a.add_keyframe_dev(f.s, kf["stamp"], nodes, dists, st, SELF, False)


def test_capture_follows_new_keyframes_and_enable():
    f = Flight(40)
    for k in range(20):
        f.keyframe(k, finish_init=k >= 5)
    f.rows(1e6, 1e6)                                                    # uncaptured first calls acquire everything
    c = f.chain
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=c.stream):
        c.observe(f.a, 0, SELF, 0.0, 0.0)
        c.compact(0, keep=False)
        c.distances(f.a, c.factors.type.numel(), SELF, distance_measurement_cov=PRM["distance_measurement_cov"])
    for k in range(20, 40, 5):
        for j in range(k, k + 5):
            f.keyframe(j, finish_init=True, check=False)
        win = f.window()
        with torch.cuda.stream(c.stream):
            g.replay()
        got = c.factors.on_host(c.stream)
        want = kr.distance_rows(win, f.store, f.a.observability()["enable"].tolist() + [False] * 248, PRM)
        same_rows(got, want)
        ref = f.rows(0.0, 0.0)[0]                                       # the same calls uncaptured
        same_rows(got, ref)


def test_threshold_edges_null_pointers_and_distance_launches():
    """the outlier threshold and minimum_distance at one ulp on the device (exact fp64 there, no transcendental
    decides), a null pointer refused at once, and one launch per distance_factors_dev"""
    a = host.LoopAnchor(8, 64, 64, 256, 1.0, 0.01, 0.01, max_keyframes=4)
    s = host.PoseGraphSolver(64, 256)
    s.graph_add_nodes(np.zeros((6, 4)))
    thr, md = float(np.float32(0.3)), float(np.float32(0.2))
    up = lambda x: float(np.nextafter(x, np.inf))                     # noqa: E731
    down = lambda x: float(np.nextafter(x, -np.inf))                  # noqa: E731
    d = [down(5.0 + thr), 5.0 + thr, up(5.0 + thr), down(md), md]    # node i + 1 -> peer 0
    want = [0, 0, 1, 1, 0]
    est = [5.0, 5.0, 5.0, down(md), md]                              # node i + 1's distance to node 0 (at the origin)
    nodes = np.zeros(6, _l.KEYFRAME_NODE_DTYPE)
    nodes["drone_id"] = nodes["block"] = np.arange(6)
    nodes["new_block"], nodes["prev_block"] = 1, -1
    nodes["vo_available"] = nodes["frame_available"] = nodes["dists_available"] = 1
    nodes["pose"][:, 3] = 1.0
    nodes["n_distances"][1:] = 1
    dists = np.zeros(5, _l.KEYFRAME_DISTANCE_DTYPE)
    dists["distance"] = d
    st = torch.cuda.current_stream().cuda_stream
    a.add_keyframe_dev(s, 1000, nodes, dists, st, SELF, False, **{k: PRM[k] for k in ("outlier_threshold",
                                                                                       "elevation_threshold",
                                                                                       "minimum_distance")})
    poses = np.zeros((6, 4))
    poses[1:, 0] = est
    s.graph_set_poses(0, poses)
    nodes["new_block"] = 0                                            # the same blocks: the resident poses decide
    a.add_keyframe_dev(s, 2000, nodes, dists, st, SELF, True, **{k: PRM[k] for k in ("outlier_threshold",
                                                                                      "elevation_threshold",
                                                                                      "minimum_distance")})
    got = a.keyframe_flags(2000)
    assert got.tolist() == want
    assert got.tolist() == kr.outlier_flags(nodes, dists, poses, nodes, dict(PRM, finish_init=True)).tolist()
    L = _l.load()
    p = _l.KeyframeParams(SELF, 1, 1, 0, 0.3, 0.5, 0.2, 0, 0)
    assert L.osb_anchor_add_keyframe_dev(a._h, s._h, 3000, 6, None, 5, _l.ptr(dists), ctypes.byref(p), None) == _l.ERR_INVALID
    assert L.osb_anchor_add_keyframe_dev(a._h, None, 3000, 6, _l.ptr(nodes), 5, _l.ptr(dists), ctypes.byref(p), None) \
        == _l.ERR_INVALID
    assert L.osb_anchor_add_keyframe_dev(a._h, s._h, 3000, 6, _l.ptr(nodes), 5, None, ctypes.byref(p), None) == _l.ERR_INVALID
    e = np.zeros(6, _l.WINDOW_ENTRY_DTYPE)
    e["drone_id"], e["block"], e["vo_available"], e["stamp"] = np.arange(6), np.arange(6), 1, 2000
    a.set_window([2000], np.array([0, 6], np.int32), e)
    rows = host.FactorRows(64)
    a.observe_dev(rows.type.data_ptr(), 0, st, SELF, -1.0, -1.0)   # self's empty extent passes: every node enabled
    rows.count.zero_()
    n0 = host.launch_count()
    a.distance_factors_dev(rows, 64, st, SELF)
    assert host.launch_count() - n0 == 1
    r = rows.on_host()
    assert r["ia"].tolist() == [1, 2, 5] and r["ib"].tolist() == [0, 0, 0]   # the flagged nodes 3 and 4 have none
