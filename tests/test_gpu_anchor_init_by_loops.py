"""osb_anchor_record_loops_dev / osb_anchor_init_by_loops_dev: the loop map of every solve and the pre-motion init start
(init_pose_by_loops) on the device.  Over rounds of the pre-motion branch (run_dev -> record_loops -> observe ->
reject_anchored -> compact -> distance_factors -> init_by_loops -> multistart with one trial and no scattered block ->
sync_dev) on a swarm that has not moved, in both PCM modes, with set_inliers sets, a window slide and a drone joining:
the poses against tests/init_by_loops_ref.py, the loop map and the estimated flags identical, an accepted round
bit-identical to the host-start round, refusals, launches, resources, no synchronisation, and the whole branch as one
CUDA graph against the same calls uncaptured."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l, synth
import init_by_loops_ref as ib
from backend_harness import feed, make_anchor, options, pcm_state, resident
from test_publish_ref import flight, frames_of

SELF, XY, Z, WIN = 0, 1e6, 1e6, 30           # movement thresholds no flight reaches: the swarm is not initialised by motion
ROUNDS = [(0, 8), (0, 10), (1, 12), (3, 14), (5, 16)]           # drone 2 joins at frame 10


def scenario(seed=3):
    g = synth.anchor_swarm(4, 24, 300, seed=seed, with_orphans=False)
    return g, synth.anchor_window_graph(g)


def close(got, want):
    return got.shape == want.shape and bool(np.all(np.abs(got - want) <= 1e-12 * np.maximum(1.0, np.abs(want))))


class Rig:
    """an anchor fed with scenario g, a PCM state, a solver holding its window graph, a chain, and the oracle's map"""

    def __init__(self, g, base, redundant=True):
        self.g = g
        self.a = make_anchor(g, max_meas=4096)
        feed(self.a, g)
        self.pcm = pcm_state(g, 16, 512, SELF, redundant)
        self.dev = host.PoseGraphSolver(4096, 32768)
        resident(self.dev, base)
        self.o = options(self.dev, "default")
        self.chain = host.AnchoredChain(4096)
        self.n_nodes = len(base["init"])
        self.lmap = ib.LoopMapVec(g["max_drones"], _l.LOOP_RECORD_DTYPE)
        self.book = ib.LoopBook(SELF, redundant)
        self.estimated = set()

    def front(self, win):
        """set_window, then the branch up to the distance rows -> the row count"""
        self.a.set_window(*win)
        c = self.chain
        n = c.run(self.a)
        c.record_loops(self.a, n)
        c.observe(self.a, n, SELF, XY, Z)
        c.reject(self.pcm, n)
        c.compact(n)
        c.distances(self.a, 4096, SELF)
        return n

    def back(self, host_start=None):
        """init_by_loops (or the given start written from the host), the one-trial multistart, sync_dev"""
        c = self.chain
        if host_start is None:
            c.init_by_loops(self.a, self.pcm, self.dev, SELF, self.n_nodes)
        else:                                                      # today's adapter path: the start from the host
            if c.mask is None or c.mask.numel() < self.n_nodes:
                c.mask = torch.zeros(self.n_nodes, dtype=torch.uint8, device="cuda")
                c.yaw = torch.zeros(self.n_nodes, dtype=torch.float64, device="cuda")
            torch.cuda.synchronize()
            c.stream.synchronize()
            self.dev.graph_set_poses(0, host_start)
        c.init_solve(self.dev, 4096, 1, 7, WIN, np.inf, options=self.o)
        self.a.sync_dev(self.dev, c.stream.cuda_stream, SELF, np.inf, WIN, True, False)

    def rows(self, n):
        with torch.cuda.stream(self.chain.stream):
            raw = self.chain.rows[:n * _l.ANCHOR_RESULT_DTYPE.itemsize].cpu().numpy()
        return raw.view(_l.ANCHOR_RESULT_DTYPE)

    def oracle_inputs(self, win):
        D = self.g["max_drones"]
        good = {}
        for a in range(D):
            for b in range(a, D):
                s = self.pcm.inliers(a, b)
                if s is not None:
                    good[(a, b)] = s
        kf = {d: p for d in range(D) if (p := self.a.paths(d)) is not None}
        est = set(self.estimated)
        if np.any(win[2]["drone_id"] == SELF):
            est.add(SELF)
        to_init = self.a.observability()["to_init"]
        return good, kf, est, to_init

    def close(self):
        for h in (self.a, self.pcm, self.dev):
            h.close()


def round_against_oracle(r, win):
    n = r.front(win)
    rows = r.rows(n)
    r.book.record(rows)
    r.lmap.record_vec(rows)
    before = r.dev.graph_get_poses()
    good, kf, est, to_init = r.oracle_inputs(win)
    r.chain.init_by_loops(r.a, r.pcm, r.dev, SELF, r.n_nodes)
    got = r.dev.graph_get_poses()
    D = r.g["max_drones"]
    est_mask = np.isin(np.arange(D), list(est))
    want = ib.init_by_loops_vec(to_init, good, r.lmap, est_mask, kf, r.g["trajs"], SELF, win, before)
    lit = ib.init_pose_by_loops(set(np.nonzero(to_init)[0].tolist()), ib.good_from_sets(good), r.book, est, kf,
                                ib.Trajs(r.g["trajs"]), SELF, win, before)
    assert close(want, lit)
    assert r.a.init_by_loops_result() == _l.OK
    assert close(got, want)
    m = r.a.loop_map()
    for f in r.lmap.recs.dtype.names:
        assert np.array_equal(m["records"][f], r.lmap.recs[f]), f
    assert np.array_equal(m["pair_min"], r.lmap.pair_min)
    assert set(np.nonzero(m["estimated"])[0].tolist()) == r.estimated
    r.chain.init_solve(r.dev, 4096, 1, 7, WIN, np.inf, options=r.o)
    r.a.sync_dev(r.dev, r.chain.stream.cuda_stream, SELF, np.inf, WIN, True, False)
    applied, st = r.a.sync_result()
    assert st == _l.OK
    if applied:
        r.estimated |= set(np.unique(win[2]["drone_id"]).tolist())
    return to_init, got, before


@pytest.mark.gpu
@pytest.mark.parametrize("redundant", [True, False])
def test_rounds_against_the_oracle(gpu, redundant):
    g, base = scenario()
    r = Rig(g, base, redundant)
    w = flight(g["window"])
    placed = 0
    for k, (lo, hi) in enumerate(ROUNDS):
        if k == 3:                                                 # inlier sets received from another drone
            rows = r.lmap.recs
            r.pcm.set_inliers(1, 3, rows["id"][((rows["id_a"] == 1) & (rows["id_b"] == 3)) |
                                               ((rows["id_a"] == 3) & (rows["id_b"] == 1))][:2])
            r.pcm.set_inliers(2, 3, [])
        to_init, got, before = round_against_oracle(r, frames_of(w, lo, hi))
        placed += int(to_init.any() and not np.array_equal(got, before))
    assert placed >= 1
    assert len(r.lmap.recs) > 0 and r.estimated >= {0, 1, 2}
    r.close()


@pytest.mark.gpu
def test_accepted_round_is_bit_identical_to_a_host_start(gpu):
    g, base = scenario()
    w = flight(g["window"])
    dev, hst = Rig(g, base), Rig(g, base)
    for lo, hi in ROUNDS[:3]:
        win = frames_of(w, lo, hi)
        for r in (dev, hst):
            r.front(win)
        dev.chain.init_by_loops(dev.a, dev.pcm, dev.dev, SELF, dev.n_nodes)
        start = dev.dev.graph_get_poses()
        dev.chain.init_solve(dev.dev, 4096, 1, 7, WIN, np.inf, options=dev.o)
        dev.a.sync_dev(dev.dev, dev.chain.stream.cuda_stream, SELF, np.inf, WIN, True, False)
        hst.back(host_start=start)
        for r in (dev, hst):
            r.chain.stream.synchronize()
        c1, c2 = dev.dev.last_multistart()[0], hst.dev.last_multistart()[0]
        assert c1 == c2 == 0
        assert np.array_equal(dev.dev.graph_get_poses(), hst.dev.graph_get_poses())
        assert dev.a.sync_result() == hst.a.sync_result() == (True, _l.OK)
    dev.close()
    hst.close()


@pytest.mark.gpu
def test_refusals_launches_resources_and_no_synchronisation(gpu):
    live0 = host.live_resources()
    g, base = scenario()
    r = Rig(g, base)
    w = flight(g["window"])
    win = frames_of(w, 0, 8)
    fresh = pcm_state(g, 16, 512, SELF, True)
    r.a.set_window(*win)
    with pytest.raises(_l.OsbError) as e:                          # no observe yet
        r.a.init_by_loops_dev(r.pcm, r.dev, SELF, r.chain.stream.cuda_stream)
    assert e.value.status == _l.ERR_INVALID
    n = r.front(win)
    n0 = host.launch_count()
    with pytest.raises(_l.OsbError) as e:                          # a PCM state without a device copy
        r.a.init_by_loops_dev(fresh, r.dev, SELF, r.chain.stream.cuda_stream)
    assert e.value.status == _l.ERR_INVALID
    for bad in (-1, g["max_drones"]):
        with pytest.raises(_l.OsbError):
            r.a.init_by_loops_dev(r.pcm, r.dev, bad, r.chain.stream.cuda_stream)
    with pytest.raises(_l.OsbError):
        r.a.record_loops_dev(r.chain.rows.data_ptr(), -1, r.chain.stream.cuda_stream)
    assert host.launch_count() == n0
    r.back()                                                       # the first calls acquire
    r.chain.stream.synchronize()
    assert r.a.init_by_loops_result() == _l.OK
    live1 = host.live_resources()
    torch.cuda.synchronize()
    with torch.cuda.stream(r.chain.stream):                        # the calls return while the stream is busy
        torch.cuda._sleep(1_000_000_000)
    n0 = host.launch_count()
    r.chain.record_loops(r.a, n)
    assert host.launch_count() - n0 == 2
    n0 = host.launch_count()
    r.chain.init_by_loops(r.a, r.pcm, r.dev, SELF, r.n_nodes)
    assert host.launch_count() - n0 == 1
    assert not r.chain.stream.query()
    r.chain.stream.synchronize()
    assert host.live_resources() == live1
    # a set whose smallest id is not in the loop map: refused on the device, every pose unchanged
    r2 = Rig(g, base, redundant=True)
    n = r2.front(win)
    r2.chain.stream.synchronize()
    to_init = r2.a.observability()["to_init"]
    d = int(np.nonzero(to_init & (np.arange(len(to_init)) != SELF))[0][0])
    other = next(x for x in np.unique(win[2]["drone_id"]).tolist() if x not in (SELF, d))
    r2.pcm.set_inliers(d, other, [-5])                             # -5: no row carries it
    before = r2.dev.graph_get_poses()
    # with self_id = other, `other` is estimated (it has a keyframe in the window), so d's set (d, other) qualifies
    r2.chain.init_by_loops(r2.a, r2.pcm, r2.dev, other, r2.n_nodes)
    assert r2.a.init_by_loops_result() == _l.ERR_INVALID
    assert np.array_equal(r2.dev.graph_get_poses(), before)
    for h in (r, r2):
        h.close()
    fresh.close()
    del r, r2, fresh
    torch.cuda.synchronize()
    assert host.live_resources() == live0


@pytest.mark.gpu
def test_capture_of_the_pre_motion_branch(gpu):
    g, base = scenario()
    w = flight(g["window"])
    extra = {d: (s[-1] + 10_000_000 * np.arange(1, 41, dtype=np.int64), np.repeat(p[-1:], 40, axis=0))
             for d, (s, p) in g["trajs"].items()}

    def step(r):
        c = r.chain
        n = c.run(r.a)
        c.record_loops(r.a, n)
        c.observe(r.a, n, SELF, XY, Z)
        c.reject(r.pcm, n)
        c.compact(n)
        c.distances(r.a, 4096, SELF)
        r.back()

    def state(r):
        D = g["max_drones"]
        m = r.a.loop_map()
        return ([r.a.sync_result(), r.a.init_by_loops_result(), r.dev.graph_get_poses()] +
                [m["records"].tobytes(), m["pair_min"], m["estimated"]] + [r.a.paths(d) for d in range(D)])

    def same(x, y):
        if isinstance(x, tuple) and len(x) == 2 and isinstance(x[0], np.ndarray):
            return y is not None and np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
        if isinstance(x, np.ndarray):
            return np.array_equal(x, y)
        return x == y

    ref, cap = Rig(g, base), Rig(g, base)
    for r in (ref, cap):
        r.front(frames_of(w, 0, 8))
        r.back()
        r.chain.stream.synchronize()
        r.dev.last_multistart()
        r.a.set_window(*frames_of(w, 0, 10))
        step(r)                                                    # warm: every first call is behind
        r.chain.stream.synchronize()
        r.dev.last_multistart()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=cap.chain.stream, capture_error_mode="global"):
        step(cap)
    for k, (lo, hi) in enumerate(((1, 11), (1, 12), (2, 12))):
        for r in (ref, cap):
            for d, (s, p) in extra.items():
                r.a.push_odometry(d, s[10 * k:10 * k + 10], p[10 * k:10 * k + 10])
            r.a.set_window(*frames_of(w, lo, hi))
        step(ref)
        ref.chain.stream.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        s1, s2 = state(ref), state(cap)
        assert s1[0] == s2[0] and s1[1] == s2[1] == _l.OK
        assert all(same(x, y) for x, y in zip(s1[2:], s2[2:]))
    ref.close()
    cap.close()
