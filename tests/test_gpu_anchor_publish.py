"""osb_anchor_sync_dev / osb_anchor_paths / osb_anchor_predict: what the back-end publishes after each accepted solve
(sync_est_poses and PredictSwarm), on the device after the solver's device call.  Against tests/publish_ref.py over
rounds of the real chain (run_dev -> observe -> compact -> solve_resident_dev or the multistart branch), rejected solves,
an init sync after steady ones, predict's conditions, the full path at 2e5 samples per drone, refusals, launch and
memory accounting, and one CUDA graph from run_dev through sync_dev against the same calls uncaptured."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l, synth
from oracle import anchor_ref as ar
import publish_ref as pb
from backend_harness import feed, make_anchor, options, resident
from test_publish_ref import SLICES, flight, frames_of

SELF, XY, Z, WIN = 0, 1.0, 0.3, 30


def scenario(n_drones=4, n_frames=24, seed=3):
    g = synth.anchor_swarm(n_drones, n_frames, 300, seed=seed, with_orphans=False)
    return g, synth.anchor_window_graph(g)


def close(got, want):
    return got.shape == want.shape and bool(np.all(np.abs(got - want) <= 1e-12 * np.maximum(1.0, np.abs(want))))


def check_paths(a, st, max_drones, full=True):
    for d in range(max_drones):
        for is_full, ref in ((False, st.kf), (True, st.full)):
            if is_full and not full:
                continue
            got = a.paths(d, is_full)
            if d not in ref:
                assert got is None, (d, is_full)
                continue
            assert got is not None and np.array_equal(got[0], ref[d][0]), (d, is_full)
            assert close(got[1], ref[d][1]), (d, is_full)


def check_predict(a, st, T, max_drones, finish_init=True):
    drones = np.arange(max_drones, dtype=np.int32)
    vo = np.stack([T[d].poses[len(T[d].poses) // 2] if d in T else np.r_[0, 0, 0, 1.0, 0, 0, 0] for d in drones])
    got = a.predict(drones, vo, SELF, finish_init)
    want = st.predict(list(zip(drones.tolist(), vo)), finish_init, SELF, a.observability()["enable"])
    for d in drones.tolist():
        w = want.get(d, (None, None))
        for x, y in zip(got[d], w):
            assert (x is None) == (y is None), d
            if x is not None:
                assert close(x, y), d


class Rig:
    """an anchor fed with scenario g, a solver holding its window graph, a chain, and the oracle's state"""

    def __init__(self, g, base, full=True):
        self.g, self.base, self.full = g, base, full
        self.a = make_anchor(g, max_meas=4096)
        feed(self.a, g)
        self.dev = host.PoseGraphSolver(4096, 32768)
        resident(self.dev, base)
        self.o = options(self.dev, "default")
        self.chain = host.AnchoredChain(4096)
        self.T = {int(d): ar.Trajectory(*v) for d, v in g["trajs"].items() if len(v[0])}
        self.st = pb.PublishState()
        self.n_nodes = len(base["init"])

    def solve(self, win, init, acpt, sync=True):
        """one solve() of window `win` through the chain, then sync_dev -> whether solve() accepts it (host rule)"""
        self.a.set_window(*win)
        c = self.chain
        n = c.run(self.a)
        c.observe(self.a, n, SELF, XY, Z)
        c.compact(n, keep=False)
        if init:
            c.init_mask(self.a, SELF, self.n_nodes)
            c.init_solve(self.dev, 4096, 3, 7, WIN, acpt, options=self.o)
        else:
            c.solve(self.dev, 4096, self.o)
        if sync:
            self.a.sync_dev(self.dev, c.stream.cuda_stream, SELF, acpt, WIN, True, self.full)
        c.stream.synchronize()
        if init:
            accepted = self.dev.last_multistart()[0] >= 0
        else:
            s = self.dev.last_summary()
            accepted = not (np.sqrt(s.final_cost) / s.n_residuals / WIN > acpt)
        if accepted and sync:
            self.st.sync(win, self.dev.graph_get_poses(), self.T, init, self.full)
        return accepted

    def close(self):
        for h in (self.a, self.dev):
            h.close()


@pytest.mark.gpu
def test_rounds_against_the_oracle(gpu):
    g, base = scenario()
    r = Rig(g, base)
    w = flight(g["window"])
    check_paths(r.a, r.st, g["max_drones"])                        # before any sync: no path
    check_predict(r.a, r.st, r.T, g["max_drones"])
    applied = []
    for lo, hi, init in SLICES:
        acc = r.solve(frames_of(w, lo, hi), init, np.inf)
        assert acc
        applied.append(r.a.sync_result())
        check_paths(r.a, r.st, g["max_drones"])
        check_predict(r.a, r.st, r.T, g["max_drones"])
        check_predict(r.a, r.st, r.T, g["max_drones"], finish_init=False)
    assert applied == [(True, _l.OK)] * len(SLICES)
    assert len(r.st.kf) >= 3 and 3 not in r.st.kf                  # drone 3 left the window
    shared = w[2]["block"]
    assert len(np.unique(shared)) < len(shared)                    # blocks shared by frames that did not move
    r.close()


@pytest.mark.gpu
def test_rejected_solves_change_nothing(gpu):
    g, base = scenario()
    r = Rig(g, base)
    w = flight(g["window"])
    assert r.solve(frames_of(w, 0, 12), True, np.inf)
    assert r.solve(frames_of(w, 2, 14), False, np.inf)
    before = {d: (r.a.paths(d), r.a.paths(d, True)) for d in range(g["max_drones"])}
    drones = np.arange(g["max_drones"], dtype=np.int32)
    vo = np.tile(np.r_[1.0, 2.0, 0.5, 1.0, 0, 0, 0], (len(drones), 1))
    pred = r.a.predict(drones, vo, SELF)
    for win, init in ((frames_of(w, 4, 16), False), (frames_of(w, 5, 17), True)):   # over acpt_cost; no trial chosen
        assert not r.solve(win, init, 1e-300)
        assert r.a.sync_result() == (False, _l.OK)
        for d in range(g["max_drones"]):
            for x, y in zip((r.a.paths(d), r.a.paths(d, True)), before[d]):
                assert (x is None) == (y is None)
                if x is not None:
                    assert np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
        got = r.a.predict(drones, vo, SELF)
        assert all(all((p is None and q is None) or np.array_equal(p, q) for p, q in zip(got[d], pred[d])) for d in got)
    check_paths(r.a, r.st, g["max_drones"])                        # the oracle did not sync either
    r.close()


@pytest.mark.gpu
def test_long_full_path_and_disabled(gpu):
    g, base = scenario(5, 20, seed=5)
    n_long = 200_000
    g2 = dict(g)
    rng = np.random.default_rng(2)
    trajs = {}
    for d, (s, p) in g["trajs"].items():                           # the flight continues after the window
        k = n_long - len(s)
        st = s[-1] + 10_000_000 * np.arange(1, k + 1, dtype=np.int64)
        pos = p[-1, :3] + np.cumsum(rng.normal(0, 0.01, (k, 3)), axis=0)
        q = p[-1, 3:] + rng.normal(0, 0.02, (k, 4))
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        trajs[d] = (np.concatenate([s, st]), np.concatenate([p, np.c_[pos, q]]))
    g2["trajs"] = trajs
    r = Rig(g2, base, full=False)
    assert r.solve(g["window"], True, np.inf)
    check_paths(r.a, r.st, g["max_drones"], full=False)
    assert all(r.a.paths(d, True) is None for d in range(g["max_drones"]))   # disabled: no full path
    r.a.sync_dev(r.dev, r.chain.stream.cuda_stream, SELF, np.inf, WIN, True, True)
    r.chain.stream.synchronize()
    for d, (s, p) in trajs.items():
        got = r.a.paths(d, True)
        want = pb.full_path_vec(r.st.kf[d], s, p)
        assert len(got[0]) == 20_000 and np.array_equal(got[0], want[0]) and close(got[1], want[1])
    r.close()


@pytest.mark.gpu
def test_refusals_launches_and_memory(gpu):
    live0 = host.live_resources()
    g, base = scenario()
    r = Rig(g, base)
    w = flight(g["window"])
    sync = lambda **k: r.a.sync_dev(r.dev, r.chain.stream.cuda_stream, k.get("self_id", SELF), k.get("acpt", np.inf),
                                    k.get("win", WIN), True, True)        # noqa: E731
    with pytest.raises(_l.OsbError) as e:                          # no device call yet
        sync()
    assert e.value.status == _l.ERR_INVALID
    assert r.solve(frames_of(w, 0, 12), True, np.inf)
    live1 = host.live_resources()
    n0 = host.launch_count()
    sync()
    assert host.launch_count() - n0 == 3 and host.live_resources() == live1
    n0 = host.launch_count()
    for bad in (dict(self_id=-1), dict(self_id=g["max_drones"]), dict(win=0), dict(acpt=float("nan"))):
        with pytest.raises(_l.OsbError) as e:
            sync(**bad)
        assert e.value.status == _l.ERR_INVALID
    L = _l.load()
    p = _l.SyncParams(SELF, 1, 1, WIN, np.inf)
    import ctypes as C
    assert L.osb_anchor_sync_dev(None, r.dev._h, C.byref(p), None) == _l.ERR_INVALID
    assert L.osb_anchor_sync_dev(r.a._h, None, C.byref(p), None) == _l.ERR_INVALID
    assert L.osb_anchor_sync_dev(r.a._h, r.dev._h, None, None) == _l.ERR_INVALID
    r.dev.graph_set_poses(0, r.dev.graph_get_poses(0, 1))          # a host-side pose change
    with pytest.raises(_l.OsbError):
        sync()
    assert host.launch_count() == n0
    assert r.solve(frames_of(w, 2, 14), False, np.inf)            # a window block beyond the solver's nodes
    big = frames_of(w, 2, 14)
    big[2]["block"][-1] = r.n_nodes
    r.a.set_window(*big)
    n0 = host.launch_count()
    with pytest.raises(_l.OsbError):
        sync()
    assert host.launch_count() == n0
    r.close()
    # a window drone without odometry: refused on the device, nothing changes
    g3 = synth.anchor_swarm(4, 24, 300, seed=3, with_orphans=True)
    r3 = Rig(g3, synth.anchor_window_graph(g3))
    w3 = g3["window"]
    e3 = [w3[2][w3[1][f]:w3[1][f + 1]] for f in range(len(w3[0]))]
    e3 = [x[x["drone_id"] != 4] for x in e3]
    no_orphan = (w3[0], np.cumsum([0] + [len(x) for x in e3]).astype(np.int32), np.concatenate(e3))
    assert r3.solve(no_orphan, True, np.inf)
    before = [r3.a.paths(d) for d in range(g3["max_drones"])]
    assert r3.solve(w3, False, np.inf, sync=False)
    r3.a.sync_dev(r3.dev, r3.chain.stream.cuda_stream, SELF, np.inf, WIN, True, True)
    assert r3.a.sync_result() == (False, _l.ERR_INVALID)
    after = [r3.a.paths(d) for d in range(g3["max_drones"])]
    assert all((x is None and y is None) or (np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1]))
               for x, y in zip(before, after))
    r3.close()
    del r, r3
    torch.cuda.synchronize()
    assert host.live_resources() == live0


@pytest.mark.gpu
def test_capture_from_run_to_sync(gpu):
    g, base = scenario()
    w = flight(g["window"])
    extra = {d: (s[-1] + 10_000_000 * np.arange(1, 41, dtype=np.int64), np.repeat(p[-1:], 40, axis=0))
             for d, (s, p) in g["trajs"].items()}

    def step(r):
        c = r.chain
        n = c.run(r.a)
        c.observe(r.a, n, SELF, XY, Z)
        c.compact(n, keep=False)
        c.solve(r.dev, 4096, r.o)
        r.a.sync_dev(r.dev, c.stream.cuda_stream, SELF, np.inf, WIN, True, True)

    def state(r):
        drones = np.arange(g["max_drones"], dtype=np.int32)
        vo = np.tile(np.r_[1.0, 2.0, 0.5, 1.0, 0, 0, 0], (len(drones), 1))
        out = [r.a.sync_result()]
        for d in drones.tolist():
            out += [r.a.paths(d), r.a.paths(d, True)]
        pred = r.a.predict(drones, vo, SELF)
        return out, pred

    def same(x, y):
        if isinstance(x, tuple) and len(x) == 2 and isinstance(x[0], np.ndarray):
            return y is not None and np.array_equal(x[0], y[0]) and np.array_equal(x[1], y[1])
        return x == y

    ref, cap = Rig(g, base), Rig(g, base)
    for r in (ref, cap):
        assert r.solve(frames_of(w, 0, 12), True, np.inf)
        r.a.set_window(*frames_of(w, 1, 13))
        step(r)                                                    # warm: the steady path's host work
        r.chain.stream.synchronize()
        r.dev.last_summary()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=cap.chain.stream, capture_error_mode="global"):
        step(cap)
    for k, (lo, hi) in enumerate(((2, 14), (3, 15), (5, 17))):
        for r in (ref, cap):
            for d, (s, p) in extra.items():
                r.a.push_odometry(d, s[10 * k:10 * k + 10], p[10 * k:10 * k + 10])
            r.a.set_window(*frames_of(w, lo, hi))
        step(ref)
        ref.chain.stream.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        (o1, p1), (o2, p2) = state(ref), state(cap)
        assert o1[0] == o2[0] == (True, _l.OK)
        assert all(same(x, y) for x, y in zip(o1[1:], o2[1:]))
        assert all(all((a is None and b is None) or np.array_equal(a, b) for a, b in zip(p1[d], p2[d])) for d in p1)
        n_odom = len(g["trajs"][0][0]) + 10 * (k + 1)              # the replay read the odometry pushed before it
        assert len(o2[2][0]) == (n_odom + 9) // 10
    ref.close()
    cap.close()
