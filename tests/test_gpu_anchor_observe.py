"""GPU: the observability estimate of a solve on the device (osb_anchor_observe_dev / osb_anchor_observability) against
its oracle (oracle/observability_ref.py): rows rewritten to run_dev's with the oracle's yaw mask, byte for byte, and the
state and flags equal to the oracle's, over rounds in which drones join late and are linked one by one, with a VOID tail,
at 256 drones, with no row, under stream capture and on to the resident solve."""
import ctypes as C

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l, synth
from oracle import observability_ref as orf
from backend_harness import make_anchor, options, pcm_state, resident

pytestmark = pytest.mark.gpu
ROW = _l.ANCHOR_RESULT_DTYPE.itemsize
SELF = 0
XY, Z = 1.2, 0.5                         # init_xy_movement, init_z_movement
KEYS = ("nodes", "yaw", "pos", "enable", "to_init")


def shaped_window(g, drones, step, n_frames=None):
    """g's window restricted to `drones`: self_id moves `step` per frame on x and y and step / 2 on z, drone 4 keeps its
    flight (a box over 1 m), the others barely move (no box over 1 m)"""
    stamps, first, entries = g["window"]
    n_frames = len(stamps) if n_frames is None else n_frames
    frames = []
    for f in range(n_frames):
        e = entries[first[f]:first[f + 1]]
        e = e[np.isin(e["drone_id"], list(drones))].copy()
        e["self_pose"][:, :3] *= np.where(e["drone_id"] == 4, 1.0, 0.01)[:, None]
        e["self_pose"][e["drone_id"] == SELF, :3] = [step * f, step * f, 0.5 * step * f]
        frames.append(e)
    return (stamps[:n_frames].copy(), np.cumsum([0] + [len(e) for e in frames]).astype(np.int32), np.concatenate(frames))


def pairs_in(meas, links):
    key = {tuple(sorted(p)) for p in links}
    return np.array([tuple(sorted((int(a), int(b)))) in key for a, b in zip(meas["id_a"], meas["id_b"])], bool)


def rows_of(t, n):
    return np.frombuffer(t[:n * ROW].cpu().numpy().tobytes(), _l.ANCHOR_RESULT_DTYPE)


def same_outcome(got, want):
    for k in KEYS:
        assert np.array_equal(got[k], want[k]), k
    for k in ("solve_master", "motion", "motion_new"):
        assert got[k] == want[k], k


def device_rows(meas):
    return torch.from_numpy(np.ascontiguousarray(meas).view(np.uint8).copy()).cuda()


# per round: drones in the window, pairs a measurement may join, self_id's step per frame
ROUNDS = [({0, 1}, [(0, 0), (1, 1)], 0.005),
          ({0, 1, 2}, [(0, 1)], 0.01),
          ({0, 1, 2, 3, 4}, [(1, 2), (3, 4), (2, 2)], 0.02),
          ({0, 1, 2, 3, 4}, [], 0.04),                           # the self box crosses both thresholds
          ({0, 1, 2, 3, 4}, [(2, 3)], 0.05),
          ({0, 1, 2, 3, 4}, [(0, 4), (1, 3)], 0.06)]             # appended on the device


def test_rounds_match_the_oracle(gpu):
    g = synth.anchor_swarm(5, 40, 600, seed=13, with_orphans=False)
    D = g["max_drones"]
    a = make_anchor(g, max_meas=2048)
    for d, (s, p) in g["trajs"].items():
        a.push_odometry(d, s, p)
    ref = orf.ObservabilityRef(D)
    chain = host.AnchoredChain(2048)
    out = torch.zeros(2048 * ROW, dtype=torch.uint8, device="cuda")
    added = np.zeros(len(g["meas"]), bool)
    links, seen = [], {k: False for k in ("motion_off", "motion", "motion_new", "late", "masked", "void")}
    keep_alive = []
    for r, (drones, new_links, step) in enumerate(ROUNDS):
        links += new_links
        new = pairs_in(g["meas"], links) & ~added
        added |= new
        win = shaped_window(g, drones, step)
        a.set_window(*win)
        ref.set_window(*win)
        n_true = sum(a.size()) + int(new.sum())
        if r == len(ROUNDS) - 1:                                  # a device append: run_dev launches over its bound
            buf = device_rows(g["meas"][new])
            cnt = torch.tensor([int(new.sum())], dtype=torch.int32, device="cuda")
            keep_alive += [buf, cnt]
            torch.cuda.synchronize()
            torch.cuda._sleep(20_000_000)                         # the append has not run when run_dev sizes its grid
            a.add_measurements_dev(buf.data_ptr(), cnt.data_ptr(), int(new.sum()) + 40, 1e6,
                                   torch.cuda.current_stream().cuda_stream)
            chain.stream.wait_stream(torch.cuda.current_stream())
        else:
            a.add_measurements(g["meas"][new])
        n = chain.run(a, np.zeros(D, np.uint8))
        chain.observe(a, n, SELF, XY, Z)
        chain.stream.synchronize()
        got = rows_of(chain.rows, n)
        want = ref.observe(got[:n_true], SELF, XY, Z)
        same_outcome(a.observability(), want)
        # run_dev with the oracle's mask writes the same rows (its bound may have come down to the true count)
        st = torch.cuda.Stream()
        n2 = a.run_dev(out.data_ptr(), st.cuda_stream, want["yaw"].astype(np.uint8))
        st.synchronize()
        assert n_true <= n2 <= n and sum(a.size()) == n_true
        assert rows_of(out, n2).tobytes() == got[:n2].tobytes()
        void = np.zeros(n - n_true, _l.ANCHOR_RESULT_DTYPE)
        void["status"], void["skip"] = _l.ANCHOR_VOID, 1
        assert got[n_true:].tobytes() == void.tobytes()
        assert np.array_equal(got["skip"][:n_true], orf.skip(got[:n_true], want["yaw"]))
        ok = got["status"][:n_true] == _l.ANCHOR_OK
        seen["motion_off"] |= not want["motion"]
        seen["motion"] |= want["motion"]
        seen["motion_new"] |= want["motion_new"]
        seen["late"] |= bool(set(np.flatnonzero(want["to_init"])) - {SELF}) and not want["motion_new"]
        seen["masked"] |= bool((ok & (got["skip"][:n_true] == 1) & (got["node_a"][:n_true] != got["node_b"][:n_true])).any())
        seen["void"] |= n > n_true
    assert a.status() == _l.OK
    assert all(seen.values()), seen
    assert want["yaw"][:5].all() and want["solve_master"]
    a.close()


def window_of(drones, D):
    """one frame holding every drone of `drones` at rest"""
    e = np.zeros(len(drones), _l.WINDOW_ENTRY_DTYPE)
    e["drone_id"] = drones
    e["vo_available"] = 1
    e["block"] = np.arange(len(drones))
    e["stamp"] = 1000
    e["self_pose"][:, 3] = 1.0
    return np.array([1000], np.int64), np.array([0, len(drones)], np.int32), e


def hand_rows(specs):
    rows = np.zeros(len(specs), _l.ANCHOR_RESULT_DTYPE)
    for i, (status, x, y) in enumerate(specs):
        rows[i]["status"] = status
        rows[i]["edge"]["id_a"], rows[i]["edge"]["id_b"] = x, y
        rows[i]["node_a"], rows[i]["node_b"] = 2 * i, 2 * i + 1
        rows[i]["skip"] = 1
        rows[i]["payload"][:] = i
    return rows


def test_256_drones_word_boundaries_and_a_long_path(gpu):
    live0 = host.live_resources()
    D = 256
    a = host.LoopAnchor(D, 8, 8, 512, 1.0, 1e-3, 1e-3)
    win = window_of(np.arange(D), D)
    win[2]["self_pose"][win[2]["drone_id"] == 200, 0] = 5000.0        # one far sample: a box from the +-1000 start
    a.set_window(*win)
    ref = orf.ObservabilityRef(D)
    ref.set_window(*win)
    chain = host.AnchoredChain(4096)
    # n = 0: only the box rules act
    n0 = host.launch_count()
    chain.observe(a, 0, 255, XY, Z)
    assert host.launch_count() - n0 == 3
    want = ref.observe(hand_rows([]), 255, XY, Z)
    same_outcome(a.observability(), want)
    assert set(np.flatnonzero(want["yaw"])) == {200, 255} and set(np.flatnonzero(want["to_init"])) == {255}
    live = host.live_resources()
    # a path 255 -> 254 -> ... -> 150 (105 hops), branches to 63 / 64 / 127 / 128, rows that do not link, in shuffled order
    specs = [(_l.ANCHOR_OK, d, d - 1) for d in range(255, 150, -1)]
    specs += [(_l.ANCHOR_OK, 150, 128), (_l.ANCHOR_OK, 127, 128), (_l.ANCHOR_OK, 64, 127), (_l.ANCHOR_OK, 63, 63),
              (_l.ANCHOR_OK, 64, 63), (_l.ANCHOR_DPOS, 0, 255), (_l.ANCHOR_NO_FRAME, 1, 255), (_l.ANCHOR_VOID, 2, 255),
              (_l.ANCHOR_BEFORE_WINDOW, 3, 255), (_l.ANCHOR_OK, 5, 6)]
    specs = [specs[i] for i in np.random.default_rng(3).permutation(len(specs))] * 30
    rows = hand_rows(specs)
    for k in range(2):
        chain.upload(rows)
        n0 = host.launch_count()
        chain.observe(a, len(rows), 255, XY, Z)
        assert host.launch_count() - n0 == 3 and host.live_resources() == live
        want = ref.observe(rows, 255, XY, Z)
        same_outcome(a.observability(), want)
        got = rows_of(chain.rows, len(rows))
        expect = rows.copy()
        expect["skip"] = orf.skip(rows, want["yaw"])
        assert got.tobytes() == expect.tobytes()
        assert set(np.flatnonzero(want["yaw"])) == set(range(150, 256)) | {63, 64, 127, 128, 200}
        assert want["to_init"].sum() == (109 if k == 0 else 0)
    a.close()
    assert host.live_resources() == live0


def test_captured_chain_follows_the_window(gpu):
    """run_dev -> observe_dev -> reject_anchored -> compact_factors_dev captured once; drone 3 joins the window between
    replays, so its rows re-anchor OK, and the next replay links it to self_id and keeps its rows, with nothing recomputed
    on the host"""
    g = synth.anchor_swarm(5, 40, 400, seed=17, with_orphans=False)
    D = g["max_drones"]
    a = make_anchor(g, max_meas=1024)
    for d, (s, p) in g["trajs"].items():
        a.push_odometry(d, s, p)
    link = pairs_in(g["meas"], [(0, 1), (1, 3), (0, 0), (3, 3)])
    a.add_measurements(g["meas"][link])
    ref = orf.ObservabilityRef(D)
    st = pcm_state(g, 16, 1024)
    chain = host.AnchoredChain(1024)
    w_before, w_after = shaped_window(g, {0, 1, 2}, 0.005), shaped_window(g, {0, 1, 2, 3}, 0.005)
    a.set_window(*w_before)
    ref.set_window(*w_before)
    n = chain.run(a, np.zeros(D, np.uint8))                         # the first calls acquire, outside the capture
    chain.observe(a, n, SELF, XY, Z)
    chain.reject(st, n)
    chain.compact(n)
    chain.stream.synchronize()
    ref.observe(rows_of(chain.rows, n), SELF, XY, Z)
    live = host.live_resources()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=chain.stream, capture_error_mode="global"):
        n = chain.run(a, np.zeros(D, np.uint8))
        chain.observe(a, n, SELF, XY, Z)
        chain.reject(st, n)
        chain.compact(n)
    assert host.live_resources() == live
    for win, linked in ((w_before, False), (w_after, True)):
        a.run()                                   # re-records the run event, which the capture left recorded in the graph
        a.set_window(*win)
        ref.set_window(*win)
        graph.replay()
        chain.stream.synchronize()
        got = rows_of(chain.rows, n)
        want = ref.observe(got, SELF, XY, Z)
        same_outcome(a.observability(), want)
        assert want["yaw"][3] == linked and want["to_init"][3] == linked
        three = (got["status"] == _l.ANCHOR_OK) & ((got["edge"]["id_a"] == 3) | (got["edge"]["id_b"] == 3)) & \
            (got["node_a"] != got["node_b"])
        assert three.any() == linked and (got["skip"][three] == 0).all()
        assert np.array_equal(got["skip"], orf.skip(got, want["yaw"]))
    assert st.status() == _l.OK
    del graph
    for h in (st, a):
        h.close()


def test_the_solve_equals_the_oracle_mask_chain(gpu):
    """run_dev (no drone) -> observe_dev -> reject -> compact -> solve_resident_dev against run_dev with the oracle's mask
    -> reject -> compact -> solve on a twin: the same poses, bit for bit"""
    g = synth.anchor_swarm(5, 30, 400, seed=19, with_orphans=False)
    D = g["max_drones"]
    base = synth.anchor_window_graph(g)
    anchors = [make_anchor(g) for _ in range(2)]
    win = shaped_window(g, {0, 1, 2, 3, 4}, 0.005)
    link = pairs_in(g["meas"], [(0, 1), (1, 2), (3, 4), (0, 0), (2, 2), (3, 3)])
    for h in anchors:
        for d, (s, p) in g["trajs"].items():
            h.push_odometry(d, s, p)
        h.add_measurements(g["meas"][link])
        h.set_window(*win)
    ref = orf.ObservabilityRef(D)
    ref.set_window(*win)
    states = [pcm_state(g, 16, 1024) for _ in range(2)]
    solvers = [host.PoseGraphSolver(4096, 32768) for _ in range(2)]
    chains = [host.AnchoredChain(1024) for _ in range(2)]
    o = options(solvers[0], "tight")
    for s in solvers:
        resident(s, base)
    n = chains[0].run(anchors[0], np.zeros(D, np.uint8))
    chains[0].observe(anchors[0], n, SELF, XY, Z)
    chains[0].reject(states[0], n)
    chains[0].compact(n)
    chains[0].solve(solvers[0], 1024, o)
    chains[0].stream.synchronize()
    want = ref.observe(rows_of(chains[0].rows, n), SELF, XY, Z)
    assert not want["yaw"][3] and want["yaw"][1] and want["yaw"][4]    # 3 is neither linked nor moving
    chains[1](anchors[1], states[1], want["yaw"].astype(np.uint8))
    chains[1].solve(solvers[1], 1024, o)
    torch.cuda.synchronize()
    fa, fb = (c.factors.on_host(c.stream) for c in chains)
    assert len(fa["ftype"]) > 0 and all(fa[k].tobytes() == fb[k].tobytes() for k in fa)
    pa, pb = solvers[0].graph_get_poses(), solvers[1].graph_get_poses()
    assert pa.tobytes() == pb.tobytes() and not np.array_equal(pa, base["init"])
    for h in anchors + states + solvers:
        h.close()


def test_argument_errors_enqueue_nothing(gpu):
    L = _l.load()
    a = host.LoopAnchor(4, 8, 8, 8, 1.0, 1e-3, 1e-3)
    buf = torch.zeros(ROW, dtype=torch.uint8, device="cuda")
    p = C.c_void_p(buf.data_ptr())
    live, n0 = host.live_resources(), host.launch_count()

    def prm(self_id):
        return C.byref(_l.ObserveParams(self_id, 1.0, 1.0, 0))

    assert L.osb_anchor_observe_dev(None, prm(0), p, 1, None) == _l.ERR_INVALID
    assert L.osb_anchor_observe_dev(a._h, None, p, 1, None) == _l.ERR_INVALID
    assert L.osb_anchor_observe_dev(a._h, prm(0), None, 1, None) == _l.ERR_INVALID
    assert L.osb_anchor_observe_dev(a._h, prm(0), p, -1, None) == _l.ERR_INVALID
    assert L.osb_anchor_observe_dev(a._h, prm(-1), p, 1, None) == _l.ERR_INVALID
    assert L.osb_anchor_observe_dev(a._h, prm(4), p, 1, None) == _l.ERR_INVALID
    assert L.osb_anchor_observability(a._h, None) == _l.ERR_INVALID
    assert L.osb_anchor_observability(None, C.byref(_l.Observability())) == _l.ERR_INVALID
    assert host.launch_count() == n0 and host.live_resources() == live
    before = a.observability()                                       # nothing observed yet: all zero
    assert not any(before[k].any() for k in KEYS) and not before["solve_master"]
    a.close()
