"""The back-end's per-drone kernels (anchor.cu) at the sizes they are built for: 256 drone ids across the four 64-bit words
of a drone set, keyframes of 256 nodes and 4096 distances (16 passes of the keyframe kernel's stride, four tiles of the
distance rows), a keyframe store that wraps several times, a one-slot store, and the re-anchoring's tie and threshold
rules on hand-built stamps.  Every device result is checked against the float64 oracles (oracle/anchor_ref.py,
oracle/observability_ref.py, tests/init_mask_ref.py, tests/publish_ref.py, tests/keyframe_ref.py), and every scenario
asserts that it reaches the pass, tile, wrap or word it is there for.  The CPU test pins the literal oracle forms to the
numpy forms the GPU tests use, at these shapes."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l, synth
from oracle import anchor_ref as ar, observability_ref as orf
import init_mask_ref as mr
import keyframe_ref as kr
import publish_ref as pb
from backend_harness import feed, options, resident
from test_gpu_anchor import check, close

NS = ar.NS
ROW = _l.ANCHOR_RESULT_DTYPE.itemsize
IDS = (0, 1, 31, 32, 63, 64, 65, 127, 128, 191, 192, 200, 254, 255)   # both sides of every word boundary
CLEARED = (32, 127, 191, 254)                                          # one yaw-unobservable drone per word
SELF_HI = 200
XY, Z = 1.0, 0.3


def relabel(g, ids):
    """synth.anchor_swarm scenario g with drone d renamed ids[d] (a monotone map, so every order is kept) and room for
    256 drones"""
    m = np.asarray(ids, np.int32)
    stamps, first, entries = g["window"]
    assert np.all(np.diff(m) > 0) and len(m) > max(max(g["trajs"]), int(entries["drone_id"].max()))
    entries = entries.copy()
    entries["drone_id"] = m[entries["drone_id"]]
    meas = g["meas"].copy()
    meas["id_a"], meas["id_b"] = m[meas["id_a"]], m[meas["id_b"]]
    return dict(g, trajs={int(m[d]): v for d, v in g["trajs"].items()}, window=(stamps, first, entries), meas=meas,
                max_drones=256)


def without(win, drone):
    """window `win` with every entry of `drone` removed"""
    stamps, first, entries = win
    fr = [entries[first[f]:first[f + 1]] for f in range(len(stamps))]
    fr = [e[e["drone_id"] != drone] for e in fr]
    return stamps, np.cumsum([0] + [len(e) for e in fr]).astype(np.int32), np.concatenate(fr)


def frames_of(win, lo, hi):
    stamps, first, entries = win
    fr = [entries[first[f]:first[f + 1]] for f in range(lo, hi)]
    return stamps[lo:hi].copy(), np.cumsum([0] + [len(e) for e in fr]).astype(np.int32), np.concatenate(fr)


def rows_of(t, n):
    return np.frombuffer(t[:n * ROW].cpu().numpy().tobytes(), _l.ANCHOR_RESULT_DTYPE)


def near(got, want):
    return got.shape == want.shape and bool(np.all(np.abs(got - want) <= 1e-12 * np.maximum(1.0, np.abs(want))))


# ---- 1. sparse high ids through run -> observe -> init_mask -> sync -> paths / predict ---------------------------------
@pytest.mark.gpu
@pytest.mark.parametrize("with_255", [True, False])
def test_sparse_high_ids_through_the_chain(gpu, with_255):
    g = relabel(synth.anchor_swarm(14, 26, 700, seed=21, with_orphans=False), IDS)
    if not with_255:
        g["window"] = without(g["window"], 255)
    win = g["window"]
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    max_full = 8 * sms + 64                              # more full-path slots per drone than sync_full_kernel's grid covers
    a = host.LoopAnchor(256, 10 * max_full, len(g["meas"]) + 64, len(win[2]) + 64, g["prm"]["det_dpos_thres"],
                        g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"], g["prm"]["begin_min_loop_dt_s"])
    feed(a, g)

    # run / run_dev against the literal walk, a yaw mask with one drone cleared in every word
    yaw = np.ones(256, np.uint8)
    yaw[list(CLEARED)] = 0
    res = a.run(yaw)
    ref = ar.anchor(g["trajs"], win, g["meas"], yaw, g["prm"])
    check(res, ref)
    ok = ref["status"] == ar.OK
    ia, ib = ref["edge"]["id_a"], ref["edge"]["id_b"]
    for w in range(4):
        mine = ok & ((ia >> 6 == w) | (ib >> 6 == w))
        cleared = (ia == CLEARED[w]) | (ib == CLEARED[w])
        assert (mine & (ref["skip"] == 0)).any(), w
        assert (cleared & ok & (ref["skip"] == 1) & (ref["node_a"] != ref["node_b"])).any(), w
    hit_255 = (g["meas"]["id_a"] == 255) | (g["meas"]["id_b"] == 255)
    assert hit_255.any()
    assert ok[np.isin(ref["id"], g["meas"]["id"][hit_255])].any() == with_255
    out = torch.zeros(len(res) * ROW, dtype=torch.uint8, device="cuda")
    st = torch.cuda.Stream()
    assert a.run_dev(out.data_ptr(), st.cuda_stream, yaw) == len(res)
    st.synchronize()
    assert out.cpu().numpy().tobytes() == res.tobytes()

    # the chain: an init solve over frames 6..25 (blocks past 255 among them), then a steady one over frames 10..25
    base = synth.anchor_window_graph(g)
    n_nodes = len(base["init"])
    assert n_nodes > 256                                 # init_mask_kernel runs more than one CTA
    dev = host.PoseGraphSolver(4096, 32768)
    resident(dev, base)
    o = options(dev, "default")
    chain = host.AnchoredChain(len(g["meas"]) + 64)
    obs = orf.ObservabilityRef(256)
    T = {d: ar.Trajectory(*v) for d, v in g["trajs"].items()}
    pub = pb.PublishState()
    drones = np.arange(256, dtype=np.int32)
    vo_now = np.stack([T[d].poses[len(T[d].poses) // 2] if d in T else np.r_[0, 0, 0, 1.0, 0, 0, 0] for d in range(256)])
    for lo, hi, init in ((6, 26, True), (10, 26, False)):
        sub = frames_of(win, lo, hi)
        a.set_window(*sub)
        obs.set_window(*sub)
        n = chain.run(a)
        chain.observe(a, n, SELF_HI, XY, Z)
        chain.compact(n, keep=False)
        if init:
            chain.init_mask(a, SELF_HI, n_nodes)
            chain.init_solve(dev, len(g["meas"]) + 64, 3, 7, 30, np.inf, options=o)
        else:
            chain.solve(dev, len(g["meas"]) + 64, o)
        a.sync_dev(dev, chain.stream.cuda_stream, SELF_HI, np.inf, 30, True, True)
        chain.stream.synchronize()
        rows = rows_of(chain.rows, n)
        want = obs.observe(rows, SELF_HI, XY, Z)
        got = a.observability()
        for k in ("nodes", "yaw", "pos", "enable", "to_init"):
            assert np.array_equal(got[k], want[k]), k
        assert np.array_equal(rows["skip"], orf.skip(rows, want["yaw"]))
        if init:
            assert set(np.flatnonzero(want["to_init"])) - {SELF_HI} and want["to_init"][192:].any()
            with torch.cuda.stream(chain.stream):
                mask, ymask = chain.mask[:n_nodes].cpu().numpy(), chain.yaw[:n_nodes].cpu().numpy()
            wm, wy = mr.init_mask(sub[1], sub[2], want["to_init"], SELF_HI, n_nodes)
            assert np.array_equal(mask, wm)
            close(ymask, wy)
            assert wm[256:].any() and not wm[sub[2]["block"][sub[2]["drone_id"] == SELF_HI]].any()
            assert dev.last_multistart()[0] >= 0
        assert a.sync_result() == (True, _l.OK)
        pub.sync(sub, dev.graph_get_poses(), T, init, True)
        assert (255 in pub.kf) == with_255 and 254 in pub.full
        for d in range(256):                             # every drone's keyframe and full path
            for full, paths in ((False, pub.kf), (True, pub.full)):
                p = a.paths(d, full)
                assert (p is None) == (d not in paths), (d, full)
                if p is not None:
                    assert np.array_equal(p[0], paths[d][0]) and near(p[1], paths[d][1]), (d, full)
        pred = a.predict(drones, vo_now, SELF_HI)
        wpred = pub.predict(list(zip(drones.tolist(), vo_now)), True, SELF_HI, got["enable"])
        for d in range(256):
            for x, y in zip(pred[d], wpred[d]):
                assert (x is None) == (y is None), d
                if x is not None:
                    assert near(x, y), d
        assert pred[200][1] is not None and (pred[255][1] is not None) == with_255
    grid = min(-(-256 * max_full // 256), 8 * sms)       # sync_full_kernel's launch: drone 254's slots are on a later pass
    assert 254 * max_full >= grid * 256
    dev.close()
    a.close()


# ---- 2. the re-anchoring's ties and thresholds on exact stamps -------------------------------------------------------
@pytest.mark.gpu
def test_reanchoring_ties_and_thresholds_by_hand(gpu):
    """two drones whose odometry steps 0.25 m along x once a second (every length exact in fp64), a window of 40 frames at
    samples 10..49 holding both; each measurement sits on one rule"""
    T0 = 1_700_000_000 * NS
    K, F0, NF = 100, 10, 40
    stamps = T0 + NS * np.arange(K, dtype=np.int64)
    poses = np.zeros((K, 7))
    poses[:, 0] = 0.25 * np.arange(K)
    poses[:, 3] = 1.0
    trajs = {0: (stamps, poses), 1: (stamps, poses.copy())}
    fs = stamps[F0:F0 + NF]
    e = np.zeros(2 * NF, _l.WINDOW_ENTRY_DTYPE)
    e["drone_id"] = np.tile([0, 1], NF)
    e["block"] = np.arange(2 * NF)
    e["vo_available"] = 1
    e["stamp"] = np.repeat(fs, 2)
    e["self_pose"] = np.repeat(poses[F0:F0 + NF], 2, axis=0)
    win = (fs, np.arange(0, 2 * NF + 1, 2, dtype=np.int32), e)
    begin_dt_ns = 17_250_000_000
    prm = dict(begin_min_loop_dt_s=17.25, det_dpos_thres=3.0, odom_pos_cov_per_m=1e-3, odom_ang_cov_per_m=2e-4, huber=True)
    at = lambda k: int(T0 + k * NS)                                    # noqa: E731  odometry sample k
    fr = lambda f: int(fs[f])                                          # noqa: E731  frame f (= sample 10 + f)
    half = NS // 2
    OK, NO_FRAME, BEFORE, DPOS = ar.OK, ar.NO_FRAME, ar.BEFORE_WINDOW, ar.DPOS
    # (id_a, id_b, stamp_a, stamp_b) -> (status, frame_a, frame_b, dpos)
    cases = [
        ((0, 1, fr(31) + half, fr(5)), (OK, 31, 5, 0.0)),              # equidistant frames: lane 31 against the next pass
        ((0, 1, fr(32) + half, fr(5)), (OK, 32, 5, 0.0)),              # ... lanes 0 and 1 of the second pass
        ((0, 1, fr(5), fr(31) + half), (OK, 5, 31, 0.0)),              # b's entries start at 40, the lanes as a's
        ((0, 1, fr(0) + half, fr(5)), (OK, 0, 5, 0.0)),
        ((0, 1, at(55) + half, fr(0)), (OK, NF - 1, 0, 1.5)),          # midway between samples 55 and 56: 55
        ((0, 1, at(8) + half, fr(39)), (OK, 0, NF - 1, 0.5)),          # midway between samples 8 and 9: 8
        ((0, 1, T0 - 5 * NS, fr(0)), (OK, 0, 0, 2.5)),                 # before the first sample: sample 0
        ((0, 1, at(130), fr(39)), (DPOS, NF - 1, NF - 1, 12.5)),       # after the last sample: sample 99
        ((0, 1, fr(39), at(120)), (DPOS, NF - 1, NF - 1, 12.5)),
        ((0, 1, fr(39) + 10000 * NS, fr(0)), (NO_FRAME, -1, 0, 0.0)),  # the 10000 s bound is strict
        ((0, 1, fr(39) + 10000 * NS - 1, fr(0)), (DPOS, NF - 1, 0, 12.5)),
        ((0, 1, fr(0) - begin_dt_ns, fr(0)), (OK, 0, 0, 2.5)),         # frame0 - stamp_a > begin_dt is strict
        ((0, 1, fr(0) - begin_dt_ns - 1, fr(0)), (BEFORE, -1, -1, 0.0)),
        ((0, 1, at(56), at(54)), (OK, NF - 1, NF - 1, 3.0)),           # dpos > det_dpos_thres is strict
        ((0, 1, at(56), at(55)), (DPOS, NF - 1, NF - 1, 3.25)),
        ((0, 0, fr(7), fr(7)), (OK, 7, 7, 0.0)),                       # a == b on one block: no factor
        ((0, 0, fr(7), fr(9)), (OK, 7, 9, 0.0)),
    ]
    m = np.zeros(len(cases), _l.MEASUREMENT_DTYPE)
    for i, ((ida, idb, sa, sb), _) in enumerate(cases):
        m[i]["id"], m[i]["type"], m[i]["id_a"], m[i]["id_b"], m[i]["stamp_a"], m[i]["stamp_b"] = i, ar.LOOP, ida, idb, sa, sb
        m[i]["relative_pose"][3] = m[i]["self_pose_a"][3] = m[i]["self_pose_b"][3] = 1.0
        m[i]["cov"] = np.diag([0.01, 0.012, 0.02, 1e-3, 1e-3, 2e-3])
    a = host.LoopAnchor(4, K, 64, 2 * NF, prm["det_dpos_thres"], prm["odom_pos_cov_per_m"], prm["odom_ang_cov_per_m"],
                        prm["begin_min_loop_dt_s"])
    for d, (s, p) in trajs.items():
        a.push_odometry(d, s, p)
    a.add_measurements(m)
    a.set_window(*win)
    res = a.run()
    ref = ar.anchor(trajs, win, m, np.ones(4, np.uint8), prm)
    check(res, ref)
    for i, (_, (status, fa, fb, dpos)) in enumerate(cases):
        assert (res["status"][i], res["frame_a"][i], res["frame_b"][i]) == (status, fa, fb), i
        assert res["dpos"][i] == dpos, i
    same = (res["status"] == OK) & (res["node_a"] == res["node_b"])
    assert same.tolist() == [i == len(cases) - 2 for i in range(len(cases))]
    assert (res["skip"] == ~((res["status"] == OK) & ~same)).all()
    a.close()


# ---- 3 and 4. keyframes of 256 nodes and 4096 distances, and a store that wraps ---------------------------------------
PRM = dict(outlier_threshold=0.3, elevation_threshold=0.5, minimum_distance=0.2, enable_distance=True,
           debug_no_rejection=False, distance_measurement_cov=0.2, self_id=SELF_HI)
KF_PRM = {k: PRM[k] for k in ("outlier_threshold", "elevation_threshold", "minimum_distance")}
SEED = 5


def trim(nodes, dists, n):
    """the keyframe cut after its first n distances"""
    nodes = nodes.copy()
    first = np.concatenate([[0], np.cumsum(nodes["n_distances"])])
    nodes["n_distances"] = np.clip(n - first[:-1], 0, nodes["n_distances"])
    return nodes, dists[:n].copy()


def entries_of(nodes, stamp):
    e = np.zeros(len(nodes), _l.WINDOW_ENTRY_DTYPE)
    e["drone_id"], e["block"], e["vo_available"], e["stamp"] = nodes["drone_id"], nodes["block"], nodes["vo_available"], stamp
    e["self_pose"] = nodes["pose"]
    return e


class Flight:
    """256 drones, each node with 16 peers: a LoopAnchor with a max_keyframes ring, a solver that gains one node per new
    block, a chain, and the oracle's record of every keyframe stored"""

    def __init__(self, n_kf, max_keyframes, trims=None, late=(3, 130, 255), static=(2, 129), cap=32768):
        self.kfs = kr.random_keyframes(256, n_kf, SEED, self_id=SELF_HI, late=late, static=static, max_peers=16)
        self.a = host.LoopAnchor(256, 8, 8, 256 * 8, 1.0, 0.01, 0.01, max_keyframes=max_keyframes,
                                 max_keyframe_distances=4096)
        self.s = host.PoseGraphSolver(256 * (n_kf + 2), 64)
        self.chain = host.AnchoredChain(cap)
        self.asg = kr.BlockAssigner()
        self.trims = trims or {}
        self.frames, self.store, self.last, self.n_blocks = [], {}, None, 0
        self.n_dists = []

    def records(self, k, finish_init):
        nodes, dists = kr.keyframe_records(self.kfs[k], self.asg, SELF_HI, finish_init)
        if k in self.trims:
            nodes, dists = trim(nodes, dists, self.trims[k])
        grow = self.asg.next - self.n_blocks
        if grow:
            self.s.graph_add_nodes(np.zeros((grow, 4)))
            self.n_blocks = self.asg.next
        return nodes, dists

    def keyframe(self, k, finish_init, recs=None):
        """add keyframe k (recs: its records, already built); its initial poses and flags against the oracle"""
        kf = self.kfs[k]
        nodes, dists = self.records(k, finish_init) if recs is None else recs
        before = self.s.graph_get_poses()
        self.a.add_keyframe_dev(self.s, kf["stamp"], nodes, dists, self.chain.stream.cuda_stream, SELF_HI, finish_init,
                                seed=SEED, **KF_PRM)
        after = self.s.graph_get_poses()
        close(after, kr.init_poses_vec(nodes, before, kf["stamp"], SELF_HI, finish_init, SEED))
        flags = self.a.keyframe_flags(kf["stamp"])
        want = kr.outlier_flags_vec(nodes, dists, after, self.last, dict(PRM, finish_init=finish_init))
        assert flags.tobytes() == want.tobytes(), k
        self.store[kf["stamp"]] = (nodes, dists, flags)
        self.last = nodes
        self.frames.append((kf["stamp"], nodes))
        self.n_dists.append(len(dists))
        return nodes, dists

    def window(self, lo, hi):
        fr = self.frames[lo:hi]
        first = np.concatenate([[0], np.cumsum([len(n) for _, n in fr])]).astype(np.int32)
        ent = np.concatenate([entries_of(n, ts) for ts, n in fr]) if fr else np.zeros(0, _l.WINDOW_ENTRY_DTYPE)
        self.a.set_window([ts for ts, _ in fr], first, ent)
        return [(ts, {int(x["drone_id"]): int(x["block"]) for x in n}) for ts, n in fr]

    def rows(self, win, xy, max_tail=None):
        """observe (no loop rows) -> compact -> distance_factors_dev -> (device rows, oracle rows)"""
        c = self.chain
        c.observe(self.a, 0, SELF_HI, xy, xy)
        c.compact(0, keep=False)
        c.distances(self.a, c.factors.type.numel() if max_tail is None else max_tail, SELF_HI,
                    distance_measurement_cov=PRM["distance_measurement_cov"])
        got = c.factors.on_host(c.stream)
        want = kr.distance_rows_vec(win, self.store, self.a.observability()["enable"], PRM)
        return got, want

    def close(self):
        for h in (self.a, self.s):
            h.close()


def same_rows(got, want):
    for k in host.FACTOR_KEYS:
        assert np.asarray(got[k]).tobytes() == np.asarray(want[k]).tobytes(), k


def kept_k(win, store, enable, prm):
    """the distance index k (within its keyframe) of every row distance_rows_vec gives, in row order"""
    out = []
    en = np.asarray(enable, bool).copy()
    en[prm["self_id"]] = True
    for ts, blocks in win:
        nodes, dists, flags = store[ts]
        blk = np.full(256, -1)
        for d, b in blocks.items():
            blk[d] = b
        owner = np.repeat(np.arange(len(nodes)), nodes["n_distances"])
        a, b = nodes["drone_id"][owner], dists["peer"]
        ok = ((nodes["frame_available"][owner] != 0) & (nodes["dists_available"][owner] != 0) & en[a] & (blk[a] >= 0)
              & (b < a) & (blk[b] >= 0) & (flags != 1))
        out.append(np.flatnonzero(ok))
    return np.concatenate(out)


@pytest.mark.gpu
def test_keyframes_of_256_nodes_and_4096_distances(gpu):
    """late and static drones, finish_init from keyframe 3, keyframes cut at 255 / 256 / 257 and 1023 / 1024 / 1025
    distances; rows of 3-frame windows; max_tail at, below and inside the third tile; a 4097-distance keyframe refused"""
    trims = {1: 255, 2: 256, 4: 257, 6: 1023, 7: 1024, 8: 1025}
    f = Flight(11, 128, trims)
    n_rows = []
    for k in range(11):
        nodes, dists = f.keyframe(k, finish_init=k >= 3)
        if k >= 2:
            win = f.window(k - 2, k + 1)
            got, want = f.rows(win, 1e6 if k < 5 else -1.0)          # self_id's box: no motion, then motion enables all
            same_rows(got, want)
            n_rows.append(len(want["ia"]))
    assert f.n_dists == [16 * 253, 255, 256, 16 * 253, 257, 4096, 1023, 1024, 1025, 4096, 4096]   # up to 16 passes
    assert len(f.frames[10][1]) == 256 and len(f.frames[0][1]) == 253             # the late drones join at 5
    assert min(n_rows) > 0 and max(n_rows) > 3 * 1024                            # several distance tiles per solve

    # max_tail on a one-frame window of 4096 distances
    win = f.window(10, 11)
    got, want = f.rows(win, -1.0)
    same_rows(got, want)
    n = len(want["ia"])
    ks = kept_k(win, f.store, f.a.observability()["enable"], PRM)
    cut = int(np.flatnonzero(ks >= 2048)[0]) + 5                                 # the cut falls in the third tile
    assert len(ks) == n and 2048 <= ks[cut] < 3072
    c = f.chain
    for tail, count in ((n, n), (n - 1, -1), (cut, -1)):
        c.factors.ia.fill_(-7)
        c.stream.wait_stream(torch.cuda.current_stream())
        c.compact(0, keep=False)
        c.distances(f.a, tail, SELF_HI, distance_measurement_cov=PRM["distance_measurement_cov"])
        c.stream.synchronize()
        assert int(c.factors.count.cpu()[0]) == count, tail
        ia = c.factors.ia.cpu().numpy()
        m = min(tail, n)
        assert np.array_equal(ia[:m], want["ia"][:m]) and (ia[m:n + 1] == -7).all(), tail
        assert np.array_equal(c.factors.ib.cpu().numpy()[:m], want["ib"][:m])
        assert c.factors.payload.cpu().numpy()[:m * _l.PAYLOAD_LEN].tobytes() == want["payload"][:m].tobytes()

    # 4097 distances: refused before anything is stored
    kf = dict(f.kfs[10], stamp=f.kfs[10]["stamp"] + 250_000_000)
    nodes, dists = kr.keyframe_records(kf, kr.BlockAssigner(), SELF_HI, True)
    nodes["block"] = nodes["drone_id"]
    assert len(dists) == 4096 and nodes["n_distances"][-1] == 16
    last = nodes["drone_id"][-1]
    extra = np.zeros(1, kr.DIST_DTYPE)
    extra["peer"], extra["distance"] = last - 1, 3.0
    assert dists["peer"][-1] < last - 1
    dists = np.concatenate([dists, extra])
    nodes["n_distances"][-1] += 1
    flags_before = {ts: f.a.keyframe_flags(ts).tobytes() for ts in f.store}
    poses_before = f.s.graph_get_poses()
    with pytest.raises(_l.OsbError) as e:
        f.a.add_keyframe_dev(f.s, kf["stamp"], nodes, dists, c.stream.cuda_stream, SELF_HI, True, seed=SEED, **KF_PRM)
    assert e.value.status == _l.ERR_CAPACITY
    assert f.a.keyframe_flags(kf["stamp"]) is None
    assert {ts: f.a.keyframe_flags(ts).tobytes() for ts in f.store} == flags_before
    assert f.s.graph_get_poses().tobytes() == poses_before.tobytes()
    got, want = f.rows(f.window(8, 11), -1.0)
    same_rows(got, want)
    f.close()


@pytest.mark.gpu
def test_the_keyframe_ring_wraps(gpu):
    """max_keyframes = the window length (3) over 11 keyframes: the window slides before each keyframe, so the slot it
    takes holds a keyframe that has left; rows against the oracle after every keyframe.  Then a keyframe added while the
    oldest stored one is still in the window is refused and changes nothing."""
    W = 3
    f = Flight(11, W)
    for k in range(11):
        if k >= W:
            f.window(k - W + 1, k)                                    # the oldest keyframe leaves the window first
        f.keyframe(k, finish_init=k >= 3)
        win = f.window(max(0, k - W + 1), k + 1)
        got, want = f.rows(win, -1.0)
        same_rows(got, want)
        assert len(want["ia"]) > 0
    assert len(f.frames) >= 3 * W + 2                                 # three wraps and more
    assert all(f.a.keyframe_flags(ts) is None for ts, _ in f.frames[:-W])
    # the window still holds the slot's keyframe: refused, nothing changes
    f.kfs.append(dict(f.kfs[-1], stamp=f.kfs[-1]["stamp"] + 500_000_000))
    nodes, dists = f.records(11, True)
    poses = f.s.graph_get_poses()
    flags = {ts: f.a.keyframe_flags(ts).tobytes() for ts, _ in f.frames[-W:]}
    with pytest.raises(_l.OsbError) as e:
        f.a.add_keyframe_dev(f.s, f.kfs[11]["stamp"], nodes, dists, f.chain.stream.cuda_stream, SELF_HI, True, seed=SEED,
                             **KF_PRM)
    assert e.value.status == _l.ERR_CAPACITY
    assert f.s.graph_get_poses().tobytes() == poses.tobytes()
    assert {ts: f.a.keyframe_flags(ts).tobytes() for ts, _ in f.frames[-W:]} == flags
    got, want = f.rows(f.window(8, 11), -1.0)
    same_rows(got, want)
    # after the slide the same keyframe is taken, its flags read the last keyframe
    f.window(9, 11)
    f.keyframe(11, finish_init=True, recs=(nodes, dists))
    got, want = f.rows(f.window(9, 12), -1.0)
    same_rows(got, want)
    f.close()


@pytest.mark.gpu
def test_one_slot_store(gpu):
    """max_keyframes = 1 with a one-frame window: each keyframe reads the last one's nodes from the slot it then
    overwrites, so the flags after finish_init depend on that read"""
    f = Flight(8, 1)
    differs = 0
    for k in range(8):
        f.window(0, 0)                                                # the slot's keyframe leaves the window
        prev = f.last
        nodes, _ = f.keyframe(k, finish_init=k >= 2)
        got, want = f.rows(f.window(k, k + 1), -1.0)
        same_rows(got, want)
        if k >= 2:                                                    # the previous keyframe decides: not this one
            self_read = kr.outlier_flags_vec(nodes, f.store[f.frames[k][0]][1], f.s.graph_get_poses(), nodes,
                                             dict(PRM, finish_init=True))
            differs += int(self_read.tobytes() != f.store[f.frames[k][0]][2].tobytes())
            assert prev is not None
    assert differs >= 3
    assert all(f.a.keyframe_flags(ts) is None for ts, _ in f.frames[:-1])
    f.close()


# ---- 5. the literal oracle forms against the numpy forms at these shapes (CPU) -----------------------------------------
def test_literal_oracles_equal_the_numpy_forms_at_scale():
    # the re-anchoring: 14 sparse ids up to 255, one cleared per word
    g = relabel(synth.anchor_swarm(14, 12, 250, seed=21, with_orphans=False), IDS)
    yaw = np.ones(256, np.uint8)
    yaw[list(CLEARED)] = 0
    r1 = ar.anchor(g["trajs"], g["window"], g["meas"], yaw, g["prm"])
    r2 = ar.anchor_vec(g["trajs"], g["window"], g["meas"], yaw, g["prm"])
    for k in ("id", "status", "frame_a", "frame_b", "node_a", "node_b", "stamp_a", "stamp_b", "dt_err_ns", "skip", "ia", "ib"):
        assert np.array_equal(r1[k], r2[k]), k
    assert np.array_equal(r1["dpos"], r2["dpos"])
    np.testing.assert_allclose(r2["payload"], r1["payload"], rtol=1e-12, atol=1e-12)
    assert (r1["status"] == ar.OK).sum() > 50 and (r1["edge"]["id_a"] >= 192).any()
    # the keyframe oracle: 256 nodes, 4096 distances, self_id 200, finish_init switching on
    kfs = kr.random_keyframes(256, 5, SEED, self_id=SELF_HI, late=(3, 255), static=(2, 129), max_peers=16)
    asg = kr.BlockAssigner()
    poses = np.zeros((256 * 5, 4))
    last, store, written = None, {}, False
    for k, kf in enumerate(kfs):
        fi = k >= 2
        nodes, dists = kr.keyframe_records(kf, asg, SELF_HI, fi)
        p1 = kr.init_poses(nodes, poses, kf["stamp"], SELF_HI, fi, SEED)
        assert p1.tobytes() == kr.init_poses_vec(nodes, poses, kf["stamp"], SELF_HI, fi, SEED).tobytes()
        poses = p1
        prm = dict(PRM, finish_init=fi)
        f1 = kr.outlier_flags(nodes, dists, poses, last, prm)
        assert f1.tobytes() == kr.outlier_flags_vec(nodes, dists, poses, last, prm).tobytes(), k
        store[kf["stamp"]] = (nodes, dists, f1)
        written |= bool((f1[256:] != -1).any())
        last = nodes
    assert len(dists) == 4096 and len(nodes) == 256 and written
    win = [(ts, {int(x["drone_id"]): int(x["block"]) for x in n}) for ts, (n, _, _) in store.items()]
    enable = np.random.default_rng(1).random(256) < 0.7
    d1, d2 = kr.distance_rows(win, store, enable, PRM), kr.distance_rows_vec(win, store, enable, PRM)
    for k in d1:
        assert d1[k].tobytes() == d2[k].tobytes(), k
    assert len(d1["ia"]) > 1024
    # the full path: the literal walk against the nearest-sample form, for drone 255's odometry
    st, ps = g["trajs"][255]
    T = ar.Trajectory(st, ps)
    kf_st = g["window"][0][::3]
    kf = (kf_st, np.stack([ps[T.nearest(t)] for t in kf_st]), np.stack([ps[T.nearest(t) - 7] for t in kf_st]))
    l1, l2 = pb.full_path(kf, T), pb.full_path_vec(kf, st, ps)
    assert np.array_equal(l1[0], l2[0]) and np.allclose(l1[1], l2[1], rtol=0, atol=1e-12)
