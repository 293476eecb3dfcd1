"""The whole solve() chain with the UWB half on the device, against the same chain with the poses, flags and distance rows
built on the host from tests/keyframe_ref.py:
  add_keyframe_dev -> run_dev -> observe_dev -> reject_anchored -> compact_factors_dev -> distance_factors_dev ->
  solve_multistart_resident_dev (init branch) or solve_resident_dev (steady) -> sync_dev,
over 100 keyframes with the window sliding at 50 frames, and the same chain captured into one CUDA graph and replayed
after new keyframes and a flipped enable, against the calls uncaptured.

The host form reads the device's initial poses of predicted blocks only after checking them against the oracle to
1e-12 relative (the yaw algebra's atan2 / sin / cos are CUDA's on the device and glibc's in numpy); every other start,
every flag and every distance row it builds itself.  From there each solve's poses, rows and published paths must match
bit for bit."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l
from oracle import pnp_ref as pn, pcm_ref as pr
import keyframe_ref as kr

pytestmark = pytest.mark.gpu
SELF, N_DRONES, WIN, SEED, CAP = 0, 6, 50, 11, 8192
PRM = dict(outlier_threshold=0.3, elevation_threshold=0.5, minimum_distance=0.2, enable_distance=True,
           debug_no_rejection=False, distance_measurement_cov=0.2, self_id=SELF)
KF_ARGS = {k: PRM[k] for k in ("outlier_threshold", "elevation_threshold", "minimum_distance")}


def flight(n_kf):
    """keyframes, their node records (blocks assigned, finish_init from keyframe 10), the odometry factors between a
    drone's consecutive blocks, and loops between the drones of every keyframe"""
    kfs = kr.random_keyframes(N_DRONES, n_kf, SEED, self_id=SELF, late=(4,), static=(5,))
    asg = kr.BlockAssigner()
    recs, odo, meas, last = [], [], [], {}
    rng = np.random.default_rng(5)
    for k, kf in enumerate(kfs):
        nodes, dists = kr.keyframe_records(kf, asg, SELF, k >= 10)
        recs.append((nodes, dists))
        for nd in nodes:
            d, b = int(nd["drone_id"]), int(nd["block"])
            if d in last and last[d][0] != b:
                dp = pn.delta_pose(last[d][1], nd["pose"], True)
                pl = np.zeros(_l.PAYLOAD_LEN)
                pl[:4] = [dp[0], dp[1], dp[2], kr.yaw(dp[3:])]
                pl[4:20] = (10.0 * np.eye(4)).ravel()
                odo.append((k, last[d][0], b, pl))
            last[d] = (b, np.array(nd["pose"]))
        ids = [int(d) for d in kf["drones"]]
        for i in range(1, len(ids)):
            if rng.random() < 0.5:
                continue
            m = np.zeros(1, _l.MEASUREMENT_DTYPE)[0]
            m["id"], m["type"], m["id_a"], m["id_b"] = len(meas), _l.MEAS_LOOP, ids[0], ids[i]
            m["stamp_a"] = m["stamp_b"] = kf["stamp"]
            pa, pb = np.asarray(kf["poses"][0]), np.asarray(kf["poses"][i])
            m["relative_pose"] = pr.pose_mul(pr.pose_inv(pa), pb) + np.r_[rng.normal(0, 0.02, 3), 0, 0, 0, 0]
            m["cov"] = np.diag([0.01] * 3 + [0.003] * 3)
            m["self_pose_a"], m["self_pose_b"] = pa, pb
            meas.append(m)
    return kfs, recs, odo, np.array(meas, _l.MEASUREMENT_DTYPE), asg.next


class Rig:
    """one back-end: anchor, PCM state, solver and chain; form "dev" runs the UWB half on the device, "host" on the
    host from the oracle"""

    def __init__(self, form, kfs, meas, stream=None):
        self.form = form
        self.a = host.LoopAnchor(8, 4096, 4096, 4096, 1.0, 0.01, 0.01, max_keyframes=128)
        self.pcm = host.PcmState(SELF, True, 15.0, 0.01, 0.01, max_pairs=36, pair_capacity=512)
        self.s = host.PoseGraphSolver(4096, 32768)
        self.chain = host.AnchoredChain(CAP, stream)
        self.frames, self.store, self.last, self.n_blocks = [], {}, None, 0
        for d in range(N_DRONES):                                      # odometry and loops up front: all on the device
            st = [kf["stamp"] for kf in kfs if d in kf["drones"]]
            po = [kf["poses"][kf["drones"].index(d)] for kf in kfs if d in kf["drones"]]
            if st:
                self.a.push_odometry(d, st, po)
        self.a.add_measurements(meas)

    def add_blocks(self, n_total, odo):
        if n_total > self.n_blocks:
            first = self.s.graph_add_nodes(np.zeros((n_total - self.n_blocks, 4)))
            if first == 0:
                self.s.graph_set_fixed(0, True)
            self.n_blocks = n_total
        if odo:
            self.s.graph_add_factors(np.full(len(odo), 1, np.int32), np.array([o[1] for o in odo], np.int32),
                                     np.array([o[2] for o in odo], np.int32), np.stack([o[3] for o in odo]),
                                     np.zeros(len(odo), np.uint8))

    def keyframe(self, kf, nodes, dists, finish_init, dev_poses=None):
        if self.form == "dev":
            self.a.add_keyframe_dev(self.s, kf["stamp"], nodes, dists, self.chain.stream.cuda_stream, SELF, finish_init,
                                    seed=SEED, **KF_ARGS)
            flags = self.a.keyframe_flags(kf["stamp"])
        else:
            before = self.s.graph_get_poses()
            want = kr.init_poses(nodes, before, kf["stamp"], SELF, finish_init, SEED)
            new = nodes[nodes["new_block"] != 0]
            pred = new[(new["prev_block"] >= 0) & (new["is_static"] == 0) & ((new["drone_id"] != SELF) | finish_init)]
            scale = np.maximum(1.0, np.abs(want[pred["block"]]))
            assert np.all(np.abs(dev_poses[pred["block"]] - want[pred["block"]]) <= 1e-12 * scale)
            want[pred["block"]] = dev_poses[pred["block"]]
            assert want.tobytes() == dev_poses.tobytes()              # every other start is the oracle's, bit for bit
            self.s.graph_set_poses(0, want)
            flags = kr.outlier_flags(nodes, dists, want, self.last, dict(PRM, finish_init=finish_init))
        self.store[kf["stamp"]] = (nodes, dists, flags)
        self.last = nodes
        self.frames.append((kf["stamp"], nodes))
        return flags

    def window(self):
        fr = self.frames[-WIN:]
        first = np.concatenate([[0], np.cumsum([len(n) for _, n in fr])]).astype(np.int32)
        ent = np.zeros(int(first[-1]), _l.WINDOW_ENTRY_DTYPE)
        for (ts, n), lo in zip(fr, first):
            e = ent[lo:lo + len(n)]
            e["drone_id"], e["block"], e["vo_available"], e["stamp"], e["self_pose"] = (
                n["drone_id"], n["block"], n["vo_available"], ts, n["pose"])
        self.a.set_window([ts for ts, _ in fr], first, ent)
        return [(ts, {int(x["drone_id"]): int(x["block"]) for x in n}) for ts, n in fr]

    def chain_calls(self, xy, init, win=None):
        """run -> observe -> reject -> compact -> distances (dev) -> solve or init solve -> sync, on the chain's stream"""
        c = self.chain
        n = c.run(self.a)
        c.observe(self.a, n, SELF, xy, xy)
        c.reject(self.pcm, n)
        c.compact(n)
        if self.form == "dev":
            c.distances(self.a, CAP, SELF, distance_measurement_cov=PRM["distance_measurement_cov"])
        else:                                                          # the host tail: the loop rows + the oracle's
            rows = c.factors.on_host(c.stream)
            enable = list(self.a.observability()["enable"]) + [False] * 248
            dist = kr.distance_rows(win, self.store, enable, PRM)
            with torch.cuda.stream(c.stream):
                c.factors.set({k: np.concatenate([rows[k], dist[k]]) for k in host.FACTOR_KEYS})
        if init:
            c.init_mask(self.a, SELF, self.n_blocks)
            c.init_solve(self.s, CAP, 3, 7, WIN, 1e9)
        else:
            c.solve(self.s, CAP, self.s.default_options())
        self.a.sync_dev(self.s, c.stream.cuda_stream, SELF, 1e9, WIN, full_path=True)

    def outcome(self):
        torch.cuda.synchronize()
        paths = [self.a.paths(d, full) for d in range(N_DRONES) for full in (False, True)]
        return self.s.graph_get_poses(), self.chain.factors.on_host(self.chain.stream), paths


def same(x, y):
    px, rx, ax = x
    py, ry, ay = y
    assert px.tobytes() == py.tobytes()
    for k in host.FACTOR_KEYS:
        assert np.asarray(rx[k]).tobytes() == np.asarray(ry[k]).tobytes(), k
    for p, q in zip(ax, ay):
        assert (p is None) == (q is None) and (p is None or (p[0].tobytes() == q[0].tobytes() and
                                                             p[1].tobytes() == q[1].tobytes()))


def test_chain_against_the_host_built_tail():
    kfs, recs, odo, meas, _ = flight(100)
    dev, hst = Rig("dev", kfs, meas), Rig("host", kfs, meas)
    n_solves = n_init = 0
    for k, kf in enumerate(kfs):
        nodes, dists = recs[k]
        blocks = max(int(nodes["block"].max()) + 1, dev.n_blocks)
        for r in (dev, hst):
            r.add_blocks(blocks, [o for o in odo if o[0] == k])
        f_dev = dev.keyframe(kf, nodes, dists, k >= 10)
        f_hst = hst.keyframe(kf, nodes, dists, k >= 10, dev_poses=dev.s.graph_get_poses())
        assert np.array_equal(f_dev, f_hst), k
        if k % 5 == 4:
            init = k < 10
            xy = 1e6 if k < 40 else 0.0                                 # enable flips at keyframe 44
            for r in (dev, hst):
                win = r.window()
                r.chain_calls(xy, init, win)
            same(dev.outcome(), hst.outcome())
            n_solves += 1
            n_init += init
    assert n_solves == 20 and n_init == 2
    assert any(p is not None for p in dev.outcome()[2])


def test_one_graph_from_run_to_sync():
    kfs, recs, odo, meas, n_total = flight(45)
    a, b = Rig("dev", kfs, meas), Rig("dev", kfs, meas)
    for r in (a, b):                                                    # every block and odometry factor up front:
        r.add_blocks(n_total, odo)                                      # a captured solve needs a fixed topology
    for k in range(18):
        for r in (a, b):
            r.keyframe(kfs[k], *recs[k], k >= 10)
    for r in (a, b):
        r.window()
        r.chain_calls(1e6, False)                                       # uncaptured first calls acquire everything
    same(a.outcome(), b.outcome())
    c = a.chain
    g = torch.cuda.CUDAGraph()
    with torch.cuda.graph(g, stream=c.stream):
        a.chain_calls(1e6, False)
    enable0 = a.a.observability()["enable"].copy()
    for k in range(18, 45):
        for r in (a, b):
            r.keyframe(kfs[k], *recs[k], True)
        if k % 3 == 2:
            for r in (a, b):
                r.window()
            with torch.cuda.stream(c.stream):
                g.replay()
            b.chain_calls(1e6, False)
            same(a.outcome(), b.outcome())
    assert not np.array_equal(a.a.observability()["enable"], enable0)   # the late drone's loops flipped its enable
