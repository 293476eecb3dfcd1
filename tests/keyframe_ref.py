"""ORACLE (test infrastructure, NOT product code) -- float64 restatement of the UWB half of add_new_swarm_frame and of
every solve's distance factors (osb_anchor_add_keyframe_dev / osb_anchor_distance_factors_dev).

Follows (paths relative to the reference's swarm_localization/src):
  * init_dynamic_nf_in_keyframe / init_static_nf_in_keyframe  swarm_localization_solver.cpp:272-339, with Predict_By_VO
      (:104-106): est_last * DeltaPose(last_vo, now_vo, yaw_only), the noisy start of a drone without an earlier block,
      self_id's odometry before finish_init;
  * the block assignment the caller keeps (:279-298, :326-327): the not-moving merge (|dpose.pos| < NOT_MOVING_THRES and
      |dpose.yaw| < NOT_MOVING_YAW, both strict) and a static node's first block are reused;
  * outlier_rejection_frame  :408-515, including its quirks: after finish_init a node absent from the last keyframe is
      skipped, the first node without VO there ends the walk (`return`), a NaN asin compares false;
  * setup_problem_with_sferror  :1102-1154, gated by enable_to_init_by_drone and NodeFrame::distance_available.

Two definitions, not pinned (swarm_msgs is not in the reference tree): distance_available(b) is "has a distance to b that
is not flagged an outlier, an unwritten flag counting as not", since cutting_edges enables every distance (:1225-1297);
and rand() is replaced by the counter draw below.  The pose algebra is pnp_ref's / pcm_ref's (no FMA; numpy's libm).

`init_poses` / `outlier_flags` / `distance_rows` walk node by node as the reference does; the `_vec` forms compute the
same with numpy over all nodes and distances at once.
"""
from __future__ import annotations

import numpy as np

from oracle import pcm_ref as pr
from oracle import pnp_ref as pn
from oracle.multistart_ref import _splitmix64

NOT_MOVING_THRES = 0.02                  # :46
NOT_MOVING_YAW = 0.05                    # :47
RAND_INIT_XY = 5.0                       # :51
FACTOR_DISTANCE = 0
PAYLOAD_LEN = 24

NODE_DTYPE = np.dtype([("drone_id", "<i4"), ("block", "<i4"), ("new_block", "<i4"), ("prev_block", "<i4"),
                       ("vo_available", "<i4"), ("is_static", "<i4"), ("frame_available", "<i4"),
                       ("dists_available", "<i4"), ("n_distances", "<i4"), ("reserved", "<i4"),
                       ("pose", "<f8", 7), ("prev_pose", "<f8", 7)])
DIST_DTYPE = np.dtype([("peer", "<i4"), ("reserved", "<i4"), ("distance", "<f8")])


def draw(seed: int, stamp, drone, comp) -> np.ndarray:
    """rand_FloatRange(-RAND_INIT_XY, RAND_INIT_XY) replaced: [-5, 5) from (seed, splitmix64(stamp) ^ (drone << 2 | comp))"""
    stamp = np.asarray(stamp, np.int64).astype(np.uint64)
    drone, comp = np.asarray(drone, np.uint64), np.asarray(comp, np.uint64)
    key = _splitmix64(stamp) ^ ((drone << np.uint64(2)) | comp)
    u = (_splitmix64(np.uint64(seed) ^ _splitmix64(key)) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return (2.0 * RAND_INIT_XY) * u + (-RAND_INIT_XY)


def yaw(q) -> float:
    return float(pn.quat2eulers(np.asarray(q, np.float64))[2])


def pose4(p):
    """Pose(double[4], true)"""
    return np.concatenate([np.asarray(p[:3], np.float64), pn.quat_from_rotvec(np.array([0.0, 0.0, p[3]]))])


def effective(prm: dict) -> dict:
    """the thresholds as the solver holds them: the float parameters, overridden by debug_no_rejection (:89-96)"""
    f = np.float32
    if prm.get("debug_no_rejection"):
        return dict(thr=float(f(1e8)), elev=float(f(1e8)), min_d=-1.0)
    return dict(thr=float(f(prm["outlier_threshold"])), elev=float(f(prm["elevation_threshold"])),
                min_d=float(f(prm["minimum_distance"])))


# ---- the caller's part: which block a node takes ---------------------------------------------------------------------
class BlockAssigner:
    """est_poses_idts' pointer sharing (:279-298, :326-327) as block ids: per drone its latest block and odometry, and
    a static drone's first block"""

    def __init__(self):
        self.last, self.first, self.next = {}, {}, 0

    def assign(self, drones, poses, is_static, self_id: int, finish_init: bool) -> np.ndarray:
        """one keyframe's nodes (ascending drone id) -> NODE_DTYPE records with block / new_block / prev_*"""
        out = np.zeros(len(drones), NODE_DTYPE)
        for i, (d, p, st) in enumerate(zip(drones, poses, is_static)):
            d = int(d)
            r = out[i]
            r["drone_id"], r["pose"], r["is_static"], r["prev_block"] = d, p, int(st), -1
            if st:
                if d in self.first:
                    r["block"], r["new_block"] = self.first[d], 0
                else:
                    r["block"], r["new_block"] = self.next, 1
                    self.next += 1
            else:
                reuse = False
                if (d != self_id or finish_init) and d in self.last:
                    blk, vo = self.last[d]
                    r["prev_block"], r["prev_pose"] = blk, vo
                    dp = pn.delta_pose(vo, np.asarray(p, np.float64), True)
                    reuse = bool(np.sqrt(dp[0] * dp[0] + dp[1] * dp[1] + dp[2] * dp[2]) < NOT_MOVING_THRES and
                                 abs(yaw(dp[3:])) < NOT_MOVING_YAW)
                    if reuse:
                        r["block"], r["new_block"] = blk, 0
                if not reuse:
                    r["block"], r["new_block"] = self.next, 1
                    self.next += 1
            self.first.setdefault(d, int(r["block"]))
            self.last[d] = (int(r["block"]), np.array(p, np.float64))
        return out


# ---- a. initial poses -----------------------------------------------------------------------------------------------
def init_pose(nd, poses, stamp: int, self_id: int, finish_init: bool, seed: int) -> np.ndarray | None:
    """the x y z yaw a node's new block starts from, or None for a reused block"""
    if not nd["new_block"]:
        return None
    vo = np.asarray(nd["pose"], np.float64)
    d = int(nd["drone_id"])
    if not nd["is_static"] and (d != self_id or finish_init) and nd["prev_block"] >= 0:       # :279-298
        p = pr.pose_mul(pose4(poses[nd["prev_block"]]), pn.delta_pose(np.asarray(nd["prev_pose"]), vo, True))
        return np.array([p[0], p[1], p[2], yaw(p[3:])])
    if not nd["is_static"] and d == self_id and not finish_init:                               # :306-310
        return np.array([vo[0], vo[1], vo[2], yaw(vo[3:])])
    noise = draw(seed, stamp, d, np.arange(3))                                                 # :300-305, :329-335
    return np.array([vo[0] + noise[0], vo[1] + noise[1], vo[2] + noise[2], yaw(vo[3:])])


def init_poses(nodes, poses, stamp: int, self_id: int, finish_init: bool, seed: int) -> np.ndarray:
    out = np.array(poses, np.float64)
    for nd in nodes:
        p = init_pose(nd, out, stamp, self_id, finish_init, seed)
        if p is not None:
            out[nd["block"]] = p
    return out


def init_poses_vec(nodes, poses, stamp: int, self_id: int, finish_init: bool, seed: int) -> np.ndarray:
    out = np.array(poses, np.float64)
    new = nodes["new_block"] != 0
    dyn = nodes["is_static"] == 0
    d = nodes["drone_id"]
    pred = new & dyn & ((d != self_id) | finish_init) & (nodes["prev_block"] >= 0)
    selfvo = new & dyn & (d == self_id) & (not finish_init)
    noisy = new & ~pred & ~selfvo
    vo = nodes["pose"]
    yaws = np.array([yaw(q) for q in vo[:, 3:]]) if len(vo) else np.zeros(0)
    res = np.zeros((len(nodes), 4))
    res[:, 3] = yaws
    res[:, :3] = vo[:, :3]
    nz = np.nonzero(noisy)[0]
    if len(nz):
        res[nz, :3] = vo[nz, :3] + draw(seed, stamp, d[nz][:, None], np.arange(3)[None, :])
    for i in np.nonzero(pred)[0]:       # reads blocks that no node of this keyframe writes (prev blocks are older)
        p = pr.pose_mul(pose4(out[nodes["prev_block"][i]]), pn.delta_pose(nodes["prev_pose"][i], vo[i], True))
        res[i] = [p[0], p[1], p[2], yaw(p[3:])]
    out[nodes["block"][new]] = res[new]
    return out


# ---- b. outlier_distance --------------------------------------------------------------------------------------------
def outlier_flags(nodes, dists, poses, last_nodes, prm: dict) -> np.ndarray:
    """int8 per distance (dists order): 1 outlier, 0 not, -1 not written.  poses: after init_poses; last_nodes: the
    previous keyframe's records (None: none)"""
    e = effective(prm)
    flags = np.full(len(dists), -1, np.int8)
    here = {int(n["drone_id"]): n for n in nodes}
    last = {} if last_nodes is None else {int(n["drone_id"]): n for n in last_nodes}
    first = np.concatenate([[0], np.cumsum(nodes["n_distances"])]).astype(int)
    with np.errstate(all="ignore"):
        for i, nd in enumerate(nodes):
            if prm["finish_init"]:
                ln = last.get(int(nd["drone_id"]))
                if ln is None:                                   # :454-457
                    continue
                if not ln["vo_available"]:                       # :459-460
                    return flags
            for k in range(first[i], first[i + 1]):
                j = int(dists[k]["peer"])
                if j not in here or not here[j]["vo_available"]:
                    continue
                dis = float(dists[k]["distance"])
                if not prm["finish_init"]:                       # :427-438
                    dh = here[j]["pose"][2] - nd["pose"][2]
                    out = abs(np.arcsin(dh / dis)) > e["elev"] or not prm["enable_distance"]
                else:                                            # :489-507
                    pa, pb = poses[nd["block"]], poses[here[j]["block"]]
                    dx, dy, dz = pb[0] - pa[0], pb[1] - pa[1], pb[2] - pa[2]
                    est = np.sqrt((dx * dx + dy * dy) + dz * dz)
                    out = (abs(dis - est) > e["thr"] or dis < e["min_d"] or abs(np.arcsin(dz / dis)) > e["elev"]
                           or not prm["enable_distance"])
                flags[k] = 1 if out else 0
    return flags


def outlier_flags_vec(nodes, dists, poses, last_nodes, prm: dict) -> np.ndarray:
    e = effective(prm)
    n = len(nodes)
    owner = np.repeat(np.arange(n), nodes["n_distances"])
    idx = np.full(256, -1)
    idx[nodes["drone_id"]] = np.arange(n)
    jn = idx[dists["peer"]]
    has = (jn >= 0)
    has[has] = nodes["vo_available"][jn[has]] != 0
    active = np.ones(n, bool)
    if prm["finish_init"]:
        lv = np.full(256, -1)
        if last_nodes is not None:
            lv[last_nodes["drone_id"]] = last_nodes["vo_available"] != 0
        st = lv[nodes["drone_id"]]
        stop = np.nonzero(st == 0)[0]
        active = (st == 1) & (np.arange(n) < (stop[0] if len(stop) else n))
    sel = has & active[owner]
    dis = dists["distance"]
    jj = np.where(jn >= 0, jn, 0)
    with np.errstate(all="ignore"):
        if not prm["finish_init"]:
            dh = nodes["pose"][jj, 2] - nodes["pose"][owner, 2]
            out = (np.abs(np.arcsin(dh / dis)) > e["elev"]) | (not prm["enable_distance"])
        else:
            pa, pb = poses[nodes["block"][owner]], poses[nodes["block"][jj]]
            d = pb[:, :3] - pa[:, :3]
            est = np.sqrt((d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1]) + d[:, 2] * d[:, 2])
            out = ((np.abs(dis - est) > e["thr"]) | (dis < e["min_d"]) | (np.abs(np.arcsin(d[:, 2] / dis)) > e["elev"])
                   | (not prm["enable_distance"]))
    return np.where(sel, out.astype(np.int8), np.int8(-1)).astype(np.int8)


# ---- setup_problem_with_sferror ---------------------------------------------------------------------------------------
def sqrt_inf(cov: float) -> float:
    """1 / sqrt(distance_measurement_cov): the float parameter widened, then fp64"""
    return 1.0 / np.sqrt(float(np.float32(cov)))


def distance_rows(window, store: dict, enable, prm: dict) -> dict:
    """window: [(frame stamp, {drone: block})] in frame order; store: {stamp: (nodes, dists, flags)}; enable [drones]
    -> the appended rows as FactorRows dicts (ftype, ia, ib, payload, huber)"""
    rows = []
    si = sqrt_inf(prm["distance_measurement_cov"])
    for ts, blocks in window:
        if ts not in store:
            continue
        nodes, dists, flags = store[ts]
        first = np.concatenate([[0], np.cumsum(nodes["n_distances"])]).astype(int)
        for i, nd in enumerate(nodes):
            a = int(nd["drone_id"])
            if a not in blocks or not (enable[a] or a == prm["self_id"]):
                continue
            if not (prm["enable_distance"] and nd["frame_available"] and nd["dists_available"]):
                continue
            for k in range(first[i], first[i + 1]):
                b = int(dists[k]["peer"])
                if b < a and b in blocks and flags[k] != 1:
                    rows.append((blocks[a], blocks[b], float(dists[k]["distance"])))
    return _rows(rows, si, not prm.get("debug_no_rejection"))


def _rows(rows, si, huber):
    m = len(rows)
    pl = np.zeros((m, PAYLOAD_LEN))
    if m:
        pl[:, 0] = [r[2] for r in rows]
        pl[:, 1] = si
    return {"ftype": np.full(m, FACTOR_DISTANCE, np.int32), "ia": np.array([r[0] for r in rows], np.int32),
            "ib": np.array([r[1] for r in rows], np.int32), "payload": pl, "huber": np.full(m, int(huber), np.uint8)}


def distance_rows_vec(window, store: dict, enable, prm: dict) -> dict:
    parts = []
    en = np.asarray(enable, bool).copy()
    en[prm["self_id"]] = True
    for ts, blocks in window:
        if ts not in store:
            continue
        nodes, dists, flags = store[ts]
        blk = np.full(256, -1)
        for d, b in blocks.items():
            blk[d] = b
        owner = np.repeat(np.arange(len(nodes)), nodes["n_distances"])
        a = nodes["drone_id"][owner]
        b = dists["peer"]
        ok = (bool(prm["enable_distance"]) & (nodes["frame_available"][owner] != 0) & (nodes["dists_available"][owner] != 0)
              & en[a] & (blk[a] >= 0) & (b < a) & (blk[b] >= 0) & (flags != 1))
        parts.append(np.stack([blk[a[ok]], blk[b[ok]]], 1).astype(np.float64))
        parts[-1] = np.concatenate([parts[-1], dists["distance"][ok][:, None]], 1)
    rows = [tuple(r) for p in parts for r in p]
    rows = [(int(r[0]), int(r[1]), r[2]) for r in rows]
    return _rows(rows, sqrt_inf(prm["distance_measurement_cov"]), not prm.get("debug_no_rejection"))


# ---- a scenario generator shared by the CPU and GPU tests --------------------------------------------------------------
def random_keyframes(n_drones: int, n_kf: int, seed: int, self_id: int = 0, late=(), static=(), still_prob=0.2,
                     max_peers=None):
    """n_kf keyframes of a swarm: per keyframe (stamp ns, drones, odometry poses [7], is_static, vo_available,
    frame_available, dists_available, distances {drone: [(peer, metres)]}).  Drones in `late` join half way; drones in
    `static` do not move; a dynamic drone stays put with probability still_prob (a not-moving merge)."""
    rng = np.random.default_rng(seed)
    pos = rng.uniform(-10, 10, (n_drones, 3))
    yw = rng.uniform(-np.pi, np.pi, n_drones)
    out = []
    for k in range(n_kf):
        stamp = 1_000_000_000 + k * 500_000_000
        drones = [d for d in range(n_drones) if d not in late or k >= n_kf // 2]
        for d in drones:
            if d in static or rng.random() < still_prob:
                continue
            pos[d] += rng.normal(0, 0.3, 3)
            yw[d] += rng.normal(0, 0.1)
        poses = []
        for d in drones:
            q = pn.quat_from_rotvec(np.array([rng.normal(0, 0.02), rng.normal(0, 0.02), yw[d]]))
            poses.append(np.concatenate([pos[d], q]))
        dist = {}
        for d in drones:
            peers = [p for p in range(n_drones) if p != d and rng.random() < 0.8]
            if max_peers is not None:
                peers = peers[:max_peers]
            dist[d] = [(p, float(np.linalg.norm(pos[p] - pos[d]) + rng.normal(0, 0.1) + (3.0 if rng.random() < 0.1 else 0)))
                       for p in peers]
        out.append(dict(stamp=stamp, drones=drones, poses=poses, is_static=[d in static for d in drones],
                        vo=[bool(rng.random() > 0.05) or d == self_id for d in drones],
                        frame=[bool(rng.random() > 0.05) for d in drones], dists_ok=[bool(rng.random() > 0.05) for d in drones],
                        dist=dist))
    return out


def keyframe_records(kf: dict, assigner: BlockAssigner, self_id: int, finish_init: bool):
    """one generated keyframe -> (nodes NODE_DTYPE with blocks assigned, dists DIST_DTYPE)"""
    nodes = assigner.assign(kf["drones"], kf["poses"], kf["is_static"], self_id, finish_init)
    nodes["vo_available"] = kf["vo"]
    nodes["frame_available"] = kf["frame"]
    nodes["dists_available"] = kf["dists_ok"]
    ds = []
    for i, d in enumerate(kf["drones"]):
        pairs = sorted(kf["dist"].get(d, []))
        nodes[i]["n_distances"] = len(pairs)
        ds += pairs
    dists = np.zeros(len(ds), DIST_DTYPE)
    if ds:
        dists["peer"] = [p for p, _ in ds]
        dists["distance"] = [m for _, m in ds]
    return nodes, dists
