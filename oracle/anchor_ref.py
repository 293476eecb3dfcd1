"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the re-anchoring of loops and detections onto the
sliding window that every solve() of the back-end performs (SURVEY.md section 8f-4).

Follows (paths relative to the reference's swarm_localization/src):
  * SwarmLocalizationSolver::find_available_loops_detections  swarm_localization_solver.cpp:1594-1666 -- every entry of
      all_loops, then every entry of all_detections_6d, through loop_from_src_loop_connection;
  * loop_from_src_loop_connection  :1464-1553 -- empty window (:1479-1482), the strict `(sf_sld_win[0].stamp - stamp_a) >
      BEGIN_MIN_LOOP_DT` test on stamp_a only (:1484, BEGIN_MIN_LOOP_DT = 1000 s at :56), the anchor search, the odometry
      covariance of both sides, detection self poses from the trajectories (Detection4d: yaw only), new_loop =
      DeltaPose(nf_a.self_pose, self_pose_a, true) * relative_pose * DeltaPose(self_pose_b, nf_b.self_pose, true), the
      `dpos > det_dpos_thres` rejection, and the output edge;
  * find_node_frame_for_measurement_2drones  :1429-1462 -- frames in order, a candidate is a vo_available node of the drone,
      taken when |stamp - stamp_x| < min_err (strict, min_err starts at 10000 s), so ties keep the earliest frame;
  * setup_problem_with_loops_and_detections  :1064-1100 -- no factor when either drone is not yaw-observable or both ends
      are the same pose block; otherwise RelativePoseFactor4d with get_sqrt_information_4d(), Huber unless
      debug_no_rejection.

DroneTrajectory, NodeFrame and LoopEdge belong to HKUST-Swarm/swarm_msgs, which is not in the reference tree.  They are
DEFINED here, not pinned:
  * a trajectory is a list of (int64 ns stamp, 7-double pose) samples pushed in increasing stamp order; length[k] is the
    sequential fp64 sum of |p_j - p_(j-1)| for j <= k;
  * `*_by_appro_ts(t)` uses the sample nearest to t, ties to the earlier one, stamps outside clamp to the first / last;
  * covariance_between_appro_ts(t1, t2) = |length(t2) - length(t1)| * diag(pos x3, ang x3) per metre (pcm_ref's rule);
  * trajectory_length_by_appro_ts(t1, t2) = |length(t2) - length(t1)|;
  * set_yaw_only keeps position and yaw, roll and pitch become 0;
  * DeltaPose(.., true) is pnp_ref.delta_pose(yaw_only=True), `*` is pcm_ref.pose_mul;
  * get_sqrt_information_4d is the CreateCov6d rule (solver_ref.create_cov6d_sqrt_inf);
  * stamps are int64 ns throughout, so every comparison is exact (1000 s and 10000 s become ns);
  * a drone without a trajectory is a status (NO_TRAJECTORY) where the reference would throw from ego_motion_trajs.at().

`anchor` is the literal restatement (one measurement at a time, frames in order); `anchor_vec` computes the same with numpy
over all measurements at once (the CPU timing of scripts/bench_anchor.py), and tests/test_anchor_ref.py checks they agree.
"""
from __future__ import annotations

import bisect

import numpy as np

from . import pcm_ref as pr
from . import pnp_ref as pn
from .solver_ref import create_cov6d_sqrt_inf, FACTOR_RELPOSE

LOOP, DET4D, DET6D = 0, 1, 2
OK, EMPTY_WINDOW, BEFORE_WINDOW, NO_FRAME, NO_TRAJECTORY, DPOS = range(6)
NS = 1_000_000_000
MIN_TS_ERR_START_NS = 10000 * NS

EDGE_DTYPE = np.dtype([("id_a", "<i4"), ("id_b", "<i4"), ("rel_pose", "<f8", 7), ("cov", "<f8", (6, 6)),
                       ("odom_a", "<f8", 7), ("odom_b", "<f8", 7), ("len_a", "<f8"), ("len_b", "<f8")])
RESULT_DTYPE = np.dtype([("id", "<i8"), ("type", "<i4"), ("status", "<i4"), ("frame_a", "<i4"), ("frame_b", "<i4"),
                         ("node_a", "<i4"), ("node_b", "<i4"), ("stamp_a", "<i8"), ("stamp_b", "<i8"), ("dt_err_ns", "<i8"),
                         ("dpos", "<f8"), ("edge", EDGE_DTYPE), ("skip", "<i4"), ("factor_type", "<i4"), ("ia", "<i4"),
                         ("ib", "<i4"), ("huber", "<i4"), ("reserved", "<i4"), ("payload", "<f8", 24)])
MEAS_DTYPE = np.dtype([("id", "<i8"), ("type", "<i4"), ("id_a", "<i4"), ("id_b", "<i4"), ("reserved", "<i4"),
                       ("stamp_a", "<i8"), ("stamp_b", "<i8"), ("relative_pose", "<f8", 7), ("cov", "<f8", (6, 6)),
                       ("self_pose_a", "<f8", 7), ("self_pose_b", "<f8", 7)])
ENTRY_DTYPE = np.dtype([("drone_id", "<i4"), ("vo_available", "<i4"), ("block", "<i4"), ("reserved", "<i4"),
                        ("stamp", "<i8"), ("self_pose", "<f8", 7)])


def trajectory_lengths(poses) -> np.ndarray:
    """length[k] = sum_{j<=k} |p_j - p_(j-1)|, summed in sample order (np.cumsum accumulates sequentially)"""
    p = np.asarray(poses, np.float64)
    if len(p) == 0:
        return np.zeros(0)
    d = p[1:, :3] - p[:-1, :3]
    step = np.sqrt(d[:, 0] * d[:, 0] + d[:, 1] * d[:, 1] + d[:, 2] * d[:, 2])
    return np.concatenate([[0.0], np.cumsum(step)])


class Trajectory:
    """DroneTrajectory as defined above"""

    def __init__(self, stamps, poses):
        self.stamps = [int(s) for s in stamps]
        assert all(b > a for a, b in zip(self.stamps, self.stamps[1:])), "stamps must increase strictly"
        self.poses = np.asarray(poses, np.float64).reshape(len(self.stamps), 7)
        self.length = trajectory_lengths(self.poses)

    def nearest(self, t: int) -> int:
        k = bisect.bisect_left(self.stamps, t)
        if k == 0:
            return 0
        if k == len(self.stamps):
            return k - 1
        return k - 1 if t - self.stamps[k - 1] <= self.stamps[k] - t else k

    def pose_by_appro_ts(self, t):
        return self.poses[self.nearest(t)].copy()

    def length_at(self, t) -> float:
        return float(self.length[self.nearest(t)])

    def trajectory_length_by_appro_ts(self, t1, t2) -> float:
        return abs(self.length_at(t2) - self.length_at(t1))

    def covariance_between_appro_ts(self, t1, t2, pos_cov, ang_cov):
        return self.trajectory_length_by_appro_ts(t1, t2) * np.diag([pos_cov] * 3 + [ang_cov] * 3)


def set_yaw_only(p):
    out = np.array(p, np.float64)
    out[3:] = pn.quat_from_rotvec(np.array([0.0, 0.0, pn.quat2eulers(p[3:])[2]]))
    return out


def window_frames(frame_stamps, frame_first, entries):
    """sf_sld_win: [(frame stamp, {drone_id: NodeFrame dict})]"""
    frames = []
    for f in range(len(frame_stamps)):
        nodes = {}
        for e in entries[int(frame_first[f]):int(frame_first[f + 1])]:
            nodes[int(e["drone_id"])] = dict(stamp=int(e["stamp"]), vo=bool(e["vo_available"]), block=int(e["block"]),
                                             self_pose=np.array(e["self_pose"], np.float64))
        frames.append((int(frame_stamps[f]), nodes))
    return frames


def find_node_frame(frames, id_a, id_b, tsa, tsb):
    """find_node_frame_for_measurement_2drones (:1429-1462) -> (index_a, index_b, min_err_a, min_err_b); -1 if not found"""
    ia = ib = -1
    ea = eb = MIN_TS_ERR_START_NS
    for i, (_, nodes) in enumerate(frames):
        na = nodes.get(id_a)
        if na is not None and na["vo"] and abs(na["stamp"] - tsa) < ea:
            ea, ia = abs(na["stamp"] - tsa), i
        nb = nodes.get(id_b)
        if nb is not None and nb["vo"] and abs(nb["stamp"] - tsb) < eb:
            eb, ib = abs(nb["stamp"] - tsb), i
    return ia, ib, ea, eb


def loop_from_src_loop_connection(m, frames, trajs, prm):
    """one measurement (a MEAS_DTYPE record or a dict with its fields) -> result dict (RESULT_DTYPE fields)"""
    r = dict(id=int(m["id"]), type=int(m["type"]), status=OK, frame_a=-1, frame_b=-1, node_a=-1, node_b=-1, stamp_a=0,
             stamp_b=0, dt_err_ns=0, dpos=0.0, edge=None, payload=np.zeros(24))
    ida, idb, tsa, tsb = int(m["id_a"]), int(m["id_b"]), int(m["stamp_a"]), int(m["stamp_b"])
    if not frames:                                                                      # :1479-1482
        r["status"] = EMPTY_WINDOW
        return r
    if frames[0][0] - tsa > int(round(prm["begin_min_loop_dt_s"] * NS)):                 # :1484
        r["status"] = BEFORE_WINDOW
        return r
    fa, fb, ea, eb = find_node_frame(frames, ida, idb, tsa, tsb)
    r["dt_err_ns"] = ea + eb
    if fa >= 0:
        nf_a = frames[fa][1][ida]
        r.update(frame_a=fa, node_a=nf_a["block"], stamp_a=nf_a["stamp"])
    if fb >= 0:
        nf_b = frames[fb][1][idb]
        r.update(frame_b=fb, node_b=nf_b["block"], stamp_b=nf_b["stamp"])
    if fa < 0 or fb < 0:
        r["status"] = NO_FRAME
        return r
    if ida not in trajs or idb not in trajs:                                            # ego_motion_trajs.at() would throw
        r["status"] = NO_TRAJECTORY
        return r
    ta, tb = trajs[ida], trajs[idb]
    pos, ang = prm["odom_pos_cov_per_m"], prm["odom_ang_cov_per_m"]
    cov_odom = ta.covariance_between_appro_ts(nf_a["stamp"], tsa, pos, ang) \
        + tb.covariance_between_appro_ts(nf_b["stamp"], tsb, pos, ang)
    self_a, self_b = np.array(m["self_pose_a"], np.float64), np.array(m["self_pose_b"], np.float64)
    if r["type"] in (DET4D, DET6D):                                                     # :1510-1517
        self_a, self_b = ta.pose_by_appro_ts(tsa), tb.pose_by_appro_ts(tsb)
        if r["type"] == DET4D:
            self_a, self_b = set_yaw_only(self_a), set_yaw_only(self_b)
    dpose_self_a = pn.delta_pose(nf_a["self_pose"], self_a, True)
    dpose_self_b = pn.delta_pose(self_b, nf_b["self_pose"], True)
    new_loop = pr.pose_mul(pr.pose_mul(dpose_self_a, np.array(m["relative_pose"], np.float64)), dpose_self_b)
    r["dpos"] = ta.trajectory_length_by_appro_ts(tsa, nf_a["stamp"]) + tb.trajectory_length_by_appro_ts(tsb, nf_b["stamp"])
    if r["dpos"] > prm["det_dpos_thres"]:
        r["status"] = DPOS
    cov = np.asarray(m["cov"], np.float64).reshape(6, 6) + cov_odom
    r["edge"] = dict(id_a=ida, id_b=idb, rel=new_loop, cov=cov, odom_a=nf_a["self_pose"].copy(),
                     odom_b=nf_b["self_pose"].copy(), len_a=ta.length_at(nf_a["stamp"]), len_b=tb.length_at(nf_b["stamp"]))
    r["payload"][:3] = new_loop[:3]
    r["payload"][3] = pn.quat2eulers(new_loop[3:])[2]
    r["payload"][4:20] = create_cov6d_sqrt_inf(cov).reshape(-1)
    return r


def measurement_order(meas):
    """all_loops in arrival order, then all_detections_6d in arrival order (:1600-1645)"""
    t = np.asarray(meas["type"])
    return np.concatenate([np.nonzero(t == LOOP)[0], np.nonzero(t != LOOP)[0]])


def _finish(r, yaw_observable):
    """setup_problem_with_loops_and_detections' choice (:1066-1073) and the factor row"""
    obs = lambda d: d < len(yaw_observable) and bool(yaw_observable[d])           # noqa: E731
    ok = r["status"] == OK and obs(r["ida"]) and obs(r["idb"])
    r["skip"] = 0 if ok and r["node_a"] != r["node_b"] else 1
    r["ia"], r["ib"] = r["node_a"], r["node_b"]


def anchor(trajs: dict, window, meas, yaw_observable, prm: dict) -> np.ndarray:
    """The literal walk.  trajs {drone: (stamps int64 [n], poses [n,7])}; window = (frame_stamps [F], frame_first [F+1],
    entries ENTRY_DTYPE); meas MEAS_DTYPE; yaw_observable indexed by drone id; prm: begin_min_loop_dt_s, det_dpos_thres,
    odom_pos_cov_per_m, odom_ang_cov_per_m, huber -> RESULT_DTYPE [n], loops first."""
    T = {int(d): Trajectory(*v) for d, v in trajs.items() if len(v[0])}
    frames = window_frames(*window)
    order = measurement_order(meas)
    out = np.zeros(len(order), RESULT_DTYPE)
    for k, i in enumerate(order):
        m = meas[i]
        r = loop_from_src_loop_connection(m, frames, T, prm)
        r["ida"], r["idb"] = int(m["id_a"]), int(m["id_b"])
        _finish(r, yaw_observable)
        o = out[k]
        for f in ("id", "type", "status", "frame_a", "frame_b", "node_a", "node_b", "stamp_a", "stamp_b", "dt_err_ns", "dpos",
                  "skip", "ia", "ib", "payload"):
            o[f] = r[f]
        o["factor_type"] = FACTOR_RELPOSE
        o["huber"] = 1 if prm.get("huber", True) else 0
        e = r["edge"]
        if e is not None:
            o["edge"]["id_a"], o["edge"]["id_b"] = e["id_a"], e["id_b"]
            o["edge"]["rel_pose"], o["edge"]["cov"] = e["rel"], e["cov"]
            o["edge"]["odom_a"], o["edge"]["odom_b"] = e["odom_a"], e["odom_b"]
            o["edge"]["len_a"], o["edge"]["len_b"] = e["len_a"], e["len_b"]
    return out


# ---- the same with numpy over all measurements ------------------------------------------------------------------------
def _nearest_vec(stamps, t):
    k = np.searchsorted(stamps, t, side="left")
    n = len(stamps)
    lo = np.clip(k - 1, 0, n - 1)
    hi = np.clip(k, 0, n - 1)
    pick_lo = (t - stamps[lo]) <= (stamps[hi] - t)
    return np.where(k == 0, 0, np.where(k == n, n - 1, np.where(pick_lo, lo, hi)))


def _yaw_vec(q):
    return np.arctan2(2.0 * (q[:, 0] * q[:, 3] + q[:, 1] * q[:, 2]), 1.0 - 2.0 * (q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3]))


def _yaw_quat_vec(yaw):
    """quat_from_rotvec([0, 0, yaw]) row by row"""
    a = np.sqrt(yaw * yaw)
    small = a < 1e-12
    with np.errstate(invalid="ignore", divide="ignore"):
        s = np.where(small, 0.5, np.sin(0.5 * a) / a)
    q = np.zeros((len(yaw), 4))
    q[:, 0] = np.where(small, 1.0, np.cos(0.5 * a))
    q[:, 3] = s * yaw
    return q / np.sqrt(q[:, 0] * q[:, 0] + q[:, 3] * q[:, 3])[:, None]


def _delta_pose4_vec(a, b):
    ya, yb = _yaw_vec(a[:, 3:]), _yaw_vec(b[:, 3:])
    d = b[:, :3] - a[:, :3]
    c, s = np.cos(ya), np.sin(ya)
    out = np.zeros_like(a)
    out[:, 0] = c * d[:, 0] + s * d[:, 1]
    out[:, 1] = -s * d[:, 0] + c * d[:, 1]
    out[:, 2] = d[:, 2]
    out[:, 3:] = _yaw_quat_vec(pn.wrap(yb - ya))
    return out


def _q_mul_vec(a, b):
    aw, ax, ay, az = a.T
    bw, bx, by, bz = b.T
    return np.stack([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw], axis=1)


def _pose_mul_vec(a, b):
    q, v = a[:, 3:], b[:, :3]
    u = q[:, 1:]
    c = np.cross(u, v)
    rot = v + 2.0 * (q[:, :1] * c + np.cross(u, c))
    return np.concatenate([a[:, :3] + rot, _q_mul_vec(a[:, 3:], b[:, 3:])], axis=1)


def _search_vec(e_stamp, e_idx, t, chunk=4096):
    """per measurement: the entry of minimal |stamp - t| below 10000 s, the earliest on ties -> (index or -1, err)"""
    n = len(t)
    idx = np.full(n, -1, np.int64)
    err = np.full(n, MIN_TS_ERR_START_NS, np.int64)
    if len(e_stamp) == 0:
        return idx, err
    for s in range(0, n, chunk):
        d = np.abs(e_stamp[None, :] - t[s:s + chunk, None])
        j = np.argmin(d, axis=1)                                   # the first minimum: entries are in frame order
        best = d[np.arange(len(j)), j]
        hit = best < MIN_TS_ERR_START_NS
        idx[s:s + chunk] = np.where(hit, e_idx[j], -1)
        err[s:s + chunk] = np.where(hit, best, MIN_TS_ERR_START_NS)
    return idx, err


def anchor_vec(trajs: dict, window, meas, yaw_observable, prm: dict) -> np.ndarray:
    """anchor() computed with numpy over all measurements at once"""
    frame_stamps, frame_first, entries = window
    meas = meas[measurement_order(meas)]
    n = len(meas)
    out = np.zeros(n, RESULT_DTYPE)
    out["id"], out["type"] = meas["id"], meas["type"]
    out["factor_type"], out["huber"] = FACTOR_RELPOSE, 1 if prm.get("huber", True) else 0
    out["frame_a"] = out["frame_b"] = out["node_a"] = out["node_b"] = -1
    ida, idb = meas["id_a"].astype(np.int64), meas["id_b"].astype(np.int64)
    tsa, tsb = meas["stamp_a"].astype(np.int64), meas["stamp_b"].astype(np.int64)
    status = np.zeros(n, np.int32)
    if len(frame_stamps) == 0:
        status[:] = EMPTY_WINDOW
    else:
        status[int(frame_stamps[0]) - tsa > int(round(prm["begin_min_loop_dt_s"] * NS))] = BEFORE_WINDOW
    live = status == OK
    frame_of = np.repeat(np.arange(len(frame_stamps)), np.diff(np.asarray(frame_first)))
    ent_a = np.full(n, -1, np.int64)
    ent_b = np.full(n, -1, np.int64)
    err_a = np.full(n, MIN_TS_ERR_START_NS, np.int64)
    err_b = np.full(n, MIN_TS_ERR_START_NS, np.int64)
    vo = np.nonzero(entries["vo_available"] != 0)[0] if len(entries) else np.zeros(0, np.int64)
    drones = np.unique(np.concatenate([ida, idb]))
    for d in drones:
        e_idx = vo[entries["drone_id"][vo] == d]                   # entries are stored frame by frame: frame order
        e_stamp = entries["stamp"][e_idx].astype(np.int64)
        for ids, ts, ent, err in ((ida, tsa, ent_a, err_a), (idb, tsb, ent_b, err_b)):
            sel = np.nonzero(live & (ids == d))[0]
            ent[sel], err[sel] = _search_vec(e_stamp, e_idx, ts[sel])
    out["dt_err_ns"] = np.where(live, err_a + err_b, 0)
    for ent, fr, nd, st in ((ent_a, "frame_a", "node_a", "stamp_a"), (ent_b, "frame_b", "node_b", "stamp_b")):
        f = ent >= 0
        out[fr][f] = frame_of[ent[f]]
        out[nd][f] = entries["block"][ent[f]]
        out[st][f] = entries["stamp"][ent[f]]
    status[live & ((ent_a < 0) | (ent_b < 0))] = NO_FRAME
    has_traj = np.array([int(d) in trajs and len(trajs[int(d)][0]) > 0 for d in range(int(drones.max()) + 1)]) \
        if len(drones) else np.zeros(0, bool)
    live = status == OK
    status[live & ~(has_traj[ida] & has_traj[idb])] = NO_TRAJECTORY
    live = np.nonzero(status == OK)[0]
    if len(live):
        L = {int(d): (np.asarray(trajs[int(d)][0], np.int64), np.asarray(trajs[int(d)][1], np.float64),
                      trajectory_lengths(trajs[int(d)][1])) for d in drones if has_traj[d]}
        m = meas[live]
        ea, eb = ent_a[live], ent_b[live]
        nfa_pose, nfb_pose = entries["self_pose"][ea], entries["self_pose"][eb]
        self_a = np.array(m["self_pose_a"], np.float64)
        self_b = np.array(m["self_pose_b"], np.float64)
        len_nfa, len_a, len_nfb, len_b = (np.zeros(len(live)) for _ in range(4))
        for d, (ts, poses, length) in L.items():
            for side, ids, t_x, nf_ent, l_nf, l_x, selfp in ((0, m["id_a"], m["stamp_a"], ea, len_nfa, len_a, self_a),
                                                             (1, m["id_b"], m["stamp_b"], eb, len_nfb, len_b, self_b)):
                sel = np.nonzero(ids == d)[0]
                if len(sel) == 0:
                    continue
                k_nf = _nearest_vec(ts, entries["stamp"][nf_ent[sel]].astype(np.int64))
                k_x = _nearest_vec(ts, t_x[sel].astype(np.int64))
                l_nf[sel], l_x[sel] = length[k_nf], length[k_x]
                det = m["type"][sel] != LOOP
                selfp[sel[det]] = poses[k_x[det]]
        for selfp in (self_a, self_b):
            d4 = np.nonzero(m["type"] == DET4D)[0]
            if len(d4):
                selfp[d4, 3:] = _yaw_quat_vec(_yaw_vec(selfp[d4, 3:]))
        da, db = np.abs(len_a - len_nfa), np.abs(len_b - len_nfb)
        new_loop = _pose_mul_vec(_pose_mul_vec(_delta_pose4_vec(nfa_pose, self_a), np.array(m["relative_pose"])),
                                 _delta_pose4_vec(self_b, nfb_pose))
        dpos = da + db
        status[live[dpos > prm["det_dpos_thres"]]] = DPOS
        per_m = np.diag([prm["odom_pos_cov_per_m"]] * 3 + [prm["odom_ang_cov_per_m"]] * 3)
        cov = np.array(m["cov"]) + (da[:, None, None] * per_m + db[:, None, None] * per_m)
        out["dpos"][live] = dpos
        e = out["edge"]
        e["id_a"][live], e["id_b"][live] = m["id_a"], m["id_b"]
        e["rel_pose"][live], e["cov"][live] = new_loop, cov
        e["odom_a"][live], e["odom_b"][live] = nfa_pose, nfb_pose
        e["len_a"][live], e["len_b"][live] = len_nfa, len_nfb
        cov4 = np.zeros((len(live), 4, 4))
        cov4[:, :3, :3] = cov[:, :3, :3]
        cov4[:, 3, 3] = cov[:, 5, 5]
        pl = np.zeros((len(live), 24))
        pl[:, :3] = new_loop[:, :3]
        pl[:, 3] = _yaw_vec(new_loop[:, 3:])
        pl[:, 4:20] = np.sqrt(np.abs(np.linalg.inv(cov4))).reshape(-1, 16)
        out["payload"][live] = pl
    out["status"] = status
    yaw = np.asarray(yaw_observable, bool)
    obs = lambda ids: (ids < len(yaw)) & yaw[np.minimum(ids, len(yaw) - 1)]     # noqa: E731
    out["ia"], out["ib"] = out["node_a"], out["node_b"]
    out["skip"] = ~((status == OK) & obs(ida) & obs(idb) & (out["node_a"] != out["node_b"]))
    return out
