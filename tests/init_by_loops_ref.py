"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the pre-motion init start:
SwarmLocalizationSolver::init_pose_by_loops / init_pose_by_loop (swarm_localization_solver.cpp:218-269) over the loop
bookkeeping of SwarmLocalOutlierRejection::OutlierRejectionLoopEdges (swarm_outlier_rejection.cpp:106-120).

`LoopBook` keeps what the reference keeps, as dict-of-dicts: all_loops_set (the ids PCM has stored: the routed pairs'
ids, :122-139), all_loop_map (id -> the re-anchored edge as first seen) and all_loops_set_by_pair[a][b]; `good` is
good_loops_set[a][b] (a PCM result or a set_inliers set, both directions).  `init_pose_by_loops` is the literal walk:
drones to initialise ascending; the good sets of _id replace its all-loops pairs as a whole; pairs by ascending id2,
skipped when empty or id2 not estimated, each later one overwriting; the loop of the set's smallest id, inverted when
id_a != id2; pose0 from id2's keyframe path, else (id2 == self) its odometry, else identity; every est_poses frame of
_id gets pose0 * odoma * rel * odomb with both odometries on id2's trajectory and odomb ending at the FRAME stamp.
Trajectory definitions are oracle/anchor_ref.py's (nearest sample, ties to the earlier) and the relative pose is
pose(t1)^-1 pose(t2) (tests/loop_candidates_ref.py).  Where the reference throws (all_loop_map.at(),
ego_motion_trajs.at()) this raises Refused.

`record_vec` / `init_by_loops_vec` compute the same with numpy over the device's representation: the map as sorted
records, each ordered pair's smallest id in a [D, D] matrix, the window as (drone, frame)-ordered entries.
tests/test_init_by_loops_ref.py checks the two forms against each other.
"""
from __future__ import annotations

import copy

import numpy as np

from oracle import anchor_ref as ar
from oracle import pcm_ref as pr

I64_MAX = np.iinfo(np.int64).max
IDENTITY = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])


class Refused(Exception):
    """where the reference throws: an id missing from all_loop_map, or id2 without odometry"""


def yaw(q):
    return float(np.arctan2(2.0 * (q[0] * q[3] + q[1] * q[2]), 1.0 - 2.0 * (q[2] * q[2] + q[3] * q[3])))


def edge_of(row) -> dict:
    """the Swarm::LoopEdge init_pose_by_loop reads, from one re-anchored row (lib.ANCHOR_RESULT_DTYPE)"""
    return dict(id=int(row["id"]), id_a=int(row["edge"]["id_a"]), id_b=int(row["edge"]["id_b"]),
                ts_a=int(row["stamp_a"]), ts_b=int(row["stamp_b"]), rel=np.array(row["edge"]["rel_pose"], np.float64))


def invert_loop(e: dict) -> dict:
    return dict(id=e["id"], id_a=e["id_b"], id_b=e["id_a"], ts_a=e["ts_b"], ts_b=e["ts_a"], rel=pr.pose_inv(e["rel"]))


class LoopBook:
    """OutlierRejectionLoopEdges' bookkeeping (:106-120), fed the OK rows of each solve in row order"""

    def __init__(self, self_id: int, redundant: bool):
        self.self_id, self.redundant = self_id, redundant
        self.all_loops_set = set()
        self.all_loop_map = {}
        self.all_loops_set_by_pair = {}

    def record(self, rows):
        routed = []
        for row in rows:
            if int(row["status"]) != ar.OK:
                continue
            e = edge_of(row)
            if e["id"] in self.all_loops_set:
                continue
            if e["id"] not in self.all_loop_map:
                self.all_loop_map[e["id"]] = e
            a, b = e["id_a"], e["id_b"]
            self.all_loops_set_by_pair.setdefault(a, {}).setdefault(b, set()).add(e["id"])
            self.all_loops_set_by_pair.setdefault(b, {}).setdefault(a, set()).add(e["id"])
            if self.redundant or a == self.self_id or b == self.self_id:
                routed.append(e["id"])
        self.all_loops_set.update(routed)                          # OutlierRejectionLoopEdgesPCM stores them


class Trajs:
    """ego_motion_trajs: {drone: anchor_ref.Trajectory}; a missing drone raises Refused"""

    def __init__(self, trajs: dict):
        self.t = {int(d): ar.Trajectory(*v) for d, v in trajs.items() if len(v[0])}

    def at(self, d) -> ar.Trajectory:
        if d not in self.t:
            raise Refused(f"drone {d} has no odometry")
        return self.t[d]

    def relative(self, d, t1, t2):
        tr = self.at(d)
        return pr.pose_mul(pr.pose_inv(tr.poses[tr.nearest(t1)]), tr.poses[tr.nearest(t2)])


def est_poses_of(window, poses) -> dict:
    """est_poses_tsid over the window: {frame stamp: {drone: the block's row of `poses` (a view: shared blocks alias)}}"""
    out = {}
    for ts, nodes in ar.window_frames(*window):
        for d, nf in nodes.items():
            out.setdefault(ts, {})[d] = poses[nf["block"]]
    return out


def init_pose_by_loop(est, _id, id2, loc, kf: dict, trajs: Trajs, self_id):
    if loc["id_a"] != id2:
        loc = invert_loop(loc)
    t0, pose0 = loc["ts_a"], IDENTITY.copy()
    if id2 in kf and len(kf[id2][0]) > 0:
        stamps, kposes = kf[id2]
        k = ar.Trajectory(stamps, kposes).nearest(t0)
        t0, pose0 = int(stamps[k]), np.array(kposes[k], np.float64)
    elif id2 == self_id:
        tr = trajs.at(id2)
        k = tr.nearest(t0)
        t0, pose0 = tr.stamps[k], tr.poses[k].copy()
    for ts in sorted(est):
        odoma = trajs.relative(id2, t0, loc["ts_a"])
        odomb = trajs.relative(id2, loc["ts_b"], ts)
        for d, p in est[ts].items():
            if d == _id:
                pose = pr.pose_mul(pr.pose_mul(pr.pose_mul(pose0, odoma), loc["rel"]), odomb)
                p[:3] = pose[:3]
                p[3] = yaw(pose[3:])


def init_pose_by_loops(ids_to_init, good: dict, book: LoopBook, estimated, kf: dict, trajs: Trajs, self_id, window,
                       poses) -> np.ndarray:
    """the literal walk -> the new poses [n_blocks, 4]; raises Refused (the poses given are never changed)"""
    poses = np.array(poses, np.float64, copy=True)
    est = est_poses_of(window, poses)
    for _id in sorted(ids_to_init):
        loop_sets = copy.deepcopy(book.all_loops_set_by_pair.get(_id, {}))
        if _id in good:
            loop_sets = good[_id]
        for id2 in sorted(loop_sets):
            s = loop_sets[id2]
            if len(s) == 0 or id2 not in estimated:
                continue
            if min(s) not in book.all_loop_map:
                raise Refused(f"loop {min(s)} is not in all_loop_map")
            init_pose_by_loop(est, _id, id2, book.all_loop_map[min(s)], kf, trajs, self_id)
    return poses


def good_from_sets(sets: dict) -> dict:
    """{(a, b) unordered: ids} -> good_loops_set[a][b] and [b][a]"""
    good = {}
    for (a, b), ids in sets.items():
        good.setdefault(a, {})[b] = set(int(i) for i in ids)
        good.setdefault(b, {})[a] = set(int(i) for i in ids)
    return good


# ---- the same with numpy over the device's representation ------------------------------------------------------------
class LoopMapVec:
    """the map as records sorted by id (lib.LOOP_RECORD_DTYPE) and pair_min [D, D] (I64_MAX: none)"""

    def __init__(self, max_drones: int, dtype):
        self.recs = np.zeros(0, dtype)
        self.pair_min = np.full((max_drones, max_drones), I64_MAX, np.int64)

    def record_vec(self, rows):
        """every OK row whose id is not recorded: the first row of each id wins; both pair orders take the minimum"""
        ok = rows[rows["status"] == ar.OK]
        fresh = ~np.isin(ok["id"], self.recs["id"])
        ok = ok[fresh]
        if len(ok) == 0:
            return
        _, first = np.unique(ok["id"], return_index=True)
        new = np.zeros(len(first), self.recs.dtype)
        w = ok[first]
        new["id"], new["id_a"], new["id_b"] = w["id"], w["edge"]["id_a"], w["edge"]["id_b"]
        new["stamp_a"], new["stamp_b"], new["rel_pose"] = w["stamp_a"], w["stamp_b"], w["edge"]["rel_pose"]
        self.recs = np.sort(np.concatenate([self.recs, new]), order="id")
        a, b = ok["edge"]["id_a"].astype(np.int64), ok["edge"]["id_b"].astype(np.int64)
        np.minimum.at(self.pair_min, (a, b), ok["id"])
        np.minimum.at(self.pair_min, (b, a), ok["id"])


def _inv_vec(p):
    q = p[:, 3:] * np.array([1.0, -1.0, -1.0, -1.0])
    t = ar._pose_mul_vec(np.concatenate([np.zeros((len(p), 3)), q], axis=1), np.concatenate([p[:, :3], q], axis=1))[:, :3]
    return np.concatenate([-t, q], axis=1)


def _rel_vec(stamps, tposes, t1, t2):
    return ar._pose_mul_vec(_inv_vec(tposes[ar._nearest_vec(stamps, t1)]), tposes[ar._nearest_vec(stamps, t2)])


def init_by_loops_vec(to_init, good_sets: dict, lmap: LoopMapVec, estimated, kf: dict, trajs: dict, self_id, window,
                      poses) -> np.ndarray:
    """init_pose_by_loops with numpy: good_sets {(lo, hi): ids} (the PCM directory), estimated bool [D], kf {drone:
    (stamps, poses)}, trajs {drone: (stamps, poses)} -> new poses; raises Refused"""
    D = lmap.pair_min.shape[0]
    frame_stamps, frame_first, entries = window
    frame_of = np.repeat(np.arange(len(frame_stamps)), np.diff(np.asarray(frame_first)))
    has_traj = np.array([d in trajs and len(trajs[d][0]) > 0 for d in range(D)])
    est = np.asarray(estimated, bool)
    choice = {}
    for d in np.nonzero(np.asarray(to_init, bool)[:D])[0]:
        d = int(d)
        mine = {(b if a == d else a): np.asarray(ids, np.int64) for (a, b), ids in good_sets.items() if d in (a, b)}
        if mine:
            cand = [(j, int(ids.min())) for j, ids in sorted(mine.items()) if len(ids)]
        else:
            js = np.nonzero(lmap.pair_min[d] != I64_MAX)[0]
            cand = [(int(j), int(lmap.pair_min[d, j])) for j in js]
        cand = [(j, i) for j, i in cand if est[j]]
        for j, i in cand:
            has_path = j in kf and len(kf[j][0]) > 0
            if not np.isin(i, lmap.recs["id"]) or (not has_traj[j] and (len(entries) > 0 or (j == self_id and not has_path))):
                raise Refused(f"drone {d}: pair with {j}, loop {i}")
        if cand:
            choice[d] = cand[-1]
    out = np.array(poses, np.float64, copy=True)
    for d, (j, lid) in choice.items():
        if not has_traj[j]:
            continue
        r = lmap.recs[np.searchsorted(lmap.recs["id"], lid)]
        ta, tb, rel = int(r["stamp_a"]), int(r["stamp_b"]), np.array(r["rel_pose"], np.float64)
        if int(r["id_a"]) != j:
            ta, tb, rel = tb, ta, pr.pose_inv(rel)
        ts_j, tp_j = np.asarray(trajs[j][0], np.int64), np.asarray(trajs[j][1], np.float64)
        t0, pose0 = ta, IDENTITY.copy()
        if j in kf and len(kf[j][0]) > 0:
            k = int(ar._nearest_vec(np.asarray(kf[j][0], np.int64), np.array([ta]))[0])
            t0, pose0 = int(kf[j][0][k]), np.array(kf[j][1][k], np.float64)
        elif j == self_id:
            k = int(ar._nearest_vec(ts_j, np.array([ta]))[0])
            t0, pose0 = int(ts_j[k]), tp_j[k].copy()
        pre = ar._pose_mul_vec(ar._pose_mul_vec(pose0[None], _rel_vec(ts_j, tp_j, np.array([t0]), np.array([ta]))),
                               rel[None])
        sel = np.nonzero(entries["drone_id"] == d)[0]               # frame order: a shared block keeps its latest frame
        if len(sel) == 0:
            continue
        fts = np.asarray(frame_stamps, np.int64)[frame_of[sel]]
        p = ar._pose_mul_vec(np.repeat(pre, len(sel), 0), _rel_vec(ts_j, tp_j, np.full(len(sel), tb), fts))
        blk = entries["block"][sel]
        _, rev = np.unique(blk[::-1], return_index=True)
        last = len(blk) - 1 - rev                                    # each block's latest entry
        out[blk[last], :3] = p[last, :3]
        out[blk[last], 3] = ar._yaw_vec(p[last, 3:])
    return out
