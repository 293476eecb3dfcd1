"""ORACLE (test infrastructure, NOT product code) -- what a round of loop edges hands from the front-end to the back-end:

  loop_measurements        the success branch of LoopDetector::compute_loop that fills the LoopEdge
                           (swarm_loop/src/loop_detector.cpp:787-829) for every candidate of a round, in candidate order,
                           with its two counters: loop_count numbers the ids (ret.id = self_id * MAX_LOOP_ID + loop_count,
                           :811, :814) and inter_drone_loop_count[new][old] / [old][new] grow by one each (:824-827);
  add_new_loop_connection  SwarmLocalizationSolver::add_new_loop_connection's gate (swarm_localization_solver.cpp:558-588):
                           a loop whose relative_pose.pos().norm() exceeds loop_outlier_distance_threshold is dropped.

Deliberate deviation: the id is computed in int64; the reference computes it in int and overflows for self_id >= 22.
The threshold is a float in the reference's parameters (swarm_localization_params.hpp:25) and is widened to double for the
comparison.  Rows are numpy records laid out as osb_measurement (include/omniswarm_b200.h), restated here.
"""
from __future__ import annotations

import numpy as np

MAX_LOOP_ID = 100000000               # loop_detector.cpp:9
PAIR_DRONES = 256                     # the counters are kept for drone ids 0..255
LOOP_ACCEPTED = 0
MEAS_LOOP = 0
MEASUREMENT_DTYPE = np.dtype([("id", "<i8"), ("type", "<i4"), ("id_a", "<i4"), ("id_b", "<i4"), ("reserved", "<i4"),
                              ("stamp_a", "<i8"), ("stamp_b", "<i8"), ("relative_pose", "<f8", 7), ("cov", "<f8", (6, 6)),
                              ("self_pose_a", "<f8", 7), ("self_pose_b", "<f8", 7)])


def new_counters():
    """the two counters as a fresh LoopDetector holds them: (loop_count, inter_drone_loop_count [256, 256])"""
    return 0, np.zeros((PAIR_DRONES, PAIR_DRONES), np.int64)


def loop_measurements(edges, swapped, cands, stamps, self_id, loop_cov_pos, loop_cov_ang, counters):
    """edges [n]: dicts with status, drone_id_a (old), drone_id_b (new), relative_pose [7]; swapped [n]: the query result's
    roles (1: old = the query keyframe); cands [n]: dicts with pose_query, pose_hit [7]; stamps [n]: (stamp_query_ns,
    stamp_hit_ns); counters: (loop_count, pair_counts) before the round
    -> (rows [k] of MEASUREMENT_DTYPE, counters after the round)"""
    loop_count, pairs = counters
    pairs = pairs.copy()
    rows = []
    for e, sw, c, (t_query, t_hit) in zip(edges, swapped, cands, stamps):
        if e["status"] != LOOP_ACCEPTED:          # only a loop that passed every check is published (:813-829)
            continue
        old_is_query = bool(sw)
        r = np.zeros((), MEASUREMENT_DTYPE)
        r["id"] = int(self_id) * MAX_LOOP_ID + loop_count
        r["type"] = MEAS_LOOP
        r["id_a"], r["id_b"] = e["drone_id_a"], e["drone_id_b"]
        r["stamp_a"], r["stamp_b"] = (t_query, t_hit) if old_is_query else (t_hit, t_query)
        r["self_pose_a"] = c["pose_query"] if old_is_query else c["pose_hit"]
        r["self_pose_b"] = c["pose_hit"] if old_is_query else c["pose_query"]
        r["relative_pose"] = e["relative_pose"]
        r["cov"] = np.diag([loop_cov_pos] * 3 + [loop_cov_ang] * 3)
        rows.append(r)
        loop_count += 1
        old, new = int(e["drone_id_a"]), int(e["drone_id_b"])
        if 0 <= old < PAIR_DRONES and 0 <= new < PAIR_DRONES:
            pairs[new, old] += 1
            pairs[old, new] += 1
    return np.array(rows, MEASUREMENT_DTYPE).reshape(-1), (loop_count, pairs)


def loop_distance(row):
    """relative_pose.pos().norm() as Eigen sums it: sqrt((x*x + y*y) + z*z), every operation rounded on its own"""
    x, y, z = (np.float64(v) for v in row["relative_pose"][:3])
    return np.sqrt((x * x + y * y) + z * z)


def add_new_loop_connection(rows, loop_outlier_distance_threshold):
    """the rows the solver stores, in order: loops no farther than the float threshold, and every detection"""
    thres = np.float64(np.float32(loop_outlier_distance_threshold))
    keep = [r["type"] != MEAS_LOOP or not (loop_distance(r) > thres) for r in rows]
    return np.asarray(rows, MEASUREMENT_DTYPE)[np.array(keep, bool)] if len(rows) else np.asarray(rows, MEASUREMENT_DTYPE)
