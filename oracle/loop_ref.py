"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the step from a loop hit to a LoopEdge
(paths relative to /root/reference/swarm_loop/src):
  * LoopDetector::compute_loop                                 loop_detector.cpp:627-836 -- gates on landmark_num (:632) and on
      the correspondences (:664-693), compute_relative_pose (:355-413), the LoopEdge fields (:787-811) and
      check_loop_odometry_consistency (:813);
  * the frame-level compute_correspond_features                 :431-537 -- direction pairs in dirs_new order, the per-pair
      lists appended in that order whatever the per-image function returned (:488: its `return false` after pushing 1-3
      flagged matches, :598-600, is ignored), MIN_MATCH_PRE_DIR per pair, MIN_DIRECTION_LOOP, and the old side's normalised
      points rotated into the old main direction by rotate_pt_norm2d (:415-428, :516-523);
  * PnP-RANSAC and the checks are oracle/pnp_ref.py's.
The inputs are what the device holds: per direction pair the filtered lists (geo_valid = 1) or the raw matches, the new side's
landmarks_flag / landmarks_3d and the old side's pixel keypoints, lifted through a distortion-free pinhole
(liftProjective(x, y) = ((x - cx) / fx, (y - cy) / fy, 1), rounded to float as toCV does).  Quaternions are unit quaternions,
so the inverse of :515-516 is the conjugate.  The PnP prior is (pose_now^-1 pose_old extrinsic)^-1 evaluated left to right
with pcm_ref's pose algebra; the device evaluates it in the same order without fused multiply-adds, so the two are equal bit
for bit.
"""
from __future__ import annotations

import numpy as np

from . import pcm_ref as pr
from . import pnp_ref as pn

(ACCEPTED, NO_HIT, NO_FRAME, FEW_LANDMARKS, CORRESPONDENCE_FAILED, TOO_FEW_COMMON, PNP_FAILED, NOT_VERIFIED,
 ODOMETRY_INCONSISTENT) = range(9)
MAX_DIRS = 4

DEFAULT_PARAMS = dict(min_loop_num=15, init_mode_min_loop_num=10, min_match_per_dir=15, min_direction_loop=3, is_4dof=1,
                      reproj_thresh=3.0, seed=0, rperr_thres=10 * np.pi / 180, accept_loop_yaw_rad=30 * np.pi / 180,
                      max_loop_dis=5.0, odometry_consistency_threshold=2.0)


def lift(kpt, K):
    """liftProjective of the pinhole K = (fx, fy, cx, cy), in float64, rounded to float (toCV)"""
    fx, fy, cx, cy = (float(v) for v in K)
    return np.float32((float(kpt[0]) - cx) / fx), np.float32((float(kpt[1]) - cy) / fy)


def rotate_pt_norm2d(pt, q):
    """loop_detector.cpp:415-428: (x, y, 1) rotated by q in float64 from the float point, z clamped to +-1e-3, -> float"""
    r = pr.q_rot(np.asarray(q, np.float64), np.array([float(pt[0]), float(pt[1]), 1.0]))
    z = r[2]
    if 0 < z < 1e-3:
        z = 1e-3
    if -1e-3 < z < 0:
        z = -1e-3
    return np.float32(r[0] / z), np.float32(r[1] / z)


def pnp_prior(pose_now, pose_old, extrinsic):
    """(pose_now^-1 pose_old extrinsic)^-1, left to right"""
    now, old, ext = (np.asarray(p, np.float64) for p in (pose_now, pose_old, extrinsic))
    return pr.pose_inv(pr.pose_mul(pr.pose_mul(pr.pose_inv(now), old), ext))


def relative_pose(pose_cam, extrinsic, pose_now, is_4dof):
    """DP_old_to_new (:393-400) as a 7-pose x y z, qw qx qy qz (LoopEdge::relative_pose, :788)"""
    p_drone_old_in_new = pr.pose_mul(pr.pose_inv(np.asarray(pose_cam, np.float64)),
                                     pr.pose_inv(np.asarray(extrinsic, np.float64)))
    return pn.delta_pose(p_drone_old_in_new, np.asarray(pose_now, np.float64), bool(is_4dof))


def compute_correspond_features(slots, new, old, K, ext_old, main_dir_old, min_match_per_dir):
    """slots: the direction pairs in dirs_new order, dicts dir_new, dir_old, geo_valid and geo_new / geo_old (geo_valid) or
    match_new / match_old; new: dict flags[d] [n], l3d[d] [n,3]; old: dict kpts[d] [n,2] (pixels).
    -> dict(X [m,3] f32, uv [m,2] f32, dir_new, idx_new, dir_old, idx_old [m], matched_dir_count)"""
    X, uv, dn_l, qi_l, do_l, ti_l = [], [], [], [], [], []
    matched = 0
    q_main_inv = pr.q_conj(np.asarray(ext_old[main_dir_old], np.float64)[3:])
    for s in slots:
        dn, do = int(s["dir_new"]), int(s["dir_old"])
        if s["geo_valid"]:
            pairs = list(zip(s["geo_new"], s["geo_old"]))
        else:          # what the per-image function pushed before returning false: the flagged matches (fewer than 4)
            pairs = [(q, t) for q, t in zip(s["match_new"], s["match_old"]) if new["flags"][dn][q]]
        if len(pairs) >= min_match_per_dir:
            matched += 1
        dq = pr.q_mul(q_main_inv, np.asarray(ext_old[do], np.float64)[3:])
        for q, t in pairs:
            X.append(np.asarray(new["l3d"][dn][q], np.float32))
            uv.append(rotate_pt_norm2d(lift(old["kpts"][do][t], K), dq))
            dn_l.append(dn); qi_l.append(int(q)); do_l.append(do); ti_l.append(int(t))
    return dict(X=np.array(X, np.float32).reshape(-1, 3), uv=np.array(uv, np.float32).reshape(-1, 2),
                dir_new=np.array(dn_l, np.int32), idx_new=np.array(qi_l, np.int32), dir_old=np.array(do_l, np.int32),
                idx_old=np.array(ti_l, np.int32), matched_dir_count=matched)


def compute_loop(hit, new, old, K, ext_old, main_dir_new, main_dir_old, cand, params=None):
    """LoopDetector::compute_loop for one hit.
    hit: dict accepted, has_frame (False for a row without a keyframe: put in with db_load, or without 3-D landmarks), slots
    (compute_correspond_features); new / old: dicts drone_id, msg_id, n_kpts [dirs] plus what compute_correspond_features
    reads; ext_old [dirs][7]: the old camera's extrinsics; cand: pose_now, pose_old [7], init_mode, and for same-drone loops
    odom_rel [7] and cov [6,6].  -> dict(status, n_corr, matched_dir_count, the correspondence lists, pnp_params, pnp,
    loop, relative_pose)"""
    p = dict(DEFAULT_PARAMS, **(params or {}))
    init = bool(cand.get("init_mode", False))
    out = dict(status=None, n_corr=0, matched_dir_count=0, pnp=None, loop=None, relative_pose=np.zeros(7),
               drone_id_a=old["drone_id"] if old else -1, drone_id_b=new["drone_id"] if new else -1,
               main_dir_new=main_dir_new, main_dir_old=main_dir_old)
    if not hit["accepted"]:
        out["status"] = NO_HIT
        return out
    if not hit.get("has_frame", True):
        out["status"] = NO_FRAME
        return out
    if int(np.sum(new["n_kpts"])) < p["min_loop_num"]:                     # :632
        out["status"] = FEW_LANDMARKS
        return out
    corr = compute_correspond_features(hit["slots"], new, old, K, ext_old, main_dir_old, p["min_match_per_dir"])
    n = len(corr["X"])
    out.update(corr)
    out["n_corr"] = n
    if not (n > 0 and corr["matched_dir_count"] >= p["min_direction_loop"]):    # :532
        out["status"] = CORRESPONDENCE_FAILED
        return out
    if not (n > p["min_loop_num"] or (init and n > p["init_mode_min_loop_num"])):    # :671
        out["status"] = TOO_FEW_COMMON
        return out
    same = old["drone_id"] == new["drone_id"]
    ext = np.asarray(ext_old[main_dir_old], np.float64)
    prm = dict(iterations=1000 if init else 100, thresh=float(np.float32(p["reproj_thresh"])), seed=int(p["seed"]),
               is_4dof=int(p["is_4dof"]), min_loop_num=p["init_mode_min_loop_num"] if init else p["min_loop_num"],
               same_drone=int(same), rperr_thres=p["rperr_thres"], accept_loop_yaw_rad=p["accept_loop_yaw_rad"],
               max_loop_dis=p["max_loop_dis"], odometry_consistency_threshold=p["odometry_consistency_threshold"],
               prior=pnp_prior(cand["pose_now"], cand["pose_old"], ext), extrinsic=ext,
               drone_pose_now=np.asarray(cand["pose_now"], np.float64), drone_pose_old=np.asarray(cand["pose_old"], np.float64),
               odom_rel=np.asarray(cand.get("odom_rel", [0, 0, 0, 1, 0, 0, 0]), np.float64),
               cov=np.asarray(cand.get("cov", np.eye(6)), np.float64), X=corr["X"], uv=corr["uv"])
    out["pnp_params"] = prm
    res = pn.pnp_ransac(corr["X"], corr["uv"], prm["prior"], prm["iterations"], prm["thresh"], prm["seed"])
    out["pnp"] = res
    if not res["success"]:
        out["status"] = PNP_FAILED
        return out
    v = pn.loop_from_pnp(res, prm)
    out["loop"] = v
    out["relative_pose"] = relative_pose(res["pose"], ext, prm["drone_pose_now"], prm["is_4dof"])
    out["status"] = ACCEPTED if v["verified"] and v["odometry_consistent"] else \
        NOT_VERIFIED if not v["verified"] else ODOMETRY_INCONSISTENT
    return out
