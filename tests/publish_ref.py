"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of what the back-end publishes after each accepted
solve: SwarmLocalizationSolver::sync_est_poses (swarm_localization_solver.cpp:962-1057) and PredictSwarm / PredictNode /
NodeCooridnateOffset (:673-765).

`PublishState` keeps what the reference keeps across solves (est_poses_tsid_saved, last_saved_est_kf_ts, the frames'
odometry poses of all_sf, keyframe_trajs and full_trajs) and restates both literally:
  * sync: every window entry, frames in order, writes its solved block pose (x y z yaw) to the saved state and a sample of
    its drone's keyframe path, stamped with the FRAME stamp, pose = Pose(block, yaw) with att = att * (AngleAxis(-yaw_ego,
    Z) * att_ego), ego = the drone's odometry at the frame stamp; an init sync pushes every frame's stamp, a steady one
    the last frame that has entries; the full path takes every 10th odometry sample (FULL_PATH_STEP, :66), walks to the
    nearest keyframe sample as :1034-1040 do (bounded at the last sample: the reference reads index + 1 before it tests
    the bound) and predicts pose = kf_pose * DeltaPose(vo_ref, ego_i, true), then att = att * att_no_yaw(ego at ts_kf);
  * predict: nothing without finish_init; per drone the latest pushed stamp whose saved frame holds it; node_pose =
    Pose(saved, yaw) * DeltaPose(set_yaw_only(vo), vo_now, false), given only for an enabled drone (self_id always);
    base_pose = set_yaw_only(Pose(saved, yaw)) * set_yaw_only(vo)^-1.
A window drone without odometry raises NoOdometry before anything changes (the reference throws from
ego_motion_trajs.at()).

`full_path_vec` computes the full path with numpy (the host form of scripts/bench_publish.py); `record_sync` is the
per-drone "last pushed frame holding d" record the device keeps instead of the stamp list.  tests/test_publish_ref.py
checks they agree with the literal forms.  Pose algebra is oracle/pcm_ref's, oracle/pnp_ref's and oracle/anchor_ref's.
"""
from __future__ import annotations

import numpy as np

from oracle import anchor_ref as ar
from oracle import pcm_ref as pr
from oracle import pnp_ref as pn

FULL_PATH_STEP = 10


class NoOdometry(KeyError):
    pass


def pose4(p):
    """Pose(double[4], true): x y z yaw -> x y z, qw qx qy qz"""
    return np.concatenate([np.asarray(p[:3], np.float64), pn.quat_from_rotvec(np.array([0.0, 0.0, p[3]]))])


def att_no_yaw(ego):
    """AngleAxisd(-ego.yaw(), Z) * ego.att()"""
    return pr.q_mul(pn.quat_from_rotvec(np.array([0.0, 0.0, -pn.quat2eulers(ego[3:])[2]])), ego[3:])


def walk(kf_stamps, ts_vo, index):
    """the nearest-keyframe walk of :1034-1040 from `index`, bounded at the last sample"""
    n = len(kf_stamps)
    if n > 1:
        while index + 1 < n and abs(ts_vo - kf_stamps[index]) > abs(ts_vo - kf_stamps[index + 1]):
            index += 1
    return index


def full_path(kf, traj: ar.Trajectory):
    """the literal loop of :1026-1053 for one drone: kf = (stamps, poses, vo) of its keyframe path -> (stamps, poses)"""
    kf_stamps, kf_poses, kf_vo = kf
    index, stamps, poses = 0, [], []
    for i in range(0, len(traj.stamps), FULL_PATH_STEP):
        ts_vo = traj.stamps[i]
        index = walk(kf_stamps, ts_vo, index)
        pose = pr.pose_mul(kf_poses[index], pn.delta_pose(kf_vo[index], traj.poses[i], True))
        pose[3:] = pr.q_mul(pose[3:], att_no_yaw(traj.pose_by_appro_ts(kf_stamps[index])))
        stamps.append(ts_vo)
        poses.append(pose)
    return np.array(stamps, np.int64), np.array(poses).reshape(-1, 7)


def full_path_vec(kf, traj_stamps, traj_poses):
    """full_path with numpy: every sample's keyframe by a nearest-sample search (ties to the earlier)"""
    kf_stamps, kf_poses, kf_vo = (np.asarray(x) for x in kf)
    ts = np.asarray(traj_stamps, np.int64)
    tp = np.asarray(traj_poses, np.float64)
    sel = np.arange(0, len(ts), FULL_PATH_STEP)
    k = ar._nearest_vec(kf_stamps.astype(np.int64), ts[sel])
    pose = ar._pose_mul_vec(kf_poses[k], ar._delta_pose4_vec(kf_vo[k], tp[sel]))
    ego = tp[ar._nearest_vec(ts, kf_stamps.astype(np.int64))]                  # per keyframe sample
    q_ego = ar._q_mul_vec(ar._yaw_quat_vec(-ar._yaw_vec(ego[:, 3:])), ego[:, 3:])
    pose[:, 3:] = ar._q_mul_vec(pose[:, 3:], q_ego[k])
    return ts[sel], pose


class PublishState:
    """the reference's state across solves; trajs {drone: anchor_ref.Trajectory} are the odometry at each sync"""

    def __init__(self):
        self.saved = {}            # est_poses_tsid_saved: ts -> {drone: [4]}
        self.vo = {}               # all_sf[ts].id2nodeframe[drone].pose()
        self.pushed = []           # last_saved_est_kf_ts
        self.kf = {}               # keyframe_trajs: drone -> (stamps [n], poses [n, 7], entry self poses [n, 7])
        self.full = {}             # full_trajs: drone -> (stamps, poses)

    def sync(self, window, poses, trajs: dict, is_init: bool, full: bool):
        frames = ar.window_frames(*window)
        for _, nodes in frames:
            for d in nodes:
                if d not in trajs:
                    raise NoOdometry(d)
        poses = np.asarray(poses, np.float64)
        kf = {}
        last_ts = frames[-1][0] if frames else None
        for ts, nodes in frames:
            for d in sorted(nodes):                               # id2nodeframe is a std::map
                nf = nodes[d]
                blk = poses[nf["block"]]
                self.saved.setdefault(ts, {})[d] = blk.copy()
                self.vo.setdefault(ts, {})[d] = nf["self_pose"].copy()
                p = pose4(blk)
                p[3:] = pr.q_mul(p[3:], att_no_yaw(trajs[d].pose_by_appro_ts(ts)))
                s = kf.setdefault(d, ([], [], []))
                s[0].append(ts); s[1].append(p); s[2].append(nf["self_pose"].copy())
                last_ts = ts
                if is_init:
                    self.pushed.append(ts)
        if not is_init and frames:
            self.pushed.append(last_ts)
        self.kf = {d: (np.array(s[0], np.int64), np.array(s[1]), np.array(s[2])) for d, s in kf.items()}
        self.full = {d: full_path(self.kf[d], trajs[d]) for d in self.kf} if full else {}

    def lookup(self, d):
        """the reverse scan of last_saved_est_kf_ts (:679-681, :704-706) -> (ts, saved [4], vo [7]) or None"""
        for ts in reversed(self.pushed):
            if d in self.saved[ts]:
                return ts, self.saved[ts][d], self.vo[ts][d]
        return None

    def predict(self, frame, finish_init: bool, self_id: int, enable) -> dict:
        """frame [(drone, vo pose [7])], enable [drone] of the last observe -> {drone: (node_pose or None, base_pose or
        None)}"""
        if not finish_init:
            return {}
        out = {}
        for d, vo_now in frame:
            node = base = None
            hit = self.lookup(d)
            if hit is not None:
                _, saved, vo = hit
                est, vo4 = pose4(saved), ar.set_yaw_only(vo)
                if d == self_id or enable[d]:
                    node = pr.pose_mul(est, pn.delta_pose(vo4, np.asarray(vo_now, np.float64), False))
                base = pr.pose_mul(ar.set_yaw_only(est), pr.pose_inv(vo4))
            out[d] = (node, base)
        return out


def record_sync(rec: dict, window, poses, is_init: bool):
    """the device's record, updated in place for one applied sync: rec {drone: (ts, saved [4], vo [7])}.  The last frame
    holding d among the frames this sync pushes takes over; otherwise a record whose frame is still in the window is
    rewritten from it; otherwise it stays."""
    frames = ar.window_frames(*window)
    poses = np.asarray(poses, np.float64)
    with_entries = [ts for ts, nodes in frames if nodes]
    pushed = set(with_entries) if is_init else set(with_entries[-1:])
    last = {}
    for ts, nodes in frames:
        for d, nf in nodes.items():
            last[d] = (ts, nf)
    for d, (ts, nf) in last.items():
        if ts in pushed:
            rec[d] = (ts, poses[nf["block"]].copy(), nf["self_pose"].copy())
        elif d in rec:
            for ts2, nodes in frames:
                if ts2 == rec[d][0] and d in nodes:
                    rec[d] = (ts2, poses[nodes[d]["block"]].copy(), nodes[d]["self_pose"].copy())
                    break
    return rec
