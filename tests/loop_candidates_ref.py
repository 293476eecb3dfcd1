"""ORACLE (test infrastructure, NOT product code) -- the keyframe metadata the device keeps and a round's loop candidates
built from it (osb_frontend_ingest_meta, osb_frontend_loop_candidates_dev, osb_frontend_init_modes_dev):

  stores       each database's frame slots as add_to_database assigns them (loop_detector.cpp:150-173): a frame per
               ingested record, a row per direction with landmarks, and the osb_keyframe_meta of the frame when one was
               ingested beside the record with the record's drone_id and msg_id (fisheyeframe_database[msg_id]);
  trajectory   ego_motion_traj (:27), own keyframes only, in ingest order: a stamp not after the last sample is refused;
               length[k] = length[k-1] + sqrt((dx*dx + dy*dy) + dz*dz); a look-up takes the nearest sample (ties to the
               earlier, clamped); relative pose (ta, tb) = pose(ta)^-1 * pose(tb) (oracle/pcm_ref.py's algebra, every
               operation rounded on its own), covariance |len(tb) - len(ta)| * diag(pos x3, ang x3);
  init_mode    on_image_recv's rule (:65-72) on inter_drone_loop_count [256][256] ([new][old]);
  candidates   the osb_loop_candidate / osb_loop_stamps bytes of each query result: query side from the round's metas, hit
               side from the hit's frame, odometry for same-drone hits (check_loop_odometry_consistency, :294-303) plus the
               loop covariance; reserved = 1 marks an accepted candidate whose query or hit has no meta.

The status codes and byte layouts restate include/omniswarm_b200.h.
"""
from __future__ import annotations

import numpy as np

from oracle import pcm_ref as pr

OK, ERR_INVALID, ERR_CAPACITY = 0, 1, 3
REMOTE_MAGIN_NUMBER = 1000000
PAIR_DRONES = 256
MAX_DIRS = 4
IDENTITY = np.array([0, 0, 0, 1, 0, 0, 0], np.float64)
META_DTYPE = np.dtype([("drone_id", "<i4"), ("msg_id", "<i4"), ("stamp_ns", "<i8"), ("pose_drone", "<f8", 7)])
CAND_DTYPE = np.dtype([("init_mode", "<i4"), ("reserved", "<i4"), ("pose_query", "<f8", 7), ("pose_hit", "<f8", 7),
                       ("odom_rel", "<f8", 7), ("odom_edge_cov", "<f8", (6, 6))])
STAMPS_DTYPE = np.dtype([("stamp_query_ns", "<i8"), ("stamp_hit_ns", "<i8")])


def _get(o, k):
    return o[k] if isinstance(o, dict) else getattr(o, k)


def metas(items):
    """[(drone_id, msg_id, stamp_ns, pose [7])] -> META_DTYPE array"""
    out = np.zeros(len(items), META_DTYPE)
    for m, (d, msg, t, p) in zip(out, items):
        m["drone_id"], m["msg_id"], m["stamp_ns"], m["pose_drone"] = d, msg, t, p
    return out


class Trajectory:
    """the own keyframes' ego-motion trajectory as the device keeps it"""

    def __init__(self, cap: int):
        self.cap = cap
        self.stamps, self.poses, self.length = [], [], []

    def append(self, stamp: int, pose) -> int:
        n = len(self.stamps)
        if n and stamp <= self.stamps[-1]:
            return ERR_INVALID
        if n >= self.cap:
            return ERR_CAPACITY
        p = np.asarray(pose, np.float64).copy()
        ln = 0.0
        if n:
            q = self.poses[-1]
            dx, dy, dz = p[0] - q[0], p[1] - q[1], p[2] - q[2]
            ln = self.length[-1] + np.sqrt((dx * dx + dy * dy) + dz * dz)
        self.stamps.append(int(stamp)); self.poses.append(p); self.length.append(np.float64(ln))
        return OK

    def nearest(self, t: int) -> int:
        s, n = self.stamps, len(self.stamps)
        lo = next((k for k in range(n) if s[k] >= t), n)          # first sample at or after t
        if lo == 0:
            return 0
        if lo == n:
            return n - 1
        return lo - 1 if t - s[lo - 1] <= s[lo] - t else lo

    def relative(self, ta: int, tb: int, pos_per_m: float, ang_per_m: float):
        """(pose(ta)^-1 pose(tb), |len(tb) - len(ta)|, the covariance diag) of get_relative_pose_by_ts"""
        ka, kb = self.nearest(ta), self.nearest(tb)
        rel = pr.pose_mul(pr.pose_inv(self.poses[ka]), self.poses[kb])
        dl = abs(self.length[kb] - self.length[ka])
        return rel, dl, [dl * pos_per_m] * 3 + [dl * ang_per_m] * 3


class MetaStores:
    """both databases' frame slots and metas, and the trajectory, fed the records' headers as ingest feeds the device"""

    def __init__(self, self_id: int, cap: int):
        self.self_id, self.cap = self_id, cap
        self.traj = Trajectory(cap)
        self.status = OK
        self.reset()

    def reset(self):
        """osb_frontend_db_reset: the stores empty, the trajectory kept"""
        self.frames = [[], []]          # per store: meta (a META_DTYPE record) or None per frame slot
        self.rows = [[], []]            # per store: frame slot per row

    def ingest(self, recs, metas_=None, skip=-1):
        """recs: records (drone_id, msg_id, n_dirs, n_kpts); metas_: META_DTYPE [n] (ingest_meta) or None (ingest)"""
        status = OK
        for r, rec in enumerate(recs):
            if r == skip:
                continue
            remote = int(_get(rec, "drone_id") != self.self_id)
            fr = self.frames[remote]
            if len(fr) >= self.cap:
                continue
            meta = None
            if metas_ is not None:
                m = metas_[r]
                if m["drone_id"] == _get(rec, "drone_id") and m["msg_id"] == _get(rec, "msg_id"):
                    meta = m.copy()
                    if not remote:
                        s = self.traj.append(int(m["stamp_ns"]), m["pose_drone"])
                        status = status if status != OK or s == OK else s
                else:
                    status = status if status != OK else ERR_INVALID
            fs = len(fr)
            fr.append(meta)
            nk = _get(rec, "n_kpts")
            for d in range(MAX_DIRS):
                if d < _get(rec, "n_dirs") and nk[d] > 0 and len(self.rows[remote]) < self.cap:
                    self.rows[remote].append(fs)
        if metas_ is not None:
            self.status = status

    def hit_meta(self, res):
        hid = _get(res, "hit_id")
        remote = int(hid >= REMOTE_MAGIN_NUMBER)
        return self.frames[remote][self.rows[remote][hid - REMOTE_MAGIN_NUMBER if remote else hid]]


def init_mode(drone: int, self_id: int, pairs, init_frames: int) -> bool:
    if drone == self_id:
        return False
    inside = 0 <= drone < PAIR_DRONES and 0 <= self_id < PAIR_DRONES
    return not ((int(pairs[drone, self_id]) if inside else 0) >= init_frames)


def init_modes(recs, skip, self_id, pairs, init_frames) -> np.ndarray:
    return np.array([0 if r == skip else int(init_mode(_get(rec, "drone_id"), self_id, pairs, init_frames))
                     for r, rec in enumerate(recs)], np.uint8)


def candidates(stores: MetaStores, recs, metas_, results, pairs, prm: dict, init_flags=None):
    """-> (CAND_DTYPE [n], STAMPS_DTYPE [n]).  prm: inter_drone_init_frames, pos_covariance_per_meter,
    yaw_covariance_per_meter, loop_cov_pos, loop_cov_ang"""
    n = len(recs)
    cand, stamps = np.zeros(n, CAND_DTYPE), np.zeros(n, STAMPS_DTYPE)
    for i, (rec, mq, res) in enumerate(zip(recs, metas_, results)):
        c = cand[i]
        drone = _get(rec, "drone_id")
        q_ok = mq["drone_id"] == drone and mq["msg_id"] == _get(rec, "msg_id")
        accepted = bool(_get(res, "accepted"))
        mh = stores.hit_meta(res) if accepted else None
        c["init_mode"] = int(init_flags[i] != 0) if init_flags is not None else \
            int(init_mode(drone, stores.self_id, pairs, prm["inter_drone_init_frames"]))
        sq = int(mq["stamp_ns"]) if q_ok else 0
        sh = int(mh["stamp_ns"]) if mh is not None else 0
        c["pose_query"] = mq["pose_drone"] if q_ok else IDENTITY
        c["pose_hit"] = mh["pose_drone"] if mh is not None else IDENTITY
        c["odom_rel"] = IDENTITY
        mark = accepted and (not q_ok or mh is None)
        if accepted and not mark and drone == _get(res, "hit_drone_id"):
            if not stores.traj.stamps:
                mark = True
            else:
                sw = bool(_get(res, "swapped"))                  # a = the old side, b = the new side
                rel, dl, diag = stores.traj.relative(sq if sw else sh, sh if sw else sq, prm["pos_covariance_per_meter"],
                                                     prm["yaw_covariance_per_meter"])
                c["odom_rel"] = rel
                loop = [prm["loop_cov_pos"]] * 3 + [prm["loop_cov_ang"]] * 3
                for k in range(6):
                    c["odom_edge_cov"][k, k] = diag[k] + loop[k]
        c["reserved"] = int(mark)
        stamps[i] = (sq, sh)
    return cand, stamps
