"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the data association branch of solve():
LocalizationDAInit (localization_DA_init.cpp, .hpp) as swarm_localization_solver.cpp:893-916 calls it.

`DAInit` is the literal form over dicts and sets: try_data_association's bookkeeping (the LAST detection of an
anonymous id in raw_dets / uniden_detector, drone_dets_by_pair[id_b][id_a] in store order), t0 and est_poses_t0, the
recursive DFS with its quirks kept (verify() always 0 because of `dis = max_dis`, drone 0 guessed but never estimated,
the first success of a level kept while its other candidates are still searched, the next id tried after a failed one,
the `est_poses_t0.size() == available_nodes.size()` leaf test), estimate_path from the smallest detector's first
detection, and the in-place renaming.  Where the reference throws (a map's at()), it raises Refused; past 32 anonymous
ids or max_nodes DFS calls it raises Capacity (the device's bounds, DESIGN.md section 7b).

`da_vec` computes the same over the device's representation: the store's detection rows in order, the estimates as a
[D, 7] array with a mask, and the DFS as the explicit stack the kernel walks.  tests/test_da_init_ref.py checks the two
forms against each other and pins each quirk.

swarm_msgs is not in the reference tree.  Pose product, inverse and log_map are oracle/pcm_ref.py's; a trajectory look-up
is the nearest sample, ties to the earlier (oracle/anchor_ref.py), and get_relative_pose_by_appro_ts(t1, t2) =
pose(t1)^-1 pose(t2).  Pose::MahalanobisDistance(a, b, cov) = computeSquaredMahalanobisDistance(log_map(a^-1 b), cov),
the squared form verify() uses against the same accept_thres, with oracle/pcm_ref.py's unpivoted Cholesky.
"""
from __future__ import annotations

import numpy as np

from oracle import anchor_ref as ar
from oracle import pcm_ref as pr

MAX_IDS = 32
DET_TYPES = (1, 2)                     # OSB_MEAS_DET4D, OSB_MEAS_DET6D: add_new_detection pushes both


class Refused(Exception):
    """where the reference throws"""


class Capacity(Exception):
    """more than 32 anonymous ids, or more DFS calls than the budget"""


def smd(v, C):
    """computeSquaredMahalanobisDistance: oracle/pcm_ref.py's unpivoted Cholesky (inf when C is not SPD)"""
    return pr.cholesky_smd(np.asarray(v, np.float64), np.asarray(C, np.float64))


def mahalanobis(a, b, cov):
    """Pose::MahalanobisDistance(a, b, cov)"""
    return smd(pr.log_map(pr.pose_mul(pr.pose_inv(a), b)), cov)


def gate(nodes, enable, n_detections) -> bool:
    """has_node_not_inited && all_nodes.size() > 1 && all_detections_6d.size() > 0 (enable_data_association given)"""
    nodes, enable = np.asarray(nodes, bool), np.asarray(enable, bool)
    return bool(np.any(nodes & ~enable)) and int(nodes.sum()) > 1 and n_detections > 0


def det_of(row) -> dict:
    return dict(id_a=int(row["id_a"]), id_b=int(row["id_b"]), ts_a=int(row["stamp_a"]), ts_b=int(row["stamp_b"]),
                rel=np.array(row["relative_pose"], np.float64), cov=np.array(row["cov"], np.float64).reshape(6, 6))


class DAInit:
    """LocalizationDAInit over dicts and sets.  trajs {drone: (stamps, poses)}, kf {drone: (stamps, poses)} (the keyframe
    paths), dets: the detection rows of the store in order (lib.MEASUREMENT_DTYPE)"""

    def __init__(self, self_id, trajs: dict, kf: dict, dets, accept_thres: float, anon_min=1000, max_nodes=1 << 20):
        self.self_id = self_id
        self.ego = {int(d): ar.Trajectory(*v) for d, v in trajs.items() if len(v[0])}
        self.kf = {int(d): v for d, v in kf.items() if len(v[0])}
        self.dets = [det_of(r) for r in dets]
        self.accept_thres = float(np.float32(accept_thres))       # a float parameter held as a double member
        self.anon_min, self.max_nodes = anon_min, max_nodes
        self.available_nodes = sorted(self.ego)
        self.drone_dets_pair, self.drone_dets_by_pair, self.uniden_detector = {}, {}, {}
        self.nodes = self.gates = 0                                 # DFS calls and Mahalanobis gate evaluations

    def ego_at(self, d) -> ar.Trajectory:
        if d not in self.ego:
            raise Refused(f"ego_motions.at({d})")
        return self.ego[d]

    def rel(self, d, t1, t2):
        tr = self.ego_at(d)
        return pr.pose_mul(pr.pose_inv(tr.poses[tr.nearest(t1)]), tr.poses[tr.nearest(t2)])

    @staticmethod
    def at(m: dict, k):
        if k not in m:
            raise Refused(f"at({k})")
        return m[k]

    def try_data_association(self):
        """-> (success, guess {anonymous id: drone}, the renamed id_b of every detection)"""
        unidentified, raw = set(), {}
        for det in self.dets:
            if det["id_b"] >= self.anon_min and det["id_a"] in self.ego:
                unidentified.add(det["id_b"])
                raw[det["id_b"]] = det
                self.uniden_detector[det["id_b"]] = det["id_a"]
                self.drone_dets_pair.setdefault(det["id_a"], {}).setdefault(det["id_b"], []).append(det)
                self.drone_dets_by_pair.setdefault(det["id_b"], {}).setdefault(det["id_a"], []).append(det)
        ids = [d["id_b"] for d in self.dets]
        if not unidentified or self.self_id not in self.ego:
            return False, {}, ids
        t0 = max(int(tr.stamps[0]) for tr in self.ego.values())
        tr = self.ego[self.self_id]
        est = {self.self_id: tr.poses[tr.nearest(t0)].copy()}
        for d in sorted(self.kf):
            stamps, poses = self.kf[d]
            k = ar.Trajectory(stamps, poses).nearest(t0)
            est[d] = pr.pose_mul(np.asarray(poses[k], np.float64), self.rel(d, int(stamps[k]), t0))
        if len(unidentified) > MAX_IDS:
            raise Capacity(f"{len(unidentified)} anonymous ids")
        guess = {}
        ok, _ = self.dfs(est, guess, unidentified, raw, t0)
        if not ok:
            return False, {}, ids
        out = [self.at(guess, i) if i >= self.anon_min else i for i in ids]
        return True, dict(guess), out

    def verify(self, est, guess):
        max_dis = 0.0
        for detector in sorted(self.drone_dets_pair):
            for target_u in sorted(self.drone_dets_pair[detector]):
                target = self.at(guess, target_u)
                if target >= 0:
                    edge = self.drone_dets_pair[detector][target_u][0]
                    est_rel = pr.pose_mul(pr.pose_inv(self.at(est, detector)), self.at(est, target))
                    dis = smd(pr.log_map(pr.pose_mul(pr.pose_inv(est_rel), edge["rel"])), edge["cov"])
                    if dis > max_dis:
                        dis = max_dis                              # the reference's bug: max_dis stays 0
        return max_dis

    def estimate_path(self, u, guess, est, t0):
        new_id = guess[u]
        det_id_a = min(self.drone_dets_by_pair[u])                 # .begin(): the smallest detector
        edge = self.drone_dets_by_pair[u][det_id_a][0]              # its first detection
        odoma = self.rel(edge["id_a"], t0, edge["ts_a"])
        odomb = self.rel(new_id, edge["ts_b"], t0)
        return pr.pose_mul(pr.pose_mul(pr.pose_mul(self.at(est, edge["id_a"]), odoma), edge["rel"]), odomb)

    def dfs(self, est, guess, unidentified, raw, t0):
        self.nodes += 1
        if self.nodes > self.max_nodes:
            raise Capacity("the DFS budget")
        if not unidentified:
            cost = self.verify(est, guess)
            if cost >= 0 and cost < self.accept_thres and len(est) == len(self.available_nodes):
                return True, cost
            return False, -1
        for u in sorted(unidentified):
            if self.uniden_detector[u] not in est or u in guess:
                continue
            best_cost, best_guess, best_est = 1000000, None, None
            cov = raw[u]["cov"]
            for i in range(len(self.available_nodes) + 1):
                new_id = self.available_nodes[i] if i < len(self.available_nodes) else -1
                if self.uniden_detector[u] == new_id or new_id not in self.ego or raw[u]["id_a"] not in self.ego:
                    continue
                new_guess = dict(guess)
                new_guess[u] = new_id
                new_est = dict(est)
                if new_id > 0:
                    pose = self.estimate_path(u, new_guess, new_est, t0)
                    if new_id in new_est:
                        self.gates += 1
                        if not mahalanobis(new_est[new_id], pose, cov) < self.accept_thres:
                            continue
                    new_est[new_id] = pose
                ok, c = self.dfs(new_est, new_guess, unidentified - {u}, raw, t0)
                if ok and c < best_cost:
                    best_cost, best_guess, best_est = c, new_guess, new_est
            if best_cost < 1000000:
                guess.clear(); guess.update(best_guess)
                est.clear(); est.update(best_est)
                return True, best_cost
        return False, -1


def da_literal(self_id, trajs, kf, dets, accept_thres, anon_min=1000, max_nodes=1 << 20, stats=None):
    """-> (applied, status, guess, id_b after the call) with status 'ok' / 'invalid' / 'capacity'; stats (a dict) gets
    the search's DFS calls ("nodes") and Mahalanobis gate evaluations ("gates")"""
    ids = [int(r["id_b"]) for r in dets]
    lit = DAInit(self_id, trajs, kf, dets, accept_thres, anon_min, max_nodes)
    try:
        ok, guess, out = lit.try_data_association()
    except Refused:
        ok, guess, out, status = False, {}, ids, "invalid"
    except Capacity:
        ok, guess, out, status = False, {}, ids, "capacity"
    else:
        status = "ok"
    if stats is not None:
        stats.update(nodes=min(lit.nodes, max_nodes), gates=lit.gates)
    return ok, status, guess, out


# ---- the same over the device's representation ------------------------------------------------------------------
def da_vec(self_id, trajs: dict, kf: dict, dets, accept_thres, anon_min=1000, max_nodes=1 << 20, max_drones=256,
           stats=None):
    """the kernel's walk: detection rows in store order, est as [D, 7] with a mask, the DFS as an explicit stack; stats
    (a dict) gets the DFS calls ("nodes", at most max_nodes) and Mahalanobis gate evaluations ("gates")"""
    D = max_drones
    count = stats if stats is not None else {}
    count.update(nodes=0, gates=0)
    thres = float(np.float32(accept_thres))
    id_a = np.asarray(dets["id_a"], np.int64)
    id_b = np.asarray(dets["id_b"], np.int64)
    ts = {d: (np.asarray(v[0], np.int64), np.asarray(v[1], np.float64)) for d, v in trajs.items() if len(v[0])}
    avail = np.array([d in ts for d in range(D)])
    anon = id_b >= anon_min
    with_traj = anon & np.array([bool(avail[a]) for a in id_a], bool)
    u_ids = np.unique(id_b[with_traj])
    if len(u_ids) == 0 or not avail[self_id]:
        return False, "ok", {}, id_b.tolist()
    n_u = len(u_ids)
    last = np.array([np.nonzero(with_traj & (id_b == u))[0].max() for u in u_ids])
    det_min = np.array([id_a[with_traj & (id_b == u)].min() for u in u_ids])
    first = np.array([np.nonzero(with_traj & (id_b == u) & (id_a == m))[0].min() for u, m in zip(u_ids, det_min)])
    need = np.zeros(D, bool)
    need[id_a[with_traj]] = True
    orphan = bool(np.any(anon & ~np.isin(id_b, u_ids)))

    def ego(d, t):
        s, p = ts[d]
        return p[int(ar._nearest_vec(s, np.array([t]))[0])]

    def rel(d, t1, t2):
        return pr.pose_mul(pr.pose_inv(ego(d, t1)), ego(d, t2))

    t0 = max(int(v[0][0]) for v in ts.values())
    est = np.zeros((D, 7))
    has = np.zeros(D, bool)
    est[self_id], has[self_id] = ego(self_id, t0), True
    for d in sorted(kf):
        s, p = np.asarray(kf[d][0], np.int64), np.asarray(kf[d][1], np.float64)
        if len(s) == 0:
            continue
        if not avail[d]:
            return False, "invalid", {}, id_b.tolist()
        k = int(ar._nearest_vec(s, np.array([t0]))[0])
        est[d], has[d] = pr.pose_mul(p[k], rel(d, int(s[k]), t0)), True
    if n_u > MAX_IDS:
        return False, "capacity", {}, id_b.tolist()
    detector = id_a[last]
    rem = [(1 << n_u) - 1] + [0] * n_u
    u_at, c_at, g = [0] * (n_u + 1), [0] * (n_u + 1), [0] * (n_u + 1)
    found, had, old = [False] * (n_u + 1), [False] * (n_u + 1), [None] * (n_u + 1)
    lvl, nodes, ret, result, step = 0, 0, False, None, "enter"
    while True:
        if step == "enter":
            nodes += 1
            if nodes > max_nodes:
                return False, "capacity", {}, id_b.tolist()
            count["nodes"] = nodes
            if rem[lvl] == 0:
                want = need.copy()
                want[g[:lvl]] = True
                if np.any(want & ~has):
                    return False, "invalid", {}, id_b.tolist()
                ret = thres > 0.0 and bool(np.array_equal(has, avail))
                if ret and result is None:
                    result = {int(u_ids[u_at[l]]): int(g[l]) for l in range(lvl)}
                step = "return"
                continue
            u_at[lvl] = -1
            step = "next_u"
            continue
        if step == "return":
            if lvl == 0:
                break
            lvl -= 1
            c = c_at[lvl]
            if c > 0:
                if had[lvl]:
                    est[c] = old[lvl]
                else:
                    has[c] = False
            found[lvl] = found[lvl] or ret
            step = "next_c"
            continue
        if step == "next_u":
            u = u_at[lvl] + 1
            while u < n_u and (not (rem[lvl] >> u) & 1 or not has[detector[u]]):
                u += 1
            if u >= n_u:
                ret, step = False, "return"
                continue
            u_at[lvl], c_at[lvl], found[lvl] = u, -1, False
            step = "next_c"
            continue
        u = u_at[lvl]
        c = c_at[lvl] + 1
        while c < D and (not avail[c] or c == detector[u]):
            c += 1
        if c >= D:
            if found[lvl]:
                ret, step = True, "return"
            else:
                step = "next_u"
            continue
        c_at[lvl], had[lvl] = c, False
        if c > 0:
            e = dets[first[u]]
            a = int(e["id_a"])
            if not has[a]:
                return False, "invalid", {}, id_b.tolist()
            pose = pr.pose_mul(pr.pose_mul(pr.pose_mul(est[a], rel(a, t0, int(e["stamp_a"]))),
                                           np.asarray(e["relative_pose"], np.float64)), rel(c, int(e["stamp_b"]), t0))
            had[lvl] = bool(has[c])
            if had[lvl]:
                cov = np.asarray(dets[last[u]]["cov"], np.float64).reshape(6, 6)
                count["gates"] += 1
                if not mahalanobis(est[c], pose, cov) < thres:
                    continue
                old[lvl] = est[c].copy()
            est[c], has[c] = pose, True
        g[lvl] = c
        rem[lvl + 1] = rem[lvl] & ~(1 << u)
        lvl += 1
        step = "enter"
    if not ret:
        return False, "ok", {}, id_b.tolist()
    if orphan:
        return False, "invalid", {}, id_b.tolist()
    return True, "ok", result, [result[int(i)] if i >= anon_min else int(i) for i in id_b]
