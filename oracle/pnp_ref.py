"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the relative-pose stage that turns a matched
keyframe pair into a LoopEdge (SURVEY.md section 8f-1, second half).

Follows (paths relative to /root/reference/swarm_loop/src):
  * LoopDetector::compute_relative_pose  loop_detector.cpp:355-413 -- cv::solvePnPRansac(matched_3d_now, matched_2d_norm_old,
      K = I, no distortion, iterations 100 (1000 in init mode, :385-391), reprojection error 3 (:393), confidence 0.99),
      p_cam_old_in_new = PnPRestoCamPose(rvec, t), p_drone_old_in_new = p_cam_old_in_new * extrinsic^-1 (:396-397),
      DP_old_to_new = DeltaPose(p_drone_old_in_new, drone_pose_now, is_4dof) (:403), RPerror (:405), pnp_result_verify (:407);
  * RPerror  loop_detector.cpp:338-351;  pnp_result_verify  :317-336;
  * LoopDetector::check_loop_odometry_consistency  :294-315 (same-drone loops only).

OpenCV's solvePnPRansac draws its minimal samples from cv::RNG and solves them with EPnP / P3P, so its inlier set is not
reproducible; its RESULT, however, is well defined: the pose that minimises the squared reprojection error over the inliers
of the best model (final cv::solvePnP(..., SOLVEPNP_ITERATIVE) = Levenberg-Marquardt).  The library defines a DETERMINISTIC
RANSAC with the same error (squared reprojection error in the normalised image plane, no cheirality test -- cv::projectPoints
has none), the same threshold rule (err <= thresh^2) and the same result definition:
  * hypothesis h = 0..iterations-1 draws 4 distinct correspondences from the counter-based hash of geometry_ref.draw4;
  * its model is the LM minimiser of those 4 reprojection errors started from the caller's prior (R0, t0) -- the odometry
    prediction the reference computes and leaves unused, initial_old_cam_pose :377-382 -- with a FIXED schedule (HYP_ITERS
    iterations, lambda x10 on reject, /10 on accept), so it is a pure function of (points, seed, prior);
  * the winner has the most inliers, ties to the smaller h; the inlier set is the winner's;
  * the pose is refined by REFINE_ITERS LM iterations over those inliers.
Pinned against the real OpenCV (cv2.solvePnPRansac) in tests/test_oracle_pins.py on data whose outliers are gross: same
inliers, same pose to 1e-6.  Swarm::Pose / DeltaPose / quat2eulers come from HKUST-Swarm/swarm_msgs, which is not in the
reference tree; they are defined here (pose = (t, unit quaternion wxyz), eulers = ZYX roll-pitch-yaw).
"""
from __future__ import annotations

import numpy as np

from .geometry_ref import draw4
from . import pcm_ref as pr

HYP_ITERS = 8
REFINE_ITERS = 12


def quat_from_rotvec(rv):
    a = float(np.sqrt(rv[0] * rv[0] + rv[1] * rv[1] + rv[2] * rv[2]))
    if a < 1e-12:
        q = np.array([1.0, 0.5 * rv[0], 0.5 * rv[1], 0.5 * rv[2]])
    else:
        s = np.sin(0.5 * a) / a
        q = np.array([np.cos(0.5 * a), s * rv[0], s * rv[1], s * rv[2]])
    return q / np.sqrt(np.dot(q, q))


def quat2eulers(q):
    """ZYX (roll, pitch, yaw) of a unit quaternion wxyz"""
    w, x, y, z = q
    roll = np.arctan2(2.0 * (w * x + y * z), 1.0 - 2.0 * (x * x + y * y))
    pitch = np.arcsin(np.clip(2.0 * (w * y - z * x), -1.0, 1.0))
    yaw = np.arctan2(2.0 * (w * z + x * y), 1.0 - 2.0 * (y * y + z * z))
    return np.array([roll, pitch, yaw])


def wrap(a):
    return a - 2.0 * np.pi * np.floor((a + np.pi) / (2.0 * np.pi))


def reproj_sq(pose, X, uv):
    """squared reprojection errors of points X [n,3] under x_cam = R X + t, normalised plane, no cheirality test"""
    Y = np.stack([pr.q_rot(pose[3:], x) for x in X]) + pose[:3]
    du = Y[:, 0] / Y[:, 2] - uv[:, 0]
    dv = Y[:, 1] / Y[:, 2] - uv[:, 1]
    return du * du + dv * dv


def _normal_eq(pose, X, uv):
    """J^T J (6x6), J^T r (6) and the cost of the reprojection residuals; unknowns (d_theta, d_t), left perturbation"""
    A = np.zeros((6, 6)); g = np.zeros(6); cost = 0.0
    for x, m in zip(X, uv):
        y = pr.q_rot(pose[3:], x)
        p = y + pose[:3]
        iz = 1.0 / p[2]
        r0, r1 = p[0] * iz - m[0], p[1] * iz - m[1]
        cost += r0 * r0 + r1 * r1
        # d p = -[y]x d_theta + d_t ;  d(u,v) = [[iz, 0, -p0 iz^2], [0, iz, -p1 iz^2]] d p
        a = np.array([iz, 0.0, -p[0] * iz * iz]); b = np.array([0.0, iz, -p[1] * iz * iz])
        J0 = np.concatenate([np.cross(y, a), a])          # a^T (-[y]x) = (y x a)^T
        J1 = np.concatenate([np.cross(y, b), b])
        A += np.outer(J0, J0) + np.outer(J1, J1)
        g += J0 * r0 + J1 * r1
    return A, g, cost


def _cost(pose, X, uv):
    return float(np.sum(reproj_sq(pose, X, uv)))


def _solve6(A, b):
    """unpivoted Cholesky solve of the damped normal equations; None if not positive definite"""
    n = 6
    L = np.zeros((n, n))
    for j in range(n):
        s = A[j, j] - np.dot(L[j, :j], L[j, :j])
        if not s > 0:
            return None
        L[j, j] = np.sqrt(s)
        for i in range(j + 1, n):
            L[i, j] = (A[i, j] - np.dot(L[i, :j], L[j, :j])) / L[j, j]
    y = np.zeros(n)
    for i in range(n):
        y[i] = (b[i] - np.dot(L[i, :i], y[:i])) / L[i, i]
    x = np.zeros(n)
    for i in range(n - 1, -1, -1):
        x[i] = (y[i] - np.dot(L[i + 1:, i], x[i + 1:])) / L[i, i]
    return x


def lm_pose(pose0, X, uv, iters):
    """fixed-schedule Levenberg-Marquardt on the reprojection error; -> pose (t, q)"""
    pose = pose0.astype(np.float64).copy()
    lam = 1e-3
    A, g, cost = _normal_eq(pose, X, uv)
    for _ in range(iters):
        Ad = A + lam * np.diag(np.diag(A)) + 1e-12 * np.eye(6)
        d = _solve6(Ad, -g)
        ok = False
        if d is not None and np.all(np.isfinite(d)):
            dq = quat_from_rotvec(d[:3])
            cand = np.concatenate([pr.q_rot(dq, pose[:3]) + d[3:], pr.q_mul(dq, pose[3:])])
            cand[3:] /= np.sqrt(np.dot(cand[3:], cand[3:]))
            c = _cost(cand, X, uv)
            ok = np.isfinite(c) and c < cost
        if ok:
            pose = cand
            A, g, cost = _normal_eq(pose, X, uv)
            lam = max(lam * 0.1, 1e-9)
        else:
            lam = min(lam * 10.0, 1e6)
    return pose


def pnp_ransac(X, uv, prior, iterations=100, thresh=3.0, seed=0):
    """X [n,3] (matched_3d_now), uv [n,2] (matched_2d_norm_old), prior = (t, q) with x_cam_old = R X + t
    -> dict(success, pose (t,q), mask uint8 [n], n_inliers, winner)"""
    X = np.asarray(X, np.float64); uv = np.asarray(uv, np.float64)
    n = len(X)
    if n < 4:
        return dict(success=False, pose=np.asarray(prior, np.float64), mask=np.zeros(n, np.uint8), n_inliers=0, winner=-1)
    t2 = float(thresh) * float(thresh)
    best, best_h, best_pose, best_mask = -1, -1, None, None
    for h in range(iterations):
        idx = draw4(seed, h, n)
        if idx is None:
            continue
        pose = lm_pose(np.asarray(prior, np.float64), X[idx], uv[idx], HYP_ITERS)
        e = reproj_sq(pose, X, uv)
        mask = e <= t2                                   # NaN compares false
        c = int(mask.sum())
        if c > best:
            best, best_h, best_pose, best_mask = c, h, pose, mask
    if best < 4:
        return dict(success=False, pose=np.asarray(prior, np.float64), mask=np.zeros(n, np.uint8), n_inliers=max(best, 0),
                    winner=best_h)
    pose = lm_pose(best_pose, X[best_mask], uv[best_mask], REFINE_ITERS)
    return dict(success=True, pose=pose, mask=best_mask.astype(np.uint8), n_inliers=best, winner=best_h)


# ---- the same RANSAC vectorised over hypotheses and points --------------------------------------------------------
# pnp_ransac's arithmetic, operation by operation, on a leading batch axis: every hypothesis runs the same fixed LM
# schedule with its own lambda, and a hypothesis whose damped system is not positive definite rejects that step alone.
def _q_rot_b(q, v):
    u = q[..., 1:]
    c = np.cross(u, v)
    return v + 2.0 * (q[..., :1] * c + np.cross(u, c))


def _q_mul_b(a, b):
    aw, ax, ay, az = (a[..., i] for i in range(4))
    bw, bx, by, bz = (b[..., i] for i in range(4))
    return np.stack([aw * bw - ax * bx - ay * by - az * bz,
                     aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw], -1)


def _reproj_sq_b(P, X, uv):
    """P [B,7], X [B|1,m,3], uv [B|1,m,2] -> squared reprojection errors [B,m]"""
    Y = _q_rot_b(P[:, None, 3:], X) + P[:, None, :3]
    du = Y[..., 0] / Y[..., 2] - uv[..., 0]
    dv = Y[..., 1] / Y[..., 2] - uv[..., 1]
    return du * du + dv * dv


def _normal_eq_b(P, X, uv):
    """_normal_eq of B poses over their own m points; m = 4 accumulates point by point as _normal_eq does"""
    Y = _q_rot_b(P[:, None, 3:], X)
    p = Y + P[:, None, :3]
    iz = 1.0 / p[..., 2]
    r0, r1 = p[..., 0] * iz - uv[..., 0], p[..., 1] * iz - uv[..., 1]
    zero = np.zeros_like(iz)
    a = np.stack([iz, zero, -p[..., 0] * iz * iz], -1)
    b = np.stack([zero, iz, -p[..., 1] * iz * iz], -1)
    J0 = np.concatenate([np.cross(Y, a), a], -1)
    J1 = np.concatenate([np.cross(Y, b), b], -1)
    Ak = J0[..., :, None] * J0[..., None, :] + J1[..., :, None] * J1[..., None, :]
    gk = J0 * r0[..., None] + J1 * r1[..., None]
    ck = r0 * r0 + r1 * r1
    m = X.shape[1]
    if m <= 4:
        A = np.zeros((len(P), 6, 6)); g = np.zeros((len(P), 6)); cost = np.zeros(len(P))
        for k in range(m):
            A += Ak[:, k]; g += gk[:, k]; cost += ck[:, k]
        return A, g, cost
    return Ak.sum(1), gk.sum(1), ck.sum(1)


def _solve6_b(A, b):
    """_solve6 of B systems -> (x [B,6], ok [B]); ok is False where _solve6 returns None or x is not finite"""
    B = len(A)
    L = np.zeros((B, 6, 6))
    ok = np.ones(B, bool)
    for j in range(6):
        s = A[:, j, j] - np.vecdot(L[:, j, :j], L[:, j, :j])
        ok &= s > 0
        L[:, j, j] = np.sqrt(np.where(ok, s, 1.0))
        for i in range(j + 1, 6):
            L[:, i, j] = (A[:, i, j] - np.vecdot(L[:, i, :j], L[:, j, :j])) / L[:, j, j]
    y = np.zeros((B, 6))
    for i in range(6):
        y[:, i] = (b[:, i] - np.vecdot(L[:, i, :i], y[:, :i])) / L[:, i, i]
    x = np.zeros((B, 6))
    for i in range(5, -1, -1):
        x[:, i] = (y[:, i] - np.vecdot(L[:, i + 1:, i], x[:, i + 1:])) / L[:, i, i]
    return x, ok & np.all(np.isfinite(x), 1)


def _quat_from_rotvec_b(rv):
    a = np.sqrt(rv[:, 0] * rv[:, 0] + rv[:, 1] * rv[:, 1] + rv[:, 2] * rv[:, 2])
    small = a < 1e-12
    ha = np.where(small, 1.0, a)
    s = np.sin(0.5 * ha) / ha
    q = np.where(small[:, None], np.concatenate([np.ones((len(rv), 1)), 0.5 * rv], 1),
                 np.concatenate([np.cos(0.5 * ha)[:, None], s[:, None] * rv], 1))
    return q / np.sqrt(np.vecdot(q, q))[:, None]


def lm_pose_batched(P0, X, uv, iters):
    """lm_pose of B poses P0 [B,7], each over its own points X [B,m,3], uv [B,m,2]"""
    P = np.array(P0, np.float64)
    B = len(P)
    lam = np.full(B, 1e-3)
    A, g, cost = _normal_eq_b(P, X, uv)
    r = np.arange(6)
    for _ in range(iters):
        D = np.zeros_like(A)
        D[:, r, r] = A[:, r, r]
        Ad = A + lam[:, None, None] * D + 1e-12 * np.eye(6)
        d, ok = _solve6_b(Ad, -g)
        d = np.where(ok[:, None], d, 0.0)
        dq = _quat_from_rotvec_b(d[:, :3])
        cand = np.concatenate([_q_rot_b(dq, P[:, :3]) + d[:, 3:], _q_mul_b(dq, P[:, 3:])], 1)
        cand[:, 3:] /= np.sqrt(np.vecdot(cand[:, 3:], cand[:, 3:]))[:, None]
        c = _reproj_sq_b(cand, X, uv).sum(1)
        ok &= np.isfinite(c) & (c < cost)
        if ok.any():
            P[ok] = cand[ok]
            A[ok], g[ok], cost[ok] = _normal_eq_b(P[ok], X[ok], uv[ok])
        lam = np.where(ok, np.maximum(lam * 0.1, 1e-9), np.minimum(lam * 10.0, 1e6))
    return P


def pnp_ransac_batched(X, uv, prior, iterations=100, thresh=3.0, seed=0):
    """pnp_ransac with every hypothesis fitted and scored at once; the same result, plus
    margin = min over hypotheses and points of |e - thresh^2| / thresh^2 (finite errors only; inf if there are none): how
    far the data keep every inlier decision from the threshold, i.e. how much rounding an implementation may differ by
    without changing a mask.  ties counts the finite errors exactly at thresh^2 and margin_untied is the margin without
    them: data built from exactly representable values can put errors on the threshold in every implementation."""
    X = np.asarray(X, np.float64); uv = np.asarray(uv, np.float64)
    prior = np.asarray(prior, np.float64)
    n = len(X)
    out = dict(success=False, pose=prior, mask=np.zeros(n, np.uint8), n_inliers=0, winner=-1, margin=np.inf,
               margin_untied=np.inf, ties=0)
    if n < 4:
        return out
    t2 = float(thresh) * float(thresh)
    hs, idx = [], []
    for h in range(iterations):
        s = draw4(seed, h, n)
        if s is not None:
            hs.append(h); idx.append(s)
    if not hs:
        return out
    idx = np.asarray(idx)
    with np.errstate(all="ignore"):
        P = lm_pose_batched(np.broadcast_to(prior, (len(hs), 7)), X[idx], uv[idx], HYP_ITERS)
        e = _reproj_sq_b(P, X[None], uv[None])
        fin = np.isfinite(e)
        if fin.any():
            rel = np.abs(e[fin] - t2) / t2
            out["margin"] = float(rel.min())
            out["ties"] = int((rel == 0).sum())
            out["margin_untied"] = float(rel[rel > 0].min()) if (rel > 0).any() else np.inf
        inl = e <= t2                                    # NaN compares false
        cnt = inl.sum(1)
        w = int(np.argmax(cnt))                          # first best
        best = int(cnt[w])
        out["winner"] = hs[w]
        out["n_inliers"] = best
        if best < 4:
            return out
        m = inl[w]
        pose = lm_pose_batched(P[w:w + 1], X[None, m], uv[None, m], REFINE_ITERS)[0]
    out.update(success=True, pose=pose, mask=m.astype(np.uint8))
    return out


# ---- what compute_relative_pose does with the PnP result (:396-407) -------------------------------------------------
def delta_pose(a, b, yaw_only):
    """Swarm::Pose::DeltaPose(a, b, use_yaw_only): 6-DoF a^-1 b, or the 4-DoF form of swarm_localization_factors.hpp:139-149"""
    if not yaw_only:
        return pr.pose_mul(pr.pose_inv(a), b)
    ya, yb = quat2eulers(a[3:])[2], quat2eulers(b[3:])[2]
    d = b[:3] - a[:3]
    c, s = np.cos(ya), np.sin(ya)
    pos = np.array([c * d[0] + s * d[1], -s * d[0] + c * d[1], d[2]])
    dy = wrap(yb - ya)
    return np.concatenate([pos, quat_from_rotvec(np.array([0.0, 0.0, dy]))])


def rp_error(p_drone_old_in_new, drone_pose_old, drone_pose_now):
    """RPerror (loop_detector.cpp:338-351)"""
    dp6 = delta_pose(p_drone_old_in_new, drone_pose_now, False)
    predict = pr.pose_mul(drone_pose_old, dp6)
    att_old = predict[3:] / np.linalg.norm(predict[3:])
    att_new = drone_pose_now[3:] / np.linalg.norm(drone_pose_now[3:])
    dyaw = quat2eulers(att_new)[2] - quat2eulers(att_old)[2]
    att_old = pr.q_mul(quat_from_rotvec(np.array([0.0, 0.0, dyaw])), att_old)
    return float(np.linalg.norm(quat2eulers(att_old) - quat2eulers(att_new)))


def loop_from_pnp(res, prm):
    """-> dict(verified, dp (x, y, z, yaw), rperr, odometry_consistent, md): loop_detector.cpp:396-407 + :294-315.
    prm: extrinsic, drone_pose_now, drone_pose_old (poses (t,q)), is_4dof, min_loop_num, rperr_thres, accept_loop_yaw_rad,
    max_loop_dis; for same-drone loops also odom_rel (pose), cov (6x6 = odometry + edge covariance),
    odometry_consistency_threshold."""
    out = dict(verified=False, dp=np.zeros(4), rperr=0.0, odometry_consistent=True, md=0.0)
    if not res["success"]:
        return out
    pose = res["pose"]
    p_cam_old_in_new = pr.pose_inv(pose)                               # PnPRestoCamPose: the camera pose is (R, t)^-1
    p_drone_old_in_new = pr.pose_mul(p_cam_old_in_new, pr.pose_inv(prm["extrinsic"]))
    dp = delta_pose(p_drone_old_in_new, prm["drone_pose_now"], bool(prm["is_4dof"]))
    yaw = quat2eulers(dp[3:])[2]
    out["dp"] = np.array([dp[0], dp[1], dp[2], yaw])
    out["rperr"] = rp_error(p_drone_old_in_new, prm["drone_pose_old"], prm["drone_pose_now"])
    out["verified"] = verify(out["rperr"], res["n_inliers"], yaw, loop_distance(dp), prm)
    if prm.get("same_drone"):                                          # :294-315
        d = delta_pose(dp if prm["is_4dof"] else dp, prm["odom_rel"], False)
        out["md"] = pr.cholesky_smd(pr.log_map(d), np.asarray(prm["cov"], np.float64))
        out["odometry_consistent"] = odometry_consistent(out["md"], prm)
    return out


def loop_distance(dp):
    """|DP_old_to_new.pos()|, summed and rounded in this order (the kernel's order too), so that the distance check is
    reproducible from a returned (x, y, z)"""
    return float(np.sqrt((dp[0] * dp[0] + dp[1] * dp[1]) + dp[2] * dp[2]))


def verify(rperr, n_inliers, yaw, dist, prm):
    """pnp_result_verify (:317-336): fails when rperr > RPERR_THRES (:323-326), too few inliers, |yaw| too large or the
    loop too long (:328-332)"""
    return bool(rperr <= prm["rperr_thres"] and n_inliers >= prm["min_loop_num"] and abs(yaw) < prm["accept_loop_yaw_rad"]
                and dist < prm["max_loop_dis"])


def odometry_consistent(md, prm):
    """check_loop_odometry_consistency (:294-315): inconsistent when the squared Mahalanobis distance exceeds the threshold
    (an infinite one, from a covariance that is not positive definite, always does)"""
    return bool(not md > prm["odometry_consistency_threshold"])
