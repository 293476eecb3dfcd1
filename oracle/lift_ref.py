"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of how the reference lifts keypoints to 3-D landmarks
and sets `landmarks_flag` (SURVEY.md section 8f-3), paths relative to /root/reference/swarm_loop/src:
  * triangulatePoint                           loop_cam.cpp:73-106   (4x4 DLT, smallest right singular vector by SVD, error =
                                                                      |design * [p;1]| / 4)
  * stereo lift in generate_stereo_image_descriptor  :393-432        (liftProjective of both keypoints, normalise, triangulate
                                                                      between pose_up and pose_down, keep iff err <=
                                                                      TRIANGLE_THRES and the point is in front of the up camera;
                                                                      both images' landmark gets the same 3-D point and flag 1)
  * depth lift in generate_gray_depth_image_descriptor   :276-302    (depth image in mm, DEPTH_NEAR_THRES < dep < DEPTH_FAR_THRES,
                                                                      p = pose_cam * (ray * dep))
camodocal's camera model is not part of the hot path: the flattened virtual cameras are distortion-free pinholes, for which
liftProjective(x, y) = ((x - cx) / fx, (y - cy) / fy, 1).  Eigen's JacobiSVD and numpy's LAPACK SVD agree to rounding (the
3-D point is a ratio of singular-vector components, so the sign convention cancels).
"""
from __future__ import annotations

import numpy as np

from . import pcm_ref as pr


def rot(q):
    return np.stack([pr.q_rot(q, e) for e in np.eye(3)], 1)


def triangulate_point(pose0, pose1, p0, p1):
    """loop_cam.cpp:73-106 -> (point_3d [3], err)"""
    R0, R1 = rot(pose0[3:]), rot(pose1[3:])
    P0 = np.concatenate([R0.T, (-R0.T @ pose0[:3])[:, None]], 1)
    P1 = np.concatenate([R1.T, (-R1.T @ pose1[:3])[:, None]], 1)
    D = np.stack([p0[0] * P0[2] - P0[0], p0[1] * P0[2] - P0[1], p1[0] * P1[2] - P1[0], p1[1] * P1[2] - P1[1]])
    v = np.linalg.svd(D)[2][-1]
    p = v[:3] / v[3]
    err = np.linalg.norm(D @ np.append(p, 1.0)) / 4.0
    return p, float(err)


def stereo_lift(kp_up, kp_down, stereo_match, K, pose_up, pose_down, triangle_thres, accept_min_3d_pts=0):
    """-> (pts3d [n_up,3] f32, flag_up [n_up] u8, flag_down [n_down] u8); K = (fx, fy, cx, cy).

    An image with n_up <= accept_min_3d_pts keypoints is not lifted at all (:385-391).  A match index outside
    [0, n_down) means "no stereo partner": the reference's indices come from its own matcher and never leave the range, the
    device kernel skips them, and so does this statement."""
    fx, fy, cx, cy = K
    n_up, n_down = len(kp_up), len(kp_down)
    pts = np.zeros((n_up, 3), np.float32); fu = np.zeros(n_up, np.uint8); fd = np.zeros(n_down, np.uint8)
    if n_up <= accept_min_3d_pts:
        return pts, fu, fd
    Ru = rot(pose_up[3:])
    for i in range(n_up):
        j = int(stereo_match[i])
        if j < 0 or j >= n_down:
            continue
        a = np.array([(kp_up[i][0] - cx) / fx, (kp_up[i][1] - cy) / fy], np.float64)
        b = np.array([(kp_down[j][0] - cx) / fx, (kp_down[j][1] - cy) / fy], np.float64)
        p, err = triangulate_point(pose_up, pose_down, a, b)
        pc = Ru.T @ (p - pose_up[:3])
        if err > triangle_thres or pc[2] < 0 or not np.all(np.isfinite(p)):
            continue
        pts[i] = p; fu[i] = 1; fd[j] = 1
    return pts, fu, fd


def depth_lift(kp, depth_mm, K, pose_cam, near, far, accept_min_3d_pts=0):
    """-> (pts3d [n,3] f32, flag [n] u8); nothing is lifted when n <= accept_min_3d_pts (:267)"""
    fx, fy, cx, cy = K
    H, W = depth_mm.shape
    n = len(kp)
    pts = np.zeros((n, 3), np.float32); fl = np.zeros(n, np.uint8)
    if n <= accept_min_3d_pts:
        return pts, fl
    for i in range(n):
        x, y = float(kp[i][0]), float(kp[i][1])
        if x < 0 or x > W or y < 0 or y > H:                          # :282 (the reference hard-codes 640 x 480)
            continue
        xi, yi = int(round(x)), int(round(y))                          # cv::Mat::at(Point2f -> Point): rounds
        if xi >= W or yi >= H:
            continue                                                   # (the reference would read out of bounds here)
        dep = depth_mm[yi, xi] / 1000.0
        if dep > near and dep < far:
            ray = np.array([(x - cx) / fx, (y - cy) / fy, 1.0]) * dep
            pts[i] = pr.q_rot(pose_cam[3:], ray) + pose_cam[:3]
            fl[i] = 1
    return pts, fl
