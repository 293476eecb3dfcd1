"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of one direction of a stereo keyframe record, with the
reference's LOWER_CAM_AS_MAIN switch (swarm_loop.cpp:243), built only from the pinned pieces of oracle/ (paths relative to
/root/reference/swarm_loop/src):
  * generate_stereo_image_descriptor, loop_cam.cpp:341-523.  ides = extractor_img_desc_deepnet(up, LOWER_CAM_AS_MAIN) and
    ides_down = extractor_img_desc_deepnet(down, !LOWER_CAM_AS_MAIN) (:350-351): NetVLAD runs on the image whose
    superpoint_mode is false (:553-556), the up image by default and the down image with the lower camera as main;
  * the stereo stage runs iff the UP count > ACCEPT_MIN_3D_PTS (:385), otherwise :390 returns ides, the up descriptor;
  * the cross-check match up -> down (:388, frontend_ref.bf_crosscheck) and the triangulation of every pair between pose_up
    and pose_down with the in-front test on the up camera (:393-432, lift_ref.stereo_lift); a kept point goes to
    ides.landmarks_3d[idx] and ides_down.landmarks_3d[idx_down] (:441-444);
  * the direction's descriptor is ides_down with the lower camera as main, ides otherwise (:517-521); its camera_extrinsic is
    the right extrinsic (:372), which is what compute_loop lifts the old frame through (oracle/loop_ref.py's ext_old).
Defined here where the reference is undefined: with the lower camera as main, the early return of :390 hands
add_to_database (loop_detector.cpp:153-166) a descriptor without image_desc.  The record carries the up keypoints and
descriptors, no flags, stereo_match -1 and a ZERO global descriptor, so its row keeps the reference's ntotal numbering and no
positive threshold accepts it.
Record fields (as osb_keyframe_record): kpts, desc, n_kpts_down, g, stereo (stereo_match), flag, l3d.  With the lower camera
as main, n_kpts_down is the up count and stereo[j] the up index matched to down keypoint j.
"""
from __future__ import annotations

import numpy as np

from oracle import frontend_ref as fr, lift_ref as lr, pcm_ref as pr

DEEP_DESC_SIZE = 4096


def inverse_stereo_map(stereo_match, n_down):
    """up -> down map of the cross-check pairs (one-to-one) -> down -> up map, -1 where a down keypoint is unmatched"""
    inv = -np.ones(n_down, np.int64)
    for i, j in enumerate(np.asarray(stereo_match)):
        if j >= 0:
            assert inv[j] < 0, "cross-check pairs are one-to-one"
            inv[j] = i
    return inv


def stereo_lift_down(kp_up, kp_down, stereo_match, K, pose_up, pose_down, triangle_thres):
    """lift_ref.stereo_lift with the point scattered to the down keypoint (:443-444) -> (pts3d [n_down,3] f32, flag [n_down])"""
    pts_up, flag_up, flag_down = lr.stereo_lift(kp_up, kp_down, stereo_match, K, pose_up, pose_down, triangle_thres)
    pts = np.zeros((len(kp_down), 3), np.float32)
    for i, j in enumerate(np.asarray(stereo_match)):
        if j >= 0 and flag_up[i]:
            pts[j] = pts_up[i]
    return pts, flag_down


def direction_record(ku, du, kd, dd, g_up, g_down, accept_min_3d_pts, lower_cam_as_main, cams=None):
    """one direction from the SuperPoint outputs of both images (keypoints [n,2], descriptors [n,64]) and the NetVLAD
    descriptor of each image (only the main one is read; None is allowed for the other).  cams: None, or dict(K, pose_up,
    pose_down, triangle_thres) for the triangulation (pose_* = pose_drone * left / right extrinsic)."""
    n_up, n_down = len(ku), len(kd)
    stereo_stage = n_up > accept_min_3d_pts                                   # :385
    m = -np.ones(n_up, np.int64)
    if stereo_stage:
        qi, ti, _ = fr.bf_crosscheck(du, dd)                                  # :388
        m[qi] = ti
    if not lower_cam_as_main:
        if cams is not None and stereo_stage:
            l3d, flag, _ = lr.stereo_lift(ku, kd, m, cams["K"], cams["pose_up"], cams["pose_down"], cams["triangle_thres"])
        else:
            l3d, flag = np.zeros((n_up, 3), np.float32), (m >= 0).astype(np.uint8)
        return dict(kpts=ku, desc=du, n_kpts_down=n_down, g=np.asarray(g_up, np.float32), stereo=m, flag=flag, l3d=l3d)
    if not stereo_stage:                                                      # :390 returns the up descriptor
        return dict(kpts=ku, desc=du, n_kpts_down=n_up, g=np.zeros(DEEP_DESC_SIZE, np.float32), stereo=m,
                    flag=np.zeros(n_up, np.uint8), l3d=np.zeros((n_up, 3), np.float32))
    inv = inverse_stereo_map(m, n_down)
    if cams is not None:
        l3d, flag = stereo_lift_down(ku, kd, m, cams["K"], cams["pose_up"], cams["pose_down"], cams["triangle_thres"])
    else:
        l3d, flag = np.zeros((n_down, 3), np.float32), (inv >= 0).astype(np.uint8)
    return dict(kpts=kd, desc=dd, n_kpts_down=n_up, g=np.asarray(g_down, np.float32), stereo=inv, flag=flag, l3d=l3d)


def stereo_keyframe(up, down, sp_w, nv_w, thres, max_num, pca_comp, pca_mean, accept_min_3d_pts, lower_cam_as_main,
                    zero_bottom_quarter=True, K=None, pose_drone=None, left_ext=None, right_ext=None, triangle_thres=0.006):
    """up / down [n_dirs,H,W] u8 -> list of direction_record dicts.  The networks run on the blanked images (:535-538);
    NetVLAD only on the main image of each pair.  With K, pose_drone and the extrinsics the pairs are triangulated."""
    out = []
    for d in range(len(up)):
        u, dn = up[d].copy(), down[d].copy()
        if zero_bottom_quarter:
            h = u.shape[0]
            u[h * 3 // 4:] = 0
            dn[h * 3 // 4:] = 0
        ku, du, _, _ = fr.superpoint_inference(u, sp_w, thres, max_num, pca_comp, pca_mean)
        kd, dd, _, _ = fr.superpoint_inference(dn, sp_w, thres, max_num, pca_comp, pca_mean)
        g_up = None if lower_cam_as_main else fr.netvlad_net(u, nv_w)
        g_down = fr.netvlad_net(dn, nv_w) if lower_cam_as_main else None
        cams = None
        if K is not None:
            pd = np.asarray(pose_drone, np.float64)
            cams = dict(K=K, triangle_thres=triangle_thres,
                        pose_up=pr.pose_mul(pd, np.asarray(left_ext[d], np.float64)),
                        pose_down=pr.pose_mul(pd, np.asarray(right_ext[d], np.float64)))
        out.append(direction_record(ku, du, kd, dd, g_up, g_down, accept_min_3d_pts, lower_cam_as_main, cams))
    return out
