"""ORACLE (test infrastructure, NOT product code) -- CPU composition of a PINHOLE_DEPTH keyframe, built only from the
pinned pieces of oracle/: LoopCam::on_flattened_images -> generate_gray_depth_image_descriptor (swarm_loop/src/
loop_cam.cpp:189-196, 231-302, with LOWER_CAM_AS_MAIN = false, swarm_loop.cpp:243) and extractor_img_desc_deepnet (:525-556).

Per direction d:
  * SuperPoint keypoints + descriptors and the NetVLAD descriptor of the gray image (:525-556); the bottom quarter is not
    blanked (:536 blanks only in STEREO_FISHEYE);
  * if landmarks_2d.size() > ACCEPT_MIN_3D_PTS (:267): the depth look-up lift of lift_ref.depth_lift through
    pose_cam = pose_drone * extrinsic[d] (:273-300); otherwise no landmark is flagged;
  * no stereo match.
"""
from __future__ import annotations

import numpy as np

from oracle import frontend_ref as fr, lift_ref as lr, pcm_ref as pr


def depth_keyframe(images, depth_mm, sp_w, nv_w, thres, max_num, pca_comp, pca_mean, K, pose_drone, extrinsics,
                   near=0.3, far=10.0, accept_min_3d_pts=10):
    """images [n_dirs,H,W] u8, depth_mm [n_dirs,H,W] u16, K = (fx, fy, cx, cy), poses 7 doubles (x y z, qw qx qy qz) ->
    list of dicts per direction: kpts [n,2], desc [n,64], g [4096], flag [n] u8, l3d [n,3] f32"""
    out = []
    for d in range(len(images)):
        kpts, desc, _, _ = fr.superpoint_inference(images[d], sp_w, thres, max_num, pca_comp, pca_mean)
        g = fr.netvlad_net(images[d], nv_w)
        n = len(kpts)
        if n > accept_min_3d_pts:
            pose_cam = pr.pose_mul(np.asarray(pose_drone, np.float64), np.asarray(extrinsics[d], np.float64))
            l3d, flag = lr.depth_lift(kpts, depth_mm[d], K, pose_cam, near, far)
        else:
            l3d, flag = np.zeros((n, 3), np.float32), np.zeros(n, np.uint8)
        out.append(dict(kpts=kpts, desc=desc, g=g, flag=flag, l3d=l3d))
    return out
