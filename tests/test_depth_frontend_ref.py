"""CPU: the depth-image generator (synth.depth_image) and the PINHOLE_DEPTH keyframe oracle (depth_frontend_ref)."""
import numpy as np

from omniswarm_b200 import synth
from oracle import pcm_ref as pr

import depth_frontend_ref as dfr

W0, H0 = 96, 64
K = np.array([80.0, 80.0, 48.0, 32.0])


def test_depth_image_is_seeded_and_has_every_case():
    a, b, c = synth.depth_image(3, H0, W0), synth.depth_image(3, H0, W0), synth.depth_image(4, H0, W0)
    assert a.dtype == np.uint16 and a.shape == (H0, W0)
    assert np.array_equal(a, b) and not np.array_equal(a, c)
    m = a / 1000.0
    assert (a == 0).any()                                   # holes
    assert (m >= 10.0).any() and ((m > 0) & (m <= 0.3)).any()   # beyond far, below near
    assert ((m > 0.3) & (m < 10.0)).mean() > 0.4            # mostly valid
    full = synth.depth_image(0)
    assert full.shape == (480, 640)


def _keyframe(seed, accept_min_3d_pts=3, nd=2):
    comp, mean = synth.pca_matrices(0)
    imgs = np.stack([synth.image(seed * 10 + d, H0, W0) for d in range(nd)])
    deps = np.stack([synth.depth_image(seed * 10 + d, H0, W0) for d in range(nd)])
    pose_drone = np.concatenate([[0.5, -1.0, 0.2], synth._quat_from_rotvec(np.array([0.0, 0.0, 0.7]))])
    ext = np.array([np.concatenate([[0.1 * d, 0.0, 0.05], synth._quat_from_rotvec(np.array([0.0, 0.0, d * np.pi / 2]))
                                    ]) for d in range(nd)])
    ref = dfr.depth_keyframe(imgs, deps, synth.superpoint_weights(0), synth.netvlad_weights(0), 0.015, 200, comp, mean, K,
                             pose_drone, ext, 0.3, 10.0, accept_min_3d_pts)
    return imgs, deps, pose_drone, ext, ref


def test_depth_keyframe_lifts_through_pose_cam():
    """every flagged landmark, taken back into its camera, sits on the ray of its keypoint at the looked-up depth; the
    unflagged ones looked up a hole or a depth outside (near, far)"""
    imgs, deps, pose_drone, ext, ref = _keyframe(1)
    n_flag = n_unflag = 0
    for d, r in enumerate(ref):
        n = len(r["kpts"])
        assert n > 3 and r["desc"].shape == (n, 64) and r["g"].shape == (4096,)
        pc = pr.pose_mul(pose_drone, ext[d])
        for i in range(n):
            x, y = r["kpts"][i]
            dep = deps[d][int(round(y)), int(round(x))] / 1000.0
            if r["flag"][i]:
                p = pr.q_rot(pr.q_conj(pc[3:]), r["l3d"][i].astype(np.float64) - pc[:3])
                assert abs(p[2] - dep) < 1e-5
                assert abs(p[0] - (x - K[2]) / K[0] * dep) < 1e-5 and abs(p[1] - (y - K[3]) / K[1] * dep) < 1e-5
                n_flag += 1
            else:
                assert not (0.3 < dep < 10.0) and not r["l3d"][i].any()
                n_unflag += 1
    assert n_flag > 0 and n_unflag > 0


def test_depth_keyframe_gate_flags_nothing_on_sparse_images():
    _, _, _, _, ref = _keyframe(1, accept_min_3d_pts=200)
    for r in ref:
        assert not r["flag"].any() and not r["l3d"].any()
