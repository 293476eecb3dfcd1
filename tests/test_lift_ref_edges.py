"""CPU: the edges of oracle/lift_ref that the device lift kernels define -- the ACCEPT_MIN_3D_PTS gate of both lifts
(loop_cam.cpp:267, :385-391: an image with n <= ACCEPT_MIN_3D_PTS keypoints is not lifted) and a stereo match index outside
[0, n_down), which has no partner."""
import numpy as np

from oracle import lift_ref as lr, pcm_ref as pr

K = np.array([80.0, 80.0, 48.0, 32.0])
POSE_UP = np.array([0.0, 0.0, 0.06, 0.5, -0.5, 0.5, -0.5])       # camera z = body x, 12 cm above the down camera
POSE_DOWN = np.array([0.0, 0.0, -0.06, 0.5, -0.5, 0.5, -0.5])


def _pixel(pose, pw):
    pc = pr.q_rot(pr.q_conj(pose[3:]), pw - pose[:3])
    return [K[0] * pc[0] / pc[2] + K[2], K[1] * pc[1] / pc[2] + K[3]]


def _scene(n):
    """n exact stereo pairs of points 2-4 m in front; down keypoint i is the partner of up keypoint i"""
    rng = np.random.default_rng(n)
    pw = [pr.q_rot(POSE_UP[3:], np.array([rng.uniform(-1, 1), rng.uniform(-0.5, 0.5), rng.uniform(2, 4)])) + POSE_UP[:3]
          for _ in range(n)]
    ku = np.array([_pixel(POSE_UP, p) for p in pw], np.float32)
    kd = np.array([_pixel(POSE_DOWN, p) for p in pw], np.float32)
    return ku, kd, np.arange(n, dtype=np.int32)


def test_stereo_lift_gate_and_match_bounds():
    ku, kd, sm = _scene(11)
    # n_up == ACCEPT_MIN_3D_PTS: nothing; one more: every exact pair is lifted
    pts, fu, fd = lr.stereo_lift(ku[:10], kd, sm[:10], K, POSE_UP, POSE_DOWN, 1e-3, accept_min_3d_pts=10)
    assert not fu.any() and not fd.any() and not pts.any()
    pts, fu, fd = lr.stereo_lift(ku, kd, sm, K, POSE_UP, POSE_DOWN, 1e-3, accept_min_3d_pts=10)
    assert fu.all() and fd.all() and np.isfinite(pts).all() and (pts != 0).any(axis=1).all()
    # the default gate (0) lifts everything, as before the gate was stated
    assert np.array_equal(lr.stereo_lift(ku, kd, sm, K, POSE_UP, POSE_DOWN, 1e-3)[1], fu)
    # indices -1, n_down - 1 and n_down: only the one inside [0, n_down) has a partner
    m = sm.copy()
    m[0], m[1], m[2] = -1, len(kd) - 1, len(kd)
    kd2 = kd.copy(); kd2[-1] = kd[1]                                  # keypoint 1's partner moved to slot n_down - 1
    pts, fu, fd = lr.stereo_lift(ku, kd2, m, K, POSE_UP, POSE_DOWN, 1e-3)
    assert fu.tolist()[:3] == [0, 1, 0] and fd[-1] == 1 and not pts[[0, 2]].any()
    assert np.allclose(pts[1], lr.stereo_lift(ku, kd, sm, K, POSE_UP, POSE_DOWN, 1e-3)[0][1])


def test_depth_lift_gate():
    kp = np.array([[10.0, 10.0]] * 4, np.float32)
    depth = np.full((20, 20), 2000, np.uint16)
    pose = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
    assert not lr.depth_lift(kp, depth, K, pose, 0.3, 10.0, accept_min_3d_pts=4)[1].any()
    pts, fl = lr.depth_lift(kp, depth, K, pose, 0.3, 10.0, accept_min_3d_pts=3)
    assert fl.all() and np.allclose(pts[0], [(10 - 48) / 80 * 2.0, (10 - 32) / 80 * 2.0, 2.0])
