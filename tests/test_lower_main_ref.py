"""CPU: oracle/lower_main_ref.py -- a stereo direction with the lower camera as main (LOWER_CAM_AS_MAIN,
loop_cam.cpp:341-523) -- pinned on hand-built cases: the inverse stereo map, points and flags on the down keypoints, the
in-front test on the up camera, the early return of :390 and NetVLAD taken from the down image."""
import numpy as np

from omniswarm_b200 import synth
from oracle import frontend_ref as fr, lift_ref as lr, lower_main_ref as lm

K = (100.0, 100.0, 50.0, 40.0)
POSE_UP = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])


def project(X, pose):
    """pixel of world point X in the distortion-free pinhole K at pose (x y z, qw qx qy qz)"""
    R = lr.rot(pose[3:])
    pc = R.T @ (np.asarray(X, np.float64) - pose[:3])
    return np.array([K[0] * pc[0] / pc[2] + K[2], K[1] * pc[1] / pc[2] + K[3]])


def unit_desc(n, seed):
    d = np.random.default_rng(seed).normal(size=(n, 64)).astype(np.float32)
    return d / np.linalg.norm(d, axis=1, keepdims=True)


def test_inverse_map():
    m = np.array([3, -1, 0, 5, -1])
    inv = lm.inverse_stereo_map(m, 7)
    assert inv.tolist() == [2, -1, -1, 0, -1, 3, -1]
    assert lm.inverse_stereo_map(-np.ones(4, int), 2).tolist() == [-1, -1]
    assert lm.inverse_stereo_map(np.zeros(0, int), 3).tolist() == [-1, -1, -1]


def test_points_and_flags_land_on_the_down_keypoints():
    pose_down = np.array([0.2, 0.05, 0.0, 1.0, 0.0, 0.0, 0.0])
    X = np.array([[0.5, 0.25, 4.0], [-0.75, 0.5, 3.0], [0.25, -0.5, 6.0], [1.0, 1.0, 5.0]])
    ku = np.array([project(x, POSE_UP) for x in X], np.float32)
    order = np.array([2, 0, 3, 1])                                  # down keypoint j shows point order[j]
    kd = np.array([project(X[i], pose_down) for i in order], np.float32)
    m = np.array([1, 3, 0, -1])                                     # up 0 <-> down 1 (point 0), ..., up 3 unmatched
    pts, flag = lm.stereo_lift_down(ku, kd, m, K, POSE_UP, pose_down, 1e-3)
    assert flag.tolist() == [1, 1, 0, 1]                            # down 2 shows point 3, whose up keypoint is unmatched
    for j in (0, 1, 3):
        assert np.abs(pts[j] - X[order[j]]).max() < 1e-5
    assert not pts[2].any()
    up_pts, fu, fd = lr.stereo_lift(ku, kd, m, K, POSE_UP, pose_down, 1e-3)
    assert np.array_equal(fd, flag) and fu.tolist() == [1, 1, 1, 0]
    for i, j in enumerate(m):
        if j >= 0:
            assert np.array_equal(pts[j], up_pts[i])               # the same point, at idx_down instead of idx


def test_in_front_test_is_on_the_up_camera():
    """a point in front of the down camera but behind the up camera is dropped; in front of both, kept"""
    pose_down = np.array([0.3, 0.0, -3.0, 1.0, 0.0, 0.0, 0.0])
    behind_up, front_both = np.array([0.5, 0.25, -1.0]), np.array([0.5, 0.25, 2.0])
    for X, keep in ((behind_up, 0), (front_both, 1)):
        assert (lr.rot(pose_down[3:]).T @ (X - pose_down[:3]))[2] > 0          # in front of the down camera
        # pixels from the normalised coordinates, also for the point behind the up camera
        a = X[:2] / X[2]
        pc = X - pose_down[:3]
        b = pc[:2] / pc[2]
        ku = np.array([[K[0] * a[0] + K[2], K[1] * a[1] + K[3]]], np.float32)
        kd = np.array([[K[0] * b[0] + K[2], K[1] * b[1] + K[3]]], np.float32)
        pts, flag = lm.stereo_lift_down(ku, kd, np.array([0]), K, POSE_UP, pose_down, 1e-3)
        assert flag.tolist() == [keep]
        if keep:
            assert np.abs(pts[0] - X).max() < 1e-5


def test_early_return_gives_a_zero_global_row():
    acc = 5
    g_up, g_down = np.full(4096, 1 / 64, np.float32), np.full(4096, -1 / 64, np.float32)
    kd, dd = np.arange(16, dtype=np.float32).reshape(8, 2), unit_desc(8, 1)
    for n_up in (acc, acc + 1):
        ku = np.arange(2 * n_up, dtype=np.float32).reshape(n_up, 2) + 0.5
        du = dd[:n_up] + 0.01 * unit_desc(n_up, 2)                 # up i matches down i
        r = lm.direction_record(ku, du, kd, dd, g_up, g_down, acc, True)
        assert r["n_kpts_down"] == n_up
        if n_up == acc:                                            # :390 returns the up descriptor
            assert np.array_equal(r["kpts"], ku) and np.array_equal(r["desc"], du)
            assert not r["g"].any() and r["g"].shape == (4096,)
            assert (r["stereo"] == -1).all() and not r["flag"].any() and len(r["stereo"]) == n_up
        else:
            assert np.array_equal(r["kpts"], kd) and np.array_equal(r["desc"], dd)
            assert np.array_equal(r["g"], g_down)
            assert r["stereo"].tolist() == list(range(n_up)) + [-1] * (8 - n_up)
            assert np.array_equal(r["flag"], (r["stereo"] >= 0).astype(np.uint8))
        up = lm.direction_record(ku, du, kd, dd, g_up, g_down, acc, False)
        assert np.array_equal(up["kpts"], ku) and np.array_equal(up["g"], g_up) and up["n_kpts_down"] == 8
        assert up["stereo"].tolist() == (list(range(n_up)) if n_up > acc else [-1] * n_up)


def test_netvlad_is_taken_from_the_down_image():
    H, W = 64, 96
    comp, mean = synth.pca_matrices(0)
    w, nvw = synth.superpoint_weights(0), synth.netvlad_weights(0)
    up = np.stack([synth.image(11, H, W)])
    down = np.stack([synth.image(12, H, W)])
    recs = {lo: lm.stereo_keyframe(up, down, w, nvw, 0.015, 200, comp, mean, 3, lo)[0] for lo in (False, True)}
    blank = lambda a: np.concatenate([a[:H * 3 // 4], np.zeros((H // 4, W), np.uint8)])
    g_up, g_down = fr.netvlad_net(blank(up[0]), nvw), fr.netvlad_net(blank(down[0]), nvw)
    assert np.array_equal(recs[False]["g"], g_up) and np.array_equal(recs[True]["g"], g_down)
    assert np.linalg.norm(g_up - g_down) > 0.1
    kd, _, _, _ = fr.superpoint_inference(blank(down[0]), w, 0.015, 200, comp, mean)
    ku, _, _, _ = fr.superpoint_inference(blank(up[0]), w, 0.015, 200, comp, mean)
    assert len(ku) > 3 and np.array_equal(recs[True]["kpts"], kd) and recs[True]["n_kpts_down"] == len(ku)
    # the two modes describe the same cross-check pairs
    pairs_up = {(i, j) for i, j in enumerate(recs[False]["stereo"]) if j >= 0}
    pairs_down = {(i, j) for j, i in enumerate(recs[True]["stereo"]) if i >= 0}
    assert pairs_up == pairs_down and len(pairs_up) > 0
