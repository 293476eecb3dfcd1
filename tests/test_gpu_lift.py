"""GPU parity of the 3-D lift of keypoints (osb_stereo_lift / osb_depth_lift, and the same inside osb_frontend extract)
against oracle/lift_ref.py (loop_cam.cpp:73-106, 276-302, 393-432)."""
import numpy as np
import pytest

from omniswarm_b200 import synth, host, lib
from oracle import lift_ref as lr, pcm_ref as pr
from frontend_harness import H0, W0
import frontend_harness as fh

pytestmark = pytest.mark.gpu
K = np.array([80.0, 80.0, 48.0, 32.0])            # 96 x 64 flattened pinhole


def rig(nd=4):
    """virtual stereo rig: per direction an up camera and a down camera 12 cm below it, yawed by 90 degrees per direction"""
    left, right = [], []
    for d in range(nd):
        yaw = synth._quat_from_rotvec(np.array([0.0, 0.0, d * np.pi / 2]))
        cam = np.array([0.5, -0.5, 0.5, -0.5])                                   # camera z = body x, x = -body y, y = -body z
        q = pr.q_mul(yaw, cam)
        left.append(np.concatenate([pr.q_rot(yaw, np.array([0.05, 0.0, 0.06])), q]))
        right.append(np.concatenate([pr.q_rot(yaw, np.array([0.05, 0.0, -0.06])), q]))
    return np.array(left), np.array(right)


def synth_stereo(seed, nd=4, mn=64):
    rng = np.random.default_rng(seed)
    left, right = rig(nd)
    pose_drone = np.concatenate([[1.0, 2.0, 0.5], synth._quat_from_rotvec(np.array([0.02, -0.01, 0.4]))])
    pu = np.array([pr.pose_mul(pose_drone, e) for e in left]); pd = np.array([pr.pose_mul(pose_drone, e) for e in right])
    ku = np.zeros((nd, mn, 2), np.float32); kd = np.zeros((nd, mn, 2), np.float32)
    sm = -np.ones((nd, mn), np.int32); nu = np.zeros(nd, np.int32); ndn = np.zeros(nd, np.int32)
    for d in range(nd):
        n = int(rng.integers(20, mn))
        nu[d] = n; ndn[d] = n
        perm = rng.permutation(n)
        for i in range(n):
            pc = np.array([rng.uniform(-1.0, 1.0), rng.uniform(-0.6, 0.6), rng.uniform(1.0, 6.0)])       # in the up camera
            pw = pr.q_rot(pu[d][3:], pc) + pu[d][:3]
            pdn = pr.q_rot(pr.q_conj(pd[d][3:]), pw - pd[d][:3])
            ku[d, i] = np.round([K[0] * pc[0] / pc[2] + K[2], K[1] * pc[1] / pc[2] + K[3]])            # integer pixels
            j = perm[i]
            kd[d, j] = np.round([K[0] * pdn[0] / pdn[2] + K[2], K[1] * pdn[1] / pdn[2] + K[3]])
            r = rng.uniform()
            if r < 0.7:
                sm[d, i] = j                                                       # a true stereo pair
            elif r < 0.85:
                sm[d, i] = perm[(i + 7) % n]                                       # a wrong pair: large triangulation error
    return ku, kd, sm, nu, ndn, pu, pd, pose_drone, left, right


def test_stereo_lift_matches_oracle(gpu):
    ku, kd, sm, nu, ndn, pu, pd, *_ = synth_stereo(0)
    pts, fu, fd = host.stereo_lift(ku, kd, sm, nu, ndn, K, pu, pd, triangle_thres=0.006)
    n_flag = 0
    for d in range(4):
        rp, rfu, rfd = lr.stereo_lift(ku[d, :nu[d]], kd[d, :ndn[d]], sm[d, :nu[d]], K, pu[d], pd[d], 0.006)
        # borderline triangulation errors (within 1e-9 of the threshold) would be the only legitimate disagreement: none here
        assert np.array_equal(fu[d, :nu[d]], rfu) and np.array_equal(fd[d, :ndn[d]], rfd)
        assert np.allclose(pts[d, :nu[d]], rp, rtol=1e-5, atol=1e-5)
        assert not fu[d, nu[d]:].any() and not pts[d, nu[d]:].any()
        n_flag += int(rfu.sum())
    assert 40 < n_flag < sum(nu)                                        # true pairs triangulate, wrong pairs are rejected
    # sparse image: nothing is lifted when landmarks_2d.size() <= ACCEPT_MIN_3D_PTS (loop_cam.cpp:385-391)
    pts2, fu2, fd2 = host.stereo_lift(ku, kd, sm, nu, ndn, K, pu, pd, accept_min_3d_pts=int(nu.max()))
    assert not fu2.any() and not fd2.any() and not pts2.any()


def test_depth_lift_matches_oracle(gpu):
    rng = np.random.default_rng(1)
    H, W, nd, mn = 64, 96, 2, 50
    depth = rng.integers(0, 12000, (nd, H, W)).astype(np.uint16)        # mm; some below DEPTH_NEAR, some beyond DEPTH_FAR
    kp = np.zeros((nd, mn, 2), np.float32); n = np.array([50, 37], np.int32)
    for d in range(nd):
        kp[d, :n[d], 0] = rng.integers(0, W, n[d]); kp[d, :n[d], 1] = rng.integers(0, H, n[d])
    pose = np.array([np.concatenate([[0.3, -0.2, 1.0], synth._quat_from_rotvec(np.array([0.1, 0.2, 0.3 + d]))]) for d in range(nd)])
    pts, fl = host.depth_lift(kp, n, depth, K, pose, near=0.3, far=10.0)
    for d in range(nd):
        rp, rf = lr.depth_lift(kp[d, :n[d]], depth[d], K, pose[d], 0.3, 10.0)
        assert np.array_equal(fl[d, :n[d]], rf) and np.allclose(pts[d, :n[d]], rp, rtol=1e-6, atol=1e-6)
        assert 0 < rf.sum() < n[d]


def test_frontend_record_carries_triangulated_landmarks(gpu):
    """osb_frontend_set_cameras: extract triangulates the cross-check stereo pairs on the device and the record's
    landmarks_flag / landmarks_3d are the reference's (loop_cam.cpp:393-432), not the stereo_match >= 0 superset."""
    spw, comp, mean, _ = synth.frontend_weights()
    fe = fh.make_frontend(db_capacity=64, match_index_dist=5)
    left, right = rig(4)
    pose_drone = np.concatenate([[1.0, 2.0, 0.5], synth._quat_from_rotvec(np.array([0.02, -0.01, 0.4]))])
    up = np.stack([synth.image(300 + d, H0, W0) for d in range(4)])
    down = np.stack([np.roll(up[d], 3, axis=0) for d in range(4)])       # the down camera sees the scene shifted vertically
    rec0, _ = fe.process(up, down, msg_id=1)                              # without cameras: flag = stereo_match >= 0
    for d in range(4):
        smv = np.ctypeslib.as_array(rec0.stereo_match[d])
        assert np.array_equal(np.ctypeslib.as_array(rec0.landmarks_flag[d]) != 0, smv >= 0)
        assert not np.ctypeslib.as_array(rec0.landmarks_3d[d]).any()
    fe.set_cameras(K, left, right, triangle_thres=0.02)
    fe.set_drone_pose(pose_drone)
    rec, _ = fe.process(up, down, msg_id=2)
    # the down keypoints are not part of the record: a stand-alone handle on the same images gives them (same kernels)
    sp = host.SuperPoint(spw, comp, mean, W0, H0, 0.015, 200, max_batch=8)
    imgs = np.concatenate([up, down]).copy(); imgs[:, H0 * 3 // 4:] = 0
    alone = sp.inference_batch(imgs)
    n_flag = 0
    for d in range(4):
        ku, kd = alone[d][0], alone[4 + d][0]
        n = rec.n_kpts[d]
        assert n == len(ku) and np.array_equal(np.ctypeslib.as_array(rec.kpts[d])[:n], ku)
        smv = np.ctypeslib.as_array(rec.stereo_match[d])[:n]
        pu, pd = pr.pose_mul(pose_drone, left[d]), pr.pose_mul(pose_drone, right[d])
        rp, rfu, _ = lr.stereo_lift(ku, kd, smv, K, pu, pd, 0.02)
        fl = np.ctypeslib.as_array(rec.landmarks_flag[d])[:n]
        assert np.array_equal(fl != 0, rfu != 0)
        assert np.allclose(np.ctypeslib.as_array(rec.landmarks_3d[d])[:n], rp, rtol=1e-5, atol=1e-5)
        assert (fl != 0).sum() <= (smv >= 0).sum()
        n_flag += int(rfu.sum())
    assert n_flag > 0
    sp.close(); fe.close()
