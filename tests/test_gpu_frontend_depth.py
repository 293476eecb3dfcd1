"""GPU: depth-camera keyframes (PINHOLE_DEPTH) through the device front-end -- osb_frontend_set_depth_camera,
extract_depth(_dev), process_depth -- against the stereo path's network outputs, osb_depth_lift, and the oracle composed as
LoopCam::generate_gray_depth_image_descriptor (loop_cam.cpp:231-302, 525-556)."""
import ctypes as C

import numpy as np
import pytest

from omniswarm_b200 import synth, host, lib
from oracle import geometry_ref as gr, lift_ref as lr, pcm_ref as pr

import depth_frontend_ref as dfr
from frontend_harness import H0, RB, RS, W0, depth_frame
import frontend_harness as fh

pytestmark = pytest.mark.gpu

K0 = np.array([80.0, 80.0, 48.0, 32.0])
# pose_drone without translation: pose_drone * extrinsic is then the same double on the host and in pcm_ref.pose_mul
POSE_DRONE = np.concatenate([[0.0, 0.0, 0.0], synth._quat_from_rotvec(np.array([0.05, -0.02, 0.8]))])


def extrinsics(nd):
    cam = np.array([0.5, -0.5, 0.5, -0.5])                   # camera z = body x, x = -body y, y = -body z
    return np.array([np.concatenate([pr.q_rot(synth._quat_from_rotvec(np.array([0.0, 0.0, d * np.pi / 2])),
                                              np.array([0.08, 0.0, 0.03])),
                                     pr.q_mul(synth._quat_from_rotvec(np.array([0.0, 0.0, d * np.pi / 2])), cam)])
                     for d in range(nd)])


CONFIG = dict(db_capacity=256, match_index_dist=2, zero_bottom_quarter=False)


def make_frontend(nd=2, W=W0, H=H0, K=K0, depth_camera=True, **kw):
    fe = fh.make_frontend(CONFIG, n_dirs=nd, width=W, height=H, **kw)
    if depth_camera:
        fe.set_depth_camera(K, extrinsics(nd), 0.3, 10.0)
        fe.set_drone_pose(POSE_DRONE)
    return fe


def frame(seed, nd=2, W=W0, H=H0):
    return depth_frame(seed, nd, W, H)


def arr(x):
    return np.ctypeslib.as_array(x)


def test_network_outputs_equal_the_stereo_up_side(gpu):
    """the same gray images as the up images of a stereo extract: keypoints, descriptors and NetVLAD bit-identical"""
    import torch
    fe = make_frontend()
    st = fh.stream()
    imgs, deps = frame(1)
    down = np.ascontiguousarray(np.stack([synth.image(900 + d, H0, W0) for d in range(2)]))
    t_st = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    t_dp = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    up = np.ascontiguousarray(imgs)
    fe.extract(up.ctypes.data, down.ctypes.data, 1, t_st.data_ptr(), st)
    fe.extract_depth(imgs, deps, 2, t_dp.data_ptr(), st)
    fe.finish(st)
    rs, rd = fh.records(t_st, 1)[0], fh.records(t_dp, 1)[0]
    assert (rd.drone_id, rd.msg_id, rd.n_dirs) == (1, 2, 2)
    assert list(rd.n_kpts) == list(rs.n_kpts) and min(rd.n_kpts[:2]) > 3
    for f in ("kpts", "local_desc", "global_desc"):
        assert arr(getattr(rd, f))[:2].tobytes() == arr(getattr(rs, f))[:2].tobytes(), f
    # directions >= n_dirs: only the counts are written (as in a stereo record)
    assert (arr(rd.stereo_match)[:2] == -1).all() and list(rd.n_kpts_down) == [0, 0, 0, 0]
    assert list(rd.n_kpts[2:]) == [0, 0]
    fe.close()


def test_landmarks_equal_depth_lift(gpu):
    """landmarks_3d / landmarks_flag bit-identical to osb_depth_lift on the record's own keypoints, and the oracle's lift"""
    import torch
    fe = make_frontend()
    st = fh.stream()
    imgs, deps = frame(2)
    t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    fe.extract_depth(imgs, deps, 5, t.data_ptr(), st)
    fe.finish(st)
    rec = fh.records(t, 1)[0]
    ext = extrinsics(2)
    pose_cam = np.array([pr.pose_mul(POSE_DRONE, ext[d]) for d in range(2)])
    n = np.array(rec.n_kpts[:2], np.int32)
    pts, fl = host.depth_lift(arr(rec.kpts)[:2], n, deps, K0, pose_cam, 0.3, 10.0, accept_min_3d_pts=3)
    assert arr(rec.landmarks_3d)[:2].tobytes() == pts.tobytes()
    assert np.array_equal(arr(rec.landmarks_flag)[:2], fl.astype(np.int32))
    n_flag = n_unflag = 0
    for d in range(2):
        k = arr(rec.kpts[d])[:n[d]]
        rp, rf = lr.depth_lift(k, deps[d], K0, pose_cam[d], 0.3, 10.0)
        f = arr(rec.landmarks_flag[d])[:n[d]]
        assert np.array_equal(f, rf.astype(np.int32))
        assert np.allclose(arr(rec.landmarks_3d[d])[:n[d]], rp, rtol=1e-6, atol=1e-6)
        n_flag += int(rf.sum()); n_unflag += int(n[d] - rf.sum())
    assert n_flag > 0 and n_unflag > 0
    fe.close()


def test_accept_min_3d_pts_gate(gpu):
    import torch
    fe = make_frontend(accept_min_3d_pts=200)
    st = fh.stream()
    imgs, deps = frame(2)
    t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    fe.extract_depth(imgs, deps, 5, t.data_ptr(), st)
    fe.finish(st)
    rec = fh.records(t, 1)[0]
    assert min(rec.n_kpts[:2]) > 3
    assert not arr(rec.landmarks_flag)[:2].any() and not arr(rec.landmarks_3d)[:2].any()
    fe.close()


def test_record_vs_oracle_640x480(gpu):
    """PINHOLE_DEPTH at full size (the RealSense configuration, n_dirs = 1), at the bars of the stereo record test"""
    W, H = 640, 480
    K = np.array([380.0, 380.0, 320.0, 240.0])
    pose_drone = np.concatenate([[1.0, -2.0, 0.5], synth._quat_from_rotvec(np.array([0.02, 0.01, 1.2]))])
    fe = make_frontend(nd=1, W=W, H=H, K=K, accept_min_3d_pts=10, match_index_dist=5)
    fe.set_drone_pose(pose_drone)
    imgs, deps = frame(7, nd=1, W=W, H=H)
    rec, res = fe.process_depth(imgs, deps, msg_id=4242)
    comp, mean = synth.pca_matrices(0)
    ref = dfr.depth_keyframe(imgs, deps, synth.superpoint_weights(0), synth.netvlad_weights(0), 0.015, 200, comp, mean, K,
                             pose_drone, extrinsics(1), 0.3, 10.0, 10)[0]
    assert (rec.drone_id, rec.msg_id, rec.n_dirs) == (1, 4242, 1)
    n = rec.n_kpts[0]
    k = arr(rec.kpts[0])[:n]
    same = {tuple(x) for x in k.tolist()} & {tuple(x) for x in ref["kpts"].tolist()}
    assert n > 10 and len(same) >= 0.9 * len(ref["kpts"])
    g = arr(rec.global_desc[0])
    assert np.linalg.norm(g - ref["g"]) < 1e-3 and abs(np.linalg.norm(g) - 1) < 1e-5
    assert rec.n_kpts_down[0] == 0 and (arr(rec.stereo_match[0]) == -1).all()
    if np.array_equal(k, ref["kpts"]):
        ld = arr(rec.local_desc[0])[:n]
        assert np.linalg.norm(ld - ref["desc"]) / np.linalg.norm(ref["desc"]) < 1e-3
        assert np.array_equal(arr(rec.landmarks_flag[0])[:n], ref["flag"].astype(np.int32))
        assert np.allclose(arr(rec.landmarks_3d[0])[:n], ref["l3d"], rtol=1e-5, atol=1e-5)
        assert 0 < ref["flag"].sum() < n
    assert fe.db_size(False) == 1 and res.accepted == 0
    fe.close()


def test_loop_on_revisit_with_geometric_filter(gpu):
    """a revisit is accepted and the device geometric filter reads the depth record's flags (loop_detector.cpp:569-598);
    with an all-zero depth image nothing is flagged and the pair is not geometrically valid"""
    fe = make_frontend(nd=1, geometric_filter=True, ransac_seed=3)
    frames = [frame(20 + s, nd=1) for s in range(4)]
    recs = [fe.process_depth(*f, msg_id=i)[0] for i, f in enumerate(frames)]
    rec, res = fe.process_depth(*frames[0], msg_id=99)
    assert res.accepted == 1 and res.hit_id == 0 and res.hit_msg_id == 0 and res.swapped == 0
    assert res.dir_new[0] == 0 and res.dir_old[0] == 0
    n = res.n_matches[0]
    mn, mo = list(res.match_new[0][:n]), list(res.match_old[0][:n])
    assert n == rec.n_kpts[0] == recs[0].n_kpts[0] and mn == list(range(n)) == mo
    flags = arr(rec.landmarks_flag[0]).astype(np.uint8)
    ref = gr.loop_pair_filter(mn, mo, flags, arr(rec.kpts[0]).copy(), arr(recs[0].kpts[0]).copy(), 3.0, seed=3)
    assert ref is not None
    qn, qo = ref
    g = res.n_geo[0]
    assert res.geo_valid[0] == 1 and g == len(qn) == int(flags[:n].sum())
    assert list(res.geo_new[0][:g]) == qn.tolist() and list(res.geo_old[0][:g]) == qo.tolist()
    _, res0 = fe.process_depth(frames[0][0], np.zeros_like(frames[0][1]), msg_id=100)
    assert res0.accepted == 1 and res0.geo_valid[0] == 0 and res0.n_geo[0] == 0
    fe.close()


def test_host_and_device_paths_agree(gpu):
    """process_depth == extract_depth_dev + ingest_own + query + finish, record and loop result bit for bit"""
    import torch
    frames = [frame(30 + s) for s in range(3)] + [frame(30)]
    fa = make_frontend(match_index_dist=1, geometric_filter=True)
    fb = make_frontend(match_index_dist=1, geometric_filter=True)
    st = fh.stream()
    rec_t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    res_t = torch.zeros(RS, dtype=torch.uint8, device="cuda")
    accepted = 0
    for i, (imgs, deps) in enumerate(frames):
        ra, sa = fa.process_depth(imgs, deps, msg_id=i)
        img_d = torch.from_numpy(imgs).cuda()
        dep_d = torch.from_numpy(deps.view(np.int16)).cuda()
        fb.extract_depth(img_d.data_ptr(), dep_d.data_ptr(), i, rec_t.data_ptr(), st, device_images=True)
        fb.ingest_own(rec_t.data_ptr(), st)
        fb.query(rec_t.data_ptr(), res_t.data_ptr(), st)
        fb.finish(st)
        assert bytes(ra) == rec_t.cpu().numpy().tobytes()
        assert bytes(sa) == res_t.cpu().numpy().tobytes()
        accepted += sa.accepted
    assert accepted >= 1
    fa.close(); fb.close()


def test_errors_and_stereo_unchanged(gpu):
    import torch
    L = lib.load()
    st = fh.stream()
    imgs, deps = frame(3)
    t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    fe = make_frontend(depth_camera=False)
    for call in (lambda: fe.extract_depth(imgs, deps, 1, t.data_ptr(), st),
                 lambda: fe.extract_depth(t.data_ptr(), t.data_ptr(), 1, t.data_ptr(), st, device_images=True),
                 lambda: fe.process_depth(imgs, deps, 1)):
        with pytest.raises(lib.OsbError) as e:
            call()
        assert e.value.status == lib.ERR_INVALID and b"set_depth_camera" in L.osb_last_error()
    K = np.ascontiguousarray(K0); ext = np.ascontiguousarray(extrinsics(2))
    for near, far in ((0.5, 0.5), (2.0, 1.0)):
        with pytest.raises(lib.OsbError) as e:
            fe.set_depth_camera(K0, ext, near, far)
        assert e.value.status == lib.ERR_INVALID
    assert L.osb_frontend_set_depth_camera(fe._h, None, lib.ptr(ext), 0.3, 10.0) == lib.ERR_INVALID
    assert L.osb_frontend_set_depth_camera(fe._h, lib.ptr(K), None, 0.3, 10.0) == lib.ERR_INVALID
    fe.set_depth_camera(K0, ext, 0.3, 10.0)
    img_c, dep_c = np.ascontiguousarray(imgs), np.ascontiguousarray(deps)
    assert L.osb_frontend_extract_depth(fe._h, None, lib.ptr(dep_c), 1, C.c_void_p(t.data_ptr()), C.c_void_p(st)) \
        == lib.ERR_INVALID
    assert L.osb_frontend_extract_depth(fe._h, lib.ptr(img_c), None, 1, C.c_void_p(t.data_ptr()), C.c_void_p(st)) \
        == lib.ERR_INVALID
    assert L.osb_frontend_process_depth(fe._h, lib.ptr(img_c), None, 1, None, None) == lib.ERR_INVALID
    fe.close()
    # the stereo step does not depend on whether a depth camera has been set
    up, down = frame(4)[0], frame(5)[0]
    out = []
    for depth_camera in (False, True):
        fe = make_frontend(depth_camera=False, zero_bottom_quarter=True)
        if depth_camera:
            fe.set_depth_camera(K0, ext, 0.3, 10.0)
        rec, res = fe.process(up, down, msg_id=3)
        rec2, res2 = fe.process(up, down, msg_id=4)
        out.append((bytes(rec), bytes(res), bytes(rec2), bytes(res2)))
        fe.close()
    assert out[0] == out[1]
