"""GPU: stereo keyframes with the lower camera as main (osb_frontend_set_main_camera(OSB_MAIN_CAMERA_DOWN), the reference's
LOWER_CAM_AS_MAIN, loop_cam.cpp:341-523) against oracle/lower_main_ref.py, in the STEREO_FISHEYE (4 directions) and the
STEREO_PINHOLE (1 direction) configurations; the query stages on such records against the oracle pipeline; compute_loop
through the right extrinsics against the ground truth of synth.loop_scene."""
import functools

import numpy as np
import pytest
import torch

from omniswarm_b200 import synth, host, lib
from oracle import frontend_ref as fr, lower_main_ref as lm, pcm_ref as pr
from frontend_harness import H0, W0, RB, RS, EB
import frontend_harness as fh

pytestmark = pytest.mark.gpu

MN = 200
K = np.array([80.0, 80.0, 48.0, 32.0])
POSE_DRONE = np.concatenate([[1.0, 2.0, 0.5], synth._quat_from_rotvec(np.array([0.02, -0.01, 0.4]))])
CONFIG = dict(db_capacity=64, match_index_dist=2, geometric_filter=True)
CONFIGS = {"fisheye": dict(n_dirs=4, zero_bottom_quarter=True), "pinhole": dict(n_dirs=1, zero_bottom_quarter=False)}
arr = np.ctypeslib.as_array


def rig(nd):
    """per direction an up camera and a down camera 12 cm below it that looks the other way (turned by pi about its y axis):
    a triangulated point in front of one of them is behind the other, so the in-front test decides which camera it uses"""
    left, right = [], []
    for d in range(nd):
        yaw = synth._quat_from_rotvec(np.array([0.0, 0.0, d * np.pi / 2]))
        q = pr.q_mul(yaw, np.array([0.5, -0.5, 0.5, -0.5]))
        left.append(np.concatenate([pr.q_rot(yaw, np.array([0.05, 0.0, 0.06])), q]))
        right.append(np.concatenate([pr.q_rot(yaw, np.array([0.05, 0.0, -0.06])), pr.q_mul(q, np.array([0.0, 0.0, 1.0, 0.0]))]))
    return np.array(left), np.array(right)


def make_frontend(cfg, cameras=True, main="down", **kw):
    fe = fh.make_frontend(dict(CONFIG, **CONFIGS[cfg]), **kw)
    if cameras:
        left, right = rig(fe.cfg.n_dirs)
        fe.set_cameras(K, left, right, triangle_thres=10.0)
        fe.set_drone_pose(POSE_DRONE)
    if main != "up":
        fe.set_main_camera(main)
    return fe


def frame(seed, nd, shift=0):
    up = np.stack([synth.image(seed * 10 + d, H0, W0) for d in range(nd)])
    if shift:
        rng = np.random.default_rng(seed)
        up = np.clip(np.roll(up, shift, axis=2).astype(np.int16) + rng.integers(-3, 4, up.shape), 0, 255).astype(np.uint8)
    down = np.stack([np.roll(up[d], 3, axis=0) for d in range(nd)])     # the down camera sees the scene shifted vertically
    return np.ascontiguousarray(up), np.ascontiguousarray(down)


def sp_alone(up, down, blank):
    """the SuperPoint outputs of every image from a stand-alone handle (the same kernels as the front-end's batch)"""
    comp, mean = synth.pca_matrices(0)
    nd = len(up)
    imgs = np.concatenate([up, down]).copy()
    if blank:
        imgs[:, H0 * 3 // 4:] = 0
    sp = host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, W0, H0, 0.015, MN,
                         max_batch=2 * nd)
    out = sp.inference_batch(imgs)
    sp.close()
    return imgs, out


def oracle_records(up, down, cfg, acc, lower=True, cameras=True):
    nd, blank = CONFIGS[cfg]["n_dirs"], CONFIGS[cfg]["zero_bottom_quarter"]
    imgs, alone = sp_alone(up, down, blank)
    nvw = synth.netvlad_weights(0)
    left, right = rig(nd)
    out = []
    for d in range(nd):
        (ku, du), (kd, dd) = alone[d], alone[nd + d]
        cams = dict(K=K, triangle_thres=10.0, pose_up=pr.pose_mul(POSE_DRONE, left[d]),
                    pose_down=pr.pose_mul(POSE_DRONE, right[d])) if cameras else None
        g = fr.netvlad_net(imgs[nd + d] if lower else imgs[d], nvw)
        out.append(lm.direction_record(ku, du, kd, dd, g, g, acc, lower, cams))
    return out


def check_record(rec, ref):
    n_flag = 0
    for d, r in enumerate(ref):
        n = rec.n_kpts[d]
        assert n == len(r["kpts"]) and rec.n_kpts_down[d] == r["n_kpts_down"]
        assert np.array_equal(arr(rec.kpts[d])[:n], r["kpts"]) and np.array_equal(arr(rec.local_desc[d])[:n], r["desc"])
        assert not arr(rec.kpts[d])[n:].any() and not arr(rec.local_desc[d])[n:].any()
        sm = arr(rec.stereo_match[d])
        assert np.array_equal(sm[:n], r["stereo"]) and (sm[n:] == -1).all()
        fl = arr(rec.landmarks_flag[d])
        assert np.array_equal(fl[:n], r["flag"].astype(np.int32)) and not fl[n:].any()
        l3d = arr(rec.landmarks_3d[d])
        assert np.allclose(l3d[:n], r["l3d"], rtol=1e-5, atol=1e-5) and not l3d[n:].any()
        assert not l3d[:n][fl[:n] == 0].any()
        g = arr(rec.global_desc[d])
        if r["g"].any():
            assert np.linalg.norm(g - r["g"]) <= 1e-4 * np.linalg.norm(r["g"]) and abs(np.linalg.norm(g) - 1) < 1e-5
        else:
            assert not g.any()
        n_flag += int(fl.sum())
    return n_flag


@pytest.mark.parametrize("cfg", ["fisheye", "pinhole"])
def test_down_records_match_oracle(gpu, cfg):
    nd = CONFIGS[cfg]["n_dirs"]
    up, down = frame(3, nd)
    fe = make_frontend(cfg)
    rec, _ = fe.process(up, down, msg_id=7)
    ref = oracle_records(up, down, cfg, 3)
    assert check_record(rec, ref) > 0
    up_ref = oracle_records(up, down, cfg, 3, lower=False)
    # the two modes differ: down keypoints, NetVLAD of the down image, and the in-front test keeps other pairs' points
    assert any(not np.array_equal(r["kpts"], u["kpts"]) for r, u in zip(ref, up_ref))
    assert any((arr(rec.landmarks_flag[d])[:rec.n_kpts[d]] != 0).any() for d in range(nd))
    # without cameras: flag = stereo_match >= 0
    fe2 = make_frontend(cfg, cameras=False)
    rec2, _ = fe2.process(up, down, msg_id=7)
    check_record(rec2, oracle_records(up, down, cfg, 3, cameras=False))
    # the early return: accept_min_3d_pts at the up count of direction 0 -- that direction carries the up image and a zero
    # global descriptor, the others (more up keypoints) the down image
    _, alone = sp_alone(up, down, CONFIGS[cfg]["zero_bottom_quarter"])
    acc = len(alone[0][0])
    fe3 = make_frontend(cfg, accept_min_3d_pts=acc)
    rec3, _ = fe3.process(up, down, msg_id=8)
    ref3 = oracle_records(up, down, cfg, acc)
    check_record(rec3, ref3)
    assert not arr(rec3.global_desc[0]).any() and rec3.n_kpts[0] == acc and rec3.n_kpts_down[0] == acc
    if nd > 1:
        assert any(len(alone[d][0]) > acc for d in range(nd)), "no direction above the threshold"
    assert fe3.db_size(False) == sum(1 for d in range(nd) if rec3.n_kpts[d] > 0)   # the zero row still takes its number
    for f in (fe, fe2, fe3):
        f.close()


def test_switch_back_to_up_is_byte_identical(gpu):
    st = fh.stream()
    up, down = frame(4, 4)
    out = torch.zeros(3 * RB, dtype=torch.uint8, device="cuda")
    a, b = make_frontend("fisheye", main="down"), make_frontend("fisheye", main="up")
    a.extract(up.ctypes.data, down.ctypes.data, 5, out.data_ptr(), st)
    a.set_main_camera("up")
    a.extract(up.ctypes.data, down.ctypes.data, 5, out.data_ptr() + RB, st)
    b.extract(up.ctypes.data, down.ctypes.data, 5, out.data_ptr() + 2 * RB, st)
    a.finish(st); b.finish(st)
    raw = out.cpu().numpy().reshape(3, -1)
    assert np.array_equal(raw[1], raw[2]) and not np.array_equal(raw[0], raw[1])
    a.close(); b.close()


def test_process_equals_extract_ingest_query(gpu):
    st = fh.stream()
    frames = [frame(5, 4), frame(6, 4), frame(5, 4, shift=2)]
    a, b = make_frontend("fisheye", match_index_dist=5), make_frontend("fisheye", match_index_dist=5)
    rt = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    qt = torch.zeros(RS, dtype=torch.uint8, device="cuda")
    accepted = 0
    for i, (up, down) in enumerate(frames):
        rec, res = a.process(up, down, msg_id=i)
        b.extract(up.ctypes.data, down.ctypes.data, i, rt.data_ptr(), st)
        b.ingest_own(rt.data_ptr(), st)
        b.query(rt.data_ptr(), qt.data_ptr(), st)
        b.finish(st)
        assert rt.cpu().numpy().tobytes() == bytes(rec) and qt.cpu().numpy().tobytes() == bytes(res)
        accepted += res.accepted
    assert accepted >= 1                                              # the revisit hits its first visit
    a.close(); b.close()


def test_query_and_query_received_read_the_record(gpu):
    """DOWN records through ingest, query and query_received against LoopDetectorDB + bf_crosscheck on the records' own
    global and local descriptors"""
    st = fh.stream()
    fe = make_frontend("fisheye", match_index_dist=1)
    frames = [frame(7, 4), frame(8, 4), frame(7, 4, shift=2)]
    recs_t = torch.zeros(3 * RB, dtype=torch.uint8, device="cuda")
    for i, (up, down) in enumerate(frames):
        fe.extract(up.ctypes.data, down.ctypes.data, 50 + i, recs_t.data_ptr() + i * RB, st)
    fe.finish(st)
    recs = fh.records(recs_t, 3)
    db = fr.LoopDetectorDB(1, inner_product_thres=0.3, match_index_dist=1)
    fe.ingest(recs_t.data_ptr(), 2, -1, st)                         # the two first keyframes, own
    for r in recs[:2]:
        db.add_frame(r.msg_id, 1, [arr(r.global_desc[d]) for d in range(4)], list(r.n_kpts))
    res_t = torch.zeros(2 * RS, dtype=torch.uint8, device="cuda")
    fe.query(recs_t.data_ptr() + 2 * RB, res_t.data_ptr(), st)
    r3 = recs[2]
    foreign = lib.KeyframeRecord.from_buffer_copy(bytes(r3)); foreign.drone_id = 2
    ft = fh.upload([foreign])
    fe.query_received(ft.data_ptr(), 1, -1, res_t.data_ptr() + RS, st)
    fe.finish(st)
    res_own, res_rcv = fh.results(res_t, 2)
    q = arr(r3.global_desc[1])
    for res, drone in ((res_own, 1), (res_rcv, 2)):
        hid, dist = db.query(drone, q, False, False)
        assert res.accepted == 1 and res.hit_id == hid and abs(res.hit_score - dist) < 1e-4
        assert res.hit_msg_id == 50 and res.swapped == 0
        hit = recs[0]
        for j in range(4):
            dn, do = res.dir_new[j], res.dir_old[j]
            if dn < 0:
                continue
            qi, ti, _ = fr.bf_crosscheck(arr(r3.local_desc[dn])[:r3.n_kpts[dn]], arr(hit.local_desc[do])[:hit.n_kpts[do]])
            n = res.n_matches[j]
            assert n == len(qi) and list(res.match_new[j][:n]) == qi.tolist() and list(res.match_old[j][:n]) == ti.tolist()
            # the geometric filter keeps flagged new landmarks only: the DOWN record's flags
            fl = arr(r3.landmarks_flag[dn])
            assert all(fl[res.geo_new[j][k]] for k in range(res.n_geo[j]))
    fe.close()


# ---- compute_loop: the old frame is lifted through the RIGHT extrinsics -------------------------------------------------
SC = synth.LOOP_SCENE                       # its cameras are the right (lower) ones
RIGHT = SC["ext"]
# the upper cameras: 10 cm above, pitched by 0.1 rad about the camera x axis -- a loop edge through them is wrong
LEFT = np.array([np.concatenate([e[:3] + np.array([0.0, 0.0, 0.1]),
                                 pr.q_mul(e[3:], synth._quat_from_rotvec(np.array([0.1, 0.0, 0.0])))]) for e in RIGHT])
PARAMS = dict(odometry_consistency_threshold=10.0, seed=3)
scene_record = functools.partial(synth.loop_record, n_outliers=0)


@pytest.mark.parametrize("hit", ["local", "swapped_remote"])
def test_loop_edge_uses_the_right_extrinsics(gpu, hit):
    st = fh.stream()
    fe = make_frontend("fisheye", cameras=False, main="up", match_index_dist=5)
    fe.set_cameras(SC["K"], LEFT, RIGHT, 0.006)
    fe.set_main_camera("down")
    fe.set_loop_params(**PARAMS)
    if hit == "local":
        old, new = scene_record(1, 100, "old"), scene_record(1, 101, "new", seed=1, g=synth.loop_noisy_g(1))
        ot = fh.upload([old]); fe.ingest_own(ot.data_ptr(), st)
        qrec, hrec = new, old
        cand = dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"], odom_rel=SC["delta_true"], cov=np.eye(6) * 0.01)
        nonkf = False
    else:
        remote = scene_record(2, 200, "new", seed=2, g=synth.loop_noisy_g(2))
        t = fh.upload([remote]); fe.ingest(t.data_ptr(), 1, -1, st)
        qrec, hrec = scene_record(1, 100, "old"), remote
        cand = dict(pose_query=SC["pose_old"], pose_hit=SC["pose_new"])
        nonkf = True
    rt = fh.upload([qrec]); fe.ingest_own(rt.data_ptr(), st)
    res_t = torch.zeros(RS, dtype=torch.uint8, device="cuda")
    fe.query(rt.data_ptr(), res_t.data_ptr(), st, nonkeyframe=nonkf)
    fe.finish(st)
    res = fh.results(res_t, 1)[0]
    assert res.accepted and bool(res.swapped) == (hit != "local")
    out = torch.zeros(EB, dtype=torch.uint8, device="cuda")
    fe.compute_loop(rt.data_ptr(), res_t.data_ptr(), [cand], out.data_ptr(), st)
    fe.finish(st)
    e = lib.LoopEdgeResult.from_buffer_copy(fh.edges(out, 1)[0])
    ref = fh.loop_oracle(res, qrec, hrec, cand, SC["K"], RIGHT, PARAMS)
    assert e.status == ref["status"] == lib.LOOP_ACCEPTED and e.n_corr == ref["n_corr"]
    n = e.n_corr
    assert list(e.corr_idx_new[:n]) == ref["idx_new"].tolist() and list(e.corr_idx_old[:n]) == ref["idx_old"].tolist()
    assert np.array_equal(np.array(e.inlier[:n], np.uint8), ref["pnp"]["mask"])
    assert np.abs(np.array(e.pnp.pose_cam) - ref["pnp"]["pose"]).max() < 1e-8
    assert np.abs(np.array(e.relative_pose) - ref["relative_pose"]).max() < 1e-8
    assert np.abs(np.array(e.relative_pose) - SC["delta_true"]).max() < 1e-5          # the ground truth
    fe.close()


def test_depth_refusals_launches_and_resources(gpu):
    st = fh.stream()
    base = host.live_resources()
    up, down = frame(9, 4)
    rt = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    fe = make_frontend("fisheye", main="up")
    fe.extract(up.ctypes.data, down.ctypes.data, 1, rt.data_ptr(), st)        # warm-up
    fe.finish(st)
    live = host.live_resources()
    counts = {}
    for main in ("up", "down", "up"):
        fe.set_main_camera(main)
        c = host.launch_count()
        fe.extract(up.ctypes.data, down.ctypes.data, 1, rt.data_ptr(), st)
        counts.setdefault(main, set()).add(host.launch_count() - c)
    fe.finish(st)
    assert counts["up"] == counts["down"] and len(counts["up"]) == 1, counts
    assert host.live_resources() == live                                     # switching allocates nothing
    L = fe._lib
    assert L.osb_frontend_set_main_camera(fe._h, 2) == lib.ERR_INVALID
    assert L.osb_frontend_set_main_camera(fe._h, -1) == lib.ERR_INVALID
    assert L.osb_frontend_set_main_camera(None, lib.MAIN_CAMERA_DOWN) == lib.ERR_INVALID
    with pytest.raises(ValueError):
        fe.set_main_camera("left")
    # a DOWN handle refuses the depth camera and the depth extracts
    fe.set_main_camera("down")
    ext = np.tile(np.array([0.0, 0, 0, 1, 0, 0, 0]), (4, 1))
    img = np.zeros((4, H0, W0), np.uint8); dep = np.zeros((4, H0, W0), np.uint16)
    for call in (lambda: fe.set_depth_camera(K, ext), lambda: fe.extract_depth(img, dep, 1, rt.data_ptr(), st),
                 lambda: fe.process_depth(img, dep, 1)):
        with pytest.raises(lib.OsbError) as ei:
            call()
        assert ei.value.status == lib.ERR_INVALID
    fe.close()
    # a depth handle refuses the main camera
    fd = make_frontend("fisheye", cameras=False, main="up")
    fd.set_depth_camera(K, ext)
    for which in (lib.MAIN_CAMERA_DOWN, lib.MAIN_CAMERA_UP):
        assert fd._lib.osb_frontend_set_main_camera(fd._h, which) == lib.ERR_INVALID
    fd.close()
    assert host.live_resources() == base
