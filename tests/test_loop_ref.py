"""CPU: oracle/loop_ref.py -- compute_loop and the frame-level compute_correspond_features -- pinned on hand-built cases:
the 1-3-match quirk of a failed homography pair, the strict and non-strict gates, the concatenation order of wrapped
direction pairs, rotate_pt_norm2d, and a noiseless planar four-direction scene whose loop edge is the true 4-DoF delta."""
import numpy as np

from omniswarm_b200 import synth
from oracle import loop_ref as lr, pcm_ref as pr, pnp_ref as pn

ND = 4


def pairing(main_new, main_old):
    """the direction pairs of compute_correspond_features (loop_detector.cpp:455-465), in dirs_new order"""
    return [(dn % ND, ((main_old - main_new + ND) % ND + dn) % ND) for dn in range(main_new, main_new + ND)]


def scene_case(sc, main_new=1, main_old=1, drop=0):
    """the scene as a hit: every direction pair's filtered list = all its points (minus the last `drop`)"""
    n = len(sc["X"][0]) - drop
    slots = [dict(dir_new=dn, dir_old=do, geo_valid=1, geo_new=np.arange(n), geo_old=np.arange(n))
             for dn, do in pairing(main_new, main_old)]
    new = dict(drone_id=1, msg_id=101, n_kpts=[len(x) for x in sc["X"]], flags=[np.ones(len(x), np.int32) for x in sc["X"]],
               l3d=sc["X"])
    old = dict(drone_id=1, msg_id=100, kpts=sc["kp_old"])
    cand = dict(pose_now=sc["pose_new"], pose_old=sc["pose_old"], odom_rel=sc["pose_new"], cov=np.eye(6) * 0.01)
    return dict(accepted=1, slots=slots), new, old, cand


def test_rotate_pt_norm2d_identity_quarter_turn_and_clamp():
    one = np.array([1.0, 0.0, 0.0, 0.0])
    for pt in [(0.125, -0.375), (-1.5, 2.25), (1e-4, 3.0)]:
        assert lr.rotate_pt_norm2d(pt, one) == (np.float32(pt[0]), np.float32(pt[1]))
    # 90 degrees about the camera y axis: (x, y, z) -> (z, y, -x), so (u, v, 1) -> (1 / -u, v / -u)
    qy = np.array([np.sqrt(0.5), 0.0, np.sqrt(0.5), 0.0])
    x, y = lr.rotate_pt_norm2d((0.5, 0.25), qy)
    assert abs(x + 2.0) < 1e-6 and abs(y + 0.5) < 1e-6
    # |z| < 1e-3 is clamped to +-1e-3 with its sign
    x, y = lr.rotate_pt_norm2d((1e-4, 0.25), qy)
    assert abs(x + 1000.0) < 1e-2 and abs(y + 250.0) < 1e-2
    x, y = lr.rotate_pt_norm2d((-1e-4, 0.25), qy)
    assert abs(x - 1000.0) < 1e-2 and abs(y - 250.0) < 1e-2
    # the lift is fp64 then float: (x - cx) / fx
    assert lr.lift((112.0, 40.0), (64.0, 64.0, 48.0, 32.0)) == (np.float32(1.0), np.float32(0.125))
    assert lr.lift((np.float32(100.3), np.float32(7.7)), (61.0, 59.0, 48.5, 31.5)) == (np.float32((float(np.float32(100.3)) - 48.5) / 61.0),
                                                             np.float32((float(np.float32(7.7)) - 31.5) / 59.0))


def test_failed_pair_appends_its_flagged_matches():
    """geo_valid = 0: the per-image function pushed the flagged matches (fewer than 4) before returning false, and the frame
    level appends them; a failed pair without flagged matches adds nothing.  geo_valid = 1 lists go in as they are."""
    rng = np.random.default_rng(0)
    flags = [np.zeros(50, np.int32) for _ in range(ND)]
    flags[2][[7, 30]] = 1
    l3d = [rng.normal(size=(50, 3)).astype(np.float32) for _ in range(ND)]
    kp = [rng.uniform(0, 90, (50, 2)).astype(np.float32) for _ in range(ND)]
    ext = [np.array([0, 0, 0, 1.0, 0, 0, 0])] * ND
    slots = [dict(dir_new=1, dir_old=1, geo_valid=1, geo_new=[4, 9, 2, 5], geo_old=[0, 3, 8, 1]),
             dict(dir_new=2, dir_old=2, geo_valid=0, match_new=[1, 7, 12, 30, 44], match_old=[5, 6, 7, 8, 9]),
             dict(dir_new=3, dir_old=3, geo_valid=0, match_new=[1, 2, 3], match_old=[4, 5, 6])]
    c = lr.compute_correspond_features(slots, dict(flags=flags, l3d=l3d), dict(kpts=kp), (64.0, 64.0, 48.0, 32.0), ext, 1,
                                       min_match_per_dir=2)
    assert c["dir_new"].tolist() == [1, 1, 1, 1, 2, 2]
    assert c["idx_new"].tolist() == [4, 9, 2, 5, 7, 30] and c["idx_old"].tolist() == [0, 3, 8, 1, 6, 8]
    assert c["dir_old"].tolist() == [1, 1, 1, 1, 2, 2]
    assert c["matched_dir_count"] == 2                         # 4 >= 2 and 2 >= 2 (non-strict); the empty pair not
    assert np.array_equal(c["X"][4], l3d[2][7]) and np.array_equal(c["X"][5], l3d[2][30])
    assert c["uv"][5].tolist() == list(lr.lift(kp[2][8], (64.0, 64.0, 48.0, 32.0)))


def test_wrapped_directions_concatenate_in_dirs_new_order():
    """main_dir_new 3, main_dir_old 1: pairs (3,1) (0,2) (1,3) (2,0) in that order, and each old point rotated by
    q_main_old^-1 q_dir_old"""
    sc = synth.loop_scene()
    hit, new, old, cand = scene_case(sc, 3, 1, drop=70)
    c = lr.compute_correspond_features(hit["slots"], new, old, sc["K"], sc["ext"], 1, 2)
    n = len(sc["X"][0]) - 70
    assert c["dir_new"].tolist() == [3] * n + [0] * n + [1] * n + [2] * n
    assert c["dir_old"].tolist() == [1] * n + [2] * n + [3] * n + [0] * n
    assert c["idx_new"].tolist() == list(range(n)) * 4
    k = 2 * n + 3                                               # pair (1, 3): old direction 3 seen from main direction 1
    dq = pr.q_mul(pr.q_conj(sc["ext"][1][3:]), sc["ext"][3][3:])
    assert c["uv"][k].tolist() == list(lr.rotate_pt_norm2d(lr.lift(sc["kp_old"][3][3], sc["K"]), dq))


def test_planar_scene_gives_the_true_delta():
    """noiseless: every correspondence is exact in float32, PnP keeps them all and DP_old_to_new is the true 4-DoF delta"""
    sc = synth.loop_scene()
    hit, new, old, cand = scene_case(sc)
    out = lr.compute_loop(hit, new, old, sc["K"], sc["ext"], 1, 1, cand, dict(odometry_consistency_threshold=10.0))
    assert out["status"] == lr.ACCEPTED, out["status"]
    assert out["n_corr"] == 4 * 78 and out["matched_dir_count"] == 4
    assert out["pnp"]["n_inliers"] == out["n_corr"]
    assert np.abs(out["relative_pose"] - sc["delta_true"]).max() < 1e-9
    assert np.abs(out["loop"]["dp"][:3] - sc["delta_true"][:3]).max() < 1e-9
    # the 6-DoF form is the same pose here (the old drone is level at the origin)
    out6 = lr.compute_loop(hit, new, old, sc["K"], sc["ext"], 1, 1, cand, dict(is_4dof=0, odometry_consistency_threshold=10.0))
    assert np.abs(out6["relative_pose"] - sc["delta_true"]).max() < 1e-9
    # the prior is (pose_now^-1 pose_old extrinsic)^-1 of the old main camera
    want = pr.pose_inv(pr.pose_mul(pr.pose_mul(pr.pose_inv(sc["pose_new"]), sc["pose_old"]), sc["ext"][1]))
    assert np.array_equal(out["pnp_params"]["prior"], want)


def test_gates_strict_and_non_strict():
    sc = synth.loop_scene()
    hit, new, old, cand = scene_case(sc)
    n = 4 * 78
    run = lambda **p: lr.compute_loop(hit, new, old, sc["K"], sc["ext"], 1, 1, cand,
                                      dict(dict(odometry_consistency_threshold=10.0), **p))
    assert run(min_loop_num=n)["status"] == lr.TOO_FEW_COMMON          # n_corr > MIN_LOOP_NUM is strict (:671)
    assert run(min_loop_num=n - 1)["status"] == lr.ACCEPTED
    # landmark_num (= n here) < MIN_LOOP_NUM is strict (:632): equal passes to the next gate
    assert run(min_loop_num=n + 1)["status"] == lr.FEW_LANDMARKS
    # init mode: n_corr > INIT_MODE_MIN_LOOP_NUM also passes, strictly
    c_init = dict(cand, init_mode=True)
    f = lambda m: lr.compute_loop(hit, new, old, sc["K"], sc["ext"], 1, 1, c_init,
                                  dict(min_loop_num=n, init_mode_min_loop_num=m, odometry_consistency_threshold=10.0))
    assert f(n - 1)["status"] != lr.TOO_FEW_COMMON and f(n)["status"] == lr.TOO_FEW_COMMON
    # MIN_MATCH_PRE_DIR is non-strict per pair, MIN_DIRECTION_LOOP non-strict over pairs (:503, :532)
    assert run(min_match_per_dir=78, min_direction_loop=4)["status"] == lr.ACCEPTED
    assert run(min_match_per_dir=79)["status"] == lr.CORRESPONDENCE_FAILED
    assert run(min_direction_loop=5)["status"] == lr.CORRESPONDENCE_FAILED
    # no hit, no frame
    assert lr.compute_loop(dict(accepted=0), new, old, sc["K"], sc["ext"], 1, 1, cand)["status"] == lr.NO_HIT
    assert lr.compute_loop(dict(accepted=1, has_frame=False), new, old, sc["K"], sc["ext"], 1, 1, cand)["status"] == lr.NO_FRAME
    # the checks after PnP: distance gate, odometry consistency (same drone), PnP without a model
    assert run(max_loop_dis=0.1)["status"] == lr.NOT_VERIFIED
    bad = dict(cand, odom_rel=np.concatenate([sc["pose_new"][:3] + 1.0, sc["pose_new"][3:]]), cov=np.eye(6) * 1e-4)
    assert lr.compute_loop(hit, new, old, sc["K"], sc["ext"], 1, 1, bad)["status"] == lr.ODOMETRY_INCONSISTENT
    rng = np.random.default_rng(1)
    scrambled = dict(new, l3d=[rng.normal(0, 3, x.shape).astype(np.float32) for x in sc["X"]])
    out = lr.compute_loop(hit, scrambled, old, sc["K"], sc["ext"], 1, 1, cand, dict(reproj_thresh=1e-4))
    assert out["status"] == lr.PNP_FAILED and not out["pnp"]["success"]
