"""PnP-RANSAC and the loop acceptance checks (pnp_ransac_kernel, through osb_pnp_ransac and osb_pnp_ransac_dev) on every
launch shape and at their numerical edges, against the float64 reference oracle/pnp_ref.pnp_ransac_batched.

Masks, inlier counts, winners and flags are compared exactly.  That is only meaningful where rounding cannot move a point
across the threshold: the kernel fuses multiply-adds and multiplies by 1/z where the reference divides, so each error
differs by a few ulps.  Every case therefore has a reference margin (min over hypotheses and points of |e - t^2| / t^2) of
at least MARGIN, and its generator redraws until it has.  The one exception is built from exactly representable values,
so that both sides compute errors exactly ON the threshold (test_scoring_threshold_is_inclusive)."""
import ctypes as C

import numpy as np
import pytest
import torch

from omniswarm_b200 import lib as _l
from oracle import pnp_ref as pn, pcm_ref as pr

pytestmark = pytest.mark.gpu

MAXN = 1024                      # PNP_MAXN
THREADS = 256                    # PNP_THREADS: one hypothesis per thread per pass
MARGIN = 1e-9
IDENT = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
# camera-in-body extrinsic: camera z = body x, camera x = -body y, camera y = -body z (synth.pnp_case's)
EXT = np.array([0.05, 0.0, 0.03, 0.5, -0.5, 0.5, -0.5])
PASS = dict(rperr_thres=10.0, min_loop_num=4, accept_loop_yaw_rad=4.0, max_loop_dis=1e3,
            odometry_consistency_threshold=1e30)


# ---- geometry ---------------------------------------------------------------------------------------------------------
def quat_euler(roll, pitch, yaw):
    """ZYX: the quaternion whose pn.quat2eulers is (roll, pitch, yaw)"""
    q = pn.quat_from_rotvec(np.array([0.0, 0.0, yaw]))
    q = pr.q_mul(q, pn.quat_from_rotvec(np.array([0.0, pitch, 0.0])))
    return pr.q_mul(q, pn.quat_from_rotvec(np.array([roll, 0.0, 0.0])))


def pose(t, q):
    return np.concatenate([np.asarray(t, np.float64), q])


def scene(rng, n, out=0.25, noise=0.002, rp=np.radians(60.0), prior_error=0.15, yaw_now=None, yaw_rel=None):
    """n landmarks in the NEW drone's frame seen by the OLD camera (normalised coordinates).  The new drone and the old
    one relative to it have any yaw and roll / pitch up to rp; the orientations whose yaw the checks read stay 15 degrees
    or more from gimbal lock, where yaw is ill-posed."""
    while True:
        eul = lambda y: quat_euler(rng.uniform(-rp, rp), rng.uniform(-rp, rp), rng.uniform(-np.pi, np.pi) if y is None else y)
        now = pose(rng.uniform(-5, 5, 3), eul(yaw_now))
        rel = pose(rng.uniform(-1.5, 1.5, 3), eul(yaw_rel))                 # the old drone in the new one's body frame
        old_in_wn = pr.pose_mul(now, rel)
        if max(abs(pn.quat2eulers(q[3:])[1]) for q in (now, old_in_wn, pr.pose_inv(rel))) < np.radians(75.0):
            break
    old = pr.pose_mul(pose(rng.uniform(-5, 5, 3), quat_euler(0.0, 0.0, rng.uniform(-np.pi, np.pi))), old_in_wn)
    cam = pr.pose_mul(old_in_wn, EXT)
    truth = pr.pose_inv(cam)
    Pc = np.stack([rng.uniform(-2.5, 2.5, n), rng.uniform(-1.5, 1.5, n), rng.uniform(2.0, 9.0, n)], 1)
    X = np.array([pr.q_rot(cam[3:], p) + cam[:3] for p in Pc]).reshape(n, 3)
    uv = Pc[:, :2] / Pc[:, 2:3] + rng.normal(0, noise, (n, 2))
    bad = rng.uniform(size=n) < out
    uv[bad] = rng.uniform(-1.2, 1.2, (int(bad.sum()), 2))
    prior = pr.pose_mul(pose(rng.normal(0, prior_error, 3), pn.quat_from_rotvec(rng.normal(0, prior_error * 0.5, 3))), truth)
    return dict(X=X.astype(np.float32), uv=uv.astype(np.float32), prior=prior, extrinsic=EXT, drone_pose_now=now,
                drone_pose_old=old)


def degenerate(c, rng):
    """duplicated correspondences, a collinear run and a coplanar run of landmarks among the generic ones"""
    n = len(c["X"])
    k = max(n // 5, 1)
    c["X"][k:2 * k] = c["X"][:k]; c["uv"][k:2 * k] = c["uv"][:k]
    s = np.linspace(0.0, 1.0, k, dtype=np.float32)[:, None]
    c["X"][2 * k:3 * k] = c["X"][0] + s * (c["X"][-1] - c["X"][0])
    c["X"][3 * k:4 * k, 2] = c["X"][0, 2]
    return c


def on_camera_plane(rng, n):
    """the prior is the identity, so landmarks with z = 0 sit exactly on its camera plane: inf / NaN errors, and a sample
    holding one keeps its model at the prior (its normal equations are not finite); some landmarks lie behind it"""
    c = scene(rng, n)
    truth = pose(rng.normal(0, 0.02, 3), pn.quat_from_rotvec(rng.normal(0, 0.01, 3)))
    Pc = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(2.0, 8.0, n)], 1)
    inv = pr.pose_inv(truth)
    X = np.array([pr.q_rot(inv[3:], p) + inv[:3] for p in Pc]).reshape(n, 3).astype(np.float32)
    uv = (Pc[:, :2] / Pc[:, 2:3] + rng.normal(0, 0.002, (n, 2))).astype(np.float32)
    k = max(n // 10, 1)
    X[:k, 2] = 0.0
    X[k:k + 2, :] = 0.0                                              # 0 / 0
    X[k + 2:2 * k + 2] *= -1.0
    c.update(X=X, uv=uv, prior=IDENT.copy())
    return c


# ---- cases and the reference ---------------------------------------------------------------------------------------
def f32(x):
    return float(np.float32(x))


def reference(c):
    """the reference's PnP (thresh as the kernel reads it, a float) and checks, cached in the case"""
    if "ref" not in c:
        c["ref"] = pn.pnp_ransac_batched(c["X"], c["uv"], c["prior"], c["iterations"], f32(c["thresh"]), c["seed"])
    return c["ref"]


def checks(c):
    return pn.loop_from_pnp(reference(c), c)


def p_drone_old_in_new(ref):
    return pr.pose_mul(pr.pose_inv(ref["pose"]), pr.pose_inv(EXT))


def new_case(rng, kind, n, iterations, is_4dof=None, same_drone=None, min_winner=None, out=None):
    """one candidate of the given kind; redrawn until the reference keeps every inlier decision MARGIN from the threshold
    (and, with min_winner, until a hypothesis at or past min_winner wins)"""
    for _ in range(50):
        c = dict(iterations=iterations, thresh=float(rng.choice([0.01, 0.03, 0.05])), seed=int(rng.integers(0, 2 ** 32)),
                 is_4dof=int(rng.integers(0, 2)) if is_4dof is None else is_4dof,
                 same_drone=int(rng.integers(0, 2)) if same_drone is None else same_drone)
        if kind == "generic":
            c.update(scene(rng, n, out=rng.uniform(0.0, 0.6) if out is None else out))
        elif kind == "exact":                                        # noise 0: every hypothesis fits every point
            c.update(scene(rng, n, out=0.0, noise=0.0, prior_error=0.05))
        elif kind == "yaw_pi":
            c.update(scene(rng, n, out=0.2, noise=0.0005), is_4dof=1)
        elif kind == "degenerate":
            c.update(degenerate(scene(rng, n, out=0.2), rng))
        elif kind == "camera_plane":
            c.update(on_camera_plane(rng, n))
        elif kind == "outliers":                                     # nothing fits: fewer than 4 inliers everywhere
            c.update(scene(rng, n, out=1.0), thresh=1e-4)
        else:
            raise ValueError(kind)
        r = reference(c)
        if r["margin"] < MARGIN or (min_winner is not None and r["winner"] < min_winner):
            continue
        if kind == "exact" and r["success"] and (r["winner"] != 0 or r["n_inliers"] != n):
            continue
        if kind == "yaw_pi":
            near_pi(c, rng)
        thresholds(c, rng)
        return c
    raise AssertionError(f"no {kind} case with n={n} met the margin")


def near_pi(c, rng):
    """set the new drone's yaw so that it minus the yaw of the old drone's pose in the new frame is within 1e-6 of +-pi,
    on either side and either end (drone_pose_now enters the checks only, not the PnP)"""
    ea = pn.quat2eulers(p_drone_old_in_new(c["ref"])[3:])[2]
    off = float(rng.choice([-1e-6, -1e-7, -1e-12, 0.0, 1e-12, 1e-7, 1e-6]))
    eb = ea + (np.pi + off if ea < 0 else -np.pi - off)
    r, p, _ = pn.quat2eulers(c["drone_pose_now"][3:])
    c["drone_pose_now"] = pose(c["drone_pose_now"][:3], quat_euler(r, p, eb))


def thresholds(c, rng):
    """each check's threshold a random factor (at least ~10 % away) from the reference's value, so either verdict occurs
    and rounding cannot decide it; half of the cases pass every check.  Same-drone loops get an odometry pose near DP."""
    r = c["ref"]
    c.update(PASS)
    c["odom_rel"], c["cov"] = IDENT.copy(), np.eye(6)
    if not r["success"]:
        return
    dp = pn.delta_pose(p_drone_old_in_new(r), c["drone_pose_now"], bool(c["is_4dof"]))
    if c["same_drone"]:
        c["odom_rel"] = pr.pose_mul(dp, pose(rng.normal(0, 0.05, 3), pn.quat_from_rotvec(rng.normal(0, 0.02, 3))))
        M = rng.normal(0, 0.1, (6, 6))
        c["cov"] = M @ M.T + np.diag(rng.uniform(0.001, 0.01, 6))
    v = checks(c)
    f = lambda: float(np.exp(rng.choice([-1.0, 1.0]) * rng.uniform(0.1, 1.0)))
    if rng.uniform() < 0.5:
        c.update(rperr_thres=v["rperr"] * f(), min_loop_num=max(r["n_inliers"] + int(rng.integers(-8, 3)), 0),
                 accept_loop_yaw_rad=abs(v["dp"][3]) * f(), max_loop_dis=pn.loop_distance(v["dp"]) * f())
    if c["same_drone"] and np.isfinite(v["md"]) and rng.uniform() < 0.7:
        c["odometry_consistency_threshold"] = v["md"] * f()


# ---- launches ----------------------------------------------------------------------------------------------------------
def params(cases):
    prm = (_l.PnpParams * len(cases))()
    for p, c in zip(prm, cases):
        p.iterations, p.reproj_thresh, p.seed = int(c["iterations"]), float(c["thresh"]), int(c["seed"])
        p.is_4dof, p.min_loop_num, p.same_drone = int(c["is_4dof"]), int(c["min_loop_num"]), int(c["same_drone"])
        p.rperr_thres, p.accept_loop_yaw_rad = float(c["rperr_thres"]), float(c["accept_loop_yaw_rad"])
        p.max_loop_dis, p.odometry_consistency_threshold = float(c["max_loop_dis"]), float(c["odometry_consistency_threshold"])
        for name in ("prior", "extrinsic", "drone_pose_now", "drone_pose_old", "odom_rel"):
            getattr(p, name)[:] = [float(x) for x in c[name]]
        p.odom_edge_cov[:] = [float(x) for x in np.asarray(c["cov"], np.float64).reshape(-1)]
    return prm


def inputs(cases, max_n):
    """[n_cand][max_n] point arrays whose rows past each candidate's n are NaN"""
    nc = len(cases)
    p3 = np.full((nc, max_n, 3), np.nan, np.float32)
    p2 = np.full((nc, max_n, 2), np.nan, np.float32)
    n = np.array([len(c["X"]) for c in cases], np.int32)
    for i, c in enumerate(cases):
        p3[i, :n[i]] = c["X"]; p2[i, :n[i]] = c["uv"]
    return p3, p2, n


def launch(cases, max_n=MAXN):
    """osb_pnp_ransac -> (mask [n_cand][max_n], results)"""
    p3, p2, n = inputs(cases, max_n)
    mask = np.full((len(cases), max_n), 0xAB, np.uint8)
    res = (_l.PnpResult * len(cases))()
    _l.check(_l.load().osb_pnp_ransac(_l.ptr(p3), _l.ptr(p2), _l.ptr(n), len(cases), max_n, params(cases), _l.ptr(mask), res))
    return mask, res


def result_bytes(r):
    """an osb_pnp_result's bytes but for the unused `reserved` field"""
    r = _l.PnpResult.from_buffer_copy(bytes(r))
    r.reserved = 0
    return bytes(r)


def wrap(a):
    return (a + np.pi) % (2.0 * np.pi) - np.pi


def check(c, mask_row, r, margin="margin"):
    """one candidate's kernel output against the reference: decisions exactly, values within 1e-8 (yaw modulo 2 pi)"""
    ref = reference(c)
    n = len(c["X"])
    assert ref[margin] >= MARGIN, "test data has a point on the threshold"
    assert (bool(r.pnp_success), r.n_inliers, r.winner) == (ref["success"], ref["n_inliers"], ref["winner"])
    assert np.array_equal(mask_row[:n], ref["mask"])
    assert not mask_row[n:].any(), "the mask is not zero between n and max_n"
    if not ref["success"]:
        assert (r.verified, r.odometry_consistent, r.rperr, r.md) == (0, 1, 0.0, 0.0)
        assert np.array_equal(np.array(r.pose_cam), np.asarray(c["prior"], np.float64))
        assert not np.array(r.dp_old_to_new).any()
        return
    v = checks(c)
    assert np.all(np.isfinite(r.pose_cam)) and np.abs(np.array(r.pose_cam) - ref["pose"]).max() <= 1e-8
    dp = np.array(r.dp_old_to_new)
    assert np.abs(dp[:3] - v["dp"][:3]).max() <= 1e-8 and abs(wrap(dp[3] - v["dp"][3])) <= 1e-9
    assert abs(r.rperr - v["rperr"]) <= 1e-8
    if np.isinf(v["md"]):
        assert r.md == v["md"]
    else:
        assert abs(r.md - v["md"]) <= 1e-8 * max(1.0, v["md"])
    assert (bool(r.verified), bool(r.odometry_consistent)) == (v["verified"], v["odometry_consistent"])


# ---- tests -------------------------------------------------------------------------------------------------------------
def test_scoring_threshold_is_inclusive(gpu):
    """err <= thresh^2 counts an error exactly on the threshold.  Landmarks at dyadic unit-depth rays and depths 1, 2, 4 and
    an identity prior that is the truth: a sample of exact correspondences fits with zero residual, so its model stays the
    prior exactly, and there the errors of the correspondences shifted by exactly thresh are exactly thresh^2 -- in both
    implementations, whatever they fuse or reciprocate."""
    rng = np.random.default_rng(101)
    th = 2.0 ** -6
    for _ in range(20):
        cells = rng.choice(17 * 13, 100, replace=False)
        a, b = (cells % 17 - 8) / 8.0, (cells // 17 - 6) / 8.0
        z = rng.choice([1.0, 2.0, 4.0], 100)
        X = np.stack([a * z, b * z, z], 1).astype(np.float32)
        uv = np.stack([a, b], 1)
        uv[60:80] += th * np.array([[1, 0], [-1, 0], [0, 1], [0, -1]])[np.arange(20) % 4]
        uv[80:] = rng.uniform(-1.2, 1.2, (20, 2))
        uv[80:] += np.sign(uv[80:] - np.stack([a, b], 1)[80:]) * 0.25       # gross outliers
        c = dict(scene(rng, 4), X=X, uv=uv.astype(np.float32), prior=IDENT.copy(), iterations=300, thresh=th,
                 seed=int(rng.integers(0, 2 ** 32)), is_4dof=1, same_drone=0)
        r = reference(c)
        if r["margin_untied"] >= MARGIN:
            break
    assert r["ties"] > 0 and r["margin_untied"] >= MARGIN and r["n_inliers"] == 80 and r["mask"][60:80].all()
    thresholds(c, rng)
    mask, res = launch([c])
    check(c, mask[0], res[0], margin="margin_untied")     # the ties are exact on both sides, all else keeps its margin


def test_exact_data_ties_every_hypothesis_to_the_first(gpu):
    rng = np.random.default_rng(102)
    cases = [new_case(rng, "exact", n, it) for n, it in [(40, 100), (300, 257), (1024, 1000), (5, 50)]]
    mask, res = launch(cases)
    for c, m, r in zip(cases, mask, res):
        check(c, m, r)
        assert r.winner == 0 and r.n_inliers == len(c["X"])


def test_launch_shapes_points_and_hypotheses(gpu):
    """every n at a warp / CTA boundary and every hypothesis count either side of a pass of PNP_THREADS, in one launch of
    max_n = PNP_MAXN whose padding is NaN"""
    rng = np.random.default_rng(103)
    cases = [new_case(rng, "generic", n, 257) for n in (3, 4, 5, 31, 32, 33, 255, 256, 257, 1023, 1024)]
    cases += [new_case(rng, "generic", 300, it, min_winner=THREADS if it >= 1000 else None, out=0.75 if it >= 1000 else None)
              for it in (0, 1, 4, 255, 256, 257, 1000, 4096)]     # a good sample is rare: some winners come after a pass
    mask, res = launch(cases)
    for c, m, r in zip(cases, mask, res):
        check(c, m, r)
    assert max(r.winner for r in res) >= THREADS


def test_dev_entry_on_a_caller_stream(gpu):
    """osb_pnp_ransac_dev on torch buffers and a stream of the caller's: byte for byte what osb_pnp_ransac gives, and the
    mask written over its whole [n_cand][max_n] extent (it starts as 0xAB here)"""
    rng = np.random.default_rng(104)
    cases = [new_case(rng, k, n, it) for k, n, it in [("generic", 0, 100), ("generic", 2, 100), ("generic", 200, 100),
                                                      ("outliers", 120, 100), ("degenerate", 500, 1000),
                                                      ("generic", 1024, 257), ("camera_plane", 100, 100)]]
    mask, res = launch(cases)
    p3, p2, n = inputs(cases, MAXN)
    dev = torch.device("cuda")
    prm = params(cases)
    t3, t2, tn = (torch.from_numpy(a).to(dev) for a in (p3, p2, n))
    tp = torch.frombuffer(bytearray(bytes(prm)), dtype=torch.uint8).to(dev)
    tm = torch.full((len(cases), MAXN), 0xAB, dtype=torch.uint8, device=dev)
    tr = torch.zeros(C.sizeof(_l.PnpResult) * len(cases), dtype=torch.uint8, device=dev)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    ptr = lambda t: C.c_void_p(t.data_ptr())
    _l.check(_l.load().osb_pnp_ransac_dev(ptr(t3), ptr(t2), ptr(tn), len(cases), MAXN, ptr(tp), ptr(tm), ptr(tr),
                                          C.c_void_p(s.cuda_stream)))
    s.synchronize()
    dres = (_l.PnpResult * len(cases)).from_buffer_copy(tr.cpu().numpy().tobytes())
    assert np.array_equal(tm.cpu().numpy(), mask)
    for c, m, a, b in zip(cases, mask, res, dres):
        assert result_bytes(a) == result_bytes(b)
        check(c, m, a)


def test_acceptance_checks_flip_exactly_at_their_thresholds(gpu):
    """each of pnp_result_verify's four comparisons and the odometry check, rerun with its threshold set to the kernel's own
    value and to the doubles either side of it: the verdicts flip where the reference's comparisons put them"""
    rng = np.random.default_rng(105)
    base = [new_case(rng, "generic", 400, 100, is_4dof=k % 2, same_drone=1) for k in range(8)]
    for c in base:
        assert c["ref"]["success"]
        c.update(PASS)
    mask, res = launch(base)
    for c, m, r in zip(base, mask, res):
        check(c, m, r)
        assert r.verified == 1
        dp = np.array(r.dp_old_to_new)
        at = dict(rperr_thres=r.rperr, accept_loop_yaw_rad=abs(dp[3]), max_loop_dis=pn.loop_distance(dp),
                  odometry_consistency_threshold=r.md)
        variants = [dict(min_loop_num=k) for k in (r.n_inliers - 1, r.n_inliers, r.n_inliers + 1)]
        for name, x in at.items():
            assert np.isfinite(x) and x > 0
            variants += [{name: y} for y in (np.nextafter(x, -np.inf), x, np.nextafter(x, np.inf))]
        runs = [dict(c, **v) for v in variants]
        # a covariance that is not positive definite: md = inf, inconsistent whatever the threshold
        cov = np.array(c["cov"]); cov[2, 2] = -cov[2, 2]
        runs.append(dict(c, cov=cov))
        rmask, rres = launch(runs)
        for cr, rr in zip(runs, rres):
            same = _l.PnpResult.from_buffer_copy(bytes(rr))
            same.verified, same.odometry_consistent, same.md = r.verified, r.odometry_consistent, r.md
            assert result_bytes(same) == result_bytes(r)                     # only the verdicts (and md) may change
            d = np.array(rr.dp_old_to_new)
            assert bool(rr.verified) == pn.verify(rr.rperr, rr.n_inliers, d[3], pn.loop_distance(d), cr)
            assert bool(rr.odometry_consistent) == pn.odometry_consistent(rr.md, cr)
        flips = [(bool(x.verified), bool(x.odometry_consistent)) for x in rres]
        assert flips[:3] == [(True, True), (True, True), (False, True)]                  # n_inliers >= MIN_LOOP_NUM
        assert flips[3:6] == [(False, True), (True, True), (True, True)]                 # rperr <= RPERR_THRES
        assert flips[6:9] == [(False, True), (False, True), (True, True)]                # |yaw| < ACCEPT_LOOP_YAW_RAD
        assert flips[9:12] == [(False, True), (False, True), (True, True)]               # dist < MAX_LOOP_DIS
        assert flips[12:15] == [(True, False), (True, True), (True, True)]               # md > threshold: inconsistent
        assert np.isinf(rres[-1].md) and rres[-1].odometry_consistent == 0
        assert pr.cholesky_smd(np.ones(6), cov) == np.inf
        check(runs[-1], rmask[-1], rres[-1])        # the others sit on the kernel's values, not the reference's


def test_yaw_difference_near_pi(gpu):
    """4-DoF DeltaPose wraps yaw(now) - yaw(old in new) into [-pi, pi): put that difference within 1e-6 of +-pi"""
    rng = np.random.default_rng(106)
    cases = [new_case(rng, "yaw_pi", int(n), 100, same_drone=int(i % 2)) for i, n in enumerate(rng.integers(60, 600, 14))]
    mask, res = launch(cases)
    for c, m, r in zip(cases, mask, res):
        check(c, m, r)
        if r.pnp_success:
            assert abs(abs(r.dp_old_to_new[3]) - np.pi) < 1e-5


def test_mixed_launch_of_many_waves(gpu):
    """more than two waves of CTAs on 132 SMs, every kind of candidate mixed: each one's result and mask bytes are those of
    the same candidate launched alone (with max_n = its own n), and the reference's"""
    rng = np.random.default_rng(107)
    kinds = ["generic"] * 6 + ["exact", "yaw_pi", "degenerate", "camera_plane", "outliers"]
    cases = []
    for i in range(320):
        kind = kinds[i % len(kinds)]
        n = int(rng.integers(0, 4)) if i % 29 == 0 else int(np.exp(rng.uniform(np.log(4), np.log(MAXN + 1))))
        if kind in ("camera_plane", "degenerate") and n < 20:
            n = 20
        it = int(rng.choice([0, 1, 4, 100, 100, 100, 255, 256, 257, 1000]))
        cases.append(new_case(rng, kind, n, it))
    mask, res = launch(cases)
    for c, m, r in zip(cases, mask, res):
        n = len(c["X"])
        am, ar = launch([c], max(n, 1))
        assert result_bytes(ar[0]) == result_bytes(r) and np.array_equal(am[0, :n], m[:n])
        check(c, m, r)
    kinds_seen = {(bool(r.pnp_success), bool(r.verified), bool(r.odometry_consistent)) for r in res}
    assert len(kinds_seen) >= 4
