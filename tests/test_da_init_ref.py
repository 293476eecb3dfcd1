"""tests/da_init_ref.py: the literal LocalizationDAInit and the device-form walk agree on random flights and on hand-built
cases for every quirk the device keeps."""
import numpy as np
import pytest

from omniswarm_b200 import lib as _l
from oracle import pcm_ref as pr
import da_init_ref as da

STEP = 100_000_000                                                 # 0.1 s odometry


def yaw_pose(x, y, z, yaw):
    return np.array([x, y, z, np.cos(yaw / 2), 0.0, 0.0, np.sin(yaw / 2)])


def case(n_drones, anon, seed=0, kf_drones=(), n_samples=40, start=None):
    """a static swarm seen through odometry: drone d sits at world pose T_d, its odometry starts at start[d] and moves
    slowly.  anon = [(detector, true target, anonymous id, sample index)] detections in store order.  -> (trajs, kf,
    dets lib.MEASUREMENT_DTYPE, world) with the keyframe paths of kf_drones true at their odometry stamps"""
    rng = np.random.default_rng(seed)
    world = {d: yaw_pose(*rng.uniform(-8, 8, 2), rng.uniform(0, 2), rng.uniform(-np.pi, np.pi)) for d in range(n_drones)}
    start = start or {}
    trajs = {}
    for d in range(n_drones):
        t = start.get(d, 0) + STEP * np.arange(n_samples, dtype=np.int64)
        p = np.stack([yaw_pose(0.01 * k * np.cos(d), 0.01 * k * np.sin(d), 0.0, 0.002 * k) for k in range(n_samples)])
        trajs[d] = (t, p)

    def wpose(d, k):
        return pr.pose_mul(world[d], trajs[d][1][k])

    kf = {d: (trajs[d][0][::5].copy(), np.stack([wpose(d, k) for k in range(0, n_samples, 5)])) for d in kf_drones}
    dets = np.zeros(len(anon), _l.MEASUREMENT_DTYPE)
    for i, (a, b, aid, k) in enumerate(anon):
        dets[i]["id"] = 10_000 + i
        dets[i]["type"] = _l.MEAS_DET6D if i % 2 else _l.MEAS_DET4D
        dets[i]["id_a"], dets[i]["id_b"] = a, aid
        dets[i]["stamp_a"], dets[i]["stamp_b"] = trajs[a][0][k], trajs[b][0][k]
        dets[i]["relative_pose"] = pr.pose_mul(pr.pose_inv(wpose(a, k)), wpose(b, k))
        dets[i]["cov"] = np.diag([0.04, 0.04, 0.04, 0.01, 0.01, 0.01])
    return trajs, kf, dets, world


def random_case(seed):
    rng = np.random.default_rng(seed)
    n = int(rng.integers(3, 9))
    n_anon = int(rng.integers(2, min(8, n) + 1))
    targets = rng.permutation(np.arange(1, n))[:n_anon - 1].tolist() + [0]
    anon = []
    for j, b in enumerate(targets):
        for _ in range(int(rng.integers(1, 3))):
            a = int(rng.choice([d for d in range(n) if d != b]))
            anon.append((a, b, 1000 + 7 * j, int(rng.integers(0, 40))))
    rng.shuffle(anon)
    return case(n, anon, seed=seed, kf_drones=tuple(range(n)))


def both(*args, **kw):
    lit = da.da_literal(*args, **kw)
    vec = da.da_vec(*args, **kw)
    assert lit == vec
    return lit


@pytest.mark.parametrize("seed", range(12))
def test_forms_agree_on_random_flights(seed):
    trajs, kf, dets, _ = random_case(seed)
    applied, status, guess, ids = both(0, trajs, kf, dets, 3.345)
    assert status == "ok" and applied
    assert all(i < 1000 for i in ids)


def hand(n, anon, kf_drones, **kw):
    """case() with drone 0 left without odometry: drone 0 is tried first at every level and never checked, so with
    odometry it would be every id's first success"""
    trajs, kf, dets, world = case(n, anon, kf_drones=kf_drones, **kw)
    trajs[0] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    return trajs, kf, dets, world


def test_drone0_first_success_when_it_has_odometry():
    trajs, kf, dets, _ = case(4, [(1, 2, 1001, 5), (2, 3, 1002, 7)], kf_drones=(0, 1, 2, 3))
    assert both(0, trajs, kf, dets, 3.345)[:3] == (True, "ok", {1001: 0, 1002: 0})


def test_true_targets_found_and_renamed():
    trajs, kf, dets, _ = hand(5, [(1, 2, 1001, 5), (2, 3, 1002, 7), (3, 4, 1003, 9), (4, 1, 1004, 9)], (1, 2, 3, 4))
    applied, status, guess, ids = both(1, trajs, kf, dets, 3.345)
    assert (applied, status) == (True, "ok")
    assert guess == {1001: 2, 1002: 3, 1003: 4, 1004: 1}
    assert ids == [2, 3, 4, 1]


def test_verify_is_always_zero():
    """a second detection of the id that contradicts the guess: verify() would reject it, but its cost is always 0"""
    trajs, kf, dets, _ = hand(4, [(1, 2, 1001, 5), (3, 2, 1001, 6)], (1, 2, 3))
    dets[1]["relative_pose"][:3] += 50.0                            # detector 3's row; the path uses detector 1's
    dets = dets[::-1].copy()                                        # ... and the last row (the gate's covariance) is 1's
    assert both(1, trajs, kf, dets, 3.345)[:3] == (True, "ok", {1001: 2})


def test_drone0_is_guessed_but_never_estimated():
    """drone 0 needs no pose to be guessed: estimated (self), it succeeds unchecked; not estimated, verify() throws"""
    trajs, kf, dets, _ = case(3, [(1, 2, 1001, 5)], kf_drones=(0, 1, 2))
    assert both(0, trajs, kf, dets, 3.345)[:3] == (True, "ok", {1001: 0})
    trajs, kf, dets, _ = case(3, [(1, 0, 1001, 5)], kf_drones=(1, 2))
    assert both(1, trajs, kf, dets, 3.345)[:2] == (False, "invalid")


def test_last_detection_gives_the_detector_first_gives_the_path():
    """raw_dets / uniden_detector take the LAST detection; estimate_path the smallest detector's FIRST one"""
    trajs, kf, dets, _ = hand(4, [(2, 3, 1001, 5), (1, 3, 1001, 6), (1, 3, 1001, 7), (2, 3, 1001, 8)], (1, 2, 3))
    lit = da.DAInit(1, trajs, kf, dets, 3.345)
    assert lit.try_data_association()[1] == {1001: 3}
    assert lit.uniden_detector[1001] == 2
    assert lit.drone_dets_by_pair[1001][1][0]["ts_a"] == int(dets[1]["stamp_a"])
    assert both(1, trajs, kf, dets, 3.345)[:3] == (True, "ok", {1001: 3})
    spoiled = dets.copy()
    spoiled[2]["relative_pose"][:3] += 40.0                         # detector 1's second row: not read
    assert both(1, trajs, kf, spoiled, 3.345)[:3] == (True, "ok", {1001: 3})
    spoiled = dets.copy()
    spoiled[1]["relative_pose"][:3] += 40.0                         # detector 1's first row: the path fails the gate
    assert both(1, trajs, kf, spoiled, 3.345)[:2] == (False, "ok")


def test_first_success_is_kept():
    """1001's drone 3 has no estimate, so both 2 and 3 pass for it; 2 is estimated and fails the second id ... while 3
    succeeds: the first successful candidate decides"""
    trajs, kf, dets, _ = hand(4, [(1, 3, 1001, 5)], (1,))
    # only 1 is estimated: a guess of c estimates c alone, no leaf covers every drone
    assert both(1, trajs, kf, dets, 3.345)[:2] == (False, "ok")
    trajs, kf, dets, _ = hand(3, [(1, 2, 1001, 5), (1, 2, 1002, 6)], (1,))
    # 1001 -> 2 estimates 2; 1002 -> 2 passes the gate against it: the first success
    assert both(1, trajs, kf, dets, 3.345)[:3] == (True, "ok", {1001: 2, 1002: 2})


def test_next_id_after_a_failed_one():
    """1001's detector (3) has no estimate at first, so the level starts with 1002, whose guess estimates 3; one level
    down 1001 is searched"""
    trajs, kf, dets, _ = hand(4, [(3, 2, 1001, 5), (1, 3, 1002, 6)], (1, 2))
    assert both(1, trajs, kf, dets, 3.345)[:3] == (True, "ok", {1001: 2, 1002: 3})
    trajs, kf, dets, _ = hand(4, [(1, 2, 1001, 5), (1, 3, 1002, 6)], (1, 2, 3))
    dets[0]["relative_pose"][:3] += 40.0                            # 1001 finds no candidate: on to 1002 at level 0
    lit = da.DAInit(1, trajs, kf, dets, 3.345)
    assert lit.try_data_association()[0] is False
    assert lit.nodes > 1
    assert both(1, trajs, kf, dets, 3.345)[:2] == (False, "ok")


def test_leaf_needs_every_drone_estimated():
    trajs, kf, dets, _ = hand(4, [(1, 2, 1001, 5)], (1,))
    assert both(1, trajs, kf, dets, 3.345)[:2] == (False, "ok")     # est {1, c}: drone 2 or 3 is missing
    trajs, kf, dets, _ = hand(4, [(1, 2, 1001, 5)], (1, 3))
    assert both(1, trajs, kf, dets, 3.345)[:3] == (True, "ok", {1001: 2})


def test_throws_become_refusals():
    # a keyframe-path drone without odometry
    trajs, kf, dets, _ = hand(3, [(1, 2, 1001, 5)], (1, 2))
    kf[0] = kf[1]
    assert both(1, trajs, kf, dets, 3.345)[:2] == (False, "invalid")
    # estimate_path of a smallest detector (2) without an estimate; the detector of the LAST row (3) has one
    trajs, kf, dets, _ = hand(4, [(2, 1, 1001, 5), (3, 1, 1001, 6)], (1, 3))
    assert both(1, trajs, kf, dets, 3.345)[:2] == (False, "invalid")
    # verify() reads every detector's estimate: detector 3 of 1001 never gets one
    trajs, kf, dets, _ = hand(4, [(3, 2, 1001, 4), (1, 2, 1001, 5)], (1,))
    assert both(1, trajs, kf, dets, 3.345)[:2] == (False, "invalid")
    # guess.at() of an anonymous row whose detector has no odometry and whose id no searched row has
    trajs, kf, dets, _ = hand(3, [(1, 2, 1001, 5)], (1, 2))
    extra = dets.copy()
    extra["id_a"], extra["id_b"] = 0, 1005
    assert both(1, trajs, kf, np.concatenate([dets, extra]), 3.345)[:2] == (False, "invalid")
    extra["id_b"] = 1001                                            # the id is searched through another row: fine
    assert both(1, trajs, kf, np.concatenate([dets, extra]), 3.345)[:3] == (True, "ok", {1001: 2})


def test_threshold_is_the_float():
    """DA_accept_thres is the float 3.345f compared as a double: a distance between 3.345 and (double)3.345f passes"""
    thr = float(np.float32(3.345))
    assert thr > 3.345
    trajs, kf, dets, _ = hand(3, [(1, 2, 1001, 5), (1, 2, 1002, 6)], (1,))
    dets[1]["relative_pose"][0] += 0.05                             # 1002's path lands 5 cm off 1001's estimate of 2
    lit = da.DAInit(1, trajs, kf, dets, 3.345)
    t0 = max(int(v.stamps[0]) for v in lit.ego.values())
    est = {1: pr.pose_mul(kf[1][1][0], lit.rel(1, int(kf[1][0][0]), t0))}
    lit.drone_dets_by_pair = {1001: {1: [da.det_of(dets[0])]}, 1002: {1: [da.det_of(dets[1])]}}
    est[2] = lit.estimate_path(1001, {1001: 2}, est, t0)
    pose = lit.estimate_path(1002, {1002: 2}, est, t0)
    unit = da.mahalanobis(est[2], pose, np.eye(6))
    d = dets.copy()
    d["cov"] = np.eye(6) * unit / ((3.345 + thr) / 2)                # both rows: the search in either order meets it
    assert 3.345 < da.mahalanobis(est[2], pose, d[1]["cov"]) < thr
    assert both(1, trajs, kf, d, 3.345)[:3] == (True, "ok", {1001: 2, 1002: 2})
    assert both(1, trajs, kf, d, 3.3449)[:2] == (False, "ok")


def test_budget_and_capacity():
    trajs, kf, dets, _ = hand(5, [(1, 2, 1001, 5), (2, 3, 1002, 7), (3, 4, 1003, 9), (4, 1, 1004, 9)], (1, 2, 3, 4))
    lit = da.DAInit(1, trajs, kf, dets, 3.345)
    assert lit.try_data_association()[0]
    n = lit.nodes
    assert both(1, trajs, kf, dets, 3.345, max_nodes=n)[0] is True
    assert both(1, trajs, kf, dets, 3.345, max_nodes=n - 1)[:2] == (False, "capacity")
    anon = [(1, 2, 1000 + j, j % 40) for j in range(33)]
    trajs, kf, dets, _ = hand(3, anon, (1, 2))
    assert both(1, trajs, kf, dets, 3.345)[:2] == (False, "capacity")
    out = both(1, trajs, kf, dets[:32], 3.345)
    assert out[:2] == (True, "ok") and set(out[2].values()) == {2}


def test_no_association_without_anonymous_ids_or_self_odometry():
    trajs, kf, dets, _ = case(3, [(1, 2, 1001, 5)], kf_drones=(0, 1, 2))
    d = dets.copy()
    d["id_b"] = 2
    assert both(0, trajs, kf, d, 3.345) == (False, "ok", {}, [2])
    t = dict(trajs)
    t[0] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    assert both(0, t, {1: kf[1], 2: kf[2]}, dets, 3.345)[:2] == (False, "ok")


def test_gate():
    nodes = np.array([1, 1, 1, 0], bool)
    assert da.gate(nodes, [1, 1, 0, 0], 1)
    assert not da.gate(nodes, [1, 1, 1, 0], 1)
    assert not da.gate(nodes, [1, 1, 0, 0], 0)
    assert not da.gate([1, 0, 0, 0], [0, 0, 0, 0], 3)
