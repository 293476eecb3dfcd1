"""CPU: tests/keyframe_ref.py -- the literal walks and the vectorised forms agree over random swarms, and each quirk of
outlier_rejection_frame and setup_problem_with_sferror has its own case."""
import numpy as np
import pytest

import keyframe_ref as kr

PRM = dict(outlier_threshold=0.3, elevation_threshold=0.5, minimum_distance=0.2, enable_distance=True,
           debug_no_rejection=False, distance_measurement_cov=0.2, self_id=0)


def run(n_drones, n_kf, seed, finish_at=3, **kw):
    """the oracle over a generated flight: per keyframe (nodes, dists, poses after init, flags)"""
    kfs = kr.random_keyframes(n_drones, n_kf, seed, **kw)
    asg = kr.BlockAssigner()
    poses = np.zeros((n_drones * n_kf, 4))
    last, out = None, []
    for k, kf in enumerate(kfs):
        fi = k >= finish_at
        nodes, dists = kr.keyframe_records(kf, asg, 0, fi)
        p1 = kr.init_poses(nodes, poses, kf["stamp"], 0, fi, 7)
        p2 = kr.init_poses_vec(nodes, poses, kf["stamp"], 0, fi, 7)
        assert p1.tobytes() == p2.tobytes()
        poses = p1
        prm = dict(PRM, finish_init=fi)
        f1 = kr.outlier_flags(nodes, dists, poses, last, prm)
        f2 = kr.outlier_flags_vec(nodes, dists, poses, last, prm)
        assert np.array_equal(f1, f2), k
        out.append((kf["stamp"], nodes, dists, f1))
        last = nodes
    return out, poses


@pytest.mark.parametrize("seed", range(4))
def test_literal_and_vectorised_agree(seed):
    kfs, _ = run(6, 12, seed, late=(4,), static=(5,))
    store = {ts: (n, d, f) for ts, n, d, f in kfs}
    window = [(ts, {int(x["drone_id"]): int(x["block"]) for x in n}) for ts, n, _, _ in kfs[-8:]]
    enable = np.random.default_rng(seed).random(256) < 0.7
    r1 = kr.distance_rows(window, store, enable, PRM)
    r2 = kr.distance_rows_vec(window, store, enable, PRM)
    for k in r1:
        assert r1[k].tobytes() == r2[k].tobytes(), k
    assert len(r1["ia"]) > 0


def test_draw_is_the_multistart_hash_keyed_by_stamp():
    v = kr.draw(3, 1_000_000_000, np.arange(5)[:, None], np.arange(3)[None, :])
    assert v.shape == (5, 3) and np.all(v >= -5.0) and np.all(v < 5.0) and len(np.unique(v)) == 15
    assert kr.draw(3, 1_000_000_000, 2, 1) == v[2, 1] and kr.draw(4, 1_000_000_000, 2, 1) != v[2, 1]


def two_nodes(z1=0.0, dis=5.0, vo=(1, 1), n_d=(0, 1), peers=(0,)):
    nodes = np.zeros(2, kr.NODE_DTYPE)
    nodes["drone_id"] = [0, 1]
    nodes["block"] = [0, 1]
    nodes["vo_available"] = vo
    nodes["frame_available"] = nodes["dists_available"] = 1
    nodes["n_distances"] = n_d
    nodes["pose"][:, 3] = 1.0
    nodes["pose"][1, 2] = z1
    dists = np.zeros(len(peers), kr.DIST_DTYPE)
    dists["peer"] = peers
    dists["distance"] = dis
    poses = np.zeros((2, 4))
    poses[1, 2] = z1
    return nodes, dists, poses


def test_asin_nan_is_not_an_outlier():
    nodes, dists, poses = two_nodes(z1=-3.0, dis=1.0, n_d=(0, 1))        # |dz| > d: asin is NaN
    for fi in (False, True):
        prm = dict(PRM, finish_init=fi, minimum_distance=0.0, outlier_threshold=100.0)
        f = kr.outlier_flags(nodes, dists, poses, nodes, prm)
        assert f.tolist() == [0] and kr.outlier_flags_vec(nodes, dists, poses, nodes, prm).tolist() == [0]


def test_early_return_and_absent_node():
    nodes, dists, poses = two_nodes(z1=0.0, dis=0.1, n_d=(1, 1), peers=(1, 0))
    prm = dict(PRM, finish_init=True)
    last = nodes.copy()
    last["vo_available"] = [0, 1]                                        # node 0 without VO last time: return
    assert kr.outlier_flags(nodes, dists, poses, last, prm).tolist() == [-1, -1]
    last["vo_available"] = [1, 0]                                        # node 1: only its flags stay unwritten
    assert kr.outlier_flags(nodes, dists, poses, last, prm).tolist() == [1, -1]
    assert kr.outlier_flags(nodes, dists, poses, last[1:], prm).tolist() == [-1, -1]   # node 0 absent: skipped, then return
    last["drone_id"] = [1, 2]
    last["vo_available"] = [1, 1]
    assert kr.outlier_flags(nodes, dists, poses, last, prm).tolist() == [-1, 1]        # node 0 absent: skipped only
    for l in (last, last[1:]):
        assert np.array_equal(kr.outlier_flags_vec(nodes, dists, poses, l, prm), kr.outlier_flags(nodes, dists, poses, l, prm))


def test_peer_absent_or_without_vo_is_skipped():
    nodes, dists, poses = two_nodes(n_d=(0, 2), peers=(0, 7))
    nodes["vo_available"] = [0, 1]
    f = kr.outlier_flags(nodes, dists, poses, nodes, dict(PRM, finish_init=False))
    assert f.tolist() == [-1, -1]


def at(x, ulps):
    x = np.float64(x)
    for _ in range(abs(ulps)):
        x = np.nextafter(x, np.inf if ulps > 0 else -np.inf)
    return float(x)


@pytest.mark.parametrize("side,want", [(-1, 0), (0, 0), (1, 1)])
def test_outlier_threshold_at_one_ulp(side, want):
    """|d - est| against the float threshold: 5 + 0.3f is exact in fp64, so d - 5 is the threshold itself at side 0"""
    thr = float(np.float32(0.3))
    nodes, dists, poses = two_nodes(dis=at(5.0 + thr, side))
    poses[1, 0] = 5.0
    prm = dict(PRM, finish_init=True, elevation_threshold=10.0)
    assert kr.outlier_flags(nodes, dists, poses, nodes, prm).tolist() == [want]
    assert kr.outlier_flags_vec(nodes, dists, poses, nodes, prm).tolist() == [want]


@pytest.mark.parametrize("side,want", [(-1, 1), (0, 0), (1, 0)])
def test_minimum_distance_at_one_ulp(side, want):
    md = float(np.float32(0.2))
    nodes, dists, poses = two_nodes(dis=at(md, side))
    poses[1, 0] = float(dists["distance"][0])                   # est == d: only d < minimum_distance decides
    prm = dict(PRM, finish_init=True, elevation_threshold=10.0)
    assert kr.outlier_flags(nodes, dists, poses, nodes, prm).tolist() == [want]


@pytest.mark.parametrize("rel,want", [(-1e-9, 0), (1e-9, 1)])
def test_elevation_threshold_edges(rel, want):
    el = float(np.float32(0.5))
    nodes, dists, poses = two_nodes(z1=float(np.sin(el * (1.0 + rel))), dis=1.0)
    for fi in (False, True):
        prm = dict(PRM, finish_init=fi, elevation_threshold=el, outlier_threshold=100.0, minimum_distance=0.0)
        assert kr.outlier_flags(nodes, dists, poses, nodes, prm).tolist() == [want]


@pytest.mark.parametrize("side", [-1, 1])
def test_not_moving_thres_at_one_ulp(side):
    asg = kr.BlockAssigner()
    p0 = np.array([0.0, 0, 0, 1, 0, 0, 0])
    asg.assign([1], [p0], [False], 0, True)
    p1 = p0.copy()
    p1[0] = at(kr.NOT_MOVING_THRES, side)                       # yaw 0: the delta's x is exact
    assert asg.assign([1], [p1], [False], 0, True)["new_block"][0] == (0 if side < 0 else 1)


@pytest.mark.parametrize("rel,want", [(-1e-9, 0), (1e-9, 1)])
def test_not_moving_yaw_edges(rel, want):
    asg = kr.BlockAssigner()
    p0 = np.array([0.0, 0, 0, 1, 0, 0, 0])
    asg.assign([1], [p0], [False], 0, True)
    p2 = np.concatenate([[0.0, 0, 0], kr.pn.quat_from_rotvec(np.array([0, 0, kr.NOT_MOVING_YAW * (1.0 + rel)]))])
    assert asg.assign([1], [p2], [False], 0, True)["new_block"][0] == want


def test_static_and_self_blocks():
    asg = kr.BlockAssigner()
    p = np.array([1.0, 2, 3, 1, 0, 0, 0])
    a = asg.assign([0, 1], [p, p], [False, True], 0, False)
    b = asg.assign([0, 1], [p, p], [False, True], 0, False)
    assert b["new_block"].tolist() == [1, 0] and b["block"][1] == a["block"][1]     # self before finish_init: new
    poses = kr.init_poses(b, np.zeros((4, 4)), 5, 0, False, 1)
    assert poses[b["block"][0]].tolist() == [1.0, 2.0, 3.0, 0.0]


def test_debug_no_rejection_and_disabled_distance():
    nodes, dists, poses = two_nodes(dis=50.0)
    f = kr.outlier_flags(nodes, dists, poses, nodes, dict(PRM, finish_init=True, debug_no_rejection=True))
    assert f.tolist() == [0]
    f = kr.outlier_flags(nodes, dists, poses, nodes, dict(PRM, finish_init=True, enable_distance=False))
    assert f.tolist() == [1]
    store = {5: (nodes, dists, np.array([0], np.int8))}
    window = [(5, {0: 0, 1: 1})]
    en = np.ones(256, bool)
    assert len(kr.distance_rows(window, store, en, dict(PRM, enable_distance=False))["ia"]) == 0
    r = kr.distance_rows(window, store, en, dict(PRM, debug_no_rejection=True))
    assert r["huber"].tolist() == [0] and r["ia"].tolist() == [1] and r["ib"].tolist() == [0]


def test_row_gates():
    nodes, dists, poses = two_nodes(n_d=(1, 1), peers=(1, 0))       # 0 -> 1 has b > a: no row
    store = {5: (nodes, dists, np.array([-1, -1], np.int8))}
    en = np.zeros(256, bool)
    assert kr.distance_rows([(5, {0: 0, 1: 1})], store, en, PRM)["ia"].tolist() == []   # drone 1 not enabled
    en[1] = True
    assert kr.distance_rows([(5, {0: 0, 1: 1})], store, en, PRM)["ia"].tolist() == [1]
    assert kr.distance_rows([(5, {1: 1})], store, en, PRM)["ia"].tolist() == []          # peer absent from the frame
    nodes["dists_available"][1] = 0
    assert kr.distance_rows([(5, {0: 0, 1: 1})], store, en, PRM)["ia"].tolist() == []
