"""CPU: the publication oracle of tests/publish_ref.py (sync_est_poses and PredictSwarm) -- the bounded nearest-keyframe
walk, the numpy full path against the literal one, the per-drone record the device keeps against the reference's reverse
scan of last_saved_est_kf_ts, and the conditions of predict."""
import numpy as np
import pytest

from omniswarm_b200 import synth
from oracle import anchor_ref as ar
import publish_ref as pb


def trajectories(g):
    return {int(d): ar.Trajectory(*v) for d, v in g["trajs"].items() if len(v[0])}


def frames_of(win, lo, hi):
    """frames [lo, hi) of window `win`"""
    stamps, first, entries = win
    fr = [entries[first[f]:first[f + 1]] for f in range(lo, min(hi, len(stamps)))]
    return (np.asarray(stamps[lo:hi], np.int64), np.cumsum([0] + [len(e) for e in fr]).astype(np.int32),
            np.concatenate(fr) if fr else entries[:0])


def flight(win):
    """the scenario's frames with drone 2 joining at frame 10 and drone 3 leaving after frame 14: a frame keeps its
    drones whichever window holds it, as a SwarmFrame does"""
    stamps, first, entries = win
    fr = []
    for f in range(len(stamps)):
        e = entries[first[f]:first[f + 1]]
        fr.append(e[~(((e["drone_id"] == 2) & (f < 10)) | ((e["drone_id"] == 3) & (f >= 15)))])
    return stamps, np.cumsum([0] + [len(e) for e in fr]).astype(np.int32), np.concatenate(fr)


SLICES = [(0, 8, True), (0, 10, False), (1, 12, False), (3, 14, False), (5, 15, False), (6, 16, True), (7, 18, False),
          (9, 19, False), (16, 22, False), (17, 24, False)]


def rounds(win):
    """steady syncs of a growing and sliding window, drone 2 joining, drone 3 leaving the window, and an init sync
    between steady ones (its pushed stamps go backwards)"""
    w = flight(win)
    return [(frames_of(w, lo, hi), init) for lo, hi, init in SLICES]


def scenario():
    g = synth.anchor_swarm(4, 24, 8, seed=3, with_orphans=False)
    n_blocks = int(g["window"][2]["block"].max()) + 1
    rng = np.random.default_rng(0)
    return g, n_blocks, rng


def test_walk_is_a_nearest_sample_search():
    rng = np.random.default_rng(1)
    for _ in range(50):
        kf = np.unique(rng.integers(0, 10_000, rng.integers(1, 30)))
        q = np.sort(rng.integers(-500, 10_500, 200))
        q = np.sort(np.concatenate([q, (kf[:-1] + kf[1:]) // 2 * (((kf[1:] - kf[:-1]) % 2) == 0)]))   # ties
        q = q[q != 0]
        index = 0
        for t in q:
            index = pb.walk(list(kf), int(t), index)
            assert index == int(ar._nearest_vec(kf, np.array([t]))[0])


def test_full_path_vec_equals_the_literal_loop():
    g, n_blocks, rng = scenario()
    T = trajectories(g)
    st = pb.PublishState()
    poses = np.c_[rng.normal(0, 5, (n_blocks, 3)), rng.uniform(-np.pi, np.pi, n_blocks)]
    st.sync(g["window"], poses, T, True, True)
    assert set(st.full) == set(st.kf) and len(st.full) == 4
    for d, (s, p) in st.full.items():
        s2, p2 = pb.full_path_vec(st.kf[d], *g["trajs"][d])
        assert np.array_equal(s, s2) and len(s) == (len(g["trajs"][d][0]) + 9) // 10
        assert np.abs(p - p2).max() <= 1e-12


def test_record_equals_the_reverse_scan():
    g, n_blocks, rng = scenario()
    T = trajectories(g)
    st, rec = pb.PublishState(), {}
    backwards = False
    for win, is_init in rounds(g["window"]):
        poses = np.c_[rng.normal(0, 5, (n_blocks, 3)), rng.uniform(-np.pi, np.pi, n_blocks)]
        before = list(st.pushed)
        st.sync(win, poses, T, is_init, False)
        backwards |= bool(before) and st.pushed[len(before)] < before[-1]
        pb.record_sync(rec, win, poses, is_init)
        for d in range(g["max_drones"]):
            hit = st.lookup(d)
            if hit is None:
                assert d not in rec
            else:
                ts, saved, vo = rec[d]
                assert ts == hit[0] and np.array_equal(saved, hit[1]) and np.array_equal(vo, hit[2])
        present = set(int(x) for x in win[2]["drone_id"])
        assert set(st.kf) == present                                # a drone that left has no path
    assert backwards                                                # the init sync pushed older stamps


def test_missing_odometry_changes_nothing():
    g, n_blocks, rng = scenario()
    T = trajectories(g)
    del T[2]
    st = pb.PublishState()
    with pytest.raises(pb.NoOdometry):
        st.sync(g["window"], np.zeros((n_blocks, 4)), T, True, True)
    assert st.saved == {} and st.pushed == [] and st.kf == {} and st.full == {}


def test_predict_conditions():
    g, n_blocks, rng = scenario()
    T = trajectories(g)
    st = pb.PublishState()
    stamps, first, entries = frames_of(flight(g["window"]), 10, 14)
    e = [entries[first[f]:first[f + 1]] for f in range(len(stamps))]
    e = [x[x["drone_id"] != 3] for x in e]                         # drone 3 in no saved frame
    win = (stamps, np.cumsum([0] + [len(x) for x in e]).astype(np.int32), np.concatenate(e))
    poses = np.c_[rng.normal(0, 5, (n_blocks, 3)), rng.uniform(-np.pi, np.pi, n_blocks)]
    frame = [(d, T[d].poses[500 + d]) for d in (0, 1, 2, 3)]
    enable = np.array([0, 1, 0, 1], bool)
    assert st.predict(frame, True, 0, enable) == {0: (None, None), 1: (None, None), 2: (None, None), 3: (None, None)}
    st.sync(win, poses, T, True, False)
    assert st.predict(frame, False, 0, enable) == {}
    out = st.predict(frame, True, 0, enable)
    assert out[0][0] is not None and out[0][1] is not None          # self_id: always enabled
    assert out[1][0] is not None and out[1][1] is not None
    assert out[2][0] is None and out[2][1] is not None              # not enabled: the offset only
    assert out[3] == (None, None)                                   # in no saved frame
    # node_pose composes back: base-frame pose of vo_now = node_pose when the vo at the saved frame is yaw-only
    ts, saved, vo = st.lookup(1)
    vo_now = ar.set_yaw_only(vo)
    node, base = st.predict([(1, vo_now)], True, 0, enable)[1]
    assert np.abs(node - pb.pose4(saved)).max() <= 1e-12
