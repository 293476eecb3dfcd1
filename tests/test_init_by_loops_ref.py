"""The pre-motion init start's oracle (tests/init_by_loops_ref.py): the literal walk of init_pose_by_loops over the
dict-of-dict bookkeeping against the vectorised form over the device's representation, and each of the reference's
quirks pinned on a small hand-made swarm."""
import numpy as np
import pytest

from oracle import anchor_ref as ar
from oracle import pcm_ref as pr
from omniswarm_b200 import lib, synth

import init_by_loops_ref as ib

NS = 1_000_000_000
T0 = 1_700_000_000 * NS


def _quat(yaw):
    return np.array([np.cos(yaw / 2), 0.0, 0.0, np.sin(yaw / 2)])


def world(n_frames=4, shared=False):
    """drones 0..3 flying straight lines with a yawing odometry frame; one frame per second, every drone in every frame
    (drone d, frame f -> block 4 f + d; with `shared`, drone 3 keeps block 3 in frames 0 and 1)"""
    trajs = {}
    for d in range(4):
        st = T0 + np.arange(0, (n_frames + 2) * 10) * (NS // 10) + d * 1000
        t = (st - T0) / NS
        poses = np.stack([np.r_[0.5 * t[i] + d, 0.2 * t[i] * d, 1.0 + 0.1 * d, _quat(0.3 * d + 0.05 * t[i])]
                          for i in range(len(st))])
        trajs[d] = (st, poses)
    frame_stamps = T0 + np.arange(n_frames) * NS + NS // 2
    entries = []
    for f in range(n_frames):
        for d in range(4):
            blk = 3 if (shared and d == 3 and f == 1) else 4 * f + d
            st = int(frame_stamps[f]) + 7_000 * d
            entries.append((d, 1, blk, 0, st, trajs[d][1][int((st - T0) // (NS // 10))]))
    entries = np.array(entries, lib.WINDOW_ENTRY_DTYPE)
    first = np.arange(0, 4 * n_frames + 1, 4, dtype=np.int32)
    return trajs, (frame_stamps, first, entries), np.zeros((4 * n_frames, 4))


def row(i, a, b, ta, tb, rel, status=ar.OK):
    r = np.zeros(1, ar.RESULT_DTYPE)
    r["id"], r["status"], r["stamp_a"], r["stamp_b"] = i, status, ta, tb
    r["edge"]["id_a"], r["edge"]["id_b"], r["edge"]["rel_pose"] = a, b, rel
    return r


def rel_pose(x, y, yaw):
    return np.r_[x, y, 0.1, _quat(yaw)]


def run_both(rows_by_solve, to_init, good_sets, estimated, kf, trajs, window, poses, self_id=0, redundant=True):
    book = ib.LoopBook(self_id, redundant)
    lmap = ib.LoopMapVec(4, lib.LOOP_RECORD_DTYPE)
    for rows in rows_by_solve:
        book.record(rows)
        lmap.record_vec(rows)
    est_mask = np.zeros(4, bool)
    est_mask[list(estimated)] = True
    outs = []
    for f in (lambda: ib.init_pose_by_loops(to_init, ib.good_from_sets(good_sets), book, estimated, kf, ib.Trajs(trajs),
                                            self_id, window, poses),
              lambda: ib.init_by_loops_vec(np.isin(np.arange(4), list(to_init)), good_sets, lmap, est_mask, kf, trajs,
                                           self_id, window, poses)):
        try:
            outs.append(f())
        except ib.Refused:
            outs.append(None)
    lit, vec = outs
    assert (lit is None) == (vec is None)
    if lit is not None:
        np.testing.assert_allclose(vec, lit, rtol=1e-12, atol=1e-12)
    return lit, book, lmap


def expected(trajs, window, d, id2, e, pose0=None, t0=None):
    """placement of drone d from loop e (already oriented id2 -> d) by hand -> {block: [4]}"""
    tr = ib.Trajs(trajs)
    t0 = e["ts_a"] if t0 is None else t0
    pose0 = ib.IDENTITY if pose0 is None else pose0
    out = {}
    for ts, nodes in ar.window_frames(*window):
        if d in nodes:
            p = pr.pose_mul(pr.pose_mul(pr.pose_mul(pose0, tr.relative(id2, t0, e["ts_a"])), e["rel"]),
                            tr.relative(id2, e["ts_b"], ts))
            out[nodes[d]["block"]] = np.r_[p[:3], ib.yaw(p[3:])]
    return out


@pytest.mark.parametrize("redundant", [True, False])
@pytest.mark.parametrize("seed", [0, 1, 2])
def test_forms_agree_on_a_swarm(seed, redundant):
    g = synth.anchor_swarm(n_drones=4, n_frames=16, n_meas=160, seed=seed, with_orphans=False)
    y = np.ones(g["max_drones"], np.uint8)
    frame_stamps, first, entries = g["window"]
    half = (frame_stamps[:10], first[:11], entries[:first[10]])
    rows1 = ar.anchor_vec(g["trajs"], half, g["meas"][:80], y, g["prm"])
    rows2 = ar.anchor_vec(g["trajs"], g["window"], g["meas"], y, g["prm"])
    rng = np.random.default_rng(seed)
    n_blk = int(entries["block"].max()) + 1
    poses = rng.normal(0, 1, (n_blk, 4))
    kf = {0: (frame_stamps[:5], np.stack([g["trajs"][0][1][k * 50] for k in range(5)]))}
    good = {(0, 2): [int(i) for i in rows2["id"][rows2["status"] == ar.OK][:3]]} if seed == 1 else {}
    lit, book, lmap = run_both([rows1, rows2], {1, 2, 3}, good, {0, 1}, kf, g["trajs"], g["window"], poses,
                               redundant=redundant)
    assert lit is not None and not np.array_equal(lit, poses)
    assert sorted(book.all_loop_map) == list(lmap.recs["id"])
    for r in lmap.recs:                                            # the records are the first-seen edges
        e = book.all_loop_map[int(r["id"])]
        assert (e["id_a"], e["id_b"], e["ts_a"], e["ts_b"]) == (r["id_a"], r["id_b"], r["stamp_a"], r["stamp_b"])
        assert np.array_equal(e["rel"], r["rel_pose"])
    for a in range(4):
        for b in range(4):
            s = book.all_loops_set_by_pair.get(a, {}).get(b)
            assert lmap.pair_min[a, b] == (min(s) if s else ib.I64_MAX)


def test_good_set_replaces_the_whole_map():
    trajs, win, poses = world()
    rows = [np.concatenate([row(10, 0, 1, T0 + NS, T0 + NS, rel_pose(1, 0, 0.1))])]
    lit, _, _ = run_both(rows, {1}, {}, {0}, {}, trajs, win, poses)
    assert not np.array_equal(lit, poses)
    lit, _, _ = run_both(rows, {1}, {(1, 2): [10]}, {0}, {}, trajs, win, poses)   # 2 is not estimated: nothing
    assert np.array_equal(lit, poses)


def test_last_qualifying_id2_wins_and_skips():
    trajs, win, poses = world()
    r02 = row(20, 2, 3, T0 + NS, T0 + 2 * NS, rel_pose(0, 1, 0.2))
    r00 = row(21, 0, 3, T0 + NS, T0 + NS, rel_pose(1, 0, 0.1))
    both, _, _ = run_both([np.concatenate([r00, r02])], {3}, {}, {0, 2}, {}, trajs, win, poses)
    only2, _, _ = run_both([r02], {3}, {}, {0, 2}, {}, trajs, win, poses)
    assert np.array_equal(both, only2)
    only0, _, _ = run_both([r00], {3}, {}, {0}, {}, trajs, win, poses)
    not_est, _, _ = run_both([np.concatenate([r00, r02])], {3}, {}, {0}, {}, trajs, win, poses)
    assert np.array_equal(not_est, only0)                          # 2 not estimated: 0 decides
    empty, _, _ = run_both([np.concatenate([r00, r02])], {3}, {(3, 2): [], (3, 0): [21]}, {0, 2}, {}, trajs, win,
                           poses)
    assert np.array_equal(empty, only0)                            # an empty set is skipped


def test_inversion_and_pose0_sources():
    trajs, win, poses = world()
    e = dict(id=30, id_a=1, id_b=2, ts_a=T0 + NS, ts_b=T0 + 2 * NS, rel=rel_pose(0.5, -0.5, 0.4))
    r = row(30, 1, 2, e["ts_a"], e["ts_b"], e["rel"])
    # drone 1 placed from 2: the loop's id_a is 1 != 2, so it is inverted; 2 has no path and is not self: identity
    lit, _, _ = run_both([r], {1}, {}, {2}, {}, trajs, win, poses)
    for blk, p in expected(trajs, win, 1, 2, ib.invert_loop(e)).items():
        np.testing.assert_allclose(lit[blk], p, rtol=1e-13, atol=1e-13)
    # drone 2 from 1: no inversion; 1 == self_id and has no path: its odometry nearest to ts_a
    lit, _, _ = run_both([r], {2}, {}, {1}, {}, trajs, win, poses, self_id=1)
    tr = ib.Trajs(trajs).at(1)
    k = tr.nearest(e["ts_a"])
    for blk, p in expected(trajs, win, 2, 1, e, tr.poses[k], tr.stamps[k]).items():
        np.testing.assert_allclose(lit[blk], p, rtol=1e-13, atol=1e-13)
    # a keyframe path of 1 comes first
    kf = {1: (np.array([T0 + NS - 3, T0 + 3 * NS]), np.stack([rel_pose(9, 9, 1.0), rel_pose(-9, 0, -1.0)]))}
    lit, _, _ = run_both([r], {2}, {}, {1}, kf, trajs, win, poses, self_id=1)
    for blk, p in expected(trajs, win, 2, 1, e, kf[1][1][0], int(kf[1][0][0])).items():
        np.testing.assert_allclose(lit[blk], p, rtol=1e-13, atol=1e-13)


def test_odomb_is_taken_on_id2s_trajectory():
    trajs, win, poses = world()
    r = row(40, 0, 3, T0 + NS, T0 + NS, rel_pose(1, 1, 0.3))
    a, _, _ = run_both([r], {3}, {}, {0}, {}, trajs, win, poses)
    moved = dict(trajs)
    moved[3] = (trajs[3][0], trajs[3][1] + np.r_[5.0, 0, 0, 0, 0, 0, 0])
    b, _, _ = run_both([r], {3}, {}, {0}, {}, moved, win, poses)
    assert np.array_equal(a, b)                                    # _id's own odometry is never read
    moved = dict(trajs)
    moved[0] = (trajs[0][0], trajs[0][1] * np.r_[2.0, 1, 1, 1, 1, 1, 1])
    c, _, _ = run_both([r], {3}, {}, {0}, {}, moved, win, poses)
    assert not np.array_equal(a, c)


def test_shared_blocks_take_the_latest_frame():
    trajs, win, poses = world(shared=True)
    e = dict(id=50, id_a=0, id_b=3, ts_a=T0 + NS, ts_b=T0 + NS, rel=rel_pose(1, 0, 0.2))
    lit, _, _ = run_both([row(50, 0, 3, e["ts_a"], e["ts_b"], e["rel"])], {3}, {}, {0}, {}, trajs, win, poses,
                         self_id=2)
    frames = ar.window_frames(*win)
    tr = ib.Trajs(trajs)
    p = pr.pose_mul(pr.pose_mul(pr.pose_mul(ib.IDENTITY, tr.relative(0, e["ts_a"], e["ts_a"])), e["rel"]),
                    tr.relative(0, e["ts_b"], frames[1][0]))
    np.testing.assert_allclose(lit[3], np.r_[p[:3], ib.yaw(p[3:])], rtol=1e-13, atol=1e-13)


def test_first_seen_values_survive_reanchoring():
    trajs, win, poses = world()
    r1 = row(60, 0, 1, T0 + NS, T0 + NS, rel_pose(1, 0, 0.1))
    r2 = row(60, 0, 1, T0 + 2 * NS, T0 + 2 * NS, rel_pose(2, 0, 0.5))         # the next solve re-anchors it
    dup = row(60, 0, 1, T0 + 3 * NS, T0 + 3 * NS, rel_pose(3, 0, 0.5))        # and holds it twice: the first row wins
    _, book, lmap = run_both([r1, np.concatenate([r2, dup])], {1}, {}, {0}, {}, trajs, win, poses)
    assert book.all_loop_map[60]["ts_a"] == T0 + NS and lmap.recs["stamp_a"][0] == T0 + NS
    _, book, lmap = run_both([np.concatenate([r2, dup])], {1}, {}, {0}, {}, trajs, win, poses)
    assert book.all_loop_map[60]["ts_a"] == T0 + 2 * NS and lmap.recs["stamp_a"][0] == T0 + 2 * NS


def test_unrouted_pairs_are_recorded_in_non_redundant_mode():
    trajs, win, poses = world()
    r = row(70, 1, 2, T0 + NS, T0 + NS, rel_pose(1, 0, 0.1))
    lit, book, lmap = run_both([r, r], {2}, {}, {1}, {}, trajs, win, poses, self_id=0, redundant=False)
    assert 70 not in book.all_loops_set and book.all_loops_set_by_pair[2][1] == {70} and lmap.pair_min[2, 1] == 70
    assert not np.array_equal(lit, poses)


def test_refusals():
    trajs, win, poses = world()
    r = row(80, 0, 1, T0 + NS, T0 + NS, rel_pose(1, 0, 0.1))
    lit, _, _ = run_both([r], {1}, {(0, 1): [81]}, {0}, {}, trajs, win, poses)     # 81 is not in all_loop_map
    assert lit is None
    no0 = {d: v for d, v in trajs.items() if d != 0}
    lit, _, _ = run_both([r], {1}, {}, {0}, {}, no0, win, poses)                   # id2 without odometry
    assert lit is None
    empty = (win[0][:0], win[1][:1], win[2][:0])                                   # ... unless nothing reads it
    lit, _, _ = run_both([r], {1}, {}, {0}, {}, no0, empty, poses, self_id=2)
    assert lit is not None and np.array_equal(lit, poses)
    lit, _, _ = run_both([r], {1}, {}, {0}, {}, no0, empty, poses, self_id=0)      # self's start needs it
    assert lit is None
