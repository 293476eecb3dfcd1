"""CPU: the hand-over of a round's loop edges from the front-end to the back-end's store (tests/loop_measurements_ref.py):
ids and counters across rounds, which statuses count, the roles of a swapped hit, the intra-drone +2, and the solver's
float distance gate."""
import numpy as np

from omniswarm_b200 import lib
import loop_measurements_ref as lm

COV_POS, COV_ANG = 0.02, 0.005


def edge(status, a, b, t=(0.3, -0.1, 0.05)):
    return dict(status=status, drone_id_a=a, drone_id_b=b, relative_pose=np.r_[t, 1.0, 0.0, 0.0, 0.0])


def cand(k):
    return dict(pose_query=np.r_[k, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0], pose_hit=np.r_[0.0, k, 0.0, 1.0, 0.0, 0.0, 0.0])


def round_(edges, swapped=None, self_id=3, counters=None):
    n = len(edges)
    return lm.loop_measurements(edges, swapped or [0] * n, [cand(k) for k in range(n)],
                                [(1000 + k, 2000 + k) for k in range(n)], self_id, COV_POS, COV_ANG,
                                counters or lm.new_counters())


def test_layout_is_the_headers():
    assert lm.MEASUREMENT_DTYPE == lib.MEASUREMENT_DTYPE and lm.MEASUREMENT_DTYPE.itemsize == 496
    assert (lm.MAX_LOOP_ID, lm.LOOP_ACCEPTED, lm.MEAS_LOOP) == (100000000, lib.LOOP_ACCEPTED, lib.MEAS_LOOP)


def test_ids_across_rounds_with_a_rejected_candidate_between():
    rows, c = round_([edge(lib.LOOP_ACCEPTED, 3, 5), edge(lib.LOOP_PNP_FAILED, 3, 6), edge(lib.LOOP_ACCEPTED, 3, 7)])
    assert rows["id"].tolist() == [300000000, 300000001] and rows["id_b"].tolist() == [5, 7]
    rows, c = round_([edge(lib.LOOP_NO_HIT, 3, 5), edge(lib.LOOP_ACCEPTED, 3, 4)], counters=c)
    assert rows["id"].tolist() == [300000002] and c[0] == 3
    rows, c = round_([], counters=c)                          # an empty round changes nothing
    assert len(rows) == 0 and c[0] == 3


def test_only_accepted_counts():
    statuses = list(range(9))
    rows, (n, pairs) = round_([edge(s, 3, 4) for s in statuses])
    assert len(rows) == 1 and n == 1 and pairs.sum() == 2
    for s in (lib.LOOP_ODOMETRY_INCONSISTENT, lib.LOOP_PNP_FAILED, lib.LOOP_NOT_VERIFIED):
        rows, (n, pairs) = round_([edge(s, 3, 4)])
        assert len(rows) == 0 and n == 0 and pairs.sum() == 0


def test_swapped_roles():
    """swapped: the query keyframe is the old side, so stamp_a / self_pose_a are the query's"""
    rows, _ = round_([edge(lib.LOOP_ACCEPTED, 3, 8), edge(lib.LOOP_ACCEPTED, 3, 8)], swapped=[1, 0])
    s, u = rows
    c0, c1 = cand(0), cand(1)
    assert (s["stamp_a"], s["stamp_b"]) == (1000, 2000) and (u["stamp_a"], u["stamp_b"]) == (2001, 1001)
    assert np.array_equal(s["self_pose_a"], c0["pose_query"]) and np.array_equal(s["self_pose_b"], c0["pose_hit"])
    assert np.array_equal(u["self_pose_a"], c1["pose_hit"]) and np.array_equal(u["self_pose_b"], c1["pose_query"])
    assert (s["id_a"], s["id_b"], s["type"], s["reserved"]) == (3, 8, lib.MEAS_LOOP, 0)
    assert np.array_equal(s["cov"], np.diag([COV_POS] * 3 + [COV_ANG] * 3))


def test_pair_counts_and_the_intra_drone_plus_two():
    rows, (n, pairs) = round_([edge(lib.LOOP_ACCEPTED, 3, 3), edge(lib.LOOP_ACCEPTED, 3, 9), edge(lib.LOOP_ACCEPTED, 300, 3)])
    assert n == 3 and len(rows) == 3                          # an id outside 0..255 is emitted, not counted
    assert pairs[3, 3] == 2 and pairs[9, 3] == 1 and pairs[3, 9] == 1 and pairs.sum() == 4


def test_large_self_id_does_not_overflow():
    rows, _ = round_([edge(lib.LOOP_ACCEPTED, 30, 31)], self_id=30)
    assert rows["id"][0] == 3_000_000_000                     # beyond int32: the reference's int would wrap


def loops_at(distances, direction=(0.6, 0.0, 0.8)):
    rows = np.zeros(len(distances), lm.MEASUREMENT_DTYPE)
    for r, d in zip(rows, distances):
        r["relative_pose"][:3] = np.asarray(direction) * d if d is not None else 0
    rows["relative_pose"][:, 3] = 1.0
    return rows


def test_gate_at_two_and_one_ulp_either_side():
    below, above = np.nextafter(2.0, 0.0), np.nextafter(2.0, 4.0)
    rows = loops_at([0.0, 0.0, 0.0])
    rows["relative_pose"][:, 0] = [below, 2.0, above]         # a norm that is exactly x
    assert [lm.loop_distance(r) for r in rows] == [below, 2.0, above]
    kept = lm.add_new_loop_connection(rows, 2.0)
    assert kept["relative_pose"][:, 0].tolist() == [below, 2.0]


def test_gate_compares_with_the_float_threshold():
    t32 = np.float64(np.float32(0.1))                         # 0.100000001490116...
    rows = loops_at([0.0, 0.0])
    rows["relative_pose"][:, 1] = [t32, np.nextafter(t32, 1.0)]
    assert 0.1 < t32                                          # a double threshold of 0.1 would drop the first
    kept = lm.add_new_loop_connection(rows, 0.1)
    assert kept["relative_pose"][:, 1].tolist() == [t32]


def test_detections_are_not_gated_and_dropped_rows_keep_their_ids():
    rows, c = round_([edge(lib.LOOP_ACCEPTED, 3, 4, t=(3.0, 0, 0)), edge(lib.LOOP_ACCEPTED, 3, 4),
                      edge(lib.LOOP_ACCEPTED, 3, 4, t=(0, 2.5, 0))])
    kept = lm.add_new_loop_connection(rows, 2.0)
    assert kept["id"].tolist() == [300000001] and c[0] == 3   # the dropped loops used up ids 0 and 2
    rows, c = round_([edge(lib.LOOP_ACCEPTED, 3, 4)], counters=c)
    assert rows["id"].tolist() == [300000003]
    det = rows.copy()
    det["type"] = lib.MEAS_DET6D
    det["relative_pose"][:, 0] = 50.0
    assert len(lm.add_new_loop_connection(det, 2.0)) == 1
