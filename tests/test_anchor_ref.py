"""CPU: the re-anchoring oracle (oracle/anchor_ref.py) rule by rule on hand-built swarms, its numpy form and the C
stand-in (oracle/c/anchor_ref.c) against the literal walk."""
import numpy as np
import pytest

from omniswarm_b200 import synth
from oracle import anchor_ref as ar, anchor_c, pnp_ref as pn, solver_ref as sr

NS = ar.NS
T0 = 1_700_000_000 * NS
INT_FIELDS = ("id", "type", "status", "frame_a", "frame_b", "node_a", "node_b", "stamp_a", "stamp_b", "dt_err_ns", "skip",
              "ia", "ib", "huber", "factor_type")
PRM = dict(begin_min_loop_dt_s=1000.0, det_dpos_thres=5.0, odom_pos_cov_per_m=1e-3, odom_ang_cov_per_m=2e-4, huber=True)


def pose(x, y, z, yaw, roll=0.0, pitch=0.0):
    return np.concatenate([[x, y, z], pn.quat_from_rotvec(np.array([roll, pitch, yaw]))])


def line_traj(drone, t_from_s=-2.0, t_to_s=30.0, hz=100):
    """1 m/s along x with a slow yaw and some roll/pitch"""
    k = np.arange(int((t_to_s - t_from_s) * hz) + 1)
    t = t_from_s + k / hz
    stamps = T0 + np.round(t * NS).astype(np.int64)
    return stamps, np.stack([pose(tt, 2.0 * drone, 1.0, 0.05 * tt + drone, 0.1, -0.05) for tt in t])


def entry(d, stamp_ns, block, vo=1, traj=None):
    p = traj[1][ar.Trajectory(*traj).nearest(stamp_ns)] if traj is not None else pose(0, 0, 0, 0)
    return (d, vo, block, 0, stamp_ns, p)


def window(frames):
    """frames: [(frame stamp, [entry tuples])] -> (frame_stamps, frame_first, entries)"""
    stamps = np.array([f[0] for f in frames], np.int64)
    first = np.cumsum([0] + [len(f[1]) for f in frames]).astype(np.int32)
    entries = np.array([e for f in frames for e in f[1]], dtype=ar.ENTRY_DTYPE)
    return stamps, first, entries


def meas(rows):
    """rows: dicts with id, type, id_a, id_b, stamp_a, stamp_b and optional rel, cov, self_a, self_b"""
    m = np.zeros(len(rows), ar.MEAS_DTYPE)
    for i, r in enumerate(rows):
        m[i] = (r["id"], r.get("type", ar.LOOP), r["id_a"], r["id_b"], 0, r["stamp_a"], r["stamp_b"],
                r.get("rel", pose(1.0, 0.5, 0.1, 0.3)), r.get("cov", np.diag([0.01, 0.012, 0.02, 1e-3, 1e-3, 2e-3])),
                r.get("self_a", pose(0, 0, 0, 0)), r.get("self_b", pose(0, 0, 0, 0)))
    return m


def run(trajs, win, m, prm=PRM, yaw=None):
    """the literal walk, checked against its numpy form and the C stand-in"""
    yaw = np.ones(8, np.uint8) if yaw is None else yaw
    ref = ar.anchor(trajs, win, m, yaw, prm)
    for other in (ar.anchor_vec(trajs, win, m, yaw, prm), anchor_c.anchor(trajs, win, m, yaw, prm)):
        for f in INT_FIELDS:
            assert np.array_equal(ref[f], other[f]), f
        assert np.array_equal(ref["dpos"], other["dpos"])
        np.testing.assert_allclose(other["payload"], ref["payload"], rtol=1e-12, atol=1e-12)
        np.testing.assert_allclose(other["edge"]["rel_pose"], ref["edge"]["rel_pose"], rtol=1e-12, atol=1e-12)
        assert np.array_equal(other["edge"]["cov"], ref["edge"]["cov"])
    return ref


TR = {0: line_traj(0), 1: line_traj(1)}


def s(t):
    return T0 + int(round(t * NS))


def test_frame_tie_keeps_the_earliest_frame():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.0), 1, traj=TR[1])]),
                  (s(2.0), [entry(0, s(2.0), 2, traj=TR[0]), entry(1, s(2.0), 3, traj=TR[1])])])
    r = run(TR, win, meas([dict(id=1, id_a=0, id_b=1, stamp_a=s(1.5), stamp_b=s(1.5)),
                           dict(id=2, id_a=0, id_b=1, stamp_a=s(1.5) + 1, stamp_b=s(1.5) - 1)]))
    assert r["status"].tolist() == [ar.OK, ar.OK]
    assert (r["frame_a"].tolist(), r["frame_b"].tolist()) == ([0, 1], [0, 0])
    assert (r["node_a"].tolist(), r["node_b"].tolist()) == ([0, 2], [1, 1])
    assert r["dt_err_ns"].tolist() == [NS, NS - 2]


def test_min_err_starts_at_10000_s_strictly():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.0), 1, traj=TR[1])])])
    far = 10000 * NS
    r = run(TR, win, meas([dict(id=1, id_a=0, id_b=1, stamp_a=s(1.0), stamp_b=s(1.0) + far),
                           dict(id=2, id_a=0, id_b=1, stamp_a=s(1.0), stamp_b=s(1.0) + far - 1)]))
    assert r["status"][0] == ar.NO_FRAME and r["frame_b"][0] == -1 and r["frame_a"][0] == 0
    assert r["dt_err_ns"][0] == far
    assert r["status"][1] == ar.DPOS and r["frame_b"][1] == 0 and r["dt_err_ns"][1] == far - 1


def test_vo_unavailable_entries_are_ignored():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.0), 1, traj=TR[1])]),
                  (s(2.0), [entry(0, s(2.0), 2, vo=0, traj=TR[0]), entry(1, s(2.0), 3, traj=TR[1])])])
    r = run(TR, win, meas([dict(id=1, id_a=0, id_b=1, stamp_a=s(2.0), stamp_b=s(2.0))]))
    assert (r["frame_a"][0], r["frame_b"][0], r["node_a"][0]) == (0, 1, 0)
    win = window([(s(1.0), [entry(0, s(1.0), 0, vo=0, traj=TR[0]), entry(1, s(1.0), 1, traj=TR[1])])])
    assert run(TR, win, meas([dict(id=1, id_a=0, id_b=1, stamp_a=s(1.0), stamp_b=s(1.0))]))["status"][0] == ar.NO_FRAME


def test_before_window_is_strict_and_tests_stamp_a_only():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.0), 1, traj=TR[1])])])
    k = 1000 * NS
    r = run(TR, win, meas([dict(id=1, id_a=0, id_b=1, stamp_a=s(1.0) - k, stamp_b=s(1.0)),
                           dict(id=2, id_a=0, id_b=1, stamp_a=s(1.0) - k - 1, stamp_b=s(1.0)),
                           dict(id=3, id_a=0, id_b=1, stamp_a=s(1.0), stamp_b=s(1.0) - 5 * k)]))
    assert r["status"][0] != ar.BEFORE_WINDOW and r["frame_a"][0] == 0
    assert r["status"][1] == ar.BEFORE_WINDOW and r["frame_a"][1] == -1 and r["dt_err_ns"][1] == 0
    assert r["status"][2] != ar.BEFORE_WINDOW and r["frame_b"][2] == 0


def test_dpos_boundary():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.0), 1, traj=TR[1])])])
    m = meas([dict(id=1, id_a=0, id_b=1, stamp_a=s(1.37), stamp_b=s(0.81))])
    dpos = run(TR, win, m, dict(PRM, det_dpos_thres=100.0))["dpos"][0]
    assert 0.5 < dpos < 0.6
    assert run(TR, win, m, dict(PRM, det_dpos_thres=float(dpos)))["status"][0] == ar.OK
    assert run(TR, win, m, dict(PRM, det_dpos_thres=float(np.nextafter(dpos, 0.0))))["status"][0] == ar.DPOS


def test_detections_take_self_poses_from_the_trajectories_and_det4d_is_yaw_only():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.0), 1, traj=TR[1])])])
    junk_a, junk_b = pose(9, 9, 9, 2.0, 0.4, 0.3), pose(-9, 3, 1, -1.0, -0.2, 0.1)
    rows = [dict(id=i, type=t, id_a=0, id_b=1, stamp_a=s(1.2), stamp_b=s(1.2), self_a=junk_a, self_b=junk_b)
            for i, t in enumerate((ar.LOOP, ar.DET4D, ar.DET6D))]
    r = run(TR, win, meas(rows))
    loop, d4, d6 = r["edge"]["rel_pose"]
    np.testing.assert_allclose(d4, d6, rtol=0, atol=1e-13)                 # DeltaPose(.., true) reads yaw and position only
    assert np.abs(loop - d4).max() > 1.0
    t = ar.Trajectory(*TR[0])
    sp = t.pose_by_appro_ts(s(1.2))
    yo = ar.set_yaw_only(sp)
    assert np.array_equal(yo[:3], sp[:3]) and abs(pn.quat2eulers(yo[3:])[2] - pn.quat2eulers(sp[3:])[2]) < 1e-15
    assert np.abs(pn.quat2eulers(yo[3:])[:2]).max() < 1e-15 and np.abs(pn.quat2eulers(sp[3:])[:2]).max() > 0.04
    want = ar.pr.pose_mul(ar.pr.pose_mul(pn.delta_pose(win[2]["self_pose"][0], yo, True), pose(1.0, 0.5, 0.1, 0.3)),
                          pn.delta_pose(ar.set_yaw_only(ar.Trajectory(*TR[1]).pose_by_appro_ts(s(1.2))),
                                        win[2]["self_pose"][1], True))
    np.testing.assert_allclose(d4, want, rtol=0, atol=1e-15)


def test_missing_trajectory_is_a_status_after_the_frame_search():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.0), 1, traj=TR[1]), entry(2, s(1.0), 2)])])
    r = run(TR, win, meas([dict(id=1, id_a=0, id_b=2, stamp_a=s(1.0), stamp_b=s(1.0)),
                           dict(id=2, id_a=3, id_b=0, stamp_a=s(1.0), stamp_b=s(1.0)),
                           dict(id=3, id_a=2, id_b=2, stamp_a=s(1.0), stamp_b=s(1.0))]))
    assert r["status"].tolist() == [ar.NO_TRAJECTORY, ar.NO_FRAME, ar.NO_TRAJECTORY]
    assert r["frame_b"][0] == 0 and r["node_b"][0] == 2 and r["skip"].tolist() == [1, 1, 1]


def test_anchored_measurement_comes_back_unchanged():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.03), 1, traj=TR[1])]),
                  (s(1.5), [entry(0, s(1.5), 2, traj=TR[0]), entry(1, s(1.5), 3, traj=TR[1])])])
    e = win[2]
    rel, cov = pose(1.0, -2.0, 0.3, 0.7), np.diag([0.01, 0.012, 0.02, 1e-3, 1e-3, 2e-3]) + 1e-4
    r = run(TR, win, meas([dict(id=1, id_a=0, id_b=1, stamp_a=s(1.5), stamp_b=s(1.03), rel=rel, cov=cov,
                                self_a=e["self_pose"][2], self_b=e["self_pose"][1])]))
    assert r["status"][0] == ar.OK and r["dt_err_ns"][0] == 0 and r["dpos"][0] == 0.0
    assert (r["frame_a"][0], r["frame_b"][0], r["node_a"][0], r["node_b"][0]) == (1, 0, 2, 1)
    np.testing.assert_allclose(r["edge"]["rel_pose"][0], rel, rtol=0, atol=1e-12)
    assert np.array_equal(r["edge"]["cov"][0], cov)                        # cov_odom = 0


def test_sqrt_information_is_the_create_cov6d_rule():
    r = run(*(lambda g: (g["trajs"], g["window"], g["meas"]))(synth.anchor_swarm(3, 12, 60, seed=4)))
    ok = r["status"] == ar.OK
    assert ok.sum() > 10
    for row in r[ok]:
        np.testing.assert_allclose(row["payload"][4:20], sr.create_cov6d_sqrt_inf(row["edge"]["cov"]).reshape(-1),
                                   rtol=1e-15, atol=0)
        assert row["payload"][3] == pn.quat2eulers(row["edge"]["rel_pose"][3:])[2]


def test_skip_rules():
    win = window([(s(1.0), [entry(0, s(1.0), 0, traj=TR[0]), entry(1, s(1.0), 0, traj=TR[1])]),
                  (s(1.5), [entry(0, s(1.5), 1, traj=TR[0]), entry(1, s(1.5), 2, traj=TR[1])])])
    m = meas([dict(id=1, id_a=0, id_b=1, stamp_a=s(1.0), stamp_b=s(1.0)),        # both ends on shared block 0
              dict(id=2, id_a=0, id_b=1, stamp_a=s(1.5), stamp_b=s(1.5))])
    assert run(TR, win, m)["skip"].tolist() == [1, 0]
    yaw = np.ones(8, np.uint8)
    yaw[1] = 0
    r = run(TR, win, m, yaw=yaw)
    assert r["skip"].tolist() == [1, 1] and r["status"].tolist() == [ar.OK, ar.OK]


def test_empty_window_and_output_order():
    win = window([])
    m = meas([dict(id=1, type=ar.DET6D, id_a=0, id_b=1, stamp_a=s(1.0), stamp_b=s(1.0)),
              dict(id=2, id_a=0, id_b=1, stamp_a=s(1.0), stamp_b=s(1.0)),
              dict(id=3, type=ar.DET4D, id_a=0, id_b=1, stamp_a=s(1.0), stamp_b=s(1.0)),
              dict(id=4, id_a=1, id_b=0, stamp_a=s(1.0), stamp_b=s(1.0))])
    r = run(TR, win, m)
    assert r["id"].tolist() == [2, 4, 1, 3]                                # loops, then detections, each in arrival order
    assert (r["status"] == ar.EMPTY_WINDOW).all() and (r["skip"] == 1).all()


@pytest.mark.parametrize("seed", [0, 1])
def test_c_standin_and_numpy_form_equal_the_oracle_on_a_synthetic_swarm(seed):
    g = synth.anchor_swarm(5, 40, 800, seed=seed)
    r = run(g["trajs"], g["window"], g["meas"], g["prm"], np.ones(g["max_drones"], np.uint8))
    counts = np.bincount(r["status"], minlength=6)
    assert counts[ar.OK] > 100 and counts[ar.BEFORE_WINDOW] > 0 and counts[ar.NO_FRAME] > 0
    assert counts[ar.NO_TRAJECTORY] > 0 and counts[ar.DPOS] > 0
