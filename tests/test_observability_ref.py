"""CPU: the observability oracle (oracle/observability_ref.py) rule by rule on hand-built windows and rows: the closure
over OK rows (loops and detections) only when there is more than one node, self_id's first sight, the bounding boxes'
+-1000 start and strict thresholds, the float parameters, the single-drone rule and the state kept across calls."""
import numpy as np

from oracle import anchor_ref as ar, observability_ref as orf

D = 8


def window(*frames):
    """frames: lists of (drone, x, y, z[, vo_available]) -> set_window's (frame_stamps, frame_first, entries)"""
    entries, first = [], [0]
    for f, frame in enumerate(frames):
        for k, e in enumerate(frame):
            d, x, y, z = e[:4]
            vo = e[4] if len(e) > 4 else 1
            entries.append((d, vo, 100 * f + k, 0, 1000 + f, np.r_[x, y, z, 1.0, 0, 0, 0]))
        first.append(len(entries))
    return (np.arange(len(frames), dtype=np.int64), np.array(first, np.int32), np.array(entries, ar.ENTRY_DTYPE))


def still(drones, n_frames=2):
    """n_frames frames holding each drone at one point"""
    return window(*[[(d, float(d), 0.0, 1.0) for d in drones]] * n_frames)


def rows(*specs):
    """specs: (status, id_a, id_b[, node_a, node_b]) -> anchor rows"""
    out = np.zeros(len(specs), ar.RESULT_DTYPE)
    for i, s in enumerate(specs):
        out[i]["status"] = s[0]
        out[i]["edge"]["id_a"], out[i]["edge"]["id_b"] = s[1], s[2]
        out[i]["node_a"], out[i]["node_b"] = (s[3], s[4]) if len(s) > 3 else (10 * i, 10 * i + 1)
    return out


def ids(mask):
    return set(np.flatnonzero(mask).tolist())


def test_closure_runs_over_ok_rows_only_when_there_is_more_than_one_node():
    o = orf.ObservabilityRef(D)
    o.set_window(*still([0]))
    r = o.observe(rows((ar.OK, 0, 1)), 0, 5.0, 5.0)                    # one node: L = {self_id}
    assert ids(r["yaw"]) == {0} and ids(r["pos"]) == {0} and not r["solve_master"]
    o = orf.ObservabilityRef(D)
    o.set_window(*still([0, 1, 2, 3, 4, 5]))
    rr = rows((ar.OK, 1, 0), (ar.OK, 1, 2), (ar.OK, 2, 2), (ar.DPOS, 2, 3), (ar.NO_FRAME, 0, 3),
              (ar.BEFORE_WINDOW, 3, 0), (ar.NO_TRAJECTORY, 4, 0), (ar.OK, 5, 5))
    r = o.observe(rr, 0, 5.0, 5.0)                                      # 0 -loop- 1 -detection- 2; 3, 4, 5 not linked
    assert ids(r["yaw"]) == {0, 1, 2} and ids(r["to_init"]) == {0, 1, 2} and ids(r["enable"]) == {0, 1, 2}
    assert r["solve_master"] and not r["motion"] and ids(r["nodes"]) == {0, 1, 2, 3, 4, 5}
    assert orf.skip(rr, r["yaw"]).tolist() == [0, 0, 0, 1, 1, 1, 1, 1]
    assert orf.skip(rows((ar.OK, 0, 1, 7, 7)), r["yaw"]).tolist() == [1]   # one pose block at both ends
    # a longer chain, found level by level, in any row order
    o = orf.ObservabilityRef(D)
    o.set_window(*still(range(D)))
    r = o.observe(rows(*[(ar.OK, d + 1, d) for d in reversed(range(D - 1))]), 3, 5.0, 5.0)
    assert ids(r["yaw"]) == set(range(D))


def test_self_id_is_new_on_the_first_call_only_and_the_state_sticks():
    o = orf.ObservabilityRef(D)
    o.set_window(*still([0, 1, 2]))
    r = o.observe(rows(), 0, 5.0, 5.0)
    assert ids(r["to_init"]) == {0} and ids(r["pos"]) == {0} and not r["solve_master"]
    r = o.observe(rows(), 0, 5.0, 5.0)
    assert ids(r["to_init"]) == set() and ids(r["pos"]) == {0}
    r = o.observe(rows((ar.OK, 0, 2)), 0, 5.0, 5.0)
    assert ids(r["to_init"]) == {2} and r["solve_master"]
    r = o.observe(rows((ar.DPOS, 0, 2)), 0, 5.0, 5.0)                   # the link is gone: pos, enable, master stay
    assert ids(r["yaw"]) == {0} and ids(r["pos"]) == {0, 2} and ids(r["enable"]) == {0, 2} and r["solve_master"]
    assert ids(r["to_init"]) == set()
    # the node set keeps every drone of every window, vo_available or not
    o.set_window(*window([(5, 0, 0, 0, 0)], [(0, 0, 0, 0)]))
    r = o.observe(rows(), 0, 5.0, 5.0)
    assert ids(r["nodes"]) == {0, 1, 2, 5}


def test_self_box_thresholds_are_strict_and_float():
    def motion(dx, dy, dz, xy=0.5, z=0.25, self_id=0):
        o = orf.ObservabilityRef(D)
        o.set_window(*window([(0, 0.0, 0.0, 0.0), (1, 0.0, 0.0, 0.0)], [(0, dx, dy, dz), (2, 0.0, 0.0, 0.0, 0)]))
        return o.observe(rows(), self_id, xy, z)

    assert not motion(0.5, 0.6, 0.3)["motion"]                          # x exactly at the threshold
    assert not motion(0.6, 0.5, 0.3)["motion"]
    assert not motion(0.6, 0.6, 0.25)["motion"]
    r = motion(0.5000001, 0.6, 0.2500001)
    assert r["motion"] and r["motion_new"] and r["solve_master"]
    assert ids(r["to_init"]) == {0, 1, 2} and ids(r["pos"]) == {0, 1, 2} and ids(r["enable"]) == {0, 1, 2}
    assert ids(r["yaw"]) == {0}                                         # the box gives pos, not yaw
    # 0.1 as a float is 0.10000000149: an extent between the two is not above it
    assert 0.1000000005 > 0.1 and not motion(0.1000000005, 0.2, 0.2, xy=0.1, z=0.1)["motion"]
    assert not motion(0.2, 0.2, 0.1000000005, xy=0.1, z=0.1)["motion"]
    assert motion(0.1000000020, 0.2, 0.1000000020, xy=0.1, z=0.1)["motion"]
    assert not motion(3.0, 3.0, 3.0, self_id=1)["motion"]                # another drone's box does not count


def test_motion_new_only_finds_drones_not_yet_positioned():
    o = orf.ObservabilityRef(D)
    moving = window([(0, 0.0, 0.0, 0.0), (1, 0.0, 0.0, 0.0)], [(0, 2.0, 2.0, 2.0), (1, 0.0, 0.0, 0.0)])
    o.set_window(*moving)
    r = o.observe(rows((ar.OK, 0, 1)), 0, 1.0, 1.0)
    assert r["motion"] and not r["motion_new"] and ids(r["to_init"]) == {0, 1}   # the closure positioned both first
    o.set_window(*window([(0, 0.0, 0.0, 0.0), (3, 0.0, 0.0, 0.0)], [(0, 2.0, 2.0, 2.0)]))
    r = o.observe(rows(), 0, 1.0, 1.0)
    assert r["motion"] and r["motion_new"] and ids(r["to_init"]) == {3} and ids(r["pos"]) == {0, 1, 3}
    r = o.observe(rows(), 0, 1.0, 1.0)
    assert r["motion"] and not r["motion_new"] and ids(r["to_init"]) == set()


def test_yaw_box_starts_at_plus_minus_1000():
    def yaw(frames):
        o = orf.ObservabilityRef(D)
        o.set_window(*window(*frames))
        return ids(o.observe(rows(), 0, 5.0, 5.0)["yaw"]) - {0}

    assert yaw([[(1, 0.0, 0.0, 0.0)], [(1, 1.0, 0.5, 0.0)]]) == set()            # exactly 1 m: not above it
    assert yaw([[(1, 0.0, 0.0, 0.0)], [(1, 0.0, 1.0 + 2 ** -52, 0.0)]]) == {1}
    assert yaw([[(1, 0.0, 0.0, 0.0)], [(1, 0.0, 0.0, 9.0)]]) == set()            # z does not count
    assert yaw([[(1, 0.5, 0.5, 0.0)]]) == set()                                  # one sample near the origin
    assert yaw([[(1, 5000.0, 0.0, 0.0)]]) == {1}                                 # xmin stays at +1000
    assert yaw([[(1, 0.0, -3000.0, 0.0)]]) == {1}                                # ymax stays at -1000
    assert yaw([[(1, 0.0, 0.0, 0.0)], [(1, 5.0, 5.0, 0.0, 0)]]) == set()         # not vo_available
    assert orf.bounding_box(window([(1, 0.0, 0.0, 0.0, 0)])[2], 1) == ([1000.0] * 3, [-1000.0] * 3)


def test_single_drone_solves_after_more_than_three_frames():
    for n_frames, want in ((3, False), (4, True)):
        o = orf.ObservabilityRef(D)
        o.set_window(*still([2], n_frames))
        assert o.observe(rows(), 2, 5.0, 5.0)["solve_master"] == want
    o = orf.ObservabilityRef(D)
    o.set_window(*still([0, 1], 6))                                     # two nodes: no single-drone rule
    assert not o.observe(rows(), 0, 5.0, 5.0)["solve_master"]
    o.set_window(*still([0], 6))                                        # drone 1 stays a node
    assert not o.observe(rows(), 0, 5.0, 5.0)["solve_master"]
