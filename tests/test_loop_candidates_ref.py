"""CPU: the keyframe-metadata oracle (tests/loop_candidates_ref.py) -- role routing of the candidates, the init-mode rule,
trajectory look-ups and the refusals of metas and stamps."""
import numpy as np

from oracle import pcm_ref as pr
import loop_candidates_ref as lc

SELF = 1
PRM = dict(inter_drone_init_frames=3, pos_covariance_per_meter=0.01, yaw_covariance_per_meter=0.003, loop_cov_pos=0.013,
           loop_cov_ang=2.5e-4)


def rec(drone, msg, nk=(5, 5, 5, 5)):
    return dict(drone_id=drone, msg_id=msg, n_dirs=4, n_kpts=list(nk))


def pose(x, yaw=0.0):
    return np.array([x, 0.5 * x, 0.0, np.cos(yaw / 2), 0.0, 0.0, np.sin(yaw / 2)])


def res(hit_id=-1, hit_drone=-1, swapped=0):
    return dict(accepted=int(hit_id >= 0), hit_id=hit_id, hit_drone_id=hit_drone, swapped=swapped)


def no_pairs():
    return np.zeros((lc.PAIR_DRONES, lc.PAIR_DRONES), np.int64)


def test_candidates_route_own_received_and_swapped_hits():
    s = lc.MetaStores(SELF, 64)
    own = [rec(SELF, 10), rec(SELF, 11, nk=(5, 0, 5, 5))]
    s.ingest(own[:1], lc.metas([(SELF, 10, 1000, pose(0.0))]))
    s.ingest(own[1:], lc.metas([(SELF, 11, 2000, pose(3.0, 0.3))]))
    remote = rec(2, 50)
    s.ingest([remote], lc.metas([(2, 50, 1500, pose(9.0))]))
    assert s.status == lc.OK and len(s.traj.stamps) == 2 and len(s.rows[0]) == 7 and len(s.rows[1]) == 4
    q_own = lc.metas([(SELF, 11, 2000, pose(3.0, 0.3))])[0]
    q_recv = lc.metas([(3, 70, 2500, pose(5.0))])[0]
    recs = [own[1], rec(3, 70), own[1], rec(3, 70)]
    ms = np.array([q_own, q_recv, q_own, q_recv])
    results = [res(2, SELF), res(5, SELF), res(lc.REMOTE_MAGIN_NUMBER + 3, 2, swapped=1), res()]
    cand, st = lc.candidates(s, recs, ms, results, no_pairs(), PRM)
    # own keyframe hitting own row 2 (frame 0): odometry from the hit (old, a) to the query (new, b)
    assert np.array_equal(cand[0]["pose_query"], pose(3.0, 0.3)) and np.array_equal(cand[0]["pose_hit"], pose(0.0))
    assert tuple(st[0]) == (2000, 1000) and cand[0]["reserved"] == 0 and cand[0]["init_mode"] == 0
    rel = pr.pose_mul(pr.pose_inv(pose(0.0)), pose(3.0, 0.3))
    assert cand[0]["odom_rel"].tobytes() == rel.tobytes()
    dl = abs(s.traj.length[1] - s.traj.length[0])
    assert np.array_equal(np.diag(cand[0]["odom_edge_cov"]), [dl * 0.01 + 0.013] * 3 + [dl * 0.003 + 2.5e-4] * 3)
    assert np.count_nonzero(cand[0]["odom_edge_cov"]) == 6
    # received keyframe hitting own row 5 (frame 1, the second keyframe's third row): no odometry, init mode
    assert np.array_equal(cand[1]["pose_hit"], pose(3.0, 0.3)) and tuple(st[1]) == (2500, 2000)
    assert cand[1]["init_mode"] == 1 and np.array_equal(cand[1]["odom_rel"], lc.IDENTITY) and not cand[1]["odom_edge_cov"].any()
    # own keyframe hitting remote row 3 (frame 0 of the remote store): swapped, cross-drone
    assert np.array_equal(cand[2]["pose_hit"], pose(9.0)) and tuple(st[2]) == (2000, 1500)
    assert cand[2]["reserved"] == 0 and np.array_equal(cand[2]["odom_rel"], lc.IDENTITY)
    # a miss: identity hit side, stamp 0, not marked
    assert np.array_equal(cand[3]["pose_hit"], lc.IDENTITY) and st[3]["stamp_hit_ns"] == 0 and cand[3]["reserved"] == 0


def test_init_mode_flips_at_exactly_inter_drone_init_frames():
    pairs = no_pairs()
    recs = [rec(2, 1), rec(SELF, 2), rec(300, 3), rec(2, 4)]
    for cnt in range(5):
        pairs[2, SELF] = cnt
        got = lc.init_modes(recs, 3, SELF, pairs, PRM["inter_drone_init_frames"])
        assert got.tolist() == [int(cnt < 3), 0, 1, 0]
    pairs[SELF, 2] = 99                                       # the rule reads [drone][self] only
    pairs[2, SELF] = 2
    assert lc.init_mode(2, SELF, pairs, 3)


def test_trajectory_lookups_at_and_between_samples():
    t = lc.Trajectory(8)
    for k, x in enumerate([0.0, 1.0, 3.0, 6.0]):
        assert t.append(100 * (k + 1), pose(x)) == lc.OK
    assert [t.nearest(v) for v in (0, 100, 149, 150, 151, 400, 10**9)] == [0, 0, 0, 0, 1, 3, 3]
    step = np.sqrt(1.0 + 0.25)
    assert t.length[1] == step and t.length[3] == (step + 2 * step) + 3 * step
    rel, dl, diag = t.relative(100, 400, 0.01, 0.003)
    assert rel.tobytes() == pr.pose_mul(pr.pose_inv(pose(0.0)), pose(6.0)).tobytes()
    assert dl == t.length[3] and diag == [dl * 0.01] * 3 + [dl * 0.003] * 3
    rel2, dl2, _ = t.relative(260, 149, 0.01, 0.003)        # between samples: nearest 300 and 100
    assert np.allclose(rel2, pr.pose_mul(pr.pose_inv(pose(3.0)), pose(0.0))) and dl2 == t.length[2]


def test_refused_metas_and_stamps():
    s = lc.MetaStores(SELF, 64)
    s.ingest([rec(SELF, 10), rec(2, 20)], lc.metas([(SELF, 10, 1000, pose(0.0)), (2, 21, 5, pose(1.0))]))
    assert s.status == lc.ERR_INVALID and s.frames[1][0] is None and s.frames[0][0] is not None
    s.ingest([rec(SELF, 11)], lc.metas([(SELF, 11, 1000, pose(1.0))]))      # stamp not after the last: meta kept
    assert s.status == lc.ERR_INVALID and len(s.traj.stamps) == 1 and s.frames[0][1] is not None
    s.ingest([rec(SELF, 12)], lc.metas([(SELF, 12, 1001, pose(1.0))]))
    assert s.status == lc.OK and len(s.traj.stamps) == 2
    s.ingest([rec(SELF, 13)])                                 # the plain ingest: no meta, status untouched
    assert s.frames[0][3] is None and s.status == lc.OK
    # an accepted candidate whose hit has no meta (or whose query meta mismatches its record) is marked
    q = lc.metas([(2, 20, 3000, pose(2.0))])[0]
    cand, _ = lc.candidates(s, [rec(2, 20)] * 2, np.array([q, q]), [res(12, SELF), res(0, SELF)], no_pairs(), PRM)
    assert cand["reserved"].tolist() == [1, 0]
    bad = lc.metas([(2, 99, 3000, pose(2.0))])[0]
    cand, st = lc.candidates(s, [rec(2, 20)], np.array([bad]), [res(0, SELF)], no_pairs(), PRM)
    assert cand["reserved"][0] == 1 and st["stamp_query_ns"][0] == 0
    # db_reset keeps the trajectory
    s.reset()
    assert len(s.traj.stamps) == 2 and s.frames == [[], []]
    tiny = lc.MetaStores(SELF, 1)
    tiny.traj.append(1, pose(0.0))
    tiny.reset()
    tiny.ingest([rec(SELF, 1)], lc.metas([(SELF, 1, 2, pose(0.0))]))
    assert tiny.status == lc.ERR_CAPACITY
