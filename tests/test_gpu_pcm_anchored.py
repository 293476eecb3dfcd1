"""GPU: the solve's chain from re-anchoring to factor rows on the device -- osb_pcm_state_reject_anchored reading
osb_anchor_run_dev's rows in place and osb_anchor_compact_factors_dev -- against the host sequence it replaces
(osb_anchor_run, the OK rows through osb_pcm_state_reject, the keep mask scattered back, add_anchored_factors' rows):
keep masks, factor rows and every pair's state byte-identical, over solve rounds, mixed with the host calls, across the
clique kernel's shared-memory bound, at capacity, under stream capture."""
import ctypes as C

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l, synth
from oracle.pcm_state_ref import PcmStateRef
from backend_harness import THRES, make_anchor, pcm_state
from oracle import pcm_ref as pr
import pcm_edges_ref as R

pytestmark = pytest.mark.gpu
DRONES = 5
PAIRS = [(a, b) for a in range(DRONES + 2) for b in range(DRONES + 2) if a <= b]
ROW = _l.ANCHOR_RESULT_DTYPE.itemsize


def outliers(meas, frac, seed):
    """pcm_edges-style gross errors on a fraction of the measurements' relative poses"""
    rng = np.random.default_rng(seed)
    for i in np.flatnonzero(rng.uniform(size=len(meas)) < frac):
        rel = meas[i]["relative_pose"]
        rel[:3] += rng.uniform(-3, 3, 3)
        q = synth._quat_from_rotvec(rng.uniform(-0.8, 0.8, 3))
        rel[3:] = synth._PoseAlgebra.pose_mul(np.r_[0, 0, 0, rel[3:]], np.r_[0, 0, 0, q])[3:]
        rel[3:] /= np.linalg.norm(rel[3:])
    return meas


def solve_rounds(seed=0, rounds=4):
    """The inputs of successive solves: per round (new measurements, window).  Every round adds measurements, one of them
    re-submitting an earlier id with other values, and slides the window by two frames, so earlier ids re-anchor to other
    values too; drone 2 is not yaw-observable (skip rows), drone DRONES has no odometry, old and far measurements are not OK."""
    g = synth.anchor_swarm(DRONES, 40, 60 * rounds, seed=seed)
    meas = outliers(g["meas"], 0.25, seed + 1)
    stamps, first, entries = g["window"]
    frames = [(int(stamps[f]), entries[first[f]:first[f + 1]].copy()) for f in range(len(stamps))]
    out = []
    for r in range(rounds):
        new = meas[60 * r:60 * (r + 1)].copy()
        if r > 0:
            again = meas[60 * (r - 1):60 * r][meas[60 * (r - 1):60 * r]["type"] == _l.MEAS_LOOP][:1].copy()
            again["relative_pose"][:, :3] += 0.05
            new = np.concatenate([new, again])
        frames = frames[2:]
        win = (np.array([f[0] for f in frames], np.int64), np.cumsum([0] + [len(f[1]) for f in frames]).astype(np.int32),
               np.concatenate([f[1] for f in frames]))
        out.append((new, win))
    return g, out


def same_state(a, b, pairs=PAIRS):
    for p in pairs:
        for x, y in zip(a.pair(*p), b.pair(*p)):
            assert np.array_equal(x, y), p
        ia, ib = a.inliers(*p), b.inliers(*p)
        assert (ia is None) == (ib is None) and (ia is None or np.array_equal(ia, ib)), p


def ref_edges(rows):
    e = rows["edge"]
    return [dict(id_a=int(x["id_a"]), id_b=int(x["id_b"]), rel=x["rel_pose"], cov=x["cov"], odom_a=x["odom_a"],
                 odom_b=x["odom_b"], len_a=float(x["len_a"]), len_b=float(x["len_b"])) for x in e]


@pytest.mark.parametrize("redundant", [True, False])
def test_solve_rounds_match_the_host_sequence(gpu, redundant):
    g, rounds = solve_rounds(seed=3)
    a = make_anchor(g, 4096, 4096, traj_margin=8)
    for d, (s, p) in g["trajs"].items():
        a.push_odometry(d, s, p)
    yaw = np.ones(g["max_drones"], np.uint8)
    yaw[2] = 0
    ha, hb = (pcm_state(g, len(PAIRS), 512, 0, redundant) for _ in range(2))
    ref = PcmStateRef(0, redundant, THRES, g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"])
    chain = host.AnchoredChain(4096)
    seen_status, set_on = set(), {}
    for r, (new, win) in enumerate(rounds):
        a.add_measurements(new)
        a.set_window(*win)
        n = chain.run(a, yaw)
        chain.stream.synchronize()
        rows = np.frombuffer(chain.rows[:n * ROW].cpu().numpy().tobytes(), _l.ANCHOR_RESULT_DTYPE)
        keep_a = host.anchored_keep(ha, rows)
        ok = rows["status"] == _l.ANCHOR_OK
        assert np.array_equal(keep_a[ok], ref.reject(ref_edges(rows[ok]), rows["id"][ok]))
        chain.reject(hb, n)
        chain.compact(n)
        fb = chain.factors.on_host(chain.stream).values()
        assert chain.keep_on_host(n).tobytes() == keep_a.tobytes()
        fa = host.anchored_factor_rows(rows, keep_a)
        assert len(fa[0]) > 0 and all(x.tobytes() == y.tobytes() for x, y in zip(fa, fb))
        same_state(ha, hb)
        for key, p in ref.pairs.items():                             # correlated covariances: against float64
            smd, bnd = R.bound_matrix(p["edges"], ref.pos, ref.ang)
            fin = np.isfinite(smd)
            assert np.all(np.abs(smd[fin] - THRES) > 2 * bnd[fin]), "a pair within the bound of the threshold"
            _, adj_d, clique_d = hb.pair(*key)
            radj, _ = pr.consistency_matrix_batched(p["edges"], THRES, ref.pos, ref.ang)
            assert np.array_equal(adj_d, radj) and np.array_equal(adj_d, p["adj"])
            assert clique_d.tolist() == p["clique"]
        if r == 1:                                                   # other drones' sets, replaced when their pair grows
            for p in PAIRS:
                if 0 not in p:
                    set_on[p] = hb.pair(*p)[0].size
                    for h in (ha, hb, ref):
                        h.set_inliers(*p, rows["id"][ok][:2])
        seen_status |= set(rows["status"].tolist())
        ids, counts = np.unique(rows["id"], return_counts=True)
        assert r == 0 or counts.max() > 1                            # a re-submitted id
        assert (rows["skip"][ok] == 1).any()
    assert ref.min_margin > 1e-6, "test data has a pair on the threshold"
    assert {_l.ANCHOR_OK, _l.ANCHOR_BEFORE_WINDOW, _l.ANCHOR_NO_TRAJECTORY} <= seen_status
    if redundant:
        assert any(hb.pair(*p)[0].size > n0 for p, n0 in set_on.items())
    else:                                                            # unrouted pairs stay unstored, keep their set
        assert all(hb.pair(*p)[0].size == 0 and hb.inliers(*p) is not None for p in set_on)
    for h in (a, ha, hb):
        h.close()


def test_host_and_anchored_calls_mix_on_one_handle(gpu):
    g, rounds = solve_rounds(seed=5, rounds=5)
    a = make_anchor(g, 4096, 4096, traj_margin=8)
    for d, (s, p) in g["trajs"].items():
        a.push_odometry(d, s, p)
    hh, hm = (pcm_state(g, len(PAIRS), 512, 1) for _ in range(2))
    chain = host.AnchoredChain(4096)
    for r, (new, win) in enumerate(rounds):
        a.add_measurements(new)
        a.set_window(*win)
        rows = a.run()
        chain.upload(rows)
        keep_h = host.anchored_keep(hh, rows)
        if r % 2 == 0:
            chain.reject(hm, len(rows))
            keep_m = chain.keep_on_host(len(rows))
        else:
            keep_m = host.anchored_keep(hm, rows)
        assert keep_m.tobytes() == keep_h.tobytes(), r
        ok_ids = rows["id"][rows["status"] == _l.ANCHOR_OK]
        for h in (hh, hm):                                           # other drones' sets between the calls
            h.set_inliers(2, 3, ok_ids[r:r + 3])
            h.set_inliers(0, 4, np.r_[ok_ids[:5], np.arange(600) + (9 << 40)])   # larger than pair_capacity = 512
        if r in (1, 2):
            same_state(hh, hm)
    same_state(hh, hm)
    for h in (a, hh, hm):
        h.close()


def pcm_rows(edges, ids):
    """osb_anchor_result rows carrying the given edges and ids, status OK"""
    rows = np.zeros(len(ids), _l.ANCHOR_RESULT_DTYPE)
    rows["id"] = ids
    rows["status"] = _l.ANCHOR_OK
    rows["skip"] = 1
    rows["edge"] = host.loop_edges(edges).view(_l.LOOP_EDGE_DTYPE).reshape(len(ids))
    return rows


def stateless(edges):
    clique, adj, _ = host.pcm_outlier_rejection(edges, THRES, 1e-4, 1e-5, want_matrices=True)
    return clique, adj


def test_sizes_across_the_shared_memory_bound_and_to_capacity(gpu):
    """in one anchored call: a pair growing across n = 1280 (the clique leaves shared memory), a pair filled to 4096 and
    a pair gaining a few loops -- each equal to osb_pcm on its whole list"""
    big = synth.pcm_edges(4096, 0.4, 21, id_a=1, id_b=2)
    mid = synth.pcm_edges(1300, 0.4, 22, id_a=1, id_b=3)
    small = synth.pcm_edges(5, 0.2, 23, id_a=3, id_b=3)
    idb = np.arange(4096, dtype=np.int64) + (5 << 32)
    idm = np.arange(1300, dtype=np.int64) + (6 << 32)
    ids_s = np.arange(5, dtype=np.int64) + (7 << 32)
    st = host.PcmState(1, True, THRES, 1e-4, 1e-5, max_pairs=3, pair_capacity=4096)
    chain = host.AnchoredChain(4096 + 1300 + 5)
    first = pcm_rows(big[:3000] + mid[:1270] + small[:2], np.concatenate([idb[:3000], idm[:1270], ids_s[:2]]))
    chain.upload(first)
    chain.reject(st, len(first))
    rows = pcm_rows(big + mid[:1290] + small, np.concatenate([idb, idm[:1290], ids_s]))
    chain.upload(rows)
    chain.reject(st, len(rows))
    keep = chain.keep_on_host(len(rows))
    for (a, b), edges in (((1, 2), big), ((1, 3), mid[:1290]), ((3, 3), small)):
        ids, adj, clique = st.pair(a, b)
        rclique, radj = stateless(edges)
        assert len(ids) == len(edges) and np.array_equal(adj, radj) and np.array_equal(clique, rclique), (a, b)
        assert np.array_equal(np.sort(st.inliers(a, b)), np.unique(ids[clique]))
    good = np.concatenate([st.inliers(1, 2), st.inliers(1, 3), st.inliers(3, 3)])
    assert np.array_equal(keep.astype(bool), np.isin(rows["id"], good))
    st.close()


def test_capacity_is_refused_on_the_device_and_changes_nothing(gpu):
    e12 = synth.pcm_edges(70, 0.3, 31, id_a=1, id_b=2)
    e13 = synth.pcm_edges(20, 0.3, 32, id_a=1, id_b=3)
    i12 = np.arange(70, dtype=np.int64) + (3 << 32)
    i13 = np.arange(20, dtype=np.int64) + (4 << 32)
    st = host.PcmState(1, True, THRES, 1e-4, 1e-5, max_pairs=2, pair_capacity=64)
    chain = host.AnchoredChain(256)
    chain.upload(pcm_rows(e12[:60] + e13[:10], np.concatenate([i12[:60], i13[:10]])))
    chain.reject(st, 70)
    assert st.status() == _l.OK
    before = [st.pair(*p) for p in [(1, 2), (1, 3)]]
    good = [st.inliers(*p) for p in [(1, 2), (1, 3)]]
    for edges, ids in ((e12[:65] + e13[:10], np.concatenate([i12[:65], i13[:10]])),        # 65 loops in (1, 2)
                       (e12[:60] + synth.pcm_edges(1, 0.0, 33, id_a=2, id_b=4), np.r_[i12[:60], 9 << 32])):  # a third pair
        chain.keep.fill_(0xAB)
        chain.upload(pcm_rows(edges, ids))
        chain.reject(st, len(ids))
        assert (chain.keep_on_host(len(chain.keep)) == 0xAB).all()       # not written
        assert st.status() == _l.ERR_CAPACITY
        with pytest.raises(_l.OsbError) as e:                        # the next host-side call reports it once
            st.inliers(1, 2)
        assert e.value.status == _l.ERR_CAPACITY
        for p, b, g in zip([(1, 2), (1, 3)], before, good):
            assert all(np.array_equal(x, y) for x, y in zip(st.pair(*p), b)) and np.array_equal(st.inliers(*p), g)
    rows = pcm_rows(e12[:64] + e13, np.concatenate([i12[:64], i13]))   # the next valid call succeeds
    chain.upload(rows)
    chain.reject(st, len(rows))
    assert st.status() == _l.OK
    ids, adj, clique = st.pair(1, 3)
    rclique, radj = stateless(e13)
    assert np.array_equal(adj, radj) and np.array_equal(clique, rclique) and st.pair(1, 2)[0].size == 64
    st.close()


def test_capturable_constant_launches_and_resources(gpu):
    live0 = host.live_resources()
    g, rounds = solve_rounds(seed=7, rounds=3)
    a = make_anchor(g, 4096, 4096, traj_margin=8)
    for d, (s, p) in g["trajs"].items():
        a.push_odometry(d, s, p)
    st, ref = (pcm_state(g, len(PAIRS), 512) for _ in range(2))
    chain = host.AnchoredChain(4096)
    launches, live = [], None
    for r, (new, win) in enumerate(rounds[:2]):
        a.add_measurements(new)
        a.set_window(*win)
        host.anchored_keep(ref, a.run())
        n = chain.run(a)
        live = host.live_resources()
        n0 = host.launch_count()
        chain.reject(st, n)
        launches.append(host.launch_count() - n0)
        n0 = host.launch_count()
        chain.compact(n)
        assert host.launch_count() - n0 == 1
        assert st.status() == _l.OK
        assert r == 0 or host.live_resources() == live              # nothing acquired after the first call
    # a steady call (nothing new): no pair changes, other n
    live = host.live_resources()
    n0 = host.launch_count()
    chain.reject(st, n - 7)
    launches.append(host.launch_count() - n0)
    assert len(set(launches)) == 1 and launches[0] > 0, launches
    assert st.status() == _l.OK and host.live_resources() == live
    # the chain of a solve under stream capture (global mode): a synchronisation or an allocation would fail the capture
    new, win = rounds[2]
    a.add_measurements(new)
    a.set_window(*win)
    rows_now = a.run()
    keep_ref = host.anchored_keep(ref, rows_now)
    graph = torch.cuda.CUDAGraph()
    live = host.live_resources()
    with torch.cuda.graph(graph, stream=chain.stream, capture_error_mode="global"):
        n = chain.run(a)
        chain.reject(st, n)
        chain.compact(n)
    assert host.live_resources() == live
    graph.replay()
    chain.stream.synchronize()
    torch.cuda.synchronize()
    assert chain.keep_on_host(n).tobytes() == keep_ref.tobytes()
    fa = host.anchored_factor_rows(rows_now, keep_ref)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(fa, chain.factors.on_host(chain.stream).values()))
    same_state(ref, st)
    del graph
    for h in (st, ref, a):
        h.close()
    assert host.live_resources() == live0


def test_argument_errors(gpu):
    L = _l.load()
    st = host.PcmState(1, True, THRES, 1e-4, 1e-5, max_pairs=2, pair_capacity=16)
    buf = torch.zeros(ROW, dtype=torch.uint8, device="cuda")
    keep = torch.zeros(1, dtype=torch.uint8, device="cuda")
    p, k = C.c_void_p(buf.data_ptr()), C.c_void_p(keep.data_ptr())
    n0 = host.launch_count()
    assert L.osb_pcm_state_reject_anchored(None, p, 1, k, None) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject_anchored(st._h, p, -1, k, None) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject_anchored(st._h, None, 1, k, None) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject_anchored(st._h, p, 1, None, None) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject_anchored(st._h, None, 0, None, None) == _l.OK
    assert L.osb_pcm_state_status(st._h, None) == _l.ERR_INVALID
    assert host.launch_count() == n0 and st.status() == _l.OK
    assert L.osb_anchor_compact_factors_dev(p, -1, None, p, p, p, p, p, k, None) == _l.ERR_INVALID
    assert L.osb_anchor_compact_factors_dev(p, 1, None, None, p, p, p, p, k, None) == _l.ERR_INVALID
    st.close()
