"""osb_anchor_data_association_dev and the predicated second run / observe: LocalizationDAInit on the device.  Flights
with 2-8 anonymous ids among 4-16 drones: the outcome and the renamed store against tests/da_init_ref.py (both forms),
the rows of the pass after it byte-identical to a handle fed the oracle's renamed detections, a handle whose store has
no anonymous row byte-identical to one without the setter, the predicated pass writing nothing when nothing is applied,
refusals and bounds, launches, no synchronisation, and the whole pre-init branch captured as one CUDA graph."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l
import da_init_ref as da
from test_da_init_ref import case

XY, Z = 1e6, 1e6                                 # no motion: the swarm is not initialised, has_node_not_inited holds
FRAMES = range(0, 40, 5)


def window(trajs, drones, frames=FRAMES):
    """one frame per odometry index in frames, holding every given drone that has odometry"""
    stamps, first, ents = [], [0], []
    for f in frames:
        stamps.append(int(f) * 100_000_000)
        for d in drones:
            s, p = trajs[d]
            if len(s) == 0:
                continue
            e = np.zeros(1, _l.WINDOW_ENTRY_DTYPE)
            e["drone_id"], e["vo_available"], e["block"] = d, 1, len(ents)
            e["stamp"], e["self_pose"] = s[f], p[f]
            ents.append(e)
        first.append(len(ents))
    return np.array(stamps, np.int64), np.array(first, np.int32), np.concatenate(ents)


def anchor(trajs, dets, max_drones, with_da=True, max_nodes=1 << 20):
    a = host.LoopAnchor(max_drones, 64, 512, 1024, 1.0, 0.0015, 0.0015)
    if with_da:
        a.set_data_association(3.345, 1000, max_nodes)
    for d, (s, p) in trajs.items():
        if len(s):
            a.push_odometry(d, s, p)
    if len(dets):
        a.add_measurements(dets)
    return a


def flight(n, n_anon, seed):
    """drone 0 without odometry (else it is every id's unchecked first success); self 1 and drones 2.. detect the
    others as anonymous targets"""
    rng = np.random.default_rng(seed)
    targets = rng.permutation(np.arange(2, n))[:n_anon]
    anon = []
    for j, b in enumerate(targets):
        for _ in range(int(rng.integers(1, 3))):
            a = int(rng.choice([d for d in [1] + targets.tolist() if d != b]))   # self or a drone found itself
            anon.append((a, int(b), 1000 + 11 * j, int(rng.integers(0, 40))))
    rng.shuffle(anon)
    trajs, kf, dets, _ = case(n, anon, seed=seed)
    trajs[0] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    return trajs, dets


def front(a, chain, win, self_id):
    a.set_window(*win)
    n = chain.run(a)
    chain.observe(a, n, self_id, XY, Z)
    return n


def rows(chain, n):
    torch.cuda.synchronize()
    chain.stream.synchronize()
    return chain.rows[:n * _l.ANCHOR_RESULT_DTYPE.itemsize].cpu().numpy().copy()


def obs_bytes(a):
    o = a.observability()
    return b"".join(np.asarray(o[k]).tobytes() for k in sorted(o))


@pytest.mark.gpu
@pytest.mark.parametrize("n,n_anon,seed", [(5, 3, 1), (4, 2, 1), (6, 4, 2), (10, 8, 5), (10, 8, 6), (12, 8, 4), (16, 8, 5)])
def test_flights_against_the_oracle(gpu, n, n_anon, seed):
    trajs, dets = flight(n, min(n_anon, n - 2), seed)
    win = window(trajs, range(n))
    a, c = anchor(trajs, dets, n), host.AnchoredChain(512)
    m = front(a, c, win, 1)
    pos1 = a.observability()["pos"]                                 # what the first observe set
    n2 = c.data_association(a, 1, XY, Z)
    applied, status, guess = a.data_association_result()
    want = da.da_vec(1, trajs, {}, dets, 3.345, max_drones=n)
    assert want == da.da_literal(1, trajs, {}, dets, 3.345)
    codes = {"ok": _l.OK, "invalid": _l.ERR_INVALID, "capacity": _l.ERR_CAPACITY}
    assert (applied, status, guess) == (want[0], codes[want[1]], want[2])
    assert applied or (n, seed) not in ((5, 1), (4, 1), (6, 2), (10, 5))   # these flights resolve
    got = rows(c, n2)
    # the same window through a handle fed the oracle's renamed store, without data association
    renamed = dets.copy()
    renamed["id_b"] = want[3]
    b, cb = anchor(trajs, renamed, n, with_da=not applied), host.AnchoredChain(512)
    m2 = front(b, cb, win, 1)
    assert m2 == n2
    assert np.array_equal(got, rows(cb, m2))
    r = got.view(_l.ANCHOR_RESULT_DTYPE)
    if applied:                                                     # every renamed row now finds its frames
        assert np.all(r["status"] == _l.ANCHOR_OK) and np.all(r["edge"]["id_b"] < n)
    else:                                                           # the anonymous rows stay NO_FRAME
        assert np.all(r["status"][renamed["id_b"] >= 1000] == _l.ANCHOR_NO_FRAME)
    # the record is the second observe's: ids_to_init leaves out what the first one set pos for (self at least)
    oa, ob = a.observability(), b.observability()
    for k in oa:
        want_k = ob[k] & ~pos1 if k == "to_init" and applied else ob[k]
        assert np.array_equal(oa[k], want_k), k
    for h in (a, b):
        h.close()


@pytest.mark.gpu
def test_no_anonymous_rows_change_nothing(gpu):
    trajs, dets = flight(6, 3, 7)
    named = dets.copy()
    named["id_b"] = np.where(named["id_b"] >= 1000, 2, named["id_b"])
    win = window(trajs, range(6))
    a, ca = anchor(trajs, named, 6), host.AnchoredChain(512)
    b, cb = anchor(trajs, named, 6, with_da=False), host.AnchoredChain(512)
    na, nb = front(a, ca, win, 1), front(b, cb, win, 1)
    before_rows, before_obs = rows(ca, na), obs_bytes(a)
    assert np.array_equal(before_rows, rows(cb, nb)) and before_obs == obs_bytes(b)
    n2 = ca.data_association(a, 1, XY, Z)               # the gate holds, but no id is anonymous: nothing applied
    assert a.data_association_result() == (False, _l.OK, {})
    assert n2 == na and np.array_equal(rows(ca, n2), before_rows) and obs_bytes(a) == before_obs
    for h in (a, b):
        h.close()


@pytest.mark.gpu
def test_refusals_and_bounds(gpu):
    trajs, dets = flight(6, 4, 8)
    win = window(trajs, range(6))
    a, c = anchor(trajs, dets, 6, max_nodes=1), host.AnchoredChain(512)
    n = front(a, c, win, 1)
    before, obs = rows(c, n), obs_bytes(a)
    assert c.data_association(a, 1, XY, Z) == n
    assert a.data_association_result() == (False, _l.ERR_CAPACITY, {})
    assert np.array_equal(rows(c, n), before) and obs_bytes(a) == obs
    a.close()
    # 33 anonymous ids
    anon = [(1, 2, 1000 + j, j % 40) for j in range(33)]
    trajs, _, dets, _ = case(3, anon)
    a, c = anchor(trajs, dets, 3), host.AnchoredChain(512)
    n = front(a, c, window(trajs, range(3)), 1)
    c.data_association(a, 1, XY, Z)
    assert a.data_association_result()[:2] == (False, _l.ERR_CAPACITY)
    # a leaf that reads a detector without an estimate (drone 0 guessed, verify()'s at())
    trajs, _, dets, _ = case(3, [(1, 0, 1001, 5)])
    a2, c2 = anchor(trajs, dets, 3), host.AnchoredChain(512)
    n = front(a2, c2, window(trajs, range(3)), 1)
    c2.data_association(a2, 1, XY, Z)
    assert da.da_vec(1, trajs, {}, dets, 3.345, max_drones=3)[1] == "invalid"
    assert a2.data_association_result()[:2] == (False, _l.ERR_INVALID)
    # refused at once: anonymous rows without the setter, loops with anonymous ids, no observe, a bad self_id
    b = anchor(trajs, dets[:0], 3, with_da=False)
    with pytest.raises(_l.OsbError):
        b.add_measurements(dets)
    with pytest.raises(_l.OsbError):
        b.data_association_dev(1, 0)
    loop = dets.copy()
    loop["type"] = _l.MEAS_LOOP
    with pytest.raises(_l.OsbError):
        a.add_measurements(loop)
    fresh = anchor(trajs, dets, 3)
    with pytest.raises(_l.OsbError):
        fresh.data_association_dev(1, 0)                            # no observe yet
    with pytest.raises(_l.OsbError):
        a.data_association_dev(3, 0)
    with pytest.raises(_l.OsbError):
        b.set_data_association(3.345, 2, 10)                        # anon_min below max_drones
    for h in (a, a2, b, fresh):
        h.close()


@pytest.mark.gpu
def test_launches_and_no_synchronisation(gpu):
    trajs, dets = flight(6, 4, 9)
    a, c = anchor(trajs, dets, 6), host.AnchoredChain(512)
    n = front(a, c, window(trajs, range(6)), 1)
    c.data_association(a, 1, XY, Z)                              # the first call acquires
    c.stream.synchronize()
    live = host.live_resources()
    torch.cuda.synchronize()
    with torch.cuda.stream(c.stream):
        torch.cuda._sleep(1_000_000_000)
    n0 = host.launch_count()
    c.data_association(a, 1, XY, Z)
    assert host.launch_count() - n0 == 1 + 1 + 3                    # DA, run_if, observe_if
    assert not c.stream.query()
    c.stream.synchronize()
    assert host.live_resources() == live
    a.close()


def with_drone0(win, pose=(0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0)):
    """the window with drone 0 (no odometry) in every frame: a node that never becomes enabled, so the gate holds"""
    stamps, first, ents = win
    out, f2 = [], [0]
    for f in range(len(stamps)):
        out.extend(ents[first[f]:first[f + 1]])
        e = np.zeros(1, _l.WINDOW_ENTRY_DTYPE)[0]
        e["drone_id"], e["vo_available"], e["stamp"], e["self_pose"] = 0, 1, stamps[f], pose
        out.append(e)
        f2.append(len(out))
    ents2 = np.array(out, _l.WINDOW_ENTRY_DTYPE)
    ents2["block"] = np.arange(len(ents2))
    return stamps, np.array(f2, np.int32), ents2


@pytest.mark.gpu
def test_capture_of_the_pre_init_branch(gpu):
    """append_dev -> run -> observe -> DA -> run_if -> observe_if captured once and replayed after new odometry, a new
    window and new anonymous detections appended on the device; every replay applies and is byte-identical to the
    same calls uncaptured"""
    n_dr, rounds, max_n = 4, 3, 8
    anon = [(1, b, 1000, k) for k in range(2 + 3 * rounds) for b in (2, 3)]
    trajs, _, pool, _ = case(n_dr, anon)
    trajs[0] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    ref, cap = [anchor({d: (s[:10], p[:10]) for d, (s, p) in trajs.items()}, pool[:0], n_dr) for _ in range(2)]
    cr, cc = host.AnchoredChain(512), host.AnchoredChain(512)
    bufs = {id(a): (torch.zeros(max_n * _l.MEASUREMENT_DTYPE.itemsize, dtype=torch.uint8, device="cuda"),
                    torch.zeros(1, dtype=torch.int32, device="cuda")) for a in (ref, cap)}

    def fill(a, k):
        """round k's rows: drones 2 and 3 detected by self under the fresh ids 2000 + 10 k and 2001 + 10 k"""
        rows_k = pool[4 * k:4 * k + 4].copy()
        rows_k["id"] = 50_000 + 10 * k + np.arange(4)
        rows_k["id_b"] = 2000 + 10 * k + (rows_k["id_b"] == 1000) * (np.arange(4) % 2)
        m, cnt = bufs[id(a)]
        m[:len(rows_k) * _l.MEASUREMENT_DTYPE.itemsize].copy_(torch.from_numpy(rows_k.view(np.uint8).copy()))
        cnt.fill_(len(rows_k))
        torch.cuda.synchronize()

    def step(a, c):
        m, cnt = bufs[id(a)]
        a.add_measurements_dev(m.data_ptr(), cnt.data_ptr(), max_n, 1e9, c.stream.cuda_stream)
        n = c.run(a)
        c.observe(a, n, 1, XY, Z)
        return c.data_association(a, 1, XY, Z)

    def win_of(k):
        return with_drone0(window(trajs, range(n_dr), range(0, 10 + 10 * k, 5)))

    for a, c in ((ref, cr), (cap, cc)):
        a.set_window(*win_of(0))
        fill(a, 0)
        step(a, c)                                                  # warm: every first call is behind
        c.stream.synchronize()
    assert ref.data_association_result()[:2] == (True, _l.OK)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=cc.stream, capture_error_mode="global"):
        step(cap, cc)
    for k in range(1, rounds):
        for a in (ref, cap):
            for d, (s, p) in trajs.items():
                if len(s):
                    a.push_odometry(d, s[10 * k:10 * k + 10], p[10 * k:10 * k + 10])
            a.set_window(*win_of(k))
            fill(a, k)
        step(ref, cr)
        cr.stream.synchronize()
        graph.replay()
        torch.cuda.synchronize()
        n = sum(ref.size())                                         # the rows both hold; the replayed appends are
                                                                    # counted on the device only
        got = ref.data_association_result()
        assert got[:2] == (True, _l.OK) and set(got[2]) == {2000 + 10 * k, 2001 + 10 * k}
        assert cap.data_association_result() == got
        assert np.array_equal(rows(cr, n), rows(cc, n))
        assert obs_bytes(ref) == obs_bytes(cap)
    for h in (ref, cap):
        h.close()


@pytest.mark.gpu
def test_keyframe_paths_of_an_applied_sync(gpu):
    """est_poses_t0 from the keyframe paths of an applied sync_dev: the search against both oracle forms with the same
    paths, and a store without anonymous rows byte-identical to a handle without the setter through sync_dev"""
    n_dr = 6
    targets = [2, 3, 4, 5]
    named = [(1, 2, 2, 3), (2, 3, 3, 4), (3, 4, 4, 6), (4, 5, 5, 8)]     # detections that tie the swarm together
    anon = named + [(1 if b == 2 else b - 1, b, 1000 + 7 * j, 12 + j) for j, b in enumerate(targets)]
    trajs, _, dets, world = case(n_dr, anon, seed=3)
    trajs[0] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    win = window(trajs, range(n_dr))

    def synced(store, with_da):
        a, c = anchor(trajs, store, n_dr, with_da=with_da), host.AnchoredChain(512)
        n = front(a, c, win, 1)
        ents = win[2]
        init = np.zeros((len(ents), 4))
        for e, ent in enumerate(ents):
            d = int(ent["drone_id"])
            k = int(np.searchsorted(trajs[d][0], ent["stamp"]))
            wp = da.pr.pose_mul(world[d], trajs[d][1][k])
            init[e, :3] = wp[:3]
            init[e, 3] = 2.0 * np.arctan2(wp[6], wp[3])
        solver = host.PoseGraphSolver(4096, 32768)
        solver.graph_clear()
        solver.graph_add_nodes(init, (np.arange(len(init)) == 0).astype(np.uint8))
        ft, ia, ib, pay = [], [], [], []            # OSB_FACTOR_RELPOSE (1) between each drone's consecutive blocks, exact
        for d in range(1, n_dr):
            blk = np.nonzero(ents["drone_id"] == d)[0]
            for i, j in zip(blk[:-1], blk[1:]):
                cy, sy = np.cos(init[i, 3]), np.sin(init[i, 3])
                dx, dy = init[j, 0] - init[i, 0], init[j, 1] - init[i, 1]
                p = np.zeros(_l.PAYLOAD_LEN)
                p[:4] = [cy * dx + sy * dy, -sy * dx + cy * dy, init[j, 2] - init[i, 2],
                         np.arctan2(np.sin(init[j, 3] - init[i, 3]), np.cos(init[j, 3] - init[i, 3]))]
                p[4:20] = np.eye(4).ravel()
                ft.append(1); ia.append(i); ib.append(j); pay.append(p)
        solver.graph_add_factors(ft, ia, ib, np.array(pay), np.zeros(len(ft), np.uint8))
        c.compact(n, keep=False)
        c.mask = torch.zeros(len(init), dtype=torch.uint8, device="cuda")
        c.yaw = torch.zeros(len(init), dtype=torch.float64, device="cuda")
        c.stream.wait_stream(torch.cuda.current_stream())
        c.init_solve(solver, 4096, 1, 7, 30, np.inf)
        a.sync_dev(solver, c.stream.cuda_stream, 1, np.inf, 30, True, False)
        c.stream.synchronize()
        assert a.sync_result() == (True, _l.OK)
        return a, c, solver

    win0 = with_drone0(win)                     # the named rows enable every drone with odometry; drone 0 keeps the gate
    a, c, solver = synced(dets, True)
    kf = {d: p for d in range(n_dr) if (p := a.paths(d)) is not None}
    assert sorted(kf) == [1, 2, 3, 4, 5]
    front(a, c, win0, 1)
    det_rows = dets[dets["type"] != _l.MEAS_LOOP]
    c.data_association(a, 1, XY, Z)
    want = da.da_vec(1, trajs, kf, det_rows, 3.345, max_drones=n_dr)
    assert want == da.da_literal(1, trajs, kf, det_rows, 3.345)
    assert want[:3] == (True, "ok", {1000: 2, 1007: 3, 1014: 4, 1021: 5})   # the gates check against the paths
    assert a.data_association_result() == (want[0], _l.OK, want[2])
    # a wrong relative pose now fails the gate against the path's estimate of its drone: the search changes
    bad = dets.copy()
    bad[len(named) + 1]["relative_pose"][:3] += 3.0
    b, cb, sb = synced(bad, True)
    front(b, cb, win0, 1)
    cb.data_association(b, 1, XY, Z)
    bad_rows = bad[bad["type"] != _l.MEAS_LOOP]
    want_b = da.da_vec(1, trajs, kf, bad_rows, 3.345, max_drones=n_dr)
    assert want_b == da.da_literal(1, trajs, kf, bad_rows, 3.345) and want_b[:2] != want[:2]
    assert b.data_association_result() == (want_b[0], {"ok": _l.OK, "invalid": _l.ERR_INVALID}[want_b[1]], want_b[2])
    # no anonymous row: with and without the setter, byte for byte through a second sync
    plain = dets[:len(named)].copy()
    outs = []
    for with_da in (True, False):
        h, ch, sh = synced(plain, with_da)
        m = front(h, ch, win, 1)
        if with_da:
            assert ch.data_association(h, 1, XY, Z) == m
            assert h.data_association_result() == (False, _l.OK, {})
        ch.compact(m, keep=False)
        ch.init_solve(sh, 4096, 1, 7, 30, np.inf)
        h.sync_dev(sh, ch.stream.cuda_stream, 1, np.inf, 30, True, True)
        outs.append((rows(ch, m).tobytes(), obs_bytes(h), h.sync_result(),
                     [(p[0].tobytes(), p[1].tobytes()) if (p := h.paths(d, full)) is not None else None
                      for d in range(n_dr) for full in (False, True)]))
        for x in (h, sh):
            x.close()
    assert outs[0] == outs[1]
    for x in (a, solver, b, sb):
        x.close()


@pytest.mark.gpu
def test_the_double_observe_keeps_motion_new(gpu):
    """observe_dev_if after an observe that raised motion_new: the record is the reference's second
    estimate_observability with motion_new of either call; a word of 0 leaves every byte"""
    trajs, dets = flight(5, 3, 1)
    win = window(trajs, range(5))
    xy, z = 0.01, -1.0                                              # self's box passes: motion, motion_new
    a, c = anchor(trajs, dets, 5), host.AnchoredChain(512)
    b, cb = anchor(trajs, dets, 5), host.AnchoredChain(512)
    for h, ch in ((a, c), (b, cb)):
        h.set_window(*win)
    n = c.run(a)
    c.observe(a, n, 1, xy, z)
    first = a.observability()
    assert first["motion_new"] and first["motion"]
    zero = torch.zeros(1, dtype=torch.int32, device="cuda")
    one = torch.ones(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    before = obs_bytes(a)
    a.observe_dev_if(c.rows.data_ptr(), n, zero.data_ptr(), c.stream.cuda_stream, 1, xy, z)
    c.stream.synchronize()
    assert obs_bytes(a) == before
    a.observe_dev_if(c.rows.data_ptr(), n, one.data_ptr(), c.stream.cuda_stream, 1, xy, z)
    # the reference's two calls, on the twin: the record of the second, motion_new of the first kept by the caller
    nb = cb.run(b)
    cb.observe(b, nb, 1, xy, z)
    cb.observe(b, nb, 1, xy, z)
    second = b.observability()
    assert not second["motion_new"]
    got = a.observability()
    for k in second:
        want = (first[k] or second[k]) if k == "motion_new" else second[k]
        assert np.array_equal(got[k], want), k
    assert np.array_equal(rows(c, n), rows(cb, nb))
    for h in (a, b):
        h.close()


@pytest.mark.gpu
@pytest.mark.parametrize("redundant", [True, False])
def test_loop_map_and_pcm_in_the_reference_order(gpu, redundant):
    """loops and named detections, plus anonymous detections of the same pairs that the search renames: the branch with
    its predicated pass and the loop map and PCM after each observe ends in the state of the reference's order (the
    second pass only when applied), decided on the host; with nothing applied, the second pair changes nothing"""
    from backend_harness import THRES
    n_dr = 5
    anon = [(1, 2, 2, 4), (1, 2, 1000, 6), (1, 2, 2, 8), (2, 3, 3, 5), (2, 3, 1007, 9), (3, 4, 4, 7), (1, 4, 1014, 11),
            (2, 3, 3, 13), (1, 2, 1000, 15)]
    trajs, _, dets, _ = case(n_dr, anon, seed=4)
    trajs[0] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    loops = dets[[0, 3, 5]].copy()                                  # loops of the same pairs
    loops["type"] = _l.MEAS_LOOP
    loops["id"] = [7, 8, 9]
    for r in loops:
        for side, d, t in (("self_pose_a", r["id_a"], r["stamp_a"]), ("self_pose_b", r["id_b"], r["stamp_b"])):
            r[side] = trajs[d][1][int(np.searchsorted(trajs[d][0], t))]
    store = np.concatenate([loops, dets])
    win = with_drone0(window(trajs, range(n_dr)))   # drone 0 never enabled: the gate holds on every solve

    def handle():
        a, c = anchor(trajs, store, n_dr), host.AnchoredChain(512)
        pcm = host.PcmState(1, redundant, THRES, 0.0015, 0.0015, max_pairs=16, pair_capacity=64)
        return a, c, pcm

    def state(a, c, pcm, n):
        m = a.loop_map()
        pairs = [(x, y, pcm.inliers(x, y), pcm.pair(x, y)) for x in range(n_dr) for y in range(x + 1, n_dr)]
        pairs = [(x, y, None if s is None else s.tobytes(), p[0].tobytes(), p[1].tobytes(), np.asarray(p[2]).tobytes())
                 for x, y, s, p in pairs]
        with torch.cuda.stream(c.stream):
            keep = c.keep[:n].cpu().numpy().tobytes()
        return m["records"].tobytes(), m["pair_min"].tobytes(), pairs, keep, rows(c, n).tobytes()

    def first_pass(a, c, pcm):
        n = front(a, c, win, 1)
        c.record_loops(a, n)
        c.reject(pcm, n)
        return n

    a, c, pa = handle()                                             # the branch as captured: launches fixed
    first_pass(a, c, pa)
    n = c.data_association(a, 1, XY, Z)
    c.record_loops(a, n)
    c.reject(pa, n)
    applied = a.data_association_result()[0]
    assert applied
    b, cb, pb = handle()                                            # the reference's order, decided on the host
    first_pass(b, cb, pb)
    b.data_association_dev(1, cb.stream.cuda_stream)
    assert b.data_association_result()[0]
    nb = first_pass(b, cb, pb)
    assert state(a, c, pa, n) == state(b, cb, pb, nb)
    # nothing applied (every anonymous id already renamed): the second pair of calls leaves every byte
    a2, c2, p2 = a, c, pa
    m = first_pass(a2, c2, p2)
    before = state(a2, c2, p2, m)
    assert c2.data_association(a2, 1, XY, Z) == m
    assert a2.data_association_result()[0] is False
    c2.record_loops(a2, m)
    c2.reject(p2, m)
    assert state(a2, c2, p2, m) == before
    for h in (a, pa, b, pb):
        h.close()
