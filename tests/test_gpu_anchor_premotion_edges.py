"""The pre-motion branch's kernels at the sizes they are built for: the loop map (record_claim_kernel /
record_write_kernel) past one pass of its grid, with duplicates across CTAs and passes, ids chosen against its hash, a
full store and an overflow; init_by_loops_kernel at 256 drones with more than 256 window entries, a shared block, yaws
near +-pi and both id2 sources; data_association_kernel with detectors and candidates in every 64-bit word, more than
256 detections, 32 and 33 ids, the exact acceptance threshold, the budget boundary, and the time a search takes per DFS
call.  Every device result is checked against tests/init_by_loops_ref.py and tests/da_init_ref.py, and every scenario
asserts that it reached the pass, word, wrap or boundary it is there for.  tests/test_premotion_ref_edges.py pins the
oracle forms to each other at the same shapes."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l
import da_init_ref as da
import init_by_loops_ref as ib
from test_gpu_anchor_data_association import window
from test_da_init_ref import case
from test_premotion_ref_edges import (BAD_COV, DRONES, I64_MAX, SELF, TO_INIT, book_view, budget_scene, close_yaw,
                                      da_scene, device_order, exact_scene, home, ibl_scene, loop_rows, scale_rows,
                                      special_ids, table_size, unshared, worst_gates, worst_scene)

ROW = _l.ANCHOR_RESULT_DTYPE.itemsize
XY, Z = 1e6, 1e6                                   # no motion: has_node_not_inited holds, to_init comes from the loops
BUDGETS = (8, 64)                                  # the worst case's search budgets timed here (64: about 3 s)
CODES = {"ok": _l.OK, "invalid": _l.ERR_INVALID, "capacity": _l.ERR_CAPACITY}


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def upload(rows):
    t = torch.from_numpy(rows.view(np.uint8).copy()).cuda()
    torch.cuda.synchronize()
    return t


def record(a, t, lo, hi, stream):
    a.record_loops_dev(t.data_ptr() + lo * ROW, hi - lo, stream.cuda_stream)


# ---- 1. the loop map --------------------------------------------------------------------------------------------------
@pytest.mark.gpu
def test_loop_map_past_one_grid_pass_against_both_forms(gpu):
    """a first call of more rows than one pass of record_*_kernel's grid: every special id first in the first CTA and
    again, with other values, on the second pass; then a call of more rows and one of re-sent ids"""
    D, max_meas = 256, 4096
    H = table_size(max_meas)
    n1 = 4 * sms() * 256 + 4_000
    grid_rows = min(-(-n1 // 256), 4 * sms()) * 256                 # record_loops_dev's grid for n1 rows, in rows
    assert n1 > grid_rows                                           # the first call takes two passes
    rows = np.concatenate([scale_rows(n1, H, 1), scale_rows(8_000, H, 2, n_ids=500)])
    spec = special_ids(H)
    for i in spec:                                                  # in the first call: once in the first CTA, once
        at = np.nonzero(rows["id"][:n1] == i)[0]                    # on the second pass, with other values
        assert at[0] < 256 and at[-1] >= grid_rows and rows["stamp_a"][at[0]] != rows["stamp_a"][at[-1]], i
    assert [home(i, H) for i in spec[-4:]] == [H - 1] * 4           # their probes wrap past slot H - 1
    a = host.LoopAnchor(D, 8, max_meas, 64, 1.0, 0.0015, 0.0015)
    st = torch.cuda.Stream()
    t = upload(rows)
    book, vec = ib.LoopBook(200, True), ib.LoopMapVec(D, _l.LOOP_RECORD_DTYPE)
    for lo, hi in ((0, n1), (n1, len(rows))):
        record(a, t, lo, hi, st)
        book.record(rows[lo:hi])
        vec.record_vec(rows[lo:hi])
    resent = loop_rows(vec.recs["id"][::3], 128, 255, 9)            # recorded ids again, other pair and values
    t2 = upload(resent)
    record(a, t2, 0, len(resent), st)
    book.record(resent)
    vec.record_vec(resent)
    st.synchronize()
    m = a.loop_map()
    assert m["records"].tobytes() == vec.recs.tobytes()
    assert np.array_equal(m["pair_min"], vec.pair_min)
    recs, pair = book_view(book, D)
    assert recs.tobytes() == m["records"].tobytes() and np.array_equal(pair, m["pair_min"])
    r = m["records"]
    for i in spec:                                                  # the first call's lowest row wrote the record
        k = int(np.nonzero(rows["id"] == i)[0][0])
        assert r["stamp_a"][np.searchsorted(r["id"], i)] == rows["stamp_a"][k]
    assert len(r) < max_meas
    assert m["pair_min"].min() == np.iinfo(np.int64).min            # INT64_MIN is a pair's minimum: the sign flip holds
    a.close()


@pytest.mark.gpu
def test_loop_map_divergences(gpu):
    """INT64_MAX is recorded but is no pair's loop; a recorded id on another pair changes no pair (DESIGN.md section 5)"""
    a = host.LoopAnchor(256, 8, 64, 64, 1.0, 0.0015, 0.0015)
    st = torch.cuda.Stream()
    rows = np.concatenate([loop_rows([I64_MAX], 64, 200, 3), loop_rows([77], 63, 64, 4)])
    record(a, upload(rows), 0, 2, st)
    record(a, upload(loop_rows([77], 128, 255, 5)), 0, 1, st)
    st.synchronize()
    m = a.loop_map()
    assert m["records"]["id"].tolist() == [77, I64_MAX]
    assert m["records"]["id_a"].tolist() == [63, 64]
    assert m["pair_min"][64, 200] == I64_MAX and m["pair_min"][128, 255] == I64_MAX and m["pair_min"][63, 64] == 77
    a.close()


# ---- a swarm that has synced: estimated flags and keyframe paths ------------------------------------------------------
def synced(trajs, store, drones, self_id, world, max_entries=4096, max_meas=1024, frames=range(0, 40, 5), later=()):
    """a 256-drone anchor holding `store`, whose sync_dev of a window of `drones` (one frame per odometry index in
    `frames`, solver poses true in the world) applied, then one of each drone list in `later`: every drone of any of
    them estimated, and those of the last one with a keyframe path -> (anchor, chain, the last solver, its window)"""
    a = host.LoopAnchor(256, 64, max_meas, max_entries, 1.0, 0.0015, 0.0015)
    a.set_data_association(3.345, 256, 4096)
    for d, (s, p) in trajs.items():
        if len(s):
            a.push_odometry(d, s, p)
    if len(store):
        a.add_measurements(store)
    c = host.AnchoredChain(max_meas)
    solver = None
    for sync_drones in [drones, *later]:
        if solver is not None:
            solver.close()
        win = window(trajs, sync_drones, frames)
        a.set_window(*win)
        n = c.run(a)
        c.observe(a, n, self_id, XY, Z)
        ents = win[2]
        init = np.zeros((len(ents), 4))
        for e, ent in enumerate(ents):
            d = int(ent["drone_id"])
            k = int(np.searchsorted(trajs[d][0], ent["stamp"]))
            wp = da.pr.pose_mul(world[d], trajs[d][1][k])
            init[e, :3] = wp[:3]
            init[e, 3] = 2.0 * np.arctan2(wp[6], wp[3])
        solver = host.PoseGraphSolver(max(4096, len(init)), 32768)
        solver.graph_clear()
        solver.graph_add_nodes(init, (np.arange(len(init)) == 0).astype(np.uint8))
        ft, ia, ibb, pay = [], [], [], []
        for d in sync_drones:
            blk = np.nonzero(ents["drone_id"] == d)[0]
            for i, j in zip(blk[:-1], blk[1:]):
                cy, sy = np.cos(init[i, 3]), np.sin(init[i, 3])
                dx, dy = init[j, 0] - init[i, 0], init[j, 1] - init[i, 1]
                p = np.zeros(_l.PAYLOAD_LEN)
                p[:4] = [cy * dx + sy * dy, -sy * dx + cy * dy, init[j, 2] - init[i, 2],
                         np.arctan2(np.sin(init[j, 3] - init[i, 3]), np.cos(init[j, 3] - init[i, 3]))]
                p[4:20] = np.eye(4).ravel()
                ft.append(1); ia.append(i); ibb.append(j); pay.append(p)
        solver.graph_add_factors(ft, ia, ibb, np.array(pay), np.zeros(len(ft), np.uint8))
        c.compact(n, keep=False)
        c.mask = torch.zeros(len(init), dtype=torch.uint8, device="cuda")
        c.yaw = torch.zeros(len(init), dtype=torch.float64, device="cuda")
        c.stream.wait_stream(torch.cuda.current_stream())
        c.init_solve(solver, 4096, 1, 7, 30, np.inf)
        a.sync_dev(solver, c.stream.cuda_stream, self_id, np.inf, 30, True, False)
        c.stream.synchronize()
        assert a.sync_result() == (True, _l.OK)
    return a, c, solver, win


def kf_of(a, drones=range(256)):
    return {d: p for d in drones if (p := a.paths(d)) is not None}


# ---- 2. init_by_loops at 256 drones -----------------------------------------------------------------------------------
T_FIRST = ibl_scene()[0][5][0][0]                  # the scene's first odometry stamp


def world_of(trajs):
    return {d: np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]) for d in trajs}


def ibl_rig(self_id, trajs, rows, win, link_to):
    """drones 5, 127 and 254 synced, then 127 and 254 alone: 5 stays estimated without a keyframe path, and self,
    never synced, holds window entries without one.  Then the window `win`, the loop map and observe from `rows` plus
    a loop from each of 5, 127, 254 and link_to to self (every drone loop-connected to self), and PCM's
    (redundant = false) directory of those loops -> (anchor, chain, the loops, the PCM state, the other solver)"""
    link = loop_rows([40, 41, 42, 43], [5, 127, 254, link_to], self_id, 8, stamps=[[T_FIRST, T_FIRST]] * 4)
    loops = np.concatenate([rows, link])
    a, c, s0, _ = synced(trajs, [], [5, 127, 254], self_id, world_of(trajs), max_entries=512, frames=range(0, 12, 3),
                         later=([127, 254],))
    a.set_window(*win)
    t = upload(loops)
    record(a, t, 0, len(loops), c.stream)
    a.observe_dev(t.data_ptr(), len(loops), c.stream.cuda_stream, self_id, XY, Z)
    pcm = host.PcmState(self_id, False, 15.0, 0.0015, 0.0015, max_pairs=64, pair_capacity=64)
    pcm.reject_anchored(t.data_ptr(), len(loops), c.keep.data_ptr(), c.stream.cuda_stream)   # acquires the device copy
    c.stream.synchronize()
    return a, c, loops, pcm, s0


def resident_poses(n_blocks):
    solver = host.PoseGraphSolver(max(4096, n_blocks), 64)
    solver.graph_clear()
    solver.graph_add_nodes(np.random.default_rng(3).uniform(-1, 1, (n_blocks, 4)), np.zeros(n_blocks, np.uint8))
    return solver


def oracle_inputs(a, pcm, loops, self_id):
    good = {}
    for x in range(256):
        for y in DRONES:
            if x <= y and (s := pcm.inliers(x, y)) is not None:
                good[(x, y)] = s
    m = a.loop_map()
    est = m["estimated"].copy()
    est[self_id] = True                                             # self holds window entries
    vec = ib.LoopMapVec(256, _l.LOOP_RECORD_DTYPE)
    vec.record_vec(loops)
    book = ib.LoopBook(self_id, False)
    book.record(loops)
    assert m["records"].tobytes() == vec.recs.tobytes()
    return good, est, vec, book


@pytest.mark.gpu
@pytest.mark.parametrize("self_id,source", [(SELF, "pairs"), (SELF, "directory"), (0, "pairs")])
def test_init_by_loops_at_256_drones(gpu, self_id, source):
    trajs, win, rows, _ = ibl_scene(self_id=self_id)
    a, c, loops, pcm, s0 = ibl_rig(self_id, trajs, rows, win, 255 if self_id == SELF else 200)
    if source == "directory":                                       # descending id2: (0, 200) before (0, 5)
        pcm.set_inliers(0, 200 if self_id == SELF else 254, [11])
        pcm.set_inliers(0, 5, [10])
        pcm.set_inliers(128, 255, [])
        pcm.set_inliers(127, 127, [16])
    solver = resident_poses(len(win[2]))
    before = solver.graph_get_poses()
    torch.cuda.synchronize()
    a.init_by_loops_dev(pcm, solver, self_id, c.stream.cuda_stream)
    c.stream.synchronize()
    assert a.init_by_loops_result() == _l.OK
    got = solver.graph_get_poses()
    to_init = a.observability()["to_init"]
    assert set(TO_INIT) - {self_id} <= set(np.flatnonzero(to_init).tolist())
    good, est, vec, book = oracle_inputs(a, pcm, loops, self_id)
    kf = kf_of(a, DRONES)
    assert sorted(kf) == [127, 254] and est[5] and est[self_id]     # pose0: paths, identity (5), self's odometry
    want = ib.init_by_loops_vec(to_init, good, vec, est, kf, trajs, self_id, win, before)
    lit = ib.init_pose_by_loops(set(np.flatnonzero(to_init).tolist()), ib.good_from_sets(good), book,
                                set(np.flatnonzero(est).tolist()), kf, ib.Trajs(trajs), self_id, win, before)
    assert close_yaw(want, lit) and close_yaw(got, want)
    moved_rows = np.any(got != before, axis=1)
    moved = set(win[2]["drone_id"][moved_rows].tolist())
    assert {63, 64} <= moved and moved & {128, 254, 255}             # drones in every word past the first placed
    if source == "pairs":
        assert 128 in moved and not good.get((5, 128))               # id2 5: estimated, no path -> identity pose0
        y = got[win[2]["drone_id"] == 128, 3]                       # its loop's and 5's odometry yaws cross +-pi
        assert y.max() > np.pi - 0.01 and y.min() < -np.pi + 0.01
        if self_id == SELF:                                         # drone 0's pairs: estimated 5 and 254, the larger
            assert 0 in moved and not good.get((0, 5)) and not good.get((0, 254))
    # drone 63's id2 is self (no path: pose0 from self's odometry); its shared blocks hold their later frames' poses,
    # one pair on different passes of the entry loop (more than 256 entries apart in the device's order)
    e63 = np.nonzero(win[2]["drone_id"] == 63)[0]
    pos = device_order(win)
    assert (pos[e63[-1]] - pos[e63[0]] > 256) and pos[e63[-1]] // 256 != pos[e63[0]] // 256
    own = ib.init_by_loops_vec(to_init, good, vec, est, kf, trajs, self_id, unshared(win), before)
    for lo, hi in ((0, -1), (40, 100)):
        assert close_yaw(got[e63[[lo]]], own[e63[[hi]]]) and not close_yaw(own[e63[[lo]]], own[e63[[hi]]])
    for h in (a, pcm, solver, s0):
        h.close()


@pytest.mark.gpu
def test_init_by_loops_refuses_an_id2_without_odometry(gpu):
    """self 255 holds window entries but has no odometry; drone 254's loop to it makes 255 its id2, so reading 255's
    odometry refuses the whole call: every pose byte-identical, in both oracle forms too"""
    trajs, win, rows, _ = ibl_scene(self_id=255)
    del trajs[255]
    a, c, loops, pcm, s0 = ibl_rig(255, trajs, rows, win, 0)
    solver = resident_poses(len(win[2]))
    before = solver.graph_get_poses()
    torch.cuda.synchronize()
    a.init_by_loops_dev(pcm, solver, 255, c.stream.cuda_stream)
    c.stream.synchronize()
    assert a.init_by_loops_result() == _l.ERR_INVALID
    assert solver.graph_get_poses().tobytes() == before.tobytes()
    to_init = a.observability()["to_init"]
    assert to_init[254]
    good, est, vec, book = oracle_inputs(a, pcm, loops, 255)
    kf = kf_of(a, DRONES)
    with pytest.raises(ib.Refused):
        ib.init_by_loops_vec(to_init, good, vec, est, kf, trajs, 255, win, before)
    with pytest.raises(ib.Refused):
        ib.init_pose_by_loops(set(np.flatnonzero(to_init).tolist()), ib.good_from_sets(good), book,
                              set(np.flatnonzero(est).tolist()), kf, ib.Trajs(trajs), 255, win, before)
    for h in (a, pcm, solver, s0):
        h.close()


@pytest.mark.gpu
def test_overflowed_map_refuses_every_later_init(gpu):
    trajs, win, rows, _ = ibl_scene()
    a, c, s0, _ = synced(trajs, [], [5, 127, 254, SELF], SELF, world_of(trajs), max_entries=512, max_meas=64,
                         frames=range(0, 12, 3))
    H = table_size(64)
    a.set_window(*win)
    st = c.stream
    t = upload(rows)
    record(a, t, 0, len(rows), st)
    a.observe_dev(t.data_ptr(), len(rows), st.cuda_stream, SELF, XY, Z)
    pcm = host.PcmState(SELF, False, 15.0, 0.0015, 0.0015, max_pairs=64, pair_capacity=64)
    pcm.reject_anchored(t.data_ptr(), len(rows), c.keep.data_ptr(), st.cuda_stream)
    solver = host.PoseGraphSolver(4096, 64)
    solver.graph_clear()
    solver.graph_add_nodes(np.random.default_rng(3).uniform(-1, 1, (len(win[2]), 4)), np.zeros(len(win[2]), np.uint8))
    # the store's capacity in distinct ids, over rounds: half the table, no overflow
    fill = loop_rows(np.arange(1000, 1000 + 64 - len(rows)), 44, 7, 2)
    for k in range(0, len(fill), 16):
        record(a, upload(fill[k:k + 16]), 0, len(fill[k:k + 16]), st)
    torch.cuda.synchronize()
    a.init_by_loops_dev(pcm, solver, SELF, st.cuda_stream)
    st.synchronize()
    assert a.init_by_loops_result() == _l.OK and len(a.loop_map()["records"]) == 64
    # more distinct ids than the table holds
    over = loop_rows(np.arange(5000, 5000 + H + 1), 7, 8, 4)
    record(a, upload(over), 0, len(over), st)
    for _ in range(2):
        before = solver.graph_get_poses()
        torch.cuda.synchronize()
        a.init_by_loops_dev(pcm, solver, SELF, st.cuda_stream)
        st.synchronize()
        assert a.init_by_loops_result() == _l.ERR_CAPACITY
        assert solver.graph_get_poses().tobytes() == before.tobytes()
        record(a, upload(rows[:1]), 0, 1, st)                      # a later record does not clear it
    for h in (a, pcm, solver, s0):
        h.close()


# ---- 3. the data-association search -----------------------------------------------------------------------------------
def da_run(a, c, self_id, thres=3.345, max_nodes=4096, anon_min=256):
    a.set_data_association(thres, anon_min, max_nodes)
    n = c.run(a)
    c.observe(a, n, self_id, XY, Z)
    c.stream.synchronize()
    before = c.rows[:n * ROW].cpu().numpy().tobytes()
    n2 = c.data_association(a, self_id, XY, Z)
    c.stream.synchronize()
    return a.data_association_result(), before, c.rows[:n2 * ROW].cpu().numpy().tobytes()


@pytest.mark.gpu
@pytest.mark.parametrize("self_id,n_ids", [(200, 32), (0, 6)])
def test_da_in_every_word(gpu, self_id, n_ids):
    trajs, _, dets, targets, avail = da_scene(self_id, n_ids)
    _, _, _, world = case(256, [], seed=2)
    a, c, s, _ = synced(trajs, dets, avail, self_id, world, max_meas=512)
    kf = kf_of(a, avail)
    assert sorted(kf) == avail and len(dets) > 256
    (applied, status, guess), _, _ = da_run(a, c, self_id)
    want = da.da_vec(self_id, trajs, kf, dets, 3.345, anon_min=256)
    assert want == da.da_literal(self_id, trajs, kf, dets, 3.345, anon_min=256)
    assert (applied, status, guess) == (want[0], CODES[want[1]], want[2])
    assert applied and len(guess) == n_ids
    if self_id == 200:
        assert guess == targets                                     # 64, 127, 128, 255 among them
    for h in (a, s):
        h.close()
    if n_ids == 32:                                                 # a 33rd id: refused, nothing renamed
        more = dets[:1].copy()
        more["id_b"], more["id"] = 256 + 32, 99_999
        a, c, s, _ = synced(trajs, np.concatenate([dets, more]), avail, self_id, world, max_meas=512)
        (applied, status, guess), b0, b1 = da_run(a, c, self_id)
        assert (applied, status, guess) == (False, _l.ERR_CAPACITY, {}) and b0 == b1
        for h in (a, s):
            h.close()


def plain_anchor(trajs, dets, self_id, drones):
    a = host.LoopAnchor(256, 64, 64, 1024, 1.0, 0.0015, 0.0015)
    for d, (s, p) in trajs.items():
        if len(s):
            a.push_odometry(d, s, p)
    a.set_data_association(3.345, 256, 4096)
    a.add_measurements(dets)
    a.set_window(*window(trajs, drones, range(0, 8, 2)))
    return a, host.AnchoredChain(64)


@pytest.mark.gpu
def test_da_threshold_at_the_exact_float(gpu):
    four = float(np.float32(4.0))
    above = float(np.nextafter(np.float32(4.0), np.float32(np.inf)))
    for cov, thres, want in ((np.eye(6), four, (False, _l.OK, {})), (np.eye(6), above, (True, _l.OK, {256: 255, 257: 255})),
                             (BAD_COV, 1e30, (False, _l.OK, {}))):
        trajs, dets = exact_scene(cov)
        a, c = plain_anchor(trajs, dets, 200, (200, 255))
        got = da_run(a, c, 200, thres=thres)[0]
        assert got == want
        w = da.da_vec(200, trajs, {}, dets, thres, anon_min=256)
        assert (w[0], CODES[w[1]], w[2]) == want
        a.close()


@pytest.mark.gpu
def test_da_budget_boundary_at_256_drones(gpu):
    trajs, dets = budget_scene()
    st = {}
    da.da_vec(200, trajs, {}, dets, 3.345, anon_min=256, stats=st)
    n = st["nodes"]
    for budget, want in ((n, True), (n - 1, False)):
        a, c = plain_anchor(trajs, dets, 200, (64, 128, 200, 255))
        (applied, status, guess), b0, b1 = da_run(a, c, 200, max_nodes=budget)
        assert applied == want and status == (_l.OK if want else _l.ERR_CAPACITY)
        if not want:
            assert guess == {} and b0 == b1
        a.close()


@pytest.mark.gpu
def test_da_search_time_per_call(gpu):
    """worst_scene on the device: every call gates about 32 x 255 candidates.  Times one search at each budget"""
    trajs, _, dets = worst_scene()
    _, _, _, world = case(256, [], seed=7)
    a, c, s, _ = synced(trajs, dets, list(range(256)), 200, world, max_meas=512)
    assert len(kf_of(a)) == 256
    n = c.run(a)
    c.observe(a, n, 200, XY, Z)
    out = {}
    name = torch.cuda.get_device_name(0)
    for budget in BUDGETS:
        a.set_data_association(3.345, 256, budget)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        c.stream.synchronize()
        e0.record(c.stream)
        a.data_association_dev(200, c.stream.cuda_stream)
        e1.record(c.stream)
        c.stream.synchronize()
        assert a.data_association_result() == (False, _l.ERR_CAPACITY, {})
        ms = e0.elapsed_time(e1)
        out[budget] = ms
        print(f"DA worst case on {name}: budget {budget}: {ms:.2f} ms, {worst_gates(budget)} gates, "
              f"{1e6 * ms / worst_gates(budget):.1f} ns a gate")
    assert out[BUDGETS[-1]] > out[BUDGETS[0]]
    for h in (a, s):
        h.close()
