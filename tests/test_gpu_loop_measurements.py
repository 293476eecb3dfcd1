"""GPU: a round's accepted loop edges handed from the front-end to the back-end's store on the device.
osb_frontend_loop_measurements against tests/loop_measurements_ref.py fed the device's own edge results (mixed statuses,
n = 0 / 1 / 64, swapped and unswapped roles, the counters over several rounds); osb_anchor_add_measurements_dev against a
handle fed the same rows from the host (run, VOID rows past the true count, PCM and factor compaction); refusals, launch
counts and resources; and a whole round from query_received to the solve against the same round with a host hop."""
import ctypes as C

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib, synth
from frontend_harness import EB, LOOP_COV, RS, SC, cand_own, filled, loop_frontend, own_query, upload
import frontend_harness as fh
import loop_measurements_ref as lm
from backend_harness import make_anchor, options, pcm_state, resident

pytestmark = pytest.mark.gpu

MB, ROW = lib.MEASUREMENT_DTYPE.itemsize, lib.ANCHOR_RESULT_DTYPE.itemsize
COV_POS, COV_ANG = 0.02, 0.005
SELF = fh.FRONTEND["self_id"]
record, noisy_g = synth.loop_record, synth.loop_noisy_g


def edge_dicts(raw):
    out = []
    for b in raw:
        e = lib.LoopEdgeResult.from_buffer_copy(b)
        out.append(dict(status=e.status, drone_id_a=e.drone_id_a, drone_id_b=e.drone_id_b,
                        relative_pose=np.array(e.relative_pose)))
    return out


def stamps_for(n, base):
    return [(base + 1000 * k + 7, base + 1000 * k + 3) for k in range(n)]


def compute_loop(fe, st, rec_ptr, res_ptr, cands):
    out = filled(max(len(cands), 1) * EB)
    if cands:
        fe.compute_loop(rec_ptr, res_ptr, cands, out.data_ptr(), st)
    torch.cuda.synchronize()
    return out, fh.edges(out, len(cands))


def emit(fe, st, res_ptr, edges_ptr, cands, stamps):
    """loop_measurements into FILL-initialised buffers -> (rows on the host, device rows, device count)"""
    out = filled(max(len(cands), 1) * MB)
    cnt = torch.full((1,), -7, dtype=torch.int32, device="cuda")
    fe.loop_measurements(res_ptr, edges_ptr, cands, stamps, COV_POS, COV_ANG, out.data_ptr(), cnt.data_ptr(), st)
    torch.cuda.synchronize()
    k = int(cnt.cpu()[0])
    return np.frombuffer(out.cpu().numpy().tobytes()[:k * MB], lib.MEASUREMENT_DTYPE), out, cnt


def check_round(fe, st, res_t, results, edges_t, raw, cands, stamps, counters):
    got, _, _ = emit(fe, st, res_t.data_ptr(), edges_t.data_ptr(), cands, stamps)
    ref, counters = lm.loop_measurements(edge_dicts(raw), [r.swapped for r in results], cands, stamps, SELF, COV_POS,
                                         COV_ANG, counters)
    assert got.tobytes() == ref.tobytes()
    n, pairs = fe.loop_counts()
    assert n == counters[0] and np.array_equal(pairs, counters[1])
    return got, counters


def test_rows_and_counters_equal_the_oracle(gpu):
    st = fh.stream()
    fe = loop_frontend()
    counters = lm.new_counters()
    assert fe.loop_counts()[0] == 0
    # round 1: an own keyframe hits an own one (intra-drone, unswapped); the second candidate fails the odometry check
    old, new = record(1, 100, "old"), record(1, 101, "new", seed=1, g=noisy_g(1))
    rt, res_t, res = own_query(fe, st, old, new)
    far = np.concatenate([SC["delta_true"][:3] + 1.0, SC["delta_true"][3:]])
    cands = [cand_own(), cand_own(odom=far)]
    rt2, res2 = upload([new, new]), upload([res, res])
    edges_t, raw = compute_loop(fe, st, rt2.data_ptr(), res2.data_ptr(), cands)
    statuses = [e["status"] for e in edge_dicts(raw)]
    assert statuses == [lib.LOOP_ACCEPTED, lib.LOOP_ODOMETRY_INCONSISTENT]
    rows, counters = check_round(fe, st, res2, [res, res], edges_t, raw, cands, stamps_for(2, 10**18), counters)
    assert len(rows) == 1 and counters[1][1, 1] == 2
    # round 2: ten received keyframes, hits and misses, unswapped
    recs, cands = [], []
    for r in range(10):
        g = noisy_g(10 + r) if r % 5 != 4 else synth.descriptor_db(4, 4096, 300 + r)
        recs.append(record(2 + r % 3, 300 + r, "new", seed=20 + r, g=g, n_outliers=2 + r % 4))
        cands.append(dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"], cov=LOOP_COV))
    rt = upload(recs)
    res_t = filled(10 * RS)
    fe.query_received(rt.data_ptr(), 10, -1, res_t.data_ptr(), st)
    fe.finish(st)
    results = fh.results(res_t, 10)
    edges_t, raw = compute_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), cands)
    statuses = [e["status"] for e in edge_dicts(raw)]
    assert statuses.count(lib.LOOP_ACCEPTED) >= 4 and lib.LOOP_NO_HIT in statuses, statuses
    rows, counters = check_round(fe, st, res_t, results, edges_t, raw, cands, stamps_for(10, 2 * 10**18), counters)
    assert rows["id"].tolist() == [SELF * lm.MAX_LOOP_ID + 1 + k for k in range(len(rows))]
    # round 3: nothing; round 4: 64 candidates, every one accepted
    rows, counters = check_round(fe, st, res_t, [], edges_t, [], [], [], counters)
    assert len(rows) == 0
    rt64, res64 = upload([new] * 64), upload([res] * 64)
    cands = [cand_own()] * 64
    edges_t, raw = compute_loop(fe, st, rt64.data_ptr(), res64.data_ptr(), cands)
    rows, counters = check_round(fe, st, res64, [res] * 64, edges_t, raw, cands, stamps_for(64, 3 * 10**18), counters)
    assert len(rows) == 64
    fe.db_reset()                                             # the reference never resets the counters
    n, pairs = fe.loop_counts()
    assert n == counters[0] and np.array_equal(pairs, counters[1])
    fe.close()
    # a swapped round, n = 1: the own keyframe hits a remote one, so the query record is the old side
    fe = loop_frontend()
    remote = record(2, 200, "new", seed=2, g=noisy_g(2))
    t = upload([remote])
    fe.ingest(t.data_ptr(), 1, -1, st)
    own = record(1, 100, "old")
    rt, res_t, res = own_query(fe, st, None, own, nonkeyframe=True, ingest_old=False)
    assert res.swapped
    cands = [dict(pose_query=SC["pose_old"], pose_hit=SC["pose_new"])]
    edges_t, raw = compute_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), cands)
    rows, counters = check_round(fe, st, res_t, [res], edges_t, raw, cands, [(555, 999)], lm.new_counters())
    assert len(rows) == 1 and (rows["stamp_a"][0], rows["stamp_b"][0]) == (555, 999)
    assert (rows["id_a"][0], rows["id_b"][0]) == (1, 2) and counters[1][2, 1] == counters[1][1, 2] == 1
    fe.close()


def prepare(a, g):
    for d, (s, p) in g["trajs"].items():
        a.push_odometry(d, s, p)
    a.set_window(*g["window"])


def loop_distances(meas):
    loops = meas[meas["type"] == lib.MEAS_LOOP]
    return np.array([lm.loop_distance(r) for r in loops])


def device_rows(rows):
    return torch.frombuffer(bytearray(np.ascontiguousarray(rows).tobytes() or b"\0"), dtype=torch.uint8).cuda()


def test_device_appends_equal_host_appends(gpu):
    g = synth.anchor_swarm(4, 30, 300, seed=11, with_orphans=False)
    meas = g["meas"]
    thr = float(np.float32(np.median(loop_distances(meas))))
    a, b = make_anchor(g, max_meas=1024), make_anchor(g, max_meas=1024)
    for h in (a, b):
        prepare(h, g)
    st = fh.stream()
    keep_alive = []
    chunks = np.array_split(meas, 6)
    for k, ch in enumerate(chunks):
        if k % 2 == 0:                                        # host appends, interleaved with the device ones
            a.add_measurements(ch)
            b.add_measurements(ch)
            continue
        a.add_measurements(lm.add_new_loop_connection(ch, thr))
        buf, cnt = device_rows(ch), torch.tensor([len(ch)], dtype=torch.int32, device="cuda")
        keep_alive += [buf, cnt]
        if k == len(chunks) - 1:
            torch.cuda._sleep(20_000_000)                     # the last append has not run when run_dev sizes its grid
        c0 = host.launch_count()
        b.add_measurements_dev(buf.data_ptr(), cnt.data_ptr(), len(ch) + 5, thr, st)
        assert host.launch_count() - c0 == 1
    cap = len(meas) + 64
    ca, cb = (host.AnchoredChain(cap, torch.cuda.current_stream()) for _ in range(2))
    nb = cb.run(b)                                            # before anything synchronises: the bound
    na = ca.run(a)
    assert na == sum(a.size()) and na < nb <= na + len(chunks[-1]) + 5
    ra = ca.rows[:na * ROW].cpu().numpy().tobytes()
    rb = cb.rows[:nb * ROW].cpu().numpy().tobytes()
    assert rb[:na * ROW] == ra
    void = np.frombuffer(rb[na * ROW:], lib.ANCHOR_RESULT_DTYPE)
    ref = np.zeros(nb - na, lib.ANCHOR_RESULT_DTYPE)
    ref["status"], ref["skip"] = lib.ANCHOR_VOID, 1
    assert void.tobytes() == ref.tobytes()
    # PCM and the factor compaction pass over the VOID rows
    pa, pb = (pcm_state(g, 16, 1024) for _ in range(2))
    for c, h, n in ((ca, pa, na), (cb, pb, nb)):
        c.keep.fill_(9)
        c.reject(h, n)
        c.compact(n)
    torch.cuda.synchronize()
    assert pa.status() == pb.status() == lib.OK
    ka, kb = ca.keep_on_host(na), cb.keep_on_host(nb)
    assert ka.tobytes() == kb[:na].tobytes() and not kb[na:nb].any()
    assert ka.any()
    fa, fb = ca.factors.on_host(), cb.factors.on_host()
    k = len(fa["ftype"])
    assert k > 0 and len(fb["ftype"]) == k
    for key in fa:
        assert fa[key].tobytes() == fb[key].tobytes()
    for i in range(4):
        for j in range(i, 4):
            assert [x.tobytes() for x in pa.pair(i, j)] == [x.tobytes() for x in pb.pair(i, j)]
    # after a synchronising call the counts are exact: run and size agree with the host-fed handle
    assert b.status() == lib.OK and b.size() == a.size()
    assert b.run().tobytes() == a.run().tobytes()
    assert cb.run(b) == na
    # a host append after device appends continues from the device's counts
    extra = synth.anchor_swarm(4, 30, 40, seed=12, with_orphans=False)["meas"]
    extra["id"] += 50_000
    a.add_measurements(extra)
    b.add_measurements(extra)
    assert b.run().tobytes() == a.run().tobytes()
    for h in (pa, pb, a, b):
        h.close()


def test_refusals_launches_and_resources(gpu):
    live0 = host.live_resources()
    st = fh.stream()
    g = synth.anchor_swarm(3, 20, 100, seed=7)
    a = make_anchor(g, 96, len(g["window"][2]), traj_margin=0)
    prepare(a, g)
    a.add_measurements(g["meas"][:90])
    assert a.status() == lib.OK                               # no device append yet
    before, size = a.run(), a.size()
    good = g["meas"][90:100].copy()
    bad_type, bad_drone = good.copy(), good.copy()
    bad_type["type"][3] = 7
    bad_drone["id_b"][5] = g["max_drones"]
    cases = ((good, 10, 10, lib.ERR_CAPACITY), (bad_type, 10, 10, lib.ERR_INVALID), (bad_drone, 10, 10, lib.ERR_INVALID),
             (good, 11, 10, lib.ERR_INVALID), (good, -1, 10, lib.ERR_INVALID))
    for rows, count, max_n, code in cases:
        buf, cnt = device_rows(rows), torch.tensor([count], dtype=torch.int32, device="cuda")
        c0 = host.launch_count()
        a.add_measurements_dev(buf.data_ptr(), cnt.data_ptr(), max_n, 1e9, st)
        assert host.launch_count() - c0 == 1
        assert a.status() == code
        assert a.size() == size and a.run().tobytes() == before.tobytes()
    live1 = host.live_resources()
    L = a._lib
    buf, cnt = device_rows(good[:6]), torch.tensor([6], dtype=torch.int32, device="cuda")
    c0 = host.launch_count()
    vp = C.c_void_p
    for args in ((a._h, None, vp(cnt.data_ptr()), 6), (a._h, vp(buf.data_ptr()), None, 6), (None, vp(buf.data_ptr()),
                 vp(cnt.data_ptr()), 6), (a._h, vp(buf.data_ptr()), vp(cnt.data_ptr()), -1)):
        assert L.osb_anchor_add_measurements_dev(*args, 1e9, vp(st)) == lib.ERR_INVALID
    assert L.osb_anchor_status(None, C.byref(C.c_int(0))) == lib.ERR_INVALID
    assert host.launch_count() == c0
    a.add_measurements_dev(buf.data_ptr(), cnt.data_ptr(), 6, 1e9, st)      # exactly fills the store
    assert a.status() == lib.OK and sum(a.size()) == 96 and host.live_resources() == live1
    a.close()
    # the front-end's call: one launch whatever n, refusals before anything is enqueued, counters acquired once
    fe = loop_frontend()
    old, new = record(1, 100, "old"), record(1, 101, "new", seed=1, g=noisy_g(1))
    rt, res_t, res = own_query(fe, st, old, new)
    edges_t, _ = compute_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), [cand_own()])
    out, cnt = filled(65 * MB), torch.zeros(1, dtype=torch.int32, device="cuda")
    live2 = host.live_resources()
    cands, stamps = host.KeyframeFrontend.loop_candidates([cand_own()] * 65), host.KeyframeFrontend.loop_stamps([(1, 2)] * 65)
    c0 = host.launch_count()
    for args in ((fe._h, vp(res_t.data_ptr()), vp(edges_t.data_ptr()), 65, cands, stamps, vp(out.data_ptr()), vp(cnt.data_ptr())),
                 (fe._h, vp(res_t.data_ptr()), vp(edges_t.data_ptr()), -1, cands, stamps, vp(out.data_ptr()), vp(cnt.data_ptr())),
                 (fe._h, None, vp(edges_t.data_ptr()), 1, cands, stamps, vp(out.data_ptr()), vp(cnt.data_ptr())),
                 (fe._h, vp(res_t.data_ptr()), vp(edges_t.data_ptr()), 1, None, stamps, vp(out.data_ptr()), vp(cnt.data_ptr())),
                 (fe._h, vp(res_t.data_ptr()), vp(edges_t.data_ptr()), 1, cands, None, vp(out.data_ptr()), vp(cnt.data_ptr())),
                 (fe._h, vp(res_t.data_ptr()), vp(edges_t.data_ptr()), 1, cands, stamps, None, vp(cnt.data_ptr())),
                 (None, vp(res_t.data_ptr()), vp(edges_t.data_ptr()), 1, cands, stamps, vp(out.data_ptr()), vp(cnt.data_ptr()))):
        h, r, e, n, cd, sp, o, k = args
        assert L.osb_frontend_loop_measurements(h, r, e, n, cd, sp, 0.1, 0.1, o, k, vp(st)) == lib.ERR_INVALID
    assert L.osb_frontend_loop_counts(fe._h, None, None) == lib.ERR_INVALID
    assert host.launch_count() == c0 and host.live_resources() == live2
    for n in (1, 0, 1):
        c0 = host.launch_count()
        fe.loop_measurements(res_t.data_ptr(), edges_t.data_ptr(), [cand_own()] * n, [(1, 2)] * n, 0.1, 0.1,
                             out.data_ptr(), cnt.data_ptr(), st)
        assert host.launch_count() - c0 == 1
    assert host.live_resources() > live2                      # the first call acquired the counters, the others nothing
    live3 = host.live_resources()
    fe.loop_measurements(res_t.data_ptr(), edges_t.data_ptr(), [cand_own()], [(1, 2)], 0.1, 0.1, out.data_ptr(),
                         cnt.data_ptr(), st)
    assert fe.loop_counts()[0] == 3 and host.live_resources() == live3
    fe.close()
    assert host.live_resources() == live0


def entry_stamp(g, drone, frame):
    """the stamp of drone's vo_available window entry nearest to frame"""
    stamps, first, e = g["window"]
    for f in list(range(frame, len(stamps))) + list(range(frame - 1, -1, -1)):
        row = e[first[f]:first[f + 1]]
        row = row[(row["drone_id"] == drone) & (row["vo_available"] == 1)]
        if len(row):
            return int(row["stamp"][0])
    raise AssertionError("no entry")


def test_device_round_solves_as_the_host_hop_round(gpu):
    g = synth.anchor_swarm(5, 30, 300, seed=9, with_orphans=False)
    base = synth.anchor_window_graph(g)
    st = fh.stream()
    fe = loop_frontend()
    old = record(1, 100, "old")
    ot = upload([old])
    fe.ingest_own(ot.data_ptr(), st)
    n = 6
    recs = [record(2 + r % 3, 300 + r, "new", seed=20 + r, g=noisy_g(10 + r)) for r in range(n)]
    cands = [dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"], cov=LOOP_COV) for _ in range(n)]
    stamps = [(entry_stamp(g, 2 + r % 3, 4 + 3 * r), entry_stamp(g, 1, 2 + 3 * r)) for r in range(n)]
    rt, res_t = upload(recs), filled(n * RS)
    fe.query_received(rt.data_ptr(), n, -1, res_t.data_ptr(), st)
    edges_t, raw = compute_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), cands)
    assert sum(e["status"] == lib.LOOP_ACCEPTED for e in edge_dicts(raw)) >= 3
    anchors = [make_anchor(g, max_meas=1024) for _ in range(2)]
    for h in anchors:
        prepare(h, g)
        h.add_measurements(g["meas"][:200])
    states = [pcm_state(g, 32, 1024) for _ in range(2)]
    solvers = [host.PoseGraphSolver(4096, 32768) for _ in range(2)]
    o = options(solvers[0], "tight")
    chains = [host.AnchoredChain(2048) for _ in range(2)]
    for s in solvers:
        resident(s, base)
    # (B) the device round: loop_measurements -> add_measurements_dev -> run_dev -> reject_anchored -> compact -> solve
    s = chains[1].stream.cuda_stream
    meas_t, cnt_t = filled(n * MB), torch.zeros(1, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()                                  # the buffers were written on the current stream
    fe.loop_measurements(res_t.data_ptr(), edges_t.data_ptr(), cands, stamps, COV_POS, COV_ANG, meas_t.data_ptr(),
                         cnt_t.data_ptr(), s)
    anchors[1].add_measurements_dev(meas_t.data_ptr(), cnt_t.data_ptr(), n, 2.0, s)
    chains[1](anchors[1], states[1])
    chains[1].solve(solvers[1], 2048, o)
    # (A) the host hop: download the edge and query results, build the rows, add them on the host
    results = fh.results(res_t, n)
    rows, _ = lm.loop_measurements(edge_dicts(raw), [r.swapped for r in results], cands, stamps, SELF, COV_POS, COV_ANG,
                                   lm.new_counters())
    anchors[0].add_measurements(lm.add_new_loop_connection(rows, 2.0))
    chains[0](anchors[0], states[0])
    chains[0].solve(solvers[0], 2048, o)
    torch.cuda.synchronize()
    assert anchors[1].status() == lib.OK and anchors[1].size() == anchors[0].size()
    ta, tb = (c.factors.on_host(c.stream) for c in chains)
    assert len(ta["ftype"]) > 0 and all(ta[k].tobytes() == tb[k].tobytes() for k in ta)
    ok = anchors[0].run()
    assert (ok["status"][ok["type"] == lib.MEAS_LOOP][-len(rows):] == lib.ANCHOR_OK).any()
    pa, pb = solvers[0].graph_get_poses(), solvers[1].graph_get_poses()
    assert np.array_equal(pa, pb) and not np.array_equal(pa, base["init"])
    for h in anchors + states + solvers + [fe]:
        h.close()
