"""GPU: osb_frontend_receive_dev -- every keyframe received from the swarm as LoopNet delivers it (only its flagged 3-D
landmarks, only the directions that have some) and as on_image_recv's gates keep it.  Output bytes against
oracle/loop_net_ref.py (extracted stereo records with and without cameras, depth and lower-camera-as-main records, random
records, n = 1 / 8 / 64, skip and own records mixed in); a whole received round from receive to the anchor's store against
the same round fed the oracle's delivered records, with the loop edges checked against oracle/loop_ref.py; a swapped own
query onto a delivered remote row; a round where an unflagged landmark steals a mutual nearest neighbour, so delivery
changes the matches; fp16 rows; capture; launches, resources and refusals."""
import ctypes as C

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib, synth
from oracle import loop_net_ref as ln
from frontend_harness import EB, RB, RS, SC, filled, loop_frontend, make_frontend, upload
import frontend_harness as fh
import loop_candidates_ref as lc
from backend_harness import make_anchor

pytestmark = pytest.mark.gpu

CB, SB, MB = lib.CANDIDATE_BYTES, lib.STAMPS_BYTES, lib.MEASUREMENT_DTYPE.itemsize
SELF = fh.FRONTEND["self_id"]
PRM = dict(inter_drone_init_frames=2, pos_covariance_per_meter=0.01, yaw_covariance_per_meter=0.003, loop_cov_pos=0.013,
           loop_cov_ang=2.5e-4)
GATES = dict(min_loop_num=15, min_direction_loop=3)        # set_loop_params' defaults
COV_POS, COV_ANG = 0.02, 0.005
record, noisy_g = synth.loop_record, synth.loop_noisy_g
vp = C.c_void_p


def random_record(seed, drone, msg, p_flag=0.6):
    """noise in every plane (beyond n_kpts too), random counts and flags"""
    rng = np.random.default_rng(seed)
    r = ln.empty_record()
    r["drone_id"], r["msg_id"], r["n_dirs"] = drone, msg, int(rng.integers(1, 5))
    for f in ("global_desc", "local_desc", "kpts", "landmarks_3d"):
        r[f] = rng.normal(size=r[f].shape)
    r["stereo_match"] = rng.integers(-1, 200, r["stereo_match"].shape)
    r["landmarks_flag"] = (rng.random(r["landmarks_flag"].shape) < p_flag) * rng.integers(1, 3, r["landmarks_flag"].shape)
    r["n_kpts"] = rng.integers(0, 201, 4)
    r["n_kpts_down"] = rng.integers(0, 201, 4)
    return r.tobytes()


def extracted_records():
    """records extract writes on four other drones: stereo without and with cameras, depth, lower camera as main"""
    st = fh.stream()
    out, keep = [], []
    plain = make_frontend(dict(db_capacity=64), self_id=2)
    cams = make_frontend(dict(db_capacity=64), self_id=3)
    cams.set_cameras(SC["K"], SC["ext"], SC["ext"], 0.006)
    depth = make_frontend(dict(db_capacity=64), self_id=4)
    depth.set_depth_camera(SC["K"], SC["ext"])
    down = make_frontend(dict(db_capacity=64), self_id=5)
    down.set_main_camera("down")
    for k, fe in enumerate((plain, cams, depth, down)):
        for j in range(2):
            t = filled(RB)
            if fe is depth:
                img, dep = fh.depth_frame(40 + 2 * k + j)
                fe.extract_depth(img, dep, 500 + 10 * k + j, t.data_ptr(), st)
            else:
                up, dn = fh.frame_images(40 + 2 * k + j)
                up, dn = np.ascontiguousarray(up), np.ascontiguousarray(dn)
                keep += [up, dn]
                fe.extract(up.ctypes.data, dn.ctypes.data, 500 + 10 * k + j, t.data_ptr(), st)
            fe.finish(st)
            out.append(t.cpu().numpy().tobytes())
    for fe in (plain, cams, depth, down):
        fe.close()
    return out


def receiver():
    """the receiving drone: the loop scene's cameras, loop parameters and candidate parameters"""
    fe = loop_frontend()
    fe.set_candidate_params(**PRM)
    return fe


def receive(fe, recs_bytes, skip, st):
    n = len(recs_bytes)
    src, out = upload(recs_bytes), filled(n * RB)
    c0 = host.launch_count()
    fe.receive_dev(src.data_ptr(), n, skip, out.data_ptr(), st)
    assert host.launch_count() - c0 == 1
    return src, out


def oracle_round(recs_bytes, skip, db_rows, gates=GATES):
    return [r.tobytes() for r in ln.receive_round(recs_bytes, skip, SELF, db_rows, gates["min_direction_loop"],
                                                  gates["min_loop_num"])]


def test_bytes_equal_the_oracle(gpu):
    st = fh.stream()
    ext = extracted_records()
    assert any(ln.as_record(b)["landmarks_flag"].any() for b in ext)
    fe = receiver()
    own = record(SELF, 100, "old")
    # gate (a): an empty store drops every foreign record, own and skipped ones travel
    mixed = [ext[0], bytes(own), ext[1], random_record(1, 3, 7, 0.9)]
    _, out = receive(fe, mixed, 2, st)
    torch.cuda.synchronize()
    got = fh._split(out, 4, RB)
    want = oracle_round(mixed, 2, 0)
    assert got == want and got[0] == ln.dropped(ln.as_record(ext[0])).tobytes() and got[1] == bytes(own)
    ot = upload([own])
    fe.ingest_own(ot.data_ptr(), st)
    fe.finish(st)
    rows = fe.db_size() + fe.db_size(remote=True)
    assert rows > 0
    pool = ext + [random_record(s, 2 + s % 4, 600 + s, p_flag=[0.02, 0.3, 0.9, 1.0][s % 4]) for s in range(60)]
    pool[5] = bytes(record(SELF, 101, "new", seed=1))             # own records mixed in
    pool[20] = bytes(record(3, 102, "new", seed=2))               # loop-scene records: kept
    kept = 0
    for n, skip in ((1, -1), (1, 0), (8, 3), (64, 17), (64, -1)):
        recs = pool[:n] if n < 64 else pool[:64]
        _, out = receive(fe, recs, skip, st)
        torch.cuda.synchronize()
        got = fh._split(out, n, RB)
        want = oracle_round(recs, skip, rows)
        for r in range(n):
            assert got[r] == want[r], (n, skip, r)
        kept += sum(1 for r in range(n) if r != skip and ln.as_record(recs[r])["drone_id"] != SELF
                    and ln.as_record(got[r])["n_kpts"].any())
    assert kept > 0
    fe.close()


def entry_stamp(g, drone, frame):
    """the stamp of drone's vo_available window entry nearest to frame"""
    stamps, first, e = g["window"]
    for f in list(range(frame, len(stamps))) + list(range(frame - 1, -1, -1)):
        row = e[first[f]:first[f + 1]]
        row = row[(row["drone_id"] == drone) & (row["vo_available"] == 1)]
        if len(row):
            return int(row["stamp"][0])
    raise AssertionError("no entry")


def stealing_record(drone, msg, seed, old):
    """a loop-scene record whose unflagged landmark 0 of every direction carries exactly the old descriptor that flagged
    landmark 1 matches: undelivered, landmark 0 is the old point's mutual nearest neighbour and removes landmark 1's match"""
    rec = record(drone, msg, "new", seed=seed, g=noisy_g(seed))
    a = np.ctypeslib.as_array
    for d in range(4):
        n_old = old.n_kpts[d]
        od = a(old.local_desc[d])[:n_old]
        nd = a(rec.local_desc[d])
        assert rec.landmarks_flag[d][0] == 0 and rec.landmarks_flag[d][1] == 1
        p = int(np.argmax(od @ nd[1]))
        nd[0] = od[p]
    return rec


def chain(fe, anchor, rt, mt, n, b, s):
    """receive's consumers, as INTEGRATION.md 2.5 orders them, from the records at rt (device pointer)"""
    fe.init_modes_dev(rt, n, -1, b["init"].data_ptr(), s)
    fe.query_received_dev(rt, n, -1, b["init"].data_ptr(), b["res"].data_ptr(), s)
    fe.ingest_meta(rt, mt, n, -1, s)
    fe.loop_candidates_dev(rt, mt, b["res"].data_ptr(), n, b["init"].data_ptr(), b["cand"].data_ptr(),
                           b["stamps"].data_ptr(), s)
    fe.compute_loop_dev(rt, b["res"].data_ptr(), n, b["cand"].data_ptr(), b["edges"].data_ptr(), s)
    fe.loop_measurements_dev(b["res"].data_ptr(), b["edges"].data_ptr(), n, b["cand"].data_ptr(), b["stamps"].data_ptr(),
                             COV_POS, COV_ANG, b["meas"].data_ptr(), b["cnt"].data_ptr(), s)
    anchor.add_measurements_dev(b["meas"].data_ptr(), b["cnt"].data_ptr(), n, 2.0, s)


def buffers(n):
    return dict(init=filled(n), res=filled(n * RS), cand=filled(n * CB), stamps=filled(n * SB), edges=filled(n * EB),
                meas=filled(n * MB), cnt=torch.zeros(1, dtype=torch.int32, device="cuda"))


def check_edges_against_loop_ref(b, recs_bytes, n, old):
    """every candidate with a hit: compute_loop of the delivered frames (oracle/loop_ref.py) gives the device's edge"""
    res, cands = fh.results(b["res"], n), (lib.LoopCandidate * n).from_buffer_copy(b["cand"].cpu().numpy().tobytes())
    accepted = 0
    for i, raw in enumerate(fh.edges(b["edges"], n)):
        e, r, c = lib.LoopEdgeResult.from_buffer_copy(raw), res[i], cands[i]
        if not r.accepted:
            assert e.status == lib.LOOP_NO_HIT
            continue
        assert r.hit_msg_id == old.msg_id and not r.swapped
        rec = lib.KeyframeRecord.from_buffer_copy(recs_bytes[i])
        cand = dict(pose_query=np.array(c.pose_query), pose_hit=np.array(c.pose_hit), init_mode=c.init_mode,
                    odom_rel=np.array(c.odom_rel), cov=np.array(c.odom_edge_cov).reshape(6, 6))
        ref = fh.loop_oracle(r, rec, old, cand, SC["K"], SC["ext"], dict(fh.LOOP_PARAMS, **GATES))
        assert e.status == ref["status"] and e.n_corr == ref["n_corr"]
        k = e.n_corr
        assert list(e.corr_idx_new[:k]) == ref["idx_new"].tolist() and list(e.corr_idx_old[:k]) == ref["idx_old"].tolist()
        if ref["pnp"] is not None and ref["pnp"]["success"]:
            assert np.array_equal(np.array(e.inlier[:k], np.uint8), ref["pnp"]["mask"])
            assert np.abs(np.array(e.relative_pose) - ref["relative_pose"]).max() < 1e-8
        accepted += e.status == lib.LOOP_ACCEPTED
    return accepted


@pytest.mark.parametrize("storage", ["fp32", "fp16"])
def test_received_round_equals_the_delivered_oracle_round(gpu, storage):
    """A: receive on the device, then the round; B: the same round fed the oracle's delivered records; C: the round fed
    the records as sent (no delivery).  Then an own query swapped onto a delivered remote row."""
    g = synth.anchor_swarm(5, 30, 300, seed=9, with_orphans=False)
    st = torch.cuda.Stream()
    s = st.cuda_stream
    fes, anchors = [], []
    for _ in range(3):
        fe = loop_frontend()
        if storage == "fp16":
            fe.set_db_storage("fp16")
        fe.set_candidate_params(**PRM)
        fes.append(fe)
        a = make_anchor(g, max_meas=1024)
        for d, (ts, p) in g["trajs"].items():
            a.push_odometry(d, ts, p)
        a.set_window(*g["window"])
        anchors.append(a)
    old = record(1, 100, "old")
    m_old = lc.metas([(1, 100, entry_stamp(g, 1, 2), SC["pose_old"])])
    ot, omt = upload([old]), torch.frombuffer(bytearray(m_old.tobytes()), dtype=torch.uint8).cuda()
    n = 8
    recs, items = [], []
    for r in range(n):
        d = 2 + r % 3
        rec = stealing_record(d, 300 + r, 20 + r, old) if r % 4 == 1 else record(d, 300 + r, "new", seed=20 + r,
                                                                                  g=noisy_g(10 + r))
        if r == 6:
            for k in range(4):                                    # one frame with a single non-empty direction: dropped
                if k != 1:
                    rec.landmarks_flag[k][:] = [0] * 200
        recs.append(bytes(rec))
        items.append((d, 300 + r, entry_stamp(g, d, 4 + 3 * r), SC["pose_new"]))
    metas = lc.metas(items)
    mt = torch.frombuffer(bytearray(metas.tobytes()), dtype=torch.uint8).cuda()
    with torch.cuda.stream(st):
        for fe in fes:
            fe.ingest_own_meta(ot.data_ptr(), omt.data_ptr(), s)
    st.synchronize()
    rows = fes[0].db_size()
    delivered = oracle_round(recs, -1, rows)
    assert ln.as_record(delivered[6])["n_kpts"].sum() == 0
    sent_t, deliv_t = upload(recs), upload(delivered)
    out_t = filled(n * RB)
    bufs = [buffers(n) for _ in range(3)]
    with torch.cuda.stream(st):
        fes[0].receive_dev(sent_t.data_ptr(), n, -1, out_t.data_ptr(), s)
        chain(fes[0], anchors[0], out_t.data_ptr(), mt.data_ptr(), n, bufs[0], s)
        chain(fes[1], anchors[1], deliv_t.data_ptr(), mt.data_ptr(), n, bufs[1], s)
        chain(fes[2], anchors[2], sent_t.data_ptr(), mt.data_ptr(), n, bufs[2], s)
    st.synchronize()
    assert fh._split(out_t, n, RB) == delivered
    for key in ("init", "res", "cand", "stamps", "edges", "cnt"):
        assert bufs[0][key].cpu().numpy().tobytes() == bufs[1][key].cpu().numpy().tobytes(), key
    k = int(bufs[0]["cnt"].cpu()[0])
    assert k >= 2 and bufs[0]["meas"].cpu().numpy().tobytes()[:k * MB] == bufs[1]["meas"].cpu().numpy().tobytes()[:k * MB]
    assert fes[0].db_size(remote=True) == fes[1].db_size(remote=True) < fes[2].db_size(remote=True)
    assert check_edges_against_loop_ref(bufs[0], delivered, n, old) == k
    # delivery matters: in the undelivered round landmark 0 (unflagged) takes landmark 1's old point; delivered, landmark 1
    # keeps its match.  Matches are compared in the sent record's landmark indices.
    ra, rc = fh.results(bufs[0]["res"], n), fh.results(bufs[2]["res"], n)
    stolen = 0
    for r in range(1, n, 4):
        if not (ra[r].accepted and rc[r].accepted):
            continue
        sent = ln.as_record(recs[r])
        for j in range(4):
            d = ra[r].dir_new[j]
            if d < 0:
                continue
            idx = np.nonzero(sent["landmarks_flag"][d][:sent["n_kpts"][d]] > 0)[0]
            got = {int(idx[m]) for m in ra[r].match_new[j][:ra[r].n_matches[j]]}
            jc = list(rc[r].dir_new).index(d)
            undelivered = set(int(m) for m in rc[r].match_new[jc][:rc[r].n_matches[jc]])
            assert 0 in undelivered and 0 not in got
            stolen += (1 in got) and (1 not in undelivered)
    assert stolen > 0
    # swapped: an own keyframe whose hit is a delivered remote row, its edge's new side read from the remote store
    own = record(1, 102, "old")
    ow = upload([own])
    m_own = lc.metas([(1, 102, entry_stamp(g, 1, 28), SC["pose_old"])])
    omt2 = torch.frombuffer(bytearray(m_own.tobytes()), dtype=torch.uint8).cuda()
    b1 = [buffers(1) for _ in range(2)]
    with torch.cuda.stream(st):
        for fe, b, a in zip(fes[:2], b1, anchors[:2]):
            fe.ingest_own_meta(ow.data_ptr(), omt2.data_ptr(), s)
            fe.query(ow.data_ptr(), b["res"].data_ptr(), s, nonkeyframe=True)
            fe.loop_candidates_dev(ow.data_ptr(), omt2.data_ptr(), b["res"].data_ptr(), 1, None, b["cand"].data_ptr(),
                                   b["stamps"].data_ptr(), s)
            fe.compute_loop_dev(ow.data_ptr(), b["res"].data_ptr(), 1, b["cand"].data_ptr(), b["edges"].data_ptr(), s)
    st.synchronize()
    res_own = fh.results(b1[0]["res"], 1)[0]
    assert res_own.accepted and res_own.swapped
    for key in ("res", "cand", "edges"):
        assert b1[0][key].cpu().numpy().tobytes() == b1[1][key].cpu().numpy().tobytes(), key
    e = lib.LoopEdgeResult.from_buffer_copy(fh.edges(b1[0]["edges"], 1)[0])
    hit = lib.KeyframeRecord.from_buffer_copy(delivered[res_own.hit_msg_id - 300])
    c = lib.LoopCandidate.from_buffer_copy(b1[0]["cand"].cpu().numpy().tobytes())
    ref = fh.loop_oracle(res_own, own, hit, dict(pose_query=np.array(c.pose_query), pose_hit=np.array(c.pose_hit),
                                                  init_mode=c.init_mode), SC["K"], SC["ext"], dict(fh.LOOP_PARAMS, **GATES))
    assert e.status == ref["status"] and e.n_corr == ref["n_corr"]
    if ref["pnp"] is not None and ref["pnp"]["success"]:
        assert np.abs(np.array(e.relative_pose) - ref["relative_pose"]).max() < 1e-8
    for a in anchors:
        assert a.status() == lib.OK
    assert anchors[0].size() == anchors[1].size() and anchors[0].run().tobytes() == anchors[1].run().tobytes()
    for h in fes + anchors:
        h.close()


def test_captured_round_replays_the_direct_bytes(gpu):
    """receive + the round captured into a CUDA graph (any host synchronisation fails the capture) and replayed"""
    g = synth.anchor_swarm(5, 30, 300, seed=9, with_orphans=False)
    st = torch.cuda.Stream()
    s = st.cuda_stream
    fes, anchors = [receiver(), receiver()], []
    for _ in range(2):
        a = make_anchor(g, max_meas=1024)
        for d, (ts, p) in g["trajs"].items():
            a.push_odometry(d, ts, p)
        a.set_window(*g["window"])
        anchors.append(a)
    old = record(1, 100, "old")
    ot = upload([old])
    omt = torch.frombuffer(bytearray(lc.metas([(1, 100, entry_stamp(g, 1, 2), SC["pose_old"])]).tobytes()),
                           dtype=torch.uint8).cuda()
    n = 8
    rounds = []
    for k in range(2):                                           # a warm-up round, then the captured one
        recs, items = [], []
        for r in range(n):
            d = 2 + r % 3
            recs.append(bytes(stealing_record(d, 300 + 10 * k + r, 20 + r, old) if r % 3 == 0 else
                              record(d, 300 + 10 * k + r, "new", seed=20 + r, g=noisy_g(10 + r))))
            items.append((d, 300 + 10 * k + r, entry_stamp(g, d, 4 + 3 * r + k), SC["pose_new"]))
        rounds.append((upload(recs), torch.frombuffer(bytearray(lc.metas(items).tobytes()), dtype=torch.uint8).cuda()))
    bufs = [dict(buffers(n), out=filled(n * RB)) for _ in range(2)]
    with torch.cuda.stream(st):
        for fe in fes:
            fe.ingest_own_meta(ot.data_ptr(), omt.data_ptr(), s)

    def step(fe, anchor, b, k):
        rt, mt = rounds[k]
        fe.receive_dev(rt.data_ptr(), n, -1, b["out"].data_ptr(), s)
        chain(fe, anchor, b["out"].data_ptr(), mt.data_ptr(), n, b, s)

    with torch.cuda.stream(st):
        for fe, a, b in zip(fes, anchors, bufs):
            step(fe, a, b, 0)
            fe.finish(s)
    st.synchronize()
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=st, capture_error_mode="global"):
        step(fes[1], anchors[1], bufs[1], 1)
    with torch.cuda.stream(st):
        step(fes[0], anchors[0], bufs[0], 1)
    graph.replay()
    torch.cuda.synchronize()
    for key in ("out", "res", "edges", "cnt"):
        assert bufs[0][key].cpu().numpy().tobytes() == bufs[1][key].cpu().numpy().tobytes(), key
    assert int(bufs[0]["cnt"].cpu()[0]) > 0
    assert anchors[0].run().tobytes() == anchors[1].run().tobytes()
    for h in fes + anchors:
        h.close()


def test_refusals_launches_and_resources(gpu):
    live0 = host.live_resources()
    st = fh.stream()
    fe = make_frontend(dict(db_capacity=64))
    src, out = upload([record(2, 1, "new")] * 4), filled(4 * RB)
    L, h = fe._lib, fe._h
    sp, op = vp(src.data_ptr()), vp(out.data_ptr())
    c0, live1 = host.launch_count(), host.live_resources()
    assert L.osb_frontend_receive_dev(h, sp, 1, -1, op, vp(st)) == lib.ERR_INVALID      # no loop parameters yet
    assert host.launch_count() == c0 and host.live_resources() == live1
    fe.set_loop_params()
    c0, live1 = host.launch_count(), host.live_resources()
    calls = [lambda: L.osb_frontend_receive_dev(None, sp, 1, -1, op, vp(st)),
             lambda: L.osb_frontend_receive_dev(h, sp, 65, -1, op, vp(st)),
             lambda: L.osb_frontend_receive_dev(h, sp, -1, -1, op, vp(st)),
             lambda: L.osb_frontend_receive_dev(h, None, 1, -1, op, vp(st)),
             lambda: L.osb_frontend_receive_dev(h, sp, 1, -1, None, vp(st)),
             lambda: L.osb_frontend_receive_dev(h, sp, 2, -1, vp(src.data_ptr() + RB), vp(st)),     # overlapping
             lambda: L.osb_frontend_receive_dev(h, vp(out.data_ptr() + RB), 2, -1, op, vp(st)),
             lambda: L.osb_frontend_receive_dev(h, sp, 1, -1, sp, vp(st))]
    for i, call in enumerate(calls):
        assert call() == lib.ERR_INVALID, i
    assert host.launch_count() == c0 and host.live_resources() == live1
    for n in (0, 1, 4):
        c0 = host.launch_count()
        fe.receive_dev(src.data_ptr(), n, -1, out.data_ptr(), st)
        assert host.launch_count() - c0 == (1 if n else 0)
    assert L.osb_frontend_receive_dev(h, sp, 2, -1, vp(src.data_ptr() + 2 * RB), vp(st)) == lib.OK   # adjacent, not overlapping
    torch.cuda.synchronize()
    assert host.live_resources() == live1
    fe.close()
    assert host.live_resources() == live0
