"""GPU: each keyframe's stamp and drone pose kept on the device and a round's loop candidates built there.
osb_frontend_loop_candidates_dev against tests/loop_candidates_ref.py bit for bit (own, received and swapped hits, misses,
n = 1 / 8 / 64, init mode from the device counters); compute_loop_dev / loop_measurements_dev against the host-array calls
fed the device's candidates on a twin handle fed by the plain calls; refusals, launch counts, resources; the whole round
from query_received to the anchor captured into a CUDA graph; osb_swarm_exchange_meta at world 1."""
import ctypes as C

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib, synth
from frontend_harness import EB, RS, SC, filled, loop_frontend, upload
import frontend_harness as fh
import loop_candidates_ref as lc
import loop_measurements_ref as lm
from backend_harness import make_anchor

pytestmark = pytest.mark.gpu

CB, SB, MB, META = lib.CANDIDATE_BYTES, lib.STAMPS_BYTES, lib.MEASUREMENT_DTYPE.itemsize, lib.META_BYTES
SELF = fh.FRONTEND["self_id"]
CAP = fh.LOOP_CONFIG["db_capacity"]
PRM = dict(inter_drone_init_frames=2, pos_covariance_per_meter=0.01, yaw_covariance_per_meter=0.003, loop_cov_pos=0.013,
           loop_cov_ang=2.5e-4)
COV_POS, COV_ANG = 0.02, 0.005
record, noisy_g = synth.loop_record, synth.loop_noisy_g
vp = C.c_void_p


def meta_t(metas):
    return torch.frombuffer(bytearray(metas.tobytes()), dtype=torch.uint8).cuda()


def received(n, msg0, seed0):
    """n records of drones 2..4 (every fifth a miss) and their metas"""
    recs, items = [], []
    for r in range(n):
        g = noisy_g(seed0 + r) if r % 5 != 4 else synth.descriptor_db(4, 4096, 300 + seed0 + r)
        d = 2 + r % 3
        recs.append(record(d, msg0 + r, "new", seed=seed0 + r, g=g, n_outliers=2 + r % 4))
        p = SC["pose_new"].copy()
        p[:3] += 0.01 * r
        items.append((d, msg0 + r, 10**12 + msg0 * 1000 + r, p))
    return recs, lc.metas(items)


class Twin:
    """A (metas, device candidates) and B (plain calls, the host-array calls) fed the same keyframes, and the oracle"""

    def __init__(self):
        self.st = fh.stream()
        self.a, self.b = loop_frontend(), loop_frontend()
        self.a.set_candidate_params(**PRM)
        self.ref = lc.MetaStores(SELF, CAP)
        self.counters = lm.new_counters()
        self.keep = []

    def ingest(self, recs, metas, own=False):
        rt, mt = upload(recs), meta_t(metas)
        self.keep += [rt, mt]
        if own:
            self.a.ingest_own_meta(rt.data_ptr(), mt.data_ptr(), self.st)
            self.b.ingest_own(rt.data_ptr(), self.st)
        else:
            self.a.ingest_meta(rt.data_ptr(), mt.data_ptr(), len(recs), -1, self.st)
            self.b.ingest(rt.data_ptr(), len(recs), -1, self.st)
        self.ref.ingest(recs, metas)
        assert self.a.meta_status() == lib.OK

    def round(self, recs, metas, rt, res_a, res_b, init_dev=None, init_flags=None):
        """candidates of the round on A vs the oracle; compute_loop_dev / loop_measurements_dev on A vs the host calls on B
        fed A's candidates -> the number of accepted edges"""
        n, st = len(recs), self.st
        mt = meta_t(metas)
        cand, stamps = filled(n * CB), filled(n * SB)
        c0 = host.launch_count()
        self.a.loop_candidates_dev(rt.data_ptr(), mt.data_ptr(), res_a.data_ptr(), n, init_dev, cand.data_ptr(),
                                   stamps.data_ptr(), st)
        assert host.launch_count() - c0 == 1
        torch.cuda.synchronize()
        results = fh.results(res_a, n)
        want_c, want_s = lc.candidates(self.ref, recs, metas, results, self.counters[1], PRM, init_flags)
        got_c, got_s = cand.cpu().numpy().tobytes(), stamps.cpu().numpy().tobytes()
        assert got_c == want_c.tobytes() and got_s == want_s.tobytes()
        edges_a, edges_b = filled(n * EB), filled(n * EB)
        c0 = host.launch_count()
        self.a.compute_loop_dev(rt.data_ptr(), res_a.data_ptr(), n, cand.data_ptr(), edges_a.data_ptr(), st)
        assert host.launch_count() - c0 == 3
        ca, sa = (lib.LoopCandidate * n).from_buffer_copy(got_c), (lib.LoopStamps * n).from_buffer_copy(got_s)
        lib.check(self.b._lib.osb_frontend_compute_loop(self.b._h, vp(rt.data_ptr()), vp(res_b.data_ptr()), n, ca,
                                                        vp(edges_b.data_ptr()), vp(st)))
        meas_a, meas_b = filled(n * MB), filled(n * MB)
        cnt_a, cnt_b = (torch.full((1,), -7, dtype=torch.int32, device="cuda") for _ in range(2))
        c0 = host.launch_count()
        self.a.loop_measurements_dev(res_a.data_ptr(), edges_a.data_ptr(), n, cand.data_ptr(), stamps.data_ptr(), COV_POS,
                                     COV_ANG, meas_a.data_ptr(), cnt_a.data_ptr(), st)
        assert host.launch_count() - c0 == 1
        self.b.loop_measurements(res_b.data_ptr(), edges_b.data_ptr(), ca, sa, COV_POS, COV_ANG, meas_b.data_ptr(),
                                 cnt_b.data_ptr(), st)
        torch.cuda.synchronize()
        assert edges_a.cpu().numpy().tobytes() == edges_b.cpu().numpy().tobytes()
        k = int(cnt_a.cpu()[0])
        assert k == int(cnt_b.cpu()[0])
        assert meas_a.cpu().numpy().tobytes()[:k * MB] == meas_b.cpu().numpy().tobytes()[:k * MB]
        (na, pa), (nb, pb) = self.a.loop_counts(), self.b.loop_counts()
        assert na == nb and np.array_equal(pa, pb)
        # the counters the oracle's init-mode rule reads next round
        eds = [lib.LoopEdgeResult.from_buffer_copy(b) for b in fh.edges(edges_a, n)]
        ed = [dict(status=e.status, drone_id_a=e.drone_id_a, drone_id_b=e.drone_id_b, relative_pose=np.array(e.relative_pose))
              for e in eds]
        cd = [dict(pose_query=c["pose_query"], pose_hit=c["pose_hit"]) for c in want_c]
        _, self.counters = lm.loop_measurements(ed, [r.swapped for r in results], cd, [tuple(s) for s in want_s], SELF,
                                                COV_POS, COV_ANG, self.counters)
        assert na == self.counters[0] and np.array_equal(pa, self.counters[1])
        return sum(e.status == lib.LOOP_ACCEPTED for e in eds), [e.status for e in eds]

    def received_round(self, recs, metas):
        n, st = len(recs), self.st
        rt = upload(recs)
        init = torch.full((n,), 0x5A, dtype=torch.uint8, device="cuda")
        self.a.init_modes_dev(rt.data_ptr(), n, -1, init.data_ptr(), st)
        res_a, res_b = filled(n * RS), filled(n * RS)
        self.a.query_received_dev(rt.data_ptr(), n, -1, init.data_ptr(), res_a.data_ptr(), st)
        torch.cuda.synchronize()
        flags = init.cpu().numpy()
        assert flags.tolist() == lc.init_modes(recs, -1, SELF, self.counters[1], PRM["inter_drone_init_frames"]).tolist()
        self.b.query_received(rt.data_ptr(), n, -1, res_b.data_ptr(), st, init_mode=flags.astype(bool))
        torch.cuda.synchronize()
        assert res_a.cpu().numpy().tobytes() == res_b.cpu().numpy().tobytes()
        self.ingest(recs, metas)                             # on_image_recv adds the received keyframes
        return flags, self.round(recs, metas, rt, res_a, res_b, init_dev=init.data_ptr(), init_flags=flags)

    def own_query(self, rec, meta, nonkeyframe=False):
        self.ingest([rec], meta, own=True)
        rt = upload([rec])
        res_a, res_b = filled(RS), filled(RS)
        self.a.query(rt.data_ptr(), res_a.data_ptr(), self.st, nonkeyframe=nonkeyframe)
        self.b.query(rt.data_ptr(), res_b.data_ptr(), self.st, nonkeyframe=nonkeyframe)
        self.a.finish(self.st); self.b.finish(self.st)
        assert res_a.cpu().numpy().tobytes() == res_b.cpu().numpy().tobytes()
        return rt, res_a, res_b

    def close(self):
        self.a.close(); self.b.close()


def test_candidates_and_rounds_equal_the_oracle_and_the_host_calls(gpu):
    t = Twin()
    accepted = 0
    # own keyframes: old, then new (own-own hit, odometry from the device trajectory), n = 1
    old, new = record(1, 100, "old"), record(1, 101, "new", seed=1, g=noisy_g(1))
    m_old, m_new = lc.metas([(1, 100, 1000, SC["pose_old"])]), lc.metas([(1, 101, 2000, SC["pose_new"])])
    t.ingest([old], m_old, own=True)
    rt, ra, rb = t.own_query(new, m_new)
    res_new = fh.results(ra, 1)[0]
    assert res_new.accepted and not res_new.swapped and res_new.hit_drone_id == SELF
    k, _ = t.round([new], m_new, rt, ra, rb)
    accepted += k
    # two received rounds of n = 8 (hits and misses): init mode from the device counters flips for drone 2 in between
    recs, metas = received(8, 300, 10)
    f1, (k, s1) = t.received_round(recs, metas)
    accepted += k
    assert lib.LOOP_NO_HIT in s1 and f1[0] == 1
    recs2, metas2 = received(8, 400, 10)
    f2, (k, _) = t.received_round(recs2, metas2)
    accepted += k
    assert t.counters[1][2, SELF] >= PRM["inter_drone_init_frames"] and f2[0] == 0 and f1.tolist() != f2.tolist()
    # an own keyframe hitting a remote one: swapped, cross-drone, n = 1
    own = record(1, 102, "old")
    rt, ra, rb = t.own_query(own, lc.metas([(1, 102, 3000, SC["pose_old"])]), nonkeyframe=True)
    assert fh.results(ra, 1)[0].swapped
    k, s = t.round([own], lc.metas([(1, 102, 3000, SC["pose_old"])]), rt, ra, rb)
    accepted += k
    assert s[0] != lib.LOOP_NO_FRAME
    # n = 64 own-own candidates of one result
    rt64, ra64 = upload([new] * 64), upload([res_new] * 64)
    k, s = t.round([new] * 64, np.repeat(m_new, 64), rt64, ra64, ra64)
    accepted += k
    assert len(set(s)) == 1
    assert accepted >= 4
    t.close()


def test_refusals_launches_and_resources(gpu):
    live0 = host.live_resources()
    st = fh.stream()
    fm, fp = loop_frontend(), loop_frontend()               # meta calls / the plain calls
    ref = lc.MetaStores(SELF, CAP)
    old, mid, new = (record(1, 100, "old"), record(1, 105, "old", seed=5, g=synth.descriptor_db(4, 4096, 77)),
                     record(1, 101, "new", seed=1, g=noisy_g(1)))
    metas = [lc.metas([(1, 999, 1000, SC["pose_old"])]),    # msg_id differs from the record's: not stored
             lc.metas([(1, 105, 2000, SC["pose_old"])]),
             lc.metas([(1, 101, 2000, SC["pose_new"])])]     # stamp not after the last sample: stored, not appended
    codes = [lib.ERR_INVALID, lib.OK, lib.ERR_INVALID]
    assert fm.meta_status() == lib.OK                        # nothing ingested with a meta yet
    keep = []
    for rec, m, code in zip((old, mid, new), metas, codes):
        rt, mt = upload([rec]), meta_t(m)
        keep += [rt, mt]
        c0 = host.launch_count()
        fm.ingest_own_meta(rt.data_ptr(), mt.data_ptr(), st)
        assert host.launch_count() - c0 == 2
        fp.ingest_own(rt.data_ptr(), st)
        ref.ingest([rec], m)
        assert fm.meta_status() == code == ref.status
    assert fm.db_size() == fp.db_size() and fm.db_size(remote=True) == fp.db_size(remote=True)
    rt = upload([new])
    ra, rb = filled(RS), filled(RS)
    fm.query(rt.data_ptr(), ra.data_ptr(), st)
    fp.query(rt.data_ptr(), rb.data_ptr(), st)
    torch.cuda.synchronize()
    assert ra.cpu().numpy().tobytes() == rb.cpu().numpy().tobytes()
    res = fh.results(ra, 1)[0]
    assert res.accepted and res.hit_msg_id == 100
    # the hit's frame has no meta: the candidate is marked and compute_loop_dev gives NO_FRAME
    cand, stamps, mt = filled(CB), filled(SB), meta_t(metas[2])
    with pytest.raises(lib.OsbError):                        # before set_candidate_params
        fm.loop_candidates_dev(rt.data_ptr(), mt.data_ptr(), ra.data_ptr(), 1, None, cand.data_ptr(), stamps.data_ptr(), st)
    fm.set_candidate_params(**PRM)
    fm.loop_candidates_dev(rt.data_ptr(), mt.data_ptr(), ra.data_ptr(), 1, None, cand.data_ptr(), stamps.data_ptr(), st)
    torch.cuda.synchronize()
    want, want_s = lc.candidates(ref, [new], metas[2], [res], lm.new_counters()[1], PRM)
    assert want["reserved"][0] == 1 and cand.cpu().numpy().tobytes() == want.tobytes()
    assert stamps.cpu().numpy().tobytes() == want_s.tobytes()
    edges = filled(EB)
    fm.compute_loop_dev(rt.data_ptr(), ra.data_ptr(), 1, cand.data_ptr(), edges.data_ptr(), st)
    torch.cuda.synchronize()
    assert lib.LoopEdgeResult.from_buffer_copy(fh.edges(edges, 1)[0]).status == lib.LOOP_NO_FRAME
    # null pointers and n outside 0..64: refused before anything is enqueued
    L, h = fm._lib, fm._h
    p = [vp(x.data_ptr()) for x in (rt, mt, ra, cand, stamps, edges)]
    rtp, mtp, rap, cp, sp, ep = p
    out, cnt = filled(65 * MB), torch.zeros(1, dtype=torch.int32, device="cuda")
    op, kp = vp(out.data_ptr()), vp(cnt.data_ptr())
    c0, live1 = host.launch_count(), host.live_resources()
    calls = [lambda: L.osb_frontend_ingest_meta(h, rtp, None, 1, -1, vp(st)),
             lambda: L.osb_frontend_ingest_meta(h, None, mtp, 1, -1, vp(st)),
             lambda: L.osb_frontend_ingest_meta(h, rtp, mtp, 65, -1, vp(st)),
             lambda: L.osb_frontend_ingest_own_meta(h, rtp, None, vp(st)),
             lambda: L.osb_frontend_ingest_own_meta(None, rtp, mtp, vp(st)),
             lambda: L.osb_frontend_meta_status(h, None),
             lambda: L.osb_frontend_set_candidate_params(h, None),
             lambda: L.osb_frontend_loop_candidates_dev(h, rtp, mtp, rap, 65, None, cp, sp, vp(st)),
             lambda: L.osb_frontend_loop_candidates_dev(h, rtp, mtp, rap, -1, None, cp, sp, vp(st)),
             lambda: L.osb_frontend_loop_candidates_dev(h, rtp, None, rap, 1, None, cp, sp, vp(st)),
             lambda: L.osb_frontend_loop_candidates_dev(h, rtp, mtp, rap, 1, None, cp, None, vp(st)),
             lambda: L.osb_frontend_compute_loop_dev(h, rtp, rap, 1, None, ep, vp(st)),
             lambda: L.osb_frontend_compute_loop_dev(h, rtp, rap, 0, cp, ep, vp(st)),
             lambda: L.osb_frontend_compute_loop_dev(h, rtp, rap, 65, cp, ep, vp(st)),
             lambda: L.osb_frontend_loop_measurements_dev(h, rap, ep, 1, cp, None, 0.1, 0.1, op, kp, vp(st)),
             lambda: L.osb_frontend_loop_measurements_dev(h, rap, ep, 65, cp, sp, 0.1, 0.1, op, kp, vp(st)),
             lambda: L.osb_frontend_loop_measurements_dev(h, rap, ep, 1, cp, sp, 0.1, 0.1, None, kp, vp(st)),
             lambda: L.osb_frontend_init_modes_dev(h, rtp, 65, -1, cp, vp(st)),
             lambda: L.osb_frontend_init_modes_dev(h, rtp, 1, -1, None, vp(st)),
             lambda: L.osb_frontend_query_received_dev(h, rtp, 65, -1, None, rap, vp(st)),
             lambda: L.osb_frontend_query_received_dev(h, None, 1, -1, None, rap, vp(st))]
    for i, call in enumerate(calls):
        assert call() == lib.ERR_INVALID, i
    assert host.launch_count() == c0 and host.live_resources() == live1
    # launches: one for the candidates and one for the init modes whatever n (none for n = 0)
    init = filled(64)
    for n in (0, 1):
        c0 = host.launch_count()
        fm.loop_candidates_dev(rt.data_ptr(), mt.data_ptr(), ra.data_ptr(), n, None, cand.data_ptr(), stamps.data_ptr(), st)
        assert host.launch_count() - c0 == n
        c0 = host.launch_count()
        fm.init_modes_dev(rt.data_ptr(), n, -1, init.data_ptr(), st)
        assert host.launch_count() - c0 == n
    rrecs, _ = received(8, 300, 10)
    rrt = upload(rrecs)
    r8 = filled(8 * RS)
    c0 = host.launch_count()
    fp.query_received(rrt.data_ptr(), 8, -1, r8.data_ptr(), st)
    n_plain = host.launch_count() - c0
    c0 = host.launch_count()
    fm.query_received_dev(rrt.data_ptr(), 8, -1, None, r8.data_ptr(), st)
    assert host.launch_count() - c0 == n_plain
    torch.cuda.synchronize()
    fm.close(); fp.close()
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


def test_round_captured_into_a_graph_equals_direct_calls_and_the_host_path(gpu):
    g = synth.anchor_swarm(5, 30, 300, seed=9, with_orphans=False)
    st = torch.cuda.Stream()
    s = st.cuda_stream
    fes = [loop_frontend() for _ in range(3)]                # host path from the oracle's candidates / direct / graph
    anchors = [make_anchor(g, max_meas=1024) for _ in range(3)]
    for a in anchors:
        for d, (ts, p) in g["trajs"].items():
            a.push_odometry(d, ts, p)
        a.set_window(*g["window"])
    ref = lc.MetaStores(SELF, CAP)
    old = record(1, 100, "old")
    m_old = lc.metas([(1, 100, entry_stamp(g, 1, 2), SC["pose_old"])])
    ot, omt = upload([old]), meta_t(m_old)
    n = 8
    rounds = []
    for k in range(2):                                       # a warm-up round (acquires every buffer), then the round
        recs, items = [], []
        for r in range(n):
            d = 2 + r % 3
            recs.append(record(d, 300 + 10 * k + r, "new", seed=20 + r, g=noisy_g(10 + r)))
            items.append((d, 300 + 10 * k + r, entry_stamp(g, d, 4 + 3 * r + k), SC["pose_new"]))
        rounds.append((recs, lc.metas(items)))
    bufs = dict(rt=[upload(r) for r, _ in rounds], mt=[meta_t(m) for _, m in rounds], init=filled(n), res=filled(n * RS),
                cand=filled(n * CB), stamps=filled(n * SB), edges=filled(n * EB), meas=filled(n * MB),
                cnt=torch.zeros(1, dtype=torch.int32, device="cuda"))
    dev_bufs = [dict(bufs, init=filled(n), res=filled(n * RS), cand=filled(n * CB), stamps=filled(n * SB),
                     edges=filled(n * EB), meas=filled(n * MB), cnt=torch.zeros(1, dtype=torch.int32, device="cuda"))
                for _ in range(2)]
    with torch.cuda.stream(st):
        for fe in fes:
            fe.set_candidate_params(**PRM)
            fe.ingest_own_meta(ot.data_ptr(), omt.data_ptr(), s)
    ref.ingest([old], m_old)
    st.synchronize()

    def device_round(fe, anchor, b, k):
        rt, mt = b["rt"][k].data_ptr(), b["mt"][k].data_ptr()
        fe.init_modes_dev(rt, n, -1, b["init"].data_ptr(), s)
        fe.query_received_dev(rt, n, -1, b["init"].data_ptr(), b["res"].data_ptr(), s)
        fe.ingest_meta(rt, mt, n, -1, s)
        fe.loop_candidates_dev(rt, mt, b["res"].data_ptr(), n, b["init"].data_ptr(), b["cand"].data_ptr(),
                               b["stamps"].data_ptr(), s)
        fe.compute_loop_dev(rt, b["res"].data_ptr(), n, b["cand"].data_ptr(), b["edges"].data_ptr(), s)
        fe.loop_measurements_dev(b["res"].data_ptr(), b["edges"].data_ptr(), n, b["cand"].data_ptr(), b["stamps"].data_ptr(),
                                 COV_POS, COV_ANG, b["meas"].data_ptr(), b["cnt"].data_ptr(), s)
        anchor.add_measurements_dev(b["meas"].data_ptr(), b["cnt"].data_ptr(), n, 2.0, s)

    counters = lm.new_counters()
    for k in range(2):
        recs, metas = rounds[k]
        # (A) the host path: finish, copy the results, the oracle's candidates, the host-array calls, the host append
        fe = fes[0]
        rt = bufs["rt"][k].data_ptr()
        flags = lc.init_modes(recs, -1, SELF, counters[1], PRM["inter_drone_init_frames"])
        with torch.cuda.stream(st):
            fe.query_received(rt, n, -1, bufs["res"].data_ptr(), s, init_mode=flags.astype(bool))
            fe.ingest(rt, n, -1, s)
            fe.finish(s)
        results = fh.results(bufs["res"], n)
        ref.ingest(recs, metas)
        cand, stamps = lc.candidates(ref, recs, metas, results, counters[1], PRM, flags)
        ca, sa = (lib.LoopCandidate * n).from_buffer_copy(cand.tobytes()), (lib.LoopStamps * n).from_buffer_copy(stamps.tobytes())
        lib.check(fe._lib.osb_frontend_compute_loop(fe._h, vp(rt), vp(bufs["res"].data_ptr()), n, ca,
                                                    vp(bufs["edges"].data_ptr()), vp(s)))
        fe.loop_measurements(bufs["res"].data_ptr(), bufs["edges"].data_ptr(), ca, sa, COV_POS, COV_ANG,
                             bufs["meas"].data_ptr(), bufs["cnt"].data_ptr(), s)
        st.synchronize()
        kk = int(bufs["cnt"].cpu()[0])
        rows = np.frombuffer(bufs["meas"].cpu().numpy().tobytes()[:kk * MB], lib.MEASUREMENT_DTYPE)
        anchors[0].add_measurements(lm.add_new_loop_connection(rows, 2.0))
        counters = (fes[0].loop_counts()[0], fes[0].loop_counts()[1].astype(np.int64))
        # (B) direct calls; (C) the same round captured into a graph and replayed (the warm-up round runs directly)
        device_round(fes[1], anchors[1], dev_bufs[0], k)
        if k == 0:
            device_round(fes[2], anchors[2], dev_bufs[1], k)
        else:
            fes[2].finish(s)                                 # exact row bounds: the captured ingest needs no refresh
            graph = torch.cuda.CUDAGraph()
            c0 = host.launch_count()
            with torch.cuda.graph(graph, stream=st):
                device_round(fes[2], anchors[2], dev_bufs[1], k)
            launches = host.launch_count() - c0
            graph.replay()
        st.synchronize()
        assert kk >= 3
        for b in dev_bufs:
            assert b["meas"].cpu().numpy().tobytes()[:kk * MB] == rows.tobytes()
            assert int(b["cnt"].cpu()[0]) == kk
    assert launches > 0
    for a in anchors:
        assert a.status() == lib.OK
    want = anchors[0].run()
    assert (want["status"] == lib.ANCHOR_OK).any()
    for a in anchors[1:]:
        assert a.size() == anchors[0].size() and a.run().tobytes() == want.tobytes()
    for fe in fes[1:]:
        n1, p1 = fe.loop_counts()
        assert n1 == counters[0] and np.array_equal(p1, counters[1])
    for h in fes + anchors:
        h.close()


def test_exchange_meta_at_world_one(gpu):
    sw = host.Swarm(None, 0, 1)
    m = lc.metas([(3, 44, 123456789, SC["pose_new"])])
    src, dst = meta_t(m), filled(META)
    c0 = host.launch_count()
    sw.exchange_meta(src.data_ptr(), dst.data_ptr(), fh.stream())
    torch.cuda.synchronize()
    assert dst.cpu().numpy().tobytes() == m.tobytes() and host.launch_count() == c0
    assert sw._lib.osb_swarm_exchange_meta(sw._h, None, vp(dst.data_ptr()), vp(fh.stream())) == lib.ERR_INVALID
    sw.close()
