"""GPU: osb_frontend_query_received -- the keyframes of a swarm round received from other drones, queried against the
own-keyframe (local) store in one pass (loop_detector.cpp:98-119, 191-195).  Every result must be byte-identical to what
osb_frontend_query writes for that record alone, hits and matches must agree with the oracle's LoopDetectorDB and
cross-check matcher, and the batch must not read the remote store, whatever it holds."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import synth, host, lib
from oracle import frontend_ref as fr
from frontend_harness import FILL, RB, RS, filled, frame_images, upload
import frontend_harness as fh

pytestmark = pytest.mark.gpu

ND, MN = 4, 200
QDIR = 1
N_OWN = 4
SIGMAS = [0.0, 0.5, 2.5, 3.5, 6.0]      # inner product with the source ~ 1, 0.89, 0.37, 0.27, 0.16
CONFIG = dict(db_capacity=256, init_mode_product_thres=0.2, match_index_dist=2)


def make_frontend(**kw):
    return fh.make_frontend(CONFIG, **kw)


def shifted(seed):
    """frame `seed` seen again: shifted by two pixels with a little pixel noise"""
    rng = np.random.default_rng(seed + 50)
    sh = lambda a: np.clip(np.roll(a, 2, axis=2).astype(np.int16) + rng.integers(-3, 4, a.shape), 0, 255).astype(np.uint8)
    return tuple(np.ascontiguousarray(sh(a)) for a in frame_images(seed))


def coop_rows():
    """rows up to which a search takes the cooperative scan kernel: DB_COOP_CHUNK (64) rows x 2 CTAs per SM"""
    return 64 * 2 * torch.cuda.get_device_properties(0).multi_processor_count


def closed_result_ok(r, geometric_filter):
    ok = (r.hit_id, r.hit_dir, r.hit_score, r.accepted, r.swapped, r.hit_msg_id, r.hit_drone_id) == (-1, -1, -1.0, 0, 0, -1, -1)
    ok &= list(r.dir_new) == [-1] * ND and list(r.dir_old) == [-1] * ND and list(r.n_matches) == [0] * ND
    if geometric_filter:
        ok &= list(r.n_geo) == [0] * ND and list(r.geo_valid) == [0] * ND
    return ok


class Round:
    """A drone (self_id 1) with N_OWN own keyframes (extract + ingest_own) and `n_loaded` rows from db_load, and a pool
    of 64 foreign records: re-labelled extracts of revisits (own frames seen again) and of new places, and synthetic
    records whose query descriptor is a noisy loaded row, at the noise levels of SIGMAS."""

    def __init__(self, n_loaded, geometric_filter, local_desc=True, ingest_pool=True):
        self.gf = geometric_filter
        self.fe = make_frontend(db_capacity=n_loaded + N_OWN * ND + 64 * ND, geometric_filter=geometric_filter)
        fe, st = self.fe, fh.stream()
        self.stream = st
        rec_t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
        self.own = []
        for i in range(N_OWN):
            up, down = (np.ascontiguousarray(a) for a in frame_images(i))
            fe.extract(up.ctypes.data, down.ctypes.data, 100 + i, rec_t.data_ptr(), st)
            fe.ingest_own(rec_t.data_ptr(), st)
            fe.finish(st)
            self.own.append(fh.records(rec_t, 1)[0])
        self.n_own_rows = sum(1 for r in self.own for d in range(ND) if r.n_kpts[d] > 0)
        self.g = synth.descriptor_db(n_loaded, 4096, 11)
        self.ld = synth.local_descriptors(MN, 77)[None].repeat(n_loaded, 0) if local_desc else None
        self.nk = np.full(n_loaded, 150, np.int32)
        fe.db_load(self.g, self.ld, self.nk if local_desc else None)
        kp = np.random.default_rng(3).uniform(0, 90, (n_loaded, MN, 2)).astype(np.float32)
        fe.db_set_geometry(self.n_own_rows, kp, np.zeros((n_loaded, MN), np.int32))
        # foreign extracts: revisits of the own frames and new places
        pool = []
        for s in list(range(N_OWN)) + [20, 21, 22]:
            up, down = shifted(s) if s < N_OWN else (np.ascontiguousarray(a) for a in frame_images(s))
            fe.extract(up.ctypes.data, down.ctypes.data, 0, rec_t.data_ptr(), st)
            fe.finish(st)
            pool.append(rec_t.cpu().numpy().tobytes())
        rng = np.random.default_rng(9)
        recs = []
        for r in range(64):
            if r % 4 == 3:          # synthetic: a noisy loaded row, the loaded rows' local descriptors
                rec = lib.KeyframeRecord()
                rec.n_dirs = ND
                rec.n_kpts[QDIR] = 150
                row = int(rng.integers(0, n_loaded))
                np.ctypeslib.as_array(rec.global_desc[QDIR])[:] = synth.noisy_queries(
                    self.g, np.array([row]), sigma=SIGMAS[r % 5], seed=r)[0]
                np.ctypeslib.as_array(rec.local_desc[QDIR])[:150] = synth.local_descriptors(150, r, base=self.ld[row]) \
                    if local_desc else 0
                np.ctypeslib.as_array(rec.kpts[QDIR])[:150] = kp[row, :150] + np.float32(1.0)
                np.ctypeslib.as_array(rec.landmarks_flag[QDIR])[:150] = 1
            else:
                rec = lib.KeyframeRecord.from_buffer_copy(pool[r % len(pool)])
                if r >= len(pool):  # later copies: noise on the queried descriptor
                    gq = np.ctypeslib.as_array(rec.global_desc[QDIR])
                    gq += rng.standard_normal(4096).astype(np.float32) * np.float32(SIGMAS[r % 5] / 64.0)
                    gq /= np.linalg.norm(gq)
            rec.drone_id, rec.msg_id = 2 + r % 3, 1000 + r
            recs.append(bytes(rec))
        self.recs = [lib.KeyframeRecord.from_buffer_copy(b) for b in recs]
        self.recs_t = upload(recs)
        if ingest_pool:             # the remote store holds copies of the first 16 records
            fe.ingest(self.recs_t.data_ptr(), 16, -1, st)
            fe.finish(st)

    def rec_ptr(self, r=0):
        return self.recs_t.data_ptr() + r * RB

    def batch(self, n, skip=-1, init=None, recs_ptr=None):
        out = filled(max(n, 1) * RS)
        self.fe.query_received(self.rec_ptr() if recs_ptr is None else recs_ptr, n, skip, out.data_ptr(), self.stream,
                               init_mode=init)
        self.fe.finish(self.stream)
        raw = out.cpu().numpy().tobytes()
        return [raw[r * RS:(r + 1) * RS] for r in range(n)]

    def single(self, r, init_mode=False):
        out = filled(RS)
        self.fe.query(self.rec_ptr(r), out.data_ptr(), self.stream, init_mode=init_mode, nonkeyframe=False)
        self.fe.finish(self.stream)
        return out.cpu().numpy().tobytes()

    def oracle(self):
        """LoopDetectorDB holding the same local rows in the same order"""
        det = fr.LoopDetectorDB(self_id=1, dim=4096, inner_product_thres=0.3, init_mode_product_thres=0.2,
                                match_index_dist=2)
        for i, o in enumerate(self.own):
            det.add_frame(100 + i, 1, [np.ctypeslib.as_array(o.global_desc[d]) for d in range(ND)], list(o.n_kpts))
        for j in range(len(self.g)):
            det.add_frame(10000 + j, 1, [self.g[j]], [1])
        return det

    def row_local(self, row, d_old):
        """local descriptors of local row `row` in direction d_old's frame row"""
        if row < self.n_own_rows:
            rows = [(f, d) for f in range(N_OWN) for d in range(ND) if self.own[f].n_kpts[d] > 0]
            f = rows[row][0]
            n = self.own[f].n_kpts[d_old]
            return np.ctypeslib.as_array(self.own[f].local_desc[d_old])[:n]
        j = row - self.n_own_rows
        return self.ld[j, :self.nk[j]]


def res_of(raw):
    return lib.LoopResult.from_buffer_copy(raw)


@pytest.mark.parametrize("large", [False, True], ids=["coop_scan", "row_scan"])
@pytest.mark.parametrize("geometric_filter", [0, 1])
def test_batch_equals_single_queries(gpu, large, geometric_filter):
    """Every result of a batch equals, byte for byte, osb_frontend_query of that record alone with its init flag: n from 1
    to 64 (one scan pass, the 8-query pass boundary, the limit), stores on both sides of the cooperative-scan limit."""
    n_loaded = coop_rows() + 3000 if large else 300
    rd = Round(n_loaded, geometric_filter, local_desc=not large)
    assert (n_loaded + rd.n_own_rows > coop_rows()) == large
    seen = dict(hit=0, miss=0, matched=0, geo=0, init_only=0)
    for n in (1, 2, 7, 8, 9, 17, 64):
        init = [r % 3 == 1 for r in range(n)]
        got = rd.batch(n, -1, init)
        for r in range(n):
            want = rd.single(r, init[r])
            assert got[r] == want, f"n={n}: record {r} differs from its single query"
            res = res_of(got[r])
            seen["hit" if res.accepted else "miss"] += 1
            seen["matched"] += int(res.accepted and sum(res.n_matches) > 0)
            seen["geo"] += int(bool(geometric_filter) and sum(res.geo_valid) > 0)     # untouched without the filter
            seen["init_only"] += int(res.accepted and init[r] and res.hit_score <= 0.3)
    # the batch exercised hits and misses, the matcher, init mode and (when on) the geometric filter
    assert seen["hit"] > 0 and seen["miss"] > 0 and seen["matched"] > 0 and seen["init_only"] > 0, seen
    assert (seen["geo"] > 0) == bool(geometric_filter), seen
    rd.fe.close()


def test_hits_and_matches_against_oracle(gpu):
    """Hits against LoopDetectorDB.query(drone, q, init_mode, nonkeyframe=False), matches against bf_crosscheck with the
    foreign record as the new side.  Record 3 scores between INIT_MODE_PRODUCT_THRES and INNER_PRODUCT_THRES: it hits
    only with its own init flag set, and its neighbours keep theirs."""
    rd = Round(300, 0)
    det = rd.oracle()
    # record 3 of the batch: a loaded row at inner product ~0.25
    rec = lib.KeyframeRecord.from_buffer_copy(bytes(rd.recs[3]))
    np.ctypeslib.as_array(rec.global_desc[QDIR])[:] = synth.noisy_queries(rd.g, np.array([40]), sigma=np.sqrt(15.0),
                                                                            seed=1)[0]
    raw = bytearray(rd.recs_t.cpu().numpy().tobytes())
    raw[3 * RB:4 * RB] = bytes(rec)
    rd.recs_t.copy_(torch.frombuffer(raw, dtype=torch.uint8))
    rd.recs[3] = rec
    q3 = np.ctypeslib.as_array(rec.global_desc[QDIR])
    assert 0.2 < float(rd.g[40] @ q3) < 0.3
    n = 12
    base = [r % 2 == 0 and r != 3 for r in range(n)]
    runs = {}
    for on in (False, True):
        init = list(base)
        init[3] = on
        got = [res_of(x) for x in rd.batch(n, -1, init)]
        runs[on] = got
        for r in range(n):
            res, rc = got[r], rd.recs[r]
            q = np.ctypeslib.as_array(rc.global_desc[QDIR])
            rid, rdist = det.query(rc.drone_id, q, init[r], False)
            assert res.hit_id == rid, (on, r, res.hit_id, rid)
            assert res.accepted == int(rid != -1 and rdist > -1)
            if not res.accepted:
                continue
            assert abs(res.hit_score - rdist) < 1e-4 and res.swapped == 0 and res.hit_drone_id == 1
            main_new, main_old, slot = QDIR, res.hit_dir, 0
            for _dn in range(main_new, main_new + ND):
                dn, do = _dn % ND, ((main_old - main_new + ND) % ND + _dn) % ND
                nq = rc.n_kpts[dn]
                old = rd.row_local(res.hit_id, do) if res.hit_id < rd.n_own_rows or do == QDIR else np.zeros((0, 64))
                if nq <= 0 or len(old) == 0:
                    continue
                assert (res.dir_new[slot], res.dir_old[slot]) == (dn, do)
                qi, ti, _ = fr.bf_crosscheck(np.ctypeslib.as_array(rc.local_desc[dn])[:nq], old)
                m = res.n_matches[slot]
                assert m == len(qi) and list(res.match_new[slot][:m]) == qi.tolist()
                assert list(res.match_old[slot][:m]) == ti.tolist()
                slot += 1
            assert all(res.dir_new[s] == -1 for s in range(slot, ND))
    assert runs[True][3].accepted == 1 and runs[True][3].hit_id == rd.n_own_rows + 40
    assert runs[False][3].accepted == 0
    for r in range(n):
        if r != 3:
            assert bytes(runs[True][r]) == bytes(runs[False][r]), f"record {r} changed with record 3's flag"
    assert sum(x.accepted for x in runs[True]) >= 4 and sum(sum(x.n_matches) > 0 for x in runs[True]) >= 2
    rd.fe.close()


def test_skip_and_own_records_stay_closed(gpu):
    """`skip` and an own-drone record in the batch get the gate-closed result; the others are unaffected by them."""
    for gf in (0, 1):
        rd = Round(300, gf)
        n = 12
        ref = rd.batch(n)
        raw = bytearray(rd.recs_t.cpu().numpy().tobytes())
        lib.KeyframeRecord.from_buffer(raw, 7 * RB).drone_id = 1               # record 7 is this drone's own
        recs2 = upload([raw])
        assert res_of(ref[7]).accepted == 1 and res_of(ref[11]).accepted == 1  # synthetic records at scores 0.37, 0.89
        got = rd.batch(n, skip=11, recs_ptr=recs2.data_ptr())
        for r in range(n):
            if r in (7, 11):
                assert closed_result_ok(res_of(got[r]), gf), r
            else:
                assert got[r] == ref[r], r
        rd.fe.close()


def test_remote_store_and_ingest_order_do_not_matter(gpu):
    """The batch reads the local store only: the same bytes before and after the records are ingested, with the remote
    store empty, and with it full of the records' own descriptors (which a remote scan would hit at score 1).  The remote
    top-k left by an own non-keyframe query right before does not leak in either."""
    rd = Round(300, 1, ingest_pool=False)
    fe, st = rd.fe, rd.stream
    n = 16
    init = [r % 5 == 0 for r in range(n)]
    assert fe.db_size(True) == 0
    before = rd.batch(n, -1, init)
    fe.ingest(rd.rec_ptr(), n, -1, st)
    fe.finish(st)
    assert fe.db_size(True) > 0
    after = rd.batch(n, -1, init)
    # fill the rest of the remote store with the queried descriptors themselves
    qs = np.stack([np.ctypeslib.as_array(rd.recs[r].global_desc[QDIR]) for r in range(n)])
    fe.db_load(qs, remote=True)
    # an own non-keyframe query whose remote top-k is a perfect remote hit
    own = lib.KeyframeRecord.from_buffer_copy(bytes(rd.recs[0]))
    own.drone_id = 1
    own_t = upload([own])
    res_t = torch.zeros(RS, dtype=torch.uint8, device="cuda")
    fe.query(own_t.data_ptr(), res_t.data_ptr(), st, nonkeyframe=True)
    fe.finish(st)
    assert res_of(res_t.cpu().numpy().tobytes()).hit_id >= lib.REMOTE_MAGIN_NUMBER
    full = rd.batch(n, -1, init)
    assert before == after == full
    assert all(res_of(x).hit_id < lib.REMOTE_MAGIN_NUMBER for x in full)
    fe.close()


def test_empty_local_store_gives_no_hits(gpu):
    rd = Round(64, 0)
    fe = make_frontend()
    fe.db_load(np.stack([np.ctypeslib.as_array(rd.recs[r].global_desc[QDIR]) for r in range(8)]), remote=True)
    st = fh.stream()
    out = filled(9 * RS)
    fe.query_received(rd.rec_ptr(), 9, -1, out.data_ptr(), st, init_mode=[1] * 9)
    fe.finish(st)
    raw = out.cpu().numpy().tobytes()
    for r in range(9):
        res = res_of(raw[r * RS:(r + 1) * RS])
        assert res.accepted == 0 and res.hit_id == -1 and list(res.n_matches) == [0] * ND
    fe.close(); rd.fe.close()


def test_arguments_and_structure(gpu):
    """n = 0 does nothing; n = 65 and null pointers are refused.  One call launches the same kernels for n = 2 and n = 8
    (one scan pass) and one more at n = 9 (the second pass).  The scratch is acquired by the first call only, and destroy
    gives it back."""
    n_start = host.live_resources()
    rd = Round(300, 1)
    fe, st = rd.fe, rd.stream
    out = filled(65 * RS)
    L = fe._lib
    c0, live0 = host.launch_count(), host.live_resources()
    fe.query_received(rd.rec_ptr(), 0, -1, out.data_ptr(), st)
    L.osb_frontend_query_received(fe._h, None, 0, -1, None, None, None)
    assert host.launch_count() == c0 and host.live_resources() == live0
    for args in ((rd.rec_ptr(), 65), (None, 2), (rd.rec_ptr(), -1)):
        assert L.osb_frontend_query_received(fe._h, args[0], args[1], -1, None, out.data_ptr(), st) == lib.ERR_INVALID
    assert L.osb_frontend_query_received(fe._h, rd.rec_ptr(), 2, -1, None, None, st) == lib.ERR_INVALID
    assert L.osb_frontend_query_received(None, rd.rec_ptr(), 2, -1, None, out.data_ptr(), st) == lib.ERR_INVALID
    torch.cuda.synchronize()
    assert (out == FILL).all() and host.launch_count() == c0 and host.live_resources() == live0
    rd.batch(1)
    live1 = host.live_resources()
    assert live1 > live0                     # the first call acquired the batch scratch, not create
    counts = {}
    for n in (2, 8, 9, 64, 2):
        c = host.launch_count()
        rd.batch(n)
        counts[n] = host.launch_count() - c
    assert counts[2] == counts[8] and counts[9] == counts[8] + 1 and counts[64] == counts[8] + 7, counts
    assert host.live_resources() == live1
    fe.close()
    assert host.live_resources() == n_start
