"""GPU: fp16 row storage of the keyframe databases (OSB_DB_STORAGE_FP16).

The contract: an fp16 store returns byte-identical ids and scores to an fp32 store holding the same rows already rounded to
fp16 (numpy float16, round to nearest even) -- on both scan kernels, both merges, every pass width -- and a front-end in
fp16 writes byte-identical results to an fp32 front-end fed copies of the same records with pre-rounded global
descriptors, while both are queried with the original records.  Small-integer rows are exact in fp16, so with them the
fp16 store must equal oracle/frontend_ref.py::IndexFlatIP bit for bit."""
import ctypes as C

import numpy as np
import pytest

from omniswarm_b200 import host, lib, synth
from oracle import db_storage_ref as dsr
from oracle import frontend_ref as fr
from frontend_harness import EB, RS, filled, upload
import frontend_harness as fh

pytestmark = pytest.mark.gpu

DB_CHUNK_MAX, DB_COOP_CHUNK, DB_MERGE_MAX = 512, 64, 3584
KS = (1, 6, 16, 17, 64)
NQS = (1, 2, 5, 8, 9, 130)


@pytest.fixture(scope="module")
def sms(gpu):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def layout(n, sms):
    """(grid, chunk) of a search over n rows, as csrc/match.cu's db_scan_grid sizes it"""
    grid, chunk = 2 * sms, -(-max(n, 1) // (2 * sms))
    if chunk > DB_CHUNK_MAX:
        chunk, grid = DB_CHUNK_MAX, -(-n // DB_CHUNK_MAX)
    return grid, chunk


def special_rows(n, dim, seed):
    """unit-norm Gaussian rows; in some rows +-0, fp16 subnormals, exact halfway cases (which round to even) and one
    element >= 65520 (-> +-inf: one per row, so that no score is inf - inf)"""
    rng = np.random.default_rng(seed)
    x = rng.standard_normal((n, dim), dtype=np.float32)
    x /= np.linalg.norm(x, axis=1, keepdims=True)
    m = min(n, 40)
    rows = rng.choice(n, m, replace=False)
    for i, r in enumerate(rows):
        cols = rng.choice(dim, min(dim, 8), replace=False)
        kind = i % 4
        if kind == 0:
            x[r, cols] = np.array([0.0, -0.0] * 4, np.float32)[: len(cols)]
        elif kind == 1:          # subnormal halves (below 2^-14) and halfway points between them
            x[r, cols] = (rng.integers(1, 1023, len(cols)) * 2.0 ** -24 + 2.0 ** -25).astype(np.float32) * \
                rng.choice([-1, 1], len(cols))
        elif kind == 2:          # halfway between two normal halves: 2^e (1 + (2j + 1) 2^-11)
            e = rng.integers(-10, 0, len(cols))
            j = rng.integers(0, 1023, len(cols))
            x[r, cols] = (2.0 ** e * (1 + (2 * j + 1) * 2.0 ** -11)).astype(np.float32) * rng.choice([-1, 1], len(cols))
        else:
            x[r, cols[0]] = np.float32(rng.choice([65520.0, -70000.0, 1e30]))
    return x


def both(dim, n, rows):
    """an fp16 store of `rows` and an fp32 store of the rows rounded to fp16"""
    a, b = host.IndexFlatIP(dim, n, storage="fp16"), host.IndexFlatIP(dim, n)
    a.add(rows)
    b.add(dsr.round_rows_fp16(rows))
    return a, b


def same_search(a, b, q, ks, nqs):
    for k in ks:
        for nq in nqs:
            Da, Ia = a.search(q[:nq], k)
            Db, Ib = b.search(q[:nq], k)
            assert Ia.tobytes() == Ib.tobytes(), f"ids differ (nq {nq}, k {k})"
            assert Da.tobytes() == Db.tobytes(), f"scores differ (nq {nq}, k {k})"


# (path, n, dim): n as a function of the SM count
SHAPES = [("coop", lambda s: DB_COOP_CHUNK * 2 * s, 4096), ("coop", lambda s: 1000, 4096),
          ("stream", lambda s: 65 * 2 * s, 4096), ("stream", lambda s: 5000, 256), ("stream", lambda s: 3000, 64)]


@pytest.mark.parametrize("kind,nfn,dim", SHAPES, ids=["coop_full", "coop_1000", "stream_4096", "stream_256", "stream_64"])
def test_identity_with_prerounded_fp32_store(sms, kind, nfn, dim):
    n = nfn(sms)
    grid, chunk = layout(n, sms)
    assert (dim == 4096 and chunk <= DB_COOP_CHUNK) == (kind == "coop")
    rows = special_rows(n, dim, seed=n + dim)
    q = np.random.default_rng(dim).standard_normal((130, dim)).astype(np.float32)
    a, b = both(dim, n, rows)
    same_search(a, b, q, KS, NQS)
    D, _ = a.search(q[:9], 64)
    assert np.isinf(D).any() and np.isfinite(D).any()          # the overflowed rows were scanned as +-inf
    a.close(); b.close()


def test_identity_unfused_merge_forced_by_grid(sms):
    """more than 512 x 3584 rows: the grid exceeds the fused merge's limit"""
    n = DB_CHUNK_MAX * DB_MERGE_MAX + 1000
    assert layout(n, sms)[0] > DB_MERGE_MAX
    rows = special_rows(n, 64, seed=3)
    q = np.random.default_rng(4).standard_normal((9, 64)).astype(np.float32)
    a, b = both(64, n, rows)
    same_search(a, b, q, (1, 16, 17, 64), (1, 2, 5, 9))
    a.close(); b.close()


def plant_ties(rows, q, chunk, k):
    """rows chunk-1 and chunk (across the first CTA boundary) are query 0's best row, and 2k + 8 copies of a weaker row
    straddle the k-th slot, next to the boundary and spread over the store"""
    n, dim = rows.shape
    best = np.sign(q[0]) * 3
    rows[chunk - 1] = rows[chunk] = best
    mid = best.copy()
    mid[: dim // 2] = 0
    rows[chunk + 1: chunk + 1 + k + 4] = mid
    rows[np.linspace(chunk + k + 5, n - 1, k + 4).astype(int)] = mid


@pytest.mark.parametrize("kind,nfn,dim", [SHAPES[0], SHAPES[2], SHAPES[3]], ids=["coop", "stream_4096", "stream_256"])
def test_exact_selection_against_oracle(sms, kind, nfn, dim):
    n = nfn(sms)
    _, chunk = layout(n, sms)
    rng = np.random.default_rng(n)
    rows = rng.integers(-3, 4, (n, dim)).astype(np.float32)
    q = rng.integers(-3, 4, (130, dim)).astype(np.float32)
    plant_ties(rows, q, chunk, 64)
    idx = host.IndexFlatIP(dim, n, storage="fp16")
    idx.add(rows)
    ref = fr.IndexFlatIP(dim)
    ref.add(rows)
    Dr, Ir = ref.search(q, 64)
    for k in KS:
        for nq in NQS:
            D, I = idx.search(q[:nq], k)
            assert np.array_equal(I, Ir[:nq, :k]) and np.array_equal(D, Dr[:nq, :k]), (nq, k)
    assert idx.search(q[:1], 2)[1][0].tolist() == [chunk - 1, chunk]
    idx.close()


def test_add_paths_capacity_and_reset(gpu):
    import torch
    dim, n = 4096, 1000
    rows = special_rows(n, dim, seed=11)
    q = np.random.default_rng(12).standard_normal((9, dim)).astype(np.float32)
    ref = host.IndexFlatIP(dim, n)
    ref.add(dsr.round_rows_fp16(rows))
    one = host.IndexFlatIP(dim, n, storage="fp16")
    assert one.add(rows) == 0
    ragged = host.IndexFlatIP(dim, n, storage="fp16")         # host adds staged 64 rows at a time, ragged ends
    for a, b in ((0, 1), (1, 65), (65, 193), (193, 700), (700, n)):
        assert ragged.add(rows[a:b]) == a
    dev = host.IndexFlatIP(dim, n, storage="fp16")
    t = torch.from_numpy(rows).cuda()
    st = torch.cuda.current_stream().cuda_stream
    assert dev.add_dev(t.data_ptr(), 300, st) == 0
    assert dev.add_dev(t[300:].data_ptr(), n - 300, st) == 300
    torch.cuda.synchronize()
    for idx in (one, ragged, dev):
        assert idx.ntotal == n
        same_search(idx, ref, q, (6, 17), (1, 9))
    # capacity: refused, nothing added
    with pytest.raises(lib.OsbError) as e:
        one.add(rows[:1])
    assert e.value.status == lib.ERR_CAPACITY and one.ntotal == n
    # reset keeps the storage
    one.reset()
    assert one.ntotal == 0 and (one.search(q[:2], 6)[1] == -1).all()
    one.add(rows[:500])
    ref.reset()
    ref.add(dsr.round_rows_fp16(rows[:500]))
    same_search(one, ref, q, (6, 64), (1, 9))
    h = C.c_void_p()
    for bad in (2, -1):
        assert gpu.osb_db_create_storage(C.byref(h), dim, 16, bad) == lib.ERR_INVALID
    for idx in (ref, one, ragged, dev):
        idx.close()


# ---------------------------------------------------------------------------------------------------------------------
# front-end
# ---------------------------------------------------------------------------------------------------------------------
ND, MN = 4, 200
QDIR = 1
SC, NPT, DESC = synth.LOOP_SCENE, synth.LOOP_NPT, synth.LOOP_DESC
CONFIG = dict(init_mode_product_thres=0.2, match_index_dist=2, ransac_seed=0)


def make_frontend(cap, gf, storage=None):
    fe = fh.make_frontend(CONFIG, db_capacity=cap, geometric_filter=bool(gf))
    if storage:
        fe.set_db_storage(storage)
    if gf:
        fe.set_cameras(SC["K"], SC["ext"], SC["ext"], 0.006)
        fe.set_loop_params(odometry_consistency_threshold=10.0, seed=3)
    return fe


def record(drone, msg, side, g, seed=0):
    """a keyframe of synth.loop_scene without outlier matches; global descriptor g [ND][4096]"""
    return synth.loop_record(drone, msg, side, seed, g, n_outliers=0)


def rounded(rec):
    """a copy of the record whose global descriptors are what an fp16 store keeps of them"""
    c = lib.KeyframeRecord.from_buffer_copy(bytes(rec))
    g = np.ctypeslib.as_array(c.global_desc)
    g[:] = dsr.round_rows_fp16(g)
    return c


class Pair:
    """an fp32 front-end fed pre-rounded copies and an fp16 one fed the originals, built the same way: own keyframes,
    rows from db_load (with local descriptors and geometry unless `large`), foreign keyframes ingested into the remote
    store"""

    def __init__(self, n_loaded, gf, large):
        self.gf = gf
        self.st = fh.stream()
        cap = n_loaded + 64 * ND + 16 * ND
        self.a, self.b = make_frontend(cap, gf), make_frontend(cap, gf, "fp16")
        self.g = synth.descriptor_db(n_loaded, 4096, 11)
        g_old = synth.descriptor_db(ND, 4096, 5)
        self.old = record(1, 100, "old", g_old)
        own = [self.old] + [record(1, 101 + i, "old", synth.descriptor_db(ND, 4096, 60 + i)) for i in range(3)]
        for r in own:
            self.each(lambda fe, rec: fe.ingest_own(upload([rec]).data_ptr(), self.st), r)
        n_own = len(own) * ND
        for fe, g in ((self.a, dsr.round_rows_fp16(self.g)), (self.b, self.g)):
            if large:
                fe.db_load(g)
                continue
            ld = np.zeros((n_loaded, MN, 64), np.float32)
            ld[:, :NPT] = DESC[QDIR]
            kp = np.zeros((n_loaded, MN, 2), np.float32)
            kp[:, :NPT] = SC["kp_old"][QDIR]
            sm = np.full((n_loaded, MN), -1, np.int32)
            sm[:, :NPT] = 0
            fe.db_load(g, ld, np.full(n_loaded, NPT, np.int32))
            fe.db_set_geometry(n_own, kp, sm)
        # foreign keyframes: near the old keyframe, near loaded rows, and unrelated; the first 16 go to the remote store
        rng = np.random.default_rng(9)
        self.recs = []
        for r in range(64):
            if r % 3 == 0:
                g = g_old + rng.normal(0, (0.05 + 0.3 * (r % 4)) / 64, g_old.shape).astype(np.float32)
            elif r % 3 == 1:
                g = np.stack([synth.noisy_queries(self.g, np.array([int(rng.integers(0, n_loaded))]),
                                                  sigma=[0.3, 2.0, 3.2, 6.0][r % 4], seed=r)[0]] * ND)
            else:
                g = synth.descriptor_db(ND, 4096, 300 + r)
            g = g / np.linalg.norm(g, axis=1, keepdims=True)
            self.recs.append(record(2 + r % 3, 300 + r, "new", g.astype(np.float32), seed=20 + r))
        self.recs_t = upload(self.recs)
        self.each(lambda fe, t: fe.ingest(t.data_ptr(), 16, -1, self.st), self.recs[:16], upload)
        self.a.finish(self.st); self.b.finish(self.st)

    def each(self, fn, recs, conv=lambda r: r):
        """fn(fp32 handle, pre-rounded records); fn(fp16 handle, original records)"""
        pre = [rounded(r) for r in recs] if isinstance(recs, list) else rounded(recs)
        fn(self.a, conv(pre))
        fn(self.b, conv(recs))

    def query(self, rec_t, nonkeyframe):
        out = []
        for fe in (self.a, self.b):
            res = filled(RS)
            fe.query(rec_t.data_ptr(), res.data_ptr(), self.st, nonkeyframe=nonkeyframe)
            fe.finish(self.st)
            out.append(res)
        return out

    def received(self, n, init):
        out = []
        for fe in (self.a, self.b):
            res = filled(n * RS)
            fe.query_received(self.recs_t.data_ptr(), n, -1, res.data_ptr(), self.st, init_mode=init)
            fe.finish(self.st)
            out.append(res)
        return out

    def loop(self, rec_t, res_pair, cands):
        out = []
        for fe, res in zip((self.a, self.b), res_pair):
            e = filled(len(cands) * EB)
            fe.compute_loop(rec_t.data_ptr(), res.data_ptr(), cands, e.data_ptr(), self.st)
            fe.finish(self.st)
            out.append(e.cpu().numpy().tobytes())
        return out


@pytest.mark.parametrize("large", [False, True], ids=["coop_scan", "row_scan"])
@pytest.mark.parametrize("gf", [0, 1])
def test_frontend_identity(gpu, large, gf):
    import torch
    coop = 64 * 2 * torch.cuda.get_device_properties(0).multi_processor_count
    p = Pair(coop + 3000 if large else 300, gf, large)
    accepted = 0
    # own keyframe: ingest (pre-rounded copy into the fp32 handle), then query with the original record.  Its descriptors
    # are the old keyframe's at inner product ~0.86, so that the received keyframes near the old one hit the old one.
    g_new = synth.descriptor_db(ND, 4096, 5) + np.random.default_rng(1).normal(0, 0.6 / 64, (ND, 4096))
    new = record(1, 200, "new", (g_new / np.linalg.norm(g_new, axis=1, keepdims=True)).astype(np.float32), seed=1)
    nt = upload([new])
    p.each(lambda fe, rec: fe.ingest_own(upload([rec]).data_ptr(), p.st), new)
    for nonkey in (False, True):
        a, b = p.query(nt, nonkey)
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), f"query (nonkeyframe {nonkey}) differs"
        r = fh.results(a, 1)[0]
        accepted += r.accepted
        if gf and r.accepted:
            cand = dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"], odom_rel=SC["delta_true"], cov=np.eye(6) * 0.01)
            ea, eb = p.loop(nt, (a, b), [cand])
            assert ea == eb, "compute_loop of the own query differs"
    # a round received from the swarm
    for n in (1, 8, 9, 64):
        init = [r % 3 == 1 for r in range(n)]
        a, b = p.received(n, init)
        assert a.cpu().numpy().tobytes() == b.cpu().numpy().tobytes(), f"query_received n={n} differs"
        res = fh.results(a, n)
        accepted += sum(x.accepted for x in res)
        if gf and n == 64:
            cands = [dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"], init_mode=init[r]) for r in range(n)]
            ea, eb = p.loop(p.recs_t, (a, b), cands)
            assert ea == eb, "compute_loop of the received round differs"
            edges = [lib.LoopEdgeResult.from_buffer_copy(ea[i * EB:(i + 1) * EB]) for i in range(n)]
            assert any(e.status == lib.LOOP_ACCEPTED for e in edges)
        if n == 64:   # hits on own keyframes and on db_load rows, and misses
            hits = {x.hit_msg_id for x in res if x.accepted}
            assert 100 in hits and -1 in hits and not all(x.accepted for x in res), hits
    assert accepted >= 10
    p.a.close(); p.b.close()


def test_setter_rules_memory_and_resources(gpu):
    import torch
    st = torch.cuda.current_stream().cuda_stream
    live0 = host.live_resources()
    g = synth.descriptor_db(8, 4096, 3)
    # bad values
    fe = make_frontend(64, 0)
    for bad in (2, -1):
        assert fe._lib.osb_frontend_set_db_storage(fe._h, bad) == lib.ERR_INVALID
    with pytest.raises(ValueError):
        fe.set_db_storage("bf16")
    # after db_load, in either store; db_reset makes it valid again and keeps the storage
    fe.set_db_storage("fp16")
    for remote in (False, True):
        fe.db_load(g, remote=remote)
        assert fe._lib.osb_frontend_set_db_storage(fe._h, lib.DB_STORAGE_FP32) == lib.ERR_INVALID
        fe.db_reset()
    # after an ingest that has not been synchronised
    rt = upload([record(1, 5, "old", g[:ND])])
    fe.ingest_own(rt.data_ptr(), st)
    assert fe._lib.osb_frontend_set_db_storage(fe._h, lib.DB_STORAGE_FP32) == lib.ERR_INVALID
    fe.finish(st)
    # the refused calls changed nothing: the store still rounds to fp16 -- it answers like a pre-rounded fp32 store
    ref = make_frontend(64, 0)
    rr = upload([rounded(record(1, 5, "old", g[:ND]))])
    ref.ingest_own(rr.data_ptr(), st)
    q = upload([record(2, 9, "new", g[:ND] + np.float32(1e-3), seed=3)])
    outs = []
    for h in (fe, ref):
        o = filled(RS)
        h.query_received(q.data_ptr(), 1, -1, o.data_ptr(), st)
        h.finish(st)
        outs.append(o.cpu().numpy().tobytes())
    assert outs[0] == outs[1] and lib.LoopResult.from_buffer_copy(outs[0]).accepted
    fe.close(); ref.close()
    # fp32 -> fp16 -> fp32 while empty: an fp32 handle
    t1, t2 = make_frontend(64, 0), make_frontend(64, 0)
    t1.set_db_storage("fp16"); t1.set_db_storage("fp32")
    r0 = upload([record(1, 5, "old", g[:ND])])
    outs = []
    for h in (t1, t2):
        h.ingest_own(r0.data_ptr(), st)
        o = filled(RS)
        h.query_received(q.data_ptr(), 1, -1, o.data_ptr(), st)
        h.finish(st)
        outs.append(o.cpu().numpy().tobytes())
    assert outs[0] == outs[1]
    t1.close(); t2.close()
    # device memory: the two row planes shrink by cap x 8 KB each; the resource count is unchanged
    cap = 20000
    big = make_frontend(cap, 0)
    live1 = host.live_resources()
    torch.cuda.synchronize()
    free0 = torch.cuda.mem_get_info()[0]
    big.set_db_storage("fp16")
    free1 = torch.cuda.mem_get_info()[0]
    want = 2 * cap * 4096 * 2
    assert abs((free1 - free0) - want) <= 8 << 20, (free1 - free0, want)
    assert host.live_resources() == live1
    big.set_db_storage("fp32")
    assert abs(torch.cuda.mem_get_info()[0] - free0) <= 8 << 20
    big.close()
    assert host.live_resources() == live0
