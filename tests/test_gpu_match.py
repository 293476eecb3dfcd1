"""GPU parity: keyframe database (faiss::IndexFlatIP replacement) and cross-check matcher (cv::BFMatcher replacement)
against the oracle, through the C ABI."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from omniswarm_b200 import synth, host
from oracle import frontend_ref as fr

pytestmark = pytest.mark.gpu


def test_db_search_matches_oracle(gpu):
    db = synth.descriptor_db(3000, 4096, 1)
    idx = host.IndexFlatIP(4096, capacity=4096)
    assert idx.add(db[:1000]) == 0 and idx.add(db[1000:]) == 1000 and idx.ntotal == 3000
    ref = fr.IndexFlatIP(4096); ref.add(db)
    rows = np.array([0, 17, 1500, 2999, 42, 43, 44, 45, 46, 47, 48])      # 11 queries: exercises Q=8 + Q=4 paths
    q = synth.noisy_queries(db, rows)
    for k in (1, 6, 10, 32):
        D, I = idx.search(q, k)
        Dr, Ir = ref.search(q, k)
        assert np.array_equal(I, Ir), f"ids differ at k={k}"                # bit-exact indices
        assert np.allclose(D, Dr, rtol=1e-5, atol=1e-6)
        assert (I[:, 0] == rows).all()
    for nq in (1, 2, 3, 5):
        D, I = idx.search(q[:nq], 6)
        assert np.array_equal(I, ref.search(q[:nq], 6)[1])


def test_db_search_golden(gpu):
    z = np.load(os.path.join(GOLDEN, "db_search.npz"))
    db = synth.descriptor_db(300, 4096, 1)
    idx = host.IndexFlatIP(4096, capacity=512); idx.add(db)
    D, I = idx.search(synth.noisy_queries(db, z["rows"]), 10)
    assert np.array_equal(I, z["I"]) and np.allclose(D, z["D"], rtol=1e-5, atol=1e-6)


def test_db_edge_cases(gpu):
    idx = host.IndexFlatIP(64, capacity=16)
    q = np.ones((1, 64), np.float32)
    D, I = idx.search(q, 5)                                    # empty database
    assert (I == -1).all() and np.isneginf(D).all()
    rows = np.zeros((3, 64), np.float32); rows[:, 0] = [1, 1, 2]   # exact tie between rows 0 and 1
    idx.add(rows)
    D, I = idx.search(q, 5)                                    # fewer rows than k: -1 / -inf padding
    assert I[0].tolist() == [2, 0, 1, -1, -1] and D[0, :3].tolist() == [2.0, 1.0, 1.0] and np.isneginf(D[0, 3:]).all()
    with pytest.raises(host._l.OsbError) as e:                # capacity
        idx.add(np.zeros((14, 64), np.float32))
    assert e.value.status == host._l.ERR_CAPACITY
    idx.reset(); assert idx.ntotal == 0


def test_db_full_size_property(gpu):
    """BASELINE size (10k rows): every row queried as itself comes back first (self inner product = 1)."""
    db = synth.descriptor_db(10000, 4096, 1)
    idx = host.IndexFlatIP(4096, capacity=10000); idx.add(db)
    rows = np.arange(0, 10000, 397)
    D, I = idx.search(db[rows], 6)
    assert (I[:, 0] == rows).all() and np.allclose(D[:, 0], 1.0, atol=1e-5)
    assert (np.diff(D, axis=1) <= 0).all()                     # descending


def test_db_streaming_path_with_ties(gpu):
    """> 64 rows per CTA: the warp-per-row streaming kernel (the 50 k-row sweep's path), fused and unfused merge; exact
    duplicates far apart must come back in ascending row order."""
    n = 24000
    db = synth.descriptor_db(n, 4096, 3)
    db[23000] = db[5]; db[12000] = db[5]
    idx = host.IndexFlatIP(4096, capacity=n); idx.add(db)
    ref = fr.IndexFlatIP(4096); ref.add(db)
    q = synth.noisy_queries(db, np.array([5, 9000, 23999]))
    for k in (6, 10, 40):                                      # 296 CTAs x 40 candidates > 4096: separate merge kernel
        D, I = idx.search(q, k)
        Dr, Ir = ref.search(q, k)
        assert np.array_equal(I, Ir), f"ids differ at k={k}"
        assert np.allclose(D, Dr, rtol=1e-5, atol=1e-6)
    assert idx.search(db[5][None], 3)[1][0].tolist() == [5, 12000, 23000]


def test_db_repeated_searches_reuse_the_ticket(gpu):
    """the fused merge's ticket counter must be back at zero after every search (same handle, many searches)."""
    db = synth.descriptor_db(2000, 4096, 4)
    idx = host.IndexFlatIP(4096, capacity=2048); idx.add(db)
    ref = fr.IndexFlatIP(4096); ref.add(db)
    for i in range(6):
        q = synth.noisy_queries(db, np.array([i * 300, i * 300 + 1]))
        assert np.array_equal(idx.search(q, 7)[1], ref.search(q, 7)[1])


def test_row_sharded_merge(gpu):
    """SURVEY 8e alternative: three shards scanned separately, candidates merged by osb_topk_merge_dev == unsharded."""
    import ctypes as C
    import torch
    from omniswarm_b200 import swarm, lib
    n, k = 1000, 8
    db = synth.descriptor_db(n, 4096, 6)
    db[900] = db[10]                                           # tie across shards
    ref = fr.IndexFlatIP(4096); ref.add(db)
    q = np.concatenate([synth.noisy_queries(db, np.array([10, 500])), db[900][None]])
    Dr, Ir = ref.search(q, k)
    spans = [swarm.shard_rows(n, r, 3) for r in range(3)]
    cs, ci = [], []
    for a, b in spans:
        sh = host.IndexFlatIP(4096, capacity=b - a); sh.add(db[a:b])
        D, I = sh.search(q, k)
        cs.append(D); ci.append(I); sh.close()
    cand_s = torch.from_numpy(np.stack(cs, 1).copy()).cuda()    # [nq][n_lists][k]
    cand_i = torch.from_numpy(np.stack(ci, 1).copy()).cuda()
    offs = torch.tensor([a for a, _ in spans], dtype=torch.int64).cuda()
    out_s = torch.empty(3, k, dtype=torch.float32, device="cuda"); out_i = torch.empty(3, k, dtype=torch.int64, device="cuda")
    L = lib.load()
    lib.check(L.osb_topk_merge_dev(3, 3, k, C.c_void_p(cand_s.data_ptr()), C.c_void_p(cand_i.data_ptr()),
                                   C.c_void_p(offs.data_ptr()), C.c_void_p(out_s.data_ptr()), C.c_void_p(out_i.data_ptr()),
                                   C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert np.array_equal(out_i.cpu().numpy(), Ir) and np.allclose(out_s.cpu().numpy(), Dr, rtol=1e-5, atol=1e-6)
    assert out_i[2, :2].tolist() == [10, 900]
    # the single-rank RowShardedIndex is the same machinery with one list
    rs = swarm.RowShardedIndex(db, n, device="cuda")
    s1, i1 = rs.search(torch.from_numpy(q[0]).cuda(), k)
    torch.cuda.synchronize()
    assert np.array_equal(i1.cpu().numpy(), Ir[0])
    rs.close()


def test_matcher_matches_oracle_and_cv2(gpu):
    m = host.BFMatcher(max_pairs=8, max_n=200)
    qs, ts = [], []
    for seed, (nq, nt) in enumerate([(200, 200), (57, 43), (1, 5), (5, 1), (0, 10), (10, 0), (200, 13), (64, 200)]):
        a = synth.local_descriptors(max(nq, 1), 30 + seed)[:nq]
        b = (synth.local_descriptors(nt, 40 + seed, base=a) if 0 < nt <= nq else synth.local_descriptors(max(nt, 1), 40 + seed)[:nt])
        qs.append(a); ts.append(b)
    out = m.match_batch(qs, ts)
    for (qi, ti, dist), a, b in zip(out, qs, ts):
        rq, rt, rd = fr.bf_crosscheck(a, b)
        assert np.array_equal(qi, rq) and np.array_equal(ti, rt)   # bit-exact index pairs
        assert np.array_equal(dist, rd)                            # same f32 accumulation order -> same bits
    try:
        import cv2
        ms = sorted(cv2.BFMatcher(cv2.NORM_L2, True).match(qs[0], ts[0]), key=lambda x: x.queryIdx)
        assert [x.queryIdx for x in ms] == out[0][0].tolist() and [x.trainIdx for x in ms] == out[0][1].tolist()
    except ImportError:
        pass


def test_matcher_golden_and_ties(gpu):
    z = np.load(os.path.join(GOLDEN, "matcher.npz"))
    m = host.BFMatcher(max_pairs=2, max_n=200)
    qi, ti, dist = m.match(z["q"], z["t"])
    assert np.array_equal(qi, z["qi"]) and np.array_equal(ti, z["ti"]) and np.array_equal(dist, z["dist"])
    # duplicated train rows: the FIRST minimum wins in both directions
    a = synth.local_descriptors(20, 7)
    b = np.concatenate([a[:10], a[:10]], 0)
    qi, ti, dist = m.match(a, b)
    assert qi.tolist() == list(range(10)) and ti.tolist() == list(range(10)) and (dist == 0).all()


def test_matcher_at_its_cap(gpu):
    """max_n = 256, the largest the matcher accepts: 256 x 256 and 256 x 1 pairs, bit-exact"""
    m = host.BFMatcher(max_pairs=2, max_n=256)
    a = synth.local_descriptors(256, 50)
    qs = [a, synth.local_descriptors(256, 51)]
    ts = [synth.local_descriptors(256, 52, base=a), synth.local_descriptors(1, 53)]
    for (qi, ti, dist), q, t in zip(m.match_batch(qs, ts), qs, ts):
        rq, rt, rd = fr.bf_crosscheck(q, t)
        assert np.array_equal(qi, rq) and np.array_equal(ti, rt) and np.array_equal(dist, rd)
    assert len(rq) == 1
    m.close()
