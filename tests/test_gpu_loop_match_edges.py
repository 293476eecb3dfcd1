"""GPU: the loop matcher's stage between the database scan and PnP -- the cross-check matcher (match.cu), the homography
RANSAC of the geometric filter (geom.cu) and the front-end's filter path around it (keyframe.cu), and the stereo / depth
lift that sets landmarks_flag and landmarks_3d (lift.cu) -- on every launch shape and at their numerical edges, against
oracle/frontend_ref.bf_crosscheck, oracle/geometry_ref and oracle/lift_ref.

Every scenario also asserts that it reaches what it is built for (a tie, a second warp pass, a clamp, a zero-disparity
pair, ...), so that a change to the synthetic data cannot quietly disarm it."""
import ctypes as C

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib, synth
from oracle import frontend_ref as fr, geometry_ref as gr, lift_ref as lr, pcm_ref as pr
from test_oracle_pins import _homography_case
import frontend_harness as fh

pytestmark = pytest.mark.gpu

DIM = 64
NS = (0, 1, 15, 16, 17, 31, 32, 33, 63, 64, 65, 199, 200, 255, 256)      # around the 16-row tile and the 32 stride


def _vp(t):
    return C.c_void_p(t.data_ptr())


# ---- 1. cross-check matcher ------------------------------------------------------------------------------------------
def _desc_pair(nq, nt, seed):
    """random query / train rows; three quarters of the smaller side have a noisy partner on the other"""
    rng = np.random.default_rng(seed)
    q = rng.standard_normal((nq, DIM)).astype(np.float32)
    t = rng.standard_normal((nt, DIM)).astype(np.float32)
    k = min(nq, nt) * 3 // 4
    if k:
        t[rng.choice(nt, k, replace=False)] = q[rng.choice(nq, k, replace=False)] + \
            np.float32(0.15) * rng.standard_normal((k, DIM)).astype(np.float32)
    return q, t


def _shapes(max_n):
    """every value of NS up to max_n meets its neighbour, one of the three largest and one of the three smallest values"""
    v = [x for x in NS if x <= max_n]
    out = []
    for i, a in enumerate(v):
        out += [(a, v[(i + 1) % len(v)]), (v[(i + 1) % len(v)], a), (a, v[-1 - i % 3]), (v[i % 3], a)]
    return out


def _match_dev(m, qs, ts, stream):
    """osb_matcher_match_dev on torch tensors and `stream` -> [(qi, ti, dist)], n_out; outputs start as sentinels"""
    P, mn = len(qs), m.max_n
    q = torch.zeros(P, mn, DIM, device="cuda"); t = torch.zeros(P, mn, DIM, device="cuda")
    for p in range(P):
        if len(qs[p]):
            q[p, :len(qs[p])] = torch.from_numpy(qs[p])
        if len(ts[p]):
            t[p, :len(ts[p])] = torch.from_numpy(ts[p])
    nq = torch.tensor([len(x) for x in qs], dtype=torch.int32, device="cuda")
    nt = torch.tensor([len(x) for x in ts], dtype=torch.int32, device="cuda")
    qi = torch.full((P * mn,), -7, dtype=torch.int32, device="cuda"); ti = torch.full_like(qi, -7)
    dist = torch.full((P * mn,), float("nan"), device="cuda"); n_out = torch.full((P,), -7, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    lib.check(lib.load().osb_matcher_match_dev(m._h, P, _vp(q), _vp(nq), _vp(t), _vp(nt), _vp(qi), _vp(ti), _vp(dist),
                                               _vp(n_out), C.c_void_p(stream.cuda_stream)))
    stream.synchronize()
    qi, ti, dist, n = qi.cpu().numpy(), ti.cpu().numpy(), dist.cpu().numpy(), n_out.cpu().numpy()
    return [(qi[p * mn:p * mn + n[p]], ti[p * mn:p * mn + n[p]], dist[p * mn:p * mn + n[p]]) for p in range(P)]


def _check_matches(m, qs, ts, stream):
    """host and _dev forms of one batch, both bit-identical to bf_crosscheck -> the oracle's matches"""
    ref = [fr.bf_crosscheck(a, b) for a, b in zip(qs, ts)]
    got = m.match_batch(qs, ts)
    dev = _match_dev(m, qs, ts, stream)
    for p, (r, g, d) in enumerate(zip(ref, got, dev)):
        for k in range(3):
            assert np.array_equal(g[k], r[k]), (p, len(qs[p]), len(ts[p]), k)
            assert np.array_equal(d[k], g[k]), (p, len(qs[p]), len(ts[p]), k)
        assert g[2].dtype == np.float32 and np.array_equal(g[2].view(np.uint32), r[2].view(np.uint32))
    return ref


@pytest.mark.parametrize("max_n", [17, 200, 256])
def test_matcher_shapes(gpu, max_n):
    """(n_q, n_t) on both sides of the 16-row tile, the 32-column lane stride and the 32-row warp stride, one batch per
    handle, then the same shapes in reverse order on the same handle: every pair's distance block then holds a larger
    pair's stale rows and columns"""
    shapes = _shapes(max_n)
    assert len(shapes) <= 64
    m = host.BFMatcher(max_pairs=64, max_n=max_n)
    stream = torch.cuda.Stream()
    data = [_desc_pair(a, b, 1000 * max_n + i) for i, (a, b) in enumerate(shapes)]
    ref = _check_matches(m, [d[0] for d in data], [d[1] for d in data], stream)
    rev = data[::-1]
    _check_matches(m, [d[0] for d in rev], [d[1] for d in rev], stream)
    assert any(a * b > c * d for (a, b), (c, d) in zip(shapes[::-1], shapes))        # stale, larger blocks underneath
    assert all(len(r[0]) > 0 for (a, b), r in zip(shapes, ref) if a and b)
    if max_n == 256:      # a second row pass of the warps, and matches in the 2nd and the 8th column of a lane
        qi = np.concatenate([r[0] for r in ref]); ti = np.concatenate([r[1] for r in ref])
        assert qi.max() >= 224 and (ti >= 32).any() and (ti >= 224).any()
    # a batch of 64 mixed pairs
    mixed = [_desc_pair(int(a), int(b), 77 + i) for i, (a, b) in
             enumerate(np.random.default_rng(max_n).choice([x for x in NS if x <= max_n], (64, 2)))]
    _check_matches(m, [d[0] for d in mixed], [d[1] for d in mixed], stream)
    m.close()


def _row_ties():
    """query rows 0..3 have two equally near train rows: columns j, j + 32 and j, j + 224 (one lane, different c) and
    j, j + 1 and j, j + 33 (different lanes)"""
    rng = np.random.default_rng(5)
    q = rng.standard_normal((8, DIM)).astype(np.float32)
    t = rng.standard_normal((256, DIM)).astype(np.float32)
    want = {}
    for i, (j, k) in enumerate([(5, 37), (10, 234), (20, 21), (40, 73)]):
        t[j] = t[k] = q[i] + np.float32(0.05) * rng.standard_normal(DIM).astype(np.float32)
        want[i] = j
    return q, t, want


def _col_ties():
    """query rows with identical descriptors -- 0 and 1, 31 and 32 (different warps), 5, 37 and 229 (one warp, passes 1, 2
    and 8): each pair or triple is at the same distance from every train row, so only its smallest row survives"""
    rng = np.random.default_rng(6)
    q = rng.standard_normal((256, DIM)).astype(np.float32)
    for a, b in [(0, 1), (31, 32), (5, 37), (5, 229)]:
        q[b] = q[a]
    t = q[rng.permutation(256)[:200]] + np.float32(0.1) * rng.standard_normal((200, DIM)).astype(np.float32)
    return q, t, [(0, 1), (31, 32), (5, 37), (5, 229)]


def test_matcher_ties(gpu):
    m = host.BFMatcher(max_pairs=8, max_n=256)
    stream = torch.cuda.Stream()
    rq, rt, rwant = _row_ties()
    cq, ct, cdup = _col_ties()
    same = np.repeat(np.random.default_rng(7).standard_normal((1, DIM)).astype(np.float32), 256, 0)
    trains = np.random.default_rng(8).standard_normal((50, DIM)).astype(np.float32)
    zq, zt = np.zeros((40, DIM), np.float32), np.zeros((70, DIM), np.float32)
    qs = [rq, cq, same, same[:33], zq]
    ts = [rt, ct, trains, trains, zt]
    ref = _check_matches(m, qs, ts, stream)
    # row ties resolve to the smaller column, and those are the matches
    qi, ti, _ = ref[0]
    got = {int(a): int(b) for a, b in zip(qi, ti)}
    assert all(got.get(i) == j for i, j in rwant.items()), got
    # column ties: only the smallest of equal rows survives, and it does match
    qi, ti, _ = ref[1]
    for a, b in cdup:
        assert a in qi and b not in qi
        assert fr.l2_distance_matrix(cq[[a]], ct).argmin() == fr.l2_distance_matrix(cq[[b]], ct).argmin()
    # every query row identical: exactly one survivor, row 0
    for r in ref[2:4]:
        assert r[0].tolist() == [0]
    # all-zero descriptors: every distance is +0; the only match is (0, 0)
    assert ref[4][0].tolist() == [0] and ref[4][1].tolist() == [0] and ref[4][2].view(np.uint32).tolist() == [0]
    m.close()


# ---- 2. homography RANSAC --------------------------------------------------------------------------------------------
NH = (3, 4, 5, 31, 32, 33, 199, 200, 255, 256)
SEEDS = (0, 1, 0xFFFFFFFF)
_HG_CACHE = {}


def _hg_ref(src, dst, seed, thresh=3.0):
    key = (src.tobytes(), dst.tobytes(), seed, thresh)
    if key not in _HG_CACHE:
        _HG_CACHE[key] = gr.homography_ransac_mask(src, dst, thresh, seed)
    return _HG_CACHE[key]


def _hg_pack(cases, max_n):
    P = len(cases)
    src = np.zeros((P, max_n, 2), np.float32); dst = np.zeros((P, max_n, 2), np.float32)
    for p, (s, d) in enumerate(cases):
        k = min(len(s), max_n)
        src[p, :k] = s[:k]; dst[p, :k] = d[:k]
    return src, dst


def _hg_host(cases, max_n, seed, thresh=3.0):
    """osb_homography_ransac with an explicit max_n -> (mask [P][max_n], n_inl, winner)"""
    P = len(cases)
    src, dst = _hg_pack(cases, max_n)
    n = np.array([len(s) for s, _ in cases], np.int32)
    mask = np.full((P, max_n), 0xAB, np.uint8); ninl = np.full(P, -7, np.int32); win = np.full(P, -7, np.int32)
    lib.check(lib.load().osb_homography_ransac(lib.ptr(src), lib.ptr(dst), lib.ptr(n), P, max_n, float(thresh), int(seed),
                                               lib.ptr(mask), lib.ptr(ninl), lib.ptr(win)))
    return mask, ninl, win


def _hg_dev(cases, max_n, seed, n_dev=None, thresh=3.0):
    """osb_homography_ransac_dev on a caller stream; n_dev may exceed max_n (the kernel clamps, buffers stay max_n long)"""
    P = len(cases)
    src, dst = _hg_pack(cases, max_n)
    n = np.array([len(s) for s, _ in cases] if n_dev is None else n_dev, np.int32)
    ts, td, tn = (torch.from_numpy(a).cuda() for a in (src, dst, n))
    mask = torch.full((P, max_n), 0xAB, dtype=torch.uint8, device="cuda")
    ninl = torch.full((P,), -7, dtype=torch.int32, device="cuda"); win = torch.full_like(ninl, -7)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    lib.check(lib.load().osb_homography_ransac_dev(_vp(ts), _vp(td), _vp(tn), P, max_n, float(thresh), int(seed), _vp(mask),
                                                   _vp(ninl), _vp(win), C.c_void_p(stream.cuda_stream)))
    stream.synchronize()
    return mask.cpu().numpy(), ninl.cpu().numpy(), win.cpu().numpy()


def _check_hg(out, cases, max_n, seed, thresh=3.0):
    mask, ninl, win = out
    for p, (s, d) in enumerate(cases):
        k = min(len(s), max_n)
        rm, rc, rw = _hg_ref(s[:k], d[:k], seed, thresh)
        assert np.array_equal(mask[p, :k], rm) and ninl[p] == rc and win[p] == rw, (p, len(s), max_n, seed)
        assert not mask[p, k:].any(), (p, len(s), max_n)                   # the tail of a short pair is zero


def _hg_cases(ns, salt):
    return [_homography_case(salt + i, n=n, n_out=max(1, n // 3))[:2] for i, n in enumerate(ns)]


@pytest.mark.parametrize("max_n", [4, 37, 200, 256])
def test_homography_shapes(gpu, max_n):
    cases = _hg_cases([n for n in NH if n <= max_n], 100 + max_n)
    for seed in SEEDS:
        _check_hg(_hg_host(cases, max_n, seed), cases, max_n, seed)
        _check_hg(_hg_dev(cases, max_n, seed), cases, max_n, seed)
    assert any(len(s) < max_n for s, _ in cases)                           # a mask tail to check
    assert any(_hg_ref(s, d, 0)[2] >= 0 for s, d in cases) == (max_n >= 4)


def test_homography_256_pairs_in_one_launch(gpu):
    """256 pairs x 8 CTAs in one grid (64 distinct pairs, each four times at different grid positions)"""
    base = _hg_cases([NH[i % len(NH)] for i in range(64)], 500)
    cases = [base[(p * 37) % 64] for p in range(256)]
    _check_hg(_hg_dev(cases, 256, 0xFFFFFFFF), cases, 256, 0xFFFFFFFF)
    assert len({len(s) for s, _ in cases}) == len(NH)


def test_homography_clamps_device_counts(gpu):
    """n_dev above max_n: the kernel uses the first max_n points, as the oracle is given them"""
    cases = _hg_cases([37, 37, 37, 37], 900)
    n_dev = [38, 200, 256, 1000]
    mask, ninl, win = _hg_dev(cases, 37, 1, n_dev=n_dev)
    _check_hg((mask, ninl, win), cases, 37, 1)
    assert (win >= 0).all() and all(n > 37 for n in n_dev)


def _grid(nx, ny, step, x0, y0):
    return np.array([(x0 + step * i, y0 + step * j) for j in range(ny) for i in range(nx)], np.float32)


def _twice_areas(p):
    """|twice-area| of the four triangles of a quadruple"""
    out = []
    for a, b, c in [(0, 1, 2), (3, 1, 2), (0, 3, 2), (0, 1, 3)]:
        out.append(abs((p[b, 0] - p[a, 0]) * (p[c, 1] - p[a, 1]) - (p[c, 0] - p[a, 0]) * (p[b, 1] - p[a, 1])))
    return np.array(out, np.float64)


def _division_free(h, s, d, thresh=3.0):
    """(lhs, rhs) of the oracle's inlier test of one point"""
    x, y = np.float64(s[0]), np.float64(s[1])
    w = (h[6] * x + h[7] * y) + h[8]
    px = (h[0] * x + h[1] * y) + h[2]
    py = (h[3] * x + h[4] * y) + h[5]
    ex = np.float64(d[0]) * w - px
    ey = np.float64(d[1]) * w - py
    t2 = np.float64(thresh) * np.float64(thresh)
    return ex * ex + ey * ey, t2 * (w * w), w


def _winner_h(src, dst, seed, hyp):
    return gr.solve_h(src[gr.draw4(seed, hyp, len(src))], dst[gr.draw4(seed, hyp, len(src))])


def test_homography_numerical_edges(gpu):
    T = np.float32([5.0, 7.0])
    cases, checks = [], []
    # (a) a pure translation of a square's corners and its centre moved exactly 3 px: an inlier (err^2 <= t^2 w^2 holds with
    # equality, every product exact); the next float32 offset is not.  A sample with the centre has two opposite corners,
    # so a collinear triangle: only the corners make a hypothesis
    g = _grid(2, 2, 4, 10, 10)
    for off in (np.float32(3.0), None):
        s = np.concatenate([g, np.float32([[12.0, 12.0]])])
        d = s + T
        d[-1, 0] = d[-1, 0] + off if off is not None else np.nextafter(d[-1, 0] + np.float32(3.0), np.float32(np.inf))
        cases.append((s, d)); checks.append("exact3" if off is not None else "next")
    # (b) a quadruple whose smallest triangle has twice-area exactly 1 px^2 (degenerate) and one with exactly 2 px^2
    for a in (1.0, 2.0):
        s = np.float32([[0, 0], [a, 0], [0, 1], [7, 5]])
        cases.append((s, s + T)); checks.append(f"area{int(a)}")
    # (c) collinear data: every hypothesis degenerate
    x = np.arange(40, dtype=np.float32)
    s = np.stack([x, 2 * x + 1], 1).astype(np.float32)
    cases.append((s, s + T)); checks.append("collinear")
    # (d) a projective map with w = 1 + x / 16 and a source point on its line at infinity (x = -16)
    s = np.float32([[0, 0], [0, 8], [16, 0], [16, 8], [48, 4], [-8, 4], [-12, 8], [0, 4], [16, 4], [-16, 5]])
    w0 = 1.0 + s[:, 0].astype(np.float64) / 16.0
    d = np.zeros_like(s)
    d[:-1] = (s[:-1] / w0[:-1, None]).astype(np.float32)
    d[-1] = (30.0, 30.0)
    cases.append((s, d)); checks.append("w0")
    # (e) two disjoint sets of 8 interleaved in one region, each a translation of its own
    s = np.random.default_rng(1).choice(41 * 41, 16, replace=False)
    s = np.stack([s % 41, s // 41], 1).astype(np.float32)
    d = s.copy(); d[0::2] += np.float32([5, 3]); d[1::2] += np.float32([-40, 25])
    cases.append((s, d)); checks.append("two_sets")
    seed = 0
    max_n = max(len(c[0]) for c in cases)
    for out in (_hg_host(cases, max_n, seed), _hg_dev(cases, max_n, seed)):
        _check_hg(out, cases, max_n, seed)
    mask, ninl, win = _hg_host(cases, max_n, seed)
    for p, what in enumerate(checks):
        s, d = cases[p]
        rm, rc, rw = _hg_ref(s, d, seed)
        if what in ("exact3", "next"):
            lhs, rhs, _ = _division_free(_winner_h(s, d, seed, rw), s[-1], d[-1])
            assert rc == len(s) - (what == "next") and bool(rm[-1]) == (what == "exact3")
            assert (lhs == rhs) if what == "exact3" else (lhs > rhs)
        elif what.startswith("area"):
            assert _twice_areas(s).min() == float(what[-1]) and _twice_areas(s + T).min() == float(what[-1])
            assert (rw, rc) == ((-1, 0) if what == "area1" else (0, 4))
        elif what == "collinear":
            assert rw == -1 and rc == 0 and not mask[p].any()
        elif what == "w0":
            _, _, w = _division_free(_winner_h(s, d, seed, rw), s[-1], d[-1])
            assert w == 0.0 and rm[-1] == 0 and rc == len(s) - 1
        else:
            # hypotheses of both sets reach the full count 8; the smallest index wins
            best = {}
            for hyp in range(gr.N_HYP):
                idx = gr.draw4(seed, hyp, len(s))
                h = None if idx is None else gr.solve_h(s[idx], d[idx])
                if h is not None:
                    m = gr.inliers(h, s, d, 3.0)
                    if m.sum() == 8:
                        best.setdefault("a" if m[0] else "b", []).append(hyp)
            assert rc == 8 and sorted(best) == ["a", "b"] and rw == min(best["a"] + best["b"])
            assert np.array_equal(rm.astype(bool), np.arange(16) % 2 == (0 if rw in best["a"] else 1))


# ---- 3. the matcher and the filter as the front-end launches them ---------------------------------------------------
QDIR, SELF, N_OWN, N_LOAD = 1, 1, 48, 16
RANSAC_SEED = 0xC0FFEE


def _unit_rows(n, seed):
    return synth.descriptor_db(n, 4096, seed)


class FilterRig:
    """a front-end with the geometric filter: N_OWN own 4-direction frames put in through ingest and N_LOAD one-direction
    rows through db_load + db_set_geometry; each round queries 64 foreign records as one received batch, every record
    hitting a planned frame, each direction pair carrying its own case"""

    CASES = ("few", "four", "ties", "full", "empty", "mid", "few", "empty")

    def __init__(self, max_num):
        self.mn = mn = max_num
        self.fe = fh.make_frontend(db_capacity=512, match_index_dist=1, geometric_filter=True, ransac_seed=RANSAC_SEED,
                                   max_num=mn)
        self.st = fh.stream()
        rng = np.random.default_rng(mn)
        g = _unit_rows(N_OWN * 4 + N_LOAD, 31 + mn)
        # stored direction rows: n, local descriptors, integer key points
        self.rows = {}                       # (frame, dir) -> (desc [n,64], kpts [n,2])
        recs = []
        for f in range(N_OWN):
            rec = lib.KeyframeRecord()
            rec.drone_id, rec.msg_id, rec.n_dirs = SELF, 10 + f, 4
            for d in range(4):
                n = mn if (f + d) % 3 == 0 else int(rng.integers(max(4, mn // 2), mn + 1))
                desc = rng.standard_normal((n, DIM)).astype(np.float32)
                kp = rng.integers(0, 90, (n, 2)).astype(np.float32)
                rec.n_kpts[d] = n
                np.ctypeslib.as_array(rec.global_desc[d])[:] = g[4 * f + d]
                np.ctypeslib.as_array(rec.local_desc[d])[:n] = desc
                np.ctypeslib.as_array(rec.kpts[d])[:n] = kp
                np.ctypeslib.as_array(rec.landmarks_flag[d])[:n] = 1
                self.rows[(f, d)] = (desc, kp)
            recs.append(rec)
        t = fh.upload(recs)
        self.fe.ingest(t.data_ptr(), N_OWN, -1, self.st)
        self.fe.finish(self.st)
        assert self.fe.db_size(False) == 4 * N_OWN
        ld = np.zeros((N_LOAD, mn, DIM), np.float32); nk = np.zeros(N_LOAD, np.int32)
        kp = np.zeros((N_LOAD, mn, 2), np.float32)
        for j in range(N_LOAD):
            n = mn if j % 2 else int(rng.integers(4, mn + 1))
            nk[j] = n
            ld[j, :n] = rng.standard_normal((n, DIM)).astype(np.float32)
            kp[j, :n] = rng.integers(0, 90, (n, 2)).astype(np.float32)
            self.rows[(N_OWN + j, QDIR)] = (ld[j, :n], kp[j, :n])
        self.fe.db_load(g[4 * N_OWN:], ld, nk)
        self.fe.db_set_geometry(4 * N_OWN, kp, np.zeros((N_LOAD, mn), np.int32))
        self.g = g

    def target_desc(self, f):
        return self.g[4 * f + QDIR] if f < N_OWN else self.g[4 * N_OWN + f - N_OWN]

    def side(self, case, stored, rng):
        """the new side of one direction pair against stored (desc, kpts) -> (n, desc, kpts, flags)"""
        sd, sk = stored
        mn = self.mn
        if case == "empty":
            return 0, None, None, None
        n = {"few": min(mn, 12), "four": min(mn, 16), "ties": min(mn, 40), "full": mn}.get(case, int(rng.integers(5, mn + 1)))
        desc = rng.standard_normal((n, DIM)).astype(np.float32)
        kp = rng.integers(0, 90, (n, 2)).astype(np.float32)
        k = min(n, len(sd))
        src = rng.permutation(len(sd))[:k]
        dst = rng.permutation(n)[:k]
        desc[dst] = sd[src] + np.float32(0.1) * rng.standard_normal((k, DIM)).astype(np.float32)
        shift = rng.integers(-6, 7, 2).astype(np.float32)
        kp[dst] = sk[src] + shift
        out = rng.uniform(size=k) < 0.25
        kp[dst[out]] += rng.integers(10, 40, (int(out.sum()), 2)).astype(np.float32)
        flags = np.ones(n, np.int32)
        if case == "few":
            flags[:] = 0
            flags[dst[:int(rng.integers(0, 4))]] = 1
        elif case == "four":
            flags[:] = 0
            flags[dst[:4]] = 1
        elif case == "ties" and n >= 4:
            desc[1] = desc[0]; desc[n - 1] = desc[n // 2]                 # equal rows: a column-minimum tie
        elif case == "mid":
            flags = (rng.uniform(size=n) < 0.8).astype(np.int32)
        return n, desc, kp, flags

    def round(self, rnd):
        rng = np.random.default_rng(1000 * self.mn + rnd)
        recs, plan = [], []
        for r in range(64):
            f = (r * 5 + rnd * 17) % (N_OWN + N_LOAD)
            rec = lib.KeyframeRecord()
            rec.drone_id, rec.msg_id, rec.n_dirs = 2 + r % 3, 5000 + 64 * rnd + r, 4
            np.ctypeslib.as_array(rec.global_desc[QDIR])[:] = self.target_desc(f)
            sides = {}
            for d in range(4):
                case = self.CASES[(r + 3 * d + rnd) % len(self.CASES)]
                if d == QDIR and case == "empty":
                    case = "full"                                            # the queried direction has landmarks
                stored = self.rows.get((f, d), self.rows[(f, QDIR)])
                n, desc, kp, flags = self.side(case, stored, rng)
                rec.n_kpts[d] = n
                if n:
                    np.ctypeslib.as_array(rec.local_desc[d])[:n] = desc
                    np.ctypeslib.as_array(rec.kpts[d])[:n] = kp
                    np.ctypeslib.as_array(rec.landmarks_flag[d])[:n] = flags
                sides[d] = (case, n, desc, kp, flags)
            recs.append(rec)
            plan.append((f, sides))
        t = fh.upload(recs)
        out = fh.filled(64 * fh.RS)
        self.fe.query_received(t.data_ptr(), 64, -1, out.data_ptr(), self.st)
        self.fe.finish(self.st)
        return plan, fh.results(out, 64)


def _check_round(rig, plan, res, seen):
    for r, ((f, sides), x) in enumerate(zip(plan, res)):
        assert x.accepted == 1 and x.hit_dir == QDIR and x.swapped == 0, r
        slot = 0
        for dn in [(QDIR + k) % 4 for k in range(4)]:
            case, n, desc, kp, flags = sides[dn]
            stored = rig.rows.get((f, dn))
            if n == 0 or stored is None:
                seen["empty"] += 1
                continue
            assert (x.dir_new[slot], x.dir_old[slot]) == (dn, dn), (r, slot)
            qi, ti, _ = fr.bf_crosscheck(desc, stored[0])
            m = x.n_matches[slot]
            assert m == len(qi) and list(x.match_new[slot][:m]) == qi.tolist(), (r, slot, case)
            assert list(x.match_old[slot][:m]) == ti.tolist(), (r, slot, case)
            ref = gr.loop_pair_filter(qi.tolist(), ti.tolist(), flags, kp, stored[1], 3.0, seed=RANSAC_SEED)
            g = x.n_geo[slot]
            if ref is None:
                assert x.geo_valid[slot] == 0 and g == 0, (r, slot, case)
                seen["invalid"] += 1
            else:
                qn, qo = ref
                assert x.geo_valid[slot] == 1 and g == len(qn), (r, slot, case, g, len(qn))
                assert list(x.geo_new[slot][:g]) == qn.tolist() and list(x.geo_old[slot][:g]) == qo.tolist(), (r, slot)
                seen["valid"] += 1
                seen["four"] += int(int(sum(flags[q] for q in qi)) == 4)
                seen["reduced"] += int(0 < g < int(sum(flags[q] for q in qi)))
            seen["ties"] += int(case == "ties" and n >= 4 and 1 not in qi.tolist() and 0 in qi.tolist())
            seen["full"] += int(n == rig.mn and len(stored[0]) == rig.mn)
            slot += 1
        assert all(x.dir_new[s] == -1 and x.n_matches[s] == 0 and x.geo_valid[s] == 0 for s in range(slot, 4)), r


@pytest.mark.parametrize("max_num", [200, 37])
def test_frontend_filter_rounds(gpu, max_num):
    """osb_frontend_query_received with the geometric filter: 64 records, 256 direction-pair slots in the grouped layout
    (max_n = max_num, which at 37 is neither the output stride 200 nor a multiple of the 16-row tile), three rounds of
    different data on one handle -- the RANSAC keys and tickets must be back at zero after every launch"""
    rig = FilterRig(max_num)
    seen = dict(empty=0, invalid=0, valid=0, four=0, reduced=0, ties=0, full=0)
    for rnd in range(3):
        plan, res = rig.round(rnd)
        _check_round(rig, plan, res, seen)
    assert all(v > 0 for v in seen.values()), seen
    rig.fe.close()


# ---- 4. stereo and depth lift ----------------------------------------------------------------------------------------
KL = np.array([80.0, 80.0, 48.0, 32.0])             # 96 x 64 flattened pinhole
MIN_PTS = 10


def _rig(nd):
    """up and down cameras 12 cm apart along the camera's y axis, yawed by 90 degrees per direction, on a drone pose"""
    pose_drone = np.concatenate([[1.0, 2.0, 0.5], synth._quat_from_rotvec(np.array([0.02, -0.01, 0.4]))])
    pu, pd = [], []
    for d in range(nd):
        yaw = synth._quat_from_rotvec(np.array([0.0, 0.0, d * np.pi / 2]))
        q = pr.q_mul(yaw, np.array([0.5, -0.5, 0.5, -0.5]))
        pu.append(pr.pose_mul(pose_drone, np.concatenate([pr.q_rot(yaw, np.array([0.05, 0.0, 0.06])), q])))
        pd.append(pr.pose_mul(pose_drone, np.concatenate([pr.q_rot(yaw, np.array([0.05, 0.0, -0.06])), q])))
    return np.array(pu), np.array(pd)


def _project(pose, pw):
    pc = pr.q_rot(pr.q_conj(pose[3:]), pw - pose[:3])
    return np.round([KL[0] * pc[0] / pc[2] + KL[2], KL[1] * pc[1] / pc[2] + KL[3]]).astype(np.float32)


def _stereo_scene(nu_list, max_n, seed):
    """per direction n_up keypoints of points 1 m to 1000 m deep (integer pixels, so far points have zero disparity),
    exact zero-disparity pairs, points behind the up camera, wrong pairs, -1, n_down - 1 and n_down (a partner parked
    just past n_down, where only the kernel's bound keeps it out)"""
    nd = len(nu_list)
    rng = np.random.default_rng(seed)
    pu, pd = _rig(nd)
    ku = np.zeros((nd, max_n, 2), np.float32); kd = np.zeros((nd, max_n, 2), np.float32)
    sm = np.full((nd, max_n), -1, np.int32); ndn = np.zeros(nd, np.int32)
    for d, nu in enumerate(nu_list):
        n_down = min(max_n - 1, nu + 1 + int(rng.integers(0, 8)))
        ndn[d] = n_down
        slots = list(rng.permutation(n_down - 1))
        wrong = [i for i in range(2, nu) if i % 8 == 6]
        for i in range(nu):
            u = np.array([rng.uniform(2, 94), rng.uniform(2, 62)])
            ray = np.array([(u[0] - KL[2]) / KL[0], (u[1] - KL[3]) / KL[1], 1.0])
            kind = i % 8
            z = {0: 3.0, 1: np.exp(rng.uniform(0, np.log(1000))),
                 2: rng.uniform(20, 1000), 3: 100.0, 4: -rng.uniform(1, 50), 5: 5.0, 6: 5.0, 7: rng.uniform(1, 6)}[kind]
            pw = pr.q_rot(pu[d][3:], ray * z) + pu[d][:3]
            ku[d, i] = _project(pu[d], pw)
            if kind == 5 and i > 1:
                continue                                                     # stereo_match -1
            j = n_down - 1 if i == 0 else (n_down if i == 1 else slots.pop())
            kd[d, j] = ku[d, i] if kind == 3 else _project(pd[d], pw)        # kind 3: exactly zero disparity
            sm[d, i] = j
        # wrong pairs: the partners of the kind-6 keypoints rotated among themselves (still one to one)
        if len(wrong) > 1:
            js = [sm[d, i] for i in wrong]
            for i, j in zip(wrong, js[1:] + js[:1]):
                sm[d, i] = j
    return ku, kd, sm, np.array(nu_list, np.int32), ndn, pu, pd


def _stereo_dev(ku, kd, sm, nu, ndn, pu, pd, thres, min_pts):
    nd, mn = sm.shape
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (ku, kd, sm, nu, ndn, pu, pd)]
    pts = torch.full((nd, mn, 3), float("nan"), device="cuda")
    fu = torch.full((nd, mn), 7, dtype=torch.uint8, device="cuda"); fd = torch.full_like(fu, 7)
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    K = np.ascontiguousarray(KL, np.float64)
    lib.check(lib.load().osb_stereo_lift_dev(*[_vp(x) for x in t[:5]], nd, mn, lib.ptr(K), _vp(t[5]), _vp(t[6]),
                                             float(thres), int(min_pts), _vp(pts), _vp(fu), _vp(fd),
                                             C.c_void_p(stream.cuda_stream)))
    stream.synchronize()
    return pts.cpu().numpy(), fu.cpu().numpy(), fd.cpu().numpy()


def _ulps(a, b):
    """distance in float32 steps (across zero too)"""
    def ordered(x):
        i = np.ascontiguousarray(x, np.float32).view(np.int32).astype(np.int64)
        return np.where(i < 0, -(i & 0x7FFFFFFF), i)
    return np.abs(ordered(a) - ordered(b))


STEREO_SHAPES = [(1, 64), (4, 64), (1, 200), (4, 200), (1, 256), (4, 256)]


@pytest.mark.parametrize("nd,max_n", STEREO_SHAPES)
def test_stereo_lift_edges(gpu, nd, max_n):
    """flags equal to lift_ref wherever its error is not within 1e-9 relative of the threshold, and on every zero-disparity
    pair; accepted points within one float32 step of the oracle's; the host and device forms byte-identical"""
    nu_list = [max_n - 1] if nd == 1 else [MIN_PTS, MIN_PTS + 1, max_n - 1, max_n // 2 + 3]
    scene = _stereo_scene(nu_list, max_n, 7 * max_n + nd)
    ku, kd, sm, nu, ndn, pu, pd = scene
    seen = dict(zero_disp=0, behind=0, last=0, lifted=0, far=0)
    excluded = total = 0
    for thres in (0.006, 0.02):
        pts, fu, fd = host.stereo_lift(ku, kd, sm, nu, ndn, KL, pu, pd, thres, MIN_PTS)
        dpts, dfu, dfd = _stereo_dev(ku, kd, sm, nu, ndn, pu, pd, thres, MIN_PTS)
        assert np.array_equal(dfu, fu) and np.array_equal(dfd, fd)
        assert np.array_equal(dpts.view(np.uint32), pts.view(np.uint32))
        for d in range(nd):
            n, m = nu[d], ndn[d]
            rp, rfu, rfd = lr.stereo_lift(ku[d, :n], kd[d, :m], sm[d, :n], KL, pu[d], pd[d], thres, MIN_PTS)
            assert not fu[d, n:].any() and not fd[d, m:].any() and not pts[d, n:].any()
            if n <= MIN_PTS:
                assert not fu[d].any() and not fd[d].any() and not pts[d].any()
                continue
            assert rfu.sum() > 0                                             # MIN_PTS + 1 keypoints are lifted
            ok = np.ones(n, bool)
            for i in range(n):
                j = int(sm[d, i])
                if j < 0 or j >= m:
                    continue
                a = np.array([(ku[d, i, 0] - KL[2]) / KL[0], (ku[d, i, 1] - KL[3]) / KL[1]])
                b = np.array([(kd[d, j, 0] - KL[2]) / KL[0], (kd[d, j, 1] - KL[3]) / KL[1]])
                zero = bool(np.array_equal(ku[d, i], kd[d, j]))
                with np.errstate(all="ignore"):
                    p, err = lr.triangulate_point(pu[d], pd[d], a, b)
                total += 1
                near = abs(err - thres) <= 1e-9 * thres
                if near and not zero:                                        # zero-disparity pairs are never excused
                    ok[i] = False
                    excluded += 1
                seen["zero_disp"] += int(zero)
                zc = (lr.rot(pu[d][3:]).T @ (p - pu[d][:3]))[2]
                seen["behind"] += int(err <= thres and zc < 0)
                seen["last"] += int(j == m - 1 and rfu[i] == 1)
                seen["far"] += int(rfu[i] == 1 and zc > 9.0)                  # one pixel of disparity: 9.6 m
            assert np.array_equal(fu[d, :n][ok], rfu[ok]), (d, thres)
            down_ok = np.ones(m, bool)
            down_ok[[int(sm[d, i]) for i in range(n) if not ok[i]]] = False
            assert np.array_equal(fd[d, :m][down_ok], rfd[down_ok]), (d, thres)
            both = (fu[d, :n] == 1) & (rfu == 1)
            seen["lifted"] += int(both.sum())
            assert _ulps(pts[d, :n][both], rp[both]).max(initial=0) <= 1, (d, thres)
            assert not pts[d, :n][fu[d, :n] == 0].any()
            # the partner parked at n_down is never read
            assert sm[d, 1] == m and fu[d, 1] == 0 and rfu[1] == 0
    assert all(v > 0 for v in seen.values()), seen
    assert excluded <= max(1, total // 100), (excluded, total)


def _depth_dev(kp, n, depth, pose, near, far, min_pts):
    nd, mn = kp.shape[:2]
    t = [torch.from_numpy(np.ascontiguousarray(a)).cuda() for a in (kp, n, depth, pose)]
    pts = torch.full((nd, mn, 3), float("nan"), device="cuda"); fl = torch.full((nd, mn), 7, dtype=torch.uint8, device="cuda")
    stream = torch.cuda.Stream()
    torch.cuda.synchronize()
    K = np.ascontiguousarray(KL, np.float64)
    lib.check(lib.load().osb_depth_lift_dev(_vp(t[0]), _vp(t[1]), nd, mn, _vp(t[2]), depth.shape[1], depth.shape[2],
                                            lib.ptr(K), _vp(t[3]), near, far, int(min_pts), _vp(pts), _vp(fl),
                                            C.c_void_p(stream.cuda_stream)))
    stream.synchronize()
    return pts.cpu().numpy(), fl.cpu().numpy()


def test_depth_lift_edges(gpu):
    """key points at 0, at W - 0.5 (rounds half to even, onto W), W - 1.5, the float32 below W and W itself, on .5 ties of
    odd and even pixels, outside the image; W = 90 is not a multiple of 32; depths 0, near and far in mm and one mm inside
    each, 65535; n = ACCEPT_MIN_3D_PTS and one more"""
    H, W, nd, mn = 50, 90, 3, 64                    # W not a multiple of 32
    near, far = 0.3, 10.0
    rng = np.random.default_rng(11)
    depth = rng.integers(0, 12000, (nd, H, W)).astype(np.uint16)
    f32 = np.float32
    xs = [0.0, W - 0.5, W - 1.5, float(np.nextafter(f32(W), f32(0))), float(W), 0.5, 1.5, 2.5, 3.5, 44.5, 45.5, W + 0.25,
          -0.25, 17.7, 60.2]
    ys = [0.0, H - 0.5, H - 1.5, float(np.nextafter(f32(H), f32(0))), float(H), 0.5, 1.5, 2.5, 3.5, 24.5, 25.5, H + 0.25,
          -0.25, 33.3, 8.9]
    kp = np.zeros((nd, mn, 2), np.float32)
    k = [(x, y) for x in xs for y in ys]
    sel = rng.permutation(len(k))[:mn]
    kp[0] = np.array([k[i] for i in sel], np.float32)
    kp[0, :len(xs)] = np.array(list(zip(xs, ys[::-1])), np.float32)
    kp[1:, :, 0] = rng.uniform(0, W, (nd - 1, mn)); kp[1:, :, 1] = rng.uniform(0, H, (nd - 1, mn))
    n = np.array([mn, MIN_PTS, MIN_PTS + 1], np.int32)
    special = [0, int(near * 1000), int(near * 1000) + 1, int(far * 1000) - 1, int(far * 1000), 65535]
    for d in range(nd):
        for i in range(n[d]):
            x, y = float(kp[d, i, 0]), float(kp[d, i, 1])
            xi, yi = int(round(x)), int(round(y))
            if 0 <= x <= W and 0 <= y <= H and xi < W and yi < H and i % 2 == 0:
                depth[d, yi, xi] = special[(i // 2) % len(special)]
    pose = np.array([np.concatenate([[0.3, -0.2, 1.0], synth._quat_from_rotvec(np.array([0.1, 0.2, 0.3 + d]))])
                     for d in range(nd)])
    pts, fl = host.depth_lift(kp, n, depth, KL, pose, near, far, MIN_PTS)
    dpts, dfl = _depth_dev(kp, n, depth, pose, near, far, MIN_PTS)
    assert np.array_equal(dfl, fl) and np.array_equal(dpts.view(np.uint32), pts.view(np.uint32))
    seen = set()
    for d in range(nd):
        rp, rf = lr.depth_lift(kp[d, :n[d]], depth[d], KL, pose[d], near, far, MIN_PTS)
        assert np.array_equal(fl[d, :n[d]], rf) and not fl[d, n[d]:].any()
        assert _ulps(pts[d, :n[d]][rf == 1], rp[rf == 1]).max(initial=0) <= 1
        assert not pts[d, :n[d]][rf == 0].any()
        if n[d] <= MIN_PTS:
            assert not fl[d].any()
            continue
        assert rf.sum() > 0
        for i in range(n[d]):
            x, y = float(kp[d, i, 0]), float(kp[d, i, 1])
            if 0 <= x <= W and 0 <= y <= H:
                xi, yi = int(round(x)), int(round(y))
                if xi < W and yi < H:
                    seen.add(int(depth[d, yi, xi]))
                else:
                    seen.add("rounds_to_edge")
                if x - np.floor(x) == 0.5 and round(x) != np.floor(x + 0.5):
                    seen.add("half_to_even")
    assert set(special) | {"rounds_to_edge", "half_to_even"} <= seen, seen
