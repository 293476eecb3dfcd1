"""The pre-motion oracles at the device's edges, on the CPU: tests/init_by_loops_ref.py's loop map (LoopBook, the literal
bookkeeping, and LoopMapVec, the device's representation) over rows in every 64-bit word of a drone set, duplicate ids
with different values, re-sent ids and ids chosen against the device's hash; init_pose_by_loops against
init_by_loops_vec at 256 drones with more than 256 window entries and yaws near +-pi; tests/da_init_ref.py's two forms
at 256 drones with 32 anonymous ids, at the exact acceptance threshold and at the budget, and the work a search does per
DFS call.  The two places where the device's loop map differs from the reference's bookkeeping are pinned here
(DESIGN.md section 5)."""
import numpy as np
import pytest

from omniswarm_b200 import lib as _l
from oracle import anchor_ref as ar
from oracle import pcm_ref as pr
import da_init_ref as da
import init_by_loops_ref as ib
from test_da_init_ref import STEP, case, yaw_pose

I64_MIN, I64_MAX = np.iinfo(np.int64).min, np.iinfo(np.int64).max
M64 = (1 << 64) - 1
WORD_EDGES = (0, 1, 63, 64, 127, 128, 254, 255)                    # both sides of every 64-bit word boundary


def splitmix64(x: int) -> int:
    """common.cuh's splitmix64 of an id taken as uint64: the loop map's hash"""
    z = (x + 0x9E3779B97F4A7C15) & M64
    z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & M64
    z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & M64
    return z ^ (z >> 31)


def home(i: int, H: int) -> int:
    return splitmix64(i & M64) & (H - 1)


def table_size(max_measurements: int) -> int:
    """the loop map's H: the least power of two >= 2 max_measurements"""
    H = 1
    while H < 2 * max_measurements:
        H <<= 1
    return H


def ids_at_home(slot: int, H: int, n: int, start: int = 1) -> list:
    """the first n positive ids from start whose home slot is `slot`"""
    out, i = [], start
    while len(out) < n:
        if home(i, H) == slot:
            out.append(i)
        i += 1
    return out


def wrap(a):
    return (np.asarray(a, np.float64) + np.pi) % (2 * np.pi) - np.pi


def close_yaw(got, want, rel=1e-12):
    """poses [n, 4]: x y z to rel relative, yaw as an angle (a difference of 2 pi is none)"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    if got.shape != want.shape:
        return False
    tol = rel * np.maximum(1.0, np.abs(want))
    return bool(np.all(np.abs(got[:, :3] - want[:, :3]) <= tol[:, :3]) and
                np.all(np.abs(wrap(got[:, 3] - want[:, 3])) <= tol[:, 3]))


def loop_rows(ids, id_a, id_b, seed, stamps=None):
    """OK osb_anchor_result rows with the given ids and drone pairs, each with its own stamps and relative pose"""
    rng = np.random.default_rng(seed)
    n = len(ids)
    rows = np.zeros(n, _l.ANCHOR_RESULT_DTYPE)
    rows["id"] = np.asarray(ids, np.int64)
    rows["status"] = _l.ANCHOR_OK
    rows["edge"]["id_a"], rows["edge"]["id_b"] = id_a, id_b
    if stamps is None:
        stamps = rng.integers(0, 1 << 40, (n, 2))
    rows["stamp_a"], rows["stamp_b"] = np.asarray(stamps)[:, 0], np.asarray(stamps)[:, 1]
    q = rng.normal(size=(n, 4))
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    rows["edge"]["rel_pose"] = np.concatenate([rng.uniform(-5, 5, (n, 3)), q], axis=1)
    return rows


def special_ids(H):
    """ids the map must handle by value: -1 (the empty key, kept in record H), INT64_MIN, 0, negatives, and ids whose
    home slot is H - 1, so the later ones' probes wrap to slot 0"""
    return [-1, int(I64_MIN), 0, -7, -(1 << 40), 5, 1 << 40] + ids_at_home(H - 1, H, 4)


def scale_rows(n, H, seed, n_ids=3000):
    """n rows over n_ids distinct ids plus special_ids(H), drone ids in every word and self-pairs; every special id and
    a tenth of the others appear again far apart (other CTAs and other grid-stride passes) with other values"""
    rng = np.random.default_rng(seed)
    spec = special_ids(H)
    pool = np.concatenate([np.array(spec, np.int64), rng.integers(-(1 << 50), 1 << 50, n_ids)])
    ids = pool[rng.integers(0, len(pool), n)]
    ids[:len(spec)] = spec                                          # each special id first in the first CTA ...
    for k, i in enumerate(spec):                                    # ... and again in the last quarter
        ids[n - 1 - 97 * k] = i
    drones = np.array(WORD_EDGES + (5, 31, 32, 65, 191, 192, 200))
    a, b = drones[rng.integers(0, len(drones), n)], drones[rng.integers(0, len(drones), n)]
    a[::53] = b[::53]                                               # self-pairs (a, a)
    return loop_rows(ids, a, b, seed)


def book_view(book: ib.LoopBook, D: int):
    """LoopBook in LoopMapVec's form: (records ascending by id, pair minima [D, D] with INT64_MAX as none)"""
    recs = np.zeros(len(book.all_loop_map), _l.LOOP_RECORD_DTYPE)
    for k, i in enumerate(sorted(book.all_loop_map)):
        e = book.all_loop_map[i]
        recs[k] = (i, e["id_a"], e["id_b"], e["ts_a"], e["ts_b"], e["rel"])
    pair = np.full((D, D), I64_MAX, np.int64)
    for a, m in book.all_loops_set_by_pair.items():
        for b, s in m.items():
            pair[a, b] = min(s)
    return recs, pair


def same_map(recs, pair, vec: ib.LoopMapVec):
    return recs.tobytes() == vec.recs.tobytes() and np.array_equal(pair, vec.pair_min)


def test_hash_edges_are_what_they_claim():
    H = table_size(4096)
    assert H == 8192
    wraps = ids_at_home(H - 1, H, 4)
    assert all(home(i, H) == H - 1 for i in wraps)
    assert splitmix64(0) == 0xE220A8397B1DCDAF                      # the published first output of splitmix64(seed 0)


def test_loop_map_forms_agree_at_scale():
    """three calls of duplicates in every word, the special ids, and every id re-sent later with new values: the first
    row of an id in the first call that has it wins, both pair orders take its minimum"""
    D, H = 256, table_size(4096)
    rows = scale_rows(30_000, H, 1)
    book, vec = ib.LoopBook(200, True), ib.LoopMapVec(D, _l.LOOP_RECORD_DTYPE)
    for lo, hi in ((0, 12_000), (12_000, 24_000), (24_000, 30_000)):
        book.record(rows[lo:hi])
        vec.record_vec(rows[lo:hi])
    resent = loop_rows(vec.recs["id"][::3], 1, 2, 9)                # every third id again, on another pair
    book.record(resent)
    vec.record_vec(resent)
    assert same_map(*book_view(book, D), vec)
    r = vec.recs
    first = {}
    for k in range(len(rows)):
        first.setdefault(int(rows["id"][k]), k)
    for i in special_ids(H):                                        # the lowest row wrote each special id's record
        rec = r[np.searchsorted(r["id"], i)]
        assert rec["id"] == i and rec["stamp_a"] == rows["stamp_a"][first[i]]
    neg = r["id"] < 0                                               # negative ids order below positive ones
    assert np.all(vec.pair_min[r["id_a"][neg], r["id_b"][neg]] <= r["id"][neg])
    assert vec.pair_min.min() == I64_MIN
    assert vec.pair_min[np.diag_indices(D)][list(WORD_EDGES)].min() < I64_MAX    # self-pairs in every word


def test_int64_max_is_no_pair_loop_on_the_device():
    """divergence 1: the id INT64_MAX is the pair table's "none", so a pair whose smallest id it is reads as no loop
    (LoopMapVec, as the device); the reference's std::set uses it"""
    D = 256
    rows = loop_rows([I64_MAX], 64, 200, 3, stamps=[[0, 0]])
    book, vec = ib.LoopBook(200, True), ib.LoopMapVec(D, _l.LOOP_RECORD_DTYPE)
    book.record(rows)
    vec.record_vec(rows)
    recs, pair = book_view(book, D)
    assert recs.tobytes() == vec.recs.tobytes()                     # the record itself is kept
    assert pair[64, 200] == I64_MAX == vec.pair_min[64, 200]        # the two views cannot tell it from none ...
    assert book.all_loops_set_by_pair[64][200] == {I64_MAX}         # ... but the reference's set holds it
    trajs = {200: (np.array([0, STEP]), np.stack([yaw_pose(0, 0, 0, 0), yaw_pose(1, 0, 0, 0)]))}
    ents = np.zeros(1, _l.WINDOW_ENTRY_DTYPE)
    ents["drone_id"], ents["block"] = 64, 0
    win = (np.array([STEP]), np.array([0, 1], np.int32), ents)
    before = np.zeros((1, 4))
    lit = ib.init_pose_by_loops({64}, {}, book, {200}, {}, ib.Trajs(trajs), 200, win, before)
    to_init = np.zeros(D, bool)
    to_init[64] = True
    vec_out = ib.init_by_loops_vec(to_init, {}, vec, np.arange(D) == 200, {}, trajs, 200, win, before)
    assert not np.array_equal(lit, before) and np.array_equal(vec_out, before)


def test_recorded_id_on_another_pair():
    """divergence 2: with redundant = false an id of a pair without self is recorded but not stored by PCM, so when it
    arrives again on another pair the reference adds it to that pair's set; the device skips every recorded id"""
    D = 256
    first = loop_rows([77], 63, 64, 4)
    again = loop_rows([77], 128, 255, 5)
    for redundant, diverges in ((False, True), (True, False)):
        book, vec = ib.LoopBook(200, redundant), ib.LoopMapVec(D, _l.LOOP_RECORD_DTYPE)
        for r in (first, again):
            book.record(r)
            vec.record_vec(r)
        recs, pair = book_view(book, D)
        assert recs.tobytes() == vec.recs.tobytes()                 # the record is the first row's either way
        assert vec.pair_min[128, 255] == I64_MAX
        assert (pair[128, 255] == 77) == diverges


# ---- init_pose_by_loops at 256 drones ---------------------------------------------------------------------------------
SELF = 200
DRONES = (0, 5, 63, 64, 127, 128, 200, 254, 255)
TO_INIT = (0, 63, 64, 127, 128, 255)
T0 = 1_000 * STEP


N_FRAMES, EVERY = 280, 35                                          # drone 63 in every frame, the others in every 35th


def ibl_scene(self_id=SELF, seed=11):
    """9 drones across the words, 12 odometry samples each with yaws near +-pi; a window of N_FRAMES frames 1/20 of a
    sample apart, from before the first sample to past the last (some exactly midway between two), with drone 63 in
    every frame and the others in every EVERY-th, so drone 63 alone holds more than 256 entries.  Two of drone 63's
    blocks are shared: its first frame's with its last (more than 256 entries apart in the device's (drone, frame)
    order, so on different passes of the entry loop) and its frame 40's with its frame 100's.  Loops with stamps
    midway between samples, before the first and after the last"""
    rng = np.random.default_rng(seed)
    trajs = {}
    for d in DRONES:
        k = np.arange(12)
        yaw = np.pi - 1e-3 + 2e-4 * k + (d % 3) * 1e-4                # crosses +pi at k = 5
        t = T0 + STEP * k
        trajs[d] = (t, np.stack([yaw_pose(*rng.uniform(-3, 3, 2), 0.1 * j, y) for j, y in zip(k, yaw)]))
    fs = T0 - STEP + (STEP // 20) * np.arange(N_FRAMES)
    frames = [np.array([63]) if f % EVERY else np.array(DRONES) for f in range(N_FRAMES)]
    ents = np.zeros(sum(map(len, frames)), _l.WINDOW_ENTRY_DTYPE)
    ents["drone_id"] = np.concatenate(frames)
    ents["block"] = np.arange(len(ents))
    e63 = np.nonzero(ents["drone_id"] == 63)[0]
    for lo, hi in ((0, -1), (40, 100)):
        ents["block"][e63[hi]] = ents["block"][e63[lo]]
    win = (fs.astype(np.int64), np.cumsum([0] + [len(f) for f in frames]).astype(np.int32), ents)
    assert np.any(fs == T0 + STEP // 2)                             # a frame stamp midway between samples 0 and 1
    mid = T0 + STEP // 2                                            # midway between samples 0 and 1: ties go to 0
    loops = [  # (id, a, b, stamp_a, stamp_b, yaw of the relative pose)
        (10, 0, 5, mid, mid + STEP, np.pi - 1e-9),
        (11, 0, 254, T0 - 5 * STEP, T0 + 30 * STEP, -np.pi + 1e-9),  # before the first / after the last sample
        (12, 63, self_id, mid + 3 * STEP, mid, 3.0),
        (13, 64, 127, mid, T0 + 2 * STEP, -np.pi + 3e-4),                      # id_a != id2 = 127: inverted
        (14, 128, 5, T0 + 7 * STEP, mid + 9 * STEP, np.pi - 2e-4),
        (15, 255, 254, mid + 11 * STEP, T0 + 4 * STEP, np.pi),
        (16, 127, 127, T0, T0 + 3 * STEP, 0.5),                        # a self-pair
        (9, 255, 0, mid, mid, 2.0),                                    # a smaller id of an unestimated pair
    ]
    rows = loop_rows([x[0] for x in loops], [x[1] for x in loops], [x[2] for x in loops], seed,
                     stamps=[[x[3], x[4]] for x in loops])
    for r, x in zip(rows, loops):
        r["edge"]["rel_pose"] = yaw_pose(*rng.uniform(-2, 2, 3), x[5])
    kf = {254: (trajs[254][0][::3].copy(), trajs[254][1][::3].copy())}
    return trajs, win, rows, kf


def ibl_both(trajs, win, rows, kf, good_sets, estimated, self_id, to_init=TO_INIT):
    D = 256
    book, vec = ib.LoopBook(self_id, True), ib.LoopMapVec(D, _l.LOOP_RECORD_DTYPE)
    book.record(rows)
    vec.record_vec(rows)
    before = np.random.default_rng(5).uniform(-1, 1, (len(win[2]), 4))
    mask = np.isin(np.arange(D), to_init)
    est = np.isin(np.arange(D), list(estimated))
    want = ib.init_by_loops_vec(mask, good_sets, vec, est, kf, trajs, self_id, win, before)
    lit = ib.init_pose_by_loops(set(to_init), ib.good_from_sets(good_sets), book, set(estimated), kf, ib.Trajs(trajs),
                                self_id, win, before)
    return want, lit, before


@pytest.mark.parametrize("source", ["pairs", "directory"])
def test_init_by_loops_forms_agree_at_256(source):
    trajs, win, rows, kf = ibl_scene()
    good = {}
    if source == "directory":                                       # sets replace the pairs; empty sets and a self-pair
        good = {(0, 5): [10], (0, 200): [], (64, 127): [13], (127, 127): [16], (128, 255): [], (5, 128): [14]}
    estimated = {5, 127, SELF, 254}
    want, lit, before = ibl_both(trajs, win, rows, kf, good, estimated, SELF)
    assert close_yaw(want, lit)
    moved = np.nonzero(np.any(want != before, axis=1))[0]
    assert set(win[2]["drone_id"][moved].tolist()) == ({0, 63, 64, 127, 128, 255} if source == "pairs"
                                                         else {0, 63, 64, 127, 128})   # 255: only an empty set
    y = want[moved, 3]
    assert y.max() > np.pi - 0.01 and y.min() < -np.pi + 0.01       # yaws on both sides of the branch cut
    e63 = np.nonzero(win[2]["drone_id"] == 63)[0]
    assert device_order(win)[e63[-1]] - device_order(win)[e63[0]] > 256
    if source == "pairs":                                           # each shared block holds its later frame's pose
        vec = ib.LoopMapVec(256, _l.LOOP_RECORD_DTYPE)
        vec.record_vec(rows)
        own = ib.init_by_loops_vec(np.arange(256) == 63, {}, vec, np.isin(np.arange(256), [SELF]), kf, trajs, SELF,
                                   unshared(win), before)
        for lo, hi in ((0, -1), (40, 100)):
            assert np.array_equal(want[e63[lo]], own[e63[hi]]) and not np.array_equal(own[e63[lo]], own[e63[hi]])


def device_order(win):
    """each entry's index in the device's window, ordered by (drone, frame)"""
    pos = np.empty(len(win[2]), np.int64)
    pos[np.argsort(win[2]["drone_id"], kind="stable")] = np.arange(len(win[2]))
    return pos


def unshared(win):
    ents = win[2].copy()
    ents["block"] = np.arange(len(ents))
    return win[0], win[1], ents


def test_init_by_loops_pose0_sources_and_refusal():
    """pose0 from a keyframe path (254), from self's odometry (self without a path), identity (5); the largest
    estimated id2 decides; self 0 in place of 200"""
    trajs, win, rows, kf = ibl_scene(self_id=0)
    want, lit, before = ibl_both(trajs, win, rows, kf, {}, {0, 5, 127, 254}, 0)
    assert close_yaw(want, lit)


def test_init_by_loops_refuses_an_id2_without_odometry():
    """self 255 holds window entries but no odometry: drone 254's id2 is 255 (a loop to self), and reading its
    odometry throws in the reference, so both forms refuse"""
    trajs, win, rows, kf = ibl_scene(self_id=255)
    del trajs[255]
    with pytest.raises(ib.Refused):
        ibl_both(trajs, win, rows, kf, {}, {5, 127, 254, 255}, 255, to_init=(0, 254))
    book = ib.LoopBook(255, True)
    book.record(rows)
    with pytest.raises(ib.Refused):                                 # the literal walk alone, drone 254 only
        ib.init_pose_by_loops({254}, {}, book, {5, 127, 254, 255}, kf, ib.Trajs(trajs), 255, win,
                              np.zeros((len(win[2]), 4)))


# ---- the data-association search at 256 drones ------------------------------------------------------------------------
WORDS = (1, 63, 64, 127, 128, 255)                                  # detectors and candidates in every 64-bit word
BAD_COV = np.diag([-1.0, 1, 1, 1, 1, 1])                            # not positive definite: +inf, no candidate passes


def da_both(*args, **kw):
    """both oracle forms, which must agree on the outcome, the DFS calls and the gate evaluations -> (outcome, stats)"""
    s1, s2 = {}, {}
    lit = da.da_literal(*args, **kw, stats=s1)
    vec = da.da_vec(*args, **kw, stats=s2)
    assert lit == vec and s1 == s2, (s1, s2)
    return lit, s1


def da_scene(self_id, n_ids, n_det=300, seed=2):
    """256 drones of which only self, the detectors WORDS and n_ids targets have odometry and keyframe paths (every one
    estimated, so every candidate meets the gate and only the true target passes).  Anonymous ids 256.. in store
    order: each id's first row is by its largest detector with a covariance that is not positive definite, its smallest
    detector's first row follows in the first 256 rows, filler rows follow, and its last row lies past row 256.
    -> (trajs, kf, dets, targets {anonymous id: drone}, avail)"""
    rng = np.random.default_rng(seed)
    others = [d for d in range(2, 255) if d not in WORDS + (self_id,)]
    targets = list(WORDS) + [int(x) for x in rng.choice(others, n_ids - len(WORDS), replace=False)]
    dets_of = {}
    for j, b in enumerate(targets[:n_ids]):
        cand = [d for d in WORDS + (self_id,) if d != b]
        dets_of[256 + j] = (b, min(cand), max(cand), cand[j % len(cand)])
    first = [(big, b, u, 1) for u, (b, small, big, last) in dets_of.items()]
    smallest = [(small, b, u, 2) for u, (b, small, big, last) in dets_of.items()]
    lasts = [(last, b, u, 30) for u, (b, small, big, last) in dets_of.items()]
    keys = list(dets_of)
    fill = [(dets_of[u][3], dets_of[u][0], u, 3 + k % 20) for k, u in
            enumerate(rng.choice(keys, n_det - 3 * len(keys)))]
    order = first + smallest + fill + lasts
    avail = sorted(set(targets[:n_ids]) | set(WORDS) | {self_id})
    trajs, kf, dets, _ = case(256, order, seed=seed, kf_drones=tuple(avail))
    for d in range(256):
        if d not in avail:
            trajs[d] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    dets["cov"][:len(first)] = BAD_COV
    assert len(first) + len(smallest) <= 256 < n_det - len(lasts)  # the smallest detector's row and the last one: two passes
    return trajs, kf, dets, {u: v[0] for u, v in dets_of.items()}, avail


@pytest.mark.parametrize("self_id,n_ids", [(200, 32), (0, 6)])
def test_da_forms_agree_at_256_drones(self_id, n_ids):
    """32 ids with self 200 (past the first word) resolve to their true targets in 33 calls; with self 0 drone 0 is a
    candidate that passes unchecked, so 6 ids take many more calls and resolve as the first success decides"""
    trajs, kf, dets, targets, _ = da_scene(self_id, n_ids)
    (applied, status, guess, ids), st = da_both(self_id, trajs, kf, dets, 3.345, anon_min=256)
    assert (applied, status) == (True, "ok") and len(guess) == n_ids
    if self_id == 200:
        assert guess == targets and st["nodes"] == 33
        assert st["gates"] >= 32 * 30                                # every other candidate met the gate and failed
    else:
        assert 0 in guess.values() and st["nodes"] > 2 * n_ids
    more = dets[:1].copy()                                          # a 33rd id: refused
    more["id_b"] = 256 + 32
    if n_ids == 32:
        out, _ = da_both(self_id, trajs, kf, np.concatenate([dets, more]), 3.345, anon_min=256)
        assert out[:2] == (False, "capacity")


def exact_scene(cov=np.eye(6)):
    """self 200 and drone 255 with odometry at dyadic positions and identity rotations; ids 256 and 257 both detected by
    self, their paths for 255 exactly 2 m apart: with unit covariance the squared Mahalanobis distance is exactly 4"""
    stamps = T0 + STEP * np.arange(8, dtype=np.int64)
    trajs = {d: (np.zeros(0, np.int64), np.zeros((0, 7))) for d in range(256)}
    for d, x in ((200, 0.5), (255, -1.25)):
        trajs[d] = (stamps.copy(), np.array([[x + 0.25 * k, 0.125, 0.0, 1.0, 0.0, 0.0, 0.0] for k in range(8)]))
    dets = np.zeros(2, _l.MEASUREMENT_DTYPE)
    dets["id"] = [70, 71]
    dets["type"] = _l.MEAS_DET6D
    dets["id_a"], dets["id_b"] = 200, [256, 257]
    dets["stamp_a"], dets["stamp_b"] = stamps[2], stamps[5]
    dets["relative_pose"] = [[8.0, 0.0, 0.5, 1.0, 0, 0, 0], [8.0, 2.0, 0.5, 1.0, 0, 0, 0]]
    dets["cov"] = cov
    return trajs, dets


def test_da_threshold_is_strict_at_the_exact_float():
    trajs, dets = exact_scene()
    four = float(np.float32(4.0))
    above = float(np.nextafter(np.float32(4.0), np.float32(np.inf)))
    assert da_both(200, trajs, {}, dets, four, anon_min=256)[0][:3] == (False, "ok", {})
    assert da_both(200, trajs, {}, dets, above, anon_min=256)[0][:3] == (True, "ok", {256: 255, 257: 255})
    lit = da.DAInit(200, trajs, {}, dets, four, anon_min=256)
    t0 = max(int(v.stamps[0]) for v in lit.ego.values())
    est = {200: lit.ego[200].poses[lit.ego[200].nearest(t0)]}
    lit.drone_dets_by_pair = {u: {200: [da.det_of(r)]} for u, r in zip((256, 257), dets)}
    p1 = lit.estimate_path(256, {256: 255}, est, t0)
    p2 = lit.estimate_path(257, {257: 255}, est, t0)
    assert da.mahalanobis(p1, p2, np.eye(6)) == 4.0                  # exactly: every product is exact
    trajs, dets = exact_scene(BAD_COV)                               # +inf: skipped whatever the threshold
    assert da_both(200, trajs, {}, dets, 1e30, anon_min=256)[0][:2] == (False, "ok")


def budget_scene():
    """self 200 detects drones 64, 128 and 255 (ids 256..258), no keyframe paths: the search walks every order of the
    three ids before it returns its first success"""
    anon = [(200, 64, 256, 5), (200, 128, 257, 9), (200, 255, 258, 13)]
    trajs, kf, dets, _ = case(256, anon, seed=5)
    for d in range(256):
        if d not in (64, 128, 200, 255):
            trajs[d] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    return trajs, dets


def test_da_budget_at_256_drones():
    trajs, dets = budget_scene()
    out, st = da_both(200, trajs, {}, dets, 3.345, anon_min=256)
    n = st["nodes"]
    assert out[:2] == (True, "ok") and n > 4
    assert da_both(200, trajs, {}, dets, 3.345, anon_min=256, max_nodes=n)[0][:2] == (True, "ok")
    out, st = da_both(200, trajs, {}, dets, 3.345, anon_min=256, max_nodes=n - 1)
    assert out[:2] == (False, "capacity") and st["nodes"] == n - 1


# ---- the work of a search per DFS call --------------------------------------------------------------------------------
N_SPINE = 7


def worst_scene(seed=7):
    """every one of 256 drones has odometry and a keyframe path (all estimated, drone 0 too); 32 ids, all detections
    30 m off.  Ids 256..280 are seen by drone 0: all 255 candidates meet the gate and fail.  Ids 281..287 are seen by
    self 200: drone 0 is their one candidate that passes (it is never gated), so the search goes deeper through them.
    No leaf is ever reached, every DFS call gates at least 25 x 255 candidates, and the budget ends the search."""
    n_dead = 32 - N_SPINE
    anon = [(0 if j < n_dead else 200, 1 + (7 * j) % 250, 256 + j, 4 + j) for j in range(32)]
    trajs, kf, dets, _ = case(256, anon, seed=seed, kf_drones=tuple(range(256)))
    dets["relative_pose"][:, 0] += 30.0
    return trajs, kf, dets


class _Stop(Exception):
    pass


def worst_gates(max_nodes, n_spine=N_SPINE, n_u=32, D=256):
    """the gate evaluations of worst_scene's search cut at max_nodes calls, counted from its order: a call gates the
    D - 1 candidates of each of the n_u - n_spine ids seen by drone 0, then for each remaining id seen by self enters
    drone 0's call and gates its D - 2 other candidates; the walk stops at the first call past the budget"""
    st = dict(nodes=0, gates=0)

    def call(spine):
        st["nodes"] += 1
        if st["nodes"] > max_nodes:
            raise _Stop
        st["gates"] += (n_u - n_spine) * (D - 1)
        for _ in range(spine):
            call(spine - 1)
            st["gates"] += D - 2

    try:
        call(n_spine)
    except _Stop:
        return st["gates"]
    raise AssertionError("the search ended within the budget")


@pytest.mark.parametrize("max_nodes", [2])
def test_da_gate_work_per_call(max_nodes):
    """divergence 3: max_nodes bounds DFS calls, not gate evaluations.  The oracles' count equals worst_gates, and a
    call costs close to n_u x (D - 1) gates"""
    trajs, kf, dets = worst_scene()
    out, st = da_both(200, trajs, kf, dets, 3.345, anon_min=256, max_nodes=max_nodes)
    assert out[:2] == (False, "capacity") and st["nodes"] == max_nodes
    assert st["gates"] == worst_gates(max_nodes) >= max_nodes * 25 * 255


def test_gate_work_at_the_documented_budgets():
    """the figures DESIGN.md section 5 quotes for worst_scene (estimates from the count rule above)"""
    got = {n: worst_gates(n) for n in (8, 64, 256, 1024, 4096)}
    assert got == {8: 51_508, 64: 422_732, 256: 1_695_500, 1024: 6_786_318, 4096: 27_151_368}
    assert all(got[n] <= n * 32 * 255 for n in got)                 # within the bound max_nodes x n_u x (D - 1)
