"""GPU: the keyframe database's scan kernels (db_scan_coop_kernel<Q>, db_scan_kernel<Q,4>) and both merges (the fused
last-CTA merge and db_merge_kernel) against oracle/frontend_ref.py::IndexFlatIP.

Selection logic is tested with exact arithmetic: small-integer rows and queries make every fp32 score exact in any
summation order, so ids and scores must equal the oracle's bit for bit, with exact ties resolved by ascending id.
Arithmetic is tested with random real data against oracle/fp32_bounds.py::ip_ref's float64 score and bound.

Which path runs follows from the shapes, as csrc/match.cu chooses it: the grid is 2 x SMs CTAs with
chunk = ceil(n / grid) rows each, or 512-row chunks and a larger grid once n > 512 x 2 x SMs; dim 4096 with
chunk <= 64 takes the cooperative kernel; grids above 3584 CTAs or k > 16 take the separate merge kernel; queries go 8
per pass while 8 x (dim + 512) floats fit the kernel's 200 KB of shared memory, else 4, and the host splits them into
passes of 64."""
import numpy as np
import pytest

from omniswarm_b200 import host
from oracle import fp32_bounds as fb
from oracle import frontend_ref as fr

pytestmark = pytest.mark.gpu

DB_CHUNK_MAX, DB_COOP_CHUNK, DB_MERGE_MAX = 512, 64, 3584


@pytest.fixture(scope="module")
def sms(gpu):
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def layout(n, sms):
    """(grid, chunk) of a search over n rows (db_scan_grid)"""
    grid = 2 * sms
    chunk = -(-max(n, 1) // grid)
    if chunk > DB_CHUNK_MAX:
        chunk = DB_CHUNK_MAX
        grid = -(-n // chunk)
    return grid, chunk


def int_data(n, dim, nq, seed):
    rng = np.random.default_rng(seed)
    return (rng.integers(-3, 4, (n, dim)).astype(np.float32), rng.integers(-3, 4, (nq, dim)).astype(np.float32))


def exact_check(idx, rows, q, ks, nqs):
    """every (k, nq) against the oracle's top 64 of all queries (a top k is the first k of a top 64)"""
    ref = fr.IndexFlatIP(rows.shape[1])
    ref.add(rows)
    Dr, Ir = ref.search(q, 64)
    for k in ks:
        for nq in nqs:
            D, I = idx.search(q[:nq], k)
            assert np.array_equal(I, Ir[:nq, :k]), f"ids differ (nq {nq}, k {k})"
            assert np.array_equal(D, Dr[:nq, :k]), f"scores differ (nq {nq}, k {k})"


def plant_ties(rows, q, chunk, k):
    """rows chunk-1 and chunk (the last row of CTA 0 and the first of CTA 1) become the best row for query 0, and k + 4
    copies of one row score just below it: the copies straddle the k-th slot, in the rows right after the boundary (so
    inside one CTA where chunks are long) and spread over the database"""
    n, dim = rows.shape
    best = np.sign(q[0]) * 3
    rows[chunk - 1] = rows[chunk] = best
    mid = best.copy()
    mid[: dim // 2] = 0
    rows[chunk + 1: chunk + 1 + k + 4] = mid
    rows[np.linspace(chunk + k + 5, n - 1, k + 4).astype(int)] = mid


# (name, n, dim): the path each shape selects is asserted from `layout`
SHAPES = [("coop", "full", 4096), ("coop", 1000, 4096), ("stream", "65", 4096), ("stream", 5000, 256),
          ("stream", "512", 256), ("wide", 300_000, 256)]


def shape_rows(kind, n, sms):
    if n == "full":
        return DB_COOP_CHUNK * 2 * sms                 # 64 rows in every CTA
    if n == "65":
        return 65 * 2 * sms                            # the smallest chunk of the streaming kernel at dim 4096
    if n == "512":
        return DB_CHUNK_MAX * 2 * sms                  # the largest chunk of a 2 x SMs grid
    return n


@pytest.mark.parametrize("kind,n,dim", SHAPES, ids=lambda v: str(v))
def test_exact_selection(sms, kind, n, dim):
    n = shape_rows(kind, n, sms)
    grid, chunk = layout(n, sms)
    assert (dim == 4096 and chunk <= DB_COOP_CHUNK) == (kind == "coop")
    assert (grid > 2 * sms) == (kind == "wide")
    rows, q = int_data(n, dim, 130, seed=n + dim)
    plant_ties(rows, q, chunk, 64)
    idx = host.IndexFlatIP(dim, capacity=n)
    idx.add(rows)
    exact_check(idx, rows, q, (1, 16, 17, 64), (1, 2, 3, 4, 5, 8, 9, 64, 65, 130))
    D, I = idx.search(q[:1], 64)
    assert I[0, :2].tolist() == [chunk - 1, chunk]          # the tie across the CTA boundary, in id order
    idx.close()


def test_exact_selection_unfused_merge_forced_by_grid(sms):
    """more than 512 x 3584 rows: the grid exceeds the fused merge's limit, so even k <= 16 uses db_merge_kernel"""
    n = DB_CHUNK_MAX * DB_MERGE_MAX + 160_000
    assert layout(n, sms)[0] > DB_MERGE_MAX
    rows, q = int_data(n, 4, 9, seed=5)
    idx = host.IndexFlatIP(4, capacity=n)
    idx.add(rows)
    exact_check(idx, rows, q, (1, 16, 17, 64), (1, 2, 4, 5, 9))   # 7^4 distinct rows: ~800 exact ties per score
    idx.close()


@pytest.mark.parametrize("dim", [4096, 64])
def test_empty_and_short_databases(gpu, dim):
    """an empty database (dim 4096 takes the cooperative kernel) and k > ntotal: -inf / -1 padding"""
    rows, q = int_data(10, dim, 9, seed=dim)
    idx = host.IndexFlatIP(dim, capacity=16)
    for k in (1, 17, 64):
        D, I = idx.search(q, k)
        assert (I == -1).all() and np.isneginf(D).all()
    idx.add(rows)
    exact_check(idx, rows, q, (1, 10, 11, 17, 64), (1, 2, 4, 8, 9))
    idx.close()


def bounded_check(D, I, rows, q, k):
    """(a) each score within its bound of the float64 score of its id; (b) sorted by score, ties by ascending id;
    (c) no row left out beats the k-th by more than both bounds; (d) ids equal the oracle's where all gaps exceed the
    bounds.  Returns the largest fraction of the bound used."""
    s64, b = fb.ip_ref(rows, q)
    worst = 0.0
    for r in range(len(q)):
        ids = I[r]
        assert (ids >= 0).all() and len(set(ids.tolist())) == k
        worst = max(worst, fb.ratio(D[r], s64[r, ids], b[r, ids]))
        d = D[r]
        assert ((d[:-1] > d[1:]) | ((d[:-1] == d[1:]) & (ids[:-1] < ids[1:]))).all(), "not in (score, id) order"
        out = np.ones(len(rows), bool)
        out[ids] = False
        assert (s64[r, out] <= s64[r, ids[-1]] + b[r, out] + b[r, ids[-1]]).all(), "a better row was left out"
        order = np.argsort(-s64[r], kind="stable")[: k + 1]
        lo, hi = s64[r, order] - b[r, order], s64[r, order] + b[r, order]
        if (lo[:-1] > hi[1:]).all():
            assert np.array_equal(ids, order[:k])
    assert worst <= 1.0
    return worst


REAL = [(4096, 2000), (4096, 17_000), (256, 40_000), (64, 3000)]


@pytest.mark.parametrize("regime", ["spread", "near_tie"])
@pytest.mark.parametrize("dim,n", REAL, ids=lambda v: str(v))
def test_real_scores_within_bound(gpu, dim, n, regime):
    rng = np.random.default_rng(dim + n)
    if regime == "spread":
        rows = rng.standard_normal((n, dim)).astype(np.float32)
    else:                                          # a base vector plus a 1e-7 perturbation: scores within their bounds
        base = rng.standard_normal(dim)
        rows = (base + 1e-7 * rng.standard_normal((n, dim))).astype(np.float32)
    q = rng.standard_normal((9, dim)).astype(np.float32)
    idx = host.IndexFlatIP(dim, capacity=n)
    idx.add(rows)
    for k in (1, 16, 17, 64):
        D, I = idx.search(q, k)
        w = bounded_check(D, I, rows, q, k)
        print(f"dim {dim} n {n} {regime} k {k}: {w:.3e} of the bound")
    idx.close()


@pytest.mark.parametrize("dim", [5888, 5892, 8192])
def test_wide_rows_take_four_queries_per_pass(gpu, dim):
    """above dim 5888, eight queries' rows no longer fit the streaming kernel's shared memory: 5 to 8 queries must
    still be answered (in passes of four)"""
    rows, q = int_data(3000, dim, 8, seed=dim)
    rows[17] = rows[2900] = 3 * np.sign(q[5])
    idx = host.IndexFlatIP(dim, capacity=3000)
    idx.add(rows)
    exact_check(idx, rows, q, (1, 16, 17, 64), (5, 6, 7, 8))
    assert idx.search(q[5:6], 2)[1][0].tolist() == [17, 2900]
    rng = np.random.default_rng(dim)
    real = rng.standard_normal((3000, dim)).astype(np.float32)
    qr = rng.standard_normal((8, dim)).astype(np.float32)
    idx.reset()
    idx.add(real)
    D, I = idx.search(qr, 17)
    bounded_check(D, I, real, qr, 17)
    idx.close()
