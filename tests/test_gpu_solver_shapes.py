"""Every launch shape of the pose-graph solve against the float64 oracle: one LM step against the oracle's linear system
and the converged window.

graph_solve_kernel picks its path from the graph's size (solve_shape): one 16-CTA cluster or a cooperative grid of up to
one CTA per SM, the fast CG path (node state in registers, factor indices preloaded, slots gathered 16 at a time) or the
strided slow path, Jacobians in shared memory or in the global store, the chain preconditioner or block-Jacobi, fp32 or
fp64 inner arithmetic, and the multi-trial (MT) and device-tail (DT) variants.  Each row below builds a graph that lands in
one shape, asserts that it did, and checks:
  1. the initial cost against the oracle's (the cost reduction across every CTA);
  2. one LM step: the backward error |(H + D / radius) delta + grad| / |grad| of the kernel's step in the oracle's system.
     A converged-pose comparison cannot see a wrong J^T J in the CG (the minimum depends only on the residuals); this can;
  3. (CPU) that the tolerance of 2 can fail: dropping one factor from H (fp32 rows: every factor of one node) moves the
     oracle's own exact step ten times further than the tolerance;
  4. the converged window: fp64 rows against the oracle's solve, fp32 rows against the fp64-inner solve.
Every graph has all three detection flag modes, Huber-active outliers, a hub of degree > 32, a free node without factors,
a fixed node besides node 0, and shuffled node and factor order."""
import functools
import math
import time

import numpy as np
import pytest

from omniswarm_b200 import host, synth
from oracle import multistart_ref as mr
from oracle import solver_ref as sr

KEYS = host.FACTOR_KEYS
THREADS, MAX_CLUSTER, KF = 256, 16, 3            # graph.cu: GS_THREADS, GS_MAX_CLUSTER, GS_KF
FAST_FPC = KF * THREADS                          # 768 factors per CTA on the fast path
SMEM_J = 200 * 1024                              # GS_SMEM_J_MAX: shared-memory bytes of a CTA's Jacobian block
SMS = 132                                        # H100 SXM; the GPU tests take the count from the device
HUB_DEGREE = 40
U32 = float(np.finfo(np.float32).eps)

# inner tolerances of the one-step check: the CG runs to PCG64 / PCG32 relative residual
PCG64, PCG32 = 1e-13, 1e-6
TOL64 = 1e-9                                     # backward error of an fp64-inner step
C32 = 8.0                                        # fp32: C32 u32 |J|^T |J| |delta| / |grad|, see tol32


# ---------------------------------------------------------------------------------------------------------------------
# graphs
# ---------------------------------------------------------------------------------------------------------------------
def _decorated(nd, nf, n_uwb, n_loop, n_det, n_bearing, seed, m_target=None):
    """synth.pose_graph plus a hub of HUB_DEGREE ranges, a second fixed node, a free node without factors; trimmed to
    m_target factors by dropping plain ranges.  Unshuffled; `hub` marks the hub's factors."""
    g = synth.pose_graph(nd, nf, n_uwb=n_uwb, n_loop=n_loop, n_det=n_det, n_bearing=n_bearing, seed=seed,
                         outlier_frac=0.1)
    rng = np.random.default_rng(seed + 500)
    n, gt = g["n_nodes"], g["gt"]
    hub_node = (nf // 2) * nd + 1
    fixed_node = (nf // 3) * nd + 2
    others = rng.choice(np.setdiff1d(np.arange(n), [hub_node]), HUB_DEGREE, replace=False)
    sd = math.sqrt(0.0014)
    pl = np.zeros((HUB_DEGREE, g["payload"].shape[1]))
    pl[:, 0] = np.linalg.norm(gt[hub_node, :3] - gt[others, :3], axis=1) + rng.standard_normal(HUB_DEGREE) * sd
    pl[:, 1] = 1.0 / sd
    out = {"ftype": np.concatenate([g["ftype"], np.full(HUB_DEGREE, sr.FACTOR_DISTANCE, np.int32)]),
           "ia": np.concatenate([g["ia"], np.full(HUB_DEGREE, hub_node, np.int32)]),
           "ib": np.concatenate([g["ib"], others.astype(np.int32)]),
           "huber": np.concatenate([g["huber"], np.ones(HUB_DEGREE, np.uint8)]),
           "payload": np.concatenate([g["payload"], pl])}
    hub = np.zeros(len(out["ftype"]), bool); hub[-HUB_DEGREE:] = True
    if m_target is not None:
        plain = np.nonzero((out["ftype"] == sr.FACTOR_DISTANCE) & ~hub)[0]
        drop = rng.permutation(plain)[:len(hub) - m_target]     # nested: a smaller m drops more
        keep = np.setdiff1d(np.arange(len(hub)), drop)
        out = {k: v[keep] for k, v in out.items()}
        hub = hub[keep]
    iso = gt[n - 1] + np.array([0.5, 0.5, 0.5, 0.1])            # the free node without factors
    out["gt"] = np.concatenate([gt, iso[None]])
    out["init"] = np.concatenate([g["init"], iso[None]])
    out["fixed"] = np.concatenate([g["fixed"], [0]]).astype(np.uint8)
    out["fixed"][fixed_node] = 1
    out["init"][fixed_node] = gt[fixed_node]
    out["n_nodes"] = n + 1
    out["hub"] = hub
    out["hub_node"], out["isolated"] = hub_node, n
    return out


def _union(parts):
    """disjoint copies: node ids offset, each copy keeping its own fixed nodes"""
    off = np.cumsum([0] + [p["n_nodes"] for p in parts])
    g = {k: np.concatenate([p[k] for p in parts]) for k in ("ftype", "huber", "payload", "gt", "init", "fixed", "hub")}
    g["ia"] = np.concatenate([p["ia"] + o for p, o in zip(parts, off)]).astype(np.int32)
    g["ib"] = np.concatenate([p["ib"] + o for p, o in zip(parts, off)]).astype(np.int32)
    g["n_nodes"] = int(off[-1])
    g["hub_node"] = np.array([p["hub_node"] + o for p, o in zip(parts, off)])
    g["isolated"] = np.array([p["isolated"] + o for p, o in zip(parts, off)])
    g["copies"] = [(int(o), int(o + p["n_nodes"])) for p, o in zip(parts, off[:-1])]
    return g


def _shuffled(g, seed):
    """node ids and factor order permuted, so that every CTA's block mixes factor types and nodes"""
    rng = np.random.default_rng(seed + 900)
    n, m = g["n_nodes"], len(g["ftype"])
    perm = rng.permutation(n)                  # old id -> new id
    fo = rng.permutation(m)
    out = dict(g)
    for k in ("ftype", "huber", "payload", "hub"):
        out[k] = g[k][fo]
    out["ia"] = perm[g["ia"][fo]].astype(np.int32); out["ib"] = perm[g["ib"][fo]].astype(np.int32)
    for k in ("gt", "init", "fixed"):
        arr = np.empty_like(g[k]); arr[perm] = g[k]; out[k] = arr
    out["hub_node"] = perm[np.atleast_1d(g["hub_node"])]
    out["isolated"] = perm[np.atleast_1d(g["isolated"])]
    out["copy_of"] = np.zeros(n, np.int64)
    for c, (a, b) in enumerate(g.get("copies", [(0, n)])):
        out["copy_of"][perm[a:b]] = c
    out["n_copies"] = len(g.get("copies", [(0, n)]))
    return out


@functools.lru_cache(maxsize=None)
def graph(name):
    """the pose graph of a row; n and m in the windows that put it in the row's shape (see ROWS)"""
    if name == "c5":        # 2001 nodes, 12 060 factors: one cluster, fast path
        g, seed = _decorated(5, 400, 4000, 4000, 1965, 60, seed=0), 1
    elif name == "m20k":    # 2001 nodes, 20 000 factors: one cluster, slow factor loop (fp32 Jacobians fit)
        g, seed = _decorated(5, 400, 6000, 8000, 3905, 60, seed=1), 2
    elif name in ("m12288", "m12289", "m12800"):   # 2001 nodes, m = 12 288 / 12 289 / 12 800: one graph, ranges dropped
        g, seed = _decorated(5, 400, 4800, 4000, 1965, 60, seed=2, m_target=int(name[1:])), int(name[1:])
    elif name == "n6k":     # 6 copies: 6006 nodes, 12 120 factors: one cluster, slow node loop only
        g, seed = _union([_decorated(5, 200, 400, 400, 170, 15, seed=20 + k) for k in range(6)]), 3
    elif name == "m13k":    # 2001 nodes, 13 000 factors: cooperative, fast path
        g, seed = _decorated(5, 400, 5000, 4000, 1905, 60, seed=4), 4
    elif name == "m110k":   # 10 copies: 5010 nodes, 110 650 factors: cooperative, slow factor loop
        g, seed = _union([_decorated(5, 100, 5000, 4000, 1500, 30, seed=10 + k) for k in range(10)]), 5
    elif name == "n34k":    # 36 copies: 34 236 nodes, 48 744 factors: cooperative, slow node loop
        g, seed = _union([_decorated(5, 190, 150, 150, 60, 9, seed=100 + k) for k in range(36)]), 6
    else:
        raise KeyError(name)
    return _shuffled(g, seed)


def shape_of(n, m, f32, sms=SMS):
    """solve_shape's choice for n nodes, m factors (the cluster always fits the device here) -> dict"""
    tsz = 4 if f32 else 8
    G = max(1, min(MAX_CLUSTER, -(-max(n, m) // THREADS)))
    fpc = -(-m // G)
    if fpc * 32 * tsz <= SMEM_J and -(-n // THREADS) <= 4 * G:
        return dict(cluster=1, ctas=G, fpc=fpc, j_in_smem=1, fast=fpc <= FAST_FPC and n <= G * THREADS)
    G0 = max(1, min(sms, -(-max(n, m) // THREADS)))
    fpc = -(-m // G0)
    return dict(cluster=0, ctas=G0, fpc=fpc, j_in_smem=int(fpc * 32 * tsz <= SMEM_J),
                fast=fpc <= FAST_FPC and n <= G0 * THREADS)


# row -> (graph, inner precision, preconditioner, expected shape).  The expectation names the path: "fast" False with
# "slow" = "factors" (ceil(m / ctas) > 768) or "nodes" (n > ctas * 256, ceil(m / ctas) <= 768).  E64 is the fp64
# twin of the fp32 row E; G's path (cooperative, slow) runs in fp64 in rows H (J global) and I (J shared).
ROWS = {
    "A64": ("c5", "fp64", "auto", dict(cluster=1, fast=True, j_in_smem=1, chain=1)),
    "A32": ("c5", "fp32", "auto", dict(cluster=1, fast=True, j_in_smem=1, chain=1)),
    "B": ("c5", "fp64", "jacobi", dict(cluster=1, fast=True, j_in_smem=1, chain=0)),
    "C": ("m20k", "fp32", "auto", dict(cluster=1, fast=False, slow="factors", j_in_smem=1, chain=0)),
    "D12288": ("m12288", "fp64", "auto", dict(cluster=1, fast=True, j_in_smem=1, chain=1)),
    "D12289": ("m12289", "fp64", "auto", dict(cluster=1, fast=False, slow="factors", j_in_smem=1, chain=0)),
    "D12800": ("m12800", "fp64", "auto", dict(cluster=1, fast=False, slow="factors", j_in_smem=1, chain=0)),
    "E": ("n6k", "fp32", "auto", dict(cluster=1, fast=False, slow="nodes", j_in_smem=1, chain=0)),
    "E64": ("n6k", "fp64", "auto", dict(cluster=1, fast=False, slow="nodes", j_in_smem=1, chain=0)),
    "F": ("m13k", "fp64", "auto", dict(cluster=0, fast=True, j_in_smem=1, chain=0)),
    "G": ("m110k", "fp32", "auto", dict(cluster=0, fast=False, slow="factors", j_in_smem=1, chain=0)),
    "H": ("m110k", "fp64", "auto", dict(cluster=0, fast=False, slow="factors", j_in_smem=0, chain=0)),
    "I": ("n34k", "fp64", "auto", dict(cluster=0, fast=False, slow="nodes", j_in_smem=1, chain=0)),
}
# the MT (J) and DT (K) rows run on row C's graph in fp32 and on row D12800's in fp64 (both one cluster, slow factor loop):
# name -> (shape row, DT tail rows, DT max_tail)
MT_TRIALS = 4
MT_DT = {"32": ("C", 400, 600), "64": ("D12800", 400, 400)}


# ---------------------------------------------------------------------------------------------------------------------
# the one-step check and its sensitivity
# ---------------------------------------------------------------------------------------------------------------------
def step_vector(sysm, x0, x1):
    """the step x1 - x0 of the free nodes in lm_system's column layout"""
    return (x1[sysm["free"]] - x0[sysm["free"]]).reshape(-1)


def backward_error(sysm, delta):
    A = sysm["H"] @ delta + (sysm["D"] / sysm["radius"]) * delta
    return float(np.linalg.norm(A + sysm["grad"]) / np.linalg.norm(sysm["grad"]))


def tol32(sysm, delta):
    """the backward error an fp32-inner step may have: its H is the product of fp32-rounded Jacobians, which moves
    H delta by up to a few u32 |J|^T |J| |delta| (componentwise); the CG stops at PCG32 relative residual"""
    aJ = abs(sysm["J"])
    return C32 * U32 * float(np.linalg.norm(aJ.T @ (aJ @ np.abs(delta))) / np.linalg.norm(sysm["grad"])) + PCG32


@functools.lru_cache(maxsize=None)
def oracle_step(name):
    """(lm_system at init with the default initial trust radius, its exact step)"""
    g = graph(name)
    sysm = sr.lm_system(g, g["init"], 1e4)
    return sysm, sr.lm_step(sysm)


def tolerance(row):
    name, inner = ROWS[row][0], ROWS[row][1]
    if inner == "fp64":
        return TOL64
    sysm, delta = oracle_step(name)
    return tol32(sysm, delta)


def drop_errors(sysm, g, unit, n_sample=50, seed=0):
    """backward errors, in the full system, of the oracle's own exact steps with H missing one unit: one factor's
    J^T J (unit "factor") or those of one node's first 16 factors, one slot batch of the fast path (unit "batch"), for
    about n_sample units including the one of smallest |J| (Woodbury on one factorisation of A = H + D / radius)"""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    J = sysm["J"]
    A = (sysm["H"] + sp.diags(sysm["D"] / sysm["radius"])).tocsc()
    lu = spla.splu(A, permc_spec="MMD_AT_PLUS_A", diag_pivot_thresh=0.0, options=dict(SymmetricMode=True))
    delta = lu.solve(-sysm["grad"])
    base = A @ delta + sysm["grad"]
    m = J.shape[0] // 4
    fsq = np.add.reduceat(J.multiply(J).sum(1).A1, np.arange(0, 4 * m, 4))
    if unit == "factor":
        groups = [np.array([f]) for f in range(m)]
    else:
        order = np.argsort(np.concatenate([g["ia"], g["ib"]]), kind="stable")
        ends = np.searchsorted(np.concatenate([g["ia"], g["ib"]])[order], np.arange(g["n_nodes"] + 1))
        groups = [order[ends[v]:min(ends[v + 1], ends[v] + 16)] % m for v in range(g["n_nodes"])]
    size = np.array([np.sqrt(fsq[grp].sum()) for grp in groups])
    live = np.nonzero(size > 0)[0]
    rng = np.random.default_rng(seed)
    pick = np.unique(np.concatenate([[live[np.argmin(size[live])]], rng.choice(live, n_sample - 1, replace=False)]))
    gn = np.linalg.norm(sysm["grad"])
    errs = []
    for u in pick:
        rows = (4 * groups[u][:, None] + np.arange(4)[None, :]).reshape(-1)
        Jk = J[rows].toarray()                                         # A_k = A - Jk^T Jk, Jk nonzero on `cols` only
        cols = np.nonzero(np.abs(Jk).sum(0))[0]
        Uk = Jk[:, cols]
        rhs = np.zeros((A.shape[0], len(Uk)))
        rhs[cols] = Uk.T
        W = Uk @ lu.solve(rhs)[cols]                                   # Jk A^-1 Jk^T
        y = np.linalg.solve(np.eye(len(Uk)) - W, Uk @ delta[cols])    # delta_k = delta + A^-1 Jk^T y
        r = base.copy()
        r[cols] += Uk.T @ y                                            # A delta_k + grad = base + Jk^T y
        errs.append(np.linalg.norm(r) / gn)
    return np.array(errs), pick, size


# ---------------------------------------------------------------------------------------------------------------------
# CPU part
# ---------------------------------------------------------------------------------------------------------------------
def test_lm_system_reproduces_solve_fast_first_step():
    g = graph("c5")
    ref = sr.solve_fast(g, max_iters=1)
    sysm = sr.lm_system(g, g["init"], 1e4)
    delta = sr.lm_step(sysm)
    step = step_vector(sysm, g["init"], ref["poses"])
    assert ref["iterations"] == 1 and np.abs(step).max() > 1e-3          # the first step was accepted
    assert np.abs(step - delta).max() <= 1e-12 * np.abs(delta).max() + 1e-14
    assert sysm["cost"] == ref["initial_cost"]
    assert backward_error(sysm, delta) < 1e-12
    assert len(sysm["free"]) == g["n_nodes"] - int(g["fixed"].sum()) and np.all(sysm["col_of"][g["fixed"] != 0] < 0)


@pytest.mark.parametrize("name", sorted({r[0] for r in ROWS.values()}))
def test_graph_builders(name):
    g = graph(name)
    n, m = g["n_nodes"], len(g["ftype"])
    rows = [r for r, v in ROWS.items() if v[0] == name]
    for r in rows:                                                     # the (n, m) window of each row on 132 SMs
        _, inner, _, want = ROWS[r]
        s = shape_of(n, m, inner == "fp32")
        assert s["cluster"] == want["cluster"] and s["fast"] == want["fast"] and s["j_in_smem"] == want["j_in_smem"], (r, s)
        assert {sr.FACTOR_DISTANCE, sr.FACTOR_RELPOSE} <= set(g["ftype"][: s["fpc"]]), r     # CTA 0's block mixes types
        blocks = np.flatnonzero(g["ftype"] == sr.FACTOR_DETECTION) // s["fpc"]                # detections in many blocks
        assert len(np.unique(blocks)) >= min(s["ctas"], 8), r
        if want.get("slow") == "factors":
            assert s["fpc"] > FAST_FPC, (r, s)
        elif want.get("slow") == "nodes":
            assert s["fpc"] <= FAST_FPC < n and n > s["ctas"] * THREADS, (r, s)
    if name in ("m12288", "m12289", "m12800"):
        assert m == int(name[1:])
    deg = np.bincount(np.concatenate([g["ia"], g["ib"]]), minlength=n)
    assert np.all(deg[g["hub_node"]] > 2 * 16)                          # more than two 16-slot batches
    assert np.all(deg[g["isolated"]] == 0) and np.all(g["fixed"][g["isolated"]] == 0)
    for c in range(g["n_copies"]):                                     # each copy: its own node 0 and one more fixed
        fx = np.nonzero((g["fixed"] != 0) & (g["copy_of"] == c))[0]
        assert len(fx) == 2
    assert np.all(g["copy_of"][g["ia"]] == g["copy_of"][g["ib"]])      # copies are disjoint
    det = g["ftype"] == sr.FACTOR_DETECTION                            # all three detection flag modes
    assert set(g["payload"][det, 10].astype(int)) == {0, 1, 3}
    _, r, _, _ = sr.evaluate_vec(g, g["init"], want_jac=False)
    assert np.sum((g["huber"] != 0) & ((r * r).sum(1) > 1.0)) >= 10     # Huber-active at init
    assert not np.all(np.diff(g["ia"]) >= 0) and np.flatnonzero(g["fixed"])[0] != 0     # numbering shuffled


@pytest.mark.parametrize("row", list(ROWS))
def test_one_step_tolerance_can_fail(row):
    """fp64 rows: dropping any one of ~50 factors (the one of smallest |J| among them) from H makes the oracle's own exact
    step miss the full system by >= 10x the tolerance of the one-step check.  fp32 rows: one factor sits at the level of
    the fp32 Jacobians' own rounding (a few 1e-7 of |grad| on these graphs), so the unit is one node's 16-slot batch --
    what a skipped node or a lost slot batch would drop; the fp64 rows of the same code paths see single factors."""
    name, inner = ROWS[row][0], ROWS[row][1]
    sysm, _ = oracle_step(name)
    if inner == "fp64":
        errs, pick, size = drop_errors(sysm, graph(name), "factor")
    else:
        errs, pick, size = drop_errors(sysm, graph(name), "batch", n_sample=25)
    tol = tolerance(row)
    print(f"SHAPES {row}: smallest drop error {errs.min():.3e} tol {tol:.3e}")
    assert errs.min() >= 10.0 * tol, (row, errs.min(), tol, size[pick[np.argmin(errs)]])


# ---------------------------------------------------------------------------------------------------------------------
# GPU part
# ---------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def solver(gpu):
    s = host.PoseGraphSolver(40000, 120000)
    yield s
    s.close()


def device_sms():
    import torch
    return torch.cuda.get_device_properties(0).multi_processor_count


def options(solver, inner, precond="auto", kind="default"):
    o = solver.default_options()
    o.inner_precision = 2 if inner == "fp32" else 1                    # OSB_INNER_FP32 / OSB_INNER_FP64
    if precond == "jacobi":
        o.preconditioner = 1                                           # OSB_PRECOND_BLOCK_JACOBI
    if kind == "step":                                                 # one LM step, the CG run to its tolerance
        o.max_iterations = 1
        o.pcg_tolerance = PCG32 if inner == "fp32" else PCG64
        o.max_pcg_iterations = 20000
    elif kind == "tight":
        o.function_tolerance = 1e-14; o.gradient_tolerance = 1e-11; o.parameter_tolerance = 1e-12
        o.pcg_tolerance = 1e-8; o.max_pcg_iterations = 2000; o.max_iterations = 300
    return o


def assert_shape(solver, row, n, m):
    _, inner, _, want = ROWS[row]
    c = solver.phase_cycles()
    expect = shape_of(n, m, inner == "fp32", device_sms())
    got = dict(cluster=int(c["cluster"]), ctas=int(c["ctas"]), j_in_smem=int(c["j_in_smem"]),
               chain=int(c["chain_preconditioner"]), f32=int(c["inner_fp32"]))
    assert got["ctas"] == expect["ctas"] and got["cluster"] == expect["cluster"] == want["cluster"], (row, got, expect)
    assert got["j_in_smem"] == want["j_in_smem"] and got["chain"] == want["chain"], (row, got)
    assert got["f32"] == int(inner == "fp32"), (row, got)
    fpc = -(-m // got["ctas"])
    fast = fpc <= FAST_FPC and n <= got["ctas"] * THREADS
    assert fast == want["fast"], (row, fpc, n, got)
    if want.get("slow") == "factors":
        assert fpc > FAST_FPC
    elif want.get("slow") == "nodes":
        assert fpc <= FAST_FPC and n > got["ctas"] * THREADS
    return got


def check_step(sysm, x0, poses, s, g, tol, label):
    """check 2 on a step the kernel took from x0: accepted, fixed nodes and the free nodes without factors (whose
    1e-10 diagonal would hide a move from the backward error) bit-unchanged, backward error <= tol"""
    assert s.iterations == 1, (label, s.iterations, s.termination)
    assert np.array_equal(poses[g["fixed"] != 0], x0[g["fixed"] != 0]), label
    assert np.array_equal(poses[g["isolated"]], x0[g["isolated"]]), label
    delta = step_vector(sysm, x0, poses)
    assert np.abs(delta).max() > 1e-3, label                            # the step was accepted
    err = backward_error(sysm, delta)
    print(f"SHAPES {label}: backward error {err:.3e} tol {tol:.3e} pcg {s.pcg_iterations}")
    assert err <= tol, (label, err, tol)
    return err


@functools.lru_cache(maxsize=None)
def converged_vs_oracle(name):
    """solve_fast at the tight tolerances, each disjoint copy of graph(name) alone -> (poses, final cost)"""
    g = graph(name)
    poses = g["init"].copy()
    cost = 0.0
    for c in range(g["n_copies"]):
        nodes = np.flatnonzero(g["copy_of"] == c)
        local = -np.ones(g["n_nodes"], np.int64); local[nodes] = np.arange(len(nodes))
        sel = g["copy_of"][g["ia"]] == c
        sub = {k: g[k][sel] for k in ("ftype", "huber", "payload")}
        sub["ia"] = local[g["ia"][sel]].astype(np.int32); sub["ib"] = local[g["ib"][sel]].astype(np.int32)
        sub["init"], sub["fixed"] = g["init"][nodes], g["fixed"][nodes]
        ref = sr.solve_fast(sub, max_iters=300, function_tol=1e-14, gradient_tol=1e-11, param_tol=1e-12)
        poses[nodes] = ref["poses"]
        cost += ref["final_cost"]
    return poses, cost


@pytest.mark.gpu
@pytest.mark.parametrize("row", list(ROWS))
def test_shape_row(solver, row):
    t0 = time.perf_counter()
    name, inner, precond, _ = ROWS[row]
    g = graph(name)
    n, m = g["n_nodes"], len(g["ftype"])
    sysm, _ = oracle_step(name)
    # 1 + 2: the initial cost and one LM step
    poses, s = solver.solve(g, options(solver, inner, precond, "step"))
    assert_shape(solver, row, n, m)
    assert abs(s.initial_cost - sysm["cost"]) <= 1e-12 * sysm["cost"], (s.initial_cost, sysm["cost"])
    check_step(sysm, g["init"], poses, s, g, tolerance(row), row)
    # 4: the converged window
    if inner == "fp64":
        p, s = solver.solve(g, options(solver, inner, precond, "tight"))
        assert_shape(solver, row, n, m)
        ref_poses, ref_cost = converged_vs_oracle(name)
        assert s.termination in (0, 1, 2), s.termination
        assert abs(s.final_cost - ref_cost) <= 1e-8 * ref_cost, (s.final_cost, ref_cost)
        assert np.abs(p - ref_poses).max() <= 1e-4
        assert s.n_residuals == sr.num_residuals(g)
    else:
        p32, s32 = solver.solve(g, options(solver, "fp32", precond))
        assert_shape(solver, row, n, m)
        p64, s64 = solver.solve(g, options(solver, "fp64", precond))
        assert s32.iterations == s64.iterations and s32.termination == s64.termination
        assert abs(s32.final_cost - s64.final_cost) <= 1e-7 * s64.final_cost, (s32.final_cost, s64.final_cost)
        assert np.abs(p32 - p64).max() <= 1e-5
    print(f"SHAPES {row}: {solver.phase_cycles()} wall {time.perf_counter() - t0:.1f} s")


def mt_setup(prec):
    """row J's inputs: (graph, restart mask, seed, rand_xy, rand_z, the K starting poses).  The restarted nodes are the
    few that start near the origin, so every trial's first step is accepted."""
    g = graph(ROWS[MT_DT[prec][0]][0])
    mask = np.zeros(g["n_nodes"], np.uint8)
    mask[np.argsort(np.linalg.norm(g["gt"][:, :3], axis=1))[:12]] = 1
    seed, rxy, rz = 31, 0.4, 0.3
    return g, mask, seed, rxy, rz, mr.multistart_initial_poses(g["init"], mask, g["fixed"], MT_TRIALS, seed, rxy, rz)


def dt_split(prec):
    """row K's inputs: the row's graph as a resident base and a tail of plain ranges between nodes inside their drone's
    odometry chain (never a chain end, so the tail leaves the chain plan as it is) -> (base, tail, full)"""
    g = graph(ROWS[MT_DT[prec][0]][0])
    deg_ego = np.bincount(np.concatenate([g["ia"][g["huber"] == 0], g["ib"][g["huber"] == 0]]), minlength=g["n_nodes"])
    inner = (deg_ego[g["ia"]] == 2) & (deg_ego[g["ib"]] == 2)
    cand = np.flatnonzero((g["ftype"] == sr.FACTOR_DISTANCE) & ~g["hub"] & inner)
    tail_idx = cand[:MT_DT[prec][1]]
    keep = np.setdiff1d(np.arange(len(g["ftype"])), tail_idx)
    base = {k: g[k][keep] for k in KEYS}
    tail = {k: g[k][tail_idx] for k in KEYS}
    full = {k: np.concatenate([base[k], tail[k]]) for k in KEYS}
    for d in (base, full):
        d["init"], d["fixed"], d["isolated"] = g["init"], g["fixed"], g["isolated"]
    return base, tail, full


@functools.lru_cache(maxsize=None)
def dt_system(prec):
    """the oracle's system of row K's step: the concatenated list at init"""
    full = dt_split(prec)[2]
    return sr.lm_system(full, full["init"], 1e4)


def step_tolerance(prec, sysm):
    return TOL64 if prec == "64" else tol32(sysm, sr.lm_step(sysm))


@pytest.mark.parametrize("prec", list(MT_DT))
def test_one_step_tolerance_can_fail_multi_trial(prec):
    """check 3 for row J's system, from a restart (row K's is its row's system: the same factors in another order):
    in fp64 one dropped factor, in fp32 one node's slot batch, as for the rows"""
    g, _, _, _, _, starts = mt_setup(prec)
    sysm = sr.lm_system(g, starts[0], 1e4)                             # trial 0's start stands for every trial's
    if prec == "64":
        errs, _, _ = drop_errors(sysm, g, "factor")
    else:
        errs, _, _ = drop_errors(sysm, g, "batch", n_sample=25)
    tol = step_tolerance(prec, sysm)
    print(f"SHAPES J{prec}: smallest drop error {errs.min():.3e} tol {tol:.3e}")
    assert errs.min() >= 10.0 * tol, (prec, errs.min(), tol)


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(MT_DT))
def test_multi_trial_row(solver, prec):
    """row J: solve_multistart, every trial in one launch of MT_TRIALS clusters (the MT kernel): trials bit-identical to
    single solves, the chosen trial's first step against the oracle's system"""
    t0 = time.perf_counter()
    row = MT_DT[prec][0]
    g, mask, seed, rxy, rz, starts = mt_setup(prec)
    n, m = g["n_nodes"], len(g["ftype"])
    inner = ROWS[row][1]
    for kind in ("default", "step"):
        o = options(solver, inner, kind=kind)
        poses, chosen, summ, _ = solver.solve_multistart(g, mask, MT_TRIALS, seed, window_size=100, acpt_cost=math.inf,
                                                         options=o, rand_xy=rxy, rand_z=rz)
        assert_shape(solver, row, n, m)
        assert 0 <= chosen < MT_TRIALS
        for t in range(MT_TRIALS):
            p, s = solver.solve(g, o, init=starts[t])
            for f in ("final_cost", "initial_cost", "iterations", "pcg_iterations", "termination", "n_residuals"):
                assert getattr(s, f) == getattr(summ[t], f), (kind, t, f)
            if t == chosen:
                assert np.array_equal(p, poses)
        if kind == "step":
            sysm = sr.lm_system(g, starts[chosen], 1e4)
            assert abs(summ[chosen].initial_cost - sysm["cost"]) <= 1e-12 * sysm["cost"]
            check_step(sysm, starts[chosen], poses, summ[chosen], g, step_tolerance(prec, sysm), "J" + prec)
    print(f"SHAPES J{prec}: wall {time.perf_counter() - t0:.1f} s")


@pytest.mark.gpu
@pytest.mark.parametrize("prec", list(MT_DT))
def test_device_tail_row(gpu, prec):
    """row K: FactorRows.solve on the row's base with a tail (the DT kernel): bit-identical to the one-shot solve of the
    concatenated list, its first step against the oracle's system"""
    from backend_harness import resident
    t0 = time.perf_counter()
    row, n_tail, max_tail = MT_DT[prec]
    base, tail, full = dt_split(prec)
    n, m = len(full["init"]), len(full["ftype"])
    plan = host.PoseGraphSolver.chain_plan
    assert all(np.array_equal(a, b) for a, b in zip(plan(base), plan(full)))
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    buf = host.FactorRows(max_tail)
    buf.set(tail)
    try:
        for kind in ("default", "step"):
            o = options(dev, ROWS[row][1], kind=kind)
            resident(dev, base)
            buf.solve(dev, max_tail, o)
            poses = dev.graph_get_poses()
            s = dev.last_summary()
            got = assert_shape(dev, row, n, m - n_tail + max_tail)
            ref, s1 = flat.solve(full, o)
            assert got == assert_shape(flat, row, n, m)
            assert np.array_equal(poses, ref)
            assert (s.initial_cost, s.final_cost, s.iterations, s.pcg_iterations, s.n_residuals, s.termination) == \
                (s1.initial_cost, s1.final_cost, s1.iterations, s1.pcg_iterations, s1.n_residuals, s1.termination)
            if kind == "step":
                sysm = dt_system(prec)
                assert abs(s.initial_cost - sysm["cost"]) <= 1e-12 * sysm["cost"]
                check_step(sysm, full["init"], poses, s, full, step_tolerance(prec, sysm), "K" + prec)
    finally:
        for h in (dev, flat):
            h.close()
    print(f"SHAPES K{prec}: wall {time.perf_counter() - t0:.1f} s")
