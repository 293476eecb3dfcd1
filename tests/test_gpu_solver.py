"""GPU parity of the pose-graph path: factor residuals / Jacobians and the converged solve vs the oracle."""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from omniswarm_b200 import synth, host
from oracle import solver_ref as sr

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def solver(gpu):
    s = host.PoseGraphSolver(4096, 32768)
    yield s
    s.close()


def tight(solver):
    o = solver.default_options()
    o.function_tolerance = 1e-14; o.gradient_tolerance = 1e-11; o.parameter_tolerance = 1e-12
    o.pcg_tolerance = 1e-8; o.max_pcg_iterations = 2000; o.max_iterations = 300
    return o


def test_linearize_matches_oracle(solver):
    g = synth.pose_graph(3, 12, n_uwb=20, n_loop=15, n_det=8, n_bearing=9, seed=3)
    z = np.load(os.path.join(GOLDEN, "graph_small.npz"))
    r, Ja, Jb = solver.linearize(g, g["init"])
    assert np.allclose(r, z["r"], rtol=1e-10, atol=1e-10)
    assert np.allclose(Ja, z["Ja"], rtol=1e-9, atol=1e-9) and np.allclose(Jb, z["Jb"], rtol=1e-9, atol=1e-9)
    # yaw wrap: poses shifted by 2*pi give the same residuals (NormalizeAngle, factors.hpp:34-40)
    p2 = g["init"].copy(); p2[::2, 3] += 2 * np.pi
    r2, _, _ = solver.linearize(g, p2)
    assert np.allclose(r2, r, atol=1e-8)


def test_solve_small_graph_converged_poses(solver):
    g = synth.pose_graph(3, 12, n_uwb=20, n_loop=15, n_det=8, n_bearing=9, seed=3)
    z = np.load(os.path.join(GOLDEN, "graph_small.npz"))
    poses, s = solver.solve(g, tight(solver))
    assert s.termination in (0, 1, 2), s.termination
    assert abs(s.initial_cost - z["initial_cost"]) < 1e-6 * z["initial_cost"]
    assert abs(s.final_cost - z["final_cost"]) < 1e-8 * max(1.0, z["final_cost"])
    assert np.abs(poses - z["poses"]).max() < 1e-5            # 1e-4 rel on metre-scale poses
    assert np.array_equal(poses[0], g["init"][0])             # constant block untouched (solver.cpp:1196-1199)
    assert s.n_residuals == sr.num_residuals(g)


@pytest.mark.parametrize("seed,outliers", [(0, 0.0), (1, 0.1)])
def test_solve_c1_window(solver, seed, outliers):
    """BASELINE config 1: 5 drones x 100 swarm frames (default max_keyframe_num), Huber active with outliers."""
    g = synth.pose_graph(5, 100, seed=seed, outlier_frac=outliers)
    ref = sr.solve(g, max_iters=300)
    poses, s = solver.solve(g, tight(solver))
    assert abs(s.final_cost - ref["final_cost"]) < 1e-7 * max(1.0, ref["final_cost"])
    assert np.abs(poses - ref["poses"]).max() < 1e-4
    assert s.final_cost < s.initial_cost


def test_solve_default_options_and_time_limit(solver):
    g = synth.pose_graph(5, 60, seed=2)
    poses, s = solver.solve(g)                                 # Ceres-default tolerances
    assert s.termination in (0, 1, 2) and s.final_cost < 1e-2 * s.initial_cost
    assert np.abs(poses - g["gt"]).max() < 0.5
    o = solver.default_options(); o.max_iterations = 2
    _, s2 = solver.solve(g, o)
    assert s2.iterations <= 2 and s2.termination == 3
    # solves are reproducible bit for bit (no atomics in the reduction / gather paths)
    p3, s3 = solver.solve(g)
    assert np.array_equal(p3, poses) and s3.final_cost == s.final_cost


def test_solver_argument_errors(solver):
    g = synth.pose_graph(2, 4, n_uwb=2, n_loop=2, n_det=1, seed=0)
    bad = dict(g); bad["ib"] = g["ia"].copy()                  # both blocks coincide: the adapter must skip these
    with pytest.raises(host._l.OsbError):
        solver.solve(bad)
    bad = dict(g); bad["ia"] = g["ia"].copy(); bad["ia"][0] = 10 ** 6
    with pytest.raises(host._l.OsbError):
        solver.solve(bad)


def test_solve_c5_full_size_properties(solver):
    """BASELINE config 5 graph (2000 nodes / 12000 factors): cost decreases monotonically to a fixed point that a
    second solve from the solution does not move (idempotence), and lands near ground truth."""
    g = synth.pose_graph_c5(0)
    poses, s = solver.solve(g)
    assert s.termination in (0, 1, 2) and s.final_cost < s.initial_cost * 1e-2
    assert np.abs(poses[:, :3] - g["gt"][:, :3]).max() < 0.5
    p2, s2 = solver.solve(g, init=poses)
    assert s2.iterations <= 3 and np.abs(p2 - poses).max() < 1e-3


def test_solve_c5_converged_poses_vs_oracle(solver):
    """The graph the bench times (BASELINE config 5: 2000 pose nodes, 12 000 factors) against the oracle run to the same
    tight tolerances: converged poses <= 1e-4, final cost <= 1e-8 relative, residual count equal."""
    g = synth.pose_graph_c5(0)
    ref = sr.solve_fast(g, max_iters=300, function_tol=1e-14, gradient_tol=1e-11, param_tol=1e-12)
    poses, s = solver.solve(g, tight(solver))
    assert s.termination in (0, 1, 2), s.termination
    assert abs(s.initial_cost - ref["initial_cost"]) < 1e-9 * ref["initial_cost"]
    assert abs(s.final_cost - ref["final_cost"]) < 1e-8 * ref["final_cost"], (s.final_cost, ref["final_cost"])
    assert np.abs(poses - ref["poses"]).max() < 1e-4
    assert s.n_residuals == ref["n_residuals"]
    # the default (Ceres-tolerance, fp32-inner) solve that the bench reports stops near the same point
    p_def, s_def = solver.solve(g)
    assert abs(s_def.final_cost - ref["final_cost"]) < 1e-6 * ref["final_cost"]
    assert np.abs(p_def - ref["poses"]).max() < 2e-2


def test_chain_preconditioner_same_answer_fewer_iterations(solver):
    """The chain (block-tridiagonal path) preconditioner and block-Jacobi solve the same normal equations: converged
    poses agree, the inner iteration count drops several-fold, and node ids in arbitrary order (the path cover has to find
    the chains) change nothing."""
    g = synth.pose_graph_c5(0)
    o_bj = solver.default_options(); o_bj.preconditioner = 1
    p_bj, s_bj = solver.solve(g, o_bj)
    assert solver.phase_cycles()["chain_preconditioner"] == 0.0
    p_ch, s_ch = solver.solve(g)
    assert solver.phase_cycles()["chain_preconditioner"] == 1.0
    assert s_ch.termination in (0, 1, 2)
    assert abs(s_ch.final_cost - s_bj.final_cost) < 1e-5 * s_bj.final_cost
    assert np.abs(p_ch - p_bj).max() < 2e-2                   # both stopped by the Ceres-default function tolerance
    assert s_ch.pcg_iterations * 3 < s_bj.pcg_iterations, (s_ch.pcg_iterations, s_bj.pcg_iterations)
    # tight solves agree to parity tolerance
    pt_ch, st_ch = solver.solve(g, tight(solver))
    ot = tight(solver); ot.preconditioner = 1
    pt_bj, st_bj = solver.solve(g, ot)
    assert np.abs(pt_ch - pt_bj).max() < 1e-5 and abs(st_ch.final_cost - st_bj.final_cost) < 1e-8 * st_bj.final_cost
    # shuffled node numbering
    rng = np.random.default_rng(1)
    perm = rng.permutation(g["n_nodes"])
    g2 = dict(g)
    g2["ia"] = perm[g["ia"]].astype(np.int32); g2["ib"] = perm[g["ib"]].astype(np.int32)
    for key in ("init", "gt", "fixed"):
        arr = np.empty_like(g[key]); arr[perm] = g[key]; g2[key] = arr
    p2, s2 = solver.solve(g2, tight(solver))
    assert np.abs(p2[perm] - pt_ch).max() < 1e-5
    assert s2.pcg_iterations < 2 * st_ch.pcg_iterations + 50


def test_fp32_inner_solve_matches_fp64_inner_solve(solver):
    """Default options run the PCG in fp32 (LM needs an inexact step only); forcing fp64 inside must give the same outer
    iterations, (almost) the same inner iteration count and the same poses far inside the parity tolerance."""
    for g in (synth.pose_graph_c5(0), synth.pose_graph(5, 100, seed=1, outlier_frac=0.1)):
        p32, s32 = solver.solve(g)
        assert solver.phase_cycles()["inner_fp32"] == 1.0
        o = solver.default_options(); o.inner_precision = 1
        p64, s64 = solver.solve(g, o)
        assert solver.phase_cycles()["inner_fp32"] == 0.0
        assert s32.iterations == s64.iterations and s32.termination == s64.termination
        assert abs(s32.pcg_iterations - s64.pcg_iterations) <= max(10, s64.pcg_iterations // 20)
        assert abs(s32.final_cost - s64.final_cost) < 1e-7 * s64.final_cost
        assert np.abs(p32 - p64).max() < 1e-5


def _frames_of(g, n_drones):
    return (np.maximum(g["ia"], g["ib"]) // n_drones)


def test_resident_graph_incremental_equals_one_shot(solver):
    """SURVEY 8f-4: nodes and factors appended frame by frame (as add_new_swarm_frame / add_new_loop_connection would)
    give bit-for-bit the one-shot solve of the same arrays; poses persist; the one-shot entry point can be mixed in."""
    nd = 5
    g = synth.pose_graph(nd, 60, seed=4)
    # stream the graph in 4 chunks of frames; a factor is added once both of its nodes exist (factor order is kept)
    fr_of = _frames_of(g, nd)
    order = np.argsort(fr_of, kind="stable")
    g2 = dict(g)
    for k in ("ftype", "ia", "ib", "huber"):
        g2[k] = g[k][order]
    g2["payload"] = g["payload"][order]
    ref_poses, ref_s = solver.solve(g2)
    solver.graph_clear()
    bounds = [0, 15, 30, 45, 60]
    fr2 = fr_of[order]
    for a, b in zip(bounds[:-1], bounds[1:]):
        first = solver.graph_add_nodes(g["init"][a * nd:b * nd], g["fixed"][a * nd:b * nd])
        assert first == a * nd
        sel = (fr2 >= a) & (fr2 < b)
        solver.graph_add_factors(g2["ftype"][sel], g2["ia"][sel], g2["ib"][sel], g2["payload"][sel], g2["huber"][sel])
    assert solver.graph_size() == (g["n_nodes"], len(g["ftype"]))
    s = solver.solve_resident()
    poses = solver.graph_get_poses()
    assert np.array_equal(poses, ref_poses) and s.final_cost == ref_s.final_cost and s.pcg_iterations == ref_s.pcg_iterations
    # unchanged topology: the second solve re-uses the cached path cover / index tables (host and device) and must be
    # bit-identical when restarted from the same poses
    solver.graph_set_poses(0, g["init"])
    s1b = solver.solve_resident()
    assert np.array_equal(solver.graph_get_poses(), ref_poses) and s1b.final_cost == ref_s.final_cost
    assert s1b.pcg_iterations == ref_s.pcg_iterations
    # poses persist: a second solve starts from the solution and stops at once
    s2 = solver.solve_resident()
    assert s2.iterations <= 2 and np.abs(solver.graph_get_poses() - poses).max() < 1e-3
    # a one-shot solve on the same handle in between must not corrupt the resident factor arrays
    other = synth.pose_graph(3, 12, n_uwb=20, n_loop=15, n_det=8, seed=3)
    solver.solve(other)
    solver.graph_set_poses(0, g["init"])
    s3 = solver.solve_resident()
    assert np.array_equal(solver.graph_get_poses(), ref_poses) and s3.final_cost == ref_s.final_cost
    # ... and neither may a linearize of another graph, with the resident topology (and its cached tables) unchanged
    solver.linearize(other, other["init"])
    solver.graph_set_poses(0, g["init"])
    s4 = solver.solve_resident()
    assert np.array_equal(solver.graph_get_poses(), ref_poses) and s4.final_cost == ref_s.final_cost
    assert s4.pcg_iterations == ref_s.pcg_iterations


def test_resident_graph_sliding_window(solver):
    """drop_oldest (solver.cpp:186-202 trims the window) == solving the sub-graph of the remaining frames"""
    nd = 5
    g = synth.pose_graph(nd, 40, seed=6)
    solver.graph_clear()
    solver.graph_add_nodes(g["init"], g["fixed"])
    solver.graph_add_factors(g["ftype"], g["ia"], g["ib"], g["payload"], g["huber"])
    drop = 10 * nd
    solver.graph_drop_oldest(drop)
    keep = (g["ia"] >= drop) & (g["ib"] >= drop)
    sub = dict(n_nodes=g["n_nodes"] - drop, init=g["init"][drop:].copy(), gt=g["gt"][drop:], fixed=g["fixed"][drop:].copy(),
               ftype=g["ftype"][keep], ia=g["ia"][keep] - drop, ib=g["ib"][keep] - drop, huber=g["huber"][keep],
               payload=g["payload"][keep])
    sub["fixed"][0] = 1                                    # the new oldest pose of drone 0 anchors the gauge
    solver.graph_set_fixed(0, True)
    assert solver.graph_size() == (sub["n_nodes"], int(keep.sum()))
    s = solver.solve_resident()
    ref_poses, ref_s = solver.solve(sub)
    assert np.array_equal(solver.graph_get_poses(), ref_poses) and s.final_cost == ref_s.final_cost
    with pytest.raises(host._l.OsbError):
        solver.graph_add_factors(sub["ftype"][:1], np.array([10 ** 6], np.int32), sub["ib"][:1], sub["payload"][:1], sub["huber"][:1])
