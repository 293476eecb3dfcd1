"""GPU: the random-restart initialisation (osb_solver_solve_multistart, solve_with_multiple_init in
swarm_localization_solver.cpp:781-845): every trial of a batch is bit-identical to a single osb_solver_solve from the
same starting poses, and the device selects the trial the reference's acceptance walk selects."""
import ctypes as C
import math
import subprocess

import numpy as np
import pytest

from omniswarm_b200 import host, lib, synth
from oracle import multistart_ref as mr
from oracle import solver_ref as sr
from test_multistart_rules import build_multistart_smoke

pytestmark = pytest.mark.gpu

FIELDS = ("final_cost", "initial_cost", "iterations", "pcg_iterations", "termination", "n_residuals")


@pytest.fixture(scope="module")
def solver(gpu):
    s = host.PoseGraphSolver(4096, 32768)
    yield s
    s.close()


def c1_with_loops():
    g = synth.pose_graph(5, 100, seed=0)                      # C1: ego motion, UWB, loops, detections
    mask = (np.arange(g["n_nodes"]) % 5 != 0).astype(np.uint8)  # drones 1-4
    return g, mask


def equv_oracle(s, window):
    return math.sqrt(s.final_cost) / s.n_residuals / window


def check_trials_match_single_solves(solver, g, mask, K, seed, opt, window=100):
    poses, chosen, summ, equv = solver.solve_multistart(g, mask, K, seed, window, acpt_cost=math.inf, options=opt)
    starts = mr.multistart_initial_poses(g["init"], mask, g["fixed"], K, seed)
    singles = []
    for t in range(K):
        p, s = solver.solve(g, opt, init=starts[t])
        for f in FIELDS:
            assert getattr(s, f) == getattr(summ[t], f), (t, f, getattr(s, f), getattr(summ[t], f))
        singles.append(p)
    assert chosen == mr.select_trial(equv, math.inf)
    assert np.array_equal(poses, singles[chosen])
    return poses, chosen, summ, equv, singles


@pytest.mark.parametrize("inner", ["default", "fp64"])
def test_trials_bit_identical_to_single_solves(solver, inner):
    g, mask = c1_with_loops()
    opt = solver.default_options()
    if inner == "fp64":
        opt.inner_precision = 1                                        # OSB_INNER_FP64
    check_trials_match_single_solves(solver, g, mask, 8, seed=2024, opt=opt)
    assert solver.phase_cycles()["cluster"] == 1


def test_selection_follows_the_reference_rule(solver):
    g, mask = c1_with_loops()
    opt = solver.default_options()
    starts = mr.multistart_initial_poses(g["init"], mask, g["fixed"], 8, 77)
    poses, chosen, summ, equv = solver.solve_multistart(g, mask, 8, 77, window_size=100, acpt_cost=math.inf,
                                                        options=opt)
    ref = np.array([equv_oracle(s, 100) for s in summ])
    assert np.array_equal(equv, ref)                                   # bit for bit
    # an acpt_cost between the costs: only trials below it may be chosen, the lowest wins
    acpt = float(np.median(equv))
    poses2, chosen2, summ2, equv2 = solver.solve_multistart(g, mask, 8, 77, window_size=100, acpt_cost=acpt,
                                                            options=opt)
    assert np.array_equal(equv2, equv)
    assert chosen2 == mr.select_trial(equv, acpt) and chosen == mr.select_trial(equv, math.inf)
    assert chosen2 == chosen and equv[chosen] < acpt
    single, _ = solver.solve(g, opt, init=starts[chosen])
    assert np.array_equal(poses, single) and np.array_equal(poses2, single)
    # normalise off: equv_cost is the final cost itself
    _, chosen3, summ3, equv3 = solver.solve_multistart(g, mask, 8, 77, window_size=100, acpt_cost=math.inf,
                                                       normalise=False, options=opt)
    assert np.array_equal(equv3, np.array([s.final_cost for s in summ3]))
    assert chosen3 == mr.select_trial(equv3, math.inf)


def test_rejection_leaves_poses_untouched(solver):
    g, mask = c1_with_loops()
    init = g["init"].copy()
    init[5, 0] = np.nextafter(init[5, 0], 1.0)                          # a pose block that is not a round number
    _, _, summ_ok, _ = solver.solve_multistart(g, mask, 4, 5, 100, acpt_cost=math.inf, init=init)
    poses, chosen, summ, equv = solver.solve_multistart(g, mask, 4, 5, 100, acpt_cost=-1.0, init=init)
    assert chosen == -1
    assert np.array_equal(poses, init) and poses.tobytes() == init.tobytes()
    for t in range(4):
        assert summ[t].final_cost == summ_ok[t].final_cost and summ[t].iterations == summ_ok[t].iterations
        assert summ[t].iterations > 0 and equv[t] > 0.0


def test_finds_the_ground_truth_basin(solver):
    """UWB + odometry init graph, drone 0 at ground truth, drones 1-4 scattered: of the oracle's 32 starts for this
    seed, 3 reach the ground-truth basin (cost 310.06) and the others stop in a higher minimum (364.02)."""
    g = synth.init_graph()
    K, seed = 32, 1
    poses, chosen, summ, equv = solver.solve_multistart(g, g["mask"], K, seed, window_size=100, acpt_cost=10.0)
    assert chosen >= 0
    err = np.linalg.norm(poses[:, :3] - g["gt"][:, :3], axis=1).max()
    assert err < 0.5, err
    starts = mr.multistart_initial_poses(g["init"], g["mask"], g["fixed"], K, seed)
    ref = []
    for t in range(K):
        gg = dict(g); gg["init"] = starts[t]
        ref.append(sr.solve_fast(gg)["final_cost"])
    best = min(ref)
    assert abs(summ[chosen].final_cost - best) <= 1e-6 * best
    costs = np.array([s.final_cost for s in summ])
    reached = int(np.sum(costs <= best * (1 + 1e-3)))
    higher = int(np.sum(costs > best * 1.05))
    print(f"\nground-truth basin: {reached} of {K} trials on the GPU ({sum(c <= best * (1 + 1e-3) for c in ref)} "
          f"in the oracle), {higher} in a higher minimum; chosen trial {chosen}, max error {err:.3f} m")
    assert higher >= 1


def test_cooperative_fallback_runs_trials_in_turn(solver):
    # 13 000 factors with fp64 inner arithmetic: the Jacobians of a 16-CTA cluster exceed shared memory, so each
    # trial runs as a cooperative grid
    g = synth.pose_graph(5, 400, n_uwb=4000, n_loop=5000, n_det=2005, seed=4)
    assert len(g["ftype"]) > 12288
    mask = (np.arange(g["n_nodes"]) % 5 != 0).astype(np.uint8)
    opt = solver.default_options()
    opt.inner_precision = 1                                            # OSB_INNER_FP64
    opt.max_iterations = 30
    check_trials_match_single_solves(solver, g, mask, 2, seed=8, opt=opt, window=400)
    assert solver.phase_cycles()["cluster"] == 0


def _raw_call(solver, g, mask, ms, n_trials_buf=4, poses=None):
    L = lib.load()
    fixed, ftype, ia, ib, payload, huber = host.PoseGraphSolver._arrays(g)
    poses = np.ascontiguousarray(g["init"] if poses is None else poses, np.float64).copy()
    mask = None if mask is None else np.ascontiguousarray(mask, np.uint8)
    summ = (lib.SolveSummary * n_trials_buf)()
    equv = np.zeros(n_trials_buf)
    chosen = C.c_int32(0)
    opt = solver.default_options()
    return L.osb_solver_solve_multistart(solver._h, poses.shape[0], lib.ptr(poses), lib.ptr(fixed), lib.ptr(mask),
                                         len(ftype), lib.ptr(ftype), lib.ptr(ia), lib.ptr(ib), lib.ptr(payload),
                                         lib.ptr(huber), C.byref(opt), C.byref(ms), C.cast(summ, C.c_void_p),
                                         lib.ptr(equv), C.byref(chosen))


def test_invalid_arguments(solver):
    g = synth.pose_graph(3, 12, n_uwb=20, n_loop=15, n_det=8, seed=3)
    mask = (np.arange(g["n_nodes"]) % 3 != 0).astype(np.uint8)
    before, s_before = solver.solve(g)

    def ms(**kw):
        d = dict(n_trials=3, normalise=1, window_size=12, seed=1, rand_xy=5.0, rand_z=1.0, acpt_cost=10.0)
        d.update(kw)
        return lib.MultistartOptions(**d)

    assert _raw_call(solver, g, mask, ms()) == lib.OK
    assert _raw_call(solver, g, None, ms()) == lib.ERR_INVALID
    for bad in (dict(n_trials=0), dict(n_trials=257), dict(n_trials=-1), dict(window_size=0), dict(window_size=-3),
                dict(rand_xy=-1.0), dict(rand_xy=math.inf), dict(rand_xy=math.nan), dict(rand_z=-0.5),
                dict(rand_z=math.nan), dict(acpt_cost=math.nan)):
        assert _raw_call(solver, g, mask, ms(**bad)) == lib.ERR_INVALID, bad
    assert _raw_call(solver, g, mask, ms(normalise=0, window_size=0)) == lib.OK    # window unused without normalise
    bad_g = dict(g); bad_g["ia"] = g["ia"].copy(); bad_g["ia"][3] = g["n_nodes"]
    assert _raw_call(solver, bad_g, mask, ms()) == lib.ERR_INVALID
    self_g = dict(g); self_g["ib"] = g["ib"].copy(); self_g["ib"][2] = g["ia"][2]
    assert _raw_call(solver, self_g, mask, ms()) == lib.ERR_INVALID
    after, s_after = solver.solve(g)
    assert np.array_equal(before, after) and s_before.final_cost == s_after.final_cost
    assert s_before.iterations == s_after.iterations


def test_adapter_solve_with_multiple_init(gpu, tmp_path):
    exe = build_multistart_smoke(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "multistart ok" in r.stdout, r.stdout + r.stderr
