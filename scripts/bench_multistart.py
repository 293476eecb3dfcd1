"""GPU: the random-restart initialisation (osb_solver_solve_multistart, solve_with_multiple_init in
swarm_localization_solver.cpp:781-845) -- K restarts in one launch against the same K starts as K sequential
osb_solver_solve calls.  Prints one JSON line; writes nothing.

Graphs: the init graph (synth.init_graph: 5 drones x 100 frames of odometry + UWB, drones 1-4 scattered) and C5
(drones 1-4 scattered), acpt_cost 10.  For K = 3 and 32: device ms of the batched call (CUDA events) and its wall ms,
the K sequential solves (device ms summed, wall), the chosen trial, its equv_cost and the largest position error
against ground truth; on the init graph at K = 3 also K x the oracle's solve_fast on one thread (the CPU stand-in).

    python scripts/bench_multistart.py [--reps 3]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
for _v in ("OMP_NUM_THREADS", "OPENBLAS_NUM_THREADS", "MKL_NUM_THREADS"):
    os.environ.setdefault(_v, "1")                   # the CPU stand-in runs on one thread, as the reference's solver
import numpy as np  # noqa: E402

from gpu_env import gpu_name_and_power  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402
from oracle import multistart_ref as mr  # noqa: E402
from oracle import solver_ref as sr  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=3)
    args = ap.parse_args()
    assert lib.load().osb_device_count() > 0, "needs a CUDA device"
    solver = host.PoseGraphSolver(2048, 12288)
    c5 = synth.pose_graph_c5(0)
    graphs = {"init": (synth.init_graph(), 100),
              "C5": (dict(c5, mask=(np.arange(c5["n_nodes"]) % 5 != 0).astype(np.uint8)), 400)}
    out = {"metric": "multistart solve ms", "gpu": gpu_name_and_power()}
    for name, (g, window) in graphs.items():
        res = {"graph": f"{g['n_nodes']} nodes / {len(g['ftype'])} factors, drones 1-4 masked, acpt_cost 10"}
        for K in (3, 32):
            seed = 1
            solver.solve_multistart(g, g["mask"], K, seed, window, 10.0)                  # warm-up (arena)
            walls, devs = [], []
            for _ in range(args.reps):
                tw = time.perf_counter()
                poses, chosen, summ, equv = solver.solve_multistart(g, g["mask"], K, seed, window, 10.0)
                walls.append((time.perf_counter() - tw) * 1e3)
                devs.append(summ[0].solve_ms)
            starts = mr.multistart_initial_poses(g["init"], g["mask"], g["fixed"], K, seed)
            solver.solve(g, init=starts[0])                                                # warm-up
            tw = time.perf_counter()
            seq_dev = sum(solver.solve(g, init=starts[t])[1].solve_ms for t in range(K))
            seq_wall = (time.perf_counter() - tw) * 1e3
            r = {"batched_ms": float(np.median(devs)), "batched_wall_ms": float(np.median(walls)),
                 "sequential_ms": float(seq_dev), "sequential_wall_ms": float(seq_wall),
                 "speedup_device": float(seq_dev / np.median(devs)), "chosen": int(chosen),
                 "equv_cost": float(equv[chosen]) if chosen >= 0 else None,
                 "max_err_vs_gt_m": float(np.linalg.norm(poses[:, :3] - g["gt"][:, :3], axis=1).max()),
                 "trial_final_costs": [float(s.final_cost) for s in summ]}
            if name == "init" and K == 3:
                tw = time.perf_counter()
                cpu = [sr.solve_fast(dict(g, init=starts[t]))["final_cost"] for t in range(K)]
                r["cpu_standin_ms"] = (time.perf_counter() - tw) * 1e3
                r["cpu_standin_kind"] = "K x oracle solve_fast (scipy SuperLU LM, Ceres-default tolerances), 1 thread"
                r["cpu_standin_best_cost"] = float(min(cpu))
            res[f"K{K}"] = r
        out[name] = res
    solver.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
