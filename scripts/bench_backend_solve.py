"""GPU: one back-end solve, from re-anchoring to solved poses, on the C5 window (5 drones x 400 keyframes,
synth.anchor_swarm(5, 400, 6005)) with its odometry + UWB factors resident.  Prints one JSON line; writes nothing.

  (A) today's path: the device chain (run_dev -> reject_anchored -> compact_factors_dev), the count and the SoA rows
      copied to the host, then osb_solver_solve of the whole window (resident factors + rows), as FlatPoseGraph does it;
  (B) the device chain, then osb_solver_solve_resident_dev on the same stream, then graph_get_poses;
  (C) (B) captured once into a CUDA graph and replayed, then graph_get_poses (steady case only: a captured run_dev has a
      fixed row count).

Each path has its own PCM state and solver handle and starts from the same poses.  Cases: steady (no new measurement)
and grow (every drone pair gains 4 loops before each solve).  Host wall time per solve and the solve kernel's event time
(summary.solve_ms), medians over --reps after --warmup, the paths alternating which goes first; each path's launch shape;
and how far (B) and (C) are from (A).  The card's name and power limit are read in the same run.

    python scripts/bench_backend_solve.py [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gpu_env import smi  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402

THRES = 15.0
NEW_PER_PAIR = 4
KEYS = host.FACTOR_KEYS


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    L = lib.load()
    assert L.osb_device_count() > 0, "needs a CUDA device"
    g = synth.anchor_swarm(5, 400, 6005, seed=0, with_orphans=False)
    base = synth.anchor_window_graph(g)
    n_nodes, m_base = len(base["init"]), len(base["ftype"])
    rounds = args.warmup + args.reps
    cap = len(g["meas"]) + 15 * NEW_PER_PAIR * rounds + 64
    a = host.LoopAnchor(g["max_drones"], max(len(v[0]) for v in g["trajs"].values()), cap, len(g["window"][2]),
                        g["prm"]["det_dpos_thres"], g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"])
    for d, (s, p) in g["trajs"].items():
        a.push_odometry(d, s, p)
    a.set_window(*g["window"])
    a.add_measurements(g["meas"])
    states = [host.PcmState(0, True, THRES, g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"],
                            max_pairs=15, pair_capacity=4096) for _ in range(3)]
    solvers = [host.PoseGraphSolver(4096, 32768) for _ in range(3)]
    chains = [host.AnchoredChain(cap) for _ in range(3)]
    for s in solvers[1:]:
        s.graph_add_nodes(base["init"], base["fixed"])
        s.graph_add_factors(*(base[k] for k in KEYS))
    o = solvers[0].default_options()
    rows0 = a.run()
    # sized to the window: every row the re-anchoring keeps (skip == 0), plus what the grow case adds
    max_tail = int((rows0["skip"] == 0).sum()) + 15 * NEW_PER_PAIR * rounds
    pose_a = base["init"].copy()

    def path_a():
        nonlocal pose_a
        c = chains[0]
        c(a, states[0])
        tail = c.factors.on_host(c.stream)
        gg = {key: np.concatenate([base[key], tail[key]]) for key in KEYS}
        gg["fixed"] = base["fixed"]
        pose_a, s = solvers[0].solve(gg, o, init=pose_a)
        return s, len(tail["ftype"])

    def path_b():
        c = chains[1]
        c(a, states[1])
        c.solve(solvers[1], max_tail, o)
        p = solvers[1].graph_get_poses()
        return solvers[1].last_summary(), p

    graph = None

    def path_c():
        nonlocal graph
        c = chains[2]
        if graph is None:                                    # the first solve runs uncaptured, then the chain is captured
            c(a, states[2])
            c.solve(solvers[2], max_tail, o)
            p = solvers[2].graph_get_poses()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=c.stream, capture_error_mode="global"):
                c(a, states[2])
                c.solve(solvers[2], max_tail, o)
            return None, p
        graph.replay()
        torch.cuda.synchronize()                             # a replay is not a library call: the caller waits for it
        return None, solvers[2].graph_get_poses()

    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm"),
           "drones": 5, "frames": 400, "measurements": len(g["meas"]), "nodes": n_nodes, "resident_factors": m_base,
           "max_tail": max_tail, "reps": args.reps, "warmup": args.warmup}
    next_id = 1 << 40
    ok_loops = rows0[(rows0["status"] == lib.ANCHOR_OK) & (rows0["type"] == lib.MEAS_LOOP)]
    by_pair = {}
    for r in ok_loops:
        by_pair.setdefault((min(r["edge"]["id_a"], r["edge"]["id_b"]), max(r["edge"]["id_a"], r["edge"]["id_b"])),
                           []).append(int(r["id"]))
    id_to_meas = {int(m["id"]): m for m in g["meas"]}
    for case in ("steady", "grow"):
        forms = (0, 1, 2) if case == "steady" else (0, 1)
        t = {f: [] for f in forms}
        kern = {0: [], 1: []}
        diff = {f: 0.0 for f in forms[1:]}
        for r in range(rounds):
            if case == "grow":
                add = []
                for ids in by_pair.values():
                    for q in range(NEW_PER_PAIR):
                        m = id_to_meas[ids[(r * NEW_PER_PAIR + q) % len(ids)]].copy()
                        m["id"] = next_id
                        next_id += 1
                        add.append(m)
                a.add_measurements(np.array(add, lib.MEASUREMENT_DTYPE))
            order = forms if r % 2 == 0 else forms[::-1]
            res = {}
            for f in order:
                t0 = time.perf_counter()
                res[f] = (path_a, path_b, path_c)[f]()
                ms = (time.perf_counter() - t0) * 1e3
                if r >= args.warmup:
                    t[f].append(ms)
            if r >= args.warmup:
                kern[0].append(res[0][0].solve_ms)
                kern[1].append(res[1][0].solve_ms)
            for f in forms[1:]:
                if res[f][1] is not None:
                    diff[f] = max(diff[f], float(np.abs(res[f][1] - pose_a).max()))
            if case == "steady" and r == 0:
                k_rows = res[0][1]
        row = {"wall_ms": {("A", "B", "C")[f]: float(np.median(t[f])) for f in forms},
               "wall_ms_min": {("A", "B", "C")[f]: float(np.min(t[f])) for f in forms},
               "solve_kernel_ms": {"A": float(np.median(kern[0])), "B": float(np.median(kern[1]))},
               "solve_kernel_ms_minmax": {"A": [float(np.min(kern[0])), float(np.max(kern[0]))],
                                          "B": [float(np.min(kern[1])), float(np.max(kern[1]))]},
               "max_abs_pose_diff_vs_A": {("A", "B", "C")[f]: diff[f] for f in forms[1:]}}
        out[case] = row
        print(json.dumps({case: row}), file=sys.stderr)
    out["tail_rows_first_steady_solve"] = int(k_rows)
    shapes = {}
    for name, s in zip("ABC", solvers):
        c = s.phase_cycles()
        shapes[name] = {k: c[k] for k in ("ctas", "cluster", "j_in_smem", "chain_preconditioner", "inner_fp32")}
    out["shape"] = shapes
    print(json.dumps(out))
    for h in states + solvers + [a]:
        h.close()


if __name__ == "__main__":
    main()
