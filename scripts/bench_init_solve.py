"""GPU: the random-restart initialisation (solve_with_multiple_init) for an adapter on the device chain, two ways:

  (A) today's path: osb_anchor_run on the host, the mask walked out of the window on the host (with the odometry yaw
      written into the masked blocks), the resident window + rows flattened into osb_solver_solve_multistart, and the
      chosen poses written back with graph_set_poses;
  (B) osb_anchor_init_mask_dev + osb_solver_solve_multistart_resident_dev + graph_get_poses: no row reaches the host.

Graphs: the C5 window (5 drones x 400 keyframes, synth.anchor_swarm(5, 400, 6005)) with its anchored rows as the tail,
the mask from the first observe of a fresh anchor (every drone reached from self_id is to_init); and synth.init_graph
(5 drones x 100 frames, odometry + UWB, drones 1-4 to init) resident with an empty tail, its mask uploaded once (there is
no window, so (B) is the multistart call + graph_get_poses and (A) skips the anchor).  K = 3 (INIT_TRIAL) and 32.
Per (graph, K): host wall time of each path and the trials' kernel time (CUDA events, summary.solve_ms), medians over
--reps after --warmup with the paths alternating which goes first; the trial chosen; the largest pose difference between
the paths.  The card's name and power limit are read in the same run.  Prints one JSON line per (graph, K); writes nothing.

    python scripts/bench_init_solve.py [--reps 10] [--warmup 2]
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

KEYS = host.FACTOR_KEYS
SELF, XY, Z = 0, 1.0, 0.3
SEED, ACPT = 7, float("inf")


def quat_yaw(q):
    return np.arctan2(2.0 * (q[:, 0] * q[:, 3] + q[:, 1] * q[:, 2]), 1.0 - 2.0 * (q[:, 2] * q[:, 2] + q[:, 3] * q[:, 3]))


def host_mask(entries, to_init, n):
    """the adapter's walk of the window: each block's latest entry decides its drone and odometry yaw"""
    last = len(entries) - 1 - np.unique(entries["block"][::-1], return_index=True)[1]
    e = entries[last]
    mask = np.zeros(n, np.uint8)
    yaw = np.zeros(n)
    sel = to_init[e["drone_id"]] & (e["drone_id"] != SELF)
    mask[e["block"][sel]] = 1
    yaw[e["block"][sel]] = quat_yaw(e["self_pose"][sel, 3:7])
    return mask, yaw


class Case:
    """one graph: a resident solver per path, the tail for (B) on the device and for (A) from the host"""

    def __init__(self, base, window_size, anchor=None, mask=None):
        self.base, self.window_size, self.anchor = base, window_size, anchor
        self.n = len(base["init"])
        self.solvers = [host.PoseGraphSolver(4096, 32768) for _ in range(2)]
        for s in self.solvers:
            s.graph_add_nodes(base["init"], base["fixed"])
            s.graph_add_factors(*(base[k] for k in KEYS))
        self.o = self.solvers[0].default_options()
        self.chain = host.AnchoredChain(max(1, len(anchor.run()) if anchor else 1))
        if anchor is not None:
            n = self.chain.run(anchor)
            self.chain.observe(anchor, n, SELF, XY, Z)
            self.chain.compact(n, keep=False)
            self.obs = anchor.observability()
            self.max_tail = int(self.chain.factors.on_host(self.chain.stream)["ftype"].shape[0])
        else:
            self.chain.factors.set({k: base[k][:0] for k in KEYS})
            self.chain.mask = torch.from_numpy(mask).cuda()
            yaw = base["init"][:, 3].copy()
            self.chain.yaw = torch.from_numpy(yaw).cuda()
            self.host_mask = (mask, yaw)
            self.max_tail = 0
        torch.cuda.synchronize()
        self.pose_a = base["init"].copy()

    def path_a(self, K):
        t0 = time.perf_counter()
        if self.anchor is not None:
            rows = self.anchor.run(self.obs["yaw"])
            ft, ia, ib, pl, hb = host.anchored_factor_rows(rows)
            mask, yaw = host_mask(self.anchor_window[2], self.obs["to_init"], self.n)
        else:
            ft, ia, ib, pl, hb = (self.base[k][:0] for k in KEYS)
            mask, yaw = self.host_mask
        g = {"ftype": np.concatenate([self.base["ftype"], ft]), "ia": np.concatenate([self.base["ia"], ia]),
             "ib": np.concatenate([self.base["ib"], ib]), "payload": np.concatenate([self.base["payload"], pl]),
             "huber": np.concatenate([self.base["huber"], hb]), "fixed": self.base["fixed"]}
        start = self.pose_a.copy()
        sel = (mask != 0) & (self.base["fixed"] == 0)
        start[sel, 3] = yaw[sel]
        poses, chosen, summ, _ = self.solvers[0].solve_multistart(g, mask, K, SEED, self.window_size, ACPT, True, self.o,
                                                                  init=start)
        if chosen >= 0:
            self.solvers[0].graph_set_poses(0, poses)
            self.pose_a = poses
        return (time.perf_counter() - t0) * 1e3, summ[0].solve_ms, chosen

    def path_b(self, K):
        t0 = time.perf_counter()
        c, s = self.chain, self.solvers[1]
        if self.anchor is not None:
            c.init_mask(self.anchor, SELF, self.n)
        c.init_solve(s, self.max_tail, K, SEED, self.window_size, ACPT, True, self.o)
        self.pose_b = s.graph_get_poses()
        chosen, summ, _ = s.last_multistart()
        return (time.perf_counter() - t0) * 1e3, summ[0].solve_ms, chosen

    def close(self):
        for h in self.solvers:
            h.close()


def run(case, K, reps, warmup):
    t = {"A": [], "B": []}
    kern = {"A": [], "B": []}
    chosen = {}
    diff = 0.0
    for r in range(warmup + reps):
        order = ("A", "B") if r % 2 == 0 else ("B", "A")
        for p in order:
            ms, km, c = (case.path_a if p == "A" else case.path_b)(K)
            chosen[p] = c
            if r >= warmup:
                t[p].append(ms)
                kern[p].append(km)
        diff = max(diff, float(np.abs(case.pose_b - case.pose_a).max()))
    return {"K": K, "wall_ms": {p: float(np.median(v)) for p, v in t.items()},
            "wall_ms_minmax": {p: [float(np.min(v)), float(np.max(v))] for p, v in t.items()},
            "trials_kernel_ms": {p: float(np.median(v)) for p, v in kern.items()},
            "chosen_last": chosen, "max_abs_pose_diff_A_B": diff, "tail_rows": case.max_tail}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    L = lib.load()
    assert L.osb_device_count() > 0, "needs a CUDA device"
    card = {"gpu": smi("name"), "power_limit_w": smi("power.limit")}
    # C5: the window, its anchored rows as the tail, the mask from a fresh anchor's first observe
    g = synth.anchor_swarm(5, 400, 6005, seed=0, with_orphans=False)
    base = synth.anchor_window_graph(g)
    a = host.LoopAnchor(g["max_drones"], max(len(v[0]) for v in g["trajs"].values()), len(g["meas"]) + 64,
                        len(g["window"][2]), g["prm"]["det_dpos_thres"], g["prm"]["odom_pos_cov_per_m"],
                        g["prm"]["odom_ang_cov_per_m"])
    for d, (s, p) in g["trajs"].items():
        a.push_odometry(d, s, p)
    a.set_window(*g["window"])
    a.add_measurements(g["meas"])
    c5 = Case(base, len(g["window"][0]), anchor=a)
    c5.anchor_window = g["window"]
    ig = synth.init_graph(5, 100, seed=0)
    init = Case(ig, 100, mask=ig["mask"])
    for name, case, extra in (("C5", c5, {"nodes": c5.n, "resident_factors": len(base["ftype"]),
                                          "to_init": np.flatnonzero(c5.obs["to_init"]).tolist()}),
                              ("init_graph", init, {"nodes": init.n, "resident_factors": len(ig["ftype"])})):
        for K in (3, 32):
            row = {"graph": name, **extra, **run(case, K, args.reps, args.warmup), **card}
            print(json.dumps(row), flush=True)
    for h in (c5, init):
        h.close()
    a.close()


if __name__ == "__main__":
    main()
