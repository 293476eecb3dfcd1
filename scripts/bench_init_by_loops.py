"""GPU: the start of the pre-motion init solve (init_pose_by_loops) on the device (osb_anchor_init_by_loops_dev) against
the host form an adapter computes today (the keyframe paths, the PCM inlier sets, to_init and the solve's rows read back,
the loop map kept and tests/init_by_loops_ref.py's numpy form run on the host, the start written with graph_set_poses),
and the whole pre-motion branch (run_dev -> record_loops -> observe -> reject_anchored -> compact -> distance_factors ->
init_by_loops -> multistart with one trial -> sync_dev) replayed as one CUDA graph against the same calls uncaptured.
Prints one JSON line; writes nothing.

Set-up per size (5 drones x 50 and 100 keyframes, 16 drones x 100 keyframes; synth.anchor_swarm, 4 measurements per
keyframe, non-redundant PCM): the swarm's first solve, whose observe marks every drone seen from self to be initialised
while only self is estimated (no sync has applied), so every such drone is placed from a loop to self.
After --warmup runs, medians of --reps:
  * start, device: host clock around init_by_loops_dev plus one stream synchronise, and CUDA events around it (1 launch);
  * start, host: host clock around the reads, the numpy form and graph_set_poses;
  * branch: host clock and CUDA events around the uncaptured calls and around one graph replay.
The device start is checked against the numpy form (1e-12 relative).  The card's name, power limit and SM clock are read
in the same run.

    python scripts/bench_init_by_loops.py [--reps 20] [--warmup 3]
"""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gpu_env import ClockSampler, smi  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402
import init_by_loops_ref as ib  # noqa: E402

SIZES = ((5, 50), (5, 100), (16, 100))
SELF, XY, Z, WIN = 0, 1e6, 1e6, 400


class Rig:
    def __init__(self, g, base):
        self.g = g
        cap = len(g["meas"]) + 64
        self.a = host.LoopAnchor(g["max_drones"], len(g["trajs"][0][0]) + 64, cap, len(g["window"][2]) + 64,
                                 g["prm"]["det_dpos_thres"], g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"])
        for d, (s, p) in g["trajs"].items():
            self.a.push_odometry(d, s, p)
        self.a.add_measurements(g["meas"])
        self.a.set_window(*g["window"])
        D = g["max_drones"]
        self.pcm = host.PcmState(SELF, False, 15.0, g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"],
                                 max_pairs=D, pair_capacity=1024)
        self.dev = host.PoseGraphSolver(8192, 65536)
        self.dev.graph_add_nodes(base["init"], base["fixed"])
        self.dev.graph_add_factors(*(base[k] for k in host.FACTOR_KEYS))
        self.o = self.dev.default_options()
        self.chain = host.AnchoredChain(cap)
        self.n_nodes = len(base["init"])
        self.cap = cap

    def front(self):
        c = self.chain
        n = c.run(self.a)
        c.record_loops(self.a, n)
        c.observe(self.a, n, SELF, XY, Z)
        c.reject(self.pcm, n)
        c.compact(n)
        c.distances(self.a, self.cap, SELF)
        return n

    def branch(self):
        self.front()
        c = self.chain
        c.init_by_loops(self.a, self.pcm, self.dev, SELF, self.n_nodes)
        c.init_solve(self.dev, self.cap, 1, 7, WIN, np.inf, options=self.o)
        self.a.sync_dev(self.dev, c.stream.cuda_stream, SELF, np.inf, WIN, True, False)

    def host_start(self, n):
        """today's adapter path for the start: everything read back, the numpy form, graph_set_poses"""
        g, D = self.g, self.g["max_drones"]
        with torch.cuda.stream(self.chain.stream):
            rows = self.chain.rows[:n * lib.ANCHOR_RESULT_DTYPE.itemsize].cpu().numpy().view(lib.ANCHOR_RESULT_DTYPE)
        lm = ib.LoopMapVec(D, lib.LOOP_RECORD_DTYPE)                # the adapter's map, fed this solve's rows
        lm.record_vec(rows)
        good = {}
        for a in range(D):
            for b in range(a, D):
                s = self.pcm.inliers(a, b)
                if s is not None:
                    good[(a, b)] = s
        kf = {d: p for d in range(D) if (p := self.a.paths(d)) is not None}
        to_init = self.a.observability()["to_init"]
        est = np.zeros(D, bool)
        est[SELF] = True                                           # no sync has applied yet
        poses = ib.init_by_loops_vec(to_init, good, lm, est, kf, g["trajs"], SELF, g["window"],
                                     self.dev.graph_get_poses())
        self.dev.graph_set_poses(0, poses)
        return poses

    def close(self):
        for h in (self.a, self.pcm, self.dev):
            h.close()


def med(x):
    return float(np.median(x))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    L = lib.load()
    assert L.osb_device_count() > 0, "needs a CUDA device"
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm"),
           "reps": args.reps, "sizes": []}
    for n_drones, n_frames in SIZES:
        g = synth.anchor_swarm(n_drones, n_frames, 4 * n_frames, seed=0, with_orphans=False)
        base = synth.anchor_window_graph(g)
        r = Rig(g, base)
        s = r.chain.stream
        n = r.front()                                              # the first solve: to_init holds the drones seen
        s.synchronize()                                            # from self, which alone is estimated
        start0 = r.dev.graph_get_poses()
        dev_wall, dev_ev, host_wall, br_wall, br_ev, gr_wall, gr_ev = ([] for _ in range(7))
        ok = True
        graph = torch.cuda.CUDAGraph()
        with ClockSampler() as clk:
            for k in range(args.warmup + args.reps):
                r.dev.graph_set_poses(0, start0)
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record(s)
                r.a.init_by_loops_dev(r.pcm, r.dev, SELF, s.cuda_stream)
                e1.record(s)
                s.synchronize()
                t1 = time.perf_counter()
                got = r.dev.graph_get_poses()
                r.dev.graph_set_poses(0, start0)
                t2 = time.perf_counter()
                want = r.host_start(n)
                t3 = time.perf_counter()
                ok = ok and bool(np.all(np.abs(got - want) <= 1e-12 * np.maximum(1.0, np.abs(want))))
                if k >= args.warmup:
                    dev_wall.append((t1 - t0) * 1e3)
                    dev_ev.append(e0.elapsed_time(e1))
                    host_wall.append((t3 - t2) * 1e3)
            torch.cuda.synchronize()
            for k in range(args.warmup + args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record(s)
                r.branch()
                e1.record(s)
                s.synchronize()
                t1 = time.perf_counter()
                if k >= args.warmup:
                    br_wall.append((t1 - t0) * 1e3)
                    br_ev.append(e0.elapsed_time(e1))
            with torch.cuda.graph(graph, stream=s, capture_error_mode="global"):
                r.branch()
            for k in range(args.warmup + args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                e0.record()
                graph.replay()
                e1.record()
                torch.cuda.synchronize()
                t1 = time.perf_counter()
                if k >= args.warmup:
                    gr_wall.append((t1 - t0) * 1e3)
                    gr_ev.append(e0.elapsed_time(e1))
        row = {"drones": n_drones, "frames": n_frames, "window_entries": int(len(g["window"][2])), "rows": int(n),
               "start_device_ms_wall": med(dev_wall), "start_device_ms_events": med(dev_ev),
               "start_host_ms_wall": med(host_wall), "start_host_over_device": med(host_wall) / med(dev_wall),
               "branch_uncaptured_ms_wall": med(br_wall), "branch_uncaptured_ms_events": med(br_ev),
               "branch_graph_ms_wall": med(gr_wall), "branch_graph_ms_events": med(gr_ev),
               "sm_clock_mhz_median": med(clk.samples) if clk.samples else None, "start_equal_to_numpy": ok}
        out["sizes"].append(row)
        print(json.dumps(row), file=sys.stderr)
        del graph
        r.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
