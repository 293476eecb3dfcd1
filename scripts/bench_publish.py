"""GPU: what the back-end publishes after an accepted solve -- sync_est_poses' keyframe and full paths and the prediction
record -- computed on the device (osb_anchor_sync_dev) against the host form (the solved poses read back with
graph_get_poses, then tests/publish_ref.py's sync and numpy full path).  Prints one JSON line; writes nothing.

Set-up: the C5 window, 5 drones x 400 keyframes 0.5 s apart (synth.anchor_swarm), solved once through the device chain
(run_dev -> observe -> compact -> solve_resident_dev).  Each drone's odometry is cut or continued to 1e4, 1e5 and 2e5
samples (100 Hz; 2e5 is a flight of 33 minutes), so the full path has 1e3 .. 2e4 samples per drone.  The full path's
work grows with the flight; the keyframe paths' with the window.
Per size, after --warmup runs, medians of --reps:
  * device: host clock around sync_dev plus one stream synchronise, and CUDA events around sync_dev (3 launches);
  * host: host clock around graph_get_poses plus the numpy sync and full path.
The device paths are checked against the host form's (stamps identical, poses to 1e-12 relative).  The card's name,
power limit and SM clock are read in the same run.

    python scripts/bench_publish.py [--reps 20] [--warmup 3]
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
from oracle import anchor_ref as ar  # noqa: E402
import publish_ref as pb  # noqa: E402

SIZES = (10_000, 100_000, 200_000)
SELF, WIN = 0, 400


def odometry(g, n, seed=0):
    """each drone's odometry cut to n samples, or continued at 100 Hz with a small random walk"""
    rng = np.random.default_rng(seed)
    out = {}
    for d, (s, p) in g["trajs"].items():
        if n <= len(s):
            out[d] = (s[:n].copy(), p[:n].copy())
            continue
        k = n - len(s)
        st = s[-1] + 10_000_000 * np.arange(1, k + 1, dtype=np.int64)
        pos = p[-1, :3] + np.cumsum(rng.normal(0, 0.01, (k, 3)), axis=0)
        q = p[-1, 3:] + rng.normal(0, 0.02, (k, 4))
        q /= np.linalg.norm(q, axis=1, keepdims=True)
        out[d] = (np.concatenate([s, st]), np.concatenate([p, np.c_[pos, q]]))
    return out


def host_form(dev, win, trajs, T):
    st = pb.PublishState()
    st.sync(win, dev.graph_get_poses(), T, False, False)
    full = {d: pb.full_path_vec(st.kf[d], *trajs[d]) for d in st.kf}
    return st, full


def same(a, st, full, drones):
    for d in drones:
        for got, want in ((a.paths(d), st.kf.get(d)), (a.paths(d, True), full.get(d))):
            if (got is None) != (want is None):
                return False
            if got is None:
                continue
            if not np.array_equal(got[0], want[0]) or got[1].shape != want[1].shape:
                return False
            if np.any(np.abs(got[1] - want[1]) > 1e-12 * np.maximum(1.0, np.abs(want[1]))):
                return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    L = lib.load()
    assert L.osb_device_count() > 0, "needs a CUDA device"
    g = synth.anchor_swarm(5, 400, 2000, seed=0, with_orphans=False)
    base = synth.anchor_window_graph(g)
    win = g["window"]
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm"),
           "drones": 5, "frames": 400, "window_entries": int(len(win[2])), "reps": args.reps, "sizes": []}
    for n in SIZES:
        trajs = odometry(g, n)
        T = {d: ar.Trajectory(*v) for d, v in trajs.items()}
        a = host.LoopAnchor(g["max_drones"], n, len(g["meas"]), len(win[2]), g["prm"]["det_dpos_thres"],
                            g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"])
        for d, (s, p) in trajs.items():
            a.push_odometry(d, s, p)
        a.add_measurements(g["meas"])
        a.set_window(*win)
        dev = host.PoseGraphSolver(4096, 32768)
        dev.graph_add_nodes(base["init"], base["fixed"])
        dev.graph_add_factors(*(base[k] for k in host.FACTOR_KEYS))
        chain = host.AnchoredChain(len(g["meas"]) + 64)
        m = chain.run(a)
        chain.observe(a, m, SELF, 1.0, 0.3)
        chain.compact(m, keep=False)
        chain.solve(dev, len(g["meas"]) + 64)
        dev.last_summary()
        s = chain.stream
        dev_wall, dev_ev, host_ms = [], [], []
        with ClockSampler() as clk:
            for r in range(args.warmup + args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                t0 = time.perf_counter()
                e0.record(s)
                a.sync_dev(dev, s.cuda_stream, SELF, np.inf, WIN, True, True)
                e1.record(s)
                s.synchronize()
                t1 = time.perf_counter()
                st, full = host_form(dev, win, trajs, T)
                t2 = time.perf_counter()
                if r >= args.warmup:
                    dev_wall.append((t1 - t0) * 1e3)
                    dev_ev.append(e0.elapsed_time(e1))
                    host_ms.append((t2 - t1) * 1e3)
        applied, status = a.sync_result()
        ok = applied and status == lib.OK and same(a, st, full, range(g["max_drones"]))
        row = {"odometry_per_drone": n, "full_path_per_drone": (n + 9) // 10,
               "device_ms_wall": float(np.median(dev_wall)), "device_ms_events": float(np.median(dev_ev)),
               "host_ms_wall": float(np.median(host_ms)), "host_over_device": float(np.median(host_ms) /
                                                                                     np.median(dev_wall)),
               "sm_clock_mhz_median": float(np.median(clk.samples)) if clk.samples else None, "outputs_equal": bool(ok)}
        out["sizes"].append(row)
        print(json.dumps(row), file=sys.stderr)
        a.close()
        dev.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
