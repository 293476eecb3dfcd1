"""GPU: the re-anchoring of every loop and detection onto the window before a solve -- osb_anchor_run on the device
against the single-threaded C stand-in of the reference's walk (oracle/c/anchor_ref.c) and the numpy oracle
(oracle/anchor_ref.anchor_vec), on the same inputs.  Prints one JSON line; writes nothing.

Set-up: the C5 window, 5 drones x 400 keyframes 0.5 s apart, 100 Hz odometry (synth.anchor_swarm), and L = 6 005,
60 050 and 600 050 measurements in all_loops / all_detections_6d (a long flight: the lists only grow).  The 6 005
distinct measurements are generated once and tiled, with new ids, to 600 050.
Per size, after --warmup runs:
  * device: CUDA events around osb_anchor_run_dev (one launch) on a caller stream, median of --reps;
  * wall: host clock around the blocking osb_anchor_run (launch, copy of the rows to the host, synchronise);
  * C stand-in: host clock around one walk (inputs packed beforehand), median of --c-reps;
  * numpy oracle: host clock around one anchor_vec call.
The device rows are checked against the C stand-in's (integer fields identical, floats to 1e-12 relative).  The card's
name and power limit are read in the same run.

    python scripts/bench_anchor.py [--reps 20] [--warmup 3] [--c-reps 3]
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
from oracle import anchor_c, anchor_ref as ar  # noqa: E402

SIZES = (6005, 60050, 600050)
INT_FIELDS = ("status", "frame_a", "frame_b", "node_a", "node_b", "dt_err_ns", "skip", "ia", "ib")


def same(res, ref):
    if any(not np.array_equal(res[f], ref[f]) for f in INT_FIELDS):
        return False
    for got, want in ((res["payload"], ref["payload"]), (res["edge"]["rel_pose"], ref["edge"]["rel_pose"]),
                      (res["edge"]["cov"], ref["edge"]["cov"]), (res["dpos"], ref["dpos"])):
        if np.any(np.abs(got - want) > 1e-12 * np.maximum(np.abs(want), 1.0)):
            return False
    return True


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--c-reps", type=int, default=3)
    args = ap.parse_args()
    L = lib.load()
    assert L.osb_device_count() > 0, "needs a CUDA device"
    g = synth.anchor_swarm(5, 400, SIZES[0], seed=0, with_orphans=False)
    base = g["meas"]
    yaw = np.ones(g["max_drones"], np.uint8)
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm"),
           "drones": 5, "frames": 400, "window_entries": int(len(g["window"][2])), "reps": args.reps, "sizes": []}
    stream = torch.cuda.Stream()
    for n in SIZES:
        reps = -(-n // len(base))
        meas = np.concatenate([base] * reps)[:n].copy()
        meas["id"] = np.arange(n) + (1 << 32)
        a = host.LoopAnchor(g["max_drones"], max(len(v[0]) for v in g["trajs"].values()), n, len(g["window"][2]),
                            g["prm"]["det_dpos_thres"], g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"])
        for d, (st, p) in g["trajs"].items():
            a.push_odometry(d, st, p)
        a.add_measurements(meas)
        a.set_window(*g["window"])
        buf = torch.empty(n * lib.ANCHOR_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        dev_ms, wall_ms = [], []
        for r in range(args.warmup + args.reps):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            a.run_dev(buf.data_ptr(), stream.cuda_stream, yaw)
            e1.record(stream)
            e1.synchronize()
            t0 = time.perf_counter()
            res = a.run(yaw)
            ms = (time.perf_counter() - t0) * 1e3
            if r >= args.warmup:
                dev_ms.append(e0.elapsed_time(e1))
                wall_ms.append(ms)
        walk = anchor_c.Walk(g["trajs"], g["window"], meas, yaw, g["prm"])
        c_ms = [walk.run() for _ in range(args.c_reps)]
        t0 = time.perf_counter()
        ref_np = ar.anchor_vec(g["trajs"], g["window"], meas, yaw, g["prm"])
        np_ms = (time.perf_counter() - t0) * 1e3
        ok = same(res, walk.out) and same(ref_np, walk.out)
        ok = ok and buf.cpu().numpy().tobytes() == res.tobytes()
        a.close()
        row = {"measurements": n, "device_ms_events": float(np.median(dev_ms)), "device_ms_min": float(np.min(dev_ms)),
               "run_ms_wall": float(np.median(wall_ms)), "c_standin_ms": float(np.median(c_ms)),
               "numpy_oracle_ms": np_ms, "c_over_device": float(np.median(c_ms) / np.median(dev_ms)),
               "c_over_run_wall": float(np.median(c_ms) / np.median(wall_ms)),
               "statuses": np.bincount(res["status"], minlength=6).tolist(), "rows_identical": bool(ok)}
        out["sizes"].append(row)
        print(json.dumps(row), file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
