"""GPU: the observability estimate of a solve -- the mask that decides which loops and detections become factors -- in
its faithful host form against the device form (osb_anchor_observe_dev).  Prints one JSON line; writes nothing.

Set-up: the C5 window of scripts/bench_anchor.py, 5 drones x 400 keyframes 0.5 s apart, 100 Hz odometry
(synth.anchor_swarm), and L = 6 005, 60 050 and 600 050 measurements (6 005 distinct ones tiled with new ids).
Per size, after --warmup rounds, --reps rounds alternating:
  (A) host form: the blocking osb_anchor_run (rows to the host), the mask in numpy (the drone pairs of the OK rows, the
      closure from self_id, the window boxes), then osb_anchor_run_dev with that mask and a synchronisation;
  (B) device form: osb_anchor_run_dev with no drone observable, osb_anchor_observe_dev, one synchronisation.
Reported: host wall medians of (A) and (B), and the CUDA-event time of observe_dev alone (its three launches).  The rows
of (B) are checked byte for byte against (A)'s.  The card's name, power limit and SM clock are read in the same run.

    python scripts/bench_observability.py [--reps 20] [--warmup 3]
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

SIZES = (6005, 60050, 600050)
SELF, XY, Z = 0, 5.0, 2.0                # self_id, init_xy_movement, init_z_movement


def window_boxes(window, D):
    """per drone max - min of x, y, z over its vo_available entries, from -1000 / +1000 (boundingbox_sldwin)"""
    _, first, e = window
    e = e[: first[-1]]
    vo = e[e["vo_available"] != 0]
    hi, lo = np.full((D, 3), -1000.0), np.full((D, 3), 1000.0)
    np.maximum.at(hi, vo["drone_id"], vo["self_pose"][:, :3])
    np.minimum.at(lo, vo["drone_id"], vo["self_pose"][:, :3])
    return hi - lo, np.unique(e["drone_id"])


def host_mask(rows, ext, nodes, D):
    """the yaw mask of estimate_observability from rows on the host"""
    ok = rows["status"] == lib.ANCHOR_OK
    key = rows["edge"]["id_a"][ok].astype(np.int64) * D + rows["edge"]["id_b"][ok]
    adj = (np.bincount(key, minlength=D * D) > 0).reshape(D, D)
    adj |= adj.T
    seen = np.zeros(D, bool)
    seen[SELF] = True
    if len(nodes) > 1:
        front = seen.copy()
        while front.any():
            front = adj[front].any(0) & ~seen
            seen |= front
    yaw = seen.copy()
    node = np.zeros(D, bool)
    node[nodes] = True
    yaw |= node & ((ext[:, 0] > 1.0) | (ext[:, 1] > 1.0))
    return yaw.astype(np.uint8)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    L = lib.load()
    assert L.osb_device_count() > 0, "needs a CUDA device"
    g = synth.anchor_swarm(5, 400, SIZES[0], seed=0, with_orphans=False)
    base = g["meas"]
    D = g["max_drones"]
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm"),
           "drones": 5, "frames": 400, "window_entries": int(len(g["window"][2])), "reps": args.reps, "sizes": []}
    stream = torch.cuda.Stream()
    none = np.zeros(D, np.uint8)
    for n in SIZES:
        reps = -(-n // len(base))
        meas = np.concatenate([base] * reps)[:n].copy()
        meas["id"] = np.arange(n) + (1 << 32)
        a = host.LoopAnchor(D, max(len(v[0]) for v in g["trajs"].values()), n, len(g["window"][2]),
                            g["prm"]["det_dpos_thres"], g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"])
        for d, (st, p) in g["trajs"].items():
            a.push_odometry(d, st, p)
        a.add_measurements(meas)
        a.set_window(*g["window"])
        buf_a = torch.empty(n * lib.ANCHOR_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        buf_b = torch.empty_like(buf_a)
        host_ms, dev_ms, obs_ms = [], [], []
        same = True
        for r in range(args.warmup + args.reps):
            t0 = time.perf_counter()                             # (A)
            rows = a.run(none)
            ext, nodes = window_boxes(g["window"], D)
            yaw = host_mask(rows, ext, nodes, D)
            a.run_dev(buf_a.data_ptr(), stream.cuda_stream, yaw)
            stream.synchronize()
            t1 = time.perf_counter()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t2 = time.perf_counter()                             # (B)
            nb = a.run_dev(buf_b.data_ptr(), stream.cuda_stream, none)
            e0.record(stream)
            a.observe_dev(buf_b.data_ptr(), nb, stream.cuda_stream, SELF, XY, Z)
            e1.record(stream)
            stream.synchronize()
            t3 = time.perf_counter()
            if r >= args.warmup:
                host_ms.append((t1 - t0) * 1e3)
                dev_ms.append((t3 - t2) * 1e3)
                obs_ms.append(e0.elapsed_time(e1))
        same = buf_a.cpu().numpy().tobytes() == buf_b.cpu().numpy().tobytes()
        same = same and np.array_equal(a.observability()["yaw"], yaw.astype(bool))
        a.close()
        row = {"measurements": n, "host_form_ms_wall": float(np.median(host_ms)),
               "device_form_ms_wall": float(np.median(dev_ms)), "observe_ms_events": float(np.median(obs_ms)),
               "observe_ms_events_min": float(np.min(obs_ms)), "yaw_observable": int(yaw.sum()),
               "rows_identical": bool(same)}
        out["sizes"].append(row)
        print(json.dumps(row), file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
