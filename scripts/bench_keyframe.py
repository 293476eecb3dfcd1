"""Timing of the back-end's UWB half: add_as_keyframe's initial poses and outlier flags once per keyframe, and
setup_problem_with_sferror's rows once per solve.

  device form: LoopAnchor.add_keyframe_dev per keyframe and distance_factors_dev per solve, timed with CUDA events on
               the chain's stream (each window of calls ends in an event the host waits for);
  host form:   per keyframe the solver's poses read back, tests/keyframe_ref.py's vectorised initial poses and flags on
               the host, the poses uploaded again; per solve the vectorised rows on the host and one upload of the tail;
               timed with the host clock around work that ends in a device synchronise.

Windows: C5-sized (5 drones, 50 and 100 frames) and 16 drones (100 frames).  Prints one JSON line per window with the
GPU's name and power limit.  Needs a CUDA device; there is no CPU fall-back.
    python scripts/bench_keyframe.py [--reps 20]
"""
import argparse
import json
import os
import subprocess
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import torch  # noqa: E402

from omniswarm_b200 import host, lib as _l  # noqa: E402
import keyframe_ref as kr  # noqa: E402

SELF, SEED = 0, 3
KF = dict(outlier_threshold=0.3, elevation_threshold=0.5, minimum_distance=0.2)
PRM = dict(KF, enable_distance=True, debug_no_rejection=False, distance_measurement_cov=0.2, self_id=SELF)


def gpu_info() -> str:
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"],
                              capture_output=True, text=True, timeout=30).stdout.strip().splitlines()[0]
    except (OSError, subprocess.SubprocessError, IndexError):
        return torch.cuda.get_device_name(0)


def records(n_drones, n_kf):
    kfs = kr.random_keyframes(n_drones, n_kf, SEED, self_id=SELF)
    asg = kr.BlockAssigner()
    recs = [kr.keyframe_records(kf, asg, SELF, k >= 3) for k, kf in enumerate(kfs)]
    return kfs, recs, asg.next


def window_of(kfs, recs, stamp_offset=0):
    first = np.concatenate([[0], np.cumsum([len(n) for n, _ in recs])]).astype(np.int32)
    ent = np.zeros(int(first[-1]), _l.WINDOW_ENTRY_DTYPE)
    for (n, _), lo, kf in zip(recs, first, kfs):
        e = ent[lo:lo + len(n)]
        e["drone_id"], e["block"], e["vo_available"], e["self_pose"] = n["drone_id"], n["block"], n["vo_available"], n["pose"]
        e["stamp"] = kf["stamp"] + stamp_offset
    stamps = [kf["stamp"] + stamp_offset for kf in kfs]
    win = [(ts, {int(x["drone_id"]): int(x["block"]) for x in n}) for ts, (n, _) in zip(stamps, recs)]
    return stamps, first, ent, win


def run(n_drones, n_frames, reps):
    kfs, recs, n_blocks = records(n_drones, n_frames)
    chain = host.AnchoredChain(8192)
    st = chain.stream
    # device form: every keyframe of the window through add_keyframe_dev, then reps solves' rows; repeated on fresh
    # stamps (the ring holds 4 windows), the first pass a warm-up
    a = host.LoopAnchor(max(n_drones, 8), 64, 64, 8192, 1.0, 0.01, 0.01, max_keyframes=4 * n_frames)
    s = host.PoseGraphSolver(8192, 32768)
    s.graph_add_nodes(np.zeros((n_blocks, 4)))
    kf_ms, df_ms = [], []
    for rep in range(4):
        off = rep * 10_000_000_000_000
        ev0, ev1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        ev0.record(st)
        for k, kf in enumerate(kfs):
            a.add_keyframe_dev(s, kf["stamp"] + off, *recs[k], st.cuda_stream, SELF, k >= 3, seed=SEED, **KF)
        ev1.record(st)
        ev1.synchronize()
        stamps, first, ent, _ = window_of(kfs, recs, off)
        a.set_window(stamps, first, ent)
        chain.observe(a, 0, SELF, 0.0, 0.0)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record(st)
        for _ in range(reps):
            chain.compact(0, keep=False)
            chain.distances(a, 8192, SELF, distance_measurement_cov=PRM["distance_measurement_cov"])
        e1.record(st)
        e1.synchronize()
        if rep > 0:
            kf_ms.append(ev0.elapsed_time(ev1) / len(kfs))
            df_ms.append(e0.elapsed_time(e1) / reps)
    n_rows = len(chain.factors.on_host(st)["ia"])
    # host form: the same keyframes and solves
    s2 = host.PoseGraphSolver(8192, 32768)
    s2.graph_add_nodes(np.zeros((n_blocks, 4)))
    rows = host.FactorRows(8192)
    enable = np.ones(256, bool)
    hk_ms, hd_ms = [], []
    for rep in range(4):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        store, last = {}, None
        for k, kf in enumerate(kfs):
            nodes, dists = recs[k]
            p = kr.init_poses_vec(nodes, s2.graph_get_poses(), kf["stamp"], SELF, k >= 3, SEED)
            s2.graph_set_poses(0, p)
            store[kf["stamp"]] = (nodes, dists, kr.outlier_flags_vec(nodes, dists, p, last, dict(PRM, finish_init=k >= 3)))
            last = nodes
        torch.cuda.synchronize()
        t1 = time.perf_counter()
        win = window_of(kfs, recs)[3]
        for _ in range(reps):
            rows.set(kr.distance_rows_vec(win, store, enable, PRM))
        torch.cuda.synchronize()
        t2 = time.perf_counter()
        if rep > 0:
            hk_ms.append((t1 - t0) * 1e3 / len(kfs))
            hd_ms.append((t2 - t1) * 1e3 / reps)
    med = lambda v: float(np.median(v))  # noqa: E731
    return dict(drones=n_drones, frames=n_frames, rows_per_solve=n_rows,
                device_keyframe_ms=med(kf_ms), device_rows_ms=med(df_ms),
                host_keyframe_ms=med(hk_ms), host_rows_ms=med(hd_ms),
                spread_device_rows_ms=[min(df_ms), max(df_ms)], spread_host_rows_ms=[min(hd_ms), max(hd_ms)])


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    args = ap.parse_args()
    if not torch.cuda.is_available():
        sys.exit("bench_keyframe.py needs a CUDA device")
    gpu = gpu_info()
    for d, f in ((5, 50), (5, 100), (16, 100)):
        print(json.dumps(dict(run(d, f, args.reps), gpu=gpu)), flush=True)


if __name__ == "__main__":
    main()
