"""Times osb_anchor_data_association_dev plus the predicated second run / observe (CUDA events, median of --reps) at
1/4/8/32 anonymous ids and 5/16/64 drones, and the same search in the CPU oracle (tests/da_init_ref.py's literal form,
a stand-in for the reference's C++ DFS, not the reference itself).  Prints one JSON line per shape."""
import argparse
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

from omniswarm_b200 import host  # noqa: E402
import da_init_ref as da  # noqa: E402
from test_da_init_ref import case  # noqa: E402
from test_gpu_anchor_data_association import XY, Z, front, window  # noqa: E402


def shape(n, n_anon):
    """self 1 detects n_anon drones; drone 0 has no odometry; each anonymous id has one detection"""
    targets = list(range(2, 2 + n_anon))
    anon = [(1, b, 1000 + j, 5 + j % 30) for j, b in enumerate(targets)]
    trajs, _, dets, _ = case(n, anon)
    trajs[0] = (np.zeros(0, np.int64), np.zeros((0, 7)))
    return trajs, dets


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--budget", type=int, default=1 << 12,
                    help="DFS calls: with no keyframe path every drone without an estimate passes the gate, so most "
                         "shapes end at this bound")
    args = ap.parse_args()
    budget = args.budget
    for n in (5, 16, 64):
        for n_anon in (1, 4, 8, 32):
            if n_anon > n - 2:
                continue
            trajs, dets = shape(n, n_anon)
            a = host.LoopAnchor(n, 64, 512, 4096, 1.0, 0.0015, 0.0015)
            a.set_data_association(3.345, 1000, budget)
            for d, (s, p) in trajs.items():
                if len(s):
                    a.push_odometry(d, s, p)
            a.add_measurements(dets)
            c = host.AnchoredChain(512)
            m = front(a, c, window(trajs, range(n)), 1)
            w = a.data_association_word()
            a.data_association_dev(1, c.stream.cuda_stream)        # the first call acquires
            c.stream.synchronize()
            applied = a.data_association_result()[0]
            ts = []
            for _ in range(args.reps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(c.stream):
                    e0.record()
                    # after a success the store holds no anonymous id: the gate and the scan run, the search does not
                    a.data_association_dev(1, c.stream.cuda_stream)
                    n2 = a.run_dev_if(c.rows.data_ptr(), w, c.stream.cuda_stream)
                    a.observe_dev_if(c.rows.data_ptr(), n2, w, c.stream.cuda_stream, 1, XY, Z)
                    e1.record()
                e1.synchronize()
                ts.append(e0.elapsed_time(e1))
            a.close()
            # the first search on a fresh store (its first calls' acquisitions made beforehand), device and oracle
            a = host.LoopAnchor(n, 64, 512, 4096, 1.0, 0.0015, 0.0015)
            a.set_data_association(3.345, 1000, budget)
            for d, (s, p) in trajs.items():
                if len(s):
                    a.push_odometry(d, s, p)
            w = a.data_association_word()
            front(a, c, window(trajs, range(n)), 1)
            a.data_association_dev(1, c.stream.cuda_stream)        # no detection yet: the gate fails
            a.observe_dev_if(c.rows.data_ptr(), 0, w, c.stream.cuda_stream, 1, XY, Z)
            a.add_measurements(dets)
            m = front(a, c, window(trajs, range(n)), 1)
            torch.cuda.synchronize()
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            with torch.cuda.stream(c.stream):
                e0.record()
                a.data_association_dev(1, c.stream.cuda_stream)
                n2 = a.run_dev_if(c.rows.data_ptr(), w, c.stream.cuda_stream)
                e1.record()
            e1.synchronize()
            first_ms = e0.elapsed_time(e1)
            status = a.data_association_result()[1]
            a.close()
            t = time.perf_counter()
            lit = da.da_literal(1, trajs, {}, dets, 3.345, max_nodes=budget)
            cpu_ms = (time.perf_counter() - t) * 1e3
            print(json.dumps(dict(drones=n, anon=n_anon, applied=applied, oracle_applied=lit[0], search_status=status,
                                  oracle_status=lit[1], rows=m, steady_ms=float(np.median(ts)), search_ms=first_ms, cpu_oracle_ms=cpu_ms,
                                  device=torch.cuda.get_device_name())), flush=True)


if __name__ == "__main__":
    main()
