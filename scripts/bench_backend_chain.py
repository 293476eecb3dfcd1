"""GPU: one solve's chain from re-anchoring to factor rows -- the host sequence (A) against the device chain (B), on the same
anchor handle and two PCM states fed the same rounds.  Prints one JSON line; writes nothing.

  (A) osb_anchor_run (every row copied to the host), the OK rows through osb_pcm_state_reject, the keep mask scattered
      back and the kept rows with skip == 0 gathered as the solver's SoA (host.anchored_factor_rows);
  (B) osb_anchor_run_dev -> osb_pcm_state_reject_anchored -> osb_anchor_compact_factors_dev on one stream, then one copy
      of the count and one copy of that many SoA rows.

Set-up: the C5 window (5 drones x 400 keyframes, synth.anchor_swarm) and L = 6 005, 60 050 and 600 050 measurements as in
bench_anchor.py, except that the tiles keep the 6 005 base ids, so every row's id is one the PCM state has seen (the
first call on the 6 005 base rows stores them).  PCM state: redundant, 15 drone pairs, pair_capacity 4096.  Two cases per
size, host wall clock per solve, medians over --reps after --warmup, (A) and (B) alternating which goes first:
  * steady: no new measurement, every row's id already seen;
  * grow: before each solve every pair gains 4 loops (copies of the pair's OK loops under new ids).
Each solve's keep mask and SoA of (B) are checked byte-identical to (A)'s.  The card's name and power limit are read in
the same run.

    python scripts/bench_backend_chain.py [--reps 10] [--warmup 2]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402

from gpu_env import smi  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402

SIZES = (6005, 60050, 600050)
THRES = 15.0
NEW_PER_PAIR = 4


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    L = lib.load()
    assert L.osb_device_count() > 0, "needs a CUDA device"
    g = synth.anchor_swarm(5, 400, SIZES[0], seed=0, with_orphans=False)
    base = g["meas"]
    yaw = np.ones(g["max_drones"], np.uint8)
    rounds = args.warmup + args.reps
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "sm_clock_max_mhz": smi("clocks.max.sm"),
           "drones": 5, "frames": 400, "pairs": 15, "pair_capacity": 4096, "new_per_pair": NEW_PER_PAIR,
           "reps": args.reps, "warmup": args.warmup, "sizes": []}
    for n_meas in SIZES:
        meas = np.concatenate([base] * -(-n_meas // len(base)))[:n_meas].copy()
        cap = n_meas + 15 * NEW_PER_PAIR * rounds + 64
        a = host.LoopAnchor(g["max_drones"], max(len(v[0]) for v in g["trajs"].values()), cap, len(g["window"][2]),
                            g["prm"]["det_dpos_thres"], g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"])
        for d, (s, p) in g["trajs"].items():
            a.push_odometry(d, s, p)
        a.set_window(*g["window"])
        a.add_measurements(base)
        sa, sb = (host.PcmState(0, True, THRES, g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"],
                                max_pairs=15, pair_capacity=4096) for _ in range(2))
        dev = host.AnchoredChain(cap)
        first_rows = a.run(yaw)
        host.anchored_keep(sa, a.run(yaw))                           # both states store the base ids
        dev(a, sb, yaw)
        a.add_measurements(meas[len(base):])
        # per pair, its OK loops: the grow case re-submits them under new ids
        ok_loops = first_rows[(first_rows["status"] == lib.ANCHOR_OK) & (first_rows["type"] == lib.MEAS_LOOP)]
        by_pair = {}
        for r in ok_loops:
            by_pair.setdefault((min(r["edge"]["id_a"], r["edge"]["id_b"]), max(r["edge"]["id_a"], r["edge"]["id_b"])),
                               []).append(int(r["id"]))
        id_to_meas = {int(m["id"]): m for m in base}
        next_id = 1 << 40
        row = {"measurements": n_meas}
        same = True
        for case in ("steady", "grow"):
            ta, tb = [], []
            for r in range(rounds):
                if case == "grow":
                    add = []
                    for ids in by_pair.values():
                        for k in range(NEW_PER_PAIR):
                            m = id_to_meas[ids[(r * NEW_PER_PAIR + k) % len(ids)]].copy()
                            m["id"] = next_id
                            next_id += 1
                            add.append(m)
                    a.add_measurements(np.array(add, lib.MEASUREMENT_DTYPE))
                for form in ((0, 1) if r % 2 == 0 else (1, 0)):
                    t0 = time.perf_counter()
                    if form == 0:
                        rows = a.run(yaw)
                        keep_a = host.anchored_keep(sa, rows)
                        fa = host.anchored_factor_rows(rows, keep_a)
                    else:
                        n = dev(a, sb, yaw)
                        fb = dev.factors.on_host(dev.stream)         # the solve's one synchronisation, one copy of the rows
                    ms = (time.perf_counter() - t0) * 1e3
                    if r >= args.warmup:
                        (ta if form == 0 else tb).append(ms)
                same &= dev.keep_on_host(n).tobytes() == keep_a.tobytes()
                same &= all(x.tobytes() == y.tobytes() for x, y in zip(fa, fb.values()))
            row[case] = {"host_sequence_ms_wall": float(np.median(ta)), "host_sequence_ms_min": float(np.min(ta)),
                         "device_chain_ms_wall": float(np.median(tb)), "device_chain_ms_min": float(np.min(tb)),
                         "speedup": float(np.median(ta) / np.median(tb)), "rows": int(n),
                         "factors": int(len(fb["ftype"]))}
        row["identical"] = bool(same and sb.status() == lib.OK)
        out["sizes"].append(row)
        print(json.dumps(row), file=sys.stderr)
        for h in (sa, sb, a):
            h.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
