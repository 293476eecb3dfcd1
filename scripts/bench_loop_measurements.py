"""GPU: a round's accepted loop edges into the back-end's store -- osb_frontend_loop_measurements +
osb_anchor_add_measurements_dev against the host hop they replace.  Prints one JSON line; writes nothing.

Set-up: the front-end of bench_loop_edge.py (4 directions, max_num 200, geometric filter, one own keyframe in the local
store) and 64 received records of the same place (every one a hit that compute_loop accepts); the back-end of a 5-drone
swarm (synth.anchor_swarm(5, 60, 600)): trajectories, window, the 600 measurements, a redundant PCM state and the window's
pose graph resident in the solver.  Each loop's two stamps are window-entry stamps of its two drones.  For n in {1, 8, 64}
candidates:
  * calls: the CUDA-event time of loop_measurements + add_measurements_dev with the candidates' ctypes arrays built once
    (median of --reps after --warmup), against the
    host path: download the n edge and query results, build the rows in numpy, gate them, osb_anchor_add_measurements
    (wall clock, median of --host-reps);
  * round: query_received -> compute_loop -> loop_measurements -> add_measurements_dev -> run_dev -> reject_anchored ->
    compact_factors_dev -> solve_resident_dev, against the same round with the host hop in place of the two new calls;
    wall clock to the end of the solve, median of --round-reps, the two forms alternating which goes first.
Both round forms run on their own anchor, PCM state and solver, fed the same rounds; their solved poses are compared bit for
bit.  The card's name and power limit are read in the same run.

    python scripts/bench_loop_measurements.py [--reps 50] [--warmup 5] [--host-reps 20] [--round-reps 10]
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

ND, MN = 4, 200
RB, RS, EB = lib.RECORD_BYTES, lib.RESULT_BYTES, lib.EDGE_BYTES
MB = lib.MEASUREMENT_DTYPE.itemsize
SC = synth.LOOP_SCENE
SELF, MAX_LOOP_ID = 1, 100000000
COV_POS, COV_ANG, THRES = 0.02, 0.005, 2.0


def host_rows(edges_t, res_t, n, cands, stamps, loop_count):
    """the host hop: download the edge and query results and build the LoopEdge rows (loop_detector.cpp:787-829), then the
    solver's distance gate (swarm_localization_solver.cpp:558-588) -> (rows, loop_count)"""
    raw_e, raw_r = edges_t[:n * EB].cpu().numpy().tobytes(), res_t[:n * RS].cpu().numpy().tobytes()
    rows = []
    for i in range(n):
        e = lib.LoopEdgeResult.from_buffer_copy(raw_e[i * EB:(i + 1) * EB])
        if e.status != lib.LOOP_ACCEPTED:
            continue
        sw = lib.LoopResult.from_buffer_copy(raw_r[i * RS:(i + 1) * RS]).swapped
        r = np.zeros((), lib.MEASUREMENT_DTYPE)
        r["id"] = SELF * MAX_LOOP_ID + loop_count
        loop_count += 1
        r["type"], r["id_a"], r["id_b"] = lib.MEAS_LOOP, e.drone_id_a, e.drone_id_b
        q, h = stamps[i]
        r["stamp_a"], r["stamp_b"] = (q, h) if sw else (h, q)
        c = cands[i]
        r["self_pose_a"], r["self_pose_b"] = (c["pose_query"], c["pose_hit"]) if sw else (c["pose_hit"], c["pose_query"])
        r["relative_pose"] = e.relative_pose
        r["cov"] = np.diag([COV_POS] * 3 + [COV_ANG] * 3)
        x, y, z = r["relative_pose"][:3]
        if not (np.sqrt((x * x + y * y) + z * z) > np.float64(np.float32(THRES))):
            rows.append(r)
    return np.array(rows, lib.MEASUREMENT_DTYPE).reshape(-1), loop_count


def entry_stamps(g, drone):
    _, _, e = g["window"]
    return e["stamp"][(e["drone_id"] == drone) & (e["vo_available"] == 1)]


class Backend:
    """anchor + PCM state + resident solver, and one solve's chain on the current stream"""

    def __init__(self, g, base, cap):
        self.a = host.LoopAnchor(g["max_drones"], max(len(v[0]) for v in g["trajs"].values()), cap, len(g["window"][2]),
                                 g["prm"]["det_dpos_thres"], g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"])
        for d, (s, p) in g["trajs"].items():
            self.a.push_odometry(d, s, p)
        self.a.set_window(*g["window"])
        self.a.add_measurements(g["meas"])
        self.pcm = host.PcmState(0, True, 15.0, g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"], max_pairs=15,
                                 pair_capacity=4096)
        self.solver = host.PoseGraphSolver(4096, 65536)
        self.solver.graph_add_nodes(base["init"], base["fixed"])
        self.solver.graph_add_factors(base["ftype"], base["ia"], base["ib"], base["payload"], base["huber"])
        self.o = self.solver.default_options()
        self.cap = cap
        self.chain = host.AnchoredChain(cap, torch.cuda.current_stream())

    def solve(self):
        self.chain(self.a, self.pcm)
        self.chain.solve(self.solver, self.cap, self.o)

    def close(self):
        for h in (self.pcm, self.solver, self.a):
            h.close()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    ap.add_argument("--host-reps", type=int, default=20)
    ap.add_argument("--round-reps", type=int, default=10)
    a = ap.parse_args()
    assert lib.load().osb_device_count() > 0, "needs a CUDA device"
    fe = host.KeyframeFrontend(*synth.frontend_weights(), width=96, height=64, n_dirs=ND, max_num=MN, self_id=SELF,
                               db_capacity=64, match_index_dist=5, geometric_filter=True)
    fe.set_cameras(SC["K"], SC["ext"], SC["ext"], 0.006)
    fe.set_loop_params(odometry_consistency_threshold=10.0)
    st = torch.cuda.current_stream().cuda_stream
    old = synth.loop_record(SELF, 100, "old", 0, g_noise=1e-3)
    ot = torch.frombuffer(bytearray(bytes(old)), dtype=torch.uint8).cuda()
    fe.ingest_own(ot.data_ptr(), st)
    recs = [synth.loop_record(2 + r % 3, 200 + r, "new", 10 + r, g_noise=1e-3) for r in range(64)]
    rt = torch.frombuffer(bytearray(b"".join(bytes(r) for r in recs)), dtype=torch.uint8).cuda()
    res_t = torch.zeros(64 * RS, dtype=torch.uint8, device="cuda")
    edges_t = torch.zeros(64 * EB, dtype=torch.uint8, device="cuda")
    meas_t = torch.zeros(64 * MB, dtype=torch.uint8, device="cuda")
    cnt_t = torch.zeros(1, dtype=torch.int32, device="cuda")
    fe.query_received(rt.data_ptr(), 64, -1, res_t.data_ptr(), st)
    cands = [dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"])] * 64
    fe.compute_loop(rt.data_ptr(), res_t.data_ptr(), cands, edges_t.data_ptr(), st)
    fe.finish(st)
    g = synth.anchor_swarm(5, 60, 600, seed=0, with_orphans=False)
    base = synth.anchor_window_graph(g)
    own = entry_stamps(g, SELF)
    stamps = [(int(entry_stamps(g, 2 + r % 3)[(7 * r + 3) % 40]), int(own[(5 * r + 1) % 40])) for r in range(64)]
    calls = a.warmup + a.reps + 1 + a.host_reps
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    out = {"bench": "loop_measurements", "gpu": smi("name"), "power_limit_w": smi("power.limit"),
           "sm_clock_max_mhz": smi("clocks.max.sm"), "reps": a.reps, "warmup": a.warmup, "host_reps": a.host_reps,
           "round_reps": a.round_reps, "calls": {}, "round": {}}
    identical = True
    loop_count = 0
    for n in (1, 8, 64):
        cap = 600 + 64 * (calls + 2 * (1 + a.round_reps)) + 64
        dev, hop = Backend(g, base, cap), Backend(g, base, cap)
        ts = []
        c_arr, s_arr = fe.loop_candidates(cands[:n]), fe.loop_stamps(stamps[:n])      # built once, as a node would
        for i in range(a.warmup + a.reps):
            e0.record()
            fe.loop_measurements(res_t.data_ptr(), edges_t.data_ptr(), c_arr, s_arr, COV_POS, COV_ANG,
                                 meas_t.data_ptr(), cnt_t.data_ptr(), st)
            dev.a.add_measurements_dev(meas_t.data_ptr(), cnt_t.data_ptr(), n, THRES, st)
            e1.record()
            e1.synchronize()
            if i >= a.warmup:
                ts.append(e0.elapsed_time(e1))
        th = []
        for i in range(1 + a.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rows, loop_count = host_rows(edges_t, res_t, n, cands, stamps, loop_count)
            hop.a.add_measurements(rows)
            if i >= 1:
                th.append((time.perf_counter() - t0) * 1e3)
        out["calls"][n] = {"device_ms_events": float(np.median(ts)), "host_hop_ms_wall": float(np.median(th)),
                           "speedup": float(np.median(th) / np.median(ts)), "rows": int(cnt_t.cpu()[0])}
        # whole rounds; both back-ends start again from the same store
        dev.close()
        hop.close()
        dev, hop = Backend(g, base, cap), Backend(g, base, cap)
        lc_host = int(fe.loop_counts()[0])                    # the host hop numbers its ids from where the device's are
        tr = {0: [], 1: []}
        for r in range(1 + a.round_reps):
            for form in ((0, 1) if r % 2 == 0 else (1, 0)):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                fe.query_received(rt.data_ptr(), n, -1, res_t.data_ptr(), st)
                fe.compute_loop(rt.data_ptr(), res_t.data_ptr(), cands[:n], edges_t.data_ptr(), st)
                if form == 0:
                    fe.loop_measurements(res_t.data_ptr(), edges_t.data_ptr(), cands[:n], stamps[:n], COV_POS, COV_ANG,
                                         meas_t.data_ptr(), cnt_t.data_ptr(), st)
                    dev.a.add_measurements_dev(meas_t.data_ptr(), cnt_t.data_ptr(), n, THRES, st)
                    dev.solve()
                else:
                    rows, lc_host = host_rows(edges_t, res_t, n, cands, stamps, lc_host)
                    hop.a.add_measurements(rows)
                    hop.solve()
                (dev if form == 0 else hop).solver.graph_get_poses()             # synchronises with the solve
                if r >= 1:
                    tr[form].append((time.perf_counter() - t0) * 1e3)
            # the device path's rows use ids from the front-end's counter; the host hop's copy of it follows one round behind
            lc_host = int(fe.loop_counts()[0])
        identical &= bool(np.array_equal(dev.solver.graph_get_poses(), hop.solver.graph_get_poses()))
        identical &= dev.a.status() == lib.OK and dev.a.size() == hop.a.size()
        out["round"][n] = {"device_round_ms_wall": float(np.median(tr[0])), "host_hop_round_ms_wall": float(np.median(tr[1])),
                           "speedup": float(np.median(tr[1]) / np.median(tr[0]))}
        print(json.dumps({"n": n, "calls": out["calls"][n], "round": out["round"][n]}), file=sys.stderr)
        dev.close()
        hop.close()
    out["identical_poses"] = bool(identical)
    fe.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
