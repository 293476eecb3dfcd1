"""GPU: a received round from the query to the measurement rows, with the loop candidates built on the host (today's round)
and on the device.  Prints one JSON line; writes nothing.

Set-up (tests/frontend_harness.py): the loop scene's stereo front-end with loop parameters, one own keyframe ingested with
its meta, and n received records of the same place (every one a hit) with their metas; three such front-ends fed alike.
For n in {1, 8, 64} the three forms alternate, one round each per repetition:
  (A) today's round: inter_drone_loop_count read back (a synchronising call), init flags in numpy, query_received, finish,
      the results copied to the host, the candidates and stamps built in numpy from the host's keyframe table
      (msg_id -> stamp, pose), compute_loop and loop_measurements with the host arrays;
  (B) the device round: init_modes_dev -> query_received_dev -> loop_candidates_dev -> compute_loop_dev ->
      loop_measurements_dev, then one synchronisation;
  (C) (B) captured once into a CUDA graph and replayed.
Each form reports the wall clock of the round (to its end on the host) and the CUDA-event time between its first and last
enqueue on the stream, medians over --reps after --warmup.  Every repetition's rows and counts of (A), (B) and (C) are
compared byte for byte.  The card's name, power limit and maximum SM clock are read in the same run.

    python scripts/bench_loop_round.py [--reps 50] [--warmup 5]
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

from gpu_env import smi  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402
import frontend_harness as fh  # noqa: E402

RS, EB, CB, SB, MB = lib.RESULT_BYTES, lib.EDGE_BYTES, lib.CANDIDATE_BYTES, lib.STAMPS_BYTES, lib.MEASUREMENT_DTYPE.itemsize
SC, SELF = fh.SC, fh.FRONTEND["self_id"]
COV_POS, COV_ANG, INIT_FRAMES = 0.02, 0.005, 50


def meta_bytes(items):
    return bytes(host.KeyframeFrontend.keyframe_metas(items))


class Round:
    """one front-end and the buffers of a round of n received keyframes"""

    def __init__(self, n, st):
        self.n, self.st, s = n, st, st.cuda_stream
        self.fe = fh.loop_frontend()
        self.fe.set_candidate_params(inter_drone_init_frames=INIT_FRAMES)
        own = synth.loop_record(SELF, 100, "old", 0, g_noise=1e-3)
        self.table = {100: (10**12, SC["pose_old"])}              # the host's fisheyeframe_database: msg_id -> stamp, pose
        self.own = [fh.upload([own]), self._dev(meta_bytes([(SELF, 100, 10**12, SC["pose_old"])]))]
        recs = [synth.loop_record(2 + r % 3, 200 + r, "new", 10 + r, g_noise=1e-3) for r in range(n)]
        self.items = [(2 + r % 3, 200 + r, 2 * 10**12 + r, SC["pose_new"]) for r in range(n)]
        self.drones = [it[0] for it in self.items]
        self.rt, self.mt = fh.upload(recs), self._dev(meta_bytes(self.items))
        self.init, self.res = fh.filled(n), fh.filled(n * RS)
        self.cand, self.stamps = fh.filled(n * CB), fh.filled(n * SB)
        self.edges, self.meas = fh.filled(n * EB), fh.filled(n * MB)
        self.cnt = torch.zeros(1, dtype=torch.int32, device="cuda")
        with torch.cuda.stream(st):
            self.fe.ingest_own_meta(self.own[0].data_ptr(), self.own[1].data_ptr(), s)
            self.fe.finish(s)

    @staticmethod
    def _dev(b):
        return torch.frombuffer(bytearray(b), dtype=torch.uint8).cuda()

    def host_round(self):
        """(A)"""
        fe, n, s = self.fe, self.n, self.st.cuda_stream
        _, pairs = fe.loop_counts()
        flags = np.array([pairs[d, SELF] < INIT_FRAMES for d in self.drones], bool)
        fe.query_received(self.rt.data_ptr(), n, -1, self.res.data_ptr(), s, init_mode=flags)
        fe.finish(s)
        raw = self.res.cpu().numpy().tobytes()
        ca, sa = (lib.LoopCandidate * n)(), (lib.LoopStamps * n)()
        for i in range(n):
            r = lib.LoopResult.from_buffer_copy(raw[i * RS:(i + 1) * RS])
            _, _, tq, pq = self.items[i]
            th, ph = self.table.get(r.hit_msg_id, (0, (0, 0, 0, 1, 0, 0, 0))) if r.accepted else (0, (0, 0, 0, 1, 0, 0, 0))
            ca[i].init_mode = int(flags[i])
            ca[i].pose_query[:], ca[i].pose_hit[:] = [float(x) for x in pq], [float(x) for x in ph]
            ca[i].odom_rel[:] = [0, 0, 0, 1, 0, 0, 0]               # received rounds hit own keyframes: no same-drone loop
            sa[i].stamp_query_ns, sa[i].stamp_hit_ns = tq, th
        lib.check(fe._lib.osb_frontend_compute_loop(fe._h, lib.ptr(self.rt.data_ptr()), lib.ptr(self.res.data_ptr()), n, ca,
                                                    lib.ptr(self.edges.data_ptr()), lib.ptr(s)))
        fe.loop_measurements(self.res.data_ptr(), self.edges.data_ptr(), ca, sa, COV_POS, COV_ANG, self.meas.data_ptr(),
                             self.cnt.data_ptr(), s)

    def device_round(self):
        """(B)"""
        fe, n, s = self.fe, self.n, self.st.cuda_stream
        fe.init_modes_dev(self.rt.data_ptr(), n, -1, self.init.data_ptr(), s)
        fe.query_received_dev(self.rt.data_ptr(), n, -1, self.init.data_ptr(), self.res.data_ptr(), s)
        fe.loop_candidates_dev(self.rt.data_ptr(), self.mt.data_ptr(), self.res.data_ptr(), n, self.init.data_ptr(),
                               self.cand.data_ptr(), self.stamps.data_ptr(), s)
        fe.compute_loop_dev(self.rt.data_ptr(), self.res.data_ptr(), n, self.cand.data_ptr(), self.edges.data_ptr(), s)
        fe.loop_measurements_dev(self.res.data_ptr(), self.edges.data_ptr(), n, self.cand.data_ptr(), self.stamps.data_ptr(),
                                 COV_POS, COV_ANG, self.meas.data_ptr(), self.cnt.data_ptr(), s)

    def rows(self):
        k = int(self.cnt.cpu()[0])
        return k, self.meas.cpu().numpy().tobytes()[:k * MB]


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=50)
    ap.add_argument("--warmup", type=int, default=5)
    a = ap.parse_args()
    assert lib.load().osb_device_count() > 0, "needs a CUDA device"
    st = torch.cuda.Stream()
    out = {"bench": "loop_round", "gpu": smi("name"), "power_limit_w": smi("power.limit"),
           "sm_clock_max_mhz": smi("clocks.max.sm"), "reps": a.reps, "warmup": a.warmup, "rounds": {}}
    identical = True
    for n in (1, 8, 64):
        forms = {"A_host": Round(n, st), "B_device": Round(n, st), "C_graph": Round(n, st)}
        c = forms["C_graph"]
        with torch.cuda.stream(st):
            c.device_round()                                     # acquires every buffer before the capture
            forms["A_host"].host_round()
            forms["B_device"].device_round()
            st.synchronize()
            graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(graph, stream=st):
                c.device_round()
        run = {"A_host": forms["A_host"].host_round, "B_device": forms["B_device"].device_round, "C_graph": graph.replay}
        wall = {k: [] for k in run}
        ev = {k: [] for k in run}
        accepted = None
        for i in range(a.warmup + a.reps):
            order = list(run) if i % 2 == 0 else list(reversed(run))
            got = {}
            for k in order:
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                with torch.cuda.stream(st):
                    st.synchronize()
                    t0 = time.perf_counter()
                    e0.record(st)
                    run[k]()
                    e1.record(st)
                    st.synchronize()
                    t1 = time.perf_counter()
                if i >= a.warmup:
                    wall[k].append((t1 - t0) * 1e3)
                    ev[k].append(e0.elapsed_time(e1))
                got[k] = forms[k].rows()
            identical &= got["A_host"] == got["B_device"] == got["C_graph"]
            accepted = got["A_host"][0]
        out["rounds"][str(n)] = {"accepted_per_round": accepted,
                                 **{k: {"wall_ms_median": float(np.median(wall[k])), "event_ms_median": float(np.median(ev[k]))}
                                    for k in run}}
        for f in forms.values():
            f.fe.close()
    out["rows_identical"] = bool(identical)
    print(json.dumps(out))
    assert identical, "the device round's rows differ from the host round's"


if __name__ == "__main__":
    main()
