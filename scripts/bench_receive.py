"""GPU: osb_frontend_receive_dev -- a received round's records as LoopNet delivers them.  Prints one JSON line; writes nothing.

Set-up (tests/frontend_harness.py): the loop scene's stereo front-end with loop parameters and one own keyframe in its local
store; the round's records are loop-scene keyframes of drones 2..4 (every fifth a miss), each with its meta.
  * per call, n in {1, 8, 64}: --calls receive_dev calls captured into one CUDA graph, against the same number of
    device-to-device cudaMemcpyAsync of the same n records (torch's copy_) in another; CUDA-event time of a replay over
    --calls, the two graphs alternating --reps times after --warmup.  The calls rotate over 4 source / destination rounds
    (150 MB), so their bytes come from HBM rather than L2.  Achieved GB/s counts the bytes read plus the bytes written
    (2 x n x 292,784).
  * per round, n = 8: two front-ends fed alike, one with the call and one without, alternating: receive (or not) ->
    init_modes_dev -> query_received_dev -> ingest_meta -> loop_candidates_dev -> compute_loop_dev -> loop_measurements_dev
    -> osb_anchor_add_measurements_dev, CUDA-event time from the first enqueue to the last, medians over --rounds.
  * information only: the remote-store rows the first round adds and the inter-drone loops it accepts, with and without
    the call.
The card's name and power limit are read in the same run.

    python scripts/bench_receive.py [--reps 20] [--calls 200] [--rounds 30] [--warmup 3]
"""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
sys.path.insert(0, os.path.join(ROOT, "tests"))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gpu_env import smi  # noqa: E402
from omniswarm_b200 import lib, synth  # noqa: E402
import frontend_harness as fh  # noqa: E402
import loop_candidates_ref as lc  # noqa: E402
from backend_harness import make_anchor  # noqa: E402

RB, RS, EB, CB, SB = lib.RECORD_BYTES, lib.RESULT_BYTES, lib.EDGE_BYTES, lib.CANDIDATE_BYTES, lib.STAMPS_BYTES
MB = lib.MEASUREMENT_DTYPE.itemsize
SC = fh.SC
POOL = 4
PRM = dict(inter_drone_init_frames=2, pos_covariance_per_meter=0.01, yaw_covariance_per_meter=0.003, loop_cov_pos=0.013,
           loop_cov_ang=2.5e-4)


def entry_stamp(g, drone, frame):
    stamps, first, e = g["window"]
    for f in list(range(frame, len(stamps))) + list(range(frame - 1, -1, -1)):
        row = e[first[f]:first[f + 1]]
        row = row[(row["drone_id"] == drone) & (row["vo_available"] == 1)]
        if len(row):
            return int(row["stamp"][0])
    raise AssertionError("no entry")


def round_records(g, n, msg0):
    recs, items = [], []
    for r in range(n):
        d = 2 + r % 3
        gd = synth.loop_noisy_g(10 + r) if r % 5 != 4 else synth.descriptor_db(4, 4096, 300 + r)
        recs.append(synth.loop_record(d, msg0 + r, "new", seed=20 + r, g=gd))
        items.append((d, msg0 + r, entry_stamp(g, d, 4 + (3 * r) % 20), SC["pose_new"]))
    return fh.upload(recs), torch.frombuffer(bytearray(lc.metas(items).tobytes()), dtype=torch.uint8).cuda()


def timed(st, fn, k):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record(st)
    for _ in range(k):
        fn()
    b.record(st)
    b.synchronize()
    return a.elapsed_time(b) / k


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20)
    ap.add_argument("--calls", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=30)
    ap.add_argument("--warmup", type=int, default=3)
    a = ap.parse_args()
    assert torch.cuda.is_available(), "bench_receive.py measures on the GPU"
    st = torch.cuda.Stream()
    s = st.cuda_stream
    g = synth.anchor_swarm(5, 30, 300, seed=9, with_orphans=False)
    old = synth.loop_record(1, 100, "old")
    ot = fh.upload([old])
    omt = torch.frombuffer(bytearray(lc.metas([(1, 100, entry_stamp(g, 1, 2), SC["pose_old"])]).tobytes()),
                           dtype=torch.uint8).cuda()
    out = {"gpu": smi("name,power.limit"), "record_bytes": RB, "per_call": {}, "per_round": {}}

    # ---- per call ------------------------------------------------------------------------------------------------
    fe = fh.loop_frontend()
    with torch.cuda.stream(st):
        fe.ingest_own(ot.data_ptr(), s)
    fe.finish(s)
    # POOL source / destination rounds in rotation (4 x 2 x 18.7 MB), so that a call's bytes do not sit in the 50 MB L2
    src = [round_records(g, 64, 300 + 100 * i)[0] for i in range(POOL)]
    dst = [fh.filled(64 * RB) for _ in range(POOL)]
    for n in (1, 8, 64):
        # a.calls calls (or copies) captured into one CUDA graph each, so the events time the device and not the enqueue
        graphs = {}
        for kind in ("call", "copy"):
            gr = torch.cuda.CUDAGraph()
            with torch.cuda.graph(gr, stream=st):
                for i in range(a.calls):
                    x, y = src[i % POOL], dst[i % POOL]
                    if kind == "call":
                        fe.receive_dev(x.data_ptr(), n, -1, y.data_ptr(), s)
                    else:
                        y[:n * RB].copy_(x[:n * RB])
            graphs[kind] = gr
        with torch.cuda.stream(st):
            for _ in range(a.warmup):
                timed(st, graphs["call"].replay, 1); timed(st, graphs["copy"].replay, 1)
            tc, tm = [], []
            for _ in range(a.reps):
                tc.append(timed(st, graphs["call"].replay, 1) / a.calls)
                tm.append(timed(st, graphs["copy"].replay, 1) / a.calls)
        us_c, us_m = 1e3 * float(np.median(tc)), 1e3 * float(np.median(tm))
        nbytes = 2 * n * RB
        out["per_call"][n] = dict(receive_us=round(us_c, 2), d2d_copy_us=round(us_m, 2),
                                  receive_gbps=round(nbytes / us_c / 1e3, 1), d2d_copy_gbps=round(nbytes / us_m / 1e3, 1),
                                  receive_us_spread=[round(1e3 * float(min(tc)), 2), round(1e3 * float(max(tc)), 2)])
    fe.close()

    # ---- per round -----------------------------------------------------------------------------------------------
    n = 8
    fes, anchors = [], []
    for _ in range(2):
        f = fh.loop_frontend(db_capacity=4096)
        f.set_candidate_params(**PRM)
        fes.append(f)
        an = make_anchor(g, max_meas=65536)
        for d, (ts, p) in g["trajs"].items():
            an.push_odometry(d, ts, p)
        an.set_window(*g["window"])
        anchors.append(an)
    with torch.cuda.stream(st):
        for f in fes:
            f.ingest_own_meta(ot.data_ptr(), omt.data_ptr(), s)
    rounds = [round_records(g, n, 1000 + 10 * k) for k in range(a.rounds + a.warmup)]
    bufs = dict(out=fh.filled(n * RB), init=fh.filled(n), res=fh.filled(n * RS), cand=fh.filled(n * CB),
                stamps=fh.filled(n * SB), edges=fh.filled(n * EB), meas=fh.filled(n * MB),
                cnt=torch.zeros(1, dtype=torch.int32, device="cuda"))

    def one_round(f, an, k, deliver):
        rt, mt = rounds[k][0].data_ptr(), rounds[k][1].data_ptr()
        if deliver:
            f.receive_dev(rt, n, -1, bufs["out"].data_ptr(), s)
            rt = bufs["out"].data_ptr()
        f.init_modes_dev(rt, n, -1, bufs["init"].data_ptr(), s)
        f.query_received_dev(rt, n, -1, bufs["init"].data_ptr(), bufs["res"].data_ptr(), s)
        f.ingest_meta(rt, mt, n, -1, s)
        f.loop_candidates_dev(rt, mt, bufs["res"].data_ptr(), n, bufs["init"].data_ptr(), bufs["cand"].data_ptr(),
                              bufs["stamps"].data_ptr(), s)
        f.compute_loop_dev(rt, bufs["res"].data_ptr(), n, bufs["cand"].data_ptr(), bufs["edges"].data_ptr(), s)
        f.loop_measurements_dev(bufs["res"].data_ptr(), bufs["edges"].data_ptr(), n, bufs["cand"].data_ptr(),
                                bufs["stamps"].data_ptr(), 0.02, 0.005, bufs["meas"].data_ptr(), bufs["cnt"].data_ptr(), s)
        an.add_measurements_dev(bufs["meas"].data_ptr(), bufs["cnt"].data_ptr(), n, 2.0, s)

    t = {True: [], False: []}
    info = {}
    with torch.cuda.stream(st):
        for k in range(a.rounds + a.warmup):
            for deliver, f, an in ((True, fes[0], anchors[0]), (False, fes[1], anchors[1])):
                r0 = f.db_size(remote=True)
                ms = timed(st, lambda: one_round(f, an, k, deliver), 1)
                f.finish(s)
                if k == 0:
                    edges = [lib.LoopEdgeResult.from_buffer_copy(b) for b in fh.edges(bufs["edges"], n)]
                    info["with_call" if deliver else "without_call"] = dict(
                        remote_rows_added=f.db_size(remote=True) - r0,
                        loops_accepted=sum(e.status == lib.LOOP_ACCEPTED for e in edges))
                if k >= a.warmup:
                    t[deliver].append(ms)
    st.synchronize()
    out["per_round"] = dict(n=n, with_call_ms=round(float(np.median(t[True])), 4),
                            without_call_ms=round(float(np.median(t[False])), 4), first_round=info)
    for h in fes + anchors:
        h.close()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
