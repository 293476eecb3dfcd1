"""GPU: a round's keyframes received from other drones, queried against the own-keyframe store -- W-1 osb_frontend_query
calls against one osb_frontend_query_received call on the same records, alternated in one process.  Prints one JSON line;
writes nothing.

Set-up per case: a 4-direction 640x480 front-end (max_num 200) whose local store holds 4 own keyframes (extract +
ingest_own) and --rows loaded rows (db_load + db_set_geometry); W-1 foreign records, re-labelled extracts alternating
between noisy revisits of the own keyframes (they hit, so the matcher and, with the geometric filter, the RANSAC run) and
new places.  Cases: rows in {10 000, 50 000} x W-1 in {1, 3, 7} x geometric filter off / on.

Per case, the median over --reps repetitions after --warmup (CUDA events on one stream, the two forms alternating which goes
first) of the device time of one round in each form, a check that the two wrote byte-identical results, and the scan alone:
osb_db_search_dev with nq = W-1, k = 6 on a store of the same rows (the search the batched call makes), reported as the
store's bytes over the scan time, as a fraction of the H100 SXM's 3.35 TB/s.  The card's name, power limit and SM clock
(sampled by nvidia-smi during the timed loops) are read in the same run.

    python scripts/bench_received_query.py [--reps 200] [--warmup 20]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gpu_env import ClockSampler, smi  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402

W, H, N_DIRS, MAX_NUM, QDIR = 640, 480, 4, 200, 1
N_OWN = 4
HBM_TBS = 3.35
RB, RS = lib.RECORD_BYTES, lib.RESULT_BYTES


def images(seed, noisy=False):
    rng = np.random.default_rng(seed + 77)
    out = []
    for k in (0, 5):
        a = np.stack([synth.image(seed * 10 + d + k, H, W) for d in range(N_DIRS)])
        if noisy:       # the same place seen again: two pixels to the side, a little pixel noise
            a = np.clip(np.roll(a, 2, axis=2).astype(np.int16) + rng.integers(-3, 4, a.shape), 0, 255).astype(np.uint8)
        out.append(np.ascontiguousarray(a))
    return out


def make_frontend(rows, geometric_filter):
    return host.KeyframeFrontend(*synth.frontend_weights(), width=W, height=H, n_dirs=N_DIRS, max_num=MAX_NUM, self_id=1,
                                 db_capacity=rows + 64, match_index_dist=5, geometric_filter=bool(geometric_filter),
                                 ransac_seed=1)


def build_store(fe, rows, g, stream):
    rec_t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    for i in range(N_OWN):
        up, down = images(i)
        fe.extract(up.ctypes.data, down.ctypes.data, 100 + i, rec_t.data_ptr(), stream)
        fe.ingest_own(rec_t.data_ptr(), stream)
        fe.finish(stream)
    first = fe.db_size(False)
    fe.db_load(g[:rows])
    kp = np.random.default_rng(3).uniform(0, 600, (rows, MAX_NUM, 2)).astype(np.float32)
    fe.db_set_geometry(first, kp, np.zeros((rows, MAX_NUM), np.int32))


def foreign_records(fe, n, stream):
    """n records of drones 2.. : even positions noisy revisits of own keyframes, odd ones new places"""
    rec_t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    raw = []
    for r in range(n):
        up, down = images(r // 2 % N_OWN, noisy=True) if r % 2 == 0 else images(50 + r)
        fe.extract(up.ctypes.data, down.ctypes.data, 1000 + r, rec_t.data_ptr(), stream)
        fe.finish(stream)
        b = bytearray(rec_t.cpu().numpy().tobytes())
        lib.KeyframeRecord.from_buffer(b).drone_id = 2 + r
        raw.append(bytes(b))
    return torch.frombuffer(bytearray(b"".join(raw)), dtype=torch.uint8).cuda()


def time_case(fe, recs, n, reps, warmup, stream):
    single = torch.full((n * RS,), 0x5A, dtype=torch.uint8, device="cuda")
    batch = single.clone()
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(3)]
    t_single, t_batch = [], []

    def run_single():
        for r in range(n):
            fe.query(recs.data_ptr() + r * RB, single.data_ptr() + r * RS, stream)

    def run_batch():
        fe.query_received(recs.data_ptr(), n, -1, batch.data_ptr(), stream)

    for i in range(warmup + reps):
        first, second = (run_single, run_batch) if i % 2 == 0 else (run_batch, run_single)
        ev[0].record()
        first()
        ev[1].record()
        second()
        ev[2].record()
        ev[2].synchronize()
        if i >= warmup:
            a, b = ev[0].elapsed_time(ev[1]), ev[1].elapsed_time(ev[2])
            (t_single if first is run_single else t_batch).append(a)
            (t_batch if first is run_single else t_single).append(b)
    fe.finish(stream)
    same = bool(torch.equal(single, batch))
    res = [lib.LoopResult.from_buffer_copy(batch[r * RS:(r + 1) * RS].cpu().numpy().tobytes()) for r in range(n)]
    return float(np.median(t_single)), float(np.median(t_batch)), same, res


def time_scan(idx, q, n, reps, warmup, stream):
    scores = torch.zeros(n * 6, dtype=torch.float32, device="cuda")
    ids = torch.zeros(n * 6, dtype=torch.int64, device="cuda")
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    t = []
    for i in range(warmup + reps):
        ev[0].record()
        idx.search_dev(q.data_ptr(), n, 6, scores.data_ptr(), ids.data_ptr(), stream)
        ev[1].record()
        ev[1].synchronize()
        if i >= warmup:
            t.append(ev[0].elapsed_time(ev[1]))
    return float(np.median(t))


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    args = p.parse_args()
    stream = torch.cuda.current_stream().cuda_stream
    g = synth.descriptor_db(50_000, 4096, 11)
    cases, clocks = [], ClockSampler()
    with clocks:
        for rows in (10_000, 50_000):
            idx = host.IndexFlatIP(4096, capacity=rows + N_OWN * N_DIRS)
            idx.add(g[:rows + N_OWN * N_DIRS])
            for gf in (0, 1):
                fe = make_frontend(rows + N_OWN * N_DIRS, gf)
                build_store(fe, rows, g, stream)
                store_rows = fe.db_size(False)
                for n in (1, 3, 7):
                    recs = foreign_records(fe, n, stream)
                    ms_single, ms_batch, same, res = time_case(fe, recs, n, args.reps, args.warmup, stream)
                    q = torch.from_numpy(g[:n] * np.float32(0.5)).cuda()
                    ms_scan = time_scan(idx, q, n, args.reps, args.warmup, stream) if gf == 0 else None
                    case = {"rows": store_rows, "received": n, "geometric_filter": gf,
                            "ms_per_round_single_queries": round(ms_single, 4), "ms_per_round_batched": round(ms_batch, 4),
                            "byte_identical": same, "hits": sum(r.accepted for r in res),
                            "matched_pairs": sum(1 for r in res for s in range(N_DIRS) if r.n_matches[s] > 0),
                            "geo_valid_pairs": sum(sum(r.geo_valid) for r in res) if gf else 0}
                    if ms_scan is not None:
                        case["scan_ms"] = round(ms_scan, 4)
                        case["scan_hbm_fraction"] = round(idx.ntotal * 4096 * 4 / (ms_scan * 1e-3) / (HBM_TBS * 1e12), 3)
                    cases.append(case)
                    print(json.dumps(case), file=sys.stderr, flush=True)
                fe.close()
            idx.close()
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"),
           "sm_clock_mhz_median": float(np.median(clocks.samples)) if clocks.samples else None,
           "reps": args.reps, "warmup": args.warmup, "cases": cases}
    print(json.dumps(out))
    if not all(c["byte_identical"] for c in cases):
        sys.exit(1)


if __name__ == "__main__":
    main()
