"""GPU: the keyframe database's fp32 and fp16 row storage (OSB_DB_STORAGE_FP32 / _FP16) side by side, alternated in one
process.  Prints one JSON line; writes nothing.

Scan: osb_db_search_dev with k = 6 at nq = 1 and 8 on stores of 10 000 / 50 000 / 200 000 unit-norm Gaussian rows of dim
4096 (the same rows in both storages).  Per case the median device time over --reps searches after --warmup (CUDA events on
one stream, the two storages alternating which goes first), and the algorithmic bytes (rows x 4096 x 4 or x 2) over that
time as a fraction of the H100 SXM's 3.35 TB/s.  An fp16 store of 10 000 rows (82 MB) is already larger than the 50 MB L2,
so no store here is served from cache between repeats.

Front-end: osb_frontend_query of an own keyframe (both stores scanned) and osb_frontend_query_received of a 7-record round
(the local store scanned once for all 7) on handles whose two stores hold 50 016 rows from db_load (no local descriptors,
so the matcher finds nothing: the time is the scans and the acceptance rule), one handle per storage, alternated.

Agreement on C3-like data (SURVEY.md 8d: unit-norm Gaussian rows, queries = rows + noise of norm 0.1, renormalised):
the share of 2000 queries against 50 000 rows whose top-6 ids, and whose accepted hit (the best row if its score is above
the threshold, else none) at thresholds 0.3 and 0.6, are the same in the two storages.

The card's name, power limit and SM clock (sampled by nvidia-smi during the timed loops) are read in the same run.

    python scripts/bench_db_storage.py [--reps 200] [--warmup 20]
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

DIM, K, QDIR, N_DIRS = 4096, 6, 1, 4
HBM_TBS = 3.35
FE_ROWS = 50_016
RB, RS = lib.RECORD_BYTES, lib.RESULT_BYTES
STORAGES = ("fp32", "fp16")


def unit_rows(n, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(n, DIM, generator=g, device="cuda")
    return x / x.norm(dim=1, keepdim=True)


def alternated(fns, reps, warmup):
    """median device time (ms) of each of the callables, called alternately, the first one rotating"""
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(len(fns) + 1)]
    times = [[] for _ in fns]
    for i in range(warmup + reps):
        order = [(i + j) % len(fns) for j in range(len(fns))]
        ev[0].record()
        for j, f in enumerate(order):
            fns[f]()
            ev[j + 1].record()
        ev[-1].synchronize()
        if i >= warmup:
            for j, f in enumerate(order):
                times[f].append(ev[j].elapsed_time(ev[j + 1]))
    return [float(np.median(t)) for t in times]


def scan_cases(reps, warmup, stream):
    cases = []
    for n in (10_000, 50_000, 200_000):
        rows = unit_rows(n, n)
        idx = {s: host.IndexFlatIP(DIM, n, storage=s) for s in STORAGES}
        for s in STORAGES:
            idx[s].add_dev(rows.data_ptr(), n, stream)
        for nq in (1, 8):
            q = unit_rows(nq, 7 + nq)
            out = {s: (torch.empty(nq * K, device="cuda"), torch.empty(nq * K, dtype=torch.int64, device="cuda"))
                   for s in STORAGES}
            fns = [lambda s=s: idx[s].search_dev(q.data_ptr(), nq, K, out[s][0].data_ptr(), out[s][1].data_ptr(), stream)
                   for s in STORAGES]
            ms = alternated(fns, reps, warmup)
            case = {"rows": n, "nq": nq, "k": K}
            for s, t in zip(STORAGES, ms):
                b = n * DIM * (4 if s == "fp32" else 2)
                case[f"{s}_ms"] = round(t, 4)
                case[f"{s}_hbm_fraction"] = round(b / (t * 1e-3) / (HBM_TBS * 1e12), 3)
            case["speedup"] = round(ms[0] / ms[1], 3)
            cases.append(case)
            print(json.dumps(case), file=sys.stderr, flush=True)
        for s in STORAGES:
            idx[s].close()
        del rows
    return cases


def agreement(stream):
    n, nq = 50_000, 2000
    rows = unit_rows(n, 1)
    src = torch.randint(0, n, (nq,), generator=torch.Generator(device="cuda").manual_seed(2), device="cuda")
    noise = torch.randn(nq, DIM, generator=torch.Generator(device="cuda").manual_seed(3), device="cuda")
    q = rows[src] + noise * (0.1 / DIM ** 0.5)
    q = (q / q.norm(dim=1, keepdim=True)).contiguous()
    res = {}
    for s in STORAGES:
        idx = host.IndexFlatIP(DIM, n, storage=s)
        idx.add_dev(rows.data_ptr(), n, stream)
        D = torch.empty(nq * K, device="cuda")
        I = torch.empty(nq * K, dtype=torch.int64, device="cuda")
        idx.search_dev(q.data_ptr(), nq, K, D.data_ptr(), I.data_ptr(), stream)
        torch.cuda.synchronize()
        res[s] = (D.view(nq, K).cpu().numpy(), I.view(nq, K).cpu().numpy())
        idx.close()
    (D32, I32), (D16, I16) = res["fp32"], res["fp16"]
    out = {"rows": n, "queries": nq, "noise_norm": 0.1, "top6_ids_same": float((I32 == I16).all(1).mean()),
           "max_score_change": float(np.abs(D32[:, 0] - D16[:, 0]).max())}
    for th in (0.3, 0.6):
        h32 = np.where(D32[:, 0] > th, I32[:, 0], -1)
        h16 = np.where(D16[:, 0] > th, I16[:, 0], -1)
        out[f"hit_same_thres_{th}"] = float((h32 == h16).mean())
    return out


def record(drone, g_row, seed):
    rec = lib.KeyframeRecord()
    rec.drone_id, rec.msg_id, rec.n_dirs = drone, 1000 + seed, N_DIRS
    rec.n_kpts[QDIR] = 150
    np.ctypeslib.as_array(rec.global_desc[QDIR])[:] = g_row
    np.ctypeslib.as_array(rec.local_desc[QDIR])[:150] = synth.local_descriptors(150, seed)
    return bytes(rec)


def frontend_cases(reps, warmup, stream):
    g = synth.descriptor_db(FE_ROWS, DIM, 11)
    fes = {}
    for s in STORAGES:
        fe = host.KeyframeFrontend(*synth.frontend_weights(), width=640, height=480, n_dirs=N_DIRS, max_num=200, self_id=1,
                                   db_capacity=FE_ROWS, match_index_dist=5)
        fe.set_db_storage(s)
        fe.db_load(g)
        fe.db_load(g, remote=True)
        fes[s] = fe
    qs = synth.noisy_queries(g, np.arange(8) * 5000, sigma=0.5)
    own = torch.frombuffer(bytearray(record(1, qs[0], 0)), dtype=torch.uint8).cuda()
    rnd = torch.frombuffer(bytearray(b"".join(record(2 + r, qs[1 + r], 1 + r) for r in range(7))), dtype=torch.uint8).cuda()
    out = {s: torch.zeros(7 * RS, dtype=torch.uint8, device="cuda") for s in STORAGES}
    cases = []
    forms = {"query": lambda s: fes[s].query(own.data_ptr(), out[s].data_ptr(), stream),
             "query_received_7": lambda s: fes[s].query_received(rnd.data_ptr(), 7, -1, out[s].data_ptr(), stream)}
    for name, f in forms.items():
        ms = alternated([lambda s=s: f(s) for s in STORAGES], reps, warmup)
        for s in STORAGES:
            fes[s].finish(stream)
        hits = {s: [lib.LoopResult.from_buffer_copy(out[s][r * RS:(r + 1) * RS].cpu().numpy().tobytes()).hit_id
                    for r in range(1 if name == "query" else 7)] for s in STORAGES}
        case = {"form": name, "rows_per_store": FE_ROWS, "fp32_ms": round(ms[0], 4), "fp16_ms": round(ms[1], 4),
                "speedup": round(ms[0] / ms[1], 3), "same_hits": hits["fp32"] == hits["fp16"]}
        cases.append(case)
        print(json.dumps(case), file=sys.stderr, flush=True)
    for fe in fes.values():
        fe.close()
    return cases


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--reps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    args = p.parse_args()
    stream = torch.cuda.current_stream().cuda_stream
    clocks = ClockSampler()
    with clocks:
        scans = scan_cases(args.reps, args.warmup, stream)
        agree = agreement(stream)
        fe = frontend_cases(args.reps, args.warmup, stream)
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"),
           "sm_clock_mhz_median": float(np.median(clocks.samples)) if clocks.samples else None,
           "reps": args.reps, "warmup": args.warmup, "scan": scans, "agreement": agree, "frontend": fe}
    print(json.dumps(out))


if __name__ == "__main__":
    main()
