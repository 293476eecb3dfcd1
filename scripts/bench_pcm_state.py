"""GPU: the outlier rejection before a solve, with the PCM state resident (osb_pcm_state_reject) against the per-pair
recompute (osb_pcm_dev on every pair's whole list), alternated in one process.  Prints one JSON line; writes nothing.

Set-up: five drones, redundant mode, so 15 drone pairs (5 of them intra-drone).  Every pair holds `size` loop edges
(synth.pcm_edges, 40 % outliers); then each round adds 4 new edges per pair and re-submits every earlier edge, as
find_available_loops_detections does.  Sizes 250, 1 000, 2 000 and 4 000 edges per pair.

Per size and round, alternating which goes first:
  * state: the wall time of one blocking osb_pcm_state_reject call (host clock; the edges are packed beforehand);
  * recompute: osb_pcm_dev once per pair on its full list, already resident on the device (CUDA events around the 15
    calls on one stream) -- what an adapter without the state does before every solve.
Medians over --reps rounds after --warmup.  At the end every pair's clique of the state is checked against the last
recompute's.  The card's name and power limit are read in the same run.

    python scripts/bench_pcm_state.py [--reps 10] [--warmup 2]
"""
import argparse
import ctypes as C
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gpu_env import smi  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402

THRES, POS, ANG = 15.0, 1e-4, 1e-5
NEW_PER_ROUND = 4
SIZES = (250, 1000, 2000, 4000)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    L = lib.load()
    assert L.osb_device_count() > 0, "needs a CUDA device"
    rounds = args.warmup + args.reps
    pairs = [(a, b) for a in range(1, 6) for b in range(1, 6) if a <= b]
    total = max(SIZES) + NEW_PER_ROUND * rounds
    assert total <= 4096, "too many rounds for the largest size"
    per_pair = [host.loop_edges(synth.pcm_edges(total, 0.4, 100 + p, id_a=a, id_b=b)) for p, (a, b) in enumerate(pairs)]
    ids = [(1 << 32) + (p << 16) + np.arange(total, dtype=np.int64) for p in range(len(pairs))]
    stream = torch.cuda.Stream()
    st_ptr = C.c_void_p(stream.cuda_stream)
    dev_edges = [torch.from_numpy(e.view(np.uint8).copy()).cuda() for e in per_pair]
    dev_out = [torch.zeros(total + 1, dtype=torch.int32, device="cuda") for _ in pairs]
    out = {"gpu": smi("name"), "power_limit_w": smi("power.limit"), "pairs": len(pairs), "new_per_pair": NEW_PER_ROUND,
           "reps": args.reps, "warmup": args.warmup, "sizes": []}
    for size in SIZES:
        # submission order: every pair's first `size` edges, then round by round 4 new edges per pair
        order = [(p, k) for p in range(len(pairs)) for k in range(size)]
        for r in range(rounds):
            order += [(p, size + NEW_PER_ROUND * r + k) for p in range(len(pairs)) for k in range(NEW_PER_ROUND)]
        sub_edges = np.stack([per_pair[p][k] for p, k in order])
        sub_ids = np.array([ids[p][k] for p, k in order], np.int64)
        state = host.PcmState(1, True, THRES, POS, ANG, max_pairs=len(pairs), pair_capacity=4096)
        n0 = len(pairs) * size
        state.reject(sub_edges[:n0], sub_ids[:n0])

        def recompute(n_each):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record(stream)
            for p in range(len(pairs)):
                lib.check(L.osb_pcm_dev(C.c_void_p(dev_edges[p].data_ptr()), n_each, THRES, POS, ANG,
                                        C.c_void_p(dev_out[p].data_ptr()), C.c_void_p(dev_out[p].data_ptr() + 4 * n_each),
                                        None, None, st_ptr))
            e1.record(stream)
            e1.synchronize()
            return e0.elapsed_time(e1)

        t_state, t_rec = [], []
        for r in range(rounds):
            n_sub = n0 + len(pairs) * NEW_PER_ROUND * (r + 1)
            n_each = size + NEW_PER_ROUND * (r + 1)
            for form in ((0, 1) if r % 2 == 0 else (1, 0)):
                if form == 0:
                    t0 = time.perf_counter()
                    state.reject(sub_edges[:n_sub], sub_ids[:n_sub])
                    ms = (time.perf_counter() - t0) * 1e3
                    if r >= args.warmup:
                        t_state.append(ms)
                else:
                    ms = recompute(n_each)
                    if r >= args.warmup:
                        t_rec.append(ms)
        same = True
        for p, (a, b) in enumerate(pairs):
            n, cs = C.c_int32(0), C.c_int32(0)
            clique = np.zeros(total, np.int32)
            lib.check(L.osb_pcm_state_pair(state._h, a, b, C.byref(n), None, None, lib.ptr(clique), C.byref(cs)))
            ref = dev_out[p].cpu().numpy()
            same &= n.value == n_each and np.array_equal(clique[:cs.value], ref[:ref[n_each]])
        state.close()
        out["sizes"].append({"edges_per_pair": size, "state_reject_ms_wall": float(np.median(t_state)),
                             "state_reject_ms_min": float(np.min(t_state)),
                             "recompute_ms_events": float(np.median(t_rec)), "recompute_ms_min": float(np.min(t_rec)),
                             "pair_checks_recompute": int(len(pairs) * n_each * (n_each - 1) // 2),
                             "speedup": float(np.median(t_rec) / np.median(t_state)), "cliques_identical": bool(same)})
        print(json.dumps(out["sizes"][-1]), file=sys.stderr)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
