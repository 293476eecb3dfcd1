"""GPU: the split-fp16 (default) and plain-fp16 precisions of the tensor-core networks, alternated in one process on the
same seeded inputs.  Prints one JSON line; writes nothing.

Per precision, the median over --rounds of
  * layer_ms: every SuperPoint layer of an 8-image 640x480 batch (CUDA events between the launches, osb_superpoint_layer_ms),
    and the executed tensor-core rate of each convolution: MMAs per K step (3 split, 1 fp16) x 2 x pixels x N x K over
    the layer time, with N the layer's padded width (64 / 80 / 128 per item) and K = Cin x taps -- conv1a runs in fp32
    FFMA and has no rate;
  * netvlad_ms: one 4-image 640x480 NetVLAD batch (host call with its 1.2 MB upload, synchronised);
  * keyframes/s of extract_dev + ingest_own + query on a 4-direction 640x480 front-end holding a 10 000-row database
    (CUDA events around --steps keyframes, as scripts/bench_depth_frontend.py);
and the card's name, power limit and SM clock, sampled by nvidia-smi while the keyframe windows run.

    python scripts/bench_precision.py [--steps 100] [--warmup 10] [--rounds 3]
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

W, H, N_DIRS, MAX_NUM, SP_BATCH, NV_BATCH = 640, 480, 4, 200, 8, 4
DB_ROWS = 10_000
POOL = 4
MODES = ("split_fp16", "fp16")
MMAS_PER_KSTEP = {"split_fp16": 3, "fp16": 1}
# SuperPoint layers after conv1a: (cin, n_pad, taps, resolution divisor)
SP_CONVS = {"conv1b+pool": (64, 64, 9, 1), "conv2a": (64, 64, 9, 2), "conv2b+pool": (64, 64, 9, 2),
            "conv3a": (64, 128, 9, 4), "conv3b+pool": (128, 128, 9, 4), "conv4a": (128, 128, 9, 8),
            "conv4b": (128, 128, 9, 8), "convPa": (128, 256, 9, 8), "convPb": (256, 80, 1, 8), "convDa": (128, 256, 9, 8),
            "convDb": (256, 256, 1, 8)}


def mma_tflops(layer, ms, mode):
    cin, n_pad, taps, div = SP_CONVS[layer]
    pixels = SP_BATCH * (H // div) * (W // div)
    return MMAS_PER_KSTEP[mode] * 2.0 * pixels * n_pad * cin * taps / (ms * 1e-3) / 1e12


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=100, help="keyframes per timed window")
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--layer-reps", type=int, default=5, help="profiled SuperPoint batches per round and precision")
    args = ap.parse_args()
    assert lib.load().osb_device_count() > 0, "needs a CUDA device"
    name, power = smi("name"), smi("power.limit")
    st = torch.cuda.current_stream().cuda_stream
    spw, comp, mean, nvw = synth.frontend_weights()

    sp = host.SuperPoint(spw, comp, mean, W, H, 0.015, MAX_NUM, max_batch=SP_BATCH)
    nv = host.NetVLAD(nvw, W, H, max_batch=NV_BATCH)
    sp_imgs = np.stack([synth.image(300 + i, H, W, zero_bottom_quarter=bool(i & 1)) for i in range(SP_BATCH)])
    nv_imgs = sp_imgs[:NV_BATCH]
    per_round = N_DIRS * (args.warmup + args.steps)
    fe = host.KeyframeFrontend(spw, comp, mean, nvw, width=W, height=H, n_dirs=N_DIRS, max_num=MAX_NUM, sp_thres=0.015,
                               self_id=0, db_capacity=DB_ROWS + 2 * args.rounds * per_round + 64, match_index_dist=5)
    for s in range(0, DB_ROWS, 2000):
        fe.db_load(synth.descriptor_db(2000, 4096, 50 + s), np.random.default_rng(s).standard_normal(
            (2000, MAX_NUM, 64)).astype(np.float32), np.full(2000, MAX_NUM, np.int32))
    frames = [torch.from_numpy(np.stack([synth.image(500 + 10 * j + d, H, W) for d in range(2 * N_DIRS)])).cuda()
              for j in range(POOL)]
    half = N_DIRS * H * W
    rec = torch.zeros(lib.RECORD_BYTES, dtype=torch.uint8, device="cuda")
    res = torch.zeros(lib.RESULT_BYTES, dtype=torch.uint8, device="cuda")

    def step(i):
        f = frames[i % POOL]
        fe.extract(f.data_ptr(), f.data_ptr() + half, i, rec.data_ptr(), st, device_images=True)
        fe.ingest_own(rec.data_ptr(), st)
        fe.query(rec.data_ptr(), res.data_ptr(), st)

    out = {m: {"layer_ms": [], "netvlad_ms": [], "kf_per_s": []} for m in MODES}
    clocks = ClockSampler()
    i = 0
    for r in range(args.rounds):
        for mode in MODES:
            sp.set_precision(mode); nv.set_precision(mode); fe.set_precision(mode)
            for _ in range(args.layer_reps):
                out[mode]["layer_ms"].append(sp.layer_ms(sp_imgs))
            nv.inference_batch(nv_imgs)
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            t = []
            for _ in range(10):
                e0.record(); nv.inference_batch(nv_imgs); e1.record(); torch.cuda.synchronize()
                t.append(e0.elapsed_time(e1))
            out[mode]["netvlad_ms"].append(float(np.median(t)))
            for _ in range(args.warmup):
                step(i); i += 1
            fe.finish(st)
            with clocks:
                e0.record()
                for _ in range(args.steps):
                    step(i); i += 1
                e1.record()
                fe.finish(st)
                torch.cuda.synchronize()
            out[mode]["kf_per_s"].append(args.steps * 1e3 / e0.elapsed_time(e1))

    result = {"metric": "split-fp16 vs plain-fp16 networks, 640x480", "gpu": name, "power_limit": power,
              "sm_clock_mhz_median": float(np.median(clocks.samples)) if clocks.samples else None,
              "sm_clock_mhz_range": [min(clocks.samples), max(clocks.samples)] if clocks.samples else None,
              "rounds": args.rounds, "steps": args.steps, "db_rows": DB_ROWS}
    for mode in MODES:
        o = out[mode]
        layers = {k: float(np.median([d[k] for d in o["layer_ms"]])) for k in host.SuperPoint.LAYERS}
        result[mode] = {
            "layer_ms": {k: round(v, 4) for k, v in layers.items()},
            "network_ms": round(sum(layers.values()), 4),
            "mma_tflops": {k: round(mma_tflops(k, v, mode), 1) for k, v in layers.items() if k in SP_CONVS},
            "netvlad_ms": round(float(np.median(o["netvlad_ms"])), 4),
            "kf_per_s": round(float(np.median(o["kf_per_s"])), 2),
            "kf_per_s_rounds": [round(x, 2) for x in o["kf_per_s"]],
            "netvlad_ms_rounds": [round(x, 4) for x in o["netvlad_ms"]],
        }
    result["speedup_network"] = result["split_fp16"]["network_ms"] / result["fp16"]["network_ms"]
    result["speedup_kf_per_s"] = result["fp16"]["kf_per_s"] / result["split_fp16"]["kf_per_s"]
    sp.close(); nv.close(); fe.close()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
