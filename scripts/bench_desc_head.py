"""GPU: what the keypoint kernel and SuperPoint's descriptor head cost on the benchmark's 8-image 640x480 batch (4 up, 4 down
images with the bottom quarter blanked, max_num 200).  Prints one JSON line; writes nothing.

Each form of the network's tail (the descriptor head convDa + convDb + l2norm_cells, and sp_keypoints_kernel) is run
  * "forked" (the default): the keypoint kernel on its own stream beside the head, the head on head_ctas = SMs - B CTAs;
  * "serial" (a handle created under OSB_SP_OVERLAP=0): the head on every SM, then the keypoint kernel on the same stream;
both in a standalone SuperPoint handle (nothing else on the GPU) and in a front-end keyframe created under
OSB_SP_SPARSE_HEAD=0 (NetVLAD runs beside it on its second stream).  The front-end's default, "sparse" (the keypoint kernel,
then the head at the sampled cells only, on the network's stream), is the third front-end form.  Per form and setting:
the keypoint kernel's time (kp_ms), the head's span from its first kernel's start to its last one's end (head_ms) and
each of its kernels, and the tail from the first of the head and the keypoint kernel to start to the last to end (tail_ms:
what the tail adds to the keyframe).  So
  * the keypoint kernel alone is standalone.serial.kp_ms;
  * the head under the head_ctas cap is standalone.forked.head_ms (frontend.forked.head_ms beside NetVLAD);
  * frontend.<form>.stage_ms holds the front-end's stages of a keyframe (osb_frontend_stage_ms).
Kernel times come from torch.profiler (CUDA activities), median over --reps batches or keyframes.  The card's name, power
limit and SM clock, sampled while the runs go, are recorded beside the numbers.

    python scripts/bench_desc_head.py [--reps 20] [--precision split_fp16]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402
from torch.profiler import ProfilerActivity, profile  # noqa: E402

from gpu_env import ClockSampler, smi  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402

W, H, N_DIRS, MAX_NUM, THRES = 640, 480, 4, 200, 0.015
KP, L2, GATHER = "sp_keypoints_kernel", "l2norm_cells_kernel", "sp_cell_gather_kernel"


def keyframe_images(seed):
    """bench.py's keyframe: 4 up and 4 down images"""
    up = np.stack([synth.image(1000 * seed + d, H, W) for d in range(N_DIRS)])
    down = np.stack([synth.image(1000 * seed + 100 + d, H, W) for d in range(N_DIRS)])
    return up, down


def kernels(prof):
    """[(name, stream, start_ns, end_ns)] of every kernel in the trace, by start"""
    out = []
    for e in prof.profiler.kineto_results.events():
        if e.device_type() != torch.autograd.DeviceType.CUDA or e.name().startswith(("Memcpy", "Memset")):
            continue
        out.append((e.name(), e.device_resource_id(), e.start_ns(), e.end_ns()))
    return sorted(out, key=lambda k: k[2])


def tail_rows(ks):
    """per keyframe or batch: {kp_ms, head_ms, tail_ms} and the head's kernels.  The dense head is the l2norm_cells launch
    and the two kernels before it on its stream (convDa, convDb); the sparse head is the sp_cell_gather_kernel launch and
    the two after it (convDa as a 1x1 layer, convDb), the L2 norm being taken inside the descriptor kernels.  The keypoint
    kernel is the one that starts nearest to the head (beside it when forked, right before or after it otherwise)."""
    rows = []
    kps = [k for k in ks if KP in k[0]]
    ms = lambda t: t * 1e-6  # noqa: E731
    for i, k in enumerate(ks):
        if L2 in k[0]:
            da, db = [x for x in ks[:i] if x[1] == k[1]][-2:]
            head = {"convDa": da, "convDb": db, "l2norm_cells": k}
        elif GATHER in k[0]:
            da, db = [x for x in ks[i + 1:] if x[1] == k[1]][:2]
            head = {"gather": k, "convDa": da, "convDb": db}
        else:
            continue
        first, last = min(x[2] for x in head.values()), max(x[3] for x in head.values())
        kp = min(kps, key=lambda x: abs(x[2] - first))
        rows.append({"kp_ms": ms(kp[3] - kp[2]), "head_ms": ms(last - first),
                     "tail_ms": ms(max(kp[3], last) - min(kp[2], first)),
                     **{n: ms(x[3] - x[2]) for n, x in head.items()}})
    return rows


def summary(rows, stages=None):
    out = {k: round(float(np.median([r[k] for r in rows])), 4) for k in rows[0]}
    if stages:
        out["stage_ms"] = {k: round(float(np.median(v)), 4) for k, v in stages.items()}
    return out


def profiled(fn, reps):
    """torch.profiler around reps calls of fn(i) -> tail_rows of the trace"""
    with profile(activities=[ProfilerActivity.CUDA]) as prof:
        for i in range(reps):
            fn(i)
        torch.cuda.synchronize()
    return tail_rows(kernels(prof))


def standalone(images, reps, precision):
    sp = host.SuperPoint(*synth.frontend_weights()[:3], W, H, THRES, MAX_NUM, max_batch=len(images))
    sp.set_precision(precision)
    for _ in range(3):
        sp.inference_batch(images)
    rows = profiled(lambda i: sp.inference_batch(images), reps)
    sp.close()
    return summary(rows)


def frontend(up, down, reps, precision):
    fe = host.KeyframeFrontend(*synth.frontend_weights(), width=W, height=H, n_dirs=N_DIRS, max_num=MAX_NUM,
                               sp_thres=THRES, db_capacity=64, zero_bottom_quarter=True, accept_min_3d_pts=10)
    fe.set_precision(precision)
    st = torch.cuda.current_stream().cuda_stream
    dev_up, dev_dn = torch.from_numpy(up).cuda(), torch.from_numpy(down).cuda()
    rec = torch.zeros(lib.RECORD_BYTES, dtype=torch.uint8, device="cuda")

    def keyframe(i):          # extract only: nothing is ingested, so the database stays empty
        fe.extract(dev_up.data_ptr(), dev_dn.data_ptr(), i, rec.data_ptr(), st, device_images=True)
        fe.finish(st)

    for i in range(3):
        keyframe(i)
    fe.set_profiling(True)
    stages = {}
    for i in range(reps):
        keyframe(100 + i)
        for k, v in fe.stage_ms().items():
            stages.setdefault(k, []).append(v)
    fe.set_profiling(False)
    rows = profiled(lambda i: keyframe(200 + i), reps)
    fe.close()
    return summary(rows, stages)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=20, help="profiled batches / keyframes per form and setting")
    ap.add_argument("--precision", default="split_fp16", choices=sorted(host.PRECISIONS))
    args = ap.parse_args()
    assert lib.load().osb_device_count() > 0, "needs a CUDA device"
    name, power = smi("name"), smi("power.limit")
    up, down = keyframe_images(0)
    images = np.concatenate([up, down])
    images[:, H * 3 // 4:, :] = 0        # the front-end blanks the bottom quarter (loop_cam.cpp:536-539)
    result = {"metric": "keypoint kernel vs descriptor head, 8 x 640x480", "precision": args.precision, "gpu": name,
              "power_limit": power, "reps": args.reps}
    clocks = ClockSampler()
    with clocks:
        # the handles read OSB_SP_OVERLAP and OSB_SP_SPARSE_HEAD when they are created
        result["frontend"] = {"sparse": frontend(up, down, args.reps, args.precision)}
        os.environ["OSB_SP_SPARSE_HEAD"] = "0"
        for form in ("forked", "serial"):
            if form == "serial":
                os.environ["OSB_SP_OVERLAP"] = "0"
            result.setdefault("standalone", {})[form] = standalone(images, args.reps, args.precision)
            result["frontend"][form] = frontend(up, down, args.reps, args.precision)
        os.environ.pop("OSB_SP_OVERLAP", None)
        os.environ.pop("OSB_SP_SPARSE_HEAD", None)
    result["sm_clock_mhz_median"] = float(np.median(clocks.samples)) if clocks.samples else None
    result["sm_clock_mhz_range"] = [min(clocks.samples), max(clocks.samples)] if clocks.samples else None
    print(json.dumps(result))


if __name__ == "__main__":
    main()
