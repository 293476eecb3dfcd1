"""GPU: depth-camera keyframes (PINHOLE_DEPTH, the RealSense configuration: one 640x480 gray image + aligned 16-bit depth,
n_dirs = 1) through the keyframe front-end, against the stereo pinhole step (n_dirs = 1, up + down image) on a handle
with the same settings.  Both handles hold a 10 000-row database put in with db_load before the first keyframe.
Prints one JSON line; writes nothing.

Per mode, keyframes/s of
  * the host-buffer step (process_depth / process) from pinned host memory: wall clock, the call synchronises;
  * the resident step (extract_depth_dev / extract_dev + ingest_own + query) with images in device memory: CUDA events
    around --steps keyframes, one synchronisation at the end;
and the median stage_ms of a profiled pass.  The modes alternate --rounds times; the medians over rounds are reported with
every round's value beside them.

    python scripts/bench_depth_frontend.py [--steps 200] [--warmup 20] [--rounds 3]
"""
import argparse
import json
import os
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gpu_env import gpu_name_and_power  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402

W, H, N_DIRS, MAX_NUM = 640, 480, 1, 200
DB_ROWS = 10_000
POOL = 8                  # distinct keyframes cycled through; from the second cycle on every query is a revisit
STAGE_KF = 20
K = np.array([380.0, 380.0, 320.0, 240.0])          # fx fy cx cy of the 640x480 pinhole
EXTRINSIC = np.array([[0.08, 0.0, 0.03, 0.5, -0.5, 0.5, -0.5]])   # camera z = body x
POSE_DRONE = np.array([1.0, -2.0, 0.5, 1.0, 0.0, 0.0, 0.0])


def make_frontend(capacity, depth):
    fe = host.KeyframeFrontend(*synth.frontend_weights(), width=W, height=H, n_dirs=N_DIRS, max_num=MAX_NUM, sp_thres=0.015,
                               self_id=0, db_capacity=capacity, inner_product_thres=0.3, match_index_dist=5,
                               zero_bottom_quarter=False, accept_min_3d_pts=10)
    if depth:
        fe.set_depth_camera(K, EXTRINSIC, 0.3, 10.0)
        fe.set_drone_pose(POSE_DRONE)
    n, chunk = DB_ROWS, 2000
    for s in range(0, n, chunk):
        m = min(chunk, n - s)
        g = synth.descriptor_db(m, 4096, 50 + s)
        ld = np.random.default_rng(s).standard_normal((m, MAX_NUM, 64)).astype(np.float32)
        fe.db_load(g, ld, np.full(m, MAX_NUM, np.int32), remote=False)
    return fe


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--steps", type=int, default=200, help="keyframes per timed window")
    ap.add_argument("--warmup", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=3)
    args = ap.parse_args()
    assert lib.load().osb_device_count() > 0, "needs a CUDA device"
    gpu = gpu_name_and_power()
    st = torch.cuda.current_stream().cuda_stream
    # every ingest charges OSB_MAX_DIRS rows to the host's bound until the next synchronisation: size the stores so that the
    # timed windows never hit the capacity check
    per_round = 2 * (args.warmup + args.steps)
    capacity = DB_ROWS + 4 * (args.rounds * per_round + STAGE_KF) + 64

    gray = [synth.image(500 + s, H, W)[None] for s in range(POOL)]
    second = [synth.image(700 + s, H, W)[None] for s in range(POOL)]          # the stereo pair's down image
    depth = [synth.depth_image(500 + s, H, W)[None] for s in range(POOL)]
    pin = lambda a: torch.from_numpy(np.ascontiguousarray(a)).pin_memory()
    p_gray, p_second = [pin(a) for a in gray], [pin(a) for a in second]
    p_depth = [pin(a.view(np.int16)) for a in depth]                          # uint16 bytes carried as int16
    d_gray, d_second, d_depth = [t.cuda() for t in p_gray], [t.cuda() for t in p_second], [t.cuda() for t in p_depth]
    rec_host = torch.zeros(lib.RECORD_BYTES, dtype=torch.uint8).pin_memory()
    res_host = torch.zeros(lib.RESULT_BYTES, dtype=torch.uint8).pin_memory()
    rec_dev = torch.zeros(lib.RECORD_BYTES, dtype=torch.uint8, device="cuda")
    res_dev = torch.zeros(lib.RESULT_BYTES, dtype=torch.uint8, device="cuda")

    fes = {"depth": make_frontend(capacity, True), "stereo": make_frontend(capacity, False)}

    def host_step(mode, i):
        j = i % POOL
        if mode == "depth":
            fes[mode].process_depth_raw(p_gray[j].data_ptr(), p_depth[j].data_ptr(), i, rec_host.data_ptr(),
                                        res_host.data_ptr())
        else:
            fes[mode].process_raw(p_gray[j].data_ptr(), p_second[j].data_ptr(), i, rec_host.data_ptr(), res_host.data_ptr())

    def resident_step(mode, i):
        j, fe = i % POOL, fes[mode]
        if mode == "depth":
            fe.extract_depth(d_gray[j].data_ptr(), d_depth[j].data_ptr(), i, rec_dev.data_ptr(), st, device_images=True)
        else:
            fe.extract(d_gray[j].data_ptr(), d_second[j].data_ptr(), i, rec_dev.data_ptr(), st, device_images=True)
        fe.ingest_own(rec_dev.data_ptr(), st)
        fe.query(rec_dev.data_ptr(), res_dev.data_ptr(), st)

    def kf_per_s_host(mode, base):
        for i in range(args.warmup):
            host_step(mode, base + i)
        t0 = time.perf_counter()
        for i in range(args.steps):
            host_step(mode, base + args.warmup + i)
        return args.steps / (time.perf_counter() - t0)

    def kf_per_s_resident(mode, base):
        fe = fes[mode]
        for i in range(args.warmup):
            resident_step(mode, base + i)
        fe.finish(st)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(args.steps):
            resident_step(mode, base + args.warmup + i)
        e1.record()
        fe.finish(st)
        torch.cuda.synchronize()
        return args.steps * 1e3 / e0.elapsed_time(e1)

    rates = {m: {"host": [], "resident": []} for m in fes}
    for r in range(args.rounds):
        for mode in ("depth", "stereo"):
            rates[mode]["host"].append(kf_per_s_host(mode, 100_000 * r))
            rates[mode]["resident"].append(kf_per_s_resident(mode, 100_000 * r + 50_000))

    out = {"metric": "keyframes/s, 640x480, n_dirs 1, 10000-row database", "gpu": gpu,
           "steps": args.steps, "warmup": args.warmup, "rounds": args.rounds}
    for mode, fe in fes.items():
        fe.set_profiling(True)
        acc = {}
        for i in range(STAGE_KF):
            resident_step(mode, 900_000 + i)
            fe.finish(st)
            for k, v in fe.stage_ms().items():
                acc.setdefault(k, []).append(v)
        fe.set_profiling(False)
        stages = {k: float(np.median(v)) for k, v in acc.items()}
        if mode == "depth":                                    # stage [3] is the depth lift + pack there
            stages = {("depth_lift_pack" if k == "stereo_pack" else k): v for k, v in stages.items()}
        rec = lib.KeyframeRecord.from_buffer_copy(rec_dev.cpu().numpy().tobytes())
        out[mode] = {
            "host_pinned_kf_per_s": float(np.median(rates[mode]["host"])),
            "resident_kf_per_s": float(np.median(rates[mode]["resident"])),
            "host_pinned_rounds": [round(x, 1) for x in rates[mode]["host"]],
            "resident_rounds": [round(x, 1) for x in rates[mode]["resident"]],
            "stage_ms": stages,
            "db_rows": fe.db_size(False),
            "last_keyframe": {"n_kpts": int(rec.n_kpts[0]), "n_flagged": int(sum(rec.landmarks_flag[0][:rec.n_kpts[0]]))},
        }
        fe.close()
    out["depth_over_stereo_resident"] = out["depth"]["resident_kf_per_s"] / out["stereo"]["resident_kf_per_s"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
