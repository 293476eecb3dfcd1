"""GPU: stereo keyframes with the upper camera as main (the default) against the lower camera as main
(osb_frontend_set_main_camera, the reference's LOWER_CAM_AS_MAIN) on ONE handle: 4-direction 640x480 STEREO_FISHEYE, the
cameras set (triangulation inside extract), a 10 000-row database put in with db_load before the first keyframe.  The two
modes run the same kernels on the same images, so their throughput should agree within run-to-run spread.
Prints one JSON line; writes nothing.

Per mode, keyframes/s of the resident step (extract_dev + ingest_own + query) with images in device memory: CUDA events
around --steps keyframes, one synchronisation at the end.  The modes alternate --rounds times; the medians over rounds are
reported with every round's value beside them, and the SM clock sampled after the last round.

    python scripts/bench_lower_main.py [--steps 200] [--warmup 20] [--rounds 3]
"""
import argparse
import json
import os
import sys

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from gpu_env import gpu_name_and_power, smi  # noqa: E402
from omniswarm_b200 import host, lib, synth  # noqa: E402

W, H, N_DIRS, MAX_NUM = 640, 480, 4, 200
DB_ROWS = 10_000
POOL = 8                  # distinct keyframes cycled through
K = np.array([320.0, 320.0, 320.0, 240.0])


def rig():
    left, right = [], []
    for d in range(N_DIRS):
        yaw = synth._quat_from_rotvec(np.array([0.0, 0.0, d * np.pi / 2]))
        q = synth._PoseAlgebra.q_mul(yaw, np.array([0.5, -0.5, 0.5, -0.5]))
        left.append(np.concatenate([synth._PoseAlgebra.q_rot(yaw, np.array([0.05, 0.0, 0.06])), q]))
        right.append(np.concatenate([synth._PoseAlgebra.q_rot(yaw, np.array([0.05, 0.0, -0.06])), q]))
    return np.array(left), np.array(right)


def make_frontend():
    fe = host.KeyframeFrontend(*synth.frontend_weights(), width=W, height=H, n_dirs=N_DIRS, max_num=MAX_NUM, sp_thres=0.015,
                               self_id=0, db_capacity=DB_ROWS + 4096, inner_product_thres=0.3, match_index_dist=5,
                               zero_bottom_quarter=True, accept_min_3d_pts=10)
    left, right = rig()
    fe.set_cameras(K, left, right, 0.006)
    fe.set_drone_pose(np.array([1.0, -2.0, 0.5, 1.0, 0.0, 0.0, 0.0]))
    for s in range(0, DB_ROWS, 2000):
        g = synth.descriptor_db(2000, 4096, 50 + s)
        ld = np.random.default_rng(s).standard_normal((2000, MAX_NUM, 64)).astype(np.float32)
        fe.db_load(g, ld, np.full(2000, MAX_NUM, np.int32), remote=False)
    return fe


def run(fe, imgs, steps, st, rec, res, msg0):
    torch.cuda.synchronize()
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for i in range(steps):
        up, down = imgs[i % POOL]
        fe.extract(up.data_ptr(), down.data_ptr(), msg0 + i, rec.data_ptr(), st, device_images=True)
        fe.ingest_own(rec.data_ptr(), st)
        fe.query(rec.data_ptr(), res.data_ptr(), st)
    b.record()
    fe.finish(st)
    return steps / (a.elapsed_time(b) / 1000.0)


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--steps", type=int, default=200)
    p.add_argument("--warmup", type=int, default=20)
    p.add_argument("--rounds", type=int, default=3)
    args = p.parse_args()
    st = torch.cuda.current_stream().cuda_stream
    imgs = []
    for k in range(POOL):
        up = np.stack([synth.image(1000 + 10 * k + d, H, W) for d in range(N_DIRS)])
        down = np.stack([np.roll(up[d], 6, axis=0) for d in range(N_DIRS)])
        imgs.append((torch.from_numpy(up).cuda(), torch.from_numpy(down).cuda()))
    rec = torch.zeros(lib.RECORD_BYTES, dtype=torch.uint8, device="cuda")
    res = torch.zeros(lib.RESULT_BYTES, dtype=torch.uint8, device="cuda")
    fe = make_frontend()
    kfs = {"up": [], "down": []}
    msg = 0
    for r in range(args.rounds):
        for mode in ("up", "down"):
            fe.set_main_camera(mode)
            run(fe, imgs, args.warmup, st, rec, res, msg); msg += args.warmup
            kfs[mode].append(run(fe, imgs, args.steps, st, rec, res, msg)); msg += args.steps
            fe.db_reset()
            for s in range(0, DB_ROWS, 2000):        # the same database for every round and mode
                g = synth.descriptor_db(2000, 4096, 50 + s)
                ld = np.random.default_rng(s).standard_normal((2000, MAX_NUM, 64)).astype(np.float32)
                fe.db_load(g, ld, np.full(2000, MAX_NUM, np.int32), remote=False)
    clock = smi("clocks.sm")
    fe.close()
    out = {"bench": "lower_main", "gpu": gpu_name_and_power(), "sm_clock": clock, "steps": args.steps,
           "rounds": args.rounds, "db_rows": DB_ROWS, "images": f"{N_DIRS}x2 {W}x{H}"}
    for mode in ("up", "down"):
        out[f"kf_per_s_{mode}"] = float(np.median(kfs[mode]))
        out[f"kf_per_s_{mode}_rounds"] = [round(v, 1) for v in kfs[mode]]
    out["down_over_up"] = out["kf_per_s_down"] / out["kf_per_s_up"]
    print(json.dumps(out))


if __name__ == "__main__":
    main()
