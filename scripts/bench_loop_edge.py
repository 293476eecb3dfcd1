"""GPU: the loop edges of a round's hits -- osb_frontend_compute_loop against the host path it replaces.  Prints one JSON
line; writes nothing.

Set-up: a 4-direction front-end (max_num 200, geometric filter on, stereo cameras set) whose local store holds one own
keyframe, and 64 received records of the same place (synth.loop_scene: 78 landmarks per direction, outlier matches and
unflagged landmarks), queried with osb_frontend_query_received: 64 hits, each with ~280 correspondences over four direction
pairs.  For n in {1, 8, 64} candidates:
  * device: the CUDA-event time of one osb_frontend_compute_loop call (assemble + PnP-RANSAC + finalise), median of --reps
    after --warmup;
  * host path: what an integrator did before -- download the n query results, assemble the correspondences in numpy from
    host copies of the records (ordered concatenation, lift, rotate_pt_norm2d, the PnP prior) and call osb_pnp_ransac on all
    n at once (upload, kernel, download, synchronise); wall-clock time, median of --host-reps.
The card's name and power limit are read in the same run.

    python scripts/bench_loop_edge.py [--reps 100] [--warmup 10] [--host-reps 10]
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
from oracle.pcm_ref import pose_inv, pose_mul, q_mul, q_rot  # noqa: E402

ND, MN, QDIR = 4, 200, 1
RB, RS, EB = lib.RECORD_BYTES, lib.RESULT_BYTES, lib.EDGE_BYTES
SC = synth.LOOP_SCENE


# ---- the host path: numpy assembly of compute_correspond_features + the PnP prior ------------------------------------
def host_assemble(res, rec, old, K, ext, pose_new, pose_old):
    Xs, uvs = [], []
    main_old = res.hit_dir
    qmi = ext[main_old][3:] * np.array([1.0, -1.0, -1.0, -1.0])
    for j in range(ND):
        dn, do = res.dir_new[j], res.dir_old[j]
        if dn < 0:
            continue
        if res.geo_valid[j]:
            qi = np.array(res.geo_new[j][:res.n_geo[j]]); ti = np.array(res.geo_old[j][:res.n_geo[j]])
        else:
            qi = np.array(res.match_new[j][:res.n_matches[j]]); ti = np.array(res.match_old[j][:res.n_matches[j]])
            keep = np.ctypeslib.as_array(rec.landmarks_flag[dn])[qi] != 0
            qi, ti = qi[keep], ti[keep]
        Xs.append(np.ctypeslib.as_array(rec.landmarks_3d[dn])[qi])
        kp = np.ctypeslib.as_array(old.kpts[do])[ti].astype(np.float64)
        u = ((kp - K[2:]) / K[:2]).astype(np.float32).astype(np.float64)
        p = q_rot(q_mul(qmi, ext[do][3:]), np.concatenate([u, np.ones((len(u), 1))], 1))
        z = p[:, 2].copy()
        z[(z < 1e-3) & (z > 0)] = 1e-3
        z[(z > -1e-3) & (z < 0)] = -1e-3
        uvs.append((p[:, :2] / z[:, None]).astype(np.float32))
    prior = pose_inv(pose_mul(pose_mul(pose_inv(pose_new), pose_old), ext[main_old]))
    return dict(X=np.concatenate(Xs), uv=np.concatenate(uvs), prior=prior, extrinsic=ext[main_old], drone_pose_now=pose_new,
                drone_pose_old=pose_old, iterations=100, thresh=3.0, seed=0, is_4dof=1, min_loop_num=15,
                rperr_thres=10 * np.pi / 180, accept_loop_yaw_rad=30 * np.pi / 180, max_loop_dis=5.0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--reps", type=int, default=100)
    ap.add_argument("--warmup", type=int, default=10)
    ap.add_argument("--host-reps", type=int, default=10)
    a = ap.parse_args()
    fe = host.KeyframeFrontend(*synth.frontend_weights(), width=96, height=64, n_dirs=ND, max_num=MN, self_id=1, db_capacity=64,
                               match_index_dist=5, geometric_filter=True)
    fe.set_cameras(SC["K"], SC["ext"], SC["ext"], 0.006)
    fe.set_loop_params(odometry_consistency_threshold=10.0)
    st = torch.cuda.current_stream().cuda_stream
    old = synth.loop_record(1, 100, "old", 0, g_noise=1e-3)
    ot = torch.frombuffer(bytearray(bytes(old)), dtype=torch.uint8).cuda()
    fe.ingest_own(ot.data_ptr(), st)
    recs = [synth.loop_record(2 + r % 3, 200 + r, "new", 10 + r, g_noise=1e-3) for r in range(64)]
    rt = torch.frombuffer(bytearray(b"".join(bytes(r) for r in recs)), dtype=torch.uint8).cuda()
    res_t = torch.zeros(64 * RS, dtype=torch.uint8, device="cuda")
    fe.query_received(rt.data_ptr(), 64, -1, res_t.data_ptr(), st)
    fe.finish(st)
    cands = [dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"])] * 64
    out = torch.zeros(64 * EB, dtype=torch.uint8, device="cuda")
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    device_ms, host_ms, accepted, n_corr = {}, {}, {}, {}
    for n in (1, 8, 64):
        ts = []
        for i in range(a.warmup + a.reps):
            e0.record()
            fe.compute_loop(rt.data_ptr(), res_t.data_ptr(), cands[:n], out.data_ptr(), st)
            e1.record()
            e1.synchronize()
            if i >= a.warmup:
                ts.append(e0.elapsed_time(e1))
        device_ms[n] = float(np.median(ts))
        raw = out.cpu().numpy().tobytes()
        edges = [lib.LoopEdgeResult.from_buffer_copy(raw[i * EB:(i + 1) * EB]) for i in range(n)]
        accepted[n] = sum(e.status == lib.LOOP_ACCEPTED for e in edges)
        n_corr[n] = float(np.mean([e.n_corr for e in edges]))
        ts = []
        for i in range(1 + a.host_reps):
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            rawr = res_t[:n * RS].cpu().numpy().tobytes()
            results = [lib.LoopResult.from_buffer_copy(rawr[i * RS:(i + 1) * RS]) for i in range(n)]
            cases = [host_assemble(results[i], recs[i], old, SC["K"], SC["ext"], SC["pose_new"], SC["pose_old"])
                     for i in range(n)]
            host.pnp_ransac(cases, max_n=lib.LOOP_MAXN)
            if i >= 1:
                ts.append((time.perf_counter() - t0) * 1e3)
        host_ms[n] = float(np.median(ts))
    fe.close()
    print(json.dumps(dict(bench="loop_edge", device_compute_loop_ms=device_ms, host_path_ms=host_ms,
                          speedup={n: host_ms[n] / device_ms[n] for n in device_ms}, accepted=accepted,
                          mean_correspondences=n_corr, gpu=smi("name"), power_limit=smi("power.limit"),
                          reps=a.reps, warmup=a.warmup, host_reps=a.host_reps)))


if __name__ == "__main__":
    main()
