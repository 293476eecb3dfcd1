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
import subprocess
import sys
import time

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))
import numpy as np  # noqa: E402
import torch  # noqa: E402

from omniswarm_b200 import host, lib, synth  # noqa: E402

ND, MN, QDIR = 4, 200, 1
RB, RS, EB = lib.RECORD_BYTES, lib.RESULT_BYTES, lib.EDGE_BYTES
SC = synth.loop_scene()
NPT = len(SC["X"][0])
G = synth.descriptor_db(ND, 4096, 5)
DESC = [synth.local_descriptors(NPT, 40 + d) for d in range(ND)]


def smi(query):
    r = subprocess.run(["nvidia-smi", f"--query-gpu={query}", "--format=csv,noheader"], capture_output=True, text=True,
                       timeout=30)
    return r.stdout.strip().splitlines()[0]


def record(drone, msg, side, seed):
    rng = np.random.default_rng(seed)
    r = lib.KeyframeRecord()
    r.drone_id, r.msg_id, r.n_dirs = drone, msg, ND
    for d in range(ND):
        perm = np.arange(NPT) if side == "old" else rng.permutation(NPT)
        kp = (SC["kp_old"][d] if side == "old" else SC["kp_new"][d])[perm].copy()
        X = SC["X"][d][perm].copy()
        desc = DESC[d][perm] + (0 if side == "old" else rng.normal(0, 0.02, (NPT, 64)).astype(np.float32))
        desc /= np.linalg.norm(desc, axis=1, keepdims=True)
        flag = np.ones(NPT, np.int32)
        if side == "new":
            flag[::11] = 0
            out = rng.choice(NPT, 4, replace=False)
            kp[out] = rng.uniform(0, 96, (4, 2))
            X[out] = rng.normal(0, 3, (4, 3))
        g = G[d] + (0 if side == "old" else rng.normal(0, 1e-3, 4096).astype(np.float32))
        r.n_kpts[d] = NPT
        np.ctypeslib.as_array(r.global_desc[d])[:] = g / np.linalg.norm(g)
        np.ctypeslib.as_array(r.local_desc[d])[:NPT] = desc
        np.ctypeslib.as_array(r.kpts[d])[:NPT] = kp
        np.ctypeslib.as_array(r.landmarks_3d[d])[:NPT] = X
        np.ctypeslib.as_array(r.landmarks_flag[d])[:NPT] = flag
        np.ctypeslib.as_array(r.stereo_match[d])[:NPT] = np.where(flag > 0, 0, -1)
    return r


# ---- the host path: numpy assembly of compute_correspond_features + the PnP prior ------------------------------------
def q_mul(a, b):
    aw, ax, ay, az = a; bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw])


def q_rot(q, v):
    u = np.broadcast_to(q[1:], v.shape)
    c = np.cross(u, v)
    return v + 2.0 * (q[0] * c + np.cross(u, c))


def pose_mul(a, b):
    return np.concatenate([a[:3] + q_rot(a[3:], b[:3]), q_mul(a[3:], b[3:])])


def pose_inv(a):
    qc = a[3:] * np.array([1.0, -1.0, -1.0, -1.0])
    return np.concatenate([-q_rot(qc, a[:3]), qc])


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
    comp, mean = synth.pca_matrices(0)
    fe = host.KeyframeFrontend(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean,
                               synth.flatten_nv_weights(synth.netvlad_weights(0)), width=96, height=64, n_dirs=ND,
                               max_num=MN, self_id=1, db_capacity=64, match_index_dist=5, geometric_filter=True)
    fe.set_cameras(SC["K"], SC["ext"], SC["ext"], 0.006)
    fe.set_loop_params(odometry_consistency_threshold=10.0)
    st = torch.cuda.current_stream().cuda_stream
    old = record(1, 100, "old", 0)
    ot = torch.frombuffer(bytearray(bytes(old)), dtype=torch.uint8).cuda()
    fe.ingest_own(ot.data_ptr(), st)
    recs = [record(2 + r % 3, 200 + r, "new", 10 + r) for r in range(64)]
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
