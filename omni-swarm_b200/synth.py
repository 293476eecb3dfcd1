"""Seeded synthetic inputs shared by the product, the tests, the oracle and bench.py.

Nothing here computes any part of the hot path: it only *generates data* (network weights,
PCA matrices, images, descriptor databases, pose graphs).  The reference ships no weights, bags
or fixtures (SURVEY.md section 8c): weights are a Dropbox download
(/root/reference/README.md:27), so every run of the path uses seeded stand-ins fed identically
to the oracle and to the CUDA kernels.

All generators use numpy's PCG64 (`np.random.default_rng(seed)`), which is bit-reproducible across
machines for a given numpy version (the GPU box runs this same image).
"""
from __future__ import annotations

import math
import numpy as np

# ----------------------------------------------------------------------------------------------
# SuperPoint (layer table follows /root/reference/swarm_loop/superpoint.ipynb:135-160)
# ----------------------------------------------------------------------------------------------
# (name, Cin, Cout, ksize)
SP_LAYERS = [
    ("conv1a", 1, 64, 3), ("conv1b", 64, 64, 3),
    ("conv2a", 64, 64, 3), ("conv2b", 64, 64, 3),
    ("conv3a", 64, 128, 3), ("conv3b", 128, 128, 3),
    ("conv4a", 128, 128, 3), ("conv4b", 128, 128, 3),
    ("convPa", 128, 256, 3), ("convPb", 256, 65, 1),
    ("convDa", 128, 256, 3), ("convDb", 256, 256, 1),
]


def sp_num_weights() -> int:
    return sum(co * ci * k * k + co for _, ci, co, k in SP_LAYERS)


def superpoint_weights(seed: int = 0, pb_gain: float = 8.0, dustbin_bias: float = 11.0) -> dict:
    """He-initialised SuperPoint weights, OIHW float32, plus biases.

    `pb_gain` / `dustbin_bias` shape the detector head so that the 65-way softmax is not
    degenerate (uniform 1/65 would put every pixel above the reference's 0.015 threshold):
    with these values a textured 640x480 image yields ~3500 candidates above
    thres=0.015 and ~320 above 0.2, i.e. the regime of SURVEY.md section 8d C2.
    """
    rng = np.random.default_rng(seed)
    w = {}
    for name, ci, co, k in SP_LAYERS:
        std = math.sqrt(2.0 / (ci * k * k))
        W = rng.standard_normal((co, ci, k, k)).astype(np.float32) * np.float32(std)
        b = (rng.standard_normal(co) * 0.05).astype(np.float32)
        if name == "convPb":
            W = W * np.float32(pb_gain)
            b[64] += np.float32(dustbin_bias)
        w[name + ".weight"] = np.ascontiguousarray(W)
        w[name + ".bias"] = b
    return w


def flatten_sp_weights(w: dict) -> np.ndarray:
    """The C-ABI weight blob: for each layer in SP_LAYERS order, weight (OIHW) then bias."""
    parts = []
    for name, *_ in SP_LAYERS:
        parts.append(w[name + ".weight"].reshape(-1))
        parts.append(w[name + ".bias"].reshape(-1))
    out = np.concatenate(parts).astype(np.float32)
    assert out.size == sp_num_weights()
    return out


def pca_matrices(seed: int = 0):
    """Stand-in for components_.csv (64x256) / mean_.csv (256) written by
    /root/reference/swarm_loop/pca.ipynb cells 2-3: orthonormal rows + small mean."""
    rng = np.random.default_rng(seed + 1000)
    q, _ = np.linalg.qr(rng.standard_normal((256, 64)))
    comp = np.ascontiguousarray(q.T.astype(np.float32))          # [64,256]
    mean = (rng.standard_normal(256) * 0.02).astype(np.float32)  # [256]
    return comp, mean


# ----------------------------------------------------------------------------------------------
# NetVLAD stand-in ("MobileNetVLAD-lite"; the real hfnet architecture is absent from the
# reference, SURVEY.md section 8c).  I/O contract: mobilenetvlad_tensorrt.h:9-15 (HxW f32 0..255
# in, 4096 f32 out).
# ----------------------------------------------------------------------------------------------
# backbone: conv0 3x3 s2 (1->32) + ReLU6, then depthwise-separable blocks (dw3x3 stride s, pw 1x1)
NV_BLOCKS = [  # (Cin, Cout, stride)
    (32, 64, 1), (64, 128, 2), (128, 128, 1), (128, 256, 2), (256, 256, 1), (256, 512, 2),
    (512, 512, 1),
]
NV_K = 32     # clusters
NV_D = 128    # descriptor dim  -> K*D = 4096 = DEEP_DESC_SIZE (loop_defines.h:30)
NV_INPUT_SCALE = 1.0 / 255.0  # folded into conv0 (engine input is unscaled 0..255)


def netvlad_layer_table():
    """[(name, shape)] in blob order."""
    t = [("conv0.weight", (32, 1, 3, 3)), ("conv0.bias", (32,))]
    for i, (ci, co, s) in enumerate(NV_BLOCKS):
        t += [(f"b{i}.dw.weight", (ci, 1, 3, 3)), (f"b{i}.dw.bias", (ci,)),
              (f"b{i}.pw.weight", (co, ci, 1, 1)), (f"b{i}.pw.bias", (co,))]
    t += [("proj.weight", (NV_D, 512, 1, 1)), ("proj.bias", (NV_D,)),
          ("assign.weight", (NV_K, NV_D, 1, 1)), ("assign.bias", (NV_K,)),
          ("centroids", (NV_K, NV_D))]
    return t


def nv_num_weights() -> int:
    return sum(int(np.prod(s)) for _, s in netvlad_layer_table())


def netvlad_weights(seed: int = 0) -> dict:
    rng = np.random.default_rng(seed + 2000)
    w = {}
    for name, shape in netvlad_layer_table():
        if name.endswith(".bias"):
            w[name] = (rng.standard_normal(shape) * 0.05).astype(np.float32)
        elif name == "centroids":
            # small centroids: residuals x - c stay image-specific (real NetVLAD centroids are data cluster centres)
            w[name] = (rng.standard_normal(shape) * 0.01).astype(np.float32)
        else:
            fan_in = int(np.prod(shape[1:]))
            gain = 8.0 if name.startswith("assign") else 1.0
            w[name] = (rng.standard_normal(shape) * math.sqrt(2.0 / fan_in) * gain).astype(np.float32)
    return w


def flatten_nv_weights(w: dict) -> np.ndarray:
    out = np.concatenate([w[n].reshape(-1) for n, _ in netvlad_layer_table()]).astype(np.float32)
    assert out.size == nv_num_weights()
    return out


# ----------------------------------------------------------------------------------------------
# Images, descriptor databases
# ----------------------------------------------------------------------------------------------
def image(seed: int, H: int = 480, W: int = 640, zero_bottom_quarter: bool = False) -> np.ndarray:
    """Textured uint8 image: smoothed noise at two scales + sharp blobs + pixel noise
    (SURVEY.md section 8d C2).  `zero_bottom_quarter` reproduces loop_cam.cpp:536-539."""
    from scipy import ndimage
    rng = np.random.default_rng(seed + 3000)
    a = ndimage.gaussian_filter(rng.standard_normal((H, W)), 6.0)
    b = ndimage.gaussian_filter(rng.standard_normal((H, W)), 1.5)
    img = a / a.std() * 40.0 + b / b.std() * 25.0 + 128.0
    nb = 120
    ys = rng.integers(0, H, nb)
    xs = rng.integers(0, W, nb)
    rad = rng.integers(2, 9, nb)
    val = rng.uniform(-90, 90, nb)
    yy, xx = np.mgrid[0:H, 0:W]
    for y, x, r, v in zip(ys, xs, rad, val):
        y0, y1, x0, x1 = max(0, y - r), min(H, y + r + 1), max(0, x - r), min(W, x + r + 1)
        m = (yy[y0:y1, x0:x1] - y) ** 2 + (xx[y0:y1, x0:x1] - x) ** 2 <= r * r
        img[y0:y1, x0:x1][m] += v
    img += rng.uniform(-6, 6, (H, W))
    img = np.clip(img, 0, 255).astype(np.uint8)
    if zero_bottom_quarter:
        img[H * 3 // 4:, :] = 0
    return img


def depth_image(seed: int, H: int = 480, W: int = 640, near: float = 0.3, far: float = 10.0) -> np.ndarray:
    """Aligned 16-bit depth image in mm for a PINHOLE_DEPTH keyframe (loop_cam.cpp:231-302): a slanted plane inside
    (near, far), with holes (0, no return), one patch beyond `far` and one below `near`, so that a keyframe's keypoints
    fall on both valid and rejected depths."""
    rng = np.random.default_rng(seed + 7000)
    lo, hi = 1000.0 * near, 1000.0 * far
    yy, xx = np.mgrid[0:H, 0:W]
    a, b = rng.uniform(0.2, 0.8, 2)
    plane = lo + (hi - lo) * (0.1 + 0.3 * a * xx / W + 0.5 * b * yy / H)          # stays within (near, far)
    dep = np.round(plane).astype(np.uint16)

    def patch():
        h, w = max(1, H // 4), max(1, W // 4)
        y0, x0 = int(rng.integers(0, H - h + 1)), int(rng.integers(0, W - w + 1))
        return slice(y0, y0 + h), slice(x0, x0 + w)

    dep[patch()] = np.uint16(min(65535, int(1.5 * hi)))                              # beyond DEPTH_FAR_THRES
    dep[patch()] = np.uint16(0.5 * lo)                                               # below DEPTH_NEAR_THRES
    dep[patch()] = 0                                                                 # a hole
    dep[rng.uniform(size=(H, W)) < 0.1] = 0                                          # scattered missing returns
    return dep


def descriptor_db(n: int, dim: int = 4096, seed: int = 1) -> np.ndarray:
    """n unit-norm Gaussian rows, float32 (SURVEY.md section 8d C3)."""
    rng = np.random.default_rng(seed + 4000)
    out = np.empty((n, dim), np.float32)
    step = 4096
    for s in range(0, n, step):
        x = rng.standard_normal((min(step, n - s), dim)).astype(np.float32)
        x /= np.linalg.norm(x, axis=1, keepdims=True)
        out[s:s + x.shape[0]] = x
    return out


def noisy_queries(db: np.ndarray, rows: np.ndarray, sigma: float = 0.5, seed: int = 2) -> np.ndarray:
    """Queries = chosen DB rows + Gaussian noise of total norm ~sigma, renormalised, so that the
    inner product with the source row is ~1/sqrt(1+sigma^2) (0.89 for 0.5): hits exist."""
    rng = np.random.default_rng(seed + 5000)
    dim = db.shape[1]
    noise = rng.standard_normal((len(rows), dim)).astype(np.float32) * np.float32(sigma / math.sqrt(dim))
    q = (db[rows] + noise).astype(np.float32)
    q /= np.linalg.norm(q, axis=1, keepdims=True)
    return np.ascontiguousarray(q)


def local_descriptors(n: int, seed: int, dim: int = 64, base: np.ndarray | None = None,
                      sigma: float = 0.15) -> np.ndarray:
    """n x dim float32 local descriptors; with `base`, a noisy permuted copy (so matches exist)."""
    rng = np.random.default_rng(seed + 6000)
    if base is None:
        return rng.standard_normal((n, dim)).astype(np.float32)
    idx = rng.permutation(base.shape[0])[:n]
    d = base[idx] + sigma * rng.standard_normal((len(idx), dim)).astype(np.float32)
    return np.ascontiguousarray(d.astype(np.float32))


# ----------------------------------------------------------------------------------------------
# Pose graphs (recipe: /root/reference/swarm_localization/test/swarm_local_sim.cpp, SURVEY A.7)
# ----------------------------------------------------------------------------------------------
FACTOR_DISTANCE = 0    # DistanceMeasurementFactor        factors.hpp:203-224
FACTOR_RELPOSE = 1     # RelativePoseFactor4d             factors.hpp:226-271
FACTOR_DETECTION = 2   # DroneDetection4dFactor           factors.hpp:273-367
PAYLOAD_LEN = 24       # doubles per factor (layout: include/omniswarm_b200.h)


def _wrap(a):
    return a - 2.0 * math.pi * np.floor((a + math.pi) / (2.0 * math.pi))


def _delta_pose(pa, pb):
    """a^-1 . b  for 4-DoF poses [x,y,z,yaw]  (factors.hpp:139-149)."""
    c, s = math.cos(pa[3]), math.sin(pa[3])
    d = pb[:3] - pa[:3]
    return np.array([c * d[0] + s * d[1], -s * d[0] + c * d[1], d[2], _wrap(pb[3] - pa[3])])


def pose_graph(n_drones: int = 5, n_frames: int = 100, n_uwb: int | None = None,
               n_loop: int | None = None, n_det: int | None = None, n_bearing: int = 0,
               seed: int = 0, init_sigma_pos: float = 0.3, init_sigma_yaw: float = 0.05,
               outlier_frac: float = 0.0) -> dict:
    """Synthetic swarm pose graph in the flat layout `osb_graph_solve` consumes.

    Ground truth follows swarm_local_sim.cpp:589-604 (`ParalCirc`: radius 5 m, z amplitude 2 m,
    period 50 s, drones offset on a grid), plus a slow yaw so that yaw is exercised.
    Node index = frame * n_drones + drone.  Factor mix (SURVEY.md section 8d C5): ego-motion
    edges between consecutive frames of each drone (no loss), UWB distances between drones in the
    same frame (Huber), loop edges from a keyframe to one of its 4 nearest stored keyframes (Huber) and
    detections-as-relative-pose between drones in the same frame (Huber).
    Noise model: simulator.launch:33-62 / swarm_local_sim.cpp:532-550,349-353.
    """
    rng = np.random.default_rng(seed + 7000)
    nd, nf = n_drones, n_frames
    n_nodes = nd * nf
    R, Rz, T = 5.0, 2.0, 50.0
    cols = 3
    d0 = 2.0
    t = np.arange(nf) * 0.5  # one swarm frame every 0.5 s
    gt = np.zeros((nf, nd, 4))
    for i in range(nd):
        gt[:, i, 0] = R * np.sin(2 * math.pi * t / T) + (i // cols) * d0
        gt[:, i, 1] = R * (1 - np.cos(2 * math.pi * t / T)) + (i % cols) * d0
        gt[:, i, 2] = Rz * np.sin(2 * math.pi * t / T) + 0.3 * i
        gt[:, i, 3] = _wrap(0.4 * np.sin(2 * math.pi * t / T + i))
    gt = gt.reshape(n_nodes, 4)

    n_ego = nd * (nf - 1)
    if n_uwb is None:
        n_uwb = 2 * nf
    if n_loop is None:
        n_loop = 2 * nf
    if n_det is None:
        n_det = nf

    types, ia, ib, huber = [], [], [], []
    payload = []

    def add(tp, a, b, pl, hub):
        types.append(tp); ia.append(a); ib.append(b); huber.append(hub)
        p = np.zeros(PAYLOAD_LEN); p[:len(pl)] = pl
        payload.append(p)

    # ego motion: RelativePoseFactor4d::CreateCov6d (factors.hpp:255-263): S = sqrt(|inv(cov4)|)
    vo_cov_pos, vo_cov_yaw = 1e-4, 1e-5
    for f in range(nf - 1):
        for i in range(nd):
            a, b = f * nd + i, (f + 1) * nd + i
            step = max(np.linalg.norm(gt[b, :3] - gt[a, :3]), 0.05)
            cov = np.diag([vo_cov_pos * step] * 3 + [vo_cov_yaw * step])
            meas = _delta_pose(gt[a], gt[b]) + rng.standard_normal(4) * np.sqrt(np.diag(cov))
            meas[3] = _wrap(meas[3])
            S = np.sqrt(np.abs(np.linalg.inv(cov)))
            add(FACTOR_RELPOSE, a, b, np.concatenate([meas, S.reshape(-1)]), 0)
    # UWB distances (solver.cpp:1136-1144): r = (|Ta-Tb| - d) / sqrt(cov)
    uwb_cov = 0.0014
    cnt = 0
    while cnt < n_uwb:
        f = int(rng.integers(0, nf)); i, j = rng.choice(nd, 2, replace=False)
        a, b = f * nd + int(max(i, j)), f * nd + int(min(i, j))   # pairs with idb < ida (:1131)
        d = np.linalg.norm(gt[a, :3] - gt[b, :3]) + rng.standard_normal() * math.sqrt(uwb_cov)
        add(FACTOR_DISTANCE, a, b, [d, 1.0 / math.sqrt(uwb_cov)], 1)
        cnt += 1
    # loops: relative pose with sqrt-information diag(1/sigma) (swarm_local_sim.cpp:459-465)
    loop_cov_pos, loop_cov_yaw = 0.003, 5.2e-4
    S_loop = np.diag([1 / math.sqrt(loop_cov_pos)] * 3 + [1 / math.sqrt(loop_cov_yaw)])
    # as the simulator does (swarm_local_sim.cpp:474-529): a keyframe is linked to one of its nearest stored
    # keyframe positions (any drone), excluding its own temporal neighbours
    frame_of = np.arange(n_nodes) // nd
    drone_of = np.arange(n_nodes) % nd
    for _ in range(n_loop):
        a = int(rng.integers(0, n_nodes))
        dist = np.linalg.norm(gt[:, :3] - gt[a, :3], axis=1)
        dist[(drone_of == drone_of[a]) & (np.abs(frame_of - frame_of[a]) <= 3)] = np.inf
        near = np.argsort(dist, kind="stable")[:4]
        b = int(near[int(rng.integers(0, 4))])
        meas = _delta_pose(gt[a], gt[b]) + rng.standard_normal(4) * np.sqrt([loop_cov_pos] * 3 + [loop_cov_yaw])
        if rng.uniform() < outlier_frac:
            meas[:3] += rng.uniform(-3, 3, 3)
        meas[3] = _wrap(meas[3])
        add(FACTOR_RELPOSE, a, b, np.concatenate([meas, S_loop.reshape(-1)]), 1)
    # detections-as-relative-pose (solver.cpp:542-551): same frame, two drones
    det_cov_pos, det_cov_yaw = 0.01, 0.01
    S_det = np.diag([1 / math.sqrt(det_cov_pos)] * 3 + [1 / math.sqrt(det_cov_yaw)])
    for _ in range(n_det):
        f = int(rng.integers(0, nf)); i, j = rng.choice(nd, 2, replace=False)
        a, b = f * nd + int(i), f * nd + int(j)
        meas = _delta_pose(gt[a], gt[b]) + rng.standard_normal(4) * np.sqrt([det_cov_pos] * 3 + [det_cov_yaw])
        meas[3] = _wrap(meas[3])
        add(FACTOR_RELPOSE, a, b, np.concatenate([meas, S_det.reshape(-1)]), 1)
    # bearing / inverse-depth detections (DroneDetection4dFactor, factors.hpp:273-367)
    for k in range(n_bearing):
        f = int(rng.integers(0, nf)); i, j = rng.choice(nd, 2, replace=False)
        a, b = f * nd + int(i), f * nd + int(j)
        mode = k % 3   # 0: extrinsic-z, no depth; 1: extrinsic-z + inverse depth; 2: dposes + depth
        ext_z = 0.05
        if mode == 2:
            dpa = np.array([0.02, -0.01, 0.03, 0.01]); dpb = np.array([-0.01, 0.02, 0.0, -0.02])
            def mul(p, q):
                c, s = math.cos(p[3]), math.sin(p[3])
                return np.array([p[0] + c * q[0] - s * q[1], p[1] + s * q[0] + c * q[1], p[2] + q[2], _wrap(p[3] + q[3])])
            pa, pb = mul(gt[a], dpa), mul(gt[b], dpb)
        else:
            dpa = dpb = np.zeros(4)
            pa = gt[a].copy(); pa[2] += ext_z; pb = gt[b]
        rel = _delta_pose(pa, pb)[:3]
        rho = 1.0 / np.linalg.norm(rel)
        dirv = rel * rho + rng.standard_normal(3) * 0.01
        dirv /= np.linalg.norm(dirv)
        # tangent base: two unit vectors orthogonal to dir
        tmp = np.array([0, 0, 1.0]) if abs(dirv[2]) < 0.9 else np.array([1.0, 0, 0])
        b0 = np.cross(dirv, tmp); b0 /= np.linalg.norm(b0); b1 = np.cross(dirv, b0)
        inv_dep = rho + rng.standard_normal() * 0.01
        flags = (1 if mode >= 1 else 0) | (2 if mode == 2 else 0)
        sphere_std, invdep_std = 0.03, 0.1
        pl = np.concatenate([dirv, b0, b1, [inv_dep, float(flags), ext_z], dpa, dpb, [sphere_std, invdep_std]])
        add(FACTOR_DETECTION, a, b, pl, 1)

    init = gt.copy()
    init[:, :3] += rng.standard_normal((n_nodes, 3)) * init_sigma_pos
    init[:, 3] = _wrap(init[:, 3] + rng.standard_normal(n_nodes) * init_sigma_yaw)
    fixed = np.zeros(n_nodes, np.uint8)
    fixed[0] = 1                     # first pose of self_id constant (solver.cpp:1196-1199)
    init[0] = gt[0]
    return dict(
        n_nodes=n_nodes, gt=gt, init=init, fixed=fixed,
        ftype=np.array(types, np.int32), ia=np.array(ia, np.int32), ib=np.array(ib, np.int32),
        huber=np.array(huber, np.uint8), payload=np.ascontiguousarray(np.array(payload, np.float64)),
    )


def init_graph(n_drones: int = 5, n_frames: int = 100, seed: int = 0) -> dict:
    """The graph of the swarm's initialisation solve (solve_with_multiple_init, solver.cpp:781-845): odometry chains
    and UWB ranges only (every drone to drone 0 and to the previous drone, every frame), before any loop or detection.  Each drone flies its
    own circle (radius, phase, height), so the ranges change over time and fix the drones' offsets; in pose_graph()
    all drones fly the same circle and constant ranges would leave them free.  `init`: drone 0 at ground truth
    (its first pose constant), the others at the origin with their ground-truth (odometry) yaw; `mask` marks drones
    1 ... n_drones-1 for random initialisation."""
    rng = np.random.default_rng(seed + 9100)
    nd, nf = n_drones, n_frames
    n_nodes = nd * nf
    t = np.arange(nf) * 0.5
    gt = np.zeros((nf, nd, 4))
    for i in range(nd):
        r, ph, w = 1.0 + 0.2 * i, 1.3 * i, 2 * math.pi / (30.0 + 7.0 * i)
        gt[:, i, 0] = r * np.cos(w * t + ph) + 4.0 * (i % 3)
        gt[:, i, 1] = r * np.sin(w * t + ph) - 4.0 * (i // 3)
        gt[:, i, 2] = 1.0 + 0.4 * i + 0.1 * np.sin(w * t * 2 + ph)
        gt[:, i, 3] = _wrap(w * t + ph + math.pi / 2)
    gt = gt.reshape(n_nodes, 4)
    types, ia, ib, huber, payload = [], [], [], [], []

    def add(tp, a, b, pl, hub):
        types.append(tp); ia.append(a); ib.append(b); huber.append(hub)
        p = np.zeros(PAYLOAD_LEN); p[:len(pl)] = pl
        payload.append(p)

    vo_cov_pos, vo_cov_yaw = 1e-4, 1e-5
    for f in range(nf - 1):
        for i in range(nd):
            a, b = f * nd + i, (f + 1) * nd + i
            step = max(np.linalg.norm(gt[b, :3] - gt[a, :3]), 0.05)
            cov = np.diag([vo_cov_pos * step] * 3 + [vo_cov_yaw * step])
            meas = _delta_pose(gt[a], gt[b]) + rng.standard_normal(4) * np.sqrt(np.diag(cov))
            meas[3] = _wrap(meas[3])
            add(FACTOR_RELPOSE, a, b, np.concatenate([meas, np.sqrt(np.abs(np.linalg.inv(cov))).reshape(-1)]), 0)
    uwb_cov = 0.0014
    for f in range(nf):
        for i in range(1, nd):
            for j in sorted({0, i - 1}):
                a, b = f * nd + i, f * nd + j
                d = np.linalg.norm(gt[a, :3] - gt[b, :3]) + rng.standard_normal() * math.sqrt(uwb_cov)
                add(FACTOR_DISTANCE, a, b, [d, 1.0 / math.sqrt(uwb_cov)], 1)
    drone = np.arange(n_nodes) % nd
    init = gt.copy()
    init[drone != 0, :3] = 0.0
    fixed = np.zeros(n_nodes, np.uint8)
    fixed[0] = 1
    return dict(
        n_nodes=n_nodes, gt=gt, init=init, fixed=fixed, mask=(drone != 0).astype(np.uint8),
        ftype=np.array(types, np.int32), ia=np.array(ia, np.int32), ib=np.array(ib, np.int32),
        huber=np.array(huber, np.uint8), payload=np.ascontiguousarray(np.array(payload, np.float64)),
    )


def pose_graph_c5(seed: int = 0) -> dict:
    """BASELINE.json C5 graph: 5 drones x 400 frames = 2000 nodes, 12 000 factors
    = 1995 ego + 4000 UWB + 4000 loop + 2005 detection-as-relative-pose."""
    return pose_graph(5, 400, n_uwb=4000, n_loop=4000, n_det=2005, seed=seed)


# ----------------------------------------------------------------------------------------------------------------
# loop edges of one drone pair for the PCM outlier rejection (SURVEY.md 8f-2)
# ----------------------------------------------------------------------------------------------------------------
def _quat_from_rotvec(rv):
    a = np.linalg.norm(rv)
    if a < 1e-12:
        return np.array([1.0, 0.5 * rv[0], 0.5 * rv[1], 0.5 * rv[2]])
    return np.concatenate([[np.cos(a / 2)], np.sin(a / 2) * rv / a])


class _PoseAlgebra:
    """(t, unit quaternion wxyz) poses: compose / invert (generator-side helper, independent of the oracle)"""

    @staticmethod
    def q_mul(a, b):
        aw, ax, ay, az = a; bw, bx, by, bz = b
        return np.array([aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
                         aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw])

    @staticmethod
    def q_rot(q, v):
        u = q[1:]
        c = np.cross(u, v)
        return v + 2.0 * (q[0] * c + np.cross(u, c))

    @classmethod
    def pose_mul(cls, a, b):
        return np.concatenate([a[:3] + cls.q_rot(a[3:], b[:3]), cls.q_mul(a[3:], b[3:])])

    @classmethod
    def pose_inv(cls, a):
        qc = np.array([a[3], -a[4], -a[5], -a[6]])
        return np.concatenate([-cls.q_rot(qc, a[:3]), qc])


def pcm_edges(n: int = 60, outlier_frac: float = 0.3, seed: int = 0, flip_frac: float = 0.3, id_a: int = 1, id_b: int = 2,
              other_pair: int = 0):
    """n loop edges between drones id_a and id_b flying the circles of swarm_local_sim.cpp (:589-604) with yaw and small
    roll/pitch: inliers = true relative pose + noise of the labelled covariance, outliers = gross errors; a fraction of
    the edges is stored b -> a (LoopEdge::same_robot_pair == 2); `other_pair` extra edges belong to another drone pair.
    Edge dicts as oracle/pcm_ref.py and host.pcm_outlier_rejection take them; e["inlier"] is the ground truth."""
    rng = np.random.default_rng(seed + 7000)
    T, R = 50.0, 5.0
    pr = _PoseAlgebra

    def gt(drone, t):
        ph = 2 * np.pi * t / T
        pos = np.array([R * np.sin(ph) + 2.0 * drone, R * (1 - np.cos(ph)) - 1.5 * drone, 2.0 * np.sin(ph) + 0.3 * drone])
        q = _quat_from_rotvec(np.array([0.03 * np.sin(ph), 0.02 * np.cos(ph), 0.6 * ph + 0.2 * drone]))
        return np.concatenate([pos, q])

    def path_len(t):                          # arc length of the circle (constant speed), metres
        return np.hypot(2 * np.pi * R / T, 2 * np.pi * 2.0 / T * 0.7) * t

    sig_p, sig_a = 0.03, 0.01
    cov = np.diag([sig_p ** 2] * 3 + [sig_a ** 2] * 3)
    edges = []
    for i in range(n + other_pair):
        ta, tb = rng.uniform(0, 40), rng.uniform(0, 40)
        a, b = (id_a, id_b) if i < n else (id_a, id_b + 5)
        pa, pb = gt(a, ta), gt(b, tb)
        rel = pr.pose_mul(pr.pose_inv(pa), pb)
        inlier = rng.uniform() >= outlier_frac
        if inlier:
            noise = np.concatenate([rng.normal(0, sig_p, 3), _quat_from_rotvec(rng.normal(0, sig_a, 3))])
        else:
            noise = np.concatenate([rng.uniform(-3, 3, 3), _quat_from_rotvec(rng.uniform(-0.8, 0.8, 3))])
        rel = pr.pose_mul(rel, noise)
        rel[3:] /= np.linalg.norm(rel[3:])
        e = dict(id_a=a, id_b=b, rel=rel, cov=cov * rng.uniform(0.8, 1.3), odom_a=pa, odom_b=pb, len_a=path_len(ta),
                 len_b=path_len(tb), inlier=bool(inlier) and i < n)
        if i < n and rng.uniform() < flip_frac:                      # the same loop reported b -> a
            e = dict(id_a=b, id_b=a, rel=pr.pose_inv(rel), cov=e["cov"], odom_a=pb, odom_b=pa, len_a=e["len_b"],
                     len_b=e["len_a"], inlier=e["inlier"])
        edges.append(e)
    order = rng.permutation(len(edges))
    return [edges[i] for i in order]


def pcm_swarm_rounds(n_drones: int = 5, rounds: int = 6, per_round: int = 8, outlier_frac: float = 0.3, seed: int = 0,
                     n_duplicates: int = 2, n_perturbed: int = 2):
    """The loop edges OutlierRejectionLoopEdges receives before successive solves of a swarm of drones 1..n_drones: every
    unordered pair {a, b} (a == b: intra-drone loops) gains 1..per_round new loops per round (pcm_edges of that pair).  As
    find_available_loops_detections does, every round re-submits every earlier loop before its new ones; `n_perturbed` of
    the re-submitted loops carry perturbed values (re-anchoring gives the same id other values), and `n_duplicates` of the
    round's new loops are submitted twice with the same id.  Ids are above 2^32.
    -> [(edges, ids int64 [n])] per round."""
    rng = np.random.default_rng(seed + 9100)
    drones = range(1, n_drones + 1)
    pairs = [(a, b) for a in drones for b in drones if a <= b]
    counts = rng.integers(1, per_round + 1, size=(len(pairs), rounds))
    per_pair = []
    for pi, (a, b) in enumerate(pairs):
        es = pcm_edges(int(counts[pi].sum()), outlier_frac, seed * 1000 + pi, id_a=a, id_b=b)
        per_pair.append([(e, (1 << 32) + (pi << 20) + 7 * k + 3) for k, e in enumerate(es)])
    out, earlier, taken = [], [], np.zeros(len(pairs), int)
    for r in range(rounds):
        new = []
        for pi in range(len(pairs)):
            c = int(counts[pi, r])
            new += per_pair[pi][taken[pi]:taken[pi] + c]
            taken[pi] += c
        new = [new[i] for i in rng.permutation(len(new))]
        old = list(earlier)
        for i in (rng.choice(len(old), min(n_perturbed, len(old)), replace=False) if old else []):
            e, lid = old[i]
            moved = dict(e, rel=e["rel"] + np.array([0.4, -0.3, 0.2, 0, 0, 0, 0]))
            old[i] = (moved, lid)
        dup = [new[i] for i in rng.choice(len(new), min(n_duplicates, len(new)), replace=False)]
        sub = old + new + dup
        out.append(([e for e, _ in sub], np.array([i for _, i in sub], np.int64)))
        earlier += new
    return out


# ----------------------------------------------------------------------------------------------------------------
# 3-D / 2-D correspondences of one loop candidate for the PnP stage (SURVEY.md 8f-1, second half)
# ----------------------------------------------------------------------------------------------------------------
def pnp_case(n: int = 200, outlier_frac: float = 0.25, seed: int = 0, noise: float = 0.002, yaw: float = 0.3,
             prior_error: float = 0.15):
    """n landmarks in the NEW drone's odometry frame (matched_3d_now) seen by the OLD camera (matched_2d_norm_old, normalised
    coordinates, K = I): the old drone sits ~1.5 m away with a yaw offset, its camera looks along body +x (extrinsic
    rotation of the usual camera convention).  Returns dict(X [n,3] f32, uv [n,2] f32, inlier [n] bool, pose_true (t,q) with
    x_cam_old = R X + t, prior (t,q) = the truth disturbed by `prior_error` (what odometry would predict), extrinsic,
    drone_pose_now, drone_pose_old)."""
    pa = _PoseAlgebra
    rng = np.random.default_rng(seed + 9000)
    # camera-in-body extrinsic: camera z = body x, camera x = -body y, camera y = -body z
    Rcb = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])

    def quat_from_R(R):
        w = np.sqrt(max(0.0, 1.0 + R[0, 0] + R[1, 1] + R[2, 2])) / 2.0
        return np.array([w, (R[2, 1] - R[1, 2]) / (4 * w), (R[0, 2] - R[2, 0]) / (4 * w), (R[1, 0] - R[0, 1]) / (4 * w)])

    extrinsic = np.concatenate([[0.05, 0.0, 0.03], quat_from_R(Rcb)])
    # everything the PnP sees lives in the NEW drone's odometry (world) frame Wn: its own pose, the landmarks
    # (matched_3d_now) and therefore the solved old-camera pose; the OLD drone reports its pose in its own gravity-aligned
    # frame Wo, which differs from Wn by a yaw and a translation
    drone_pose_now = np.concatenate([[2.0, -1.0, 1.2], _quat_from_rotvec(np.array([0.01, -0.02, 0.7]))])
    d_old_in_new = np.concatenate([[-1.2, 0.6, 0.1], _quat_from_rotvec(np.array([0.0, 0.0, yaw]))])
    old_in_wn = pa.pose_mul(drone_pose_now, d_old_in_new)
    wo_from_wn = np.concatenate([[4.0, 2.5, -0.4], _quat_from_rotvec(np.array([0.0, 0.0, -1.1]))])
    drone_pose_old = pa.pose_mul(wo_from_wn, old_in_wn)
    cam_old_in_new = pa.pose_mul(old_in_wn, extrinsic)                # old camera pose in Wn
    pose_true = pa.pose_inv(cam_old_in_new)                            # x_cam_old = R X + t
    # landmarks in front of the old camera, expressed in Wn
    Pc = np.stack([rng.uniform(-2.5, 2.5, n), rng.uniform(-1.5, 1.5, n), rng.uniform(2.0, 9.0, n)], 1)
    X = np.stack([pa.q_rot(cam_old_in_new[3:], p) + cam_old_in_new[:3] for p in Pc])
    uv = Pc[:, :2] / Pc[:, 2:3] + rng.normal(0, noise, (n, 2))
    inlier = rng.uniform(size=n) >= outlier_frac
    uv[~inlier] = rng.uniform(-1.2, 1.2, ((~inlier).sum(), 2))
    far = np.linalg.norm(uv - Pc[:, :2] / Pc[:, 2:3], axis=1) < 0.2
    inlier = inlier | far                                              # a random "outlier" that happens to fit is an inlier
    prior = pa.pose_mul(np.concatenate([rng.normal(0, prior_error, 3), _quat_from_rotvec(rng.normal(0, prior_error * 0.5, 3))]),
                        pose_true)
    return dict(X=X.astype(np.float32), uv=uv.astype(np.float32), inlier=inlier, pose_true=pose_true, prior=prior,
                extrinsic=extrinsic, drone_pose_now=drone_pose_now, drone_pose_old=drone_pose_old)


# ----------------------------------------------------------------------------------------------------------------
# A four-direction loop candidate with exactly representable geometry (osb_frontend_compute_loop)
# ----------------------------------------------------------------------------------------------------------------
def loop_scene(yaw: float = 0.15, t_new=(0.25, -0.125, 0.0625), depths=(2.0, 4.0, 2.0, 4.0), fx: float = 64.0,
               cx: float = 48.0, cy: float = 32.0):
    """The old drone at the origin of the shared odometry frame, four cameras at its centre looking along body +x rotated
    by 0, 90, 180 and 270 degrees of yaw; direction d sees a fronto-parallel plane at depth depths[d].  The points of a
    direction sit at unit-depth ray (a, b, 1) with a in {+-1/4, +-1/2, +-1} and b a multiple of 1/8, so the old pixels, their
    lift, the rotation into any other direction and the 3-D points are all exact in float32.  The new drone is at
    (t_new, yaw).  Returns dict(K (fx fy cx cy), ext [4,7], pose_old, pose_new, delta_true (x y z, qw qx qy qz: the 4-DoF
    DP_old_to_new), and per direction kp_old [n,2], kp_new [n,2] (pixels, the new camera), X [n,3] (float32))."""
    Rcb = np.array([[0.0, 0.0, 1.0], [-1.0, 0.0, 0.0], [0.0, -1.0, 0.0]])     # camera z = body x, x = -body y, y = -body z
    q_base = np.array([0.5, -0.5, 0.5, -0.5])                                  # the quaternion of Rcb
    pa = _PoseAlgebra
    K = np.array([fx, fx, cx, cy])
    ext, kp_old, kp_new, X = [], [], [], []
    pose_old = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
    pose_new = np.concatenate([np.asarray(t_new, np.float64), _quat_from_rotvec(np.array([0.0, 0.0, yaw]))])
    a_vals = np.array([-1.0, -0.5, -0.25, 0.25, 0.5, 1.0])
    b_vals = np.arange(-6, 7) / 8.0
    for d in range(4):
        qd = pa.q_mul(_quat_from_rotvec(np.array([0.0, 0.0, d * np.pi / 2])), q_base)
        ext.append(np.concatenate([[0.0, 0.0, 0.0], qd]))
        Rz = np.rint(np.array([[np.cos(d * np.pi / 2), -np.sin(d * np.pi / 2), 0], [np.sin(d * np.pi / 2), np.cos(d * np.pi / 2), 0],
                               [0, 0, 1]]))
        R = Rz @ Rcb                                                           # exact: entries 0, +-1
        a, b = np.meshgrid(a_vals, b_vals, indexing="ij")
        ray = np.stack([a.ravel(), b.ravel(), np.ones(a.size)], 1)
        pc = ray * depths[d]
        Xw = pc @ R.T
        X.append(Xw.astype(np.float32))
        kp_old.append(np.stack([fx * ray[:, 0] + cx, fx * ray[:, 1] + cy], 1).astype(np.float32))
        cam_new = pa.pose_mul(pose_new, ext[-1])
        qc = cam_new[3:] * np.array([1.0, -1.0, -1.0, -1.0])
        pn = np.stack([pa.q_rot(qc, x - cam_new[:3]) for x in Xw])
        kp_new.append(np.stack([fx * pn[:, 0] / pn[:, 2] + cx, fx * pn[:, 1] / pn[:, 2] + cy], 1).astype(np.float32))
    delta = pose_new.copy()                                                   # the old drone is the origin
    return dict(K=K, ext=np.array(ext), pose_old=pose_old, pose_new=pose_new, delta_true=delta, kp_old=kp_old, kp_new=kp_new,
                X=X)


# ----------------------------------------------------------------------------------------------------------------
# Inputs of the keyframe front-end: its networks, and keyframe records of loop_scene() built on the host
# ----------------------------------------------------------------------------------------------------------------
def frontend_weights(seed: int = 0):
    """(sp_weights_flat, pca_comp, pca_mean, nv_weights_flat): the first four arguments of host.KeyframeFrontend"""
    comp, mean = pca_matrices(seed)
    return flatten_sp_weights(superpoint_weights(seed)), comp, mean, flatten_nv_weights(netvlad_weights(seed))


LOOP_SCENE = loop_scene()
LOOP_NPT = len(LOOP_SCENE["X"][0])                                  # landmarks per direction
LOOP_G_OLD = descriptor_db(4, 4096, 5)                              # the old keyframe's global descriptor per direction
LOOP_DESC = [local_descriptors(LOOP_NPT, 40 + d) for d in range(4)]  # the old keyframe's local descriptors per direction


def loop_noisy_g(seed: int, sigma: float = 0.05) -> np.ndarray:
    """LOOP_G_OLD with Gaussian noise of norm ~sigma per direction, renormalised"""
    rng = np.random.default_rng(seed)
    g = LOOP_G_OLD + rng.normal(0, sigma / 64, LOOP_G_OLD.shape).astype(np.float32)
    return g / np.linalg.norm(g, axis=1, keepdims=True)


def loop_record(drone: int, msg: int, side: str, seed: int = 0, g: np.ndarray | None = None, n_outliers: int = 4,
                unflag_every: int = 11, few_flags_dir: int | None = None, scramble: bool = False, g_noise: float = 0.0):
    """A four-direction keyframe record (lib.KeyframeRecord) of LOOP_SCENE.  side 'old': the old camera's pixels; 'new':
    the new camera's, points permuted, descriptors noisy, every `unflag_every`-th landmark unflagged and `n_outliers`
    points per direction moved to random pixels / 3-D (their descriptors still match the old point: outlier matches).
    few_flags_dir: only two landmarks of that direction flagged (a failed homography pair); scramble: random 3-D points.
    Global descriptors: g [4][4096] (LOOP_G_OLD if None); with g_noise, a 'new' record adds Gaussian noise of that
    sigma per element, and either side is renormalised."""
    from . import lib
    rng = np.random.default_rng(seed)
    sc, n = LOOP_SCENE, LOOP_NPT
    r = lib.KeyframeRecord()
    r.drone_id, r.msg_id, r.n_dirs = drone, msg, 4
    for d in range(4):
        perm = np.arange(n) if side == "old" else rng.permutation(n)
        kp = (sc["kp_old"][d] if side == "old" else sc["kp_new"][d])[perm].copy()
        X = sc["X"][d][perm].copy()
        desc = LOOP_DESC[d][perm] + (0 if side == "old" else rng.normal(0, 0.02, (n, 64)).astype(np.float32))
        desc /= np.linalg.norm(desc, axis=1, keepdims=True)
        flag = np.ones(n, np.int32)
        if side == "new":
            flag[::unflag_every] = 0
            out = rng.choice(n, n_outliers, replace=False)
            kp[out] = rng.uniform(0, 96, (n_outliers, 2))
            X[out] = rng.normal(0, 3, (n_outliers, 3))
        if few_flags_dir == d:
            flag[:] = 0
            flag[[3, 17]] = 1
        if scramble:
            X = rng.normal(0, 3, X.shape).astype(np.float32)
        gd = LOOP_G_OLD[d] if g is None else g[d]
        if g_noise:
            if side == "new":
                gd = gd + rng.normal(0, g_noise, 4096).astype(np.float32)
            gd = gd / np.linalg.norm(gd)
        r.n_kpts[d] = n
        np.ctypeslib.as_array(r.global_desc[d])[:] = gd
        np.ctypeslib.as_array(r.local_desc[d])[:n] = desc
        np.ctypeslib.as_array(r.kpts[d])[:n] = kp
        np.ctypeslib.as_array(r.landmarks_3d[d])[:n] = X
        np.ctypeslib.as_array(r.landmarks_flag[d])[:n] = flag
        np.ctypeslib.as_array(r.stereo_match[d])[:n] = np.where(flag > 0, 0, -1)
    return r


def anchor_swarm(n_drones: int = 5, n_frames: int = 60, n_meas: int = 400, seed: int = 0, kf_dt_s: float = 0.5,
                 hz: float = 100.0, pre_s: float = 20.0, frac_old: float = 0.05, frac_far: float = 0.1,
                 with_orphans: bool = True):
    """A swarm as find_available_loops_detections sees it before a solve (inputs of host.LoopAnchor and of
    oracle/anchor_ref.anchor).  Drones 0..n_drones-1 fly smooth 3-D curves with yaw and small roll/pitch; each drone's
    odometry (100 Hz, int64 ns stamps from a realistic epoch) is its ground truth in a per-drone odometry frame.  The window
    holds n_frames keyframes kf_dt_s apart: each drone appears with its own stamp jitter, 5 % of its entries are missing,
    5 % have vo_available = 0, and 10 % reuse the previous frame's pose block (a keyframe that did not move).  Measurements
    (loops, Detection4d, Detection6d; loops may be intra-drone) carry noisy true relative poses and correlated covariances at
    off-keyframe stamps, mostly inside the window, `frac_far` of them up to 3 s outside it (dpos rejections) and `frac_old`
    more than 1000 s before it.  With `with_orphans`, drone n_drones has window entries but no odometry and drone
    n_drones + 1 has odometry but no window entry.
    -> dict(trajs {drone: (stamps, poses)}, window (frame_stamps, frame_first, entries), meas, max_drones, prm)"""
    from . import lib as _lib
    rng = np.random.default_rng(seed + 9100)
    NS = 1_000_000_000
    t_epoch = 1_700_000_000 * NS
    pa = _PoseAlgebra
    span = n_frames * kf_dt_s

    def gt(d, t):
        ph = 0.12 * t + 0.9 * d
        pos = np.array([5.0 * np.sin(ph) + 2.0 * d, 5.0 * (1 - np.cos(ph)) - 1.5 * d, 1.0 + 0.5 * np.sin(0.3 * t + d)])
        q = _quat_from_rotvec(np.array([0.04 * np.sin(0.7 * t), 0.03 * np.cos(0.5 * t), 0.3 * t + d]))
        return np.concatenate([pos, q])

    odom_frame = {d: np.concatenate([rng.uniform(-3, 3, 3), _quat_from_rotvec(np.array([0, 0, rng.uniform(-3, 3)]))])
                  for d in range(n_drones + 2)}

    def odom(d, t):
        return pa.pose_mul(odom_frame[d], gt(d, t))

    flying = list(range(n_drones)) + ([n_drones + 1] if with_orphans else [])
    in_window = list(range(n_drones)) + ([n_drones] if with_orphans else [])
    n_samples = int((pre_s + span + 4.0) * hz)
    trajs = {}
    for d in flying:
        k = np.arange(n_samples)
        stamps = t_epoch + (k * (NS / hz)).astype(np.int64) + d * 1000
        trajs[d] = (stamps, np.stack([odom(d, (s - t_epoch) / NS) for s in stamps]))
    t_win = pre_s
    frame_stamps = t_epoch + ((t_win + kf_dt_s * np.arange(n_frames)) * NS).astype(np.int64)
    entries, first, last_block, block = [], [0], {}, 0
    for f in range(n_frames):
        for d in in_window:
            if f > 0 and rng.uniform() < 0.05:
                continue
            st = int(frame_stamps[f]) + int(rng.integers(-3_000_000, 3_000_000))
            if d in last_block and rng.uniform() < 0.1:
                b = last_block[d]
            else:
                b, block = block, block + 1
            last_block[d] = b
            entries.append((d, 0 if rng.uniform() < 0.05 else 1, b, 0, st, odom(d, (st - t_epoch) / NS)))
        first.append(len(entries))
    entries = np.array(entries, dtype=_lib.WINDOW_ENTRY_DTYPE)
    meas = np.zeros(n_meas, _lib.MEASUREMENT_DTYPE)
    ids = list(range(n_drones + (2 if with_orphans else 0)))
    for i in range(n_meas):
        typ = int(rng.integers(0, 3))
        a = int(rng.choice(ids))
        b = a if (typ == 0 and rng.uniform() < 0.2) else int(rng.choice([x for x in ids if x != a]))
        u = rng.uniform()
        if u < frac_old:
            ta = t_win - 1000.0 - rng.uniform(0.001, 50.0)
        elif u < frac_old + frac_far:
            ta = t_win + (span + rng.uniform(0.5, 3.0) if rng.uniform() < 0.5 else -rng.uniform(0.5, 3.0))
        else:
            ta = t_win + rng.uniform(-0.2, span)
        tb = ta if typ != 0 else t_win + rng.uniform(-0.2, span)
        sa, sb = t_epoch + int(ta * NS), t_epoch + int(tb * NS)
        rel = pa.pose_mul(pa.pose_inv(gt(a, ta)), gt(b, tb))
        rel = pa.pose_mul(rel, np.concatenate([rng.normal(0, 0.02, 3), _quat_from_rotvec(rng.normal(0, 0.01, 3))]))
        rel[3:] /= np.linalg.norm(rel[3:])
        L = np.tril(rng.normal(0, 0.004, (6, 6)), -1) + np.diag(rng.uniform(0.02, 0.06, 6))
        meas[i] = (i + (1 << 32), typ, a, b, 0, sa, sb, rel, L @ L.T, odom(a, ta), odom(b, tb))
    prm = dict(begin_min_loop_dt_s=1000.0, det_dpos_thres=1.0, odom_pos_cov_per_m=1e-3, odom_ang_cov_per_m=2e-4, huber=True)
    return dict(trajs=trajs, window=(frame_stamps, np.array(first, np.int32), entries), meas=meas,
                max_drones=n_drones + 2, prm=prm)


def _quat_yaw(q):
    """the yaw of a unit quaternion wxyz (the z angle of its ZYX Euler angles)"""
    w, x, y, z = q
    return np.arctan2(2.0 * (w * z + x * y), 1.0 - 2.0 * (y * y + z * z))


def anchor_window_graph(g: dict) -> dict:
    """The pose graph of an anchor_swarm window, in the layout osb_solver_solve takes: one block per window pose block at
    its entries' self pose (x, y, z, yaw), perturbed except the first, fixed one; an odometry factor (RELPOSE, the
    4-DoF delta) between consecutive blocks of each drone and a UWB distance between the blocks of each frame."""
    stamps, first, entries = g["window"]
    rng = np.random.default_rng(1)
    n = int(entries["block"].max()) + 1
    truth = np.zeros((n, 4))
    for e in entries:
        truth[e["block"]] = np.r_[e["self_pose"][:3], _quat_yaw(e["self_pose"][3:])]
    ftype, ia, ib, payload, huber, last = [], [], [], [], [], {}
    for f in range(len(stamps)):
        fe = entries[first[f]:first[f + 1]]
        for e in fe:
            d, b = int(e["drone_id"]), int(e["block"])
            if d in last and last[d] != b:
                pl = np.zeros(PAYLOAD_LEN)
                pl[:4], pl[4:20] = _delta_pose(truth[last[d]], truth[b]), (np.eye(4) * 50.0).reshape(-1)
                ftype.append(FACTOR_RELPOSE); ia.append(last[d]); ib.append(b); payload.append(pl); huber.append(0)
            last[d] = b
        for i in range(len(fe)):
            for j in range(i + 1, len(fe)):
                if fe[i]["block"] == fe[j]["block"]:
                    continue
                pl = np.zeros(PAYLOAD_LEN)
                pl[0], pl[1] = np.linalg.norm(truth[fe[i]["block"], :3] - truth[fe[j]["block"], :3]), 10.0
                ftype.append(FACTOR_DISTANCE); ia.append(int(fe[i]["block"])); ib.append(int(fe[j]["block"]))
                payload.append(pl); huber.append(1)
    fixed = np.zeros(n, np.uint8)
    fixed[int(entries["block"][0])] = 1
    init = truth + np.c_[rng.normal(0, 0.05, (n, 3)), rng.normal(0, 0.01, n)] * (1 - fixed[:, None])
    return dict(init=init, fixed=fixed, ftype=np.array(ftype, np.int32), ia=np.array(ia, np.int32),
                ib=np.array(ib, np.int32), payload=np.array(payload), huber=np.array(huber, np.uint8))
