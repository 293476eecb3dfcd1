"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the PCM outlier rejection that runs immediately
upstream of the pose-graph solve (SURVEY.md section 8f-2).

Follows (paths relative to /root/reference):
  * SwarmLocalOutlierRejection::OutlierRejectionLoopEdgesPCM
      swarm_localization/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:173-297 -- pairwise consistency of the
      loop edges of one drone pair: err = odom_a * p_edge2 * odom_b^-1 * p_edge1^-1 (:227), 6-D log map (:228), squared
      Mahalanobis distance against cov_1 + cov_2 + cov(odom_a) + cov(odom_b) (:193,212,224,229), edge in the consistency
      graph iff smd < pcm_thres (:231-235); edge1 is the LATER-inserted loop of the pair (:180,190);
  * FMC::maxCliqueHeu (Josh Mangelson's variant that returns the clique)
      swarm_localization/src/swarm_outlier_rejection/third_party/fast_max-clique_finder/src/findCliqueHeu.cpp:120-244
      -- restated literally, prunings 1/3/5 and the "last element of S" choice (:185) included; PINNED against the
      reference's own library compiled from these very sources (oracle/fmc_ref.py, oracle/_ref/libfmc_ref.so):
      tests/test_oracle_pins.py::test_max_clique_restatement_equals_the_references_own_library.

Third-party arithmetic that is ABSENT from the reference tree (HKUST-Swarm/swarm_msgs, un-vendored, no commit pinned):
`Swarm::Pose` composition / inverse / `log_map`, `LoopEdge::get_covariance`, `computeSquaredMahalanobisDistance` and
`DroneTrajectory::get_relative_pose_by_ts`.  They are DEFINED here (parity unpinned at that boundary, as for the factors):
  * Pose = (t, unit quaternion wxyz); a*b = (t_a + R_a t_b, q_a q_b); inverse = (-R^T t, q*);
  * log_map(T) = [t ; rotation vector of q]  (6-vector, translation first -- the order of get_covariance's blocks);
  * smd(v, C) = v^T C^-1 v;
  * the covariances and the ego-motion poses are INPUTS: every loop edge carries its 6x6 covariance, the ego-motion
    (odometry-frame) pose of both drones at its two stamps and the accumulated trajectory length there; the odometry
    between two stamps of a drone is pose(ts1)^-1 * pose(ts2) with covariance |len(ts2) - len(ts1)| * diag(pos_cov_per_m x3,
    ang_cov_per_m x3) -- the per-metre model of the simulator's labels (swarm_local_sim.cpp:532-550).
"""
from __future__ import annotations

import os

import numpy as np


# ---- Swarm::Pose algebra (defined here; swarm_msgs is not in the tree) ----------------------------------------
def q_mul(a, b):
    aw, ax, ay, az = a; bw, bx, by, bz = b
    return np.array([aw * bw - ax * bx - ay * by - az * bz,
                     aw * bx + ax * bw + ay * bz - az * by,
                     aw * by - ax * bz + ay * bw + az * bx,
                     aw * bz + ax * by - ay * bx + az * bw])


def q_conj(q):
    return np.array([q[0], -q[1], -q[2], -q[3]])


def q_rot(q, v):
    """R(q) v, expanded (no matrix): v + 2 w (u x v) + 2 u x (u x v)"""
    u = q[1:]
    c = np.cross(u, v)
    return v + 2.0 * (q[0] * c + np.cross(u, c))


def pose_mul(a, b):
    return np.concatenate([a[:3] + q_rot(a[3:], b[:3]), q_mul(a[3:], b[3:])])


def pose_inv(a):
    qc = q_conj(a[3:])
    return np.concatenate([-q_rot(qc, a[:3]), qc])


def log_map(p):
    """[translation ; rotation vector]"""
    q = p[3:]
    if q[0] < 0:
        q = -q
    n = np.sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    if n < 1e-12:
        rv = 2.0 * q[1:]
    else:
        rv = (2.0 * np.arctan2(n, q[0]) / n) * q[1:]
    return np.concatenate([p[:3], rv])


def cholesky_smd(v, C):
    """v^T C^-1 v through an unpivoted Cholesky factorisation, the arithmetic the kernel performs"""
    n = len(v)
    L = np.zeros((n, n))
    for j in range(n):
        s = C[j, j] - np.dot(L[j, :j], L[j, :j])
        if not s > 0:
            return np.inf
        L[j, j] = np.sqrt(s)
        for i in range(j + 1, n):
            L[i, j] = (C[i, j] - np.dot(L[i, :j], L[j, :j])) / L[j, j]
    y = np.zeros(n)
    for i in range(n):
        y[i] = (v[i] - np.dot(L[i, :i], y[:i])) / L[i, i]
    return float(np.dot(y, y))


def same_robot_pair(e1, e2):
    """LoopEdge::same_robot_pair: 1 same orientation, 2 swapped, 0 another pair"""
    if e1["id_a"] == e2["id_a"] and e1["id_b"] == e2["id_b"]:
        return 1
    if e1["id_a"] == e2["id_b"] and e1["id_b"] == e2["id_a"]:
        return 2
    return 0


def pair_smd(e1, e2, pos_cov_per_m, ang_cov_per_m):
    """squared Mahalanobis consistency error of (edge1 = later loop, edge2 = earlier loop), or None for another pair
    (swarm_outlier_rejection.cpp:190-229)"""
    srp = same_robot_pair(e1, e2)
    if srp == 0:
        return None
    if srp == 1:                                                   # :200-212
        p2 = e2["rel"]
        a2, la2, b2, lb2 = e2["odom_a"], e2["len_a"], e2["odom_b"], e2["len_b"]
    else:                                                          # :214-224 edge2 runs b -> a
        p2 = pose_inv(e2["rel"])
        a2, la2, b2, lb2 = e2["odom_b"], e2["len_b"], e2["odom_a"], e2["len_a"]
    odom_a = pose_mul(pose_inv(e1["odom_a"]), a2)                  # drone id_a: ts_a(edge1) -> its stamp on edge2
    odom_b = pose_mul(pose_inv(e1["odom_b"]), b2)
    da, db = abs(la2 - e1["len_a"]), abs(lb2 - e1["len_b"])
    C = e1["cov"] + e2["cov"] + np.diag([pos_cov_per_m] * 3 + [ang_cov_per_m] * 3) * (da + db)
    err = pose_mul(pose_mul(pose_mul(odom_a, p2), pose_inv(odom_b)), pose_inv(e1["rel"]))          # :227
    return cholesky_smd(log_map(err), C)


def consistency_matrix(edges, pcm_thres, pos_cov_per_m, ang_cov_per_m):
    """adj [n,n] uint8, symmetric, zero diagonal: 1 iff smd < pcm_thres (:231-235); smd [n,n] (inf where undefined)"""
    n = len(edges)
    adj = np.zeros((n, n), np.uint8)
    smd = np.full((n, n), np.inf)
    for i in range(n):
        for j in range(i):
            s = pair_smd(edges[i], edges[j], pos_cov_per_m, ang_cov_per_m)     # edge1 = the later one
            if s is None:
                continue
            smd[i, j] = smd[j, i] = s
            if s < pcm_thres:
                adj[i, j] = adj[j, i] = 1
    return adj, smd


def max_clique_heu(adj):
    """FMC::maxCliqueHeu (findCliqueHeu.cpp:120-244) on the adjacency matrix; neighbour lists ascending (the order in which
    OutlierRejectionLoopEdgesPCM fills pcm_graph).  -> (clique vertex list in the reference's order, maxClq)"""
    n = adj.shape[0]
    nbr = [np.nonzero(adj[v])[0].tolist() for v in range(n)]
    deg = [len(x) for x in nbr]
    max_clq, best = -1, []
    for v in range(n):
        if max_clq > deg[v]:                                        # pruning 1 (:149)
            continue
        S = [v] + [u for u in nbr[v] if max_clq <= deg[u]]          # :156-165 pruning 3
        inter = [v]                                                 # :174
        icc = 0
        while S:                                                    # :176
            icc += 1
            imdv = S[-1]                                            # :185
            row = adj[imdv]
            S1 = [u for u in S if row[u] and max_clq <= deg[u]]     # :190-203 pruning 5
            if S1:
                inter.append(imdv)                                  # :218-221
            S = S1
        if max_clq < icc:                                           # :236-239
            max_clq, best = icc, inter
    return best, max_clq


def pcm(edges, pcm_thres, pos_cov_per_m, ang_cov_per_m):
    """-> (indices of the loops kept (good_loops_set, :291-296), adjacency, clique size)"""
    adj, _ = consistency_matrix(edges, pcm_thres, pos_cov_per_m, ang_cov_per_m)
    clique, size = max_clique_heu(adj)
    return clique, adj, size


def max_clique_exact(adj):
    """brute force, for pinning the heuristic on small graphs"""
    n = adj.shape[0]
    best = 0
    for mask in range(1 << n):
        vs = [i for i in range(n) if mask >> i & 1]
        if len(vs) <= best:
            continue
        if all(adj[a, b] for k, a in enumerate(vs) for b in vs[k + 1:]):
            best = len(vs)
    return best


# ---- the same arithmetic over arrays of pairs (a full 4096 x 4096 matrix, not a sample) ------------------------------
# A pose is a tuple of 7 arrays (tx ty tz qw qx qy qz); every expression is the scalar one above, term for term.
def _cross_v(a, b):
    return (a[1] * b[2] - a[2] * b[1], a[2] * b[0] - a[0] * b[2], a[0] * b[1] - a[1] * b[0])


def _q_mul_v(a, b):
    aw, ax, ay, az = a
    bw, bx, by, bz = b
    return (aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
            aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw)


def _q_rot_v(q, v):
    u = q[1:]
    c = _cross_v(u, v)
    d = _cross_v(u, c)
    return tuple(v[k] + 2.0 * (q[0] * c[k] + d[k]) for k in range(3))


def _pose_mul_v(a, b):
    r = _q_rot_v(a[3:], b[:3])
    return tuple(a[k] + r[k] for k in range(3)) + _q_mul_v(a[3:], b[3:])


def _pose_inv_v(a):
    qc = (a[3], -a[4], -a[5], -a[6])
    r = _q_rot_v(qc, a[:3])
    return (-r[0], -r[1], -r[2]) + qc


def _log_map_v(p):
    neg = p[3] < 0
    q = tuple(np.where(neg, -x, x) for x in p[3:])
    n = np.sqrt(q[1] * q[1] + q[2] * q[2] + q[3] * q[3])
    with np.errstate(divide="ignore", invalid="ignore"):
        k = np.where(n < 1e-12, 2.0, 2.0 * np.arctan2(n, q[0]) / n)
    return p[:3] + (k * q[1], k * q[2], k * q[3])


def edge_arrays(edges):
    """edge dicts -> dict of arrays (ids [n], rel / odom_a / odom_b [n, 7], cov [n, 6, 6], len_a / len_b [n])"""
    return dict(id_a=np.array([e["id_a"] for e in edges], np.int64), id_b=np.array([e["id_b"] for e in edges], np.int64),
                rel=np.array([e["rel"] for e in edges], np.float64).reshape(-1, 7),
                cov=np.array([np.asarray(e["cov"], np.float64).reshape(6, 6) for e in edges]).reshape(-1, 6, 6),
                odom_a=np.array([e["odom_a"] for e in edges], np.float64).reshape(-1, 7),
                odom_b=np.array([e["odom_b"] for e in edges], np.float64).reshape(-1, 7),
                len_a=np.array([e["len_a"] for e in edges], np.float64),
                len_b=np.array([e["len_b"] for e in edges], np.float64))


def pair_smd_batched(E, I, J, pos_cov_per_m, ang_cov_per_m, terms=False):
    """pair_smd(edges[I[k]], edges[J[k]]) for every k (edge1 = I, the later loop), E = edge_arrays(edges): +inf for
    another drone pair or a C that is not positive definite.  The same operations in the same order as pair_smd and
    cholesky_smd, each one elementwise numpy operation.  With terms, also the quantities a forward-error bound of the
    pair needs (tests/pcm_edges_ref.py)."""
    ia, ib, ja, jb = E["id_a"][I], E["id_b"][I], E["id_a"][J], E["id_b"][J]
    srp = np.where((ia == ja) & (ib == jb), 1, np.where((ia == jb) & (ib == ja), 2, 0))
    two = srp == 2
    pose = lambda a, idx: tuple(a[idx, k] for k in range(7))                      # noqa: E731
    rel2 = pose(E["rel"], J)
    inv2 = _pose_inv_v(rel2)
    p2 = tuple(np.where(two, x, y) for x, y in zip(inv2, rel2))
    oa2, ob2 = pose(E["odom_a"], J), pose(E["odom_b"], J)
    a2 = tuple(np.where(two, x, y) for x, y in zip(ob2, oa2))
    b2 = tuple(np.where(two, x, y) for x, y in zip(oa2, ob2))
    la2 = np.where(two, E["len_b"][J], E["len_a"][J])
    lb2 = np.where(two, E["len_a"][J], E["len_b"][J])
    oa1, ob1, rel1 = pose(E["odom_a"], I), pose(E["odom_b"], I), pose(E["rel"], I)
    odom_a = _pose_mul_v(_pose_inv_v(oa1), a2)
    odom_b = _pose_mul_v(_pose_inv_v(ob1), b2)
    dl = np.abs(la2 - E["len_a"][I]) + np.abs(lb2 - E["len_b"][I])
    err = _pose_mul_v(_pose_mul_v(_pose_mul_v(odom_a, p2), _pose_inv_v(odom_b)), _pose_inv_v(rel1))
    v = _log_map_v(err)
    covI, covJ = E["cov"].reshape(-1, 36)[I], E["cov"].reshape(-1, 36)[J]
    per_m = [pos_cov_per_m] * 3 + [ang_cov_per_m] * 3
    C = [[covI[:, 6 * i + j] + covJ[:, 6 * i + j] + (np.diag(per_m)[i, j] * dl if i == j else 0.0) for j in range(6)]
         for i in range(6)]
    ok = srp > 0
    L = [[None] * 6 for _ in range(6)]
    y = [None] * 6
    with np.errstate(invalid="ignore", divide="ignore"):
        for j in range(6):
            s = C[j][j]
            for k in range(j):
                s = s - L[j][k] * L[j][k]
            ok &= s > 0
            L[j][j] = np.sqrt(np.where(ok, s, 1.0))
            for i in range(j + 1, 6):
                c = C[i][j]
                for k in range(j):
                    c = c - L[i][k] * L[j][k]
                L[i][j] = c / L[j][j]
        smd = 0.0
        for i in range(6):
            c = v[i]
            for k in range(i):
                c = c - L[i][k] * y[k]
            y[i] = c / L[i][i]
            smd = smd + y[i] * y[i]
    smd = np.where(ok, smd, np.inf)
    if not terms:
        return smd
    tn = lambda p: np.sqrt(p[0] * p[0] + p[1] * p[1] + p[2] * p[2])                   # noqa: E731
    return smd, dict(T=tn(oa1) + tn(ob1) + tn(rel1) + tn(a2) + tn(b2) + tn(p2),
                     Lsum=np.abs(E["len_a"][I]) + np.abs(E["len_b"][I]) + np.abs(la2) + np.abs(lb2), dl=dl,
                     covF=np.linalg.norm(covI, axis=1) + np.linalg.norm(covJ, axis=1),
                     C=np.stack([np.stack(np.broadcast_arrays(*row), -1) for row in C], -2),
                     rv=np.sqrt(v[3] * v[3] + v[4] * v[4] + v[5] * v[5]), srp=srp)


def consistency_matrix_batched(edges, pcm_thres, pos_cov_per_m, ang_cov_per_m, pairs_per_chunk=1 << 18, workers=None):
    """consistency_matrix over arrays, a chunk of rows at a time (chunks on `workers` threads: numpy releases the GIL in
    its elementwise loops): the same adjacency and smd matrices"""
    from concurrent.futures import ThreadPoolExecutor
    n = len(edges)
    E = edge_arrays(edges)
    adj = np.zeros((n, n), np.uint8)
    smd = np.full((n, n), np.inf)
    chunks, i0 = [], 1
    while i0 < n:
        i1 = i0 + 1
        while i1 < n and (i1 * (i1 - 1) - i0 * (i0 - 1)) // 2 < pairs_per_chunk:
            i1 += 1
        chunks.append((i0, i1))
        i0 = i1

    def run(c):
        i0, i1 = c
        I, J = np.nonzero(np.tril(np.ones((i1 - i0, i1), bool), i0 - 1))
        I += i0
        s = pair_smd_batched(E, I, J, pos_cov_per_m, ang_cov_per_m)
        smd[I, J] = s
        smd[J, I] = s
        a = (s < pcm_thres).astype(np.uint8)
        adj[I, J] = a
        adj[J, I] = a

    with ThreadPoolExecutor(workers or min(16, os.cpu_count() or 1)) as ex:
        list(ex.map(run, chunks))
    return adj, smd
