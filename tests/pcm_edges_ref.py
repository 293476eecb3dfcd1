"""Test infrastructure for the PCM edge tests (tests/test_pcm_ref_edges.py on the CPU, tests/test_gpu_pcm_edges.py on the
device): a 50-digit statement of the pair error, a forward-error bound for any float64 evaluation of it, the seeded case
families and graph families both files use, and defective variants of the float64 pair error and of maxCliqueHeu that the
CPU tests show the checks can tell apart.

pair_smd_mp(e1, e2) is oracle/pcm_ref.pair_smd (swarm_outlier_rejection.cpp:190-229) computed with mpmath at 50 digits
from the exact float64 inputs, with v^T C^-1 v by an LU solve (mpmath.lu_solve, partial pivoting): it shares no rounding
with the Cholesky form the kernel and the float64 oracle use.

The bound.  Let u = 2^-53.  A float64 evaluation differs from the exact smd through
  * v (the 6-D log map of err): the translation part is a sum of rotated translations, so its error is at most
    K_T u T with T the sum of the norms of the six translations that enter (both loops' relative poses and odometry);
    the error quaternion's components are off by at most K_Q u after its five products, and the log map's rotation vector
    moves by at most (2 pi + 4) per unit of quaternion error (theta / sin(theta / 2) <= pi for w >= 0) plus 16 u |rv| of
    its own rounding;  ||dv|| <= K_T u T + (2 pi + 4) K_Q u + 16 u |rv|;
  * C: forming it rounds each entry (2 u |cov_1 + cov_2| and 3 u of the odometry term, whose dl is itself off by
    3 u (|len| sum)), and the unpivoted Cholesky solve is backward stable, (C + dC) y = v with
    ||dC|| <= 2 (n + 1) n u ||C|| = 84 u ||C|| (Higham, Thm 10.4, n = 6);  eps_C = the sum of those;
  * smd = v^T C^-1 v then moves by  smd r / (1 - r), r = ||C^-1|| eps_C   (the kappa(C) term),
    and by 2 sqrt(smd) ||L^-1|| ||dv|| + ||L^-1||^2 ||dv||^2, ||L^-1||^2 = ||C^-1||   (the 2 sqrt(smd) ||L^-1|| ||dv|| term),
    plus 8 u smd for the final sum of squares.
  bound = 2 x their sum (the factor 2 covers the second-order terms the first-order propagation drops).
It holds for any order of the operations and with or without fused multiply-adds, so it needs no model of the device's
instruction selection.  Where the error quaternion's |w| is within K_Q u of 0 the log map's sign flip (w < 0) is not
determined by the inputs: either branch (+theta u or -theta u, theta ~ pi) is a correct float64 result, so the reference
returns both branches' smd and a value within the bound of either passes.
"""
from __future__ import annotations

import math

import mpmath
import numpy as np

from oracle import pcm_ref as pr

U = 2.0 ** -53
K_T, K_Q = 512.0, 64.0
DPS = 50


# ---- the bound ------------------------------------------------------------------------------------------------------
def bound(smd, T, Lsum, dl, covF, C_norm, Cinv_norm, rv, per_m):
    """the forward-error bound of a float64 pair error (module docstring); arrays or scalars; +inf where C is too close to
    singular for the bound to hold (r >= 1/2)"""
    smd = np.abs(np.asarray(smd, np.float64))
    dv = K_T * U * T + (2 * math.pi + 4) * K_Q * U + 16 * U * rv
    eps_C = 84 * U * C_norm + 2 * U * covF + math.sqrt(6) * per_m * (3 * U * dl + 3 * U * Lsum)
    r = Cinv_norm * eps_C
    with np.errstate(invalid="ignore", divide="ignore", over="ignore"):
        d_C = np.where(r < 0.5, smd * r / (1 - r), np.inf)
        d_v = 2 * np.sqrt(smd) * np.sqrt(Cinv_norm) * dv + Cinv_norm * dv * dv
    return 2 * (d_C + d_v + 8 * U * smd)


def norms(C):
    """(||C||_2, ||C^-1||_2, lambda_min) of symmetric 6x6 matrices [..., 6, 6]"""
    lam = np.linalg.eigvalsh(C)
    with np.errstate(divide="ignore"):
        return np.abs(lam).max(-1), np.where(lam[..., 0] > 0, 1.0 / lam[..., 0], np.inf), lam[..., 0]


def batched_bound(E, I, J, pos, ang):
    """(float64 smd, bound) of the pairs (I[k], J[k]) of E = pcm_ref.edge_arrays(edges), I the later loop"""
    s, t = pr.pair_smd_batched(E, I, J, pos, ang, terms=True)
    fin = np.isfinite(s)
    cn, ci = np.full(len(I), np.nan), np.full(len(I), np.inf)
    if fin.any():                                                  # Frobenius norms: upper bounds of the 2-norms
        Cf = t["C"][fin]
        cn[fin] = np.sqrt((Cf * Cf).sum((1, 2)))
        Ci = np.linalg.inv(Cf)
        ci[fin] = np.sqrt((Ci * Ci).sum((1, 2)))
    b = np.full(len(I), np.nan)
    b[fin] = bound(s[fin], t["T"][fin], t["Lsum"][fin], t["dl"][fin], t["covF"][fin], cn[fin], ci[fin], t["rv"][fin],
                   max(pos, ang))
    return s, b


# ---- the 50-digit pair error --------------------------------------------------------------------------------------------
def _mp(x):
    return [mpmath.mpf(float(a)) for a in np.asarray(x, np.float64).reshape(-1)]


def _qmul(a, b):
    aw, ax, ay, az = a; bw, bx, by, bz = b
    return [aw * bw - ax * bx - ay * by - az * bz, aw * bx + ax * bw + ay * bz - az * by,
            aw * by - ax * bz + ay * bw + az * bx, aw * bz + ax * by - ay * bx + az * bw]


def _qrot(q, v):
    u = q[1:]
    c = [u[1] * v[2] - u[2] * v[1], u[2] * v[0] - u[0] * v[2], u[0] * v[1] - u[1] * v[0]]
    d = [u[1] * c[2] - u[2] * c[1], u[2] * c[0] - u[0] * c[2], u[0] * c[1] - u[1] * c[0]]
    return [v[k] + 2 * (q[0] * c[k] + d[k]) for k in range(3)]


def _pmul(a, b):
    r = _qrot(a[3:], b[:3])
    return [a[k] + r[k] for k in range(3)] + _qmul(a[3:], b[3:])


def _pinv(a):
    qc = [a[3], -a[4], -a[5], -a[6]]
    return [-x for x in _qrot(qc, a[:3])] + qc


def _rv(q, sign):
    w, x, y, z = [sign * c for c in q]
    n = mpmath.sqrt(x * x + y * y + z * z)
    k = mpmath.mpf(2) if n < mpmath.mpf("1e-12") else 2 * mpmath.atan2(n, w) / n
    return [k * x, k * y, k * z]


def pair_smd_mp(e1, e2, pos, ang):
    """-> (values, bound): the exact pair error rounded to float64, one value, or two when the log map's branch is not
    determined (|w| <= K_Q u); [inf] for another drone pair or a C that is not positive definite, [nan] when a pose or C
    is not finite; bound as the module docstring derives it (nan where the value is not finite)"""
    srp = pr.same_robot_pair(e1, e2)
    if srp == 0:
        return [math.inf], math.nan
    if not (np.isfinite(np.asarray(e1["cov"], np.float64)).all() and np.isfinite(np.asarray(e2["cov"], np.float64)).all()):
        return [math.inf], math.nan                                # C is not positive definite
    poses = [e1["odom_a"], e1["odom_b"], e1["rel"], e2["odom_a"], e2["odom_b"], e2["rel"]]
    finite_v = all(np.isfinite(np.asarray(x, np.float64)).all() for x in poses)
    with mpmath.workdps(DPS):
        rel2 = _mp(np.nan_to_num(e2["rel"]))
        if srp == 1:
            p2, a2, b2, la2, lb2 = rel2, _mp(np.nan_to_num(e2["odom_a"])), _mp(np.nan_to_num(e2["odom_b"])), e2["len_a"], \
                e2["len_b"]
        else:
            p2, a2, b2, la2, lb2 = _pinv(rel2), _mp(np.nan_to_num(e2["odom_b"])), _mp(np.nan_to_num(e2["odom_a"])), \
                e2["len_b"], e2["len_a"]
        oa1, ob1, rel1 = (_mp(np.nan_to_num(e1[k])) for k in ("odom_a", "odom_b", "rel"))
        odom_a = _pmul(_pinv(oa1), a2)
        odom_b = _pmul(_pinv(ob1), b2)
        dl = abs(mpmath.mpf(la2) - mpmath.mpf(e1["len_a"])) + abs(mpmath.mpf(lb2) - mpmath.mpf(e1["len_b"]))
        per_m = [pos] * 3 + [ang] * 3
        c1, c2 = _mp(e1["cov"]), _mp(e2["cov"])
        C = mpmath.matrix(6, 6)
        for i in range(6):
            for j in range(6):
                C[i, j] = c1[6 * i + j] + c2[6 * i + j] + (dl * mpmath.mpf(per_m[i]) if i == j else 0)
        Cf = np.array([[float(C[i, j]) for j in range(6)] for i in range(6)])
        C_norm, Cinv_norm, lam_min = norms(Cf)
        try:                                                       # positive definite, decided at 50 digits
            mpmath.cholesky(C)
        except ValueError:
            return [math.inf], math.nan
        if not finite_v:
            return [math.nan], math.nan
        err = _pmul(_pmul(_pmul(odom_a, p2), _pinv(odom_b)), _pinv(rel1))
        w = err[3]
        signs = [-1 if w < 0 else 1]
        if abs(w) <= K_Q * U:                                      # the flip is rounding-decided: both branches
            signs = [1, -1]
        vals, rvn = [], 0.0
        for sg in signs:
            v = err[:3] + _rv(err[3:], sg)
            x = mpmath.lu_solve(C, mpmath.matrix(v))
            vals.append(float(sum(v[k] * x[k] for k in range(6))))
            rvn = max(rvn, float(mpmath.sqrt(sum(c * c for c in v[3:]))))
        tn = lambda p: float(mpmath.sqrt(p[0] ** 2 + p[1] ** 2 + p[2] ** 2))        # noqa: E731
        T = sum(tn(p) for p in (oa1, ob1, rel1, a2, b2, p2))
        Lsum = abs(e1["len_a"]) + abs(e1["len_b"]) + abs(la2) + abs(lb2)
        covF = float(np.linalg.norm(np.asarray(e1["cov"], np.float64))) + float(np.linalg.norm(np.asarray(e2["cov"])))
        b = max(float(bound(s, T, Lsum, float(dl), covF, C_norm, Cinv_norm, rvn, max(pos, ang))) for s in vals)
    return vals, b


def within(dev, vals, b):
    """a device value agrees with the reference: both finite and within the bound of one branch, or both non-finite"""
    if not math.isfinite(vals[0]):
        return not math.isfinite(dev)
    return math.isfinite(dev) and min(abs(dev - v) for v in vals) <= b


def _mp_rows(args):
    edges, pos, ang, rows = args
    return [(i, j, *pair_smd_mp(edges[i], edges[j], pos, ang)) for i, j in rows]


def mp_matrix(edges, pos, ang, pairs=None, procs=None):
    """pair_smd_mp of every pair (i > j) or of `pairs`, on a process pool -> {(i, j): (values, bound)}"""
    import os
    from multiprocessing import get_context
    if pairs is None:
        pairs = list(zip(*all_pairs(len(edges))))
    procs = procs or min(16, os.cpu_count() or 1)
    chunks = [pairs[k::procs * 4] for k in range(procs * 4)]
    with get_context("fork").Pool(procs) as pool:
        out = pool.map(_mp_rows, [(edges, pos, ang, c) for c in chunks if c])
    return {(int(i), int(j)): (v, b) for part in out for i, j, v, b in part}


# ---- defects of the float64 pair error (each must be caught by the bound) ---------------------------------------------
DEFECTS = ["offdiag_dropped", "cov2_omitted", "signed_dl", "srp2_lengths_not_swapped", "srp2_rel_not_inverted",
           "no_w_flip", "chol_LiLi"]


def pair_smd_defect(e1, e2, pos, ang, defect):
    """oracle/pcm_ref.pair_smd with one defect built in"""
    srp = pr.same_robot_pair(e1, e2)
    if srp == 0:
        return math.inf
    if srp == 1:
        p2, a2, la2, b2, lb2 = e2["rel"], e2["odom_a"], e2["len_a"], e2["odom_b"], e2["len_b"]
    else:
        p2 = e2["rel"] if defect == "srp2_rel_not_inverted" else pr.pose_inv(e2["rel"])
        a2, la2, b2, lb2 = e2["odom_b"], e2["len_b"], e2["odom_a"], e2["len_a"]
        if defect == "srp2_lengths_not_swapped":
            la2, lb2 = e2["len_a"], e2["len_b"]
    odom_a = pr.pose_mul(pr.pose_inv(e1["odom_a"]), a2)
    odom_b = pr.pose_mul(pr.pose_inv(e1["odom_b"]), b2)
    if defect == "signed_dl":
        dl = (la2 - e1["len_a"]) + (lb2 - e1["len_b"])
    else:
        dl = abs(la2 - e1["len_a"]) + abs(lb2 - e1["len_b"])
    C = np.asarray(e1["cov"], np.float64) + (0.0 if defect == "cov2_omitted" else np.asarray(e2["cov"], np.float64))
    C = C + np.diag([pos] * 3 + [ang] * 3) * dl
    if defect == "offdiag_dropped":
        C = np.diag(np.diag(C))
    err = pr.pose_mul(pr.pose_mul(pr.pose_mul(odom_a, p2), pr.pose_inv(odom_b)), pr.pose_inv(e1["rel"]))
    v = pr.log_map(err)
    if defect == "no_w_flip":
        q = err[3:]
        n = np.sqrt(q[1] ** 2 + q[2] ** 2 + q[3] ** 2)
        v = np.concatenate([err[:3], (2.0 if n < 1e-12 else 2.0 * np.arctan2(n, q[0]) / n) * q[1:]])
    L = np.zeros((6, 6))
    for j in range(6):
        s = C[j, j] - np.dot(L[j, :j], L[j, :j])
        if not s > 0:
            return math.inf
        L[j, j] = np.sqrt(s)
        for i in range(j + 1, 6):
            L[i, j] = (C[i, j] - np.dot(L[i, :j], L[i if defect == "chol_LiLi" else j, :j])) / L[j, j]
    y = np.zeros(6)
    for i in range(6):
        y[i] = (v[i] - np.dot(L[i, :i], y[:i])) / L[i, i]
    return float(np.dot(y, y))


# ---- seeded edge families ------------------------------------------------------------------------------------------------
def _qrv(rv):
    a = float(np.linalg.norm(rv))
    if a < 1e-300:
        return np.array([1.0, 0.0, 0.0, 0.0])
    return np.concatenate([[math.cos(a / 2)], math.sin(a / 2) * np.asarray(rv) / a])


def _unit(rng):
    x = rng.normal(size=3)
    return x / np.linalg.norm(x)


def _pose(rng, tscale, ang=math.pi):
    return np.concatenate([rng.normal(size=3) * tscale, _qrv(_unit(rng) * rng.uniform(0, ang))])


def _corr_cov(rng, kappa, scale):
    """L L^T with every translation-rotation entry coupled and condition number kappa"""
    Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
    lam = scale * np.geomspace(1.0, 1.0 / kappa, 6)
    C = (Q * lam) @ Q.T
    return 0.5 * (C + C.T)


OTHER_AT = (0, 31, 32, 33, 63, 64)              # insertion positions of the other pair's loops: inf on word boundaries


def _interleave(main, other):
    """insertion order with the other pair's loops at OTHER_AT (those below the total count)"""
    out, mi, oi = [], 0, 0
    while mi < len(main) or oi < len(other):
        if oi < len(other) and (len(out) in OTHER_AT or mi == len(main)):
            out.append(other[oi]); oi += 1
        else:
            out.append(main[mi]); mi += 1
    return out


def _loop(rng, ida, idb, tscale, cov, noise_cov=None, lens=(0.0, 0.0), flip=False, gross=False):
    """one loop edge between drones on random trajectories: true relative pose x noise drawn from noise_cov (or gross)"""
    oa, ob = _pose(rng, tscale), _pose(rng, tscale)
    rel = pr.pose_mul(pr.pose_inv(oa), ob)
    nc = cov if noise_cov is None else noise_cov
    if gross:
        d = np.concatenate([rng.uniform(-3, 3, 3) * max(tscale, 1e-3), _qrv(rng.uniform(-0.8, 0.8, 3))])
    else:
        x = np.linalg.cholesky(0.5 * (nc + nc.T) + 1e-300 * np.eye(6)) @ rng.normal(size=6) * 0.6
        d = np.concatenate([x[:3], _qrv(x[3:])])
    rel = pr.pose_mul(rel, d)
    rel[3:] /= np.linalg.norm(rel[3:])
    e = dict(id_a=ida, id_b=idb, rel=rel, cov=np.array(cov), odom_a=oa, odom_b=ob, len_a=float(lens[0]),
             len_b=float(lens[1]))
    if flip:
        e = dict(id_a=idb, id_b=ida, rel=pr.pose_inv(rel), cov=e["cov"], odom_a=ob, odom_b=oa, len_a=e["len_b"],
                 len_b=e["len_a"])
    return e


def _theta_loops(rng, cov):
    """loops whose error rotation against the first is exactly theta: odometry identity, rel = (t, q_theta)"""
    ident = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])
    out = []
    axis = _unit(rng)
    for th in [0.0, 1e-13, 1e-11, 1e-3, 1.0, math.pi - 1e-3, math.pi - 1e-8]:
        out.append(np.concatenate([rng.normal(size=3) * 0.05, _qrv(axis * th) if th > 0 else [1.0, 0, 0, 0]]))
    out.append(np.concatenate([rng.normal(size=3) * 0.05, [0.0], axis]))            # theta = pi, w = +0
    out.append(np.concatenate([rng.normal(size=3) * 0.05, [-0.0], axis]))           # theta = pi, w = -0
    out.append(np.concatenate([rng.normal(size=3) * 0.05, [-0.0], -axis]))
    edges = [dict(id_a=1, id_b=2, rel=ident.copy(), cov=cov, odom_a=ident.copy(), odom_b=ident.copy(), len_a=0.0,
                  len_b=0.0)]
    for r in out:
        edges.append(dict(id_a=1, id_b=2, rel=r, cov=cov, odom_a=ident.copy(), odom_b=ident.copy(), len_a=0.0, len_b=0.0))
    return edges


def family(name, seed):
    """-> (edges in insertion order, pos_cov_per_m, ang_cov_per_m) of the case family `name`"""
    rng = np.random.default_rng(seed)
    pos, ang = 1e-4, 1e-5
    other = [_loop(rng, 1, 7, 5.0, np.diag([1e-3] * 3 + [1e-4] * 3)) for _ in range(6)]
    main = []
    if name == "correlated":                     # L L^T, kappa 1 .. 1e8, translation-rotation coupling
        for k in range(40):
            cov = _corr_cov(rng, 10.0 ** rng.uniform(0, 8), 10.0 ** rng.uniform(-4, -1))
            main.append(_loop(rng, 1, 2, 5.0, cov, lens=rng.uniform(0, 50, 2), flip=k % 3 == 0, gross=k % 5 == 4))
    elif name == "anisotropic":                  # diagonals from 1e-8 to 1e2
        for k in range(40):
            cov = np.diag(10.0 ** rng.uniform(-8, 2, 6))
            main.append(_loop(rng, 1, 2, 5.0, cov, lens=rng.uniform(0, 50, 2), flip=k % 3 == 1, gross=k % 6 == 5))
    elif name == "odometry":                     # dl = 0 exactly, dl ~ 1e4 m
        for k in range(40):
            cov = _corr_cov(rng, 10.0 ** rng.uniform(0, 4), 1e-3)
            lens = (100.0, 250.0) if k < 20 else rng.uniform(0, 2e4, 2)
            main.append(_loop(rng, 1, 2, 5.0, cov, lens=lens, flip=k % 4 == 1, gross=k % 7 == 6))
    elif name == "odometry_zero_per_m":          # zero per-metre covariances
        pos, ang = 0.0, 0.0
        for k in range(40):
            cov = _corr_cov(rng, 10.0 ** rng.uniform(0, 4), 1e-3)
            main.append(_loop(rng, 1, 2, 5.0, cov, lens=rng.uniform(0, 2e4, 2), flip=k % 4 == 1, gross=k % 7 == 6))
    elif name == "theta":                        # exact error rotations around the log map's branches
        cov = _corr_cov(rng, 1e3, 1e-2)
        main = _theta_loops(rng, cov)
    elif name == "negated_q":                    # quaternions stored as -q
        for k in range(40):
            cov = _corr_cov(rng, 10.0 ** rng.uniform(0, 5), 10.0 ** rng.uniform(-3, -1))
            e = _loop(rng, 1, 2, 5.0, cov, lens=rng.uniform(0, 50, 2), flip=k % 3 == 0, gross=k % 5 == 4)
            for key, bit in (("rel", 1), ("odom_a", 2), ("odom_b", 4)):
                if (k + 1) & bit:
                    e[key] = np.concatenate([e[key][:3], -e[key][3:]])
            main.append(e)
    elif name == "translation":                  # translations 1e-9 m .. 1e4 m
        for k in range(40):
            ts = 10.0 ** rng.uniform(-9, 4)
            cov = _corr_cov(rng, 10.0 ** rng.uniform(0, 4), max(ts, 1e-6) ** 2 * 1e-2)
            cov[3:, 3:] += np.eye(3) * 1e-4
            main.append(_loop(rng, 1, 2, ts, cov, lens=rng.uniform(0, 50, 2), flip=k % 3 == 0, gross=k % 6 == 5))
    elif name == "srp":                          # srp 1 and 2, intra-drone pairs, reversed pairs
        for k in range(24):
            cov = _corr_cov(rng, 10.0 ** rng.uniform(0, 4), 10.0 ** rng.uniform(-3, -1))
            main.append(_loop(rng, 1, 2, 5.0, cov, lens=rng.uniform(0, 500, 2), flip=k % 2 == 1, gross=k % 6 == 5))
        for k in range(16):
            cov = _corr_cov(rng, 10.0 ** rng.uniform(0, 4), 10.0 ** rng.uniform(-3, -1))
            main.append(_loop(rng, 3, 3, 5.0, cov, lens=rng.uniform(0, 500, 2), gross=k % 6 == 5))
        main = [main[i] for i in rng.permutation(len(main))]
    elif name == "not_finite":                   # C zero, indefinite or NaN; NaN / inf in a pose
        pos, ang = 0.0, 0.0
        for k in range(30):
            cov = _corr_cov(rng, 10.0 ** rng.uniform(0, 3), 1e-2)
            main.append(_loop(rng, 1, 2, 5.0, cov, lens=rng.uniform(0, 50, 2), flip=k % 3 == 0))
        main[3]["cov"] = np.zeros((6, 6)); main[4]["cov"] = np.zeros((6, 6))
        main[5]["cov"] = -main[6]["cov"]                          # C of (6, 5) = 0; of (5, x) indefinite
        main[7]["cov"] = np.diag([1.0, 1.0, -3.0, 1.0, 1.0, 1.0]) * 1e-2
        main[8]["cov"] = main[8]["cov"].copy(); main[8]["cov"][2, 4] = main[8]["cov"][4, 2] = np.nan
        main[9]["rel"] = main[9]["rel"].copy(); main[9]["rel"][1] = np.nan
        main[10]["odom_a"] = main[10]["odom_a"].copy(); main[10]["odom_a"][0] = np.inf
        main[11]["odom_b"] = main[11]["odom_b"].copy(); main[11]["odom_b"][5] = np.nan
        main[12]["rel"] = main[12]["rel"].copy(); main[12]["rel"][3] = -np.inf
    else:
        raise KeyError(name)
    return _interleave(main, other), pos, ang


FAMILIES = ["correlated", "anisotropic", "odometry", "odometry_zero_per_m", "theta", "negated_q", "translation", "srp",
            "not_finite"]


def all_pairs(n):
    """(I, J) of every i > j, row by row"""
    I, J = np.tril_indices(n, -1)
    return I, J


def choose_threshold(smd, b, want=15.0):
    """a threshold near `want` farther than 2 x bound from every finite float64 smd (so it is farther than the bound from
    every exact one): the midpoint of the widest such gap among the values next to `want`"""
    fin = np.isfinite(smd)
    s, bb = smd[fin], np.nan_to_num(b[fin], nan=0.0)
    lo, hi = s - 2 * bb - 1e-300, s + 2 * bb + 1e-300
    order = np.argsort(s)
    lo, hi = lo[order], np.maximum.accumulate(hi[order])
    k = np.searchsorted(lo, want)
    best, thres = -1.0, None
    for a in range(max(k - 64, 0), min(k + 64, len(lo)) + 1):
        left = hi[a - 1] if a > 0 else want - 1.0
        right = lo[a] if a < len(lo) else want + 1.0
        if right - left > best:
            best, thres = right - left, 0.5 * (left + right)
    assert best > 0, "no threshold clears every pair"
    return float(thres)


# ---- maxCliqueHeu over boolean rows (fast enough at n = 4096), with defects --------------------------------------------
CLIQUE_DEFECTS = ["pruning_lt", "imdv_first", "tie_later"]


def max_clique_heu_rows(adj, defect=None):
    """oracle/pcm_ref.max_clique_heu on numpy boolean rows -> (clique, maxClq).  S = [v, ascending members] is a mask
    holding v; its last element is the largest member other than v, or v when there is none (the kernel's choice)"""
    adj = np.asarray(adj).astype(bool)
    n = adj.shape[0]
    deg = adj.sum(1)
    max_clq, best = -1, []
    for v in range(n):
        if max_clq > deg[v]:                                        # pruning 1
            continue
        dm = (deg > max_clq) if defect == "pruning_lt" else (max_clq <= deg)        # prunings 3 and 5
        S = adj[v] & dm
        S[v] = True
        inter, icc = [v], 0
        while True:
            icc += 1
            if defect == "imdv_first":                               # S[0] instead of S[-1]
                imdv = v if S[v] else int(np.argmax(S))
            else:
                S[v], had_v = False, S[v]
                nz = np.flatnonzero(S)
                S[v] = had_v
                imdv = int(nz[-1]) if len(nz) else v
            S = S & adj[imdv] & dm
            if not S.any():
                break
            inter.append(imdv)
        if (max_clq <= icc) if defect == "tie_later" else (max_clq < icc):
            max_clq, best = icc, inter
    return best, max_clq


def graph_families():
    """-> list of (name, adjacency uint8 [n, n]) regenerated from fixed seeds: the clique graphs of §3"""
    rng = np.random.default_rng(20261019)
    out = [("empty_1", np.zeros((1, 1), np.uint8)), ("empty_40", np.zeros((40, 40), np.uint8))]
    for n in (1, 32, 33, 1280, 1281, 4096):
        out.append((f"complete_{n}", (1 - np.eye(n, dtype=np.uint8))))
    for n, k, sz in ((60, 3, 6), (200, 4, 9), (1300, 5, 33)):       # disjoint equal cliques: the first one wins
        a = np.zeros((n, n), np.uint8)
        perm = rng.permutation(n)
        for c in range(k):
            idx = perm[c * sz:(c + 1) * sz]
            a[np.ix_(idx, idx)] = 1
        np.fill_diagonal(a, 0)
        out.append((f"equal_cliques_{n}", a))
    a = np.zeros((4096, 4096), np.uint8)                             # a clique across words and lanes
    idx = np.array([31, 32, 63, 64, 1023, 1024, 4095])
    a[np.ix_(idx, idx)] = 1
    r = np.triu(rng.uniform(size=(4096, 4096)) < 0.001, 1)
    a |= (r | r.T).astype(np.uint8)
    np.fill_diagonal(a, 0)
    out.append(("clique_on_word_edges", a))
    n = 70                                                           # candidates larger than all their neighbours
    a = np.zeros((n, n), np.uint8)
    for v in range(40, 70, 3):
        nb = rng.choice(40, 5, replace=False)
        a[v, nb] = a[nb, v] = 1
    for i in range(8):
        for j in range(i + 1, 8):
            a[i, j] = a[j, i] = 1
    out.append(("largest_last", a))
    for p in (1, 3, 5):                                              # degrees exactly maxClq at each pruning
        n = 80
        a = np.zeros((n, n), np.uint8)
        K = 6
        a[:K, :K] = 1                                                # clique {0..5}: maxClq = 6 after v = 0
        if p == 1:                                                   # later v of degree 6 (= maxClq): not skipped
            for v in range(20, 80, 7):
                nb = list(range(v + 1, min(v + 7, n)))
                a[v, nb] = a[nb, v] = 1
        elif p == 3:                                                 # neighbours of degree exactly 6 stay in S
            hub = 30
            for u in range(31, 40):
                a[hub, u] = a[u, hub] = 1
                for w in range(41 + 6 * (u - 31), 41 + 6 * (u - 31) + 5):
                    if w < n:
                        a[u, w] = a[w, u] = 1
        else:                                                        # members of degree 6 kept by pruning 5
            grp = list(range(40, 47))
            a[np.ix_(grp, grp)] = 1
            for u in grp[:3]:
                a[u, 60] = a[60, u] = 1
        np.fill_diagonal(a, 0)
        out.append((f"degree_eq_maxclq_p{p}", a))
    for n in (33, 1025):                                             # stars and paths
        a = np.zeros((n, n), np.uint8)
        a[0, 1:] = a[1:, 0] = 1
        out.append((f"star_{n}", a))
        b = np.zeros((n, n), np.uint8)
        i = np.arange(n - 1)
        b[i, i + 1] = b[i + 1, i] = 1
        out.append((f"path_{n}", b))
    for n in (1025, 2049, 3073, 4096):                               # G(n, p), sparse to dense
        for p in (0.002, 0.05, 0.5, 0.95):
            r = np.triu(rng.uniform(size=(n, n)) < p, 1)
            out.append((f"gnp_{n}_{p}", (r | r.T).astype(np.uint8)))
    for s in range(2):                                               # PCM-shaped: a consistent block plus false links
        n = 4096
        a = np.zeros((n, n), bool)
        idx = rng.choice(n, int(rng.uniform(0.08, 0.12) * n), replace=False)
        a[np.ix_(idx, idx)] = True
        a |= rng.uniform(size=(n, n)) < 0.02
        a = np.triu(a, 1)
        out.append((f"pcm_shaped_{s}", (a | a.T).astype(np.uint8)))
    return out


def pack_bits(adj, stride=None):
    """adjacency [n, n] -> uint32 rows [n, stride] (bit j % 32 of word j / 32), stride >= ceil(n / 32)"""
    n = adj.shape[0]
    stride = stride or (n + 31) // 32
    padded = np.zeros((n, stride * 32), np.uint8)
    padded[:, :n] = adj
    return np.packbits(padded, axis=1, bitorder="little").view("<u4").astype(np.uint32)


# ---- the launch-shape list and its reference ------------------------------------------------------------------------------
SHAPES = [1, 2, 31, 32, 33, 63, 64, 65, 127, 128, 129, 1025, 1279, 1280, 1281, 2049, 3073, 4064, 4065, 4095, 4096]
SHAPE_POS, SHAPE_ANG = 1e-4, 1e-5


def shape_edges(seed=9):
    """4096 loops (another pair's among them) with correlated covariances: every shape is a prefix, so its consistency
    matrix is the top-left block of the 4096 one"""
    from omniswarm_b200 import synth
    edges = synth.pcm_edges(4096 - 64, 0.85, seed, other_pair=64)
    rng = np.random.default_rng(seed)
    for e in edges:                                                # couple translation and rotation (correlation <= 0.3)
        d = np.sqrt(np.diag(e["cov"]))
        Q, _ = np.linalg.qr(rng.normal(size=(6, 6)))
        R = np.eye(6) + 0.3 * (Q @ np.diag(rng.uniform(-1, 1, 6)) @ Q.T - np.diag(np.diag(Q @ np.diag(rng.uniform(-1, 1, 6)) @ Q.T)))
        R = 0.5 * (R + R.T)
        if np.linalg.eigvalsh(R)[0] <= 0.1:
            R = np.eye(6)
        e["cov"] = d[:, None] * R * d[None, :]
    return edges


def bound_matrix(edges, pos, ang, pairs_per_chunk=1 << 17, workers=None):
    """float64 smd [n, n] and its bound [n, n] (nan where the smd is not finite), chunks of rows on threads"""
    import os
    from concurrent.futures import ThreadPoolExecutor
    n = len(edges)
    E = pr.edge_arrays(edges)
    smd, bnd = np.full((n, n), np.inf), np.full((n, n), np.nan)
    chunks, i0 = [], 1
    while i0 < n:
        i1 = i0 + 1
        while i1 < n and (i1 * (i1 - 1) - i0 * (i0 - 1)) // 2 < pairs_per_chunk:
            i1 += 1
        chunks.append((i0, i1))
        i0 = i1

    def run(c):
        I, J = np.nonzero(np.tril(np.ones((c[1] - c[0], c[1]), bool), c[0] - 1))
        I += c[0]
        s, b = batched_bound(E, I, J, pos, ang)
        smd[I, J] = smd[J, I] = s
        bnd[I, J] = bnd[J, I] = b

    with ThreadPoolExecutor(workers or min(16, os.cpu_count() or 1)) as ex:
        list(ex.map(run, chunks))
    return smd, bnd
