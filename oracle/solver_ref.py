"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the swarm_localization
factor graph: residuals, analytic Jacobians, Huber robustification and a direct-solve LM.

Follows /root/reference/swarm_localization/include/swarm_localization/swarm_localization_factors.hpp
(functors) and src/swarm_localization_solver.cpp:1064-1214,1668-1725 (graph assembly, solve).
Ceres and swarm_msgs are absent from /root/reference (un-vendored, unpinned: SURVEY.md section 8c):
  * the sqrt-information matrices S that `LoopEdge::get_sqrt_information_4d()` would return are INPUTS;
  * the solve is a "Ceres stand-in": Levenberg-Marquardt on the normal equations with a sparse direct
    solver (scipy SuperLU), Huber(1.0) as Ceres' corrector does it when rho''<=0 (residual and
    Jacobian scaled by sqrt(rho')), run to tight convergence.  Parity is on CONVERGED POSES
    (SURVEY.md section 8 item 4), not on iterates.  parity unpinned: no Ceres output exists to check.
The Jacobians are pinned against central finite differences in tests/test_oracle_pins.py.

Flat graph layout (same arrays as include/omniswarm_b200.h::osb_graph_solve):
  poses [n,4] f64 (x,y,z,yaw);  fixed [n] u8;  ftype/ia/ib [m] i32;  huber [m] u8;  payload [m,24] f64
  payload DISTANCE : [d, sqrt_inf]
          RELPOSE  : [meas x,y,z,yaw, S row-major 16]
          DETECTION: [dir 3, B0 3, B1 3, inv_dep, flags(bit0 depth, bit1 dpose), ext_z, dposea 4,
                      dposeb 4, sphere_std, inv_dep_std]
"""
from __future__ import annotations

import math
import numpy as np

FACTOR_DISTANCE, FACTOR_RELPOSE, FACTOR_DETECTION = 0, 1, 2
TWO_PI = 2.0 * math.pi


def normalize_angle(a):
    """factors.hpp:34-40"""
    return a - TWO_PI * np.floor((a + math.pi) / TWO_PI)


def factor_residual_jacobian(ftype: int, pa: np.ndarray, pb: np.ndarray, pl: np.ndarray):
    """-> (r [nr], Ja [nr,4], Jb [nr,4]) for one factor, un-robustified."""
    if ftype == FACTOR_DISTANCE:                       # factors.hpp:203-224
        d = pa[:3] - pb[:3]
        nrm = math.sqrt(float(d @ d))
        r = np.array([(nrm - pl[0]) * pl[1]])
        Ja = np.zeros((1, 4)); Jb = np.zeros((1, 4))
        Ja[0, :3] = pl[1] * d / nrm
        Jb[0, :3] = -pl[1] * d / nrm
        return r, Ja, Jb
    if ftype == FACTOR_RELPOSE:                        # factors.hpp:226-271, DeltaPose :139-149
        c, s = math.cos(pa[3]), math.sin(pa[3])
        d = pb[:3] - pa[:3]
        est = np.array([c * d[0] + s * d[1], -s * d[0] + c * d[1], d[2], normalize_angle(pb[3] - pa[3])])
        e = pl[0:4] - est                              # pose_error_4d :52-61: err = meas - est
        e[3] = normalize_angle(e[3])
        S = pl[4:20].reshape(4, 4)
        r = S @ e
        dEa = np.zeros((4, 4)); dEb = np.zeros((4, 4))  # d est / d pose
        R = np.array([[c, s, 0], [-s, c, 0], [0, 0, 1.0]])
        dEb[:3, :3] = R
        dEa[:3, :3] = -R
        dEa[0, 3] = -s * d[0] + c * d[1]
        dEa[1, 3] = -c * d[0] - s * d[1]
        dEa[3, 3] = -1.0
        dEb[3, 3] = 1.0
        return r, -S @ dEa, -S @ dEb
    if ftype == FACTOR_DETECTION:                      # factors.hpp:273-367
        dirv, B = pl[0:3], pl[3:9].reshape(2, 3)
        inv_dep, flags, ext_z = pl[9], int(pl[10]), pl[11]
        dpa, dpb = pl[12:16], pl[16:20]
        sphere_std, invdep_std = pl[20], pl[21]
        # primed poses and their Jacobians wrt the raw poses
        Ga = np.eye(4); Gb = np.eye(4)
        if flags & 2:                                  # PoseMulti (:165-172)
            def mul(p, q):
                c, s = math.cos(p[3]), math.sin(p[3])
                out = np.array([p[0] + c * q[0] - s * q[1], p[1] + s * q[0] + c * q[1], p[2] + q[2],
                                normalize_angle(p[3] + q[3])])
                G = np.eye(4)
                G[0, 3] = -s * q[0] - c * q[1]
                G[1, 3] = c * q[0] - s * q[1]
                return out, G
            A, Ga = mul(pa, dpa)
            Bp, Gb = mul(pb, dpb)
        else:                                          # :319-321
            A = pa.copy(); A[2] += ext_z
            Bp = pb
        c, s = math.cos(A[3]), math.sin(A[3])
        d = Bp[:3] - A[:3]
        rel = np.array([c * d[0] + s * d[1], -s * d[0] + c * d[1], d[2]])   # DeltaPose_Naive :153-160
        R = np.array([[c, s, 0], [-s, c, 0], [0, 0, 1.0]])
        dRelA = np.zeros((3, 4)); dRelB = np.zeros((3, 4))
        dRelA[:, :3] = -R; dRelB[:, :3] = R
        dRelA[0, 3] = -s * d[0] + c * d[1]
        dRelA[1, 3] = -c * d[0] - s * d[1]
        rho = 1.0 / math.sqrt(float(rel @ rel))
        u = rel * rho - dirv                           # unit_position_error :73-103
        dU = rho * (np.eye(3) - np.outer(rel, rel) * rho * rho)
        nr = 3 if (flags & 1) else 2
        r = np.zeros(nr); Jrel = np.zeros((nr, 3))
        r[0:2] = (B @ u) / sphere_std
        Jrel[0:2] = (B @ dU) / sphere_std
        if flags & 1:
            r[2] = (inv_dep - rho) / invdep_std        # :97
            Jrel[2] = (rho ** 3) * rel / invdep_std
        return r, Jrel @ dRelA @ Ga, Jrel @ dRelB @ Gb
    raise ValueError(ftype)


def huber_scale(sq_norm: float, delta: float = 1.0):
    """sqrt(rho'(s)) for ceres::HuberLoss(delta): rho(s)=s (s<=d^2), 2 d sqrt(s) - d^2 otherwise."""
    if sq_norm <= delta * delta:
        return 1.0
    return math.sqrt(delta / math.sqrt(sq_norm))


def huber_rho(sq_norm: float, delta: float = 1.0):
    if sq_norm <= delta * delta:
        return sq_norm
    return 2.0 * delta * math.sqrt(sq_norm) - delta * delta


def evaluate(g: dict, poses: np.ndarray, want_jac: bool = True):
    """-> cost, list of (a, b, r_rob [nr], Ja_rob, Jb_rob)."""
    cost = 0.0
    out = []
    for f in range(len(g["ftype"])):
        a, b = int(g["ia"][f]), int(g["ib"][f])
        r, Ja, Jb = factor_residual_jacobian(int(g["ftype"][f]), poses[a], poses[b], g["payload"][f])
        s = float(r @ r)
        if g["huber"][f]:
            cost += 0.5 * huber_rho(s)
            w = huber_scale(s)
            r, Ja, Jb = r * w, Ja * w, Jb * w
        else:
            cost += 0.5 * s
        if want_jac:
            out.append((a, b, r, Ja, Jb))
    return cost, out


def cost_only(g: dict, poses: np.ndarray) -> float:
    return evaluate(g, poses, want_jac=False)[0]


def num_residuals(g: dict) -> int:
    n = 0
    for f in range(len(g["ftype"])):
        t = int(g["ftype"][f])
        n += 1 if t == FACTOR_DISTANCE else 4 if t == FACTOR_RELPOSE else (3 if int(g["payload"][f][10]) & 1 else 2)
    return n


def _spd_solve(A, b):
    """Sparse direct solve of the SPD normal equations (stand-in for Ceres' SPARSE_NORMAL_CHOLESKY,
    solver.cpp:1698): SuperLU in symmetric mode with a minimum-degree ordering on A^T + A."""
    import scipy.sparse.linalg as spla
    return spla.splu(A, permc_spec="MMD_AT_PLUS_A", diag_pivot_thresh=0.0, options=dict(SymmetricMode=True)).solve(b)


def solve(g: dict, max_iters: int = 200, function_tol: float = 1e-14, gradient_tol: float = 1e-11,
          param_tol: float = 1e-12, verbose: bool = False):
    """Levenberg-Marquardt (Ceres-style step control) with a sparse direct solve.

    -> dict(poses, final_cost, initial_cost, iterations).  Constant blocks: fixed[n]==1
    (solver.cpp:1196-1199).
    """
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla

    x = g["init"].astype(np.float64).copy()
    n = x.shape[0]
    free = np.nonzero(g["fixed"] == 0)[0]
    col_of = -np.ones(n, np.int64); col_of[free] = np.arange(len(free))
    nv = 4 * len(free)
    radius = 1e4
    decrease = 2.0
    cost, lin = evaluate(g, x)
    initial_cost = cost
    it = 0
    for it in range(1, max_iters + 1):
        rows, cols, vals = [], [], []
        rr = []
        ro = 0
        for (a, b, r, Ja, Jb) in lin:
            nr = len(r)
            for node, J in ((a, Ja), (b, Jb)):
                cidx = col_of[node]
                if cidx < 0:
                    continue
                for i in range(nr):
                    for j in range(4):
                        rows.append(ro + i); cols.append(4 * cidx + j); vals.append(J[i, j])
            rr.append(r); ro += nr
        rvec = np.concatenate(rr)
        J = sp.csr_matrix((vals, (rows, cols)), shape=(ro, nv))
        grad = J.T @ rvec
        if np.max(np.abs(grad)) < gradient_tol:
            break
        H = (J.T @ J).tocsc()
        diag = np.clip(H.diagonal(), 1e-6, 1e32)
        while True:
            A = H + sp.diags(diag / radius)
            delta = _spd_solve(A.tocsc(), -grad)
            xn = x.copy()
            xn[free] += delta.reshape(-1, 4)
            new_cost = cost_only(g, xn)
            model = -(grad @ delta) - 0.5 * (delta @ (H @ delta))
            rho = (cost - new_cost) / model if model > 0 else -1.0
            if rho > 1e-3:
                radius = min(radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3), 1e16)
                decrease = 2.0
                break
            radius /= decrease
            decrease *= 2.0
            if radius < 1e-32:
                break
        if radius < 1e-32:
            break
        step_norm = np.linalg.norm(delta)
        dcost = cost - new_cost
        x = xn
        cost, lin = evaluate(g, x)
        if verbose:
            print(f"it {it} cost {cost:.12e} d {dcost:.3e} |step| {step_norm:.3e} radius {radius:.3e}")
        if abs(dcost) < function_tol * cost or step_norm < param_tol * (np.linalg.norm(x[free]) + param_tol):
            break
    return dict(poses=x, final_cost=cost, initial_cost=initial_cost, iterations=it,
                n_residuals=num_residuals(g))


def equv_cost(final_cost: float, n_residuals: int, window_size: int) -> float:
    """solve_once return value (solver.cpp:1721-1725)."""
    return math.sqrt(final_cost) / n_residuals / window_size


def create_cov6d_sqrt_inf(cov6: np.ndarray) -> np.ndarray:
    """RelativePoseFactor4d::CreateCov6d (factors.hpp:255-263): S = sqrt(|inv(cov4)|) element-wise."""
    cov4 = np.zeros((4, 4))
    cov4[:3, :3] = cov6[:3, :3]
    cov4[3, 3] = cov6[5, 5]
    return np.sqrt(np.abs(np.linalg.inv(cov4)))


# --------------------------------------------------------------------------------------------------------------
# Vectorised evaluation (same arithmetic as factor_residual_jacobian, batched with numpy) so that the CPU
# baseline of bench.py is a fair "Ceres stand-in" rather than a Python-loop artefact.  DETECTION factors (rare)
# fall back to the scalar routine.  tests/test_oracle_pins.py checks it against the scalar path.
# --------------------------------------------------------------------------------------------------------------
def evaluate_vec(g: dict, x: np.ndarray, want_jac: bool = True):
    """-> cost, r [m,4], Ja [m,4,4], Jb [m,4,4] (robustified, rows beyond the factor's residual count zero)."""
    ft, ia, ib, pl = g["ftype"], g["ia"], g["ib"], g["payload"]
    m = len(ft)
    r = np.zeros((m, 4)); Ja = np.zeros((m, 4, 4)); Jb = np.zeros((m, 4, 4))
    pa, pb = x[ia], x[ib]
    d_idx = np.nonzero(ft == FACTOR_DISTANCE)[0]
    if len(d_idx):
        d = pa[d_idx, :3] - pb[d_idx, :3]
        nrm = np.sqrt((d * d).sum(1))
        si = pl[d_idx, 1]
        r[d_idx, 0] = (nrm - pl[d_idx, 0]) * si
        if want_jac:
            Ja[d_idx, 0, :3] = d * (si / nrm)[:, None]
            Jb[d_idx, 0, :3] = -d * (si / nrm)[:, None]
    p_idx = np.nonzero(ft == FACTOR_RELPOSE)[0]
    if len(p_idx):
        A, B, P = pa[p_idx], pb[p_idx], pl[p_idx]
        c, s = np.cos(A[:, 3]), np.sin(A[:, 3])
        d = B[:, :3] - A[:, :3]
        est = np.stack([c * d[:, 0] + s * d[:, 1], -s * d[:, 0] + c * d[:, 1], d[:, 2],
                        normalize_angle(B[:, 3] - A[:, 3])], 1)
        e = P[:, 0:4] - est
        e[:, 3] = normalize_angle(e[:, 3])
        S = P[:, 4:20].reshape(-1, 4, 4)
        r[p_idx] = np.einsum("nij,nj->ni", S, e)
        if want_jac:
            n = len(p_idx)
            Ea = np.zeros((n, 4, 4)); Eb = np.zeros((n, 4, 4))
            Eb[:, 0, 0] = c; Eb[:, 0, 1] = s; Eb[:, 1, 0] = -s; Eb[:, 1, 1] = c; Eb[:, 2, 2] = 1; Eb[:, 3, 3] = 1
            Ea[:, :3, :3] = -Eb[:, :3, :3]
            Ea[:, 0, 3] = -s * d[:, 0] + c * d[:, 1]
            Ea[:, 1, 3] = -c * d[:, 0] - s * d[:, 1]
            Ea[:, 3, 3] = -1
            Ja[p_idx] = -np.einsum("nij,njk->nik", S, Ea)
            Jb[p_idx] = -np.einsum("nij,njk->nik", S, Eb)
    for f in np.nonzero(ft == FACTOR_DETECTION)[0]:
        rr, ja, jb = factor_residual_jacobian(FACTOR_DETECTION, pa[f], pb[f], pl[f])
        r[f, :len(rr)] = rr; Ja[f, :len(rr)] = ja; Jb[f, :len(rr)] = jb
    s2 = (r * r).sum(1)
    hub = (g["huber"] != 0) & (s2 > 1.0)
    cost = 0.5 * s2[~hub].sum() + 0.5 * (2.0 * np.sqrt(s2[hub]) - 1.0).sum()
    w = np.ones(m); w[hub] = 1.0 / np.sqrt(np.sqrt(s2[hub]))
    r = r * w[:, None]
    if want_jac:
        Ja *= w[:, None, None]; Jb *= w[:, None, None]
    return cost, r, Ja, Jb


def _jacobian_layout(g: dict):
    """-> (free [nf] node ids, col_of [n] (-1: fixed), masks ma / mb [m,4,4] of the free blocks, rows R and columns C of
    their entries in the [4m, 4 nf] Jacobian: factor f owns rows 4f..4f+3, free node i columns 4 col_of[i]..+3)"""
    n, m = len(g["fixed"]), len(g["ftype"])
    free = np.nonzero(g["fixed"] == 0)[0]
    col_of = -np.ones(n, np.int64); col_of[free] = np.arange(len(free))
    ia, ib = g["ia"], g["ib"]
    rows = (np.arange(m)[:, None, None] * 4 + np.arange(4)[None, :, None]) + np.zeros((1, 1, 4), np.int64)
    ca = (col_of[ia][:, None, None] * 4 + np.arange(4)[None, None, :]) + np.zeros((1, 4, 1), np.int64)
    cb = (col_of[ib][:, None, None] * 4 + np.arange(4)[None, None, :]) + np.zeros((1, 4, 1), np.int64)
    ma = np.broadcast_to((col_of[ia] >= 0)[:, None, None], (m, 4, 4))
    mb = np.broadcast_to((col_of[ib] >= 0)[:, None, None], (m, 4, 4))
    return free, col_of, ma, mb, np.concatenate([rows[ma], rows[mb]]), np.concatenate([ca[ma], cb[mb]])


def lm_system(g: dict, x: np.ndarray, radius: float) -> dict:
    """The LM step's linear system at poses x, as solve_fast builds it: robustified J (sparse [4m, 4 nf], factor f in
    rows 4f..4f+3), H = J^T J, grad = J^T r, D = diag(H) clipped to [1e-6, 1e32], the free-node map and the cost.
    The step solves (H + diag(D) / radius) delta = -grad; delta[4 col_of[i] + k] moves component k of free node i."""
    import scipy.sparse as sp
    free, col_of, ma, mb, R, Cc = _jacobian_layout(g)
    m = len(g["ftype"])
    cost, r, Ja, Jb = evaluate_vec(g, np.asarray(x, np.float64))
    J = sp.csr_matrix((np.concatenate([Ja[ma], Jb[mb]]), (R, Cc)), shape=(4 * m, 4 * len(free)))
    H = (J.T @ J).tocsc()
    return dict(J=J, H=H, grad=J.T @ r.reshape(-1), D=np.clip(H.diagonal(), 1e-6, 1e32), radius=float(radius),
                free=free, col_of=col_of, cost=cost)


def lm_step(sysm: dict) -> np.ndarray:
    """the exact step of an lm_system: (H + diag(D) / radius)^-1 (-grad), by the sparse direct solve solve_fast uses"""
    import scipy.sparse as sp
    return _spd_solve((sysm["H"] + sp.diags(sysm["D"] / sysm["radius"])).tocsc(), -sysm["grad"])


def solve_fast(g: dict, max_iters: int = 200, function_tol: float = 1e-6, gradient_tol: float = 1e-10,
               param_tol: float = 1e-8, num_threads: int | None = None):
    """Same LM as solve(), vectorised; default tolerances = Ceres defaults (the configuration the reference runs,
    solver.cpp:1695-1706)."""
    import scipy.sparse as sp
    import scipy.sparse.linalg as spla
    x = g["init"].astype(np.float64).copy()
    m = len(g["ftype"])
    free, col_of, ma, mb, R, Cc = _jacobian_layout(g)
    nv = 4 * len(free)
    radius, decrease = 1e4, 2.0
    cost, r, Ja, Jb = evaluate_vec(g, x)
    initial_cost = cost
    it = 0
    for it in range(1, max_iters + 1):
        J = sp.csr_matrix((np.concatenate([Ja[ma], Jb[mb]]), (R, Cc)), shape=(4 * m, nv))
        rv = r.reshape(-1)
        grad = J.T @ rv
        if np.max(np.abs(grad)) < gradient_tol:
            break
        H = (J.T @ J).tocsc()
        diag = np.clip(H.diagonal(), 1e-6, 1e32)
        ok = False
        while radius > 1e-32:
            delta = _spd_solve((H + sp.diags(diag / radius)).tocsc(), -grad)
            xn = x.copy(); xn[free] += delta.reshape(-1, 4)
            new_cost = evaluate_vec(g, xn, want_jac=False)[0]
            model = -(grad @ delta) - 0.5 * (delta @ (H @ delta))
            rho = (cost - new_cost) / model if model > 0 else -1.0
            if rho > 1e-3:
                radius = min(radius / max(1.0 / 3.0, 1.0 - (2.0 * rho - 1.0) ** 3), 1e16); decrease = 2.0
                ok = True
                break
            radius /= decrease; decrease *= 2.0
        if not ok:
            break
        dcost, step = cost - new_cost, np.linalg.norm(delta)
        x = xn
        old = cost
        cost, r, Ja, Jb = evaluate_vec(g, x)
        if abs(dcost) < function_tol * old or step < param_tol * (np.linalg.norm(x[free]) + param_tol):
            break
    return dict(poses=x, final_cost=cost, initial_cost=initial_cost, iterations=it, n_residuals=num_residuals(g))
