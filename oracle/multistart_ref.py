"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the random-restart initialisation of
swarm_localization: solve_with_multiple_init (src/swarm_localization_solver.cpp:781-845) with random_init_pose
(:204-216).

The reference draws with rand(); the library (osb_solver_solve_multistart) draws with a counter hash so that a trial's
start depends only on (seed, trial, caller's node id, component).  This module restates that hash in numpy uint64,
and the reference's acceptance walk over the trials' equv_costs (oracle/solver_ref.py: equv_cost).
"""
from __future__ import annotations

import numpy as np


def _splitmix64(z: np.ndarray) -> np.ndarray:
    with np.errstate(over="ignore"):
        z = z + np.uint64(0x9E3779B97F4A7C15)
        z = (z ^ (z >> np.uint64(30))) * np.uint64(0xBF58476D1CE4E5B9)
        z = (z ^ (z >> np.uint64(27))) * np.uint64(0x94D049BB133111EB)
    return z ^ (z >> np.uint64(31))


def multistart_draw(seed: int, trial, node, comp, r: float) -> np.ndarray:
    """value in [-r, r) for (seed, trial, caller node id, component 0/1/2 = x/y/z); exact restatement of the kernel
    (2r * u rounded, then + (-r) rounded: no fused multiply-add)."""
    trial, node, comp = (np.asarray(v, np.uint64) for v in (trial, node, comp))
    key = (trial << np.uint64(34)) | (node << np.uint64(2)) | comp
    u = (_splitmix64(np.uint64(seed) ^ _splitmix64(key)) >> np.uint64(11)).astype(np.float64) * 2.0 ** -53
    return (2.0 * r) * u + (-r)


def multistart_initial_poses(base: np.ndarray, mask: np.ndarray, fixed: np.ndarray, n_trials: int, seed: int,
                             rand_xy: float = 5.0, rand_z: float = 1.0) -> np.ndarray:
    """[n_trials, n, 4] starting poses: random_init_pose on every masked node that is not fixed (x, y in +-rand_xy,
    z in +-rand_z, yaw kept), the base pose elsewhere."""
    base = np.asarray(base, np.float64)
    out = np.repeat(base[None], n_trials, axis=0)
    nodes = np.nonzero((np.asarray(mask) != 0) & (np.asarray(fixed) == 0))[0]
    t = np.arange(n_trials)[:, None]
    for comp, r in ((0, rand_xy), (1, rand_xy), (2, rand_z)):
        out[:, nodes, comp] = multistart_draw(seed, t, nodes[None, :], comp, r)
    return out


def select_trial(equv, acpt_cost: float) -> int:
    """The acceptance walk of solve_with_multiple_init (:783-831): cost starts at acpt_cost, a trial replaces the best
    iff its cost is strictly lower.  -1 when no trial is accepted."""
    best, chosen = acpt_cost, -1
    for t, c in enumerate(equv):
        if c < best:
            best, chosen = c, t
    return chosen
