"""What the back-end's GPU tests share: a LoopAnchor and a PcmState of a synth.anchor_swarm scenario, the anchor fed
with it, and a pose-graph solver's option presets and resident window.  Test modules import it as `backend_harness`;
the device buffers of a solve are host.AnchoredChain and host.FactorRows."""
import numpy as np

from omniswarm_b200 import host

THRES = 15.0                             # the PCM threshold of every back-end test's state
KEYS = host.FACTOR_KEYS


def make_anchor(g, max_meas=None, max_entries=None, traj_margin=64):
    """a LoopAnchor for scenario g: room for every trajectory plus traj_margin samples, max_meas measurements and
    max_entries window entries (default: the scenario's plus 64)"""
    return host.LoopAnchor(g["max_drones"], max(len(v[0]) for v in g["trajs"].values()) + traj_margin,
                           max_meas or len(g["meas"]) + 64, max_entries or len(g["window"][2]) + 64,
                           g["prm"]["det_dpos_thres"], g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"],
                           g["prm"]["begin_min_loop_dt_s"])


def feed(a, g, chunks=3):
    """the scenario's odometry in chunks, its measurements in two calls, its window"""
    for d, (st, p) in g["trajs"].items():
        for c in np.array_split(np.arange(len(st)), chunks):             # only new samples cross PCIe, length continues
            a.push_odometry(d, st[c], p[c])
    m = g["meas"]
    a.add_measurements(m[: len(m) // 3])
    a.add_measurements(m[len(m) // 3:])
    a.set_window(*g["window"])


def pcm_state(g, max_pairs, pair_capacity, self_id=0, redundant=True):
    """a PcmState with THRES and the scenario's odometry covariances"""
    return host.PcmState(self_id, redundant, THRES, g["prm"]["odom_pos_cov_per_m"], g["prm"]["odom_ang_cov_per_m"],
                         max_pairs=max_pairs, pair_capacity=pair_capacity)


def options(solver, kind):
    """the solver's defaults ("default"), or tight tolerances ("tight") with fp64 inner iterations ("fp64") or the
    block-Jacobi preconditioner ("jacobi")"""
    o = solver.default_options()
    if kind in ("tight", "fp64", "jacobi"):
        o.function_tolerance = 1e-14; o.pcg_tolerance = 1e-8; o.max_pcg_iterations = 2000
    if kind == "fp64":
        o.inner_precision = 1                                  # OSB_INNER_FP64
    if kind == "jacobi":
        o.preconditioner = 1                                   # OSB_PRECOND_BLOCK_JACOBI
    return o


def resident(solver, base):
    """the solver's resident graph replaced by the pose graph `base` (synth.anchor_window_graph's layout)"""
    solver.graph_clear()
    solver.graph_add_nodes(base["init"], base["fixed"])
    solver.graph_add_factors(*(base[k] for k in KEYS))
