"""ORACLE (test infrastructure): ctypes binding of oracle/c/anchor_ref.c, the single-threaded C restatement of the
re-anchoring walk (find_available_loops_detections, swarm_localization_solver.cpp:1594-1666).  `anchor` has the signature
of anchor_ref.anchor; `Walk` holds the inputs packed once, so that `run` times the walk alone."""
from __future__ import annotations

import ctypes as C
import os
import subprocess
import time

import numpy as np

from . import anchor_ref as ar

_DIR = os.path.join(os.path.dirname(os.path.abspath(__file__)), "c")
_SRC = os.path.join(_DIR, "anchor_ref.c")
_PATH = os.path.join(_DIR, "libanchor_ref.so")
_lib = None


class Params(C.Structure):
    _fields_ = [("begin_min_loop_dt_s", C.c_double), ("det_dpos_thres", C.c_double), ("odom_pos_cov_per_m", C.c_double),
                ("odom_ang_cov_per_m", C.c_double), ("huber", C.c_int32), ("reserved", C.c_int32)]


def build() -> str:
    """the recipe of oracle/c/Makefile: $(CC) -O2 -shared -fPIC"""
    cc = os.environ.get("CC", "gcc")
    r = subprocess.run([cc, "-O2", "-shared", "-fPIC", "-o", _PATH, _SRC, "-lm"], capture_output=True, text=True)
    if r.returncode != 0:
        raise RuntimeError("building oracle/c/anchor_ref.c failed:\n" + r.stdout + r.stderr)
    return _PATH


def load():
    global _lib
    if _lib is None:
        if not os.path.exists(_PATH):
            build()
        _lib = C.CDLL(_PATH)
        _lib.osb_ref_anchor.restype = C.c_int
        _lib.osb_ref_anchor.argtypes = [C.POINTER(Params), C.c_int] + [C.c_void_p] * 4 + [C.c_int] + [C.c_void_p] * 3 \
            + [C.c_int] + [C.c_void_p] * 3
    return _lib


def _p(a):
    return a.ctypes.data_as(C.c_void_p)


class Walk:
    """the inputs of anchor_ref.anchor packed for the C walk"""

    def __init__(self, trajs: dict, window, meas, yaw_observable, prm: dict):
        frame_stamps, frame_first, entries = window
        ids = [int(d) for d in trajs] + [int(x) for x in np.concatenate([meas["id_a"], meas["id_b"]])]
        self.n_drones = max(ids) + 1 if ids else 1
        first = np.zeros(self.n_drones + 1, np.int64)
        stamps, poses, lens = [], [], []
        for d in range(self.n_drones):
            s, p = trajs.get(d, (np.zeros(0, np.int64), np.zeros((0, 7))))
            first[d + 1] = first[d] + len(s)
            stamps.append(np.asarray(s, np.int64))
            poses.append(np.asarray(p, np.float64).reshape(-1, 7))
            lens.append(ar.trajectory_lengths(p))
        self.first = first
        self.stamps = np.ascontiguousarray(np.concatenate(stamps))
        self.poses = np.ascontiguousarray(np.concatenate(poses))
        self.lens = np.ascontiguousarray(np.concatenate(lens))
        self.frame_stamps = np.ascontiguousarray(frame_stamps, np.int64)
        self.frame_first = np.ascontiguousarray(frame_first, np.int32)
        self.entries = np.ascontiguousarray(entries, ar.ENTRY_DTYPE)
        self.meas = np.ascontiguousarray(meas, ar.MEAS_DTYPE)
        yaw = np.zeros(self.n_drones, np.uint8)
        y = np.asarray(yaw_observable, bool)[:self.n_drones]
        yaw[:len(y)] = y
        self.yaw = yaw
        self.prm = Params(float(prm["begin_min_loop_dt_s"]), float(prm["det_dpos_thres"]), float(prm["odom_pos_cov_per_m"]),
                          float(prm["odom_ang_cov_per_m"]), 1 if prm.get("huber", True) else 0, 0)
        self.out = np.zeros(len(self.meas), ar.RESULT_DTYPE)

    def run(self) -> float:
        """one walk -> its wall time in ms; the results are in self.out"""
        lib = load()
        t0 = time.perf_counter()
        n = lib.osb_ref_anchor(C.byref(self.prm), self.n_drones, _p(self.first), _p(self.stamps), _p(self.poses),
                               _p(self.lens), len(self.frame_stamps), _p(self.frame_stamps), _p(self.frame_first),
                               _p(self.entries), len(self.meas), _p(self.meas), _p(self.yaw), _p(self.out))
        ms = (time.perf_counter() - t0) * 1e3
        assert n == len(self.meas)
        return ms


def anchor(trajs: dict, window, meas, yaw_observable, prm: dict) -> np.ndarray:
    w = Walk(trajs, window, meas, yaw_observable, prm)
    w.run()
    return w.out
