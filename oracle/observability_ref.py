"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the observability estimate that every solve() of
the back-end makes before it builds its problem (osb_anchor_observe_dev).

Follows (paths relative to the reference's swarm_localization/src):
  * SwarmLocalizationSolver::estimate_observability  swarm_localization_solver.cpp:1336-1427 -- yaw_observability cleared
      (:1338), loop_edges from find_available_loops_detections (every loop and detection that comes back OK, :1600-1634),
      the single-drone rule `sf_sld_win.size() > SINGLE_DRONE_SFS_THRES && all_nodes.size() == 1` (:1364-1367, the
      threshold 3 at :62), the loop-observable set (:1369-1379), the self bounding box against init_xy_movement /
      init_z_movement (:1381-1403) and the per-drone box against THRES_YAW_OBSER_XY = 1.0 (:49, :1413-1422);
  * loop_observable_set  :1299-1334 -- {self_id}, grown by a BFS over loop_edges only when all_nodes holds more than one
      drone;
  * boundingbox_sldwin  :848-878 -- the vo_available entries of one drone over the window, max from -1000 and min from
      +1000 per axis, so a drone without such an entry has extents of -2000;
  * add_new_swarm_frame  :627-645 -- every keyframe's drone ids join all_nodes, vo_available or not; the adapter passes
      every keyframe through set_window, so all_nodes is every drone of every window since create;
      enable_to_init_by_drone[self_id] is set true on every keyframe (:640);
  * setup_problem_with_loops_and_detections  :1064-1073 -- a row becomes a factor only when both drones are
      yaw-observable and its two ends are different pose blocks (anchor_ref's skip rule, with this solve's yaw).

pos_observability is a std::map<int, bool>: a drone never written reads false, self_id included, so the first call puts
self_id into ids_to_init.  pos, enable_to_init_by_drone and enable_to_solve_master only ever become true.  init_xy_movement
and init_z_movement are float parameters compared as doubles.  finish_init and system_is_initied_by_motion stay with the
caller: `motion_new` is the branch that sets both (:1392-1396), `motion` the box test (:1400-1402).
"""
from __future__ import annotations

import numpy as np

OK = 0                                   # anchor_ref.OK (status of a usable row)
THRES_YAW_OBSER_XY = 1.0                 # :49
SINGLE_DRONE_SFS_THRES = 3               # :62


def bounding_box(entries, drone):
    """boundingbox_sldwin (:848-878) over the window's entries -> (min xyz, max xyz), each a list of 3 floats"""
    xmax, xmin, ymax, ymin, zmax, zmin = -1000.0, 1000.0, -1000.0, 1000.0, -1000.0, 1000.0
    for e in entries:
        if int(e["drone_id"]) == drone and e["vo_available"]:
            x, y, z = (float(v) for v in e["self_pose"][:3])
            if x > xmax:
                xmax = x
            if y > ymax:
                ymax = y
            if z > zmax:
                zmax = z
            if x < xmin:
                xmin = x
            if y < ymin:
                ymin = y
            if z < zmin:
                zmin = z
    return [xmin, ymin, zmin], [xmax, ymax, zmax]


def loop_observable_set(self_id, all_nodes, loop_edges):
    """:1299-1334: self_id, and when all_nodes holds more than one drone every drone its loop edges reach"""
    obs = {self_id}
    if len(all_nodes) > 1:
        queue = [self_id]
        while queue:
            d = queue.pop(0)
            for c in sorted(loop_edges.get(d, ())):
                if c not in obs:
                    obs.add(c)
                    queue.append(c)
    return obs


class ObservabilityRef:
    """The persistent part of SwarmLocalizationSolver that estimate_observability reads and writes: all_nodes,
    pos_observability, enable_to_init_by_drone, enable_to_solve_master, and the window of the last set_window."""

    def __init__(self, max_drones: int):
        self.max_drones = max_drones
        self.all_nodes: set[int] = set()
        self.pos: dict[int, bool] = {}
        self.enable: dict[int, bool] = {}
        self.solve_master = False
        self.n_frames = 0
        self.entries = np.zeros(0)
        self.last = None

    def set_window(self, frame_stamps, frame_first, entries):
        """the window of the next solves; its drones join all_nodes (:627-645)"""
        self.n_frames = len(frame_stamps)
        self.entries = np.asarray(entries)[: int(frame_first[-1]) if len(frame_first) else 0]
        self.all_nodes |= {int(d) for d in self.entries["drone_id"]} if len(self.entries) else set()

    def observe(self, rows, self_id: int, init_xy_movement: float, init_z_movement: float) -> dict:
        """estimate_observability (:1336-1427) with this solve's rows (anchor_ref's result records) -> the outcome, the
        record osb_anchor_observability writes: bool arrays [max_drones] nodes / yaw / pos / enable / to_init and the
        flags solve_master, motion, motion_new"""
        loop_edges: dict[int, set[int]] = {}
        for r in rows:                                                   # :1600-1634
            if int(r["status"]) == OK:
                a, b = int(r["edge"]["id_a"]), int(r["edge"]["id_b"])
                loop_edges.setdefault(a, set()).add(b)
                loop_edges.setdefault(b, set()).add(a)
        yaw: dict[int, bool] = {}                                        # :1338
        to_init: set[int] = set()
        observable = loop_observable_set(self_id, self.all_nodes, loop_edges)
        if self.n_frames > SINGLE_DRONE_SFS_THRES and len(self.all_nodes) == 1:   # :1364-1367
            self.solve_master = True
        for d in observable:                                             # :1369-1379
            if not self.pos.get(d, False):
                to_init.add(d)
            self.pos[d] = True
            yaw[d] = True
            self.enable[d] = True
            if d != self_id:
                self.solve_master = True
        lo, hi = bounding_box(self.entries, self_id)                     # :1381-1403
        xy, z = float(np.float32(init_xy_movement)), float(np.float32(init_z_movement))
        motion = hi[0] - lo[0] > xy and hi[1] - lo[1] > xy and hi[2] - lo[2] > z
        motion_new = False
        if motion:
            self.solve_master = True
            for d in self.all_nodes:
                if not self.pos.get(d, False):
                    motion_new = True
                    to_init.add(d)
                self.pos[d] = True
                self.enable[d] = True
        for d in self.all_nodes:                                         # :1413-1422
            lo, hi = bounding_box(self.entries, d)
            if hi[0] - lo[0] > THRES_YAW_OBSER_XY or hi[1] - lo[1] > THRES_YAW_OBSER_XY:
                yaw[d] = True
        self.enable[self_id] = True                                      # :640

        def mask(keys):
            m = np.zeros(self.max_drones, bool)
            m[[d for d in keys if 0 <= d < self.max_drones]] = True
            return m

        self.last = dict(nodes=mask(self.all_nodes), yaw=mask(d for d, v in yaw.items() if v),
                         pos=mask(d for d, v in self.pos.items() if v), enable=mask(d for d, v in self.enable.items() if v),
                         to_init=mask(to_init), solve_master=self.solve_master, motion=motion, motion_new=motion_new)
        return self.last


def skip(rows, yaw) -> np.ndarray:
    """:1064-1073 per row with this solve's yaw mask: 1 unless the row is OK, both drones are yaw-observable and its two
    ends are different pose blocks"""
    out = np.ones(len(rows), np.int32)
    for i, r in enumerate(rows):
        a, b = int(r["edge"]["id_a"]), int(r["edge"]["id_b"])
        if int(r["status"]) == OK and yaw[a] and yaw[b] and int(r["node_a"]) != int(r["node_b"]):
            out[i] = 0
    return out
