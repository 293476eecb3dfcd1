"""ORACLE (test infrastructure, NOT product code) -- random_init_pose's choice of blocks (swarm_localization_solver.cpp:
204-216) taken from the sliding window, the rule osb_anchor_init_mask_dev computes on the device."""
import numpy as np

from oracle.anchor_ref import _yaw_vec


def init_mask(frame_first, entries, to_init, self_id: int, n_nodes: int):
    """(mask uint8 [n_nodes], yaw float64 [n_nodes]).  mask[b] = 1 iff block b belongs to a window entry (vo_available or
    not: add_as_keyframe gives every node frame a block, :517-540) of a drone d with to_init[d] and d != self_id; yaw[b] =
    that entry's self_pose yaw (NodeFrame::yaw(), the quaternion -> yaw of oracle/anchor_ref.py).  Frames are walked in
    order, so a block shared by several frames takes its latest frame's pose, as the reference writes the shared block
    once per (ts, id) in stamp order.  Elsewhere 0."""
    mask = np.zeros(n_nodes, np.uint8)
    yaw = np.zeros(n_nodes, np.float64)
    to_init = np.asarray(to_init, bool)
    for f in range(len(frame_first) - 1):
        for e in entries[frame_first[f]:frame_first[f + 1]]:
            d, b = int(e["drone_id"]), int(e["block"])
            if d == self_id or not to_init[d]:
                mask[b], yaw[b] = 0, 0.0       # the block's latest entry decides (a block holds one drone)
                continue
            mask[b] = 1
            yaw[b] = _yaw_vec(np.asarray(e["self_pose"][3:7], np.float64)[None])[0]
    return mask, yaw
