"""CPU: the init-branch mask rule of tests/init_mask_ref.py (random_init_pose's blocks, the rule
osb_anchor_init_mask_dev computes on the device) on hand-built windows, and the C declarations of the init branch."""
import ctypes as C
import math
import os
import re
import shutil
import subprocess

import numpy as np
import pytest

from omniswarm_b200 import lib
import init_mask_ref as mr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def quat(yaw):
    return [math.cos(yaw / 2), 0.0, 0.0, math.sin(yaw / 2)]


def window(frames):
    """frames: list of [(drone, block, yaw, vo_available), ...] -> (frame_first, entries)"""
    rows = [r for f in frames for r in f]
    e = np.zeros(len(rows), lib.WINDOW_ENTRY_DTYPE)
    for i, (d, b, y, vo) in enumerate(rows):
        e[i]["drone_id"], e[i]["block"], e[i]["vo_available"] = d, b, vo
        e[i]["self_pose"] = [0.1 * i, 0.0, 0.0] + quat(y)
    first = np.cumsum([0] + [len(f) for f in frames]).astype(np.int32)
    return first, e


def to_init(*drones, n=8):
    t = np.zeros(n, bool)
    t[list(drones)] = True
    return t


def test_shared_block_takes_the_latest_frame():
    # drone 1 did not move between frames 0 and 2: its block 1 is shared, written once per frame in stamp order
    first, e = window([[(0, 0, 0.0, 1), (1, 1, 0.3, 1)], [(0, 2, 0.1, 1)], [(0, 3, 0.2, 1), (1, 1, -0.7, 1)]])
    mask, yaw = mr.init_mask(first, e, to_init(1), 0, 4)
    assert mask.tolist() == [0, 1, 0, 0]
    assert yaw[1] == pytest.approx(-0.7, abs=1e-15) and yaw[[0, 2, 3]].tolist() == [0.0, 0.0, 0.0]


def test_entries_without_vo_count():
    first, e = window([[(0, 0, 0.0, 1), (2, 1, 0.4, 0)], [(0, 2, 0.0, 1), (2, 3, 0.5, 0)]])
    mask, yaw = mr.init_mask(first, e, to_init(2), 0, 5)
    assert mask.tolist() == [0, 1, 0, 1, 0]
    assert yaw[1] == pytest.approx(0.4, abs=1e-15) and yaw[3] == pytest.approx(0.5, abs=1e-15)


def test_self_is_never_masked():
    first, e = window([[(0, 0, 0.2, 1), (1, 1, 0.3, 1)], [(0, 2, 0.2, 1), (1, 3, 0.3, 1)]])
    mask, _ = mr.init_mask(first, e, to_init(0, 1), 0, 4)
    assert mask.tolist() == [0, 1, 0, 1]
    mask, _ = mr.init_mask(first, e, to_init(0, 1), 1, 4)
    assert mask.tolist() == [1, 0, 1, 0]


def test_drones_not_to_init_are_untouched():
    first, e = window([[(0, 0, 0.0, 1), (1, 1, 0.3, 1), (2, 2, 0.6, 1)], [(1, 3, 0.3, 1), (3, 4, 0.9, 0)]])
    mask, yaw = mr.init_mask(first, e, to_init(2, 3), 0, 7)
    assert mask.tolist() == [0, 0, 1, 0, 1, 0, 0]
    assert yaw[[0, 1, 3, 5, 6]].tolist() == [0.0] * 5
    assert yaw[4] == pytest.approx(0.9, abs=1e-15)
    mask, yaw = mr.init_mask(first, e, to_init(), 0, 7)
    assert not mask.any() and not yaw.any()


def prototype(name):
    text = re.sub(r"/\*.*?\*/", "", open(os.path.join(ROOT, "include", "omniswarm_b200.h")).read(), flags=re.S)
    m = re.search(r"\bosb_status\s+" + name + r"\s*\((.*?)\);", text, flags=re.S)
    assert m, name
    return [a.strip() for a in m.group(1).split(",")]


@pytest.mark.parametrize("name", ["osb_anchor_init_mask_dev", "osb_solver_solve_multistart_resident_dev",
                                  "osb_solver_last_multistart"])
def test_prototypes_match_ctypes(name):
    args = prototype(name)
    assert len(lib._SIG[name][1]) == len(args), (name, args)
    assert name in lib.exported_symbols() and hasattr(lib.load(), name)


def test_struct_sizes():
    assert C.sizeof(lib.MultistartOptions) == 48 and C.sizeof(lib.SolveSummary) == 40
    assert lib.WINDOW_ENTRY_DTYPE.itemsize == 80 and C.sizeof(lib.Observability) == 5 * 256 + 16


@pytest.mark.skipif(shutil.which("gcc") is None, reason="gcc missing")
def test_header_parses_as_c():
    r = subprocess.run(["gcc", "-std=c99", "-fsyntax-only", "-Wall", "-Werror", "-x", "c",
                        os.path.join(ROOT, "include", "omniswarm_b200.h")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
