"""CPU: the rules of the random-restart initialisation (osb_solver_solve_multistart) -- the oracle's hashed draws, the
acceptance walk of solve_with_multiple_init (solver.cpp:781-845), the header and the C++ adapter."""
import ctypes as C
import math
import os
import shutil
import subprocess

import numpy as np
import pytest

from omniswarm_b200 import lib
from oracle import multistart_ref as mr

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "omni-swarm_b200", "csrc")


def _base(n, seed=0):
    rng = np.random.default_rng(seed)
    return rng.standard_normal((n, 4)) * 3.0


def test_draws_inside_range_and_deterministic():
    n, K = 40, 16
    base = _base(n)
    mask = np.ones(n, np.uint8); fixed = np.zeros(n, np.uint8)
    a = mr.multistart_initial_poses(base, mask, fixed, K, seed=123, rand_xy=5.0, rand_z=1.0)
    b = mr.multistart_initial_poses(base, mask, fixed, K, seed=123, rand_xy=5.0, rand_z=1.0)
    assert a.shape == (K, n, 4)
    assert np.array_equal(a, b)
    assert np.all(np.abs(a[..., :2]) <= 5.0) and np.all(np.abs(a[..., 2]) <= 1.0)
    assert np.all(a[..., :2] >= -5.0) and np.all(a[..., :2] < 5.0)
    # the draws spread over the range and differ between trials, nodes, components and seeds
    assert a[..., 0].min() < -4.0 and a[..., 0].max() > 4.0
    assert len(np.unique(a[..., :3])) == K * n * 3
    c = mr.multistart_initial_poses(base, mask, fixed, K, seed=124)
    assert not np.any(c[..., :3] == a[..., :3])


def test_draw_is_a_function_of_seed_trial_node_component():
    v = mr.multistart_draw(7, 3, 11, 2, 1.0)
    assert v == mr.multistart_draw(7, np.array([3]), np.array([11]), 2, 1.0)[0]
    # the exact formula: u = (sm(seed ^ sm(key)) >> 11) 2^-53, value = 2r u - r (two roundings)
    def sm(z):
        z = (z + 0x9E3779B97F4A7C15) & (2 ** 64 - 1)
        z = ((z ^ (z >> 30)) * 0xBF58476D1CE4E5B9) & (2 ** 64 - 1)
        z = ((z ^ (z >> 27)) * 0x94D049BB133111EB) & (2 ** 64 - 1)
        return z ^ (z >> 31)
    key = (3 << 34) | (11 << 2) | 2
    u = (sm(7 ^ sm(key)) >> 11) * 2.0 ** -53
    assert v == 2.0 * u + -1.0


def test_draws_unchanged_when_nodes_are_appended():
    base = _base(30)
    mask = (np.arange(30) % 3 != 0).astype(np.uint8); fixed = np.zeros(30, np.uint8)
    a = mr.multistart_initial_poses(base, mask, fixed, 5, seed=9)
    big = np.concatenate([base, _base(17, 1)])
    b = mr.multistart_initial_poses(big, np.concatenate([mask, np.ones(17, np.uint8)]),
                                    np.zeros(47, np.uint8), 5, seed=9)
    assert np.array_equal(b[:, :30], a)
    # and unchanged when more trials are asked for
    c = mr.multistart_initial_poses(base, mask, fixed, 9, seed=9)
    assert np.array_equal(c[:5], a)


def test_unmasked_and_fixed_nodes_and_every_yaw_stay_bit_equal():
    n = 25
    base = _base(n)
    mask = (np.arange(n) % 2).astype(np.uint8)
    fixed = np.zeros(n, np.uint8); fixed[[1, 3, 4]] = 1          # 1, 3: masked but fixed
    p = mr.multistart_initial_poses(base, mask, fixed, 6, seed=5, rand_xy=5.0, rand_z=1.0)
    keep = (mask == 0) | (fixed != 0)
    for t in range(6):
        assert np.array_equal(p[t, keep], base[keep])
        assert np.array_equal(p[t, :, 3], base[:, 3])
        assert not np.any(p[t, ~keep, :3] == base[~keep, :3])
    # rand = 0 puts the scattered nodes at the origin
    z = mr.multistart_initial_poses(base, mask, fixed, 2, seed=5, rand_xy=0.0, rand_z=0.0)
    assert np.all(z[:, ~keep, :3] == 0.0)


def test_select_trial_rules():
    # strict < against acpt_cost
    assert mr.select_trial([1.0, 2.0], 1.0) == -1
    assert mr.select_trial([1.0, 0.5], 1.0) == 1
    assert mr.select_trial([0.9], 1.0) == 0
    # ties go to the first index
    assert mr.select_trial([0.7, 0.3, 0.3, 0.5], 1.0) == 1
    # a NaN is never taken, and does not stop the walk
    assert mr.select_trial([math.nan, 0.4, math.nan], 1.0) == 1
    assert mr.select_trial([math.nan, math.nan], math.inf) == -1
    # nothing below acpt_cost
    assert mr.select_trial([3.0, 4.0, math.inf], 2.0) == -1
    assert mr.select_trial([], 2.0) == -1
    # an infinite acpt_cost accepts the lowest finite cost
    assert mr.select_trial([5.0, 2.0, 7.0], math.inf) == 1


def test_multistart_options_struct_layout():
    assert C.sizeof(lib.MultistartOptions) == 3 * 4 + 4 + 8 + 3 * 8
    assert lib.MultistartOptions.seed.offset == 16 and lib.MultistartOptions.rand_xy.offset == 24


@pytest.mark.skipif(shutil.which("gcc") is None, reason="gcc missing")
def test_header_parses_as_c():
    r = subprocess.run(["gcc", "-std=c99", "-fsyntax-only", "-Wall", "-Werror", "-x", "c",
                        os.path.join(ROOT, "include", "omniswarm_b200.h")], capture_output=True, text=True)
    assert r.returncode == 0, r.stderr


def build_multistart_smoke(tmp_path):
    exe = str(tmp_path / "multistart_smoke")
    cmd = ["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"),
           os.path.join(ROOT, "tests", "cpp", "multistart_smoke.cpp"), "-L", CSRC, "-lomniswarm_b200",
           f"-Wl,-rpath,{CSRC}", "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.skipif(shutil.which("g++") is None, reason="g++ missing")
def test_adapter_multistart_compiles_and_runs(tmp_path):
    exe = build_multistart_smoke(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr          # without a GPU: osb_solver_create reported no device
