"""CPU: the arithmetic behind the fp16 row storage of the keyframe databases (OSB_DB_STORAGE_FP16).

Rounding a unit-norm row of dim 4096 to fp16 moves its inner product with a unit query by at most
2^-11 sum|q_i x_i| + 2^-25 sum|q_i| <= 4.9e-4 + 1.9e-6, and numpy's float16 conversion -- the oracle's -- rounds to
nearest even like CUDA's __float2half_rn (tests/test_gpu_db_fp16.py pins the device to it)."""
import os
import re

import numpy as np
import pytest

from omniswarm_b200 import lib
from oracle import db_storage_ref as dsr

DIM = 4096
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def unit(x):
    x = np.asarray(x, np.float64)
    return (x / np.linalg.norm(x, axis=-1, keepdims=True)).astype(np.float32)


def moved(q, x):
    """exact change of <q, x> when x is rounded to fp16 (float64 sums of float32 products are exact enough)"""
    xr = dsr.round_rows_fp16(x)
    return abs(float(q.astype(np.float64) @ (xr.astype(np.float64) - x.astype(np.float64))))


def adversarial(seed):
    """a (nearly unit) row whose every element rounds with nearly the largest relative error, just below a halfway point
    of [2^-6, 2^-5), and the query that adds those errors up"""
    rng = np.random.default_rng(seed)
    x = (2.0 ** -6 * (1 + (2 * rng.integers(0, 8, DIM) + 1 - 1e-3) * 2.0 ** -11)).astype(np.float32)
    x *= rng.choice([-1, 1], DIM).astype(np.float32)
    err = dsr.round_rows_fp16(x).astype(np.float64) - x
    q = unit(np.sign(err) * np.abs(x))
    return q, x


def subnormal_heavy(seed):
    """one large element and 4095 below the fp16 normal range (2^-14)"""
    rng = np.random.default_rng(seed)
    x = rng.uniform(-2.0 ** -15, 2.0 ** -15, DIM)
    x[rng.integers(DIM)] = 1.0
    return unit(rng.standard_normal(DIM)), unit(x)


CASES = [("random", s) for s in range(4)] + [("adversarial", s) for s in range(3)] + [("subnormal", s) for s in range(3)]


@pytest.mark.parametrize("kind,seed", CASES)
def test_score_change_within_bound(kind, seed):
    if kind == "random":
        rng = np.random.default_rng(seed)
        q, x = unit(rng.standard_normal(DIM)), unit(rng.standard_normal(DIM))
    elif kind == "adversarial":
        q, x = adversarial(seed)
    else:
        q, x = subnormal_heavy(seed)
    d, b = moved(q, x), dsr.fp16_score_bound(q, x)
    assert d <= b
    assert b <= 2.0 ** -11 * np.linalg.norm(x.astype(np.float64)) + 2.0 ** -25 * np.sqrt(DIM) * 1.0001
    if kind == "adversarial":           # the bound is tight: these rows reach most of it
        assert d >= 0.9 * b, (d, b)
    if kind != "adversarial":           # unit rows
        assert b <= 4.9e-4 + 1.9e-6


def test_numpy_float16_rounds_to_nearest_even():
    u = 2.0 ** -10                                     # the spacing of halves in [1, 2)
    cases = {
        1 + u / 2: 1.0,                                # halfway, 1 is even
        1 + 3 * u / 2: 1 + 2 * u,                      # halfway, 1 + 2u is even
        1 + u / 2 + 2.0 ** -20: 1 + u,                 # just above halfway
        -(1 + 5 * u / 2): -(1 + 2 * u),
        2.0 ** -25: 0.0,                               # halfway between 0 and the smallest subnormal
        3 * 2.0 ** -25: 2.0 ** -23,                    # halfway between subnormals 1 and 2 (x 2^-24): to 2
        5 * 2.0 ** -25: 2.0 ** -23,                    # halfway between 2 and 3: to 2
        65504.0: 65504.0,                              # the largest half
        65519.99: 65504.0,                             # below halfway to 2^16
        65520.0: np.inf,                               # halfway to 2^16 rounds to even = overflow
        -65520.0: -np.inf,
        1e30: np.inf,
    }
    x = np.array(list(cases), np.float32)
    assert np.array_equal(dsr.round_rows_fp16(x), np.array(list(cases.values()), np.float32))
    z = dsr.round_rows_fp16(np.array([0.0, -0.0], np.float32))
    assert np.signbit(z).tolist() == [False, True]


def test_oracle_stores_round_on_add():
    rng = np.random.default_rng(5)
    rows = unit(rng.standard_normal((50, 64)))
    a = dsr.IndexFlatIPFP16(64)
    a.add(rows)
    assert np.array_equal(a.rows, dsr.round_rows_fp16(rows))
    det = dsr.LoopDetectorDBFP16(1, 64)
    det.add_frame(7, 2, [rows[0]], [1])
    assert np.array_equal(det.remote_index.rows[0], dsr.round_rows_fp16(rows[0]))


def test_storage_constants_match_header():
    text = open(os.path.join(ROOT, "include", "omniswarm_b200.h")).read()
    found = dict(re.findall(r"#define (OSB_DB_STORAGE_FP(?:32|16)) (\d+)", text))
    assert found == {"OSB_DB_STORAGE_FP32": str(lib.DB_STORAGE_FP32), "OSB_DB_STORAGE_FP16": str(lib.DB_STORAGE_FP16)}
