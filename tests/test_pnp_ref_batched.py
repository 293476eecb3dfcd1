"""oracle/pnp_ref.pnp_ransac_batched (every hypothesis fitted and scored at once) against pnp_ransac, the per-hypothesis
restatement it vectorises: the same mask, inlier count and winner, and the same pose."""
import time

import numpy as np
import pytest

from omniswarm_b200 import synth
from oracle import pnp_ref as pn
from oracle.geometry_ref import draw4


def same(c, iterations, thresh, seed):
    with np.errstate(all="ignore"):                   # landmarks on the camera plane give inf / NaN on purpose
        a = pn.pnp_ransac(c["X"], c["uv"], c["prior"], iterations, thresh, seed)
    b = pn.pnp_ransac_batched(c["X"], c["uv"], c["prior"], iterations, thresh, seed)
    assert b["success"] == a["success"]
    assert b["n_inliers"] == a["n_inliers"] and b["winner"] == a["winner"]
    assert np.array_equal(b["mask"], a["mask"])
    assert np.abs(np.asarray(b["pose"]) - np.asarray(a["pose"])).max() <= 1e-12
    return b


def identity_case(n, seed):
    """points in front of a camera whose prior is the identity rotation, so landmarks can sit exactly on its z = 0 plane"""
    rng = np.random.default_rng(seed)
    Pc = np.stack([rng.uniform(-2, 2, n), rng.uniform(-1.5, 1.5, n), rng.uniform(2, 8, n)], 1)
    uv = Pc[:, :2] / Pc[:, 2:3] + rng.normal(0, 0.002, (n, 2))
    return dict(X=Pc.astype(np.float32), uv=uv.astype(np.float32), prior=np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0]))


@pytest.mark.parametrize("n,out,iterations,thresh,seed", [
    (200, 0.25, 100, 0.03, 0), (40, 0.0, 100, 0.03, 2), (120, 0.6, 60, 0.03, 3), (64, 0.3, 100, 3.0, 4),
    (4, 0.0, 100, 0.03, 5), (5, 0.0, 50, 0.03, 6), (3, 0.0, 100, 0.03, 7), (0, 0.0, 100, 0.03, 8),
    (150, 0.2, 0, 0.03, 9), (150, 0.2, 1, 0.03, 10)])
def test_batched_matches_sequential(n, out, iterations, thresh, seed):
    c = synth.pnp_case(n, out, seed) if n else dict(X=np.zeros((0, 3), np.float32), uv=np.zeros((0, 2), np.float32),
                                                    prior=synth.pnp_case(4, 0.0, seed)["prior"])
    b = same(c, iterations, thresh, seed)
    if n < 4 or iterations == 0:
        assert not b["success"] and b["winner"] == -1 and b["n_inliers"] == 0
    if n == 4:                                          # 16 tries per slot do not always find 4 distinct of 4 indices
        assert any(draw4(seed, h, 4) is None for h in range(iterations))


def test_batched_degenerate_samples():
    # every correspondence the same one: each sample's normal equations have rank 2
    c = synth.pnp_case(12, 0.0, 11)
    c["X"][:] = c["X"][0]; c["uv"][:] = c["uv"][0]
    same(c, 100, 0.03, 11)
    # duplicated correspondences, collinear and coplanar landmarks among generic ones
    c = synth.pnp_case(160, 0.2, 12)
    c["X"][40:80] = c["X"][:40]; c["uv"][40:80] = c["uv"][:40]
    s = np.linspace(0.0, 1.0, 30, dtype=np.float32)[:, None]
    c["X"][80:110] = c["X"][0] + s * (c["X"][1] - c["X"][0])
    c["X"][110:140, 2] = c["X"][0, 2]
    same(c, 100, 0.03, 12)


def test_batched_points_on_and_behind_the_camera_plane():
    """landmarks at camera z = 0 under the prior give inf / NaN errors and normal equations (never inliers, the sample's
    Cholesky fails so its model stays the prior); landmarks behind the camera project like any other (no cheirality)"""
    c = identity_case(120, 13)
    c["X"][:10, 2] = 0.0
    c["X"][10:14, :2] = 0.0; c["X"][10:14, 2] = 0.0            # 0 / 0
    c["X"][14:20] *= -1.0
    b = same(c, 100, 0.03, 13)
    assert b["success"] and not b["mask"][:14].any() and np.all(np.isfinite(b["pose"]))


def test_batched_all_outliers_keep_the_prior():
    rng = np.random.default_rng(14)
    c = synth.pnp_case(60, 0.0, 14)
    c["uv"] = rng.uniform(-1, 1, (60, 2)).astype(np.float32)
    b = same(c, 100, 1e-4, 14)
    assert not b["success"] and b["n_inliers"] < 4 and b["winner"] >= 0
    assert np.array_equal(b["pose"], c["prior"])


def test_batched_margin_and_ties():
    c = synth.pnp_case(100, 0.3, 15)
    b = pn.pnp_ransac_batched(c["X"], c["uv"], c["prior"], 50, 0.03, 15)
    e = np.stack([pn.reproj_sq(pn.lm_pose(c["prior"], c["X"].astype(np.float64)[i], c["uv"].astype(np.float64)[i],
                                          pn.HYP_ITERS), c["X"].astype(np.float64), c["uv"].astype(np.float64))
                  for i in (draw4(15, h, 100) for h in range(50)) if i is not None])
    t2 = 0.03 * 0.03
    assert b["margin"] == np.abs(e - t2).min() / t2 and b["ties"] == 0 and b["margin_untied"] == b["margin"]
    # threshold exactly at one of the errors the winner scores
    w = pn.lm_pose(c["prior"], c["X"].astype(np.float64)[draw4(15, b["winner"], 100)],
                   c["uv"].astype(np.float64)[draw4(15, b["winner"], 100)], pn.HYP_ITERS)
    t = float(np.sqrt(pn.reproj_sq(w, c["X"].astype(np.float64), c["uv"].astype(np.float64))[0]))
    tb = pn.pnp_ransac_batched(c["X"], c["uv"], c["prior"], 50, t, 15)
    assert tb["margin"] <= 1e-15


def test_batched_reference_is_fast_at_the_largest_launch():
    c = synth.pnp_case(1024, 0.3, 16)
    t = time.perf_counter()
    b = pn.pnp_ransac_batched(c["X"], c["uv"], c["prior"], 1000, 0.03, 16)
    assert time.perf_counter() - t < 30.0                     # ~0.4 s on one core; the per-hypothesis form takes minutes
    assert b["success"] and b["n_inliers"] == int(b["mask"].sum()) > 600
