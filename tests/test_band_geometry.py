"""CPU: the blanked band of the front-end's SuperPoint (osb_superpoint_band_geometry) against a brute-force propagation.

Images zero from row r0 down: a trunk output pixel is constant when it depends on no non-blank input and on no padding.
The propagation marks, layer by layer, every pixel that does depend on one ("tainted"); the geometry must give exactly
the untainted pixels, exactly the untainted whole 8 x 16 tiles, and exactly the conv1a pixels that no computed conv1b tile
reads."""
import numpy as np
import pytest

from omniswarm_b200.host import SuperPoint

# conv1a, conv1b + pool, conv2a, conv2b + pool, conv3a, conv3b + pool, conv4a, conv4b (superpoint.ipynb:143-158)
TRUNK = [(3, 0), (3, 1), (3, 0), (3, 1), (3, 0), (3, 1), (3, 0), (3, 0)]
TH, TW = 8, 16


def brute(H, W, r0):
    taint = np.ones((H, W), bool)
    if 0 <= r0 < H:
        taint[r0:] = False
    layers = []
    for ks, pool in TRUNK:
        h, w = taint.shape
        k = ks // 2
        pad = np.pad(taint, k, constant_values=True)              # padding differs from the constant
        out = np.zeros_like(taint)
        for dy in range(ks):
            for dx in range(ks):
                out |= pad[dy:dy + h, dx:dx + w]
        tiles = {(ty, tx) for ty in range(h // TH) for tx in range(w // TW)
                 if not out[TH * ty:TH * ty + TH, TW * tx:TW * tx + TW].any()}
        if pool:
            out = out.reshape(h // 2, 2, w // 2, 2).any(axis=(1, 3))
        layers.append((out, tiles, (h, w)))
        taint = out
    return layers


def rect_mask(r, shape):
    m = np.zeros(shape, bool)
    y0, y1, x0, x1 = (int(v) for v in r)
    if y0 < y1 and x0 < x1:
        m[y0:y1, x0:x1] = True
    return m


def rect_tiles(r):
    y0, y1, x0, x1 = (int(v) for v in r)
    return {(ty, tx) for ty in range(y0, y1) for tx in range(x0, x1)}


def first_skip(H, W, const_tiles):
    """conv1a pixels read by no computed conv1b tile (ragged tiles included among the computed ones)"""
    read = np.zeros((H, W), bool)
    for ty in range(-(-H // TH)):
        for tx in range(-(-W // TW)):
            if (ty, tx) not in const_tiles:
                read[max(TH * ty - 1, 0):TH * ty + TH + 1, max(TW * tx - 1, 0):TW * tx + TW + 1] = True
    return ~read


GEOMETRIES = [(480, 640), (240, 320), (64, 96), (96, 64), (200, 320), (168, 248), (360, 480), (72, 640), (520, 200),
              (960, 1280)]


@pytest.mark.parametrize("H,W", GEOMETRIES)
def test_band_geometry_matches_brute_force(H, W):
    for r0 in sorted({H * 3 // 4, H // 2, H - 8, 0, 8, H, -1}):
        g = SuperPoint.band_geometry(H, W, r0)
        ref = brute(H, W, r0)
        h, w = H, W
        for l, (taint, tiles, (hl, wl)) in enumerate(ref):
            assert (hl, wl) == (h, w)
            assert np.array_equal(rect_mask(g["px"][l], taint.shape), ~taint), (H, W, r0, l)
            assert rect_tiles(g["tiles"][l]) == tiles, (H, W, r0, l, g["tiles"][l])
            h, w = taint.shape
        assert np.array_equal(rect_mask(g["first_skip"], (H, W)), first_skip(H, W, ref[1][1])), (H, W, r0)
        if r0 < 0 or r0 >= H:                                     # nothing blanked: nothing constant
            assert all(not rect_tiles(t) for t in g["tiles"]) and not rect_mask(g["first_skip"], (H, W)).any()


def test_flagship_geometry():
    """640 x 480 with the bottom quarter blanked (the front-end's STEREO_FISHEYE default)"""
    g = SuperPoint.band_geometry(480, 640, 360)
    assert g["tiles"][1].tolist() == [46, 59, 1, 39]      # conv1b: tile rows 46-58, 38 of 40 columns
    assert g["tiles"][2].tolist() == [23, 29, 1, 19] == g["tiles"][3].tolist()
    assert g["tiles"][4].tolist() == [12, 14, 1, 9] == g["tiles"][5].tolist()
    assert g["tiles"][6].tolist() == [6, 7, 1, 4]
    assert rect_tiles(g["tiles"][7]) == set()
    assert g["first_skip"].tolist() == [369, 471, 17, 623]


def test_band_geometry_refuses_bad_sizes():
    from omniswarm_b200 import lib
    with pytest.raises(lib.OsbError):
        SuperPoint.band_geometry(100, 640, 75)
