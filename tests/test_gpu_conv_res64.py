"""The 64 -> 64 channel 3x3 layers (conv_res64_kernel in csrc/conv_umma.cu) under every tile -> warpgroup assignment.

The kernel gives a CTA's i-th tile to consumer warpgroup i & 1.  Capping the persistent grid at 1 .. 8 CTAs covers CTAs
with one tile, CTAs whose last tile falls to warpgroup 1 and CTAs whose last tile falls to warpgroup 0, on 9 ragged tiles
and on 32 whole ones.  Every grid must give the same bits, in fp32 and as pooled split planes, and stay within the float64
bound of tests/test_gpu_conv_layers.py.
"""
import numpy as np
import pytest

from omniswarm_b200 import host
from oracle import split_model as sm
from test_gpu_conv_layers import LAYERS, SA, planes_of, run_and_check

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

RES64 = LAYERS[0]
assert RES64[0] == "n64_resident_64to64_k3"
GEOMS = [(1, 20, 40), (2, 26, 50)]               # (B, H, W): 3 x 3 ragged tiles; 2 x 4 x 4 tiles


def outputs(w, b, hi, lo, max_ctas):
    f32 = host.conv_layer_parity(w, b, hi, lo, SA, relu=1, max_ctas=max_ctas)
    phi, plo = host.conv_layer_parity(w, b, hi, lo, SA, relu=1, pool=1, mode="planes", out_scale=SA, max_ctas=max_ctas)
    return [t.cpu().numpy() for t in (f32, phi, plo)]


@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: "B{}_{}x{}".format(*g))
def test_every_grid_gives_the_same_bits(geom):
    B, H, W = geom
    x, w, b = sm.make_case("relu_gauss", B, H, W, 64, 64, 3, seed=12)
    hi, lo, _ = planes_of(x)
    ref = outputs(w, b, hi, lo, 0)
    for m in range(1, 9):
        for name, got, want in zip(("fp32", "hi plane", "lo plane"), outputs(w, b, hi, lo, m), ref):
            assert np.array_equal(got, want, equal_nan=True), f"max_ctas {m}: {name} differs from the full grid"


@pytest.mark.parametrize("max_ctas", [1, 2, 3, 8])
@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: "B{}_{}x{}".format(*g))
def test_capped_grid_within_float64_bound(geom, max_ctas):
    B, H, W = geom
    run_and_check(RES64, B, H, W, "relu_gauss", 1, 1, "planes", seed=13, max_ctas=max_ctas)
    run_and_check(RES64, B, H, W, "signed", 0, 0, "f32", seed=14, max_ctas=max_ctas)
