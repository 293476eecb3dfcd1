"""The 128-channel streamed layers (conv_stream_t_kernel in csrc/conv_umma.cu) under every grid and warpgroup skew.

Both consumer warpgroups of a CTA compute the same work item, 64 output channels each, from one ring of A boxes and
their own rings of weight rows; warpgroup 1 starts a box behind warpgroup 0 and the two stay apart.  Capping the
persistent grid at 1, 2, 3 or 8 CTAs gives CTAs one item or many, and an item count that does or does not divide
among them.  Every grid must give the same bits, for 3x3 and 1x1 layers, 128 channels and 256 / 512 as 2 / 4 items per
tile, pooled and unpooled planes and fp32 outputs, in both precisions, and capped grids stay within the float64 bound
of tests/test_gpu_conv_layers.py on ragged and sub-tile geometries.
"""
import numpy as np
import pytest

from omniswarm_b200 import host
from oracle import split_model as sm
from test_gpu_conv_layers import LAYERS, SA, planes_of, run_and_check
import test_gpu_fp16_mode as f16_mode

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

STREAMED = [l for l in LAYERS if l[4] >= 128]
assert [l[0] for l in STREAMED] == ["n128_64to128_k3", "n128_128to128_k3", "n128_512to128_k1", "nsplit2_128to256_k3",
                                    "nsplit2_256to256_k1", "nsplit4_256to512_k1", "nsplit4_512to512_k1"]
BITS = [STREAMED[i] for i in (0, 2, 3, 4, 5)]            # 3x3 / 1x1 x n_split 1 / 2 / 4
CAPS = [1, 2, 3, 8]
GEOM = (2, 26, 50)                                       # 2 x 4 x 4 tiles, ragged in both directions
RAGGED = [(3, 7, 17), (1, 3, 5), (1, 30, 40)]


def outputs(layer, x, w, b, fp16, max_ctas):
    """fp32, fp32 pooled, planes, planes pooled of one layer, as numpy"""
    out = []
    if fp16:
        hi, _ = f16_mode.hi_plane(x)
        run = lambda **kw: host.conv_layer_fp16_parity(w, b, hi, SA, relu=1, max_ctas=max_ctas, **kw)
        for pool in (0, 1):
            out += [run(pool=pool), run(pool=pool, mode="planes", out_scale=SA)]
    else:
        hi, lo, _ = planes_of(x)
        run = lambda **kw: host.conv_layer_parity(w, b, hi, lo, SA, relu=1, max_ctas=max_ctas, **kw)
        for pool in (0, 1):
            out += [run(pool=pool), *run(pool=pool, mode="planes", out_scale=SA)]
    return [t.cpu().numpy() for t in out]


@pytest.mark.parametrize("fp16", [False, True], ids=["split", "fp16"])
@pytest.mark.parametrize("layer", BITS, ids=[l[0] for l in BITS])
def test_every_grid_gives_the_same_bits(layer, fp16):
    name, cin, cout, ks, _ = layer
    x, w, b = sm.make_case("relu_gauss", *GEOM, cin, cout, ks, seed=21)
    ref = outputs(layer, x, w, b, fp16, 0)
    for m in CAPS:
        for i, (got, want) in enumerate(zip(outputs(layer, x, w, b, fp16, m), ref)):
            assert np.array_equal(got, want, equal_nan=True), f"{name} max_ctas {m}: output {i} differs from the full grid"


@pytest.mark.parametrize("max_ctas", CAPS)
@pytest.mark.parametrize("geom", RAGGED, ids=lambda g: "B{}_{}x{}".format(*g))
@pytest.mark.parametrize("layer", BITS, ids=[l[0] for l in BITS])
def test_capped_grid_within_float64_bound(layer, geom, max_ctas):
    B, H, W = geom
    pool = int(H % 2 == 0 and W % 2 == 0)
    run_and_check(layer, B, H, W, "relu_gauss", 1, pool, "planes", seed=22, max_ctas=max_ctas)
    run_and_check(layer, B, H, W, "signed", 0, 0, "f32", seed=23, max_ctas=max_ctas)
    f16_mode.run_and_check(layer, B, H, W, "relu_gauss", 2, pool, "planes", seed=24, max_ctas=max_ctas)
    f16_mode.run_and_check(layer, B, H, W, "signed", 0, 0, "f32", seed=25, max_ctas=max_ctas)
