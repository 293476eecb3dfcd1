"""The 16-byte plane stores of conv_umma_kernel (csrc/conv_umma.cu) when fewer channels are stored than the kernel computes.

Unpooled split planes of the N = 64 / 128 instantiations leave the kernel as one 16-byte store per 8-channel block, after
four blocks are transposed across each lane quad.  A block past `out_c` must not be written even when other blocks of its
group of four are, and the destination may be wider than `out_c` (`out_cstride`).  Every stored value must be within the
float64 bound of tests/test_gpu_conv_layers.py, and every channel the layer does not own must keep the NaN it was filled
with.
"""
import numpy as np
import pytest

from omniswarm_b200 import host
from oracle import split_model as sm
from test_gpu_conv_layers import SA, TAU, act, check_bound, check_planes, planes_of, ref64, w_rep

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

# (id, cin, cout, ks, out_c, out_cstride): out_c ends inside a group of four blocks, or inside a second channel block
CASES = [
    ("n128_64to96_k3", 64, 96, 3, 96, 104),
    ("n128_128to80_k1", 128, 112, 1, 80, 120),
    ("n64_128to48_k3", 128, 48, 3, 48, 56),
    ("nsplit2_128to256_k3", 128, 256, 3, 208, 216),
]


@pytest.mark.parametrize("geom", [(1, 8, 16), (2, 7, 17)], ids=lambda g: "B{}_{}x{}".format(*g))
@pytest.mark.parametrize("case", CASES, ids=lambda c: c[0])
def test_partial_channel_groups(case, geom):
    name, cin, cout, ks, out_c, stride = case
    B, H, W = geom
    x, w, b = sm.make_case("relu_gauss", B, H, W, cin, cout, ks, seed=31)
    hi, lo, x64 = planes_of(x)
    y64, d = ref64(x64, w_rep(w), b, ks)
    ohi, olo = host.conv_layer_parity(w, b, hi, lo, SA, relu=1, out_c=out_c, out_cstride=stride, mode="planes",
                                      out_scale=SA)
    assert torch.isnan(ohi[..., out_c:]).all() and torch.isnan(olo[..., out_c:]).all(), \
        f"{name}: channels past out_c were written"
    y = check_planes(ohi[..., :out_c], olo[..., :out_c], name)
    check_bound(y, act(y64, 1)[..., :out_c], TAU * d[..., :out_c] + 2.0 ** -25 / SA, f"{name} {geom}")
