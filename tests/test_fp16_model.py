"""CPU: the bounds of the plain-fp16 GPU tests (tests/test_gpu_fp16_mode.py) can fail.

Layers: the fp16 layer model (oracle.fp16_ref.fp16_conv_model, split_model.conv_model with zero lo planes) stays within
the split tests' float64 bound TAU * (sum |x| |w| + |b|) on the dequantised hi operands, and a dropped tap, a dropped
64-channel slab or a nonzero lo plane read by mistake each exceeds it.
Networks: the tolerance is NET_TOL_FACTOR x the difference between the float64 and the float32-accumulated emulation of
the whole network.  A dropped tap or slab exceeds it by two orders of magnitude.  A lo plane read by mistake does not:
once an accumulation order flips fp16 roundings, the flips cascade through the ReLUs and pools and move the outputs by
5e-4 .. 2e-3 relative, about what reading every activation unrounded moves them by -- so that defect is left to the layer
tests, where it exceeds the bound 20-fold.
"""
import numpy as np
import pytest

from omniswarm_b200 import synth
from oracle import fp16_ref as f16
from oracle import split_model as sm

SA, SW = f16.SA, f16.SW
SHAPES = [(64, 64, 3), (128, 128, 3), (512, 128, 1), (256, 256, 1)]


def layer_errors(cin, cout, ks):
    """{variant: max over the regimes of max |y - y64| / (sum |x||w| + |b|)}, y64 on the hi operands"""
    out = {}
    for seed, regime in enumerate(sm.REGIMES):
        x, w, b = sm.make_case(regime, 1, 5, 9, cin, cout, ks, seed=seed)
        xh, xl = sm.split(x, SA)
        wh, _ = sm.split_weights(w, SW)
        w64 = (wh.astype(np.float64) / SW).transpose(1, 2, 0).reshape(cout, cin, ks, ks)
        y64, d = sm.conv_f64(xh.astype(np.float64) / SA, w64, b, ks)
        slab_gone = xh.copy(); slab_gone[..., :64] = 0
        variants = {
            "faithful_rz": f16.fp16_conv_model(xh, wh, b, ks, SA, SW, rounding="rz"),
            "faithful_rn": f16.fp16_conv_model(xh, wh, b, ks, SA, SW, rounding="rn"),
            "slab_missing": f16.fp16_conv_model(slab_gone, wh, b, ks, SA, SW),
            "lo_read": sm.conv_model(xh, xl, wh, np.zeros_like(wh), b, ks, SA, SW),
        }
        if ks == 3:
            variants["tap_missing"] = f16.fp16_conv_model(xh, wh, b, ks, SA, SW, mutant="tap_missing")
        for name, y in variants.items():
            out[name] = max(out.get(name, 0.0), float((np.abs(y - y64) / d).max()))
    return out


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "{}to{}_k{}".format(*s))
def test_layer_bound_separates_faithful_from_defects(shape):
    e = layer_errors(*shape)
    print(shape, {k: f"{v:.2e}" for k, v in e.items()})
    assert e["faithful_rz"] < sm.TAU / 4 and e["faithful_rn"] < sm.TAU / 4, e
    for m in ("slab_missing", "lo_read", "tap_missing"):
        if m in e:
            assert e[m] > sm.TAU, f"{m} stays within the bound ({e[m]:.2e} <= {sm.TAU:.0e})"


def test_fp16_layer_model_is_the_split_model_without_lo():
    x, w, b = sm.make_case("relu_gauss", 1, 4, 6, 64, 64, 3, seed=3)
    xh, _ = sm.split(x, SA)
    wh, _ = sm.split_weights(w, SW)
    z = lambda a: np.zeros_like(a)
    assert np.array_equal(f16.fp16_conv_model(xh, wh, b, 3, SA, SW, relu=1),
                          sm.conv_model(xh, z(xh), wh, z(wh), b, 3, SA, SW, relu=1))


IMAGES = [synth.image(41, 64, 96), synth.image(42, 64, 96, zero_bottom_quarter=True)]


@pytest.fixture(scope="module")
def tolerances():
    return f16.network_tolerances(IMAGES, synth.superpoint_weights(0), synth.netvlad_weights(0))


def test_network_tolerance_separates_defects(tolerances):
    """A dropped tap or slab moves every network output by more than its tolerance; the lo-plane read is reported."""
    wsp, wnv = synth.superpoint_weights(0), synth.netvlad_weights(0)
    print({k: f"{v:.2e}" for k, v in tolerances.items()})
    for m in f16.NET_MUTANTS:
        worst = {"semi": 0.0, "desc": 0.0, "vlad": 0.0}
        for img in IMAGES:
            s, d = f16.superpoint_net_fp16(img, wsp)
            sm_, dm = f16.superpoint_net_fp16(img, wsp, mutant=m)
            worst["semi"] = max(worst["semi"], f16.rel(sm_, s))
            worst["desc"] = max(worst["desc"], f16.rel(dm, d))
            worst["vlad"] = max(worst["vlad"], f16.rel(f16.netvlad_net_fp16(img, wnv, mutant=m), f16.netvlad_net_fp16(img, wnv)))
        print(m, {k: f"{v:.2e} ({v / tolerances[k]:.1f}x)" for k, v in worst.items()})
        if m == "lo_read":
            continue
        assert worst["desc"] > tolerances["desc"] and worst["semi"] > tolerances["semi"], (m, worst)
        assert worst["vlad"] > tolerances["vlad"], (m, worst)


def test_fp16_network_is_near_the_fp32_network():
    """The emulation is the fp32 oracle up to fp16 operand rounding: 1e-3 .. 4e-3 relative.  That is below the
    emulation's own tolerance: at network level an fp16 network is only as well defined as its rounding flips."""
    from oracle import frontend_ref as fr
    wsp, wnv = synth.superpoint_weights(0), synth.netvlad_weights(0)
    for img in IMAGES:
        s, d = f16.superpoint_net_fp16(img, wsp)
        s32, d32 = fr.superpoint_net(img, wsp)
        v, v32 = f16.netvlad_net_fp16(img, wnv), fr.netvlad_net(img, wnv)
        e = {"semi": f16.rel(s, s32), "desc": f16.rel(d, d32), "vlad": f16.rel(v, v32)}
        print({k: f"{x:.2e}" for k, x in e.items()})
        assert all(1e-5 < x < 2e-2 for x in e.values()), e
