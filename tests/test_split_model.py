"""CPU: the float64 bound of the GPU layer tests (tests/test_gpu_conv_layers.py) can fail.

oracle/split_model.py models the split-fp16 arithmetic of csrc/conv_umma.cu step by step.  Over layer shapes with K from
64 to 4608 and the value regimes the GPU tests use, the faithful model (fp32 accumulation rounded toward zero, or to
nearest) must stay below TAU / 4 and each defect below must exceed TAU -- otherwise the GPU tests could pass a wrong
kernel.  The second test checks that the shipped networks use a small part of the range of the fp16 planes.
"""
import numpy as np
import pytest

from omniswarm_b200 import synth
from oracle import frontend_ref as fr
from oracle import split_model as sm

SA, SW = 16.0, 1024.0

# (cin, cout, ks): K = 64, 576, 1152, 512, 256 (two 128-channel work items) and 4608
SHAPES = [(64, 64, 1), (64, 64, 3), (128, 128, 3), (512, 128, 1), (256, 256, 1), (512, 128, 3)]


def normalised_errors(cin, cout, ks):
    """{variant: max over the regimes of max |y - y64| / (sum |x||w| + |b|)}"""
    out = {}
    for seed, regime in enumerate(sm.REGIMES):
        x, w, b = sm.make_case(regime, 1, 5, 9, cin, cout, ks, seed=seed)
        xh, xl = sm.split(x, SA)
        wh, wl = sm.split_weights(w, SW)
        w64 = sm.dequant(wh, wl, SW).transpose(1, 2, 0).reshape(cout, cin, ks, ks)
        y64, d = sm.conv_f64(sm.dequant(xh, xl, SA), w64, b, ks)
        variants = [("faithful_rz", "rz", None), ("faithful_rn", "rn", None)]
        variants += [(m, "rz", m) for m in sm.MUTANTS if m != "nsplit_rows" or cout >= 256]
        for name, rounding, mutant in variants:
            y = sm.conv_model(xh, xl, wh, wl, b, ks, SA, SW, rounding=rounding, mutant=mutant)
            out[name] = max(out.get(name, 0.0), float((np.abs(y - y64) / d).max()))
    return out


@pytest.mark.parametrize("shape", SHAPES, ids=lambda s: "{}to{}_k{}".format(*s))
def test_tolerance_separates_faithful_from_mutants(shape):
    e = normalised_errors(*shape)
    print(shape, {k: f"{v:.2e}" for k, v in e.items()})
    assert e["faithful_rz"] < sm.TAU / 4 and e["faithful_rn"] < sm.TAU / 4, e
    for m in sm.MUTANTS:
        if m in e:
            assert e[m] > sm.TAU, f"mutant {m} stays within the bound ({e[m]:.2e} <= {sm.TAU:.0e})"


def test_model_split_is_the_kernels_split():
    """hi = fp16(s x) rounded to nearest even, lo the fp16 of the exact remainder; hi + lo carries 22 bits."""
    x = np.array([1.0, 1.0 / 3.0, 4094.0, 2.0 ** -12, -0.1, 1e-6], np.float32)
    hi, lo = sm.split(x, SA)
    assert np.array_equal(hi, (x * np.float32(SA)).astype(np.float16))
    assert np.array_equal((hi.astype(np.float32) + lo.astype(np.float32)).astype(np.float16), hi)
    rel = np.abs(sm.dequant(hi, lo, SA) - x.astype(np.float64)) / np.abs(x.astype(np.float64))
    assert rel[:5].max() < 2.0 ** -21
    over, _ = sm.split(np.float32([4095.0, -4095.0]), SA)
    assert np.isinf(over).all()                               # the plane limit of conv_umma.cuh


def test_shipped_networks_have_plane_headroom():
    """Every operand the tensor-core layers of the synthetic SuperPoint and NetVLAD see stays at least 8x below the fp16
    plane limit: max |activation| * 16 and max |weight| * 1024 below 65520 / 8."""
    limit = sm.FP16_MAX_FINITE_SPLIT / 8
    sp, nv = {}, {}
    wsp, wnv = synth.superpoint_weights(0), synth.netvlad_weights(0)
    for seed in range(2):
        img = synth.image(seed, zero_bottom_quarter=bool(seed))
        tr = {}
        fr.superpoint_net(img, wsp, trace=tr)
        for k, v in tr.items():
            sp[k] = np.maximum(sp.get(k, (0.0, 0.0)), v)
        tr = {}
        fr.netvlad_net(img, wnv, trace=tr)
        for k, v in tr.items():
            nv[k] = np.maximum(nv.get(k, (0.0, 0.0)), v)
    tensor_core = {k: v for k, v in sp.items() if k != "conv1a"}      # conv1a runs in fp32 FFMA on the image
    tensor_core.update({k: v for k, v in nv.items() if k != "b0.pw"})  # block 0 runs fused in fp32
    assert len(tensor_core) == 11 + 7
    for k, (a, w) in tensor_core.items():
        print(f"{k}: max |x| {a:.3g} (x16 = {a * SA:.3g}), max |w| {w:.3g} (x1024 = {w * SW:.3g})")
        assert a * SA < limit, f"{k}: activations reach {a:.4g}, within 8x of the plane limit"
        assert w * SW < limit, f"{k}: weights reach {w:.4g}, within 8x of the plane limit"
