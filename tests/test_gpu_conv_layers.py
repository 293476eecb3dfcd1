"""The tensor-core convolutions (csrc/conv_umma.cu) layer by layer against a float64 reference.

Each test feeds one layer, through the parity hooks of the C ABI, split planes it built itself, and compares the output
with the float64 convolution of the DEQUANTISED operands (x = (hi + lo) / s, the weights rebuilt from the same split), so
that the rounding of the inputs is not charged to the kernel.  Per output element

    |y - y64| <= TAU * (sum |x| |w| + |b|)

with TAU = oracle.split_model.TAU.  tests/test_split_model.py shows, on a CPU model of the split arithmetic, that the
faithful arithmetic stays below TAU / 4 while one missing lo plane of one slab of one tap, one dropped cross product, a
missing tap, a shifted box or a wrong n_split block each exceed it.  The measured maxima are in DESIGN.md section 4.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from omniswarm_b200 import host, lib, synth
from oracle import split_model as sm

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

TAU = sm.TAU
SA, SW = 16.0, 1024.0                    # SP_ACT_SCALE / NV_ACT_SCALE, SP_W_SCALE / NV_W_SCALE
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# every instantiation of conv_umma_kernel the networks reach: (id, cin, cout, ks, out_c)
LAYERS = [
    ("n64_resident_64to64_k3", 64, 64, 3, 64),
    ("n64_streamed_64to64_k1", 64, 64, 1, 64),
    ("n64_streamed_128to64_k3", 128, 64, 3, 64),
    ("n80_f32_256to65_k1", 256, 65, 1, 80),
    ("n128_64to128_k3", 64, 128, 3, 128),
    ("n128_128to128_k3", 128, 128, 3, 128),
    ("n128_512to128_k1", 512, 128, 1, 128),
    ("nsplit2_128to256_k3", 128, 256, 3, 256),
    ("nsplit2_256to256_k1", 256, 256, 1, 256),
    ("nsplit4_256to512_k1", 256, 512, 1, 512),
    ("nsplit4_512to512_k1", 512, 512, 1, 512),
]
LAYER_IDS = [l[0] for l in LAYERS]
SMALL = [(1, 8, 16), (3, 1, 1), (1, 3, 5), (3, 7, 17)]          # (B, H, W): one tile, sub-tile maps, ragged tiles
LARGE = [(3, 26, 50), (1, 60, 80)]                             # 400 x 208 at 1/8 resolution; 640 x 480 at 1/8


def dev():
    return torch.device("cuda")


def planes_of(x):
    """fp32 numpy [B,H,W,C] -> CUDA fp16 planes at SA and the float64 value they represent"""
    hi, lo = sm.split(x, SA)
    return (torch.from_numpy(hi).to(dev()), torch.from_numpy(lo).to(dev()), sm.dequant(hi, lo, SA))


def w_rep(w):
    """the weights the kernel multiplies: the x1024 split planes, dequantised, OIHW float64"""
    hi, lo = sm.split(w, SW)
    return sm.dequant(hi, lo, SW)


def ref64(x64, w64, b, ks):
    """float64 convolution and its error scale sum |x| |w| + |b| on the GPU, [B,H,W,Cout] numpy"""
    F = torch.nn.functional
    xt = torch.from_numpy(np.ascontiguousarray(x64.transpose(0, 3, 1, 2))).to(dev())
    wt, bt = torch.from_numpy(w64).to(dev()), torch.from_numpy(np.asarray(b, np.float64)).to(dev())
    y = F.conv2d(xt, wt, bt, padding=ks // 2)
    d = F.conv2d(xt.abs(), wt.abs(), bt.abs(), padding=ks // 2)
    return y.permute(0, 2, 3, 1).cpu().numpy(), d.permute(0, 2, 3, 1).cpu().numpy()


def act(y, relu):
    if relu:
        y = np.maximum(y, 0.0)
    return np.minimum(y, 6.0) if relu == 2 else y


def pool2(a):
    B, H, W, C = a.shape
    return a.reshape(B, H // 2, 2, W // 2, 2, C).max(axis=(2, 4))


def check_bound(y, ref, bound, what):
    """every element finite and within its bound; returns the largest |y - ref| / bound * TAU (the normalised error)"""
    y = np.asarray(y, np.float64)
    assert np.isfinite(y).all(), f"{what}: {np.count_nonzero(~np.isfinite(y))} non-finite outputs"
    r = np.abs(y - ref) / bound
    worst = np.unravel_index(np.argmax(r), r.shape)
    assert r.max() <= 1.0, (f"{what}: error {np.abs(y - ref)[worst]:.3e} at {worst} is {r.max():.2f}x its bound "
                            f"(y {y[worst]:.8g}, float64 {ref[worst]:.8g})")
    return float(r.max()) * TAU


def check_planes(hi, lo, what):
    """the split invariant of stored planes: |lo| <= ulp(hi) / 2 and hi == fp16(hi + lo).  The one exception is a tie:
    when the remainder rounds to exactly half an ulp, hi + lo lies midway between two fp16 values and rounds to the even
    one, which need not be hi (numpy's own split does the same, about once in 7000 values)."""
    h, l = hi.cpu().numpy(), lo.cpu().numpy()
    assert np.isfinite(h).all() and np.isfinite(l).all(), f"{what}: non-finite planes"
    half = 0.5 * np.spacing(np.abs(h)).astype(np.float64)
    a = np.abs(l.astype(np.float64))
    assert (a <= half).all(), f"{what}: |lo| exceeds half an ulp of hi"
    s = h.astype(np.float32) + l.astype(np.float32)
    ok = (s.astype(np.float16) == h) | (a == half)
    assert ok.all(), f"{what}: {np.count_nonzero(~ok)} values where hi is not the rounded value of hi + lo"
    return sm.dequant(h, l, SA)


def run_and_check(layer, B, H, W, regime, relu, pool, mode, seed=0, max_ctas=0):
    name, cin, cout, ks, out_c = layer
    x, w, b = sm.make_case(regime, B, H, W, cin, cout, ks, seed)
    hi, lo, x64 = planes_of(x)
    y64, d = ref64(x64, w_rep(w), b, ks)
    ref, bound = act(y64, relu), TAU * d
    if pool:
        ref, bound = pool2(ref), pool2(bound)
    what = f"{name} {B}x{H}x{W} {regime} relu={relu} pool={pool} {mode}"
    if mode == "f32":
        y = host.conv_layer_parity(w, b, hi, lo, SA, relu=relu, pool=pool, out_c=out_c, max_ctas=max_ctas)
        y = y.cpu().numpy()
        assert (y[..., cout:out_c] == 0).all(), "the padding channels of the layer must be stored as 0"
        y = y[..., :cout]
    else:
        ohi, olo = host.conv_layer_parity(w, b, hi, lo, SA, relu=relu, pool=pool, out_c=out_c, mode="planes",
                                          out_scale=SA, max_ctas=max_ctas)
        y = check_planes(ohi[..., :out_c], olo[..., :out_c], what)[..., :cout]
        bound = bound + 2.0 ** -25 / SA          # the fp16 rounding of lo when the stored value is tiny
    return check_bound(y, ref[..., :cout], bound[..., :cout], what)


@pytest.mark.parametrize("geom", SMALL, ids=lambda g: "B{}_{}x{}".format(*g))
@pytest.mark.parametrize("layer", LAYERS, ids=LAYER_IDS)
def test_layer_vs_float64_small(layer, geom):
    """Every instantiation x the small geometries x every value regime, activations and output forms alternating."""
    B, H, W = geom
    worst = 0.0
    for i, regime in enumerate(sm.REGIMES):
        relu = i % 3
        mode = "planes" if (i % 2 == 1 and layer[2] == layer[4]) else "f32"
        pool = int(H % 2 == 0 and W % 2 == 0 and i % 2 == 0)
        worst = max(worst, run_and_check(layer, B, H, W, regime, relu, pool, mode, seed=i))
    print(f"{layer[0]} B{B} {H}x{W}: max normalised error {worst:.3e}")


@pytest.mark.parametrize("geom", LARGE, ids=lambda g: "B{}_{}x{}".format(*g))
@pytest.mark.parametrize("layer", LAYERS, ids=LAYER_IDS)
def test_layer_vs_float64_large(layer, geom):
    """The feature-map sizes of 400 x 208 and 640 x 480 images at 1/8 resolution: pooled planes and fp32 output."""
    B, H, W = geom
    mode = "planes" if layer[2] == layer[4] else "f32"
    e1 = run_and_check(layer, B, H, W, "relu_gauss", 1, 1, mode, seed=1)
    e2 = run_and_check(layer, B, H, W, "ramp", 0, 0, "f32", seed=2)
    print(f"{layer[0]} B{B} {H}x{W}: max normalised error {max(e1, e2):.3e}")


def test_full_resolution_resident_layer():
    """conv1b at 640 x 480 (the resident-weight N = 64 kernel over 2400 tiles), ReLU + pool into planes."""
    run_and_check(LAYERS[0], 1, 480, 640, "relu_gauss", 1, 1, "planes", seed=3)


@pytest.mark.parametrize("geom", [(1, 8, 16), (3, 3, 5), (1, 26, 50)], ids=lambda g: "B{}_{}x{}".format(*g))
@pytest.mark.parametrize("regime", ["relu_gauss", "signed", "bias_dominant"])
def test_detector_head_softmax_vs_float64(geom, regime):
    """convPb (256 -> 65) with the softmax + pixel shuffle epilogue.  A logit error of at most e moves log p by at most
    2e; the fp32 softmax itself (expf, a 65-term sum, one division) adds at most 5e-6 relative."""
    B, H, W = geom
    x, w, b = sm.make_case(regime, B, H, W, 256, 65, 1, seed=4)
    hi, lo, x64 = planes_of(x)
    z, d = ref64(x64, w_rep(w), b, 1)
    p = np.exp(z - z.max(axis=-1, keepdims=True))
    p /= p.sum(axis=-1, keepdims=True)
    dz = 2.0 * TAU * d.max(axis=-1, keepdims=True)
    bound = p * (np.expm1(dz) + 5e-6) + 1e-37
    shuffle = lambda a: a[..., :64].reshape(B, H, W, 8, 8).transpose(0, 1, 3, 2, 4).reshape(B, 8 * H, 8 * W)
    heat = host.conv_layer_parity(w, b, hi, lo, SA, mode="softmax").cpu().numpy()
    worst = check_bound(heat, shuffle(p), shuffle(bound), f"softmax head {geom} {regime}")
    print(f"softmax head {geom} {regime}: {worst / TAU:.3f} of the bound")


# ---------------------------------------------------------------------------------------------------------------------
# invariances (bit-exact)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layer", [LAYERS[0], LAYERS[3], LAYERS[7], LAYERS[10]], ids=lambda l: l[0])
def test_max_ctas_does_not_change_the_result(layer):
    """The persistent grid capped at 1 and 5 CTAs (as head_ctas caps it beside the keypoint kernel) walks the same tiles
    in another order per CTA: the output must be bit-identical."""
    name, cin, cout, ks, out_c = layer
    x, w, b = sm.make_case("relu_gauss", 2, 26, 50, cin, cout, ks, seed=5)
    hi, lo, _ = planes_of(x)
    outs = [host.conv_layer_parity(w, b, hi, lo, SA, relu=1, out_c=out_c, max_ctas=m).cpu().numpy() for m in (0, 1, 5)]
    assert np.array_equal(outs[0], outs[1], equal_nan=True) and np.array_equal(outs[0], outs[2], equal_nan=True)


@pytest.mark.parametrize("layer", [LAYERS[0], LAYERS[2], LAYERS[8]], ids=lambda l: l[0])
def test_batch_slot_does_not_change_the_result(layer):
    """An image alone and in slot 2 of a batch of 3 (other images in slots 0 and 1) gives the same bits."""
    name, cin, cout, ks, out_c = layer
    x, w, b = sm.make_case("relu_gauss", 3, 7, 17, cin, cout, ks, seed=6)
    hi, lo, _ = planes_of(x)
    batch = host.conv_layer_parity(w, b, hi, lo, SA, relu=1, out_c=out_c).cpu().numpy()
    one = host.conv_layer_parity(w, b, hi[2:].contiguous(), lo[2:].contiguous(), SA, relu=1, out_c=out_c).cpu().numpy()
    assert np.array_equal(batch[2:], one, equal_nan=True)


def _superpoint_outputs(W, H, imgs):
    comp, mean = synth.pca_matrices(0)
    sp = host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, W, H, 0.015, 200,
                         max_batch=len(imgs))
    sp.inference_batch(imgs)
    out = [(sp.read("semi", b), sp.read("desc", b)) for b in range(len(imgs))]
    sp.close()
    return out


def test_programmatic_dependent_launch_is_bit_identical(tmp_path):
    """OSB_CONV_PDL=1 (read when the library loads, hence a fresh process) must not change one bit of the network."""
    W, H = 400, 208
    imgs = np.stack([synth.image(31, H, W), synth.image(32, H, W, zero_bottom_quarter=True)])
    np.save(tmp_path / "imgs.npy", imgs)
    code = ("import sys, numpy as np; sys.path.insert(0, sys.argv[1]); "
            "from omniswarm_b200 import host, synth; "
            "imgs = np.load(sys.argv[2]); comp, mean = synth.pca_matrices(0); "
            "sp = host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, 400, 208, 0.015, "
            "200, max_batch=len(imgs)); sp.inference_batch(imgs); "
            "np.savez(sys.argv[3], **{f'{k}{b}': sp.read(k, b) for b in range(len(imgs)) for k in ('semi', 'desc')})")
    env = dict(os.environ, OSB_CONV_PDL="1")
    r = subprocess.run([sys.executable, "-c", code, ROOT, str(tmp_path / "imgs.npy"), str(tmp_path / "pdl.npz")],
                       env=env, capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    pdl = np.load(tmp_path / "pdl.npz")
    for b, (semi, desc) in enumerate(_superpoint_outputs(W, H, imgs)):
        assert np.array_equal(pdl[f"semi{b}"], semi) and np.array_equal(pdl[f"desc{b}"], desc), f"image {b}"


# ---------------------------------------------------------------------------------------------------------------------
# the kernels that write planes from fp32: depthwise 3x3 (NetVLAD) and conv1a (SuperPoint)
# ---------------------------------------------------------------------------------------------------------------------
def dw_ref(x, w, b, stride):
    F = torch.nn.functional
    xt = torch.from_numpy(np.ascontiguousarray(x.astype(np.float64).transpose(0, 3, 1, 2))).to(dev())
    wt = torch.from_numpy(w.astype(np.float64)).to(dev())
    bt = torch.from_numpy(b.astype(np.float64)).to(dev())
    C = x.shape[-1]
    y = F.conv2d(xt, wt, bt, stride=stride, padding=1, groups=C)
    d = F.conv2d(xt.abs(), wt.abs(), bt.abs(), stride=stride, padding=1, groups=C)
    return y.permute(0, 2, 3, 1).cpu().numpy(), d.permute(0, 2, 3, 1).cpu().numpy()


@pytest.mark.parametrize("shape", [(2, 7, 13, 128), (1, 26, 50, 64), (3, 1, 5, 256), (1, 48, 64, 512)],
                         ids=lambda s: "B{}_{}x{}_C{}".format(*s))
def test_depthwise_kernels_bit_identical_and_within_bound(shape):
    """dwconv3x3_split_s1x4_kernel (four pixels per thread) and dwconv3x3_split_kernel at stride 1 give the same planes
    bit for bit; both, and the stride-2 form, are within the float64 bound after ReLU6."""
    B, H, W, C = shape
    rng = np.random.default_rng(7)
    x = np.maximum(rng.standard_normal(shape), 0).astype(np.float32) * 3
    w = (rng.standard_normal((C, 1, 3, 3)) * 0.5).astype(np.float32)
    b = (rng.standard_normal(C) * 0.1).astype(np.float32)
    xt = torch.from_numpy(x).to(dev())
    h4, l4 = host.dwconv_parity(w, b, xt, SA)
    hg, lg = host.dwconv_parity(w, b, xt, SA, generic=True)
    assert torch.equal(h4, hg) and torch.equal(l4, lg), "stride-1 depthwise kernels differ"
    for stride in (1, 2):
        if stride == 2 and (H % 2 or W % 2):
            continue
        hi, lo = (h4, l4) if stride == 1 else host.dwconv_parity(w, b, xt, SA, stride=2)
        y64, d = dw_ref(x, w, b, stride)
        y = check_planes(hi, lo, f"dwconv {shape} s{stride}")
        check_bound(y, act(y64, 2), TAU * d + 2.0 ** -25 / SA, f"dwconv {shape} s{stride}")


def conv1a_ref(imgs):
    """the u8 -> fp32 input of conv1a exactly as the kernels form it: (float)v * (float)(1/255)"""
    return imgs.astype(np.float32) * np.float32(1.0 / 255.0)


@pytest.mark.parametrize("geom", [(1, 8, 16), (3, 7, 17), (2, 60, 80), (1, 480, 640)], ids=lambda g: "B{}_{}x{}".format(*g))
def test_first_layers_vs_float64(geom):
    """conv_first_split_kernel (conv1a + ReLU -> planes) within the float64 bound."""
    B, H, W = geom
    wsp = synth.superpoint_weights(0)
    w1a, b1a = wsp["conv1a.weight"], wsp["conv1a.bias"]
    rng = np.random.default_rng(8)
    imgs = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
    imgs[0, : H // 2, : W // 3] = 0
    it = torch.from_numpy(imgs).to(dev())
    hi, lo = host.conv_first_parity(w1a, b1a, it, SA)
    x = conv1a_ref(imgs)[..., None].astype(np.float64)
    y64, d = ref64(x, w1a.astype(np.float64), b1a, 3)
    a64 = check_planes(hi, lo, f"conv1a {geom}")
    check_bound(a64, act(y64, 1), TAU * d + 2.0 ** -25 / SA, f"conv1a {geom}")


# ---------------------------------------------------------------------------------------------------------------------
# the range of the planes
# ---------------------------------------------------------------------------------------------------------------------
def test_weights_outside_the_plane_range_are_rejected():
    """A weight w with fp16(1024 w) = inf cannot be split: the layer upload (and so the network constructors) fails with
    OSB_ERR_INVALID instead of computing with inf.  63.98 is the largest weight that still splits."""
    x, w, b = sm.make_case("relu_gauss", 1, 8, 16, 64, 64, 1, seed=9)
    hi, lo, x64 = planes_of(x)
    w[3, 5, 0, 0] = 63.98
    run = lambda: host.conv_layer_parity(w, b, hi, lo, SA)
    y = run().cpu().numpy()
    y64, d = ref64(x64, w_rep(w), b, 1)
    check_bound(y, y64, TAU * d, "weight 63.98")
    w[3, 5, 0, 0] = -64.0
    with pytest.raises(lib.OsbError) as e:
        run()
    assert e.value.status == lib.ERR_INVALID and "split-fp16 range" in str(e.value)

    comp, mean = synth.pca_matrices(0)
    wsp = synth.superpoint_weights(0)
    wsp["conv3a.weight"] = wsp["conv3a.weight"].copy()
    wsp["conv3a.weight"][7, 2, 1, 1] = 100.0
    with pytest.raises(lib.OsbError) as e:
        host.SuperPoint(synth.flatten_sp_weights(wsp), comp, mean, 96, 64, 0.015, 50, max_batch=1)
    assert e.value.status == lib.ERR_INVALID and "split-fp16 range" in str(e.value)
    nvw = synth.netvlad_weights(0)
    nvw["proj.weight"] = nvw["proj.weight"].copy()
    nvw["proj.weight"][0, 0, 0, 0] = -70.0
    with pytest.raises(lib.OsbError) as e:
        host.NetVLAD(synth.flatten_nv_weights(nvw), 96, 64, max_batch=1)
    assert e.value.status == lib.ERR_INVALID and "split-fp16 range" in str(e.value)


def test_activation_above_the_plane_limit_is_silently_zeroed():
    """Pins today's behaviour for an activation of 4095 or more (beyond fp16 at the x16 plane scale; conv_umma.cuh): the
    epilogue stores hi = +inf, lo = -inf; the next layer's sums at every pixel that reads it are NaN, and a ReLU there turns
    the NaN into 0 -- the overflow does not surface.  The shipped networks stay far below the limit
    (tests/test_split_model.py::test_shipped_networks_have_plane_headroom)."""
    x, w, b = sm.make_case("relu_gauss", 1, 8, 16, 64, 64, 1, seed=10)
    hi, lo, _ = planes_of(x)
    b = b.copy()
    b[9] = 5000.0                                  # channel 9 of every pixel overflows
    ohi, olo = host.conv_layer_parity(w, b, hi, lo, SA, relu=1, mode="planes", out_scale=SA)
    assert torch.isinf(ohi[..., 9]).all() and (ohi[..., 9] > 0).all() and (olo[..., 9] < 0).all() \
        and torch.isinf(olo[..., 9]).all()
    ok = torch.ones(64, dtype=torch.bool, device=dev())
    ok[9] = False
    assert torch.isfinite(ohi[..., ok]).all()
    x2, w2, b2 = sm.make_case("signed", 1, 8, 16, 64, 64, 1, seed=11)
    raw = host.conv_layer_parity(w2, b2, ohi, olo, SA, relu=0).cpu().numpy()
    assert np.isnan(raw).all()
    relu = host.conv_layer_parity(w2, b2, ohi, olo, SA, relu=1).cpu().numpy()
    assert (relu == 0).all()
