"""The fp32 CUDA-core kernels stage by stage against a float64 reference: the FFMA convolutions (csrc/conv_ffma.cu, the
OSB_SP_CONV=ffma path and the A/B reference of the tensor-core path), the first layers, depthwise 3x3, max-pool, and
NetVLAD's fused block 0 and head (csrc/netvlad.cu).

Each stage runs through a parity hook of the C ABI (the host functions the networks call) on fp32 inputs the test builds,
or on the device's own output of the previous stage, and every output element must lie within the fp32 forward-error
bound of oracle/fp32_bounds.py (the VLAD vector, per cluster and whole, and the centring against the float64 mean, per
location, are bounded normwise); tests/test_fp32_bounds.py shows on the CPU that those bounds fail for a skipped K chunk,
a shifted halo, a dropped VLAD slice or location, a lost VLAD dimension, another slot's mean, a skewed row stride or a
softmax without its max shift.
Outputs are pre-filled with NaN, so anything a kernel does not write fails.  Each test prints the largest fraction of its
bound it used (FRACTION lines); DESIGN.md section 4 records them.
"""
import numpy as np
import pytest

from omniswarm_b200 import host, lib, synth
from oracle import fp32_bounds as fb
from oracle import frontend_ref as fr

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
DEV = "cuda"


def launches(fn, expected, *args, **kw):
    """run a hook and check how many kernels it launched (each hook runs the network's own launch sequence)"""
    n0 = host.launch_count()
    out = fn(*args, **kw)
    assert host.launch_count() - n0 == expected, f"{fn.__name__} launched {host.launch_count() - n0} kernels"
    return out


def check(y, ref, bound, what):
    """every element finite and within its bound; returns the largest fraction of the bound used"""
    y = np.asarray(y, np.float64)
    assert np.isfinite(y).all(), f"{what}: {np.count_nonzero(~np.isfinite(y))} non-finite outputs"
    err = np.abs(y - ref)
    r = np.where(err == 0, 0.0, err / np.where(bound > 0, bound, 1e-300))
    worst = np.unravel_index(np.argmax(r), r.shape)
    assert r.max() <= 1.0, (f"{what}: error {err[worst]:.3e} at {worst} is {r.max():.3g}x its bound {bound[worst]:.3e} "
                            f"(y {y[worst]:.9g}, float64 {ref[worst]:.9g})")
    return float(r.max())


def check_norm(y, ref, bound, what):
    """the same normwise: ||y - ref|| over the last axis within its bound for every leading index"""
    y = np.asarray(y, np.float64)
    assert np.isfinite(y).all(), f"{what}: {np.count_nonzero(~np.isfinite(y))} non-finite outputs"
    err = np.linalg.norm(y - ref, axis=-1)
    r = np.where(err == 0, 0.0, err / np.where(bound > 0, bound, 1e-300))
    worst = np.unravel_index(np.argmax(r), r.shape)
    assert r.max() <= 1.0, f"{what}: error norm {err[worst]:.3e} at {worst} is {r.max():.3g}x its bound {bound[worst]:.3e}"
    return float(r.max())


def report(what, frac):
    print(f"FRACTION {what} {frac:.3e}")


def cuda(a):
    return torch.from_numpy(np.ascontiguousarray(a)).to(DEV)


# ---------------------------------------------------------------------------------------------------------------------
# FFMA convolutions: every (cin, cout, ks, out_cstride, act) the two networks run on the FFMA path
# ---------------------------------------------------------------------------------------------------------------------
LAYERS = [
    ("sp_64to64_k3", 64, 64, 3, 64, 1), ("sp_64to128_k3", 64, 128, 3, 128, 1), ("sp_128to128_k3", 128, 128, 3, 128, 1),
    ("sp_128to256_k3", 128, 256, 3, 256, 1), ("sp_256to256_k1", 256, 256, 1, 256, 0),
    ("sp_256to65_k1_s72", 256, 65, 1, 72, 0),
    ("nv_32to64", 32, 64, 1, 64, 2), ("nv_64to128", 64, 128, 1, 128, 2), ("nv_128to128", 128, 128, 1, 128, 2),
    ("nv_128to256", 128, 256, 1, 256, 2), ("nv_256to256", 256, 256, 1, 256, 2), ("nv_256to512", 256, 512, 1, 512, 2),
    ("nv_512to512", 512, 512, 1, 512, 2), ("nv_proj_512to128", 512, 128, 1, 128, 0),
    ("nv_assign_128to32_s32", 128, 32, 1, 32, 0),
]
GEOMS = [(1, 8, 32), (3, 1, 1), (1, 3, 5), (3, 7, 33), (1, 26, 50), (1, 60, 80)]


def layer_case(cin, cout, ks, B, H, W, seed):
    rng = np.random.default_rng(seed)
    x = np.clip(rng.standard_normal((B, H, W, cin)) * 2 + 0.5, 0, 6).astype(np.float32)
    w = (rng.standard_normal((cout, cin, ks, ks)) * np.sqrt(2.0 / (cin * ks * ks))).astype(np.float32)
    b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    return x, w, b


@pytest.mark.parametrize("geom", GEOMS, ids=lambda g: "B{}_{}x{}".format(*g))
@pytest.mark.parametrize("layer", LAYERS, ids=[l[0] for l in LAYERS])
def test_ffma_conv_vs_float64(layer, geom):
    """|y - y64| <= gamma_{K+1} (sum |x||w| + |b|); channels [cout, out_cstride) stored as 0, nothing written beyond"""
    name, cin, cout, ks, ocs, a = layer
    B, H, W = geom
    x, w, b = layer_case(cin, cout, ks, B, H, W, seed=cin + 7 * cout + H)
    worst = 0.0
    for act in sorted({a, 0}):
        y, guard = launches(host.conv_ffma_parity, 1, w, b, cuda(x), act=act, out_cstride=ocs, guard=True)
        y = y.cpu().numpy()
        assert torch.isnan(guard).all(), f"{name}: written beyond the last pixel's out_cstride channels"
        assert (y[..., cout:] == 0).all(), f"{name}: padding channels [cout, out_cstride) not stored as 0"
        y64, bound = fb.conv_ref(x, w, b, a=act, device=DEV)
        worst = max(worst, check(y[..., :cout], y64, bound, f"{name} {geom} act {act}"))
    report(f"ffma_conv {name} {geom}", worst)


def test_conv_first_vs_float64():
    """conv_first_kernel<64> stride 1 + ReLU (SuperPoint conv1a) and <32> stride 2 + ReLU6 (NetVLAD conv0); H/s x W/s
    not a multiple of the 128-pixel CTA in most cases"""
    wsp, wnv = synth.superpoint_weights(0), synth.netvlad_weights(0)
    rng = np.random.default_rng(8)
    worst = 0.0
    for (w, b, stride, act) in ((wsp["conv1a.weight"], wsp["conv1a.bias"], 1, 1),
                                (wnv["conv0.weight"], wnv["conv0.bias"], 2, 2)):
        for (B, H, W) in ((1, 8, 16), (3, 10, 34), (2, 60, 80), (2, 208, 400), (1, 480, 640)):
            imgs = rng.integers(0, 256, (B, H, W), dtype=np.uint8)
            imgs[0, : H // 2, : W // 3] = 0
            imgs[-1, H // 2:, W // 2:] = 255
            y = launches(host.conv_first_ffma_parity, 1, w, b, cuda(imgs), stride=stride, act=act).cpu().numpy()
            y64, bound = fb.first_ref(imgs, w, b, stride=stride, a=act, device=DEV)
            worst = max(worst, check(y, y64, bound, f"conv_first cout {w.shape[0]} s{stride} {B}x{H}x{W}"))
    report("conv_first", worst)


@pytest.mark.parametrize("C", [32, 64, 128, 256, 512])
def test_dwconv_and_maxpool_vs_float64(C):
    """dwconv3x3_kernel (gamma_10) at strides 1 and 2; maxpool2x2_kernel bit-exact"""
    rng = np.random.default_rng(C)
    w = (rng.standard_normal((C, 1, 3, 3)) * 0.5).astype(np.float32)
    b = (rng.standard_normal(C) * 0.1).astype(np.float32)
    worst = 0.0
    for (B, H, W) in ((2, 7, 13), (3, 8, 14), (1, 26, 50), (1, 2, 2)):
        x = (rng.standard_normal((B, H, W, C)) * 2).astype(np.float32)
        for stride in (1, 2):
            if stride == 2 and (H % 2 or W % 2):
                continue
            for act in (2, 0):
                y = launches(host.dwconv_ffma_parity, 1, w, b, cuda(x), stride=stride, act=act).cpu().numpy()
                y64, bound = fb.dwconv_ref(x, w, b, stride=stride, a=act, device=DEV)
                worst = max(worst, check(y, y64, bound, f"dwconv C{C} {B}x{H}x{W} s{stride} act {act}"))
        if H % 2 == 0 and W % 2 == 0:
            p = launches(host.maxpool_parity, 1, cuda(x)).cpu().numpy()
            assert np.array_equal(p, fb.maxpool_ref(x)), f"maxpool C{C} {B}x{H}x{W}"
    report(f"dwconv C{C}", worst)


# ---------------------------------------------------------------------------------------------------------------------
# NetVLAD block 0 (fused depthwise + pointwise)
# ---------------------------------------------------------------------------------------------------------------------
def block0_operands(seed):
    nvw = synth.netvlad_weights(seed)
    return nvw["b0.dw.weight"], nvw["b0.dw.bias"], nvw["b0.pw.weight"], nvw["b0.pw.bias"]


def block0_input(B, H, W, seed):
    rng = np.random.default_rng(seed)
    return np.clip(rng.standard_normal((B, H, W, 32)) * 2 + 1, 0, 6).astype(np.float32)


@pytest.mark.parametrize("geom", [(3, 8, 32), (1, 104, 200), (3, 13, 35), (2, 240, 320), (1, 5, 7)],
                         ids=lambda g: "B{}_{}x{}".format(*g))
def test_block0_vs_float64(geom):
    """w % 16 in {0, 8, 3}, h % 8 != 0 (guarded by the kernel though the network cannot reach it), B = 3; the depthwise
    bound composed through ReLU6 into the 33-term pointwise bound"""
    B, H, W = geom
    ops = block0_operands(0)
    x = block0_input(B, H, W, seed=H * W)
    y = launches(host.nv_block0_parity, 1, *ops, cuda(x)).cpu().numpy()
    y64, bound = fb.block0_ref(x, *ops, device=DEV)
    report(f"block0 {geom}", check(y, y64, bound, f"block0 {geom}"))


def test_block0_batch_slot_bit_exact():
    ops = block0_operands(0)
    x = block0_input(3, 13, 35, seed=11)
    batch = host.nv_block0_parity(*ops, cuda(x)).cpu().numpy()
    one = host.nv_block0_parity(*ops, cuda(x[2:])).cpu().numpy()
    assert np.array_equal(batch[2:], one)


# ---------------------------------------------------------------------------------------------------------------------
# NetVLAD head, stage by stage
# ---------------------------------------------------------------------------------------------------------------------
HEAD_LAUNCHES = 6            # colmean, centre + norm, assign conv, softmax, VLAD partial, VLAD final


def run_head(x4, ab, aw, cent):
    r = launches(host.nv_head_parity, HEAD_LAUNCHES, aw, ab, cent, cuda(x4))
    return {k: v.cpu().numpy() for k, v in r.items()}


def flat(a):
    return a.reshape(a.shape[0], -1, a.shape[-1])


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("regime", fb.HEAD_REGIMES)
@pytest.mark.parametrize("shape", fb.HEAD_SHAPES, ids=lambda s: "P{}".format(s[0] * s[1]))
def test_head_stages_vs_float64(shape, regime, B):
    h, w = shape
    P = h * w
    x4, ab, aw, cent = fb.head_case(regime, B, h, w, seed=P + B)
    x = flat(x4)
    r = run_head(x4, ab, aw, cent)
    what = f"head P{P} B{B} {regime}"
    frac = {}
    mu64, bmu = fb.mu_ref(x)
    frac["mu"] = check(r["mu"], mu64, bmu, what + " mu")
    xn = flat(r["xn"])
    frac["xn"] = check(xn, *fb.centre_ref(x, r["mu"]), what + " centred (device mu)")
    frac["xn_from_x"] = check_norm(xn, *fb.centre_from_x_ref(x), what + " centred (float64 mu)")
    if P == 1:
        assert (xn == 0).all(), "a single location centres to exactly zero"
    z64, bz = fb.conv_ref(r["xn"], aw, ab, device=DEV)
    frac["logits"] = check(r["logits"], z64, bz, what + " logits")
    p64, bp = fb.softmax_ref(r["logits"])
    frac["softmax"] = check(r["assign"], p64, bp, what + " softmax")
    v64, per, glob, ill = fb.vlad_ref(xn, flat(r["assign"]), cent)
    expect_ill = np.zeros_like(ill)
    if regime == "underflow":
        expect_ill[:, fb.DEAD] = True
        assert (r["assign"][..., fb.DEAD] == 0).all(), "the dead cluster's fp32 mass must be exactly 0"
        assert (r["out"].reshape(B, 32, 128)[:, fb.DEAD] == 0).all(), "the dead cluster's block must be 0"
        oracle = fb.head_fp32(x, aw, ab, cent)["out"].reshape(B, 32, 128)
        assert (oracle[:, fb.DEAD] == 0).all(), "the fp32 oracle's dead block must be 0"
    assert np.array_equal(ill, expect_ill), f"{what}: ill-conditioned clusters {np.argwhere(ill).tolist()}"
    out = r["out"].reshape(B, 32, 128)
    assert np.isfinite(out).all() and (np.linalg.norm(out, axis=-1) <= 1 + 1e-6).all()
    ref = v64.reshape(B, 32, 128)
    frac["vlad_cluster"] = check_norm(out[~ill], ref[~ill], per[~ill], what + " VLAD per cluster")
    frac["vlad_global"] = check_norm(r["out"], v64, glob, what + " VLAD")
    report(what, max(frac.values()))
    print("FRACTIONS", what, " ".join(f"{k} {v:.3e}" for k, v in frac.items()))


@pytest.mark.parametrize("regime", ["network", "underflow"])
def test_head_batch_slot_bit_exact(regime):
    """an image alone and in slot 2 of a batch of 3 with other means gives the same bits at every stage"""
    x4, ab, aw, cent = fb.head_case(regime, 3, 13, 25, seed=5)
    batch = run_head(x4, ab, aw, cent)
    one = run_head(x4[2:], ab, aw, cent)
    for k in batch:
        assert np.array_equal(batch[k][2:], one[k]), k


# ---------------------------------------------------------------------------------------------------------------------
# NetVLAD end to end on the FFMA path; argument checks; blank images
# ---------------------------------------------------------------------------------------------------------------------
def rel_err(a, b):
    return float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-30))


def _netvlad(mode, W, H, imgs, monkeypatch):
    with monkeypatch.context() as m:              # the switch is read when the handle is created
        m.setenv("OSB_SP_CONV", mode)
        nv = host.NetVLAD(synth.flatten_nv_weights(synth.netvlad_weights(0)), W, H, max_batch=len(imgs))
    out = nv.inference_batch(imgs)
    nv.close()
    return out


@pytest.mark.parametrize("size", [(96, 64), (400, 208), (640, 480)], ids=lambda s: "{}x{}".format(*s))
def test_netvlad_ffma_path_vs_oracle_and_default(size, monkeypatch):
    """OSB_SP_CONV=ffma (every layer in fp32 on the CUDA cores) against the fp32 oracle and the default path"""
    W, H = size
    imgs = np.stack([synth.image(40, H, W), synth.image(41, H, W, zero_bottom_quarter=True)])
    ffma, umma = _netvlad("ffma", W, H, imgs, monkeypatch), _netvlad("umma", W, H, imgs, monkeypatch)
    nvw = synth.netvlad_weights(0)
    for b in range(len(imgs)):
        o = fr.netvlad_net(imgs[b], nvw)
        e_f, e_u, e_fu = rel_err(ffma[b], o), rel_err(umma[b], o), rel_err(ffma[b], umma[b].astype(np.float64))
        print(f"MEASURED netvlad {W}x{H} image {b}: ffma vs oracle {e_f:.3e}, default vs oracle {e_u:.3e}, "
              f"ffma vs default {e_fu:.3e}")
        # an H100 measures at most 4.5e-6 / 4.6e-6 / 2.4e-6 (640x480, image 1; DESIGN.md section 4)
        assert e_f < 1.5e-5 and e_u < 1e-5 and e_fu < 1e-5


def test_netvlad_argument_errors_and_blank_images():
    nvb = synth.flatten_nv_weights(synth.netvlad_weights(0))
    for W, H in ((100, 64), (96, 60), (0, 64)):
        with pytest.raises(lib.OsbError) as e:
            host.NetVLAD(nvb, W, H, max_batch=1)
        assert e.value.status == lib.ERR_INVALID, (W, H)
    nv = host.NetVLAD(nvb, 96, 64, max_batch=2)
    for n in (0, 3):
        with pytest.raises(lib.OsbError) as e:
            nv.inference_batch(np.zeros((n, 64, 96), np.uint8))
        assert e.value.status == lib.ERR_INVALID, n
    blank = np.stack([np.zeros((64, 96), np.uint8), np.full((64, 96), 255, np.uint8)])
    v = nv.inference_batch(blank)
    nv.close()
    assert np.isfinite(v).all() and (np.linalg.norm(v, axis=1) <= 1 + 1e-6).all()
