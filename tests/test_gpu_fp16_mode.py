"""GPU: the plain-fp16 precision (OSB_PRECISION_FP16) of the tensor-core networks.

Layers, through the fp16 parity hooks, against the float64 convolution of the dequantised hi operands x = hi / 16,
w = fp16(1024 w) / 1024: fp16 x fp16 products are exact in fp32, so the split tests' bound TAU * (sum |x| |w| + |b|)
applies unchanged; a stored plane adds its fp16 rounding, 2^-11 |y| (+ 2^-25 / 16 for subnormals).  conv1a and the
depthwise kernels keep their fp32 arithmetic, so their fp16 plane is bit for bit the split kernels' hi plane.
Networks, against oracle.fp16_ref's emulation with the tolerance derived on the CPU (tests/test_fp16_model.py):
NET_TOL_FACTOR x the difference between the float64 and the float32-accumulated emulation of the same images.
"""
import os
import subprocess
import sys

import numpy as np
import pytest

from omniswarm_b200 import host, lib, synth
from oracle import fp16_ref as f16
from oracle import frontend_ref as fr
from oracle import split_model as sm
from test_gpu_conv_layers import LARGE, LAYER_IDS, LAYERS, SMALL, act, check_bound, pool2, ref64
from frontend_harness import H0, W0, frame_images
import frontend_harness as fh

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")

TAU = sm.TAU
SA, SW = f16.SA, f16.SW
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def hi_plane(x):
    """fp32 numpy [B,H,W,C] -> CUDA fp16 plane fp16(16 x) and the float64 value it represents"""
    hi, _ = sm.split(x, SA)
    return torch.from_numpy(hi).cuda(), hi.astype(np.float64) / SA


def w16(w):
    hi, _ = sm.split(w, SW)
    return hi.astype(np.float64) / SW


def plane_value(hi):
    return hi.cpu().numpy().astype(np.float64) / SA


def run_and_check(layer, B, H, W, regime, relu, pool, mode, seed=0, max_ctas=0):
    name, cin, cout, ks, out_c = layer
    x, w, b = sm.make_case(regime, B, H, W, cin, cout, ks, seed)
    hi, x64 = hi_plane(x)
    y64, d = ref64(x64, w16(w), b, ks)
    ref, bound = act(y64, relu), TAU * d
    if pool:
        ref, bound = pool2(ref), pool2(bound)
    what = f"fp16 {name} {B}x{H}x{W} {regime} relu={relu} pool={pool} {mode}"
    if mode == "f32":
        y = host.conv_layer_fp16_parity(w, b, hi, SA, relu=relu, pool=pool, out_c=out_c, max_ctas=max_ctas).cpu().numpy()
        assert (y[..., cout:out_c] == 0).all(), "the padding channels of the layer must be stored as 0"
        y = y[..., :cout]
    else:
        ohi = host.conv_layer_fp16_parity(w, b, hi, SA, relu=relu, pool=pool, out_c=out_c, mode="planes", out_scale=SA,
                                          max_ctas=max_ctas)
        y = plane_value(ohi[..., :out_c])[..., :cout]
        bound = bound + 2.0 ** -11 * (np.abs(ref) + bound) + 2.0 ** -25 / SA
    return check_bound(y, ref[..., :cout], bound[..., :cout], what)


@pytest.mark.parametrize("geom", SMALL, ids=lambda g: "B{}_{}x{}".format(*g))
@pytest.mark.parametrize("layer", LAYERS, ids=LAYER_IDS)
def test_fp16_layer_vs_float64_small(layer, geom):
    """Every instantiation x the small geometries x every value regime; ReLU / ReLU6, pooled and plane outputs alternate."""
    B, H, W = geom
    worst = 0.0
    for i, regime in enumerate(sm.REGIMES):
        relu = i % 3
        mode = "planes" if (i % 2 == 1 and layer[2] == layer[4]) else "f32"
        pool = int(H % 2 == 0 and W % 2 == 0 and i % 2 == 0)
        worst = max(worst, run_and_check(layer, B, H, W, regime, relu, pool, mode, seed=i))
    print(f"fp16 {layer[0]} B{B} {H}x{W}: max normalised error {worst:.3e}")


@pytest.mark.parametrize("geom", LARGE, ids=lambda g: "B{}_{}x{}".format(*g))
@pytest.mark.parametrize("layer", LAYERS, ids=LAYER_IDS)
def test_fp16_layer_vs_float64_large(layer, geom):
    B, H, W = geom
    mode = "planes" if layer[2] == layer[4] else "f32"
    e1 = run_and_check(layer, B, H, W, "relu_gauss", 1, 1, mode, seed=1)
    e2 = run_and_check(layer, B, H, W, "ramp", 2, 0, "f32", seed=2)
    print(f"fp16 {layer[0]} B{B} {H}x{W}: max normalised error {max(e1, e2):.3e}")


def test_fp16_full_resolution_resident_layer():
    """conv1b at 640 x 480 (conv_res64_kernel over 2400 tiles), ReLU + pool into the plane."""
    run_and_check(LAYERS[0], 1, 480, 640, "relu_gauss", 1, 1, "planes", seed=3)


@pytest.mark.parametrize("geom", [(1, 8, 16), (3, 3, 5), (1, 26, 50)], ids=lambda g: "B{}_{}x{}".format(*g))
def test_fp16_detector_head_softmax_vs_float64(geom):
    B, H, W = geom
    x, w, b = sm.make_case("relu_gauss", B, H, W, 256, 65, 1, seed=4)
    hi, x64 = hi_plane(x)
    z, d = ref64(x64, w16(w), b, 1)
    p = np.exp(z - z.max(axis=-1, keepdims=True))
    p /= p.sum(axis=-1, keepdims=True)
    bound = p * (np.expm1(2.0 * TAU * d.max(axis=-1, keepdims=True)) + 5e-6) + 1e-37
    shuffle = lambda a: a[..., :64].reshape(B, H, W, 8, 8).transpose(0, 1, 3, 2, 4).reshape(B, 8 * H, 8 * W)
    heat = host.conv_layer_fp16_parity(w, b, hi, SA, mode="softmax").cpu().numpy()
    check_bound(heat, shuffle(p), shuffle(bound), f"fp16 softmax head {geom}")


# ---------------------------------------------------------------------------------------------------------------------
# the fp32 kernels that write planes: only the hi plane, bit for bit the split kernels' hi plane
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("shape", [(2, 7, 13, 128), (1, 26, 50, 64), (1, 48, 64, 512)], ids=lambda s: "B{}_{}x{}_C{}".format(*s))
def test_fp16_depthwise_is_the_split_hi_plane(shape):
    rng = np.random.default_rng(7)
    C = shape[-1]
    x = torch.from_numpy(np.maximum(rng.standard_normal(shape), 0).astype(np.float32) * 3).cuda()
    w = (rng.standard_normal((C, 1, 3, 3)) * 0.5).astype(np.float32)
    b = (rng.standard_normal(C) * 0.1).astype(np.float32)
    for stride, generic in ((1, False), (1, True), (2, False)):
        if stride == 2 and (shape[1] % 2 or shape[2] % 2):
            continue
        hi, _ = host.dwconv_parity(w, b, x, SA, stride=stride, generic=generic)
        assert torch.equal(host.dwconv_fp16_parity(w, b, x, SA, stride=stride, generic=generic), hi), (stride, generic)


@pytest.mark.parametrize("geom", [(3, 7, 17), (1, 480, 640)], ids=lambda g: "B{}_{}x{}".format(*g))
def test_fp16_first_layer_is_the_split_hi_plane(geom):
    B, H, W = geom
    wsp = synth.superpoint_weights(0)
    imgs = torch.from_numpy(np.random.default_rng(8).integers(0, 256, (B, H, W), dtype=np.uint8)).cuda()
    hi, _ = host.conv_first_parity(wsp["conv1a.weight"], wsp["conv1a.bias"], imgs, SA)
    assert torch.equal(host.conv_first_fp16_parity(wsp["conv1a.weight"], wsp["conv1a.bias"], imgs, SA), hi)


# ---------------------------------------------------------------------------------------------------------------------
# invariances (bit-exact)
# ---------------------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("layer", [LAYERS[0], LAYERS[3], LAYERS[7], LAYERS[10]], ids=lambda l: l[0])
def test_fp16_max_ctas_does_not_change_the_result(layer):
    name, cin, cout, ks, out_c = layer
    x, w, b = sm.make_case("relu_gauss", 2, 26, 50, cin, cout, ks, seed=5)
    hi, _ = hi_plane(x)
    outs = [host.conv_layer_fp16_parity(w, b, hi, SA, relu=1, out_c=out_c, max_ctas=m).cpu().numpy()
            for m in (0, 1, 5)]
    assert np.array_equal(outs[0], outs[1], equal_nan=True) and np.array_equal(outs[0], outs[2], equal_nan=True)


@pytest.mark.parametrize("layer", [LAYERS[0], LAYERS[2], LAYERS[8]], ids=lambda l: l[0])
def test_fp16_batch_slot_does_not_change_the_result(layer):
    name, cin, cout, ks, out_c = layer
    x, w, b = sm.make_case("relu_gauss", 3, 7, 17, cin, cout, ks, seed=6)
    hi, _ = hi_plane(x)
    batch = host.conv_layer_fp16_parity(w, b, hi, SA, relu=1, out_c=out_c).cpu().numpy()
    one = host.conv_layer_fp16_parity(w, b, hi[2:].contiguous(), SA, relu=1, out_c=out_c).cpu().numpy()
    assert np.array_equal(batch[2:], one, equal_nan=True)


# (B, H, W) -> tiles of 8 x 16: 1 x 2 ragged, 3 x 3 ragged, 2 x 1 and 3 x 1 exact
@pytest.mark.parametrize("geom", [(1, 7, 17), (1, 21, 33), (1, 16, 16), (1, 24, 16)], ids=lambda g: "B{}_{}x{}".format(*g))
def test_fp16_resident_kernel_tiles_and_warpgroups(geom):
    """conv_res64_kernel: the CTA's i-th tile belongs to warpgroup i & 1.  With one CTA, an odd tile count leaves the last
    tile to warpgroup 0 and an even one to warpgroup 1; ragged tiles clip at the image edge.  Every grid gives the same
    bits, within the float64 bound, as planes and as fp32."""
    B, H, W = geom
    layer = LAYERS[0]
    for m in (0, 1, 2, 5):
        run_and_check(layer, B, H, W, "relu_gauss", 1, 0, "planes", seed=12, max_ctas=m)
    x, w, b = sm.make_case("signed", B, H, W, 64, 64, 3, seed=13)
    hi, _ = hi_plane(x)
    outs = [host.conv_layer_fp16_parity(w, b, hi, SA, relu=2, max_ctas=m).cpu().numpy() for m in (0, 1, 2, 5)]
    assert all(np.array_equal(outs[0], o, equal_nan=True) for o in outs[1:])


def test_fp16_programmatic_dependent_launch_is_bit_identical(tmp_path):
    """OSB_CONV_PDL=1 (read when the library loads, hence a fresh process) changes no bit of the fp16 network."""
    W, H = 400, 208
    imgs = np.stack([synth.image(31, H, W), synth.image(32, H, W, zero_bottom_quarter=True)])
    np.save(tmp_path / "imgs.npy", imgs)
    code = ("import sys, numpy as np; sys.path.insert(0, sys.argv[1]); "
            "from omniswarm_b200 import host, synth; "
            "imgs = np.load(sys.argv[2]); comp, mean = synth.pca_matrices(0); "
            "sp = host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, 400, 208, 0.015, "
            "200, max_batch=len(imgs)); sp.set_precision('fp16'); sp.inference_batch(imgs); "
            "np.savez(sys.argv[3], **{f'{k}{b}': sp.read(k, b) for b in range(len(imgs)) for k in ('semi', 'desc')})")
    r = subprocess.run([sys.executable, "-c", code, ROOT, str(tmp_path / "imgs.npy"), str(tmp_path / "pdl.npz")],
                       env=dict(os.environ, OSB_CONV_PDL="1"), capture_output=True, text=True, timeout=600)
    assert r.returncode == 0, r.stderr[-3000:]
    pdl = np.load(tmp_path / "pdl.npz")
    sp = make_sp(W, H, len(imgs))
    sp.set_precision("fp16")
    sp.inference_batch(imgs)
    for b in range(len(imgs)):
        assert np.array_equal(pdl[f"semi{b}"], sp.read("semi", b)) and np.array_equal(pdl[f"desc{b}"], sp.read("desc", b))
    sp.close()


# ---------------------------------------------------------------------------------------------------------------------
# whole networks
# ---------------------------------------------------------------------------------------------------------------------
NET_IMAGES = [synth.image(51, H0, W0), synth.image(52, H0, W0, zero_bottom_quarter=True), synth.image(53, H0, W0)]


def make_sp(W, H, max_batch, max_num=200):
    comp, mean = synth.pca_matrices(0)
    return host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, W, H, 0.015, max_num,
                           max_batch=max_batch)


@pytest.fixture(scope="module")
def net_tol():
    return f16.network_tolerances(NET_IMAGES, synth.superpoint_weights(0), synth.netvlad_weights(0))


def test_fp16_superpoint_vs_emulation_and_oracle(gpu, net_tol):
    """Heat map and descriptors against the fp16 emulation within the derived tolerance; against the fp32 oracle the
    figure is reported and loosely bounded; keypoints of the oracle's post-processing on the device's heat map are the
    device's, bit for bit, and so are its descriptors to 1e-4."""
    wsp = synth.superpoint_weights(0)
    comp, mean = synth.pca_matrices(0)
    sp = make_sp(W0, H0, len(NET_IMAGES), max_num=50)
    sp.set_precision("fp16")
    outs = sp.inference_batch(np.stack(NET_IMAGES))
    for b, img in enumerate(NET_IMAGES):
        semi, desc = sp.read("semi", b), sp.read("desc", b)
        es, ed = f16.superpoint_net_fp16(img, wsp)
        s32, d32 = fr.superpoint_net(img, wsp)
        e = {"semi": f16.rel(semi, es), "desc": f16.rel(desc, ed)}
        print(f"image {b}: vs emulation {e} (tolerance {net_tol}); vs fp32 oracle semi {f16.rel(semi, s32):.2e} "
              f"desc {f16.rel(desc, d32):.2e}")
        assert e["semi"] <= net_tol["semi"] and e["desc"] <= net_tol["desc"], (e, net_tol)
        assert f16.rel(semi, s32) < 2e-2 and f16.rel(desc, d32) < 2e-2
        k, d = outs[b]
        rk, _ = fr.get_keypoints(semi, 0.015, 50)
        assert np.array_equal(k, rk)
        rd = fr.compute_descriptors(desc, rk, W0, H0, comp, mean)
        assert np.linalg.norm(d - rd) <= 1e-4 * max(np.linalg.norm(rd), 1e-30)
    sp.close()


def test_fp16_netvlad_vs_emulation_and_oracle(gpu, net_tol):
    wnv = synth.netvlad_weights(0)
    nv = host.NetVLAD(synth.flatten_nv_weights(wnv), W0, H0, max_batch=len(NET_IMAGES))
    nv.set_precision("fp16")
    v = nv.inference_batch(np.stack(NET_IMAGES))
    for b, img in enumerate(NET_IMAGES):
        e, e32 = f16.rel(v[b], f16.netvlad_net_fp16(img, wnv)), f16.rel(v[b], fr.netvlad_net(img, wnv))
        print(f"image {b}: NetVLAD vs emulation {e:.2e} (tolerance {net_tol['vlad']:.2e}), vs fp32 oracle {e32:.2e}")
        assert e <= net_tol["vlad"] and e32 < 2e-2
    nv.close()


def test_switching_back_is_bit_identical_and_acquires_nothing(gpu):
    imgs = np.stack(NET_IMAGES)
    ref = make_sp(W0, H0, len(imgs))
    ref.inference_batch(imgs)
    sp = make_sp(W0, H0, len(imgs))
    live = host.live_resources()
    sp.set_precision("fp16")
    sp.inference_batch(imgs)
    fp16_semi = sp.read("semi", 0)
    sp.set_precision("split_fp16")
    sp.inference_batch(imgs)
    assert host.live_resources() == live
    assert not np.array_equal(fp16_semi, ref.read("semi", 0))
    for b in range(len(imgs)):
        assert np.array_equal(sp.read("semi", b), ref.read("semi", b)) and np.array_equal(sp.read("desc", b), ref.read("desc", b))
    with pytest.raises(ValueError):
        sp.set_precision("bf16")
    assert lib.load().osb_superpoint_set_precision(sp._h, 7) == lib.ERR_INVALID
    sp.close(); ref.close()


# ---------------------------------------------------------------------------------------------------------------------
# the front-end
# ---------------------------------------------------------------------------------------------------------------------
def make_frontend(**kw):
    return fh.make_frontend(dict(db_capacity=256, match_index_dist=1), **kw)


def blanked(a):
    a = a.copy()
    a[:, H0 * 3 // 4:] = 0
    return a


def test_fp16_frontend_records_and_query(gpu, net_tol):
    """Records of fp16 keyframes: global descriptors within the NetVLAD bound of the emulation, keypoints and local
    descriptors those of a standalone fp16 SuperPoint on the same images; the query rule on fp16 records returns the
    oracle's hit ids for the device's own descriptors."""
    wnv = synth.netvlad_weights(0)
    comp, mean = synth.pca_matrices(0)
    fe = make_frontend()
    fe.set_precision("fp16")
    sp = make_sp(W0, H0, 8)
    sp.set_precision("fp16")
    det = fr.LoopDetectorDB(self_id=1, dim=4096, inner_product_thres=0.3, match_index_dist=1)
    frames = [frame_images(s) for s in range(4)] + [frame_images(0)]
    for i, (up, down) in enumerate(frames):
        rec, res = fe.process(up, down, msg_id=i)
        up_b, down_b = blanked(up), blanked(down)
        sp.inference_batch(np.concatenate([up_b, down_b]))
        g = [np.ctypeslib.as_array(rec.global_desc[d]).copy() for d in range(4)]
        for d in range(4):
            e = f16.rel(g[d], f16.netvlad_net_fp16(up_b[d], wnv))
            assert e <= net_tol["vlad"], (i, d, e)
            n = rec.n_kpts[d]
            rk, _ = fr.get_keypoints(sp.read("semi", d), 0.015, 200)
            assert np.array_equal(np.ctypeslib.as_array(rec.kpts[d])[:n], rk)
            rd = fr.compute_descriptors(sp.read("desc", d), rk, W0, H0, comp, mean)
            ld = np.ctypeslib.as_array(rec.local_desc[d])[:n]
            assert np.linalg.norm(ld - rd) <= 1e-4 * max(np.linalg.norm(rd), 1e-30)
        det.add_frame(i, 1, g, [rec.n_kpts[d] for d in range(4)])
        rid, rdist = det.query(1, g[1], False, False)
        assert res.hit_id == rid and res.accepted == int(rid != -1 and rdist > -1), (i, res.hit_id, rid)
        if rid != -1 and rdist > -1:
            assert abs(res.hit_score - rdist) < 1e-4
    assert res.accepted == 1 and res.hit_id == 1                   # the revisit of frame 0 finds its row
    fe.close(); sp.close()


def test_frontend_switch_back_is_bit_identical(gpu):
    up, down = frame_images(2)
    fe_ref = make_frontend()
    ref, _ = fe_ref.process(up, down, msg_id=5)
    fe = make_frontend()
    live = host.live_resources()
    fe.set_precision("fp16")
    r16, _ = fe.process(up, down, msg_id=5)
    fe.set_precision("split_fp16")
    fe.db_reset()
    rec, _ = fe.process(up, down, msg_id=5)
    assert host.live_resources() == live
    assert bytes(r16) != bytes(ref)
    assert bytes(rec) == bytes(ref)
    fe.close(); fe_ref.close()


def test_cuda_core_handles_reject_fp16(gpu, monkeypatch):
    """A handle created under OSB_SP_CONV=ffma has no tensor-core layers: fp16 is OSB_ERR_INVALID, split stays valid."""
    monkeypatch.setenv("OSB_SP_CONV", "ffma")
    fe = make_frontend()
    sp = make_sp(W0, H0, 1)
    nv = host.NetVLAD(synth.flatten_nv_weights(synth.netvlad_weights(0)), W0, H0, max_batch=1)
    for h in (fe, sp, nv):
        with pytest.raises(lib.OsbError) as e:
            h.set_precision("fp16")
        assert e.value.status == lib.ERR_INVALID
        h.set_precision("split_fp16")
    fe.close(); sp.close(); nv.close()
