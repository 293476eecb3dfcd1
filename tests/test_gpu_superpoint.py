"""GPU parity of the SuperPoint path (network, keypoints/NMS, descriptors) and NetVLAD against the oracle.

Parity definition (SURVEY.md section 7 hard part 1 / section 8 item 7):
  * post-processing (threshold, NMS2, top-K, sampling, norm, PCA) given the SAME engine outputs:
    keypoints and their order bit-exact, descriptors <= 1e-4 relative;
  * network outputs: semi <= 1e-4, desc and NetVLAD <= 1e-5 relative to the fp32 oracle (a few times what an H100
    measures, DESIGN.md section 4; the kernels themselves are bounded layer by layer in test_gpu_conv_layers.py);
  * end to end: keypoints identical except where the oracle heat-map is within a margin of a decision boundary
    (threshold or a neighbour's confidence), which is reported and bounded.
"""
import os

import numpy as np
import pytest

from conftest import GOLDEN
from omniswarm_b200 import synth, host
from oracle import frontend_ref as fr

pytestmark = pytest.mark.gpu

W0, H0 = 96, 64


@pytest.fixture(scope="module")
def small_sp(gpu):
    comp, mean = synth.pca_matrices(0)
    sp = host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, W0, H0, 0.015, 50, max_batch=3)
    yield sp
    sp.close()


def rel_err(a, b):
    return float(np.linalg.norm(a.astype(np.float64) - b) / max(np.linalg.norm(b), 1e-30))


def test_postprocess_golden_bit_exact(small_sp):
    z = np.load(os.path.join(GOLDEN, "postproc.npz"))
    semi = np.stack([z[f"{n}_semi"] for n in "abc"]); desc = np.stack([z[f"{n}_desc"] for n in "abc"])
    out = small_sp.postprocess(semi, desc)
    for i, n in enumerate("abc"):
        k, d = out[i]
        assert np.array_equal(k, z[f"{n}_kpts"]), f"case {n}: keypoints / order differ"
        assert np.array_equal(small_sp.read("conf", i)[:len(k)], z[f"{n}_conf"])
        ref = z[f"{n}_out"]
        assert d.shape == ref.shape
        if len(k):
            assert rel_err(d, ref) < 1e-4
        surv = small_sp.read("survivors", i) > 0
        assert np.array_equal(surv, fr.nms_survivor_mask(z[f"{n}_semi"], 0.015))


@pytest.mark.parametrize("kind", ["dense_ties", "all_equal", "empty", "single", "chain"])
def test_postprocess_edge_cases(small_sp, kind):
    rng = np.random.default_rng(7)
    semi = np.zeros((H0, W0), np.float32)
    if kind == "dense_ties":       # few distinct values -> many equal-confidence neighbours (never suppress each other)
        semi = rng.choice(np.array([0.0, 0.02, 0.3, 0.3, 0.7], np.float32), (H0, W0))
    elif kind == "all_equal":      # every pixel a candidate with the same confidence: all survive, raster order
        semi[:] = 0.5
    elif kind == "single":
        semi[H0 - 1, W0 - 1] = 0.4
    elif kind == "chain":          # strictly decreasing along a row: long dependency chain for the fixpoint loop
        semi[10, :] = np.linspace(0.9, 0.1, W0).astype(np.float32)
        semi[30, :] = np.linspace(0.1, 0.9, W0).astype(np.float32)
    desc = rng.standard_normal((256, H0 // 8, W0 // 8)).astype(np.float32)
    desc /= np.linalg.norm(desc, axis=0, keepdims=True)
    (k, d), = small_sp.postprocess(semi, desc)
    rk, rc = fr.get_keypoints(semi, 0.015, 50)
    assert np.array_equal(k, rk)
    comp, mean = synth.pca_matrices(0)
    rd = fr.compute_descriptors(desc, rk, W0, H0, comp, mean)
    assert d.shape == rd.shape
    if len(rk):
        fin = np.isfinite(rd)
        assert np.array_equal(np.isfinite(d), fin)
        assert np.allclose(d[fin], rd[fin], rtol=1e-4, atol=1e-5)


def test_u16_index_plane_wrap(gpu):
    """More than 65535 candidates: the reference's CV_16UC1 index plane wraps (superpoint_tensorrt.cpp:246,260)."""
    comp, mean = synth.pca_matrices(0)
    H, W = 256, 320                                    # 81920 pixels, all candidates
    sp = host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, W, H, 0.015, 200, max_batch=1)
    rng = np.random.default_rng(3)
    semi = rng.uniform(0.02, 0.9, (H, W)).astype(np.float32)
    desc = rng.standard_normal((256, H // 8, W // 8)).astype(np.float32)
    desc /= np.linalg.norm(desc, axis=0, keepdims=True)
    (k, d), = sp.postprocess(semi, desc)
    rk, rc = fr.get_keypoints(semi, 0.015, 200)
    assert (semi > 0.015).sum() > 65536
    assert np.array_equal(k, rk)
    # at least one returned point is displaced by the wrap (its coordinates are not where its confidence lives)
    conf = sp.read("conf", 0)[:len(k)]
    assert np.array_equal(conf, rc)
    assert (semi[k[:, 1].astype(int), k[:, 0].astype(int)] != conf).any()
    sp.close()


def test_network_golden(small_sp):
    z = np.load(os.path.join(GOLDEN, "superpoint_net.npz"))
    small_sp.inference(z["img"])
    semi, desc = small_sp.read("semi"), small_sp.read("desc")
    assert rel_err(semi, z["semi"]) < 1e-4
    assert np.abs(semi - z["semi"]).max() < 1e-4        # probability map in [0,1]
    assert np.abs(desc - z["desc"].astype(np.float32)).max() < 2e-3      # fixture stored as fp16


@pytest.fixture(scope="module")
def full_sp(gpu):
    comp, mean = synth.pca_matrices(0)
    sp = host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, 640, 480, 0.015, 200, max_batch=2)
    yield sp
    sp.close()


def test_network_full_size_vs_oracle(full_sp):
    """640x480 (BASELINE config 2): semi / desc against the fp32 oracle; stage-wise keypoint parity bit-exact on the
    device's own heat-map; end-to-end keypoints equal up to decision-margin cases.  Tolerances: about 3x (heat-map) and
    4x (descriptors) what an H100 measures on these images (DESIGN.md section 4)."""
    comp, mean = synth.pca_matrices(0)
    w = synth.superpoint_weights(0)
    imgs = np.stack([synth.image(0), synth.image(1, zero_bottom_quarter=True)])
    out = full_sp.inference_batch(imgs)
    for b in range(2):
        semi_o, desc_o = fr.superpoint_net(imgs[b], w)
        semi, desc = full_sp.read("semi", b), full_sp.read("desc", b)
        assert rel_err(semi, semi_o) < 1e-4 and rel_err(desc, desc_o) < 1e-5      # measured 3.5e-5, 2.3e-6
        assert np.abs(semi - semi_o).max() < 7.5e-5                                # measured 2.6e-5
        # stage-wise: oracle post-processing applied to the DEVICE heat-map must agree bit-exactly
        k, d = out[b]
        rk, rc = fr.get_keypoints(semi, 0.015, 200)
        assert np.array_equal(k, rk)
        rd = fr.compute_descriptors(desc, rk, 640, 480, comp, mean)
        assert rel_err(d, rd) < 1e-4
        # end to end vs the oracle's own heat-map: identical set except margin cases
        ok, oc = fr.get_keypoints(semi_o, 0.015, 200)
        same = {tuple(x) for x in k.tolist()} & {tuple(x) for x in ok.tolist()}
        assert len(same) >= 0.97 * len(ok), f"only {len(same)}/{len(ok)} keypoints agree end to end"
        assert len(k) == 200


def test_superpoint_argument_errors(small_sp):
    with pytest.raises(AssertionError):
        small_sp.inference(np.zeros((10, 10), np.uint8))       # reference asserts the size (:122)
    with pytest.raises(host._l.OsbError):
        host.SuperPoint(np.zeros(10, np.float32), *synth.pca_matrices(0), W0, H0)   # wrong blob length


def test_netvlad_vs_oracle(gpu):
    nvw = synth.netvlad_weights(0)
    z = np.load(os.path.join(GOLDEN, "netvlad.npz"))
    nv = host.NetVLAD(synth.flatten_nv_weights(nvw), W0, H0, max_batch=2)
    v = nv.inference(z["img"])
    assert rel_err(v, z["out"]) < 1e-5 and abs(np.linalg.norm(v) - 1) < 1e-5
    nv.close()
    nv = host.NetVLAD(synth.flatten_nv_weights(nvw), 640, 480, max_batch=4)
    imgs = np.stack([synth.image(s) for s in range(3)])
    out = nv.inference_batch(imgs)
    for b in range(3):
        # an H100 measures at most 2.1e-6 (DESIGN.md section 4): about 5x margin
        assert rel_err(out[b], fr.netvlad_net(imgs[b], nvw)) < 1e-5
    # distinct images give distinct descriptors; same image gives the same descriptor regardless of batch slot
    assert np.abs(out[0] @ out[1]) < 0.9999       # (random-weight stand-in: textures of one generator stay similar)
    assert np.array_equal(nv.inference(imgs[2]), out[2])
    nv.close()


def test_onboard_resolution_400x208(gpu):
    """The reference's TX2 configuration (400x208 engines, nodelet-sfisheye.launch:45-51; the size loop_tensorrt_test.cpp
    exercises): pooled maps of 200x104, 100x52 and 50x26 leave ragged 16x8 tiles in both directions."""
    W, H = 400, 208
    comp, mean = synth.pca_matrices(0)
    w = synth.superpoint_weights(0)
    sp = host.SuperPoint(synth.flatten_sp_weights(w), comp, mean, W, H, 0.015, 200, max_batch=2)
    imgs = np.stack([synth.image(5, H, W), synth.image(6, H, W, zero_bottom_quarter=True)])
    out = sp.inference_batch(imgs)
    for b in range(2):
        semi_o, desc_o = fr.superpoint_net(imgs[b], w)
        semi, desc = sp.read("semi", b), sp.read("desc", b)
        assert rel_err(semi, semi_o) < 1e-4 and rel_err(desc, desc_o) < 1e-5      # measured 3.4e-5, 2.2e-6
        k, d = out[b]
        rk, _ = fr.get_keypoints(semi, 0.015, 200)
        assert np.array_equal(k, rk)                      # bit-exact on the device's own heat-map
        assert rel_err(d, fr.compute_descriptors(desc, rk, W, H, comp, mean)) < 1e-4
    sp.close()
    nvw = synth.netvlad_weights(0)
    nv = host.NetVLAD(synth.flatten_nv_weights(nvw), W, H, max_batch=2)
    v = nv.inference_batch(imgs)
    for b in range(2):
        assert rel_err(v[b], fr.netvlad_net(imgs[b], nvw)) < 1e-5                 # measured 1.7e-6
    nv.close()


def test_tensor_core_path_vs_cuda_core_path(gpu):
    """The tensor-core convolutions (split-fp16, 3 products per K step) and the fp32 FFMA convolutions are two
    implementations of the same network, both compared with the fp32 oracle and with each other.  Tolerances: about 3x
    what an H100 measures on these images (DESIGN.md section 4); the layer-level bound is tests/test_gpu_conv_layers.py."""
    comp, mean = synth.pca_matrices(0)
    wts = synth.flatten_sp_weights(synth.superpoint_weights(0))
    img = np.stack([synth.image(3), synth.image(4, zero_bottom_quarter=True)])
    out = {}
    for mode in ("umma", "ffma"):
        os.environ["OSB_SP_CONV"] = mode
        sp = host.SuperPoint(wts, comp, mean, 640, 480, 0.015, 200, max_batch=2)
        sp.inference_batch(img)
        out[mode] = [(sp.read("semi", b), sp.read("desc", b)) for b in range(2)]
        sp.close()
    os.environ.pop("OSB_SP_CONV")
    w = synth.superpoint_weights(0)
    for b in range(2):
        so, do = fr.superpoint_net(img[b], w)
        # measured: umma 3.5e-5 / 2.2e-6, ffma 5.4e-6 / 1.3e-6 (heat-map / descriptors, relative)
        assert rel_err(out["umma"][b][0], so) < 1e-4 and rel_err(out["umma"][b][1], do) < 1e-5
        assert rel_err(out["ffma"][b][0], so) < 2e-5 and rel_err(out["ffma"][b][1], do) < 5e-6
        assert np.abs(out["umma"][b][0] - out["ffma"][b][0]).max() < 7.5e-5      # measured 2.5e-5
        assert np.abs(out["umma"][b][1] - out["ffma"][b][1]).max() < 5e-6        # measured 1.1e-6
        print("rel err vs oracle (semi, desc):", {m: (rel_err(out[m][b][0], so), rel_err(out[m][b][1], do)) for m in out})


def test_fused_softmax_matches_two_kernel_softmax(gpu):
    """The detector head's softmax + pixel shuffle fused into convPb's epilogue (default) against convPb writing its logits
    and sp_softmax_shuffle_kernel (OSB_SP_FUSED_SOFTMAX=0).  Same logits; the fused form reduces max and sum over the four
    lanes that hold a cell, the stand-alone kernel in channel order, so the heat maps agree to rounding, not bit for bit.
    The descriptor head does not depend on the switch: bit-identical."""
    W, H = 400, 208
    comp, mean = synth.pca_matrices(0)
    wts = synth.flatten_sp_weights(synth.superpoint_weights(0))
    imgs = np.stack([synth.image(21, H, W), synth.image(22, H, W, zero_bottom_quarter=True)])
    out = {}
    for f in ("1", "0"):
        os.environ["OSB_SP_FUSED_SOFTMAX"] = f
        sp = host.SuperPoint(wts, comp, mean, W, H, 0.015, 200, max_batch=2)
        sp.inference_batch(imgs)
        out[f] = [(sp.read("semi", b), sp.read("desc", b)) for b in range(2)]
        sp.close()
    os.environ.pop("OSB_SP_FUSED_SOFTMAX")
    for b in range(2):
        (s1, d1), (s0, d0) = out["1"][b], out["0"][b]
        assert np.abs(s1 - s0).max() < 1e-6 and rel_err(s1, s0) < 1e-6
        assert np.array_equal(d1, d0)


def test_network_vs_the_references_own_module(small_sp):
    """The CUDA network against golden vectors that do NOT come from the oracle: tests/golden/ref_superpoint.npz was written
    by the reference's own `SuperPointNet` (swarm_loop/superpoint.ipynb, the module its TensorRT engine is exported from),
    executed in place by tests/golden/make_ref_superpoint.py with the seeded weights and the C++ runtime's input scaling."""
    z = np.load(os.path.join(GOLDEN, "ref_superpoint.npz"))
    img = z["img_0"]
    assert img.shape == (H0, W0)
    small_sp.inference(img)
    semi, desc = small_sp.read("semi"), small_sp.read("desc")
    assert rel_err(semi, z["semi_0"]) < 1e-4 and np.abs(semi - z["semi_0"]).max() < 1e-4
    assert rel_err(desc, z["desc_0"]) < 1e-4
