"""GPU: every handle and every host entry point gives back what it acquired.  osb_live_resources() counts the device
buffers, pinned buffers, streams and events the library holds; it must return to its starting value after create, use and
destroy of each handle type (with the lazily acquired resources exercised), after creates that fail part-way, and after
the host-buffer wrappers and the parity hooks, including one that fails in its weight upload."""
import gc

import numpy as np
import pytest

from omniswarm_b200 import host, lib, synth
from test_gpu_frontend_depth import K0, POSE_DRONE, extrinsics, frame, make_frontend
from test_gpu_lift import K as LIFT_K, synth_stereo
from test_gpu_multistart import c1_with_loops
from test_gpu_pcm import ANG, POS, THRES
from test_gpu_pnp import case as pnp_case

pytestmark = pytest.mark.gpu

torch = pytest.importorskip("torch")
W, H = 96, 64


def baseline():
    gc.collect()            # handles of earlier tests that are only reachable through a cycle close now, not mid-test
    return host.live_resources()


def test_handles_give_back_everything(gpu):
    comp, mean = synth.pca_matrices(0)
    spw = synth.flatten_sp_weights(synth.superpoint_weights(0))
    nvw = synth.flatten_nv_weights(synth.netvlad_weights(0))
    imgs = np.stack([synth.image(s, H, W) for s in range(2)])
    n0 = baseline()

    sp = host.SuperPoint(spw, comp, mean, W, H, 0.015, 50, max_batch=2)
    sp.inference_batch(imgs)
    n1 = host.live_resources()
    assert n1 > n0
    sp.layer_ms(imgs)                                           # creates the per-layer profiling events
    assert host.live_resources() > n1
    sp.close()
    assert host.live_resources() == n0, "SuperPoint"

    nv = host.NetVLAD(nvw, W, H, max_batch=2)
    nv.inference_batch(imgs)
    nv.close()
    assert host.live_resources() == n0, "NetVLAD"

    rng = np.random.default_rng(0)
    db = host.IndexFlatIP(64, 1024)
    db.add(rng.standard_normal((10, 64)))
    db.search(rng.standard_normal((2, 64)), 4)
    db.close()
    assert host.live_resources() == n0, "IndexFlatIP"

    m = host.BFMatcher(2, 200, 64)
    m.match(rng.standard_normal((30, 64)).astype(np.float32), rng.standard_normal((40, 64)).astype(np.float32))
    m.close()
    assert host.live_resources() == n0, "BFMatcher"

    g, mask = c1_with_loops()
    solver = host.PoseGraphSolver(g["n_nodes"], len(g["ftype"]))    # sized to the graph: K = 4 grows the arena
    solver.solve(g)
    solver.solve(g)
    n1 = host.live_resources()
    solver.solve_multistart(g, mask, 4, 77, window_size=100, acpt_cost=float("inf"))
    assert host.live_resources() == n1                          # the grown arena replaced the one-trial arena
    solver.close()
    assert host.live_resources() == n0, "PoseGraphSolver"

    fe = make_frontend(depth_camera=False)
    fe.set_profiling(True)                                      # creates the stage events at the first keyframe
    up, down = (np.stack([synth.image(s * 10 + d, H, W) for d in range(2)]) for s in (1, 2))
    fe.process(up, down, 1)
    fe.stage_ms()
    fe.set_depth_camera(K0, extrinsics(2), 0.3, 10.0)          # allocates the depth staging buffer
    fe.set_drone_pose(POSE_DRONE)
    fe.process_depth(*frame(3), 2)
    fe.close()
    assert host.live_resources() == n0, "KeyframeFrontend"

    sw = host.Swarm(None, 0, 1)
    stream = torch.cuda.current_stream().cuda_stream
    rec = torch.arange(lib.RECORD_BYTES, device="cuda").to(torch.uint8)
    g1 = torch.zeros_like(rec)
    g2 = torch.zeros_like(rec)
    sw.exchange(rec.data_ptr(), g1.data_ptr(), stream)
    sw.exchange_async(rec.data_ptr(), g2.data_ptr(), stream)
    sw.wait(stream)
    torch.cuda.synchronize()
    assert torch.equal(rec, g1) and torch.equal(rec, g2)
    sw.close()
    assert host.live_resources() == n0, "Swarm"


def out_of_range(weights, name, value):
    w = dict(weights)
    w[name] = w[name].copy()
    w[name].reshape(-1)[0] = value
    return w


def test_failed_creates_leave_nothing_behind(gpu):
    """an unsplittable weight in each tensor-core layer makes the create fail there, after everything before it was
    acquired; nothing of it may stay"""
    comp, mean = synth.pca_matrices(0)
    wsp, wnv = synth.superpoint_weights(0), synth.netvlad_weights(0)
    n0 = baseline()
    failures = [(lambda w=out_of_range(wsp, f"{name}.weight", 100.0):
                 host.SuperPoint(synth.flatten_sp_weights(w), comp, mean, W, H, 0.015, 50, max_batch=1), name)
                for name, *_ in synth.SP_LAYERS[1:]]                                       # conv1b ... convDb
    failures += [(lambda w=out_of_range(wnv, name, -70.0): host.NetVLAD(synth.flatten_nv_weights(w), W, H, max_batch=1),
                  name) for name in [f"b{i}.pw.weight" for i in range(1, 7)] + ["proj.weight"]]
    bad_nv = synth.flatten_nv_weights(out_of_range(wnv, "b3.pw.weight", 100.0))
    failures.append((lambda: host.KeyframeFrontend(synth.flatten_sp_weights(wsp), comp, mean, bad_nv, width=W, height=H,
                                                   n_dirs=2, db_capacity=256), "frontend NetVLAD"))
    assert len(failures) == 11 + 7 + 1
    for create, what in failures:
        with pytest.raises(lib.OsbError) as e:
            create()
        assert e.value.status == lib.ERR_INVALID and "split-fp16 range" in str(e.value), what
        assert host.live_resources() == n0, what


def test_wrappers_and_parity_hooks_give_back_everything(gpu):
    rng = np.random.default_rng(1)
    n0 = baseline()

    src = rng.uniform(0, 100, (20, 2)).astype(np.float32)
    host.homography_ransac([src], [src + 1.0])
    ku, kd, sm, nu, ndn, pu, pd, *_ = synth_stereo(0)
    host.stereo_lift(ku, kd, sm, nu, ndn, LIFT_K, pu, pd)
    kp = rng.integers(0, 64, (2, 50, 2)).astype(np.float32)
    pose = np.array([np.concatenate([[0.3, -0.2, 1.0], [1.0, 0.0, 0.0, 0.0]])] * 2)
    host.depth_lift(kp, np.array([50, 37], np.int32), rng.integers(0, 12000, (2, H, W)).astype(np.uint16), LIFT_K, pose)
    host.pnp_ransac([pnp_case(0)])
    host.pcm_outlier_rejection(synth.pcm_edges(20, 0.3, 0), THRES, POS, ANG, want_matrices=True)
    assert host.live_resources() == n0, "host-buffer wrappers"

    wsp, wnv = synth.superpoint_weights(0), synth.netvlad_weights(0)
    imgs = torch.from_numpy(np.stack([synth.image(0, H, W)])).cuda()
    x64 = torch.rand((1, 8, 16, 64), device="cuda")
    hi, lo = x64.half(), torch.zeros((1, 8, 16, 64), dtype=torch.float16, device="cuda")
    w = (rng.standard_normal((64, 64, 3, 3)) * 0.05).astype(np.float32)
    b = np.zeros(64, np.float32)
    host.conv_layer_parity(w, b, hi, lo, 16.0)
    host.conv_first_parity(wsp["conv1a.weight"], wsp["conv1a.bias"], imgs, 16.0)
    host.dwconv_parity(wnv["b1.dw.weight"], wnv["b1.dw.bias"], torch.rand((1, 8, 16, 64), device="cuda"), 16.0)
    host.conv_ffma_parity(w, b, x64)
    host.conv_first_ffma_parity(wsp["conv1a.weight"], wsp["conv1a.bias"], imgs, stride=1, act=1)
    host.dwconv_ffma_parity(wnv["b1.dw.weight"], wnv["b1.dw.bias"], torch.rand((1, 8, 16, 64), device="cuda"))
    host.nv_block0_parity(wnv["b0.dw.weight"], wnv["b0.dw.bias"], wnv["b0.pw.weight"], wnv["b0.pw.bias"],
                          torch.rand((1, 8, 16, 32), device="cuda"))
    host.nv_head_parity(wnv["assign.weight"], wnv["assign.bias"], wnv["centroids"], torch.rand((1, 4, 6, 128), device="cuda"))
    torch.cuda.synchronize()
    assert host.live_resources() == n0, "parity hooks"

    w[3, 5, 0, 0] = -64.0                                       # the hook fails in its weight upload
    with pytest.raises(lib.OsbError) as e:
        host.conv_layer_parity(w, b, hi, lo, 16.0)
    assert e.value.status == lib.ERR_INVALID
    assert host.live_resources() == n0, "failed parity hook"
