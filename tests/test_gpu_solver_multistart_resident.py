"""osb_solver_solve_multistart_resident_dev and osb_anchor_init_mask_dev: the random-restart initialisation on the
resident window with a device tail, its mask and yaw read from the device.  Against osb_solver_solve_multistart of the
concatenated list (bit-identical where both pick the same shape and plan), the mask against the oracle rule on the
observability record, rejection, refusals, stream capture of the whole init branch, the cooperative path, launch and
memory accounting, and the C++ adapter smoke program."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l
import init_mask_ref as mr
from backend_harness import KEYS, feed, make_anchor, options, pcm_state, resident
from test_gpu_solver_device_tail import candidate_rows, concat, plan_keeping_rows, same_plan, shape, window

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "omni-swarm_b200", "csrc")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")
SELF, XY, Z = 0, 1.0, 0.3


def mask_and_yaw(base, seed):
    """a quarter of the nodes masked, each with a yaw of its own"""
    rng = np.random.default_rng(seed)
    n = len(base["init"])
    mask = (rng.random(n) < 0.25).astype(np.uint8)
    yaw = rng.uniform(-np.pi, np.pi, n)
    return mask, yaw


def dev_buffers(mask, yaw):
    return torch.from_numpy(mask).cuda(), torch.from_numpy(yaw).cuda()


def one_shot_start(base, mask, yaw):
    """the starting poses of the one-shot call: the device call sets a scattered node's yaw from init_yaw_dev"""
    init = base["init"].copy()
    sel = (mask != 0) & (base["fixed"] == 0)
    init[sel, 3] = yaw[sel]
    return init


def ms_call(solver, buf, max_tail, m_dev, y_dev, K, o, acpt=np.inf, seed=5, window_size=30, stream=None):
    s = torch.cuda.current_stream() if stream is None else stream
    solver.solve_multistart_resident_dev(max_tail, *buf.ptrs(), m_dev.data_ptr(), None if y_dev is None else y_dev.data_ptr(),
                                         s.cuda_stream, K, seed, window_size, acpt, True, o)


def same_summaries(a, b):
    return all((x.initial_cost, x.final_cost, x.iterations, x.pcg_iterations, x.n_residuals, x.termination) ==
               (y.initial_cost, y.final_cost, y.iterations, y.pcg_iterations, y.n_residuals, y.termination)
               for x, y in zip(a, b))


@pytest.mark.gpu
@pytest.mark.parametrize("kind", ["default", "fp64"])
@pytest.mark.parametrize("K", [1, 3, 32])
def test_bit_identical_to_one_shot_multistart(gpu, K, kind):
    _, base = window()
    k = 24
    tail = plan_keeping_rows(base, k, seed=3)
    assert len(tail["ftype"]) == k and same_plan(base, tail)
    mask, yaw = mask_and_yaw(base, 1)
    m_dev, y_dev = dev_buffers(mask, yaw)
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    o = options(dev, kind)
    resident(dev, base)
    buf = host.FactorRows(64)
    buf.set(tail)
    ms_call(dev, buf, k, m_dev, y_dev, K, o)
    chosen, summ, equv = dev.last_multistart()
    poses = dev.graph_get_poses()
    sh = shape(dev)
    start = one_shot_start(base, mask, yaw)
    ref, c1, s1, e1 = flat.solve_multistart(concat(base, tail, start), mask, K, 5, 30, np.inf, True, o, init=start)
    assert sh == shape(flat)
    assert chosen == c1 >= 0 and np.array_equal(equv, e1) and same_summaries(summ, s1)
    assert np.array_equal(poses, ref)
    assert all(s.solve_ms > 0.0 for s in summ)
    with pytest.raises(_l.OsbError) as e:                          # the single-solve reader names the new one
        dev.last_summary()
    assert e.value.status == _l.ERR_INVALID
    ms_call(dev, buf, k, m_dev, None, K, o)                        # without a yaw the scattered nodes keep theirs
    chosen, summ, equv = dev.last_multistart()
    ref2, c2, s2, e2 = flat.solve_multistart(concat(base, tail, poses), mask, K, 5, 30, np.inf, True, o, init=poses)
    assert chosen == c2 and np.array_equal(equv, e2) and same_summaries(summ, s2)
    assert np.array_equal(dev.graph_get_poses(), ref2)
    for h in (dev, flat):
        h.close()


def renumbered(win, d):
    """the window without its blocks < d, the rest renumbered block - d (emptied frames removed)"""
    stamps, first, entries = win
    keep_f, new_e, new_first = [], [], [0]
    for f in range(len(stamps)):
        e = entries[first[f]:first[f + 1]]
        e = e[e["block"] >= d].copy()
        if len(e):
            e["block"] -= d
            keep_f.append(stamps[f]); new_e.append(e); new_first.append(new_first[-1] + len(e))
    return np.array(keep_f, np.int64), np.array(new_first, np.int32), np.concatenate(new_e)


def restricted(win, drones):
    stamps, first, entries = win
    frames = [entries[first[f]:first[f + 1]] for f in range(len(stamps))]
    frames = [e[np.isin(e["drone_id"], list(drones))] for e in frames]
    return stamps.copy(), np.cumsum([0] + [len(e) for e in frames]).astype(np.int32), np.concatenate(frames)


@pytest.mark.gpu
def test_mask_from_the_device(gpu):
    g, base = window()
    a = make_anchor(g, max_meas=4096)
    feed(a, g)
    chain = host.AnchoredChain(4096)
    n_nodes = len(base["init"]) + 5                                # blocks past the window's get 0
    full = g["window"]
    rounds = [restricted(full, {0, 1}), restricted(full, {0, 1, 2}), full, full]
    d = int(full[2]["block"][:full[1][1]].max()) + 1
    rounds.append(renumbered(full, d))                             # drop_oldest + the renumbered set_window
    seen_new = seen_mask = False
    for win in rounds:
        a.set_window(*win)
        n = chain.run(a)
        chain.observe(a, n, SELF, XY, Z)
        chain.init_mask(a, SELF, n_nodes)
        chain.stream.synchronize()
        obs = a.observability()
        want_m, want_y = mr.init_mask(win[1], win[2], obs["to_init"], SELF, n_nodes)
        got_m = chain.mask[:n_nodes].cpu().numpy()
        got_y = chain.yaw[:n_nodes].cpu().numpy()
        assert np.array_equal(got_m, want_m)
        assert np.abs(got_y - want_y).max() <= 1e-15 and np.array_equal(got_y[want_m == 0], want_y[want_m == 0])
        seen_new |= obs["motion_new"] or bool(obs["to_init"][1:].any())
        seen_mask |= bool(want_m.any())
    assert seen_new and seen_mask
    # refused at once, nothing enqueued
    n0 = host.launch_count()
    s = chain.stream.cuda_stream
    for args in ((SELF, n_nodes, 0, chain.yaw.data_ptr()), (SELF, n_nodes, chain.mask.data_ptr(), 0),
                 (SELF, 0, chain.mask.data_ptr(), chain.yaw.data_ptr()), (-1, n_nodes, chain.mask.data_ptr(), chain.yaw.data_ptr()),
                 (SELF, 3, chain.mask.data_ptr(), chain.yaw.data_ptr())):                       # a window block >= 3
        with pytest.raises(_l.OsbError) as e:
            a.init_mask_dev(*args, s)
        assert e.value.status == _l.ERR_INVALID
    fresh = make_anchor(g)
    fresh.set_window(*full)
    with pytest.raises(_l.OsbError):                               # no observe yet
        fresh.init_mask_dev(SELF, n_nodes, chain.mask.data_ptr(), chain.yaw.data_ptr(), s)
    assert host.launch_count() == n0
    for h in (a, fresh):
        h.close()


@pytest.mark.gpu
def test_rejection_leaves_the_poses(gpu):
    _, base = window()
    tail = plan_keeping_rows(base, 16, seed=5)
    mask, yaw = mask_and_yaw(base, 2)
    m_dev, y_dev = dev_buffers(mask, yaw)
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    o = options(dev, "default")
    resident(dev, base)
    buf = host.FactorRows(64)
    buf.set(tail)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    buf.solve(dev, 16, o, stream)                                  # the steady chain, then the init branch
    before = dev.graph_get_poses()
    ms_call(dev, buf, 16, m_dev, y_dev, 3, o, acpt=0.0, stream=stream)
    chosen, summ, equv = dev.last_multistart()
    assert chosen == -1 and (equv >= 0.0).all()
    assert dev.graph_get_poses().tobytes() == before.tobytes()
    # the next steady solve runs from them without host work: it can be captured
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=stream, capture_error_mode="global"):
        buf.solve(dev, 16, o, stream)
    graph.replay()
    torch.cuda.synchronize()
    ref, _ = flat.solve(concat(base, tail, before), o)
    assert np.array_equal(dev.graph_get_poses(), ref)
    for h in (dev, flat):
        h.close()


@pytest.mark.gpu
def test_refusals(gpu):
    _, base = window()
    n = len(base["init"])
    tail = plan_keeping_rows(base, 8, seed=7)
    mask, yaw = mask_and_yaw(base, 3)
    m_dev, y_dev = dev_buffers(mask, yaw)
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    o = options(dev, "default")
    resident(dev, base)
    buf = host.FactorRows(64)
    buf.set(tail)
    ms_call(dev, buf, 8, m_dev, y_dev, 3, o)
    good = dev.graph_get_poses()
    size = dev.graph_size()
    bad = {k_: v.copy() for k_, v in tail.items()}
    bad["ia"][2] = n
    for rows, count, code in ((tail, 9, _l.ERR_CAPACITY), (bad, None, _l.ERR_INVALID)):   # refused on the device
        buf.set(rows, count)
        ms_call(dev, buf, 8, m_dev, y_dev, 3, o)
        with pytest.raises(_l.OsbError) as e:
            dev.last_multistart()
        assert e.value.status == code
        assert dev.graph_get_poses().tobytes() == good.tobytes() and dev.graph_size() == size
    buf.set(tail)                                                  # the next valid call is correct
    ms_call(dev, buf, 8, m_dev, y_dev, 3, o)
    c, _, _ = dev.last_multistart()
    start = one_shot_start(dict(base, init=good), mask, yaw)
    ref, c1, _, _ = flat.solve_multistart(concat(base, tail, start), mask, 3, 5, 30, np.inf, True, o, init=start)
    assert c == c1 and np.array_equal(dev.graph_get_poses(), ref)
    # refused at once: nothing enqueued
    n0 = host.launch_count()
    s = torch.cuda.current_stream().cuda_stream
    p = buf.ptrs()
    for i in range(7):
        args = list(p) + [m_dev.data_ptr()]
        args[i] = 0
        with pytest.raises(_l.OsbError):
            dev.solve_multistart_resident_dev(8, *args, y_dev.data_ptr(), s, 3, 5, 30, np.inf, True, o)
    for K, acpt in ((0, 1.0), (257, 1.0), (3, float("nan"))):
        with pytest.raises(_l.OsbError) as e:
            dev.solve_multistart_resident_dev(8, *p, m_dev.data_ptr(), y_dev.data_ptr(), s, K, 5, 30, acpt, True, o)
        assert e.value.status == _l.ERR_INVALID
    assert host.launch_count() == n0
    # growing the arena is host work: refused under capture, the capture itself completes
    fresh = host.PoseGraphSolver(4096, 32768)
    resident(fresh, base)
    stream = torch.cuda.Stream()
    stream.wait_stream(torch.cuda.current_stream())
    buf.solve(fresh, 8, o, stream)
    fresh.last_summary()
    g2 = torch.cuda.CUDAGraph()
    x = torch.zeros(4, device="cuda")
    with torch.cuda.graph(g2, stream=stream, capture_error_mode="global"):
        with pytest.raises(_l.OsbError) as e:
            ms_call(fresh, buf, 8, m_dev, y_dev, 256, o, stream=stream)
        x += 1
    assert e.value.status == _l.ERR_INVALID
    g2.replay()
    torch.cuda.synchronize()
    assert float(x.sum()) == 4.0
    for h in (dev, flat, fresh):
        h.close()


@pytest.mark.gpu
def test_capture_of_the_init_branch(gpu):
    g, base = window()
    n_nodes = len(base["init"])
    o_ms = dict(n_trials=3, seed=11, window_size=30, acpt_cost=np.inf)

    def setup():
        a = make_anchor(g, max_meas=4096)
        feed(a, g)
        st = pcm_state(g, 32, 1024)
        dev = host.PoseGraphSolver(4096, 32768)
        resident(dev, base)
        return a, st, dev, host.AnchoredChain(4096)

    def branch(a, st, dev, chain, o):
        n = chain.run(a)
        chain.observe(a, n, SELF, XY, Z)
        chain.reject(st, n)
        chain.compact(n)
        chain.init_mask(a, SELF, n_nodes)
        chain.init_solve(dev, 2048, options=o, **o_ms)

    a, st, dev, chain = setup()
    o = options(dev, "default")
    want = []
    for _ in range(3):
        branch(a, st, dev, chain, o)
        want.append((dev.graph_get_poses(), dev.last_multistart()))
    a2, st2, dev2, chain2 = setup()
    branch(a2, st2, dev2, chain2, o)                               # warm: the plan, the tables, the arena
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=chain2.stream, capture_error_mode="global"):
        branch(a2, st2, dev2, chain2, o)
    for poses, (c, summ, equv) in want[1:]:
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(dev2.graph_get_poses(), poses)
        c2, summ2, equv2 = dev2.last_multistart()
        assert c2 == c and np.array_equal(equv2, equv) and same_summaries(summ2, summ)
        assert all(s.solve_ms == 0.0 for s in summ2)
    for h in (a, st, dev, a2, st2, dev2):
        h.close()


@pytest.mark.gpu
def test_cooperative_path(gpu):
    _, base = window()
    k, K = 26000, 2
    tail = candidate_rows(base, k, np.random.default_rng(13), kinds=(0,))
    tail["payload"][:, 1] = 0.05                                   # weak ranges
    mask, yaw = mask_and_yaw(base, 4)
    m_dev, y_dev = dev_buffers(mask, yaw)
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    o = options(dev, "default")
    resident(dev, base)
    buf = host.FactorRows(k)
    buf.set(tail)
    n0 = host.launch_count()
    ms_call(dev, buf, k, m_dev, y_dev, K, o)
    launches = host.launch_count() - n0
    chosen, summ, equv = dev.last_multistart()
    poses = dev.graph_get_poses()
    assert shape(dev)[1] == 0.0 and launches == 6 + K               # cooperative grids, the trials in turn
    start = one_shot_start(base, mask, yaw)
    ref, c1, s1, e1 = flat.solve_multistart(concat(base, tail, start), mask, K, 5, 30, np.inf, True, o, init=start)
    assert shape(dev) == shape(flat)
    assert len({s.final_cost for s in summ}) == K                  # each trial kept its own summary
    if same_plan(base, tail):
        assert chosen == c1 and np.array_equal(equv, e1) and np.array_equal(poses, ref)
    else:
        assert np.allclose(equv, e1, rtol=1e-8) and np.abs(poses - ref).max() < 1e-5
    for h in (dev, flat):
        h.close()


@pytest.mark.gpu
def test_launches_and_memory(gpu):
    g, base = window()
    live0 = host.live_resources()
    a = make_anchor(g, max_meas=4096)
    feed(a, g)
    chain = host.AnchoredChain(4096)
    dev = host.PoseGraphSolver(4096, 32768)
    resident(dev, base)
    o = options(dev, "default")
    n_nodes = len(base["init"])
    n = chain.run(a)
    chain.observe(a, n, SELF, XY, Z)
    chain.compact(n, keep=False)
    chain.init_mask(a, SELF, n_nodes)
    chain.init_solve(dev, 2048, 32, 1, 30, np.inf, options=o)      # acquires what the calls below need
    dev.last_multistart()
    live1 = host.live_resources()
    counts = []
    for K in (1, 3, 32):
        n0 = host.launch_count()
        chain.init_mask(a, SELF, n_nodes)
        counts.append(host.launch_count() - n0)
        n0 = host.launch_count()
        chain.init_solve(dev, 2048, K, 1, 30, np.inf, options=o)
        counts.append(host.launch_count() - n0)
        c, summ, _ = dev.last_multistart()
        assert len(summ) == K and 0 <= c < K and host.live_resources() == live1
    assert counts == [1, 7] * 3
    for h in (dev, a):
        h.close()
    del chain
    assert host.live_resources() == live0


def _build_cpp(tmp_path):
    exe = str(tmp_path / "multistart_resident_smoke")
    cmd = ["g++", "-std=c++17", "-Wall", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(CUDA, "include"),
           os.path.join(ROOT, "tests", "cpp", "multistart_resident_smoke.cpp"), "-L", CSRC, "-lomniswarm_b200",
           f"-Wl,-rpath,{CSRC}", "-L", os.path.join(CUDA, "lib64"), "-lcudart", f"-Wl,-rpath,{os.path.join(CUDA, 'lib64')}",
           "-o", exe]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stderr
    return exe


@pytest.mark.skipif(shutil.which("g++") is None or not os.path.isdir(os.path.join(CUDA, "include")),
                    reason="g++ or the CUDA headers missing")
def test_cpp_smoke_compiles_and_reports_no_device(tmp_path):
    exe = _build_cpp(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr


@pytest.mark.gpu
def test_cpp_smoke_on_gpu(gpu, tmp_path):
    exe = _build_cpp(tmp_path)
    r = subprocess.run([exe], capture_output=True, text=True)
    assert r.returncode == 0 and "multistart resident ok" in r.stdout, r.stdout + r.stderr
