"""osb_solver_solve_resident_dev: the resident window solved with a tail of loop / detection rows read on the device.
Against osb_solver_solve of the concatenated list (bit-identical where both pick the same shape and plan), over the real
chain run_dev -> reject_anchored -> compact_factors_dev with window slides, mixed with host calls, refused calls, launch
and memory accounting, stream capture and the cooperative path; plus the C++ adapter smoke program."""
import os
import shutil
import subprocess

import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l, synth
from oracle import solver_ref as sr
from backend_harness import KEYS, feed, make_anchor, options, pcm_state, resident

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CSRC = os.path.join(ROOT, "omni-swarm_b200", "csrc")
CUDA = os.environ.get("CUDA_HOME", "/usr/local/cuda")


def concat(base, tail, init):
    g = {k: np.concatenate([base[k], tail[k]]) if len(tail["ftype"]) else base[k].copy() for k in KEYS}
    g["fixed"], g["init"] = base["fixed"], init
    return g


def candidate_rows(base, k, rng, kinds=(0, 1)):
    """loop-like rows between random nodes: RELPOSE at the truth-ish relative pose, or a weak UWB distance"""
    init, n = base["init"], len(base["init"])
    t = {"ftype": [], "ia": [], "ib": [], "payload": [], "huber": []}
    while len(t["ftype"]) < k:
        a, b = (int(x) for x in rng.integers(0, n, 2))
        if a == b:
            continue
        ty = int(kinds[len(t["ftype"]) % len(kinds)])
        pl = np.zeros(_l.PAYLOAD_LEN)
        A, B = init[a], init[b]
        if ty == 1:
            c, s = np.cos(A[3]), np.sin(A[3])
            d = B[:3] - A[:3]
            pl[:4] = [c * d[0] + s * d[1], -s * d[0] + c * d[1], d[2], B[3] - A[3]]
            pl[:4] += rng.normal(0, 0.02, 4)
            pl[4:20] = (np.eye(4) * 2.0).reshape(-1)
        else:
            pl[0], pl[1] = np.linalg.norm(A[:3] - B[:3]) + rng.normal(0, 0.02), 3.0
        t["ftype"].append(ty); t["ia"].append(a); t["ib"].append(b); t["payload"].append(pl); t["huber"].append(1)
    return {k_: np.array(v, np.float64 if k_ == "payload" else (np.uint8 if k_ == "huber" else np.int32))
            for k_, v in t.items()}


def plan_keeping_rows(base, k, seed, kinds=(0, 1)):
    """k candidate rows, kept only while the chain plan of base + rows stays the base's"""
    rng = np.random.default_rng(seed)
    plan0 = host.PoseGraphSolver.chain_plan(base)
    cand = candidate_rows(base, 4 * k + 8, rng, kinds)
    keep = []
    for i in range(len(cand["ftype"])):
        if len(keep) == k:
            break
        trial = {k_: cand[k_][keep + [i]] for k_ in KEYS}
        p = host.PoseGraphSolver.chain_plan(concat(base, trial, base["init"]))
        if all(np.array_equal(x, y) for x, y in zip(p, plan0)):
            keep.append(i)
    return {k_: cand[k_][keep] for k_ in KEYS}


def same_plan(base, tail):
    p0 = host.PoseGraphSolver.chain_plan(base)
    p1 = host.PoseGraphSolver.chain_plan(concat(base, tail, base["init"]))
    return all(np.array_equal(x, y) for x, y in zip(p0, p1))


def shape(solver):
    c = solver.phase_cycles()
    return tuple(c[k] for k in ("ctas", "cluster", "j_in_smem", "chain_preconditioner", "inner_fp32"))


def window():
    g = synth.anchor_swarm(4, 30, 300, seed=9, with_orphans=False)
    return g, synth.anchor_window_graph(g)


@pytest.mark.gpu
@pytest.mark.parametrize("kind,k", [("default", 24), ("tight", 24), ("fp64", 24), ("jacobi", 24), ("default", 0)])
def test_bit_identical_to_one_shot(gpu, kind, k):
    _, base = window()
    tail = plan_keeping_rows(base, k, seed=3)
    assert len(tail["ftype"]) == k and same_plan(base, tail)
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    o = options(dev, kind)
    resident(dev, base)
    buf = host.FactorRows(64)
    buf.set(tail)
    buf.solve(dev, k + 3, o)
    poses = dev.graph_get_poses()
    s = dev.last_summary()
    sh = shape(dev)
    ref, s1 = flat.solve(concat(base, tail, base["init"]), o)
    assert np.array_equal(poses, ref)
    assert (s.final_cost, s.iterations, s.pcg_iterations, s.n_residuals, s.termination) == \
        (s1.final_cost, s1.iterations, s1.pcg_iterations, s1.n_residuals, s1.termination)
    assert sh == shape(flat)
    assert s.initial_cost == s1.initial_cost and s.solve_ms > 0.0
    for h in (dev, flat):
        h.close()


def slide(win, base, d):
    """drop the window's blocks < d: entries renumbered block - d, emptied frames removed; the graph as drop_oldest does"""
    stamps, first, entries = win
    keep_f, new_e, new_first = [], [], [0]
    for f in range(len(stamps)):
        e = entries[first[f]:first[f + 1]]
        e = e[e["block"] >= d].copy()
        if len(e):
            e["block"] -= d
            keep_f.append(stamps[f]); new_e.append(e); new_first.append(new_first[-1] + len(e))
    win = (np.array(keep_f, np.int64), np.array(new_first, np.int32), np.concatenate(new_e))
    sel = (base["ia"] >= d) & (base["ib"] >= d)
    nb = {k: base[k][sel].copy() for k in KEYS}
    nb["ia"] -= d; nb["ib"] -= d
    nb["fixed"] = base["fixed"][d:].copy()
    nb["fixed"][0] = 1
    nb["init"] = base["init"][d:].copy()
    return win, nb


@pytest.mark.gpu
def test_rows_from_the_device_chain(gpu):
    g, base = window()
    a = make_anchor(g, max_meas=4096)
    g0 = dict(g, meas=g["meas"][:200])
    feed(a, g0)
    st = pcm_state(g, 32, 1024)
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    resident(dev, base)
    chain = host.AnchoredChain(4096)
    o = options(dev, "tight")
    win = g["window"]
    exact = close = 0
    for r in range(4):
        if r == 1:
            a.add_measurements(g["meas"][200:])                # new measurements
        if r >= 2:                                            # the window slides by its first frame's blocks
            d = int(win[2]["block"][:win[1][1]].max()) + 1
            start = dev.graph_get_poses()
            win, base = slide(win, base, d)
            dev.graph_drop_oldest(d)
            dev.graph_set_fixed(0)
            a.set_window(*win)
            base["init"] = start[d:]
        start = dev.graph_get_poses()
        chain(a, st)
        chain.solve(dev, 2048, o)
        poses = dev.graph_get_poses()
        s = dev.last_summary()
        tail = chain.factors.on_host(chain.stream)
        assert len(tail["ftype"]) > 0
        gcat = concat(base, tail, start)
        gcat["fixed"] = base["fixed"]
        ref, s1 = flat.solve(gcat, o)
        if same_plan(base, tail) and shape(dev) == shape(flat):
            assert np.array_equal(poses, ref) and s.final_cost == s1.final_cost
            exact += 1
        else:
            assert np.abs(poses - ref).max() < 1e-5
            assert abs(s.final_cost - s1.final_cost) <= 1e-8 * abs(s1.final_cost)
            close += 1
        if r == 0:                                             # the small window against the oracle solver
            orc = sr.solve(gcat)["poses"]
            assert np.abs(poses - orc).max() < 1e-4
        base["init"] = poses
    assert exact + close == 4
    for h in (dev, flat, st, a):
        h.close()


@pytest.mark.gpu
def test_mixed_with_host_calls(gpu):
    _, base = window()
    tail = plan_keeping_rows(base, 16, seed=5)
    dev, flat, twin = (host.PoseGraphSolver(4096, 32768) for _ in range(3))
    o = options(dev, "tight")
    resident(dev, base)
    resident(twin, base)
    buf = host.FactorRows(64)
    buf.set(tail)
    buf.solve(dev, 16, o)
    p1 = dev.graph_get_poses()                                 # graph_get_poses after a device call
    r1, _ = flat.solve(concat(base, tail, base["init"]), o)
    assert np.array_equal(p1, r1)
    moved = p1 + np.r_[0.03, -0.02, 0.01, 0.005] * (1 - base["fixed"][:, None])
    dev.graph_set_poses(0, moved)                              # set_poses before a device call
    buf.solve(dev, 16, o)
    p2 = dev.graph_get_poses()
    r2, _ = flat.solve(concat(base, tail, moved), o)
    assert np.array_equal(p2, r2)
    other = synth.pose_graph(3, 12, n_uwb=20, n_loop=15, n_det=8, n_bearing=9, seed=3)
    q_dev, _ = dev.solve(other, o)                             # a one-shot solve in between ...
    q_ref, _ = flat.solve(other, o)
    assert np.array_equal(q_dev, q_ref)
    buf.solve(dev, 16, o)                                      # ... and the device call after it
    p3 = dev.graph_get_poses()
    r3, _ = flat.solve(concat(base, tail, p2), o)
    assert np.array_equal(p3, r3)
    s_dev = dev.solve_resident(o)                              # solve_resident after a device call
    twin.graph_set_poses(0, p3)
    s_twin = twin.solve_resident(o)
    assert np.array_equal(dev.graph_get_poses(), twin.graph_get_poses()) and s_dev.final_cost == s_twin.final_cost
    for h in (dev, flat, twin):
        h.close()


@pytest.mark.gpu
def test_refusals(gpu):
    _, base = window()
    n = len(base["init"])
    tail = plan_keeping_rows(base, 8, seed=7)
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    o = options(dev, "tight")
    resident(dev, base)
    buf = host.FactorRows(64)
    buf.set(tail)
    buf.solve(dev, 8, o)
    good = dev.graph_get_poses()
    size = dev.graph_size()
    bad_cases = []
    for field, value, code in (("ftype", 3, _l.ERR_INVALID), ("ftype", -1, _l.ERR_INVALID), ("ia", n, _l.ERR_INVALID),
                               ("ib", -1, _l.ERR_INVALID), ("ib", None, _l.ERR_INVALID)):
        t = {k: v.copy() for k, v in tail.items()}
        t[field][5] = t["ia"][5] if value is None else value
        bad_cases.append((t, None, code))
    bad_cases += [(tail, -1, _l.ERR_INVALID), (tail, 9, _l.ERR_CAPACITY)]
    for t, count, code in bad_cases:
        buf.set(t, count)
        buf.solve(dev, 8, o)
        with pytest.raises(_l.OsbError) as e:
            dev.last_summary()
        assert e.value.status == code
        assert np.array_equal(dev.graph_get_poses(), good) and dev.graph_size() == size
    buf.set(tail)                                              # the next valid call is correct
    buf.solve(dev, 8, o)
    ref, _ = flat.solve(concat(base, tail, good), o)
    assert np.array_equal(dev.graph_get_poses(), ref)
    # refused on the host: nothing enqueued
    n0 = host.launch_count()
    args = buf.ptrs()
    for i in range(6):
        a2 = list(args)
        a2[i] = 0
        with pytest.raises(_l.OsbError):
            dev.solve_resident_dev(8, *a2, torch.cuda.current_stream().cuda_stream, o)
    with pytest.raises(_l.OsbError) as e:
        dev.solve_resident_dev(-1, *args, 0, o)
    assert e.value.status == _l.ERR_INVALID
    with pytest.raises(_l.OsbError) as e:
        dev.solve_resident_dev(32768, *args, 0, o)
    assert e.value.status == _l.ERR_CAPACITY
    empty = host.PoseGraphSolver(64, 256)
    with pytest.raises(_l.OsbError):
        empty.solve_resident_dev(8, *args, 0, o)
    assert host.launch_count() == n0
    for h in (dev, flat, empty):
        h.close()


@pytest.mark.gpu
def test_launches_and_memory(gpu):
    _, base = window()
    live0 = host.live_resources()
    dev = host.PoseGraphSolver(4096, 32768)
    resident(dev, base)
    rng = np.random.default_rng(11)
    big = candidate_rows(base, 3000, rng)
    buf = host.FactorRows(3000)
    o = options(dev, "default")
    buf.set(big, 1)
    buf.solve(dev, 3000, o)
    dev.last_summary()
    live1 = host.live_resources()
    counts = []
    for k in (0, 1, 3000):
        buf.set(big, k)
        n0 = host.launch_count()
        buf.solve(dev, 3000, o)
        counts.append(host.launch_count() - n0)
        s = dev.last_summary()
        assert np.isfinite(s.final_cost) and s.n_residuals == sr_residuals(base) + sr_residuals(
            {k_: big[k_][:k] for k_ in KEYS})
        assert host.live_resources() == live1
    assert counts[0] == counts[1] == counts[2] == 6
    dev.close()
    assert host.live_resources() == live0


def sr_residuals(g):
    t = np.asarray(g["ftype"])
    if len(t) == 0:
        return 0
    det = np.where((np.asarray(g["payload"])[:, 10].astype(int) & 1) == 1, 3, 2)
    return int(np.sum(np.where(t == 0, 1, np.where(t == 1, 4, det))))


@pytest.mark.gpu
def test_capture_of_the_whole_chain(gpu):
    g, base = window()

    def setup():
        a = make_anchor(g, max_meas=4096)
        feed(a, g)
        st = pcm_state(g, 32, 1024)
        dev = host.PoseGraphSolver(4096, 32768)
        resident(dev, base)
        return a, st, dev, host.AnchoredChain(4096)

    a, st, dev, chain = setup()
    o = options(dev, "default")
    want = []
    for _ in range(3):                                        # the uncaptured sequence: three solves
        chain(a, st)
        chain.solve(dev, 2048, o)
        want.append(dev.graph_get_poses())
    want = want[1:]
    a2, st2, dev2, chain2 = setup()
    chain2(a2, st2)                                           # warm: the plan, the tables and the poses are on the device
    chain2.solve(dev2, 2048, o)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph, stream=chain2.stream, capture_error_mode="global"):
        chain2(a2, st2)
        chain2.solve(dev2, 2048, o)
    for w in want:                                            # every replay's poses reach the host copy
        graph.replay()
        torch.cuda.synchronize()
        assert np.array_equal(dev2.graph_get_poses(), w)
    # a call that needs host work (the poses changed on the host) is refused inside a capture, which still completes
    dev2.graph_set_poses(0, want[-1])
    g2 = torch.cuda.CUDAGraph()
    x = torch.zeros(4, device="cuda")
    with torch.cuda.graph(g2, stream=chain2.stream, capture_error_mode="global"):
        with pytest.raises(_l.OsbError) as e:
            chain2.solve(dev2, 2048, o)
        x += 1
    assert e.value.status == _l.ERR_INVALID
    g2.replay()
    torch.cuda.synchronize()
    assert float(x.sum()) == 4.0
    for h in (a, st, dev, a2, st2, dev2):
        h.close()


@pytest.mark.gpu
def test_cooperative_path(gpu):
    _, base = window()
    k = 26000
    tail = candidate_rows(base, k, np.random.default_rng(13), kinds=(0,))
    tail["payload"][:, 1] = 0.05                               # weak ranges
    dev, flat = host.PoseGraphSolver(4096, 32768), host.PoseGraphSolver(4096, 32768)
    o = options(dev, "tight")
    resident(dev, base)
    buf = host.FactorRows(k)
    buf.set(tail)
    buf.solve(dev, k, o)
    poses = dev.graph_get_poses()
    s = dev.last_summary()
    assert shape(dev)[1] == 0.0                                # cooperative grid
    ref, s1 = flat.solve(concat(base, tail, base["init"]), o)
    assert shape(dev) == shape(flat)
    if same_plan(base, tail):
        assert np.array_equal(poses, ref) and s.final_cost == s1.final_cost
    else:
        assert np.abs(poses - ref).max() < 1e-5 and abs(s.final_cost - s1.final_cost) <= 1e-8 * abs(s1.final_cost)
    for h in (dev, flat):
        h.close()


def _build_cpp(tmp_path):
    exe = str(tmp_path / "device_tail_smoke")
    cmd = ["g++", "-std=c++17", "-I", os.path.join(ROOT, "include"), "-I", os.path.join(CUDA, "include"),
           os.path.join(ROOT, "tests", "cpp", "device_tail_smoke.cpp"), "-L", CSRC, "-lomniswarm_b200",
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
    assert r.returncode == 0 and "device tail ok" in r.stdout, r.stdout + r.stderr
