"""GPU: the re-anchoring of loops and detections onto the window (osb_anchor_*) against its oracle
(oracle/anchor_ref.anchor) on synthetic swarms, across window slides, and feeding the pose-graph solve."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib as _l, synth
from oracle import anchor_ref as ar
from backend_harness import feed, make_anchor, pcm_state

pytestmark = pytest.mark.gpu
INT_FIELDS = ("id", "type", "status", "frame_a", "frame_b", "node_a", "node_b", "stamp_a", "stamp_b", "dt_err_ns", "skip",
              "ia", "ib", "huber", "factor_type")


def close(got, want):
    """agreement to 1e-12 relative: only libm-vs-CUDA transcendental ulps may differ"""
    got, want = np.asarray(got, np.float64), np.asarray(want, np.float64)
    scale = np.maximum(np.abs(want), 1.0)
    assert np.all(np.abs(got - want) <= 1e-12 * scale), float(np.max(np.abs(got - want) / scale))


def check(res, ref):
    assert len(res) == len(ref)
    for f in INT_FIELDS:
        assert np.array_equal(res[f], ref[f]), f
    close(res["dpos"], ref["dpos"])
    close(res["payload"], ref["payload"])
    for f in ("id_a", "id_b"):
        assert np.array_equal(res["edge"][f], ref["edge"][f])
    for f in ("rel_pose", "cov", "odom_a", "odom_b", "len_a", "len_b"):
        close(res["edge"][f], ref["edge"][f])


def oracle(g, yaw=None, window=None):
    yaw = np.ones(g["max_drones"], np.uint8) if yaw is None else yaw
    return ar.anchor(g["trajs"], window or g["window"], g["meas"], yaw, g["prm"])


@pytest.mark.parametrize("seed", [0, 1])
def test_matches_oracle_on_a_synthetic_swarm(gpu, seed):
    g = synth.anchor_swarm(5, 60, 600, seed=seed)
    a = make_anchor(g)
    feed(a, g)
    yaw = np.ones(g["max_drones"], np.uint8)
    yaw[2] = 0
    n0 = host.launch_count()
    res = a.run(yaw)
    assert host.launch_count() == n0 + 1
    ref = oracle(g, yaw)
    check(res, ref)
    counts = np.bincount(ref["status"], minlength=6)
    assert np.delete(counts, ar.EMPTY_WINDOW).min() > 0
    # run_dev on a caller stream gives the same rows
    out = torch.zeros(len(res) * _l.ANCHOR_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
    st = torch.cuda.Stream()
    n = a.run_dev(out.data_ptr(), st.cuda_stream, yaw)
    st.synchronize()
    assert n == len(res) and host.launch_count() == n0 + 2
    assert out.cpu().numpy().tobytes() == res.tobytes()
    a.close()


def test_window_slides_over_several_runs(gpu):
    g = synth.anchor_swarm(4, 50, 400, seed=5)
    a = make_anchor(g, max_meas=2000)
    feed(a, g)
    rng = np.random.default_rng(0)
    stamps, first, entries = g["window"]
    frames = [(int(stamps[f]), entries[first[f]:first[f + 1]].copy()) for f in range(len(stamps))]
    extra = synth.anchor_swarm(4, 50, 300, seed=6)["meas"]
    extra["id"] += 10_000
    for step in range(4):
        if step == 0:
            frames = frames[3:]                                              # front deletion
        elif step == 1:
            del frames[int(rng.integers(1, len(frames) - 1))]                # deletion at a random index
        elif step == 2:
            last = frames[-1]
            for k in range(1, 4):                                            # appended frames
                e = last[1].copy()
                e["stamp"] += k * 400_000_000
                e["block"] += 1000 * k
                frames.append((last[0] + k * 400_000_000, e))
        else:
            part = extra[:150]
            a.add_measurements(part)
            g["meas"] = np.concatenate([g["meas"], part])
        win = (np.array([f[0] for f in frames], np.int64), np.cumsum([0] + [len(f[1]) for f in frames]).astype(np.int32),
               np.concatenate([f[1] for f in frames]))
        a.set_window(*win)
        check(a.run(), oracle(g, window=win))
    a.close()


def test_capacity_and_invalid_input_leave_the_handle_unchanged(gpu):
    g = synth.anchor_swarm(3, 20, 100, seed=7)
    a = make_anchor(g, 100, len(g["window"][2]), traj_margin=0)
    feed(a, g)
    before = a.run()
    check(before, oracle(g))
    d, (st, p) = next(iter(g["trajs"].items()))
    for call, status in ((lambda: a.add_measurements(g["meas"][:1]), _l.ERR_CAPACITY),
                         (lambda: a.push_odometry(d, st[-1:] + 10, p[-1:]), _l.ERR_CAPACITY),
                         (lambda: a.set_window(g["window"][0][:1], [0, len(g["window"][2]) + 1],
                                               np.concatenate([g["window"][2], g["window"][2][:1]])), _l.ERR_CAPACITY),
                         (lambda: a.push_odometry(g["max_drones"], st[:1], p[:1]), _l.ERR_INVALID),
                         (lambda: a.set_window([1], [0, 2], np.concatenate([g["window"][2][:1]] * 2)), _l.ERR_INVALID)):
        with pytest.raises(_l.OsbError) as e:
            call()
        assert e.value.status == status
    assert a.size() == (int((g["meas"]["type"] == 0).sum()), int((g["meas"]["type"] != 0).sum()))
    assert a.run().tobytes() == before.tobytes()
    b = host.LoopAnchor(g["max_drones"], 64, 8, 8, 1.0, 1e-3, 1e-3)
    b.push_odometry(0, [5, 6], np.tile(np.r_[0, 0, 0, 1.0, 0, 0, 0], (2, 1)))
    with pytest.raises(_l.OsbError) as e:
        b.push_odometry(0, [6], np.r_[0, 0, 0, 1.0, 0, 0, 0][None])           # not after the last stamp
    assert e.value.status == _l.ERR_INVALID
    b.close()
    a.close()


def test_empty_window_and_resources(gpu):
    live = host.live_resources()
    g = synth.anchor_swarm(3, 10, 50, seed=8)
    a = make_anchor(g)
    feed(a, g)
    a.set_window(np.zeros(0, np.int64), np.zeros(1, np.int32), np.zeros(0, _l.WINDOW_ENTRY_DTYPE))
    res = a.run()
    assert (res["status"] == _l.ANCHOR_EMPTY_WINDOW).all() and (res["skip"] == 1).all()
    check(res, oracle(g, window=(np.zeros(0, np.int64), np.zeros(1, np.int32), np.zeros(0, ar.ENTRY_DTYPE))))
    a.close()
    assert host.live_resources() == live


def test_factor_rows_feed_the_solver_as_the_oracles_do(gpu):
    g = synth.anchor_swarm(4, 30, 300, seed=9, with_orphans=False)
    a = make_anchor(g)
    feed(a, g)
    res = a.run()
    ref = oracle(g)
    base = synth.anchor_window_graph(g)
    solver = host.PoseGraphSolver(4096, 32768)
    o = solver.default_options()
    o.function_tolerance = 1e-14; o.gradient_tolerance = 1e-11; o.parameter_tolerance = 1e-12
    o.pcg_tolerance = 1e-8; o.max_pcg_iterations = 2000; o.max_iterations = 300
    poses = []
    for rows in (host.anchored_factor_rows(res), host.anchored_factor_rows(ref)):
        assert len(rows[0]) > 50
        gg = dict(base, ftype=np.r_[base["ftype"], rows[0]], ia=np.r_[base["ia"], rows[1]], ib=np.r_[base["ib"], rows[2]],
                  payload=np.r_[base["payload"], rows[3]], huber=np.r_[base["huber"], rows[4]])
        p, s = solver.solve(gg, o)
        assert s.termination in (0, 1, 2), s.termination
        poses.append(p)
    assert np.abs(poses[0] - poses[1]).max() < 1e-5
    # the re-anchored edges go to the PCM state as they are
    keep = pcm_state(g, 16, 512).reject(host.anchored_loop_edges(res[res["status"] == 0]), res["id"][res["status"] == 0])
    assert keep.any()
    solver.close()
    a.close()
