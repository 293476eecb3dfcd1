"""GPU: osb_frontend_compute_loop -- the loop edge of every hit (compute_loop + the frame-level compute_correspond_features,
loop_detector.cpp:431-537, 627-836) against oracle/loop_ref.py.  Keyframe records are built on the host from a planar
four-direction scene (synth.loop_scene: exact geometry, one plane per direction) with per-point descriptors, unflagged
landmarks and outlier matches, then go through the real ingest / query / query_received.  The oracle is fed the device's
query result (the matcher and the homography filter are tested elsewhere) and must give the same status, correspondences,
inlier mask and PnP winner, the same poses to 1e-8, and the true delta within the data's float32 rounding."""
import ctypes as C

import numpy as np
import pytest

from omniswarm_b200 import synth, host, lib
from frontend_harness import (EB, LOOP_COV, LOOP_PARAMS, RB, RS, SC, cand_own, filled, loop_frontend, loop_oracle,
                              own_query, upload)
import frontend_harness as fh

pytestmark = pytest.mark.gpu

ND, MN = 4, 200
QDIR = 1
NPT = synth.LOOP_NPT
record, noisy_g = synth.loop_record, synth.loop_noisy_g


def oracle(res, query_rec, hit_rec, cand, params=None, K=None):
    return loop_oracle(res, query_rec, hit_rec, cand, SC["K"] if K is None else K, SC["ext"],
                       dict(LOOP_PARAMS, **(params or {})), QDIR)


def run_loop(fe, st, rec_ptr, res_ptr, cands):
    out = filled(len(cands) * EB)
    fe.compute_loop(rec_ptr, res_ptr, cands, out.data_ptr(), st)
    fe.finish(st)
    return fh.edges(out, len(cands))


def check(raw, ref, truth=True):
    e = lib.LoopEdgeResult.from_buffer_copy(raw)
    assert e.status == ref["status"], (e.status, ref["status"])
    assert e.n_corr == ref["n_corr"]
    n = e.n_corr
    if n:
        assert list(e.corr_dir_new[:n]) == ref["dir_new"].tolist() and list(e.corr_idx_new[:n]) == ref["idx_new"].tolist()
        assert list(e.corr_dir_old[:n]) == ref["dir_old"].tolist() and list(e.corr_idx_old[:n]) == ref["idx_old"].tolist()
        assert e.matched_dir_count == ref["matched_dir_count"]
    assert not any(e.inlier[n:])
    if ref["pnp"] is None:
        assert not any(e.inlier[:n]) and e.pnp.pnp_success == 0
        return e
    p = ref["pnp"]
    assert bool(e.pnp.pnp_success) == p["success"] and e.pnp.winner == p["winner"] and e.pnp.n_inliers == p["n_inliers"]
    assert np.array_equal(np.array(e.inlier[:n], np.uint8), p["mask"])
    if p["success"]:
        assert np.abs(np.array(e.pnp.pose_cam) - p["pose"]).max() < 1e-8
        assert np.abs(np.array(e.relative_pose) - ref["relative_pose"]).max() < 1e-8
        assert np.abs(np.array(e.pnp.dp_old_to_new) - ref["loop"]["dp"]).max() < 1e-8
        assert abs(e.pnp.rperr - ref["loop"]["rperr"]) < 1e-8
        assert abs(e.pnp.md - ref["loop"]["md"]) <= 1e-8 * max(1.0, ref["loop"]["md"])
        if truth and e.status == lib.LOOP_ACCEPTED:          # exact geometry: only float32 rounding of the inputs
            assert np.abs(np.array(e.relative_pose) - SC["delta_true"]).max() < 1e-5
    return e


def same_pnp(a, b):
    """two osb_pnp_result equal bit for bit but for the unused `reserved` field"""
    a, b = lib.PnpResult.from_buffer_copy(bytes(a)), lib.PnpResult.from_buffer_copy(bytes(b))
    a.reserved = b.reserved = 0
    return bytes(a) == bytes(b)


def test_own_query_local_hit_and_pnp_inputs(gpu):
    st = fh.stream()
    fe = loop_frontend()
    old, new = record(1, 100, "old"), record(1, 101, "new", seed=1, g=noisy_g(1))
    rt, res_t, res = own_query(fe, st, old, new)
    assert res.accepted and not res.swapped and res.hit_dir == QDIR and sum(res.geo_valid) == ND
    cand = cand_own()
    raw = run_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), [cand])[0]
    ref = oracle(res, new, old, cand)
    e = check(raw, ref)
    assert e.status == lib.LOOP_ACCEPTED and e.pnp.odometry_consistent == 1 and e.pnp.md < 1e-6
    assert (e.drone_id_a, e.drone_id_b, e.msg_id_a, e.msg_id_b) == (1, 1, 100, 101)
    assert (e.main_dir_new, e.main_dir_old) == (QDIR, QDIR)
    # the PnP stage's inputs are those of a host caller of osb_pnp_ransac: the same outputs, bit for bit
    prm = ref["pnp_params"]
    mask, pr_host = host.pnp_ransac([prm], max_n=lib.LOOP_MAXN)[0]
    assert same_pnp(pr_host, e.pnp) and np.array_equal(mask, np.array(e.inlier[:e.n_corr], np.uint8))
    fe.close()


def test_own_query_remote_hit_is_swapped(gpu):
    """the own keyframe hits a remote one: new = the remote keyframe, its 3-D landmarks read from the remote store"""
    st = fh.stream()
    fe = loop_frontend()
    remote = record(2, 200, "new", seed=2, g=noisy_g(2))
    t = upload([remote])
    fe.ingest(t.data_ptr(), 1, -1, st)
    own = record(1, 100, "old")
    # the remote record's buffer is overwritten: what compute_loop reads of it must come from the store
    t.copy_(upload([record(2, 200, "new", seed=99, scramble=True)]))
    rt, res_t, res = own_query(fe, st, None, own, nonkeyframe=True, ingest_old=False)
    assert res.accepted and res.swapped and res.hit_msg_id == 200 and res.hit_drone_id == 2
    cand = dict(pose_query=SC["pose_old"], pose_hit=SC["pose_new"])
    raw = run_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), [cand])[0]
    e = check(raw, oracle(res, own, remote, cand))
    assert e.status == lib.LOOP_ACCEPTED and (e.drone_id_a, e.drone_id_b, e.msg_id_a, e.msg_id_b) == (1, 2, 100, 200)
    assert e.pnp.md == 0.0                                         # inter-drone: no odometry check
    fe.close()


def test_received_batch_equals_single_calls(gpu):
    """a round of 10 received keyframes: hits with outliers, a failed homography pair (the 1-3-match quirk), init mode,
    misses; one call for all, each equal to its one-candidate call and to the oracle"""
    st = fh.stream()
    fe = loop_frontend()
    old = record(1, 100, "old")
    ot = upload([old])
    fe.ingest_own(ot.data_ptr(), st)
    recs, cands = [], []
    rng = np.random.default_rng(7)
    for r in range(10):
        g = noisy_g(10 + r) if r % 5 != 4 else synth.descriptor_db(ND, 4096, 300 + r)
        recs.append(record(2 + r % 3, 300 + r, "new", seed=20 + r, g=g, n_outliers=2 + r % 4,
                           few_flags_dir=(r % 4) if r in (1, 6) else None))
        cands.append(dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"], init_mode=(r == 2),
                          odom_rel=rng.normal(size=7), cov=LOOP_COV))
    rt = upload(recs)
    res_t = filled(10 * RS)
    fe.query_received(rt.data_ptr(), 10, -1, res_t.data_ptr(), st, init_mode=[c["init_mode"] for c in cands])
    fe.finish(st)
    results = fh.results(res_t, 10)
    batch = run_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), cands)
    statuses = []
    for r in range(10):
        single = run_loop(fe, st, rt.data_ptr() + r * RB, res_t.data_ptr() + r * RS, [cands[r]])[0]
        assert single == batch[r], f"candidate {r}: batch and single call differ"
        e = check(batch[r], oracle(results[r], recs[r], old, cands[r]))
        statuses.append(e.status)
        if r in (1, 6):                          # the failed pair contributed its two flagged matches
            assert any(results[r].geo_valid[j] == 0 and results[r].dir_new[j] >= 0 for j in range(ND))
    assert statuses.count(lib.LOOP_ACCEPTED) >= 6 and statuses.count(lib.LOOP_NO_HIT) == 2, statuses
    fe.close()


def test_depth_keyframe_camera(gpu):
    """a depth-camera handle lifts the old frame through set_depth_camera's pinhole and extrinsics"""
    st = fh.stream()
    K2 = np.array([80.0, 80.0, 40.0, 30.0])
    fe = loop_frontend(cameras=None, loop_params=False)
    fe.set_depth_camera(K2, SC["ext"])
    fe.set_loop_params(**LOOP_PARAMS)
    old, new = record(1, 100, "old"), record(1, 101, "new", seed=3, g=noisy_g(3))
    rt, res_t, res = own_query(fe, st, old, new)
    cand = cand_own()
    raw = run_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), [cand])[0]
    check(raw, oracle(res, new, old, cand, K=K2), truth=False)      # the pixels were made for another camera
    fe.close()


def test_every_status_code(gpu):
    st = fh.stream()
    fe = loop_frontend()
    old, new = record(1, 100, "old"), record(1, 101, "new", seed=4, g=noisy_g(4))
    rt, res_t, res = own_query(fe, st, old, new)
    seen = {}
    by_msg = {100: old, 101: new}

    def go(params, cand, rec=new, rt_=rt, res_t_=res_t, res_=res):
        fe.set_loop_params(**dict(LOOP_PARAMS, **params))
        raw = run_loop(fe, st, rt_.data_ptr(), res_t_.data_ptr(), [cand])[0]
        e = check(raw, oracle(res_, rec, by_msg.get(res_.hit_msg_id), cand, params))
        seen[e.status] = seen.get(e.status, 0) + 1
        return e

    e = go({}, cand_own())
    assert e.status == lib.LOOP_ACCEPTED
    n = e.n_corr
    assert go(dict(min_loop_num=n), cand_own()).status == lib.LOOP_TOO_FEW_COMMON
    assert go(dict(min_loop_num=n, init_mode_min_loop_num=n - 1), cand_own(init_mode=True)).status == lib.LOOP_ACCEPTED
    assert go(dict(min_loop_num=4 * NPT + 1), cand_own()).status == lib.LOOP_FEW_LANDMARKS
    assert go(dict(min_direction_loop=5), cand_own()).status == lib.LOOP_CORRESPONDENCE_FAILED
    assert go(dict(max_loop_dis=0.1), cand_own()).status == lib.LOOP_NOT_VERIFIED
    far = np.concatenate([SC["delta_true"][:3] + 1.0, SC["delta_true"][3:]])
    assert go(dict(), cand_own(odom=far)).status == lib.LOOP_ODOMETRY_INCONSISTENT
    bad = record(1, 102, "new", seed=5, g=noisy_g(5), scramble=True)
    bt, bres_t, bres = own_query(fe, st, None, bad, ingest_old=False)
    assert bres.accepted
    assert go(dict(reproj_thresh=1e-4), cand_own(), bad, bt, bres_t, bres).status == lib.LOOP_PNP_FAILED
    miss = record(1, 103, "new", seed=6, g=synth.descriptor_db(ND, 4096, 77))
    mt, mres_t, mres = own_query(fe, st, None, miss, ingest_old=False)
    assert go({}, cand_own(), miss, mt, mres_t, mres).status == lib.LOOP_NO_HIT
    fe.close()
    # a row put in with db_load has no keyframe behind it
    fe = loop_frontend()
    q = record(1, 101, "new", seed=4, g=noisy_g(4))
    fe.db_load(np.stack([np.ctypeslib.as_array(q.global_desc[QDIR])]), synth.local_descriptors(MN, 3)[None],
               np.array([NPT], np.int32))
    rt2, res_t2, res2 = own_query(fe, st, old, q)
    assert res2.accepted and res2.hit_msg_id == -1
    raw = run_loop(fe, st, rt2.data_ptr(), res_t2.data_ptr(), [cand_own()])[0]
    e = lib.LoopEdgeResult.from_buffer_copy(raw)
    assert e.status == lib.LOOP_NO_FRAME and e.n_corr == 0 and e.pnp.pnp_success == 0
    seen[e.status] = 1
    fe.close()
    assert set(seen) == set(range(9)), seen


def test_arguments_errors_and_resources(gpu):
    st = fh.stream()
    base = host.live_resources()
    fe = loop_frontend()
    L = fe._lib
    old, new = record(1, 100, "old"), record(1, 101, "new", seed=1, g=noisy_g(1))
    rt, res_t, res = own_query(fe, st, old, new)
    out = filled(65 * EB)
    cands = host.KeyframeFrontend.loop_candidates([cand_own()] * 65)
    c0, live0 = host.launch_count(), host.live_resources()
    for args in ((fe._h, rt.data_ptr(), res_t.data_ptr(), 0, cands, out.data_ptr()),
                 (fe._h, rt.data_ptr(), res_t.data_ptr(), 65, cands, out.data_ptr()),
                 (fe._h, None, res_t.data_ptr(), 1, cands, out.data_ptr()),
                 (fe._h, rt.data_ptr(), None, 1, cands, out.data_ptr()),
                 (fe._h, rt.data_ptr(), res_t.data_ptr(), 1, None, out.data_ptr()),
                 (fe._h, rt.data_ptr(), res_t.data_ptr(), 1, cands, None),
                 (None, rt.data_ptr(), res_t.data_ptr(), 1, cands, out.data_ptr())):
        h, r, q, n, cd, o = args
        vp = lambda x: None if x is None else C.c_void_p(x)
        assert L.osb_frontend_compute_loop(h, vp(r), vp(q), n, cd, vp(o), C.c_void_p(st)) == lib.ERR_INVALID
    assert L.osb_frontend_set_loop_params(fe._h, None) == lib.ERR_INVALID
    assert host.launch_count() == c0 and host.live_resources() == live0
    run_loop(fe, st, rt.data_ptr(), res_t.data_ptr(), [cand_own()])
    live1 = host.live_resources()
    assert live1 > live0                                    # the first call acquired the scratch
    rt64 = upload([new] * 64)                                # n candidates read n records and n results
    res64 = upload([res] * 64)
    for n in (1, 8, 64):
        c = host.launch_count()
        fe.compute_loop(rt64.data_ptr(), res64.data_ptr(), [cand_own()] * n, out.data_ptr(), st)
        assert host.launch_count() - c == 3
    assert host.live_resources() == live1
    fe.close()

    def refused(fe, call):
        with pytest.raises(lib.OsbError) as ei:
            call()
        assert ei.value.status == lib.ERR_INVALID
        fe.close()

    call = lambda fe: lambda: fe.compute_loop(rt.data_ptr(), res_t.data_ptr(), [cand_own()], out.data_ptr(), st)
    f = loop_frontend(loop_params=False); refused(f, call(f))                  # no loop parameters
    f = loop_frontend(cameras=None); refused(f, call(f))                       # no camera
    f = loop_frontend(cameras="both"); refused(f, call(f))                     # two cameras
    f = loop_frontend(geometric_filter=False); refused(f, call(f))             # the reference's USE_FUNDMENTAL path only
    f = loop_frontend(loop_params=False)                                       # after a remote ingest: no 3-D plane
    t = upload([record(2, 200, "new")])
    f.ingest(t.data_ptr(), 1, -1, st)
    refused(f, lambda: f.set_loop_params())
    # without set_loop_params nothing is allocated
    f = loop_frontend(loop_params=False)
    live = host.live_resources()
    f.ingest(t.data_ptr(), 1, -1, st)
    f.finish(st)
    assert host.live_resources() == live
    f.close()
    assert host.live_resources() == base
