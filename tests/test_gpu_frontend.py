"""GPU: the keyframe pipeline (extract -> add_to_database -> query -> per-direction match) against the oracle
composed the same way (LoopCam::generate_stereo_image_descriptor + LoopDetector database rule)."""
import numpy as np
import pytest

from omniswarm_b200 import synth, host, lib
from oracle import frontend_ref as fr
from frontend_harness import H0, RB, RS, W0, frame_images, upload
import frontend_harness as fh

pytestmark = pytest.mark.gpu

CONFIG = dict(db_capacity=256, match_index_dist=2)


def make_frontend(**kw):
    return fh.make_frontend(CONFIG, **kw)


def oracle_record(up, down):
    comp, mean = synth.pca_matrices(0)
    w, nvw = synth.superpoint_weights(0), synth.netvlad_weights(0)
    rec = []
    for d in range(4):
        u = up[d].copy(); u[H0 * 3 // 4:] = 0
        dn = down[d].copy(); dn[H0 * 3 // 4:] = 0
        ku, du, _, _ = fr.superpoint_inference(u, w, 0.015, 200, comp, mean)
        kd, dd, _, _ = fr.superpoint_inference(dn, w, 0.015, 200, comp, mean)
        g = fr.netvlad_net(u, nvw)
        qi, ti, _ = fr.bf_crosscheck(du, dd) if len(ku) > 3 else (np.zeros(0, int), np.zeros(0, int), None)
        m = -np.ones(len(ku), int); m[qi] = ti
        rec.append(dict(kpts=ku, desc=du, n_down=len(kd), g=g, stereo=m))
    return rec


def test_process_record_matches_oracle(gpu):
    fe = make_frontend(match_index_dist=5)      # reference default: the 4 rows a keyframe just added are skipped
    up, down = frame_images(1)
    rec, res = fe.process(up, down, msg_id=77)
    ref = oracle_record(up, down)
    assert rec.drone_id == 1 and rec.msg_id == 77 and rec.n_dirs == 4
    for d in range(4):
        n = rec.n_kpts[d]
        k = np.ctypeslib.as_array(rec.kpts[d])[:n]
        # small images + margin cases: require the keypoint sets to agree almost everywhere, exact where they do
        same = {tuple(x) for x in k.tolist()} & {tuple(x) for x in ref[d]["kpts"].tolist()}
        assert len(same) >= 0.9 * len(ref[d]["kpts"])
        g = np.ctypeslib.as_array(rec.global_desc[d])
        assert np.linalg.norm(g - ref[d]["g"]) < 1e-3 and abs(np.linalg.norm(g) - 1) < 1e-5
        if np.array_equal(k, ref[d]["kpts"]):
            ld = np.ctypeslib.as_array(rec.local_desc[d])[:n]
            assert np.linalg.norm(ld - ref[d]["desc"]) / np.linalg.norm(ref[d]["desc"]) < 1e-3
            assert rec.n_kpts_down[d] == ref[d]["n_down"]
    assert fe.db_size(False) == sum(1 for d in range(4) if rec.n_kpts[d] > 0) and fe.db_size(True) == 0
    assert res.accepted == 0                       # database_size() <= MATCH_INDEX_DIST gate / too-new rows
    fe.close()


def test_loop_is_found_on_revisit(gpu):
    """Revisit an old keyframe: the query returns its row, the per-direction match pairs keypoints with themselves."""
    fe = make_frontend(match_index_dist=1)
    frames = [frame_images(s) for s in range(4)]
    recs = [fe.process(*f, msg_id=i)[0] for i, f in enumerate(frames)]
    rec, res = fe.process(*frames[0], msg_id=99)               # same images as keyframe 0
    assert res.accepted == 1 and res.swapped == 0
    assert res.hit_id == 1 and res.hit_dir == 1               # row of (frame 0, direction 1): rows are frame*4+dir
    assert abs(res.hit_score - 1.0) < 1e-4
    assert list(res.dir_new) == [1, 2, 3, 0] and list(res.dir_old) == [1, 2, 3, 0]
    for slot in range(4):
        d = res.dir_new[slot]
        n = res.n_matches[slot]
        assert n == rec.n_kpts[d] == recs[0].n_kpts[d]
        assert list(res.match_new[slot][:n]) == list(range(n)) == list(res.match_old[slot][:n])
    fe.close()


def test_query_rule_device_vs_oracle(gpu):
    """Drive the database through db_load + ingest of synthetic records and compare the acceptance rule with the
    oracle's LoopDetectorDB for own / remote keyframes, init mode and non-keyframes."""
    import torch
    fe = make_frontend(match_index_dist=3, self_id=1)
    det = fr.LoopDetectorDB(self_id=1, dim=4096, inner_product_thres=0.3, init_mode_product_thres=0.2, match_index_dist=3)
    db = synth.descriptor_db(40, 4096, 5)
    fe.db_load(db[:30], remote=False); fe.db_load(db[30:], remote=True)
    for i in range(30):
        det.add_frame(i, 1, [db[i]], [10])
    for i in range(30, 40):
        det.add_frame(i, 2, [db[i]], [10])
    assert fe.db_size(False) == 30 and fe.db_size(True) == 10
    stream = fh.stream()
    rec_t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    res_t = torch.zeros(RS, dtype=torch.uint8, device="cuda")
    cases = [(1, 5, False, False), (1, 29, False, False), (1, 35, False, False), (1, 35, False, True),
             (2, 12, False, False), (2, 29, True, False), (1, 27, False, False), (1, 26, False, False)]
    for drone, row, init_mode, nonkf in cases:
        q = synth.noisy_queries(db, np.array([row]), sigma=0.3)[0]
        rec = lib.KeyframeRecord()
        rec.drone_id, rec.n_dirs = drone, 4
        for d in range(4):
            rec.n_kpts[d] = 5
        np.ctypeslib.as_array(rec.global_desc[1])[:] = q
        rec_t.copy_(torch.frombuffer(bytearray(bytes(rec)), dtype=torch.uint8))
        fe.query(rec_t.data_ptr(), res_t.data_ptr(), stream, init_mode, nonkf)
        fe.finish(stream)
        res = fh.results(res_t, 1)[0]
        rid, rdist = det.query(drone, q, init_mode, nonkf)
        assert res.hit_id == rid, (drone, row, init_mode, nonkf, res.hit_id, rid)
        assert abs(res.hit_score - rdist) < 1e-4
        assert res.accepted == int(rid != -1 and rdist > -1)
    fe.close()


def test_blank_keyframe_adds_nothing(gpu):
    """Empty input (no keypoints anywhere): landmark_num == 0 for every direction, so add_to_database adds no row
    (loop_detector.cpp:153), the query is skipped (:262) and nothing is NaN."""
    fe = make_frontend(match_index_dist=5)
    z = np.zeros((4, H0, W0), np.uint8)
    rec, res = fe.process(z, z, msg_id=1)
    assert list(rec.n_kpts) == [0, 0, 0, 0] and list(rec.n_kpts_down) == [0, 0, 0, 0]
    assert fe.db_size(False) == 0 and fe.db_size(True) == 0
    assert res.accepted == 0 and res.hit_id == -1 and list(res.n_matches) == [0, 0, 0, 0]
    g = np.ctypeslib.as_array(rec.global_desc)
    assert np.isfinite(g).all()
    assert (np.ctypeslib.as_array(rec.stereo_match) == -1).all()
    # a normal keyframe afterwards still works
    up, down = frame_images(2)
    rec2, _ = fe.process(up, down, msg_id=2)
    assert sum(rec2.n_kpts) > 0 and fe.db_size(False) == sum(1 for d in range(4) if rec2.n_kpts[d] > 0)
    fe.close()


def test_geometric_filter_in_query(gpu):
    """loop_detector.cpp:569-598 on the device: the query's matches are reduced to those whose NEW landmark has a 3-D flag
    and that pass the homography-RANSAC mask; compared with the oracle filter applied to the same matches and geometry."""
    from oracle import geometry_ref as gr
    fe = make_frontend(match_index_dist=1, geometric_filter=True, ransac_seed=3)
    frames = [frame_images(s) for s in range(4)]
    recs = [fe.process(*f, msg_id=i)[0] for i, f in enumerate(frames)]
    rec, res = fe.process(*frames[0], msg_id=99)               # revisit keyframe 0: identical landmarks on both sides
    assert res.accepted == 1 and res.swapped == 0
    for slot in range(4):
        d_new, d_old = res.dir_new[slot], res.dir_old[slot]
        n = res.n_matches[slot]
        mn = list(res.match_new[slot][:n]); mo = list(res.match_old[slot][:n])
        flags = (np.ctypeslib.as_array(rec.stereo_match[d_new]) >= 0).astype(np.uint8)
        k_new = np.ctypeslib.as_array(rec.kpts[d_new]).copy()
        k_old = np.ctypeslib.as_array(recs[0].kpts[d_old]).copy()
        ref = gr.loop_pair_filter(mn, mo, flags, k_new, k_old, 3.0, seed=3)
        if ref is None:
            assert res.geo_valid[slot] == 0 and res.n_geo[slot] == 0
            continue
        qn, qo = ref
        g = res.n_geo[slot]
        assert res.geo_valid[slot] == 1 and g == len(qn)
        assert list(res.geo_new[slot][:g]) == qn.tolist() and list(res.geo_old[slot][:g]) == qo.tolist()
        # identical frames: every flagged match is an exact inlier of the identity homography
        assert g == int(sum(flags[q] for q in mn))
    fe.close()
    # filter off (default): the geometry fields stay zero
    fe = make_frontend(match_index_dist=1)
    for i, f in enumerate(frames):
        fe.process(*f, msg_id=i)
    _, res = fe.process(*frames[0], msg_id=99)
    assert list(res.geo_valid) == [0, 0, 0, 0] and list(res.n_geo) == [0, 0, 0, 0]
    fe.close()


def test_geometric_filter_on_loaded_rows(gpu):
    """Rows put in with db_load get their landmarks_2d / stereo_match through db_set_geometry; a query that hits such a
    row runs the geometric filter on them (and treats every landmark as flagged when no geometry was set)."""
    import torch
    from oracle import geometry_ref as gr
    fe = make_frontend(match_index_dist=1, geometric_filter=True, ransac_seed=0)
    rng = np.random.default_rng(2)
    n_rows, mn = 12, 200
    g = synth.descriptor_db(n_rows, 4096, 9)
    ld = synth.local_descriptors(mn, 77)[None].repeat(n_rows, 0).copy()          # same 200 local descriptors in every row
    nk = np.full(n_rows, 150, np.int32)
    fe.db_load(g, ld, nk, remote=False)
    k_old = np.zeros((n_rows, mn, 2), np.float32)
    k_old[:, :150] = rng.uniform(0, 90, (n_rows, 150, 2)).astype(np.float32)
    sm = np.zeros((n_rows, mn), np.int32)
    fe.db_set_geometry(0, k_old, sm, remote=False)
    # query record: direction 1 carries row 3's descriptors; its landmarks are row 3's shifted by (5, -2), 30 of them moved far
    rec = lib.KeyframeRecord()
    rec.drone_id, rec.msg_id, rec.n_dirs = 1, 500, 4
    rec.n_kpts[1] = 150
    np.ctypeslib.as_array(rec.global_desc[1])[:] = g[3]
    np.ctypeslib.as_array(rec.local_desc[1])[:150] = ld[3, :150]
    k_new = k_old[3].copy(); k_new[:150] += np.float32([5.0, -2.0]); k_new[:30] += np.float32(40.0)
    np.ctypeslib.as_array(rec.kpts[1])[:] = k_new
    smn = np.zeros(mn, np.int32); smn[100:120] = -1                              # 20 new landmarks without a 3-D flag
    np.ctypeslib.as_array(rec.stereo_match[1])[:] = smn
    np.ctypeslib.as_array(rec.landmarks_flag[1])[:] = (smn >= 0)                 # landmarks_flag is what the filter tests (:574)
    stream = fh.stream()
    rec_t = upload([rec])
    res_t = torch.zeros(RS, dtype=torch.uint8, device="cuda")
    fe.query(rec_t.data_ptr(), res_t.data_ptr(), stream)
    fe.finish(stream)
    res = fh.results(res_t, 1)[0]
    assert res.accepted == 1 and res.hit_id == 3 and res.dir_new[0] == 1
    n = res.n_matches[0]
    mnw = list(res.match_new[0][:n]); mo = list(res.match_old[0][:n])
    assert mnw == list(range(150)) == mo                                         # identical descriptors: identity match
    qn, qo = gr.loop_pair_filter(mnw, mo, (smn >= 0).astype(np.uint8), k_new, k_old[3], 3.0, seed=0)
    gcount = res.n_geo[0]
    assert res.geo_valid[0] == 1 and gcount == len(qn) == 150 - 30 - 20
    assert list(res.geo_new[0][:gcount]) == qn.tolist() and list(res.geo_old[0][:gcount]) == qo.tolist()
    fe.close()


def test_c3_keyframe_record_vs_oracle(gpu):
    """BASELINE config C3 at full size: one 4-view fisheye keyframe = 8 x 640x480 images through osb_frontend_process,
    the whole record against the oracle composed as LoopCam::generate_stereo_image_descriptor (loop_cam.cpp:341-523):
    keypoints bit-exact on the device heat-map of every image, local descriptors and NetVLAD <= 1e-4 relative, heat-map /
    descriptor map <= 1e-4 relative to the fp32 network, stereo pairs exact given the device descriptors."""
    W, H, MN = 640, 480, 200
    comp, mean = synth.pca_matrices(0)
    w, nvw = synth.superpoint_weights(0), synth.netvlad_weights(0)
    spw = synth.flatten_sp_weights(w)
    fe = make_frontend(width=W, height=H, max_num=MN, self_id=3, db_capacity=64, match_index_dist=5, accept_min_3d_pts=10)
    up = np.stack([synth.image(100 + d, H, W) for d in range(4)])
    down = np.stack([synth.image(200 + d, H, W) for d in range(4)])
    rec, res = fe.process(up, down, msg_id=4242)
    assert (rec.drone_id, rec.msg_id, rec.n_dirs) == (3, 4242, 4)
    imgs = np.concatenate([up, down]).copy()
    imgs[:, H * 3 // 4:, :] = 0                                   # loop_cam.cpp:535-538
    sp = host.SuperPoint(spw, comp, mean, W, H, 0.015, MN, max_batch=8)
    alone = sp.inference_batch(imgs)
    n_same = n_ref = 0
    for b in range(8):
        semi, desc = sp.read("semi", b), sp.read("desc", b)
        k, dsc = alone[b]
        semi_o, desc_o = fr.superpoint_net(imgs[b], w)
        assert np.linalg.norm(semi - semi_o) <= 1e-4 * np.linalg.norm(semi_o) and np.abs(semi - semi_o).max() < 1e-4
        assert np.linalg.norm(desc - desc_o) <= 1e-4 * np.linalg.norm(desc_o)
        rk, _ = fr.get_keypoints(semi, 0.015, MN)                 # oracle NMS2 on the DEVICE heat-map: bit-exact
        assert np.array_equal(k, rk), f"image {b}: keypoints differ from the oracle NMS on the device heat-map"
        rd = fr.compute_descriptors(desc, rk, W, H, comp, mean)
        assert np.linalg.norm(dsc - rd) <= 1e-4 * np.linalg.norm(rd)
        ok, _ = fr.get_keypoints(semi_o, 0.015, MN)               # end to end: margin cases only
        n_same += len({tuple(x) for x in k.tolist()} & {tuple(x) for x in ok.tolist()}); n_ref += len(ok)
    assert n_same >= 0.97 * n_ref, f"only {n_same}/{n_ref} keypoints agree end to end"
    for d in range(4):
        ku, du = alone[d]; kd, dd = alone[4 + d]
        n = rec.n_kpts[d]
        # the front-end's batch of 8 and the stand-alone handle run the same kernels: records are bit-identical
        assert n == len(ku) and rec.n_kpts_down[d] == len(kd)
        assert np.array_equal(np.ctypeslib.as_array(rec.kpts[d])[:n], ku)
        assert np.array_equal(np.ctypeslib.as_array(rec.local_desc[d])[:n], du)
        g = np.ctypeslib.as_array(rec.global_desc[d])
        go = fr.netvlad_net(imgs[d], nvw)
        assert np.linalg.norm(g - go) <= 1e-4 * np.linalg.norm(go) and abs(np.linalg.norm(g) - 1) < 1e-5
        qi, ti, _ = fr.bf_crosscheck(du, dd)                      # loop_cam.cpp:388 on the device descriptors
        m = -np.ones(MN, np.int64); m[qi] = ti
        assert n > 10 and np.array_equal(np.ctypeslib.as_array(rec.stereo_match[d]), m)
    assert fe.db_size(False) == 4 and res.accepted == 0 and res.hit_msg_id == -1
    sp.close(); fe.close()


def test_remote_hit_swaps_matcher_roles(gpu):
    """Multi-drone path on one GPU: two keyframes extracted here are re-labelled as a foreign drone's and ingested (they go
    to the REMOTE database, ids + REMOTE_MAGIN_NUMBER); an own non-keyframe that looks like the first one must hit it, and
    because the hit is remote and the query keyframe ours the reference calls compute_loop(old, new)
    (loop_detector.cpp:113-118): the DATABASE frame is the matcher's query side.  Checked against the oracle matcher with
    the roles exchanged, direction pairing of loop_detector.cpp:455-465 included."""
    import torch
    fe = make_frontend(self_id=1, match_index_dist=5, inner_product_thres=0.3)
    stream = fh.stream()
    recs_t = torch.zeros(2 * RB, dtype=torch.uint8, device="cuda")
    frames = [frame_images(31), frame_images(32)]
    for i, (up, down) in enumerate(frames):
        up = np.ascontiguousarray(up); down = np.ascontiguousarray(down)
        fe.extract(up.ctypes.data, down.ctypes.data, 700 + i, recs_t.data_ptr() + i * RB, stream)
        fe.finish(stream)
    raw = bytearray(recs_t.cpu().numpy().tobytes())
    foreign = []
    for i in range(2):
        r = lib.KeyframeRecord.from_buffer(raw, i * RB)
        r.drone_id = 2                                            # a foreign drone's keyframe
        foreign.append(lib.KeyframeRecord.from_buffer_copy(bytes(raw[i * RB:(i + 1) * RB])))
    recs_t.copy_(torch.frombuffer(raw, dtype=torch.uint8))
    fe.ingest(recs_t.data_ptr(), 2, -1, stream)
    fe.finish(stream)
    n_rows = [sum(1 for d in range(4) if f.n_kpts[d] > 0) for f in foreign]
    assert fe.db_size(True) == sum(n_rows) and fe.db_size(False) == 0
    # own keyframe: frame 0 seen again, shifted by two pixels with a little noise (descriptors close, not identical)
    rng = np.random.default_rng(5)
    up, down = frames[0]
    shift = lambda a: np.clip(np.roll(a, 2, axis=2).astype(np.int16) + rng.integers(-3, 4, a.shape), 0, 255).astype(np.uint8)
    up2, down2 = np.ascontiguousarray(shift(up)), np.ascontiguousarray(shift(down))
    own_t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    res_t = torch.zeros(RS, dtype=torch.uint8, device="cuda")
    fe.extract(up2.ctypes.data, down2.ctypes.data, 900, own_t.data_ptr(), stream)
    fe.query(own_t.data_ptr(), res_t.data_ptr(), stream, init_mode=False, nonkeyframe=True)
    fe.finish(stream)
    own = fh.records(own_t, 1)[0]
    res = fh.results(res_t, 1)[0]
    assert own.drone_id == 1
    # expected hit: best inner product over the remote rows (max_index = 1: every row is old enough), rows in ingest order
    rows = [(f, d) for f in range(2) for d in range(4) if foreign[f].n_kpts[d] > 0]
    q = np.ctypeslib.as_array(own.global_desc[1]).astype(np.float32)
    scores = np.array([np.ctypeslib.as_array(foreign[f].global_desc[d]) @ q for f, d in rows])
    best = int(np.argmax(scores))
    assert scores[best] > 0.3 and np.sort(scores)[-1] - np.sort(scores)[-2] > 1e-4
    f_hit, d_hit = rows[best]
    assert f_hit == 0                                             # it is the frame we re-visited
    assert res.accepted == 1 and res.swapped == 1
    assert res.hit_id == lib.REMOTE_MAGIN_NUMBER + best and res.hit_dir == d_hit
    assert res.hit_msg_id == 700 + f_hit and res.hit_drone_id == 2
    assert abs(res.hit_score - scores[best]) < 1e-4
    # direction pairing with swapped roles: main_new = direction_old (database), main_old = the queried direction (1)
    main_new, main_old = d_hit, 1
    slot = 0
    for _dn in range(main_new, main_new + 4):
        dir_new = _dn % 4
        dir_old = ((main_old - main_new + 4) % 4 + _dn) % 4
        n_db, n_rec = foreign[f_hit].n_kpts[dir_new], own.n_kpts[dir_old]
        if n_db <= 0 or n_rec <= 0:
            continue
        assert (res.dir_new[slot], res.dir_old[slot]) == (dir_new, dir_old)
        qd = np.ctypeslib.as_array(foreign[f_hit].local_desc[dir_new])[:n_db]       # "new" = the DATABASE frame
        td = np.ctypeslib.as_array(own.local_desc[dir_old])[:n_rec]                 # "old" = the current keyframe
        qi, ti, _ = fr.bf_crosscheck(qd, td)
        n = res.n_matches[slot]
        assert n == len(qi) and n > 5
        assert list(res.match_new[slot][:n]) == qi.tolist() and list(res.match_old[slot][:n]) == ti.tolist()
        slot += 1
    assert slot >= 1 and all(res.dir_new[s] == -1 for s in range(slot, 4))
    fe.close()


def test_swarm_exchange_single_rank_and_ingest(gpu):
    """osb_swarm_* with world = 1 (no NCCL needed): exchange and exchange_async + wait deliver the record, and the gathered
    buffer feeds osb_frontend_ingest exactly like the record itself (own drone -> local database)."""
    import torch
    fe = make_frontend(self_id=1, match_index_dist=5)
    sw = host.Swarm(None, 0, 1)
    stream = fh.stream()
    rec_t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    g1 = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    g2 = torch.zeros(RB, dtype=torch.uint8, device="cuda")
    up, down = (np.ascontiguousarray(a) for a in frame_images(41))
    fe.extract(up.ctypes.data, down.ctypes.data, 5, rec_t.data_ptr(), stream)
    sw.exchange(rec_t.data_ptr(), g1.data_ptr(), stream)
    sw.exchange_async(rec_t.data_ptr(), g2.data_ptr(), stream)
    sw.wait(stream)
    fe.ingest(g2.data_ptr(), 1, -1, stream)
    fe.finish(stream)
    assert torch.equal(rec_t, g1) and torch.equal(rec_t, g2)
    rec = fh.records(g2, 1)[0]
    assert rec.msg_id == 5 and fe.db_size(False) == sum(1 for d in range(4) if rec.n_kpts[d] > 0) and fe.db_size(True) == 0
    with pytest.raises(host._l.OsbError):
        host.Swarm(None, 0, 2)                     # world > 1 needs the unique id
    sw.close(); fe.close()


def test_ingest_own_equals_ingest_and_remote_store_wakes_up(gpu):
    """osb_frontend_ingest_own is osb_frontend_ingest of one own record with a promise to the host's bookkeeping: the same
    rows, the same query results -- and the remote store, unscanned while nothing foreign has arrived, takes part in the
    query as soon as a foreign keyframe is ingested afterwards."""
    import torch
    stream = fh.stream()
    frames = [frame_images(40 + s) for s in range(3)]
    results = []
    for own in (False, True):
        fe = make_frontend(match_index_dist=1)
        rec_t = torch.zeros(RB, dtype=torch.uint8, device="cuda")
        res_t = torch.zeros(RS, dtype=torch.uint8, device="cuda")
        out = []
        for i, (up, down) in enumerate(frames + [frames[0]]):
            up = np.ascontiguousarray(up); down = np.ascontiguousarray(down)
            fe.extract(up.ctypes.data, down.ctypes.data, 900 + i, rec_t.data_ptr(), stream)
            if own:
                fe.ingest_own(rec_t.data_ptr(), stream)
            else:
                fe.ingest(rec_t.data_ptr(), 1, -1, stream)
            fe.query(rec_t.data_ptr(), res_t.data_ptr(), stream)
            fe.finish(stream)
            out.append(res_t.cpu().numpy().tobytes())
        assert fe.db_size(False) == 16 and fe.db_size(True) == 0
        if own:
            # a foreign copy of keyframe 1 arrives: an own NON-keyframe that looks like it must now hit the remote store
            up, down = (np.ascontiguousarray(a) for a in frames[1])
            fe.extract(up.ctypes.data, down.ctypes.data, 950, rec_t.data_ptr(), stream)
            fe.finish(stream)
            raw = bytearray(rec_t.cpu().numpy().tobytes())
            lib.KeyframeRecord.from_buffer(raw).drone_id = 7
            f_t = upload([raw])
            fe.ingest(f_t.data_ptr(), 1, -1, stream)
            fe.query(rec_t.data_ptr(), res_t.data_ptr(), stream, nonkeyframe=True)
            fe.finish(stream)
            res = fh.results(res_t, 1)[0]
            assert fe.db_size(True) == 4
            assert res.accepted == 1 and res.hit_id >= lib.REMOTE_MAGIN_NUMBER and res.hit_drone_id == 7
        results.append(out)
        fe.close()
    assert results[0] == results[1]
    last = lib.LoopResult.from_buffer_copy(results[1][-1])
    assert last.accepted == 1 and last.hit_msg_id == 900
