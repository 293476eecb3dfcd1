"""What the keyframe front-end's GPU tests share: synthetic frames, a front-end of the synthetic networks, device records
and results, the loop scene's front-end and own-keyframe query, and oracle/loop_ref.compute_loop fed a device query result.
Test modules import it as `frontend_harness`."""
import numpy as np
import torch

from omniswarm_b200 import host, lib, synth
from oracle import loop_ref

W0, H0 = 96, 64
RB, RS, EB = lib.RECORD_BYTES, lib.RESULT_BYTES, lib.EDGE_BYTES
FILL = 0x5A                              # result buffers start with this byte: unwritten fields compare equal too
# the settings every test front-end starts from; host.KeyframeFrontend's defaults apply to the rest
FRONTEND = dict(width=W0, height=H0, n_dirs=4, max_num=200, sp_thres=0.015, self_id=1, inner_product_thres=0.3,
                accept_min_3d_pts=3)


def make_frontend(config=None, **overrides):
    """a front-end of synth.frontend_weights(): FRONTEND, then a test module's `config`, then `overrides`"""
    return host.KeyframeFrontend(*synth.frontend_weights(), **{**FRONTEND, **(config or {}), **overrides})


def frame_images(seed, nd=4):
    up = np.stack([synth.image(seed * 10 + d, H0, W0) for d in range(nd)])
    down = np.stack([synth.image(seed * 10 + d + 5, H0, W0) for d in range(nd)])
    return up, down


def depth_frame(seed, nd=4, W=W0, H=H0):
    return (np.stack([synth.image(seed * 10 + d, H, W) for d in range(nd)]),
            np.stack([synth.depth_image(seed * 10 + d, H, W) for d in range(nd)]))


# ---- device records and results --------------------------------------------------------------------------------------
def stream():
    return torch.cuda.current_stream().cuda_stream


def upload(recs):
    """host records (ctypes structures or bytes), back to back in one device byte tensor"""
    return torch.frombuffer(bytearray(b"".join(bytes(r) for r in recs)), dtype=torch.uint8).cuda()


def filled(nbytes):
    """a device byte buffer holding FILL"""
    return torch.full((nbytes,), FILL, dtype=torch.uint8, device="cuda")


def _split(t, n, size):
    raw = t.cpu().numpy().tobytes()
    return [raw[i * size:(i + 1) * size] for i in range(n)]


def results(t, n):
    return [lib.LoopResult.from_buffer_copy(b) for b in _split(t, n, RS)]


def records(t, n):
    return [lib.KeyframeRecord.from_buffer_copy(b) for b in _split(t, n, RB)]


def edges(t, n):
    """the raw bytes of n loop edges"""
    return _split(t, n, EB)


# ---- the loop scene (synth.LOOP_SCENE) seen by a stereo front-end with loop parameters ------------------------------
SC = synth.LOOP_SCENE
LOOP_COV = np.eye(6) * 0.01
LOOP_PARAMS = dict(odometry_consistency_threshold=10.0, seed=3)
LOOP_CONFIG = dict(db_capacity=64, init_mode_product_thres=0.2, match_index_dist=5, geometric_filter=True, ransac_seed=0)


def loop_frontend(cameras="stereo", loop_params=True, **kw):
    """make_frontend(LOOP_CONFIG, **kw) with the scene's cameras ("stereo", "depth", "both" or None) and LOOP_PARAMS"""
    fe = make_frontend(LOOP_CONFIG, **kw)
    if cameras in ("stereo", "both"):
        fe.set_cameras(SC["K"], SC["ext"], SC["ext"], 0.006)
    if cameras in ("depth", "both"):
        fe.set_depth_camera(SC["K"], SC["ext"])
    if loop_params:
        fe.set_loop_params(**LOOP_PARAMS)
    return fe


def own_query(fe, st, old_rec, new_rec, nonkeyframe=False, ingest_old=True):
    """ingest the old record, then the new one (own, as on_image_recv does), query the new one -> (rec_t, res_t, result)"""
    if ingest_old:
        ot = upload([old_rec])
        fe.ingest_own(ot.data_ptr(), st)
    rt = upload([new_rec])
    fe.ingest_own(rt.data_ptr(), st)
    res_t = filled(RS)
    fe.query(rt.data_ptr(), res_t.data_ptr(), st, nonkeyframe=nonkeyframe)
    fe.finish(st)
    return rt, res_t, results(res_t, 1)[0]


def cand_own(init_mode=False, odom=None):
    """the candidate of an own query of the new keyframe hitting the old one"""
    return dict(pose_query=SC["pose_new"], pose_hit=SC["pose_old"], init_mode=init_mode,
                odom_rel=SC["delta_true"] if odom is None else odom, cov=LOOP_COV)


# ---- the loop-edge oracle --------------------------------------------------------------------------------------------
def loop_frame(rec):
    """what the oracle reads of a record (or of the store row made from it)"""
    n = list(rec.n_kpts)
    a = np.ctypeslib.as_array
    return dict(drone_id=rec.drone_id, msg_id=rec.msg_id, n_kpts=n,
                kpts=[a(rec.kpts[d])[:n[d]].copy() for d in range(len(n))],
                flags=[a(rec.landmarks_flag[d])[:n[d]].copy() for d in range(len(n))],
                l3d=[a(rec.landmarks_3d[d])[:n[d]].copy() for d in range(len(n))])


def loop_hit(res):
    slots = [dict(dir_new=res.dir_new[j], dir_old=res.dir_old[j], geo_valid=res.geo_valid[j],
                  geo_new=list(res.geo_new[j][:res.n_geo[j]]), geo_old=list(res.geo_old[j][:res.n_geo[j]]),
                  match_new=list(res.match_new[j][:res.n_matches[j]]), match_old=list(res.match_old[j][:res.n_matches[j]]))
             for j in range(len(res.dir_new)) if res.dir_new[j] >= 0]
    return dict(accepted=res.accepted, has_frame=res.hit_msg_id != -1, slots=slots)


def loop_oracle(res, query_rec, hit_rec, cand, K, ext, params, query_dir=1):
    """compute_loop of a device query result with the device's roles (loop_detector.cpp:113-118): a swapped hit makes the
    hit keyframe the new side.  cand: pose_query, pose_hit and optionally init_mode, odom_rel, cov"""
    sw = bool(res.swapped)
    new, old = (hit_rec, query_rec) if sw else (query_rec, hit_rec)      # old is None: a db_load row without a keyframe
    main_new, main_old = (res.hit_dir, query_dir) if sw else (query_dir, res.hit_dir)
    c = dict(init_mode=cand.get("init_mode", False), odom_rel=cand.get("odom_rel", [0, 0, 0, 1, 0, 0, 0]),
             cov=cand.get("cov", np.eye(6)),
             pose_now=cand["pose_hit"] if sw else cand["pose_query"], pose_old=cand["pose_query"] if sw else cand["pose_hit"])
    return loop_ref.compute_loop(loop_hit(res), loop_frame(new), None if old is None else loop_frame(old), K, ext,
                                 main_new, main_old, c, params)
