"""The front-end's sparse descriptor head (convDa, convDb and the L2 norm at the cells the keypoints sample) against the
dense head (OSB_SP_SPARSE_HEAD=0): records and loop results byte-identical, for stereo frames with and without the
blanked bottom quarter, depth frames, both precisions, a geometry whose cell grid is not a multiple of the 8 x 16 tile,
no keypoints and a full max_num."""
import os

import numpy as np
import pytest
import torch

import frontend_harness as fh
from omniswarm_b200 import synth

pytestmark = pytest.mark.gpu


def _frontend(dense, **kw):
    old = os.environ.get("OSB_SP_SPARSE_HEAD")
    if dense:
        os.environ["OSB_SP_SPARSE_HEAD"] = "0"
    try:
        return fh.make_frontend(**kw)
    finally:
        if old is None:
            os.environ.pop("OSB_SP_SPARSE_HEAD", None)
        else:
            os.environ["OSB_SP_SPARSE_HEAD"] = old


def _run(fe, frames, depth, precision):
    """extract, ingest and query every frame -> (record bytes, result bytes) per frame"""
    fe.set_precision(precision)
    if depth:
        fe.set_depth_camera(fh.SC["K"], np.tile(fh.SC["ext"][:1], (fe.cfg.n_dirs, 1)))
    st = fh.stream()
    out = []
    for i, (a, b) in enumerate(frames):
        rec = fh.filled(fh.RB)
        if depth:
            fe.extract_depth(a, b, i, rec.data_ptr(), st)
        else:
            fe.extract(a.ctypes.data, b.ctypes.data, i, rec.data_ptr(), st)
        fe.ingest_own(rec.data_ptr(), st)
        res = fh.filled(fh.RS)
        fe.query(rec.data_ptr(), res.data_ptr(), st)
        fe.finish(st)
        torch.cuda.synchronize()
        out.append((rec.cpu().numpy().tobytes(), res.cpu().numpy().tobytes(), fh.records(rec, 1)[0]))
    return out


CASES = {
    "fisheye_small": dict(width=96, height=64, zero_bottom_quarter=True),
    "pinhole_small": dict(width=96, height=64, zero_bottom_quarter=False),
    "fisheye_640x480": dict(width=640, height=480, zero_bottom_quarter=True, n_dirs=2),
    "full_max_num": dict(width=96, height=64, zero_bottom_quarter=False, max_num=20),
    "no_keypoints": dict(width=96, height=64, zero_bottom_quarter=False, sp_thres=2.0),
    "depth_small": dict(width=96, height=64, zero_bottom_quarter=False),
}


@pytest.mark.parametrize("precision", ["split_fp16", "fp16"])
@pytest.mark.parametrize("case", sorted(CASES))
def test_sparse_head_matches_dense(case, precision):
    kw = dict(CASES[case])
    W, H, nd = kw["width"], kw["height"], kw.get("n_dirs", 4)
    depth = case.startswith("depth")
    frames = []
    for s in range(3):
        if depth:
            frames.append((np.stack([synth.image(s * 10 + d, H, W) for d in range(nd)]),
                           np.stack([synth.depth_image(s * 10 + d, H, W) for d in range(nd)])))
        else:
            frames.append((np.stack([synth.image(s * 10 + d, H, W) for d in range(nd)]),
                           np.stack([synth.image(s * 10 + d + 5, H, W) for d in range(nd)])))
    kw.setdefault("db_capacity", 64)
    sparse = _run(_frontend(False, **kw), frames, depth, precision)
    dense = _run(_frontend(True, **kw), frames, depth, precision)
    n = [list(r[2].n_kpts)[:nd] for r in sparse]
    if case == "no_keypoints":
        assert all(k == 0 for f in n for k in f)
    else:
        assert all(k > 0 for f in n for k in f)
    if case == "full_max_num":
        assert all(k == 20 for f in n for k in f)
    if case == "fisheye_640x480":
        # some keypoint sits within half a cell of the border, so one of its taps lies outside the cell grid
        kp = np.concatenate([np.ctypeslib.as_array(r[2].kpts[d])[:k] for r, f in zip(sparse, n) for d, k in enumerate(f)])
        assert ((kp < 4.0) | (kp[:, :1] > W - 4.0) | (kp[:, 1:] > H - 4.0)).any()
    for (rs, qs, _), (rd, qd, _) in zip(sparse, dense):
        assert rs == rd
        assert qs == qd
