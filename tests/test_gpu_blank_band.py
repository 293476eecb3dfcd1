"""GPU: the blanked band.  A front-end that blanks the bottom quarter itself (zero_bottom_quarter) stores the constant
tiles of SuperPoint's trunk instead of computing them; one fed the same images already blanked, with blanking off,
computes every tile.  Their records and loop results must be byte-identical, and equal to a stand-alone SuperPoint
handle's outputs on the blanked images, in both precisions, with either main camera, in the fisheye (4 directions) and
pinhole (1 direction) configurations, across geometries, with capped grids and after switching precision back and forth."""
import numpy as np
import pytest

from omniswarm_b200 import host, lib, synth
import frontend_harness as fh

pytestmark = pytest.mark.gpu

MN = 200
CONFIG = dict(db_capacity=64, match_index_dist=2)
CONFIGS = {"fisheye": 4, "pinhole": 1}
# (W, H): the harness size, the flagship size, and sizes whose heights are not multiples of 32
GEOMETRIES = [(96, 64), (640, 480), (320, 208), (272, 176)]


def frame(seed, nd, W, H, shift=0):
    up = np.stack([synth.image(seed * 10 + d, H, W) for d in range(nd)])
    if shift:
        rng = np.random.default_rng(seed)
        up = np.clip(np.roll(up, shift, axis=2).astype(np.int16) + rng.integers(-3, 4, up.shape), 0, 255).astype(np.uint8)
    down = np.stack([np.roll(up[d], 3, axis=0) for d in range(nd)])
    return np.ascontiguousarray(up), np.ascontiguousarray(down)


def blanked(a, H):
    a = a.copy()
    a[:, H * 3 // 4:] = 0
    return a


def sp_alone(sp, up, down, H):
    return sp.inference_batch(np.concatenate([blanked(up, H), blanked(down, H)]))


@pytest.mark.parametrize("cfg", sorted(CONFIGS))
@pytest.mark.parametrize("W,H", GEOMETRIES)
def test_band_records_equal_the_computed_path(gpu, cfg, W, H):
    nd = CONFIGS[cfg]
    g = host.SuperPoint.band_geometry(H, W, H * 3 // 4)
    kw = dict(CONFIG, n_dirs=nd, width=W, height=H, max_num=MN)
    band = fh.make_frontend(kw, zero_bottom_quarter=True)
    full = fh.make_frontend(kw, zero_bottom_quarter=False)
    comp, mean = synth.pca_matrices(0)
    sp = host.SuperPoint(synth.flatten_sp_weights(synth.superpoint_weights(0)), comp, mean, W, H, 0.015, MN,
                         max_batch=2 * nd)
    seeds = [(1, 0), (2, 0), (1, 5), (3, 0), (2, 4), (1, 2)]
    steps = [(p, m) for p in ("split_fp16", "fp16", "split_fp16") for m in ("up", "down")]
    for k, ((prec, main), (seed, shift)) in enumerate(zip(steps, seeds)):
        for fe in (band, full):
            fe.set_precision(prec)
            fe.set_main_camera(main)
        sp.set_precision(prec)
        up, down = frame(seed, nd, W, H, shift)
        rb, qb = band.process(up, down, msg_id=k)
        rf, qf = full.process(blanked(up, H), blanked(down, H), msg_id=k)
        assert bytes(rb) == bytes(rf), (cfg, W, H, prec, main)
        assert bytes(qb) == bytes(qf), (cfg, W, H, prec, main)
        if main == "up":
            alone = sp_alone(sp, up, down, H)
            for d in range(nd):
                ku, du = alone[d]
                n = rb.n_kpts[d]
                assert n == len(ku) and rb.n_kpts_down[d] == len(alone[nd + d][0])
                assert np.ctypeslib.as_array(rb.kpts[d])[:n].tobytes() == ku.tobytes()
                assert np.ctypeslib.as_array(rb.local_desc[d])[:n].tobytes() == du.tobytes()
    assert band.db_size(False) == full.db_size(False) == nd * len(steps)
    if (W, H) == (640, 480):
        assert all(g["tiles"][l][0] < g["tiles"][l][1] for l in range(1, 7))     # the band is there to skip
    sp.close(); band.close(); full.close()


def test_band_with_capped_grids(gpu):
    """fewer persistent CTAs than SMs: every CTA strides over more computed items and more of the band's stores"""
    W, H, nd = 640, 480, 4
    kw = dict(CONFIG, n_dirs=nd, width=W, height=H, max_num=MN)
    band = fh.make_frontend(kw, zero_bottom_quarter=True)
    full = fh.make_frontend(kw, zero_bottom_quarter=False)
    L = lib.load()
    try:
        for k, budget in enumerate((37, 1, 0)):
            L.osb_set_sm_budget(budget)
            for prec in ("split_fp16", "fp16"):
                for fe in (band, full):
                    fe.set_precision(prec)
                up, down = frame(7 + k, nd, W, H)
                rb, qb = band.process(up, down, msg_id=2 * k + (prec == "fp16"))
                rf, qf = full.process(blanked(up, H), blanked(down, H), msg_id=2 * k + (prec == "fp16"))
                assert bytes(rb) == bytes(rf) and bytes(qb) == bytes(qf), (budget, prec)
    finally:
        L.osb_set_sm_budget(0)
        band.close(); full.close()
