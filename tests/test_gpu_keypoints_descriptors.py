"""GPU: keypoint selection (sp_keypoints_kernel) on each of its three sort paths, and the descriptor chain
(sp_desc_norm_kernel, sp_desc_pca_kernel) against float64, through the post-processing hook.

Keypoints are bit-exact against oracle/frontend_ref.py::get_keypoints.  The survivor count S picks the sort path: rank
counting for S <= 128, a bitonic sort in shared memory for S <= 8192, max_num rounds of block-wide minimum above.  Every
case checks the kernel's candidate and survivor counts against the oracle, so each case proves which path it ran.  The
heat-maps are built so that S is known by construction, and the oracle still counts it:
  * isolated peaks on a 5-pixel lattice over a zero background: one survivor each;
  * blocks whose values increase in raster order: every pixel is a candidate, and only the block's last pixel survives
    (all others have a later, stronger neighbour), so the candidate count M can exceed the u16 index plane's 65 536
    with few survivors;
  * a plateau of one confidence: every pixel survives (ties never suppress each other).
Descriptors are checked element by element within oracle/fp32_bounds.py::desc_ref's bound."""
import numpy as np
import pytest

from omniswarm_b200 import synth, host
from oracle import fp32_bounds as fb
from oracle import frontend_ref as fr

pytestmark = pytest.mark.gpu

W, H = 640, 480
THRES = 0.015
MAX_NUMS = (1, 128, 200, 8192)
LATTICE = np.array([y * W + x for y in range(0, H, 5) for x in range(0, W - 4, 5)])   # 12 288 peaks, no column wrap


def path(S):
    return "rank" if S <= 128 else ("bitonic" if S <= 8192 else "global")


def survivor_conf(n, mode, rng):
    if mode == "equal":
        return np.full(n, 0.5, np.float32)
    if mode == "two":
        return rng.choice(np.array([0.3, 0.6], np.float32), n)
    return (0.02 + 0.9 * (rng.permutation(n) + 1) / (n + 1)).astype(np.float32)


def add_peaks(semi, flat, conf):
    semi.reshape(-1)[flat] = conf


def add_blocks(semi, n, bw, bh, top, y0=5):
    """n blocks of bw x bh pixels, 5 pixels apart, values increasing in raster order up to top[i] at the last pixel"""
    per_row = (W - 10 + 5) // (bw + 5)
    ramp = (np.arange(bw * bh, dtype=np.float64) - (bw * bh - 1)) * 2e-6
    for i in range(n):
        x, y = 5 + (i % per_row) * (bw + 5), y0 + (i // per_row) * (bh + 5)
        assert x + bw <= W - 5 and y + bh <= H
        semi[y:y + bh, x:x + bw] = (top[i] + ramp).astype(np.float32).reshape(bh, bw)


def heatmap(kind, S, mode, seed=0):
    rng = np.random.default_rng(seed * 7919 + S)
    semi = np.zeros((H, W), np.float32)
    if kind == "lattice":
        add_peaks(semi, LATTICE[:S], survivor_conf(S, mode, rng))
    elif kind == "plateau":
        semi[:] = 0.5
    elif kind == "wrap_rank":          # 100 blocks of 750: M = 75 000
        add_blocks(semi, 100, 30, 25, survivor_conf(100, mode, rng))
    elif kind == "wrap_bitonic":       # 1000 blocks of 80: M = 80 000
        add_blocks(semi, 1000, 8, 10, survivor_conf(1000, mode, rng))
    elif kind == "wrap_global":        # 9216 peaks in the top 360 rows and one block of 115 x 626: M = 81 206
        n = 72 * 128
        c = survivor_conf(n + 1, mode, rng)
        add_peaks(semi, LATTICE[:n], c[:n])
        add_blocks(semi, 1, 626, 115, c[n:] if mode != "distinct" else [0.95], y0=365)   # its ramp spans 0.146
    elif kind == "threshold":          # every other peak exactly at the threshold: not a candidate
        c = survivor_conf(S, mode, rng)
        c[::2] = np.float32(THRES)
        add_peaks(semi, LATTICE[:S], c)
    return semi


@pytest.fixture(scope="module")
def sps(gpu):
    comp, mean = synth.pca_matrices(0)
    w = synth.flatten_sp_weights(synth.superpoint_weights(0))
    out = {m: host.SuperPoint(w, comp, mean, W, H, THRES, m, max_batch=3) for m in MAX_NUMS}
    yield out
    for sp in out.values():
        sp.close()


DESC = np.random.default_rng(1).standard_normal((256, H // 8, W // 8)).astype(np.float32)


def oracle(semi):
    """(M, S, keypoints of every survivor in output order, their confidences)"""
    xs, ys, conf = fr.get_candidates(semi, THRES)
    k, c = fr.nms2(xs, ys, conf, W, H, max_num=1 << 30)
    return len(xs), len(k), k, c


def check(sp, semi, b, out, ref, max_num, survivors=True):
    M, S, rk, rc = ref
    k, _ = out[b]
    assert np.array_equal(k, rk[:max_num]), f"keypoints differ (M {M}, S {S}, max_num {max_num})"
    assert np.array_equal(sp.read("conf", b)[:len(k)], rc[:max_num])
    assert sp.read("counts", b)[:2].tolist() == [M, S], "candidate / survivor counts differ"
    if survivors and M <= 65536:
        assert np.array_equal(sp.read("survivors", b) > 0, fr.nms_survivor_mask(semi, THRES))


LATTICE_S = [0, 1, 127, 128, 129, 1000, 8191, 8192, 8193, 12288]


@pytest.mark.parametrize("mode", ["distinct", "equal", "two"])
@pytest.mark.parametrize("S", LATTICE_S)
def test_keypoints_lattice(sps, S, mode):
    """S isolated peaks; every max_num, so that n_out < S, = S and > S occur on every path"""
    semi = heatmap("lattice", S, mode)
    ref = oracle(semi)
    assert ref[:2] == (S, S)
    for m, sp in sps.items():
        out = sp.postprocess(semi, DESC)
        check(sp, semi, 0, out, ref, m, survivors=(m == 8192))
    print(f"S {S} {mode}: path {path(S)}")


WRAP_CASES = [(kind, S, mode) for kind, S in (("wrap_rank", 100), ("wrap_bitonic", 1000), ("wrap_global", 9217))
              for mode in ("distinct", "equal", "two")] + [("plateau", H * W, "equal")]


@pytest.mark.parametrize("kind,S,mode", WRAP_CASES)
def test_keypoints_u16_wrap_on_every_path(sps, kind, S, mode):
    """more than 65 536 candidates: survivor coordinates come from the wrapped u16 index plane, on each sort path"""
    semi = heatmap(kind, S, mode)
    ref = oracle(semi)
    assert ref[0] > 65536 and ref[1] == S, ref[:2]
    for m, sp in sps.items():
        check(sp, semi, 0, sp.postprocess(semi, DESC), ref, m)
    print(f"{kind} {mode}: M {ref[0]} S {S} path {path(S)}")


def test_keypoints_batch_mixes_paths(sps):
    """one batch whose images take the rank, bitonic and global paths: each equals the same image run alone"""
    semis = np.stack([heatmap("wrap_rank", 100, "distinct"), heatmap("lattice", 1000, "two"),
                      heatmap("lattice", 8193, "equal")])
    descs = np.stack([DESC, DESC[::-1].copy(), -DESC])
    for m, sp in sps.items():
        out = sp.postprocess(semis, descs)
        counts = [sp.read("counts", b)[:2].tolist() for b in range(3)]
        conf = [sp.read("conf", b) for b in range(3)]
        assert [path(c[1]) for c in counts] == ["rank", "bitonic", "global"]
        for b in range(3):
            (k, d), = sp.postprocess(semis[b], descs[b])
            assert np.array_equal(out[b][0], k) and np.array_equal(out[b][1], d)
            assert sp.read("counts", 0)[:2].tolist() == counts[b]
            assert np.array_equal(sp.read("conf", 0)[:len(k)], conf[b][:len(k)])
    for b in range(3):
        check(sps[8192], semis[b], b, sps[8192].postprocess(semis, descs), oracle(semis[b]), 8192)


@pytest.mark.parametrize("S", [100, 1000, 12288])
def test_keypoints_exactly_at_threshold(sps, S):
    """prob == thres is not a candidate (the threshold is strict)"""
    semi = heatmap("threshold", S, "distinct")
    ref = oracle(semi)
    assert ref[:2] == (S // 2, S // 2)
    for m, sp in sps.items():
        check(sp, semi, 0, sp.postprocess(semi, DESC), ref, m)


# ---------------------------------------------------------------------------------------------------------------------
# descriptors
# ---------------------------------------------------------------------------------------------------------------------
DESC_CASES = [(m, n) for m in fb.DESC_MAPS for n in fb.DESC_N if n <= 200 or m == (80, 60)]


@pytest.fixture(scope="module")
def desc_sps(gpu):
    comp, mean = synth.pca_matrices(0)
    w = synth.flatten_sp_weights(synth.superpoint_weights(0))
    out = {m: host.SuperPoint(w, comp, mean, 8 * m[0], 8 * m[1], fb.DESC_THRES, 8192, max_batch=1) for m in fb.DESC_MAPS}
    yield out
    for sp in out.values():
        sp.close()


@pytest.mark.parametrize("cells", ["unit", "raw"])
@pytest.mark.parametrize("case", DESC_CASES, ids=lambda c: "{}x{}_N{}".format(*c[0], c[1]))
def test_descriptors_within_bound(desc_sps, case, cells):
    """N keypoints: corners, every edge and interior points; N covers the norm kernel's 16 groups of two and the PCA
    kernel's 8 keypoints per CTA on both sides of their multiples.  max_num is 8192, so slots past N are unused."""
    (Wc, Hc), N = case
    comp, mean = synth.pca_matrices(0)
    semi, desc = fb.desc_case(Wc, Hc, N, cells)
    sp = desc_sps[(Wc, Hc)]
    (k, d), = sp.postprocess(semi, desc)
    rk, _ = fr.get_keypoints(semi, fb.DESC_THRES, 8192)
    assert len(rk) == N and np.array_equal(k, rk)
    y64, bound = fb.desc_ref(desc, k, 8 * Wc, 8 * Hc, comp, mean)
    r = fb.ratio(d, y64, bound)
    print(f"{case} {cells}: {r:.3e} of the bound")
    assert r <= 1.0


def test_descriptors_zero_channel_norm(desc_sps):
    """a channel with norm 0 over the keypoints: the outputs are not finite exactly where the oracle's are not"""
    comp, mean = synth.pca_matrices(0)
    semi, desc = fb.desc_case(12, 8, 33, "dead")
    (k, d), = desc_sps[(12, 8)].postprocess(semi, desc)
    rd = fr.compute_descriptors(desc, k, 96, 64, comp, mean)
    assert len(k) == 33 and np.array_equal(np.isfinite(d), np.isfinite(rd)) and not np.isfinite(rd).any()
