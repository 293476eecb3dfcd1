"""CPU: the float64 bounds of the fp32 stage tests (tests/test_gpu_fp32_stages.py) hold for fp32 arithmetic and can fail.

oracle/fp32_bounds.py bounds each fp32 CUDA-core kernel -- the FFMA convolutions, the first layer, depthwise 3x3, NetVLAD's
fused block 0 and the stages of its head -- by fp32 forward-error analysis.  Here each stage is computed in fp32 by torch
on the CPU (in whatever order torch sums) and must stay within its bound, while each defect below must exceed it:
otherwise the GPU tests could pass a wrong kernel.
"""
import numpy as np
import pytest
import torch

from omniswarm_b200 import synth
from oracle import fp32_bounds as fb

F = torch.nn.functional
# (cin, cout, ks, out_cstride): 3x3 and 1x1, K from 128 to 2304, a padded output
LAYERS = [(64, 64, 3, 64), (256, 256, 3, 256), (256, 65, 1, 72), (128, 32, 1, 32), (512, 128, 1, 128)]


def t32(a):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float32)


def conv_fp32(x, w, b, a, skip_chunk=None):
    """fp32 conv as a float32 matrix product over the unfolded input; skip_chunk = c zeroes input channels [c, c + 8)"""
    cout, cin, ks, _ = w.shape
    xt = t32(x).permute(0, 3, 1, 2)
    if skip_chunk is not None:
        xt = xt.clone()
        xt[:, skip_chunk:skip_chunk + 8] = 0
    B, _, H, W = xt.shape
    cols = F.unfold(xt, ks, padding=ks // 2)                              # [B, cin ks ks, H W]
    y = (t32(w).reshape(cout, -1) @ cols).reshape(B, cout, H, W) + t32(b)[None, :, None, None]
    return fb.act(y, a).permute(0, 2, 3, 1).numpy()


def layer_case(cin, cout, ks, seed, B=3, H=7, W=33):
    rng = np.random.default_rng(seed)
    x = np.maximum(rng.standard_normal((B, H, W, cin)), 0).astype(np.float32) * 2
    w = (rng.standard_normal((cout, cin, ks, ks)) * np.sqrt(2.0 / (cin * ks * ks))).astype(np.float32)
    b = (rng.standard_normal(cout) * 0.1).astype(np.float32)
    return x, w, b


@pytest.mark.parametrize("layer", LAYERS, ids=lambda l: "{}to{}_k{}".format(*l[:3]))
def test_conv_bound(layer):
    cin, cout, ks, _ = layer
    x, w, b = layer_case(cin, cout, ks, seed=cin + cout + ks)
    for a in (0, 1, 2):
        y64, bound = fb.conv_ref(x, w, b, a=a)
        good = fb.ratio(conv_fp32(x, w, b, a), y64, bound)
        bad = fb.ratio(conv_fp32(x, w, b, a, skip_chunk=cin - 8), y64, bound)
        print(f"{layer} act {a}: fp32 {good:.2e} of the bound, one K chunk skipped {bad:.1f}x")
        assert good <= 1.0 and bad > 1.0


def test_depthwise_and_first_layer_bounds():
    rng = np.random.default_rng(3)
    x = np.maximum(rng.standard_normal((2, 9, 14, 64)), 0).astype(np.float32) * 3
    w = (rng.standard_normal((64, 1, 3, 3)) * 0.5).astype(np.float32)
    b = (rng.standard_normal(64) * 0.1).astype(np.float32)
    for stride in (1, 2):
        y64, bound = fb.dwconv_ref(x, w, b, stride=stride)
        y = fb.act(F.conv2d(t32(x).permute(0, 3, 1, 2), t32(w), t32(b), stride=stride, padding=1, groups=64), 2)
        assert fb.ratio(y.permute(0, 2, 3, 1).numpy(), y64, bound) <= 1.0
        w0 = w.copy()
        w0[:, :, 0, 0] = 0                                              # one tap missing
        y = fb.act(F.conv2d(t32(x).permute(0, 3, 1, 2), t32(w0), t32(b), stride=stride, padding=1, groups=64), 2)
        assert fb.ratio(y.permute(0, 2, 3, 1).numpy(), y64, bound) > 1.0
    imgs = rng.integers(0, 256, (2, 12, 20), dtype=np.uint8)
    nvw = synth.netvlad_weights(0)
    w1, b1 = nvw["conv0.weight"], nvw["conv0.bias"]
    for stride, a in ((1, 1), (2, 2)):
        y64, bound = fb.first_ref(imgs, w1, b1, stride=stride, a=a)
        for scale, ok in ((1.0 / 255.0, True), (1.0 / 256.0, False)):  # the u8 scale of the reference vs one off
            xin = t32(imgs.astype(np.float32) * np.float32(scale))[:, None]
            y = fb.act(F.conv2d(xin, t32(w1), t32(b1), stride=stride, padding=1), a).permute(0, 2, 3, 1).numpy()
            assert (fb.ratio(y, y64, bound) <= 1.0) == ok


def test_block0_bound():
    nvw = synth.netvlad_weights(0)
    dw_w, dw_b, pw_w, pw_b = nvw["b0.dw.weight"], nvw["b0.dw.bias"], nvw["b0.pw.weight"], nvw["b0.pw.bias"]
    rng = np.random.default_rng(4)
    x = np.clip(rng.standard_normal((2, 9, 35, 32)) * 2 + 1, 0, 6).astype(np.float32)
    y64, bound = fb.block0_ref(x, dw_w, dw_b, pw_w, pw_b)

    def run(xin):
        a = fb.act(F.conv2d(t32(xin).permute(0, 3, 1, 2), t32(dw_w), t32(dw_b), padding=1, groups=32), 2)
        return fb.act(F.conv2d(a, t32(pw_w), t32(pw_b)), 2).permute(0, 2, 3, 1).numpy()

    assert fb.ratio(run(x), y64, bound) <= 1.0
    # the input tile with its halo loaded one column off (x0 + pc instead of x0 + pc - 1) in every 16-wide tile
    shifted = np.zeros_like(x)
    shifted[:, :, :-1] = x[:, :, 1:]
    assert fb.ratio(run(shifted), y64, bound) > 1.0


def flat(a):
    B, h, w, C = a.shape
    return a.reshape(B, h * w, C)


@pytest.mark.parametrize("regime", fb.HEAD_REGIMES)
@pytest.mark.parametrize("shape", fb.HEAD_SHAPES, ids=lambda s: "{}x{}".format(*s))
def test_head_stage_bounds(regime, shape):
    """each head stage of the fp32 model within its bound on its own fp32 input, and the defects outside it"""
    h, w = shape
    P = h * w
    x4, ab, aw, cent = fb.head_case(regime, 3, h, w, seed=P)
    x = flat(x4)
    r = fb.head_fp32(x, aw, ab, cent)
    mu64, bmu = fb.mu_ref(x)
    assert fb.ratio(r["mu"], mu64, bmu) <= 1.0
    if P % 4:                                        # colmean dropping the locations after the last group of four
        assert fb.ratio(x[:, : P // 4 * 4].sum(1) / P, mu64, bmu) > 1.0
    xn64, bxn = fb.centre_ref(x, r["mu"])
    assert fb.ratio(r["xn"], xn64, bxn) <= 1.0
    c64, bc = fb.centre_from_x_ref(x)
    assert fb.norm_ratio(r["xn"], c64, bc) <= 1.0
    if P == 1:
        assert (r["xn"] == 0).all()
    else:                                            # image 0's mean used for every slot
        d = x - r["mu"][:1, None, :]
        wrong = d / np.maximum(np.linalg.norm(d, axis=-1, keepdims=True), fb.EPS)
        assert fb.ratio(wrong, xn64, bxn) > 1.0
    z64, bz = fb.conv_ref(r["xn"].reshape(3, h, w, 128), aw, ab)
    z = r["logits"]
    assert fb.ratio(z, flat(z64), flat(bz)) <= 1.0
    skewed = z.reshape(-1)[np.arange(3 * P)[:, None] * 31 + np.arange(32)].reshape(z.shape)   # row stride 31 for 32
    if P > 1:
        assert fb.ratio(skewed, flat(z64), flat(bz)) > 1.0
    p64, bp = fb.softmax_ref(z)
    assert fb.ratio(r["assign"], p64, bp) <= 1.0
    if regime == "underflow":                        # without the max shift every exp underflows: 0 / 0
        e = np.exp(z.astype(np.float32))
        with np.errstate(invalid="ignore"):
            assert fb.ratio(e / e.sum(-1, keepdims=True), p64, bp) > 1.0
        assert (r["assign"][..., fb.DEAD] == 0).all() and (p64[..., fb.DEAD] > 0).all()
    frac, ill = fb.vlad_fraction(r["out"], r["xn"], r["assign"], cent)
    assert frac <= 1.0
    expect_ill = np.zeros_like(ill)
    if regime == "underflow":
        expect_ill[:, fb.DEAD] = True
        assert (r["out"].reshape(3, 32, 128)[:, fb.DEAD] == 0).all()
    assert np.array_equal(ill, expect_ill)
    # VLAD defects: the last slice dropped, the last location of every slice dropped, one dimension lost in every cluster
    per = -(-P // fb.NV_SLICES)
    slices = [(s * per, min(P, (s + 1) * per)) for s in range(fb.NV_SLICES) if s * per < P]
    mutants = {"last location of each slice": vlad(r["xn"], drop(r["assign"], [p1 - 1 for _, p1 in slices]), cent)}
    if P > 7 * per:
        mutants["last slice"] = vlad(r["xn"], drop(r["assign"], range(7 * per, P)), cent)
    v = r["out"].reshape(3, 32, 128).copy()
    v[..., 17] = 0
    mutants["dimension 17"] = v.reshape(3, -1)
    for name, m in mutants.items():
        f, _ = fb.vlad_fraction(m, r["xn"], r["assign"], cent)
        print(f"P {P} {regime}: faithful {frac:.2e} of the VLAD bound, {name} dropped {f:.3g}x")
        assert f > 1.0, name


def drop(a, locations):
    a = a.copy()
    a[:, list(locations)] = 0
    return a


def vlad(xn, a, cent):
    """VLAD of fp32 features and assignments, as the kernels define it (float64 here: a defect, not rounding, is modelled)"""
    Uk = np.einsum("bpk,bpd->bkd", a, xn) - a.sum(1)[..., None] * cent[None]
    v = (Uk / np.maximum(np.linalg.norm(Uk, axis=-1, keepdims=True), fb.EPS)).reshape(a.shape[0], -1)
    return v / np.maximum(np.linalg.norm(v, axis=-1, keepdims=True), fb.EPS)


def test_head_model_is_the_oracle():
    """head_fp32 is the head of oracle/frontend_ref.py::netvlad_net: the same 4096-vector from the oracle's own features"""
    from oracle import frontend_ref as fr
    nvw = synth.netvlad_weights(0)
    img = synth.image(3, 64, 96)
    ref = fr.netvlad_net(img, nvw)
    # the projected features of the oracle network, rebuilt layer by layer
    x = torch.from_numpy(img.astype(np.float32))[None, None] * np.float32(synth.NV_INPUT_SCALE)
    tw = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in nvw.items()}
    with torch.no_grad():
        x = torch.clamp(F.conv2d(x, tw["conv0.weight"], tw["conv0.bias"], stride=2, padding=1), 0, 6)
        for i, (ci, co, s) in enumerate(synth.NV_BLOCKS):
            x = torch.clamp(F.conv2d(x, tw[f"b{i}.dw.weight"], tw[f"b{i}.dw.bias"], stride=s, padding=1, groups=ci), 0, 6)
            x = torch.clamp(F.conv2d(x, tw[f"b{i}.pw.weight"], tw[f"b{i}.pw.bias"]), 0, 6)
        x = F.conv2d(x, tw["proj.weight"], tw["proj.bias"])
    feats = x[0].permute(1, 2, 0).reshape(1, -1, 128).numpy()
    out = fb.head_fp32(feats, nvw["assign.weight"], nvw["assign.bias"], nvw["centroids"])["out"][0]
    assert np.abs(out - ref).max() < 1e-6


# ---------------------------------------------------------------------------------------------------------------------
# keypoint descriptors and database inner products (tests/test_gpu_keypoints_descriptors.py, tests/test_gpu_db_scan.py)
# ---------------------------------------------------------------------------------------------------------------------
def desc_defects(desc, kpts, W, H, comp, mean, max_num):
    """float64 models of wrong descriptor kernels; each must leave the bound of fb.desc_ref at these shapes"""
    N = len(kpts)
    x0, y0, w = fb.desc_taps(kpts, W, H)
    out = {}

    def chain(v, n_norm=N, extra=None, centre=True, channels=256):
        q = (v[:n_norm] ** 2).sum(0) + (0.0 if extra is None else extra)
        with np.errstate(divide="ignore", invalid="ignore"):
            z = v / np.sqrt(q) - (mean.astype(np.float64) if centre else 0.0)
        return z[:, :channels] @ comp.astype(np.float64)[:, :channels].T

    def sample(taps, clamp=False):
        return (np.asarray(taps[2], np.float64)[..., None] * fb.desc_tap_values(desc, taps[0], taps[1], clamp=clamp)).sum(1)

    v = sample((x0, y0, w))
    out["out-of-range taps clamped"] = chain(sample((x0, y0, w), clamp=True))
    out["last keypoint dropped from the norm"] = chain(v, n_norm=N - 1)
    if max_num > N:   # the unused slots of a zero-filled keypoint buffer sample at (0, 0)
        out["norm over max_num slots"] = chain(v, extra=(max_num - N) * sample(fb.desc_taps(np.zeros((1, 2)), W, H))[0] ** 2)
    out["last 8 PCA channels skipped"] = chain(v, channels=248)
    out["mean not subtracted"] = chain(v, centre=False)
    if W != H:
        out["x and y swapped"] = chain(sample(fb.desc_taps(np.asarray(kpts)[:, ::-1], H, W)))
    out["align_corners=True"] = chain(sample(fb.desc_taps(kpts, W, H, align_corners=True)))
    return out


DESC_CPU_CASES = [(m, n) for m in fb.DESC_MAPS for n in fb.DESC_N if n <= 200 or m == (80, 60)]


@pytest.mark.parametrize("cells", ["unit", "raw"])
@pytest.mark.parametrize("case", DESC_CPU_CASES, ids=lambda c: "{}x{}_N{}".format(*c[0], c[1]))
def test_descriptor_bound(case, cells):
    """the oracle's torch chain (grid_sample) and a numpy fp32 chain stay within fb.desc_ref's bound, element by element;
    the fp32 tap weights reproduce grid_sample; every defect leaves the bound"""
    from oracle import frontend_ref as fr
    (Wc, Hc), N = case
    W, H = 8 * Wc, 8 * Hc
    comp, mean = synth.pca_matrices(0)
    semi, desc = fb.desc_case(Wc, Hc, N, cells)
    kpts, _ = fr.get_keypoints(semi, fb.DESC_THRES, 8192)
    assert len(kpts) == N and tuple(kpts[0]) == (0, 0)
    y64, bound = fb.desc_ref(desc, kpts, W, H, comp, mean)
    assert np.isfinite(y64).all()
    for name, y in (("torch", fr.compute_descriptors(desc, kpts, W, H, comp, mean)),
                    ("numpy", fb.desc_fp32(desc, kpts, W, H, comp, mean))):
        r = fb.ratio(y, y64, bound)
        print(f"{case} {cells}: {name} fp32 {r:.2e} of the bound")
        assert r <= 1.0, name
    # fb.desc_taps is grid_sample's sampling: its samples agree with grid_sample's up to the sum's rounding and a few
    # ulp of the tap coordinates (ATen's vectorised CPU path rounds the unnormalisation differently); align_corners=True
    # does not
    g = torch.zeros((1, 1, N, 2))
    fk = torch.from_numpy(kpts)
    g[0, 0, :, 0] = 2.0 * fk[:, 0] / W - 1
    g[0, 0, :, 1] = 2.0 * fk[:, 1] / H - 1
    gs = F.grid_sample(t32(desc)[None], g, mode="bilinear", padding_mode="zeros", align_corners=False)[0, :, 0].T.numpy()
    for ac in (False, True):
        x0, y0, w = fb.desc_taps(kpts, W, H, align_corners=ac)
        dv = fb.desc_tap_values(desc, x0, y0)
        v64 = (w.astype(np.float64)[..., None] * dv).sum(1)
        tol = fb.gamma(4) * (np.abs(w.astype(np.float64))[..., None] * np.abs(dv)).sum(1) + \
            8 * fb.U * max(Wc, Hc) * np.abs(desc).max(axis=(1, 2))
        assert (fb.ratio(gs, v64, tol) <= 1.0) != ac
    for name, y in desc_defects(desc, kpts, W, H, comp, mean, 8192).items():
        r = fb.ratio(y, y64, bound)
        print(f"{case} {cells}: {name} {r:.3g}x")
        # one keypoint's channel norm is |v|, so v / cn = sign(v): a defect that only rescales its sample cannot show
        if N > 1 or name not in SCALE_ONLY:
            assert r > 1.0, name


SCALE_ONLY = {"out-of-range taps clamped", "x and y swapped", "align_corners=True"}


def test_descriptor_zero_channel_is_nan():
    """a channel whose norm over the keypoints is 0 makes every output NaN, in the oracle and in the reference model"""
    from oracle import frontend_ref as fr
    comp, mean = synth.pca_matrices(0)
    semi, desc = fb.desc_case(12, 8, 33, "dead")
    kpts, _ = fr.get_keypoints(semi, fb.DESC_THRES, 8192)
    y64, _ = fb.desc_ref(desc, kpts, 96, 64, comp, mean)
    assert np.isnan(y64).all() and np.isnan(fr.compute_descriptors(desc, kpts, 96, 64, comp, mean)).all()


@pytest.mark.parametrize("dim", [4, 256, 4096, 8192])
def test_inner_product_bound(dim):
    """fp32 dot products (torch and numpy, any order) within fb.ip_ref's bound; one term dropped or a row off by one ulp
    in its largest element leaves it"""
    rng = np.random.default_rng(dim)
    rows = rng.standard_normal((300, dim)).astype(np.float32)
    rows[100:200] = rows[0] + (1e-7 * rng.standard_normal((100, dim))).astype(np.float32)   # near ties
    q = rng.standard_normal((5, dim)).astype(np.float32)
    s64, bound = fb.ip_ref(rows, q)
    assert fb.ratio((t32(q) @ t32(rows).T).numpy(), s64, bound) <= 1.0
    assert fb.ratio(q @ rows.T, s64, bound) <= 1.0
    assert fb.ratio(np.cumsum(q[:, None, :] * rows[None], axis=-1, dtype=np.float32)[..., -1], s64, bound) <= 1.0
    dropped = q[:, :-1].astype(np.float64) @ rows[:, :-1].astype(np.float64).T
    assert fb.ratio(dropped, s64, bound) > 1.0
