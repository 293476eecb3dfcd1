"""Forward-error bounds of the fp32 CUDA-core kernels, and the float64 values they bound.

The fp32 convolutions (csrc/conv_ffma.cu), NetVLAD's fused block 0 and its head (csrc/netvlad.cu), the keypoint
descriptors (csrc/postproc.cu) and the database's inner products (csrc/match.cu) are compared element by element with a
float64 reference of the same operation on the same fp32 inputs.  The bounds are the standard ones of
fp32 arithmetic (Higham, Accuracy and Stability of Numerical Algorithms, ch. 3) with u = 2^-24 and
gamma_n = n u / (1 - n u); they hold for ANY summation order and assume only what the build guarantees (no fast math:
expf within 2 ulp, sqrtf and division correctly rounded):

  * a sum of n products plus a bias:  |y - y64| <= gamma_{n+1} (sum |x||w| + |b|);  ReLU / ReLU6 are 1-Lipschitz;
  * an L2 normalisation of n values:  relative error of each element <= gamma_{n/2+4} (squares, sum, sqrt, division);
  * normalising a perturbed vector:   ||U'/||U'|| - U/||U|| || <= 2 ||U' - U|| / ||U||  -- a bound on the norm of the
    error, so the outputs it governs (the VLAD vector per cluster and as a whole, the centring against the float64 mean
    per location) are checked normwise, not element by element.

tests/test_fp32_bounds.py shows on the CPU that fp32 arithmetic stays within them and that defects exceed them;
tests/test_gpu_fp32_stages.py, test_gpu_keypoints_descriptors.py and test_gpu_db_scan.py apply them to the kernels.  Every function takes NHWC numpy arrays and computes in
torch float64 on `device` ("cpu" or "cuda"); results come back as float64 numpy arrays.
"""
import numpy as np
import torch

U = 2.0 ** -24
EPS = 1e-12                              # the normalisations' eps (F.normalize; csrc/netvlad.cu)
TINY = 2.0 ** -140                       # absolute slack for fp32 subnormal results (exp underflow)
NV_K, NV_D, NV_SLICES = 32, 128, 8


def gamma(n):
    n = np.asarray(n, np.float64)
    return n * U / (1.0 - n * U)


def norm_rel(n):
    """relative error bound of one element of an fp32 L2 normalisation of n values"""
    return gamma(n // 2 + 4)


def _t(a, device):
    return torch.as_tensor(np.ascontiguousarray(a), dtype=torch.float64, device=device)


def _np(t):
    return t.detach().cpu().numpy()


def _nchw(x, device):
    return _t(x, device).permute(0, 3, 1, 2)


def act(y, a):
    """0 none, 1 ReLU, 2 ReLU6 (numpy or torch)"""
    if a == 0:
        return y
    y = y.clip(min=0.0)
    return y.clip(max=6.0) if a == 2 else y


def conv(x, w, b, *, ks, stride=1, groups=1, a=0, device="cpu"):
    """float64 act(conv(x) + b) and its error scale sum |x||w| + |b|: x [B,H,W,C], w OIHW -> two [B,Ho,Wo,Cout]"""
    F = torch.nn.functional
    xt, wt, bt = _nchw(x, device), _t(w, device), _t(b, device)
    y = F.conv2d(xt, wt, bt, stride=stride, padding=ks // 2, groups=groups)
    d = F.conv2d(xt.abs(), wt.abs(), bt.abs(), stride=stride, padding=ks // 2, groups=groups)
    return _np(act(y, a).permute(0, 2, 3, 1)), _np(d.permute(0, 2, 3, 1))


def conv_ref(x, w, b, *, a=0, device="cpu"):
    """dense conv (conv_ffma_kernel): (y64, bound) with bound = gamma_{K+1} (sum |x||w| + |b|), K = cin ks^2"""
    cout, cin, ks, _ = w.shape
    y, d = conv(x, w, b, ks=ks, a=a, device=device)
    return y, gamma(cin * ks * ks + 1) * d


def dwconv_ref(x, w, b, *, stride, a=2, device="cpu"):
    """depthwise 3x3 (dwconv3x3_kernel): 9 products + bias"""
    y, d = conv(x, w, b, ks=3, stride=stride, groups=x.shape[-1], a=a, device=device)
    return y, gamma(10) * d


def image_input(imgs):
    """the u8 -> fp32 input of the first layer exactly as the kernels form it: (float)v * (float)(1/255)"""
    return (imgs.astype(np.float32) * np.float32(1.0 / 255.0))[..., None]


def first_ref(imgs, w, b, *, stride, a, device="cpu"):
    """conv_first_kernel on u8 images [B,H,W]: 9 products + bias"""
    y, d = conv(image_input(imgs), w, b, ks=3, stride=stride, a=a, device=device)
    return y, gamma(10) * d


def maxpool_ref(x):
    B, H, W, C = x.shape
    return x[:, : H // 2 * 2, : W // 2 * 2].reshape(B, H // 2, 2, W // 2, 2, C).max(axis=(2, 4))


def block0_ref(x, dw_w, dw_b, pw_w, pw_b, device="cpu"):
    """NetVLAD block 0 (nv_block0_fused_kernel): a = ReLU6(dw(x)) with |a' - a| <= e = gamma_10 d_dw, then
    y = ReLU6(pw(a')): |y' - y64| <= gamma_33 (sum (|a| + e)|w| + |b|) + sum e |w|"""
    F = torch.nn.functional
    a64, ea = dwconv_ref(x, dw_w, dw_b, stride=1, a=2, device=device)
    at, et = _nchw(a64, device), _nchw(ea, device)
    wt, bt = _t(pw_w, device), _t(pw_b, device)
    y = act(F.conv2d(at, wt, bt), 2)
    bound = gamma(33) * F.conv2d(at.abs() + et, wt.abs(), bt.abs()) + F.conv2d(et, wt.abs())
    return _np(y.permute(0, 2, 3, 1)), _np(bound.permute(0, 2, 3, 1))


# ---------------------------------------------------------------------------------------------------------------------
# NetVLAD head; features as [B, P, D] (P = h w locations)
# ---------------------------------------------------------------------------------------------------------------------
def mu_ref(x):
    """per-image channel mean (nv_colmean_kernel): a sum of P values and one division -> gamma_P mean |x|"""
    x = np.asarray(x, np.float64)
    P = x.shape[1]
    return x.mean(axis=1), gamma(P) * np.abs(x).mean(axis=1)


def centre_ref(x, mu):
    """(x - mu) / max(||x - mu||, eps) per location (nv_center_norm_kernel) from the fp32 inputs x [B,P,D], mu [B,D]:
    one rounded subtraction per element, then a D-element normalisation"""
    d = np.asarray(x, np.float64) - np.asarray(mu, np.float64)[:, None, :]
    n = np.linalg.norm(d, axis=-1, keepdims=True)
    y = d / np.maximum(n, EPS)
    return y, (norm_rel(NV_D) + U) * np.abs(y) * (1.0 + U)


def centre_from_x_ref(x):
    """The same from x alone, float64 mean, NORMWISE per location: the mean's error bound dmu (mu_ref) moves a normalised
    location by at most 2 ||dmu|| / ||x - mu64|| -- large when the locations share a large common component (centring
    cancels).  Returns (y64 [B,P,D], bound on ||y - y64|| [B,P])."""
    mu, dmu = mu_ref(x)
    y, by = centre_ref(x, mu)
    d = np.asarray(x, np.float64) - mu[:, None, :]
    cond = 2.0 * np.linalg.norm(dmu, axis=-1)[:, None] / np.maximum(np.linalg.norm(d, axis=-1), EPS)
    return y, np.linalg.norm(by, axis=-1) + cond


def softmax_ref(z):
    """softmax over the last axis (nv_softmax_kernel) of the fp32 logits z: t = z - max rounds (relative u, so exp is off
    by u|t|), expf is within 2 ulp (4u), the 32-term sum adds gamma_31, the division u; plus TINY for subnormal results"""
    z = np.asarray(z, np.float64)
    t = z - z.max(axis=-1, keepdims=True)
    p = np.exp(t)
    p /= p.sum(axis=-1, keepdims=True)
    eta = np.expm1(U * np.abs(t)) * (1 + 4 * U) + 4 * U
    eta_max = eta.max(axis=-1, keepdims=True)
    rel = (1 + eta) * (1 + U) / ((1 - eta_max) * (1 - gamma(NV_K - 1))) - 1
    return p, rel * p + TINY


def vlad_ref(xn, a, cent):
    """VLAD from the fp32 normalised features xn [B,P,D] and assignments a [B,P,K] (nv_vlad_partial / final kernels),
    bounded NORMWISE.  U_k = sum_p a_pk (x_p - c_k), each element a sum of P products (8 slices), minus A_k c_k:
    |dU| <= gamma_{P+10} (sum_p a |x| + A |c|) elementwise.  Intra-normalisation moves v_k = U_k / ||U_k|| by at most
    e_k = r_k + its own rounding, r_k = 2 ||dU_k|| / ||U_k||.  A cluster with r_k >= 1 is ILL-CONDITIONED (its direction
    is not determined): only ||v'_k|| <= 1 is known, so e_k = ||v_k|| + 1 -- unless dU_k = 0 (all its assignments exactly
    0), then v'_k = v_k = 0.  With E = sqrt(sum_k e_k^2) >= ||v' - v|| and g = ||v||, the global normalisation gives
        ||out' - out||     <= 2 E / g                              (+ its rounding)
        ||out'_k - out_k|| <= (e_k + ||v_k|| E / g) / (g - E)      (+ its rounding).
    Returns (out64 [B,K*D], per-cluster bound [B,K], global bound [B], ill [B,K] bool)."""
    x = np.asarray(xn, np.float64)
    a = np.asarray(a, np.float64)
    c = np.asarray(cent, np.float64)
    P = x.shape[1]
    A = a.sum(axis=1)                                                      # [B,K]
    Uk = np.einsum("bpk,bpd->bkd", a, x) - A[..., None] * c[None]
    dU = gamma(P + 10) * (np.einsum("bpk,bpd->bkd", a, np.abs(x)) + A[..., None] * np.abs(c)[None])
    nU = np.linalg.norm(Uk, axis=-1)                                       # [B,K]
    ndU = np.linalg.norm(dU, axis=-1)
    v = Uk / np.maximum(nU, EPS)[..., None]
    nvk = np.linalg.norm(v, axis=-1)
    ill = nU <= 2 * ndU
    r = 2 * ndU / np.maximum(nU, EPS)
    e = np.where(ill, np.where(ndU > 0, nvk + 1.0, 0.0), r + norm_rel(NV_D) * (nvk + r))
    vf = v.reshape(v.shape[0], -1)
    g = np.linalg.norm(vf, axis=-1)                                        # [B]
    out = vf / np.maximum(g, EPS)[:, None]
    E = np.sqrt((e ** 2).sum(axis=-1))
    gs = np.maximum(g, EPS)
    glob = 2 * E / gs
    glob = glob + norm_rel(NV_K * NV_D) * (1.0 + glob)
    with np.errstate(divide="ignore", invalid="ignore"):
        per = np.where(g[:, None] > E[:, None], (e + nvk * (E / gs)[:, None]) / (g - E)[:, None], np.inf)
    per = np.where((E == 0)[:, None] & (g == 0)[:, None], 0.0, per)
    per = per + norm_rel(NV_K * NV_D) * (nvk / gs[:, None] + per)
    return out, per, glob, ill


def vlad_fraction(out, xn, a, cent):
    """The largest fraction of its VLAD bounds (vlad_ref) an fp32 4096-vector out [B,K*D] uses: every well-conditioned
    cluster and the whole vector; inf if out is not finite or an ill-conditioned cluster has norm above 1.
    Returns (fraction, ill)."""
    ref, per, glob, ill = vlad_ref(xn, a, cent)
    out = np.asarray(out, np.float64)
    if not np.isfinite(out).all():
        return float("inf"), ill
    o, r = out.reshape(ill.shape + (NV_D,)), ref.reshape(ill.shape + (NV_D,))
    if (np.linalg.norm(o[ill], axis=-1) > 1 + norm_rel(NV_K * NV_D)).any():
        return float("inf"), ill
    return max(norm_ratio(o[~ill], r[~ill], per[~ill]), norm_ratio(out, ref, glob)), ill


def head_fp32(x, aw, ab, cent):
    """The head in torch float32 on the CPU, as oracle/frontend_ref.py::netvlad_net computes it, per image:
    x [B,P,D] -> dict(mu, xn, logits, assign, out)"""
    t = lambda v: torch.as_tensor(np.ascontiguousarray(v), dtype=torch.float32)
    xt = t(x)
    mu = xt.mean(dim=1)
    d = xt - mu[:, None, :]
    xn = d / torch.clamp(torch.norm(d, dim=-1, keepdim=True), min=EPS)
    z = xn @ t(aw).reshape(NV_K, NV_D).t() + t(ab)
    a = torch.softmax(z, -1)
    Uk = torch.einsum("bpk,bpd->bkd", a, xn) - a.sum(1)[..., None] * t(cent)[None]
    v = Uk / torch.clamp(torch.norm(Uk, dim=-1, keepdim=True), min=EPS)
    v = v.reshape(v.shape[0], -1)
    v = v / torch.clamp(torch.norm(v, dim=-1, keepdim=True), min=EPS)
    return {"mu": mu.numpy(), "xn": xn.numpy(), "logits": z.numpy(), "assign": a.numpy(), "out": v.numpy()}


# ---------------------------------------------------------------------------------------------------------------------
# keypoint descriptors (sp_desc_norm_kernel, sp_desc_pca_kernel) and database inner products (db_scan kernels)
# ---------------------------------------------------------------------------------------------------------------------
def desc_taps(kpts, W, H, *, align_corners=False):
    """grid_sample's bilinear taps of keypoints kpts [N,2] (x, y pixels) on the Wc x Hc cell map, in fp32 with ATen's
    operation order, every step rounded to nearest as csrc/postproc.cu::bilinear_taps does: gx = 2 kx / W - 1,
    ix = ((gx + 1) Wc - 1) / 2.  These are INPUTS of the float64 reference; their rounding is not charged to the kernel.
    Returns (x0 [N], y0 [N], weights [N,4] for the taps (x0,y0), (x0+1,y0), (x0,y0+1), (x0+1,y0+1))."""
    f = np.float32
    one, two = f(1), f(2)
    kx, ky = np.asarray(kpts, f)[:, 0], np.asarray(kpts, f)[:, 1]
    Wc, Hc = W // 8, H // 8
    gx = two * kx / f(W) - one
    gy = two * ky / f(H) - one
    if align_corners:
        ix, iy = (gx + one) / two * f(Wc - 1), (gy + one) / two * f(Hc - 1)
    else:
        ix, iy = ((gx + one) * f(Wc) - one) / two, ((gy + one) * f(Hc) - one) / two
    fx, fy = np.floor(ix), np.floor(iy)
    ex, ey = fx + one, fy + one
    w = np.stack([(ex - ix) * (ey - iy), (ix - fx) * (ey - iy), (ex - ix) * (iy - fy), (ix - fx) * (iy - fy)], 1)
    return fx.astype(np.int64), fy.astype(np.int64), w.astype(f)


def desc_tap_values(desc, x0, y0, *, clamp=False):
    """the four tap values [N,4,256] of desc [256,Hc,Wc]: taps outside the map are 0 (zeros padding), or the nearest
    cell's with clamp=True"""
    C, Hc, Wc = desc.shape
    d = np.asarray(desc, np.float64)
    out = []
    for dx, dy in ((0, 0), (1, 0), (0, 1), (1, 1)):
        x, y = x0 + dx, y0 + dy
        inside = (x >= 0) & (x < Wc) & (y >= 0) & (y < Hc)
        v = d[:, np.clip(y, 0, Hc - 1), np.clip(x, 0, Wc - 1)].T          # [N,256]
        out.append(v if clamp else v * inside[:, None])
    return np.stack(out, 1)


def desc_ref(desc, kpts, W, H, pca_comp, pca_mean, *, taps=None, n_norm=None):
    """float64 descriptors of keypoints kpts [N,2] (computeDescriptors: bilinear sample, per-channel L2 norm over the N
    keypoints, centre by the PCA mean, project) from the fp32 map desc [256,Hc,Wc] and fp32 tap weights (desc_taps), with
    the element-wise bound of an fp32 computation in any summation order:
      sample     v = sum_t w_t d_t                      e_v  = gamma_4 sum_t |w_t||d_t|
      norm^2     q_c = sum_n v^2                        |dq| <= gamma_{N+1} sum (|v| + e_v)^2 + sum (2|v| e_v + e_v^2)
      norm       cn = sqrt(q)                           rel(cn) <= |dq| / (2 q) + u
      centred    z = v / cn - mu                        |dz| <= |v / cn| (rel(cn) + u) + e_v / cn + u |z|   (first order, x(1+2^-20))
      output     y_o = sum_c z_c W_oc                   |dy| <= gamma_257 sum_c (|z| + |dz|) |W_oc| + sum_c |W_oc| |dz_c|
    A channel whose norm is 0 makes every output NaN (0 / 0), as in the reference; its bound is then NaN too.
    `taps` = (x0, y0, weights) overrides desc_taps (defect models); `n_norm` = the number of leading keypoints in the norm.
    Returns (y64 [N,64], bound [N,64])."""
    kpts = np.asarray(kpts, np.float32)
    N = kpts.shape[0]
    x0, y0, w = desc_taps(kpts, W, H) if taps is None else taps
    dv = desc_tap_values(desc, x0, y0)                                      # [N,4,256]
    w64 = np.asarray(w, np.float64)[..., None]
    v = (w64 * dv).sum(1)                                                   # [N,256]
    ev = gamma(4) * (np.abs(w64) * np.abs(dv)).sum(1)
    nn = N if n_norm is None else n_norm
    av = np.abs(v[:nn])
    q = (v[:nn] ** 2).sum(0)
    dq = gamma(nn + 1) * ((av + ev[:nn]) ** 2).sum(0) + (2 * av * ev[:nn] + ev[:nn] ** 2).sum(0)
    with np.errstate(divide="ignore", invalid="ignore"):
        cn = np.sqrt(q)
        rel_cn = dq / (2 * q) + U
        vc = v / cn
        z = vc - np.asarray(pca_mean, np.float64)[None]
        dz = (np.abs(vc) * (rel_cn + U) + ev / cn + U * np.abs(z)) * (1 + 2.0 ** -20)
    Wo = np.asarray(pca_comp, np.float64)                                   # [64,256]
    y = z @ Wo.T
    bound = gamma(257) * ((np.abs(z) + dz) @ np.abs(Wo).T) + dz @ np.abs(Wo).T
    return y, bound


def desc_fp32(desc, kpts, W, H, pca_comp, pca_mean):
    """the descriptor chain in numpy fp32 in the kernels' order of operations (a second fp32 model beside the oracle's
    torch grid_sample): taps summed nw, ne, sw, se; squares summed over keypoints; sum over channels by matmul"""
    f = np.float32
    x0, y0, w = desc_taps(kpts, W, H)
    dv = desc_tap_values(desc, x0, y0).astype(f)
    v = np.zeros((dv.shape[0], dv.shape[2]), f)
    for t in range(4):
        v = v + dv[:, t] * w[:, t:t + 1]
    cn = np.sqrt((v * v).sum(0, dtype=f))
    with np.errstate(divide="ignore", invalid="ignore"):
        z = v / cn - np.asarray(pca_mean, f)[None]
    return z @ np.asarray(pca_comp, f).T


def ip_ref(rows, q):
    """float64 inner products s [nq, n] of fp32 rows [n, dim] and queries [nq, dim], and the bound of an fp32 dot
    product in any order: |s' - s| <= gamma_dim sum_i |q_i x_i|"""
    r, qq = np.asarray(rows, np.float64), np.asarray(q, np.float64)
    return qq @ r.T, gamma(r.shape[1]) * (np.abs(qq) @ np.abs(r).T)


def ratio(y, ref, bound):
    """max |y - ref| / bound; inf if y has a non-finite value, or the error is non-zero where the bound is 0"""
    y = np.asarray(y, np.float64)
    if not np.isfinite(y).all():
        return float("inf")
    err = np.abs(y - ref)
    with np.errstate(divide="ignore", invalid="ignore"):
        r = np.where(err == 0, 0.0, err / bound)
    return float(np.nan_to_num(r, nan=np.inf).max()) if r.size else 0.0


def norm_ratio(y, ref, bound):
    """max over the leading axes of ||y - ref|| (over the last axis) / bound; inf as for ratio()"""
    y = np.asarray(y, np.float64)
    if not np.isfinite(y).all():
        return float("inf")
    return ratio(np.linalg.norm(y - ref, axis=-1), 0.0, bound)


# ---------------------------------------------------------------------------------------------------------------------
# test operands
# ---------------------------------------------------------------------------------------------------------------------
HEAD_SHAPES = [(1, 1), (1, 2), (1, 7), (4, 6), (13, 25), (30, 40)]   # P = 1, 2, 7, 24, 325, 1200: 16x16 ... 640x480 at 1/16
HEAD_REGIMES = ["network", "common", "underflow"]
DEAD = 5                                 # the cluster whose fp32 mass is exactly 0 in the "underflow" regime


def head_weights(seed=0):
    """assign [32,128,1,1], bias [32] and centroids [32,128] of the synthetic NetVLAD"""
    from omniswarm_b200 import synth
    w = synth.netvlad_weights(seed)
    return w["assign.weight"], w["assign.bias"], w["centroids"]


def head_case(regime, B, h, w, seed=0):
    """projected features [B,h,w,128] fp32 and the assign bias for `regime`:
      network    features like the projection's output, every slot with its own, very different mean;
      common     a large component shared by all locations of a slot (|x| ~ 64, spread ~ 0.5): centring cancels;
      underflow  network features, the assign bias lowered by 120 (exp of every logit underflows without the max shift)
                 and by 300 more for cluster DEAD, whose fp32 mass is then exactly 0 everywhere."""
    rng = np.random.default_rng(1000 + seed)
    aw, ab, cent = head_weights()
    ab = ab.astype(np.float32).copy()
    means = rng.standard_normal((B, 1, 1, NV_D)) * (1.0 + 2.0 * np.arange(B))[:, None, None, None]
    if regime == "common":
        x = 64.0 * np.sign(means) + 0.5 * rng.standard_normal((B, h, w, NV_D))
    else:
        x = means + rng.standard_normal((B, h, w, NV_D)) * rng.uniform(0.3, 2.0, (1, 1, 1, NV_D))
    if regime == "underflow":
        ab -= 120.0
        ab[DEAD] -= 300.0
    return x.astype(np.float32), ab, aw, cent


DESC_MAPS = [(12, 8), (50, 26), (80, 60)]   # cell maps of 96x64, 400x208 and 640x480 images
DESC_N = [1, 15, 16, 17, 31, 32, 33, 200, 8192]
DESC_THRES = 0.015


def window_coupled(L, others, W):
    """whether flat address L lies in the 9x9 flat-address NMS window (column wrap included) of each of `others`"""
    d = np.asarray(others, np.int64) - int(L)
    return np.any([np.abs(d - k * W) <= 4 for k in range(-4, 5)], axis=0)


def desc_case(Wc, Hc, N, cells="unit", seed=0):
    """a heat-map [H,W] with exactly N NMS survivors and a descriptor map [256,Hc,Wc] (fp32).  The first survivors are
    the corners and points on every edge, in the order (0,0), (W-1,H-1), the other corners, then edges, all at one
    confidence (ties never suppress each other); the rest are interior points of a 5-pixel lattice with distinct lower
    confidences, away from the edge points' windows.  cells: "unit" (unit-norm cells like the network's), "raw" (cell
    norms spread over three decades) or "dead" (unit cells, channel 7 zero everywhere: a zero channel norm)."""
    W, H = 8 * Wc, 8 * Hc
    rng = np.random.default_rng(seed * 1000 + N)
    xs = [W // 3, W // 2, 2 * W // 3]
    ys = [H // 3, H // 2, 2 * H // 3]
    edge = [(0, 0), (W - 1, H - 1), (W - 1, 0), (0, H - 1)] + [(x, 0) for x in xs] + [(x, H - 1) for x in xs] + \
           [(0, y) for y in ys] + [(W - 1, y) for y in ys[1:]]
    edge = edge[:N]
    semi = np.zeros((H, W), np.float32)
    flat = [y * W + x for x, y in edge]
    for x, y in edge:
        semi[y, x] = 0.9
    n_in = N - len(edge)
    if n_in:
        gx, gy = np.meshgrid(np.arange(5, W - 8, 5), np.arange(5, H - 4, 5))
        lat = (gy * W + gx).reshape(-1)
        far = np.ones(lat.size, bool)
        for L in flat:
            far &= ~window_coupled(L, lat, W)
        lat = lat[far]
        assert lat.size >= n_in, "map too small for N"
        lat = rng.choice(lat, n_in, replace=False)
        conf = 0.02 + 0.85 * (rng.permutation(n_in) + 1) / (n_in + 1)
        semi.reshape(-1)[lat] = conf.astype(np.float32)
    desc = rng.standard_normal((256, Hc, Wc))
    desc /= np.linalg.norm(desc, axis=0, keepdims=True)
    # the cells under the LAST keypoint (lowest confidence; among the tied edge points the last in raster order) point
    # almost along channel 5, so that keypoint carries a visible share of that channel's norm even at N = 8192
    # (and, in "raw", have the largest norm)
    scale = 10.0 ** rng.uniform(-1.5, 1.5, (1, Hc, Wc))
    last = max(flat) if not n_in else int(lat[np.argmin(conf)])
    x0, y0, _ = desc_taps(np.array([[last % W, last // W]]), W, H)
    for dx in (0, 1):
        for dy in (0, 1):
            if 0 <= x0[0] + dx < Wc and 0 <= y0[0] + dy < Hc:
                cell = desc[:, y0[0] + dy, x0[0] + dx] + 30.0 * np.eye(256)[5]
                desc[:, y0[0] + dy, x0[0] + dx] = cell / np.linalg.norm(cell)
                scale[0, y0[0] + dy, x0[0] + dx] = 10.0 ** 1.5
    if cells == "raw":
        desc *= scale
    elif cells == "dead":
        desc[7] = 0.0
    return semi, desc.astype(np.float32)
