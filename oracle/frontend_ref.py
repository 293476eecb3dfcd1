"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of the swarm_loop front-end.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import
this module.  The product path (omniswarm_b200 + csrc/libomniswarm_b200.so) never does.

Each function cites the reference lines (relative to /root/reference) it restates.  The reference
cannot be compiled or imported here (no ROS/TensorRT/OpenCV-C++/faiss/libtorch-C++; SURVEY.md
section 8c) and ships no golden vectors, so the pins are:
  * torch.nn.functional.grid_sample  == torch::grid_sampler  (same ATen kernel)       -> PINNED
  * cv2.BFMatcher(NORM_L2, True)     == cv::BFMatcher        (same OpenCV algorithm)  -> PINNED
  * SuperPoint network: torch module of superpoint.ipynb:135-205, seeded weights      -> pinned against the reference's own
    SuperPointNet class executed in place (tests/golden/make_ref_superpoint.py, ref_superpoint.npz): 2e-7; the trained
    weights and the fp16 TensorRT engine's rounding remain unpinned
    (no reference outputs exist; the engine ran fp16 TensorRT)
  * NMS2 / getKeyPoints: literal restatement incl. flat-address wrap, u16 index plane  -> parity unpinned
    (out-of-buffer neighbour = skip; sort ties = stable raster order; both are *defined* here)
  * NetVLAD: stand-in architecture (hfnet MobileNetVLAD is not in the reference)       -> parity unpinned
  * faiss::IndexFlatIP: exact inner product, descending, ties by ascending id, -1 pad -> parity unpinned
tests/test_oracle_pins.py checks the pinned items and the committed fixtures in tests/golden/.
"""
from __future__ import annotations

import numpy as np

try:  # torch is used for the CNNs and grid_sample only
    import torch
    import torch.nn.functional as F
except Exception:  # pragma: no cover
    torch = None

REMOTE_MAGIN_NUMBER = 1000000      # loop_detector.h:22
SEARCH_NEAREST_NUM = 5             # loop_defines.h:32


# ------------------------------------------------------------------------------------------------
# SuperPoint network: superpoint.ipynb:135-205 (module), :345-352 (export; input already /255)
# ------------------------------------------------------------------------------------------------
def superpoint_net(img_u8: np.ndarray, w: dict, num_threads: int | None = None, trace: dict | None = None):
    """img_u8 [H,W] uint8 -> (semi [H,W] f32, desc [256,H/8,W/8] f32).

    Pre-processing u8 -> f32 * (1/255): superpoint_tensorrt.cpp:127.
    `trace`, if given, receives {layer: (max |input|, max |weight|)} of every convolution.
    """
    if num_threads is not None:
        torch.set_num_threads(num_threads)
    t = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in w.items()}
    # cv::Mat::convertTo(CV_32F, 1/255.0): OpenCV's cvtScale for 8U->32F computes (float)v * (float)alpha
    x = torch.from_numpy(img_u8.astype(np.float32) * np.float32(1.0 / 255.0))[None, None]
    relu = F.relu

    def conv(x, n, pad):
        if trace is not None:
            trace[n] = (float(x.abs().max()), float(t[n + ".weight"].abs().max()))
        return F.conv2d(x, t[n + ".weight"], t[n + ".bias"], padding=pad)

    with torch.no_grad():
        x = relu(conv(x, "conv1a", 1)); x = relu(conv(x, "conv1b", 1)); x = F.max_pool2d(x, 2, 2)
        x = relu(conv(x, "conv2a", 1)); x = relu(conv(x, "conv2b", 1)); x = F.max_pool2d(x, 2, 2)
        x = relu(conv(x, "conv3a", 1)); x = relu(conv(x, "conv3b", 1)); x = F.max_pool2d(x, 2, 2)
        x = relu(conv(x, "conv4a", 1)); x = relu(conv(x, "conv4b", 1))
        cPa = relu(conv(x, "convPa", 1)); semi = conv(cPa, "convPb", 0)
        cDa = relu(conv(x, "convDa", 1)); desc = conv(cDa, "convDb", 0)
        dn = torch.norm(desc, p=2, dim=1)                       # superpoint.ipynb:187
        desc = desc.div(torch.unsqueeze(dn, 1))                 # :188
        semi = torch.softmax(semi, 1)                           # :190
        semi = semi.narrow(1, 0, 64).permute((0, 2, 3, 1))      # :191-192 drop dustbin
        Hc, Wc = semi.size(1), semi.size(2)
        semi = semi.contiguous().view((-1, Hc, Wc, 8, 8)).permute((0, 1, 3, 2, 4))
        semi = semi.contiguous().view((-1, Hc * 8, Wc * 8))     # :194-198 pixel shuffle
    return semi[0].numpy().copy(), desc[0].numpy().copy()


# ------------------------------------------------------------------------------------------------
# getKeyPoints + NMS2: superpoint_tensorrt.cpp:164-189, 237-310   (SURVEY.md Appendix A.2)
# ------------------------------------------------------------------------------------------------
def get_candidates(prob: np.ndarray, thres: float):
    """mask = prob > thres (strict, f32), cv::findNonZero order = row-major. (:167-173)"""
    ys, xs = np.nonzero(prob > np.float32(thres))
    conf = prob[ys, xs].astype(np.float32)
    return xs.astype(np.int32), ys.astype(np.int32), conf


def nms2(xs, ys, conf, W: int, H: int, max_num: int, dist_thresh: int = 4, border: int = 0):
    """Literal NMS2 (:237-310).  Returns (kpts [n,2] f32 (x,y) ordered by descending conf, conf [n]).

    Defined behaviours where the reference is undefined / unspecified:
      * neighbour flat address outside [0,H*W)  -> skipped (Mat::at is unchecked in release; columns
        wrap into the adjacent row of the continuous buffer exactly as the flat address does);
      * std::sort is not stable -> the oracle uses a stable sort, ties keep raster order.
    """
    M = len(xs)
    grid = np.zeros(H * W, np.uint8)
    inds = np.zeros(H * W, np.uint16)
    confp = np.zeros(H * W, np.float32)
    flat = ys.astype(np.int64) * W + xs.astype(np.int64)
    grid[flat] = 1
    inds[flat] = (np.arange(M) & 0xFFFF).astype(np.uint16)     # :260 u16 plane wraps above 65535
    confp[flat] = conf
    offs = np.array([k * W + j for k in range(-dist_thresh, dist_thresh + 1)
                     for j in range(-dist_thresh, dist_thresh + 1) if not (j == 0 and k == 0)], np.int64)
    HW = H * W
    for i in range(M):                                         # :265-283
        L = int(flat[i])
        if grid[L] != 1:
            continue
        nb = L + offs
        nb = nb[(nb >= 0) & (nb < HW)]
        lower = nb[confp[nb] < confp[L]]                       # strict <
        grid[lower] = 0                                        # may overwrite a 2
        grid[L] = 2
    sel = np.nonzero(grid == 2)[0]                             # :287-302 raster order, border = 0
    if border > 0:
        v, u = sel // W, sel % W
        keep = (u < W - border) & (u >= border) & (v < H - border) & (v >= border)
        sel = sel[keep]
    sidx = inds[sel].astype(np.int64)
    pts = np.stack([xs[sidx], ys[sidx]], 1).astype(np.float32) if len(sel) else np.zeros((0, 2), np.float32)
    c = confp[sel]
    order = np.argsort(-c.astype(np.float64), kind="stable")   # :304 (descending; ties: raster order)
    order = order[:max_num]                                    # :305-308
    return pts[order], c[order]


def get_keypoints(prob: np.ndarray, thres: float, max_num: int):
    H, W = prob.shape
    xs, ys, conf = get_candidates(prob, thres)
    return nms2(xs, ys, conf, W, H, max_num)


def nms_survivor_mask(prob: np.ndarray, thres: float) -> np.ndarray:
    """grid==2 plane (bool [H,W]) -- used for bit-exact comparison of the NMS stage alone."""
    H, W = prob.shape
    xs, ys, conf = get_candidates(prob, thres)
    pts, _ = nms2(xs, ys, conf, W, H, max_num=1 << 30)
    m = np.zeros((H, W), bool)
    if len(xs) <= 65536 and len(pts):
        m[pts[:, 1].astype(int), pts[:, 0].astype(int)] = True
    return m


# ------------------------------------------------------------------------------------------------
# computeDescriptors: superpoint_tensorrt.cpp:192-230   (SURVEY.md Appendix A.3)
# ------------------------------------------------------------------------------------------------
def compute_descriptors(desc: np.ndarray, kpts: np.ndarray, W: int, H: int,
                        pca_comp: np.ndarray, pca_mean: np.ndarray) -> np.ndarray:
    """desc [256,Hc,Wc], kpts [N,2] (x,y) -> [N,64] f32."""
    N = kpts.shape[0]
    if N == 0:
        return np.zeros((0, pca_comp.shape[0]), np.float32)
    fk = torch.from_numpy(kpts.astype(np.float32))
    grid = torch.zeros((1, 1, N, 2))
    grid[0, 0, :, 0] = 2.0 * fk[:, 0] / W - 1                  # :204 x
    grid[0, 0, :, 1] = 2.0 * fk[:, 1] / H - 1                  # :205 y
    d = torch.from_numpy(np.ascontiguousarray(desc))[None]
    s = F.grid_sample(d, grid, mode="bilinear", padding_mode="zeros", align_corners=False)  # :209
    s = s.squeeze(0).squeeze(1)                                # [256,N]
    dn = torch.norm(s, 2, 1)                                   # :214 per-CHANNEL norm over keypoints
    s = s.div(torch.unsqueeze(dn, 1))                          # :215
    s = s.transpose(0, 1).contiguous().numpy()                 # [N,256]
    out = (s - pca_mean[None, :].astype(np.float32)) @ pca_comp.T.astype(np.float32)   # :221
    return np.ascontiguousarray(out.astype(np.float32))


def superpoint_inference(img_u8, w, thres, max_num, pca_comp, pca_mean):
    """SuperPointTensorRT::inference (superpoint_tensorrt.cpp:117-162)."""
    semi, desc = superpoint_net(img_u8, w)
    H, W = semi.shape
    kpts, conf = get_keypoints(semi, thres, max_num)
    d = compute_descriptors(desc, kpts, W, H, pca_comp, pca_mean)
    return kpts, d, semi, desc


# ------------------------------------------------------------------------------------------------
# NetVLAD stand-in (I/O contract mobilenetvlad_tensorrt.cpp:4-15; architecture is OURS, pinned in
# omniswarm_b200/synth.py::NV_BLOCKS and DESIGN.md)
# ------------------------------------------------------------------------------------------------
def netvlad_net(img_u8: np.ndarray, w: dict, trace: dict | None = None) -> np.ndarray:
    """`trace`, if given, receives {layer: (max |input|, max |weight|)} of the pointwise convolutions and the projection."""
    from omniswarm_b200 import synth
    t = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in w.items()}
    x = torch.from_numpy(img_u8.astype(np.float32))[None, None]      # u8 -> f32 UNSCALED (:8,:10)
    relu6 = lambda v: torch.clamp(v, 0.0, 6.0)

    def pointwise(x, n):
        if trace is not None:
            trace[n] = (float(x.abs().max()), float(t[n + ".weight"].abs().max()))
        return F.conv2d(x, t[n + ".weight"], t[n + ".bias"])

    with torch.no_grad():
        x = x * np.float32(synth.NV_INPUT_SCALE)
        x = relu6(F.conv2d(x, t["conv0.weight"], t["conv0.bias"], stride=2, padding=1))
        for i, (ci, co, s) in enumerate(synth.NV_BLOCKS):
            x = relu6(F.conv2d(x, t[f"b{i}.dw.weight"], t[f"b{i}.dw.bias"], stride=s, padding=1, groups=ci))
            x = relu6(pointwise(x, f"b{i}.pw"))
        x = pointwise(x, "proj")                                      # [1,D,h,w]
        x = x - x.mean(dim=(2, 3), keepdim=True)                      # per-image centring (makes random-weight
        x = x / torch.clamp(torch.norm(x, dim=1, keepdim=True), min=1e-12)   # descriptors image-specific); per-location L2
        a = torch.softmax(F.conv2d(x, t["assign.weight"], t["assign.bias"]), 1)   # [1,K,h,w]
        D, K = x.shape[1], a.shape[1]
        xf = x.reshape(D, -1)                                         # [D,P]
        af = a.reshape(K, -1)                                         # [K,P]
        vlad = af @ xf.t() - af.sum(1, keepdim=True) * t["centroids"]  # [K,D]
        vlad = vlad / torch.clamp(torch.norm(vlad, dim=1, keepdim=True), min=1e-12)   # intra-normalisation
        v = vlad.reshape(-1)
        v = v / torch.clamp(torch.norm(v), min=1e-12)              # (eps as F.normalize: blank images give 0, not NaN)
    return v.numpy().copy()


# ------------------------------------------------------------------------------------------------
# Local matcher: cv::BFMatcher(NORM_L2, crossCheck=true).match  (loop_cam.cpp:141-174,
# loop_detector.cpp:564-567; SURVEY.md Appendix A.5)
# ------------------------------------------------------------------------------------------------
def l2_distance_matrix(q: np.ndarray, t: np.ndarray) -> np.ndarray:
    """d(i,j) = sqrt(sum_k (q_ik - t_jk)^2), accumulated left-to-right in f32 (OpenCV normL2Sqr_ scalar
    order; the SIMD build reassociates -- distances are compared with a tolerance, indices exactly
    whenever the best/second-best gap exceeds it)."""
    q = q.astype(np.float32); t = t.astype(np.float32)
    d = np.zeros((q.shape[0], t.shape[0]), np.float32)
    for k in range(q.shape[1]):
        diff = q[:, k:k + 1] - t[None, :, k]
        d += diff * diff
    return np.sqrt(d)


def bf_crosscheck(q: np.ndarray, t: np.ndarray):
    """-> (qi, ti, dist): pairs (i, fwd[i]) with bwd[fwd[i]] == i, i ascending; first minimum wins."""
    if q.shape[0] == 0 or t.shape[0] == 0:
        return np.zeros(0, np.int32), np.zeros(0, np.int32), np.zeros(0, np.float32)
    d = l2_distance_matrix(q, t)
    fwd = d.argmin(1)
    bwd = d.argmin(0)
    qi = np.nonzero(bwd[fwd] == np.arange(q.shape[0]))[0]
    return qi.astype(np.int32), fwd[qi].astype(np.int32), d[qi, fwd[qi]]


# ------------------------------------------------------------------------------------------------
# Global DB: faiss::IndexFlatIP add/search + acceptance rule (loop_detector.cpp:150-287, A.4)
# ------------------------------------------------------------------------------------------------
class IndexFlatIP:
    """Exact inner product; top-k descending; ties -> ascending row id; labels -1 / scores -inf
    padded when fewer than k rows (faiss heap semantics: -inf sentinel)."""

    def __init__(self, dim: int):
        self.d = dim
        self.rows = np.zeros((0, dim), np.float32)

    @property
    def ntotal(self):
        return self.rows.shape[0]

    def add(self, x: np.ndarray):
        self.rows = np.concatenate([self.rows, x.reshape(-1, self.d).astype(np.float32)], 0)

    def scores(self, q: np.ndarray) -> np.ndarray:
        # f32 dot products accumulated in f64 then rounded: the "true" fp32-input inner product.
        return (self.rows.astype(np.float64) @ q.reshape(-1, self.d).astype(np.float64).T).T

    def search(self, q: np.ndarray, k: int):
        s = self.scores(q)                                   # [nq, n]
        nq = s.shape[0]
        D = np.full((nq, k), -np.inf, np.float32)
        I = np.full((nq, k), -1, np.int64)
        for r in range(nq):
            order = np.argsort(-s[r], kind="stable")[:k]
            D[r, :len(order)] = s[r, order].astype(np.float32)
            I[r, :len(order)] = order
        return D, I


class LoopDetectorDB:
    """LoopDetector's two databases and the literal query rule (loop_detector.cpp:150-287)."""

    def __init__(self, self_id: int, dim: int = 4096, inner_product_thres: float = 0.3,
                 init_mode_product_thres: float = 0.2, match_index_dist: int = 5):
        self.self_id = self_id
        self.local_index = IndexFlatIP(dim)
        self.remote_index = IndexFlatIP(dim)
        self.imgid2fisheye = {}
        self.imgid2dir = {}
        self.INNER_PRODUCT_THRES = inner_product_thres
        self.INIT_MODE_PRODUCT_THRES = init_mode_product_thres
        self.MATCH_INDEX_DIST = match_index_dist

    def add_image(self, drone_id: int, image_desc: np.ndarray) -> int:          # :164-173
        if drone_id == self.self_id:
            self.local_index.add(image_desc)
            return self.local_index.ntotal - 1
        self.remote_index.add(image_desc)
        return self.remote_index.ntotal - 1 + REMOTE_MAGIN_NUMBER

    def add_frame(self, msg_id: int, drone_id: int, image_descs, landmark_nums):  # :150-162
        for i, (d, n) in enumerate(zip(image_descs, landmark_nums)):
            if n > 0:
                idx = self.add_image(drone_id, d)
                self.imgid2fisheye[idx] = msg_id
                self.imgid2dir[idx] = i
        return msg_id

    def _search(self, q, index, remote_db, thres, max_index, state):           # :199-242
        off = REMOTE_MAGIN_NUMBER if remote_db else 0
        k = SEARCH_NEAREST_NUM + max_index
        D, I = index.search(q[None], k)
        ret = -1
        for i in range(k):
            lab = int(I[0, i])
            if lab < 0:
                continue
            if (lab + off) not in self.imgid2fisheye:
                continue
            ret = lab + off
            if lab <= index.ntotal - max_index and float(D[0, i]) > thres:     # :232  (<=, double thres)
                state["distance"] = float(D[0, i])
                return ret
        return ret

    def query(self, drone_id: int, q: np.ndarray, init_mode: bool, nonkeyframe: bool):   # :176-197
        """-> (id, distance).  distance starts at -1 (:263); caller accepts iff id!=-1 and distance>-1."""
        thres = self.INIT_MODE_PRODUCT_THRES if init_mode else self.INNER_PRODUCT_THRES
        st = {"distance": -1.0}
        if drone_id == self.self_id:
            r = self._search(q, self.remote_index, True, thres, 1, st)
            if not nonkeyframe:
                return self._search(q, self.local_index, False, thres, self.MATCH_INDEX_DIST, st), st["distance"]
            elif r != -1:
                return r, st["distance"]
            return -1, st["distance"]
        return self._search(q, self.local_index, False, thres, 1, st), st["distance"]
