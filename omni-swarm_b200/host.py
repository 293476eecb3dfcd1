"""Host-side mirror of the reference's C++ call sites, one class per replaced object.

Names, argument meaning and error behaviour follow the reference (paths relative to /root/reference):
  SuperPoint        <- SuperPointTensorRT            swarm_loop/include/swarm_loop/superpoint_tensorrt.h:20-28
  NetVLAD           <- MobileNetVLADTensorRT         swarm_loop/include/swarm_loop/mobilenetvlad_tensorrt.h:10-21
  IndexFlatIP       <- faiss::IndexFlatIP            swarm_loop/include/swarm_loop/loop_detector.h:27-29
  BFMatcher         <- cv::BFMatcher(NORM_L2, true)  swarm_loop/src/loop_cam.cpp:147-150
  PoseGraphSolver   <- SwarmLocalizationSolver::solve_once  swarm_localization/src/swarm_localization_solver.cpp:1668
  KeyframeFrontend  <- LoopCam::on_flattened_images + LoopDetector::on_image_recv database work
  LoopAnchor        <- SwarmLocalizationSolver::find_available_loops_detections  swarm_localization_solver.cpp:1594-1666
All compute happens in libomniswarm_b200.so; these classes only marshal numpy arrays.  FactorRows and AnchoredChain hold
the device buffers (torch tensors) that one solve's *_dev calls pass between them.
"""
from __future__ import annotations

import ctypes as C
import numpy as np

from . import lib as _l


def _f32(a):
    return np.ascontiguousarray(a, dtype=np.float32)


PRECISIONS = {"split_fp16": _l.PRECISION_SPLIT_FP16, "fp16": _l.PRECISION_FP16}


DB_STORAGES = {"fp32": _l.DB_STORAGE_FP32, "fp16": _l.DB_STORAGE_FP16}


def _db_storage(name: str) -> int:
    """'fp32' (the default: rows as given, faiss::IndexFlatIP) or 'fp16' (rows rounded to nearest-even fp16, half the bytes
    per scan; queries stay fp32) -> OSB_DB_STORAGE_*"""
    if name not in DB_STORAGES:
        raise ValueError(f"storage must be one of {sorted(DB_STORAGES)}, not {name!r}")
    return DB_STORAGES[name]


def _precision(name: str) -> int:
    """'split_fp16' (the default: two fp16 planes per operand, fp32-level accuracy) or 'fp16' (plain fp16 operands, the
    precision of the reference's fp16 TensorRT engines) -> OSB_PRECISION_*"""
    if name not in PRECISIONS:
        raise ValueError(f"precision must be one of {sorted(PRECISIONS)}, not {name!r}")
    return PRECISIONS[name]


class _Handle:
    """One library handle in `self._h`: `close()`, also run when the object is collected, destroys it once."""

    _destroy = ""        # name of the handle's osb_*_destroy

    def close(self):
        if getattr(self, "_h", None):
            getattr(self._lib, self._destroy)(self._h)
            self._h = None

    __del__ = close


class SuperPoint(_Handle):
    """`inference(image) -> (keypoints [N,2] f32 (x,y) by descending confidence, descriptors [N,64])`."""

    _destroy = "osb_superpoint_destroy"

    def __init__(self, weights: np.ndarray, pca_comp: np.ndarray, pca_mean: np.ndarray, width: int, height: int,
                 thres: float = 0.015, max_num: int = 200, max_batch: int = 8):
        self._lib = _l.load()
        self.width, self.height, self.thres, self.max_num, self.max_batch = width, height, thres, max_num, max_batch
        w, pc, pm = _f32(weights).reshape(-1), _f32(pca_comp), _f32(pca_mean)
        assert pc.shape == (64, 256) and pm.shape == (256,)
        self._h = C.c_void_p()
        _l.check(self._lib.osb_superpoint_create(C.byref(self._h), _l.ptr(w), w.size, width, height, thres, max_num,
                                                 _l.ptr(pc), _l.ptr(pm), max_batch))

    def _outputs(self, B):
        return (np.zeros(B, np.int32), np.zeros((B, self.max_num, 2), np.float32),
                np.zeros((B, self.max_num, 64), np.float32))

    def inference_batch(self, images: np.ndarray):
        """images [B,H,W] uint8 -> list of (kpts, desc)."""
        images = np.ascontiguousarray(images, dtype=np.uint8)
        # the reference asserts the image size (superpoint_tensorrt.cpp:122)
        assert images.ndim == 3 and images.shape[1:] == (self.height, self.width), \
            "Input image must have same size with network"
        B = images.shape[0]
        n, k, d = self._outputs(B)
        _l.check(self._lib.osb_superpoint_infer(self._h, _l.ptr(images), B, _l.ptr(n), _l.ptr(k), _l.ptr(d)))
        return [(k[b, :n[b]].copy(), d[b, :n[b]].copy()) for b in range(B)]

    def inference(self, image: np.ndarray):
        return self.inference_batch(image[None])[0]

    def postprocess(self, semi: np.ndarray, desc_nchw: np.ndarray):
        """parity hook: getKeyPoints + NMS2 + computeDescriptors on caller-supplied engine outputs."""
        semi, desc_nchw = _f32(semi), _f32(desc_nchw)
        if semi.ndim == 2:
            semi, desc_nchw = semi[None], desc_nchw[None]
        B = semi.shape[0]
        n, k, d = self._outputs(B)
        _l.check(self._lib.osb_superpoint_postprocess(self._h, _l.ptr(semi), _l.ptr(desc_nchw), B, _l.ptr(n),
                                                      _l.ptr(k), _l.ptr(d)))
        return [(k[b, :n[b]].copy(), d[b, :n[b]].copy()) for b in range(B)]

    LAYERS = ["conv1a", "conv1b+pool", "conv2a", "conv2b+pool", "conv3a", "conv3b+pool", "conv4a", "conv4b", "convPa",
              "convPb", "convDa", "convDb"]

    def layer_ms(self, images: np.ndarray) -> dict:
        """device time of every network layer for one batch (tensor-core path)."""
        _l.check(self._lib.osb_superpoint_set_profiling(self._h, 1))
        self.inference_batch(images)
        ms = np.zeros(12, np.float32)
        _l.check(self._lib.osb_superpoint_layer_ms(self._h, _l.ptr(ms), 12))
        _l.check(self._lib.osb_superpoint_set_profiling(self._h, 0))
        return {k: float(v) for k, v in zip(self.LAYERS, ms)}

    def set_precision(self, precision: str):
        """'split_fp16' (default) or 'fp16' for the network's tensor-core convolutions (osb_superpoint_set_precision)"""
        _l.check(self._lib.osb_superpoint_set_precision(self._h, _precision(precision)))

    def read(self, what: str, image: int = 0) -> np.ndarray:
        H, W = self.height, self.width
        shapes = {"semi": (0, (H, W)), "desc": (1, (256, H // 8, W // 8)), "conf": (2, (self.max_num,)),
                  "survivors": (3, (H, W)), "counts": (4, (8,))}
        code, shape = shapes[what]
        out = np.zeros(shape, np.float32)
        _l.check(self._lib.osb_superpoint_read(self._h, code, image, _l.ptr(out), out.size))
        return out

    @staticmethod
    def band_geometry(height: int, width: int, zero_row: int) -> dict:
        """the blanked band of images zero from row `zero_row` down (osb_superpoint_band_geometry): 'px' and 'tiles' [8, 4]
        per trunk layer conv1a .. conv4b, 'first_skip' [4]; every rectangle as y0, y1, x0, x1 of [y0, y1) x [x0, x1)"""
        out = np.zeros(68, np.int32)
        _l.check(_l.load().osb_superpoint_band_geometry(height, width, zero_row, _l.ptr(out)))
        r = out[:64].reshape(8, 2, 4)
        return {"px": r[:, 0].copy(), "tiles": r[:, 1].copy(), "first_skip": out[64:].copy()}


class NetVLAD(_Handle):
    """`inference(image) -> [4096] f32` (mobilenetvlad_tensorrt.cpp:4-15)."""

    _destroy = "osb_netvlad_destroy"

    def __init__(self, weights: np.ndarray, width: int, height: int, max_batch: int = 4):
        self._lib = _l.load()
        self.width, self.height = width, height
        w = _f32(weights).reshape(-1)
        self._h = C.c_void_p()
        _l.check(self._lib.osb_netvlad_create(C.byref(self._h), _l.ptr(w), w.size, width, height, max_batch))

    def inference_batch(self, images: np.ndarray) -> np.ndarray:
        images = np.ascontiguousarray(images, dtype=np.uint8)
        assert images.ndim == 3 and images.shape[1:] == (self.height, self.width)
        out = np.zeros((images.shape[0], _l.DEEP_DESC_SIZE), np.float32)
        _l.check(self._lib.osb_netvlad_infer(self._h, _l.ptr(images), images.shape[0], _l.ptr(out)))
        return out

    def inference(self, image: np.ndarray) -> np.ndarray:
        return self.inference_batch(image[None])[0]

    def set_precision(self, precision: str):
        """'split_fp16' (default) or 'fp16' for the pointwise convolutions (osb_netvlad_set_precision)"""
        _l.check(self._lib.osb_netvlad_set_precision(self._h, _precision(precision)))


class IndexFlatIP(_Handle):
    """faiss::IndexFlatIP look-alike: `add(x)`, `search(q, k) -> (D, I)`, `ntotal`."""

    _destroy = "osb_db_destroy"

    def __init__(self, d: int, capacity: int = 16384, storage: str = "fp32"):
        """storage 'fp16' keeps every row as float16 (round to nearest even; osb_db_create_storage)"""
        self._lib = _l.load()
        self.d = d
        self._h = C.c_void_p()
        _l.check(self._lib.osb_db_create_storage(C.byref(self._h), d, capacity, _db_storage(storage)))

    @property
    def ntotal(self) -> int:
        return int(self._lib.osb_db_size(self._h))

    def add(self, x: np.ndarray) -> int:
        x = _f32(x).reshape(-1, self.d)
        first = C.c_int64(-1)
        _l.check(self._lib.osb_db_add(self._h, x.shape[0], _l.ptr(x), C.byref(first)))
        return int(first.value)

    def search(self, q: np.ndarray, k: int):
        q = _f32(q).reshape(-1, self.d)
        D = np.zeros((q.shape[0], k), np.float32)
        I = np.zeros((q.shape[0], k), np.int64)
        _l.check(self._lib.osb_db_search(self._h, q.shape[0], _l.ptr(q), k, _l.ptr(D), _l.ptr(I)))
        return D, I

    def search_dev(self, q_ptr: int, nq: int, k: int, scores_ptr: int, ids_ptr: int, stream: int):
        """device pointers in / out, no synchronisation (osb_db_search_dev)."""
        _l.check(self._lib.osb_db_search_dev(self._h, nq, C.c_void_p(q_ptr), k, C.c_void_p(scores_ptr),
                                             C.c_void_p(ids_ptr), C.c_void_p(stream)))

    def add_dev(self, x_ptr: int, n: int, stream: int) -> int:
        first = C.c_int64(-1)
        _l.check(self._lib.osb_db_add_dev(self._h, n, C.c_void_p(x_ptr), C.byref(first), C.c_void_p(stream)))
        return int(first.value)

    def reset(self):
        _l.check(self._lib.osb_db_reset(self._h))


class BFMatcher(_Handle):
    """cv::BFMatcher(cv::NORM_L2, crossCheck=True): `match(query, train) -> (queryIdx, trainIdx, distance)`."""

    _destroy = "osb_matcher_destroy"

    def __init__(self, max_pairs: int = 8, max_n: int = 200, dim: int = 64):
        self._lib = _l.load()
        self.max_pairs, self.max_n, self.dim = max_pairs, max_n, dim
        self._h = C.c_void_p()
        _l.check(self._lib.osb_matcher_create(C.byref(self._h), max_pairs, max_n, dim))

    def match_batch(self, queries, trains):
        P = len(queries)
        q = np.zeros((P, self.max_n, self.dim), np.float32)
        t = np.zeros((P, self.max_n, self.dim), np.float32)
        nq = np.array([len(x) for x in queries], np.int32)
        nt = np.array([len(x) for x in trains], np.int32)
        for p in range(P):
            q[p, :nq[p]] = queries[p]
            t[p, :nt[p]] = trains[p]
        qi = np.zeros((P, self.max_n), np.int32); ti = np.zeros((P, self.max_n), np.int32)
        dist = np.zeros((P, self.max_n), np.float32); n = np.zeros(P, np.int32)
        _l.check(self._lib.osb_matcher_match(self._h, P, _l.ptr(q), _l.ptr(nq), _l.ptr(t), _l.ptr(nt), _l.ptr(qi),
                                             _l.ptr(ti), _l.ptr(dist), _l.ptr(n)))
        return [(qi[p, :n[p]].copy(), ti[p, :n[p]].copy(), dist[p, :n[p]].copy()) for p in range(P)]

    def match(self, query: np.ndarray, train: np.ndarray):
        return self.match_batch([query], [train])[0]


def homography_ransac(src_list, dst_list, thresh: float = 3.0, seed: int = 0):
    """cv::findHomography(old_2d, new_2d, CV_RANSAC, 3, mask) for several correspondence sets at once
    (loop_detector.cpp:589-598): src_list[i] = old_2d, dst_list[i] = new_2d, [n_i, 2] float32 ->
    list of (mask uint8 [n_i], n_inliers, winning hypothesis)."""
    lib = _l.load()
    n_pairs = len(src_list)
    max_n = max(1, max(len(a) for a in src_list))
    src = np.zeros((n_pairs, max_n, 2), np.float32); dst = np.zeros((n_pairs, max_n, 2), np.float32)
    n = np.zeros(n_pairs, np.int32)
    for i, (a, b) in enumerate(zip(src_list, dst_list)):
        n[i] = len(a)
        if len(a):
            src[i, :len(a)] = a; dst[i, :len(a)] = b
    mask = np.zeros((n_pairs, max_n), np.uint8); ninl = np.zeros(n_pairs, np.int32); win = np.zeros(n_pairs, np.int32)
    _l.check(lib.osb_homography_ransac(_l.ptr(src), _l.ptr(dst), _l.ptr(n), n_pairs, max_n, float(thresh), int(seed),
                                       _l.ptr(mask), _l.ptr(ninl), _l.ptr(win)))
    return [(mask[i, :n[i]].copy(), int(ninl[i]), int(win[i])) for i in range(n_pairs)]


class PoseGraphSolver(_Handle):
    """Flat-array form of SwarmLocalizationSolver::solve_once: `solve(graph) -> (poses, summary)`."""

    _destroy = "osb_solver_destroy"

    def __init__(self, max_nodes: int = 4096, max_factors: int = 32768):
        self._lib = _l.load()
        self._h = C.c_void_p()
        _l.check(self._lib.osb_solver_create(C.byref(self._h), max_nodes, max_factors))

    def default_options(self) -> _l.SolveOptions:
        o = _l.SolveOptions()
        self._lib.osb_solve_default_options(C.byref(o))
        return o

    @staticmethod
    def _arrays(g):
        return (np.ascontiguousarray(g["fixed"], np.uint8), np.ascontiguousarray(g["ftype"], np.int32),
                np.ascontiguousarray(g["ia"], np.int32), np.ascontiguousarray(g["ib"], np.int32),
                np.ascontiguousarray(g["payload"], np.float64), np.ascontiguousarray(g["huber"], np.uint8))

    def solve(self, g: dict, options: _l.SolveOptions | None = None, init: np.ndarray | None = None):
        fixed, ftype, ia, ib, payload, huber = self._arrays(g)
        poses = np.ascontiguousarray(g["init"] if init is None else init, np.float64).copy()
        opt = options if options is not None else self.default_options()
        summ = _l.SolveSummary()
        _l.check(self._lib.osb_solver_solve(self._h, poses.shape[0], _l.ptr(poses), _l.ptr(fixed), len(ftype),
                                            _l.ptr(ftype), _l.ptr(ia), _l.ptr(ib), _l.ptr(payload), _l.ptr(huber),
                                            C.byref(opt), C.byref(summ)))
        return poses, summ

    def solve_multistart(self, g: dict, init_mask: np.ndarray, n_trials: int, seed: int, window_size: int,
                         acpt_cost: float, normalise: bool = True, options: _l.SolveOptions | None = None,
                         rand_xy: float = 5.0, rand_z: float = 1.0, init: np.ndarray | None = None):
        """SwarmLocalizationSolver::solve_with_multiple_init (solver.cpp:781-845): n_trials solves from random
        restarts of the masked nodes, in one launch.  Returns (poses, chosen, summaries, equv): the chosen trial's poses
        (the starting poses when chosen == -1, i.e. no trial got below acpt_cost), the trial index, the K summaries and
        the K equv_costs."""
        fixed, ftype, ia, ib, payload, huber = self._arrays(g)
        poses = np.ascontiguousarray(g["init"] if init is None else init, np.float64).copy()
        mask = np.ascontiguousarray(init_mask, np.uint8)
        assert mask.shape == (poses.shape[0],)
        opt = options if options is not None else self.default_options()
        ms = _l.MultistartOptions(n_trials=n_trials, normalise=int(normalise), window_size=window_size, seed=seed,
                                  rand_xy=rand_xy, rand_z=rand_z, acpt_cost=acpt_cost)
        summ = (_l.SolveSummary * max(1, n_trials))()
        equv = np.zeros(max(1, n_trials), np.float64)
        chosen = C.c_int32(-2)
        _l.check(self._lib.osb_solver_solve_multistart(self._h, poses.shape[0], _l.ptr(poses), _l.ptr(fixed),
                                                       _l.ptr(mask), len(ftype), _l.ptr(ftype), _l.ptr(ia), _l.ptr(ib),
                                                       _l.ptr(payload), _l.ptr(huber), C.byref(opt), C.byref(ms),
                                                       C.cast(summ, C.c_void_p), _l.ptr(equv), C.byref(chosen)))
        return poses, int(chosen.value), list(summ), equv

    # ---- resident graph (SURVEY 8f-4): the factor list stays on the device between solves ----
    def graph_clear(self):
        _l.check(self._lib.osb_solver_graph_clear(self._h))

    def graph_add_nodes(self, poses: np.ndarray, fixed: np.ndarray | None = None) -> int:
        poses = np.ascontiguousarray(poses, np.float64).reshape(-1, 4)
        fx = None if fixed is None else np.ascontiguousarray(fixed, np.uint8)
        first = C.c_int32(-1)
        _l.check(self._lib.osb_solver_graph_add_nodes(self._h, poses.shape[0], _l.ptr(poses),
                                                      None if fx is None else _l.ptr(fx), C.byref(first)))
        return int(first.value)

    def graph_add_factors(self, ftype, ia, ib, payload, huber):
        ftype = np.ascontiguousarray(ftype, np.int32); ia = np.ascontiguousarray(ia, np.int32)
        ib = np.ascontiguousarray(ib, np.int32); huber = np.ascontiguousarray(huber, np.uint8)
        payload = np.ascontiguousarray(payload, np.float64)
        _l.check(self._lib.osb_solver_graph_add_factors(self._h, len(ftype), _l.ptr(ftype), _l.ptr(ia), _l.ptr(ib),
                                                        _l.ptr(payload), _l.ptr(huber)))

    def graph_set_fixed(self, node: int, fixed: bool = True):
        _l.check(self._lib.osb_solver_graph_set_fixed(self._h, node, int(fixed)))

    def graph_set_poses(self, first: int, poses: np.ndarray):
        poses = np.ascontiguousarray(poses, np.float64).reshape(-1, 4)
        _l.check(self._lib.osb_solver_graph_set_poses(self._h, first, poses.shape[0], _l.ptr(poses)))

    def graph_get_poses(self, first: int = 0, n: int | None = None) -> np.ndarray:
        if n is None:
            n = self.graph_size()[0] - first
        out = np.zeros((n, 4), np.float64)
        _l.check(self._lib.osb_solver_graph_get_poses(self._h, first, n, _l.ptr(out)))
        return out

    def graph_size(self) -> tuple[int, int]:
        a, b = C.c_int32(0), C.c_int32(0)
        _l.check(self._lib.osb_solver_graph_size(self._h, C.byref(a), C.byref(b)))
        return int(a.value), int(b.value)

    def graph_drop_oldest(self, n_nodes: int):
        _l.check(self._lib.osb_solver_graph_drop_oldest(self._h, n_nodes))

    def solve_resident(self, options: _l.SolveOptions | None = None) -> _l.SolveSummary:
        opt = options if options is not None else self.default_options()
        summ = _l.SolveSummary()
        _l.check(self._lib.osb_solver_solve_resident(self._h, C.byref(opt), C.byref(summ)))
        return summ

    def solve_resident_dev(self, max_tail: int, type_ptr: int, ia_ptr: int, ib_ptr: int, payload_ptr: int,
                           huber_ptr: int, count_ptr: int, stream: int, options: _l.SolveOptions | None = None):
        """solve the resident graph plus *count_ptr tail rows read on the device (compact_anchored_factors' arrays), on
        `stream` without synchronising; the poses stay on the device until a host-side call (see last_summary)"""
        opt = options if options is not None else self.default_options()
        _l.check(self._lib.osb_solver_solve_resident_dev(self._h, int(max_tail), C.c_void_p(type_ptr), C.c_void_p(ia_ptr),
                                                         C.c_void_p(ib_ptr), C.c_void_p(payload_ptr),
                                                         C.c_void_p(huber_ptr), C.c_void_p(count_ptr), C.byref(opt),
                                                         C.c_void_p(stream)))

    def last_summary(self) -> _l.SolveSummary:
        """synchronises with the last solve_resident_dev call -> its summary (raises its refusal code)"""
        summ = _l.SolveSummary()
        _l.check(self._lib.osb_solver_last_summary(self._h, C.byref(summ)))
        return summ

    def solve_multistart_resident_dev(self, max_tail: int, type_ptr: int, ia_ptr: int, ib_ptr: int, payload_ptr: int,
                                      huber_ptr: int, count_ptr: int, mask_ptr: int, yaw_ptr, stream: int, n_trials: int,
                                      seed: int, window_size: int, acpt_cost: float, normalise: bool = True,
                                      options: _l.SolveOptions | None = None, rand_xy: float = 5.0, rand_z: float = 1.0):
        """solve_multistart of the resident graph plus *count_ptr tail rows read on the device, started from the resident
        device poses, the nodes of the uint8 device mask at mask_ptr scattered (yaw from the float64 device array at
        yaw_ptr, or kept when it is None), on `stream` without synchronising; the chosen poses stay on the device until a
        host-side call (see last_multistart)"""
        opt = options if options is not None else self.default_options()
        ms = _l.MultistartOptions(n_trials=int(n_trials), normalise=int(normalise), window_size=int(window_size),
                                  seed=int(seed), rand_xy=rand_xy, rand_z=rand_z, acpt_cost=acpt_cost)
        _l.check(self._lib.osb_solver_solve_multistart_resident_dev(
            self._h, int(max_tail), C.c_void_p(type_ptr), C.c_void_p(ia_ptr), C.c_void_p(ib_ptr), C.c_void_p(payload_ptr),
            C.c_void_p(huber_ptr), C.c_void_p(count_ptr), C.c_void_p(mask_ptr),
            None if yaw_ptr is None else C.c_void_p(yaw_ptr), C.byref(opt), C.byref(ms), C.c_void_p(stream)))
        self._ms_trials = int(n_trials)

    def last_multistart(self):
        """synchronises with the last solve_multistart_resident_dev call -> (chosen, summaries, equv), as
        solve_multistart returns them (raises its refusal code)"""
        k = max(1, getattr(self, "_ms_trials", 1))
        summ = (_l.SolveSummary * k)()
        equv = np.zeros(k, np.float64)
        chosen = C.c_int32(-2)
        _l.check(self._lib.osb_solver_last_multistart(self._h, C.cast(summ, C.c_void_p), _l.ptr(equv), C.byref(chosen)))
        return int(chosen.value), list(summ), equv

    def phase_cycles(self) -> dict:
        c = np.zeros(12, np.float64)
        _l.check(self._lib.osb_solver_phase_cycles(self._h, _l.ptr(c)))
        names = ["factor", "barrier", "node1", "reduce1", "node2", "reduce2", "cg_iterations", "kernel", "ctas",
                 "cluster", "j_in_smem", "threads"]
        d = dict(zip(names, c.tolist()))
        d["chain_preconditioner"] = float((int(d["j_in_smem"]) >> 1) & 1)
        d["inner_fp32"] = float((int(d["j_in_smem"]) >> 2) & 1)
        d["j_in_smem"] = float(int(d["j_in_smem"]) & 1)
        return d

    def chain_cycles(self) -> np.ndarray:
        c = np.zeros(128, np.float64)
        _l.check(self._lib.osb_solver_chain_cycles(self._h, _l.ptr(c)))
        return c.reshape(16, 8)

    @staticmethod
    def chain_plan(g: dict):
        """Host-only: the solver's internal node numbering (greedy maximum-weight path cover) ->
        (order [n] internal -> caller's node id, link [n] uint8)."""
        lib = _l.load()
        fixed = np.ascontiguousarray(g["fixed"], np.uint8)
        ftype = np.ascontiguousarray(g["ftype"], np.int32)
        ia = np.ascontiguousarray(g["ia"], np.int32); ib = np.ascontiguousarray(g["ib"], np.int32)
        payload = np.ascontiguousarray(g["payload"], np.float64)
        n = fixed.shape[0]
        order = np.zeros(n, np.int32); link = np.zeros(n, np.uint8)
        _l.check(lib.osb_solver_chain_plan(n, _l.ptr(fixed), len(ftype), _l.ptr(ftype), _l.ptr(ia), _l.ptr(ib),
                                           _l.ptr(payload), _l.ptr(order), _l.ptr(link)))
        return order, link

    def linearize(self, g: dict, poses: np.ndarray):
        _, ftype, ia, ib, payload, _ = self._arrays(g)
        poses = np.ascontiguousarray(poses, np.float64)
        m = len(ftype)
        r = np.zeros((m, 4)); Ja = np.zeros((m, 4, 4)); Jb = np.zeros((m, 4, 4))
        _l.check(self._lib.osb_solver_linearize(self._h, poses.shape[0], _l.ptr(poses), m, _l.ptr(ftype), _l.ptr(ia),
                                                _l.ptr(ib), _l.ptr(payload), _l.ptr(r), _l.ptr(Ja), _l.ptr(Jb)))
        return r, Ja, Jb


class KeyframeFrontend(_Handle):
    """The per-keyframe pipeline (extract -> ingest -> query) on one GPU."""

    _destroy = "osb_frontend_destroy"

    def __init__(self, sp_weights, pca_comp, pca_mean, nv_weights, width=640, height=480, n_dirs=4, max_num=200,
                 sp_thres=0.015, self_id=0, db_capacity=16384, inner_product_thres=0.3, init_mode_product_thres=0.2,
                 match_index_dist=5, query_dir=None, zero_bottom_quarter=True, accept_min_3d_pts=10,
                 geometric_filter=False, ransac_seed=0):
        self._lib = _l.load()
        cfg = _l.FrontendConfig()
        cfg.width, cfg.height, cfg.n_dirs, cfg.max_num = width, height, n_dirs, max_num
        cfg.sp_thres, cfg.self_id, cfg.db_capacity = sp_thres, self_id, db_capacity
        cfg.inner_product_thres, cfg.init_mode_product_thres = inner_product_thres, init_mode_product_thres
        cfg.match_index_dist = match_index_dist
        cfg.query_dir = (1 if n_dirs > 1 else 0) if query_dir is None else query_dir
        cfg.zero_bottom_quarter = int(zero_bottom_quarter)
        cfg.accept_min_3d_pts = accept_min_3d_pts
        cfg.geometric_filter, cfg.ransac_seed = int(geometric_filter), int(ransac_seed)
        self.cfg = cfg
        spw, nvw = _f32(sp_weights).reshape(-1), _f32(nv_weights).reshape(-1)
        pc, pm = _f32(pca_comp), _f32(pca_mean)
        self._h = C.c_void_p()
        _l.check(self._lib.osb_frontend_create(C.byref(self._h), C.byref(cfg), _l.ptr(spw), spw.size, _l.ptr(pc),
                                               _l.ptr(pm), _l.ptr(nvw), nvw.size))

    def process(self, images_up: np.ndarray, images_down: np.ndarray, msg_id: int):
        """HOST images [n_dirs,H,W] u8 -> (KeyframeRecord, LoopResult); one synchronisation."""
        up = np.ascontiguousarray(images_up, np.uint8); down = np.ascontiguousarray(images_down, np.uint8)
        rec, res = _l.KeyframeRecord(), _l.LoopResult()
        _l.check(self._lib.osb_frontend_process(self._h, _l.ptr(up), _l.ptr(down), msg_id, C.byref(rec), C.byref(res)))
        return rec, res

    def process_raw(self, up_ptr: int, down_ptr: int, msg_id: int, rec_ptr: int, res_ptr: int):
        """same, with raw HOST pointers (pinned buffers owned by the caller)."""
        _l.check(self._lib.osb_frontend_process(self._h, C.c_void_p(up_ptr), C.c_void_p(down_ptr), msg_id,
                                                C.c_void_p(rec_ptr), C.c_void_p(res_ptr)))

    def extract(self, up_ptr: int, down_ptr: int, msg_id: int, record_dev: int, stream: int, device_images=False):
        fn = self._lib.osb_frontend_extract_dev if device_images else self._lib.osb_frontend_extract
        _l.check(fn(self._h, C.c_void_p(up_ptr), C.c_void_p(down_ptr), msg_id, C.c_void_p(record_dev), C.c_void_p(stream)))

    def ingest(self, records_dev: int, n_records: int, skip: int, stream: int):
        _l.check(self._lib.osb_frontend_ingest(self._h, C.c_void_p(records_dev), n_records, skip, C.c_void_p(stream)))

    def ingest_own(self, record_dev: int, stream: int):
        """add_to_database of the record `extract` has just written (this drone's own)"""
        _l.check(self._lib.osb_frontend_ingest_own(self._h, C.c_void_p(record_dev), C.c_void_p(stream)))

    def query(self, record_dev: int, result_dev: int, stream: int, init_mode=False, nonkeyframe=False):
        _l.check(self._lib.osb_frontend_query(self._h, C.c_void_p(record_dev), int(init_mode), int(nonkeyframe),
                                              C.c_void_p(result_dev), C.c_void_p(stream)))

    def query_received(self, records_dev: int, n_records: int, skip: int, results_dev: int, stream: int, init_mode=None):
        """query_from_database for a batch of keyframes received from other drones (osb_frontend_query_received): record r
        != skip with a foreign drone_id -> results_dev[r], one scan of the local store for the batch.  init_mode: None (all
        off) or n_records flags."""
        flags = None
        if init_mode is not None:
            flags = np.ascontiguousarray(np.asarray(init_mode, dtype=bool), np.uint8)
            assert flags.shape == (n_records,), "init_mode needs one flag per record"
        _l.check(self._lib.osb_frontend_query_received(self._h, C.c_void_p(records_dev), n_records, skip,
                                                       None if flags is None else _l.ptr(flags), C.c_void_p(results_dev),
                                                       C.c_void_p(stream)))

    def set_loop_params(self, min_loop_num=15, init_mode_min_loop_num=10, min_match_per_dir=15, min_direction_loop=3,
                        is_4dof=True, reproj_thresh=3.0, seed=0, rperr_thres=10 * np.pi / 180,
                        accept_loop_yaw_rad=30 * np.pi / 180, max_loop_dis=5.0, odometry_consistency_threshold=2.0):
        """the constants of compute_loop (swarm_loop.cpp:221-256, loop_defines.h defaults); before the first remote ingest"""
        p = _l.LoopParams(min_loop_num=min_loop_num, init_mode_min_loop_num=init_mode_min_loop_num,
                          min_match_per_dir=min_match_per_dir, min_direction_loop=min_direction_loop, is_4dof=int(is_4dof),
                          reproj_thresh=reproj_thresh, seed=seed, rperr_thres=rperr_thres,
                          accept_loop_yaw_rad=accept_loop_yaw_rad, max_loop_dis=max_loop_dis,
                          odometry_consistency_threshold=odometry_consistency_threshold)
        _l.check(self._lib.osb_frontend_set_loop_params(self._h, C.byref(p)))

    @staticmethod
    def loop_candidates(cands):
        """list of dicts (pose_query [7], pose_hit [7]; optional init_mode, odom_rel [7], cov [6,6]) -> LoopCandidate array"""
        arr = (_l.LoopCandidate * len(cands))()
        for a, c in zip(arr, cands):
            a.init_mode = int(bool(c.get("init_mode", False)))
            a.pose_query[:] = [float(x) for x in c["pose_query"]]
            a.pose_hit[:] = [float(x) for x in c["pose_hit"]]
            a.odom_rel[:] = [float(x) for x in c.get("odom_rel", [0, 0, 0, 1, 0, 0, 0])]
            a.odom_edge_cov[:] = [float(x) for x in np.asarray(c.get("cov", np.eye(6)), np.float64).reshape(-1)]
        return arr

    def compute_loop(self, records_dev: int, results_dev: int, cands, out_dev: int, stream: int):
        """loop edges of n = len(cands) query results (osb_frontend_compute_loop): records_dev / results_dev [n] as query or
        query_received wrote them, cands a list of dicts (see loop_candidates) -> LoopEdgeResult [n] at out_dev, no
        synchronisation"""
        arr = self.loop_candidates(cands)
        _l.check(self._lib.osb_frontend_compute_loop(self._h, C.c_void_p(records_dev), C.c_void_p(results_dev), len(cands),
                                                     arr, C.c_void_p(out_dev), C.c_void_p(stream)))

    @staticmethod
    def loop_stamps(stamps):
        """[(stamp_query_ns, stamp_hit_ns)] per candidate -> LoopStamps array"""
        arr = (_l.LoopStamps * len(stamps))()
        for a, (q, h) in zip(arr, stamps):
            a.stamp_query_ns, a.stamp_hit_ns = int(q), int(h)
        return arr

    def loop_measurements(self, results_dev: int, edges_dev: int, cands, stamps, loop_cov_pos: float, loop_cov_ang: float,
                          out_dev: int, count_dev: int, stream: int):
        """the LoopEdge of every ACCEPTED candidate of the preceding compute_loop (osb_frontend_loop_measurements): rows of
        lib.MEASUREMENT_DTYPE at out_dev in candidate order and their number into the int32 at count_dev, on `stream`
        without synchronising.  cands: the list compute_loop took; stamps: (stamp_query_ns, stamp_hit_ns) per candidate.
        Either may also be given as the ctypes array loop_candidates / loop_stamps made of it, built once by a caller that
        repeats the call."""
        assert len(stamps) == len(cands), "one stamp pair per candidate"
        arr = cands if isinstance(cands, C.Array) else self.loop_candidates(cands)
        st = stamps if isinstance(stamps, C.Array) else self.loop_stamps(stamps)
        _l.check(self._lib.osb_frontend_loop_measurements(self._h, C.c_void_p(results_dev), C.c_void_p(edges_dev),
                                                          len(cands), arr, st, float(loop_cov_pos), float(loop_cov_ang),
                                                          C.c_void_p(out_dev), C.c_void_p(count_dev), C.c_void_p(stream)))

    def loop_counts(self):
        """waits for the last loop_measurements -> (loop_count, inter_drone_loop_count [256, 256] int32, [new][old])"""
        n = C.c_int64(0)
        pairs = np.zeros((_l.LOOP_PAIR_DRONES, _l.LOOP_PAIR_DRONES), np.int32)
        _l.check(self._lib.osb_frontend_loop_counts(self._h, C.byref(n), _l.ptr(pairs)))
        return n.value, pairs

    # ---- keyframe metadata and a round's loop candidates on the device ------------------------------------------
    @staticmethod
    def keyframe_metas(metas):
        """list of (drone_id, msg_id, stamp_ns, pose_drone [7]) -> KeyframeMeta array (upload its bytes beside the records)"""
        arr = (_l.KeyframeMeta * len(metas))()
        for a, (drone, msg, stamp, pose) in zip(arr, metas):
            a.drone_id, a.msg_id, a.stamp_ns = int(drone), int(msg), int(stamp)
            a.pose_drone[:] = [float(x) for x in pose]
        return arr

    def ingest_meta(self, records_dev: int, metas_dev: int, n_records: int, skip: int, stream: int):
        """ingest, and each record's osb_keyframe_meta (metas_dev [n_records]) into the frame slot it takes"""
        _l.check(self._lib.osb_frontend_ingest_meta(self._h, C.c_void_p(records_dev), C.c_void_p(metas_dev), n_records, skip,
                                                    C.c_void_p(stream)))

    def ingest_own_meta(self, record_dev: int, meta_dev: int, stream: int):
        """ingest_own with the keyframe's meta; it also extends the ego-motion trajectory"""
        _l.check(self._lib.osb_frontend_ingest_own_meta(self._h, C.c_void_p(record_dev), C.c_void_p(meta_dev),
                                                        C.c_void_p(stream)))

    def meta_status(self) -> int:
        """waits for the last ingest -> the status of the last meta ingest (lib.OK, lib.ERR_INVALID, lib.ERR_CAPACITY)"""
        st = C.c_int(0)
        self._lib.osb_frontend_meta_status(self._h, C.byref(st))
        return st.value

    def set_candidate_params(self, inter_drone_init_frames=50, pos_covariance_per_meter=0.01, yaw_covariance_per_meter=0.003,
                             loop_cov_pos=0.013, loop_cov_ang=2.5e-4):
        """the constants of the device-built candidates (swarm_loop.cpp:227-256 defaults)"""
        p = _l.CandidateParams(inter_drone_init_frames=inter_drone_init_frames,
                               pos_covariance_per_meter=pos_covariance_per_meter,
                               yaw_covariance_per_meter=yaw_covariance_per_meter, loop_cov_pos=loop_cov_pos,
                               loop_cov_ang=loop_cov_ang)
        _l.check(self._lib.osb_frontend_set_candidate_params(self._h, C.byref(p)))

    def init_modes_dev(self, records_dev: int, n_records: int, skip: int, out_dev: int, stream: int):
        """init_mode bytes [n_records] of a received round from the device's inter_drone_loop_count"""
        _l.check(self._lib.osb_frontend_init_modes_dev(self._h, C.c_void_p(records_dev), n_records, skip, C.c_void_p(out_dev),
                                                       C.c_void_p(stream)))

    def receive_dev(self, records_dev: int, n_records: int, skip: int, out_dev: int, stream: int):
        """the received records as LoopNet delivers them and on_image_recv keeps them (osb_frontend_receive_dev): foreign
        records [n_records] -> their flagged landmarks only, gated frames zeroed, at out_dev; pass out_dev to the rest of
        the round"""
        _l.check(self._lib.osb_frontend_receive_dev(self._h, C.c_void_p(records_dev), n_records, skip, C.c_void_p(out_dev),
                                                    C.c_void_p(stream)))

    def query_received_dev(self, records_dev: int, n_records: int, skip: int, init_mode_dev, results_dev: int, stream: int):
        """query_received with init_mode a device byte array [n_records] (or None: all 0)"""
        _l.check(self._lib.osb_frontend_query_received_dev(self._h, C.c_void_p(records_dev), n_records, skip,
                                                           None if init_mode_dev is None else C.c_void_p(init_mode_dev),
                                                           C.c_void_p(results_dev), C.c_void_p(stream)))

    def loop_candidates_dev(self, records_dev: int, metas_dev: int, results_dev: int, n: int, init_mode_dev,
                            cand_out_dev: int, stamps_out_dev: int, stream: int):
        """LoopCandidate [n] and LoopStamps [n] of a round's results, built on the device (osb_frontend_loop_candidates_dev)"""
        _l.check(self._lib.osb_frontend_loop_candidates_dev(self._h, C.c_void_p(records_dev), C.c_void_p(metas_dev),
                                                            C.c_void_p(results_dev), n,
                                                            None if init_mode_dev is None else C.c_void_p(init_mode_dev),
                                                            C.c_void_p(cand_out_dev), C.c_void_p(stamps_out_dev),
                                                            C.c_void_p(stream)))

    def compute_loop_dev(self, records_dev: int, results_dev: int, n: int, cand_dev: int, out_dev: int, stream: int):
        """compute_loop with the candidates read from the device array cand_dev [n]"""
        _l.check(self._lib.osb_frontend_compute_loop_dev(self._h, C.c_void_p(records_dev), C.c_void_p(results_dev), n,
                                                         C.c_void_p(cand_dev), C.c_void_p(out_dev), C.c_void_p(stream)))

    def loop_measurements_dev(self, results_dev: int, edges_dev: int, n: int, cand_dev: int, stamps_dev: int,
                              loop_cov_pos: float, loop_cov_ang: float, out_dev: int, count_dev: int, stream: int):
        """loop_measurements with the candidates and stamps read from device arrays [n]"""
        _l.check(self._lib.osb_frontend_loop_measurements_dev(self._h, C.c_void_p(results_dev), C.c_void_p(edges_dev), n,
                                                              C.c_void_p(cand_dev), C.c_void_p(stamps_dev),
                                                              float(loop_cov_pos), float(loop_cov_ang), C.c_void_p(out_dev),
                                                              C.c_void_p(count_dev), C.c_void_p(stream)))

    def finish(self, stream: int):
        _l.check(self._lib.osb_frontend_finish(self._h, C.c_void_p(stream)))

    STAGES = ["superpoint_net(+keypoints beside descriptor head)", "descriptors", "netvlad_unhidden", "stereo_pack", "add_to_database", "db_scan",
              "rule_local_match"]

    def set_profiling(self, enable: bool):
        _l.check(self._lib.osb_frontend_set_profiling(self._h, int(enable)))

    def set_precision(self, precision: str):
        """'split_fp16' (default) or 'fp16' for both networks of the front-end (osb_frontend_set_precision)"""
        _l.check(self._lib.osb_frontend_set_precision(self._h, _precision(precision)))

    def set_db_storage(self, storage: str):
        """'fp32' (default) or 'fp16' for the global-descriptor rows of both databases (osb_frontend_set_db_storage); only
        while both are empty"""
        _l.check(self._lib.osb_frontend_set_db_storage(self._h, _db_storage(storage)))

    def set_main_camera(self, which: str):
        """'up' (default) or 'down': the reference's LOWER_CAM_AS_MAIN (osb_frontend_set_main_camera).  With 'down' the
        record is the down image's, NetVLAD runs on the down images and compute_loop uses the right extrinsics."""
        cams = {"up": _l.MAIN_CAMERA_UP, "down": _l.MAIN_CAMERA_DOWN}
        if which not in cams:
            raise ValueError(f"main camera must be 'up' or 'down', not {which!r}")
        _l.check(self._lib.osb_frontend_set_main_camera(self._h, cams[which]))

    def stage_ms(self) -> dict:
        ms = np.zeros(8, np.float32)
        _l.check(self._lib.osb_frontend_stage_ms(self._h, _l.ptr(ms)))
        return {k: float(v) for k, v in zip(self.STAGES, ms)}

    def set_cameras(self, intrinsics, left_extrinsics, right_extrinsics, triangle_thres=0.006):
        """stereo triangulation inside extract: the record then carries landmarks_3d / landmarks_flag (loop_cam.cpp:393-432)"""
        K = np.ascontiguousarray(intrinsics, np.float64)
        le, re = np.ascontiguousarray(left_extrinsics, np.float64), np.ascontiguousarray(right_extrinsics, np.float64)
        _l.check(self._lib.osb_frontend_set_cameras(self._h, _l.ptr(K), _l.ptr(le), _l.ptr(re), float(triangle_thres)))

    def set_drone_pose(self, pose_drone):
        p = np.ascontiguousarray(pose_drone, np.float64)
        _l.check(self._lib.osb_frontend_set_drone_pose(self._h, _l.ptr(p)))

    def set_depth_camera(self, intrinsics, extrinsics, near_thres=0.3, far_thres=10.0):
        """PINHOLE_DEPTH keyframes (loop_cam.cpp:231-302): pinhole intrinsics fx fy cx cy, extrinsics [n_dirs,7],
        DEPTH_NEAR_THRES / DEPTH_FAR_THRES in metres"""
        K = np.ascontiguousarray(intrinsics, np.float64)
        ext = np.ascontiguousarray(extrinsics, np.float64)
        assert K.shape == (4,) and ext.shape == (self.cfg.n_dirs, 7)
        _l.check(self._lib.osb_frontend_set_depth_camera(self._h, _l.ptr(K), _l.ptr(ext), float(near_thres), float(far_thres)))

    def _depth_inputs(self, images, depth_mm):
        img = np.ascontiguousarray(images, np.uint8); dep = np.ascontiguousarray(depth_mm, np.uint16)
        shape = (self.cfg.n_dirs, self.cfg.height, self.cfg.width)
        assert img.shape == shape and dep.shape == shape, "images and depth must be [n_dirs, H, W]"
        return img, dep

    def extract_depth(self, images, depth_mm, msg_id: int, record_dev: int, stream: int, device_images=False):
        """gray images [n_dirs,H,W] u8 + depth [n_dirs,H,W] u16 mm -> record_dev, no synchronisation.  HOST numpy arrays, or
        with device_images=True two device pointers (ints)."""
        if device_images:
            _l.check(self._lib.osb_frontend_extract_depth_dev(self._h, C.c_void_p(images), C.c_void_p(depth_mm), msg_id,
                                                              C.c_void_p(record_dev), C.c_void_p(stream)))
            return
        img, dep = self._depth_inputs(images, depth_mm)
        _l.check(self._lib.osb_frontend_extract_depth(self._h, _l.ptr(img), _l.ptr(dep), msg_id, C.c_void_p(record_dev),
                                                      C.c_void_p(stream)))

    def process_depth(self, images: np.ndarray, depth_mm: np.ndarray, msg_id: int):
        """HOST gray images [n_dirs,H,W] u8 + depth [n_dirs,H,W] u16 mm -> (KeyframeRecord, LoopResult); one synchronisation."""
        img, dep = self._depth_inputs(images, depth_mm)
        rec, res = _l.KeyframeRecord(), _l.LoopResult()
        _l.check(self._lib.osb_frontend_process_depth(self._h, _l.ptr(img), _l.ptr(dep), msg_id, C.byref(rec), C.byref(res)))
        return rec, res

    def process_depth_raw(self, img_ptr: int, depth_ptr: int, msg_id: int, rec_ptr: int, res_ptr: int):
        """same, with raw HOST pointers (pinned buffers owned by the caller)."""
        _l.check(self._lib.osb_frontend_process_depth(self._h, C.c_void_p(img_ptr), C.c_void_p(depth_ptr), msg_id,
                                                      C.c_void_p(rec_ptr), C.c_void_p(res_ptr)))

    def db_size(self, remote=False) -> int:
        return int(self._lib.osb_frontend_db_size(self._h, int(remote)))

    def db_reset(self):
        _l.check(self._lib.osb_frontend_db_reset(self._h))

    def db_load(self, global_desc: np.ndarray, local_desc=None, n_kpts=None, remote=False):
        g = _f32(global_desc)
        ld = None if local_desc is None else _f32(local_desc)
        nk = None if n_kpts is None else np.ascontiguousarray(n_kpts, np.int32)
        _l.check(self._lib.osb_frontend_db_load(self._h, int(remote), g.shape[0], _l.ptr(g), _l.ptr(ld), _l.ptr(nk)))

    def db_set_geometry(self, first_row: int, kpts: np.ndarray, stereo_match: np.ndarray, remote=False):
        """landmarks_2d [n][max_num][2] and stereo_match [n][max_num] of rows put in with db_load"""
        k = _f32(kpts); sm = np.ascontiguousarray(stereo_match, np.int32)
        _l.check(self._lib.osb_frontend_db_set_geometry(self._h, int(remote), first_row, k.shape[0], _l.ptr(k), _l.ptr(sm)))


def stereo_lift(kp_up, kp_down, stereo_match, n_up, n_down, intrinsics, pose_up, pose_down, triangle_thres=0.006,
                accept_min_3d_pts=0):
    """loop_cam.cpp:393-432 for n_dirs directions: kp_* [n_dirs,max_n,2] f32, stereo_match [n_dirs,max_n] i32,
    poses [n_dirs,7] -> (pts3d [n_dirs,max_n,3] f32, flag_up, flag_down [n_dirs,max_n] u8)"""
    lib = _l.load()
    ku, kd = _f32(kp_up), _f32(kp_down)
    nd, mn = ku.shape[0], ku.shape[1]
    sm = np.ascontiguousarray(stereo_match, np.int32)
    nu, ndn = np.ascontiguousarray(n_up, np.int32), np.ascontiguousarray(n_down, np.int32)
    K = np.ascontiguousarray(intrinsics, np.float64)
    pu, pd = np.ascontiguousarray(pose_up, np.float64), np.ascontiguousarray(pose_down, np.float64)
    pts = np.zeros((nd, mn, 3), np.float32); fu = np.zeros((nd, mn), np.uint8); fd = np.zeros((nd, mn), np.uint8)
    _l.check(lib.osb_stereo_lift(_l.ptr(ku), _l.ptr(kd), _l.ptr(sm), _l.ptr(nu), _l.ptr(ndn), nd, mn, _l.ptr(K), _l.ptr(pu),
                                 _l.ptr(pd), float(triangle_thres), int(accept_min_3d_pts), _l.ptr(pts), _l.ptr(fu), _l.ptr(fd)))
    return pts, fu, fd


def depth_lift(kp, n, depth_mm, intrinsics, pose_cam, near=0.3, far=10.0, accept_min_3d_pts=0):
    """loop_cam.cpp:276-302: kp [n_dirs,max_n,2], depth_mm [n_dirs,H,W] u16, pose_cam [n_dirs,7] -> (pts3d, flag)"""
    lib = _l.load()
    k = _f32(kp)
    nd, mn = k.shape[0], k.shape[1]
    nn = np.ascontiguousarray(n, np.int32)
    dep = np.ascontiguousarray(depth_mm, np.uint16)
    K = np.ascontiguousarray(intrinsics, np.float64)
    pc = np.ascontiguousarray(pose_cam, np.float64)
    pts = np.zeros((nd, mn, 3), np.float32); fl = np.zeros((nd, mn), np.uint8)
    _l.check(lib.osb_depth_lift(_l.ptr(k), _l.ptr(nn), nd, mn, _l.ptr(dep), dep.shape[1], dep.shape[2], _l.ptr(K), _l.ptr(pc),
                                float(near), float(far), int(accept_min_3d_pts), _l.ptr(pts), _l.ptr(fl)))
    return pts, fl


def pnp_ransac(cases, max_n: int | None = None):
    """LoopDetector::compute_relative_pose + check_loop_odometry_consistency (loop_detector.cpp:294-413) for a batch of loop
    candidates.  cases: list of dicts with X [n,3], uv [n,2] and the osb_pnp_params fields (prior, extrinsic, drone_pose_now,
    drone_pose_old [7]; iterations, thresh, seed, is_4dof, min_loop_num, rperr_thres, accept_loop_yaw_rad, max_loop_dis;
    optional same_drone, odom_rel [7], cov [6,6], odometry_consistency_threshold) -> list of (mask uint8 [n], PnpResult)."""
    lib = _l.load()
    nc = len(cases)
    if max_n is None:
        max_n = max(1, max(len(c["X"]) for c in cases))
    p3 = np.zeros((nc, max_n, 3), np.float32); p2 = np.zeros((nc, max_n, 2), np.float32)
    n = np.zeros(nc, np.int32)
    prm = (_l.PnpParams * nc)()
    for i, c in enumerate(cases):
        k = len(c["X"]); n[i] = k
        if k:
            p3[i, :k] = c["X"]; p2[i, :k] = c["uv"]
        p = prm[i]
        p.iterations, p.reproj_thresh, p.seed = int(c.get("iterations", 100)), float(c.get("thresh", 3.0)), int(c.get("seed", 0))
        p.is_4dof, p.min_loop_num, p.same_drone = int(c.get("is_4dof", 1)), int(c.get("min_loop_num", 15)), int(c.get("same_drone", 0))
        p.rperr_thres, p.accept_loop_yaw_rad = float(c.get("rperr_thres", 0.1)), float(c.get("accept_loop_yaw_rad", 0.8))
        p.max_loop_dis = float(c.get("max_loop_dis", 5.0))
        p.odometry_consistency_threshold = float(c.get("odometry_consistency_threshold", 10.0))
        for name in ("prior", "extrinsic", "drone_pose_now", "drone_pose_old"):
            getattr(p, name)[:] = [float(x) for x in c[name]]
        p.odom_rel[:] = [float(x) for x in c.get("odom_rel", [0, 0, 0, 1, 0, 0, 0])]
        p.odom_edge_cov[:] = [float(x) for x in np.asarray(c.get("cov", np.eye(6)), np.float64).reshape(-1)]
    mask = np.zeros((nc, max_n), np.uint8)
    res = (_l.PnpResult * nc)()
    _l.check(lib.osb_pnp_ransac(_l.ptr(p3), _l.ptr(p2), _l.ptr(n), nc, max_n, prm, _l.ptr(mask), res))
    return [(mask[i, :n[i]].copy(), res[i]) for i in range(nc)]


def loop_edges(edges):
    """edge dicts (id_a, id_b, rel [7], cov [6,6], odom_a [7], odom_b [7], len_a, len_b) -> osb_loop_edge [n] as a
    float64 array [n, 60] (word 0 holds id_a, id_b as two int32), the bytes the C ABI reads"""
    n = len(edges)
    arr = np.zeros((n, 60), np.float64)
    if n:
        ids = arr.view(np.int32)
        ids[:, 0] = [int(e["id_a"]) for e in edges]
        ids[:, 1] = [int(e["id_b"]) for e in edges]
        arr[:, 1:8] = [e["rel"] for e in edges]
        arr[:, 8:44] = np.asarray([np.asarray(e["cov"], np.float64).reshape(-1) for e in edges])
        arr[:, 44:51] = [e["odom_a"] for e in edges]
        arr[:, 51:58] = [e["odom_b"] for e in edges]
        arr[:, 58] = [float(e["len_a"]) for e in edges]
        arr[:, 59] = [float(e["len_b"]) for e in edges]
    return arr


def pcm_outlier_rejection(edges, pcm_thres: float, odom_pos_cov_per_m: float, odom_ang_cov_per_m: float,
                          want_matrices: bool = False):
    """SwarmLocalOutlierRejection::OutlierRejectionLoopEdgesPCM (swarm_outlier_rejection.cpp:173-297) for the loop edges of
    one drone pair: `edges` = list of dicts (id_a, id_b, rel [7], cov [6,6], odom_a [7], odom_b [7], len_a, len_b) in
    insertion order -> indices of the kept loops in maxCliqueHeu's order (+ adjacency and smd matrices on request)."""
    lib = _l.load()
    n = len(edges)
    arr = loop_edges(edges)
    clique = np.zeros(n, np.int32)
    size = C.c_int32(0)
    adj = np.zeros((n, n), np.uint8) if want_matrices else None
    smd = np.zeros((n, n), np.float64) if want_matrices else None
    _l.check(lib.osb_pcm(_l.ptr(arr), n, float(pcm_thres), float(odom_pos_cov_per_m), float(odom_ang_cov_per_m), _l.ptr(clique),
                         C.byref(size), _l.ptr(adj), _l.ptr(smd)))
    out = clique[:size.value].copy()
    return (out, adj, smd) if want_matrices else out


class PcmState(_Handle):
    """SwarmLocalOutlierRejection (swarm_outlier_rejection.cpp:37-56, 98-297) with its per-drone-pair PCM state resident on
    the device (osb_pcm_state_*): `reject(edges, ids)` is OutlierRejectionLoopEdges -> keep mask of good_loops,
    `inliers(a, b)` what broadcast_good_loops sends, `set_inliers(a, b, ids)` good_ids_handle, `pair(a, b)` the read-out."""

    _destroy = "osb_pcm_state_destroy"

    def __init__(self, self_id: int, redundant: bool, pcm_thres: float, odom_pos_cov_per_m: float,
                 odom_ang_cov_per_m: float, max_pairs: int = 16, pair_capacity: int = 4096):
        self._lib = _l.load()
        self._h = C.c_void_p()
        p = _l.PcmStateParams(int(self_id), int(bool(redundant)), int(max_pairs), int(pair_capacity), float(pcm_thres),
                              float(odom_pos_cov_per_m), float(odom_ang_cov_per_m))
        _l.check(self._lib.osb_pcm_state_create(C.byref(self._h), C.byref(p)))

    def reject(self, edges, ids) -> np.ndarray:
        """edges: edge dicts (as pcm_outlier_rejection) or an already packed loop_edges() array; ids: LoopEdge::id each
        -> keep [n] bool"""
        arr = edges if isinstance(edges, np.ndarray) else loop_edges(edges)
        ids = np.ascontiguousarray(ids, np.int64)
        assert arr.shape == (len(ids), 60)
        keep = np.zeros(len(ids), np.uint8)
        _l.check(self._lib.osb_pcm_state_reject(self._h, _l.ptr(arr), _l.ptr(ids), len(ids), _l.ptr(keep)))
        return keep.astype(bool)

    def inliers(self, a: int, b: int):
        """the pair's inlier ids ascending, or None when it has no set"""
        n = C.c_int32(0)
        _l.check(self._lib.osb_pcm_state_inliers(self._h, a, b, None, 0, C.byref(n)))
        if n.value < 0:
            return None
        out = np.zeros(n.value, np.int64)
        _l.check(self._lib.osb_pcm_state_inliers(self._h, a, b, _l.ptr(out), n.value, C.byref(n)))
        return out

    def set_inliers(self, a: int, b: int, ids):
        ids = np.ascontiguousarray(ids, np.int64)
        _l.check(self._lib.osb_pcm_state_set_inliers(self._h, a, b, _l.ptr(ids), len(ids)))

    def pair(self, a: int, b: int):
        """-> (ids [n] in insertion order, adjacency [n,n] uint8, last clique in maxCliqueHeu order)"""
        n = C.c_int32(0)
        _l.check(self._lib.osb_pcm_state_pair(self._h, a, b, C.byref(n), None, None, None, None))
        ids = np.zeros(n.value, np.int64)
        adj = np.zeros((n.value, n.value), np.uint8)
        clique = np.zeros(n.value, np.int32)
        size = C.c_int32(0)
        _l.check(self._lib.osb_pcm_state_pair(self._h, a, b, C.byref(n), _l.ptr(ids), _l.ptr(adj), _l.ptr(clique),
                                              C.byref(size)))
        return ids, adj, clique[:size.value].copy()

    def reject_anchored(self, rows_ptr: int, n: int, keep_ptr: int, stream: int):
        """reject() over the OK rows of osb_anchor_run_dev's output, read in place on the device: writes keep [n] uint8 at
        keep_ptr on `stream` without synchronising (not written when the call is refused; see status())"""
        _l.check(self._lib.osb_pcm_state_reject_anchored(self._h, C.c_void_p(rows_ptr), int(n), C.c_void_p(keep_ptr),
                                                         C.c_void_p(stream)))

    def status(self) -> int:
        """synchronises with the last reject_anchored call -> its status (lib.OK or lib.ERR_CAPACITY)"""
        last = C.c_int(0)
        st = self._lib.osb_pcm_state_status(self._h, C.byref(last))
        if st not in (_l.OK, last.value):
            _l.check(st)
        return last.value


class LoopAnchor(_Handle):
    """The re-anchoring walk of SwarmLocalizationSolver::find_available_loops_detections (swarm_localization_solver.cpp:
    1594-1666, 1429-1553) with ego_motion_trajs, all_loops / all_detections_6d and sf_sld_win resident on the device
    (osb_anchor_*).  Records are numpy structured arrays of lib.MEASUREMENT_DTYPE / WINDOW_ENTRY_DTYPE; `run` returns one
    lib.ANCHOR_RESULT_DTYPE row per measurement, loops first, each in arrival order."""

    _destroy = "osb_anchor_destroy"

    def __init__(self, max_drones: int, max_traj_samples: int, max_measurements: int, max_window_entries: int,
                 det_dpos_thres: float, odom_pos_cov_per_m: float, odom_ang_cov_per_m: float,
                 begin_min_loop_dt_s: float = 1000.0, huber: bool = True, max_keyframes: int = 256,
                 max_keyframe_distances: int | None = None):
        self._lib = _l.load()
        self._h = C.c_void_p()
        self.max_drones = int(max_drones)
        if max_keyframe_distances is None:                 # every ordered drone pair, up to 4096
            max_keyframe_distances = min(self.max_drones * self.max_drones, 4096)
        p = _l.AnchorParams(self.max_drones, int(max_traj_samples), int(max_measurements), int(max_window_entries),
                            float(begin_min_loop_dt_s), float(det_dpos_thres), float(odom_pos_cov_per_m),
                            float(odom_ang_cov_per_m), int(bool(huber)), int(max_keyframes),
                            int(max_keyframe_distances), 0)
        _l.check(self._lib.osb_anchor_create(C.byref(self._h), C.byref(p)))

    def push_odometry(self, drone: int, stamps_ns, poses):
        """appends samples: stamps int64 ns, strictly increasing; poses [n,7] (x y z, qw qx qy qz)"""
        stamps = np.ascontiguousarray(stamps_ns, np.int64)
        poses = np.ascontiguousarray(poses, np.float64).reshape(len(stamps), 7)
        _l.check(self._lib.osb_anchor_push_odometry(self._h, int(drone), len(stamps), _l.ptr(stamps), _l.ptr(poses)))

    def add_measurements(self, meas):
        meas = np.ascontiguousarray(meas, _l.MEASUREMENT_DTYPE)
        _l.check(self._lib.osb_anchor_add_measurements(self._h, len(meas), _l.ptr(meas)))

    def add_measurements_dev(self, meas_ptr: int, count_ptr: int, max_n: int, loop_outlier_distance_threshold: float,
                             stream: int):
        """add_new_loop_connection / add_new_detection for rows [0, *count_ptr) of lib.MEASUREMENT_DTYPE in device memory
        (osb_anchor_add_measurements_dev), on `stream` without synchronising; a refused call shows in status()"""
        _l.check(self._lib.osb_anchor_add_measurements_dev(self._h, C.c_void_p(meas_ptr), C.c_void_p(count_ptr), int(max_n),
                                                           float(loop_outlier_distance_threshold), C.c_void_p(stream)))

    def status(self) -> int:
        """waits for the last add_measurements_dev -> its status (lib.OK, lib.ERR_INVALID or lib.ERR_CAPACITY)"""
        last = C.c_int(0)
        st = self._lib.osb_anchor_status(self._h, C.byref(last))
        if st not in (_l.OK, last.value):
            _l.check(st)
        return last.value

    def size(self) -> tuple[int, int]:
        """-> (loops, detections) held"""
        a, b = C.c_int32(0), C.c_int32(0)
        _l.check(self._lib.osb_anchor_size(self._h, C.byref(a), C.byref(b)))
        return a.value, b.value

    def set_window(self, frame_stamps_ns, frame_first, entries):
        """frame f: entries[frame_first[f]:frame_first[f+1]], taken at frame_stamps_ns[f]"""
        stamps = np.ascontiguousarray(frame_stamps_ns, np.int64)
        first = np.ascontiguousarray(frame_first, np.int32)
        entries = np.ascontiguousarray(entries, _l.WINDOW_ENTRY_DTYPE)
        assert len(first) == len(stamps) + 1
        _l.check(self._lib.osb_anchor_set_window(self._h, len(stamps), _l.ptr(stamps), _l.ptr(first),
                                                 _l.ptr(entries) if len(entries) else None))

    def _yaw(self, yaw_observable):
        y = np.zeros(self.max_drones, np.uint8)
        if yaw_observable is None:
            y[:] = 1
        else:
            y[:] = np.asarray(yaw_observable, bool)
        return y

    def run(self, yaw_observable=None) -> np.ndarray:
        """yaw_observable [max_drones] (None: every drone) -> results [n] of lib.ANCHOR_RESULT_DTYPE"""
        y = self._yaw(yaw_observable)
        out = np.zeros(sum(self.size()), _l.ANCHOR_RESULT_DTYPE)
        n = C.c_int32(0)
        _l.check(self._lib.osb_anchor_run(self._h, _l.ptr(y), _l.ptr(out) if len(out) else None, C.byref(n)))
        return out[:n.value]

    def run_dev(self, out_ptr: int, stream: int, yaw_observable=None) -> int:
        """writes the results to device memory at out_ptr on `stream` without synchronising -> their count"""
        y = self._yaw(yaw_observable)
        n = C.c_int32(0)
        _l.check(self._lib.osb_anchor_run_dev(self._h, _l.ptr(y), C.c_void_p(out_ptr), C.byref(n), C.c_void_p(stream)))
        return n.value

    def observe_dev(self, rows_ptr: int, n: int, stream: int, self_id: int, init_xy_movement: float,
                    init_z_movement: float):
        """estimate_observability on the device (osb_anchor_observe_dev) from the n rows run_dev wrote at rows_ptr: updates
        the handle's observability state and rewrites each row's skip with this solve's yaw-observable drones, on `stream`
        without synchronising"""
        p = _l.ObserveParams(int(self_id), float(init_xy_movement), float(init_z_movement), 0)
        _l.check(self._lib.osb_anchor_observe_dev(self._h, C.byref(p), C.c_void_p(rows_ptr), int(n), C.c_void_p(stream)))

    def init_mask_dev(self, self_id: int, n_nodes: int, mask_ptr: int, yaw_ptr: int, stream: int):
        """random_init_pose's blocks from the window and the last observe_dev's to_init (osb_anchor_init_mask_dev): uint8
        mask [n_nodes] at mask_ptr and float64 odometry yaw [n_nodes] at yaw_ptr, on `stream` without synchronising"""
        _l.check(self._lib.osb_anchor_init_mask_dev(self._h, int(self_id), int(n_nodes), C.c_void_p(mask_ptr),
                                                    C.c_void_p(yaw_ptr), C.c_void_p(stream)))

    def sync_dev(self, solver: PoseGraphSolver, stream: int, self_id: int, acpt_cost: float, window_size: int,
                 normalise: bool = True, full_path: bool = False):
        """sync_est_poses on the device (osb_anchor_sync_dev): the keyframe paths, the full paths (full_path) and the
        prediction record from the solver's last device call, applied only if solve() would accept that call, on
        `stream` without synchronising"""
        p = _l.SyncParams(int(self_id), int(bool(full_path)), int(bool(normalise)), int(window_size), float(acpt_cost))
        _l.check(self._lib.osb_anchor_sync_dev(self._h, solver._h, C.byref(p), C.c_void_p(stream)))

    def sync_result(self) -> tuple[bool, int]:
        """waits for the last sync_dev -> (applied, status): status lib.ERR_INVALID for a window drone without odometry"""
        applied, last = C.c_int32(0), C.c_int(0)
        _l.check(self._lib.osb_anchor_sync_result(self._h, C.byref(applied), C.byref(last)))
        return bool(applied.value), last.value

    def paths(self, drone: int, full: bool = False):
        """waits for the last sync_dev -> drone's keyframe path (or full path) as (stamps int64 [n], poses [n, 7]), or
        None when the drone has none"""
        n = C.c_int32(0)
        _l.check(self._lib.osb_anchor_paths(self._h, int(full), int(drone), None, None, 0, C.byref(n)))
        if n.value < 0:
            return None
        stamps = np.zeros(n.value, np.int64)
        poses = np.zeros((n.value, 7), np.float64)
        _l.check(self._lib.osb_anchor_paths(self._h, int(full), int(drone), _l.ptr(stamps), _l.ptr(poses), n.value,
                                            C.byref(n)))
        return stamps, poses

    def record_loops_dev(self, rows_ptr: int, n: int, stream: int):
        """the loop map of OutlierRejectionLoopEdges (osb_anchor_record_loops_dev) from the n rows run_dev wrote at
        rows_ptr: every OK row's id the first time it is seen, and each drone pair's smallest id, on `stream` without
        synchronising"""
        _l.check(self._lib.osb_anchor_record_loops_dev(self._h, C.c_void_p(rows_ptr), int(n), C.c_void_p(stream)))

    def init_by_loops_dev(self, pcm: "PcmState", solver: PoseGraphSolver, self_id: int, stream: int):
        """init_pose_by_loops on the device (osb_anchor_init_by_loops_dev): the window blocks of the last observe's
        to_init drones placed from their loops to estimated drones, written into the solver's resident poses on `stream`
        without synchronising; a refusal shows in init_by_loops_result()"""
        _l.check(self._lib.osb_anchor_init_by_loops_dev(self._h, pcm._h, solver._h, int(self_id), C.c_void_p(stream)))

    def init_by_loops_result(self) -> int:
        """waits for the last init_by_loops_dev -> its status (lib.OK, lib.ERR_INVALID or lib.ERR_CAPACITY)"""
        last = C.c_int(0)
        _l.check(self._lib.osb_anchor_init_by_loops_result(self._h, C.byref(last)))
        return last.value

    def loop_map(self) -> dict:
        """waits for the last record_loops_dev and sync_dev -> dict(records: lib.LOOP_RECORD_DTYPE [n] ascending by id,
        pair_min: int64 [max_drones, max_drones] (INT64_MAX: no id), estimated: bool [max_drones])"""
        D = self.max_drones
        n = C.c_int32(0)
        pair = np.zeros((D, D), np.int64)
        est = np.zeros(D, np.uint8)
        _l.check(self._lib.osb_anchor_loop_map(self._h, None, 0, C.byref(n), _l.ptr(pair), _l.ptr(est)))
        recs = np.zeros(n.value, _l.LOOP_RECORD_DTYPE)
        if n.value:
            _l.check(self._lib.osb_anchor_loop_map(self._h, _l.ptr(recs), n.value, C.byref(n), None, None))
        return dict(records=recs, pair_min=pair, estimated=est.astype(bool))

    def set_data_association(self, accept_thres: float = 3.345, anon_min: int = 1000, max_nodes: int = 4096):
        """enables data association (osb_anchor_set_data_association): detections with id_b >= anon_min are accepted
        as anonymous; accept_thres is the reference's float DA_accept_thres; max_nodes bounds each search's DFS calls,
        not its gate evaluations: a call can gate up to n_u x (max_drones - 1) candidates, so a search does up to
        max_nodes x n_u x (max_drones - 1) of them, on one thread at about 7.5 us each (measured on an H100 80GB HBM3
        at 700 W).  At 32 ids and 256 drones that bounds a call by about 61 ms and 4096 calls by about 250 s (a measured
        worst case took about 50 ms a call)"""
        p = _l.DaParams(float(accept_thres), int(anon_min), int(max_nodes), 0)
        _l.check(self._lib.osb_anchor_set_data_association(self._h, C.byref(p)))

    def data_association_dev(self, self_id: int, stream: int):
        """LocalizationDAInit on the device (osb_anchor_data_association_dev): on success the store's anonymous detections
        are renamed in place, on `stream` without synchronising; the outcome shows in data_association_result()"""
        _l.check(self._lib.osb_anchor_data_association_dev(self._h, int(self_id), C.c_void_p(stream)))

    def data_association_result(self) -> tuple[bool, int, dict]:
        """waits for the last data_association_dev -> (applied, status, {anonymous id: drone} of an applied call)"""
        applied, status, n = C.c_int32(0), C.c_int(0), C.c_int32(0)
        pairs = np.zeros((32, 2), np.int32)
        _l.check(self._lib.osb_anchor_data_association_result(self._h, C.byref(applied), C.byref(status), _l.ptr(pairs),
                                                              32, C.byref(n)))
        return bool(applied.value), status.value, {int(a): int(d) for a, d in pairs[:n.value]}

    def data_association_word(self) -> int:
        """the device address of the applied word that run_dev_if / observe_dev_if read"""
        w = C.c_void_p()
        _l.check(self._lib.osb_anchor_data_association_word(self._h, C.byref(w)))
        return int(w.value)

    def run_dev_if(self, out_ptr: int, pred_ptr: int, stream: int, yaw_observable=None) -> int:
        """run_dev predicated on the int32 at pred_ptr, read on the device (0 writes nothing) -> the row count"""
        y = self._yaw(yaw_observable)
        n = C.c_int32(0)
        _l.check(self._lib.osb_anchor_run_dev_if(self._h, _l.ptr(y), C.c_void_p(out_ptr), C.byref(n), C.c_void_p(pred_ptr),
                                                 C.c_void_p(stream)))
        return n.value

    def observe_dev_if(self, rows_ptr: int, n: int, pred_ptr: int, stream: int, self_id: int, init_xy_movement: float,
                       init_z_movement: float):
        """observe_dev predicated on the int32 at pred_ptr (0 writes nothing); a motion_new the record holds is kept"""
        p = _l.ObserveParams(int(self_id), float(init_xy_movement), float(init_z_movement), 0)
        _l.check(self._lib.osb_anchor_observe_dev_if(self._h, C.byref(p), C.c_void_p(rows_ptr), int(n), C.c_void_p(pred_ptr),
                                                     C.c_void_p(stream)))

    def predict(self, drones, vo_poses, self_id: int, finish_init: bool = True) -> dict:
        """PredictSwarm for one frame (osb_anchor_predict): drones [n], their odometry poses [n, 7] now -> {drone:
        (node_pose [7] or None, base_pose [7] or None)}"""
        d = np.ascontiguousarray(drones, np.int32)
        vo = np.ascontiguousarray(vo_poses, np.float64).reshape(len(d), 7)
        out = (_l.PredictResult * max(1, len(d)))()
        p = _l.PredictParams(int(self_id), int(bool(finish_init)))
        _l.check(self._lib.osb_anchor_predict(self._h, C.byref(p), len(d), _l.ptr(d), _l.ptr(vo), C.cast(out, C.c_void_p)))
        return {int(d[i]): (np.array(out[i].node_pose) if out[i].node_valid else None,
                            np.array(out[i].base_pose) if out[i].base_valid else None) for i in range(len(d))}

    def add_keyframe_dev(self, solver: PoseGraphSolver, stamp_ns: int, nodes, dists, stream: int, self_id: int,
                         finish_init: bool, enable_distance: bool = True, outlier_threshold: float = 0.3,
                         elevation_threshold: float = 0.5, minimum_distance: float = 0.2,
                         debug_no_rejection: bool = False, seed: int = 0):
        """add_as_keyframe on the device (osb_anchor_add_keyframe_dev): nodes [n] of lib.KEYFRAME_NODE_DTYPE in
        ascending drone id, dists of lib.KEYFRAME_DISTANCE_DTYPE (each node's n_distances in turn, ascending peer).  Writes
        the new blocks' initial poses into the solver's resident device poses, flags the distances and stores the
        keyframe, on `stream` without synchronising"""
        nodes = np.ascontiguousarray(nodes, _l.KEYFRAME_NODE_DTYPE)
        dists = np.ascontiguousarray(dists, _l.KEYFRAME_DISTANCE_DTYPE)
        p = _l.KeyframeParams(int(self_id), int(bool(finish_init)), int(bool(enable_distance)),
                              int(bool(debug_no_rejection)), float(outlier_threshold), float(elevation_threshold),
                              float(minimum_distance), 0, int(seed) & (2 ** 64 - 1))
        _l.check(self._lib.osb_anchor_add_keyframe_dev(self._h, solver._h, int(stamp_ns), len(nodes), _l.ptr(nodes),
                                                       len(dists), _l.ptr(dists) if len(dists) else None, C.byref(p),
                                                       C.c_void_p(stream)))

    def keyframe_flags(self, stamp_ns: int):
        """waits for the last add_keyframe_dev -> the stored keyframe's outlier flags (int8: 1, 0, -1 not written) in
        its dists order, or None when the stamp is not stored"""
        n = C.c_int32(0)
        _l.check(self._lib.osb_anchor_keyframe_flags(self._h, int(stamp_ns), None, 0, C.byref(n)))
        if n.value < 0:
            return None
        out = np.zeros(n.value, np.int8)
        _l.check(self._lib.osb_anchor_keyframe_flags(self._h, int(stamp_ns), _l.ptr(out) if n.value else None, n.value,
                                                     C.byref(n)))
        return out

    def distance_factors_dev(self, rows: "FactorRows", max_tail: int, stream: int, self_id: int,
                             enable_distance: bool = True, debug_no_rejection: bool = False,
                             distance_measurement_cov: float = 0.2):
        """setup_problem_with_sferror on the device (osb_anchor_distance_factors_dev): the window's distance rows
        appended to `rows` at its count, on `stream` without synchronising; a count past max_tail becomes -1"""
        p = _l.DistanceParams(int(self_id), int(bool(enable_distance)), int(bool(debug_no_rejection)),
                              float(distance_measurement_cov))
        ty, ia, ib, pl, hu, cnt = rows.ptrs()
        _l.check(self._lib.osb_anchor_distance_factors_dev(self._h, C.byref(p), C.c_void_p(ty), C.c_void_p(ia),
                                                           C.c_void_p(ib), C.c_void_p(pl), C.c_void_p(hu),
                                                           C.c_void_p(cnt), int(max_tail), C.c_void_p(stream)))

    def observability(self) -> dict:
        """waits for the last observe_dev -> its outcome: bool arrays [max_drones] nodes, yaw, pos, enable, to_init and
        the flags solve_master, motion, motion_new"""
        o = _l.Observability()
        _l.check(self._lib.osb_anchor_observability(self._h, C.byref(o)))
        out = {k: np.frombuffer(bytes(getattr(o, k)), np.uint8)[:self.max_drones].astype(bool)
               for k in ("nodes", "yaw", "pos", "enable", "to_init")}
        out.update(solve_master=bool(o.solve_master), motion=bool(o.motion), motion_new=bool(o.motion_new))
        return out


def anchored_factor_rows(res: np.ndarray, keep=None):
    """the solver rows of the results with skip == 0 (and keep[i], e.g. the PCM keep mask) -> (ftype, ia, ib, payload,
    huber), the arrays osb_solver_solve takes"""
    sel = res["skip"] == 0
    if keep is not None:
        sel &= np.asarray(keep, bool)
    r = res[sel]
    return (r["factor_type"].astype(np.int32), r["ia"].astype(np.int32), r["ib"].astype(np.int32),
            np.ascontiguousarray(r["payload"]), r["huber"].astype(np.uint8))


def compact_anchored_factors(rows_ptr: int, n: int, keep_ptr, type_ptr: int, ia_ptr: int, ib_ptr: int, payload_ptr: int,
                             huber_ptr: int, count_ptr: int, stream: int):
    """anchored_factor_rows on the device (osb_anchor_compact_factors_dev): the rows with skip == 0 and keep[i] (keep_ptr
    may be None) in row order into device arrays of n rows each -- type / ia / ib int32, payload [n, PAYLOAD_LEN] float64,
    huber uint8 -- and their number into the int32 at count_ptr, on `stream` without synchronising"""
    _l.check(_l.load().osb_anchor_compact_factors_dev(C.c_void_p(rows_ptr), int(n),
                                                      None if keep_ptr is None else C.c_void_p(keep_ptr),
                                                      C.c_void_p(type_ptr), C.c_void_p(ia_ptr), C.c_void_p(ib_ptr),
                                                      C.c_void_p(payload_ptr), C.c_void_p(huber_ptr),
                                                      C.c_void_p(count_ptr), C.c_void_p(stream)))


def anchored_loop_edges(res: np.ndarray) -> np.ndarray:
    """the re-anchored edges as the packed [n, 60] array PcmState.reject takes"""
    return np.ascontiguousarray(res["edge"]).view(np.float64).reshape(len(res), 60)


def anchored_keep(state: PcmState, res: np.ndarray) -> np.ndarray:
    """the keep mask PcmState.reject_anchored writes, on the host: the OK rows through state.reject, scattered back to
    one uint8 per row"""
    ok = res["status"] == _l.ANCHOR_OK
    keep = np.zeros(len(res), np.uint8)
    keep[ok] = state.reject(anchored_loop_edges(res[ok]), res["id"][ok])
    return keep


FACTOR_KEYS = ("ftype", "ia", "ib", "payload", "huber")


class FactorRows:
    """cap solver rows in device memory, laid out as compact_anchored_factors writes them and
    PoseGraphSolver.solve_resident_dev reads them: type / ia / ib int32, payload [cap, PAYLOAD_LEN] float64, huber uint8,
    and their count in one int32.  Host-side rows are dicts of FACTOR_KEYS arrays, in anchored_factor_rows' order."""

    def __init__(self, cap: int):
        import torch
        cap = max(cap, 1)
        self.type, self.ia, self.ib = (torch.zeros(cap, dtype=torch.int32, device="cuda") for _ in range(3))
        self.payload = torch.zeros(cap * _l.PAYLOAD_LEN, dtype=torch.float64, device="cuda")
        self.huber = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        self.count = torch.zeros(1, dtype=torch.int32, device="cuda")

    def ptrs(self) -> tuple:
        """the six device pointers, in the order compact_anchored_factors and solve_resident_dev take them"""
        return tuple(t.data_ptr() for t in (self.type, self.ia, self.ib, self.payload, self.huber, self.count))

    def set(self, rows: dict, count: int | None = None):
        """copies host rows in on the current stream; count: the count stored (default: the number of rows)"""
        import torch
        k = len(rows["ftype"])
        if k:
            self.type[:k] = torch.from_numpy(np.asarray(rows["ftype"], np.int32)).cuda()
            self.ia[:k] = torch.from_numpy(np.asarray(rows["ia"], np.int32)).cuda()
            self.ib[:k] = torch.from_numpy(np.asarray(rows["ib"], np.int32)).cuda()
            self.payload[:k * _l.PAYLOAD_LEN] = torch.from_numpy(np.ascontiguousarray(rows["payload"]).reshape(-1)).cuda()
            self.huber[:k] = torch.from_numpy(np.asarray(rows["huber"], np.uint8)).cuda()
        self.count.fill_(k if count is None else count)

    def on_host(self, stream=None) -> dict:
        """waits for `stream` (a torch stream; None: the current one), the stream that wrote the rows -> the first count
        rows"""
        import torch
        with torch.cuda.stream(stream):
            k = int(self.count.cpu()[0])
            return {"ftype": self.type[:k].cpu().numpy(), "ia": self.ia[:k].cpu().numpy(), "ib": self.ib[:k].cpu().numpy(),
                    "payload": self.payload[:k * _l.PAYLOAD_LEN].cpu().numpy().reshape(k, _l.PAYLOAD_LEN),
                    "huber": self.huber[:k].cpu().numpy()}

    def solve(self, solver: PoseGraphSolver, max_tail: int, options=None, stream=None):
        """solver.solve_resident_dev with these rows as its tail, on `stream` (a torch stream; None: the current one)"""
        import torch
        s = torch.cuda.current_stream() if stream is None else stream
        solver.solve_resident_dev(max_tail, *self.ptrs(), s.cuda_stream, options)


class AnchoredChain:
    """The device buffers of one solve's chain and the stream it runs on: LoopAnchor.run_dev's rows (cap of them),
    PcmState.reject_anchored's keep mask and the FactorRows compact_anchored_factors fills.  Each step is one method;
    calling the chain runs run -> reject -> compact, nothing copied between them."""

    def __init__(self, cap: int, stream=None):
        import torch
        self.rows = torch.zeros(cap * _l.ANCHOR_RESULT_DTYPE.itemsize, dtype=torch.uint8, device="cuda")
        self.keep = torch.zeros(cap, dtype=torch.uint8, device="cuda")
        self.factors = FactorRows(cap)
        self.mask = self.yaw = None                                  # init_mask's buffers, acquired by its first call
        self.stream = torch.cuda.Stream() if stream is None else stream
        self.stream.wait_stream(torch.cuda.current_stream())        # the buffers are zeroed on the current stream

    def upload(self, res: np.ndarray):
        """host rows of lib.ANCHOR_RESULT_DTYPE in place of run's, copied on the current stream, which the chain's stream
        then waits for (so does everything else written there before)"""
        import torch
        self.rows[:len(res) * _l.ANCHOR_RESULT_DTYPE.itemsize].copy_(torch.from_numpy(res.view(np.uint8).copy()))
        self.stream.wait_stream(torch.cuda.current_stream())

    def run(self, anchor: LoopAnchor, yaw_observable=None) -> int:
        return anchor.run_dev(self.rows.data_ptr(), self.stream.cuda_stream, yaw_observable)

    def observe(self, anchor: LoopAnchor, n: int, self_id: int, init_xy_movement: float, init_z_movement: float):
        """the observability of the first n rows, their skip rewritten in place (LoopAnchor.observe_dev)"""
        anchor.observe_dev(self.rows.data_ptr(), n, self.stream.cuda_stream, self_id, init_xy_movement, init_z_movement)

    def reject(self, state: PcmState, n: int):
        state.reject_anchored(self.rows.data_ptr(), n, self.keep.data_ptr(), self.stream.cuda_stream)

    def compact(self, n: int, keep: bool = True):
        """the factor rows of the first n rows, with the keep mask or without it"""
        compact_anchored_factors(self.rows.data_ptr(), n, self.keep.data_ptr() if keep else None, *self.factors.ptrs(),
                                 self.stream.cuda_stream)

    def solve(self, solver: PoseGraphSolver, max_tail: int, options=None):
        self.factors.solve(solver, max_tail, options, self.stream)

    def init_mask(self, anchor: LoopAnchor, self_id: int, n_nodes: int):
        """the init branch's mask and yaw of n_nodes blocks into the chain's buffers (LoopAnchor.init_mask_dev), after
        observe; the buffers are (re)acquired on the current stream when n_nodes outgrows them"""
        import torch
        if self.mask is None or self.mask.numel() < n_nodes:
            self.mask = torch.zeros(n_nodes, dtype=torch.uint8, device="cuda")
            self.yaw = torch.zeros(n_nodes, dtype=torch.float64, device="cuda")
            self.stream.wait_stream(torch.cuda.current_stream())
        anchor.init_mask_dev(self_id, n_nodes, self.mask.data_ptr(), self.yaw.data_ptr(), self.stream.cuda_stream)

    def init_solve(self, solver: PoseGraphSolver, max_tail: int, n_trials: int, seed: int, window_size: int,
                   acpt_cost: float, normalise: bool = True, options=None):
        """the init branch's last step: solver.solve_multistart_resident_dev with the chain's rows as its tail and
        init_mask's mask and yaw, on the chain's stream"""
        solver.solve_multistart_resident_dev(max_tail, *self.factors.ptrs(), self.mask.data_ptr(), self.yaw.data_ptr(),
                                             self.stream.cuda_stream, n_trials, seed, window_size, acpt_cost, normalise,
                                             options)

    def record_loops(self, anchor: LoopAnchor, n: int):
        """the loop map from the first n rows (LoopAnchor.record_loops_dev), after run"""
        anchor.record_loops_dev(self.rows.data_ptr(), n, self.stream.cuda_stream)

    def init_by_loops(self, anchor: LoopAnchor, state: PcmState, solver: PoseGraphSolver, self_id: int, n_nodes: int):
        """the pre-motion init branch's start (LoopAnchor.init_by_loops_dev), after reject and observe; the chain's mask
        and yaw become n_nodes zeros (no block scattered), acquired on the current stream when n_nodes outgrows them"""
        import torch
        if self.mask is None or self.mask.numel() < n_nodes:
            self.mask = torch.zeros(n_nodes, dtype=torch.uint8, device="cuda")
            self.yaw = torch.zeros(n_nodes, dtype=torch.float64, device="cuda")
            self.stream.wait_stream(torch.cuda.current_stream())
        else:
            with torch.cuda.stream(self.stream):
                self.mask.zero_()
        anchor.init_by_loops_dev(state, solver, self_id, self.stream.cuda_stream)

    def data_association(self, anchor: LoopAnchor, self_id: int, init_xy_movement: float, init_z_movement: float) -> int:
        """the DA branch (solve(), :893-916) after the first run -> observe -> record_loops -> reject:
        LoopAnchor.data_association_dev, then run and observe again predicated on its applied word, the same launches
        whatever the outcome -> the row count.  record_loops and reject follow it again, as the reference's second
        estimate_observability runs them (with nothing applied they see the same rows and change nothing)"""
        anchor.data_association_dev(self_id, self.stream.cuda_stream)
        w = anchor.data_association_word()
        n2 = anchor.run_dev_if(self.rows.data_ptr(), w, self.stream.cuda_stream)
        anchor.observe_dev_if(self.rows.data_ptr(), n2, w, self.stream.cuda_stream, self_id, init_xy_movement,
                              init_z_movement)
        return n2

    def distances(self, anchor: LoopAnchor, max_tail: int, self_id: int, **kw):
        """the window's distance rows appended to the chain's rows (LoopAnchor.distance_factors_dev), after compact"""
        anchor.distance_factors_dev(self.factors, max_tail, self.stream.cuda_stream, self_id, **kw)

    def keep_on_host(self, n: int) -> np.ndarray:
        import torch
        with torch.cuda.stream(self.stream):
            return self.keep[:n].cpu().numpy()

    def __call__(self, anchor: LoopAnchor, state: PcmState, yaw_observable=None) -> int:
        """run -> reject -> compact on the chain's stream, without synchronising -> the number of rows"""
        n = self.run(anchor, yaw_observable)
        self.reject(state, n)
        self.compact(n)
        return n


class Swarm(_Handle):
    """The swarm-wide keyframe exchange behind the C ABI (osb_swarm_*): one ncclAllGather of the fixed-size keyframe
    record per round; replaces LoopNet::broadcast_fisheye_desc / image_desc_callback (loop_net.cpp:20-120,142-172).
    `unique_id()` on rank 0, hand the 128 bytes to the other ranks, then `Swarm(id, rank, world)` everywhere."""

    _destroy = "osb_swarm_destroy"

    @staticmethod
    def unique_id() -> bytes:
        buf = (C.c_uint8 * _l.SWARM_ID_BYTES)()
        _l.check(_l.load().osb_swarm_unique_id(buf))
        return bytes(buf)

    def __init__(self, uid: bytes | None, rank: int, world: int):
        self._lib = _l.load()
        self._h = C.c_void_p()
        idbuf = None
        if uid is not None:
            assert len(uid) == _l.SWARM_ID_BYTES
            idbuf = (C.c_uint8 * _l.SWARM_ID_BYTES).from_buffer_copy(uid)
        _l.check(self._lib.osb_swarm_init(C.byref(self._h), idbuf, rank, world))
        self.rank, self.world = rank, world
        self.transport = "p2p copy engines" if self._lib.osb_swarm_transport(self._h) == 1 else "nccl"

    def exchange(self, record_dev: int, gathered_dev: int, stream: int):
        """this rank's record -> gathered[world] in rank order, enqueued on `stream` (osb_swarm_exchange)"""
        _l.check(self._lib.osb_swarm_exchange(self._h, C.c_void_p(record_dev), C.c_void_p(gathered_dev), C.c_void_p(stream)))

    def exchange_async(self, record_dev: int, gathered_dev: int, stream: int):
        """the same on the handle's own stream, behind an event of `stream` (osb_swarm_exchange_async)"""
        _l.check(self._lib.osb_swarm_exchange_async(self._h, C.c_void_p(record_dev), C.c_void_p(gathered_dev), C.c_void_p(stream)))

    def wait(self, stream: int):
        """`stream` waits for the last exchange_async (osb_swarm_wait)"""
        _l.check(self._lib.osb_swarm_wait(self._h, C.c_void_p(stream)))

    def exchange_meta(self, meta_dev: int, gathered_dev: int, stream: int):
        """this drone's KeyframeMeta -> gathered_dev [world] in rank order (osb_swarm_exchange_meta)"""
        _l.check(self._lib.osb_swarm_exchange_meta(self._h, C.c_void_p(meta_dev), C.c_void_p(gathered_dev), C.c_void_p(stream)))


def conv_layer_parity(w, bias, in_hi, in_lo, act_scale: float, *, w_scale: float = 1024.0, relu: int = 0, pool: int = 0,
                      out_c: int | None = None, out_cstride: int | None = None, max_ctas: int = 0, mode: str = "f32",
                      out_scale: float = 1.0):
    """One tensor-core convolution layer (osb_conv_layer_parity).  w [cout,cin,ks,ks], bias [cout] float32 (numpy);
    in_hi / in_lo: CUDA torch.float16 [B,H,W,cin] split planes at act_scale.  Outputs are CUDA tensors pre-filled with NaN,
    so anything the kernel did not write stays NaN:  mode "f32" -> [B,Ho,Wo,out_cstride] float32; "planes" -> (hi, lo)
    [B,Ho,Wo,out_cstride] float16 at out_scale; "softmax" (the 65-logit detector head) -> heat map [B,8H,8W] float32."""
    import torch
    w, b = _f32(w), _f32(bias)
    cout, cin, ks = w.shape[0], w.shape[1], w.shape[2]
    B, H, W, c = in_hi.shape
    assert c == cin and in_hi.dtype == torch.float16 and in_lo.shape == in_hi.shape and in_hi.is_contiguous() \
        and in_lo.is_contiguous()
    n_pad = 64 if cout <= 64 else 80 if cout <= 80 else 128 if cout <= 128 else 256 if cout <= 256 else 512
    out_c = n_pad if out_c is None else out_c
    out_cstride = out_c if out_cstride is None else out_cstride
    Ho, Wo = (H // 2, W // 2) if pool else (H, W)
    dev = in_hi.device
    f32 = hi = lo = None
    if mode == "softmax":
        f32 = torch.full((B, 8 * H, 8 * W), float("nan"), dtype=torch.float32, device=dev)
    elif mode == "f32":
        f32 = torch.full((B, Ho, Wo, out_cstride), float("nan"), dtype=torch.float32, device=dev)
    else:
        hi = torch.full((B, Ho, Wo, out_cstride), float("nan"), dtype=torch.float16, device=dev)
        lo = torch.full_like(hi, float("nan"))
    code = {"f32": 0, "planes": 1, "softmax": 2}[mode]
    dp = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    _l.check(_l.load().osb_conv_layer_parity(
        _l.ptr(w), _l.ptr(b), cin, cout, ks, float(w_scale), dp(in_hi), dp(in_lo), B, H, W, float(act_scale), int(relu),
        int(pool), out_c, out_cstride, int(max_ctas), code, dp(f32), dp(hi), dp(lo), float(out_scale),
        C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)))
    return (hi, lo) if mode == "planes" else f32


def conv_first_parity(w1a, b1a, images, act_scale: float):
    """SuperPoint's first layer (osb_conv_first_parity): images CUDA torch.uint8 [B,H,W] -> conv1a + ReLU as (hi, lo)
    float16 planes [B,H,W,64] at act_scale."""
    import torch
    B, H, W = images.shape
    hi = torch.full((B, H, W, 64), float("nan"), dtype=torch.float16, device=images.device)
    lo = torch.full_like(hi, float("nan"))
    w1a, b1a = _f32(w1a), _f32(b1a)
    _l.check(_l.load().osb_conv_first_parity(
        _l.ptr(w1a), _l.ptr(b1a), C.c_void_p(images.data_ptr()), B, H, W, float(act_scale), C.c_void_p(hi.data_ptr()),
        C.c_void_p(lo.data_ptr()), C.c_void_p(torch.cuda.current_stream(images.device).cuda_stream)))
    return hi, lo


def dwconv_parity(w, bias, x, out_scale: float, *, stride: int = 1, generic: bool = False):
    """Depthwise 3x3 + bias + ReLU6 into split planes (osb_dwconv_parity): w [C,1,3,3], x CUDA float32 [B,H,W,C] ->
    (hi, lo) float16 [B,H/stride,W/stride,C] at out_scale; generic=True runs the one-pixel kernel at stride 1."""
    import torch
    B, H, W, Cn = x.shape
    hi = torch.full((B, H // stride, W // stride, Cn), float("nan"), dtype=torch.float16, device=x.device)
    lo = torch.full_like(hi, float("nan"))
    w, b = _f32(w), _f32(bias)
    _l.check(_l.load().osb_dwconv_parity(
        _l.ptr(w), _l.ptr(b), C.c_void_p(x.data_ptr()), B, H, W, Cn, int(stride), int(generic), float(out_scale),
        C.c_void_p(hi.data_ptr()), C.c_void_p(lo.data_ptr()), C.c_void_p(torch.cuda.current_stream(x.device).cuda_stream)))
    return hi, lo


def conv_layer_fp16_parity(w, bias, in_hi, act_scale: float, *, w_scale: float = 1024.0, relu: int = 0, pool: int = 0,
                           out_c: int | None = None, out_cstride: int | None = None, max_ctas: int = 0, mode: str = "f32",
                           out_scale: float = 1.0):
    """conv_layer_parity in plain fp16 (osb_conv_layer_fp16_parity): one input plane in_hi = fp16(act_scale * x); mode
    "planes" returns the one output plane [B,Ho,Wo,out_cstride] float16, "f32" / "softmax" as conv_layer_parity."""
    import torch
    w, b = _f32(w), _f32(bias)
    cout, cin, ks = w.shape[0], w.shape[1], w.shape[2]
    B, H, W, c = in_hi.shape
    assert c == cin and in_hi.dtype == torch.float16 and in_hi.is_contiguous()
    n_pad = 64 if cout <= 64 else 80 if cout <= 80 else 128 if cout <= 128 else 256 if cout <= 256 else 512
    out_c = n_pad if out_c is None else out_c
    out_cstride = out_c if out_cstride is None else out_cstride
    Ho, Wo = (H // 2, W // 2) if pool else (H, W)
    dev = in_hi.device
    f32 = hi = None
    if mode == "softmax":
        f32 = torch.full((B, 8 * H, 8 * W), float("nan"), dtype=torch.float32, device=dev)
    elif mode == "f32":
        f32 = torch.full((B, Ho, Wo, out_cstride), float("nan"), dtype=torch.float32, device=dev)
    else:
        hi = torch.full((B, Ho, Wo, out_cstride), float("nan"), dtype=torch.float16, device=dev)
    code = {"f32": 0, "planes": 1, "softmax": 2}[mode]
    dp = lambda t: None if t is None else C.c_void_p(t.data_ptr())
    _l.check(_l.load().osb_conv_layer_fp16_parity(
        _l.ptr(w), _l.ptr(b), cin, cout, ks, float(w_scale), dp(in_hi), B, H, W, float(act_scale), int(relu), int(pool),
        out_c, out_cstride, int(max_ctas), code, dp(f32), dp(hi), float(out_scale), _stream(dev)))
    return hi if mode == "planes" else f32


def conv_first_fp16_parity(w1a, b1a, images, act_scale: float):
    """conv_first_parity in plain fp16 (osb_conv_first_fp16_parity): -> the hi plane [B,H,W,64] float16 only."""
    import torch
    B, H, W = images.shape
    hi = torch.full((B, H, W, 64), float("nan"), dtype=torch.float16, device=images.device)
    _l.check(_l.load().osb_conv_first_fp16_parity(_l.ptr(_f32(w1a)), _l.ptr(_f32(b1a)), C.c_void_p(images.data_ptr()), B,
                                                  H, W, float(act_scale), C.c_void_p(hi.data_ptr()), _stream(images.device)))
    return hi


def dwconv_fp16_parity(w, bias, x, out_scale: float, *, stride: int = 1, generic: bool = False):
    """dwconv_parity in plain fp16 (osb_dwconv_fp16_parity): -> the hi plane [B,H/stride,W/stride,C] float16 only."""
    import torch
    B, H, W, Cn = x.shape
    hi = torch.full((B, H // stride, W // stride, Cn), float("nan"), dtype=torch.float16, device=x.device)
    _l.check(_l.load().osb_dwconv_fp16_parity(_l.ptr(_f32(w)), _l.ptr(_f32(bias)), C.c_void_p(x.data_ptr()), B, H, W, Cn,
                                              int(stride), int(generic), float(out_scale), C.c_void_p(hi.data_ptr()),
                                              _stream(x.device)))
    return hi


_GUARD = 64          # floats after an fp32 hook output, pre-filled with NaN like the output: a store past the end shows


def _nan_out(shape, dev):
    """a NaN-filled CUDA float32 tensor of `shape` followed by _GUARD NaN floats: (view, guard)"""
    import torch
    n = int(np.prod(shape))
    buf = torch.full((n + _GUARD,), float("nan"), dtype=torch.float32, device=dev)
    return buf[:n].view(shape), buf[n:]


def _stream(dev):
    import torch
    return C.c_void_p(torch.cuda.current_stream(dev).cuda_stream)


def conv_ffma_parity(w, bias, x, *, act: int = 0, out_cstride: int | None = None, guard: bool = False):
    """One fp32 CUDA-core convolution (osb_conv_ffma_parity): w [cout,cin,ks,ks], bias [cout] float32 (numpy); x CUDA
    float32 [B,H,W,cin] -> [B,H,W,out_cstride] float32, pre-filled with NaN (guard=True also returns the NaN-filled
    floats behind it)."""
    w, b = _f32(w), _f32(bias)
    cout, cin, ks = w.shape[0], w.shape[1], w.shape[2]
    B, H, W, c = x.shape
    assert c == cin and x.is_contiguous()
    out_cstride = cout if out_cstride is None else out_cstride
    y, g = _nan_out((B, H, W, out_cstride), x.device)
    _l.check(_l.load().osb_conv_ffma_parity(_l.ptr(w), _l.ptr(b), cin, cout, ks, C.c_void_p(x.data_ptr()), B, H, W,
                                            int(act), out_cstride, C.c_void_p(y.data_ptr()), _stream(x.device)))
    return (y, g) if guard else y


def conv_first_ffma_parity(w, bias, images, *, stride: int, act: int):
    """The fp32 first layer (osb_conv_first_ffma_parity): w [cout,1,3,3] (cout 32 or 64), images CUDA torch.uint8 [B,H,W]
    -> [B,H/stride,W/stride,cout] float32."""
    w, b = _f32(w), _f32(bias)
    B, H, W = images.shape
    cout = w.shape[0]
    y, _ = _nan_out((B, H // stride, W // stride, cout), images.device)
    _l.check(_l.load().osb_conv_first_ffma_parity(_l.ptr(w), _l.ptr(b), cout, int(stride), int(act),
                                                  C.c_void_p(images.data_ptr()), B, H, W, C.c_void_p(y.data_ptr()),
                                                  _stream(images.device)))
    return y


def dwconv_ffma_parity(w, bias, x, *, stride: int = 1, act: int = 2):
    """fp32 depthwise 3x3 (osb_dwconv_ffma_parity): w [C,1,3,3], x CUDA float32 [B,H,W,C] -> [B,H/s,W/s,C] float32."""
    w, b = _f32(w), _f32(bias)
    B, H, W, Cn = x.shape
    y, _ = _nan_out((B, H // stride, W // stride, Cn), x.device)
    _l.check(_l.load().osb_dwconv_ffma_parity(_l.ptr(w), _l.ptr(b), C.c_void_p(x.data_ptr()), B, H, W, Cn, int(stride),
                                              int(act), C.c_void_p(y.data_ptr()), _stream(x.device)))
    return y


def maxpool_parity(x):
    """2x2 max-pool (osb_maxpool_parity): x CUDA float32 [B,H,W,C] -> [B,H/2,W/2,C] float32."""
    B, H, W, Cn = x.shape
    y, _ = _nan_out((B, H // 2, W // 2, Cn), x.device)
    _l.check(_l.load().osb_maxpool_parity(C.c_void_p(x.data_ptr()), B, H, W, Cn, C.c_void_p(y.data_ptr()),
                                          _stream(x.device)))
    return y


def nv_block0_parity(dw_w, dw_b, pw_w, pw_b, x):
    """NetVLAD block 0 as the default path runs it, one fused kernel (osb_nv_block0_parity): dw_w [32,1,3,3], pw_w
    [64,32,1,1]; x CUDA float32 [B,H,W,32] -> [B,H,W,64] float32."""
    B, H, W, c = x.shape
    assert c == 32 and x.is_contiguous()
    y, _ = _nan_out((B, H, W, 64), x.device)
    _l.check(_l.load().osb_nv_block0_parity(_l.ptr(_f32(dw_w)), _l.ptr(_f32(dw_b)), _l.ptr(_f32(pw_w)), _l.ptr(_f32(pw_b)),
                                            C.c_void_p(x.data_ptr()), B, H, W, C.c_void_p(y.data_ptr()),
                                            _stream(x.device)))
    return y


def nv_head_parity(assign_w, assign_b, centroids, x):
    """The NetVLAD head (osb_nv_head_parity) on projected features x CUDA float32 [B,h,w,128] -> dict of CUDA float32
    tensors: mu [B,128], xn [B,h,w,128] (centred, L2-normalised), logits and assign [B,h,w,32], out [B,4096]."""
    B, h, w, c = x.shape
    assert c == 128 and x.is_contiguous()
    r = {"mu": _nan_out((B, 128), x.device)[0], "xn": _nan_out((B, h, w, 128), x.device)[0],
         "logits": _nan_out((B, h, w, 32), x.device)[0], "assign": _nan_out((B, h, w, 32), x.device)[0],
         "out": _nan_out((B, 4096), x.device)[0]}
    _l.check(_l.load().osb_nv_head_parity(
        _l.ptr(_f32(assign_w)), _l.ptr(_f32(assign_b)), _l.ptr(_f32(centroids)), C.c_void_p(x.data_ptr()), B, h, w,
        *(C.c_void_p(r[k].data_ptr()) for k in ("mu", "xn", "logits", "assign", "out")), _stream(x.device)))
    return r


def launch_count() -> int:
    return int(_l.load().osb_launch_count())


def live_resources() -> int:
    """device buffers, pinned buffers, streams and events the library holds right now (osb_live_resources)"""
    return int(_l.load().osb_live_resources())
