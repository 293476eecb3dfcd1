"""Oracle of the keyframe databases' fp16 row storage (OSB_DB_STORAGE_FP16).

An fp16 store holds every global-descriptor element rounded to the nearest fp16 (ties to even, overflow to +-inf): numpy's
astype(np.float16), the rule of CUDA's __float2half_rn.  Queries stay fp32 and a score is the inner product with the
rounded row converted exactly back to fp32, so the fp16 forms below are frontend_ref's IndexFlatIP and LoopDetectorDB fed
the rounded rows.
"""
from __future__ import annotations

import numpy as np

from . import frontend_ref as fr


def round_rows_fp16(x: np.ndarray) -> np.ndarray:
    """fp32 rows -> the fp32 values an fp16 store holds for them"""
    with np.errstate(over="ignore"):
        return np.asarray(x, np.float32).astype(np.float16).astype(np.float32)


def fp16_score_bound(q: np.ndarray, x: np.ndarray) -> float:
    """largest change of <q, x> when x is rounded to fp16: each element moves by at most 2^-11 |x_i| (normal range) or
    2^-25 (half the spacing of fp16 subnormals), so |d| <= 2^-11 sum|q_i x_i| + 2^-25 sum|q_i|"""
    q, x = np.abs(np.asarray(q, np.float64)), np.abs(np.asarray(x, np.float64))
    return float(2.0 ** -11 * (q * x).sum() + 2.0 ** -25 * q.sum())


class IndexFlatIPFP16(fr.IndexFlatIP):
    """IndexFlatIP of an fp16 store: rows are rounded when added"""

    def add(self, x: np.ndarray):
        super().add(round_rows_fp16(np.asarray(x, np.float32).reshape(-1, self.d)))


class LoopDetectorDBFP16(fr.LoopDetectorDB):
    """LoopDetectorDB whose two databases are fp16 stores"""

    def __init__(self, self_id: int, dim: int = 4096, **kw):
        super().__init__(self_id, dim, **kw)
        self.local_index = IndexFlatIPFP16(dim)
        self.remote_index = IndexFlatIPFP16(dim)
