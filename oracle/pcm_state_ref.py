"""ORACLE (test infrastructure, NOT product code) -- CPU restatement of SwarmLocalOutlierRejection's persistent PCM state,
the reference of osb_pcm_state_* (SURVEY.md section 8f-2).

Follows (paths relative to /root/reference), swarm_localization/src/swarm_outlier_rejection/swarm_outlier_rejection.cpp:
  * OutlierRejectionLoopEdges (:98-167): a loop whose id is in all_loops_set is skipped (:106-107); the others are grouped
    per drone pair in call order (:108-111); with `redundant` every pair runs the PCM, otherwise only the pairs that contain
    self_id (:122-139); good_loops keeps a loop when its pair has no inlier set or its id is in the set (:141-157);
  * OutlierRejectionLoopEdgesPCM (:173-297): every new loop of a pair is checked against every loop stored before it
    (edge1 = the new one), appended to all_loops and put into all_loops_set (:271-272); maxCliqueHeu then runs on the
    pair's whole graph and the clique's ids replace the pair's inlier set (:277-297);
  * good_ids_handle (:37-56): another drone's set replaces the pair's, unless the pair contains self_id (:40-43).  The
    reference inserts the indices 0..inlier_id_size-1 there (:51-53); this restatement takes the ids the adapter passes.
The reference keys its maps by ordered (a, b) and writes both orders; one unordered pair (lo, hi) here is the same state.
Incremental like the reference: a call computes only the new rows of each pair's consistency matrix, built on
oracle/pcm_ref.py's pair_smd and max_clique_heu.
"""
from __future__ import annotations

import numpy as np

from oracle import pcm_ref


class PcmStateRef:
    def __init__(self, self_id, redundant, pcm_thres, pos_cov_per_m, ang_cov_per_m):
        self.self_id, self.redundant = int(self_id), bool(redundant)
        self.thres, self.pos, self.ang = float(pcm_thres), float(pos_cov_per_m), float(ang_cov_per_m)
        self.pairs = {}          # (lo, hi) -> {"edges": [...], "ids": [...], "adj": uint8 [n, n], "clique": [...]}
        self.seen = set()        # all_loops_set
        self.good = {}           # good_loops_set, (lo, hi) -> set of ids
        self.min_margin = np.inf  # smallest |smd - pcm_thres| of every pair check so far

    @staticmethod
    def key(a, b):
        return (min(int(a), int(b)), max(int(a), int(b)))

    def routed(self, k):
        return self.redundant or self.self_id in k

    def reject(self, edges, ids):
        """-> keep [n] bool: edge i is in the returned good_loops"""
        fresh = {}
        for e, i in zip(edges, ids):                                 # :106-120
            i = int(i)
            if i in self.seen:
                continue
            k = self.key(e["id_a"], e["id_b"])
            if self.routed(k):                                       # :122-139
                fresh.setdefault(k, []).append((e, i))
        for k, new in fresh.items():
            self._pcm(k, new)
        keep = np.zeros(len(ids), bool)
        for t, (e, i) in enumerate(zip(edges, ids)):                 # :141-157
            g = self.good.get(self.key(e["id_a"], e["id_b"]))
            keep[t] = g is None or int(i) in g
        return keep

    def _pcm(self, k, new):
        """OutlierRejectionLoopEdgesPCM (:173-297) for the pair k and its new loops in call order"""
        p = self.pairs.setdefault(k, {"edges": [], "ids": [], "adj": np.zeros((0, 0), np.uint8), "clique": []})
        m, n = len(p["edges"]), len(p["edges"]) + len(new)
        adj = np.zeros((n, n), np.uint8)
        adj[:m, :m] = p["adj"]
        for r, (e, i) in enumerate(new):
            row = m + r
            for j in range(row):                                     # against everything stored before it (:191)
                s = pcm_ref.pair_smd(e, p["edges"][j], self.pos, self.ang)
                if s is None:
                    continue
                self.min_margin = min(self.min_margin, abs(s - self.thres))
                if s < self.thres:
                    adj[row, j] = adj[j, row] = 1
            p["edges"].append(e)
            p["ids"].append(i)
        p["adj"] = adj
        clique, _ = pcm_ref.max_clique_heu(adj)
        p["clique"] = list(clique)
        self.good[k] = {p["ids"][c] for c in clique}
        self.seen.update(i for _, i in new)

    def inliers(self, a, b):
        """good_loops_set[a][b] ascending (broadcast_good_loops), None when the pair has none"""
        g = self.good.get(self.key(a, b))
        return None if g is None else sorted(g)

    def set_inliers(self, a, b, ids):
        """good_ids_handle (:37-56)"""
        if int(a) == self.self_id or int(b) == self.self_id:
            return
        self.good[self.key(a, b)] = {int(i) for i in ids}

    def pair(self, a, b):
        """-> (ids in insertion order, adjacency, last clique), or None for a pair never stored"""
        p = self.pairs.get(self.key(a, b))
        if p is None:
            return None
        return list(p["ids"]), p["adj"], list(p["clique"])
