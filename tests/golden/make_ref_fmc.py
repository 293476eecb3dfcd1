"""Golden vectors from the reference's own max-clique finder (FMC::maxCliqueHeu, plain C++ in the reference tree, compiled
from its sources in place by oracle/ref_build/Makefile into oracle/_ref/libfmc_ref.so): the clique it returns, vertex by
vertex, for

  * the random and PCM-shaped graphs of tests/test_oracle_pins.py::test_max_clique_restatement_equals_the_references_own_library
    (regenerated there from the same seed), and
  * the consistency graphs of tests/test_gpu_pcm.py (oracle/pcm_ref.py's consistency matrix of the seeded loop edges),

so that both tests keep comparing with the reference where the reference tree is absent.

    python tests/golden/make_ref_fmc.py        (needs the reference tree to build the library; writes tests/golden/ref_fmc.npz)
"""
import os
import sys
from multiprocessing import Pool

import numpy as np

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT)

from omniswarm_b200 import synth  # noqa: E402
from oracle import fmc_ref, pcm_ref as pr  # noqa: E402

THRES, POS, ANG = 15.0, 1e-4, 1e-5
PCM_CASES = [(60, 0.3, 0, 3), (150, 0.5, 1, 3), (33, 0.0, 2, 3), (1, 0.0, 3, 0)]   # (n, outlier fraction, seed, other_pair)
PCM_LARGE = (1500, 0.4, 5)


def pin_graphs():
    """the graphs of test_max_clique_restatement_equals_the_references_own_library, in its order"""
    rng = np.random.default_rng(1)
    graphs = [np.zeros((1, 1), np.uint8), np.zeros((7, 7), np.uint8), (1 - np.eye(9, dtype=np.uint8))]
    for _ in range(400):
        n = int(rng.integers(2, 60))
        a = np.triu(rng.uniform(size=(n, n)) < rng.uniform(0.02, 0.95), 1)
        graphs.append((a | a.T).astype(np.uint8))
    for _ in range(20):                       # PCM-shaped graphs: a big consistent block plus scattered false links
        n = int(rng.integers(30, 120)); k = int(0.5 * n)
        a = np.zeros((n, n), bool)
        idx = rng.choice(n, k, replace=False)
        a[np.ix_(idx, idx)] = True
        a |= np.triu(rng.uniform(size=(n, n)) < 0.05, 1); a = np.triu(a, 1); a = a | a.T
        graphs.append(a.astype(np.uint8))
    return graphs


def pack(cliques):
    """list of vertex lists -> (concatenated vertices, offsets)"""
    offs = np.zeros(len(cliques) + 1, np.int64)
    offs[1:] = np.cumsum([len(c) for c in cliques])
    return np.array([v for c in cliques for v in c], np.int32), offs


_EDGES = None


def _row(i):
    return i, [(j, pr.pair_smd(_EDGES[i], _EDGES[j], POS, ANG)) for j in range(i)]


def main():
    global _EDGES
    assert fmc_ref.build(), "oracle/_ref/libfmc_ref.so could not be built (is the reference tree present?)"
    out = {}
    pin = [fmc_ref.max_clique_heu(a) for a in pin_graphs()]
    out["pin_verts"], out["pin_offs"] = pack([c for c, _ in pin])
    out["pin_sizes"] = np.array([s for _, s in pin], np.int32)
    pcm = []
    for n, frac, seed, other in PCM_CASES:
        adj, _ = pr.consistency_matrix(synth.pcm_edges(n, frac, seed, other_pair=other), THRES, POS, ANG)
        pcm.append(fmc_ref.max_clique_heu(adj)[0])
    n, frac, seed = PCM_LARGE
    _EDGES = synth.pcm_edges(n, frac, seed)
    adj = np.zeros((n, n), np.uint8)
    with Pool() as p:                          # the oracle's pairwise loop, row by row in parallel (fork: workers see _EDGES)
        for i, row in p.imap_unordered(_row, range(n), chunksize=8):
            for j, s in row:
                if s is not None and s < THRES:
                    adj[i, j] = adj[j, i] = 1
    pcm.append(fmc_ref.max_clique_heu(adj)[0])
    out["pcm_verts"], out["pcm_offs"] = pack(pcm)
    np.savez_compressed(os.path.join(HERE, "ref_fmc.npz"), **out)


if __name__ == "__main__":
    main()
