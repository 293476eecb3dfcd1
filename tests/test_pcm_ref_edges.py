"""CPU: the references of tests/test_gpu_pcm_edges.py checked against each other, and shown to fail.

  * oracle/pcm_ref.consistency_matrix_batched equals the literal consistency_matrix (adjacency identical, smd to 1e-15);
  * the float64 oracle lies within the derived bound of the 50-digit pair error on every case family;
  * each listed defect of the pair error exceeds the bound on at least one pair of the families, and each listed defect of
    maxCliqueHeu changes the clique of at least one graph of the graph families, so the GPU checks can tell them apart;
  * the boolean-row maxCliqueHeu the GPU tests use equals the literal restatement and the reference library's stored
    answers (tests/golden/ref_fmc.npz, ref_fmc_edges.npz)."""
import math
import os
import sys

import numpy as np
import pytest

from conftest import GOLDEN
from omniswarm_b200 import synth
from oracle import pcm_ref as pr

import pcm_edges_ref as R

THRES, POS, ANG = 15.0, 1e-4, 1e-5


@pytest.fixture(scope="module")
def families():
    out = {}
    for name in R.FAMILIES:
        edges, pos, ang = R.family(name, 11)
        out[name] = (edges, pos, ang, R.mp_matrix(edges, pos, ang))
    return out


@pytest.mark.parametrize("case", [(60, 0.3, 0, 3), (150, 0.5, 1, 3), (33, 0.0, 2, 3), (1, 0.0, 3, 0), (2, 0.0, 4, 1)])
def test_batched_consistency_matrix_equals_the_literal_one(case):
    n, frac, seed, other = case
    edges = synth.pcm_edges(n, frac, seed, other_pair=other)
    adj, smd = pr.consistency_matrix(edges, THRES, POS, ANG)
    adj_b, smd_b = pr.consistency_matrix_batched(edges, THRES, POS, ANG, pairs_per_chunk=257)
    fin = np.isfinite(smd)
    assert np.array_equal(adj, adj_b) and np.array_equal(fin, np.isfinite(smd_b))
    assert np.all(np.abs(smd_b[fin] - smd[fin]) <= 1e-15 * np.abs(smd[fin]))


@pytest.mark.parametrize("name", R.FAMILIES)
def test_batched_form_on_the_families(families, name):
    edges, pos, ang, _ = families[name]
    adj, smd = pr.consistency_matrix(edges, THRES, pos, ang)
    adj_b, smd_b = pr.consistency_matrix_batched(edges, THRES, pos, ang)
    fin = np.isfinite(smd)
    assert np.array_equal(adj, adj_b) and np.array_equal(fin, np.isfinite(smd_b))
    assert np.all(np.abs(smd_b[fin] - smd[fin]) <= 1e-12 * np.abs(smd[fin]))


@pytest.mark.parametrize("name", R.FAMILIES)
def test_float64_oracle_within_the_bound_of_the_exact_value(families, name):
    edges, pos, ang, ref = families[name]
    s64, b64 = R.batched_bound(pr.edge_arrays(edges), *R.all_pairs(len(edges)), pos, ang)
    for k, ((i, j), (vals, b)) in enumerate(sorted(ref.items(), key=lambda kv: (kv[0][0], kv[0][1]))):
        s = pr.pair_smd(edges[i], edges[j], pos, ang)
        s = math.inf if s is None else s
        assert R.within(s, vals, b), (name, i, j, s, vals, b)
    I, J = R.all_pairs(len(edges))
    for k in range(len(I)):                                        # the cheap batched bound never undercuts the exact one
        vals, b = ref[(int(I[k]), int(J[k]))]
        if math.isfinite(vals[0]):
            assert b64[k] >= 0.99 * b


def test_theta_family_has_undetermined_branches(families):
    assert any(len(v) == 2 for v, _ in families["theta"][3].values())


@pytest.mark.parametrize("defect", R.DEFECTS)
def test_each_pair_error_defect_exceeds_the_bound(families, defect):
    caught = []
    for name, (edges, pos, ang, ref) in families.items():
        for (i, j), (vals, b) in ref.items():
            if not math.isfinite(vals[0]):
                continue
            with np.errstate(all="ignore"):
                d = R.pair_smd_defect(edges[i], edges[j], pos, ang, defect)
            if not R.within(d, vals, b):
                caught.append(name)
                break
    assert caught, f"{defect} stays within the bound on every case"


def test_the_unmodified_pair_error_is_not_flagged(families):
    for name, (edges, pos, ang, ref) in families.items():
        for (i, j), (vals, b) in ref.items():
            with np.errstate(all="ignore"):
                d = R.pair_smd_defect(edges[i], edges[j], pos, ang, None)
            assert R.within(d, vals, b), (name, i, j)


SMALL_GRAPHS = [(nm, a) for nm, a in R.graph_families() if a.shape[0] <= 1300]


@pytest.mark.parametrize("defect", R.CLIQUE_DEFECTS)
def test_each_clique_defect_changes_a_graph_family_answer(defect):
    assert any(R.max_clique_heu_rows(a, defect) != R.max_clique_heu_rows(a) for _, a in SMALL_GRAPHS), defect


def test_row_clique_equals_the_literal_restatement_and_the_library():
    sys.path.insert(0, GOLDEN)
    import make_ref_fmc as M
    z = np.load(os.path.join(GOLDEN, "ref_fmc.npz"))
    for k, a in enumerate(M.pin_graphs()):
        got = R.max_clique_heu_rows(a)
        assert got == pr.max_clique_heu(a)
        assert got[0] == z["pin_verts"][z["pin_offs"][k]:z["pin_offs"][k + 1]].tolist()
    e = np.load(os.path.join(GOLDEN, "ref_fmc_edges.npz"))
    names = [str(x) for x in e["names"]]
    for nm, a in SMALL_GRAPHS:
        k = names.index(nm)
        assert R.max_clique_heu_rows(a)[0] == e["verts"][e["offs"][k]:e["offs"][k + 1]].tolist(), nm
        if a.shape[0] <= 80:
            assert R.max_clique_heu_rows(a) == pr.max_clique_heu(a), nm


def test_pack_bits_layout():
    a = np.zeros((40, 40), np.uint8)
    a[0, 33] = a[33, 0] = a[1, 31] = a[31, 1] = 1
    b = R.pack_bits(a, 4)
    assert b.shape == (40, 4) and b[0, 1] == 2 and b[33, 0] == 1 and b[1, 0] == 1 << 31 and b[31, 0] == 2
