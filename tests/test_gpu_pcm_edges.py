"""GPU: the PCM consistency error and maxCliqueHeu at their numerical edges and on every launch shape.

  * every device smd of the case families of tests/pcm_edges_ref.py within the derived forward-error bound of the 50-digit
    pair error, the finite / non-finite pattern equal, the adjacency bit-exact (each family's threshold clears every
    pair by more than the bound), and the threshold strict at the device's own value;
  * osb_pcm at every launch shape (the consistency grid's last partial block, the last partial word, each lane's second,
    third and fourth bitset word, both sides of the 200 KiB shared-memory bound, capacity) against the full float64 matrix;
  * pcm_max_clique_kernel in each of its three launch forms (osb_pcm_clique_parity) on the pin graphs and the graph
    families, against the reference library's answers (tests/golden/ref_fmc.npz, ref_fmc_edges.npz);
  * the state's grow kernel at word and shared-memory boundaries against float64."""
import math
import os

import numpy as np
import pytest

from conftest import GOLDEN
from omniswarm_b200 import host, synth, lib as _l
from oracle import fmc_ref, pcm_ref as pr

import pcm_edges_ref as R

pytestmark = pytest.mark.gpu
FAM_SEED = 11


@pytest.fixture(scope="module")
def families():
    out = {}
    for name in R.FAMILIES:
        edges, pos, ang = R.family(name, FAM_SEED)
        n = len(edges)
        s64, b64 = R.batched_bound(pr.edge_arrays(edges), *R.all_pairs(n), pos, ang)
        out[name] = (edges, pos, ang, R.choose_threshold(s64, b64), R.mp_matrix(edges, pos, ang))
    return out


@pytest.mark.parametrize("name", R.FAMILIES)
def test_family_smd_within_the_bound_and_adjacency_exact(gpu, families, name):
    edges, pos, ang, thres, ref = families[name]
    clique, adj, smd = host.pcm_outlier_rejection(edges, thres, pos, ang, want_matrices=True)
    worst, n_fin = 0.0, 0
    for (i, j), (vals, b) in ref.items():
        d = smd[i, j]
        assert d == smd[j, i] or (math.isnan(d) and math.isnan(smd[j, i]))
        assert R.within(d, vals, b), f"{name} ({i}, {j}): device {d!r}, exact {vals}, bound {b:.3g}"
        assert adj[i, j] == adj[j, i] == (d < thres)
        if math.isfinite(vals[0]):
            n_fin += 1
            worst = max(worst, min(abs(d - v) for v in vals) / b)
            if all(abs(v - thres) > b for v in vals) and len({v < thres for v in vals}) == 1:
                assert adj[i, j] == (vals[0] < thres), f"{name} ({i}, {j}) on the wrong side of {thres}"
        else:
            assert adj[i, j] == 0
    assert adj.diagonal().sum() == 0
    assert clique.tolist() == R.max_clique_heu_rows(adj)[0]
    assert n_fin >= (60 if name in ("theta", "not_finite") else 400)
    print(f"{name}: {n_fin} finite pairs, largest fraction of the bound used {worst:.3e}")


def test_theta_family_reaches_every_log_map_branch(families):
    """the theta family's error rotations: both sides of the 1e-12 switch, w < 0, and pi with an undetermined sign"""
    edges, pos, ang, _, ref = families["theta"]
    assert any(len(v) == 2 for v, _ in ref.values())               # |w| within its rounding bound: both branches


def test_threshold_is_strict_at_the_device_value(gpu, families):
    edges, pos, ang, thres, _ = families["correlated"]
    _, _, smd = host.pcm_outlier_rejection(edges, thres, pos, ang, want_matrices=True)
    fin = np.argwhere(np.isfinite(np.tril(smd, -1)) & (np.tril(np.ones_like(smd), -1) > 0))
    for i, j in fin[:: max(len(fin) // 4, 1)][:4]:
        t = float(smd[i, j])
        _, a0, s0 = host.pcm_outlier_rejection(edges, t, pos, ang, want_matrices=True)
        assert s0[i, j] == t and a0[i, j] == 0 and a0[j, i] == 0
        _, a1, _ = host.pcm_outlier_rejection(edges, np.nextafter(t, np.inf), pos, ang, want_matrices=True)
        assert a1[i, j] == 1 and a1[j, i] == 1


# ---- launch shapes ----------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def shapes():
    edges = R.shape_edges()
    smd, bnd = R.bound_matrix(edges, R.SHAPE_POS, R.SHAPE_ANG)
    low = np.tril_indices(len(edges), -1)
    thres = R.choose_threshold(smd[low], bnd[low])
    return edges, smd, bnd, thres


@pytest.mark.parametrize("n", R.SHAPES)
def test_osb_pcm_every_launch_shape_against_the_full_float64_matrix(gpu, shapes, n):
    edges, smd_r, bnd_r, thres = shapes
    clique, adj, smd = host.pcm_outlier_rejection(edges[:n], thres, R.SHAPE_POS, R.SHAPE_ANG, want_matrices=True)
    s_r, b_r = smd_r[:n, :n], bnd_r[:n, :n]
    fin = np.isfinite(s_r)
    assert np.array_equal(np.isfinite(smd), fin)
    assert np.all(np.abs(smd[fin] - s_r[fin]) <= 2 * b_r[fin]), "device smd outside the bound of the float64 value"
    assert np.array_equal(adj, (s_r < thres).astype(np.uint8))
    if n > 1:
        worst = float(np.max(np.abs(smd[fin] - s_r[fin]) / (2 * b_r[fin]))) if fin.any() else 0.0
        print(f"n = {n}: largest fraction of twice the bound used {worst:.3e}")
    assert clique.tolist() == R.max_clique_heu_rows(adj)[0]
    if fmc_ref.available() and n <= 1281:                          # (the library takes minutes on the larger graphs)
        assert clique.tolist() == fmc_ref.max_clique_heu(adj)[0]


# ---- the clique kernel's three launch forms ---------------------------------------------------------------------------
def clique_parity(form, graphs, slot_rows=None, stride=None, n_ctas=0):
    """osb_pcm_clique_parity on adjacency matrices -> list of cliques"""
    L = _l.load()
    slot_rows = slot_rows or max(a.shape[0] for a in graphs)
    stride = stride or (slot_rows + 31) // 32
    bits = np.zeros((len(graphs), slot_rows, stride), np.uint32)
    for g, a in enumerate(graphs):
        bits[g, :a.shape[0]] = R.pack_bits(a, stride)
    ns = np.array([a.shape[0] for a in graphs], np.int32)
    out = np.zeros((len(graphs), 1 + slot_rows), np.int32)
    _l.check(L.osb_pcm_clique_parity(form, _l.ptr(bits), len(graphs), _l.ptr(ns), slot_rows, stride, n_ctas,
                                     _l.ptr(out)))
    return [out[g, 1:1 + out[g, 0]].tolist() for g in range(len(graphs))]


def every_form(graphs):
    """the cliques of every graph from form 0 (one launch each, stride W), form 1 (one launch, slot stride 3 words more
    than the largest W) and form 2 (one launch, 200 KiB, 37 CTAs more than graphs); all three must agree"""
    one = [clique_parity(0, [a])[0] for a in graphs]
    nmax = max(a.shape[0] for a in graphs)
    jobs = clique_parity(1, graphs, stride=min((nmax + 31) // 32 + 3, 128))
    dev = clique_parity(2, graphs, n_ctas=len(graphs) + 37)
    assert one == jobs == dev
    return one


def golden(name):
    return np.load(os.path.join(GOLDEN, name))


def test_pin_graphs_in_every_launch_form(gpu):
    import sys
    sys.path.insert(0, GOLDEN)
    import make_ref_fmc as M
    z = golden("ref_fmc.npz")
    graphs = M.pin_graphs()
    want = [z["pin_verts"][z["pin_offs"][k]:z["pin_offs"][k + 1]].tolist() for k in range(len(graphs))]
    assert every_form(graphs) == want


def test_graph_families_in_every_launch_form(gpu):
    z = golden("ref_fmc_edges.npz")
    fams = R.graph_families()
    assert [str(x) for x in z["names"]] == [nm for nm, _ in fams]
    want = [z["verts"][z["offs"][k]:z["offs"][k + 1]].tolist() for k in range(len(fams))]
    got = every_form([a for _, a in fams])
    for (nm, _), g, w in zip(fams, got, want):
        assert g == w, nm


def test_parity_hook_argument_errors(gpu):
    L = _l.load()
    bits = np.zeros(4, np.uint32)
    n = np.array([1, 1], np.int32)
    out = np.zeros(8, np.int32)
    for form, ng, rows, stride, ctas in [(3, 1, 1, 1, 0), (0, 2, 1, 1, 0), (1, 1, 0, 1, 0), (1, 1, 33, 1, 0),
                                         (2, 2, 1, 1, 1), (1, 1, 4097, 129, 0)]:
        assert L.osb_pcm_clique_parity(form, _l.ptr(bits), ng, _l.ptr(n), rows, stride, ctas, _l.ptr(out)) == \
            _l.ERR_INVALID


# ---- the state's grow kernel against float64 ---------------------------------------------------------------------------
def test_grow_at_word_and_smem_boundaries_against_float64(gpu):
    """pairs appended to m = 63, 64, 65, 1279, 1280 and 4064 in one call, then grown in ONE more call (one grow launch,
    several jobs of different m, so the job search meets first_item boundaries): adjacency and clique against float64"""
    steps = [(63, 70), (64, 65), (65, 97), (1279, 1281), (1280, 1300), (4064, 4096)]
    lists = []
    for k, (m, n) in enumerate(steps):
        e = synth.pcm_edges(n, 0.85, 300 + k, id_a=1, id_b=3 + k)
        s, b = R.bound_matrix(e, R.SHAPE_POS, R.SHAPE_ANG)
        lists.append((1, 3 + k, e, s, b))
    allv = np.concatenate([s[np.tril_indices(len(s), -1)] for *_, s, _ in lists])
    allb = np.concatenate([b[np.tril_indices(len(b), -1)] for *_, b in lists])
    thres = R.choose_threshold(allv, allb)
    st = host.PcmState(1, True, thres, R.SHAPE_POS, R.SHAPE_ANG, max_pairs=len(steps), pair_capacity=4096)
    for phase in (0, 1):
        edges, ids = [], []
        for k, ((m, n), (a, b, e, _, _)) in enumerate(zip(steps, lists)):
            lo, hi = (0, m) if phase == 0 else (m, n)
            edges += e[lo:hi]
            ids += [(k << 40) + i for i in range(lo, hi)]
        n0 = host.launch_count()
        st.reject(edges, np.array(ids, np.int64))
        assert host.launch_count() - n0 == 2
    for (m, n), (a, b, e, s, _) in zip(steps, lists):
        _, adj, clique = st.pair(a, b)
        assert np.array_equal(adj, (s[:n, :n] < thres).astype(np.uint8)), (m, n)
        assert clique.tolist() == R.max_clique_heu_rows(adj)[0]
    st.close()
