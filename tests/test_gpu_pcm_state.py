"""GPU: the persistent PCM state (osb_pcm_state_*) against its oracle (oracle/pcm_state_ref.py) and the stateless path
(osb_pcm on each pair's stored list): keep mask, inlier sets, adjacency bit-identical, clique identical, and the state's
errors, launches and resources."""
import ctypes as C

import numpy as np
import pytest

from omniswarm_b200 import synth, host, lib as _l
from oracle import pcm_ref as pr
from oracle import fmc_ref
from oracle.pcm_state_ref import PcmStateRef

pytestmark = pytest.mark.gpu
THRES, POS, ANG = 15.0, 1e-4, 1e-5
PAIRS5 = [(a, b) for a in range(1, 6) for b in range(1, 6) if a <= b]


def stateless(edges):
    """osb_pcm on a pair's whole insertion-ordered list -> (clique, adj)"""
    clique, adj, _ = host.pcm_outlier_rejection(edges, THRES, POS, ANG, want_matrices=True)
    return clique, adj


def check_pair_against_stateless(st, a, b, edges):
    ids, adj, clique = st.pair(a, b)
    assert len(ids) == len(edges)
    rclique, radj = stateless(edges)
    assert np.array_equal(adj, radj), f"pair {a},{b}: adjacency differs from osb_pcm"
    assert np.array_equal(clique, rclique)
    return ids, adj, clique


@pytest.mark.parametrize("redundant", [True, False])
def test_rounds_match_oracle_and_stateless(gpu, redundant):
    st = host.PcmState(1, redundant, THRES, POS, ANG, max_pairs=15, pair_capacity=256)
    ref = PcmStateRef(1, redundant, THRES, POS, ANG)
    for edges, ids in synth.pcm_swarm_rounds(5, 6, 8, 0.3, seed=3):
        keep = st.reject(edges, ids)
        assert np.array_equal(keep, ref.reject(edges, ids))
        assert ref.min_margin > 1e-6, "test data has a pair on the threshold"
        for a, b in PAIRS5:
            got = st.inliers(a, b)
            want = ref.inliers(a, b)
            assert (got is None) == (want is None) and (got is None or got.tolist() == want)
            rp = ref.pair(a, b)
            if rp is None:
                assert st.pair(a, b)[0].size == 0
                continue
            ids_d, adj_d, clique_d = check_pair_against_stateless(st, a, b, ref.pairs[(a, b)]["edges"])
            assert ids_d.tolist() == rp[0] and np.array_equal(adj_d, rp[1]) and clique_d.tolist() == rp[2]
            if fmc_ref.available():
                assert clique_d.tolist() == fmc_ref.max_clique_heu(rp[1])[0]
    assert len(ref.pairs) == (15 if redundant else 5)


def test_new_rows_at_word_boundaries(gpu):
    """rows appended at m = 0, 31, 32, 33 (the first old-row word that is recomputed: floor(m / 32))"""
    edges = synth.pcm_edges(40, 0.3, 11)
    ids = np.arange(40, dtype=np.int64) + (1 << 33)
    st = host.PcmState(1, True, THRES, POS, ANG, max_pairs=2, pair_capacity=64)
    ref = PcmStateRef(1, True, THRES, POS, ANG)
    for lo, hi in [(0, 31), (31, 32), (32, 33), (33, 40)]:
        keep = st.reject(edges[:hi], ids[:hi])
        assert np.array_equal(keep, ref.reject(edges[:hi], ids[:hi]))
        ids_d, adj_d, clique_d = check_pair_against_stateless(st, 1, 2, edges[:hi])
        assert clique_d.tolist() == ref.pair(1, 2)[2] and np.array_equal(adj_d, ref.pair(1, 2)[1])
    assert ref.min_margin > 1e-6


def test_sizes_across_the_shared_memory_bound_and_to_capacity(gpu):
    """in one launch: a pair growing across n = 1280 (the clique kernel leaves shared memory), a pair filled to 4096 and
    a pair of a few loops; then a call that would overflow the full pair fails and changes nothing"""
    big = synth.pcm_edges(4096, 0.4, 21, id_a=1, id_b=2)
    mid = synth.pcm_edges(1300, 0.4, 22, id_a=1, id_b=3)
    small = synth.pcm_edges(5, 0.2, 23, id_a=3, id_b=3)
    idb = np.arange(4096, dtype=np.int64) + (5 << 32)
    idm = np.arange(1300, dtype=np.int64) + (6 << 32)
    ids_s = np.arange(5, dtype=np.int64) + (7 << 32)
    st = host.PcmState(1, True, THRES, POS, ANG, max_pairs=3, pair_capacity=4096)
    st.reject(big[:3000] + mid[:1270] + small[:2], np.concatenate([idb[:3000], idm[:1270], ids_s[:2]]))
    ev = np.concatenate([idb, idm[:1290], ids_s])
    n0 = host.launch_count()
    st.reject(big + mid[:1290] + small, ev)
    assert host.launch_count() - n0 == 2
    _, adj_b, clique_b = check_pair_against_stateless(st, 1, 2, big)
    _, adj_m, clique_m = check_pair_against_stateless(st, 3, 1, mid[:1290])
    check_pair_against_stateless(st, 3, 3, small)
    assert clique_m.tolist() == pr.max_clique_heu(adj_m)[0]
    rng = np.random.default_rng(0)
    for _ in range(100):                                             # sampled pairs of the big graph against the oracle
        i, j = sorted(rng.choice(4096, 2, replace=False))[::-1]
        assert adj_b[i, j] == (pr.pair_smd(big[i], big[j], POS, ANG) < THRES)
    before = [st.pair(*p) for p in [(1, 2), (1, 3), (3, 3)]]
    good = [st.inliers(*p) for p in [(1, 2), (1, 3), (3, 3)]]
    extra = synth.pcm_edges(12, 0.0, 24, id_a=1, id_b=2)
    n0 = host.launch_count()
    with pytest.raises(_l.OsbError) as e:                            # 4097 loops in pair (1, 2)
        st.reject(extra[:1] + mid[1290:], np.concatenate([[9 << 32], idm[1290:]]))
    assert e.value.status == _l.ERR_CAPACITY and host.launch_count() == n0
    with pytest.raises(_l.OsbError) as e:                            # a fourth pair
        st.reject(synth.pcm_edges(1, 0.0, 25, id_a=4, id_b=5), [10 << 32])
    assert e.value.status == _l.ERR_CAPACITY
    for p, b, g in zip([(1, 2), (1, 3), (3, 3)], before, good):
        a = st.pair(*p)
        assert all(np.array_equal(x, y) for x, y in zip(a, b)) and np.array_equal(st.inliers(*p), g)
    st.reject(mid[1290:], idm[1290:])                                # the refused loops are still new
    check_pair_against_stateless(st, 1, 3, mid)


def test_pair_without_new_loops_keeps_its_clique_and_empty_calls_launch_nothing(gpu):
    e12 = synth.pcm_edges(50, 0.3, 31, id_a=1, id_b=2)
    e13 = synth.pcm_edges(20, 0.3, 32, id_a=1, id_b=3)
    i12 = np.arange(50, dtype=np.int64) + (3 << 32)
    i13 = np.arange(20, dtype=np.int64) + (4 << 32)
    st = host.PcmState(1, False, THRES, POS, ANG, max_pairs=4, pair_capacity=128)
    st.reject(e12 + e13[:10], np.concatenate([i12, i13[:10]]))
    before = st.pair(1, 2)
    good = np.concatenate([st.inliers(1, 2), st.inliers(1, 3)])
    n0 = host.launch_count()
    keep = st.reject(e12 + e13[:10], np.concatenate([i12, i13[:10]]))       # everything seen
    assert host.launch_count() == n0
    assert st.reject([], []).size == 0 and host.launch_count() == n0
    keep2 = st.reject(synth.pcm_edges(4, 0.0, 33, id_a=2, id_b=3), [1, 2, 3, 4])  # unrouted: nothing launched
    assert keep2.all() and host.launch_count() == n0
    st.reject(e12 + e13, np.concatenate([i12, i13]))                 # only (1, 3) gains loops
    assert host.launch_count() - n0 == 2
    after = st.pair(1, 2)
    assert all(np.array_equal(x, y) for x, y in zip(before, after))
    assert np.array_equal(keep, np.isin(np.concatenate([i12, i13[:10]]), good))
    check_pair_against_stateless(st, 1, 3, e13)


def test_unrouted_loops_stay_new(gpu):
    """without `redundant`, a loop of a pair without self_id is neither stored nor marked as seen: the same id arriving
    later on a pair that contains self_id is stored there"""
    e23 = synth.pcm_edges(3, 0.0, 45, id_a=2, id_b=3)
    e12 = synth.pcm_edges(3, 0.0, 46, id_a=1, id_b=2)
    ids = np.array([11, 12, 13], np.int64) + (1 << 36)
    st = host.PcmState(1, False, THRES, POS, ANG, max_pairs=2, pair_capacity=16)
    ref = PcmStateRef(1, False, THRES, POS, ANG)
    for edges in (e23, e12):
        assert np.array_equal(st.reject(edges, ids), ref.reject(edges, ids))
    assert st.pair(2, 3)[0].size == 0 and st.pair(1, 2)[0].tolist() == ids.tolist() == ref.pair(1, 2)[0]


def test_inlier_sets_from_other_drones(gpu):
    e23 = synth.pcm_edges(6, 0.0, 41, id_a=2, id_b=3)
    ids = np.arange(6, dtype=np.int64) + (1 << 40)
    st = host.PcmState(1, False, THRES, POS, ANG, max_pairs=2, pair_capacity=16)
    assert st.inliers(2, 3) is None and st.reject(e23, ids).all()
    st.set_inliers(3, 2, ids[[1, 4]])
    assert st.inliers(2, 3).tolist() == ids[[1, 4]].tolist()
    assert st.reject(e23, ids).tolist() == [False, True, False, False, True, False]
    st.set_inliers(1, 2, ids[:1])                                    # contains self: ignored
    assert st.inliers(1, 2) is None
    st.set_inliers(2, 3, [])
    assert st.inliers(2, 3).size == 0 and not st.reject(e23, ids).any()


def test_argument_errors_and_resources(gpu):
    L = _l.load()
    live0 = host.live_resources()
    h = C.c_void_p()
    for cap, pairs in [(0, 1), (4097, 1), (16, 0), (16, -1)]:
        p = _l.PcmStateParams(1, 1, pairs, cap, THRES, POS, ANG)
        assert L.osb_pcm_state_create(C.byref(h), C.byref(p)) == _l.ERR_INVALID
    assert L.osb_pcm_state_create(None, C.byref(_l.PcmStateParams(1, 1, 1, 16, THRES, POS, ANG))) == _l.ERR_INVALID
    assert L.osb_pcm_state_create(C.byref(h), None) == _l.ERR_INVALID
    assert host.live_resources() == live0
    st = host.PcmState(1, True, THRES, POS, ANG, max_pairs=3, pair_capacity=64)
    live1 = host.live_resources()
    arr = host.loop_edges(synth.pcm_edges(2, 0.0, 51))
    ids = np.array([1, 2], np.int64)
    keep = np.zeros(2, np.uint8)
    n = C.c_int32(0)
    assert L.osb_pcm_state_reject(st._h, _l.ptr(arr), _l.ptr(ids), -1, _l.ptr(keep)) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject(st._h, None, _l.ptr(ids), 2, _l.ptr(keep)) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject(st._h, _l.ptr(arr), None, 2, _l.ptr(keep)) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject(st._h, _l.ptr(arr), _l.ptr(ids), 2, None) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject(None, _l.ptr(arr), _l.ptr(ids), 2, _l.ptr(keep)) == _l.ERR_INVALID
    assert L.osb_pcm_state_reject(st._h, None, None, 0, None) == _l.OK
    assert L.osb_pcm_state_inliers(st._h, 1, 2, None, -1, C.byref(n)) == _l.ERR_INVALID
    assert L.osb_pcm_state_inliers(st._h, 1, 2, None, 0, None) == _l.ERR_INVALID
    assert L.osb_pcm_state_set_inliers(st._h, 2, 3, None, 1) == _l.ERR_INVALID
    assert L.osb_pcm_state_set_inliers(st._h, 2, 3, _l.ptr(ids), -1) == _l.ERR_INVALID
    assert L.osb_pcm_state_pair(st._h, 1, 2, None, None, None, None, None) == _l.ERR_INVALID
    assert host.live_resources() == live1
    rounds = synth.pcm_swarm_rounds(2, 4, 6, 0.3, seed=5)            # pairs (1,1), (1,2), (2,2)
    st.reject(*rounds[0])
    live2 = host.live_resources()
    assert live2 == live1 + 3                                        # one slot per pair, at its first use
    for edges, r_ids in rounds[1:]:
        st.reject(edges, r_ids)
        st.inliers(1, 2); st.pair(1, 2)
    assert host.live_resources() == live2                            # nothing acquired after a pair's first use
    ids_big = np.zeros(5, np.int64)
    assert L.osb_pcm_state_inliers(st._h, 1, 2, _l.ptr(ids_big), 0, C.byref(n)) == _l.ERR_CAPACITY
    st.close()
    assert host.live_resources() == live0
