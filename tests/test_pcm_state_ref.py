"""CPU: the oracle of the persistent PCM state (oracle/pcm_state_ref.py) on hand-built cases -- incremental equals a
from-scratch oracle/pcm_ref.pcm on each pair's stored list, routing, seen ids, duplicates, and the keep rule."""
import numpy as np

from omniswarm_b200 import synth
from oracle import pcm_ref
from oracle.pcm_state_ref import PcmStateRef

THRES, POS, ANG = 15.0, 1e-4, 1e-5


def edge(a, b, seed=0, k=0):
    """one inlier loop edge between drones a and b"""
    return synth.pcm_edges(k + 1, 0.0, seed, flip_frac=0.0, id_a=a, id_b=b)[k]


def test_incremental_equals_from_scratch_after_every_round():
    for redundant in (True, False):
        ref = PcmStateRef(1, redundant, THRES, POS, ANG)
        for edges, ids in synth.pcm_swarm_rounds(3, 4, 4, 0.3, seed=1):
            keep = ref.reject(edges, ids)
            assert len(keep) == len(ids)
            for k, p in ref.pairs.items():
                clique, adj, _ = pcm_ref.pcm(p["edges"], THRES, POS, ANG)
                assert np.array_equal(p["adj"], adj)
                assert p["clique"] == clique
                assert ref.inliers(*k) == sorted({p["ids"][c] for c in clique})
        stored = {k for k in ref.pairs}
        if redundant:
            assert stored == {(a, b) for a in (1, 2, 3) for b in (1, 2, 3) if a <= b}
        else:
            assert stored == {(1, 1), (1, 2), (1, 3)}


def test_routing_self_only_and_unrouted_edges_stay_new():
    ref = PcmStateRef(2, False, THRES, POS, ANG)
    es = [edge(1, 3), edge(2, 2), edge(3, 2)]
    keep = ref.reject(es, [10, 11, 12])
    assert keep.all()                                                # no pair has a set before its first PCM
    assert set(ref.pairs) == {(2, 2), (2, 3)}
    assert ref.seen == {11, 12} and 10 not in ref.seen               # the (1, 3) loop was not processed: still new
    assert ref.inliers(1, 3) is None and ref.inliers(3, 2) == [12]
    ref.reject(es, [10, 11, 12])
    assert ref.pair(1, 3) is None and len(ref.pair(2, 3)[0]) == 1
    red = PcmStateRef(2, True, THRES, POS, ANG)
    red.reject(es, [10, 11, 12])
    assert set(red.pairs) == {(1, 3), (2, 2), (2, 3)} and red.seen == {10, 11, 12}


def test_duplicates_within_one_call_are_both_appended():
    ref = PcmStateRef(1, True, THRES, POS, ANG)
    e0, e1 = edge(1, 2, k=0), edge(1, 2, k=1)
    ref.reject([e0, e1, e0], [5, 6, 5])
    ids, adj, clique = ref.pair(1, 2)
    assert ids == [5, 6, 5] and adj.shape == (3, 3)
    ref.reject([e0], [5])                                            # seen now
    assert ref.pair(1, 2)[0] == [5, 6, 5]


def test_resubmitted_id_with_new_values_changes_nothing():
    ref = PcmStateRef(1, True, THRES, POS, ANG)
    es = [edge(1, 2, k=k) for k in range(4)]
    ref.reject(es, [1, 2, 3, 4])
    ids, adj, clique = ref.pair(1, 2)
    good = ref.inliers(1, 2)
    moved = dict(es[2], rel=es[2]["rel"] + np.array([3.0, 0, 0, 0, 0, 0, 0]))
    keep = ref.reject([es[0], es[1], moved, es[3]], [1, 2, 3, 4])
    ids2, adj2, clique2 = ref.pair(1, 2)
    assert ids2 == ids and np.array_equal(adj2, adj) and clique2 == clique and ref.inliers(1, 2) == good
    assert ref.pairs[(1, 2)]["edges"][2] is es[2]                    # the first-seen values stay
    assert keep.tolist() == [i in good for i in (1, 2, 3, 4)]


def test_keep_rule_no_set_pcm_set_set_inliers_and_overwrite():
    ref = PcmStateRef(1, False, THRES, POS, ANG)
    inl = [edge(1, 2, k=k) for k in range(5)]
    out = dict(inl[4], rel=inl[4]["rel"] + np.array([2.5, -2.0, 1.0, 0, 0, 0, 0]))     # a gross outlier
    other = [edge(2, 3, k=k) for k in range(3)]
    keep = ref.reject(inl[:4] + [out] + other, [1, 2, 3, 4, 5, 20, 21, 22])
    good = ref.inliers(1, 2)                                         # PCM set: the clique's ids
    clique, _, _ = pcm_ref.pcm(inl[:4] + [out], THRES, POS, ANG)
    assert good == sorted(i + 1 for i in clique) and 5 not in good and len(good) >= 2
    assert keep.tolist() == [i in good for i in (1, 2, 3, 4, 5)] + [True] * 3      # (2, 3): no set, all kept
    ref.set_inliers(3, 2, [21, 99])                                  # another drone's set for (2, 3)
    keep = ref.reject(other, [20, 21, 22])
    assert keep.tolist() == [False, True, False] and ref.inliers(2, 3) == [21, 99]
    ref.set_inliers(2, 1, [5])                                       # contains self: ignored
    assert ref.inliers(1, 2) == good
    red = PcmStateRef(1, True, THRES, POS, ANG)
    red.reject(other[:2], [20, 21])
    red.set_inliers(2, 3, [20])
    assert red.reject(other[:2], [20, 21]).tolist() == [True, False]
    red.reject(other, [20, 21, 22])                                  # (2, 3) gains a loop: its PCM set replaces [20]
    assert red.inliers(2, 3) == [20, 21, 22]
