"""CPU: the claim osb_frontend_query_received rests on, pinned on the oracle's LoopDetectorDB.  The reference handles the
keyframes received in a round one at a time, add then query (loop_detector.cpp:89-104); a foreign keyframe is added to
remote_index and queried in local_index only (:191-195).  So querying all of a round's foreign keyframes first and adding
them afterwards -- or adding them all first -- gives the answers of the arrival order exactly."""
import numpy as np

from omniswarm_b200 import synth
from oracle import frontend_ref as fr

SELF = 1


def detector(own):
    det = fr.LoopDetectorDB(self_id=SELF, dim=4096, inner_product_thres=0.3, init_mode_product_thres=0.2,
                            match_index_dist=2)
    for i, g in enumerate(own):
        det.add_frame(i, SELF, [g], [10])
    return det


def round_of_foreign(own, n, seed):
    """n foreign keyframes: revisits of own rows at several noise levels (some only above the init-mode threshold),
    copies of each other (a later one would hit an earlier one if foreign queries read remote_index), new places"""
    rng = np.random.default_rng(seed)
    rows = rng.integers(0, len(own), n)
    sig = np.array([0.3, 2.5, 3.7, 8.0])[np.arange(n) % 4]         # inner products ~0.96, 0.37, 0.26, 0.12
    q = np.stack([synth.noisy_queries(own, rows[i:i + 1], sigma=float(sig[i]), seed=seed * 100 + i)[0] for i in range(n)])
    q[n // 2:n // 2 + 3] = q[:3]                                   # repeats inside the round
    q[-2:] = synth.descriptor_db(2, 4096, seed + 900)              # places nobody has seen
    drones = 2 + rng.integers(0, 3, n)
    init = np.arange(n) % 5 == 2                                   # record 2 in init mode, its repeat 8 not
    return q, drones, init


def test_foreign_queries_do_not_depend_on_the_adds_of_their_round():
    own = synth.descriptor_db(60, 4096, 4)
    for seed in range(3):
        q, drones, init = round_of_foreign(own, 12, seed)
        # arrival order: add(r) then query(r)
        a = detector(own)
        arrival = []
        for r in range(len(q)):
            a.add_frame(1000 + r, int(drones[r]), [q[r]], [10])
            arrival.append(a.query(int(drones[r]), q[r], bool(init[r]), False))
        # every query first, then every add
        b = detector(own)
        first = [b.query(int(drones[r]), q[r], bool(init[r]), False) for r in range(len(q))]
        for r in range(len(q)):
            b.add_frame(1000 + r, int(drones[r]), [q[r]], [10])
        # every add first, then every query
        c = detector(own)
        for r in range(len(q)):
            c.add_frame(1000 + r, int(drones[r]), [q[r]], [10])
        last = [c.query(int(drones[r]), q[r], bool(init[r]), False) for r in range(len(q))]
        assert arrival == first == last
        assert a.remote_index.ntotal == b.remote_index.ntotal == len(q) and a.local_index.ntotal == len(own)
        # the round is not trivial: hits, misses, and hits that only init mode accepts
        acc = [rid != -1 and d > -1 for rid, d in arrival]
        assert any(acc) and not all(acc)
        assert any(ok and i and d <= 0.3 for ok, i, (_, d) in zip(acc, init, arrival))


def test_an_own_keyframe_would_see_the_round():
    """The contrast: an own keyframe's query reads remote_index, so for it the adds of a round do matter -- which is why
    the batch covers foreign keyframes only."""
    own = synth.descriptor_db(10, 4096, 5)
    q = synth.descriptor_db(1, 4096, 6)[0]
    det = detector(own)
    assert det.query(SELF, q, False, True)[0] == -1
    det.add_frame(50, 3, [q], [10])
    assert det.query(SELF, q, False, True)[0] == fr.REMOTE_MAGIN_NUMBER
