"""CPU: oracle/loop_net_ref.py's two forms of a received keyframe -- the message-level restatement of LoopNet's sender and
receiver plus on_image_recv's gates, and the vectorised receive_record the GPU tests compare against -- agree on random
records, at every gate's edge, and on the corner cases; the literal per-image frame key splits frames."""
import numpy as np
import pytest

from oracle import loop_net_ref as ln

SELF = 1


def random_record(seed, drone=2, msg=7, n_dirs=4, n_kpts=None, p_flag=0.6):
    rng = np.random.default_rng(seed)
    r = ln.empty_record()
    r["drone_id"], r["msg_id"], r["n_dirs"], r["reserved"] = drone, msg, n_dirs, 0
    # every plane filled with noise, beyond n_kpts too: what lies there must not travel
    r["global_desc"] = rng.normal(size=r["global_desc"].shape)
    r["local_desc"] = rng.normal(size=r["local_desc"].shape)
    r["kpts"] = rng.uniform(0, 96, r["kpts"].shape)
    r["landmarks_3d"] = rng.normal(size=r["landmarks_3d"].shape)
    r["stereo_match"] = rng.integers(-1, 200, r["stereo_match"].shape)
    r["landmarks_flag"] = (rng.random(r["landmarks_flag"].shape) < p_flag).astype(np.int32)
    r["n_kpts"] = rng.integers(0, 201, ln.MAX_DIRS) if n_kpts is None else n_kpts
    r["n_kpts_down"] = rng.integers(0, 201, ln.MAX_DIRS)
    return r


def both(rec, db_rows=10, min_dir=3, min_lm=15):
    """(literal frames kept, vectorised record); the literal form gives [] or one frame"""
    lit = ln.receive_literal(rec, SELF, db_rows, min_dir, min_lm)
    vec = ln.receive_record(rec, SELF, db_rows, min_dir, min_lm)
    return lit, vec


def assert_agree(rec, **kw):
    lit, vec = both(rec, **kw)
    assert len(lit) <= 1
    if lit:
        assert lit[0].tobytes() == vec.tobytes()
    else:
        assert vec.tobytes() == ln.dropped(rec).tobytes()
    return bool(lit)


@pytest.mark.parametrize("seed", range(40))
def test_forms_agree_on_random_records(seed):
    rng = np.random.default_rng(1000 + seed)
    rec = random_record(seed, n_dirs=int(rng.integers(1, 5)), p_flag=float(rng.uniform(0, 1)))
    assert_agree(rec, min_dir=int(rng.integers(1, 5)), min_lm=int(rng.integers(1, 300)))


def test_kept_record_layout():
    rec = random_record(3, n_kpts=[200, 37, 0, 120])
    rec["landmarks_flag"][1][:] = 0                           # a direction with keypoints and no flagged landmark
    assert assert_agree(rec, min_dir=2, min_lm=1)
    out = ln.receive_record(rec, SELF, 10, 2, 1)
    for d, n in enumerate([200, 37, 0, 120]):
        idx = np.nonzero(rec["landmarks_flag"][d][:n] > 0)[0]
        k = len(idx)
        assert out["n_kpts"][d] == k and out["n_kpts_down"][d] == 0
        np.testing.assert_array_equal(out["local_desc"][d][:k], rec["local_desc"][d][idx])
        np.testing.assert_array_equal(out["kpts"][d][:k], rec["kpts"][d][idx])
        np.testing.assert_array_equal(out["stereo_match"][d][k:], -1)
        assert not out["local_desc"][d][k:].any() and not out["landmarks_flag"][d][k:].any()
        assert (out["global_desc"][d] == rec["global_desc"][d]).all() if k else not out["global_desc"][d].any()
    assert out["n_kpts"][1] == 0 and out["n_kpts"][2] == 0


@pytest.mark.parametrize("min_dir", [1, 2, 3, 4])
def test_direction_gate_at_equality_and_one_below(min_dir):
    nk = [50] * min_dir + [0] * (4 - min_dir)
    rec = random_record(5, n_kpts=nk, p_flag=1.0)
    assert assert_agree(rec, min_dir=min_dir, min_lm=1)       # exactly min_dir non-empty directions: kept
    rec["landmarks_flag"][min_dir - 1][:] = 0                # one below
    assert not assert_agree(rec, min_dir=min_dir, min_lm=1)


def test_landmark_gate_at_equality_and_one_below():
    rec = random_record(6, n_kpts=[40, 40, 40, 40])
    total = int((rec["landmarks_flag"][:, :40] > 0).sum())
    assert assert_agree(rec, min_dir=1, min_lm=total)
    assert not assert_agree(rec, min_dir=1, min_lm=total + 1)


def test_empty_store_then_not():
    rec = random_record(7, p_flag=1.0, n_kpts=[100] * 4)
    assert not assert_agree(rec, db_rows=0, min_dir=1, min_lm=1)
    assert assert_agree(rec, db_rows=1, min_dir=1, min_lm=1)
    own = random_record(7, drone=SELF)                        # own and skipped records travel unchanged
    assert ln.receive_record(own, SELF, 0, 3, 15).tobytes() == own.tobytes()
    assert ln.receive_record(rec, SELF, 0, 3, 15, skipped=True).tobytes() == rec.tobytes()


def test_no_flags_all_flags_and_no_keypoints():
    none = random_record(8, p_flag=0.0)
    assert not assert_agree(none, min_dir=1, min_lm=1)
    assert ln.receive_literal(none, SELF, 10, 1, 1) == []
    full = random_record(9, p_flag=1.0, n_kpts=[200] * 4)
    assert assert_agree(full, min_dir=4, min_lm=800)
    out = ln.receive_record(full, SELF, 10, 4, 800)
    for f in ("local_desc", "kpts", "stereo_match", "landmarks_3d", "landmarks_flag", "global_desc"):
        np.testing.assert_array_equal(out[f], full[f])
    zero = random_record(10, n_kpts=[0, 0, 0, 0], p_flag=1.0)
    assert not assert_agree(zero, min_dir=1, min_lm=0)
    assert ln.broadcast(zero, [1, 2, 3, 4]) == []            # nothing is sent for a direction without landmarks


def test_broadcast_messages():
    rec = random_record(11, n_kpts=[10, 0, 5, 3], p_flag=0.5)
    msgs = ln.broadcast(rec, [11, 12, 13, 14])
    heads = [m for k, m in msgs if k == "header"]
    assert [h["direction"] for h in heads] == [0, 2, 3]
    for h in heads:
        n = int(rec["n_kpts"][h["direction"]])
        assert h["feature_num"] == int((rec["landmarks_flag"][h["direction"]][:n] > 0).sum())
        lms = [m for k, m in msgs if k == "landmark" and m["header_id"] == h["msg_id"]]
        assert [m["landmark_id"] for m in lms] == list(np.nonzero(rec["landmarks_flag"][h["direction"]][:n] > 0)[0])


def test_literal_per_image_key_splits_frames():
    """image_desc_callback keys a frame by the image's own (random) msg_id: each direction becomes a frame of its own,
    which MIN_DIRECTION_LOOP = 3 then drops; keyed by frame_id the record is one frame"""
    rec = random_record(12, p_flag=1.0, n_kpts=[60] * 4)
    rx = ln.Receiver("msg_id", 3)
    frames = rx.receive(ln.broadcast(rec, [101, 202, 303, 404]))
    assert len(frames) == 4
    assert all(sum(im is not None for im in f["images"]) == 1 for f in frames)
    assert not any(ln.gate(f, SELF, 10, 3, 15) for f in frames)
    assert ln.receive_literal(rec, SELF, 10, 3, 15, key="msg_id") == []
    kept = ln.receive_literal(rec, SELF, 10, 3, 15, key="frame_id")
    assert len(kept) == 1 and list(kept[0]["n_kpts"]) == [60] * 4


def test_round_skip_and_own():
    recs = [random_record(20 + i, drone=[2, SELF, 3, 4][i], msg=i) for i in range(4)]
    out = ln.receive_round([r.tobytes() for r in recs], 2, SELF, 5, 2, 10)
    assert out[1].tobytes() == recs[1].tobytes() and out[2].tobytes() == recs[2].tobytes()
    for i in (0, 3):
        assert out[i].tobytes() == ln.receive_record(recs[i], SELF, 5, 2, 10).tobytes()
