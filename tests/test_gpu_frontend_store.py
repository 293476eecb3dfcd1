"""GPU: the front-end's two keyframe databases (local and remote) at their limits and across a reset, its stage profile,
and the number of kernels one keyframe launches.  Ingest past capacity and db_load past the row or frame table must be
refused without touching either store; db_reset must bring a handle back to its freshly created state."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import synth, host, lib
from frontend_harness import H0, RB, RS, W0, depth_frame, frame_images, upload
import frontend_harness as fh

pytestmark = pytest.mark.gpu

ND = 4
K0 = np.array([80.0, 80.0, 48.0, 32.0])
IDENT = np.array([0.0, 0.0, 0.0, 1.0, 0.0, 0.0, 0.0])

# kernels launched by one keyframe on a warm handle (96x64, n_dirs = 4, max_num = 200)
LAUNCHES_STEREO = 51          # process(): cameras set, geometric filter on
LAUNCHES_DEPTH = 48           # process_depth()


CONFIG = dict(db_capacity=8, match_index_dist=1)


def make_frontend(**kw):
    return fh.make_frontend(CONFIG, **kw)


class Dev:
    """one device record, one device result and the current torch stream"""

    def __init__(self, fe):
        self.fe = fe
        self.stream = fh.stream()
        self.rec = torch.zeros(RB, dtype=torch.uint8, device="cuda")
        self.res = torch.zeros(RS, dtype=torch.uint8, device="cuda")

    def extract(self, seed, msg_id, drone_id=None):
        up, down = (np.ascontiguousarray(a) for a in frame_images(seed))
        self.fe.extract(up.ctypes.data, down.ctypes.data, msg_id, self.rec.data_ptr(), self.stream)
        self.fe.finish(self.stream)
        if drone_id is not None:
            rec = self.record()
            rec.drone_id = drone_id
            self.rec.copy_(upload([rec]))
        return self.record()

    def record(self):
        return fh.records(self.rec, 1)[0]

    def ingest(self):
        self.fe.ingest(self.rec.data_ptr(), 1, -1, self.stream)
        self.fe.finish(self.stream)

    def query(self, nonkeyframe=False):
        self.fe.query(self.rec.data_ptr(), self.res.data_ptr(), self.stream, nonkeyframe=nonkeyframe)
        self.fe.finish(self.stream)
        return result_fields(self.res.cpu().numpy().tobytes())


def result_fields(raw):
    """the defined part of a loop result: the match / geo lists up to their counts (entries past them are not written)"""
    r = lib.LoopResult.from_buffer_copy(bytes(raw))
    a = np.ctypeslib.as_array
    out = [r.hit_id, r.hit_dir, r.hit_score, r.accepted, r.swapped, r.hit_msg_id, r.hit_drone_id, list(r.dir_new),
           list(r.dir_old), list(r.n_matches), list(r.geo_valid), list(r.n_geo)]
    for s in range(ND):
        n, g = r.n_matches[s], r.n_geo[s]
        out += [a(r.match_new[s])[:n].tolist(), a(r.match_old[s])[:n].tolist(),
                a(r.geo_new[s])[:g].tolist(), a(r.geo_old[s])[:g].tolist()]
    return out


def sizes(fe):
    return fe.db_size(False), fe.db_size(True)


def assert_capacity_error(call):
    with pytest.raises(lib.OsbError) as e:
        call()
    assert e.value.status == lib.ERR_CAPACITY
    return str(e.value)


def test_ingest_past_capacity_is_refused_and_changes_nothing(gpu):
    """8 rows per store: two four-direction keyframes fill the local store through process(), two foreign ones the remote
    store through ingest(); one more of either kind is refused, and the stores still answer the same query."""
    fe = make_frontend()
    dev = Dev(fe)
    for i in (0, 1):
        rec, _ = fe.process(*frame_images(i), msg_id=i)
        assert all(rec.n_kpts[d] > 0 for d in range(ND))
    for i in (2, 3):
        dev.extract(i, 100 + i, drone_id=7)
        dev.ingest()
    assert sizes(fe) == (8, 8)
    dev.extract(0, 50)                                           # keyframe 0 again: a local hit
    before = dev.query()
    assert before[3] == 1 and before[5] == 0                     # accepted, hit_msg_id
    before_nkf = dev.query(nonkeyframe=True)                     # an own non-keyframe also looks at the remote store
    assert "database capacity exceeded" in assert_capacity_error(lambda: fe.process(*frame_images(4), msg_id=4))
    assert sizes(fe) == (8, 8)
    dev.extract(5, 105, drone_id=7)
    assert "database capacity exceeded" in assert_capacity_error(dev.ingest)
    assert sizes(fe) == (8, 8)
    dev.extract(0, 50)
    assert dev.query() == before and dev.query(nonkeyframe=True) == before_nkf
    fe.close()


def test_db_load_past_rows_or_frames_is_refused(gpu):
    """db_load checks the row table and the frame table; a keyframe without keypoints takes a frame but no row, so the
    frame table can be the one that runs out first.  A refused load leaves both stores as they were."""
    fe = make_frontend(geometric_filter=True)
    dev = Dev(fe)
    z = np.zeros((ND, H0, W0), np.uint8)
    for i in range(3):
        fe.process(z, z, msg_id=i)                              # 3 frames, 0 rows
    assert sizes(fe) == (0, 0)
    g = synth.descriptor_db(16, 4096, 3)
    assert_capacity_error(lambda: fe.db_load(g[:9], remote=False))           # rows: 0 + 9 > 8
    assert_capacity_error(lambda: fe.db_load(g[:6], remote=False))           # frames: 3 + 6 > 8
    assert sizes(fe) == (0, 0)
    fe.db_load(g[:5], remote=False)                             # frames 3 + 5 = 8: fits exactly
    assert_capacity_error(lambda: fe.db_load(g[5:6], remote=False))          # rows 6 <= 8, frames 9 > 8
    fe.db_load(g[8:16], remote=True)                            # the remote store is full on rows and frames
    assert_capacity_error(lambda: fe.db_load(g[:1], remote=True))
    assert sizes(fe) == (5, 8)
    rec = lib.KeyframeRecord()
    rec.drone_id, rec.msg_id, rec.n_dirs = 1, 60, ND
    for d in range(ND):
        rec.n_kpts[d] = 5
    np.ctypeslib.as_array(rec.global_desc[1])[:] = g[2]
    dev.rec.copy_(upload([rec]))
    hit_id, hit_dir, _, accepted, _, hit_msg_id, hit_drone_id = dev.query()[:7]
    assert (accepted, hit_id, hit_dir, hit_msg_id, hit_drone_id) == (1, 2, 1, -1, 1)
    np.ctypeslib.as_array(rec.global_desc[1])[:] = g[12]
    dev.rec.copy_(upload([rec]))
    hit_id, _, _, accepted, _, _, hit_drone_id = dev.query(nonkeyframe=True)[:7]
    assert (accepted, hit_id, hit_drone_id) == (1, lib.REMOTE_MAGIN_NUMBER + 4, -1)
    fe.close()


def test_db_reset_replays_bit_identically(gpu):
    """db_reset empties both stores and re-initialises the remote store's unscanned top-k list: replaying the same
    keyframes afterwards gives byte-identical records and identical loop results, including a non-keyframe query made
    before any foreign keyframe has arrived."""
    fe = make_frontend(db_capacity=64, geometric_filter=True)
    dev = Dev(fe)

    def one_pass():
        out = []
        for i in range(3):
            rec, res = fe.process(*frame_images(i), msg_id=i)
            out += [bytes(rec), result_fields(res)]
        dev.extract(1, 20)
        out.append(dev.query(nonkeyframe=True))                  # remote store still empty
        dev.extract(1, 21, drone_id=7)
        dev.ingest()                                            # a foreign keyframe
        dev.extract(1, 22)
        out.append(dev.query(nonkeyframe=True))                  # now hits the remote store
        rec, res = fe.process(*frame_images(0), msg_id=3)       # revisit: a local hit
        out += [bytes(rec), result_fields(res)]
        return out

    first = one_pass()
    assert sizes(fe) == (16, 4)
    assert first[7][6] == 7 and first[-1][3] == 1                # hit_drone_id of the remote hit, accepted of the revisit
    fe.db_reset()
    assert sizes(fe) == (0, 0)
    second = one_pass()
    assert len(first) == len(second)
    for i, (a, b) in enumerate(zip(first, second)):
        assert a == b, f"output {i} differs after db_reset"
    fe.close()


def stereo_frontend():
    fe = make_frontend(db_capacity=64, geometric_filter=True)
    left = np.tile(IDENT, (ND, 1))
    right = left.copy(); right[:, 1] = 0.1
    fe.set_cameras(K0, left, right, triangle_thres=0.02)
    fe.set_drone_pose(IDENT)
    return fe


def depth_frontend():
    fe = make_frontend(db_capacity=64, geometric_filter=True, zero_bottom_quarter=False)
    fe.set_depth_camera(K0, np.tile(IDENT, (ND, 1)), 0.3, 10.0)
    fe.set_drone_pose(IDENT)
    return fe


def test_stage_ms(gpu):
    fe = stereo_frontend()
    fe.process(*frame_images(0), msg_id=0)
    assert list(fe.stage_ms().values()) == [0.0] * 7             # profiling off
    ms = np.zeros(8, np.float32)
    lib.check(fe._lib.osb_frontend_stage_ms(fe._h, lib.ptr(ms)))
    assert (ms == 0).all()
    fe.set_profiling(True)
    fe.process(*frame_images(1), msg_id=1)
    fe.set_depth_camera(K0, np.tile(IDENT, (ND, 1)), 0.3, 10.0)
    for run in (lambda: fe.process(*frame_images(2), msg_id=2), lambda: fe.process_depth(*depth_frame(3), msg_id=3)):
        run()
        lib.check(fe._lib.osb_frontend_stage_ms(fe._h, lib.ptr(ms)))
        assert np.isfinite(ms).all() and (ms[:7] >= 0).all() and ms[0] > 0 and ms[7] == 0, ms
    fe.close()


def test_launches_per_keyframe(gpu):
    """the kernels one keyframe launches; a change here is a change of the pipeline, not of its plumbing"""
    fe = stereo_frontend()
    fe.process(*frame_images(0), msg_id=0)
    n0 = host.launch_count()
    fe.process(*frame_images(1), msg_id=1)
    stereo = host.launch_count() - n0
    fe.close()
    fe = depth_frontend()
    fe.process_depth(*depth_frame(0), msg_id=0)
    n0 = host.launch_count()
    fe.process_depth(*depth_frame(1), msg_id=1)
    depth = host.launch_count() - n0
    fe.close()
    print(f"launches per keyframe: stereo {stereo}, depth {depth}")
    assert (stereo, depth) == (LAUNCHES_STEREO, LAUNCHES_DEPTH)
