"""GPU: a handle's host bound of a device-resident row count is lowered by what the appending kernel published, with no
synchronising call on the handle in between -- only the caller synchronises its own stream.  Front-end ingest (the
stores' row counts) and the back-end's device append (the measurement count)."""
import numpy as np
import pytest
import torch

from omniswarm_b200 import host, lib, synth
import frontend_harness as fh
from backend_harness import make_anchor

pytestmark = pytest.mark.gpu

ROW = lib.ANCHOR_RESULT_DTYPE.itemsize


def test_ingest_feedback_lowers_the_remote_bound(gpu):
    """a plain ingest of an own record charges both stores, so the remote store's bound is positive until the ingest's
    counts are read; once they have landed, query skips the empty remote store's scan exactly as it does after
    ingest_own (which charges the local store only), and answers the same"""
    st = fh.stream()
    plain, own = fh.make_frontend(), fh.make_frontend()
    rec_t = torch.zeros(fh.RB, dtype=torch.uint8, device="cuda")
    for i in range(2):
        up, down = (np.ascontiguousarray(a) for a in fh.frame_images(60 + i))
        plain.extract(up.ctypes.data, down.ctypes.data, 700 + i, rec_t.data_ptr(), st)
        launches, results = [], []
        for fe in (plain, own):
            if fe is plain:
                fe.ingest(rec_t.data_ptr(), 1, -1, st)
            else:
                fe.ingest_own(rec_t.data_ptr(), st)
            torch.cuda.current_stream().synchronize()
            res_t = fh.filled(fh.RS)
            c0 = host.launch_count()
            fe.query(rec_t.data_ptr(), res_t.data_ptr(), st)
            launches.append(host.launch_count() - c0)
            results.append(res_t.cpu().numpy().tobytes())
        assert launches[0] == launches[1]
        assert results[0] == results[1]
    assert plain.db_size(True) == own.db_size(True) == 0 and plain.db_size(False) == own.db_size(False) > 0
    plain.close(); own.close()


def test_append_feedback_lowers_the_run_bound(gpu):
    """add_measurements_dev charges max_n = n + 50; once the append has run, run_dev's grid covers exactly the n rows
    appended: no VOID row, and the rows of a handle fed the same measurements from the host"""
    g = synth.anchor_swarm(4, 30, 300, seed=11, with_orphans=False)
    rows = np.ascontiguousarray(g["meas"][:100])
    n = len(rows)
    dev, ref = make_anchor(g), make_anchor(g)
    for h in (dev, ref):
        for d, (s, p) in g["trajs"].items():
            h.push_odometry(d, s, p)
        h.set_window(*g["window"])
    ref.add_measurements(rows)
    st = fh.stream()
    buf = torch.frombuffer(bytearray(rows.tobytes()), dtype=torch.uint8).cuda()
    cnt = torch.tensor([n], dtype=torch.int32, device="cuda")
    dev.add_measurements_dev(buf.data_ptr(), cnt.data_ptr(), n + 50, 1e9, st)
    torch.cuda.current_stream().synchronize()
    out = fh.filled((n + 50) * ROW)
    assert dev.run_dev(out.data_ptr(), st) == n
    got = out.cpu().numpy().tobytes()
    assert got[:n * ROW] == ref.run().tobytes()
    assert set(got[n * ROW:]) == {fh.FILL}
    assert dev.status() == lib.OK and dev.size() == ref.size()
    dev.close(); ref.close()
