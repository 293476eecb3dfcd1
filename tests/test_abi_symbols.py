"""CPU: the C-ABI library builds/loads and exports every symbol include/omniswarm_b200.h declares."""
import os
import re
import ctypes as C

import pytest

from omniswarm_b200 import lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def header_symbols():
    text = open(os.path.join(ROOT, "include", "omniswarm_b200.h")).read()
    text = re.sub(r"/\*.*?\*/", "", text, flags=re.S)
    return sorted(set(re.findall(r"\b(osb_[a-z0-9_]+)\s*\(", text)))


def test_library_exports_every_declared_symbol():
    L = lib.load()
    syms = header_symbols()
    assert len(syms) >= 40
    for s in syms:
        assert hasattr(L, s), f"{s} declared in the header but not exported"
    # and the ctypes table covers the header exactly
    assert set(lib.exported_symbols()) == set(syms)


def test_struct_sizes_match_header():
    # osb_keyframe_record: 4+4+4 ints header/counts, 4*4096 + 4*200*64 + 4*200*2 floats, 4*200 ints (stereo_match),
    # 4*200*3 floats (landmarks_3d), 4*200 ints (landmarks_flag)
    assert lib.RECORD_BYTES == 4 * (4 + 4 + 4) + 4 * (4 * 4096 + 4 * 200 * 64 + 4 * 200 * 2) + 4 * 4 * 200 \
        + 4 * 4 * 200 * 3 + 4 * 4 * 200
    assert C.sizeof(lib.LoopEdge) == 8 + 59 * 8 and C.sizeof(lib.PnpResult) == 6 * 4 + 8 * (2 + 7 + 4)
    assert C.sizeof(lib.SolveOptions) == 8 + 8 * 6 + 8   # + preconditioner, reserved
    assert C.sizeof(lib.SolveSummary) == 8 * 3 + 4 * 4


def test_no_cpu_fallback_without_device():
    L = lib.load()
    if L.osb_device_count() > 0:
        pytest.skip("a GPU is visible")
    h = C.c_void_p()
    assert L.osb_db_create(C.byref(h), 4096, 16) == lib.ERR_NO_DEVICE
    assert b"no CPU path" in L.osb_last_error()
    assert L.osb_solver_create(C.byref(h), 16, 16) == lib.ERR_NO_DEVICE
    assert L.osb_matcher_create(C.byref(h), 1, 200, 64) == lib.ERR_NO_DEVICE


def test_product_never_imports_oracle():
    """The product path must not route through the oracle (prompt section 3)."""
    pkg = os.path.join(ROOT, "omni-swarm_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                src = open(os.path.join(dirpath, f)).read()
                assert "import oracle" not in src and "from oracle" not in src, f


RAW_ACQUIRE_RELEASE = re.compile(
    r"\bcuda(Malloc|Free|HostAlloc|FreeHost|StreamCreate\w*|StreamDestroy|EventCreate\w*|EventDestroy)\s*\(")


def test_cuda_resources_are_acquired_only_through_the_owner():
    """Every device buffer, pinned buffer, stream and event is acquired and released by osb::Resources (common.cuh),
    so that destroy and every error path free all of it.  The one exception is swarm.cu's copy-engine transport: the
    IPC-exported inbox and the two buffers its handles are gathered through."""
    csrc = os.path.join(ROOT, "omni-swarm_b200", "csrc")
    raw = []
    for f in sorted(os.listdir(csrc)):
        if not f.endswith((".cu", ".cuh")) or f == "common.cuh":
            continue
        for i, line in enumerate(open(os.path.join(csrc, f)), 1):
            if not RAW_ACQUIRE_RELEASE.search(line):
                continue
            if f == "swarm.cu" and re.search(r"\b(inbox|d_all|d_flag)\b", line):
                continue
            raw.append(f"{f}:{i}: {line.strip()}")
    assert not raw, "raw CUDA acquire / release outside common.cuh:\n" + "\n".join(raw)
