"""CPU: the keyframe and distance-row kernels compile for sm_90a without spills, in one CTA's worth of registers and
static shared memory (ptxas's report of the build)."""
import os
import re

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
LOG = os.path.join(ROOT, "omni-swarm_b200", "csrc", "anchor.ptxas.log")


def kernel_info(name):
    text = open(LOG).read()
    i = text.index(f"Compiling entry function '_ZN3osb{len(name)}{name}")
    block = text[i:i + 600]
    spill = re.search(r"(\d+) bytes spill stores, (\d+) bytes spill loads", block)
    res = re.search(r"Used (\d+) registers.*?(\d+) bytes smem", block)
    return int(spill.group(1)), int(spill.group(2)), int(res.group(1)), int(res.group(2))


def test_no_spills_and_resources():
    from omniswarm_b200 import lib
    lib.build(verbose=False)
    for name, threads in (("keyframe_kernel", 256), ("distance_factors_kernel", 1024)):
        st, ld, regs, smem = kernel_info(name)
        assert st == 0 and ld == 0, name
        assert regs * threads <= 65536 and smem <= 48 * 1024, (name, regs, smem)
