"""The granule-planar convolutions' output epilogues batch their global loads (host only: reads the compiled sm_90a SASS).

After the last MMA of a tile, `conv1d_gp_kernel` and the fused `resblock_gp_kernel` add the bias, the residual and, in the
accumulate modes, the old output to each accumulator register pair and store it.  The output may alias the residual, so the
compiler keeps every load behind the previous pair's store unless the source issues them first; one pair at a time, each of the
32 pairs per thread waits a full global-load latency while no warp of the CTA issues MMAs.  The kernels walk the pairs in chunks
and issue a whole chunk's residual and output loads before its first store (DESIGN.md §3.1, §3.2).  So in every instantiation,
between the last HGMMA and the first STG after it there must be at least two non-constant LDG (residual, output) per pair of
the first chunk: 4 pairs in conv1d_gp (8 at MT = 4), 2 MT pairs (one column group) in resblock_gp.
"""
import os
import re

import pytest

from emotivoice_b200 import build
from test_wgmma_pipeline_sass import _sass_text, _tools

CHUNK_PAIRS = {"conv1d_gp_kernel": lambda mt: 8 if mt == 4 else 4, "resblock_gp_kernel": lambda mt: 2 * mt}


def _instructions(sass):
    """mangled function name -> its SASS instruction lines"""
    funcs, cur = {}, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [])
            continue
        if cur is not None and re.search(r"/\*[0-9a-f]{4,}\*/", line):
            cur.append(line)
    return funcs


def _loads_before_first_store(ins):
    """non-constant LDG between the last HGMMA and the first STG after it"""
    last = max(i for i, l in enumerate(ins) if "HGMMA" in l)
    n = 0
    for l in ins[last:]:
        if "STG" in l:
            return n
        if "LDG" in l and ".CONSTANT" not in l:
            n += 1
    raise AssertionError("no STG after the last HGMMA")


@pytest.fixture(scope="module")
def functions():
    nvcc, cuobjdump = _tools()
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    return _instructions(_sass_text(nvcc, cuobjdump, [os.path.join(build.CSRC, src) for src in ("conv1d_gp.cu", "resblock_gp.cu")]))


@pytest.mark.parametrize("kernel", list(CHUNK_PAIRS))
def test_epilogue_loads_precede_stores(functions, kernel):
    mine = {f: ins for f, ins in functions.items() if kernel in f}
    assert mine, "no %s in the SASS" % kernel
    bad = []
    for f, ins in mine.items():
        mode, mt, kbg = map(int, re.search(kernel + r"ILi(\d+)ELi(\d+)ELi(\d+)E", f).groups())
        want = 2 * CHUNK_PAIRS[kernel](mt)
        got = _loads_before_first_store(ins)
        if got < want:
            bad.append("<%d, %d, %d>: %d loads before the first store, want >= %d" % (mode, mt, kbg, got, want))
    assert not bad, "%s: the epilogue waits on one global load at a time in %d of %d instantiations:\n  %s" % (
        kernel, len(bad), len(mine), "\n  ".join(bad))
