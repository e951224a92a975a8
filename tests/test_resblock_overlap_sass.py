"""The fused ResBlock kernel runs each tile's output epilogue under the next tile's c1 MMAs (host only: reads the compiled sm_90a SASS).

`resblock_gp_kernel` keeps c1 and c2 in two accumulator sets, so after c2 of tile i the consumers issue c1 of tile i + 1 tap by tap
and, between its chains, store epi2 of tile i (DESIGN.md §3.2).  The two sets only fit with `setmaxnreg`: the consumer warpgroups
take registers the transform and loader warps give back.  So in every instantiation:
  * USETMAXREG is present (the register split exists);
  * there is no local-memory traffic (STL / LDL): the accumulators and the epilogue chunk fit the consumers' registers;
  * epi2's global stores (STG) lie between HGMMAs: some STG comes after the first HGMMA and before the last one.  With the
    epilogue after c2 of the same tile, as one tile at a time, every STG follows the textually last HGMMA.
"""
import os
import re

import pytest

from emotivoice_b200 import build
from test_wgmma_pipeline_sass import _sass_text, _tools
from test_epilogue_sass import _instructions

KERNEL = "resblock_gp_kernel"


@pytest.fixture(scope="module")
def functions():
    nvcc, cuobjdump = _tools()
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    funcs = _instructions(_sass_text(nvcc, cuobjdump, [os.path.join(build.CSRC, "resblock_gp.cu")]))
    mine = {f: ins for f, ins in funcs.items() if KERNEL in f}
    assert mine, "no %s in the SASS" % KERNEL
    return mine


def _sig(name):
    return tuple(int(v) for v in re.search(KERNEL + r"ILi(\d+)ELi(\d+)ELi(\d+)ELi(\d+)E", name).groups())


def test_registers_are_reallocated(functions):
    bad = [_sig(f) for f, ins in functions.items() if not any("USETMAXREG" in l for l in ins)]
    assert not bad, "no setmaxnreg in %d of %d instantiations: %s" % (len(bad), len(functions), bad)


def test_no_local_memory(functions):
    bad = ["%s: %d" % (_sig(f), sum(1 for l in ins if re.search(r"\b(STL|LDL)\b", l))) for f, ins in functions.items()
           if any(re.search(r"\b(STL|LDL)\b", l) for l in ins)]
    assert not bad, "local-memory loads / stores (spills) in %d of %d instantiations:\n  %s" % (len(bad), len(functions), "\n  ".join(bad))


def test_epilogue_stores_lie_between_mmas(functions):
    bad = []
    for f, ins in functions.items():
        mma = [i for i, l in enumerate(ins) if "HGMMA" in l]
        stg = [i for i in range(mma[0], mma[-1]) if re.search(r"\bSTG\b", ins[i])]
        if not stg:
            bad.append(str(_sig(f)))
        # each chunk still issues its loads before its stores: a residual load between the first HGMMA and the first such STG
        elif not any(re.search(r"\bLDG\b", ins[i]) and ".CONSTANT" not in ins[i] for i in range(mma[0], stg[0])):
            bad.append("%s: no residual load before the first overlapped store" % (_sig(f),))
    assert not bad, "epi2 does not run under c1's MMAs in %d of %d instantiations:\n  %s" % (len(bad), len(functions), "\n  ".join(bad))
