"""The granule-planar convolutions issue each tap's MMAs as one unbroken wgmma chain (host only: reads the compiled sm_90a SASS).

`conv1d_gp_kernel<MODE, MT, KBG, BN>` and `resblock_gp_kernel<MODE, MT, KBG, C>` fix the N width of their MMAs at compile time, so a
tap of a full channel block is NK8 K steps x MT accumulators x m MMAs (m = 3 in 3xTF32 / bf16x3, else 1) between one
`wgmma.fence` and one `wgmma.commit_group` (DESIGN.md §3).  With N chosen at run time every K step went through a jump table
(`BRX`) and ptxas fenced each fragment with its own `WARPGROUP.ARRIVE`.  So in every instantiation:
  * no BRX lies between two HGMMA;
  * every HGMMA has the instantiation's N;
  * some run of HGMMA from a WARPGROUP.ARRIVE to the next HGMMA marked gsb0 holds the whole tap of a full block, NK8 * MT * m MMAs.
"""
import os
import re

import pytest

from emotivoice_b200 import build
from test_wgmma_pipeline_sass import _sass_text, _tools
from test_epilogue_sass import _instructions

KERNELS = ("conv1d_gp_kernel", "resblock_gp_kernel")


def _params(kernel, name):
    """(MODE, MT, KBG, N); N is None for a kernel whose N is not a template parameter"""
    m = re.search(kernel + r"ILi(\d+)ELi(\d+)ELi(\d+)E(?:Li(\d+)E)?", name)
    assert m, "%s: no <MODE, MT, KBG, ...> signature" % name
    return tuple(int(v) if v else None for v in m.groups())


def _chain_len(kernel, mode, mt, kbg, n):
    """MMAs of one tap of a full channel block"""
    cpg = 8 if mode == 2 else 4                   # activation channels per 16-byte granule
    wcpg = 8 if mode >= 2 else 4                  # operand channels per granule
    kb = cpg * kbg
    if kernel == "resblock_gp_kernel" and n:
        kb = min(kb, n)                         # n = C: a 32-channel layer is one block, shorter than KB
    m = 3 if mode in (1, 3) else 1
    return kb // (2 * wcpg) * mt * m


def _longest_chain(ins):
    """the most HGMMA between a WARPGROUP.ARRIVE and the next gsb0 HGMMA, counting only runs with nothing but non-HGMMA in between"""
    best, run = 0, None
    for l in ins:
        if "WARPGROUP.ARRIVE" in l:
            run = 0
        elif "HGMMA" in l:
            if run is not None:
                run += 1
                if "gsb0" in l:
                    best = max(best, run)
                    run = None
    return best


@pytest.fixture(scope="module")
def functions():
    nvcc, cuobjdump = _tools()
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    return _instructions(_sass_text(nvcc, cuobjdump, [os.path.join(build.CSRC, src) for src in ("conv1d_gp.cu", "resblock_gp.cu")]))


@pytest.mark.parametrize("kernel", KERNELS)
def test_no_indirect_branch_between_mmas(functions, kernel):
    mine = {f: ins for f, ins in functions.items() if kernel in f}
    assert mine, "no %s in the SASS" % kernel
    bad = []
    for f, ins in mine.items():
        idx = [i for i, l in enumerate(ins) if "HGMMA" in l]
        assert idx, "%s issues no HGMMA" % f
        brx = [i for i in range(idx[0], idx[-1]) if re.search(r"\bBRX\b", ins[i])]
        if brx:
            bad.append("%s: %d BRX between its HGMMA" % (_params(kernel, f), len(brx)))
    assert not bad, "%s: the MMAs are issued through a jump table in %d of %d instantiations:\n  %s" % (
        kernel, len(bad), len(mine), "\n  ".join(bad))


@pytest.mark.parametrize("kernel", KERNELS)
def test_one_mma_width(functions, kernel):
    mine = {f: ins for f, ins in functions.items() if kernel in f}
    assert mine, "no %s in the SASS" % kernel
    bad = []
    for f, ins in mine.items():
        n = _params(kernel, f)[3]
        # ptxas closes a commit group that may be empty with a no-op `HGMMA.64x8x16 RZ, ..., !UPT`: not an MMA of the kernel
        widths = {int(w) for w in re.findall(r"HGMMA\.64x(\d+)x\S* R(?!Z)", "\n".join(ins))}
        if widths != {n}:
            bad.append("%s: HGMMA widths %s" % (_params(kernel, f), sorted(widths)))
    assert not bad, "%s: MMAs of another N than the instantiation's in %d of %d instantiations:\n  %s" % (
        kernel, len(bad), len(mine), "\n  ".join(bad))


@pytest.mark.parametrize("kernel", KERNELS)
def test_tap_is_one_chain(functions, kernel):
    mine = {f: ins for f, ins in functions.items() if kernel in f}
    assert mine, "no %s in the SASS" % kernel
    bad, checked = [], 0
    for f, ins in mine.items():
        mode, mt, kbg, n = _params(kernel, f)
        want = _chain_len(kernel, mode, mt, kbg, n)
        if want < 2:
            continue
        checked += 1
        got = _longest_chain(ins)
        if got < want:
            bad.append("<%d, %d, %d, %d>: longest chain %d HGMMA, a tap is %d" % (mode, mt, kbg, n, got, want))
    assert checked, "%s: no instantiation with a chain to check" % kernel
    assert not bad, "%s: a tap's MMAs are split by warpgroup.arrive in %d of %d instantiations:\n  %s" % (
        kernel, len(bad), checked, "\n  ".join(bad))
