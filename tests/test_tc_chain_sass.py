"""The acoustic model's GEMM kernel issues each tap's MMAs as one unbroken wgmma chain (host only: compiles conv1d_tc.cu for sm_90a
and reads the ptxas messages and the SASS; needs nvcc and cuobjdump, no GPU).

`conv1d_tc_kernel<MODE, MT, KBG, BN>` fixes the N width of its MMAs at compile time, so a tap of a full channel block is
KBG / 2 K steps x MT accumulators x m MMAs (m = 3 in 3xTF32 / bf16x3, else 1) between one `wgmma.fence` and one
`wgmma.commit_group` (DESIGN.md §3, §3.4).  With N chosen at run time every K step went through a jump table (`BRX`) and ptxas
fenced each 1- or 3-MMA fragment with a `warpgroup.arrive` of its own (warning C7519, 1,197 lines for conv1d_tc.cu).  So:
  * ptxas injects at most one warpgroup.arrive per instantiation: at the commit after the run-time K loop of a short last channel
    block (C_in not a multiple of the block, tc::tap_chain_short), a path the full blocks never take;
  * the instantiations are exactly the tiles the planner can return: every (MODE, KBG) of the shape rule, BN a multiple of 16
    up to 128, MT in {1, 2, 4} with MT * BN <= 128;
and in every instantiation:
  * no BRX lies between its first and last HGMMA;
  * every HGMMA has the instantiation's BN;
  * some run of HGMMA from a WARPGROUP.ARRIVE to the next HGMMA marked gsb0 (the commit) holds the whole tap of a full block;
  * and, here and in conv1d_gp_kernel, such a full tap's chain is followed by its WARPGROUP.DEPBAR with no further commit group in
    between (an empty group there makes `wgmma.wait_group 1` wait for the tap just issued).
"""
import os
import re
import subprocess
import tempfile

import pytest

from emotivoice_b200 import build
from test_epilogue_sass import _instructions
from test_wgmma_chain_sass import _longest_chain, _params
from test_wgmma_pipeline_sass import _sass_text, _tools

KERNEL = "conv1d_tc_kernel"
SRC = "conv1d_tc.cu"
MODE_KBG = ((0, 4), (0, 8), (1, 4), (2, 4), (2, 8), (3, 4), (3, 8))     # tc_shape_kbg: KBG = 4 in 3xTF32, else 8 when it fits


def _tiles():
    return {(mt, bn) for bn in range(16, 129, 16) for mt in (1, 2, 4) if mt * bn <= 128}


@pytest.fixture(scope="module")
def compiled():
    """(ptxas messages, mangled function name -> SASS instruction lines) of conv1d_tc.cu compiled with the build's flags"""
    nvcc, cuobjdump = _tools()
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    with tempfile.TemporaryDirectory() as tmp:
        out = os.path.join(tmp, "conv1d_tc.cubin")
        cmd = [nvcc] + [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")] + ["-I", build.INCLUDE, "-cubin",
                                                                                          os.path.join(build.CSRC, SRC), "-o", out]
        p = subprocess.run(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT, text=True)
        assert p.returncode == 0, p.stdout
        sass = subprocess.run([cuobjdump, "-sass", out], capture_output=True, text=True, check=True).stdout
    funcs = {f: ins for f, ins in _instructions(sass).items() if KERNEL in f}
    assert funcs, "no %s in the SASS" % KERNEL
    return p.stdout, funcs


def test_at_most_one_injected_warpgroup_arrive(compiled):
    log, funcs = compiled
    per = {}
    for l in log.splitlines():
        if "C7519" in l:
            m = re.search(r"function '(\S+)'", l)
            per[m.group(1) if m else l] = per.get(m.group(1) if m else l, 0) + 1
    bad = ["%s: %d" % (_params(KERNEL, f) if KERNEL in f else f, n) for f, n in per.items() if n > 1 or KERNEL not in f]
    assert not bad, "ptxas injected warpgroup.arrive more than once per instantiation in %s:\n  %s" % (SRC, "\n  ".join(bad))


def test_instantiations_are_the_plannable_tiles(compiled):
    _, funcs = compiled
    got = {_params(KERNEL, f) for f in funcs}
    want = {(mode, mt, kbg, bn) for mode, kbg in MODE_KBG for mt, bn in _tiles()}
    assert got == want, "missing %s, unexpected %s" % (sorted(want - got), sorted(got - want))


def test_no_indirect_branch_between_mmas(compiled):
    _, funcs = compiled
    bad = []
    for f, ins in funcs.items():
        idx = [i for i, l in enumerate(ins) if "HGMMA" in l]
        assert idx, "%s issues no HGMMA" % f
        brx = [i for i in range(idx[0], idx[-1]) if re.search(r"\bBRX\b", ins[i])]
        if brx:
            bad.append("%s: %d BRX between its HGMMA" % (_params(KERNEL, f), len(brx)))
    assert not bad, "the MMAs are issued through a jump table in %d of %d instantiations:\n  %s" % (len(bad), len(funcs), "\n  ".join(bad))


def test_one_mma_width(compiled):
    _, funcs = compiled
    bad = []
    for f, ins in funcs.items():
        n = _params(KERNEL, f)[3]
        # ptxas closes a commit group that may be empty with a no-op `HGMMA.64x8x16 RZ, ..., !UPT`: not an MMA of the kernel
        widths = {int(w) for w in re.findall(r"HGMMA\.64x(\d+)x\S* R(?!Z)", "\n".join(ins))}
        if widths != {n}:
            bad.append("%s: HGMMA widths %s" % (_params(KERNEL, f), sorted(widths)))
    assert not bad, "MMAs of another N than the instantiation's in %d of %d instantiations:\n  %s" % (len(bad), len(funcs), "\n  ".join(bad))


def _full_chain_then_wait(ins, want):
    """True if some run of `want` or more HGMMA from a WARPGROUP.ARRIVE to a gsb0 HGMMA is followed by a WARPGROUP.DEPBAR before
    any further HGMMA.  Where the full and short block paths join before the commit, the commit opens a second, empty group that
    ptxas closes with a no-op `HGMMA.64x8x16 RZ ... gsb0` after the chain: `wgmma.wait_group 1` then waits for the tap's own MMAs."""
    run, closed = None, False
    for l in ins:
        if "WARPGROUP.ARRIVE" in l and not closed:
            run = 0
        elif "HGMMA" in l:
            if closed:
                closed, run = False, None
            if run is not None:
                run += 1
                if "gsb0" in l:
                    closed, run = run >= want, None
        elif "WARPGROUP.DEPBAR" in l and closed:
            return True
    return False


@pytest.fixture(scope="module")
def gp_functions():
    nvcc, cuobjdump = _tools()
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    funcs = _instructions(_sass_text(nvcc, cuobjdump, [os.path.join(build.CSRC, "conv1d_gp.cu")]))
    return {f: ins for f, ins in funcs.items() if "conv1d_gp_kernel" in f}


def test_full_tap_is_one_commit_group(compiled, gp_functions):
    _, funcs = compiled
    bad, checked = [], 0
    for kernel, fs in ((KERNEL, funcs), ("conv1d_gp_kernel", gp_functions)):
        for f, ins in fs.items():
            mode, mt, kbg, n = _params(kernel, f)
            if kernel == KERNEL:
                nk8 = kbg // 2                       # conv1d_tc stages bf16x3 operands as bf16: two granules per K step in every mode
            else:
                nk8 = (8 if mode == 2 else 4) * kbg // (2 * (8 if mode >= 2 else 4))   # conv1d_gp's bf16x3 stages fp32 granules
            want = nk8 * mt * (3 if mode in (1, 3) else 1)
            checked += 1
            if not _full_chain_then_wait(ins, want):
                bad.append("%s<%d, %d, %d, %d>" % (kernel, mode, mt, kbg, n))
    assert checked
    assert not bad, "a full tap's chain is not followed by its wait (an extra commit group in between) in %d of %d:\n  %s" % (
        len(bad), checked, "\n  ".join(bad))


def test_tap_is_one_chain(compiled):
    _, funcs = compiled
    bad = []
    for f, ins in funcs.items():
        mode, mt, kbg, n = _params(KERNEL, f)
        want = kbg // 2 * mt * (3 if mode in (1, 3) else 1)
        got = _longest_chain(ins)
        if got < want:
            bad.append("<%d, %d, %d, %d>: longest chain %d HGMMA, a tap is %d" % (mode, mt, kbg, n, got, want))
    assert not bad, "a tap's MMAs are split by warpgroup.arrive in %d of %d instantiations:\n  %s" % (len(bad), len(funcs), "\n  ".join(bad))
