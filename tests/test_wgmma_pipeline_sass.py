"""The convolution kernels' wgmma pipeline exists in the binary (host only: reads the compiled sm_90a SASS, needs no GPU).

The consumers issue a K step's MMAs, commit them and wait with `wgmma.wait_group 1`, so the tensor core always has the next step
queued while the previous one drains (DESIGN.md §3).  When ptxas cannot prove that a wgmma is issued by the whole warpgroup it
serialises every one of them instead (warning C7520): each HGMMA is followed by its own WARPGROUP.DEPBAR, and the MMAs run one at
a time with the same results.  So in every instantiation of the three convolution kernels the number of WARPGROUP.DEPBAR must not
exceed the number of `wgmma_wait<N>()` sites in its source file.

The in-tree library is used when it is current; otherwise the three sources are compiled to cubins in a temporary directory.
"""
import os
import re
import shutil
import subprocess
import tempfile
from collections import OrderedDict

import pytest

from emotivoice_b200 import build

KERNELS = OrderedDict([("conv1d_gp_kernel", "conv1d_gp.cu"), ("resblock_gp_kernel", "resblock_gp.cu"), ("conv1d_tc_kernel", "conv1d_tc.cu")])


def _tools():
    nvcc = build.nvcc_path()
    nvcc = nvcc if os.path.isabs(nvcc) else shutil.which(nvcc)
    if not nvcc or not os.path.exists(nvcc):
        return None, None
    cuobjdump = os.path.join(os.path.dirname(nvcc), "cuobjdump")
    if not os.path.exists(cuobjdump):
        cuobjdump = shutil.which("cuobjdump")
    return nvcc, cuobjdump


def _sass_text(nvcc, cuobjdump, sources):
    """SASS of the in-tree library when it is current, else of `sources` (paths of .cu files) compiled to cubins"""
    if build._up_to_date(build._digest()):
        return subprocess.run([cuobjdump, "-sass", build.LIB_PATH], capture_output=True, text=True, check=True).stdout
    with tempfile.TemporaryDirectory() as tmp:
        procs = []
        for src in sources:
            out = os.path.join(tmp, os.path.basename(src)[:-3] + ".cubin")
            cmd = [nvcc] + [f for f in build.NVCC_FLAGS if f not in ("-cudart", "static")] + ["-I", build.INCLUDE, "-cubin", src, "-o", out]
            procs.append((out, subprocess.Popen(cmd, stdout=subprocess.PIPE, stderr=subprocess.STDOUT)))
        text = []
        for out, p in procs:
            log, _ = p.communicate()
            assert p.returncode == 0, log.decode()
            text.append(subprocess.run([cuobjdump, "-sass", out], capture_output=True, text=True, check=True).stdout)
        return "\n".join(text)


def _per_function(sass):
    """mangled function name -> [WARPGROUP.DEPBAR count, HGMMA count]"""
    funcs, cur = OrderedDict(), None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            cur = funcs.setdefault(m.group(1), [0, 0])
            continue
        if cur is None:
            continue
        if "WARPGROUP.DEPBAR" in line:
            cur[0] += 1
        if "HGMMA" in line:
            cur[1] += 1
    return funcs


def _wait_sites(src):
    with open(os.path.join(build.CSRC, src)) as f:
        return len(re.findall(r"wgmma_wait<\d+>\(\)", f.read()))


@pytest.fixture(scope="module")
def functions():
    nvcc, cuobjdump = _tools()
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    return _per_function(_sass_text(nvcc, cuobjdump, [os.path.join(build.CSRC, src) for src in KERNELS.values()]))


@pytest.mark.parametrize("kernel", list(KERNELS))
def test_wgmma_not_serialised(functions, kernel):
    sites = _wait_sites(KERNELS[kernel])
    assert sites >= 1
    mine = {f: v for f, v in functions.items() if kernel in f}
    assert mine, "no %s in the SASS" % kernel
    bad = []
    for f, (depbar, hgmma) in mine.items():
        assert hgmma > 0, "%s issues no HGMMA" % f
        if depbar > sites:
            bad.append("%s: %d WARPGROUP.DEPBAR for %d HGMMA" % (f, depbar, hgmma))
    assert not bad, ("ptxas serialised the wgmma pipeline (more WARPGROUP.DEPBAR than the source's %d wgmma_wait sites) in %d of %d "
                     "instantiations:\n  %s" % (sites, len(bad), len(mine), "\n  ".join(bad)))
