"""Every kernel of the library waits for the grid before it (host only: reads the compiled sm_90a SASS, needs no GPU).

The engine launches every kernel through one helper that sets programmatic stream serialization (ev_common.cuh: launch), so a
kernel may start while its predecessor in the stream is still running.  Each kernel therefore executes
griddepcontrol.launch_dependents and griddepcontrol.wait (SASS: PREEXIT and ACQBULK) before it touches memory a predecessor
writes; a kernel without the wait would race its predecessor.  So every function in the library must contain both.

The in-tree library is used when it is current; otherwise every source of the library is compiled to a cubin in a temporary
directory.
"""
import pytest

from emotivoice_b200 import build
from test_epilogue_sass import _instructions
from test_wgmma_pipeline_sass import _sass_text, _tools


@pytest.fixture(scope="module")
def functions():
    nvcc, cuobjdump = _tools()
    if not nvcc or not cuobjdump:
        pytest.skip("needs nvcc and cuobjdump")
    return _instructions(_sass_text(nvcc, cuobjdump, build.sources()))


def test_every_kernel_waits_for_its_predecessor(functions):
    assert functions, "no function in the SASS"
    bad = [f for f, ins in functions.items()
           if not (any("PREEXIT" in l for l in ins) and any("ACQBULK" in l for l in ins))]
    assert not bad, "%d of %d functions lack PREEXIT (griddepcontrol.launch_dependents) or ACQBULK (griddepcontrol.wait):\n  %s" % (
        len(bad), len(functions), "\n  ".join(bad))
