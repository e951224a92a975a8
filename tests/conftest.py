import json
import os
import sys

import numpy as np
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
if ROOT not in sys.path:
    sys.path.insert(0, ROOT)

GOLDEN = os.path.join(ROOT, "tests", "golden")


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (an H100, sm_90a)")


def pytest_collection_modifyitems(config, items):
    """`gpu` tests need a CUDA device AND the in-tree library: on a host without one they are skipped, not errors, so a
    bare `pytest` is green on a machine without a GPU."""
    if torch.cuda.is_available():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (sm_90a); there is no CPU path")
    for it in items:
        if "gpu" in it.keywords:
            it.add_marker(skip)


@pytest.fixture(scope="session")
def conf():
    from emotivoice_b200.config import default_config
    return default_config()


@pytest.fixture(scope="session")
def sd(conf):
    from emotivoice_b200 import synth
    return synth.make_state_dict(conf)


@pytest.fixture(scope="session")
def golden_meta():
    with open(os.path.join(GOLDEN, "meta.json")) as f:
        return json.load(f)


def load_golden(name):
    z = np.load(os.path.join(GOLDEN, name + ".npz"))
    return {k: torch.from_numpy(z[k]) for k in z.files}


@pytest.fixture(scope="session")
def lib():
    from emotivoice_b200 import build, _abi
    build.build(verbose=False)
    return _abi.load()


@pytest.fixture(scope="session")
def dev():
    assert torch.cuda.is_available()
    return torch.device("cuda:0")


@pytest.fixture(scope="session")
def model(conf, sd, dev, lib):
    from emotivoice_b200.modules import JETSGenerator
    m = JETSGenerator(conf).to(dev)
    m.load_state_dict(sd)
    return m.eval()


def rel_max(a, b):
    return (a - b).abs().max().item() / max(b.abs().max().item(), 1e-30)


def rel_rms(a, b):
    return ((a - b).double().pow(2).mean().sqrt() / b.double().pow(2).mean().sqrt().clamp_min(1e-30)).item()
