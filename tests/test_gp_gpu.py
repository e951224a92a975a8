"""Granule-planar HiFi-GAN convolution kernel (csrc/conv1d_gp.cu) on the H100.

* operator level: tests/test_voc_kernels_gpu.py (every kernel and mode against fp64, plus the bitwise cross-checks);
* end to end: the vocoder on the GP path (the default) is BITWISE the round-1 time-major path (EV_VOC_LAYOUT=tm) in the
  tf32 mode and, with EV_VOC_FP32=tf32x3 on both sides, in the fp32 mode; bf16 storage against the unmodified reference's fixture within the bf16 tolerance."""
import os
import subprocess
import sys

import numpy as np
import pytest
import torch

from conftest import GOLDEN, ROOT, load_golden, rel_max, rel_rms

pytestmark = pytest.mark.gpu
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")


_TM_CHILD = r"""
import sys, numpy as np, torch
sys.path.insert(0, sys.argv[1])
from emotivoice_b200.config import default_config
from emotivoice_b200 import synth
from emotivoice_b200.modules import JETSGenerator
conf = default_config()
m = JETSGenerator(conf).to("cuda:0"); m.load_state_dict(synth.make_state_dict(conf)); m.eval()
z = np.load(sys.argv[2])
keys = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")
res = {}
for prec in ("fp32", "tf32"):
    m.precision = prec
    out = m(**{k: torch.from_numpy(z[k]).cuda() for k in keys})
    torch.cuda.synchronize()
    res[prec + "_wav"] = out["wav_predictions"].cpu().numpy(); res[prec + "_lens"] = out["mel_lengths"].cpu().numpy()
np.savez(sys.argv[3], **res)
"""


def test_vocoder_on_the_gp_path_is_bitwise_the_time_major_path(model, dev, tmp_path):
    src, dst = os.path.join(GOLDEN, "b3_padded.npz"), str(tmp_path / "tm.npz")
    subprocess.run([sys.executable, "-c", _TM_CHILD, ROOT, src, dst], env=dict(os.environ, EV_VOC_LAYOUT="tm"), check=True, timeout=300)
    got = np.load(dst)
    g = load_golden("b3_padded")
    try:
        # the fp32 mode of the GP path defaults to the bf16x3 emulation (not the same arithmetic as 3xTF32): compare it within the fp32
        # tolerance here; the bitwise 3xTF32 comparison is the operator-level check (tests/test_voc_kernels_gpu.py) plus the tf32 mode below
        model.precision = "fp32"
        out = model(**{k: g[k].to(dev) for k in KEYS})
        for b, n in enumerate(got["fp32_lens"].tolist()):
            a, r = out["wav_predictions"][b, 0, :n * 256].cpu(), torch.from_numpy(got["fp32_wav"][b, 0, :n * 256])
            assert rel_rms(a, r) <= 1e-4
        for prec in ("tf32",):
            model.precision = prec
            out = model(**{k: g[k].to(dev) for k in KEYS})
            wav = out["wav_predictions"].cpu().numpy()
            for b, n in enumerate(got[prec + "_lens"].tolist()):        # the GP path leaves rows >= len of its scratch undefined; the waveform is zero there in both
                assert np.array_equal(wav[b, 0, :n * 256], got[prec + "_wav"][b, 0, :n * 256]), (prec, b)
                assert not wav[b, 0, n * 256:].any()
    finally:
        model.precision = "fp32"


@pytest.mark.parametrize("name", ["b1_t12", "b1_t50", "b1_t100"])
def test_bf16_storage_mode_against_the_reference_fixture(model, dev, name):
    """ "bf16": bf16 operands AND bf16 activations in HBM through the vocoder (fp32 accumulation; the duration prefix
    stays 3xTF32, so durations are identical).  Tolerance (SURVEY.md s8d cfg3): mel <= 2e-2 of max|mel|, wav rms <= 2e-2 of rms."""
    g = load_golden(name)
    try:
        model.precision = "bf16"
        out = model(**{k: g[k].to(dev) for k in KEYS})
        assert torch.equal(out["log_duration_predictions"].cpu(), g["durations"])
        e_mel, e_wav = rel_max(out["dec_outputs"].cpu(), g["mel"]), rel_rms(out["wav_predictions"].cpu(), g["wav"])
        print(name, "bf16 storage: mel rel-max %.2e wav rel-rms %.2e" % (e_mel, e_wav))
        assert e_mel <= 2e-2 and e_wav <= 2e-2
    finally:
        model.precision = "fp32"


def test_generator_alone_takes_channels_first_mel_on_the_gp_path(model, dev):
    """hifigan/models.py:115: Generator.forward takes (B, n_mels, F); the GP boundary kernel reads it with strides."""
    g = load_golden("voc_b2_f40")
    wav = model.generator(g["mel"].to(dev))
    assert rel_rms(wav.cpu(), g["wav"]) <= 1e-4
