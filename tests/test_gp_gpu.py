"""Granule-planar HiFi-GAN convolution kernel (csrc/conv1d_gp.cu) on the H100.

* operator level: tests/test_voc_kernels_gpu.py (every kernel and mode against fp64, plus the bitwise cross-checks, among them
  GP == the time-major tensor-core kernel);
* end to end: bf16 storage against the unmodified reference's fixture within the bf16 tolerance, and the weight copies each
  precision needs checked when the blob is bound."""
import pytest
import torch

from conftest import load_golden, rel_max, rel_rms

pytestmark = pytest.mark.gpu
KEYS = ("inputs_ling", "input_lengths", "inputs_speaker", "inputs_style_embedding", "inputs_content_embedding")


def test_blob_without_its_bf16x3_copies_is_refused_for_fp32(conf, sd, dev, lib):
    """ "fp32" runs the decoder, to_mel and the vocoder on the two-plane bf16 copies ('.tc16x2'): a blob without them is refused
    when it is bound for "fp32" and when "fp32" is chosen for it later, instead of running those layers on another kernel."""
    from emotivoice_b200 import _abi, packing
    from emotivoice_b200.modules import _Engine
    packed = {k: v for k, v in packing.add_tc_weights(packing.pack_state_dict(sd, conf)).items() if not k.endswith(".tc16x2")}
    with pytest.raises(_abi.EvError) as e:
        _Engine(conf, packed, dev, "fp32")
    assert e.value.code == _abi.EV_ENOWEIGHT and ".tc16x2" in str(e.value)
    eng = _Engine(conf, packed, dev, "tf32")          # every copy "tf32" reads is there
    with pytest.raises(_abi.EvError) as e:
        eng.set_precision("fp32")
    assert e.value.code == _abi.EV_ENOWEIGHT and eng.precision == "tf32"


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
