"""feats.Pitch on the host: the fp64 restatement of pyworld.dio / pyworld.stonemask (oracle/pitch_oracle.py) against the
fixtures made with the reference's own glue (oracle/make_golden_pitch.py), its accuracy on signals of known F0, frame counts and
the argument errors raised before anything reaches the device."""
import glob
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from emotivoice_b200 import feats
from oracle import pitch_oracle as PO

FIXTURES = sorted(os.path.basename(p)[6:-4] for p in glob.glob(os.path.join(GOLDEN, "pitch_*.npz")))
KNOWN = ["stat90", "stat150", "stat220", "stat330", "vibrato", "glide", "sr24k"]


def load(name):
    with np.load(os.path.join(GOLDEN, "pitch_%s.npz" % name)) as z:
        return {k: z[k] for k in z.files}


def core_frames(known, edge=3):
    """Frames with a known F0 at least `edge` frames from a voicing edge or an end of the item."""
    v = known > 0
    F = len(v)
    core = np.zeros(F, bool)
    for i in range(edge, F - edge):
        core[i] = v[i - edge:i + edge + 1].all()
    return core


def test_fixture_set():
    assert len(FIXTURES) == 10 and set(KNOWN) <= set(FIXTURES) and {"noise", "b1_t100", "alternate"} <= set(FIXTURES)


@pytest.mark.parametrize("name", FIXTURES)
def test_oracle_reproduces_fixture(name):
    z = load(name)
    x, sr, hop = z["wav"].astype(np.float64), int(z["sr"]), int(z["hop"])
    f0, t = PO.dio(x, sr, 1000 * hop / sr)
    assert np.array_equal(f0, z["f0_dio"])
    ref = PO.stonemask(x, f0, t, sr)
    assert np.array_equal(ref, z["f0_refined"])
    cont = PO.continuous(ref)
    assert np.array_equal(cont, z["continuous"])
    assert np.array_equal(PO.log_pitch(cont), z["log"])
    assert np.array_equal(PO.log_pitch(ref), z["log_raw"])
    assert np.array_equal(PO.average_by_duration(cont, z["durations"]), z["token_avg"])


@pytest.mark.parametrize("name", KNOWN)
def test_known_f0_accuracy(name):
    """Refined track within 1 % of the known F0 at every voiced frame 3 or more frames from a voicing edge; those frames all voiced."""
    z = load(name)
    core = core_frames(z["known_f0"])
    assert core.sum() >= 40
    ref = z["f0_refined"]
    assert (ref[core] > 0).all(), np.nonzero(core & (ref == 0))[0]
    err = np.abs(ref[core] / z["known_f0"][core] - 1)
    assert err.max() <= 0.01, (err.max(), np.nonzero(core)[0][np.argmax(err)])


def test_noise_and_silence_are_unvoiced():
    z = load("noise")
    assert not z["f0_dio"].any() and not z["continuous"].any() and not z["log"].any()
    f0, t = PO.dio(np.zeros(8000), 16000, 16.0)
    assert f0.shape == (32,) and not f0.any() and not PO.stonemask(np.zeros(8000), f0, t, 16000).any()


def test_frame_counts():
    for n in list(range(640, 1200)) + [160000, 480000, 480001]:
        assert feats.pitch_frames(n, 16000, 256) == n // 256 + 1 == PO.frame_count(n, 16000, 16.0)
        assert feats.pitch_frames(n, 24000, 300) == n // 300 + 1 == PO.frame_count(n, 24000, 12.5)
    assert feats.pitch_frame_period(16000, 256) == 16.0 and feats.pitch_frame_period(24000, 300) == 12.5
    assert feats.pitch_min_samples(16000) == 641 and feats.pitch_min_samples(48000) == 1921


def test_band_layout():
    assert PO.n_bands() == 7
    assert PO.band_half_lengths(16000)[0] == 319 and PO.band_half_lengths(48000)[0] == 956
    assert PO.voice_range_minimum(16.0) == 3 and PO.voice_range_minimum(12.5) == 3


@pytest.mark.parametrize("sr,hop", [(7999, 256), (48001, 256), (22050.5, 256), (16000, 15), (16000, 4097), (16000, 256.5)])
def test_unsupported_config_raises(sr, hop):
    with pytest.raises(ValueError):
        feats.Pitch(sr=sr, hop_length=hop)


def test_supported_configs():
    for sr, hop in ((16000, 256), (22050, 256), (24000, 300), (48000, 300), (8000, 16), (48000, 4096)):
        p = feats.Pitch(sr=sr, hop_length=hop, pitch_min=1, pitch_max=2)
        assert (p.sr, p.hop_length, p.pitch_min, p.pitch_max) == (sr, hop, 1, 2)
    assert (feats.Pitch().sr, feats.Pitch().hop_length, feats.Pitch().pitch_min, feats.Pitch().pitch_max) == (24000, 300, 80, 7600)


def test_cpu_tensor_raises():
    with pytest.raises(RuntimeError):
        feats.Pitch(sr=16000, hop_length=256).get_pitch(torch.zeros(4000))
    with pytest.raises(RuntimeError):
        feats.pitch_track(torch.zeros(2, 4000, dtype=torch.float64), 16000, 256)
