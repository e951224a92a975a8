"""Host side of emotivoice_b200.feats (log-mel spectrograms and frame energy): the oracle against the reference fixtures
(oracle/make_golden_feats.py), the restated librosa mel basis, the kernel's band table, frame counts and argument errors.
No GPU needed: every error here is raised before anything is enqueued."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from emotivoice_b200 import feats
from oracle import feats_oracle as FO

NAMES = ["tone", "chirp", "noise_m20", "noise_m60", "silence", "square", "b1_t100"]


def _fixture(name):
    with np.load(os.path.join(GOLDEN, "feats_%s.npz" % name)) as z:
        return {k: z[k] for k in z.files}


def _basis():
    return feats.mel_filterbank(sr=16000, n_fft=1024, n_mels=80, fmin=0.0, fmax=8000.0)


@pytest.mark.parametrize("name", NAMES)
def test_oracle_reproduces_reference_fixture(name):
    g = _fixture(name)
    y = g["wav"]
    assert np.array_equal(FO.tacotron_mel(y, 256)[0], g["taco_mel"])
    assert np.array_equal(FO.mel_spectrogram(y, 256)[0], g["mt_mel"])
    assert np.array_equal(FO.energy(y, 256), g["energy"])
    basis = _basis()
    assert np.allclose(FO.tacotron64(y, 256, basis)["logmel"], g["taco_mel64"], rtol=0, atol=1e-12)
    assert np.allclose(FO.mel_spectrogram64(y, 256, basis)["logmel"], g["mt_mel64"], rtol=0, atol=1e-12)
    assert np.allclose(FO.energy64(y, 256), g["energy64"], rtol=0, atol=1e-12)
    assert np.array_equal(g["taco_dev"], np.abs(g["taco_mel"] - g["taco_mel64"]))


def test_b1_t100_fixture_is_the_model_waveform():
    g = _fixture("b1_t100")
    with np.load(os.path.join(GOLDEN, "b1_t100.npz")) as z:
        wav = z["wav"].reshape(-1)
    a, b = g["span"].tolist()
    assert np.array_equal(g["wav"], wav[a:b])


def test_mel_filterbank_matches_fixture_basis_and_torchaudio():
    basis = _basis()
    assert basis.dtype == np.float32 and basis.shape == (80, 513)
    assert int((basis != 0).sum()) == 1001
    assert np.array_equal(basis, _fixture("b1_t100")["mel_basis"])
    ta = pytest.importorskip("torchaudio")
    ref = ta.functional.melscale_fbanks(513, 0.0, 8000.0, 80, 16000, norm="slaney", mel_scale="slaney").T.numpy()
    assert np.abs(basis - ref).max() <= 1e-7
    assert np.array_equal(basis > 0, ref > 0)


@pytest.mark.parametrize("sr,n_mels,fmax", [(16000, 80, 8000.0), (22050, 80, 8000.0), (16000, 128, None), (24000, 100, 12000.0)])
def test_band_table_rebuilds_the_dense_basis(sr, n_mels, fmax):
    basis = feats.mel_filterbank(sr=sr, n_fft=1024, n_mels=n_mels, fmin=0.0, fmax=fmax)
    bands, w = feats.band_table(basis)
    assert bands.dtype == np.int32 and bands.shape == (n_mels, 3) and w.dtype == np.float32
    dense = np.zeros_like(basis)
    off = 0
    for j, (first, cnt, o) in enumerate(bands.tolist()):
        assert o == off and 0 <= first and first + cnt <= basis.shape[1]
        dense[j, first:first + cnt] = w[o:o + cnt]
        if cnt:
            assert basis[j, first] != 0 and basis[j, first + cnt - 1] != 0
        off += cnt
        nz = np.nonzero(basis[j])[0]
        assert (nz.size == 0 and cnt == 0) or (nz[0] == first and nz[-1] == first + cnt - 1)
    assert np.array_equal(dense, basis)


def test_frame_counts():
    for n in (385, 1000, 4000, 4096, 137472):
        for hop in (160, 256):
            assert feats.n_frames(n, 512, hop) == n // hop + 1
            p = (1024 - hop) // 2
            x = torch.zeros(1, n + 2 * p)
            nfr = torch.stft(x, 1024, hop_length=hop, window=torch.hann_window(1024), center=False, return_complex=True).shape[-1]
            assert feats.n_frames(n, p, hop) == nfr
    g = _fixture("b1_t100")
    assert g["taco_mel"].shape[1] == feats.n_frames(len(g["wav"]), 512, 256) == len(g["energy"])
    assert g["mt_mel"].shape[1] == feats.n_frames(len(g["wav"]), 384, 256)


def test_twiddles_and_windows():
    tw = feats.twiddles()
    assert tw.dtype == np.float32 and tw.shape == (1024, 2)
    k = np.arange(1024)
    assert np.array_equal(tw[:, 0], np.cos(2 * np.pi * k / 1024).astype(np.float32))
    w = feats.hann_window_scipy()
    assert w.dtype == np.float32 and w[0] == 0 and np.abs(w.astype(np.float64) - (0.5 - 0.5 * np.cos(2 * np.pi * k / 1024))).max() < 1e-7


def test_cpu_tensors_raise_runtime_error():
    y = torch.zeros(1, 4000)
    with pytest.raises(RuntimeError, match="CUDA"):
        feats.TacotronSTFT(sampling_rate=16000).mel_spectrogram(y)
    with pytest.raises(RuntimeError, match="CUDA"):
        feats.mel_spectrogram_torch(y, 1024, 80, 16000, 256, 1024, 0, 8000)
    with pytest.raises(RuntimeError, match="CUDA"):
        feats.Energy(sr=16000, n_fft=1024, hop_length=256).get_energy(y[0])


def test_unsupported_configurations_raise_value_error():
    with pytest.raises(ValueError, match="1024"):
        feats.TacotronSTFT(filter_length=2048)
    with pytest.raises(ValueError, match="1024"):
        feats.TacotronSTFT(win_length=800)
    with pytest.raises(ValueError, match="1024"):
        feats.Energy()                                                # the reference's default n_fft = 2048
    with pytest.raises(ValueError, match="center=True"):
        feats.Energy(n_fft=1024, hop_length=256, center=False)
    with pytest.raises(ValueError, match="reflect"):
        feats.Energy(n_fft=1024, hop_length=256, pad_mode="constant")
    with pytest.raises(ValueError, match="hann"):
        feats.Energy(n_fft=1024, hop_length=256, window="hamming")
    with pytest.raises(ValueError, match=r"\[1, 1024\]"):
        feats.TacotronSTFT(hop_length=0)
    with pytest.raises(ValueError, match=r"\[1, 1024\]"):
        feats.Energy(n_fft=1024, hop_length=1025)


def test_short_items_and_bad_lengths_raise(monkeypatch):
    """The length checks run on host ints before the device is touched (the CUDA check is bypassed here)."""
    monkeypatch.setattr(feats, "_check", lambda t, name: None)
    win = torch.zeros(1024)
    with pytest.raises(RuntimeError, match="not longer than the reflect padding"):
        feats.stft_features(torch.zeros(2, 512), 512, 256, win, 0.0, energy=True)
    with pytest.raises(RuntimeError, match="not longer than the reflect padding"):
        feats.stft_features(torch.zeros(2, 600), 512, 256, win, 0.0, energy=True, lengths=[600, 512])
    with pytest.raises(RuntimeError, match="shorter than the 1024-point frame"):
        feats.mel_spectrogram_torch(torch.zeros(1, 13), 1024, 80, 16000, 1000, 1024, 0, 8000)
    with pytest.raises(ValueError, match="exceeds"):
        feats.stft_features(torch.zeros(2, 600), 512, 256, win, 0.0, energy=True, lengths=torch.tensor([601, 600]))
    with pytest.raises(ValueError, match="2 items"):
        feats.stft_features(torch.zeros(2, 600), 512, 256, win, 0.0, energy=True, lengths=[600])
    with pytest.raises(ValueError, match="center=True is not supported"):
        feats.mel_spectrogram_torch(torch.zeros(1, 4000), 1024, 80, 16000, 256, 1024, 0, 8000, center=True)
    with pytest.raises(ValueError, match="1024"):
        feats.mel_spectrogram_torch(torch.zeros(1, 4000), 2048, 80, 16000, 256, 2048, 0, 8000)
    with pytest.raises(ValueError, match="mel bands"):
        feats.device_bands(feats.mel_filterbank(sr=16000, n_fft=1024, n_mels=129), "cpu")
    with pytest.raises(ValueError, match="1-D waveform"):
        feats.Energy(sr=16000, n_fft=1024, hop_length=256).get_energy(torch.zeros(2, 4000), duration=np.ones(3, np.int64))
