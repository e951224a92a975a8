"""TEST INFRASTRUCTURE ONLY -- torch-CPU restatements of the reference's three feature computations, and their fp64
counterparts for the operator checks of emotivoice_b200.feats.

  tacotron_mel         TacotronSTFT.mel_spectrogram (tacotron_stft.py:71-80, stft.py:98-160, audio_processing.py:50-51)
  mel_spectrogram      mel_process.mel_spectrogram_torch (mel_process.py:77-110)
  energy               feats.Energy.get_energy (feats.py:178-213)

librosa is absent from this environment.  Its two pieces the reference uses are restated: ``librosa.filters.mel`` by
``emotivoice_b200.feats.mel_filterbank`` (checked against torchaudio's ``melscale_fbanks``) and ``librosa.stft`` by
``librosa_stft`` below (checked against ``torch.stft(center=True)``).  Neither is checked against librosa itself.

The fp64 counterparts frame the fp64-cast signal exactly like the variant (same padding and hop), multiply by the variant's
fp32 window cast to fp64 and take numpy's fp64 rfft.  ``frame_l1`` gives m_f = sum_n |w_n x_n| per frame, the scale of the
operator-check bounds.
"""
import numpy as np
import torch
import torch.nn.functional as F

from emotivoice_b200.feats import N_FFT, hann_window_scipy, mel_filterbank


def _rows(y):
    y = np.asarray(y, dtype=np.float32)
    return y[None] if y.ndim == 1 else y


def tacotron_mel(y, hop=256, sr=16000, n_mels=80, fmin=0.0, fmax=8000.0):
    """(B, N) float32 -> (B, n_mels, N // hop + 1) float32, the reference's operations on torch CPU."""
    y = torch.from_numpy(_rows(y))
    B, N = y.shape
    fb = np.fft.fft(np.eye(N_FFT))
    cutoff = N_FFT // 2 + 1
    fb = np.vstack([np.real(fb[:cutoff, :]), np.imag(fb[:cutoff, :])])
    basis = torch.FloatTensor(fb[:, None, :]) * torch.from_numpy(hann_window_scipy())       # stft.py:114-126
    x = F.pad(y.view(B, 1, N).unsqueeze(1), (N_FFT // 2, N_FFT // 2, 0, 0), mode="reflect").squeeze(1)
    ft = F.conv1d(x, basis, stride=hop, padding=0)
    mag = torch.sqrt(ft[:, :cutoff, :] ** 2 + ft[:, cutoff:, :] ** 2)
    mel_basis = torch.from_numpy(mel_filterbank(sr=sr, n_fft=N_FFT, n_mels=n_mels, fmin=fmin, fmax=fmax)).float()
    return torch.log(torch.clamp(torch.matmul(mel_basis, mag), min=1e-5)).numpy()


def mel_spectrogram(y, hop=256, sr=16000, n_mels=80, fmin=0.0, fmax=8000.0):
    """(B, N) float32 -> (B, n_mels, (N + 2p - 1024) // hop + 1), p = (1024 - hop) // 2: mel_process.py:99-110 on torch CPU."""
    y = torch.from_numpy(_rows(y))
    p = int((N_FFT - hop) / 2)
    x = F.pad(y.unsqueeze(1), (p, p), mode="reflect").squeeze(1)
    spec = torch.stft(x, N_FFT, hop_length=hop, win_length=N_FFT, window=torch.hann_window(N_FFT), center=False, pad_mode="reflect",
                      normalized=False, onesided=True, return_complex=True)
    spec = torch.view_as_real(spec)
    spec = torch.sqrt(spec.pow(2).sum(-1) + 1e-6)
    mel_basis = torch.from_numpy(mel_filterbank(sr=sr, n_fft=N_FFT, n_mels=n_mels, fmin=fmin, fmax=fmax))
    return torch.log(torch.clamp(torch.matmul(mel_basis, spec), min=1e-5)).numpy()


def librosa_stft(y, n_fft=2048, hop_length=None, win_length=None, window="hann", center=True, pad_mode="constant", **_):
    """The arithmetic of librosa.stft for a float32 signal: reflect pad n_fft // 2 at both ends (center), periodic Hann window
    (scipy get_window, fftbins=True) in fp64 times the fp32 frames, fp64 rfft, stored as complex64.  (1 + n_fft // 2, F)."""
    from scipy.signal import get_window
    y = np.asarray(y)
    if win_length is None:
        win_length = n_fft
    if hop_length is None:
        hop_length = win_length // 4
    w = get_window(window, win_length, fftbins=True)
    lp = (n_fft - win_length) // 2
    w = np.pad(w, (lp, n_fft - win_length - lp))
    if center:
        y = np.pad(y, (n_fft // 2, n_fft // 2), mode=pad_mode)
    nfr = 1 + (len(y) - n_fft) // hop_length
    idx = np.arange(n_fft)[:, None] + hop_length * np.arange(nfr)[None, :]
    return np.fft.rfft(w[:, None] * y[idx], axis=0).astype(np.complex64)


def energy(wav, hop=256):
    """1-D float32 -> (N // hop + 1,) float32: feats.py:188-196 with librosa_stft."""
    x = np.asarray(wav).astype(np.float32)
    power = np.abs(librosa_stft(x, n_fft=N_FFT, hop_length=hop, win_length=N_FFT, window="hann", center=True, pad_mode="reflect")) ** 2
    return np.sqrt(np.clip(np.sum(power, axis=0), a_min=1.0e-10, a_max=float("inf")))


# ---- fp64 counterparts ------------------------------------------------------------------------------------------------------

def frames64(y, pad, hop):
    """(N,) -> (F, 1024) fp64 frames of the reflect-padded signal."""
    x = np.pad(np.asarray(y, dtype=np.float64), (pad, pad), mode="reflect")
    nfr = (len(x) - N_FFT) // hop + 1
    return x[np.arange(N_FFT)[None, :] + hop * np.arange(nfr)[:, None]]


def spectrum64(y, pad, hop, window):
    """-> (X (F, 513) complex128, m_f (F,) = sum_n |w_n x_n|)."""
    fr = frames64(y, pad, hop) * np.asarray(window, dtype=np.float64)[None, :]
    return np.fft.rfft(fr, axis=1), np.abs(fr).sum(axis=1)


def features64(y, pad, hop, window, mag_eps, basis):
    """-> dict of fp64 results of one item: mel (n_mels, F) before the log, logmel, energy (F,), m_f (F,)."""
    X, m = spectrum64(y, pad, hop, window)
    p = X.real ** 2 + X.imag ** 2
    mel = np.asarray(basis, dtype=np.float64) @ np.sqrt(p + mag_eps).T
    return {"mel": mel, "logmel": np.log(np.maximum(mel, 1e-5)), "energy": np.sqrt(np.maximum(p.sum(axis=1), 1e-10)), "m_f": m}


def tacotron64(y, hop=256, basis=None):
    return features64(y, N_FFT // 2, hop, hann_window_scipy(), 0.0, basis)


def mel_spectrogram64(y, hop=256, basis=None):
    return features64(y, (N_FFT - hop) // 2, hop, torch.hann_window(N_FFT).numpy(), 1e-6, basis)


def energy64(y, hop=256):
    return features64(y, N_FFT // 2, hop, hann_window_scipy(), 0.0, np.zeros((1, N_FFT // 2 + 1)))["energy"]


# ---- the seeded inputs of the fixtures ---------------------------------------------------------------------------------------

SR = 16000


def signals(n=4000, seed=9101):
    """name -> float32 signal in [-1, 1]: harmonic tone with vibrato, 50 Hz - 7.9 kHz chirp, white noise at -20 and -60 dBFS,
    digital silence, a +-1.0 square wave."""
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    f0 = 220.0 * (1.0 + 0.03 * np.sin(2 * np.pi * 5.0 * t))
    ph = 2 * np.pi * np.cumsum(f0) / SR
    tone = sum(np.sin(h * ph) / h for h in range(1, 11))
    tone = 0.8 * tone / np.abs(tone).max()
    dur = n / SR
    chirp = 0.7 * np.sin(2 * np.pi * (50.0 * t + 0.5 * (7900.0 - 50.0) / dur * t ** 2))
    sq = np.where(np.sin(2 * np.pi * 440.0 * t + 0.1) >= 0, 1.0, -1.0)
    return {"tone": tone.astype(np.float32), "chirp": chirp.astype(np.float32),
            "noise_m20": (0.1 * rng.standard_normal(n)).astype(np.float32), "noise_m60": (0.001 * rng.standard_normal(n)).astype(np.float32),
            "silence": np.zeros(n, np.float32), "square": sq.astype(np.float32)}
