"""TEST INFRASTRUCTURE ONLY -- generates tests/golden/feats_*.npz from the reference's own feature code and pins
oracle/feats_oracle.py against it.  Run where the reference tree is present:  python oracle/make_golden_feats.py

The unmodified TacotronSTFT (tacotron_stft.py), mel_spectrogram_torch (mel_process.py) and Energy (feats.py) are imported with
stub ``librosa`` and ``pyworld`` modules in sys.modules, since neither package is installed.  The stubs provide what those
three use: ``filters.mel`` (emotivoice_b200.feats.mel_filterbank), ``util.pad_center``, ``util.tiny``, ``util.normalize`` and
``core.stft`` (oracle.feats_oracle.librosa_stft).  The two restatements are cross-checked here against torchaudio's
``melscale_fbanks`` and against ``torch.stft(center=True)``, not against librosa.

Each fixture holds the input, the reference's fp32 outputs at the config (16 kHz, hop 256, 80 mels, 0-8000 Hz), their fp64
counterparts and the per-element deviation of the reference from fp64.
"""
import os
import sys
import types

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from emotivoice_b200.feats import mel_filterbank     # noqa: E402
from oracle import feats_oracle as FO                 # noqa: E402
from oracle import refshim                            # noqa: E402

HOP, N_MELS, FMIN, FMAX = 256, 80, 0.0, 8000.0
B1_SPAN = (40000, 48000)          # the excerpt of tests/golden/b1_t100.npz's waveform (the model's own output)


def _pad_center(data, *, size, axis=-1, **kw):
    n = data.shape[axis]
    lpad = int((size - n) // 2)
    lengths = [(0, 0)] * data.ndim
    lengths[axis] = (lpad, int(size - n - lpad))
    return np.pad(data, lengths, **kw)


def _tiny(x):
    x = np.asarray(x)
    dt = x.dtype if np.issubdtype(x.dtype, np.floating) or np.issubdtype(x.dtype, np.complexfloating) else np.float32
    return np.finfo(dt).tiny


def _normalize(S, norm=np.inf, **_):
    if norm is None:
        return S
    raise NotImplementedError("the stub only covers norm=None")


def install_stubs():
    lib = types.ModuleType("librosa")
    filters = types.ModuleType("librosa.filters")
    filters.mel = lambda sr, n_fft, n_mels=128, fmin=0.0, fmax=None, **_: mel_filterbank(sr, n_fft, n_mels, fmin, fmax)
    util = types.ModuleType("librosa.util")
    util.pad_center, util.tiny, util.normalize = _pad_center, _tiny, _normalize
    core = types.ModuleType("librosa.core")
    core.stft = FO.librosa_stft
    lib.filters, lib.util, lib.core, lib.stft = filters, util, core, FO.librosa_stft
    for name, m in (("librosa", lib), ("librosa.filters", filters), ("librosa.util", util), ("librosa.core", core)):
        sys.modules[name] = m
    sys.modules["pyworld"] = types.ModuleType("pyworld")


def cross_check_restatements():
    import torchaudio
    ours = mel_filterbank(sr=16000, n_fft=1024, n_mels=N_MELS, fmin=FMIN, fmax=FMAX)
    ta = torchaudio.functional.melscale_fbanks(513, FMIN, FMAX, N_MELS, 16000, norm="slaney", mel_scale="slaney").T.numpy()
    assert np.abs(ours - ta).max() <= 1e-7 and np.array_equal(ours > 0, ta > 0), np.abs(ours - ta).max()
    rng = np.random.default_rng(9100)
    x = (0.3 * rng.standard_normal(5000)).astype(np.float32)
    a = FO.librosa_stft(x, n_fft=1024, hop_length=HOP, win_length=1024, center=True, pad_mode="reflect")
    b = torch.stft(torch.from_numpy(x).double(), 1024, hop_length=HOP, win_length=1024, window=torch.hann_window(1024, dtype=torch.float64),
                   center=True, pad_mode="reflect", return_complex=True).numpy()
    assert a.shape == b.shape and np.abs(a - b).max() <= 1e-5 * np.abs(b).max(), np.abs(a - b).max()
    print("restatements ok: mel basis vs torchaudio %.2e, stft vs torch.stft(center=True) %.2e" % (np.abs(ours - ta).max(), np.abs(a - b).max()))


def main():
    if not refshim.reference_available():
        raise SystemExit("reference tree not present at %s" % refshim.REF_ROOT)
    install_stubs()
    if refshim.REF_ROOT not in sys.path:
        sys.path.insert(0, refshim.REF_ROOT)
    from models.prompt_tts_modified.tacotron_stft import TacotronSTFT
    from models.prompt_tts_modified import feats as RF
    import mel_process as RM
    cross_check_restatements()
    stft = TacotronSTFT(filter_length=1024, hop_length=HOP, win_length=1024, n_mel_channels=N_MELS, sampling_rate=16000, mel_fmin=FMIN,
                        mel_fmax=FMAX)
    basis = stft.mel_basis.numpy()
    assert np.array_equal(basis, mel_filterbank(sr=16000, n_fft=1024, n_mels=N_MELS, fmin=FMIN, fmax=FMAX))
    en = RF.Energy(sr=16000, n_fft=1024, hop_length=HOP, win_length=1024, window="hann")
    sigs = FO.signals()
    wav = np.load(os.path.join(ROOT, "tests", "golden", "b1_t100.npz"))["wav"].reshape(-1)
    sigs["b1_t100"] = wav[B1_SPAN[0]:B1_SPAN[1]].astype(np.float32)
    out_dir = os.path.join(ROOT, "tests", "golden")
    for name, y in sigs.items():
        yt = torch.from_numpy(y)[None]
        with torch.no_grad():
            taco = stft.mel_spectrogram(yt).numpy()[0]
            mt = RM.mel_spectrogram_torch(yt, 1024, N_MELS, 16000, HOP, 1024, FMIN, FMAX, center=False).numpy()[0]
        e = np.asarray(en.get_energy(y), dtype=np.float32)
        assert np.array_equal(FO.tacotron_mel(y, HOP)[0], taco), name
        assert np.array_equal(FO.mel_spectrogram(y, HOP)[0], mt), name
        assert np.array_equal(FO.energy(y, HOP), e), name
        t64 = FO.tacotron64(y, HOP, basis)
        m64 = FO.mel_spectrogram64(y, HOP, basis)
        e64 = FO.energy64(y, HOP)
        arrays = {"wav": y, "taco_mel": taco, "taco_mel64": t64["logmel"], "taco_dev": np.abs(taco - t64["logmel"]),
                  "mt_mel": mt, "mt_mel64": m64["logmel"], "mt_dev": np.abs(mt - m64["logmel"]),
                  "energy": e, "energy64": e64, "energy_dev": np.abs(e - e64)}
        if name == "b1_t100":
            arrays["span"] = np.asarray(B1_SPAN, np.int64)
            arrays["mel_basis"] = basis                               # the reference TacotronSTFT's mel_basis buffer
        np.savez_compressed(os.path.join(out_dir, "feats_%s.npz" % name), **arrays)
        print("feats_%s ok: %d samples, mel %s / %s, max deviation from fp64: taco %.2e mt %.2e energy %.2e" % (
            name, len(y), taco.shape, mt.shape, arrays["taco_dev"].max(), arrays["mt_dev"].max(), arrays["energy_dev"].max()))


if __name__ == "__main__":
    main()
