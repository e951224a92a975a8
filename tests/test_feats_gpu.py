"""stft_feats_kernel (csrc/feats_kernels.cu) through emotivoice_b200.feats: log-mel spectrograms and frame energy against fp64
per element, against the reference fixtures (oracle/make_golden_feats.py), exact values, batches and one chain into the
alignment helpers.

Bounds, with m_f = sum_n |w_n x_n| of the frame and tau = 2^-16 (about ten fp32 FFT stages with headroom):
  mel before the log   |mel - mel64| <= 2 tau m_f sum_k M_jk + (n_j + 2) 2^-24 mel64
  log-mel              that bound / max(mel64, 1e-5) + 2^-22 |log-mel64|
  energy               |e - e64| <= sqrt(513) tau m_f + 2^-22 e64
The FFT term vanishes with the signal; the relative terms are the fp32 rounding left when it does: the n_j-term fp32 sum of a
band (n_j = its bin count) and the square root of a magnitude that mel_spectrogram_torch's 1e-6 keeps away from 0, and the
rounding of the energy's 1e-10 floor and its square root.
"""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from emotivoice_b200 import align, feats, synth
from oracle import feats_oracle as FO

pytestmark = pytest.mark.gpu

TAU = 2.0 ** -16
DEV = "cuda"
SR = 16000


def _basis():
    return feats.mel_filterbank(sr=SR, n_fft=1024, n_mels=80, fmin=0.0, fmax=8000.0)


def _logmel_bound(r64, basis):
    n_j = feats.band_table(basis)[0][:, 1].astype(np.float64)
    mel_b = 2 * TAU * r64["m_f"][None, :] * basis.astype(np.float64).sum(axis=1)[:, None] + (n_j[:, None] + 2) * 2.0 ** -24 * r64["mel"]
    return mel_b / np.maximum(r64["mel"], 1e-5) + 2.0 ** -22 * np.abs(r64["logmel"])


def _energy_bound(r64):
    return np.sqrt(513.0) * TAU * r64["m_f"] + 2.0 ** -22 * r64["energy"]


def _run(variant, y, hop, lengths=None):
    """-> (log-mel (B, 80, F) or None, energy (B, F) or None) as numpy."""
    yt = torch.from_numpy(np.atleast_2d(np.asarray(y, np.float32))).to(DEV)
    if variant == "taco":
        return feats.TacotronSTFT(hop_length=hop, sampling_rate=SR).to(DEV).mel_spectrogram(yt, lengths=lengths).cpu().numpy(), None
    if variant == "mt":
        return feats.mel_spectrogram_torch(yt, 1024, 80, SR, hop, 1024, 0.0, 8000.0, lengths=lengths).cpu().numpy(), None
    en = feats.Energy(sr=SR, n_fft=1024, hop_length=hop, win_length=1024)
    return None, en.get_energy(yt, lengths=lengths).cpu().numpy()


def _fp64(variant, y, hop, basis):
    if variant == "taco":
        return FO.tacotron64(y, hop, basis)
    if variant == "mt":
        return FO.mel_spectrogram64(y, hop, basis)
    return FO.features64(y, 512, hop, feats.hann_window_scipy(), 0.0, basis)


def _check_item(variant, y, hop, extra=None):
    basis = _basis()
    mel, e = _run(variant, y, hop)
    r64 = _fp64(variant, np.asarray(y, np.float32), hop, basis)
    if variant == "energy":
        err, bnd = np.abs(e[0] - r64["energy"]), _energy_bound(r64) + (0 if extra is None else extra)
    else:
        err, bnd = np.abs(mel[0] - r64["logmel"]), _logmel_bound(r64, basis) + (0 if extra is None else extra)
    assert err.shape == bnd.shape
    bad = err > bnd
    assert not bad.any(), "%s hop %d: %d elements over the bound, worst err %.3e vs bound %.3e" % (
        variant, hop, int(bad.sum()), float(err[bad].max()), float(bnd[bad][np.argmax(err[bad])]))


def _signal(n, seed):
    rng = np.random.default_rng(seed)
    t = np.arange(n) / SR
    x = 0.4 * np.sin(2 * np.pi * 330.0 * t) + 0.2 * np.sin(2 * np.pi * 2900.0 * t + 1.0) + 0.05 * rng.standard_normal(n)
    return x.astype(np.float32)


@pytest.mark.parametrize("hop", [256, 160])
@pytest.mark.parametrize("variant", ["taco", "mt", "energy"])
def test_against_fp64_on_the_synthetic_signals(variant, hop):
    for name, y in FO.signals().items():
        _check_item(variant, y, hop)


@pytest.mark.parametrize("hop", [256, 160])
@pytest.mark.parametrize("variant", ["taco", "mt", "energy"])
def test_against_fp64_at_length_and_tile_edges(variant, hop):
    pad = 512 if variant != "mt" else (1024 - hop) // 2
    ns = [pad + 1 if variant == "mt" else pad + 1 + 512, 20 * hop - 1, 20 * hop, 20 * hop + 1]
    for fcount in (31, 32, 33, 65):                      # the kernel's tile is 32 frames: T - 1, T, T + 1, 2T + 1
        ns.append((fcount - 1) * hop + 1024 - 2 * pad)
    for i, n in enumerate(ns):
        y = _signal(n, 9200 + i)
        _check_item(variant, y, hop)
        if variant == "mt" and n == pad + 1:                  # a single frame at hop 256
            assert _run(variant, y, hop)[0].shape[-1] == feats.n_frames(n, pad, hop) == (1 if hop == 256 else 2)
    for fcount in (31, 32, 33, 65):
        n = (fcount - 1) * hop + 1024 - 2 * pad
        out = _run(variant, _signal(n, 1), hop)
        assert (out[0] if out[0] is not None else out[1]).shape[-1] == fcount


@pytest.mark.parametrize("variant", ["taco", "mt", "energy"])
def test_against_fp64_on_a_30s_item(variant):
    _check_item(variant, _signal(30 * SR, 9300), 256)


NAMES = ["tone", "chirp", "noise_m20", "noise_m60", "silence", "square", "b1_t100"]


@pytest.mark.parametrize("name", NAMES)
def test_against_the_reference_fixtures(name):
    """The same bounds plus the reference's own deviation from fp64."""
    with np.load(os.path.join(GOLDEN, "feats_%s.npz" % name)) as z:
        g = {k: z[k] for k in z.files}
    y, basis = g["wav"], _basis()
    for variant, key in (("taco", "taco_mel"), ("mt", "mt_mel"), ("energy", "energy")):
        mel, e = _run(variant, y, 256)
        r64 = _fp64(variant, y, 256, basis)
        if variant == "energy":
            err, bnd = np.abs(e[0] - g[key]), _energy_bound(r64) + g["energy_dev"]
        else:
            err, bnd = np.abs(mel[0] - g[key]), _logmel_bound(r64, basis) + g[key.split("_")[0] + "_dev"]
        assert (err <= bnd).all(), (name, variant, float(err.max()))


def test_silence_is_exact():
    y = torch.zeros(1, 8000, device=DEV)
    mel = feats.TacotronSTFT(sampling_rate=SR).to(DEV).mel_spectrogram(y)
    expect = torch.log(torch.full((1,), 1e-5, dtype=torch.float32, device=DEV))
    assert torch.equal(mel, expect.expand_as(mel))
    e = feats.Energy(sr=SR, n_fft=1024, hop_length=256).get_energy(y[0])
    assert torch.equal(e.cpu(), torch.full_like(e.cpu(), float(np.sqrt(np.float32(1e-10)))))


def test_range_check():
    stft = feats.TacotronSTFT(sampling_rate=SR).to(DEV)
    sq = torch.from_numpy(FO.signals()["square"]).to(DEV)[None]
    assert sq.abs().max().item() == 1.0
    stft.mel_spectrogram(sq)
    over = sq.clone()
    over[0, 1234] = float(np.nextafter(np.float32(1.0), np.float32(2.0)))
    with pytest.raises(AssertionError):
        stft.mel_spectrogram(over)
    tail = sq.clone()
    tail[0, -1] = -1.0000001                                 # the last sample, read only by the last frame
    with pytest.raises(AssertionError):
        stft.mel_spectrogram(tail)
    assert torch.equal(stft.mel_spectrogram(sq), stft.mel_spectrogram(sq))
    # past an item's length nothing is read, so nothing there is checked
    assert stft.mel_spectrogram(over, lengths=[1234]).shape[-1] == sq.shape[1] // 256 + 1


@pytest.mark.parametrize("variant", ["taco", "mt", "energy"])
def test_batch_is_bitwise_its_items(variant):
    lens = [4000, 385 + 700, 12345, 7777, 9000]
    N = max(lens)
    rng = np.random.default_rng(9400)
    y = np.full((5, N), np.nan, np.float32)                 # NaN past every item's length: must not leak
    items = []
    for b, n in enumerate(lens):
        items.append(_signal(n, 9400 + b) * np.float32(rng.uniform(0.2, 1.0)))
        y[b, :n] = items[-1]
    mel, e = _run(variant, y, 256, lengths=lens)
    out = mel if mel is not None else e
    pad = 512 if variant != "mt" else 384
    assert out.shape[-1] == feats.n_frames(N, pad, 256)
    assert np.isfinite(out).all()
    for b, n in enumerate(lens):
        m1, e1 = _run(variant, items[b], 256)
        one = (m1 if m1 is not None else e1)[0]
        fb = feats.n_frames(n, pad, 256)
        assert one.shape[-1] == fb
        assert np.array_equal(out[b][..., :fb], one)
        assert (out[b][..., fb:] == 0.0).all()


def test_chain_into_alignment():
    """Fixture waveform -> TacotronSTFT mel -> seeded AlignmentModule -> viterbi_decode; token-averaged energy."""
    with np.load(os.path.join(GOLDEN, "b1_t100.npz")) as z:
        wav = torch.from_numpy(z["wav"].reshape(-1)).to(DEV)
    mel = feats.TacotronSTFT(sampling_rate=SR).to(DEV).mel_spectrogram(wav[None])        # (1, 80, F)
    F = mel.shape[-1]
    assert F == wav.numel() // 256 + 1
    adim, odim, T = 384, 80, 40
    mod = align.AlignmentModule(adim, odim)
    mod.load_state_dict(synth.make_alignment_state_dict(adim, odim))
    mod = mod.to(DEV)
    text = torch.from_numpy(np.random.default_rng(9500).normal(size=(1, T, adim)).astype(np.float32)).to(DEV)
    tl, fl = torch.tensor([T]), torch.tensor([F])
    lp = mod(text, mel.transpose(1, 2), tl, fl)
    ds, _ = align.viterbi_decode(lp, tl, fl)
    assert int(ds.sum().item()) == F and (ds >= 1).all()
    en = feats.Energy(sr=SR, n_fft=1024, hop_length=256, win_length=1024)
    frames = en.get_energy(wav, use_token_averaged_energy=False)
    assert frames.shape == (F,)
    tok = en.get_energy(wav, duration=ds[0])
    assert torch.equal(tok, align.average_by_duration(ds, frames[None], tl, fl)[0])
    dsn = ds[0].cpu().numpy().astype(np.int64)
    assert torch.equal(tok, en.get_energy(wav, duration=dsn))
