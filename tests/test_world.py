"""WORLD spectral envelopes (CheapTrick) and SPTK mel-cepstra (sp2mc, freqt): the fp64 oracle (oracle/world_oracle.py) against
what is known independently of pyworld and pysptk, neither of which is installed: envelopes recovered from harmonic signals
whose envelope is known, independence of F0 and gain, digital silence, the FFT size per rate, sp2mc at alpha = 0 as the real
cepstrum, the all-pass warping identity of the mel-cepstrum, freqt's inverse; ``feats.sp2mc_table`` against the oracle's
recursion; argument errors of ``feats.spectral_envelope``, ``feats.sp2mc`` and ``evaluate.compare(cepstrum=)``.  No GPU.

The dB and relative bounds were measured on the oracle (numpy fp64 on x86-64) when the tests were written and carry a margin;
each says what was measured."""
import math

import numpy as np
import pytest
import torch

from emotivoice_b200 import evaluate, feats
from oracle import world_oracle as W

SR = 16000
DB = 10.0 / math.log(10.0)          # dB per neper of power


def envelope(f, fs=SR):
    """A known smooth power envelope: two resonances (600 Hz / 150 Hz wide, 2200 Hz / 250 Hz wide) of an all-pole filter."""
    out = np.ones_like(np.asarray(f, np.float64))
    z = np.exp(-2j * np.pi * np.asarray(f, np.float64) / fs)
    for fc, bw in ((600.0, 150.0), (2200.0, 250.0)):
        r, w = math.exp(-math.pi * bw / fs), 2 * math.pi * fc / fs
        out = out / np.abs(1 - 2 * r * math.cos(w) * z + r * r * z * z) ** 2
    return out


def harmonic(f0, seconds=0.4, seed=0, fs=SR):
    """Harmonics of f0 up to fs / 2 with amplitudes sqrt(envelope(h f0)) and seeded random phases."""
    rng = np.random.default_rng(seed)
    t = np.arange(int(seconds * fs)) / fs
    x = np.zeros_like(t)
    h = 1
    while h * f0 < fs / 2:
        x += math.sqrt(envelope(h * f0, fs)) * np.cos(2 * np.pi * h * f0 * t + rng.uniform(0, 2 * np.pi))
        h += 1
    return 0.5 * x / np.abs(x).max()


def log_envelope(x, f0, t=0.2):
    n_fft = W.fft_size(SR)
    return W.envelope_frame(x, len(x), SR, f0, t, n_fft, log=True)


def band(f0, n_fft):
    freqs = np.arange(n_fft // 2 + 1) * SR / n_fft
    return freqs, (freqs >= 2 * f0) & (freqs <= SR / 2 - 2 * f0)


# measured max deviation (dB) of the level-aligned estimate from the known envelope: 0.81, 1.41, 3.02, 3.75
@pytest.mark.parametrize("f0,bound_db", [(100.0, 1.0), (150.0, 1.75), (220.0, 3.5), (300.0, 4.5)])
def test_envelope_of_a_harmonic_signal_follows_the_known_one(f0, bound_db):
    x = harmonic(f0)
    n_fft = W.fft_size(SR)
    freqs, m = band(f0, n_fft)
    d = log_envelope(x, f0) - np.log(envelope(freqs))
    d = d[m] - d[m].mean()
    dev = DB * np.abs(d).max()
    print("F0 %g Hz: max deviation %.3f dB, rms %.3f dB" % (f0, dev, DB * np.sqrt((d * d).mean())))
    assert dev <= bound_db


def test_the_same_envelope_at_two_f0s_gives_matching_estimates():
    n_fft = W.fft_size(SR)
    a = log_envelope(harmonic(150.0), 150.0)
    b = log_envelope(harmonic(220.0, seed=1), 220.0)
    _, m = band(220.0, n_fft)
    d = (a - b)[m]
    d = d - d.mean()
    print("150 vs 220 Hz: max difference %.3f dB" % (DB * np.abs(d).max()))
    assert DB * np.abs(d).max() <= 4.0                      # measured 3.54 dB


@pytest.mark.parametrize("g", [0.5, 0.1])
def test_gain_moves_only_c0(g):
    """Scaling by g scales the power by g^2, so log sp moves by 2 ln g; sp2mc halves c[0], so c0 moves by ln g."""
    x = harmonic(150.0)
    f0 = np.full(10, 150.0)
    s1 = W.cheaptrick(x, SR, f0, 16.0)[3]
    s2 = W.cheaptrick(x * g, SR, f0, 16.0)[3]
    c1, c2 = W.sp2mc(s1, 24, 0.42), W.sp2mc(s2, 24, 0.42)
    print("g %g: c0 moved %.12f (ln g %.12f), c1..c24 by at most %.2e" % (g, c2[0] - c1[0], math.log(g), np.abs(c2[1:] - c1[1:]).max()))
    assert abs((c2[0] - c1[0]) - math.log(g)) <= 1e-7        # measured 3.0e-9 at g = 0.1: the eps floor
    assert np.abs(c2[1:] - c1[1:]).max() <= 1e-7             # measured 5.8e-9


def test_digital_silence_gives_finite_output():
    sp = W.cheaptrick(np.zeros(4000), SR, np.zeros(10), 16.0)
    Fb = W.frame_count(4000, SR, 16.0)
    assert np.isfinite(sp).all() and (sp[:Fb] > 0).all() and (sp[Fb:] == 0).all()
    assert np.allclose(sp[:Fb], W.EPS, rtol=1e-9)
    assert np.isfinite(W.sp2mc(sp[0], 24, 0.42)).all()


@pytest.mark.parametrize("fs,n_fft", [(8000, 512), (16000, 1024), (22050, 1024), (24000, 1024), (44100, 2048), (48000, 2048)])
def test_fft_size_per_rate(fs, n_fft):
    assert W.fft_size(fs) == feats.world_fft_size(fs) == n_fft
    assert 2 * W.matlab_round(1.5 * fs / (W.f0_floor(fs, n_fft) + 1e-9)) + 1 <= n_fft      # the longest window fits


def test_sp2mc_at_alpha_0_is_the_truncated_real_cepstrum_with_c0_halved():
    sp = W.cheaptrick(harmonic(150.0), SR, np.full(10, 150.0), 16.0)[3]
    c = np.fft.irfft(np.log(sp))
    c[0] /= 2.0
    assert np.array_equal(W.sp2mc(sp, 24, 0.0), c[:25])


def test_the_mel_cepstrum_on_the_warped_axis_reproduces_half_the_log_envelope():
    """sum_m mc_m cos(m beta(w)) = 1/2 log sp(w), beta the all-pass warping of freqt, as the order grows."""
    sp = W.cheaptrick(harmonic(150.0), SR, np.full(10, 150.0), 16.0)[3]
    n_fft = W.fft_size(SR)
    w = np.arange(n_fft // 2 + 1) * 2 * np.pi / n_fft
    beta = W.warped_frequency(w, 0.42)
    errs = []
    for order in (60, 100, 200):
        mc = W.sp2mc(sp, order, 0.42)
        errs.append(np.abs(np.cos(np.outer(beta, np.arange(order + 1))) @ mc - 0.5 * np.log(sp)).max())
    print("max error (nepers) at orders 60 / 100 / 200: %s" % errs)
    assert errs[0] > errs[1] > errs[2]
    assert errs[2] <= 0.05                                   # measured 0.032


def test_freqt_with_minus_alpha_undoes_freqt_with_alpha():
    c = np.random.default_rng(1).normal(size=30) * 0.7 ** np.arange(30)
    for alpha in (0.42, 0.55, -0.3):
        back = W.freqt(W.freqt(c, 400, alpha), 29, -alpha)
        assert np.abs(back - c).max() <= 1e-12               # measured 1.1e-16


def test_smoothing_local_sums_equal_the_running_sum_difference_and_stay_positive():
    """W6: the local sum equals WORLD's difference of interp1Q reads of the running sum where that difference is well
    conditioned (a spectrum with no quiet band), and is never negative where it is not (a band-limited spectrum)."""
    n_fft, fs = 1024, SR
    for f0 in (93.2, 150.0, 500.0, 4000.0):
        width = f0 * 2.0 / 3.0
        p = np.exp(np.random.default_rng(int(f0)).normal(size=n_fft // 2 + 1))
        half, b = n_fft // 2, int(width * n_fft / fs) + 1
        seg = np.cumsum(np.concatenate([p[b:0:-1], p[:half], p[half:half - b - 1:-1]]) * fs / n_fft)
        origin = -(b - 0.5) * fs / n_fft
        axis = np.arange(half + 1) / n_fft * fs - width / 2.0
        world = (W.interp1q(origin, fs / n_fft, seg, axis + width) - W.interp1q(origin, fs / n_fft, seg, axis)) / width
        ours = W.linear_smoothing(p, width, fs, n_fft)
        assert np.abs(ours - world).max() <= 1e-10 * np.abs(world).max(), f0
        q = p.copy()
        q[200:] = 0.0                                          # a band with nothing in it
        assert (W.linear_smoothing(q, width, fs, n_fft) >= 0.0).all(), f0


@pytest.mark.parametrize("n_fft,order,alpha", [(512, 24, 0.31), (1024, 24, 0.42), (1024, 40, 0.0), (2048, 24, 0.55), (16, 5, -0.2)])
def test_sp2mc_table_is_the_oracle_recursion(n_fft, order, alpha):
    rng = np.random.default_rng(n_fft + order)
    T = feats.sp2mc_table(n_fft, order, alpha)
    assert T.shape == (order + 1, n_fft // 2 + 1)
    for _ in range(3):
        sp = np.exp(rng.normal(size=n_fft // 2 + 1))
        want = W.sp2mc(sp, order, alpha)
        assert np.abs(T @ np.log(sp) - want).max() <= 1e-12 * max(1.0, np.abs(want).max())


def test_argument_errors():
    cpu = torch.zeros((1, 16000), dtype=torch.float32)      # the cepstrum arguments are checked before the waveforms
    for kw, msg in ((dict(cepstrum="sptk"), "cepstrum must be"), (dict(cepstrum=None), "cepstrum must be"),
                    (dict(cepstrum="mel", alpha=0.42), "alpha applies"), (dict(alpha=0.0), "alpha applies"),
                    (dict(cepstrum="world", alpha=1.0), "alpha must be"), (dict(cepstrum="world", alpha=-1.5), "alpha must be"),
                    (dict(cepstrum="world", alpha="0.42"), "alpha must be"), (dict(cepstrum="world", alpha=True), "alpha must be")):
        with pytest.raises(ValueError, match=msg):
            evaluate.compare(cpu, cpu, **kw)
    for order, alpha in ((-1, 0.42), (256, 0.42), (2.0, 0.42), (24, 1.0), (24, float("nan")), (24, None)):
        with pytest.raises(ValueError):
            feats.sp2mc(torch.ones((2, 513), dtype=torch.float64), order, alpha)
    with pytest.raises(ValueError):                           # not a CUDA tensor
        feats.sp2mc(torch.ones((2, 513), dtype=torch.float64), 24, 0.42)
    with pytest.raises(RuntimeError):                         # as pitch_track: no CPU path
        feats.spectral_envelope(cpu.double(), SR, 256)
