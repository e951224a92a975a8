"""The loudness meter on the host (no GPU): the fp64 oracle's known answers at 16 and 48 kHz (EBU Tech 3342 cases 1-4, steady
tones, a loud second inside quiet tone, a true peak between samples), its exact percentile rule, and the argument checks of
``loudness.meter``.

Signals are mono, so their levels read 3.01 dB under Tech 3341 / 3342's stereo ones; loudness ranges are unchanged."""
import math

import numpy as np
import pytest
import torch
from scipy.signal import freqz

from emotivoice_b200 import audio, loudness
from oracle import limiter_oracle
from oracle import loudness_oracle as LO
from oracle import meter_oracle as O

RATES = (16000, 48000)


def _sine(sr, dbfs, seconds, f=1000.0, phase=0.0):
    n = np.arange(int(round(seconds * sr)))
    return 10.0 ** (dbfs / 20.0) * np.sin(2 * np.pi * f * n / sr + phase)


def _k_gain_db(f, sr):
    sb, sa, hb, ha = LO.k_weighting(sr)
    w = 2 * np.pi * f / sr
    return 20 * np.log10(abs(freqz(sb, sa, [w])[1][0] * freqz(hb, ha, [w])[1][0]))


def _tone_lufs(dbfs, f, sr):
    """The loudness of a steady sine of peak level dbfs (the formula of test_loudness)."""
    return dbfs - 3.0103 + (_k_gain_db(f, sr) - 0.691)


@pytest.mark.parametrize("sr", RATES)
@pytest.mark.parametrize("levels, lra", [((-20, -30), 10.0), ((-20, -15), 5.0), ((-40, -20), 20.0),
                                         ((-50, -35, -20, -35, -50), 15.0)])
def test_tech3342_cases_read_their_range(sr, levels, lra):
    x = np.concatenate([_sine(sr, l, 20.0) for l in levels])
    got = O.loudness_range(x, sr)
    assert abs(got - lra) <= 1.0, (levels, got)


@pytest.mark.parametrize("sr", RATES)
def test_steady_tone_reads_the_same_everywhere(sr):
    x = _sine(sr, -20.0, 10.0, 997.0)
    m = O.meter(x, sr, true_peak=False)
    want = _tone_lufs(-20.0, 997.0, sr)
    for k in ("integrated", "max_momentary", "max_short_term"):
        assert abs(m[k] - want) <= 0.01, (k, m[k], want)
    assert len(m["momentary"]) == 100 - 3 and len(m["short_term"]) == 100 - 29
    assert abs(m["loudness_range"]) <= 0.01


@pytest.mark.parametrize("sr", RATES)
def test_a_loud_second_in_quiet_tone(sr):
    x = np.concatenate([_sine(sr, -36.0, 10.0), _sine(sr, -20.0, 1.0), _sine(sr, -36.0, 10.0)])
    m = O.meter(x, sr, true_peak=False)
    loud, quiet = _tone_lufs(-20.0, 1000.0, sr), _tone_lufs(-36.0, 1000.0, sr)
    assert abs(m["max_momentary"] - loud) <= 0.02, (m["max_momentary"], loud)
    mixed = 10.0 * math.log10((10.0 ** (loud / 10.0) + 2.0 * 10.0 ** (quiet / 10.0)) / 3.0)
    assert abs(m["max_short_term"] - mixed) <= 0.02, (m["max_short_term"], mixed)


def test_true_peak_between_samples():
    sr, amp = 16000, 0.5
    x = _sine(sr, 20 * math.log10(amp), 1.0, 4000.0, math.pi / 4)
    fade = int(0.1 * sr)
    ramp = 0.5 - 0.5 * np.cos(np.pi * np.arange(fade) / fade)
    x[:fade] *= ramp
    x[-fade:] *= ramp[::-1]
    tp = limiter_oracle.true_peak_db(x, sr)
    want = 20 * math.log10(amp)
    assert -0.4 <= tp - want <= 0.2, (tp, want)
    sp = 20 * math.log10(LO.peak(x))
    assert abs(sp - (want - 3.0103)) <= 0.01, sp


def test_percentiles_pick_elements_and_round_half_away():
    assert [O.round_half_away(v) for v in (0.0, 0.49, 0.5, 1.5, 2.5, 7.6)] == [0, 0, 1, 2, 3, 8]
    st = np.array([-30.0, -31.0, -25.0, -28.0, -29.0, -80.0, -27.0])    # -80: under the absolute gate
    v = np.sort(st[st > -70])                                           # all six pass the relative gate
    assert len(v) == 6 and O.round_half_away(0.10 * 5) == 1           # (n - 1) * 0.10 = 0.5 exactly: rounds up
    assert O.loudness_range(None, 16000, st) == v[5] - v[1]            # round(4.75) = 5
    assert math.isnan(O.loudness_range(None, 16000, np.array([-80.0, -75.0])))
    assert math.isnan(O.loudness_range(np.zeros(4 * 16000), 16000))
    assert math.isnan(O.loudness_range(np.ones(16000), 16000))           # shorter than one short-term window


def test_empty_and_silent_series_read_minus_infinity():
    for x in (np.zeros(16000), np.full(3000, 0.1)):
        m = O.meter(x, 16000)
        assert m["max_momentary"] == -np.inf and m["integrated"] == -np.inf and m["max_short_term"] == -np.inf
    assert O.meter(np.zeros(16000), 16000)["true_peak"] == -np.inf


def test_rates_are_checked():
    for ok in (4000, 8000, 11030, 22050, 44100, 48000, 96000, 192000, np.int64(16000)):
        assert loudness.check_rate(ok) == int(ok)
    for bad in (11025, 3990, 192010, 16005, 16000.0, "16000", True, None):
        with pytest.raises(ValueError):
            loudness.check_rate(bad)


def test_meter_refuses_what_is_not_a_cuda_float32_batch():
    for bad in (np.zeros((1, 100), np.float32), torch.zeros(1, 100), torch.zeros(100), torch.zeros(1, 100, dtype=torch.float64)):
        with pytest.raises(ValueError):
            loudness.meter(bad, 16000)


def test_detector_bank_is_the_limiters_with_phase_zero():
    assert audio.true_peak_bank(192000) is None
    for sr in (4000, 8000, 16000, 44100, 48000, 96000, 96010, 191990):
        bank = audio.true_peak_bank(sr)
        R = -(-192000 // sr)
        assert bank.shape == (R, 21) and bank.dtype == np.float32, sr
        assert np.array_equal(bank[1:], audio.limit_bank(sr, sr)[0]), sr
        assert 1.0 < bank[0, 10] < 1.001 and np.abs(np.delete(bank[0], 10)).max() < 1e-12, sr


@pytest.mark.parametrize("sr", (8000, 16000, 44100, 48000, 96000))
def test_detector_bank_reads_what_true_peak_db_reads(sr):
    """The kernels' detector, restated with the host bank: max |sum_j bank[p][j] x[s + 10 - j]| over all R phases and |x|."""
    rng = np.random.default_rng(sr)
    x = (0.02 * rng.standard_normal(3000)).astype(np.float32)
    x[1234] = 0.9                                     # a peak at a sample instant: phase 0 reads it 1 + 6.7e-4 times
    bank = audio.true_peak_bank(sr).astype(np.float64)
    xp = np.concatenate([np.zeros(10), x, np.zeros(10)]).astype(np.float64)
    phases = [np.abs(np.convolve(xp, row, mode="valid")) for row in bank]
    want = limiter_oracle.true_peak_db(x, sr)
    tp = 20 * np.log10(np.maximum(np.abs(x), np.max(phases, axis=0)).max())
    assert abs(tp - want) <= 1e-6                     # float32 taps
    limiter = 20 * np.log10(np.maximum(np.abs(x), np.max(phases[1:], axis=0)).max())
    assert 0.004 <= want - limiter <= 0.006, want - limiter