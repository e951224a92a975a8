"""The true-peak limiter on the host (no GPU): the fp64 oracle's envelope (G <= r everywhere, the prefix-minimum release equal
to the literal recurrence bit for bit, edge peaks limited, a lone peak's release rate), the true-peak bound of its output, the
host detector bank against the oracle's filter, the ceiling checks, and the MicroBatcher's format keys."""
import numpy as np
import pytest
import torch

from emotivoice_b200 import audio
from emotivoice_b200 import frontdoor as fd
from oracle import limiter_oracle as O

SR = 16000


def sine_45():
    """4 kHz at 16 kHz, 45 degree phase: sample peak -3.01 dB, true peak 0 dB."""
    n = np.arange(SR)
    return np.sin(2 * np.pi * 4000.0 * n / SR + np.pi / 4).astype(np.float32)


def voiced(plr_db, seconds=4.0, f0=120.0, seed=0):
    """Speech-like voiced signal: a pulse train through three formant resonators under a 4 Hz syllabic envelope, scaled so its
    peak-to-loudness ratio (sample peak over integrated loudness) is about ``plr_db``; the envelope's depth and sharpness set
    the ratio."""
    from scipy.signal import lfilter
    from oracle import loudness_oracle
    rng = np.random.default_rng(seed)
    n = int(seconds * SR)
    t = np.arange(n) / SR
    f = f0 * (1.0 + 0.05 * np.sin(2 * np.pi * 0.7 * t))
    phase = np.cumsum(f / SR)
    x = (np.diff(np.floor(phase), prepend=0.0) > 0).astype(np.float64)
    for fc, bw in ((700.0, 110.0), (1220.0, 120.0), (2600.0, 160.0)):
        r = np.exp(-np.pi * bw / SR)
        x = lfilter([1.0 - r], [1.0, -2.0 * r * np.cos(2 * np.pi * fc / SR), r * r], x)
    x += 1e-3 * rng.standard_normal(n)
    best = None
    syl = 0.5 + 0.5 * np.cos(2 * np.pi * 4.0 * t)
    envs = [1.0 - depth * syl ** 2 for depth in np.linspace(0.0, 0.98, 50)] + [syl ** k for k in np.linspace(0.1, 16.0, 160)]
    for env in envs:
        y = x * env
        y = y / np.abs(y).max() * 0.5
        plr = 20 * np.log10(0.5) - loudness_oracle.integrated_loudness(y, SR)
        if best is None or abs(plr - plr_db) < abs(best[0] - plr_db):
            best = (plr, y)
    return best[1].astype(np.float32)


def test_envelope_never_exceeds_the_required_gain():
    rng = np.random.default_rng(1)
    for x, g in ((sine_45(), 1.0), (np.clip(0.3 * rng.standard_normal(2 * SR), -1, 1).astype(np.float32), 3.0), (voiced(16.0), 4.0)):
        for rate in (16000, 8000, 11025, 48000):
            y, G, r = O.limit(x, SR, rate, -1.0, g)
            assert len(G) == len(r) == len(x)
            assert np.all(G <= r), (rate, np.max(G - r))
            assert np.all(G <= 0.0)


def test_prefix_minimum_release_is_the_recurrence_bit_for_bit():
    rng = np.random.default_rng(2)
    x = np.clip(0.4 * rng.standard_normal(3 * SR), -1, 1).astype(np.float32)
    for g in (1.0, 2.5):
        r = O.required(O.detect(x, SR, SR), g, -3.0)
        m = O.hold_min(r, O.lookahead(SR), O.hold(SR, SR))
        rho = O.release(SR)
        assert rho / O.Q == int(rho / O.Q)
        a, b = O.release_recurrence(m, rho), O.release_prefix(m, rho)
        assert np.array_equal(a.view(np.int64), b.view(np.int64))
        assert a.min() < -1.0


@pytest.mark.parametrize("where", ["start", "end"])
def test_peaks_at_the_item_edges_are_limited(where):
    L, M = O.lookahead(SR), O.hold(SR, SR)
    x = np.zeros(SR, np.float32)
    x[[0, 1, 2] if where == "start" else [-3, -2, -1]] = [0.9, -0.95, 0.9]
    y, G, r = O.limit(x, SR, SR, -6.0)
    edge = slice(0, L + M) if where == "start" else slice(SR - L - M, SR)
    assert np.all(G[edge][r[edge] < 0] <= r[edge][r[edge] < 0])
    assert O.true_peak_db(y, SR) <= -6.0 + 0.05


def test_a_lone_peak_releases_at_60_db_per_second():
    L, M = O.lookahead(SR), O.hold(SR, SR)
    x = np.zeros(2 * SR, np.float32)
    x[SR // 2] = 1.0
    y, G, r = O.limit(x, SR, SR, -12.0)
    assert G.min() <= -12.0
    # once the look-ahead window has passed, G rises by rho per sample, averaged over L + 1 samples: a straight line
    start = SR // 2 + M + L + 1
    stop = start + int(0.1 * SR)
    slope = np.diff(G[start:stop])
    assert np.allclose(slope, O.release(SR), rtol=0, atol=1e-9), (slope.min(), slope.max())
    assert abs(O.release(SR) * SR - 60.0) <= SR * O.Q
    assert G[-1] == 0.0


def test_true_peak_bound_of_the_oracle_output():
    from scipy.signal import resample_poly
    rng = np.random.default_rng(3)
    sig = {"sine_45": sine_45(), "pm_one": np.tile(np.array([1, 1, -1, -1], np.float32), SR // 4),
           "voiced16": voiced(16.0), "noise": np.clip(0.3 * rng.standard_normal(2 * SR), -1, 1).astype(np.float32)}
    for name, x in sig.items():
        for C in (-1.0, -3.0):
            for rate, (up, down) in ((16000, (1, 1)), (24000, (3, 2)), (48000, (3, 1))):
                y, _, _ = O.limit(x, SR, rate, C, 2.0 if name == "voiced16" else 1.0)
                z = y.astype(np.float64) if up == down else resample_poly(y.astype(np.float64), up, down)
                # a full-scale start is cut off again by the resampled output (see test_limiter_gpu.py): 0.05 dB inside
                assert O.true_peak_db(z, rate, 0.002) <= C + 0.05, (name, C, rate, O.true_peak_db(z, rate, 0.002))
                assert O.true_peak_db(z, rate) <= C + (0.05 if up == down else 0.1), (name, C, rate, O.true_peak_db(z, rate))


@pytest.mark.parametrize("rate", [8000, 11025, 16000, 22050, 44100])
def test_host_bank_is_the_oracles_filter(rate):
    bank, hold = audio.limit_bank(SR, rate)
    h, c, phases = O.detector_filter(SR, rate)
    R = O.oversampling(SR)
    assert hold == O.hold(SR, rate) and bank.shape == (len(phases), 2 * c + 1)
    for row, ph in zip(bank, phases):
        want = h[ph::R]
        assert np.array_equal(row[:len(want)], want.astype(np.float32)) and not row[len(want):].any()
    assert audio.limit_lookahead(SR) == O.lookahead(SR) == 80
    assert audio.limit_release(SR) == O.release(SR)


def test_hold_and_oversampling_per_rate():
    assert O.oversampling(16000) == 12 and O.oversampling(24000) == 8 and O.oversampling(44100) == 5
    assert [audio.limit_bank(SR, r)[1] for r in (8000, 11025, 16000, 22050, 24000, 44100, 48000)] == [30, 25, 10, 10, 10, 10, 10]


def test_true_peak_ceilings_are_checked():
    assert audio.check_true_peak(-1) == -1.0 and audio.check_true_peak(np.float32(-3.0)) == -3.0
    assert audio.check_true_peak(0) == 0.0 and audio.check_true_peak(-20.0) == -20.0
    for bad in (float("nan"), float("inf"), -float("inf"), 0.5, -20.01, -100, True, False, np.bool_(True), "-1", None, [-1]):
        with pytest.raises(ValueError):
            audio.check_true_peak(bad)


def test_microbatcher_formats_once_per_key_with_ceilings(monkeypatch):
    wav = torch.zeros(6, 1, 512)

    def forward(**kw):
        return {"wav_predictions": wav[:len(kw["inputs_ling"])], "mel_lengths": torch.full((len(kw["inputs_ling"]),), 2)}

    calls = []

    def fake_fetch(model, out, sample_rate=None, encoding="pcm16", items=None, hop=None, loudness=None, true_peak=None):
        calls.append((sample_rate, encoding, loudness, true_peak, tuple(items)))
        return [np.array([len(calls)]) for _ in items]

    monkeypatch.setattr(fd, "fetch_audio", fake_fetch)
    z = np.zeros(768, np.float32)
    reqs = [dict(loudness=-16, true_peak=-1), dict(loudness=-16, true_peak=-1.0), dict(loudness=-16), dict(true_peak=-2),
            dict(loudness=-16, true_peak=-3, sample_rate=8000, encoding="mulaw"), dict()]
    with fd.MicroBatcher(forward, max_batch=6, max_wait_s=0.5) as mb:
        for kw in (dict(true_peak=float("nan")), dict(true_peak=1.0), dict(true_peak="-1"), dict(true_peak=True), dict(true_peak=-21)):
            with pytest.raises(ValueError):
                mb.submit(np.array([1, 2]), 0, z, z, **kw)
            with pytest.raises(ValueError):
                mb.submit_joined([np.array([1, 2])], 0, z, z, **kw)
        futs = [mb.submit(np.array([1, 2, 3]), 0, z, z, **kw) for kw in reqs]
        got = [f.result(timeout=30) for f in futs]
        assert mb.batches_run == 1
    assert sorted(calls, key=str) == sorted([(16000, "pcm16", -16.0, -1.0, (0, 1)), (16000, "pcm16", -16.0, None, (2,)),
                                             (16000, "pcm16", None, -2.0, (3,)), (8000, "mulaw", -16.0, -3.0, (4,))], key=str)
    assert got[0][0] == got[1][0] and isinstance(got[5], torch.Tensor)
    assert fd.MicroBatcher._output_format(mb, None, None, -23, -1) == audio.OutputFormat(16000, 1, 1, "pcm16", -23.0, -1.0)
    assert fd.MicroBatcher._output_format(mb, None, None, None, -1) == audio.OutputFormat(16000, 1, 1, "pcm16", None, -1.0)
    assert fd.MicroBatcher._output_format(mb, None, None, -23, None) == audio.OutputFormat(16000, 1, 1, "pcm16", -23.0, None)
