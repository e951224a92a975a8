"""The watermark's definition and host side, without a GPU: the fp64 oracle's transform and pattern, the false-positive
behaviour of the detector statistic over many keys, the format checks, and the MicroBatcher's watermark plumbing.  Also holds
the seeded speech-like signals the GPU tests mark and detect."""
import numpy as np
import pytest
import torch
from scipy.signal import lfilter

from emotivoice_b200 import audio
from emotivoice_b200 import frontdoor as fd
from emotivoice_b200 import watermark
from oracle import watermark_oracle as W

SR = 16000
MASK = (1 << 64) - 1
VOWELS = ((730, 1090, 2440), (270, 2290, 3010), (300, 870, 2240), (530, 1840, 2480), (640, 1190, 2390), (490, 1350, 1690))


def speech_like(seconds, seed, peak=0.5):
    """A seeded voiced signal at 16 kHz: syllables of 120-320 ms, each a harmonic source (glottal-like 1/h spectrum, F0 gliding
    in 90-240 Hz) through three formant resonators of a vowel, under a raised-cosine envelope, grouped into phrases separated by
    pauses of digital silence (150-450 ms)."""
    rng = np.random.default_rng(seed)
    n = int(seconds * SR)
    out = np.zeros(n)
    t = 0
    while t < n:
        for _ in range(rng.integers(3, 9)):                          # one phrase
            m = int(rng.uniform(0.12, 0.32) * SR)
            f0 = np.linspace(rng.uniform(90, 240), rng.uniform(90, 240), m)
            ph = 2 * np.pi * np.cumsum(f0) / SR
            src = sum(np.sin(h * ph) / h * (h * f0 < 7000) for h in range(1, 60))
            y = src + 0.02 * rng.standard_normal(m)
            for f in VOWELS[rng.integers(len(VOWELS))]:
                r, w = np.exp(-np.pi * 90.0 / SR), 2 * np.pi * f / SR
                y = lfilter([1 - r], [1, -2 * r * np.cos(w), r * r], y)
            seg = y * np.sin(np.pi * np.arange(m) / m) ** 0.5
            end = min(n, t + m)
            out[t:end] = seg[:end - t]
            t = end
            if t >= n:
                break
        t += int(rng.uniform(0.15, 0.45) * SR)
    return (out * peak / np.max(np.abs(out))).astype(np.float32)


def _mix64(x):
    x = (x + 0x9E3779B97F4A7C15) & MASK
    x = ((x ^ (x >> 30)) * 0xBF58476D1CE4E5B9) & MASK
    x = ((x ^ (x >> 27)) * 0x94D049BB133111EB) & MASK
    return x ^ (x >> 31)


def test_oracle_mdct_reconstructs_perfectly():
    x = np.random.default_rng(0).uniform(-1, 1, 7777)
    bins = np.arange(W.H)
    C, _ = W.mclt(x, 0, bins)
    assert C.shape == (W.n_frames(len(x)), W.H) == (17, 512)
    assert np.max(np.abs(W.imdct(C, len(x), bins) - x)) < 1e-12


def test_oracle_embed_with_zero_alpha_is_the_identity():
    x = speech_like(1.0, 3).astype(np.float64)
    assert np.array_equal(W.embed(x, 12345, alpha=0.0), x)
    assert np.array_equal(W.embed(np.zeros(5000), 12345), np.zeros(5000))


def test_pattern_is_splitmix64():
    # SplitMix64 seeded with 0 returns mix64(0), mix64(golden), mix64(2 golden), ...
    g = 0x9E3779B97F4A7C15
    assert [_mix64(i * g & MASK) for i in range(3)] == [0xE220A8397B1DCDAF, 0x6E789E6AA1B965F4, 0x06C45D188009454F]
    assert [int(v) for v in W.mix64(np.array([0, g, 2 * g & MASK], np.uint64))] == [_mix64(0), _mix64(g), _mix64(2 * g & MASK)]
    for key, r, k in ((1, 0, 19), (12345, 63, 217), (2 ** 63 - 1, 17, 100)):
        want = -1.0 if _mix64(key ^ _mix64((r << 10) | k)) >> 63 else 1.0
        assert W.pattern(key)[r, k - W.K_LO] == want
    s = W.pattern(777)
    assert s.shape == (64, 199) and abs(s.mean()) < 0.03


def test_constants_match_the_oracle():
    assert (audio.WATERMARK_N, audio.WATERMARK_HOP, audio.WATERMARK_PERIOD) == (W.N, W.H, W.P)
    assert audio.WATERMARK_BAND == (W.K_LO, W.K_HI) and audio.WATERMARK_ALPHA == W.ALPHA
    assert watermark.DETECT_Z == 7.0
    assert 512 * 64 * np.exp(-watermark.DETECT_Z ** 2 / 2) < 7.7e-7      # the bound in watermark's docstring


def test_z_over_many_keys_is_standard_and_never_reaches_the_threshold():
    """2000 keys on two fixed unmarked signals: z at one hypothesis has mean ~0 and standard deviation ~1, and no key's
    full-search maximum over all 512 x 64 hypotheses reaches DETECT_Z."""
    keys = [int(k) for k in np.random.default_rng(5).integers(1, 2 ** 63 - 1, 2000, dtype=np.int64)]
    sigs = (np.random.default_rng(6).standard_normal(12000) * 0.1, speech_like(1.0, 7).astype(np.float64))
    for x in sigs:
        b = W.fold(x)
        den = np.sqrt((b[0] ** 2).sum())
        z0 = np.array([(W.pattern(k) * b[0]).sum() / den for k in keys])
        assert abs(z0.mean()) < 0.1 and abs(z0.std() - 1.0) < 0.1, (z0.mean(), z0.std())
        zmax = W.z_max_keys(b, keys)
        assert zmax.max() < watermark.DETECT_Z, zmax.max()
        assert np.isclose(zmax[0], W.z_table(b, keys[0]).max())


def test_output_format_checks_the_key_after_the_others():
    with pytest.raises(ValueError, match="sample_rate"):
        audio.output_format(3000, "pcm16", None, None, SR, watermark=True)
    with pytest.raises(ValueError, match="loudness"):
        audio.output_format(None, "pcm16", 5, None, SR, watermark=0)
    with pytest.raises(ValueError, match="true_peak"):
        audio.output_format(None, "pcm16", None, 3, SR, watermark=0)
    for bad in (True, np.bool_(True), 1.0, "7", 0, -3, 2 ** 63):
        with pytest.raises(ValueError, match="watermark"):
            audio.output_format(None, "pcm16", None, None, SR, watermark=bad)
    with pytest.raises(ValueError, match="8000"):
        audio.output_format(4000, "pcm16", None, None, SR, watermark=5)
    assert audio.output_format(8000, "mulaw", None, None, SR, watermark=np.int64(5)).watermark == 5
    assert audio.output_format(None, "pcm16", None, None, SR, watermark=2 ** 63 - 1).watermark == 2 ** 63 - 1
    assert audio.output_format(4000, "pcm16", None, None, SR).watermark is None


def test_output_format_equality_and_hash():
    six = audio.OutputFormat(48000, 3, 1, "flac", -16.0, None)
    assert six == audio.OutputFormat(48000, 3, 1, "flac", -16.0, None, None) == (48000, 3, 1, "flac", -16.0, None)
    assert audio.output_format(48000, "flac", -16, None, SR) == six and six.watermark is None and six.true_peak is None
    marked = audio.output_format(48000, "flac", -16, None, SR, watermark=9)
    assert marked != six and marked.watermark == 9 and marked.rate == 48000 and marked.loudness == -16.0
    assert marked == audio.OutputFormat(48000, 3, 1, "flac", -16.0, None, 9)
    d = {six: 1, marked: 2, audio.output_format(48000, "flac", -16, None, SR, watermark=10): 3}
    assert len(d) == 3 and d[audio.OutputFormat(48000, 3, 1, "flac", -16.0, None)] == 1
    assert hash(marked) == hash(audio.OutputFormat(48000, 3, 1, "flac", -16.0, None, 9))
    assert "watermark=9" in repr(marked)


def test_microbatcher_passes_watermark_only_when_asked(monkeypatch):
    wav = torch.zeros(6, 1, 512)

    def forward(**kw):
        return {"wav_predictions": wav[:len(kw["inputs_ling"])], "mel_lengths": torch.full((len(kw["inputs_ling"]),), 2)}

    calls = []

    def fake_fetch(model, out, sample_rate=None, encoding="pcm16", items=None, hop=None, loudness=None, true_peak=None, **kw):
        calls.append((sample_rate, encoding, tuple(sorted(kw.items())), tuple(items)))
        return [np.array([len(calls)], audio.NUMPY_DTYPES[encoding]) for _ in items]

    monkeypatch.setattr(fd, "fetch_audio", fake_fetch)
    z = np.zeros(768, np.float32)
    reqs = [dict(encoding="flac", watermark=11), dict(encoding="pcm16"), dict(watermark=11), dict(encoding="flac", watermark=12),
            dict(encoding="flac", watermark=11), dict(sample_rate=8000, encoding="mulaw", watermark=12)]
    with fd.MicroBatcher(forward, max_batch=6, max_wait_s=0.5) as mb:
        futs = [mb.submit(np.array([1, 2, 3]), 0, z, z, **kw) for kw in reqs]
        got = [f.result(timeout=30) for f in futs]
        assert mb.batches_run == 1
        with pytest.raises(ValueError, match="watermark"):
            mb.submit(np.array([1, 2, 3]), 0, z, z, watermark=True)
        with pytest.raises(ValueError, match="8000"):
            mb.submit_joined([np.array([1, 2])], 0, z, z, sample_rate=4000, watermark=3)
    assert sorted(calls, key=str) == sorted([(16000, "flac", (("watermark", 11),), (0, 4)), (16000, "pcm16", (), (1,)),
                                             (16000, "pcm16", (("watermark", 11),), (2,)), (16000, "flac", (("watermark", 12),), (3,)),
                                             (8000, "mulaw", (("watermark", 12),), (5,))], key=str)
    assert got[0][0] == got[4][0]
    assert fd.MicroBatcher._output_format(mb, None, None, None, None, 5) == audio.OutputFormat(16000, 1, 1, "pcm16", None, None, 5)
    assert fd.MicroBatcher._output_format(mb, None, None, None, None, None) is None
