"""Output formats on the host (no GPU): rate planning, the polyphase filter bank against scipy's own resample_poly filter, output
lengths and packing offsets, the WAV images, and the MicroBatcher's checks of a request's format."""
import io
import struct
import wave

import numpy as np
import pytest
from scipy.signal import firwin, resample_poly

from emotivoice_b200 import audio
from emotivoice_b200 import frontdoor as fd

SR = 16000
RATES = {8000: (1, 2), 11025: (441, 640), 12000: (3, 4), 16000: (1, 1), 22050: (441, 320), 24000: (3, 2), 32000: (2, 1),
         44100: (441, 160), 48000: (3, 1), 96000: (6, 1), 192000: (12, 1)}


@pytest.mark.parametrize("rate", sorted(RATES))
def test_listed_rates_plan_to_their_ratio(rate):
    for enc in audio.ENCODINGS:
        assert audio.plan(rate, enc, SR) == (rate,) + RATES[rate]
    assert audio.plan(np.int64(rate), "pcm16", SR) == (rate,) + RATES[rate]
    assert audio.plan(float(rate), "pcm16", SR) == (rate,) + RATES[rate]


def test_source_rate_is_the_default_and_bad_requests_raise():
    assert audio.plan(None, "pcm16", SR) == (SR, 1, 1)
    assert audio.plan(4000, "mulaw", SR) == (4000, 1, 4)
    for rate in (3999, 192001, 0, -8000, 22050.5, float("nan"), float("inf"), "24000", True, [24000],
                 4001,           # 4001/16000: factors 4001 and 16000
                 16001):         # 16001/16000
        with pytest.raises(ValueError):
            audio.plan(rate, "pcm16", SR)
    for enc in ("mp3", "PCM16", "int16", None, "ulaw", 1):
        with pytest.raises(ValueError):
            audio.plan(24000, enc, SR)


def test_output_format_checks_rate_then_loudness_then_ceiling():
    assert audio.output_format(48000, "flac", -16, np.float32(-1.0), SR) == audio.OutputFormat(48000, 3, 1, "flac", -16.0, -1.0)
    assert audio.output_format(None, "pcm16", None, None, SR) == (SR, 1, 1, "pcm16", None, None)
    assert hash(audio.output_format(8000, "mulaw", -23, None, SR)) == hash(audio.output_format(8000.0, "mulaw", -23.0, None, SR))
    for args, what in (((3999, "pcm16", 1.0, 1.0), "sample_rate"), ((None, "mp3", 1.0, 1.0), "encoding"),
                       ((None, "pcm16", 1.0, 1.0), "loudness"), ((None, "pcm16", -23, 1.0), "true_peak")):
        with pytest.raises(ValueError, match=what):
            audio.output_format(*args, SR)


def _scipy_filter(up, down):
    """resample_poly's own filter (float64, multiplied by up), read back from resample_poly: unit impulses spaced so that no
    output receives two of them, placed so that together they meet every filter tap.  Each such output is one tap times 1.0
    plus exact zeros, so it is the tap bit for bit."""
    half = 10 * max(up, down)
    N = 2 * half + 1
    M = -(-N // up) + 1
    M += (1 - M) % down                       # M = 1 (mod down): impulse r meets the taps k = half - r * up (mod down)
    P0 = -(-N // up)
    pos = P0 + M * np.arange(down)
    n = int(pos[-1]) + M
    x = np.zeros(n)
    x[pos] = 1.0
    y = resample_poly(x, up, down)
    h = np.full(N, np.nan)
    for p in pos:
        o0 = -(-(p * up - half) // down)      # outputs o with 0 <= o * down + half - p * up < N
        for o in range(max(o0, 0), len(y)):
            k = o * down + half - p * up
            if k >= N:
                break
            h[k] = y[o]
    assert not np.isnan(h).any()
    return h


@pytest.mark.parametrize("rate", sorted(r for r in RATES if r != SR))
def test_filter_bank_is_scipys_default_filter(rate):
    up, down = RATES[rate]
    h = audio.resample_filter(up, down)
    want = _scipy_filter(up, down)
    assert h.dtype == np.float64 and np.array_equal(h, want)
    ref = firwin(20 * max(up, down) + 1, 1.0 / max(up, down), window=("kaiser", 5.0))
    ref *= up
    assert np.array_equal(h, ref)
    bank = audio.polyphase_bank(up, down)
    taps = -(-len(h) // up)
    assert bank.dtype == np.float32 and bank.shape == (up, taps) and bank.flags.c_contiguous
    for p in range(up):
        row = h[p::up].astype(np.float32)
        assert np.array_equal(bank[p, :len(row)], row) and not bank[p, len(row):].any()


@pytest.mark.parametrize("rate", sorted(RATES))
def test_output_lengths_and_offsets_follow_resample_poly(rate):
    up, down = RATES[rate]
    ns = [1, 255, 256, 257, 137472]
    for n in ns:
        assert audio.resampled_length(n, up, down) == len(resample_poly(np.zeros(n), up, down))
    offs = audio.packed_offsets(ns, [4, 0, 2], up, down)
    lens = [len(resample_poly(np.zeros(ns[b]), up, down)) for b in (4, 0, 2)]
    assert offs.dtype == np.int64 and offs.tolist() == [0, lens[0], lens[0] + lens[1], sum(lens)]


@pytest.mark.parametrize("rate", [24000, 48000])
def test_pcm16_wav_image_at_other_rates_reads_back(rate):
    pcm = np.random.default_rng(rate).integers(-32768, 32768, size=rate // 10 + 1).astype(np.int16)
    img = fd.audio_to_wav_bytes(pcm, rate, "pcm16")
    assert img == fd.pcm16_to_wav_bytes(pcm, rate)
    with wave.open(io.BytesIO(img)) as w:
        assert (w.getnchannels(), w.getsampwidth(), w.getframerate(), w.getnframes()) == (1, 2, rate, len(pcm))
        assert np.array_equal(np.frombuffer(w.readframes(len(pcm)), "<i2"), pcm)


@pytest.mark.parametrize("encoding,tag", [("mulaw", 7), ("alaw", 6)])
@pytest.mark.parametrize("n", [0, 1, 8000])
def test_g711_wav_header_fields(encoding, tag, n):
    codes = np.random.default_rng(n).integers(0, 256, size=n).astype(np.uint8)
    img = fd.audio_to_wav_bytes(codes, 8000, encoding)
    pad = n & 1
    assert len(img) == 58 + n + pad
    assert img[0:4] == b"RIFF" and struct.unpack("<I", img[4:8])[0] == len(img) - 8 and img[8:12] == b"WAVE"
    assert img[12:16] == b"fmt " and struct.unpack("<I", img[16:20])[0] == 18
    fmt = struct.unpack("<HHIIHHH", img[20:38])
    assert fmt == (tag, 1, 8000, 8000, 1, 8, 0)       # tag, channels, rate, bytes/s, block align, bits, cbSize
    assert img[38:42] == b"fact" and struct.unpack("<II", img[42:50]) == (4, n)
    assert img[50:54] == b"data" and struct.unpack("<I", img[54:58])[0] == n
    assert img[58:58 + n] == codes.tobytes() and img[58 + n:] == b"\0" * pad


def test_wav_writer_rejects_what_it_cannot_hold():
    for enc, data in (("mulaw", np.zeros(4, np.int16)), ("alaw", np.zeros((2, 2), np.uint8)), ("float32", np.zeros(4, np.float32)),
                      ("mp3", np.zeros(4, np.uint8))):
        with pytest.raises(ValueError):
            fd.audio_to_wav_bytes(data, 8000, enc)


def test_microbatcher_checks_the_format_before_queueing():
    calls = []

    def forward(**kw):
        calls.append(kw)
        raise AssertionError("no request should reach the model")

    z = np.zeros(768, np.float32)
    with fd.MicroBatcher(forward, max_batch=2, max_wait_s=0.01) as mb:
        for kw in (dict(sample_rate=44100.5), dict(sample_rate=1000), dict(encoding="mp3"), dict(sample_rate=24000, encoding="ogg")):
            with pytest.raises(ValueError):
                mb.submit(np.array([1, 2]), 0, z, z, **kw)
            with pytest.raises(ValueError):
                mb.submit_joined([np.array([1, 2])], 0, z, z, **kw)
    assert not calls
