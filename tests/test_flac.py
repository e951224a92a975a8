"""FLAC output on the host (no GPU): the CRCs' catalogue values, a hand-assembled stream, encoder / decoder round trips of the
oracle over signals and lengths, sizes, corruption detection, the rate planning and frame-header rate codes, and the
MicroBatcher's grouping of flac requests."""
import numpy as np
import pytest
import torch

from emotivoice_b200 import audio
from emotivoice_b200 import frontdoor as fd
from oracle import flac_oracle as F
from test_audio_format import RATES

SR = 16000


def test_crcs_give_the_catalogue_check_values():
    assert F.crc8(b"123456789") == 0xF4          # CRC-8 (poly 0x07, init 0)
    assert F.crc16(b"123456789") == 0xFEE8       # CRC-16/UMTS (poly 0x8005, init 0)


# 4096 samples of 1000 (one CONSTANT frame), then a 20-sample ramp 100, 107, ..., 233 (one FIXED order-2 frame, zero residual)
HAND = bytes([
    0x66, 0x4C, 0x61, 0x43,                  # "fLaC" (RFC 9639 section 6)
    0x80, 0x00, 0x00, 0x22,                  # metadata block header: last block, type 0 STREAMINFO, 34 bytes (8.1)
    0x10, 0x00, 0x10, 0x00,                  # STREAMINFO (8.2): min block size 4096, max block size 4096
    0x00, 0x00, 0x0B, 0x00, 0x00, 0x12,      # min frame size 11, max frame size 18
    0x03, 0xE8, 0x00,                        # sample rate 16000 (20 bits), channels - 1 = 0 (3 bits), then
    0xF0,                                    #   bits per sample - 1 = 15 (5 bits), total samples (36 bits) ...
    0x00, 0x00, 0x10, 0x14,                  #   ... = 4116
    0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00, 0x00,   # MD5 unknown
    # frame 0 (9.1)
    0xFF, 0xF8,                              # sync 0b11111111111110, reserved 0, fixed block size 0
    0xC5,                                    # block size 1100 (4096), sample rate 0101 (16 kHz) (9.1.1, 9.1.2)
    0x08,                                    # channels 0000 (mono), sample size 100 (16 bits), reserved 0 (9.1.3, 9.1.4)
    0x00,                                    # frame number 0, coded number (9.1.5)
    0x6F,                                    # CRC-8 of the header (9.1.8)
    0x00,                                    # subframe header (9.2.1): 0, type 000000 CONSTANT, no wasted bits
    0x03, 0xE8,                              # the constant 1000 (9.2.3)
    0x6D, 0x25,                              # CRC-16 of the frame (9.3)
    # frame 1
    0xFF, 0xF8,
    0x65,                                    # block size 0110 (8-bit n - 1 follows), sample rate 0101
    0x08,
    0x01,                                    # frame number 1
    0x13,                                    # block size - 1 = 19 (9.1.6)
    0x99,                                    # CRC-8
    0x14,                                    # subframe header: 0, type 001010 FIXED order 2, no wasted bits (9.2.5)
    0x00, 0x64, 0x00, 0x6B,                  # warm-up samples 100, 107
    0x00, 0x3F, 0xFF, 0xF0,                  # residual (9.2.7): method 00, partition order 0000, Rice parameter 0000,
                                             #   18 codes "1" (zero), 4 zero bits of padding to the byte
    0xAF, 0x28,                              # CRC-16
])


def test_hand_assembled_stream():
    x = np.concatenate([np.full(4096, 1000), 100 + 7 * np.arange(20)]).astype(np.int16)
    assert F.encode(x, SR) == HAND
    rate, y, stats = F.decode(HAND)
    assert rate == SR and np.array_equal(y, x)
    assert [(s["type"], s["order"]) for s in stats] == [("CONSTANT", 0), ("FIXED", 2)]


def _q(x):
    return np.clip(np.round(x), -32768, 32767).astype(np.int16)


def signals(n=3 * SR, seed=0):
    """The test signals: silence, DC, a ramp, tones at -6 / -20 / -60 dBFS, noise at three levels, a full-scale square wave and
    samples at both int16 extremes."""
    t = np.arange(n)
    rng = np.random.default_rng(seed)
    tone = lambda db, f: 10 ** (db / 20) * 32767 * np.sin(2 * np.pi * f * t / SR)
    return {
        "silence": np.zeros(n, np.int16),
        "dc": np.full(n, -1234, np.int16),
        "ramp": ((t * 13) % 65536 - 32768).astype(np.int16),
        "tone_m6": _q(tone(-6, 440.0)),
        "tone_m20": _q(tone(-20, 997.0)),
        "tone_m60": _q(tone(-60, 220.0)),
        "noise_m10": _q(rng.normal(0, 10 ** (-10 / 20) * 32767 / 3, n)),
        "noise_m30": _q(rng.normal(0, 10 ** (-30 / 20) * 32767, n)),
        "noise_m60": _q(rng.normal(0, 10 ** (-60 / 20) * 32767, n)),
        "square": np.where((t // 37) % 2, 32767, -32768).astype(np.int16),
        "extremes": rng.choice(np.array([-32768, 32767], np.int16), n),
    }


def test_round_trip_on_signals_and_every_subframe_kind_occurs():
    kinds = set()
    for name, x in signals().items():
        img = F.encode(x, SR)
        rate, y, stats = F.decode(img)
        assert rate == SR and y.dtype == np.int16 and np.array_equal(y, x), name
        kinds |= {s["type"] for s in stats}
        for s in stats:
            assert s["bytes"] <= 16 + 1 + 2 * s["samples"] + 2, (name, s)          # never above its VERBATIM frame
    assert kinds == {"CONSTANT", "FIXED", "LPC", "VERBATIM"}


@pytest.mark.parametrize("n", list(range(1, 21)) + [4095, 4096, 4097, 8191, 8192, 8193, 12289, 256, 257])
def test_round_trip_at_length_edges(n):
    rng = np.random.default_rng(n)
    for x in (rng.integers(-40, 40, n).astype(np.int16), _q(3000 * np.sin(np.arange(n) * 0.05)), np.full(n, 7, np.int16)):
        rate, y, stats = F.decode(F.encode(x, 44100))
        assert rate == 44100 and np.array_equal(y, x)
        assert len(stats) == -(-n // F.BLOCK)
        for s in stats:
            assert s["order"] < s["samples"] or s["type"] in ("CONSTANT", "VERBATIM")


def test_round_trip_at_random_lengths():
    rng = np.random.default_rng(7)
    for n in rng.integers(1, 30000, 8):
        x = _q(rng.normal(0, 500, n) + 4000 * np.sin(np.arange(n) * 0.01))
        assert np.array_equal(F.decode(F.encode(x, 24000))[1], x)


def test_sizes():
    s = signals()
    n = len(s["silence"])
    frames = -(-n // F.BLOCK)
    assert len(F.encode(s["silence"], SR)) <= 42 + 12 * frames               # a few bytes per frame
    assert len(F.encode(s["tone_m20"], SR)) <= 0.25 * 2 * n
    assert len(F.encode(s["noise_m60"], SR)) < len(F.encode(s["noise_m30"], SR)) < 2 * n


def test_a_flipped_bit_in_a_frame_is_detected():
    rng = np.random.default_rng(3)
    x = np.concatenate([_q(2000 * np.sin(np.arange(4096) * 0.03) + rng.normal(0, 30, 4096)), rng.integers(-9, 9, 300).astype(np.int16)])
    img = F.encode(x, 22050)
    bits = 8 * (len(img) - 42)
    positions = sorted(set(range(0, 8 * 64)) | set(rng.integers(0, bits, 400).tolist()) | set(range(bits - 8 * 24, bits)))
    for p in positions:
        bad = bytearray(img)
        bad[42 + p // 8] ^= 0x80 >> (p % 8)
        with pytest.raises(F.FlacError):
            F.decode(bytes(bad))


def test_decoder_checks_streaminfo():
    img = bytearray(HAND)
    img[13] = 0x13                           # max frame size 19
    with pytest.raises(F.FlacError):
        F.decode(bytes(img))
    img = bytearray(HAND)
    img[25] = 0x15                           # total samples 4117
    with pytest.raises(F.FlacError):
        F.decode(bytes(img))


FRAME_RATE_CODES = {8000: (4, 0, 0), 11025: (13, 11025, 16), 12000: (12, 12, 8), 16000: (5, 0, 0), 22050: (6, 0, 0),
                    24000: (7, 0, 0), 32000: (8, 0, 0), 44100: (9, 0, 0), 48000: (10, 0, 0), 96000: (11, 0, 0), 192000: (3, 0, 0),
                    88200: (1, 0, 0), 176400: (2, 0, 0), 4000: (12, 4, 8), 100000: (12, 100, 8), 65535: (13, 65535, 16),
                    100010: (14, 10001, 16), 127625: (0, 0, 0), 65537: (0, 0, 0)}


@pytest.mark.parametrize("rate", sorted(RATES))
def test_plan_accepts_flac_at_every_listed_rate(rate):
    assert audio.plan(rate, "flac", SR) == (rate,) + RATES[rate]
    assert audio.flac_rate_code(rate) == FRAME_RATE_CODES[rate]


def test_frame_header_rate_codes():
    for rate, want in FRAME_RATE_CODES.items():
        assert audio.flac_rate_code(rate) == want == F.rate_code(rate), rate
    for rate in (11025, 127625, 100010):
        x = np.arange(-50, 50, dtype=np.int16)
        assert F.decode(F.encode(x, rate))[0] == rate
    assert audio.NUMPY_DTYPES["flac"] is np.uint8 and "flac" not in audio.ENCODINGS
    with pytest.raises(ValueError):
        fd.audio_to_wav_bytes(np.zeros(8, np.uint8), SR, "flac")


def test_microbatcher_groups_flac_with_other_formats(monkeypatch):
    wav = torch.zeros(4, 1, 512)
    forwards = []

    def forward(**kw):
        forwards.append(len(kw["inputs_ling"]))
        return {"wav_predictions": wav[:len(kw["inputs_ling"])], "mel_lengths": torch.full((len(kw["inputs_ling"]),), 2)}

    calls = []

    def fake_fetch(model, out, sample_rate=None, encoding="pcm16", items=None, hop=None, loudness=None, true_peak=None):
        calls.append((sample_rate, encoding, loudness, true_peak, tuple(items)))
        return [np.array([len(calls)], audio.NUMPY_DTYPES[encoding]) for _ in items]

    monkeypatch.setattr(fd, "fetch_audio", fake_fetch)
    z = np.zeros(768, np.float32)
    reqs = [dict(encoding="flac"), dict(encoding="pcm16"), dict(encoding="mulaw", sample_rate=8000), dict(encoding="flac")]
    with fd.MicroBatcher(forward, max_batch=4, max_wait_s=0.5) as mb:
        futs = [mb.submit(np.array([1, 2, 3]), 0, z, z, **kw) for kw in reqs]
        got = [f.result(timeout=30) for f in futs]
        assert mb.batches_run == 1
    assert forwards == [4]
    assert sorted(calls, key=str) == sorted([(16000, "flac", None, None, (0, 3)), (16000, "pcm16", None, None, (1,)),
                                             (8000, "mulaw", None, None, (2,))], key=str)
    assert got[0].dtype == np.uint8 and got[0][0] == got[3][0]
    assert fd.MicroBatcher._output_format(mb, 48000, "flac", -16) == audio.OutputFormat(48000, 3, 1, "flac", -16.0, None)
