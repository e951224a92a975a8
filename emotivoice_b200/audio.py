"""Host side of the output formats (``JETSGenerator.format_audio``, ``frontdoor.fetch_audio``): which rates and encodings are
accepted, the resampling ratio, the polyphase filter bank ``ev_format_audio`` runs, the loudness targets and K-weighting
filter of ``ev_loudness``, the ceiling checks, detector bank and fixed constants of ``ev_limit``, and the frame-header rate code
of ``ev_flac_encode``, and the watermark's constants and key check.  Pure host code, no CUDA.

Resampling is ``scipy.signal.resample_poly(x, up, down)`` with its defaults: the filter is
``firwin(2 * 10 * max(up, down) + 1, 1 / max(up, down), window=('kaiser', 5.0)) * up``, input outside the item is zero, and an
item of n samples gives ``ceil(n * up / down)`` samples.
"""
import collections
import math

import numpy as np

ENCODINGS = {"float32": 0, "pcm16": 1, "mulaw": 2, "alaw": 3}        # EV_AUDIO_* (include/emotivoice_b200.h)
FLAC = "flac"                   # a complete .flac file image per output (ev_flac_encode); not an EV_AUDIO_* sample encoding
NUMPY_DTYPES = {"float32": np.float32, "pcm16": np.int16, "mulaw": np.uint8, "alaw": np.uint8, FLAC: np.uint8}
RATE_RANGE = (4000, 192000)
MAX_FACTOR = 1024               # largest up or down ev_format_audio takes (the bank of up = 1024 is ~86 KB of shared memory)


def plan(sample_rate, encoding, source_rate):
    """-> (rate, up, down): the output rate (``source_rate`` for None) and the coprime resampling factors.  Accepts an integer
    rate in [4000, 192000] Hz whose ratio to ``source_rate`` reduces to up / down with both at most 1024, and an encoding of
    ``ENCODINGS`` or "flac".  Raises ValueError otherwise."""
    if encoding not in ENCODINGS and encoding != FLAC:
        raise ValueError("encoding must be one of %s, got %r" % (sorted(ENCODINGS) + [FLAC], encoding))
    if sample_rate is None:
        rate = int(source_rate)
    else:
        if isinstance(sample_rate, (bool, np.bool_)) or not isinstance(sample_rate, (int, float, np.integer, np.floating)):
            raise ValueError("sample_rate must be an integer number of Hz, got %r" % (sample_rate,))
        if not (math.isfinite(float(sample_rate)) and float(sample_rate) == int(sample_rate)):
            raise ValueError("sample_rate must be an integer number of Hz, got %r" % (sample_rate,))
        rate = int(sample_rate)
    if not RATE_RANGE[0] <= rate <= RATE_RANGE[1]:
        raise ValueError("sample_rate must lie in [%d, %d] Hz, got %d" % (RATE_RANGE + (rate,)))
    g = math.gcd(rate, int(source_rate))
    up, down = rate // g, int(source_rate) // g
    if max(up, down) > MAX_FACTOR:
        raise ValueError("%d Hz from %d Hz is the ratio %d/%d; rates whose ratio needs a factor above %d are not supported"
                         % (rate, source_rate, up, down, MAX_FACTOR))
    return rate, up, down


def resample_filter(up, down):
    """scipy.signal.resample_poly's default filter for up / down, float64, already multiplied by ``up``."""
    from scipy.signal import firwin
    max_rate = max(up, down)
    h = firwin(2 * 10 * max_rate + 1, 1.0 / max_rate, window=("kaiser", 5.0))
    h *= up
    return h


def polyphase_bank(up, down):
    """-> (up, taps_per_phase) float32 C-contiguous: row p holds the filter taps p, p + up, p + 2 up, ... (zero past its end)."""
    h = resample_filter(up, down)
    taps = -(-len(h) // up)
    padded = np.zeros(up * taps, dtype=np.float64)
    padded[:len(h)] = h
    return np.ascontiguousarray(padded.reshape(taps, up).T.astype(np.float32))


def resampled_length(n, up, down):
    """Samples ``resample_poly`` returns for n input samples: ceil(n * up / down)."""
    return (int(n) * up + down - 1) // down


def packed_offsets(n_in, items, up, down):
    """Where each listed item's output starts in the packed buffer: (len(items) + 1,) int64, the last entry the total."""
    counts = [resampled_length(n_in[b], up, down) for b in items]
    return np.concatenate([[0], np.cumsum(counts, dtype=np.int64)]).astype(np.int64)


LOUDNESS_RANGE = (-70.0, 0.0)   # LUFS: a target below the absolute gate could never be measured


def check_loudness(target):
    """A loudness target -> float LUFS.  Raises ValueError unless it is a finite real number in [-70, 0]."""
    if isinstance(target, (bool, np.bool_)) or not isinstance(target, (int, float, np.integer, np.floating)):
        raise ValueError("loudness must be a number of LUFS, got %r" % (target,))
    t = float(target)
    if not (math.isfinite(t) and LOUDNESS_RANGE[0] <= t <= LOUDNESS_RANGE[1]):
        raise ValueError("loudness must be a finite target in [%g, %g] LUFS, got %r" % (LOUDNESS_RANGE + (target,)))
    return t


TRUE_PEAK_RANGE = (-20.0, 0.0)  # dBTP


def check_true_peak(ceiling):
    """A true-peak ceiling -> float dBTP.  Raises ValueError unless it is a finite real number in [-20, 0]."""
    if isinstance(ceiling, (bool, np.bool_)) or not isinstance(ceiling, (int, float, np.integer, np.floating)):
        raise ValueError("true_peak must be a ceiling in dBTP, got %r" % (ceiling,))
    c = float(ceiling)
    if not (math.isfinite(c) and TRUE_PEAK_RANGE[0] <= c <= TRUE_PEAK_RANGE[1]):
        raise ValueError("true_peak must be a finite ceiling in [%g, %g] dBTP, got %r" % (TRUE_PEAK_RANGE + (ceiling,)))
    return c


def check_watermark(key):
    """A watermark key -> int.  Raises ValueError unless it is an integer (not a bool) in [1, 2^63 - 1]."""
    if isinstance(key, (bool, np.bool_)) or not isinstance(key, (int, np.integer)):
        raise ValueError("watermark must be an integer key, got %r" % (key,))
    if not WATERMARK_KEY_RANGE[0] <= int(key) <= WATERMARK_KEY_RANGE[1]:
        raise ValueError("watermark must be a key in [1, 2^63 - 1], got %r" % (key,))
    return int(key)


_FIELDS = ("rate", "up", "down", "encoding", "loudness", "true_peak", "watermark")


class OutputFormat(tuple):
    """A validated output format: the rate and its resampling factors from the source rate, the encoding ("flac" or one of
    ENCODINGS), the loudness target (LUFS), the true-peak ceiling (dBTP) and the watermark key, each None when not asked for.
    Hashable: the MicroBatcher formats all requests of one key with one call.  Without a watermark it is the six-tuple of the
    first six fields, so it equals the formats (and tuples) made before the mark existed; with one it has seven."""
    __slots__ = ()

    def __new__(cls, rate, up, down, encoding, loudness, true_peak, watermark=None):
        fields = (rate, up, down, encoding, loudness, true_peak)
        return tuple.__new__(cls, fields if watermark is None else fields + (watermark,))

    def __repr__(self):
        return "OutputFormat(%s)" % ", ".join("%s=%r" % (f, getattr(self, f)) for f in _FIELDS)

    def __getnewargs__(self):
        return tuple(self)


for _i, _f in enumerate(_FIELDS):
    setattr(OutputFormat, _f, property(lambda self, i=_i: self[i] if i < len(self) else None))


def output_format(sample_rate, encoding, loudness, true_peak, source_rate, *, watermark=None):
    """The arguments of ``format_audio`` -> ``OutputFormat``, checked by ``plan``, ``check_loudness``, ``check_true_peak`` and
    ``check_watermark`` in that order; a watermark also needs an output rate of at least 8000 Hz, where its band still fits.
    Raises their ValueError otherwise."""
    rate, up, down = plan(sample_rate, encoding, source_rate)
    loudness = None if loudness is None else check_loudness(loudness)
    true_peak = None if true_peak is None else check_true_peak(true_peak)
    if watermark is not None:
        watermark = check_watermark(watermark)
        if rate < WATERMARK_MIN_RATE:
            raise ValueError("a watermark needs an output rate of at least %d Hz (its band reaches 3.4 kHz), got %d"
                             % (WATERMARK_MIN_RATE, rate))
    return OutputFormat(rate, up, down, encoding, loudness, true_peak, watermark)


# The true-peak limiter of ev_limit: fixed constants, not options.
LIMIT_DETECT_RATE = 192000      # the detector oversamples by R = ceil(192000 / sr): 12 at 16 kHz
LIMIT_LOOKAHEAD_S = 0.005       # look-ahead L: 5 ms, 80 samples at 16 kHz
LIMIT_RELEASE_DB_PER_S = 60.0   # linear release in dB per second
LIMIT_GRID = 2.0 ** -32         # ev_limit's envelope grid (dB): the release step is a multiple of it


def limit_lookahead(sr):
    return int(round(LIMIT_LOOKAHEAD_S * sr))


def limit_release(sr):
    """The release per sample (dB), rounded to ev_limit's 2^-32 dB grid so the release scan is exact in fp64."""
    return round(LIMIT_RELEASE_DB_PER_S / sr / LIMIT_GRID) * LIMIT_GRID


def _kaiser_lowpass(half, cutoff):
    from scipy.signal import firwin
    return firwin(2 * half + 1, cutoff, window=("kaiser", 5.0))


def limit_bank(sr, rate):
    """The detector of ev_limit for output at ``rate`` Hz from ``sr`` -> (bank (phases, taps) float32, hold M in samples).

    The interpolator oversamples by R = ceil(192000 / sr) and is designed like resample_poly's filter,
    ``firwin(2 * 10 * R + 1, 1 / R, kaiser 5) * R``.  For a rate below sr it is convolved (at the oversampled rate) with the
    same-design low-pass at rate / 2, ``firwin(2 * ceil(10 sr / rate) + 1, rate / sr, kaiser 5)``: the down-sampler removes that
    content, and doing so can raise peaks.  Row p of the bank is phase p's taps h[p + j R], applied as sum_j bank[p][j] x[n + c - j],
    c = (taps - 1) / 2; the plain interpolator keeps phases 1 .. R - 1 (phase 0 is x[n] itself), the low-passed one all R.
    M is the larger half-span, in samples at sr, of the detector and of format_audio's resampling filter for that rate."""
    R = -(-LIMIT_DETECT_RATE // int(sr))
    h = _kaiser_lowpass(10 * R, 1.0 / R) * R
    half = 10
    if rate < sr:
        lp_half = -(-10 * int(sr) // int(rate))
        lp = _kaiser_lowpass(lp_half, float(rate) / sr)
        up = np.zeros((len(lp) - 1) * R + 1)
        up[::R] = lp
        h = np.convolve(h, up)
        half += lp_half
    taps = 2 * half + 1
    padded = np.zeros(taps * R)
    padded[:len(h)] = h
    bank = padded.reshape(taps, R).T
    if rate >= sr:
        bank = bank[1:]
    g = math.gcd(int(rate), int(sr))
    up_, down_ = int(rate) // g, int(sr) // g
    resample_half = -(-10 * max(up_, down_) // up_) if (up_, down_) != (1, 1) else 0
    return np.ascontiguousarray(bank.astype(np.float32)), max(half, resample_half)


def true_peak_bank(sr):
    """The true-peak detector of ev_meter at ``sr`` Hz -> (R, 21) float32, R = ceil(192000 / sr): every phase of the
    limiter's interpolator ``firwin(2 * 10 * R + 1, 1 / R, kaiser 5) * R``, row p = h[p + j R], phase 0 included, so the
    detector reads exactly the samples of ``resample_poly(x, R, 1)`` and |x|.  ``limit_bank(sr, sr)`` is rows 1 .. R - 1: the
    limiter takes |x[n]| for phase 0, but the filter's centre tap is 1 + 6.7e-4 (firwin's unit-gain scaling), so phase 0
    reads up to 0.0059 dB above |x[n]|.  None at R = 1 (192 kHz), where resample_poly returns x itself."""
    R = -(-LIMIT_DETECT_RATE // int(sr))
    if R == 1:
        return None
    h = _kaiser_lowpass(10 * R, 1.0 / R) * R
    padded = np.zeros(21 * R)
    padded[:len(h)] = h
    return np.ascontiguousarray(padded.reshape(21, R).T.astype(np.float32))


# The watermark of ev_watermark_embed / ev_watermark_detect (emotivoice_b200.watermark): fixed constants, not options.  They
# hold at the model's rate, 16 kHz.
WATERMARK_N = 1024              # MCLT frame (sine window); bins of 15.625 Hz, bin k centred at (k + 1/2) 15.625 Hz
WATERMARK_HOP = 512             # frame j covers samples [(j - 1) hop, (j + 1) hop), j = 0 .. ceil(n / hop)
WATERMARK_BAND = (19, 218)      # bins 19..217: about 300-3400 Hz, inside 8 kHz telephony and the resampler's passband
WATERMARK_PERIOD = 64           # P: the pattern repeats every 64 frames (about 2 s)
WATERMARK_ALPHA = 10.0 ** (-20.0 / 20.0) / math.sqrt(2.0)   # the mark 20 dB under the host's in-band energy (E[C^2] = M^2 / 2)
WATERMARK_DETECT_Z = 7.0        # detection threshold (see emotivoice_b200.watermark)
WATERMARK_MIN_RATE = 8000       # output rates below this cut into the band
WATERMARK_KEY_RANGE = (1, 2 ** 63 - 1)


def k_weighting(sr):
    """ITU-R BS.1770-4's K-weighting at ``sr`` Hz -> (10,) float64: (b0, b1, b2, a1, a2) of the high shelf, then of the high
    pass, a0 = 1.  Both come from their analog prototypes through the bilinear transform, pre-warped at f0, with the constants
    libebur128 and pyloudnorm use; at 48 kHz they are the standard's table."""
    K = math.tan(math.pi * 1681.974450955533 / sr)
    Q = 0.7071752369554196
    Vh = 10.0 ** (3.999843853973347 / 20.0)
    Vb = Vh ** 0.4996667741545416
    a0 = 1.0 + K / Q + K * K
    shelf = [(Vh + Vb * K / Q + K * K) / a0, 2.0 * (K * K - Vh) / a0, (Vh - Vb * K / Q + K * K) / a0,
             2.0 * (K * K - 1.0) / a0, (1.0 - K / Q + K * K) / a0]
    K = math.tan(math.pi * 38.13547087602444 / sr)
    Q = 0.5003270373238773
    a0 = 1.0 + K / Q + K * K
    high_pass = [1.0, -2.0, 1.0, 2.0 * (K * K - 1.0) / a0, (1.0 - K / Q + K * K) / a0]
    return np.array(shelf + high_pass, dtype=np.float64)


def restart_warmup(kcoef):
    """Samples ``ev_loudness`` filters before each 100 ms sub-block, from zero state: the smallest multiple of 32 with
    W * r^W <= 1e-10, r the largest pole radius of the cascade (2048 at 16 kHz)."""
    r = max(float(np.max(np.abs(np.roots([1.0, kcoef[i + 3], kcoef[i + 4]])))) for i in (0, 5))
    W = 32
    while math.log(W) + W * math.log(r) > math.log(1e-10):
        W += 32
    return W


FLAC_STANDARD_RATES = {88200: 1, 176400: 2, 192000: 3, 8000: 4, 16000: 5, 22050: 6, 24000: 7, 32000: 8, 44100: 9, 48000: 10, 96000: 11}


def flac_rate_code(rate):
    """The sample rate field of a FLAC frame header (RFC 9639 section 9.1.2) -> (code, value of the field that follows the
    header's fixed part, its bits).  The standard code where one exists; else 12 (8-bit kHz) for a whole number of kHz up to
    255, 13 (16-bit Hz) up to 65535 Hz, 14 (16-bit tens of Hz) for a multiple of 10; else 0: the rate is only in STREAMINFO,
    and such a stream is outside FLAC's streamable subset."""
    rate = int(rate)
    if rate in FLAC_STANDARD_RATES:
        return FLAC_STANDARD_RATES[rate], 0, 0
    if rate % 1000 == 0 and rate // 1000 <= 255:
        return 12, rate // 1000, 8
    if rate <= 65535:
        return 13, rate, 16
    if rate % 10 == 0:
        return 14, rate // 10, 16
    return 0, 0, 0
