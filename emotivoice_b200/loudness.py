"""Loudness meter of recordings and outputs on the GPU (``ev_meter``): what EBU R128, ATSC A/85 and the podcast and streaming
delivery specs ask to be reported, per recording of a batch, at the recording's own rate.

    m = loudness.meter(wav, 48000, lengths)         # wav: a CUDA (B, L) float32 tensor
    m.integrated, m.true_peak, m.loudness_range     # device float32 tensors of shape (B,)

Definitions (one channel, n valid samples at sr Hz, sr a multiple of 10 in [4000, 192000]):

- Sub-blocks: 100 ms of sr / 10 samples of the BS.1770-4 K-weighted signal (``audio.k_weighting(sr)``), mean square per
  sub-block, exactly those of ``JETSGenerator.measure_loudness`` / ``format_audio(loudness=...)``; only full sub-blocks count.
- Momentary loudness M: -0.691 + 10 log10(mean of the mean squares of 4 consecutive sub-blocks), one value per 400 ms window
  inside the item, 10 per second.  Short-term loudness S: the same over 30 sub-blocks (3 s).  ``max_momentary`` /
  ``max_short_term`` are their largest values, -inf for an item too short to hold one window, or silent.
- ``integrated``: BS.1770-4 gated loudness, bit for bit the ``lufs`` of ``measure_loudness`` for the same samples.
- ``loudness_range`` (EBU Tech 3342): take the short-term values S > -70 LUFS; keep those greater than
  10 log10(mean of 10^(S/10) over them) - 20; sort the n values left; LRA = v[round((n - 1) 0.95)] - v[round((n - 1) 0.10)],
  0-based, rounding half away from zero (Tech 3342's pseudo-code), each v the exact element.  NaN when n = 0.
- ``true_peak`` (dBTP): 20 log10 of the largest of |x| and the item oversampled by R = ceil(192000 / sr) with the output
  chain's limiter's interpolator (``audio.true_peak_bank``: ``resample_poly(x, R, 1)``'s filter, all R phases; zero outside
  the item), through the limiter's own detector code; -inf for silence.  It is what ``limiter_oracle.true_peak_db`` reads,
  the measure the limiter's ceiling is tested against.  The limiter itself skips phase 0 (``audio.limit_bank(sr, sr)``),
  whose centre tap is 1 + 6.7e-4, so on a peak at a sample instant the meter reads up to 0.0059 dB above the limiter's
  detector.  A declared choice: BS.1770-4 Annex 2's example filter is not used.
- ``sample_peak``: max |x|, linear (as ``measure_loudness``'s peak).

Every result of a recording is bitwise the same whatever else is in the batch and in which order.
"""
import collections

import numpy as np
import torch

from . import _abi, audio, recordings

Meter = collections.namedtuple("Meter", "integrated loudness_range max_momentary max_short_term true_peak sample_peak momentary short_term")
Meter.__doc__ = """Per-recording results of ``meter`` (device float32 tensors of shape (B,)): integrated (LUFS), loudness_range
(LU), max_momentary and max_short_term (LUFS), true_peak (dBTP), sample_peak (linear); momentary and short_term: (B, K)
series at 10 Hz when asked for (row b holds NaN past its own values), else None."""


def check_rate(sample_rate):
    """A meter rate -> int Hz.  Raises ValueError unless it is an integer multiple of 10 in [4000, 192000] (100 ms
    sub-blocks must hold a whole number of samples)."""
    if isinstance(sample_rate, (bool, np.bool_)) or not isinstance(sample_rate, (int, np.integer)):
        raise ValueError("sample_rate must be an integer number of Hz, got %r" % (sample_rate,))
    rate = int(sample_rate)
    if not (audio.RATE_RANGE[0] <= rate <= audio.RATE_RANGE[1] and rate % 10 == 0):
        raise ValueError("sample_rate must be a multiple of 10 Hz in [%d, %d] (100 ms sub-blocks), got %d" % (audio.RATE_RANGE + (rate,)))
    return rate


def k_weighting(rate):
    """``audio.k_weighting(rate)`` as a host float64 tensor, made once per rate: ev_loudness and ev_meter read it by address."""
    return recordings.device_table(("k_weighting", rate), lambda: audio.k_weighting(rate), "cpu")


def enqueue(base, meta_ptr, lens, rate, ws, series):
    """ev_meter of the items at base + start[k] (``meta_ptr``: device i64 start offsets followed by the lengths; ``lens``: host
    lengths) -> Meter.  ``ws(nbytes)`` returns a workspace of at least nbytes on the items' device.  Arguments must already
    be valid."""
    lib = _abi.load()
    k = len(lens)
    nb = int(lib.ev_meter_workspace_bytes(k, max(lens), rate))
    w = ws(nb)
    dev = w.device
    res = torch.empty((6, k), dtype=torch.float32, device=dev)
    cols = max(lens) // (rate // 10)
    ser = torch.empty((2, k, cols), dtype=torch.float32, device=dev) if series else None
    n_host = np.ascontiguousarray(lens, dtype=np.int64)
    bank = recordings.device_table(("true_peak_bank", rate), lambda: audio.true_peak_bank(rate), dev)   # None at 192 kHz
    phases, taps = (0, 21) if bank is None else (int(bank.shape[0]), int(bank.shape[1]))
    _abi.check(lib.ev_meter(base, meta_ptr, meta_ptr + 8 * k, n_host.ctypes.data, k, rate, k_weighting(rate).data_ptr(),
                            None if bank is None else bank.data_ptr(), phases, taps, res.data_ptr(),
                            None if ser is None or ser.numel() == 0 else ser[0].data_ptr(),
                            None if ser is None or ser.numel() == 0 else ser[1].data_ptr(), cols, w.data_ptr(), nb,
                            torch.cuda.current_stream(dev).cuda_stream))
    mom = st = None
    if series:
        mom, st = ser[0][:, :max(0, cols - 3)], ser[1][:, :max(0, cols - 29)]
    return Meter(res[0], res[1], res[2], res[3], res[4], res[5], mom, st)


@torch.no_grad()
def meter(wav, sample_rate, lengths=None, series=False):
    """Meters each recording of a batch (see the module docstring for the definitions).

    ``wav``: a CUDA (B, L) float32 tensor, one recording per row (rows may be further apart than L; samples must be
    contiguous).  ``sample_rate``: their rate, an integer multiple of 10 Hz in [4000, 192000] (so 11025 Hz is refused).
    ``lengths``: the valid samples of each row (a sequence or a CPU tensor of B integers in [0, L]); None: every row is L.
    ``series``: also return the momentary and short-term series.

    Returns a ``Meter`` of device tensors.  Four launches, no sync; invalid arguments raise ValueError before anything is
    enqueued."""
    wav = recordings.recording_batch(wav)
    B, L = wav.shape
    rate = check_rate(sample_rate)
    lens = recordings.host_lengths(lengths, B, L)
    if not isinstance(series, (bool, np.bool_)):
        raise ValueError("series must be True or False, got %r" % (series,))
    dev = wav.device
    meta, (p_meta, _) = recordings.upload([[b * wav.stride(0) for b in range(B)], lens], dev)     # start offsets, then lengths
    return enqueue(wav.data_ptr(), p_meta, lens, rate, lambda nb: torch.empty((nb,), dtype=torch.uint8, device=dev), bool(series))
