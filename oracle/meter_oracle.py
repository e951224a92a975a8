"""The EBU R128 loudness meter of ``ev_meter`` / ``emotivoice_b200.loudness.meter``, in float64 numpy, on top of the BS.1770-4
restatement of ``loudness_oracle`` (K-weighting, gating, integrated loudness, sample peak) and the true peak of
``limiter_oracle``.

- Sub-blocks: 100 ms of fs / 10 samples of the K-weighted signal; only full ones count.
- Momentary and short-term loudness: -0.691 + 10 log10(mean square) of every window of 4 (400 ms) and 30 (3 s) sub-blocks,
  stepped by one sub-block, that lies entirely inside the signal; their maxima, -inf when there is no window (or silence).
- Loudness range (EBU Tech 3342): the short-term values above -70 LUFS; of those, the values above
  10 log10(mean of 10^(S / 10)) - 20; of the n left, sorted ascending, v[round(0.95 (n - 1))] - v[round(0.10 (n - 1))],
  0-based, rounding half away from zero; NaN when n = 0.
- Integrated loudness: ``loudness_oracle.integrated_loudness``.  True peak: ``limiter_oracle.true_peak_db``.

Shares no code with ``emotivoice_b200``.
"""
import math

import numpy as np
from numpy.lib.stride_tricks import sliding_window_view

from oracle import limiter_oracle, loudness_oracle

MOMENTARY, SHORT_TERM = 4, 30   # sub-blocks per window
ABS_GATE, REL_GATE = -70.0, -20.0
LOW, HIGH = 0.10, 0.95


def subblock_energies(x, fs):
    """Sum of squares of the K-weighted signal over every full 100 ms sub-block, and the sub-block length fs / 10."""
    y = loudness_oracle.k_filter(x, fs)
    S = int(fs) // 10
    nf = len(y) // S
    return (y[:nf * S] ** 2).reshape(nf, S).sum(axis=1), S


def window_loudness(x, fs, blocks):
    """-0.691 + 10 log10(mean square) of every window of ``blocks`` sub-blocks, stepped by one, entirely inside x."""
    e, S = subblock_energies(x, fs)
    if len(e) < blocks:
        return np.zeros(0)
    z = sliding_window_view(e, blocks).sum(axis=1) / (blocks * S)
    with np.errstate(divide="ignore"):
        return loudness_oracle.OFFSET + 10.0 * np.log10(z)


def momentary(x, fs):
    return window_loudness(x, fs, MOMENTARY)


def short_term(x, fs):
    return window_loudness(x, fs, SHORT_TERM)


def round_half_away(v):
    q = math.floor(v)
    return int(q) + 1 if v - q >= 0.5 else int(q)


def loudness_range(x, fs, st=None):
    """EBU Tech 3342's loudness range (LU) of x, or of its short-term series ``st``; NaN when no value passes both gates."""
    s = short_term(x, fs) if st is None else np.asarray(st, np.float64)
    s = s[s > ABS_GATE]
    if not len(s):
        return math.nan
    rel = 10.0 * np.log10(np.mean(10.0 ** (s / 10.0))) + REL_GATE
    v = np.sort(s[s > rel])
    if not len(v):
        return math.nan
    n = len(v)
    return float(v[round_half_away((n - 1) * HIGH)] - v[round_half_away((n - 1) * LOW)])


def meter(x, fs, true_peak=True):
    """-> dict: integrated, loudness_range, max_momentary, max_short_term, true_peak (dBTP; None unless asked for),
    sample_peak (linear), and the momentary and short_term series."""
    x = np.asarray(x, np.float64)
    m, st = momentary(x, fs), short_term(x, fs)
    return dict(integrated=loudness_oracle.integrated_loudness(x, fs), loudness_range=loudness_range(x, fs, st),
                max_momentary=float(np.max(m, initial=-np.inf)), max_short_term=float(np.max(st, initial=-np.inf)),
                true_peak=limiter_oracle.true_peak_db(x, fs) if true_peak else None, sample_peak=loudness_oracle.peak(x),
                momentary=m, short_term=st)
